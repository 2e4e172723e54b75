// SPG-N: the SM-partitioned groupby kernels (groupby.cu, "SM-partitioned groupby") with NARROW bucket rows.
// Included by groupby.cu only.
//
// The two-kernel path moves 48 B/row through HBM: 16 read + 16 bucket write + 16 bucket read.  When a row's key and value both
// fit 32 bits (dictionary codes, dates, small integers — decided per ROW, sampled per operator state so the variant is only
// chosen when it pays) the owner bucket carries the row as an (int32 key, int32 value) pair: 16 + 8 + 8 = 32 B/row, K1n stages
// and copies out half the bytes, and K2n's shared table shrinks to 12-byte slots (int32 key, low sum word, count) whose
// two-slot buckets are ONE 8-byte shared load each, with 32-bit key compares.  Rows that do not fit (either value outside
// int32, or the key INT32_MIN, which marks a free slot) take the direct global path inside K1n, so the result is exact for any
// input; a.counters[CTR_WIDE] counts them and the host drops back to the 16-byte kernels when they are not rare.
// Sums stay exact mod 2^64: the sign-extended value is added as (low word, high word + carry) exactly as in spg_aggregate_kernel.
// K1n is K1's tile loop (spg_partition_tiles in groupby.cu) with its own classify / stage / copy-out; K2n's table is the shared
// two-choice table (spg_find, and spg_claim in spgn_cold_row) with int32 keys, and K2n and K2d flush through spg_flush_ticketed.
//
// The DENSE form (template flag DENSE, DESIGN §3) is for keys that lie in a small window [kbase, kbase + 2^KB), KB <= 21, chosen
// from the state's sample.  A row's key offset d = key - kbase is scrambled by a bijection sigma on KB bits and split into
// (owner, slot) = (sigma(d) mod G, sigma(d) div G): the owner's shared table is direct-mapped, so the bucket row needs no key.  It
// is ONE 4-byte word, slot << VB | (value - vbase), and K2 does one load and two 32-bit shared atomics per row with no key
// compare and no insertion: 16 + 4 + 4 = 24 B/row of HBM traffic.  A row whose key or value offset does not fit takes the
// direct path in K1 and counts in counters[CTR_DENSE_WIDE]; the host goes back to the hash form when such rows are not rare.
#pragma once

#ifndef SPGN_TILE_ROWS
#define SPGN_TILE_ROWS 4096
#endif
constexpr int SPGN_TILE = SPGN_TILE_ROWS;            // rows per K1n tile (8-byte staged rows leave room for twice the 16-byte kernels' tile)
constexpr int SPGN_CTAS = SPGN_TILE == 4096 ? 2 : 3;  // K1n CTAs per SM
constexpr int SPGN_QUEUE = 32;                                          // K2n: cold rows a warp queues before it handles them together
constexpr int SPGN_QUEUE_BYTES = SPG_THREADS / 32 * SPGN_QUEUE * 9;     // 8-byte row + one flag byte per queued row: 9 KB

// find-or-insert for a caller that already holds a group ticket: `inserted` says whether THIS call created the group (else the
// ticket goes back).  The table cannot be full: tickets bound the number of groups by cap / 2.
__device__ __forceinline__ uint64_t spgn_insert_ticketed(long long* __restrict__ tkeys, uint64_t cap, long long key, bool& inserted) {
    const uint64_t mask = cap - 1;
    uint64_t s = (key_hash(key) >> 32) & mask;
    inserted = false;
    while (true) {
        long long k = __ldcg(tkeys + s);
        if (k == EMPTY_KEY) {
            k = (long long)atomicCAS((unsigned long long*)(tkeys + s), (unsigned long long)EMPTY_KEY, (unsigned long long)key);
            if (k == EMPTY_KEY) { inserted = true; return s; }
        }
        if (k == key) return s;
        s = (s + 1) & mask;
    }
}

// The dense form's key map.  sigma(d) = xorshift(d * mul mod 2^KB) is a bijection on KB bits: an odd multiplier is invertible mod
// 2^KB, and x ^ (x >> s) with 2s >= KB is its own inverse.  It spreads keys that share a stride (all multiples of G, of 128, of
// 2^k) or a sub-range of the window over all owners.  q = umulhi(x, gmagic) with gmagic = ceil(2^32 / G) is x div G exactly for
// x < 2^21 and 2 <= G <= 256 (the error x * (gmagic * G - 2^32) / 2^32 stays below 2^29 / 2^32).  tests/test_spgn_dense_map.py
// checks all of it over every window size and owner count.
__device__ __forceinline__ unsigned int spgd_scramble(unsigned int d, unsigned int kb, unsigned int mul) {
    const unsigned int x = (d * mul) & ((1u << kb) - 1u);
    return x ^ (x >> ((kb + 1) / 2));
}
__device__ __forceinline__ long long spgd_key(const SpgDenseArgs& a, unsigned int slot, unsigned int owner) {
    unsigned int x = slot * (unsigned int)a.n_owners + owner;
    x ^= x >> ((a.d_kb + 1) / 2);
    return (long long)((unsigned long long)a.kbase + ((x * a.d_inv) & ((1u << a.d_kb) - 1u)));
}

// K1n's shared memory: spg_partition_tiles' regions with 8-byte (hash) or 4-byte (dense) staged rows, then the staged rows'
// owners (SPGN_TILE), per owner its run's destination (SPG_MAX_OWNERS pointers) and the tile_over flag
template <bool DENSE>
using SpgnK1Smem = SpgTileSmem<SPGN_TILE, SPG_MAX_OWNERS, DENSE ? 4 : 8, SPGN_TILE + SPG_MAX_OWNERS * 8 + 16>;

template <bool HAS_SUM, bool HAS_CNT, bool DENSE = false>
__global__ void __launch_bounds__(SPG_TTHREADS, SPGN_CTAS) spgn_partition_kernel(const __grid_constant__ std::conditional_t<DENSE, SpgDenseArgs, SpgArgs> a) {
    using Row = std::conditional_t<DENSE, unsigned int, int2>;  // bucket row: slot << VB | value offset, or (int32 key, int32 value)
    using L = SpgnK1Smem<DENSE>;
    extern __shared__ __align__(128) unsigned char smem_n_raw[];
    long long* raw_k = (long long*)(smem_n_raw + L::raw_k);
    long long* raw_v = (long long*)(smem_n_raw + L::raw_v);
    Row* stage = (Row*)(smem_n_raw + L::stage);
    const unsigned long long* gbase = (const unsigned long long*)(smem_n_raw + L::gbase);
    unsigned char* stage_owner = smem_n_raw + L::tail;                          // SPGN_TILE
    Row** dptr = (Row**)(stage_owner + SPGN_TILE);                              // SPG_MAX_OWNERS: run start - local start, as an address
    unsigned int* tile_over = (unsigned int*)(dptr + SPG_MAX_OWNERS);           // some run of this tile does not fit its bucket
    const int G = a.n_owners, tid = threadIdx.x;
    Row* bucket = reinterpret_cast<Row*>(a.bucket);
    unsigned int wide = 0;
    spg_partition_tiles<SPGN_TILE, SPG_TTHREADS, L>(
        smem_n_raw, a.n_rows, G, a.bucket_cnt,
        [&](int64_t r0, uint64_t* mbar) {
            mbar_expect_tx(mbar, (HAS_SUM ? 2u : 1u) * SPGN_TILE * 8u);
            tma_load_1d(raw_k, a.keys + r0, SPGN_TILE * 8u, mbar);
            if (HAS_SUM) tma_load_1d(raw_v, a.vals + r0, SPGN_TILE * 8u, mbar);
        },
        [&](int64_t r0) {
            for (int j = tid; j < SPGN_TILE; j += SPG_TTHREADS) {
                int64_t i = r0 + j;
                raw_k[j] = i < a.n_rows ? a.keys[i] : 0;
                raw_v[j] = (HAS_SUM && i < a.n_rows) ? a.vals[i] : 0;
            }
        },
        [&] { *tile_over = 0; },
        [&](int j, [[maybe_unused]] unsigned int& w) -> int {  // DENSE: w = the row's bucket word
            const long long k = raw_k[j];
            const long long v = HAS_SUM ? raw_v[j] : 0;
            if constexpr (DENSE) {
                // key and value offsets inside their windows (unsigned: below the base wraps to a large offset)
                const unsigned long long d = (unsigned long long)k - (unsigned long long)a.kbase;
                const unsigned long long e = HAS_SUM ? (unsigned long long)v - (unsigned long long)a.vbase : 0ull;
                if ((d >> a.d_kb) != 0 || (e >> a.d_vb) != 0) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, k, (unsigned long long)v, 1ull); wide++; return -1; }
                const unsigned int x = spgd_scramble((unsigned int)d, a.d_kb, a.d_mul), q = __umulhi(x, a.d_gmagic);
                w = q << a.d_vb | (unsigned int)e;
                return (int)(x - q * (unsigned int)G);
            } else {
                // both values inside int32 <=> the high words of (x + 2^31) are zero; the key INT32_MIN (low word of k + 2^31 zero) is excluded
                const unsigned long long kb = (unsigned long long)k + 0x80000000ull, vb = (unsigned long long)v + 0x80000000ull;
                const bool narrow = ((kb | vb) >> 32) == 0 && (unsigned int)kb != 0u;
                if (!narrow) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, k, (unsigned long long)v, 1ull); wide++; return -1; }
                return (int)spg_owner(spg_hash(k), G);
            }
        },
        [&](unsigned int p, int j, int o, [[maybe_unused]] unsigned int w) {
            if constexpr (DENSE) stage[p] = w;
            else stage[p] = make_int2((int)raw_k[j], HAS_SUM ? (int)raw_v[j] : 0);
            stage_owner[p] = (unsigned char)o;
        },
        [&](int ow, unsigned long long my_gbase, unsigned int my_cnt) {
            const unsigned int* lbase = (const unsigned int*)(smem_n_raw + L::lbase);
            dptr[ow] = bucket + ((size_t)ow * a.bucket_cap + my_gbase - lbase[ow]);  // staged position p of this owner's run goes to dptr[ow][p]
            if (my_gbase + my_cnt > (unsigned long long)a.bucket_cap) *tile_over = 1;
        },
        [&](unsigned int n_tile) {
            if (*tile_over == 0) {  // every run fits (the common case): one owner byte, one address and one 8-byte store per row
                unsigned int p = tid;
                for (; p + SPG_TTHREADS < n_tile; p += 2 * SPG_TTHREADS) {
                    const unsigned int o0 = stage_owner[p], o1 = stage_owner[p + SPG_TTHREADS];
                    const Row r0v = stage[p], r1v = stage[p + SPG_TTHREADS];
                    dptr[o0][p] = r0v;
                    dptr[o1][p + SPG_TTHREADS] = r1v;
                }
                if (p < n_tile) dptr[stage_owner[p]][p] = stage[p];
            } else {
                for (unsigned int p = tid; p < n_tile; p += SPG_TTHREADS) {
                    const unsigned int ow = stage_owner[p];
                    const unsigned long long off = gbase[ow] + p;
                    const Row row = stage[p];
                    if (off < (unsigned long long)a.bucket_cap) bucket[(size_t)ow * a.bucket_cap + off] = row;
                    else if constexpr (DENSE)  // bucket full (skew): the row back from its word and owner
                        spg_direct_apply<HAS_SUM, HAS_CNT>(a, spgd_key(a, row >> a.d_vb, ow),
                                                           (unsigned long long)a.vbase + (row & ((1u << a.d_vb) - 1u)), 1ull);
                    else spg_direct_apply<HAS_SUM, HAS_CNT>(a, (long long)row.x, (unsigned long long)(long long)row.y, 1ull);  // bucket full (skew)
                }
            }
            __syncthreads();  // every thread has read tile_over
            if (tid == 0) *tile_over = 0;
        });
    if (wide) atomicAdd((unsigned long long*)&a.counters[DENSE ? CTR_DENSE_WIDE : CTR_WIDE], (unsigned long long)wide);
}

// K2n's rare per-row work, for one queued row.  !added: the key is not in its two buckets (spg_claim: a free candidate slot, else
// the stash; else the direct path), then the row is added.  added: the row was added already and the low sum word
// wrapped, so the high sum word takes the sign extension plus the carry: +1 for a value >= 0, -1 for a negative one.  Either way
// a carry into the high sum word goes to the global table.
// Out of line on purpose: inlined into the row loop it made K2n slower per 2^28 rows on an H100 (scratch/spg_harness.cu): at
// eight call sites 4.5 against 3.0 ms at 1 M groups, at one call site 2.8 against 1.0 ms at 200 k groups.
template <bool HAS_SUM, bool HAS_CNT>
__device__ __noinline__ void spgn_cold_row(const SpgArgs& a, int* skeys, unsigned int* slo, unsigned int* scnt, unsigned int NB, int key, int val,
                                           bool added) {
    unsigned int old = 0;
    if (!added) {
        const int s = spg_claim(skeys, 2 * NB, spg_hash((long long)key), key);
        if (s < 0) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, (long long)key, (unsigned long long)(long long)val, 1ull); return; }
        if (HAS_SUM) old = atomicAdd(&slo[s], (unsigned int)val);
        if (HAS_CNT) atomicAdd(&scnt[s], 1u);
    }
    if (HAS_SUM) {
        const unsigned int lo = (unsigned int)val;
        const unsigned int hi = added ? (val < 0 ? 0xffffffffu : 1u) : (val < 0 ? 0xffffffffu : 0u) + (old + lo < old ? 1u : 0u);
        if (hi) spg_direct_apply<HAS_SUM, HAS_CNT>(a, (long long)key, (unsigned long long)hi << 32, 0ull);
    }
}

// scratch/spg_harness.cu builds K2n with SPGN_PHASE_CLOCKS to see where a launch's time goes: per CTA, the SM clocks of table
// init, the row loop and the flush, summed over passes.  SPGN_SKIP_FLUSH (harness ablation, wrong results) drops the flush.
#ifdef SPGN_PHASE_CLOCKS
__device__ unsigned long long spgn_phase_clocks[SPG_MAX_OWNERS * 4];  // per CTA: 3 spans, then the clock of the last mark
#define SPGN_PHASE(i)                                                                                                      \
    do {                                                                                                                   \
        if (threadIdx.x == 0) {                                                                                            \
            unsigned long long* c_ = spgn_phase_clocks + blockIdx.x * 4;                                                   \
            const unsigned long long t_ = clock64();                                                                       \
            if ((i) >= 0) c_[(i)] += t_ - c_[3];                                                                           \
            c_[3] = t_;                                                                                                    \
        }                                                                                                                  \
    } while (0)
#else
#define SPGN_PHASE(i) do {} while (0)
#endif

// The flush of K2n and K2d: one owner's n_slots-slot table, whose slot s holds a group when occupied(s), read by
// entry(s, key, sum, cnt), into the state's global table.  First flush of a state (empty global table, a.reserve_tickets):
// every occupied slot is a NEW group, and 10^6 per-insert tickets on one counter cost ~0.2 ms — the CTA takes the tickets of
// all its slots with ONE atomic and returns the few it did not need (a key that sits in two slots, or that the direct path
// inserted meanwhile).
template <bool HAS_SUM, bool HAS_CNT, typename Occupied, typename Entry>
__device__ __forceinline__ void spg_flush_ticketed(const SpgArgs& a, int n_slots, Occupied occupied, Entry entry) {
    const int tid = threadIdx.x;
    __shared__ unsigned int fl_occ, fl_dup;
    __shared__ int fl_reserved;
    if (tid == 0) { fl_occ = 0; fl_dup = 0; fl_reserved = 0; }
    __syncthreads();
    if (a.reserve_tickets && a.group_limit >= 0) {
        unsigned int mine = 0;
        for (int s = tid; s < n_slots; s += SPG_THREADS) mine += occupied(s);
        for (int d = 16; d; d >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, d);
        if ((tid & 31) == 0 && mine) atomicAdd(&fl_occ, mine);
        __syncthreads();
        if (tid == 0 && fl_occ) {
            const long long t = (long long)atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], (unsigned long long)fl_occ);
            if (t + (long long)fl_occ <= a.group_limit) fl_reserved = 1;
            else atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], (unsigned long long)(-(long long)fl_occ));  // no room: per-insert tickets
        }
        __syncthreads();
    }
    const bool reserved = fl_reserved != 0;
    unsigned int dup = 0;
    for (int s = tid; s < n_slots; s += SPG_THREADS) {
        if (!occupied(s)) continue;
        long long key;
        unsigned long long sum, cnt;
        entry(s, key, sum, cnt);
        if (!reserved) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, sum, cnt); continue; }
        // ticket already held: insert without the limit; a key that was there already gives its ticket back
        bool inserted;
        const uint64_t sl = spgn_insert_ticketed(a.tkeys, a.cap, key, inserted);
        if (!inserted) dup++;
        if (HAS_SUM && sum) atomicAdd(a.acc_sum + sl, sum);
        if (HAS_CNT && cnt) atomicAdd(a.acc_cnt + sl, cnt);
    }
    if (reserved) {
        for (int d = 16; d; d >>= 1) dup += __shfl_xor_sync(0xffffffffu, dup, d);
        if ((tid & 31) == 0 && dup) atomicAdd(&fl_dup, dup);
        __syncthreads();
        if (tid == 0 && fl_dup) atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], (unsigned long long)(-(long long)fl_dup));
    }
    __syncthreads();
}

// K2n: slot = int32 key, low sum word (biased by 2^31), count.
template <bool HAS_SUM, bool HAS_CNT>
__device__ __forceinline__ void spgn_hash_aggregate(const SpgArgs& a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SPGN_PHASE(-1);
    const int NS = a.ns, NT = a.ns + SPG_STASH, tid = threadIdx.x, me = blockIdx.x;
    int* skeys = (int*)smem_raw;                      // NT x 4
    unsigned int* slo = (unsigned int*)(skeys + NT);  // NT x 4
    unsigned int* scnt = slo + NT;                    // NT x 4, then the warps' cold-row queues (SPGN_QUEUE_BYTES)
    const unsigned int NB = (unsigned int)NS / 2;
    const unsigned int NP = (unsigned int)a.n_pass, GP = (unsigned int)gridDim.x * NP;

    unsigned long long n_in = a.bucket_cnt[me * SPG_CNT_STRIDE];
    if (n_in > (unsigned long long)a.bucket_cap) n_in = (unsigned long long)a.bucket_cap;
    const int2* src = reinterpret_cast<const int2*>(a.bucket) + (size_t)me * a.bucket_cap;  // bucket_cap is even: 16-byte aligned
    constexpr int U = 4;  // rows per thread per iteration, as two 16-byte loads of two adjacent rows
    // unit = two adjacent rows; units of this thread: first + j * SPG_THREADS, j = 0 .. U/2 - 1
    // rows of one iteration: U/2 units of two adjacent rows, unit index first + j * SPG_THREADS
    auto load_rows = [&](unsigned long long first, int2 (&row)[U], auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
#pragma unroll
        for (int j = 0; j < U / 2; j++) {
            const unsigned long long r = 2 * (first + (unsigned long long)j * SPG_THREADS);
            row[2 * j] = row[2 * j + 1] = make_int2(SPGN_EMPTY, 0);
            if (FULL || r + 1 < n_in) {
                const int4 q = __ldcs(reinterpret_cast<const int4*>(src + r));
                row[2 * j] = make_int2(q.x, q.y); row[2 * j + 1] = make_int2(q.z, q.w);
            } else if (r < n_in) row[2 * j] = __ldcs(src + r);
        }
    };
    // Rows that need spgn_cold_row (a key not in its two buckets, a low sum word that wrapped) do not call it where they are found:
    // they go to their warp's queue in shared memory, and the warp drains a full queue with one call on all lanes.  At 1 M groups a
    // warp meets such a row in most iterations (first appearances, then stashed keys: about 14 k per CTA and 2^28-row launch), and
    // calling it per row took K2n from 1.1 to 3.0 ms per launch (H100 at 400 W, scratch/spg_harness.cu), most likely because a call
    // first waits for every load in flight, the next iteration's bucket rows included.
    // queue slot i of this warp: row at q_row(i), flag "added already" at q_added(i) (computed where used: the loop has no
    // register to spare for the two addresses)
    auto q_row = [&](unsigned int i) { return reinterpret_cast<int2*>(scnt + NT) + (threadIdx.x >> 5) * SPGN_QUEUE + i; };
    auto q_added = [&](unsigned int i) {
        return reinterpret_cast<unsigned char*>(reinterpret_cast<int2*>(scnt + NT) + SPG_THREADS / 32 * SPGN_QUEUE) + (threadIdx.x >> 5) * SPGN_QUEUE + i;
    };
    unsigned int qn = 0;  // rows in this warp's queue (the same in every lane)
    auto drain = [&]() {
        __syncwarp();
        const unsigned int lane = threadIdx.x & 31;
        if (lane < qn) spgn_cold_row<HAS_SUM, HAS_CNT>(a, skeys, slo, scnt, NB, q_row(lane)->x, q_row(lane)->y, *q_added(lane) != 0);
        __syncwarp();
        qn = 0;
    };
    auto process = [&](const int2 (&row)[U], unsigned int pass, auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;
        int sl[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const uint64_t h = spg_hash((long long)row[u].x);
            unsigned int b1, b2;
            spg_buckets(h, NB, b1, b2);
            const int key = row[u].x;
            sl[u] = spg_find(skeys, b1, b2, key);
            if (!FULL && key == SPGN_EMPTY) sl[u] = -2;  // padding lane (INT32_MIN never reaches a bucket)
            if (NP > 1 && __umulhi((unsigned int)(h >> 32), GP) - (unsigned int)me * NP != pass) sl[u] = -2;
        }
        unsigned int cold = 0;  // bit u: row u goes to the queue; bit U + u: its row was added already (the low sum word wrapped)
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (sl[u] >= 0) {
                if (HAS_SUM) {
                    const unsigned int lo = (unsigned int)row[u].y, old = atomicAdd(&slo[sl[u]], lo);
                    // high sum word = sign extension + carry of the low-word add: nonzero only when the biased low word wraps
                    if ((row[u].y < 0 ? 0xffffffffu : 0u) + (old + lo < old ? 1u : 0u)) cold |= (1u << u) | (1u << (U + u));
                }
                if (HAS_CNT) atomicAdd(&scnt[sl[u]], 1u);
            } else if (sl[u] == -1) cold |= 1u << u;
        }
        if (__any_sync(0xffffffffu, cold != 0)) {
#pragma unroll 1
            for (int u = 0; u < U; u++) {
                const bool mine = (cold >> u) & 1u;
                const unsigned int m = __ballot_sync(0xffffffffu, mine);
                if (!m) continue;
                if (qn + __popc(m) > SPGN_QUEUE) drain();
                if (mine) {
                    int2 r = row[0];
#pragma unroll
                    for (int v = 1; v < U; v++)
                        if (u == v) r = row[v];
                    const unsigned int p = qn + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
                    *q_row(p) = r;
                    *q_added(p) = (cold >> (U + u)) & 1u;
                }
                qn += __popc(m);
            }
        }
    };
    const unsigned long long ustep = (unsigned long long)(U / 2) * SPG_THREADS;   // units per CTA iteration
    const unsigned long long full_units = n_in / (2 * ustep) * ustep;              // iterations whose rows are all in range
    for (unsigned int pass = 0; pass < NP; pass++) {
        for (int s = tid; s < NT; s += SPG_THREADS) { skeys[s] = SPGN_EMPTY; slo[s] = 0x80000000u; scnt[s] = 0; }
        __syncthreads();
        SPGN_PHASE(0);
        // software pipeline: the next iteration's bucket rows are in flight while the current ones are aggregated (the wait for these
        // loads was the largest single stall of the unpipelined loop, 20 % of the samples)
        if (full_units > 0) {
            int2 cur[U], nxt[U];
            load_rows(tid, cur, std::true_type{});
            for (unsigned long long ub = 0; ub < full_units; ub += ustep) {
                if (ub + ustep < full_units) load_rows(ub + ustep + tid, nxt, std::true_type{});
                process(cur, pass, std::true_type{});
#pragma unroll
                for (int u = 0; u < U; u++) cur[u] = nxt[u];
            }
        }
        for (unsigned long long ub = full_units; 2 * ub < n_in; ub += ustep) {
            int2 tail[U];
            load_rows(ub + tid, tail, std::false_type{});
            process(tail, pass, std::false_type{});
        }
        if (qn) drain();
        __syncthreads();
        SPGN_PHASE(1);
#ifdef SPGN_SKIP_FLUSH
        continue;
#endif
        spg_flush_ticketed<HAS_SUM, HAS_CNT>(a, NT, [&](int s) { return skeys[s] != SPGN_EMPTY; },
                                             [&](int s, long long& key, unsigned long long& sum, unsigned long long& cnt) {
                                                 key = (long long)skeys[s];
                                                 sum = (unsigned long long)slo[s] - 0x80000000ull;  // remove the bias (wraps mod 2^64)
                                                 cnt = (unsigned long long)scnt[s];
                                             });
        SPGN_PHASE(2);
    }
}

// K2d, the dense form of K2n (spgn_aggregate_kernel<., ., true>): slot s of owner `me` is the key kbase + sigma^-1(s * G + me).
// A slot is {low word of the sum of value offsets, count}; the count is kept for a sum-only signature too, it marks the slots
// the flush visits.  The row loop has no rare path but a wrap of the sum word, which sends its 2^32 to the global table.
template <bool HAS_SUM, bool HAS_CNT>
__device__ __noinline__ void spgd_carry(const SpgDenseArgs& a, unsigned int slot) {
    spg_direct_apply<HAS_SUM, HAS_CNT>(a, spgd_key(a, slot, blockIdx.x), 1ull << 32, 0ull);
}

template <bool HAS_SUM, bool HAS_CNT>
__device__ __forceinline__ void spgd_aggregate(const SpgDenseArgs& a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int NS = a.d_slots, tid = threadIdx.x, me = blockIdx.x;
    unsigned int* ssum = (unsigned int*)smem_raw;  // NS: sum of (value - vbase) mod 2^32
    unsigned int* scnt = ssum + NS;                // NS: rows
    for (int s = tid; s < NS; s += SPG_THREADS) { ssum[s] = 0; scnt[s] = 0; }
    __syncthreads();
    unsigned long long n_in = a.bucket_cnt[me * SPG_CNT_STRIDE];
    if (n_in > (unsigned long long)a.bucket_cap) n_in = (unsigned long long)a.bucket_cap;
    const unsigned int* src = reinterpret_cast<const unsigned int*>(a.bucket) + (size_t)me * a.bucket_cap;  // bucket_cap % 4 == 0: 16-byte aligned
    const unsigned int vb = a.d_vb, vmask = (1u << vb) - 1u;
    auto add = [&](unsigned int w) {
        const unsigned int s = w >> vb;
        if (HAS_SUM) {
            const unsigned int e = w & vmask, old = atomicAdd(&ssum[s], e);
            if (old + e < old) spgd_carry<HAS_SUM, HAS_CNT>(a, s);
        }
        atomicAdd(&scnt[s], 1u);
    };
    // software pipeline: V 16-byte loads (4 rows each) per thread in flight while the previous V are aggregated
    constexpr int V = 2;
    const uint4* src4 = reinterpret_cast<const uint4*>(src);
    const unsigned long long n4 = n_in / 4, step = (unsigned long long)V * SPG_THREADS, full = n4 / step * step;
    if (full > 0) {
        uint4 cur[V], nxt[V];
#pragma unroll
        for (int j = 0; j < V; j++) cur[j] = __ldcs(src4 + tid + j * SPG_THREADS);
        for (unsigned long long ub = 0; ub < full; ub += step) {
            if (ub + step < full) {
#pragma unroll
                for (int j = 0; j < V; j++) nxt[j] = __ldcs(src4 + ub + step + tid + j * SPG_THREADS);
            }
#pragma unroll
            for (int j = 0; j < V; j++) { add(cur[j].x); add(cur[j].y); add(cur[j].z); add(cur[j].w); }
#pragma unroll
            for (int j = 0; j < V; j++) cur[j] = nxt[j];
        }
    }
    for (unsigned long long i = 4 * full + tid; i < n_in; i += SPG_THREADS) add(__ldcs(src + i));
    __syncthreads();
    const unsigned long long vbase = (unsigned long long)a.vbase;
    spg_flush_ticketed<HAS_SUM, HAS_CNT>(a, NS, [&](int s) { return scnt[s] != 0; },
                                 [&](int s, long long& key, unsigned long long& sum, unsigned long long& cnt) {
                                     cnt = (unsigned long long)scnt[s];
                                     key = spgd_key(a, (unsigned int)s, (unsigned int)me);
                                     sum = (unsigned long long)ssum[s] + cnt * vbase;  // exact mod 2^64
                                 });
}

template <bool HAS_SUM, bool HAS_CNT, bool DENSE = false>
__global__ void __launch_bounds__(SPG_THREADS, 1) spgn_aggregate_kernel(const __grid_constant__ std::conditional_t<DENSE, SpgDenseArgs, SpgArgs> a) {
    if constexpr (DENSE) spgd_aggregate<HAS_SUM, HAS_CNT>(a);
    else spgn_hash_aggregate<HAS_SUM, HAS_CNT>(a);
}
