// spf.cuh — SPF: the SM-partitioned groupby as ONE persistent kernel (included by groupby.cu after the SPG helpers,
// inside namespace b200).
//
// Why: the two-kernel SPG (K1 partition -> owner buckets in HBM -> K2 aggregate) moves 48 B/row through HBM for 16 B/row
// of input, so it cannot pass 1/3 of the 16 B/row roofline however well the kernels are tuned (VERDICT r01 #5).  Here the
// bucket hand-off never leaves L2 and no warp ever waits at a CTA-wide barrier:
//
//   * one CTA per SM, all co-resident (cooperative launch), 32 warps with four roles:
//       loader   (1 warp)  claims 4096-row blocks from a global counter and streams them into a 4-stage shared-memory ring with
//                          TMA bulk copies (cp.async.bulk + mbarrier full/empty pairs, L2 evict-first policy);
//       producer (8 warps) takes its two rows of every 512-row stage, hashes them to their owner SM and appends them to that
//                          owner's WRITE-COMBINING BIN: two 128-byte lines of eight (key, value) rows per owner, slots handed out
//                          by a shared-memory ticket atomic; the thread that completes a line posts it to a flusher queue;
//       flusher  (3 warps) copies completed lines to the owner's ring in global memory — always whole, 128-byte aligned lines
//                          (one L2 request per eight rows), up to 16 lines per warp iteration;
//       publisher (1 warp) fences and publishes the ring heads (committed line counts) — the GPU-scope fence costs thousands of
//                          cycles under load, so it sits on no data path;
//       consumer (19 warps) polls the heads of the rings it reads, takes lines as they arrive (four lines = 32 rows per warp
//                          instruction, from whichever rings have them) and aggregates them into a shared-memory cuckoo hash
//                          table that lives for the whole launch (flushed into the state's global table ONCE, at the end).
//     A first version with a counting sort per 2048-row tile (three producer barriers per tile, 8 producer warps) was far
//     slower: every phase waited for the slowest warp and the consumers starved.
//   * every (producer SM p, owner SM o) pair has a private ring of SPF_RL lines (SMs x SMs x 2 KB:
//     132 x 132 x 2 KB = 35 MB on an H100, inside its 50 MB L2).  A
//     private ring needs no reservation atomics: p's flusher owns the head, o's consumer owns the tail; cursors are
//     monotonically increasing line counts in pub[p][o] / cons[o][p];
//   * scratch/ubench4.cu measures the ceiling of this data flow: HBM stream + L2-resident ring write + ring read, against
//     the same ring in HBM.
//
// Shared-memory table: two-choice cuckoo, two-slot buckets (two 16-byte loads + four compares per lookup), two native
// 32-bit atomics per row (low word of the sum with carry detection; count).  First appearances claim a free candidate slot
// with a CAS; a key whose four candidates are taken is parked and placed by cuckoo displacement in a short consumer-only
// quiescent phase (displacing an entry while lookups are in flight would lose updates).  Simulation: 2 x 2 cuckoo places
// every key up to 80 % load where plain two-choice leaves 3 % of them out at 66 %.
//
// Bounded scratch: rows / partials that find the GLOBAL table at its group limit go to the retry list (as in SPG).  When
// the list passes SPF_RETRY_SOFT entries the loaders stop claiming blocks (blocks are claimed from a global counter, so
// "rows < claimed blocks x 4096" is exactly what was consumed); everything in flight at that moment (rings, bins, shared
// tables: < 5 M entries) still fits behind the soft limit.  The host grows the table, merges the list and relaunches from
// the first unclaimed block.
#pragma once

constexpr int SPF_NPW = 8;                          // producer warps
constexpr int SPF_NFW = 2;                          // flusher warps
constexpr int SPF_NCW = 20;                         // consumer warps
constexpr int SPF_W_LOADER = SPF_NPW;               // warp index of the loader
constexpr int SPF_W_FLUSH0 = SPF_NPW + 1;
constexpr int SPF_W_PUB = SPF_NPW + 1 + SPF_NFW;     // the publisher warp
constexpr int SPF_W_CONS0 = SPF_NPW + 2 + SPF_NFW;
constexpr int SPF_THREADS = (SPF_NPW + 2 + SPF_NFW + SPF_NCW) * 32;   // 32 warps = 1024 threads (the CTA limit; 64 registers each)
constexpr int SPF_CT = SPF_NCW * 32;
constexpr int SPF_CHUNK = SPF_NPW * 64;             // rows per stage: two adjacent rows per producer lane
constexpr int SPF_NSTAGE = 4;
constexpr int SPF_BLOCK = 8 * SPF_CHUNK;            // rows per claimed block
constexpr int SPF_LINE = 8;                         // rows per 128-byte line
constexpr int SPF_RL = 16;                          // ring lines per (producer, owner) pair
constexpr int SPF_R = SPF_RL * SPF_LINE;            // ring rows
constexpr int SPF_MAXO = 160;                       // owners (= CTAs = SMs) supported
constexpr int SPF_FQ = 256;                         // flusher queue entries (>= 2 lines x owners of one flusher + one iteration)
constexpr int SPF_KQ = 128;                         // parked keys awaiting cuckoo placement
constexpr int SPF_MAXKICK = 96;
constexpr unsigned int SPF_FINAL = 0x80000000u;     // pub[] flag: the producer SM has published its last lines
constexpr long long SPF_RETRY_SOFT = 1ll << 21;     // retry-list entries at which loaders stop claiming blocks
constexpr long long SPF_RETRY_HARD = 1ll << 23;     // retry-list capacity (soft limit + everything that can be in flight)
static_assert(SPF_CHUNK == 512, "stage size");

struct SpfArgs {
    SpgArgs g;                    // keys / vals / n_rows, global table, counters, retry list (bucket fields unused)
    longlong2* ring;              // [owner][producer][SPF_R]
    unsigned int* pub;            // [producer][owner] lines written (| SPF_FINAL)
    unsigned int* cons;           // [owner][producer] lines consumed
    unsigned long long* tile_ctr; // [0] next block to claim (2^62 once the launch was stopped), [1] first unconsumed block of a stopped launch (host inits to ~0)
    int ns;                       // shared-memory table slots per CTA (even)
    unsigned long long* stats;    // SPF_STATS builds (scratch/spf_harness only), else unused
};
#ifdef SPF_STATS
#define SPF_STAT_T0() const long long st_t0_ = clock64()
#define SPF_STAT_ADD(i) do { if (lane == 0) atomicAdd(fa.stats + (i), (unsigned long long)(clock64() - st_t0_)); } while (0)
#define SPF_STAT_INC(i, v) do { if (lane == 0) atomicAdd(fa.stats + (i), (unsigned long long)(v)); } while (0)
#ifdef SPF_STATS_HEAVY
#define SPF_TM_DECL long long tm_[6] = {0, 0, 0, 0, 0, 0}; long long tm_t_ = clock64()
#define SPF_TM(i) do { const long long n_ = clock64(); tm_[i] += n_ - tm_t_; tm_t_ = n_; } while (0)
#define SPF_TM_FLUSH(base) do { if (lane == 0) for (int i_ = 0; i_ < 6; i_++) atomicAdd(fa.stats + (base) + i_, (unsigned long long)tm_[i_]); } while (0)
#else
#define SPF_TM_DECL do {} while (0)
#define SPF_TM(i) do {} while (0)
#define SPF_TM_FLUSH(base) do {} while (0)
#endif
#else
#define SPF_TM_DECL do {} while (0)
#define SPF_TM(i) do {} while (0)
#define SPF_TM_FLUSH(base) do {} while (0)
#define SPF_STAT_T0() do {} while (0)
#define SPF_STAT_ADD(i) do {} while (0)
#define SPF_STAT_INC(i, v) do {} while (0)
#endif

// shared-memory footprint in front of the table
struct SpfSmemLayout {
    static constexpr size_t raw_k = 0;                                                   // [NSTAGE][CHUNK] keys
    static constexpr size_t raw_v = raw_k + (size_t)SPF_NSTAGE * SPF_CHUNK * 8;          // [NSTAGE][CHUNK] values
    static constexpr size_t bins = raw_v + (size_t)SPF_NSTAGE * SPF_CHUNK * 8;           // [MAXO][2 lines][8] (key, value)
    static constexpr size_t fill = bins + (size_t)SPF_MAXO * 2 * SPF_LINE * 16;          // [MAXO] u32 ticket counters
    static constexpr size_t done = fill + SPF_MAXO * 4;                                  // [MAXO][2] u32 rows stored into the line
    static constexpr size_t slotgen = done + SPF_MAXO * 8;                               // [MAXO][2] u32 line generation the slot accepts
    static constexpr size_t headline = slotgen + SPF_MAXO * 8;                           // [MAXO] u32 lines written to ring (me -> o)
    static constexpr size_t headdone = headline + SPF_MAXO * 4;                          // [MAXO] u32 lines committed (stored) to ring (me -> o)
    static constexpr size_t ctail = headdone + SPF_MAXO * 4;                             // [MAXO] u32 cached consumer tails
    static constexpr size_t fq = ctail + SPF_MAXO * 4;                                   // [NFW][FQ] u32 flusher queues
    static constexpr size_t mbar = fq + (size_t)SPF_NFW * SPF_FQ * 4;                    // full[NSTAGE], empty[NSTAGE] u64
    static constexpr size_t ctl = mbar + 2 * SPF_NSTAGE * 8;                             // 32 u32 control words
    static constexpr size_t kq = ctl + 128;                                              // [SPF_KQ] (key, value)
    static constexpr size_t table = kq + (size_t)SPF_KQ * 16;                            // ns x 16
};
// control words
enum { SPF_CTL_KQ = 0, SPF_CTL_CDONE = 1, SPF_CTL_RNG = 2, SPF_CTL_PDONE = 3, SPF_CTL_FINAL = 4, SPF_CTL_FDONE = 5,
       SPF_CTL_FQTAIL = 8 /* [NFW] */, SPF_CTL_ROWS = 16 /* [NSTAGE] rows in the stage, -1 = end of input */ };

__device__ __forceinline__ unsigned int ld_relaxed_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u32(unsigned int* p, unsigned int v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_1d_stream(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
// the rare global-table path (marker key, high word of a sum, evicted entries, final flush): ONE out-of-line copy, so the hot
// loops stay small (inlined, each call site carries ~400 instructions of hash + probe loop)
template <bool HAS_SUM, bool HAS_CNT>
__device__ __noinline__ void spf_direct(const SpgArgs* a, long long key, unsigned long long sum, unsigned long long cnt) {
    spg_direct_apply<HAS_SUM, HAS_CNT>(*a, key, sum, cnt);
}

template <bool HAS_SUM, bool HAS_CNT>
__global__ void __launch_bounds__(SPF_THREADS, 1) spf_groupby_kernel(const __grid_constant__ SpfArgs fa) {
    extern __shared__ __align__(128) unsigned char spf_smem[];
    const SpgArgs& a = fa.g;
    using L = SpfSmemLayout;
    long long* raw_k = (long long*)(spf_smem + L::raw_k);
    long long* raw_v = (long long*)(spf_smem + L::raw_v);
    longlong2* bins = (longlong2*)(spf_smem + L::bins);
    unsigned int* fill = (unsigned int*)(spf_smem + L::fill);
    unsigned int* done = (unsigned int*)(spf_smem + L::done);
    volatile unsigned int* slotgen = (volatile unsigned int*)(spf_smem + L::slotgen);
    unsigned int* headline = (unsigned int*)(spf_smem + L::headline);
    unsigned int* headdone = (unsigned int*)(spf_smem + L::headdone);
    unsigned int* ctail = (unsigned int*)(spf_smem + L::ctail);
    volatile unsigned int* fq = (volatile unsigned int*)(spf_smem + L::fq);
    uint64_t* mb_full = (uint64_t*)(spf_smem + L::mbar);
    uint64_t* mb_empty = mb_full + SPF_NSTAGE;
    volatile unsigned int* ctl = (volatile unsigned int*)(spf_smem + L::ctl);
    volatile int* stage_rows = (volatile int*)(ctl + SPF_CTL_ROWS);
    longlong2* kq = (longlong2*)(spf_smem + L::kq);
    const int NS = fa.ns;
    long long* skeys = (long long*)(spf_smem + L::table);
    unsigned int* slo = (unsigned int*)(skeys + NS);
    unsigned int* scnt = slo + NS;
    const unsigned int NB = (unsigned int)NS / 2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = (int)gridDim.x, me = (int)blockIdx.x;

    // ---- init ----
    for (int s = tid; s < NS; s += SPF_THREADS) { skeys[s] = EMPTY_KEY; slo[s] = 0x80000000u; scnt[s] = 0; }
    for (int j = tid; j < SPF_MAXO; j += SPF_THREADS) {
        fill[j] = 0; done[2 * j] = 0; done[2 * j + 1] = 0; slotgen[2 * j] = 0; slotgen[2 * j + 1] = 1; headline[j] = 0; headdone[j] = 0; ctail[j] = 0;
    }
    for (int j = tid; j < SPF_NFW * SPF_FQ; j += SPF_THREADS) fq[j] = 0;
    if (tid < 32) ctl[tid] = 0;
    if (tid == 0) {
        for (int s = 0; s < SPF_NSTAGE; s++) { mbar_init(&mb_full[s], 1); mbar_init(&mb_empty[s], SPF_NPW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto buckets = [&](long long key, unsigned int& b1, unsigned int& b2) {
        const uint64_t h = spg_hash(key);
        b1 = __umulhi((unsigned int)(h >> 20), NB);
        b2 = __umulhi(((unsigned int)h ^ (unsigned int)(h >> 44)) * 0x9E3779B1u, NB);
        b2 = b2 == b1 ? (b1 + 1 == NB ? 0u : b1 + 1) : b2;
    };
    // add one row (or a partial) to slot s: low word with carry detection, the rare high word goes to the global table
    auto add = [&](int s, long long key, long long val) {
        if (HAS_SUM) {
            const unsigned int lo = (unsigned int)(unsigned long long)val;
            unsigned int hi = (unsigned int)((unsigned long long)val >> 32);
            const unsigned int old = atomicAdd(&slo[s], lo);
            hi += (old + lo < old) ? 1u : 0u;
            if (hi) spf_direct<HAS_SUM, HAS_CNT>(&a, key, (unsigned long long)hi << 32, 0ull);
        }
        if (HAS_CNT) atomicAdd(&scnt[s], 1u);
    };
    // a completed line (owner o, generation g) goes to the queue of the flusher that serves o
    auto post_line = [&](unsigned int o, unsigned int g) {
        const unsigned int f = o % SPF_NFW;
        const unsigned int q = atomicAdd((unsigned int*)&ctl[SPF_CTL_FQTAIL + f], 1u);
        fq[f * SPF_FQ + (q & (SPF_FQ - 1))] = ((g << 8) | o) + 1u;
    };

    if (warp < SPF_NPW) {
        // =====================================================================================================
        // producer: two adjacent rows of every stage -> owner bins
        // =====================================================================================================
        SPF_TM_DECL;
        for (unsigned int it = 0;; it++) {
            const int s = (int)(it % SPF_NSTAGE);
            const uint32_t par = (it / SPF_NSTAGE) & 1u;
            SPF_TM(3);
            while (!mbar_try_wait(&mb_full[s], par)) {}
            SPF_TM(0);
            const int n = stage_rows[s];
            if (n < 0) break;
            const int r = 2 * (warp * 32 + lane);
            long long k[2] = {EMPTY_KEY, EMPTY_KEY}, v[2] = {0, 0};
            bool in[2] = {r < n, r + 1 < n};
            if (in[0]) {
                const longlong2 kk = *reinterpret_cast<const longlong2*>(raw_k + s * SPF_CHUNK + r);
                k[0] = kk.x; k[1] = kk.y;
                if (HAS_SUM) { const longlong2 vv = *reinterpret_cast<const longlong2*>(raw_v + s * SPF_CHUNK + r); v[0] = vv.x; v[1] = vv.y; }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&mb_empty[s]);  // this warp has its rows: the stage may be refilled once all warps said so
            unsigned int o[2], pos[2];
#pragma unroll
            for (int q = 0; q < 2; q++) {
                if (in[q] && k[q] == EMPTY_KEY) { spf_direct<HAS_SUM, HAS_CNT>(&a, k[q], (unsigned long long)v[q], 1ull); in[q] = false; }
                if (in[q]) { o[q] = spg_owner(spg_hash(k[q]), G); pos[q] = atomicAdd(&fill[o[q]], 1u); }
            }
            SPF_TM(1);
#pragma unroll
            for (int q = 0; q < 2; q++) {
                if (!in[q]) continue;
                const unsigned int g = pos[q] >> 3, b = g & 1u;
#ifndef SPF_EXP_NOFLUSH
                if (slotgen[2 * o[q] + b] != g) {
                    SPF_STAT_T0();
                    unsigned int ns = 64;
                    while (slotgen[2 * o[q] + b] != g) { __nanosleep(ns); ns = ns < 1024 ? ns * 2 : ns; }
                    { const int lane = 0; SPF_STAT_ADD(40); SPF_STAT_INC(41, 1); }
                }
#endif
                SPF_TM(2);  // the line's previous occupant (generation g - 2) is not flushed yet
                bins[(o[q] * 2 + b) * SPF_LINE + (pos[q] & 7u)] = make_longlong2(k[q], v[q]);
                asm volatile("" ::: "memory");  // the row is stored before it is counted (shared-memory accesses of a warp execute in order)
                const unsigned int d = atomicAdd(&done[2 * o[q] + b], 1u);
#ifndef SPF_EXP_NOFLUSH
                if (d == SPF_LINE - 1) post_line(o[q], g);
#else
                if (d == 0x7fffffffu) post_line(o[q], g);
#endif
            }
        }
        SPF_TM_FLUSH(16);
        // end of input for this warp; the LAST producer warp pads and posts the partially filled lines
        __syncwarp();
        unsigned int prev = 0;
        if (lane == 0) { __threadfence_block(); prev = atomicAdd((unsigned int*)&ctl[SPF_CTL_PDONE], 1u); }
        prev = __shfl_sync(0xffffffffu, prev, 0);
        if (prev == SPF_NPW - 1) {
            __threadfence_block();
            for (int ow = lane; ow < G; ow += 32) {
                const unsigned int pos = *(volatile unsigned int*)&fill[ow];
                const unsigned int rem = pos & 7u;
#ifdef SPF_EXP_NOFLUSH
                if (rem > 100) {
#else
                if (rem) {
#endif
                    const unsigned int g = pos >> 3, b = g & 1u;
                    for (unsigned int j = rem; j < SPF_LINE; j++) bins[(ow * 2 + b) * SPF_LINE + j] = make_longlong2(EMPTY_KEY, 0);  // padding rows
                    __threadfence_block();
                    post_line((unsigned int)ow, g);
                }
            }
            __syncwarp();
            __threadfence_block();
            if (lane == 0) ctl[SPF_CTL_FINAL] = 1u;  // flushers: drain your queues, then publish the final cursors
        }
    } else if (warp == SPF_W_LOADER) {
        // =====================================================================================================
        // loader: block claims + TMA pipeline
        // =====================================================================================================
        const int64_t n_blocks = (a.n_rows + SPF_BLOCK - 1) / SPF_BLOCK;
        uint64_t policy;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
        // blocks are claimed one ahead: the atomic for the next block is issued when a block starts and first looked at when it ends
        unsigned long long c_cur = 0, c_next = ~0ull;
        if (lane == 0) c_cur = atomicAdd(fa.tile_ctr, 1ull);
        c_cur = __shfl_sync(0xffffffffu, c_cur, 0);
        unsigned int cnt = 0;  // stages issued so far
        auto wait_stage_free = [&](int s) {
            if (cnt >= (unsigned int)SPF_NSTAGE) { const uint32_t par = ((cnt / SPF_NSTAGE) - 1u) & 1u; while (!mbar_try_wait(&mb_empty[s], par)) {} }
        };
        while (c_cur < (unsigned long long)n_blocks) {
            if (lane == 0) {
                c_next = atomicAdd(fa.tile_ctr, 1ull);
                if (*(volatile long long*)a.retry_ctr >= SPF_RETRY_SOFT) {
                    // stop the launch: nobody claims another block; blocks below `old` were claimed and are all consumed
                    const unsigned long long old = atomicExch(fa.tile_ctr, 1ull << 62);
                    if (old < (1ull << 62)) atomicMin(fa.tile_ctr + 1, old);
                }
            }
            const int64_t b0 = (int64_t)c_cur * SPF_BLOCK;
            const int64_t b1 = min(b0 + (int64_t)SPF_BLOCK, a.n_rows);
            for (int64_t r0 = b0; r0 < b1; r0 += SPF_CHUNK, cnt++) {
                const int s = (int)(cnt % SPF_NSTAGE);
                // sweep of the consumers' tails (for the flushers' ring-space test): loads issued now, stored after the wait below
                unsigned int tl[5];
                const bool sweep = (cnt & 1u) == 0;
                if (sweep) {
#pragma unroll
                    for (int q = 0; q < 5; q++) { const int ow = lane + 32 * q; tl[q] = ow < G ? ld_relaxed_u32(fa.cons + (size_t)ow * G + me) : 0u; }
                }
                wait_stage_free(s);
                if (sweep) {
#pragma unroll
                    for (int q = 0; q < 5; q++) { const int ow = lane + 32 * q; if (ow < G) ctail[ow] = tl[q]; }
                }
                const int rows = (int)min((int64_t)SPF_CHUNK, b1 - r0);
                if (rows == SPF_CHUNK) {
                    if (lane == 0) {
                        stage_rows[s] = rows;
                        mbar_expect_tx(&mb_full[s], (HAS_SUM ? 2u : 1u) * SPF_CHUNK * 8u);
                        tma_load_1d_stream(raw_k + s * SPF_CHUNK, a.keys + r0, SPF_CHUNK * 8u, &mb_full[s], policy);
                        if (HAS_SUM) tma_load_1d_stream(raw_v + s * SPF_CHUNK, a.vals + r0, SPF_CHUNK * 8u, &mb_full[s], policy);
                    }
                } else {  // the input's last, partial chunk: ordinary loads
                    for (int j = lane; j < rows; j += 32) { raw_k[s * SPF_CHUNK + j] = a.keys[r0 + j]; if (HAS_SUM) raw_v[s * SPF_CHUNK + j] = a.vals[r0 + j]; }
                    __syncwarp();
                    if (lane == 0) { stage_rows[s] = rows; mbar_arrive(&mb_full[s]); }
                }
            }
            c_cur = __shfl_sync(0xffffffffu, c_next, 0);
        }
        // end marker
        {
            const int s = (int)(cnt % SPF_NSTAGE);
            wait_stage_free(s);
            if (lane == 0) { stage_rows[s] = -1; mbar_arrive(&mb_full[s]); }
        }
    } else if (warp < SPF_W_PUB) {
        // =====================================================================================================
        // flusher f: completed lines of the owners o with o % NFW == f -> rings.  Up to 16 lines per iteration: every 8-lane
        // group takes four queue entries whose (independent) latency chains overlap.  No fences here: the heads are published
        // by the publisher warp, which reads the committed line counts (headdone[]).
        // =====================================================================================================
        const int f = warp - SPF_W_FLUSH0;
        const int grp = lane >> 3, l8 = lane & 7;
        unsigned int qhead = 0;
        // One iteration takes up to 32 posted lines: lane i does the bookkeeping of queue entry qhead + i (ring position, commit),
        // the copy itself runs in eight passes of four lines (eight lanes x 16 bytes per line).
        while (true) {
            const unsigned int e = fq[f * SPF_FQ + ((qhead + lane) & (SPF_FQ - 1))];
            const unsigned int vm = __ballot_sync(0xffffffffu, e != 0);
            const int nv = vm == 0xffffffffu ? 32 : __ffs(~vm) - 1;  // entries are taken in queue order: the leading run of posted ones
            if (nv == 0) {
                if (ctl[SPF_CTL_FINAL] && ctl[SPF_CTL_FQTAIL + f] == qhead) break;
                __nanosleep(100);
                continue;
            }
            SPF_STAT_INC(10, nv); SPF_STAT_INC(11, 1);
            const bool act = lane < nv;
            const unsigned int o = (e - 1u) & 0xffu, g = (e - 1u) >> 8, b = g & 1u;
            unsigned int pos = 0;
            if (act) {
                pos = atomicAdd(&headline[o], 1u);  // this line's place in ring (me -> o)
                // ring full (lines written - lines consumed >= SPF_RL)?  ctail[] is kept fresh by the loader warp's sweeps
                if (pos - *(volatile unsigned int*)&ctail[o] >= (unsigned int)SPF_RL) {
                    SPF_STAT_T0();
                    const unsigned int* cp = fa.cons + (size_t)o * G + me;
                    while (true) { const unsigned int ct = ld_relaxed_u32(cp); if (pos - ct < (unsigned int)SPF_RL) { ctail[o] = ct; break; } __nanosleep(200); }
                    { const int lane = 0; SPF_STAT_ADD(42); SPF_STAT_INC(43, 1); }
                }
            }
            __syncwarp();
            const unsigned int src_word = (o * 2 + b) * SPF_LINE;                                   // first row of the line in bins[]
            const unsigned int dst_word = ((unsigned int)o * G + me) * SPF_R + (pos & (SPF_RL - 1)) * SPF_LINE;  // ... and in ring[]
#pragma unroll
            for (int p = 0; p < 8; p++) {
                const int Lq = 4 * p + grp;
                const unsigned int sw = __shfl_sync(0xffffffffu, src_word, Lq);
                const unsigned int dw = __shfl_sync(0xffffffffu, dst_word, Lq);
                if (Lq < nv) fa.ring[(size_t)dw + l8] = bins[sw + l8];
            }
            __syncwarp();  // every lane's bin reads and ring stores of this iteration are done / issued
            if (act) {
                fq[f * SPF_FQ + ((qhead + lane) & (SPF_FQ - 1))] = 0;
                done[2 * o + b] = 0;
                atomicMax(&headdone[o], pos + 1u);  // committed lines of ring (me -> o): what the publisher may announce
            }
            __threadfence_block();
            if (act) slotgen[2 * o + b] = g + 2;  // the slot accepts the line two generations on
            qhead += nv;
        }
        __syncwarp();
        SPF_TM_FLUSH(24);
        if (lane == 0) { __threadfence_block(); atomicAdd((unsigned int*)&ctl[SPF_CTL_FDONE], 1u); }
    } else if (warp == SPF_W_PUB) {
        // =====================================================================================================
        // publisher: committed line counts -> fence -> cursors.  The fence (MEMBAR at GPU scope: thousands of cycles under
        // load) is why this is its own warp; it is cumulative over the flushers' ring stores because the counts it read were
        // written after those stores (CTA-scope fence in between).
        // =====================================================================================================
        unsigned int last[5] = {0, 0, 0, 0, 0};
        while (true) {
            const bool fin = ctl[SPF_CTL_FDONE] >= (unsigned int)SPF_NFW;  // read BEFORE the counts: final means nothing more will come
            __threadfence_block();
            unsigned int cur[5];
            bool changed = false;
#pragma unroll
            for (int q = 0; q < 5; q++) { const int ow = lane + 32 * q; cur[q] = ow < G ? *(volatile unsigned int*)&headdone[ow] : 0u; changed |= cur[q] != last[q]; }
            if (!__any_sync(0xffffffffu, changed) && !fin) { __nanosleep(100); continue; }
            SPF_STAT_T0();
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
            SPF_STAT_ADD(44); SPF_STAT_INC(45, 1);
#pragma unroll
            for (int q = 0; q < 5; q++) {
                const int ow = lane + 32 * q;
                if (ow < G && (cur[q] != last[q] || fin)) st_relaxed_u32(fa.pub + (size_t)me * G + ow, cur[q] | (fin ? SPF_FINAL : 0u));
                last[q] = cur[q];
            }
            if (fin) break;
        }
    } else {
        // =====================================================================================================
        // consumer
        // =====================================================================================================
        const int cw = warp - SPF_W_CONS0;
        // rings read by this warp: producers p0 .. p0 + np - 1 (balanced split of G over the consumer warps; np <= 16)
        const int base_n = G / SPF_NCW, extra = G % SPF_NCW;
        const int np = base_n + (cw < extra ? 1 : 0);
        const int p0 = cw * base_n + min(cw, extra);
        // the cursor state of ring r of this warp (r < np) lives in lane r
        const int grp = lane >> 3, l8 = lane & 7;
        const int myring = lane;
        const bool mine = myring < np;
        const unsigned int ringrow0 = ((unsigned int)me * G + (unsigned int)(p0 + (mine ? myring : 0))) * SPF_R;  // first row of my ring in fa.ring
        volatile unsigned int* kq_cnt = ctl + SPF_CTL_KQ;
        volatile unsigned int* cdone = ctl + SPF_CTL_CDONE;

        // first appearance of a key, or a key whose candidates are all taken
        auto slow_upsert = [&](long long key, long long val) {
            unsigned int b1, b2;
            buckets(key, b1, b2);
            const unsigned long long uk = (unsigned long long)key, E = (unsigned long long)EMPTY_KEY;
            const ulonglong2 c1 = *reinterpret_cast<const ulonglong2*>(skeys + 2 * b1);
            const ulonglong2 c2 = *reinterpret_cast<const ulonglong2*>(skeys + 2 * b2);
            const int f1 = (c1.x == E) + (c1.y == E), f2 = (c2.x == E) + (c2.y == E);
            int s = c1.x == uk ? (int)(2 * b1) : c1.y == uk ? (int)(2 * b1 + 1) : c2.x == uk ? (int)(2 * b2) : c2.y == uk ? (int)(2 * b2 + 1) : -1;
            if (s < 0 && f1 + f2 > 0) {
                const unsigned int first = f2 > f1 ? b2 : b1, second = f2 > f1 ? b1 : b2;  // balanced allocation: emptier bucket first
                const unsigned int cand[4] = {2 * first, 2 * first + 1, 2 * second, 2 * second + 1};
#pragma unroll
                for (int c = 0; c < 4 && s < 0; c++) {
                    const unsigned long long old = atomicCAS((unsigned long long*)&skeys[cand[c]], E, uk);
                    if (old == E || old == uk) s = (int)cand[c];
                }
            }
            if (s >= 0) { add(s, key, val); return; }
            // all four candidates hold other keys: park for the cuckoo phase (or, queue full, the direct global path)
            const unsigned int q = atomicAdd((unsigned int*)kq_cnt, 1u);
            if (q < (unsigned int)SPF_KQ) kq[q] = make_longlong2(key, val);
            else spf_direct<HAS_SUM, HAS_CNT>(&a, key, (unsigned long long)val, 1ull);
        };
        // cuckoo placement of the parked keys; runs on ONE lane while every consumer warp waits at the named barrier
        auto place_parked = [&]() {
            const unsigned int n = min(*kq_cnt, (unsigned int)SPF_KQ);
            unsigned int rng = ctl[SPF_CTL_RNG] * 1664525u + 1013904223u;
            const unsigned long long E = (unsigned long long)EMPTY_KEY;
            for (unsigned int q = 0; q < n; q++) {
                const long long key = kq[q].x, val = kq[q].y;
                auto find = [&](long long kx) -> int {
                    unsigned int b1, b2;
                    buckets(kx, b1, b2);
                    return skeys[2 * b1] == kx ? (int)(2 * b1) : skeys[2 * b1 + 1] == kx ? (int)(2 * b1 + 1)
                         : skeys[2 * b2] == kx ? (int)(2 * b2) : skeys[2 * b2 + 1] == kx ? (int)(2 * b2 + 1) : -1;
                };
                int s = find(key);
                if (s < 0) {
                    long long ck = key; unsigned int clo = 0x80000000u, ccnt = 0;  // entry looking for a home
                    unsigned int from = 0xffffffffu;
                    bool placed = false;
                    for (int it = 0; it < SPF_MAXKICK && !placed; it++) {
                        unsigned int b1, b2;
                        buckets(ck, b1, b2);
                        const unsigned int cand[4] = {2 * b1, 2 * b1 + 1, 2 * b2, 2 * b2 + 1};
                        for (int c = 0; c < 4 && !placed; c++)
                            if ((unsigned long long)skeys[cand[c]] == E) { skeys[cand[c]] = ck; slo[cand[c]] = clo; scnt[cand[c]] = ccnt; placed = true; }
                        if (placed) break;
                        rng = rng * 1664525u + 1013904223u;
                        const unsigned int vb = from == b1 ? b2 : (from == b2 ? b1 : ((rng >> 16) & 1 ? b1 : b2));
                        const unsigned int vs = 2 * vb + ((rng >> 17) & 1);
                        const long long vk = skeys[vs]; const unsigned int vlo = slo[vs], vcnt = scnt[vs];
                        skeys[vs] = ck; slo[vs] = clo; scnt[vs] = ccnt;
                        ck = vk; clo = vlo; ccnt = vcnt; from = vb;
                    }
                    if (!placed)  // the walk did not end: the entry still in hand leaves for the global table with its partial sums
                        spf_direct<HAS_SUM, HAS_CNT>(&a, ck, (unsigned long long)clo - 0x80000000ull, (unsigned long long)ccnt);
                    s = find(key);
                }
                if (s >= 0) add(s, key, val);
                else spf_direct<HAS_SUM, HAS_CNT>(&a, key, (unsigned long long)val, 1ull);  // the new key itself was the one evicted
            }
            ctl[SPF_CTL_RNG] = rng;
            *kq_cnt = 0;
        };

        // Hand-off without consumer-side fences (the NCCL "simple" protocol): the flusher fences between its ring stores and
        // the cursor store; here the cursor is polled with a relaxed GPU-scope load and the ring lines are then read from L2
        // (ld.cg) by loads that are only ISSUED once the cursor value is known.  The tail is published after the rows have been
        // aggregated, i.e. after their values arrived, so the flusher can never overwrite a line that is still to be read.
        unsigned int tail = 0;  // lines consumed of ring p0 + lane
        unsigned int idle_ns = 50;
        bool finished = false;
        const unsigned int* pubp = fa.pub + (size_t)(p0 + (mine ? myring : 0)) * G + me;
        unsigned int hv = mine ? ld_relaxed_u32(pubp) : 0u;
        SPF_TM_DECL;
        while (true) {
            // safe point: no lookup of this warp is in flight
            if (*kq_cnt != 0) {
                SPF_TM(0);
                named_bar(2, SPF_CT);
                if (cw == 0 && lane == 0) place_parked();
                named_bar(2, SPF_CT);
                SPF_TM(4);
                SPF_STAT_INC(4, 1);
            }
            if (finished) {
                if (*cdone >= (unsigned int)SPF_NCW) break;
                __nanosleep(1000);
                SPF_TM(5);
                continue;
            }
            const bool fin = (hv & SPF_FINAL) != 0;
            const unsigned int avail = mine ? (hv & ~SPF_FINAL) - tail : 0u;  // lines waiting in my ring
            // Lines are taken four at a time (one per 8-lane group: full warps); a ring with fewer waits for more to arrive — a
            // FULL ring holds SPF_RL = 16 of them, so a flusher is never blocked by this.  After the last publication: everything.
            const unsigned int take = fin ? avail : (avail & ~3u);
            unsigned int am = __ballot_sync(0xffffffffu, take != 0);
            if (am == 0) {
                if (__all_sync(0xffffffffu, !mine || (fin && avail == 0))) {
                    finished = true;
                    if (lane == 0) atomicAdd((unsigned int*)cdone, 1u);
                    continue;
                }
                SPF_STAT_INC(6, 1);
                __nanosleep(idle_ns);
                idle_ns = idle_ns < 800 ? idle_ns * 2 : idle_ns;
                hv = mine ? ld_relaxed_u32(pubp) : 0u;
                continue;
            }
            idle_ns = 50;
            SPF_STAT_INC(7, 1);
            SPF_TM(0);
            const unsigned int hv_next = mine ? ld_relaxed_u32(pubp) : 0u;  // next poll: its latency hides behind the lines below
            constexpr int U = 2;  // batches of four lines (32 rows) in flight per warp
            while (am) {
                const int r = __ffs(am) - 1;
                am &= am - 1;
                const unsigned int n = __shfl_sync(0xffffffffu, take, r);
                const unsigned int t0 = __shfl_sync(0xffffffffu, tail, r);
                const longlong2* rbase = fa.ring + (size_t)__shfl_sync(0xffffffffu, ringrow0, r) + l8;
                for (unsigned int i0 = 0; i0 < n; i0 += 4 * U) {
                    longlong2 row[U];
                    bool act[U];
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const unsigned int li = i0 + 4 * u + grp;
                        act[u] = li < n;
                        if (act[u]) row[u] = __ldcg(rbase + ((t0 + li) & (SPF_RL - 1)) * SPF_LINE);
                    }
                    SPF_TM(1);
                    int sl[U];
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        sl[u] = -2;
#ifdef SPF_EXP_NOCONS  // experiment: consumers are a pure sink (rows loaded, not aggregated): producer-side ceiling
                        if (act[u] && row[u].x == 0x7ff123456789abcll) {
#else
                        if (act[u] && row[u].x != EMPTY_KEY) {  // (EMPTY_KEY: padding row of a final, partially filled line)
#endif
                            unsigned int b1, b2;
                            buckets(row[u].x, b1, b2);
                            const ulonglong2 k1 = *reinterpret_cast<const ulonglong2*>(skeys + 2 * b1);
                            const ulonglong2 k2 = *reinterpret_cast<const ulonglong2*>(skeys + 2 * b2);
                            const unsigned long long uk = (unsigned long long)row[u].x;
                            sl[u] = k1.x == uk ? (int)(2 * b1) : k1.y == uk ? (int)(2 * b1 + 1) : k2.x == uk ? (int)(2 * b2) : k2.y == uk ? (int)(2 * b2 + 1) : -1;
                        }
                    }
                    SPF_TM(2);
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        if (sl[u] >= 0) add(sl[u], row[u].x, row[u].y);
                        else if (sl[u] == -1) slow_upsert(row[u].x, row[u].y);
                    }
                    SPF_TM(3);
                }
            }
            SPF_STAT_INC(8, take);
            if (mine && take) { tail += take; st_relaxed_u32(fa.cons + (size_t)me * G + (p0 + myring), tail); }
            hv = hv_next;
        }
        SPF_TM_FLUSH(32);
    }
    __syncthreads();
    // ---- flush the shared table into the state's global table (once per launch) ----
    for (int s = tid; s < NS; s += SPF_THREADS) {
        const long long key = skeys[s];
        if (key == EMPTY_KEY) continue;
        const unsigned long long sum = (unsigned long long)slo[s] - 0x80000000ull;  // remove the bias (wraps mod 2^64)
        spf_direct<HAS_SUM, HAS_CNT>(&a, key, sum, (unsigned long long)scnt[s]);
    }
}
