// join.cu — streaming hash join on one GPU (H100, sm_90a).
//
// Replaces HashJoinState / JoinPartition of the reference (bodo/libs/streaming/_join.cpp):
//   build  : join_build_consume_batch (:3134-3443) appends batches to device-resident build columns; on the
//            last batch BuildHashTable (:381-437) + FinalizeGroups (:439-512) become three kernels:
//            insert+count (one table slot per distinct key, rows-per-key counter), exclusive scan (CSR
//            groups_offsets), fill (CSR groups = build row ids).  Keys with exactly one build row keep the
//            row id in the slot itself, so the common 1:N probe needs no CSR lookup.
//   probe  : join_probe_consume_batch (:3459-3900): pass A looks up every probe row and writes its match count,
//            a scan turns counts into output offsets, pass B expands the matches and gathers the kept build and
//            probe columns straight into the output columns (produce_probe_output :729-827 +
//            ChunkedTableBuilder::AppendJoinOutput fused; no (build_idx, probe_idx) pair vectors in HBM,
//            unlike the cuDF path bodo/libs/streaming/cuda_join.cpp:543-612).
//   outer  : probe_table_outer emits unmatched probe rows with NULL build columns; build_table_outer tracks
//            matched build rows and emits the unmatched ones after the last probe batch.
// NA keys: `is_na_equal` is a state option, as in the reference's HashJoinState.  true (the pandas door,
// bodo/pandas/physical/join.h:267): NA joins NA.  false (the default of join_state_init_py_entry, SQL semantics): rows
// with an NA key never match — they are filtered from the build table unless it is the outer side
// (_join.cpp:3180 filter_na_values) and only survive as NULL-extended rows of an outer join.
// Keys: the first n_keys (1..4) columns of each side; n_keys 0 is the nested-loop join (probe_nested, no table).  One key column can take the unique-key tables (Slot16 / Slot32); a
// multi-column key always takes the CSR form, whose key table holds (tuple-hash tag, first build row) words (the _mk kernels).
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <utility>
#include <vector>

#include "common.cuh"
#include "expr.cuh"

namespace b200 {

constexpr long long J_EMPTY = (long long)0x8000000000000000ULL;
constexpr int J_MAX_COLS = 32;
constexpr uint32_t J_NONE = 0xffffffffu;

// ---- exclusive scan u32 -> u64 in three launches over 2048-row tiles (common.cuh): each tile's sum, tile_carry_kernel over the
// tile sums, each tile's scan seeded by its prefix ----
__global__ void __launch_bounds__(TILE_THREADS) offsets_tile_sum_kernel(const uint32_t* in, int64_t n, unsigned long long* sums) {
    unsigned long long s = 0;
    const int64_t i0 = tile_row(blockIdx.x, 0);
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = i0 + k * TILE_THREADS;
        if (i < n) s += in[i];
    }
    s = block_reduce<SumOf<unsigned long long>>(s);
    if (threadIdx.x == 0) sums[blockIdx.x] = s;
}
__global__ void __launch_bounds__(TILE_THREADS) offsets_tile_scan_kernel(const uint32_t* in, int64_t n, const unsigned long long* carry,
                                                                         unsigned long long* out) {
    uint32_t x[TILE_ITEMS];
    unsigned long long v[TILE_ITEMS];
    const int64_t i0 = tile_row(blockIdx.x, 0);
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = i0 + k * TILE_THREADS;
        v[k] = x[k] = i < n ? in[i] : 0;
    }
    tile_scan<SumOf<unsigned long long>>(carry[blockIdx.x], v);
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = i0 + k * TILE_THREADS;
        if (i < n) out[i] = v[k] - x[k];
    }
}

Scanner::~Scanner() { pinned_release(h_total, 8); }
unsigned long long Scanner::run(const uint32_t* in, int64_t n, unsigned long long* out, cudaStream_t st, int64_t* launches) {
    if (!h_total) h_total = (unsigned long long*)pinned_acquire(8);
    if (n == 0) return 0;
    int64_t nb = (n + TILE_ROWS - 1) / TILE_ROWS;
    sums.ensure((size_t)nb * 8);
    total.ensure(8);
    offsets_tile_sum_kernel<<<(unsigned)nb, TILE_THREADS, 0, st>>>(in, n, sums.as<unsigned long long>());
    tile_carry_kernel<SumOf<unsigned long long>><<<1, 1024, 0, st>>>(sums.as<unsigned long long>(), nb, total.as<unsigned long long>());
    offsets_tile_scan_kernel<<<(unsigned)nb, TILE_THREADS, 0, st>>>(in, n, sums.as<unsigned long long>(), out);
    *launches += 3;
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(h_total, total.p, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return *h_total;
}

// ---- hash table ----
struct SlotInfo { uint32_t cnt; uint32_t first; };  // rows with this key; one of those rows (row id)

__device__ __forceinline__ uint64_t j_hash_slot(long long key, uint64_t mask) {
    return (xxh3_64_short((uint64_t)key, 8, SEED_HASH_JOIN) >> 32) & mask;
}
// capacity >= 2 * n_build, so an insert always finds a free slot
__device__ __forceinline__ uint32_t j_find_or_insert(long long* tkeys, uint64_t cap, long long key) {
    uint64_t mask = cap - 1, s = j_hash_slot(key, mask);
    while (true) {
        long long k = __ldcg(tkeys + s);
        if (k == key) return (uint32_t)s;
        if (k == J_EMPTY) {
            long long prev = (long long)atomicCAS((unsigned long long*)(tkeys + s), (unsigned long long)J_EMPTY, (unsigned long long)key);
            if (prev == J_EMPTY || prev == key) return (uint32_t)s;
        }
        s = (s + 1) & mask;
    }
}
__device__ __forceinline__ uint32_t j_find(const long long* __restrict__ tkeys, uint64_t cap, long long key) {
    uint64_t mask = cap - 1, s = j_hash_slot(key, mask);
    while (true) {
        long long k = __ldg(tkeys + s);
        if (k == key) return (uint32_t)s;
        if (k == J_EMPTY) return J_NONE;
        s = (s + 1) & mask;
    }
}

// One key row as the tables hold it, loaded once per row.  An integer key is its value.  A float key (FK: both key columns are
// float64, or both float32) is the canon_float_key encoding of its value, and a NaN key is an NA key: it joins NaN and NA keys
// exactly when NA joins NA (is_na_equal).  A non-NaN float never encodes to J_EMPTY, so float keys never use the marker-key slot
// cap + 1.  `bits` is the input's bit pattern (zero-extended), which the unique-key kernels write to the build key column.  The
// data of a row that is not `valid` is not read.
struct JoinKey { long long key; unsigned long long bits; bool na; };
template <bool FK>
__device__ __forceinline__ JoinKey load_join_key(const void* __restrict__ p, int ct, int64_t i, bool valid) {
    if constexpr (FK) {
        const unsigned long long b = !valid ? 0ull : ct == CT_FLOAT64 ? ((const unsigned long long*)p)[i] : ((const unsigned int*)p)[i];
        const long long k = canon_float_key(ct == CT_FLOAT64 ? __longlong_as_double((long long)b) : (double)__uint_as_float((unsigned int)b));
        return {k, b, !valid || k == J_EMPTY};
    } else {
        const long long k = valid ? load_int_as_i64(p, ct, i) : 0;
        return {k, (unsigned long long)k, !valid};
    }
}

// The as-of join's `on` column of one side: a build column (validity one byte per row, nullptr = none) or a probe column (Arrow
// bitmap).  A null cell and a NaN are NA: such a row takes part in no match.
struct AsofOn { const void* data; const uint8_t* valid; SortKey key; };
template <bool BYTES>
__device__ __forceinline__ uint64_t asof_word(const AsofOn& o, int64_t i, bool& na) {
    na = BYTES ? (o.valid && !o.valid[i]) : !bit_valid(o.valid, i);
    return sort_word(o.key, load_bits(o.data, o.key.size, i), na);
}

// BuildHashTable: slot per distinct key, num_rows_in_group, build_row_to_group_map (= row_slot).  ASOF: a row whose `on` cell is
// NA belongs to no group either.
template <bool FK, bool ASOF>
__global__ void join_insert_count_kernel(const void* key_data, int key_ctype, const uint8_t* key_valid_bytes, int64_t n,
                                         long long* tkeys, uint64_t cap, SlotInfo* info, uint32_t* row_slot, int na_equal, const AsofOn on) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t s;
        if constexpr (ASOF) {
            bool na;
            asof_word<true>(on, i, na);
            if (na) { row_slot[i] = J_NONE; continue; }
        }
        const JoinKey jk = load_join_key<FK>(key_data, key_ctype, i, !key_valid_bytes || key_valid_bytes[i]);
        if (jk.na) {
            if (!na_equal) { row_slot[i] = J_NONE; continue; }  // never matches: belongs to no group
            s = (uint32_t)cap;  // NA group
        } else {
            s = jk.key == J_EMPTY ? (uint32_t)cap + 1 : j_find_or_insert(tkeys, cap, jk.key);
        }
        row_slot[i] = s;
        atomicAdd(&info[s].cnt, 1u);
        info[s].first = (uint32_t)i;  // any row of the group; exact when cnt == 1
    }
}
__global__ void join_slot_counts_kernel(const SlotInfo* info, uint64_t n_slots, uint32_t* cnt_multi, uint32_t min_rows) {
    // the CSR holds the groups of at least min_rows rows: 2 for the equi-join (a group of one keeps its row in the slot), 1 for
    // the as-of join
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_slots; s += stride) {
        uint32_t c = info[s].cnt;
        cnt_multi[s] = c >= min_rows ? c : 0;
    }
}
// FinalizeGroups: groups[offs[slot] + k] = k-th build row of the slot's key
__global__ void join_fill_groups_kernel(const uint32_t* row_slot, int64_t n, const SlotInfo* info, const unsigned long long* offs,
                                        uint32_t* fill, uint32_t* groups) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t s = row_slot[i];
        if (s != J_NONE && info[s].cnt > 1) groups[offs[s] + atomicAdd(&fill[s], 1u)] = (uint32_t)i;
    }
}

// probe pass A: slot + match count per probe row
// mode 0: inner / outer join; 1: anti join (a probe row goes out, once and with NULL build columns, iff it has NO match:
// the is_anti_join template of the reference's probe, _join.cpp:763-767); 2: mark join (every probe row goes out once, without
// build columns; mark[i] says whether it has a match, _join.cpp:3668-3693)
// key_reject: the probe key is int64 / DATETIME / TIMEDELTA and the build key UINT64, or the other way round.  Keys join by value, so
// a valid probe key with its top bit set (a negative value, or a uint64 of at least 2^63) has no partner; it is not an NA key.
// The slot of probe row i's key in the single-key table (J_NONE: no such key).
template <bool FK>
__device__ __forceinline__ uint32_t probe_slot(const void* key_data, int key_ctype, const uint8_t* key_valid, int64_t i, const long long* tkeys,
                                               uint64_t cap, int na_equal, int key_reject) {
    const JoinKey jk = load_join_key<FK>(key_data, key_ctype, i, bit_valid(key_valid, i));
    if (jk.na) return na_equal ? (uint32_t)cap : J_NONE;
    if (!FK && key_reject && jk.key < 0) return J_NONE;
    return jk.key == J_EMPTY ? (uint32_t)cap + 1 : j_find(tkeys, cap, jk.key);
}
template <bool FK>
__global__ void join_probe_count_kernel(const void* key_data, int key_ctype, const uint8_t* key_valid, int64_t n,
                                        const long long* tkeys, uint64_t cap, const SlotInfo* info, int probe_outer,
                                        uint32_t* pslot, uint32_t* pcnt, int na_equal, int mode, uint8_t* mark, int key_reject) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t s = probe_slot<FK>(key_data, key_ctype, key_valid, i, tkeys, cap, na_equal, key_reject);
        uint32_t c = s == J_NONE ? 0 : info[s].cnt;
        if (c == 0) s = J_NONE;
        if (mode == 1) { pslot[i] = J_NONE; pcnt[i] = c ? 0u : 1u; continue; }
        if (mode == 2) { pslot[i] = J_NONE; pcnt[i] = 1u; mark[i] = c ? 1 : 0; continue; }
        pslot[i] = s;
        pcnt[i] = c ? c : (probe_outer ? 1u : 0u);
    }
}

struct GatherArgs {
    int64_t n_probe;
    const uint32_t* pslot;
    const unsigned long long* poff;
    const SlotInfo* info;
    const unsigned long long* goffs;
    const uint32_t* groups;
    uint8_t* bmatched;  // build_outer: matched flags per build row, else nullptr
    int n_b, n_p;       // kept build / probe columns
    const void* b_data[J_MAX_COLS]; const uint8_t* b_valid[J_MAX_COLS]; int b_size[J_MAX_COLS];
    const void* p_data[J_MAX_COLS]; const uint8_t* p_valid[J_MAX_COLS]; int p_size[J_MAX_COLS];
    void* ob_data[J_MAX_COLS]; uint8_t* ob_valid[J_MAX_COLS];  // output columns (validity: one byte per row or nullptr)
    void* op_data[J_MAX_COLS]; uint8_t* op_valid[J_MAX_COLS];
};
__device__ __forceinline__ void zero_item(void* dst, int64_t d, int size) {
    switch (size) {
        case 8: ((uint64_t*)dst)[d] = 0; break;
        case 4: ((uint32_t*)dst)[d] = 0; break;
        case 2: ((uint16_t*)dst)[d] = 0; break;
        default: ((uint8_t*)dst)[d] = 0; break;
    }
}
// probe pass B: expand matches and gather both sides into the output columns (build validity is byte-per-row)
__global__ void __launch_bounds__(256) join_probe_gather_kernel(const __grid_constant__ GatherArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n_probe; i += stride) {
        uint32_t s = a.pslot[i];
        unsigned long long o = a.poff[i];
        uint32_t c = s == J_NONE ? 0 : a.info[s].cnt;
        uint32_t reps = c ? c : (a.poff[i + 1] - o ? 1u : 0u);  // outer probe row without match: one NULL-build row
        for (uint32_t q = 0; q < reps; q++) {
            int64_t orow = (int64_t)(o + q);
            if (c) {
                uint32_t brow = c == 1 ? a.info[s].first : a.groups[a.goffs[s] + q];
                if (a.bmatched) a.bmatched[brow] = 1;
                for (int k = 0; k < a.n_b; k++) {
                    copy_cell(a.ob_data[k], orow, a.b_data[k], brow, a.b_size[k]);
                    if (a.ob_valid[k]) a.ob_valid[k][orow] = a.b_valid[k] ? a.b_valid[k][brow] : 1;
                }
            } else {
                for (int k = 0; k < a.n_b; k++) { zero_item(a.ob_data[k], orow, a.b_size[k]); a.ob_valid[k][orow] = 0; }
            }
            for (int k = 0; k < a.n_p; k++) {
                copy_cell(a.op_data[k], orow, a.p_data[k], i, a.p_size[k]);
                if (a.op_valid[k]) a.op_valid[k][orow] = bit_valid(a.p_valid[k], i) ? 1 : 0;
            }
        }
    }
}

// build_outer tail: unmatched build rows with NULL probe columns
__global__ void join_unmatched_flags_kernel(const uint8_t* bmatched, int64_t n, uint32_t* flags) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) flags[i] = bmatched[i] ? 0u : 1u;
}
struct TailArgs {
    int64_t n_build;
    const uint32_t* flags;
    const unsigned long long* off;
    int n_b, n_p;
    const void* b_data[J_MAX_COLS]; const uint8_t* b_valid[J_MAX_COLS]; int b_size[J_MAX_COLS];
    int p_size[J_MAX_COLS];
    void* ob_data[J_MAX_COLS]; uint8_t* ob_valid[J_MAX_COLS];
    void* op_data[J_MAX_COLS]; uint8_t* op_valid[J_MAX_COLS];
};
__global__ void join_unmatched_emit_kernel(const __grid_constant__ TailArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n_build; i += stride) {
        if (!a.flags[i]) continue;
        int64_t orow = (int64_t)a.off[i];
        for (int k = 0; k < a.n_b; k++) {
            copy_cell(a.ob_data[k], orow, a.b_data[k], i, a.b_size[k]);
            if (a.ob_valid[k]) a.ob_valid[k][orow] = a.b_valid[k] ? a.b_valid[k][i] : 1;
        }
        for (int k = 0; k < a.n_p; k++) { zero_item(a.op_data[k], orow, a.p_size[k]); a.op_valid[k][orow] = 0; }
    }
}

__global__ void expand_bitmap_kernel(const uint8_t* bitmap, int64_t n, uint8_t* bytes) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) bytes[i] = bit_valid(bitmap, i) ? 1 : 0;
}

// ---- fast path: unique build keys + inner join --------------------------------------------------
// One 16-byte slot {key, first_row, cnt} (one 32-byte sector per lookup instead of two), the non-key build columns
// packed row-major in 8-byte fields (one sector per matched row instead of one per column), and a single fused kernel:
// lookup -> warp-aggregated output cursor -> gather both sides straight into the output columns. No per-row slot /
// count / offset arrays and no scan. Output order follows the cursor (unspecified, as in the reference).
struct __align__(16) Slot16 { long long key; uint32_t first; uint32_t cnt; };

__global__ void join_make_slots16_kernel(const long long* tkeys, const SlotInfo* info, uint64_t n_slots, Slot16* out) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_slots; s += stride) {
        Slot16 e; e.key = tkeys[s]; e.first = info[s].first; e.cnt = info[s].cnt;
        out[s] = e;
    }
}
struct PackPayloadArgs {
    int64_t n_build;
    int n_fields;
    const void* src[J_MAX_COLS];
    int size[J_MAX_COLS];
    unsigned long long* out;  // n_build x n_fields 8-byte fields
};
__global__ void join_pack_payload_kernel(const __grid_constant__ PackPayloadArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n_build; i += stride)
        for (int f = 0; f < a.n_fields; f++) {
            unsigned long long v = 0;
            switch (a.size[f]) {
                case 8: v = ((const uint64_t*)a.src[f])[i]; break;
                case 4: v = ((const uint32_t*)a.src[f])[i]; break;
                case 2: v = ((const uint16_t*)a.src[f])[i]; break;
                default: v = ((const uint8_t*)a.src[f])[i]; break;
            }
            a.out[i * a.n_fields + f] = v;
        }
}
struct FastProbeArgs {
    int64_t n_probe;
    const void* key_data; int key_ctype; const uint8_t* key_valid;
    const Slot16* slots; uint64_t cap;
    const unsigned long long* bpack; int n_fields;
    unsigned long long* cursor;
    int n_b, n_p;
    int na_equal;
    int key_reject;                        // as in join_probe_count_kernel
    int b_field[J_MAX_COLS];               // kept build col -> payload field index, -1 = the key column
    const uint8_t* b_valid[J_MAX_COLS]; int b_size[J_MAX_COLS];
    const void* p_data[J_MAX_COLS]; const uint8_t* p_valid[J_MAX_COLS]; int p_size[J_MAX_COLS];
    void* ob_data[J_MAX_COLS]; uint8_t* ob_valid[J_MAX_COLS];
    void* op_data[J_MAX_COLS]; uint8_t* op_valid[J_MAX_COLS];
};
__device__ __forceinline__ void store_sized(void* dst, int64_t d, unsigned long long v, int size) {
    switch (size) {
        case 8: ((uint64_t*)dst)[d] = v; break;
        case 4: ((uint32_t*)dst)[d] = (uint32_t)v; break;
        case 2: ((uint16_t*)dst)[d] = (uint16_t)v; break;
        default: ((uint8_t*)dst)[d] = (uint8_t)v; break;
    }
}
template <bool FK>
__global__ void __launch_bounds__(256) join_probe_fast_kernel(const __grid_constant__ FastProbeArgs a) {
    // tile = 1024 probe rows per CTA iteration (4 per thread); ONE global cursor atomic per tile (a cursor atomic per
    // warp serialises on a single L2 address: measured 117 ms for 1e9 probe rows, dominated by that atomic)
    constexpr int R = 4, NW = 8, TILE = 256 * R;
    __shared__ unsigned int wcnt[R * NW];
    __shared__ unsigned int woff[R * NW];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t mask = a.cap - 1;
    const int64_t n_tiles = (a.n_probe + TILE - 1) / TILE;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        long long key[R];
        unsigned long long bits[R];  // the probe key's bit pattern: the build key column's value on a match
        uint32_t brow[R];
        unsigned int rank[R];
        bool match[R], kvalid[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t i = t * TILE + r * 256 + threadIdx.x;
            match[r] = false; kvalid[r] = true; key[r] = 0; bits[r] = 0; brow[r] = 0;
            if (i < a.n_probe) {
                kvalid[r] = bit_valid(a.key_valid, i);
                const JoinKey jk = load_join_key<FK>(a.key_data, a.key_ctype, i, true);  // bits under a NULL too: the output's validity hides them
                key[r] = jk.key; bits[r] = jk.bits;
                if (!kvalid[r] || jk.na) { if (a.na_equal) { Slot16 e = a.slots[a.cap]; match[r] = e.cnt > 0; brow[r] = e.first; } }
                else if (!FK && a.key_reject && key[r] < 0) {}  // a value the build key's type cannot hold: no partner
                else if (key[r] == J_EMPTY) { Slot16 e = a.slots[a.cap + 1]; match[r] = e.cnt > 0; brow[r] = e.first; }
                else {
                    uint64_t s = j_hash_slot(key[r], mask);
                    while (true) {
                        int4 raw = __ldg(reinterpret_cast<const int4*>(a.slots + s));
                        long long k = ((long long)(unsigned int)raw.x) | ((long long)raw.y << 32);
                        if (k == key[r]) { match[r] = (unsigned int)raw.w > 0; brow[r] = (unsigned int)raw.z; break; }
                        if (k == J_EMPTY) break;
                        s = (s + 1) & mask;
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            unsigned m = __ballot_sync(0xffffffffu, match[r]);
            rank[r] = __popc(m & ((1u << lane) - 1));
            if (lane == 0) wcnt[r * NW + warp] = __popc(m);
        }
        __syncthreads();
        if (warp == 0) {  // exclusive scan of the 32 (row-slot, warp) counts, one cursor atomic for the tile
            const unsigned int x = wcnt[lane], inc = warp_inclusive_scan<SumOf<unsigned int>>(x);
            woff[lane] = inc - x;
            if (lane == 31) tile_base = inc ? atomicAdd(a.cursor, (unsigned long long)inc) : 0ull;
        }
        __syncthreads();
        const unsigned long long base = tile_base;
#pragma unroll
        for (int r = 0; r < R; r++) {
            if (!match[r]) continue;
            const int64_t i = t * TILE + r * 256 + threadIdx.x;
            const int64_t orow = (int64_t)(base + woff[r * NW + warp] + rank[r]);
            const unsigned long long* fields = a.bpack + (size_t)brow[r] * a.n_fields;
            for (int k2 = 0; k2 < a.n_b; k2++) {
                int f = a.b_field[k2];
                unsigned long long v = f < 0 ? bits[r] : __ldg(fields + f);
                store_sized(a.ob_data[k2], orow, v, a.b_size[k2]);
                if (a.ob_valid[k2]) a.ob_valid[k2][orow] = f < 0 ? (kvalid[r] ? 1 : 0) : (a.b_valid[k2] ? a.b_valid[k2][brow[r]] : 1);
            }
            for (int k2 = 0; k2 < a.n_p; k2++) {
                copy_cell(a.op_data[k2], orow, a.p_data[k2], i, a.p_size[k2]);
                if (a.op_valid[k2]) a.op_valid[k2][orow] = bit_valid(a.p_valid[k2], i) ? 1 : 0;
            }
        }
        __syncthreads();
    }
}

// ---- inline-payload probe: the specialisation for all-8-byte, bitmap-free schemas with at most two build payload columns ----
// Slot32 = {key, f0, f1, first | cnt << 32}: key AND payload of a unique-key build row sit in ONE 32-byte sector, so a probe
// row costs one random sector instead of two (Slot16 + packed payload row).  All coalesced loads of a tile (key and the kept
// probe columns, 4 rows per thread) are issued before the first dependent table access.
struct __align__(32) Slot32 { long long key; unsigned long long f0, f1; uint32_t first; uint32_t cnt; };
constexpr int J_INL_MAX_P = 4;
struct InlineProbeArgs {
    int64_t n_probe;
    const long long* key;
    const Slot32* slots; uint64_t cap;
    unsigned long long* cursor;
    int n_b;                       // kept build columns (<= 3)
    int b_field[4];                // -1 = key, 0 / 1 = payload field
    unsigned long long* ob[4];
    const unsigned long long* p[J_INL_MAX_P];  // kept probe columns (the key column included when kept)
    unsigned long long* op[J_INL_MAX_P];
    int na_equal;                  // float64 keys: a NaN probe key looks up the NA slot cap
};
// Direct build of the Slot32 table (no separate key table / slot-info / CSR passes): one random 32-byte sector per build row.
// A row claims its slot with a CAS on the key word, counts itself in the slot and, when it is the first row of that key,
// writes the payload.  A second row of any key raises *dup: the host then falls back to the general build (CSR groups).
// Float64 keys (FK) are stored as their canon_float_key encoding; a NaN row takes the NA slot cap under na_equal (the marker
// slot's scheme: the key word stays the free-slot pattern) and belongs to no group otherwise.
__global__ void join_fill_slots32_kernel(Slot32* slots, uint64_t n_slots) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const ulonglong4 e = make_ulonglong4((unsigned long long)J_EMPTY, 0ull, 0ull, 0ull);
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_slots; s += stride) reinterpret_cast<ulonglong4*>(slots)[s] = e;
}
template <bool FK>
__global__ void __launch_bounds__(256) join_build_inline_kernel(const long long* __restrict__ keys, const unsigned long long* __restrict__ f0, const unsigned long long* __restrict__ f1,
                                                                int64_t n, int64_t row0, Slot32* slots, uint64_t cap, int* dup, int na_equal) {
    constexpr int R = 4;
    const uint64_t mask = cap - 1;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * R;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x * R + threadIdx.x; i0 < n; i0 += stride) {
        long long key[R], k0[R];
        uint64_t s[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t i = i0 + r * 256;
            key[r] = i < n ? __ldcs(keys + i) : 0;
            if constexpr (FK) key[r] = canon_float_key(__longlong_as_double(key[r]));
        }
#pragma unroll
        for (int r = 0; r < R; r++) {  // the R first probes are in flight together
            s[r] = key[r] == J_EMPTY ? (FK ? cap : cap + 1) : j_hash_slot(key[r], mask);
            k0[r] = __ldcg(&slots[s[r]].key);
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t i = i0 + r * 256;
            if (i >= n) continue;
            if (FK && key[r] == J_EMPTY && !na_equal) continue;  // a NaN key that never matches
            bool won = false;  // this row claimed a free slot (it is the first row of its key)
            if (key[r] != J_EMPTY) {
                long long k = k0[r];
                while (true) {
                    if (k == J_EMPTY) {
                        const long long prev = (long long)atomicCAS((unsigned long long*)&slots[s[r]].key, (unsigned long long)J_EMPTY, (unsigned long long)key[r]);
                        if (prev == J_EMPTY) { won = true; break; }
                        k = prev;
                    }
                    if (k == key[r]) break;  // another row holds this key: duplicate
                    s[r] = (s[r] + 1) & mask;
                    k = __ldcg(&slots[s[r]].key);
                }
            } else {
                won = atomicAdd(&slots[s[r]].cnt, 1u) == 0;  // marker-key slot: its key word stays the free-slot pattern
            }
            if (won) {  // the rest of the sector: f0 (8 B), then {f1, first, cnt = 1} (16 B)
                slots[s[r]].f0 = f0 ? __ldcs(f0 + i) : 0ull;
                const unsigned long long f1v = f1 ? __ldcs(f1 + i) : 0ull;
                *reinterpret_cast<ulonglong2*>(&slots[s[r]].f1) = make_ulonglong2(f1v, (unsigned long long)(uint32_t)(row0 + i) | (1ull << 32));
            } else *dup = 1;
        }
    }
}
__global__ void join_slots16_from32_kernel(const Slot32* in, uint64_t n_slots, Slot16* out) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n_slots; s += stride) {
        Slot16 e; e.key = in[s].key; e.first = in[s].first; e.cnt = in[s].cnt;
        out[s] = e;
    }
}
// One Slot32 (one 32-byte sector) through the read-only path.  sm_90 has no 256-bit load: two 128-bit loads of the same
// aligned sector, issued back to back, still cost one sector of L2 / HBM traffic.
__device__ __forceinline__ void ld_slot32(const Slot32* p, unsigned long long& w0, unsigned long long& w1, unsigned long long& w2,
                                          unsigned long long& w3) {
    asm volatile("ld.global.nc.v2.u64 {%0, %1}, [%4];\n\tld.global.nc.v2.u64 {%2, %3}, [%4+16];"
                 : "=l"(w0), "=l"(w1), "=l"(w2), "=l"(w3) : "l"(p));
}
// Float64 keys (FK): the slots hold canon_float_key encodings.  A NaN probe key looks up the NA slot cap under na_equal and
// otherwise the marker slot cap + 1, which float keys leave empty.  The build key column gets the probe key's bits.
template <bool FK, int NF, int NPK>
__global__ void __launch_bounds__(256) join_probe_inline_kernel(const __grid_constant__ InlineProbeArgs a) {
    constexpr int R = 4, NW = 8, TILE = 256 * R;
    __shared__ unsigned int wcnt[R * NW];
    __shared__ unsigned int woff[R * NW];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t mask = a.cap - 1;
    const int64_t n_tiles = (a.n_probe + TILE - 1) / TILE;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        long long key[R], ck[R];  // the probe key's bits; its table key
        unsigned long long pv[NPK][R], f0[R], f1[R];
        unsigned int rank[R];
        bool match[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t i = t * TILE + r * 256 + threadIdx.x;
            const bool in = i < a.n_probe;
            key[r] = in ? __ldcs(a.key + i) : 0;
            ck[r] = FK ? canon_float_key(__longlong_as_double(key[r])) : key[r];
#pragma unroll
            for (int c = 0; c < NPK; c++) pv[c][r] = in ? __ldcs(a.p[c] + i) : 0ull;
        }
        // first probe of all R rows: the R random 32-byte slot loads (one sector each) are in flight together;
        // a data-dependent probe loop per row would serialise them
        uint64_t sl[R];
        unsigned long long w0[R], w1[R], w2[R], w3[R];
#pragma unroll
        for (int r = 0; r < R; r++) {
            sl[r] = ck[r] == J_EMPTY ? (FK && a.na_equal ? a.cap : a.cap + 1) : j_hash_slot(ck[r], mask);
            ld_slot32(a.slots + sl[r], w0[r], w1[r], w2[r], w3[r]);
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t i = t * TILE + r * 256 + threadIdx.x;
            match[r] = false; f0[r] = 0; f1[r] = 0;
            if (i >= a.n_probe) continue;
            while (true) {
                if ((long long)w0[r] == ck[r]) {
                    if (NF >= 1) f0[r] = w1[r];
                    if (NF >= 2) f1[r] = w2[r];
                    match[r] = (unsigned int)(w3[r] >> 32) > 0;
                    break;
                }
                if ((long long)w0[r] == J_EMPTY || sl[r] > mask) break;  // free slot, or the marker-key slot (cap + 1) without a build row
                sl[r] = (sl[r] + 1) & mask;  // collision (about one row in four at this load factor): next slot
                ld_slot32(a.slots + sl[r], w0[r], w1[r], w2[r], w3[r]);
            }
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            unsigned m = __ballot_sync(0xffffffffu, match[r]);
            rank[r] = __popc(m & ((1u << lane) - 1));
            if (lane == 0) wcnt[r * NW + warp] = __popc(m);
        }
        __syncthreads();
        if (warp == 0) {
            const unsigned int x = wcnt[lane], inc = warp_inclusive_scan<SumOf<unsigned int>>(x);
            woff[lane] = inc - x;
            if (lane == 31) tile_base = inc ? atomicAdd(a.cursor, (unsigned long long)inc) : 0ull;
        }
        __syncthreads();
        const unsigned long long base = tile_base;
#pragma unroll
        for (int r = 0; r < R; r++) {
            if (!match[r]) continue;
            const int64_t orow = (int64_t)(base + woff[r * NW + warp] + rank[r]);
            for (int k2 = 0; k2 < a.n_b; k2++) {
                const int f = a.b_field[k2];
                a.ob[k2][orow] = f < 0 ? (unsigned long long)key[r] : (f == 0 ? f0[r] : f1[r]);
            }
#pragma unroll
            for (int c = 0; c < NPK; c++) a.op[c][orow] = pv[c][r];
        }
        __syncthreads();
    }
}

// ---- multi-column keys (n_keys 2..4): the key table and the key-reading kernels of the general (CSR) path ----
// Key columns are a KeySet in key order: build validity is one byte per row (nullptr = all valid), probe validity an Arrow bitmap.
// The key table holds one 8-byte word per slot: the 32-bit tag of the row's tuple hash in the high half, the first build row that
// claimed the slot in the low half; MK_EMPTY (row J_NONE) is a free slot.  Slot index and tag are independent bits of the hash.
// Two rows are one key when the tags match and every key column compares equal (build rows are complete before finalize_build,
// so the insert compares against the occupant's row without a race).  NA (and NaN) is part of the tuple: the NA slot cap and the
// marker slot cap + 1 stay unused.  From the slot id on, the single-key general path runs unchanged.
constexpr unsigned long long MK_EMPTY = ~0ull;
// One tuple in canonical form: per column the load_join_key value (0 under an NA), and bit j of `na` set when column j is NA.
// The runtime filter below reads the keys of any key count, one column included, this way.
struct MKRow { long long key[MAX_HASH_KEYS]; uint32_t na; };
template <bool BYTES>  // BYTES: validity is one byte per row (build side), else a bitmap
__device__ __forceinline__ MKRow mk_row(const KeySet& k, int64_t i) {
    MKRow r;
    r.na = 0;
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++) {
        r.key[j] = 0;
        if (j < k.n_keys && k.data[j]) {  // a runtime filter's absent column (data nullptr) reads as a valid 0
            const bool v = BYTES ? (!k.valid[j] || k.valid[j][i]) : bit_valid(k.valid[j], i);
            const JoinKey jk = ctype_is_float(k.ctype[j]) ? load_join_key<true>(k.data[j], k.ctype[j], i, v)
                                                          : load_join_key<false>(k.data[j], k.ctype[j], i, v);
            if (jk.na) r.na |= 1u << j;
            else r.key[j] = jk.key;
        }
    }
    return r;
}
__device__ __forceinline__ uint64_t mk_hash(const MKRow& r, int n_keys) {
    uint64_t h = SEED_HASH_JOIN;
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++)
        if (j < n_keys) h = mix64(h ^ (uint64_t)r.key[j]);
    return mix64(h ^ r.na);
}
__device__ __forceinline__ bool mk_equal_build(const KeySet& bk, uint32_t row, const MKRow& r) {
    const MKRow o = mk_row<true>(bk, row);
    bool eq = o.na == r.na;
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++) eq = eq && (j >= bk.n_keys || o.key[j] == r.key[j]);
    return eq;
}
// Bit j of `key_reject`: key position j compares an int64 / DATETIME / TIMEDELTA column with a UINT64 one.  A valid key there with
// its top bit set is a value the other column's type cannot hold, so the row has no partner (NA columns read as 0).
__device__ __forceinline__ bool mk_rejected(const MKRow& r, uint32_t key_reject) {
    bool x = false;
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++) x = x || ((key_reject >> j & 1) && r.key[j] < 0);
    return x;
}
__device__ __forceinline__ uint64_t mk_slot(uint64_t h, uint64_t mask) { return (h >> 32) & mask; }
__device__ __forceinline__ uint32_t mk_tag(uint64_t h) { return (uint32_t)h; }

// join_insert_count_kernel for a multi-column key: same outputs (row_slot, info[s].cnt, info[s].first)
template <bool ASOF>
__global__ void join_insert_count_mk_kernel(const KeySet bk, int64_t n, unsigned long long* table, uint64_t cap, SlotInfo* info,
                                            uint32_t* row_slot, int na_equal, const AsofOn on) {
    const uint64_t mask = cap - 1;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        if constexpr (ASOF) {
            bool na;
            asof_word<true>(on, i, na);
            if (na) { row_slot[i] = J_NONE; continue; }
        }
        const MKRow r = mk_row<true>(bk, i);
        if (r.na && !na_equal) { row_slot[i] = J_NONE; continue; }  // never matches: belongs to no group
        const uint64_t h = mk_hash(r, bk.n_keys);
        const unsigned long long mine = ((unsigned long long)mk_tag(h) << 32) | (uint32_t)i;
        uint64_t s = mk_slot(h, mask);
        while (true) {
            unsigned long long w = __ldcg(table + s);
            if (w == MK_EMPTY) {
                w = atomicCAS(table + s, MK_EMPTY, mine);
                if (w == MK_EMPTY) break;  // claimed
            }
            if ((uint32_t)(w >> 32) == mk_tag(h) && mk_equal_build(bk, (uint32_t)w, r)) break;
            s = (s + 1) & mask;
        }
        row_slot[i] = (uint32_t)s;
        atomicAdd(&info[s].cnt, 1u);
        info[s].first = (uint32_t)i;  // any row of the group; exact when cnt == 1
    }
}
// The slot of probe row i's key tuple in the multi-column key table (J_NONE: no such key).
__device__ __forceinline__ uint32_t probe_slot_mk(const KeySet& pk, const KeySet& bk, int64_t i, const unsigned long long* __restrict__ table,
                                                  uint64_t cap, int na_equal, uint32_t key_reject) {
    const uint64_t mask = cap - 1;
    const MKRow r = mk_row<false>(pk, i);
    if ((!r.na || na_equal) && !mk_rejected(r, key_reject)) {
        const uint64_t h = mk_hash(r, pk.n_keys);
        for (uint64_t t = mk_slot(h, mask);; t = (t + 1) & mask) {
            const unsigned long long w = __ldg(table + t);
            if (w == MK_EMPTY) break;
            if ((uint32_t)(w >> 32) == mk_tag(h) && mk_equal_build(bk, (uint32_t)w, r)) return (uint32_t)t;
        }
    }
    return J_NONE;
}
// join_probe_count_kernel for a multi-column key: same outputs (pslot, pcnt, mark) in modes 0, 1 and 2
__global__ void join_probe_count_mk_kernel(const KeySet pk, const KeySet bk, int64_t n, const unsigned long long* __restrict__ table,
                                           uint64_t cap, const SlotInfo* info, int probe_outer, uint32_t* pslot, uint32_t* pcnt,
                                           int na_equal, int mode, uint8_t* mark, uint32_t key_reject) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint32_t s = probe_slot_mk(pk, bk, i, table, cap, na_equal, key_reject);
        uint32_t c = s == J_NONE ? 0 : info[s].cnt;
        if (c == 0) s = J_NONE;
        if (mode == 1) { pslot[i] = J_NONE; pcnt[i] = c ? 0u : 1u; continue; }
        if (mode == 2) { pslot[i] = J_NONE; pcnt[i] = 1u; mark[i] = c ? 1 : 0; continue; }
        pslot[i] = s;
        pcnt[i] = c ? c : (probe_outer ? 1u : 0u);
    }
}

// ---- runtime join filter, any key count (reference: HashJoinState::RuntimeFilter, bodo/libs/streaming/_join.h:1060-1095; bloom
// filter bodo/libs/gpu_bloom_filter.cu:60-201; key min / max bodo/libs/streaming/_join.cpp:3199-3238) ----
// Split-block bloom filter: a key selects one 32-byte block (one sector) with the high hash word and sets / tests one bit in each
// of its eight 32-bit words (eight odd multipliers of the low hash word, the Parquet / Impala scheme).  ~8 bits per build key.
__device__ __forceinline__ void bloom_masks(uint32_t h, uint32_t (&m)[8]) {
    const uint32_t salt[8] = {0x47b6137bu, 0x44974d91u, 0x8824ad5bu, 0xa2b7289du, 0x705495c7u, 0x2df1424bu, 0x9efc4947u, 0x5c6bfb31u};
#pragma unroll
    for (int j = 0; j < 8; j++) m[j] = 1u << ((h * salt[j]) >> 27);
}
// One bloom filter over the tuple hash (mk_hash, also for one key column) of the build rows that belong to a group, and min / max
// per key column over its non-NA values (canon_float_ordered for float columns).  minmax[2j], minmax[2j + 1]: column j.
__global__ void join_bloom_add_kernel(const KeySet bk, int64_t n, int na_equal, uint32_t* bloom, uint64_t n_blocks, long long* minmax) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    long long mn[MAX_HASH_KEYS], mx[MAX_HASH_KEYS];
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++) { mn[j] = INT64_MAX; mx[j] = INT64_MIN; }
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const MKRow r = mk_row<true>(bk, i);
        if (r.na && !na_equal) continue;  // in no group
#pragma unroll
        for (int j = 0; j < MAX_HASH_KEYS; j++) {
            if (j >= bk.n_keys || (r.na >> j & 1)) continue;
            const long long ord = ctype_is_float(bk.ctype[j]) ? canon_float_ordered(r.key[j]) : r.key[j];
            mn[j] = ord < mn[j] ? ord : mn[j]; mx[j] = ord > mx[j] ? ord : mx[j];
        }
        const uint64_t h = mk_hash(r, bk.n_keys);
        uint32_t m[8];
        bloom_masks((uint32_t)h, m);
        uint32_t* blk = bloom + (size_t)(__umul64hi(h, n_blocks)) * 8;
#pragma unroll
        for (int j = 0; j < 8; j++) atomicOr(blk + j, m[j]);
    }
#pragma unroll
    for (int j = 0; j < MAX_HASH_KEYS; j++) {
        for (int d = 16; d; d >>= 1) {
            const long long a = __shfl_xor_sync(0xffffffffu, mn[j], d), b = __shfl_xor_sync(0xffffffffu, mx[j], d);
            mn[j] = a < mn[j] ? a : mn[j]; mx[j] = b > mx[j] ? b : mx[j];
        }
        if ((threadIdx.x & 31) == 0 && j < bk.n_keys && mn[j] <= mx[j]) { atomicMin(minmax + 2 * j, mn[j]); atomicMax(minmax + 2 * j + 1, mx[j]); }
    }
}
struct MKBounds { long long v[2 * MAX_HASH_KEYS]; };
// keep[i] = 1 iff probe row i can still find a partner.  A column absent from the probe table has pk.data[j] == nullptr; the host
// clears its use_minmax bit and use_bloom.  An NA column drops the row unless NA joins NA; then it skips the bounds and is hashed
// into the bloom test as the build side hashes it.
__global__ void join_runtime_filter_kernel(const KeySet pk, int64_t n, int na_equal, const uint32_t* bloom, uint64_t n_blocks,
                                           const MKBounds b, uint32_t use_minmax, int use_bloom, uint8_t* keep, uint32_t key_reject) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const MKRow r = mk_row<false>(pk, i);
        bool k = (!r.na || na_equal) && !mk_rejected(r, key_reject);
#pragma unroll
        for (int j = 0; j < MAX_HASH_KEYS; j++) {
            if (j >= pk.n_keys || !(use_minmax >> j & 1) || (r.na >> j & 1)) continue;
            const long long ord = ctype_is_float(pk.ctype[j]) ? canon_float_ordered(r.key[j]) : r.key[j];
            if (ord < b.v[2 * j] || ord > b.v[2 * j + 1]) k = false;
        }
        if (k && use_bloom) {
            const uint64_t h = mk_hash(r, pk.n_keys);
            uint32_t m[8];
            bloom_masks((uint32_t)h, m);
            const uint4* blk = reinterpret_cast<const uint4*>(bloom + (size_t)(__umul64hi(h, n_blocks)) * 8);
            const uint4 lo = __ldg(blk), hi = __ldg(blk + 1);
            k = (lo.x & m[0]) && (lo.y & m[1]) && (lo.z & m[2]) && (lo.w & m[3]) && (hi.x & m[4]) && (hi.y & m[5]) && (hi.z & m[6]) && (hi.w & m[7]);
        }
        keep[i] = k ? 1 : 0;
    }
}

// ---- non-equi condition (the reference's cond_func: join.py:991-1100, join_state_init_py_entry; cuDF's filter_join_indices) ----
// A candidate pair (probe row p, build row b of p's key group) passes when the condition program (expr.cuh) evaluates to a valid,
// true value.  The program's column argument c < J_MAX_COLS reads build column c at row b (validity one byte per row, nullptr =
// all valid), J_MAX_COLS + c reads probe column c at row p (Arrow bitmap).  A state with a condition always takes the CSR form:
// join_probe_count_kernel / _mk in mode 0 without probe_outer give each probe row its slot, then the two kernels below evaluate
// the condition on every candidate, once to count and once to gather.
struct CondArgs {
    ExprInstr prog[EX_MAX_INSTR];
    const void* b_data[J_MAX_COLS]; const uint8_t* b_valid[J_MAX_COLS]; int b_ct[J_MAX_COLS];
    const void* p_data[J_MAX_COLS]; const uint8_t* p_valid[J_MAX_COLS]; int p_ct[J_MAX_COLS];
};
__device__ __forceinline__ bool cond_pass(const CondArgs& a, int64_t p, uint32_t b) {
    const ExprVal v = expr_run(a.prog, 0, [&](int64_t arg) {
        const int c = (int)arg;
        if (c < J_MAX_COLS) return expr_load(a.b_data[c], a.b_ct[c], b, !a.b_valid[c] || a.b_valid[c][b]);
        const int q = c - J_MAX_COLS;
        return expr_load(a.p_data[q], a.p_ct[q], p, bit_valid(a.p_valid[q], p));
    });
    return v.valid && ev_true(v);
}
// build row of candidate q (0 <= q < c) of key group s, which has c rows
__device__ __forceinline__ uint32_t cand_row(const SlotInfo* info, const unsigned long long* goffs, const uint32_t* groups, uint32_t s,
                                             uint32_t c, uint32_t q) {
    return c == 1 ? info[s].first : groups[goffs[s] + q];
}
// condition pass A: each probe row's output count for the join kind.  mode 0 (inner / outer): its passing pairs, or one NULL-build
// row for a probe_outer row without one; 1 (anti): one row iff no pair passes; 2 (mark): one row, mark[i] = some pair passes.
// pairs[0] += candidate pairs evaluated, pairs[1] += pairs that passed.
__global__ void __launch_bounds__(256) join_cond_count_kernel(const __grid_constant__ CondArgs a, int64_t n, const uint32_t* pslot,
                                                              const SlotInfo* info, const unsigned long long* goffs, const uint32_t* groups,
                                                              int probe_outer, int mode, uint32_t* pcnt, uint8_t* mark, unsigned long long* pairs) {
    unsigned long long n_eval = 0, n_pass = 0;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t s = pslot[i];
        const uint32_t c = s == J_NONE ? 0 : info[s].cnt;
        uint32_t k = 0;
        for (uint32_t q = 0; q < c; q++) k += cond_pass(a, i, cand_row(info, goffs, groups, s, c, q)) ? 1 : 0;
        n_eval += c; n_pass += k;
        if (mode == 1) pcnt[i] = k ? 0u : 1u;
        else if (mode == 2) { pcnt[i] = 1u; mark[i] = k ? 1 : 0; }
        else pcnt[i] = k ? k : (probe_outer ? 1u : 0u);
    }
    for (int d = 16; d; d >>= 1) { n_eval += __shfl_xor_sync(0xffffffffu, n_eval, d); n_pass += __shfl_xor_sync(0xffffffffu, n_pass, d); }
    if ((threadIdx.x & 31) == 0 && n_eval) { atomicAdd(pairs, n_eval); atomicAdd(pairs + 1, n_pass); }
}
// condition pass B: the passing pairs of a probe row go to its output rows in candidate order (build_outer: they mark their build
// row matched); a row the count gave an output row without a passing pair (probe_outer, anti, mark) goes out NULL-extended.
__global__ void __launch_bounds__(256) join_cond_gather_kernel(const __grid_constant__ GatherArgs g, const __grid_constant__ CondArgs a, int mode) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < g.n_probe; i += stride) {
        const unsigned long long o = g.poff[i];
        if (g.poff[i + 1] == o) continue;
        uint32_t k = 0;
        const uint32_t s = g.pslot[i];
        const uint32_t c = mode != 0 || s == J_NONE ? 0 : g.info[s].cnt;
        for (uint32_t q = 0; q < c; q++) {
            const uint32_t brow = cand_row(g.info, g.goffs, g.groups, s, c, q);
            if (!cond_pass(a, i, brow)) continue;
            const int64_t orow = (int64_t)(o + k++);
            if (g.bmatched) g.bmatched[brow] = 1;
            for (int j = 0; j < g.n_b; j++) {
                copy_cell(g.ob_data[j], orow, g.b_data[j], brow, g.b_size[j]);
                if (g.ob_valid[j]) g.ob_valid[j][orow] = g.b_valid[j] ? g.b_valid[j][brow] : 1;
            }
            for (int j = 0; j < g.n_p; j++) {
                copy_cell(g.op_data[j], orow, g.p_data[j], i, g.p_size[j]);
                if (g.op_valid[j]) g.op_valid[j][orow] = bit_valid(g.p_valid[j], i) ? 1 : 0;
            }
        }
        if (k) continue;
        for (int j = 0; j < g.n_b; j++) { zero_item(g.ob_data[j], (int64_t)o, g.b_size[j]); g.ob_valid[j][o] = 0; }
        for (int j = 0; j < g.n_p; j++) {
            copy_cell(g.op_data[j], (int64_t)o, g.p_data[j], i, g.p_size[j]);
            if (g.op_valid[j]) g.op_valid[j][o] = bit_valid(g.p_valid[j], i) ? 1 : 0;
        }
    }
}

// ---- as-of join (pandas.merge_asof; SQL ASOF JOIN ... MATCH_CONDITION) ----
// Build: every key group goes into the CSR, groups of one row included (join_slot_counts_kernel with min_rows 1), and a row with
// an NA `on` cell belongs to no group (the ASOF instantiations of the insert kernels).  radix_sort_columns sorts the build row ids
// stably by (slot, on word), so groups[goffs[s] ..] lists group s's rows by ascending `on`, ties in arrival order, and
// join_asof_groups_kernel stores the rows' words beside them (gwords): a probe's binary search reads words, not `on` cells through
// row ids.  Probe: the key lookup of the equi-join (probe_slot / probe_slot_mk), a binary search of the probe's `on` word in its
// group's words, the tolerance check, then the gather.  Words order as the values do (sort_word, -0.0 equal to 0.0), and for an
// integer or temporal column the difference of two words is the exact difference of the values as a uint64.
enum { ASOF_BACKWARD = 0, ASOF_FORWARD = 1, ASOF_NEAREST = 2 };
struct AsofArgs {
    const void* key_data; int key_ctype; const uint8_t* key_valid;  // one key column
    KeySet pk, bk;                                                   // a multi-column key
    const void* table;  // the key table: int64 keys, or the multi-column key table's (tag, row) words
    uint64_t cap; int na_equal; uint32_t key_reject;
    const SlotInfo* info; const unsigned long long* goffs; const uint32_t* groups; const uint64_t* gwords;
    AsofOn on;  // the probe's `on` column
    int direction, allow_exact, has_tol;
    unsigned long long tol_w;  // integer / temporal column: the tolerance, in word (= value) units
    double tol_f;              // float column
};
// The value of a float column's word (sort_word inverted), as float64.
__device__ __forceinline__ double asof_float(int ct, uint64_t w) {
    if (ct == CT_FLOAT64) return __longlong_as_double(canon_float_ordered((long long)(w ^ 0x8000000000000000ull)));
    const uint32_t x = (uint32_t)w;
    return (double)__uint_as_float(x >> 31 ? x ^ 0x80000000u : ~x);
}
// First position k < c with w[k] > v (strict) or w[k] >= v, else c.
__device__ __forceinline__ uint32_t asof_first_above(const uint64_t* __restrict__ w, uint32_t c, uint64_t v, bool strict) {
    uint32_t lo = 0, hi = c;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const uint64_t x = __ldg(w + mid);
        if (strict ? x > v : x >= v) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}
// The build row probe row i matches, or J_NONE.  KT: 0 one integer key column, 1 one float key column, 2 a multi-column key.
template <int KT>
__device__ __forceinline__ uint32_t asof_match(const AsofArgs& a, int64_t i) {
    uint32_t s;
    if constexpr (KT == 2) s = probe_slot_mk(a.pk, a.bk, i, (const unsigned long long*)a.table, a.cap, a.na_equal, a.key_reject);
    else s = probe_slot<KT == 1>(a.key_data, a.key_ctype, a.key_valid, i, (const long long*)a.table, a.cap, a.na_equal, (int)a.key_reject);
    const uint32_t c = s == J_NONE ? 0 : a.info[s].cnt;
    if (c == 0) return J_NONE;
    bool na;
    const uint64_t v = asof_word<false>(a.on, i, na);
    if (na) return J_NONE;
    const unsigned long long g0 = a.goffs[s];
    const uint64_t* w = a.gwords + g0;
    // backward candidate: position kb - 1, the last w <= v (w < v without exact matches); forward candidate: kf, the first w >= v
    // (w > v).  Equal words keep arrival order, so these are the last and the first of a run of ties.
    const uint32_t kb = a.direction != ASOF_FORWARD ? asof_first_above(w, c, v, a.allow_exact) : 0;
    const uint32_t kf = a.direction != ASOF_BACKWARD ? asof_first_above(w, c, v, !a.allow_exact) : c;
    const bool hb = kb > 0, hf = kf < c;
    if (!hb && !hf) return J_NONE;
    bool fwd;  // the forward candidate wins: the nearer one, the backward one on a tie (pandas: bdiff <= fdiff keeps backward)
    if (ctype_is_float(a.on.key.ct)) {
        const double x = asof_float(a.on.key.ct, v);
        const double db = hb ? x - asof_float(a.on.key.ct, __ldg(w + kb - 1)) : 0.0, df = hf ? asof_float(a.on.key.ct, __ldg(w + kf)) - x : 0.0;
        fwd = !hb || (hf && !(db <= df));
        if (a.has_tol && (fwd ? df : db) > a.tol_f) return J_NONE;
    } else {
        const uint64_t db = hb ? v - __ldg(w + kb - 1) : 0, df = hf ? __ldg(w + kf) - v : 0;
        fwd = !hb || (hf && df < db);
        if (a.has_tol && (fwd ? df : db) > a.tol_w) return J_NONE;
    }
    return a.groups[g0 + (fwd ? kf : kb - 1)];
}
// Output row o from probe row i and build row brow, or NULL build cells when brow is J_NONE.
__device__ __forceinline__ void asof_emit(const GatherArgs& g, int64_t o, int64_t i, uint32_t brow) {
    for (int k = 0; k < g.n_b; k++) {
        if (brow == J_NONE) { zero_item(g.ob_data[k], o, g.b_size[k]); g.ob_valid[k][o] = 0; continue; }
        copy_cell(g.ob_data[k], o, g.b_data[k], brow, g.b_size[k]);
        if (g.ob_valid[k]) g.ob_valid[k][o] = g.b_valid[k] ? g.b_valid[k][brow] : 1;
    }
    for (int k = 0; k < g.n_p; k++) {
        copy_cell(g.op_data[k], o, g.p_data[k], i, g.p_size[k]);
        if (g.op_valid[k]) g.op_valid[k][o] = bit_valid(g.p_valid[k], i) ? 1 : 0;
    }
}
// left as-of: output row i is probe row i, in one kernel.  (256, 1): with the block size alone ptxas keeps the multi-column key
// instantiation at 32 registers and spills.
template <int KT>
__global__ void __launch_bounds__(256, 1) join_asof_left_kernel(const __grid_constant__ GatherArgs g, const __grid_constant__ AsofArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < g.n_probe; i += stride) asof_emit(g, i, i, asof_match<KT>(a, i));
}
// inner as-of: the matched build row (J_NONE: none) and a 0 / 1 output count per probe row; the scan, then join_asof_gather_kernel
template <int KT>
__global__ void __launch_bounds__(256) join_asof_match_kernel(const __grid_constant__ AsofArgs a, int64_t n, uint32_t* brow, uint32_t* cnt) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t b = asof_match<KT>(a, i);
        brow[i] = b;
        cnt[i] = b != J_NONE ? 1u : 0u;
    }
}
// g.pslot holds the matched build rows, g.poff the output offsets
__global__ void __launch_bounds__(256) join_asof_gather_kernel(const __grid_constant__ GatherArgs g) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < g.n_probe; i += stride)
        if (g.poff[i + 1] != g.poff[i]) asof_emit(g, (int64_t)g.poff[i], i, g.pslot[i]);
}
// groups[p] = the p-th build row of the sorted order (ids: the permutation, nullptr = identity), gwords[p] its `on` word
__global__ void join_asof_groups_kernel(const uint32_t* ids, int64_t n, const AsofOn on, uint32_t* groups, uint64_t* gwords) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += stride) {
        const uint32_t r = ids ? ids[p] & 0x7FFFFFFFu : (uint32_t)p;
        bool na;
        groups[p] = r;
        gwords[p] = asof_word<true>(on, r, na);
    }
}

// ---- nested-loop join: no equi-join key (the reference's NestedLoopJoinState, bodo/libs/streaming/_nested_loop_join.cpp) ----
// Every (probe row, build row) pair is a candidate.  Output order is fixed: probe rows in batch order, each probe row's pairs in
// build arrival order, a NULL-extended / anti / mark row in its probe row's place; a build-outer tail follows the last probe call.
// With a condition, the work is a 2-D grid of probe tiles (NLJ_TILE_P rows: one warp per probe row at a time, NLJ_ROWS_PER_WARP
// rows per warp) × build chunks (a multiple of NLJ_SUB rows).  The lanes of a warp take 32 consecutive build rows, so the
// interpreter's control flow and the probe cells are warp-uniform; the build columns the program reads are staged per NLJ_SUB-row
// sub-tile in shared memory (at most NLJ_MAX_STAGE columns, further ones read through L1).  Pass A writes the passing pairs of each
// (probe row, chunk) into a count matrix n_probe × (chunks + 1), the last entry of a row being its NULL-extended / anti / mark row;
// the Scanner turns it into output offsets and pass B writes the passing pairs at offset + running + popc(ballot & lanemask_lt).
constexpr int NLJ_WARPS = 8, NLJ_ROWS_PER_WARP = 4, NLJ_TILE_P = NLJ_WARPS * NLJ_ROWS_PER_WARP, NLJ_SUB = 256, NLJ_MAX_STAGE = 8;
constexpr int64_t NLJ_MAX_ROWS = 1ll << 31;  // output rows of one probe call
struct NljArgs {
    int64_t n_probe, n_build;
    int64_t chunk;             // build rows per chunk (a multiple of NLJ_SUB); gridDim.y chunks
    int n_stage;               // build columns staged in shared memory
    int stage_col[NLJ_MAX_STAGE];
    int8_t b_slot[J_MAX_COLS];  // build column -> its stage slot, -1: read from global memory
};
// Stages the NLJ_SUB build rows from s0 (up to `end`) of the staged columns: their expr_load bits, then their validity bytes.
__device__ __forceinline__ void nlj_stage(const CondArgs& a, const NljArgs& na, int64_t s0, int64_t end, long long* sbits, uint8_t* svalid) {
    const int64_t b = s0 + threadIdx.x;
    if (b < end)
        for (int s = 0; s < na.n_stage; s++) {
            const int c = na.stage_col[s];
            const ExprVal v = expr_load(a.b_data[c], a.b_ct[c], b, !a.b_valid[c] || a.b_valid[c][b]);
            sbits[s * NLJ_SUB + threadIdx.x] = v.bits;
            svalid[s * NLJ_SUB + threadIdx.x] = v.valid ? 1 : 0;
        }
}
// The condition on probe row p and build row b, the j-th row of the staged sub-tile.
__device__ __forceinline__ bool nlj_pass(const CondArgs& a, const NljArgs& na, const long long* sbits, const uint8_t* svalid, int j, int64_t p, int64_t b) {
    const ExprVal v = expr_run(a.prog, 0, [&](int64_t arg) {
        const int c = (int)arg;
        if (c < J_MAX_COLS) {
            const int s = na.b_slot[c];
            if (s >= 0) return ExprVal{sbits[s * NLJ_SUB + j], ctype_is_float(a.b_ct[c]), svalid[s * NLJ_SUB + j] != 0, a.b_ct[c] == CT_UINT64};
            return expr_load(a.b_data[c], a.b_ct[c], b, !a.b_valid[c] || a.b_valid[c][b]);
        }
        const int q = c - J_MAX_COLS;
        return expr_load(a.p_data[q], a.p_ct[q], p, bit_valid(a.p_valid[q], p));
    });
    return v.valid && ev_true(v);
}
// condition pass A: cnt[p * (gridDim.y + 1) + chunk] = the passing pairs of probe row p in build chunk blockIdx.y.  pairs[0] += pairs
// evaluated, pairs[1] += pairs passed (one atomic per warp).  Every pair is evaluated, for anti and mark joins too.
__global__ void __launch_bounds__(NLJ_WARPS * 32) nlj_count_kernel(const __grid_constant__ CondArgs a, const __grid_constant__ NljArgs na, uint32_t* cnt,
                                                                   unsigned long long* pairs) {
    extern __shared__ long long nlj_smem[];
    long long* sbits = nlj_smem;
    uint8_t* svalid = (uint8_t*)(nlj_smem + na.n_stage * NLJ_SUB);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t b0 = (int64_t)blockIdx.y * na.chunk, end = min(b0 + na.chunk, na.n_build);
    const int64_t p0 = (int64_t)blockIdx.x * NLJ_TILE_P + warp * NLJ_ROWS_PER_WARP;
    uint32_t k[NLJ_ROWS_PER_WARP] = {};
    unsigned long long n_eval = 0;
    for (int64_t s0 = b0; s0 < end; s0 += NLJ_SUB) {
        __syncthreads();
        nlj_stage(a, na, s0, end, sbits, svalid);
        __syncthreads();
#pragma unroll
        for (int r = 0; r < NLJ_ROWS_PER_WARP; r++) {
            const int64_t p = p0 + r;
            if (p >= na.n_probe) break;
            for (int j = lane; j < NLJ_SUB && s0 + j - lane < end; j += 32) {
                const int64_t b = s0 + j;
                const bool in = b < end;
                k[r] += __popc(__ballot_sync(0xffffffffu, in && nlj_pass(a, na, sbits, svalid, j, p, b)));
                n_eval += in ? 1 : 0;
            }
        }
    }
    unsigned long long n_pass = 0;
#pragma unroll
    for (int r = 0; r < NLJ_ROWS_PER_WARP; r++) {
        const int64_t p = p0 + r;
        if (p < na.n_probe && lane == 0) cnt[p * (gridDim.y + 1) + blockIdx.y] = k[r];
        n_pass += k[r];
    }
    for (int d = 16; d; d >>= 1) n_eval += __shfl_xor_sync(0xffffffffu, n_eval, d);
    if (lane == 0 && n_eval) { atomicAdd(pairs, n_eval); atomicAdd(pairs + 1, n_pass); }
}
// After pass A, per probe row: the entry after its chunk counts, by kind.  mode 0: 1 for a probe_outer row without a passing pair;
// 1 (anti): 1 without a passing pair, and the chunk counts zeroed; 2 (mark): 1, mark[p] = some pair passes, chunk counts zeroed.
__global__ void nlj_rows_kernel(int64_t n, int n_chunks, uint32_t* cnt, int probe_outer, int mode, uint8_t* mark) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += stride) {
        uint32_t* row = cnt + p * (n_chunks + 1);
        bool any = false;
        for (int c = 0; c < n_chunks; c++) any = any || row[c] != 0;
        if (mode != 0)
            for (int c = 0; c < n_chunks; c++) row[c] = 0;
        row[n_chunks] = mode == 2 ? 1u : (!any && (mode == 1 || probe_outer)) ? 1u : 0u;
        if (mode == 2) mark[p] = any ? 1 : 0;
    }
}
// condition pass B: the passing pairs of (probe row, chunk) go to their output rows in build order (build_outer: they mark their
// build row matched).  A block none of whose rows has output in its chunk skips it; so does a warp for each row without output.
__global__ void __launch_bounds__(NLJ_WARPS * 32) nlj_gather_kernel(const __grid_constant__ GatherArgs g, const __grid_constant__ CondArgs a,
                                                                    const __grid_constant__ NljArgs na) {
    extern __shared__ long long nlj_smem[];
    long long* sbits = nlj_smem;
    uint8_t* svalid = (uint8_t*)(nlj_smem + na.n_stage * NLJ_SUB);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t b0 = (int64_t)blockIdx.y * na.chunk, end = min(b0 + na.chunk, na.n_build);
    const int64_t p0 = (int64_t)blockIdx.x * NLJ_TILE_P + warp * NLJ_ROWS_PER_WARP;
    unsigned long long o[NLJ_ROWS_PER_WARP];
    bool need[NLJ_ROWS_PER_WARP], any = false;
#pragma unroll
    for (int r = 0; r < NLJ_ROWS_PER_WARP; r++) {
        const int64_t p = p0 + r, e = p * (gridDim.y + 1) + blockIdx.y;
        need[r] = p < na.n_probe && g.poff[e + 1] != g.poff[e];
        o[r] = need[r] ? g.poff[e] : 0;
        any = any || need[r];
    }
    if (!__syncthreads_or(any)) return;
    const unsigned lt = (1u << lane) - 1;
    for (int64_t s0 = b0; s0 < end; s0 += NLJ_SUB) {
        __syncthreads();
        nlj_stage(a, na, s0, end, sbits, svalid);
        __syncthreads();
#pragma unroll
        for (int r = 0; r < NLJ_ROWS_PER_WARP; r++) {
            if (!need[r]) continue;
            const int64_t p = p0 + r;
            for (int j = lane; j < NLJ_SUB && s0 + j - lane < end; j += 32) {
                const int64_t b = s0 + j;
                const bool ok = b < end && nlj_pass(a, na, sbits, svalid, j, p, b);
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                if (ok) {
                    const int64_t orow = (int64_t)(o[r] + __popc(m & lt));
                    if (g.bmatched) g.bmatched[b] = 1;
                    for (int q = 0; q < g.n_b; q++) {
                        copy_cell(g.ob_data[q], orow, g.b_data[q], b, g.b_size[q]);
                        if (g.ob_valid[q]) g.ob_valid[q][orow] = g.b_valid[q] ? g.b_valid[q][b] : 1;
                    }
                    for (int q = 0; q < g.n_p; q++) {
                        copy_cell(g.op_data[q], orow, g.p_data[q], p, g.p_size[q]);
                        if (g.op_valid[q]) g.op_valid[q][orow] = bit_valid(g.p_valid[q], p) ? 1 : 0;
                    }
                }
                o[r] += __popc(m);
            }
        }
    }
}
// The one-row entries: probe row p goes out NULL-extended (or as an anti / mark row, whose build columns are NULL or absent) at
// g.poff[p * (n_chunks + 1) + n_chunks] when that entry is 1; without offsets (g.poff nullptr) every probe row goes out at row p.
__global__ void nlj_probe_rows_kernel(const __grid_constant__ GatherArgs g, int n_chunks) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < g.n_probe; p += stride) {
        if (!g.poff) { asof_emit(g, p, p, J_NONE); continue; }
        const int64_t e = p * (n_chunks + 1) + n_chunks;
        if (g.poff[e + 1] != g.poff[e]) asof_emit(g, (int64_t)g.poff[e], p, J_NONE);
    }
}
// Cross join (no condition): output row o = (probe row o / n_build, build row o % n_build), o < rows <= NLJ_MAX_ROWS, so the
// index arithmetic is 32-bit.  Consecutive threads write consecutive output rows and read consecutive build rows; the probe cell
// of a run of n_build rows is one broadcast load.
__global__ void __launch_bounds__(256) nlj_cross_kernel(const __grid_constant__ GatherArgs g, uint32_t n_build, uint32_t rows) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < rows; o += stride) {
        const uint32_t p = o / n_build, b = o - p * n_build;
        for (int q = 0; q < g.n_b; q++) {
            copy_cell(g.ob_data[q], o, g.b_data[q], b, g.b_size[q]);
            if (g.ob_valid[q]) g.ob_valid[q][o] = g.b_valid[q] ? g.b_valid[q][b] : 1;
        }
        for (int q = 0; q < g.n_p; q++) {
            copy_cell(g.op_data[q], o, g.p_data[q], p, g.p_size[q]);
            if (g.op_valid[q]) g.op_valid[q][o] = bit_valid(g.p_valid[q], p) ? 1 : 0;
        }
    }
}

// ================================================================================================
// When `buf` holds fewer than `need` bytes, replaces it by a buffer of max(need, alloc) bytes that keeps its first `keep` bytes.
static void grow_keep(DevBuf& buf, size_t need, size_t keep, cudaStream_t st, size_t alloc = 0) {
    if (need <= buf.bytes) return;
    DevBuf nb;
    nb.alloc(std::max(need, alloc));
    if (keep) {
        B200_CUDA(cudaMemcpyAsync(nb.p, buf.p, keep, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaStreamSynchronize(st));
    }
    buf = std::move(nb);
}

struct GrowCol {  // growable device column (geometric growth, copy on grow)
    DevBuf buf;
    size_t used = 0;
    void append(const void* src, size_t nbytes, cudaStream_t st) {
        grow_keep(buf, used + nbytes, used, st, std::max<size_t>((used + nbytes) * 2, 1 << 16));
        if (nbytes) B200_CUDA(cudaMemcpyAsync((char*)buf.p + used, src, nbytes, cudaMemcpyDeviceToDevice, st));
        used += nbytes;
    }
    void reserve(size_t n) { if (n > buf.bytes) { B200_REQUIRE(used == 0, "internal: reserve after append"); buf.alloc(n); } }
};

// f(std::integral_constant<int, v>) for the one v in [0, N) equal to `v`: the kernel instantiation a runtime argument selects
template <typename F, int... I> void with_int_seq(int v, F&& f, std::integer_sequence<int, I...>) {
    ((v == I ? f(std::integral_constant<int, I>{}) : void()), ...);
}
template <int N, typename F> void with_int(int v, F&& f) {
    B200_REQUIRE(v >= 0 && v < N, "internal: no kernel instantiation for this argument");
    with_int_seq(v, f, std::make_integer_sequence<int, N>{});
}

class JoinState {
   public:
    int device; cudaStream_t stream; int sms;
    std::vector<int8_t> b_ct, b_at, p_ct, p_at;
    int n_b, n_p;
    bool build_outer, probe_outer;
    bool na_equal = false;  // is_na_equal of the reference's HashJoinState
    int n_keys = 1;         // key columns: the first n_keys of each side; more than one always takes the CSR form (the _mk kernels)
    bool float_key = false; // float64 or float32 key column (n_keys == 1): every FK-templated key kernel runs its FK instantiation
    uint32_t key_reject = 0;  // bit j: probe key position j differs from the build key in signedness at 8 bytes (signedness_differs)
    int64_t output_batch_size;
    // build side
    std::vector<GrowCol> bcol, bvalid;  // data; validity as one byte per row (empty when the column has none so far)
    std::vector<bool> b_has_valid;
    int64_t n_build = 0;
    bool build_final = false;
    uint64_t cap = 0;
    // the table the probe reads, chosen by finalize_build: the CSR key table of the general path; for unique build keys of an
    // inner join, Slot16 (+ packed payload) built from the key table, or Slot32 (inline payload) with Slot16 derived on demand
    enum class TableForm { CSR, SLOT16, SLOT32 } form = TableForm::CSR;
    DevBuf d_tkeys, d_info, d_row_slot, d_cnt_multi, d_goffs, d_groups, d_fill, d_bmatched;
    DevBuf d_slots16, d_bpack, d_cursor;  // fast path (unique build keys, inner join)
    DevBuf d_slots32;                      // inline-payload table (all-8-byte bitmap-free build schema, <= 2 payload columns)
    int64_t inline_probes = 0, inline_builds = 0;
    // join kind (set_kind, before the first build batch): mark join / probe-side anti join (reference: is_mark_join member,
    // is_anti_join template argument of the probe)
    bool mark = false, anti = false;
    DevBuf d_mark, d_mark_valid;
    // non-equi condition (set_condition, before the first build batch): one expression over build column c (arg c) and probe
    // column c (arg J_MAX_COLS + c); empty = none.  d_cond_pairs: candidate pairs evaluated, pairs passed (metrics 8, 9)
    std::vector<ExprInstr> cond;
    // as-of join (set_asof, before the first build batch): the `on` column of each side, direction, exact matches, tolerance.  The
    // build keeps every key group in the CSR, sorted by `on`; d_gwords holds the `on` words of the groups' rows.
    bool asof = false;
    int asof_b_on = -1, asof_p_on = -1, asof_dir = 0;
    bool asof_exact = true, asof_has_tol = false;
    long long asof_tol_i = 0;
    double asof_tol_f = 0;
    DevBuf d_gwords;
    DevBuf d_cond_pairs;
    unsigned long long* h_cond_pairs = nullptr;
    int64_t cond_evaluated = 0, cond_passed = 0;
    // runtime join filter, built on demand from the build keys
    DevBuf d_bloom, d_minmax;
    uint64_t bloom_blocks = 0;
    long long key_bounds[2 * MAX_HASH_KEYS];  // min, max of key column 0, then of column 1, ...
    int64_t filter_rows_in = 0, filter_rows_kept = 0;
    void* h_word = nullptr;  // pinned mirror of read_word
    int64_t fast_probes = 0;
    Scanner scan;
    // probe scratch + output
    DevBuf d_pslot, d_pcnt, d_poff, d_stage_valid;
    std::vector<DevBuf> stage_data, stage_valid;   // device copies of host probe batches
    std::vector<DevBuf> out_data, out_vbytes, out_bitmap;
    int64_t launches = 0, probe_rows = 0, out_rows_total = 0;
    bool tail_emitted = false;

    JoinState(const int8_t* bct, const int8_t* bat, int nb, const int8_t* pct, const int8_t* pat, int np, uint64_t nk,
              bool bo, bool po, bool na_eq, int64_t obs, int dev, int64_t expected_build_rows, cudaStream_t st)
        : device(dev), stream(st), n_b(nb), n_p(0), build_outer(bo), probe_outer(po), na_equal(na_eq), output_batch_size(obs) {
        B200_REQUIRE(nk <= MAX_HASH_KEYS, "b200 join: between 0 (a nested-loop join) and 4 key columns (n_keys) per side");
        n_keys = (int)nk;
        for (int j = 0; j < 2 * MAX_HASH_KEYS; j++) key_bounds[j] = j % 2 ? INT64_MIN : INT64_MAX;
        B200_REQUIRE(nb >= 1 && np >= 0 && nb <= J_MAX_COLS && np <= J_MAX_COLS, "b200 join: between 1 and 32 columns per side");
        B200_REQUIRE(nb >= n_keys && (np == 0 || np >= n_keys), "b200 join: fewer columns than key columns");
        b_ct.assign(bct, bct + nb); b_at.assign(bat, bat + nb);
        for (int c = 0; c < nb; c++) B200_REQUIRE(ctype_size(b_ct[c]) > 0, "b200 join: unsupported build column dtype");
        float_key = n_keys == 1 && ctype_is_float(b_ct[0]);
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        sms = num_sms(device);
        bcol.resize(nb); bvalid.resize(nb); b_has_valid.assign(nb, false);
        if (expected_build_rows > 0)
            for (int c = 0; c < nb; c++) bcol[c].reserve((size_t)expected_build_rows * ctype_size(b_ct[c]));
        stage_data.resize(nb); stage_valid.resize(nb);
        if (np > 0) set_probe_schema(pct, pat, np);
    }
    // The probe schema may be given at init (n_probe_arrs > 0) or adopted from the first probe batch (n_probe_arrs == 0), so
    // a host layer that only learns it from the data can feed build batches straight away.
    void set_probe_schema(const int8_t* pct, const int8_t* pat, int np) {
        B200_REQUIRE(np >= 1 && np <= J_MAX_COLS, "b200 join: between 1 and 32 columns per side");
        p_ct.assign(pct, pct + np); p_at.assign(pat, pat + np); n_p = np;
        for (int c = 0; c < np; c++) B200_REQUIRE(ctype_size(p_ct[c]) > 0, "b200 join: unsupported probe column dtype");
        B200_REQUIRE(np >= n_keys, "b200 join: fewer columns than key columns");
        for (int j = 0; j < n_keys; j++) require_key_type(j, p_ct[j], "probe");
        if (n_keys > 0) B200_REQUIRE(ctype_size(b_ct[0]) == ctype_size(p_ct[0]), "b200 join: build and probe key widths differ");
        key_reject = 0;
        for (int j = 0; j < n_keys; j++) key_reject |= signedness_differs(p_ct[j], b_ct[j]) ? 1u << j : 0u;
        if (asof) check_asof_probe();
        for (const ExprInstr& in : cond)
            B200_REQUIRE(in.op != EX_COL || in.arg < J_MAX_COLS || in.arg - J_MAX_COLS < np,
                         "b200 join: the condition reads probe column " + std::to_string(in.arg - J_MAX_COLS) + " and the probe table has " +
                             std::to_string(np) + " columns");
        out_data.resize(n_b + np); out_vbytes.resize(n_b + np); out_bitmap.resize(n_b + np);
        if ((int)stage_data.size() < std::max(n_b, np)) { stage_data.resize(std::max(n_b, np)); stage_valid.resize(std::max(n_b, np)); }
    }
    ~JoinState() { cudaSetDevice(device); scratch_set_stream(stream); cudaStreamSynchronize(stream); pinned_release(h_word, 8); pinned_release(h_cond_pairs, 16); }

    // Key position j: a float key joins a float key of the same type only; integer keys join integer keys of the same width (for
    // one key column the callers check the width with their own message)
    void require_key_type(int j, int ct, const char* what) const {
        const std::string pos = n_keys > 1 ? "key position " + std::to_string(j) + ": " : "";
        const std::string types = std::string("the ") + what + " key column is " + ctype_name(ct) + " and the build key column is " + ctype_name(b_ct[j]);
        if (ctype_is_float(b_ct[j]) || ctype_is_float(ct))
            B200_REQUIRE(ct == b_ct[j], "b200 join: " + pos + types + "; float keys join float keys of the same type");
        if (n_keys > 1) B200_REQUIRE(ctype_size(ct) == ctype_size(b_ct[j]), "b200 join: " + pos + types + "; integer keys join integer keys of the same width");
    }
    // Integer keys join by value, as pandas merge does.  Up to 4 bytes the key load sign- or zero-extends each side to int64, which
    // is the value.  At 8 bytes an int64 / DATETIME / TIMEDELTA key and a UINT64 key are the same value exactly when their bits are
    // equal and the top bit is clear, so the probe side rejects a key with that bit set (key_reject) and any build key with it is
    // then unreachable.
    static bool signedness_differs(int probe_ct, int build_ct) {
        return ctype_size(probe_ct) == 8 && !ctype_is_float(probe_ct) && !ctype_is_float(build_ct) && (probe_ct == CT_UINT64) != (build_ct == CT_UINT64);
    }
    KeySet build_keys() const {
        KeySet k{};
        k.n_keys = n_keys;
        for (int j = 0; j < n_keys; j++) { k.data[j] = bcol[j].buf.p; k.valid[j] = build_valid(j); k.ctype[j] = b_ct[j]; }
        return k;
    }
    KeySet probe_keys(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid) const {
        KeySet k{};
        k.n_keys = n_keys;
        for (int j = 0; j < n_keys; j++) { k.data[j] = data[j]; k.valid[j] = valid[j]; k.ctype[j] = p_ct[j]; }
        return k;
    }
    // f(std::bool_constant<FK>): the instantiation of a key kernel for this join's key type
    template <typename F> void with_key(F&& f) const {
        if (float_key) f(std::true_type{});
        else f(std::false_type{});
    }

    int grid_for(int64_t n) const { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sms * 8)); }
    const uint8_t* build_valid(int c) const { return b_has_valid[c] ? bvalid[c].buf.as<uint8_t>() : nullptr; }
    // the device word at `dev` (synchronises the stream)
    template <typename T> T read_word(const T* dev) {
        static_assert(sizeof(T) <= 8, "one pinned 8-byte mirror");
        if (!h_word) h_word = pinned_acquire(8);
        B200_CUDA(cudaMemcpyAsync(h_word, dev, sizeof(T), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        return *(const T*)h_word;
    }

    void set_kind(bool is_mark, bool is_anti) {
        B200_REQUIRE(n_build == 0 && !build_final, "b200 join: the join kind must be set before the first build batch");
        B200_REQUIRE(!(is_mark && is_anti), "b200 join: a join is a mark join or an anti join, not both");
        B200_REQUIRE(!(is_mark || is_anti) || !build_outer, "b200 join: mark / anti joins do not emit build rows (build_table_outer must be false)");
        B200_REQUIRE(!(is_mark || is_anti) || !asof, "b200 join: an as-of join is not a mark or anti join");
        mark = is_mark; anti = is_anti;
    }
    // The non-equi condition: one expression (ending in EX_END) over the columns of both sides.  Build columns are checked here,
    // probe columns here when the probe schema is known and otherwise when the first probe batch brings it.
    void set_condition(const ExprInstr* prog, int n_instr) {
        B200_REQUIRE(n_build == 0 && !build_final, "b200 join: the condition must be set before the first build batch");
        B200_REQUIRE(!asof, "b200 join: an as-of join takes no non-equi condition");
        const std::string who = "b200 join: set_condition";
        expr_validate(prog, n_instr, [&](int64_t c) {
            return (c >= 0 && c < n_b) || (c >= J_MAX_COLS && c < 2 * J_MAX_COLS && (n_p == 0 || c - J_MAX_COLS < n_p));
        }, who);
        for (int i = 0; i + 1 < n_instr; i++) B200_REQUIRE(prog[i].op != EX_END, who + ": the condition is one expression (one END, at the end)");
        cond.assign(prog, prog + n_instr);
    }
    // The as-of join (pandas.merge_asof): each probe row matches at most the one build row of its key group whose `on` value is the
    // latest at or before its own (backward), the earliest at or after it (forward) or the nearer of those two (nearest).
    void set_asof(int b_on, int p_on, int dir, bool exact, bool has_tol, long long tol_i, double tol_f) {
        const std::string who = "b200 join: set_asof: ";
        B200_REQUIRE(n_build == 0 && !build_final, who + "the as-of join must be set before the first build batch");
        B200_REQUIRE(n_keys > 0, who + "a nested-loop join (n_keys 0) has no as-of form; give one constant key column per side");
        B200_REQUIRE(!build_outer, who + "a build-outer as-of join is not supported");
        B200_REQUIRE(!mark && !anti && cond.empty(), who + "an as-of join is not a mark, anti or condition join");
        B200_REQUIRE(dir >= ASOF_BACKWARD && dir <= ASOF_NEAREST, who + "direction is 0 (backward), 1 (forward) or 2 (nearest)");
        B200_REQUIRE(b_on >= n_keys && b_on < n_b, who + "the build `on` column must be a non-key column of the build table (got " + std::to_string(b_on) +
                                                       "; the key columns are 0.." + std::to_string(n_keys - 1) + " of " + std::to_string(n_b) + ")");
        B200_REQUIRE(p_on >= n_keys && p_on < J_MAX_COLS, who + "the probe `on` column must be a non-key column of the probe table (got " + std::to_string(p_on) + ")");
        const int ct = b_ct[b_on];
        B200_REQUIRE(ct != CT_BOOL, who + "the `on` column is " + ctype_name(ct) + "; it must be an integer, float, date, datetime or timedelta column");
        if (has_tol && ctype_is_float(ct)) B200_REQUIRE(std::isfinite(tol_f) && tol_f >= 0, who + "the tolerance must be finite and >= 0");
        if (has_tol && !ctype_is_float(ct)) B200_REQUIRE(tol_i >= 0, who + "the tolerance must be >= 0");
        asof_b_on = b_on; asof_p_on = p_on; asof_dir = dir; asof_exact = exact; asof_has_tol = has_tol; asof_tol_i = tol_i; asof_tol_f = tol_f;
        if (n_p) check_asof_probe();  // the probe schema is known: check it now, else when the first probe batch brings it
        asof = true;
    }
    void check_asof_probe() const {
        B200_REQUIRE(asof_p_on < n_p, "b200 join: set_asof: the probe `on` column " + std::to_string(asof_p_on) + " is out of range (the probe table has " +
                                          std::to_string(n_p) + " columns)");
        B200_REQUIRE(p_ct[asof_p_on] == b_ct[asof_b_on], std::string("b200 join: set_asof: the probe `on` column is ") + ctype_name(p_ct[asof_p_on]) +
                                                              " and the build `on` column " + ctype_name(b_ct[asof_b_on]) + "; both sides need the same type");
    }
    SortKey asof_key() const { return SortKey{b_ct[asof_b_on], ctype_size(b_ct[asof_b_on]), 0, 1}; }
    AsofOn asof_build_on() const { return AsofOn{bcol[asof_b_on].buf.p, build_valid(asof_b_on), asof_key()}; }
    // groups (the CSR of every key group, `total` rows) sorted by `on`, and their words
    void build_asof_groups(unsigned long long total) {
        d_gwords.alloc((size_t)std::max<unsigned long long>(total, 1) * 8);
        if (total == 0) return;
        const void* cols[2] = {d_row_slot.p, bcol[asof_b_on].buf.p};
        const SortKey keys[2] = {SortKey{CT_UINT32, 4, 0, 1}, asof_key()};
        DevBuf ids[2];
        const uint32_t* perm = radix_sort_columns(2, cols, keys, n_build, ids, stream);
        join_asof_groups_kernel<<<grid_for((int64_t)total), 256, 0, stream>>>(perm, (int64_t)total, asof_build_on(), d_groups.as<uint32_t>(),
                                                                              d_gwords.as<uint64_t>());
        launches++;
        B200_CUDA(cudaGetLastError());
    }

    // ---- runtime join filter ----
    // n_blocks: 32-byte bloom blocks (0 = one per 32 build rows, ~8 bits per key); ranks that will OR their filters together
    // pass the same value.  Also computes the min / max of the (non-NA) build keys, per key column.
    void build_filter(uint64_t n_blocks) {
        B200_REQUIRE(build_final, "b200 join: runtime filter before the build side was finished");
        B200_REQUIRE(n_keys > 0, "b200 join: a nested-loop join (n_keys 0) has no key to build a runtime filter from");
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        bloom_blocks = n_blocks ? n_blocks : (uint64_t)n_build / 32 + 1;
        d_bloom.alloc(bloom_blocks * 32);
        B200_CUDA(cudaMemsetAsync(d_bloom.p, 0, bloom_blocks * 32, stream));
        const size_t mm_bytes = 16 * (size_t)n_keys;
        d_minmax.alloc(mm_bytes);
        long long h[2 * MAX_HASH_KEYS];
        for (int j = 0; j < 2 * n_keys; j++) h[j] = j % 2 ? INT64_MIN : INT64_MAX;
        B200_CUDA(cudaMemcpyAsync(d_minmax.p, h, mm_bytes, cudaMemcpyHostToDevice, stream));
        if (n_build > 0) {
            join_bloom_add_kernel<<<grid_for(n_build), 256, 0, stream>>>(build_keys(), n_build, na_equal ? 1 : 0, d_bloom.as<uint32_t>(), bloom_blocks,
                                                                         d_minmax.as<long long>());
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        B200_CUDA(cudaMemcpyAsync(h, d_minmax.p, mm_bytes, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        std::copy(h, h + 2 * n_keys, key_bounds);
    }
    // key_cols[j] < 0: key column j is absent from `t`; the bounds then apply to the present columns and the bloom filter only when
    // every column is present.  With no key column present every row is kept.
    void runtime_filter(const b200_table* t, const int32_t* key_cols, int nk, const int32_t* use_minmax, bool use_bloom, uint8_t* keep) {
        B200_REQUIRE(n_keys > 0, "b200 join: runtime_filter_n: a nested-loop join (n_keys 0) has no key to filter probe rows by");
        B200_REQUIRE(nk == n_keys, "b200 join: runtime_filter_n: n_keys is " + std::to_string(nk) + " and this join has " + std::to_string(n_keys) + " key columns");
        B200_REQUIRE(t->device == device, "b200 join: runtime_filter takes a device-resident table on the state's device");
        KeySet pk{};
        pk.n_keys = n_keys;
        uint32_t mm = 0, reject = 0;
        bool all = true, any = false;
        for (int j = 0; j < n_keys; j++) {
            const int c = key_cols[j];
            if (c < 0) { all = false; continue; }
            any = true;
            B200_REQUIRE(c < t->n_cols, "b200 join: runtime_filter: bad key column");
            require_key_type(j, t->cols[c].c_type, "runtime_filter");
            B200_REQUIRE(ctype_size(t->cols[c].c_type) == ctype_size(b_ct[j]), "b200 join: runtime_filter: key column type differs from the build key");
            pk.data[j] = t->cols[c].data; pk.valid[j] = t->cols[c].validity; pk.ctype[j] = t->cols[c].c_type;
            if (use_minmax[j]) mm |= 1u << j;
            if (signedness_differs(pk.ctype[j], b_ct[j])) reject |= 1u << j;
        }
        B200_CUDA(cudaSetDevice(device));
        const int64_t n = t->n_rows;
        if (!any) {
            if (n) B200_CUDA(cudaMemsetAsync(keep, 1, (size_t)n, stream));
            return;
        }
        if (!d_bloom.p) build_filter(0);
        if (n == 0) return;
        MKBounds b;
        std::copy(key_bounds, key_bounds + 2 * MAX_HASH_KEYS, b.v);
        join_runtime_filter_kernel<<<grid_for(n), 256, 0, stream>>>(pk, n, na_equal ? 1 : 0, d_bloom.as<uint32_t>(), bloom_blocks, b, mm,
                                                                    use_bloom && all ? 1 : 0, keep, reject);
        launches++;
        B200_CUDA(cudaGetLastError());
        filter_rows_in += n;
    }

    // device pointers for a batch (host batches are staged to the device first)
    void stage_batch(const b200_table* t, int ncols, const std::vector<int8_t>& cts, std::vector<const void*>& data,
                     std::vector<const uint8_t*>& valid) {
        data.assign(ncols, nullptr); valid.assign(ncols, nullptr);
        int64_t n = t->n_rows;
        for (int c = 0; c < ncols; c++) {
            B200_REQUIRE(t->cols[c].c_type == cts[c], "b200 join: batch column dtype differs from the schema");
            if (t->device >= 0) {
                B200_REQUIRE(t->device == device, "b200 join: batch lives on another device");
                data[c] = t->cols[c].data; valid[c] = t->cols[c].validity;
            } else {
                size_t nbytes = (size_t)n * ctype_size(cts[c]);
                stage_data[c].ensure(nbytes + 8);
                if (nbytes) B200_CUDA(cudaMemcpyAsync(stage_data[c].p, t->cols[c].data, nbytes, cudaMemcpyHostToDevice, stream));
                data[c] = stage_data[c].p;
                if (t->cols[c].validity) {
                    stage_valid[c].ensure((size_t)(n + 7) / 8 + 8);
                    B200_CUDA(cudaMemcpyAsync(stage_valid[c].p, t->cols[c].validity, (size_t)(n + 7) / 8, cudaMemcpyHostToDevice, stream));
                    valid[c] = stage_valid[c].as<uint8_t>();
                }
            }
        }
    }

    void build_consume(const b200_table* t, bool is_last) {
        B200_REQUIRE(!build_final, "b200 join: build batch after the build was finalized");
        B200_REQUIRE(t->n_cols == n_b, "b200 join: build batch has a different number of columns than the schema");
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        int64_t n = t->n_rows;
        // slot ids and build row ids are 32-bit; cap = next power of two >= 2 * n_build, and cap + 2 must stay below 2^32
        B200_REQUIRE(n_build + n <= (1ll << 30), "b200 join: build side is limited to 2^30 rows per GPU");
        if (n > 0) {
            std::vector<const void*> data; std::vector<const uint8_t*> valid;
            stage_batch(t, n_b, b_ct, data, valid);
            for (int c = 0; c < n_b; c++) {
                bcol[c].append(data[c], (size_t)n * ctype_size(b_ct[c]), stream);
                bool has = valid[c] != nullptr;
                if (has && !b_has_valid[c]) {  // first batch with a bitmap: earlier rows were all valid
                    b_has_valid[c] = true;
                    if (n_build) { DevBuf ones; ones.alloc((size_t)n_build); B200_CUDA(cudaMemsetAsync(ones.p, 1, (size_t)n_build, stream)); bvalid[c].append(ones.p, (size_t)n_build, stream); B200_CUDA(cudaStreamSynchronize(stream)); }
                }
                if (b_has_valid[c]) {
                    d_stage_valid.ensure((size_t)n);
                    if (has) { expand_bitmap_kernel<<<grid_for(n), 256, 0, stream>>>(valid[c], n, d_stage_valid.as<uint8_t>()); launches++; }
                    else B200_CUDA(cudaMemsetAsync(d_stage_valid.p, 1, (size_t)n, stream));
                    bvalid[c].append(d_stage_valid.p, (size_t)n, stream);
                }
            }
            B200_CUDA(cudaStreamSynchronize(stream));  // staging buffers are reused by the next batch
            n_build += n;
        }
        if (is_last) finalize_build();
    }

    // Inline-payload build attempt (unique keys expected): true when the Slot32 table is complete, false when a key repeats
    // (or the schema does not qualify) and the general build has to run.
    bool try_inline_build(uint64_t n_slots) {
        const int nf = n_b - 1;
        bool ok = n_build > 0 && nf <= 2 && !build_outer && !probe_outer && !(getenv("B200_JOIN_INLINE") && getenv("B200_JOIN_INLINE")[0] == '0');
        for (int c = 0; c < n_b; c++) ok = ok && ctype_size(b_ct[c]) == 8 && !b_has_valid[c];
        if (!ok) return false;
        d_slots32.alloc(n_slots * sizeof(Slot32));
        DevBuf dup;  // raised by the second row of any key
        dup.alloc(4);
        B200_CUDA(cudaMemsetAsync(dup.p, 0, 4, stream));
        join_fill_slots32_kernel<<<grid_for((int64_t)n_slots), 256, 0, stream>>>(d_slots32.as<Slot32>(), n_slots);
        with_key([&](auto fk) {
            join_build_inline_kernel<fk><<<(int)std::max<int64_t>(1, std::min<int64_t>((n_build + 1023) / 1024, (int64_t)sms * 8)), 256, 0, stream>>>(
                bcol[0].buf.as<long long>(), nf > 0 ? bcol[1].buf.as<unsigned long long>() : nullptr, nf > 1 ? bcol[2].buf.as<unsigned long long>() : nullptr,
                n_build, 0, d_slots32.as<Slot32>(), cap, dup.as<int>(), na_equal ? 1 : 0);
        });
        launches += 2;
        B200_CUDA(cudaGetLastError());
        if (read_word(dup.as<int>()) != 0) { d_slots32.release(); return false; }  // duplicate build keys
        return true;
    }
    // Slot16 table + packed payload of the two-sector fast kernel: from the key table when finalize_build finds unique keys, or
    // on demand from the Slot32 table when a probe batch does not qualify for the inline kernel (bitmaps, narrow columns)
    void setup_slot16() {
        const uint64_t n_slots = cap + 2;
        d_slots16.alloc(n_slots * sizeof(Slot16));
        if (form == TableForm::SLOT32)
            join_slots16_from32_kernel<<<grid_for((int64_t)n_slots), 256, 0, stream>>>(d_slots32.as<Slot32>(), n_slots, d_slots16.as<Slot16>());
        else
            join_make_slots16_kernel<<<grid_for((int64_t)n_slots), 256, 0, stream>>>(d_tkeys.as<long long>(), d_info.as<SlotInfo>(), n_slots, d_slots16.as<Slot16>());
        const int nf = n_b - 1;
        d_bpack.alloc((size_t)std::max<int64_t>(n_build * std::max(nf, 1), 1) * 8);
        if (nf > 0) {
            PackPayloadArgs pa{};
            pa.n_build = n_build; pa.n_fields = nf; pa.out = d_bpack.as<unsigned long long>();
            for (int c = 1; c < n_b; c++) { pa.src[c - 1] = bcol[c].buf.p; pa.size[c - 1] = ctype_size(b_ct[c]); }
            join_pack_payload_kernel<<<grid_for(n_build), 256, 0, stream>>>(pa);
        }
        launches += 2;
        B200_CUDA(cudaGetLastError());
    }

    void finalize_build() {
        if (n_keys == 0) {  // a nested-loop join probes the build store itself: no hash table, bloom filter or CSR
            finish_build();
            return;
        }
        cap = 1024;
        while (cap < 2ull * (uint64_t)n_build) cap <<= 1;
        uint64_t n_slots = cap + 2;
        // the unique-key tables (Slot32, Slot16) hold one int64 key: a multi-column key always takes the CSR form
        if (n_keys == 1 && !mark && !anti && cond.empty() && !asof && try_inline_build(n_slots)) {
            form = TableForm::SLOT32; inline_builds++;
            build_final = true;
            return;
        }
        d_tkeys.alloc(n_slots * 8);  // int64 keys, or the multi-column key table's (tag, row) words
        launch_fill_u64(d_tkeys.p, n_slots, n_keys > 1 ? MK_EMPTY : (unsigned long long)J_EMPTY, grid_for((int64_t)n_slots), stream);
        d_info.alloc(n_slots * sizeof(SlotInfo));
        B200_CUDA(cudaMemsetAsync(d_info.p, 0, n_slots * sizeof(SlotInfo), stream));
        d_row_slot.alloc((size_t)std::max<int64_t>(n_build, 1) * 4);
        launches++;
        if (n_build > 0) {
            const AsofOn on = asof ? asof_build_on() : AsofOn{};
            with_int<2>(asof ? 1 : 0, [&](auto as) {
                if (n_keys > 1)
                    join_insert_count_mk_kernel<decltype(as)::value == 1><<<grid_for(n_build), 256, 0, stream>>>(build_keys(), n_build, d_tkeys.as<unsigned long long>(), cap,
                                                                                           d_info.as<SlotInfo>(), d_row_slot.as<uint32_t>(), na_equal ? 1 : 0, on);
                else
                    with_key([&](auto fk) {
                        join_insert_count_kernel<fk, decltype(as)::value == 1><<<grid_for(n_build), 256, 0, stream>>>(bcol[0].buf.p, b_ct[0], build_valid(0), n_build, d_tkeys.as<long long>(),
                                                                                               cap, d_info.as<SlotInfo>(), d_row_slot.as<uint32_t>(), na_equal ? 1 : 0, on);
                    });
            });
            d_cnt_multi.alloc(n_slots * 4);
            join_slot_counts_kernel<<<grid_for((int64_t)n_slots), 256, 0, stream>>>(d_info.as<SlotInfo>(), n_slots, d_cnt_multi.as<uint32_t>(), asof ? 1u : 2u);
            launches += 2;
            d_goffs.alloc((n_slots + 1) * 8);
            unsigned long long n_multi = scan.run(d_cnt_multi.as<uint32_t>(), (int64_t)n_slots, d_goffs.as<unsigned long long>(), stream, &launches);
            d_groups.alloc((size_t)std::max<unsigned long long>(n_multi, 1) * 4);
            if (asof) build_asof_groups(n_multi);
            else if (n_multi > 0) {
                d_fill.alloc(n_slots * 4);
                B200_CUDA(cudaMemsetAsync(d_fill.p, 0, n_slots * 4, stream));
                join_fill_groups_kernel<<<grid_for(n_build), 256, 0, stream>>>(d_row_slot.as<uint32_t>(), n_build, d_info.as<SlotInfo>(), d_goffs.as<unsigned long long>(),
                                                                              d_fill.as<uint32_t>(), d_groups.as<uint32_t>());
                launches++;
            }
            d_cnt_multi.release(); d_fill.release(); d_row_slot.release();
            if (n_keys == 1 && n_multi == 0 && !build_outer && !probe_outer && !mark && !anti && cond.empty() && !asof) {
                // every key (incl. the NA / marker groups) has exactly one build row: set up the fused probe path
                form = TableForm::SLOT16;
                setup_slot16();
                d_tkeys.release(); d_info.release();  // the general-path table is not needed any more
            }
        }
        finish_build();
    }
    // what every table form needs before the first probe: the condition's pair counters, the build-outer matched flags
    void finish_build() {
        if (!cond.empty()) {
            d_cond_pairs.alloc(16);
            B200_CUDA(cudaMemsetAsync(d_cond_pairs.p, 0, 16, stream));
            h_cond_pairs = (unsigned long long*)pinned_acquire(16);
        }
        if (build_outer) { d_bmatched.alloc((size_t)std::max<int64_t>(n_build, 1)); B200_CUDA(cudaMemsetAsync(d_bmatched.p, 0, (size_t)std::max<int64_t>(n_build, 1), stream)); }
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(stream));
        build_final = true;
    }

    // One output column of a probe batch: the kept build columns come first, then the kept probe columns.
    struct OutCol {
        bool is_b;      // build side, else probe side
        int src;        // column of that side
        int size;       // item bytes
        bool nullable;  // has validity: one byte per row while the kernels write it, a bitmap in the output
    };
    // A column is nullable when its input has a bitmap or a nullable array type, or when an outer / anti join NULL-extends its side.
    std::vector<OutCol> plan_out(const std::vector<int>& kb, const std::vector<int>& kp, const std::vector<const uint8_t*>& valid) const {
        std::vector<OutCol> cols;
        for (int src : kb) {
            // the unique-key kernels write the probe's key value into the build key column, so it takes the probe key's bitmap
            const bool has_bitmap = (src == 0 && form != TableForm::CSR) ? valid[0] != nullptr : b_has_valid[src];
            cols.push_back({true, src, ctype_size(b_ct[src]), has_bitmap || b_at[src] == ARR_NULLABLE || probe_outer || anti});
        }
        for (int src : kp) cols.push_back({false, src, ctype_size(p_ct[src]), valid[src] != nullptr || p_at[src] == ARR_NULLABLE || build_outer});
        return cols;
    }
    // room for `rows` output rows; the first `keep` rows already written survive a regrowth
    void size_outputs(const std::vector<OutCol>& cols, int64_t rows, int64_t keep = 0) {
        for (size_t k = 0; k < cols.size(); k++) {
            grow_keep(out_data[k], (size_t)(rows + 32) * cols[k].size, (size_t)keep * cols[k].size, stream);
            if (cols[k].nullable) {
                grow_keep(out_vbytes[k], (size_t)rows + 32, (size_t)keep, stream);
                out_bitmap[k].ensure((size_t)((rows + 31) / 32 + 1) * 4);
            }
        }
    }
    uint8_t* out_valid(const std::vector<OutCol>& cols, size_t k) const { return cols[k].nullable ? out_vbytes[k].as<uint8_t>() : nullptr; }
    void describe_out(b200_table* out, const std::vector<OutCol>& cols, int64_t rows) {
        out->n_rows = rows; out->n_cols = (int)cols.size(); out->device = device;
        for (size_t k = 0; k < cols.size(); k++) {
            const OutCol& oc = cols[k];
            b200_column& c = out->cols[k];
            c.data = out_data[k].p; c.length = rows;
            c.c_type = oc.is_b ? b_ct[oc.src] : p_ct[oc.src];
            c.validity = oc.nullable ? out_bitmap[k].as<uint8_t>() : nullptr;
            c.arr_type = oc.nullable ? ARR_NULLABLE : (oc.is_b ? b_at[oc.src] : p_at[oc.src]);
        }
    }

    // unique build keys, inner join: one fused lookup + gather kernel, the inline-payload one when the batch qualifies
    int64_t probe_unique(int64_t n, const std::vector<OutCol>& cols, int nkb, const std::vector<const void*>& data,
                         const std::vector<const uint8_t*>& valid) {
        size_outputs(cols, n);  // matches <= probe rows
        if (n == 0) return 0;
        const int nkp = (int)cols.size() - nkb;
        d_cursor.ensure(8);
        B200_CUDA(cudaMemsetAsync(d_cursor.p, 0, 8, stream));
        // inline-payload variant: every column of this batch 8 bytes wide and bitmap-free, 1..4 kept probe columns
        // (a nullable-typed column without a bitmap still gets one); the inline kernel compares key bits, so a probe key of the
        // other signedness takes the fast kernel
        bool inl = form == TableForm::SLOT32 && valid[0] == nullptr && nkp >= 1 && nkp <= J_INL_MAX_P && nkb <= 4 && !key_reject;
        for (const OutCol& c : cols) inl = inl && c.size == 8 && !c.nullable;
        const int gridp = (int)std::min<int64_t>((int64_t)sms * 8, (n + 1023) / 1024);
        if (inl) {
            InlineProbeArgs ia{};
            ia.n_probe = n; ia.key = (const long long*)data[0]; ia.slots = d_slots32.as<Slot32>(); ia.cap = cap;
            ia.cursor = d_cursor.as<unsigned long long>(); ia.n_b = nkb; ia.na_equal = na_equal ? 1 : 0;
            for (int k = 0; k < (int)cols.size(); k++) {
                if (cols[k].is_b) { ia.b_field[k] = cols[k].src - 1; ia.ob[k] = out_data[k].as<unsigned long long>(); }
                else { ia.p[k - nkb] = (const unsigned long long*)data[cols[k].src]; ia.op[k - nkb] = out_data[k].as<unsigned long long>(); }
            }
            // <FK, NF = build payload columns (0..2), NPK = kept probe columns (1..4)>
            with_key([&](auto fk) {
                with_int<3>(n_b - 1, [&](auto nf) {
                    with_int<J_INL_MAX_P>(nkp - 1, [&](auto npk) { join_probe_inline_kernel<fk, nf, npk + 1><<<gridp, 256, 0, stream>>>(ia); });
                });
            });
            inline_probes++;
        } else {
            if (!d_slots16.p) setup_slot16();
            FastProbeArgs f{};
            f.n_probe = n; f.key_data = data[0]; f.key_ctype = p_ct[0]; f.key_valid = valid[0];
            f.slots = d_slots16.as<Slot16>(); f.cap = cap; f.bpack = d_bpack.as<unsigned long long>(); f.n_fields = std::max(n_b - 1, 1);
            f.cursor = d_cursor.as<unsigned long long>(); f.n_b = nkb; f.n_p = nkp; f.na_equal = na_equal ? 1 : 0; f.key_reject = (int)key_reject;
            for (int k = 0; k < (int)cols.size(); k++) {
                const OutCol& c = cols[k];
                if (c.is_b) {
                    f.b_field[k] = c.src - 1; f.b_size[k] = c.size; f.b_valid[k] = c.src > 0 ? build_valid(c.src) : nullptr;
                    f.ob_data[k] = out_data[k].p; f.ob_valid[k] = out_valid(cols, k);
                } else {
                    const int j = k - nkb;
                    f.p_data[j] = data[c.src]; f.p_valid[j] = valid[c.src]; f.p_size[j] = c.size;
                    f.op_data[j] = out_data[k].p; f.op_valid[j] = out_valid(cols, k);
                }
            }
            with_key([&](auto fk) { join_probe_fast_kernel<fk><<<gridp, 256, 0, stream>>>(f); });
        }
        launches++; fast_probes++;
        B200_CUDA(cudaGetLastError());
        return (int64_t)read_word(d_cursor.as<unsigned long long>());
    }

    // The gather kernels' arguments for a probe batch of n rows: the general path's per-row slots and output offsets, the CSR, and
    // the kept columns of both sides with their output columns (size_outputs first: it may move them).
    GatherArgs gather_args(int64_t n, const std::vector<OutCol>& cols, int nkb, const std::vector<const void*>& data,
                           const std::vector<const uint8_t*>& valid) const {
        GatherArgs g{};
        g.n_probe = n; g.pslot = d_pslot.as<uint32_t>(); g.poff = d_poff.as<unsigned long long>(); g.info = d_info.as<SlotInfo>();
        g.goffs = d_goffs.as<unsigned long long>(); g.groups = d_groups.as<uint32_t>(); g.bmatched = build_outer ? d_bmatched.as<uint8_t>() : nullptr;
        g.n_b = nkb; g.n_p = (int)cols.size() - nkb;
        for (int k = 0; k < (int)cols.size(); k++) {
            const OutCol& c = cols[k];
            if (c.is_b) {
                g.b_data[k] = bcol[c.src].buf.p; g.b_valid[k] = build_valid(c.src); g.b_size[k] = c.size;
                g.ob_data[k] = out_data[k].p; g.ob_valid[k] = out_valid(cols, k);
            } else {
                const int j = k - nkb;
                g.p_data[j] = data[c.src]; g.p_valid[j] = valid[c.src]; g.p_size[j] = c.size;
                g.op_data[j] = out_data[k].p; g.op_valid[j] = out_valid(cols, k);
            }
        }
        return g;
    }

    // as-of join: a left as-of batch is one kernel (output row i = probe row i); an inner one the match kernel, the scan and a
    // one-row gather
    int64_t probe_asof(int64_t n, const std::vector<OutCol>& cols, int nkb, const std::vector<const void*>& data,
                       const std::vector<const uint8_t*>& valid) {
        AsofArgs a{};
        if (n_keys > 1) { a.pk = probe_keys(data, valid); a.bk = build_keys(); }
        else { a.key_data = data[0]; a.key_ctype = p_ct[0]; a.key_valid = valid[0]; }
        a.table = d_tkeys.p; a.cap = cap; a.na_equal = na_equal ? 1 : 0; a.key_reject = key_reject;
        a.info = d_info.as<SlotInfo>(); a.goffs = d_goffs.as<unsigned long long>(); a.groups = d_groups.as<uint32_t>(); a.gwords = d_gwords.as<uint64_t>();
        a.on = AsofOn{data[asof_p_on], valid[asof_p_on], asof_key()};
        a.direction = asof_dir; a.allow_exact = asof_exact ? 1 : 0; a.has_tol = asof_has_tol ? 1 : 0;
        a.tol_w = (unsigned long long)asof_tol_i; a.tol_f = asof_tol_f;
        const int kt = n_keys > 1 ? 2 : float_key ? 1 : 0;
        unsigned long long rows = (unsigned long long)n;
        if (probe_outer) {
            size_outputs(cols, n);
            const GatherArgs g = gather_args(n, cols, nkb, data, valid);
            if (n > 0) with_int<3>(kt, [&](auto k) { join_asof_left_kernel<k><<<grid_for(n), 256, 0, stream>>>(g, a); });
        } else {
            d_pslot.ensure((size_t)(n + 1) * 4); d_pcnt.ensure((size_t)(n + 1) * 4); d_poff.ensure((size_t)(n + 2) * 8);
            rows = 0;
            if (n > 0) {
                with_int<3>(kt, [&](auto k) {
                    join_asof_match_kernel<k><<<grid_for(n), 256, 0, stream>>>(a, n, d_pslot.as<uint32_t>(), d_pcnt.as<uint32_t>());
                });
                launches++;
                B200_CUDA(cudaMemsetAsync(d_pcnt.as<uint32_t>() + n, 0, 4, stream));
                rows = scan.run(d_pcnt.as<uint32_t>(), n + 1, d_poff.as<unsigned long long>(), stream, &launches);
            }
            size_outputs(cols, (int64_t)rows);
            const GatherArgs g = gather_args(n, cols, nkb, data, valid);
            if (rows > 0) join_asof_gather_kernel<<<grid_for(n), 256, 0, stream>>>(g);
        }
        if (n > 0) launches++;
        B200_CUDA(cudaGetLastError());
        return (int64_t)rows;
    }

    // the condition program and the columns it may read: the build store and probe batch `data` / `valid`
    CondArgs cond_args(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid) const {
        CondArgs ca{};
        std::copy(cond.begin(), cond.end(), ca.prog);
        for (int c = 0; c < n_b; c++) { ca.b_data[c] = bcol[c].buf.p; ca.b_valid[c] = build_valid(c); ca.b_ct[c] = b_ct[c]; }
        for (int c = 0; c < n_p; c++) { ca.p_data[c] = data[c]; ca.p_valid[c] = valid[c]; ca.p_ct[c] = p_ct[c]; }
        return ca;
    }

    // ---- nested-loop join (n_keys 0) ----
    // The condition kernels' grid for a batch of n probe rows: build chunks of a multiple of NLJ_SUB rows, enough of them that the
    // probe tiles × chunks fill the GPU about NLJ_BLOCKS_PER_SM times over, so a probe batch of a few rows still spreads over every
    // SM; a large batch gets one chunk and a count matrix of 2 n entries.  The build columns the condition reads are staged.
    static constexpr int NLJ_BLOCKS_PER_SM = 8;
    NljArgs nlj_args(int64_t n) const {
        NljArgs na{};
        na.n_probe = n; na.n_build = n_build;
        if (n > 0 && n_build > 0) {
            const int64_t tiles = (n + NLJ_TILE_P - 1) / NLJ_TILE_P, subs = (n_build + NLJ_SUB - 1) / NLJ_SUB;
            const int64_t chunks = std::min(std::max<int64_t>(1, ((int64_t)sms * NLJ_BLOCKS_PER_SM + tiles - 1) / tiles), subs);
            na.chunk = (subs + chunks - 1) / chunks * NLJ_SUB;
        }
        std::fill(na.b_slot, na.b_slot + J_MAX_COLS, (int8_t)-1);
        for (const ExprInstr& in : cond)
            if (in.op == EX_COL && in.arg < J_MAX_COLS && na.b_slot[in.arg] < 0 && na.n_stage < NLJ_MAX_STAGE) {
                na.b_slot[in.arg] = (int8_t)na.n_stage;
                na.stage_col[na.n_stage++] = (int)in.arg;
            }
        return na;
    }
    static std::string nlj_too_many(unsigned long long rows, const std::string& how) {
        return "b200 join: this nested-loop probe call would produce " + std::to_string(rows) + " output rows (" + how +
               "); one probe call produces at most 2^31 rows: feed smaller probe batches";
    }
    // Every (probe row, build row) pair is a candidate.  Rows go out in probe order, each probe row's pairs in build arrival order, a
    // NULL-extended / anti / mark row in its probe row's place; the build-outer tail follows the last probe call.
    int64_t probe_nested(int64_t n, const std::vector<OutCol>& cols, int nkb, const std::vector<const void*>& data,
                         const std::vector<const uint8_t*>& valid, bool is_last) {
        const int mode = anti ? 1 : (mark ? 2 : 0);
        if (mark && n > 0) { d_mark.ensure((size_t)n + 32); d_mark_valid.ensure((size_t)(n + 7) / 8 + 32); B200_CUDA(cudaMemsetAsync(d_mark_valid.p, 0xff, (size_t)(n + 7) / 8 + 8, stream)); }
        int64_t rows = 0;
        if (cond.empty()) {
            // the counts are arithmetic: n × n_build pairs (inner / outer kinds), or one row per probe row: every one for a mark join,
            // every one for an anti join against an empty build side and for a left / full join that NULL-extends them
            const bool cross = mode == 0 && n_build > 0;
            if (cross) {
                B200_REQUIRE(n <= NLJ_MAX_ROWS / n_build, nlj_too_many((unsigned long long)n * (unsigned long long)n_build,
                                                                       std::to_string(n) + " probe rows x " + std::to_string(n_build) + " build rows"));
                rows = n * n_build;
            } else if (mode == 2 || (n_build == 0 && (mode == 1 || probe_outer))) {
                rows = n;
            }
            size_outputs(cols, rows);
            GatherArgs g = gather_args(n, cols, nkb, data, valid);
            g.poff = nullptr;
            if (rows > 0) {
                if (cross) nlj_cross_kernel<<<grid_for(rows), 256, 0, stream>>>(g, (uint32_t)n_build, (uint32_t)rows);
                else nlj_probe_rows_kernel<<<grid_for(n), 256, 0, stream>>>(g, 0);
                launches++;
            }
            if (mark && n > 0) B200_CUDA(cudaMemsetAsync(d_mark.p, n_build > 0 ? 1 : 0, (size_t)n, stream));
            if (build_outer && n > 0 && n_build > 0) B200_CUDA(cudaMemsetAsync(d_bmatched.p, 1, (size_t)n_build, stream));  // every pair joins
        } else {
            const NljArgs na = nlj_args(n);
            const CondArgs ca = cond_args(data, valid);
            const int chunks = na.chunk ? (int)((n_build + na.chunk - 1) / na.chunk) : 0;
            const int64_t entries = n * (chunks + 1);
            const dim3 grid((unsigned)((n + NLJ_TILE_P - 1) / NLJ_TILE_P), (unsigned)chunks);
            const size_t smem = (size_t)na.n_stage * NLJ_SUB * 9;  // bits (8 B), then validity (1 B), per staged column and row
            d_pcnt.ensure((size_t)(entries + 1) * 4); d_poff.ensure((size_t)(entries + 2) * 8);
            if (n > 0) {
                if (chunks > 0) {
                    nlj_count_kernel<<<grid, NLJ_WARPS * 32, smem, stream>>>(ca, na, d_pcnt.as<uint32_t>(), d_cond_pairs.as<unsigned long long>());
                    launches++;
                }
                nlj_rows_kernel<<<grid_for(n), 256, 0, stream>>>(n, chunks, d_pcnt.as<uint32_t>(), probe_outer ? 1 : 0, mode, mark ? d_mark.as<uint8_t>() : nullptr);
                launches++;
                B200_CUDA(cudaGetLastError());
                B200_CUDA(cudaMemsetAsync(d_pcnt.as<uint32_t>() + entries, 0, 4, stream));
                rows = (int64_t)scan.run(d_pcnt.as<uint32_t>(), entries + 1, d_poff.as<unsigned long long>(), stream, &launches);
            }
            B200_REQUIRE(rows <= NLJ_MAX_ROWS, nlj_too_many((unsigned long long)rows, "pairs that pass the condition"));
            size_outputs(cols, rows);
            const GatherArgs g = gather_args(n, cols, nkb, data, valid);
            if (rows > 0) {
                if (mode == 0 && chunks > 0) { nlj_gather_kernel<<<grid, NLJ_WARPS * 32, smem, stream>>>(g, ca, na); launches++; }
                if (mode != 0 || probe_outer) { nlj_probe_rows_kernel<<<grid_for(n), 256, 0, stream>>>(g, chunks); launches++; }
            }
        }
        B200_CUDA(cudaGetLastError());
        return rows + emit_build_tail(cols, nkb, rows, is_last);
    }

    // The unmatched build rows of a build-outer join, with NULL probe columns, after the `n_before` rows this call has written: once,
    // with the last probe batch (bmatched must be complete).  Returns the rows added.
    int64_t emit_build_tail(const std::vector<OutCol>& cols, int nkb, int64_t n_before, bool is_last) {
        if (!(is_last && build_outer && !tail_emitted && n_build > 0)) return 0;
        DevBuf tail_flags, tail_off;
        tail_flags.alloc((size_t)(n_build + 1) * 4); tail_off.alloc((size_t)(n_build + 2) * 8);
        join_unmatched_flags_kernel<<<grid_for(n_build), 256, 0, stream>>>(d_bmatched.as<uint8_t>(), n_build, tail_flags.as<uint32_t>());
        B200_CUDA(cudaMemsetAsync(tail_flags.as<uint32_t>() + n_build, 0, 4, stream));
        launches++;
        const unsigned long long n_tail = scan.run(tail_flags.as<uint32_t>(), n_build + 1, tail_off.as<unsigned long long>(), stream, &launches);
        tail_emitted = true;
        if (n_tail > 0) {
            // the tail size is only known after the gather: grow the outputs, keeping the gathered rows
            size_outputs(cols, n_before + (int64_t)n_tail, n_before);
            TailArgs ta{};
            ta.n_build = n_build; ta.flags = tail_flags.as<uint32_t>(); ta.off = tail_off.as<unsigned long long>();
            ta.n_b = nkb; ta.n_p = (int)cols.size() - nkb;
            for (int k = 0; k < (int)cols.size(); k++) {
                const OutCol& c = cols[k];
                void* od = (char*)out_data[k].p + n_before * c.size;
                uint8_t* ov = c.nullable ? out_vbytes[k].as<uint8_t>() + n_before : nullptr;
                if (c.is_b) {
                    ta.b_data[k] = bcol[c.src].buf.p; ta.b_valid[k] = build_valid(c.src); ta.b_size[k] = c.size;
                    ta.ob_data[k] = od; ta.ob_valid[k] = ov;
                } else {
                    const int j = k - nkb;
                    ta.p_size[j] = c.size; ta.op_data[j] = od; ta.op_valid[j] = ov;
                }
            }
            join_unmatched_emit_kernel<<<grid_for(n_build), 256, 0, stream>>>(ta);
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        return (int64_t)n_tail;
    }

    // general path (CSR groups: duplicate keys, outer, anti and mark joins): count + scan, then expand and gather; the unmatched
    // build rows of a build-outer join follow the last probe batch
    int64_t probe_general(int64_t n, const std::vector<OutCol>& cols, int nkb, const std::vector<const void*>& data,
                          const std::vector<const uint8_t*>& valid, bool is_last) {
        // pass A + scan; with a condition pass A gives the slot (mode 0, no probe_outer row) and the condition count kernel the counts
        const bool has_cond = !cond.empty();
        const int mode = anti ? 1 : (mark ? 2 : 0), count_mode = has_cond ? 0 : mode, count_po = probe_outer && !has_cond ? 1 : 0;
        const CondArgs ca = has_cond ? cond_args(data, valid) : CondArgs{};
        unsigned long long n_match = 0;
        d_pslot.ensure((size_t)(n + 1) * 4); d_pcnt.ensure((size_t)(n + 1) * 4); d_poff.ensure((size_t)(n + 2) * 8);
        if (n > 0) {
            if (mark) { d_mark.ensure((size_t)n + 32); d_mark_valid.ensure((size_t)(n + 7) / 8 + 32); B200_CUDA(cudaMemsetAsync(d_mark_valid.p, 0xff, (size_t)(n + 7) / 8 + 8, stream)); }
            if (n_keys > 1)
                join_probe_count_mk_kernel<<<grid_for(n), 256, 0, stream>>>(probe_keys(data, valid), build_keys(), n, d_tkeys.as<unsigned long long>(), cap,
                                                                            d_info.as<SlotInfo>(), count_po, d_pslot.as<uint32_t>(), d_pcnt.as<uint32_t>(),
                                                                            na_equal ? 1 : 0, count_mode, mark ? d_mark.as<uint8_t>() : nullptr,
                                                                            key_reject);
            else
                with_key([&](auto fk) {
                    join_probe_count_kernel<fk><<<grid_for(n), 256, 0, stream>>>(data[0], p_ct[0], valid[0], n, d_tkeys.as<long long>(), cap, d_info.as<SlotInfo>(),
                                                                                 count_po, d_pslot.as<uint32_t>(), d_pcnt.as<uint32_t>(), na_equal ? 1 : 0,
                                                                                 count_mode, mark ? d_mark.as<uint8_t>() : nullptr, (int)key_reject);
                });
            launches++;
            if (has_cond) {
                join_cond_count_kernel<<<grid_for(n), 256, 0, stream>>>(ca, n, d_pslot.as<uint32_t>(), d_info.as<SlotInfo>(), d_goffs.as<unsigned long long>(),
                                                                        d_groups.as<uint32_t>(), probe_outer ? 1 : 0, mode, d_pcnt.as<uint32_t>(),
                                                                        mark ? d_mark.as<uint8_t>() : nullptr, d_cond_pairs.as<unsigned long long>());
                launches++;
                B200_CUDA(cudaGetLastError());
            }
            B200_CUDA(cudaMemsetAsync(d_pcnt.as<uint32_t>() + n, 0, 4, stream));
            n_match = scan.run(d_pcnt.as<uint32_t>(), n + 1, d_poff.as<unsigned long long>(), stream, &launches);
        }
        // pass B needs bmatched complete before the tail is computed, so: gather first, then the tail
        size_outputs(cols, (int64_t)n_match);
        const GatherArgs g = gather_args(n, cols, nkb, data, valid);
        if (n > 0 && n_match > 0) {
            if (has_cond) join_cond_gather_kernel<<<grid_for(n), 256, 0, stream>>>(g, ca, mode);
            else join_probe_gather_kernel<<<grid_for(n), 256, 0, stream>>>(g);
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        return (int64_t)n_match + emit_build_tail(cols, nkb, (int64_t)n_match, is_last);
    }

    int64_t probe_consume(const b200_table* t, const uint64_t* kept_b, int64_t n_kb, const uint64_t* kept_p, int64_t n_kp,
                          b200_table* out, bool is_last) {
        B200_REQUIRE(build_final, "b200 join: probe before the build side was finished (is_last build batch)");
        if (n_p == 0) {  // adopt the probe schema from the first probe batch
            B200_REQUIRE(t->n_cols >= 1 && t->n_cols <= J_MAX_COLS, "b200 join: between 1 and 32 columns per side");
            std::vector<int8_t> ct(t->n_cols), at(t->n_cols);
            for (int c = 0; c < t->n_cols; c++) { ct[c] = (int8_t)t->cols[c].c_type; at[c] = (int8_t)t->cols[c].arr_type; }
            set_probe_schema(ct.data(), at.data(), t->n_cols);
        }
        B200_REQUIRE(t->n_cols == n_p, "b200 join: probe batch has a different number of columns than the schema");
        B200_REQUIRE(out->cols != nullptr, "b200 join: out->cols must point to n_kept_build + n_kept_probe descriptors");
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        std::vector<int> kb, kp;
        for (int64_t k = 0; k < n_kb; k++) { B200_REQUIRE((int)kept_b[k] < n_b, "b200 join: bad kept build column"); kb.push_back((int)kept_b[k]); }
        for (int64_t k = 0; k < n_kp; k++) { B200_REQUIRE((int)kept_p[k] < n_p, "b200 join: bad kept probe column"); kp.push_back((int)kept_p[k]); }
        int n_out_cols = (int)(kb.size() + kp.size());
        B200_REQUIRE(n_out_cols + (mark ? 1 : 0) <= J_MAX_COLS, "b200 join: too many output columns");
        B200_REQUIRE(!mark || kb.empty(), "b200 join: a mark join does not output build table columns (bodo/pandas/physical/join.h:309-316)");
        int64_t n = t->n_rows;
        std::vector<const void*> data; std::vector<const uint8_t*> valid;
        stage_batch(t, n_p, p_ct, data, valid);
        const std::vector<OutCol> cols = plan_out(kb, kp, valid);
        const int64_t rows = asof                     ? probe_asof(n, cols, (int)kb.size(), data, valid)
                             : n_keys == 0            ? probe_nested(n, cols, (int)kb.size(), data, valid, is_last)
                             : form == TableForm::CSR ? probe_general(n, cols, (int)kb.size(), data, valid, is_last)
                                                      : probe_unique(n, cols, (int)kb.size(), data, valid);
        for (int k = 0; k < n_out_cols; k++)
            if (cols[k].nullable && rows > 0) { launch_pack_bitmap(out_vbytes[k].as<uint8_t>(), rows, out_bitmap[k].as<uint32_t>(), grid_for(rows), stream); launches++; }
        B200_CUDA(cudaGetLastError());
        if (h_cond_pairs) B200_CUDA(cudaMemcpyAsync(h_cond_pairs, d_cond_pairs.p, 16, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        if (h_cond_pairs) { cond_evaluated = (int64_t)h_cond_pairs[0]; cond_passed = (int64_t)h_cond_pairs[1]; }
        describe_out(out, cols, rows);
        if (mark) {  // the mark column: BOOL, nullable array type, every row valid; output row i is probe row i
            b200_column& c = out->cols[n_out_cols];
            c.data = d_mark.p; c.validity = d_mark_valid.as<uint8_t>(); c.length = rows; c.c_type = CT_BOOL; c.arr_type = ARR_NULLABLE;
            out->n_cols = n_out_cols + 1;
        }
        probe_rows += n; out_rows_total += rows;
        return rows;
    }
};

}  // namespace b200

using b200::JoinState;

extern "C" {

void* b200_join_state_init(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                           int32_t n_build_arrs, const int8_t* probe_arr_c_types, const int8_t* probe_arr_array_types,
                           int32_t n_probe_arrs, uint64_t n_keys, int32_t build_table_outer, int32_t probe_table_outer,
                           int32_t is_na_equal, int64_t output_batch_size, int32_t device, int64_t expected_build_rows, void* stream) {
    (void)operator_id;
    try {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw b200::Error("b200 join: no CUDA device available (this path has no CPU fallback)");
        B200_REQUIRE(device >= 0 && device < ndev, "b200 join: bad device ordinal");
        return new JoinState(build_arr_c_types, build_arr_array_types, n_build_arrs, probe_arr_c_types, probe_arr_array_types, n_probe_arrs,
                             n_keys, build_table_outer != 0, probe_table_outer != 0, is_na_equal != 0, output_batch_size, device, expected_build_rows, (cudaStream_t)stream);
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return nullptr; }
}

int b200_join_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last, int32_t* request_input) {
    try {
        B200_REQUIRE(state && in_table, "b200 join: null state or table");
        ((JoinState*)state)->build_consume(in_table, is_last != 0);
        if (request_input) *request_input = 1;
        return is_last ? 1 : 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_probe_consume_batch(void* state, const b200_table* in_table, const uint64_t* kept_build_cols, int64_t n_kept_build,
                                  const uint64_t* kept_probe_cols, int64_t n_kept_probe, b200_table* out, int64_t* total_rows,
                                  int32_t is_last, int32_t* out_is_last) {
    try {
        B200_REQUIRE(state && in_table && out, "b200 join: null argument");
        int64_t rows = ((JoinState*)state)->probe_consume(in_table, kept_build_cols, n_kept_build, kept_probe_cols, n_kept_probe, out, is_last != 0);
        if (total_rows) *total_rows = rows;
        if (out_is_last) *out_is_last = is_last ? 1 : 0;
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

void b200_delete_join_state(void* state) { delete (JoinState*)state; }

int b200_join_set_kind(void* state, int32_t is_mark_join, int32_t is_anti_join) {
    try {
        B200_REQUIRE(state, "b200 join: null state");
        ((JoinState*)state)->set_kind(is_mark_join != 0, is_anti_join != 0);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_set_condition(void* state, const void* program, int32_t n_instr) {
    try {
        B200_REQUIRE(state && program, "b200 join: null argument");
        ((JoinState*)state)->set_condition((const b200::ExprInstr*)program, n_instr);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_set_asof(void* state, int32_t build_on_col, int32_t probe_on_col, int32_t direction, int32_t allow_exact_matches,
                        int32_t has_tolerance, int64_t tolerance_i64, double tolerance_f64) {
    try {
        B200_REQUIRE(state, "b200 join: null state");
        ((JoinState*)state)->set_asof(build_on_col, probe_on_col, direction, allow_exact_matches != 0, has_tolerance != 0, tolerance_i64, tolerance_f64);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_build_filter(void* state, int64_t n_bloom_blocks, void** bloom_words_dev, int64_t* n_blocks_out, int64_t* key_min_max) {
    try {
        B200_REQUIRE(state && n_bloom_blocks >= 0, "b200 join: bad arguments");
        auto* s = (JoinState*)state;
        s->build_filter((uint64_t)n_bloom_blocks);
        if (bloom_words_dev) *bloom_words_dev = s->d_bloom.p;
        if (n_blocks_out) *n_blocks_out = (int64_t)s->bloom_blocks;
        if (key_min_max) std::copy(s->key_bounds, s->key_bounds + 2 * s->n_keys, key_min_max);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_set_key_bounds_n(void* state, const int64_t* key_min_max, int32_t n_keys) {
    try {
        B200_REQUIRE(state && key_min_max, "b200 join: null argument");
        auto* s = (JoinState*)state;
        B200_REQUIRE(n_keys == s->n_keys, "b200 join: set_key_bounds_n: n_keys is " + std::to_string(n_keys) + " and this join has " +
                                              std::to_string(s->n_keys) + " key columns");
        std::copy(key_min_max, key_min_max + 2 * n_keys, s->key_bounds);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_join_runtime_filter_n(void* state, const b200_table* in_table, const int32_t* key_cols, int32_t n_keys, const int32_t* use_min_max,
                               int32_t use_bloom, uint8_t* keep_out) {
    try {
        B200_REQUIRE(state && in_table && key_cols && use_min_max && keep_out, "b200 join: null argument");
        ((JoinState*)state)->runtime_filter(in_table, key_cols, n_keys, use_min_max, use_bloom != 0, keep_out);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int64_t b200_join_get_metric(void* state, int32_t which) {
    auto* s = (JoinState*)state;
    switch (which) {
        case 0: return s->n_build;
        case 1: return (int64_t)s->cap;
        case 2: return s->probe_rows;
        case 3: return s->out_rows_total;
        case 4: return s->launches;
        case 5: return s->fast_probes;
        case 6: return s->inline_probes;
        case 7: return s->inline_builds;
        case 8: return s->cond_evaluated;
        case 9: return s->cond_passed;
        default: return -1;
    }
}

}  // extern "C"
