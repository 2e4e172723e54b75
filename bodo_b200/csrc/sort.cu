// sort.cu — streaming sort over a stream of batches (sm_90a): ORDER BY k_0 .. k_{n-1} [LIMIT limit OFFSET offset].
//
// Replaces the reference's streaming sort state (bodo/libs/streaming/_sort.cpp: stream_sort_state_init_py_entry, the
// build-consume and produce-output entries, delete_stream_sort_state), which DuckDB's ORDER BY and TopN lower to (PhysicalSort,
// bodo/pandas/physical/sort.h).  Two forms share the schema, the batch checks, the key encoding and the output side (SortState);
// each keeps its own rows:
//
//   TopkState      ORDER BY ... LIMIT: only the first K = limit + offset rows of the stable sort are ever needed, so the state
//                  keeps at most K "held" rows and a device-resident cutoff, the key tuple of the K-th held row (topk_* kernels).
//   FullSortState  ORDER BY without LIMIT: every row is appended to a chunk store and radix-sorted at is_last (fsort_* kernels).
//
// Key encoding (sort_word): each key cell becomes an unsigned integer of the key's own width whose unsigned order is the key
// order (sign bit flipped for signed integers and temporals; float32 and float64 in their ordered forms with -0.0 folded onto
// +0.0; complemented for a descending key), plus one NA-class bit: NA and NaN keys get word 0 and class 1 for
// na_position="last", 0 for "first"; other keys the opposite class.  Rows compare lexicographically over (class_0, word_0,
// class_1, word_1, ..., arrival index), so no two rows are equal.
#include <algorithm>
#include <cfloat>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace b200 {

constexpr int SORT_MAX_KEYS = 4;
constexpr int SORT_MAX_COLS = 32;

// The schema both forms sort by: one descriptor per key (the first n_keys columns, SortKey in common.cuh) and every column's
// type.
struct SortSchema {
    int n_keys, n_cols;
    SortKey key[SORT_MAX_KEYS];
    int ctype[SORT_MAX_COLS];
};

// ---- top-k (ORDER BY ... LIMIT): candidate filter, bitonic sort + merge reduce ----
//
//   topk_filter_kernel   one pass per batch over the key columns only: a row survives iff its key tuple is strictly below the
//                        cutoff (a row that ties the cutoff sorts after the held row, its arrival index is larger).  Survivors are
//                        compacted (warp ballot -> tile scan -> one cursor atomic per tile) into the candidate store together with
//                        their key words, arrival index and every column; payload bytes are read for survivors only.
//   reduce               held rows + candidates are sorted by (key words, arrival index): topk_block_sort_kernel (bitonic sort of
//                        1024-row tiles in shared memory) then topk_merge_kernel passes (merge path over pairs of sorted runs,
//                        every run cut to its first K rows); topk_gather_kernel moves the first K rows into the other store buffer
//                        and writes the new cutoff.
//
// The store keeps each key's word zero-extended to 64 bits; words of one key all have that key's width, so they compare as they
// would at it.  No two rows are equal, so the (unstable) bitonic sort still yields the stable order.
//
// K = limit + offset is capped so that store row ids (uint32, the sort permutation) and the two store buffers of max(2K, 4 Mi)
// rows stay within reach: 2^26 rows is 2 x 128 Mi rows of store, about 5 GB per 8-byte column.
constexpr int64_t TK_MAX_K = 1ll << 26;
// Store capacity: max(2K, 4 Mi rows).  At least 2K so that a reduce (down to K rows) always frees at least K rows for the next
// slice of a batch; at least 4 Mi rows so that, once a cutoff exists and few rows survive, the host needs to read the candidate
// count only about once per 4 Mi consumed rows (it keeps an upper bound and reads only when that bound could overflow).
constexpr int64_t TK_MIN_CAP = 1ll << 22;
constexpr int TK_THREADS = 256, TK_ROWS = 4, TK_TILE = TK_THREADS * TK_ROWS;
constexpr int TK_SORT_TILE = 1024, TK_SORT_THREADS = 512, TK_MERGE_ITEMS = 8;
constexpr uint32_t TK_SENTINEL = 0xFFFFFFFFu;

struct TkCutoff { uint32_t has; uint32_t cls; uint64_t w[SORT_MAX_KEYS]; };

// One buffer of rows, structure of arrays: key words, NA-class bits (bit j = key j), arrival index, every column's values and,
// for nullable columns, one validity byte per row.
struct TkStore {
    uint64_t* w[SORT_MAX_KEYS];
    uint8_t* cls;
    int64_t* seq;
    void* data[SORT_MAX_COLS];
    uint8_t* vb[SORT_MAX_COLS];
};

struct TkFilterArgs {
    SortSchema sc;
    int64_t row0, row1;      // rows [row0, row1) of the batch
    int64_t seq_base;        // arrival index of batch row 0
    const void* in_data[SORT_MAX_COLS];
    const uint8_t* in_valid[SORT_MAX_COLS];
    const TkCutoff* cutoff;
    TkStore st;
    unsigned long long* cursor;  // rows in the store
};

// Radix word of key j at batch row i; *cls receives its NA-class bit.
__device__ __forceinline__ uint64_t tk_word(const TkFilterArgs& a, int j, int64_t i, uint32_t* cls) {
    const SortKey& k = a.sc.key[j];
    bool na = !bit_valid(a.in_valid[j], i);
    const uint64_t w = sort_word(k, load_bits(a.in_data[j], k.size, i), na);
    *cls = sort_class(k, na);
    return w;
}

// The row's key tuple is strictly below the cutoff's.
__device__ __forceinline__ bool tk_below_cutoff(const TkFilterArgs& a, const TkCutoff& c, int64_t row) {
#pragma unroll
    for (int j = 0; j < SORT_MAX_KEYS; j++) {
        if (j < a.sc.n_keys) {
            uint32_t cl;
            const uint64_t w = tk_word(a, j, row, &cl);
            const uint32_t cc = (c.cls >> j) & 1;
            if (cl != cc) return cl < cc;
            if (w != c.w[j]) return w < c.w[j];
        }
    }
    return false;
}

__global__ void __launch_bounds__(TK_THREADS, 4) topk_filter_kernel(const __grid_constant__ TkFilterArgs a) {
    __shared__ unsigned int wsum[TK_ROWS][TK_THREADS / 32];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const TkCutoff cut = *a.cutoff;
    const int64_t n = a.row1 - a.row0;
    const int64_t n_tiles = (n + TK_TILE - 1) / TK_TILE;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        bool keep[TK_ROWS];
        unsigned int rank[TK_ROWS];
#pragma unroll
        for (int r = 0; r < TK_ROWS; r++) {
            const int64_t row = a.row0 + t * TK_TILE + r * TK_THREADS + threadIdx.x;
            keep[r] = row < a.row1 && (!cut.has || tk_below_cutoff(a, cut, row));
            const unsigned m = __ballot_sync(0xffffffffu, keep[r]);
            rank[r] = __popc(m & ((1u << lane) - 1));
            if (lane == 0) wsum[r][warp] = __popc(m);
        }
        __syncthreads();
        if (threadIdx.x < 32) {  // exclusive scan of the 32 (row slot, warp) counts; one cursor atomic per tile
            const int r = threadIdx.x >> 3, w = threadIdx.x & 7;
            const unsigned int x = wsum[r][w], inc = warp_inclusive_scan<SumOf<unsigned int>>(x);
            wsum[r][w] = inc - x;
            if (lane == 31) tile_base = inc ? atomicAdd(a.cursor, (unsigned long long)inc) : 0ull;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < TK_ROWS; r++) {
            if (!keep[r]) continue;
            const int64_t row = a.row0 + t * TK_TILE + r * TK_THREADS + threadIdx.x;
            const int64_t o = (int64_t)(tile_base + wsum[r][warp] + rank[r]);
            uint32_t cls = 0;
            for (int j = 0; j < a.sc.n_keys; j++) {  // survivors are rare once a cutoff exists: encode again instead of holding it
                uint32_t cl;
                a.st.w[j][o] = tk_word(a, j, row, &cl);
                cls |= cl << j;
            }
            a.st.cls[o] = (uint8_t)cls;
            a.st.seq[o] = a.seq_base + row;
            for (int c = 0; c < a.sc.n_cols; c++) {
                copy_cell(a.st.data[c], o, a.in_data[c], row, ctype_size(a.sc.ctype[c]));
                if (a.st.vb[c]) a.st.vb[c][o] = bit_valid(a.in_valid[c], row) ? 1 : 0;
            }
        }
        __syncthreads();
    }
}

// Order of two store rows: (class_0, word_0, ..., arrival index).  Never equal for two different rows.
__device__ __forceinline__ bool tk_less(const TkStore& s, int nk, uint32_t a, uint32_t b) {
    const uint32_t ca = s.cls[a], cb = s.cls[b];
#pragma unroll
    for (int j = 0; j < SORT_MAX_KEYS; j++) {
        if (j < nk) {
            const uint32_t x = (ca >> j) & 1, y = (cb >> j) & 1;
            if (x != y) return x < y;
            const uint64_t wa = s.w[j][a], wb = s.w[j][b];
            if (wa != wb) return wa < wb;
        }
    }
    return s.seq[a] < s.seq[b];
}
__device__ __forceinline__ bool tk_less_sent(const TkStore& s, int nk, uint32_t a, uint32_t b) {
    if (a == TK_SENTINEL) return false;
    if (b == TK_SENTINEL) return true;
    return tk_less(s, nk, a, b);
}

// Row ids of a sorted run starting at o of width w, cut to its first K rows.
__host__ __device__ __forceinline__ int64_t tk_run_len(int64_t o, int64_t w, int64_t n, int64_t K) {
    if (o >= n) return 0;
    const int64_t l = n - o < w ? n - o : w;
    return l < K ? l : K;
}

// Bitonic sort of the row ids of one TK_SORT_TILE-row tile; writes the tile's first min(K, rows) ids.
__global__ void __launch_bounds__(TK_SORT_THREADS) topk_block_sort_kernel(const TkStore s, int nk, int64_t n, int64_t K, uint32_t* out) {
    __shared__ uint32_t v[TK_SORT_TILE];
    const int64_t o = (int64_t)blockIdx.x * TK_SORT_TILE;
    const int len = (int)(n - o < TK_SORT_TILE ? n - o : TK_SORT_TILE);
    for (int i = threadIdx.x; i < TK_SORT_TILE; i += TK_SORT_THREADS) v[i] = i < len ? (uint32_t)(o + i) : TK_SENTINEL;
    __syncthreads();
    for (int k = 2; k <= TK_SORT_TILE; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < TK_SORT_TILE; i += TK_SORT_THREADS) {
                const int p = i ^ j;
                if (p > i) {
                    const uint32_t x = v[i], y = v[p];
                    const bool up = (i & k) == 0;
                    if (up ? tk_less_sent(s, nk, y, x) : tk_less_sent(s, nk, x, y)) { v[i] = y; v[p] = x; }
                }
            }
            __syncthreads();
        }
    }
    const int64_t keep = tk_run_len(o, TK_SORT_TILE, n, K);
    for (int i = threadIdx.x; i < keep; i += TK_SORT_THREADS) out[o + i] = v[i];
}

// Outputs [d0, min(d0 + ITEMS, m)) of the merge of two sorted runs of row ids, A(i) for i < la and B(j) for j < lb, go to out[d0 ..].
// The thread finds where its outputs start on the merge path by binary search, then merges them sequentially.  b_first(b, a):
// row b sorts strictly before row a; a row of A that ties a row of B comes first.
template <int ITEMS, typename RunA, typename RunB, typename BFirst>
__device__ __forceinline__ void merge_path_items(RunA A, int64_t la, RunB B, int64_t lb, int64_t d0, int64_t m, uint32_t* __restrict__ out,
                                                 BFirst b_first) {
    int64_t lo = d0 - lb > 0 ? d0 - lb : 0, hi = d0 < la ? d0 : la;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (b_first(B(d0 - mid - 1), A(mid))) hi = mid; else lo = mid + 1;
    }
    int64_t i = lo, j = d0 - lo;
    for (int t = 0; t < ITEMS && d0 + t < m; t++) {
        const bool take_a = j >= lb || (i < la && !b_first(B(j), A(i)));
        out[d0 + t] = take_a ? A(i++) : B(j++);
    }
}

// One merge pass: runs of width w at offsets 2pw and 2pw + w become one run of width 2w (cut to K rows).
__global__ void topk_merge_kernel(const TkStore s, int nk, int64_t n, int64_t K, int64_t w, int64_t chunks_per_pair, int64_t n_pairs,
                                  const uint32_t* __restrict__ in, uint32_t* __restrict__ out) {
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n_pairs * chunks_per_pair) return;
    const int64_t p = gid / chunks_per_pair, d0 = (gid % chunks_per_pair) * TK_MERGE_ITEMS;
    const int64_t ao = 2 * p * w, bo = ao + w;
    const int64_t la = tk_run_len(ao, w, n, K), lb = tk_run_len(bo, w, n, K);
    const int64_t m = la + lb < K ? la + lb : K;
    if (d0 >= m) return;
    const uint32_t* A = in + ao;
    const uint32_t* B = in + bo;
    merge_path_items<TK_MERGE_ITEMS>([&](int64_t i) { return A[i]; }, la, [&](int64_t j) { return B[j]; }, lb, d0, m, out + ao,
                                     [&](uint32_t b, uint32_t a) { return tk_less(s, nk, b, a); });
}

// dst row i = src row perm[i] for i < m; the K-th row becomes the cutoff; the store count becomes m.
__global__ void topk_gather_kernel(const TkStore src, const TkStore dst, const SortSchema sc, const uint32_t* __restrict__ perm, int64_t m,
                                   int64_t K, TkCutoff* cutoff, unsigned long long* cursor) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid == 0) *cursor = (unsigned long long)m;
    for (int64_t i = gid; i < m; i += stride) {
        const uint32_t si = perm[i];
        for (int j = 0; j < sc.n_keys; j++) dst.w[j][i] = src.w[j][si];
        dst.cls[i] = src.cls[si];
        dst.seq[i] = src.seq[si];
        for (int c = 0; c < sc.n_cols; c++) {
            copy_cell(dst.data[c], i, src.data[c], si, ctype_size(sc.ctype[c]));
            if (dst.vb[c]) dst.vb[c][i] = src.vb[c][si];
        }
        if (i == K - 1) {
            for (int j = 0; j < sc.n_keys; j++) cutoff->w[j] = src.w[j][si];
            cutoff->cls = src.cls[si];
            cutoff->has = 1;
        }
    }
}

// ---- full sort (ORDER BY without LIMIT): append-only chunk store, LSD radix sort at is_last ----
//
//   fsort_append_kernel  per consume call: the batch's columns, plus one validity byte per nullable column, are copied into the
//                        chunk store at rows [rows_consumed, rows_consumed + n).  Arrival order is storage order.
//   fsort_hist_kernel    at is_last: one read of the key columns builds the 256-bin histogram of every byte digit of every key's
//                        radix word and each key's NA count.  The host reads them back once and skips every pass whose digit takes
//                        a single value over all rows.
//   fsort_pass_kernel    one onesweep pass per digit that is not skipped, least significant key first: a stable in-tile rank
//                        (warp multisplit), a decoupled look-back over per-tile digit counts seeded by the global histogram, and a
//                        staged, coalesced copy-out of (radix word, row id) pairs.  The first pass of a key computes its words from
//                        the column: in row order for the first key sorted, through the current permutation for the others.
//   fsort_gather_kernel  every column and validity byte through the final permutation into the output store.
//
// A key that can hold NAs gets one more pass on its NA-class bit after its byte passes; the bit rides in bit 31 of the row id,
// which is why the store holds at most 2^31 rows.
constexpr int FS_CHUNK_LOG = 24;
constexpr int64_t FS_CHUNK = 1ll << FS_CHUNK_LOG;
constexpr int FS_MAX_CHUNKS = 128;
constexpr int64_t FS_MAX_ROWS = (int64_t)FS_MAX_CHUNKS * FS_CHUNK;  // 2^31
constexpr int FS_THREADS = 256, FS_WARPS = FS_THREADS / 32, FS_ITEMS = 16, FS_TILE = FS_THREADS * FS_ITEMS;
constexpr uint32_t FS_ID_MASK = 0x7FFFFFFFu;
constexpr int FS_HIST_WORDS = SORT_MAX_KEYS * 8 * 256 + SORT_MAX_KEYS;  // [key][byte][digit] counts, then one NA count per key
// look-back word: pass epoch (bits 34..63), AGGREGATE / INCLUSIVE flag (bits 32..33), count (bits 0..31)
constexpr unsigned long long FS_AGG = 1ull << 32, FS_INCL = 2ull << 32;
enum { FS_IN_PAIRS = 0, FS_IN_COLUMN = 1, FS_IN_GATHER = 2 };

// One chunk is one allocation: FS_CHUNK values of every column, then FS_CHUNK validity bytes of every nullable column.
struct FsLayout {
    SortSchema sc;
    int64_t coff[SORT_MAX_COLS];  // byte offset of column c's values in a chunk
    int64_t voff[SORT_MAX_COLS];  // byte offset of its validity bytes, -1 for a numpy column
};
struct FsChunks { const char* p[FS_MAX_CHUNKS]; };

// Radix word of the key cell at row `off` of `chunk`, the key's values at byte offset coff and its validity bytes at voff;
// na: the cell is NA or NaN.
__device__ __forceinline__ uint64_t fs_word(const SortKey& k, int64_t coff, int64_t voff, const char* chunk, int64_t off, bool& na) {
    na = voff >= 0 && chunk[voff + off] == 0;
    return sort_word(k, load_bits(chunk + coff, k.size, off), na);
}

template <typename W>
__device__ __forceinline__ uint32_t fs_digit(W w, uint32_t id, int shift) {
    return shift < 0 ? id >> 31 : (uint32_t)(w >> shift) & 0xFFu;
}

struct FsAppendArgs {
    int64_t src0, n, dst0;  // batch rows [src0, src0 + n) go to rows [dst0, dst0 + n) of `chunk`
    FsLayout lay;
    char* chunk;
    const void* in_data[SORT_MAX_COLS];
    const uint8_t* in_valid[SORT_MAX_COLS];
};

__global__ void __launch_bounds__(256) fsort_append_kernel(const __grid_constant__ FsAppendArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
        const int64_t s = a.src0 + i, o = a.dst0 + i;
        for (int c = 0; c < a.lay.sc.n_cols; c++) {
            copy_cell(a.chunk + a.lay.coff[c], o, a.in_data[c], s, ctype_size(a.lay.sc.ctype[c]));
            if (a.lay.voff[c] >= 0) a.chunk[a.lay.voff[c] + o] = bit_valid(a.in_valid[c], s) ? 1 : 0;
        }
    }
}

// Where the radix words come from: word(k, j, r, na) is the radix word of key j's cell at row r (key j described by k), na as
// fs_word's.  FsChunkSrc reads the full sort's chunk store; FsArraySrc plain device columns (validity one byte per row,
// nullptr = none), which is how the join's as-of build hands over its (slot, on) keys.  A pass reads one key: the host hands
// it the source of that key as key 0 (for_key), so the pass kernel indexes no parameter array.
struct FsChunkSrc {
    FsChunks ch;
    int64_t coff[SORT_MAX_KEYS], voff[SORT_MAX_KEYS];
    __device__ __forceinline__ uint64_t word(const SortKey& k, int j, uint32_t r, bool& na) const {
        return fs_word(k, coff[j], voff[j], ch.p[r >> FS_CHUNK_LOG], r & (FS_CHUNK - 1), na);
    }
    FsChunkSrc for_key(int j) const { FsChunkSrc s = *this; s.coff[0] = coff[j]; s.voff[0] = voff[j]; return s; }
};
struct FsArraySrc {
    const void* data[SORT_MAX_KEYS];
    const uint8_t* valid[SORT_MAX_KEYS];
    __device__ __forceinline__ uint64_t word(const SortKey& k, int j, uint32_t r, bool& na) const {
        na = valid[j] && !valid[j][r];
        return sort_word(k, load_bits(data[j], k.size, r), na);
    }
    FsArraySrc for_key(int j) const { FsArraySrc s = *this; s.data[0] = data[j]; s.valid[0] = valid[j]; return s; }
};

template <typename Src>
struct FsHistArgs {
    int64_t n;
    int nk;
    SortKey key[SORT_MAX_KEYS];
    uint32_t* hist;  // FS_HIST_WORDS
    Src src;
};

// Block-private histograms of every (key, byte) digit, merged into `hist` once per block.  Equal digits within a warp are
// counted by one shared atomic (match.any), so a constant byte costs one atomic per warp, not 32.
template <typename Src>
__global__ void __launch_bounds__(FS_THREADS) fsort_hist_kernel(const __grid_constant__ FsHistArgs<Src> a) {
    __shared__ uint32_t h[SORT_MAX_KEYS * 8 * 256];
    __shared__ uint32_t s_na[SORT_MAX_KEYS];
    const int lane = threadIdx.x & 31;
    const int nk = a.nk;
    for (int i = threadIdx.x; i < nk * 8 * 256; i += FS_THREADS) h[i] = 0;
    if (threadIdx.x < SORT_MAX_KEYS) s_na[threadIdx.x] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * FS_THREADS;
    for (int64_t r0 = (int64_t)blockIdx.x * FS_THREADS; r0 < a.n; r0 += stride) {
        const int64_t r = r0 + threadIdx.x;
        const unsigned act = __ballot_sync(0xffffffffu, r < a.n);
        if (r >= a.n) continue;
        const int leader = __ffs(act) - 1;
        for (int j = 0; j < nk; j++) {
            bool na;
            const uint64_t w = a.src.word(a.key[j], j, (uint32_t)r, na);
            const unsigned nam = __ballot_sync(act, na);
            if (lane == leader && nam) atomicAdd(&s_na[j], (uint32_t)__popc(nam));
            const int nb = a.key[j].size;
            for (int b = 0; b < nb; b++) {
                const uint32_t d = (uint32_t)(w >> (8 * b)) & 0xFFu;
                const unsigned peers = __match_any_sync(act, d);
                if (lane == __ffs(peers) - 1) atomicAdd(&h[(j * 8 + b) * 256 + d], (uint32_t)__popc(peers));
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nk * 8 * 256; i += FS_THREADS)
        if (h[i]) atomicAdd(&a.hist[i], h[i]);
    if (threadIdx.x < nk && s_na[threadIdx.x]) atomicAdd(&a.hist[SORT_MAX_KEYS * 8 * 256 + threadIdx.x], s_na[threadIdx.x]);
}

template <typename Src>
struct FsPassArgs {
    int64_t n;
    int shift;       // digit = (word >> shift) & 255; -1: the NA-class bit (bit 31 of the row id)
    uint32_t epoch;  // this pass's tag in the look-back words (1, 2, ...; the words start at 0)
    SortKey key;     // FS_IN_COLUMN / FS_IN_GATHER: the key the words are computed from, key 0 of `src`
    const void* w_in;
    const uint32_t* id_in;
    void* w_out;
    uint32_t* id_out;
    unsigned long long* status;  // [tile][digit] look-back words
    unsigned int* tile_counter;  // tiles are numbered in the order their blocks start
    uint32_t base[256];          // first output row of each digit: exclusive scan of the pass's global histogram
    Src src;
};

// One LSD pass over FS_TILE-row tiles.  Warp w of a tile owns its rows [w * 32 * FS_ITEMS, (w + 1) * 32 * FS_ITEMS), item k of
// lane l is row 32 k + l of that range, and items are ranked in row order, so the in-tile rank is stable.  Row ids are 32-bit;
// words are W (uint32_t for keys of <= 4 bytes, uint64_t otherwise).
template <typename W, int MODE, typename Src>
__global__ void __launch_bounds__(FS_THREADS) fsort_pass_kernel(const __grid_constant__ FsPassArgs<Src> a) {
    __shared__ uint32_t s_hist[FS_WARPS][256];  // per-warp digit counts, then each warp's offset inside the digit's tile run
    __shared__ uint32_t s_start[256];           // tile-local first position of each digit
    __shared__ uint32_t s_gofs[256];            // output row of tile-local position p of digit d: s_gofs[d] + p
    __shared__ uint32_t s_wsum[FS_WARPS];
    __shared__ W s_stage[FS_TILE];
    __shared__ uint8_t s_dig[FS_TILE];
    __shared__ uint32_t s_tile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_tile = atomicAdd(a.tile_counter, 1u);
    for (int i = threadIdx.x; i < FS_WARPS * 256; i += FS_THREADS) (&s_hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t t = s_tile;
    const int64_t tile0 = (int64_t)t * FS_TILE;
    const int tile_n = (int)(a.n - tile0 < FS_TILE ? a.n - tile0 : FS_TILE);
    const int64_t row0 = tile0 + warp * (32 * FS_ITEMS) + lane;
    const unsigned lt = (1u << lane) - 1;
    W w[FS_ITEMS];
    uint32_t id[FS_ITEMS], rk[FS_ITEMS];
#pragma unroll
    for (int k = 0; k < FS_ITEMS; k++) {
        const int64_t i = row0 + 32 * k;
        const bool valid = i < a.n;
        uint32_t d = 0;
        w[k] = 0; id[k] = 0;
        if (valid) {
            if (MODE == FS_IN_PAIRS) {
                w[k] = ((const W*)a.w_in)[i];
                id[k] = a.id_in[i];
            } else {
                const uint32_t r = MODE == FS_IN_COLUMN ? (uint32_t)i : (a.id_in[i] & FS_ID_MASK);
                bool na;
                w[k] = (W)a.src.word(a.key, 0, r, na);
                id[k] = r | (sort_class(a.key, na) << 31);
            }
            d = fs_digit(w[k], id[k], a.shift);
        }
        // warp multisplit: m = the valid lanes whose digit equals this lane's
        unsigned m = __ballot_sync(0xffffffffu, valid);
#pragma unroll
        for (int b = 0; b < 8; b++) {
            const unsigned bal = __ballot_sync(0xffffffffu, (d >> b) & 1);
            m &= ((d >> b) & 1) ? bal : ~bal;
        }
        const uint32_t before = valid ? s_hist[warp][d] : 0;
        __syncwarp();
        if (valid && (m & lt) == 0) s_hist[warp][d] = before + __popc(m);
        __syncwarp();
        rk[k] = before + __popc(m & lt);
    }
    __syncthreads();
    // thread d: digit d's warp offsets, tile count, tile-local start and look-back
    const int d = threadIdx.x;
    uint32_t cnt = 0;
#pragma unroll
    for (int q = 0; q < FS_WARPS; q++) { const uint32_t x = s_hist[q][d]; s_hist[q][d] = cnt; cnt += x; }
    const uint32_t inc = warp_inclusive_scan<SumOf<uint32_t>>(cnt);
    if (lane == 31) s_wsum[warp] = inc;
    volatile unsigned long long* status = a.status;
    const unsigned long long tag = (unsigned long long)a.epoch << 34;
    uint32_t excl = 0;
    if (t == 0) {
        status[d] = tag | FS_INCL | cnt;
    } else {
        status[(int64_t)t * 256 + d] = tag | FS_AGG | cnt;
        // Tile j < t drew its number before this one, so its block is running and publishes its aggregate without waiting.
        for (int64_t j = (int64_t)t - 1;;) {
            const unsigned long long s = status[j * 256 + d];
            if ((s >> 34) != a.epoch) continue;
            excl += (uint32_t)s;
            if (s & FS_INCL) break;
            j--;
        }
        status[(int64_t)t * 256 + d] = tag | FS_INCL | (excl + cnt);
    }
    __syncthreads();
    uint32_t wpre = 0;
    for (int q = 0; q < warp; q++) wpre += s_wsum[q];
    const uint32_t start = wpre + inc - cnt;
    s_start[d] = start;
    s_gofs[d] = a.base[d] + excl - start;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FS_ITEMS; k++) {
        if (row0 + 32 * k < a.n) {
            const uint32_t dk = fs_digit(w[k], id[k], a.shift);
            rk[k] += s_start[dk] + s_hist[warp][dk];
            s_stage[rk[k]] = w[k];
            s_dig[rk[k]] = (uint8_t)dk;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < tile_n; i += FS_THREADS) ((W*)a.w_out)[s_gofs[s_dig[i]] + (uint32_t)i] = s_stage[i];
    __syncthreads();
    uint32_t* s_id = (uint32_t*)s_stage;
#pragma unroll
    for (int k = 0; k < FS_ITEMS; k++)
        if (row0 + 32 * k < a.n) s_id[rk[k]] = id[k];
    __syncthreads();
    for (int i = threadIdx.x; i < tile_n; i += FS_THREADS) a.id_out[s_gofs[s_dig[i]] + (uint32_t)i] = s_id[i];
}

struct FsGatherArgs {
    int64_t n;
    const uint32_t* ids;  // the permutation (bit 31 ignored); nullptr: identity
    FsLayout lay;
    void* out[SORT_MAX_COLS];
    uint8_t* out_vb[SORT_MAX_COLS];
    FsChunks ch;
};

__global__ void __launch_bounds__(256) fsort_gather_kernel(const __grid_constant__ FsGatherArgs a) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
        const uint32_t r = a.ids ? (a.ids[i] & FS_ID_MASK) : (uint32_t)i;
        const char* chunk = a.ch.p[r >> FS_CHUNK_LOG];
        const int64_t off = r & (FS_CHUNK - 1);
        for (int c = 0; c < a.lay.sc.n_cols; c++) {
            copy_cell(a.out[c], i, chunk + a.lay.coff[c], off, ctype_size(a.lay.sc.ctype[c]));
            if (a.lay.voff[c] >= 0) a.out_vb[c][i] = (uint8_t)chunk[a.lay.voff[c] + off];
        }
    }
}

// ---- the full sort's sharded form (streaming/sort.py init_sharded_sort_state): every rank sorts its rows, samples them, counts
// the rows below the chosen splitters and sends each rank its slice; the receiver's store holds the runs it got, one per source
// rank, back to back, and merges them instead of sorting ----
//
//   fsort_sample_kernel       sample i of a finished sort is its output row q_i = floor(i n / s): per key (NA class, radix word),
//                             then (rank, q_i), one uint64 each.
//   fsort_count_below_kernel  per splitter (a sample record) the number of output rows whose (key, rank, row) tuple is below it,
//                             by binary search over the sorted rows.
//   fsort_merge_kernel        one pairwise merge-path round over runs of row ids (merge_path_items, as the top-k's reduce);
//                             ceil(log2 P) rounds merge P runs.  Key words are read through FsChunkSrc; two rows that tie on
//                             every key keep their store order, which is (source rank, position).
constexpr int FS_MERGE_ITEMS = 16;

// The key columns of a finished state's output: rows [0, n) of key j at data[j], its validity bitmap at bitmap[j] (nullptr: none).
struct FsOutKeys {
    int nk;
    int64_t n, rank;
    SortKey key[SORT_MAX_KEYS];
    const void* data[SORT_MAX_KEYS];
    const uint8_t* bitmap[SORT_MAX_KEYS];
    __device__ __forceinline__ uint64_t word(int j, int64_t q, uint32_t& cls) const {
        bool na = !bit_valid(bitmap[j], q);
        const uint64_t w = sort_word(key[j], load_bits(data[j], key[j].size, q), na);
        cls = sort_class(key[j], na);
        return w;
    }
};

__global__ void fsort_sample_kernel(const __grid_constant__ FsOutKeys a, int64_t s, uint64_t* __restrict__ rec) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s) return;
    const int64_t q = i * a.n / s;  // i n < 2^31 * 2^31
    uint64_t* r = rec + i * (2 * a.nk + 2);
    for (int j = 0; j < a.nk; j++) {
        uint32_t cls;
        r[2 * j + 1] = a.word(j, q, cls);
        r[2 * j] = cls;
    }
    r[2 * a.nk] = (uint64_t)a.rank;
    r[2 * a.nk + 1] = (uint64_t)q;
}

__global__ void fsort_count_below_kernel(const __grid_constant__ FsOutKeys a, const uint64_t* __restrict__ spl, int64_t n_spl,
                                         int64_t* __restrict__ counts) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_spl) return;
    const uint64_t* t = spl + k * (2 * a.nk + 2);
    // row q is below the splitter: rows are sorted, so this holds for a prefix of [0, n)
    auto below = [&](int64_t q) {
        for (int j = 0; j < a.nk; j++) {
            uint32_t cls;
            const uint64_t w = a.word(j, q, cls);
            if (cls != t[2 * j]) return cls < t[2 * j];
            if (w != t[2 * j + 1]) return w < t[2 * j + 1];
        }
        if ((uint64_t)a.rank != t[2 * a.nk]) return (uint64_t)a.rank < t[2 * a.nk];
        return (uint64_t)q < t[2 * a.nk + 1];
    };
    int64_t lo = 0, hi = a.n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (below(mid)) lo = mid + 1; else hi = mid;
    }
    counts[k] = lo;
}

// Two adjacent runs of one merge round: A is rows [off, off + la) of the round's input, B the lb rows after it; they become rows
// [off, off + la + lb) of its output, handled by threads chunk0 .. chunk0 + ceil((la + lb) / FS_MERGE_ITEMS) - 1.
struct FsMergePair { int64_t off, la, lb, chunk0; };

struct FsMergeArgs {
    int nk;
    SortKey key[SORT_MAX_KEYS];
    FsChunkSrc src;
    const FsMergePair* pair;
    int64_t n_pairs, n_chunks;
    const uint32_t* in;  // nullptr: the identity (the first round reads the store order)
    uint32_t* out;
};

__global__ void __launch_bounds__(256) fsort_merge_kernel(const __grid_constant__ FsMergeArgs a) {
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_chunks) return;
    int64_t lo = 0, hi = a.n_pairs - 1;  // the last pair whose first chunk is <= c: a pair without rows owns no chunk
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (a.pair[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    const FsMergePair p = a.pair[lo];
    const int64_t d0 = (c - p.chunk0) * FS_MERGE_ITEMS, bo = p.off + p.la;
    const uint32_t* in = a.in;
    auto A = [&](int64_t i) { return in ? in[p.off + i] : (uint32_t)(p.off + i); };
    auto B = [&](int64_t j) { return in ? in[bo + j] : (uint32_t)(bo + j); };
    auto b_first = [&](uint32_t b, uint32_t x) {
#pragma unroll
        for (int j = 0; j < SORT_MAX_KEYS; j++) {
            if (j < a.nk) {
                bool nb, nx;
                const uint64_t wb = a.src.word(a.key[j], j, b, nb), wx = a.src.word(a.key[j], j, x, nx);
                const uint32_t cb = sort_class(a.key[j], nb), cx = sort_class(a.key[j], nx);
                if (cb != cx) return cb < cx;
                if (wb != wx) return wb < wx;
            }
        }
        return false;
    };
    merge_path_items<FS_MERGE_ITEMS>(A, p.la, B, p.lb, d0, p.la + p.lb, a.out + p.off, b_first);
}

static_assert(FS_THREADS == 256, "fsort_pass_kernel: one thread per digit");

template <typename W, typename Src>
void launch_fsort_pass(int mode, int64_t n_tiles, const FsPassArgs<Src>& a, cudaStream_t st) {
    const unsigned g = (unsigned)n_tiles;
    if (mode == FS_IN_PAIRS) fsort_pass_kernel<W, FS_IN_PAIRS><<<g, FS_THREADS, 0, st>>>(a);
    else if (mode == FS_IN_COLUMN) fsort_pass_kernel<W, FS_IN_COLUMN><<<g, FS_THREADS, 0, st>>>(a);
    else fsort_pass_kernel<W, FS_IN_GATHER><<<g, FS_THREADS, 0, st>>>(a);
}

// The LSD radix sort of rows [0, n) by nk keys read from `src`: the digit histograms (one kernel), the pass plan, then one
// fsort_pass_kernel per planned digit.  Plan: least significant key first; per key its byte digits from the lowest, then its
// NA class when may_na[j].  A digit that takes one value on every row leaves the order as it is: that pass is skipped.
// Returns the permutation in ibuf[0] or ibuf[1] (bit 31 of an entry is the NA-class bit, not part of the row id), or nullptr
// when no pass ran (the identity).  Word buffers and look-back words are freed on return.
template <typename Src>
const uint32_t* fsort_rows(const Src& src, const SortKey* keys, const bool* may_na, int nk, int64_t n, DevBuf (&ibuf)[2], int hist_grid,
                           cudaStream_t stream, int64_t& passes_run, int64_t& passes_skipped) {
    DevBuf d_hist;
    d_hist.alloc(FS_HIST_WORDS * 4);
    B200_CUDA(cudaMemsetAsync(d_hist.p, 0, FS_HIST_WORDS * 4, stream));
    FsHistArgs<Src> ha{};
    ha.n = n; ha.nk = nk; ha.hist = d_hist.as<uint32_t>(); ha.src = src;
    std::copy(keys, keys + nk, ha.key);
    fsort_hist_kernel<<<hist_grid, FS_THREADS, 0, stream>>>(ha);
    B200_CUDA(cudaGetLastError());
    auto* h = (uint32_t*)pinned_acquire(FS_HIST_WORDS * 4);
    B200_CUDA(cudaMemcpyAsync(h, d_hist.p, FS_HIST_WORDS * 4, cudaMemcpyDeviceToHost, stream));
    B200_CUDA(cudaStreamSynchronize(stream));
    struct Pass { int key, shift; uint32_t base[256]; };
    std::vector<Pass> plan;
    for (int j = nk - 1; j >= 0; j--) {
        for (int b = 0; b < keys[j].size; b++) {
            const uint32_t* c = h + (j * 8 + b) * 256;
            if (std::any_of(c, c + 256, [&](uint32_t x) { return (int64_t)x == n; })) { passes_skipped++; continue; }
            Pass p{j, 8 * b, {}};
            for (uint32_t d = 0, s = 0; d < 256; s += c[d], d++) p.base[d] = s;
            plan.push_back(p);
        }
        if (may_na[j]) {
            const int64_t na = h[SORT_MAX_KEYS * 8 * 256 + j];
            if (na == 0 || na == n) { passes_skipped++; continue; }
            const int64_t class0 = keys[j].na_last ? n - na : na;  // rows whose class bit is 0
            Pass p{j, -1, {}};
            for (int d = 1; d < 256; d++) p.base[d] = (uint32_t)class0;
            plan.push_back(p);
        }
    }
    pinned_release(h, FS_HIST_WORDS * 4);
    passes_run += (int64_t)plan.size();
    if (plan.empty()) return nullptr;
    DevBuf wbuf[2], status, counters;
    size_t wb = 4;
    for (const Pass& p : plan) if (keys[p.key].size > 4) wb = 8;
    for (int b = 0; b < 2; b++) { wbuf[b].alloc((size_t)n * wb); ibuf[b].alloc((size_t)n * 4); }
    const int64_t n_tiles = (n + FS_TILE - 1) / FS_TILE;
    status.alloc((size_t)n_tiles * 256 * 8);
    counters.alloc(plan.size() * 4);
    B200_CUDA(cudaMemsetAsync(status.p, 0, (size_t)n_tiles * 256 * 8, stream));
    B200_CUDA(cudaMemsetAsync(counters.p, 0, plan.size() * 4, stream));
    const uint32_t* ids = nullptr;
    int cur_buf = -1, prev_key = -1;
    for (size_t q = 0; q < plan.size(); q++) {
        const Pass& p = plan[q];
        const int mode = p.key == prev_key ? FS_IN_PAIRS : ids ? FS_IN_GATHER : FS_IN_COLUMN;
        const int ob = cur_buf == 0 ? 1 : 0;
        FsPassArgs<Src> a{};
        a.n = n; a.shift = p.shift; a.epoch = (uint32_t)q + 1;
        a.key = keys[p.key]; a.src = src.for_key(p.key);
        a.w_in = cur_buf >= 0 ? wbuf[cur_buf].p : nullptr; a.id_in = ids;
        a.w_out = wbuf[ob].p; a.id_out = ibuf[ob].as<uint32_t>();
        a.status = status.as<unsigned long long>(); a.tile_counter = counters.as<unsigned int>() + q;
        std::copy(p.base, p.base + 256, a.base);
        if (keys[p.key].size > 4) launch_fsort_pass<uint64_t>(mode, n_tiles, a, stream);
        else launch_fsort_pass<uint32_t>(mode, n_tiles, a, stream);
        B200_CUDA(cudaGetLastError());
        cur_buf = ob; ids = ibuf[ob].as<uint32_t>(); prev_key = p.key;
    }
    return ids;
}

const uint32_t* radix_sort_columns(int n_keys, const void* const* data, const SortKey* keys, int64_t n, DevBuf (&ids)[2], cudaStream_t st,
                                   int64_t* passes_run) {
    B200_REQUIRE(n_keys >= 1 && n_keys <= SORT_MAX_KEYS && n <= FS_MAX_ROWS, "internal: radix_sort_columns: 1 to 4 keys, at most 2^31 rows");
    if (n == 0) return nullptr;
    FsArraySrc src{};
    bool may_na[SORT_MAX_KEYS] = {};
    for (int j = 0; j < n_keys; j++) src.data[j] = data[j];
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + FS_THREADS - 1) / FS_THREADS, (int64_t)num_sms(dev) * 8));
    int64_t run = 0, skipped = 0;
    const uint32_t* perm = fsort_rows(src, keys, may_na, n_keys, n, ids, grid, st, run, skipped);
    if (passes_run) *passes_run += run;
    return perm;
}

// ---- host state: a form consumes rows and at is_last points the output views at its sorted rows; the base checks batches,
// packs the output's validity bitmaps and hands out output batches ----
struct SortState {
    int device, sms;
    cudaStream_t stream;
    SortSchema sc{};
    int arr_type[SORT_MAX_COLS];
    int64_t output_batch_size;
    int64_t rows_consumed = 0;  // metric 0
    bool finished = false;
    // Output columns: the n_cols input columns, then any columns a form computes (of type sc.ctype[c] and array type
    // arr_type[c]; the window's function columns).
    int n_out_cols;
    // output views, set by the form's finish_rows: rows [0, n_out) of column c at out_data[c], for a nullable column one validity
    // byte per row at out_vb[c]
    char* out_data[SORT_MAX_COLS]{};
    uint8_t* out_vb[SORT_MAX_COLS]{};
    int64_t n_out = 0, out_cursor = 0;
    DevBuf d_bitmaps;
    std::vector<uint32_t*> out_bitmap;

    SortState(const int8_t* c_types, const int8_t* arr_types, int n_arrs, int n_keys, const int32_t* asc, const int32_t* na_last,
              int64_t obs, int dev, cudaStream_t st)
        : device(dev), stream(st), output_batch_size(obs), n_out_cols(n_arrs) {
        B200_REQUIRE(n_keys >= 1 && n_keys <= SORT_MAX_KEYS, "b200 sort: 1 to 4 sort keys");
        B200_REQUIRE(n_arrs >= n_keys && n_arrs <= SORT_MAX_COLS, "b200 sort: keys are the first n_keys of at most 32 columns");
        B200_REQUIRE(c_types && arr_types && asc && na_last, "b200 sort: null argument");
        sc.n_keys = n_keys; sc.n_cols = n_arrs;
        for (int c = 0; c < n_arrs; c++) {
            B200_REQUIRE(ctype_size(c_types[c]) > 0, "b200 sort: unsupported column dtype (fixed-width numeric, bool and temporal columns only)");
            B200_REQUIRE(arr_types[c] == ARR_NUMPY || arr_types[c] == ARR_NULLABLE, "b200 sort: unsupported array type");
            sc.ctype[c] = c_types[c]; arr_type[c] = arr_types[c];
        }
        for (int j = 0; j < n_keys; j++) sc.key[j] = SortKey{sc.ctype[j], ctype_size(sc.ctype[j]), asc[j] ? 0 : 1, na_last[j] ? 1 : 0};
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        sms = num_sms(device);
    }
    // The caller selects the state's device and stream first (b200_delete_sort_state): both forms' buffers go back to its pool.
    virtual ~SortState() = default;

    // Rows [0, n) of a checked batch, arriving with indices rows_consumed, rows_consumed + 1, ...
    virtual void consume_rows(const b200_table* t, int64_t n) = 0;
    // At is_last: sort, then set n_out, out_data and out_vb.  Validity bytes the form allocates for its output go in vbytes (one
    // slot per output column), which is freed once the bitmaps are packed.
    virtual void finish_rows(std::vector<DevBuf>& vbytes) = 0;
    // Metric 0 to 9; a metric the form does not keep reads 0.
    virtual int64_t metric(int which) const = 0;

    int grid_for(int64_t items, int per_block) const { return (int)std::max<int64_t>(1, std::min<int64_t>((items + per_block - 1) / per_block, (int64_t)sms * 8)); }

    void consume(const b200_table* t) {
        B200_REQUIRE(!finished, "b200 sort: batch consumed after is_last");
        B200_REQUIRE(t->n_cols == sc.n_cols, "b200 sort: the batch's column count differs from the state's schema");
        for (int c = 0; c < sc.n_cols; c++)
            B200_REQUIRE(t->cols[c].c_type == sc.ctype[c] && t->cols[c].arr_type == arr_type[c],
                         "b200 sort: a batch's column types differ from the state's schema");
        const int64_t n = t->n_rows;
        if (n > 0) B200_REQUIRE(t->device == device, "b200 sort: batches must be resident on the state's device (stage host batches first)");
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        consume_rows(t, n);
        rows_consumed += n;
    }

    void finish() {
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        std::vector<DevBuf> vbytes(n_out_cols);
        finish_rows(vbytes);
        finished = true;
        int n_nullable = 0;
        for (int c = 0; c < n_out_cols; c++) n_nullable += arr_type[c] == ARR_NULLABLE;
        const int64_t words = (n_out + 31) / 32 + 2;
        d_bitmaps.alloc((size_t)std::max(1, n_nullable) * words * 4);
        B200_CUDA(cudaMemsetAsync(d_bitmaps.p, 0, d_bitmaps.bytes, stream));
        out_bitmap.assign(n_out_cols, nullptr);
        for (int c = 0, k = 0; c < n_out_cols; c++) {
            if (arr_type[c] != ARR_NULLABLE) continue;
            out_bitmap[c] = d_bitmaps.as<uint32_t>() + (k++) * words;
            if (n_out > 0) launch_pack_bitmap(out_vb[c], n_out, out_bitmap[c], grid_for(n_out, 256), stream);
        }
        B200_CUDA(cudaGetLastError());
        vbytes.clear();
        B200_CUDA(cudaStreamSynchronize(stream));
    }

    int produce(b200_table* out, int32_t* out_is_last, bool produce_output) {
        B200_REQUIRE(finished, "b200 sort: output requested before the last batch was consumed");
        B200_REQUIRE(out->cols != nullptr, "b200 sort: out->cols must point to one descriptor per column");
        int64_t bs = output_batch_size > 0 ? output_batch_size : n_out;
        if (bs % 32 != 0 && bs < n_out) bs = (bs + 31) & ~31ll;  // validity bitmaps are sliced at word granularity
        const int64_t rows = produce_output ? std::min(bs, n_out - out_cursor) : 0;
        out->n_rows = rows; out->n_cols = n_out_cols; out->device = device;
        for (int c = 0; c < n_out_cols; c++) {
            b200_column& col = out->cols[c];
            col.data = out_data[c] + out_cursor * ctype_size(sc.ctype[c]);
            col.validity = out_bitmap[c] ? (uint8_t*)out_bitmap[c] + out_cursor / 8 : nullptr;
            col.length = rows; col.c_type = sc.ctype[c]; col.arr_type = arr_type[c];
        }
        out_cursor += rows;
        *out_is_last = out_cursor >= n_out ? 1 : 0;
        return 0;
    }
};

// ORDER BY ... LIMIT limit OFFSET offset.
struct TopkState : SortState {
    int64_t offset, K, cap;
    // two store buffers (cur = the one the filter appends to) and their memory
    std::vector<DevBuf> mem[2];
    TkStore store[2]{};
    int cur = 0;
    DevBuf perm[2], d_cursor, d_cutoff;
    unsigned long long* h_count = nullptr;
    int64_t held = 0;         // sorted rows at the front of the current store (<= K)
    int64_t count_bound = 0;  // upper bound on the store count: last count read + rows launched since
    bool has_cutoff = false;
    int64_t rows_admitted = 0, admitted_after_cutoff = 0, reduce_steps = 0, count_reads = 0, filter_launches = 0;

    TopkState(int64_t limit, int64_t offset_, const int8_t* c_types, const int8_t* arr_types, int n_arrs, int n_keys,
              const int32_t* asc, const int32_t* na_last, int64_t obs, int dev, cudaStream_t st)
        : SortState(c_types, arr_types, n_arrs, n_keys, asc, na_last, obs, dev, st), offset(offset_), K(limit + offset_),
          cap(std::max<int64_t>(2 * K, TK_MIN_CAP)) {
        h_count = (unsigned long long*)pinned_acquire(8);
        d_cursor.alloc(8); d_cutoff.alloc(sizeof(TkCutoff));
        B200_CUDA(cudaMemsetAsync(d_cursor.p, 0, 8, stream));
        B200_CUDA(cudaMemsetAsync(d_cutoff.p, 0, sizeof(TkCutoff), stream));
        if (K == 0) return;  // nothing is ever kept: no store
        for (int b = 0; b < 2; b++) {
            auto take = [&](size_t bytes) { mem[b].emplace_back(); mem[b].back().alloc(bytes); return mem[b].back().p; };
            TkStore& s = store[b];
            for (int j = 0; j < n_keys; j++) s.w[j] = (uint64_t*)take(cap * 8);
            s.cls = (uint8_t*)take(cap);
            s.seq = (int64_t*)take(cap * 8);
            for (int c = 0; c < n_arrs; c++) {
                s.data[c] = take(cap * ctype_size(sc.ctype[c]));
                s.vb[c] = arr_type[c] == ARR_NULLABLE ? (uint8_t*)take(cap) : nullptr;
            }
            perm[b].alloc(cap * 4);
        }
    }
    ~TopkState() override { pinned_release(h_count, 8); }

    int64_t read_count() {
        B200_CUDA(cudaMemcpyAsync(h_count, d_cursor.p, 8, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        count_reads++;
        count_bound = (int64_t)*h_count;
        return count_bound;
    }

    // Sorts held rows + candidates, keeps the first K in the other buffer and writes the cutoff.  n: the store count, if known.
    void reduce(int64_t n = -1) {
        if (n < 0) n = read_count();
        reduce_steps++;
        rows_admitted += n - held;
        if (has_cutoff) admitted_after_cutoff += n - held;
        if (n > held) {
            uint32_t* a = perm[0].as<uint32_t>();
            uint32_t* b = perm[1].as<uint32_t>();
            const TkStore& s = store[cur];
            topk_block_sort_kernel<<<(unsigned)((n + TK_SORT_TILE - 1) / TK_SORT_TILE), TK_SORT_THREADS, 0, stream>>>(s, sc.n_keys, n, K, a);
            B200_CUDA(cudaGetLastError());
            for (int64_t w = TK_SORT_TILE; w < n; w *= 2) {
                const int64_t n_pairs = (n + 2 * w - 1) / (2 * w);
                const int64_t chunks = (std::min(2 * w, K) + TK_MERGE_ITEMS - 1) / TK_MERGE_ITEMS;
                const int64_t threads = n_pairs * chunks;
                topk_merge_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(s, sc.n_keys, n, K, w, chunks, n_pairs, a, b);
                B200_CUDA(cudaGetLastError());
                std::swap(a, b);
            }
            const int64_t m = std::min(n, K);
            topk_gather_kernel<<<grid_for(m, 256), 256, 0, stream>>>(s, store[cur ^ 1], sc, a, m, K, d_cutoff.as<TkCutoff>(),
                                                                    d_cursor.as<unsigned long long>());
            B200_CUDA(cudaGetLastError());
            cur ^= 1;
            held = m;
        }
        count_bound = held;
        if (held == K) has_cutoff = true;
    }

    void consume_rows(const b200_table* t, int64_t n) override {
        if (K == 0 || n == 0) return;
        TkFilterArgs a{};
        a.sc = sc;
        a.seq_base = rows_consumed;
        for (int c = 0; c < sc.n_cols; c++) { a.in_data[c] = t->cols[c].data; a.in_valid[c] = t->cols[c].validity; }
        a.cutoff = d_cutoff.as<TkCutoff>();
        a.cursor = d_cursor.as<unsigned long long>();
        for (int64_t r0 = 0; r0 < n;) {
            int64_t r = n - r0;
            if (count_bound + r > cap) {
                read_count();
                if (count_bound + r > cap && count_bound > held) reduce(count_bound);
                r = std::min(r, cap - count_bound);
            }
            a.row0 = r0; a.row1 = r0 + r;
            a.st = store[cur];
            topk_filter_kernel<<<grid_for(r, TK_TILE), TK_THREADS, 0, stream>>>(a);
            B200_CUDA(cudaGetLastError());
            filter_launches++;
            count_bound += r;
            r0 += r;
            if (!has_cutoff && count_bound >= K) reduce();  // before a cutoff every row is admitted: the count is exactly count_bound
        }
    }

    void finish_rows(std::vector<DevBuf>&) override {
        if (K > 0) reduce();
        n_out = std::max<int64_t>(0, held - offset);
        const TkStore& s = store[cur];
        for (int c = 0; c < sc.n_cols; c++) {
            // K = 0 has no store: its zero output rows still carry a non-null data pointer
            out_data[c] = K == 0 ? d_cutoff.as<char>() : (char*)s.data[c] + offset * ctype_size(sc.ctype[c]);
            out_vb[c] = s.vb[c] ? s.vb[c] + offset : nullptr;
        }
    }

    int64_t metric(int which) const override {
        const int64_t m[10] = {rows_consumed, rows_admitted, reduce_steps, count_reads, filter_launches, admitted_after_cutoff, cap, 0, 0, 0};
        return m[which];
    }
};

// ORDER BY without LIMIT.
struct FullSortState : SortState {
    FsLayout lay{};
    int64_t chunk_bytes = 0, n_chunks = 0, passes_run = 0, passes_skipped = 0;
    std::vector<DevBuf> chunks, out_mem;

    FullSortState(const int8_t* c_types, const int8_t* arr_types, int n_arrs, int n_keys, const int32_t* asc, const int32_t* na_last,
                  int64_t obs, int dev, cudaStream_t st)
        : SortState(c_types, arr_types, n_arrs, n_keys, asc, na_last, obs, dev, st) {
        lay.sc = sc;
        for (int c = 0; c < n_arrs; c++) {
            lay.coff[c] = chunk_bytes;
            chunk_bytes += FS_CHUNK * ctype_size(sc.ctype[c]);
        }
        for (int c = 0; c < n_arrs; c++) {
            lay.voff[c] = arr_type[c] == ARR_NULLABLE ? chunk_bytes : -1;
            if (arr_type[c] == ARR_NULLABLE) chunk_bytes += FS_CHUNK;
        }
    }

    // Rows [0, n) of the batch go to rows [rows_consumed, rows_consumed + n) of the chunk store.
    void consume_rows(const b200_table* t, int64_t n) override {
        B200_REQUIRE(n <= FS_MAX_ROWS - rows_consumed, "b200 sort: a full sort holds at most 2^31 rows (32-bit row ids)");
        FsAppendArgs a{};
        a.lay = lay;
        for (int c = 0; c < sc.n_cols; c++) { a.in_data[c] = t->cols[c].data; a.in_valid[c] = t->cols[c].validity; }
        for (int64_t i = 0; i < n;) {
            const int64_t g = rows_consumed + i, k = g >> FS_CHUNK_LOG, off = g & (FS_CHUNK - 1);
            const int64_t r = std::min(n - i, FS_CHUNK - off);
            if (k == (int64_t)chunks.size()) {
                chunks.emplace_back();
                chunks.back().alloc((size_t)chunk_bytes);
                n_chunks++;
            }
            a.src0 = i; a.n = r; a.dst0 = off; a.chunk = chunks[k].as<char>();
            fsort_append_kernel<<<grid_for(r, 256), 256, 0, stream>>>(a);
            B200_CUDA(cudaGetLastError());
            i += r;
        }
    }

    FsChunkSrc key_src(const FsChunks& ch) const {
        FsChunkSrc src{};
        src.ch = ch;
        for (int j = 0; j < sc.n_keys; j++) { src.coff[j] = lay.coff[j]; src.voff[j] = lay.voff[j]; }
        return src;
    }

    // The sorted order of the n > 0 stored rows: the digit histograms, the pass plan and the digit passes.  Returns the
    // permutation in ibuf (bit 31 of an entry is not part of the row id), or nullptr for the identity.
    virtual const uint32_t* sorted_ids(const FsChunks& ch, int64_t n, DevBuf (&ibuf)[2]) {
        bool may_na[SORT_MAX_KEYS] = {};
        for (int j = 0; j < sc.n_keys; j++) may_na[j] = arr_type[j] == ARR_NULLABLE || ctype_is_float(sc.ctype[j]);
        return fsort_rows(key_src(ch), sc.key, may_na, sc.n_keys, n, ibuf, grid_for(n, FS_THREADS), stream, passes_run, passes_skipped);
    }

    // The sorted order, then the gather into the output store (out_mem; the validity bytes of nullable column c go to vbytes[c]).
    // Chunks, pair buffers and look-back words are freed on return.
    void finish_rows(std::vector<DevBuf>& vbytes) override {
        const int64_t n = rows_consumed;
        FsChunks ch{};
        for (size_t k = 0; k < chunks.size(); k++) ch.p[k] = chunks[k].as<char>();
        DevBuf ibuf[2];
        const uint32_t* ids = n > 0 ? sorted_ids(ch, n, ibuf) : nullptr;  // the permutation; nullptr: identity
        FsGatherArgs ga{};
        ga.n = n; ga.ids = ids; ga.lay = lay; ga.ch = ch;
        out_mem.resize(sc.n_cols);
        for (int c = 0; c < sc.n_cols; c++) {
            out_mem[c].alloc((size_t)n * ctype_size(sc.ctype[c]));
            ga.out[c] = out_data[c] = out_mem[c].as<char>();
            if (arr_type[c] == ARR_NULLABLE) { vbytes[c].alloc((size_t)n); ga.out_vb[c] = out_vb[c] = vbytes[c].as<uint8_t>(); }
        }
        if (n > 0) fsort_gather_kernel<<<grid_for(n, 256), 256, 0, stream>>>(ga);
        B200_CUDA(cudaGetLastError());
        n_out = n;
        chunks.clear();  // the rows now live in the output store
    }

    int64_t metric(int which) const override {
        const int64_t m[10] = {rows_consumed, 0, 0, 0, 0, 0, n_chunks * FS_CHUNK, passes_run, passes_skipped, 0};
        return m[which];
    }

    // The sorted key columns of a finished state, tagged with the caller's rank.
    FsOutKeys out_keys(int64_t rank) const {
        FsOutKeys k{};
        k.nk = sc.n_keys; k.n = n_out; k.rank = rank;
        for (int j = 0; j < sc.n_keys; j++) { k.key[j] = sc.key[j]; k.data[j] = out_data[j]; k.bitmap[j] = (const uint8_t*)out_bitmap[j]; }
        return k;
    }

    // s sample records of the sorted rows (fsort_sample_kernel) into rec (host, s (2 n_keys + 2) words).
    void sample(int64_t s, int64_t rank, uint64_t* rec) {
        B200_REQUIRE(finished, "b200 sort: samples are taken after the last batch was consumed");
        B200_REQUIRE(s >= 0 && s <= n_out && rec, "b200 sort: 0 <= samples <= rows, and a record buffer");
        if (s == 0) return;
        B200_CUDA(cudaSetDevice(device));
        const size_t bytes = (size_t)s * (2 * sc.n_keys + 2) * 8;
        DevBuf d; d.alloc(bytes);
        fsort_sample_kernel<<<(unsigned)((s + 255) / 256), 256, 0, stream>>>(out_keys(rank), s, d.as<uint64_t>());
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaMemcpyAsync(rec, d.p, bytes, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
    }

    // counts[k] = the sorted rows whose (key, rank, row) tuple is below splitter record k (fsort_count_below_kernel); host arrays.
    void count_below(const uint64_t* spl, int64_t n_spl, int64_t rank, int64_t* counts) {
        B200_REQUIRE(finished, "b200 sort: splitters are counted after the last batch was consumed");
        B200_REQUIRE(n_spl >= 0 && (n_spl == 0 || (spl && counts)), "b200 sort: null splitter or count buffer");
        if (n_spl == 0) return;
        B200_CUDA(cudaSetDevice(device));
        const size_t bytes = (size_t)n_spl * (2 * sc.n_keys + 2) * 8;
        DevBuf d_spl, d_counts;
        d_spl.alloc(bytes); d_counts.alloc((size_t)n_spl * 8);
        B200_CUDA(cudaMemcpyAsync(d_spl.p, spl, bytes, cudaMemcpyHostToDevice, stream));
        fsort_count_below_kernel<<<(unsigned)((n_spl + 127) / 128), 128, 0, stream>>>(out_keys(rank), d_spl.as<uint64_t>(), n_spl,
                                                                                        d_counts.as<int64_t>());
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaMemcpyAsync(counts, d_counts.p, (size_t)n_spl * 8, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
    }
};

// A full sort whose input is n_runs runs of the given lengths, consumed back to back, each already in the state's sorted order:
// is_last merges them (fsort_merge_kernel) instead of sorting.  Rows that tie on every key keep their store order.
struct MergeSortState : FullSortState {
    std::vector<int64_t> runs;

    MergeSortState(const int64_t* run_lengths, int n_runs, const int8_t* c_types, const int8_t* arr_types, int n_arrs, int n_keys,
                   const int32_t* asc, const int32_t* na_last, int64_t obs, int dev, cudaStream_t st)
        : FullSortState(c_types, arr_types, n_arrs, n_keys, asc, na_last, obs, dev, st), runs(run_lengths, run_lengths + n_runs) {}

    const uint32_t* sorted_ids(const FsChunks& ch, int64_t n, DevBuf (&ibuf)[2]) override {
        int64_t total = 0;
        std::vector<int64_t> len;
        for (int64_t r : runs) { total += r; if (r > 0) len.push_back(r); }
        B200_REQUIRE(total == n, "b200 sort: the rows consumed differ from the sum of the run lengths");
        if (len.size() <= 1) return nullptr;
        // every round's pairs, uploaded at once
        std::vector<FsMergePair> pairs;
        std::vector<size_t> first;
        std::vector<int64_t> n_chunks;
        while (len.size() > 1) {
            first.push_back(pairs.size());
            std::vector<int64_t> next;
            int64_t off = 0, c = 0;
            for (size_t p = 0; p < len.size(); p += 2) {
                const int64_t la = len[p], lb = p + 1 < len.size() ? len[p + 1] : 0;
                pairs.push_back(FsMergePair{off, la, lb, c});
                c += (la + lb + FS_MERGE_ITEMS - 1) / FS_MERGE_ITEMS;
                off += la + lb;
                next.push_back(la + lb);
            }
            n_chunks.push_back(c);
            len.swap(next);
        }
        first.push_back(pairs.size());
        DevBuf d_pairs;
        d_pairs.alloc(pairs.size() * sizeof(FsMergePair));
        B200_CUDA(cudaMemcpyAsync(d_pairs.p, pairs.data(), pairs.size() * sizeof(FsMergePair), cudaMemcpyHostToDevice, stream));
        for (int b = 0; b < 2; b++) ibuf[b].alloc((size_t)n * 4);
        FsMergeArgs a{};
        a.nk = sc.n_keys;
        std::copy(sc.key, sc.key + sc.n_keys, a.key);
        a.src = key_src(ch);
        const uint32_t* ids = nullptr;
        for (size_t r = 0; r + 1 < first.size(); r++) {
            a.pair = d_pairs.as<FsMergePair>() + first[r];
            a.n_pairs = (int64_t)(first[r + 1] - first[r]);
            a.n_chunks = n_chunks[r];
            a.in = ids;
            a.out = ibuf[r & 1].as<uint32_t>();
            fsort_merge_kernel<<<(unsigned)((a.n_chunks + 255) / 256), 256, 0, stream>>>(a);
            B200_CUDA(cudaGetLastError());
            ids = a.out;
        }
        B200_CUDA(cudaStreamSynchronize(stream));  // the pair list lives in host memory until its copy has run
        return ids;
    }
};

// ---- window (ranking functions OVER (PARTITION BY p ... ORDER BY o ...)): a full sort by (p ascending NA last, o), then scans
// over the sorted key columns ----
//
//   window_bounds_kernel  one pass over the sorted key columns: position i starts a partition when a partition key's (NA class,
//                         radix word) differs from position i - 1's, and a peer group when any key does (i = 0 starts both).
//                         The row at i - 1 is the tile's one-row halo.  Writes one flag byte per position and per TILE_ROWS-row
//                         tile the reduction of the scan values below, plus the tile's partition-start count.
//   tile_carry_kernel     one block (common.cuh): the exclusive scan of the tile values, and their total (the partition count).
//   window_ends_kernel    scan of the flags seeded by the tile prefix: per position the partition start P (a max-scan of the
//                         start positions), the peer start Q (a max-scan) and D, the number of peer starts up to the position.
//                         The last row of a partition writes its size into slot P and the last row of a peer group its end into
//                         slot Q; a partition's first row writes D into slot P.  No reverse scan is needed.
//   window_eval_kernel    the same scan again, then every requested function per position.
// Row positions are below 2^31 (the full sort's limit), so positions, sizes and counts are uint32.
enum { WN_ROW_NUMBER = 0, WN_RANK = 1, WN_DENSE_RANK = 2, WN_PERCENT_RANK = 3, WN_CUME_DIST = 4, WN_NTILE = 5 };
constexpr uint8_t WN_PART = 1, WN_PEER = 2;  // a partition start is also a peer-group start

// Scan value of a position: (partition start, peer start, peer starts so far) under (max, max, +).
struct WnAgg {
    using T = WnAgg;
    uint32_t p, q, d;
    __device__ __forceinline__ static WnAgg identity() { return {0, 0, 0}; }
    __device__ __forceinline__ static WnAgg combine(WnAgg a, WnAgg b) { return {max(a.p, b.p), max(a.q, b.q), a.d + b.d}; }
};
// Field by field rather than common.cuh's word-wise shfl_up: the per-row kernels then keep their registers and code.
__device__ __forceinline__ WnAgg shfl_up(WnAgg v, int o) {
    return WnAgg{__shfl_up_sync(0xffffffffu, v.p, o), __shfl_up_sync(0xffffffffu, v.q, o), __shfl_up_sync(0xffffffffu, v.d, o)};
}
// A tile's value: its WnAgg and its partition starts, so the scan's total is the partition count.
struct WnTile {
    using T = WnTile;
    WnAgg v;
    uint32_t parts;
    __device__ __forceinline__ static WnTile identity() { return {WnAgg::identity(), 0}; }
    __device__ __forceinline__ static WnTile combine(WnTile a, WnTile b) { return {WnAgg::combine(a.v, b.v), a.parts + b.parts}; }
};

struct WnArgs {
    int64_t n;
    int n_part, n_keys;
    SortKey key[SORT_MAX_KEYS];
    const char* data[SORT_MAX_KEYS];   // sorted key columns
    const uint8_t* vb[SORT_MAX_KEYS];  // their validity bytes, nullptr for a numpy column
    uint8_t* flags;
    WnTile* tile;         // per tile: its reduction (bounds), then its exclusive prefix (tile_carry_kernel)
    WnTile* total;        // the combine of every tile: .parts is the partition count
    uint32_t *psize, *pend, *pdense;  // slot P: partition size, slot Q: peer-group end, slot P: D at the partition start
    int n_funcs;
    int func[SORT_MAX_COLS];
    int64_t farg[SORT_MAX_COLS];
    void* out[SORT_MAX_COLS];
};

__device__ __forceinline__ bool wn_key_differs(const WnArgs& a, int j, int64_t i) {
    const SortKey& k = a.key[j];
    bool na0 = a.vb[j] && a.vb[j][i - 1] == 0, na1 = a.vb[j] && a.vb[j][i] == 0;
    const uint64_t w0 = sort_word(k, load_bits(a.data[j], k.size, i - 1), na0);
    const uint64_t w1 = sort_word(k, load_bits(a.data[j], k.size, i), na1);
    return na0 != na1 || w0 != w1;
}

__global__ void __launch_bounds__(TILE_THREADS) window_bounds_kernel(const __grid_constant__ WnArgs a) {
    const int64_t t = blockIdx.x;
    WnTile acc = WnTile::identity();
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        if (i >= a.n) break;
        uint8_t f = WN_PART | WN_PEER;
        if (i > 0) {
            f = 0;
            for (int j = 0; j < a.n_keys && !f; j++)
                if (wn_key_differs(a, j, i)) f = j < a.n_part ? (WN_PART | WN_PEER) : WN_PEER;
        }
        a.flags[i] = f;
        if (f & WN_PART) { acc.v.p = (uint32_t)i; acc.parts++; }
        if (f & WN_PEER) { acc.v.q = (uint32_t)i; acc.v.d++; }
    }
    acc = block_reduce<WnTile>(acc);
    if (threadIdx.x == 0) a.tile[t] = acc;
}

// Inclusive scan values of this thread's TILE_ITEMS positions of tile t, seeded by the tile's exclusive prefix; f: their flags.
__device__ __forceinline__ void wn_scan_tile(int64_t n, const uint8_t* flags, const WnTile* tile, int64_t t, uint8_t (&f)[TILE_ITEMS],
                                             WnAgg (&v)[TILE_ITEMS]) {
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        f[k] = i < n ? flags[i] : 0;
        v[k] = WnAgg{(f[k] & WN_PART) ? (uint32_t)i : 0u, (f[k] & WN_PEER) ? (uint32_t)i : 0u, (f[k] & WN_PEER) ? 1u : 0u};
    }
    tile_scan<WnAgg>(tile[t].v, v);
}

// The ranking scan of this block's tile, then body(i, v) for each of this thread's positions i < n, v its scan value.  The
// bodies have out-of-line slow paths (divisions, searches): holding every item's scan values in registers across them spills,
// so each thread parks its own values in shared memory and the item loop is not unrolled.
template <typename Body>
__device__ __forceinline__ void wn_for_rows(int64_t n, const uint8_t* flags, const WnTile* tile, Body body) {
    const int64_t t = blockIdx.x;
    uint8_t f[TILE_ITEMS];
    WnAgg v[TILE_ITEMS];
    wn_scan_tile(n, flags, tile, t, f, v);
    __shared__ WnAgg s_v[TILE_ITEMS][TILE_THREADS];
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) s_v[k][threadIdx.x] = v[k];
#pragma unroll 1
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        if (i >= n) break;
        body(i, s_v[k][threadIdx.x]);
    }
}

__global__ void __launch_bounds__(TILE_THREADS) window_ends_kernel(const __grid_constant__ WnArgs a) {
    const int64_t t = blockIdx.x;
    uint8_t f[TILE_ITEMS];
    WnAgg v[TILE_ITEMS];
    wn_scan_tile(a.n, a.flags, a.tile, t, f, v);
    const int64_t i0 = tile_row(t, 0);
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = i0 + k * TILE_THREADS;
        if (i >= a.n) break;
        const uint8_t next = i + 1 < a.n ? a.flags[i + 1] : (WN_PART | WN_PEER);
        if (f[k] & WN_PART) a.pdense[i] = v[k].d;
        if (next & WN_PART) a.psize[v[k].p] = (uint32_t)(i + 1) - v[k].p;
        if (next & WN_PEER) a.pend[v[k].q] = (uint32_t)(i + 1);
    }
}

__global__ void __launch_bounds__(TILE_THREADS) window_eval_kernel(const __grid_constant__ WnArgs a) {
    wn_for_rows(a.n, a.flags, a.tile, [&](int64_t i, const WnAgg vk) {
        const uint32_t P = vk.p, s = a.psize[P], pos = (uint32_t)i - P, rank = vk.q - P + 1;
        for (int fn = 0; fn < a.n_funcs; fn++) {
            int64_t r = 0;
            double x = 0.0;
            switch (a.func[fn]) {
                case WN_ROW_NUMBER: r = pos + 1; break;
                case WN_RANK: r = rank; break;
                case WN_DENSE_RANK: r = vk.d - a.pdense[P] + 1; break;
                case WN_PERCENT_RANK: x = s == 1 ? 0.0 : (double)(rank - 1) / (double)(s - 1); break;
                case WN_CUME_DIST: x = (double)(a.pend[vk.q] - P) / (double)s; break;
                default: {  // WN_NTILE: the first s % n buckets hold s / n + 1 rows, the others s / n.  n > s gives buckets 1..s, as
                            // n = s does, so n is capped at s and the arithmetic stays in 32 bits.
                    const uint32_t nb = (uint32_t)min(a.farg[fn], (int64_t)s), q = s / nb, rem = s % nb, big = rem * (q + 1);
                    r = pos < big ? pos / (q + 1) + 1 : rem + (pos - big) / q + 1;
                }
            }
            if (a.func[fn] == WN_PERCENT_RANK || a.func[fn] == WN_CUME_DIST) ((double*)a.out[fn])[i] = x;
            else ((int64_t*)a.out[fn])[i] = r;
        }
    });
}

// ---- value window functions: SUM / COUNT / MEAN / MIN / MAX / FIRST_VALUE / LAST_VALUE over a frame [P, e], LAG / LEAD ----
//
// They run after window_ends_kernel, over the sorted columns the gather wrote.  A frame starts at the partition start P and ends
// at e = i (WF_ROWS), the row's last peer pend[Q] - 1 (WF_RANGE) or the partition's last row P + psize[P] - 1 (WF_PARTITION).
//   window_vscan_kernel<K, false>  per scan function (sum, count of a column, mean, min, max): the segmented reduction of each
//                                  TILE_ROWS-row tile, reset at partition starts (the WN_PART flags).
//   tile_carry_kernel<Wv<K>>       one block: the exclusive scan of the tile carries.
//   window_vscan_kernel<K, true>   the tile's scan again, seeded by its carry; every position that ends a frame of the function
//                                  writes the function's final cell and validity byte there.
//   window_veval_kernel            the ranking scan of the flags (P, Q) again, then per position and value function: a scan
//                                  function whose frame ends elsewhere copies out[e] to out[i] (race-free: e(e(i)) = e(i), so only
//                                  frame ends are read and they are not written); count(*) is e - P + 1; first_value, last_value,
//                                  lag and lead gather the cell at P, e, i - k or i + k (or take the default) from the sorted column.
// A min / max scan carries (radix word, position) with ties kept on the left and resolves to that position's cell.  Float sums
// are combined in double in the scan's fixed order, which depends only on the row count: they are bit-identical across runs and
// batch splits.
enum { WN_SUM = 6, WN_COUNT = 7, WN_MEAN = 8, WN_MIN = 9, WN_MAX = 10, WN_FIRST_VALUE = 11, WN_LAST_VALUE = 12, WN_LAG = 13, WN_LEAD = 14 };
enum { WF_NONE = 0, WF_RANGE = 1, WF_ROWS = 2, WF_PARTITION = 3 };
enum { WV_ISUM = 0, WV_FSUM = 1, WV_MIN = 2, WV_MAX = 3 };  // scan kinds: 64-bit wrapping sum (and count), double sum, min, max
constexpr uint32_t WV_NONE = 0xFFFFFFFFu;                    // a min / max scan that has seen no valid cell
constexpr uint64_t WV_NEG_ZERO = 0x8000000000000000ull;      // -0.0, the identity of a double sum (x + -0.0 == x for every x)

// Scan value: x the sum (int64 bits or double bits) or the radix word; c the count of valid cells or the position of the min /
// max; f set when the segment holds a partition start.
struct WvAgg { uint64_t x; uint32_t c, f; };

// VAR / STDDEV / VAR_POP / STDDEV_POP (codes 16..19) scan kind WV_MOM: c the count of valid cells, f as WvAgg's, mean their
// mean and m2 = sum (x - mean)^2, combined by Chan's pairwise merge (Wv<WV_MOM>::combine).  wv_t<K> is kind K's scan value.
enum { WN_VAR = 16, WN_STD = 17, WN_VAR_POP = 18, WN_STD_POP = 19 };
enum { WV_MOM = 5 };
struct WvMom { uint32_t c, f; double mean, m2; };
// COVAR_SAMP / COVAR_POP / CORR / REGR_SLOPE / REGR_INTERCEPT (codes 20..24, y = the function's column, x = its second column)
// scan kind WV_CO: c the count of rows where both cells are valid and non-NaN, f as WvAgg's, mx / my their means and sxx / syy /
// sxy = sum (x - mx)^2, sum (y - my)^2, sum (x - mx)(y - my), combined by the bivariate form of Chan's merge (Wv<WV_CO>::combine).
enum { WN_COVAR_SAMP = 20, WN_COVAR_POP = 21, WN_CORR = 22, WN_REGR_SLOPE = 23, WN_REGR_INTERCEPT = 24 };
enum { WV_CO = 6 };
struct WvCo { uint32_t c, f; double mx, my, sxx, syy, sxy; };

// A function whose result comes from a scan or a tree of its scan values: sum, count, mean, min, max and the moments (the ranking
// codes are routed before this is asked).
__host__ __device__ constexpr bool wv_aggregate(int code) { return code <= WN_MAX || code >= WN_VAR; }

// One value function as the kernels see it.
struct WvFunc {
    int code, frame, ct, size, out_size, dflt_valid;  // ct / size: the value column's c-type and cell bytes (size 0: count(*))
    int64_t k;                                        // lag / lead offset
    uint64_t dflt;                                    // lag / lead default bits
    const char* data;                                 // the sorted value column and its validity bytes (nullptr: numpy)
    const uint8_t* vb;
    char* out;                                        // the output column and its validity bytes (nullptr: count, numpy)
    uint8_t* out_vb;
};

// A bivariate function's second column (x): the sorted cells and validity bytes (nullptr: numpy), c-type and cell bytes.  The
// scan, tree and frame kernels take it as a last parameter of their own (read by WV_CO only), so the argument structs and every
// other kernel parameter keep their offsets.
struct WvCol {
    const char* data;
    const uint8_t* vb;
    int ct, size;
};

struct WvArgs {
    int64_t n;
    const uint8_t* flags;
    const uint32_t *psize, *pend;
    void* carry;   // per tile: its reduction, then its exclusive prefix (wv_t<K>)
    WvFunc s;      // window_vscan_kernel: the function being scanned
    int n_funcs;   // window_veval_kernel: the value functions with work there
    WvFunc f[SORT_MAX_COLS];
};

// Kind K's scan value as a monoid (common.cuh): Wv<K>::T, identity() and combine(a, b).
template <int K>
struct Wv {
    using T = WvAgg;
    __device__ __forceinline__ static WvAgg identity() { return WvAgg{K == WV_FSUM ? WV_NEG_ZERO : 0ull, (K == WV_MIN || K == WV_MAX) ? WV_NONE : 0u, 0u}; }
    __device__ __forceinline__ static WvAgg combine(WvAgg a, WvAgg b) {
        if (b.f) return b;
        WvAgg r{b.x, b.c, a.f};
        if (K == WV_ISUM) { r.x = a.x + b.x; r.c = a.c + b.c; }
        else if (K == WV_FSUM) { r.x = (uint64_t)__double_as_longlong(__longlong_as_double((long long)a.x) + __longlong_as_double((long long)b.x)); r.c = a.c + b.c; }
        else {
            const bool take_b = a.c == WV_NONE || (b.c != WV_NONE && (K == WV_MIN ? b.x < a.x : b.x > a.x));  // ties keep the left row
            if (!take_b) { r.x = a.x; r.c = a.c; }
        }
        return r;
    }
};
// Chan's merge of (n_a, mean_a, M2_a) and (n_b, mean_b, M2_b): with d = mean_b - mean_a and n = n_a + n_b, mean = mean_a +
// d n_b / n and M2 = M2_a + M2_b + d^2 n_a n_b / n.  An empty side gives the other side's values exactly (no 0 / 0); every term
// of M2 is >= 0, and equal means give d = 0, so a frame of equal values has M2 = 0 exactly.
template <>
struct Wv<WV_MOM> {
    using T = WvMom;
    __device__ __forceinline__ static WvMom identity() { return WvMom{0u, 0u, 0.0, 0.0}; }
    __device__ __forceinline__ static WvMom combine(WvMom a, WvMom b) {
        if (b.f) return b;
        if (b.c == 0) return a;
        if (a.c == 0) { b.f = a.f; return b; }
        const uint32_t n = a.c + b.c;
        const double w = (double)b.c / (double)n, d = b.mean - a.mean;
        return WvMom{n, a.f, a.mean + d * w, a.m2 + b.m2 + d * (d * ((double)a.c * w))};
    }
};
// The bivariate merge: the means as WV_MOM's, and with t = n_a n_b / n, sxx += (dx dx) t, syy += (dy dy) t, sxy += (dx dy) t.
// The three terms are formed alike, so swapping x and y swaps sxx and syy and leaves sxy's bits (dx dy = dy dx), and x = y gives
// sxx, syy and sxy the same bits; a frame of equal x has dx = 0 at every merge, so sxx = 0 exactly.
template <>
struct Wv<WV_CO> {
    using T = WvCo;
    __device__ __forceinline__ static WvCo identity() { return WvCo{0u, 0u, 0.0, 0.0, 0.0, 0.0, 0.0}; }
    __device__ __forceinline__ static WvCo combine(WvCo a, WvCo b) {
        if (b.f) return b;
        if (b.c == 0) return a;
        if (a.c == 0) { b.f = a.f; return b; }
        const uint32_t n = a.c + b.c;
        const double w = (double)b.c / (double)n, dx = b.mx - a.mx, dy = b.my - a.my, t = (double)a.c * w;
        return WvCo{n, a.f, a.mx + dx * w, a.my + dy * w, a.sxx + b.sxx + (dx * dx) * t, a.syy + b.syy + (dy * dy) * t,
                    a.sxy + b.sxy + (dx * dy) * t};
    }
};
template <int K> using wv_t = typename Wv<K>::T;
// Field-wise shuffles, as WnAgg's: the value scans then compile as with per-field shuffles of their own.
__device__ __forceinline__ WvAgg shfl_up(WvAgg v, int o) {
    return WvAgg{__shfl_up_sync(0xffffffffu, (unsigned long long)v.x, o), __shfl_up_sync(0xffffffffu, v.c, o), __shfl_up_sync(0xffffffffu, v.f, o)};
}
__device__ __forceinline__ WvMom shfl_up(WvMom v, int o) {
    return WvMom{__shfl_up_sync(0xffffffffu, v.c, o), __shfl_up_sync(0xffffffffu, v.f, o), __shfl_up_sync(0xffffffffu, v.mean, o),
                 __shfl_up_sync(0xffffffffu, v.m2, o)};
}
__device__ __forceinline__ WvCo shfl_up(WvCo v, int o) {
    return WvCo{__shfl_up_sync(0xffffffffu, v.c, o), __shfl_up_sync(0xffffffffu, v.f, o), __shfl_up_sync(0xffffffffu, v.mx, o),
                __shfl_up_sync(0xffffffffu, v.my, o), __shfl_up_sync(0xffffffffu, v.sxx, o), __shfl_up_sync(0xffffffffu, v.syy, o),
                __shfl_up_sync(0xffffffffu, v.sxy, o)};
}
// The carry and tree buffers hold kind K's scan values.
template <int K>
__device__ __forceinline__ wv_t<K>* wv_buf(void* p) { return (wv_t<K>*)p; }

// Cell i of a column of c-type ct and `size` bytes as a double (integers and bool exactly up to 2^53), as wv_value<WV_MOM>
// converts its cells (which keeps its own copy, so the moments' kernels compile as before).
__device__ __forceinline__ double wv_double(const char* data, int ct, int size, int64_t i) {
    const uint64_t raw = load_bits(data, size, i);
    return ct == CT_FLOAT64 ? __longlong_as_double((long long)raw)
         : ct == CT_FLOAT32 ? (double)__uint_as_float((uint32_t)raw)
         : ctype_is_signed_int(ct) ? (double)((int64_t)(raw << (64 - 8 * size)) >> (64 - 8 * size))
                                   : (double)raw;
}

// Scan value of position i of the scanned function (x: its second column, read by WV_CO only); `part`: i starts a partition.
template <int K>
__device__ __forceinline__ wv_t<K> wv_value(const WvFunc& s, const WvCol& x, int64_t i, bool part) {
    WvAgg r = Wv<K>::identity();
    r.f = part;
    bool na = s.vb && s.vb[i] == 0;
    if (K == WV_ISUM && s.code == WN_COUNT && !ctype_is_float(s.ct)) { r.c = !na; return r; }  // only NaN needs the values
    const uint64_t raw = load_bits(s.data, s.size, i);
    if (K == WV_ISUM) {
        uint64_t x = raw;
        if (s.ct == CT_FLOAT64) na = na || isnan(__longlong_as_double((long long)raw));
        else if (s.ct == CT_FLOAT32) na = na || isnan(__uint_as_float((uint32_t)raw));
        else if (ctype_is_signed_int(s.ct)) x = (uint64_t)((int64_t)(raw << (64 - 8 * s.size)) >> (64 - 8 * s.size));
        if (!na) { r.x = x; r.c = 1; }
    } else if (K == WV_FSUM) {
        const double d = s.ct == CT_FLOAT64 ? __longlong_as_double((long long)raw) : (double)__uint_as_float((uint32_t)raw);
        if (!(na || isnan(d))) { r.x = (uint64_t)__double_as_longlong(d); r.c = 1; }
    } else {
        const uint64_t w = sort_word(SortKey{s.ct, s.size, 0, 1}, raw, na);
        if (!na) { r.x = w; r.c = (uint32_t)i; }
    }
    return r;
}
// (1, x, 0) for a valid, non-NaN cell x converted to double (integers and bool exactly up to 2^53); the identity otherwise.
template <>
__device__ __forceinline__ WvMom wv_value<WV_MOM>(const WvFunc& s, const WvCol&, int64_t i, bool part) {
    WvMom r = Wv<WV_MOM>::identity();
    r.f = part;
    const uint64_t raw = load_bits(s.data, s.size, i);
    const double x = s.ct == CT_FLOAT64 ? __longlong_as_double((long long)raw)
                   : s.ct == CT_FLOAT32 ? (double)__uint_as_float((uint32_t)raw)
                   : ctype_is_signed_int(s.ct) ? (double)((int64_t)(raw << (64 - 8 * s.size)) >> (64 - 8 * s.size))
                                               : (double)raw;
    if (!(s.vb && s.vb[i] == 0) && !isnan(x)) { r.c = 1; r.mean = x; }
    return r;
}
// (1, x, y, 0, 0, 0) when both cells are valid and non-NaN (pairwise deletion); the identity otherwise.
template <>
__device__ __forceinline__ WvCo wv_value<WV_CO>(const WvFunc& s, const WvCol& x, int64_t i, bool part) {
    WvCo r = Wv<WV_CO>::identity();
    r.f = part;
    const double yv = wv_double(s.data, s.ct, s.size, i), xv = wv_double(x.data, x.ct, x.size, i);
    if (!(s.vb && s.vb[i] == 0) && !(x.vb && x.vb[i] == 0) && !isnan(xv) && !isnan(yv)) { r.c = 1; r.mx = xv; r.my = yv; }
    return r;
}

// dst[i] = the low `size` bytes of bits.
__device__ __forceinline__ void wv_store_bits(void* dst, int64_t i, uint64_t bits, int size) {
    switch (size) {
        case 8: ((uint64_t*)dst)[i] = bits; break;
        case 4: ((uint32_t*)dst)[i] = (uint32_t)bits; break;
        case 2: ((uint16_t*)dst)[i] = (uint16_t)bits; break;
        default: ((uint8_t*)dst)[i] = (uint8_t)bits; break;
    }
}

// The function's result at a frame end i whose frame's scan value is v.
template <int K>
__device__ __forceinline__ void wv_write(const WvFunc& s, int64_t i, wv_t<K> v) {
    if (s.code == WN_COUNT) { ((int64_t*)s.out)[i] = v.c; return; }
    if (K == WV_MIN || K == WV_MAX) {
        const bool ok = v.c != WV_NONE;
        if (ok) copy_cell(s.out, i, s.data, v.c, s.size);
        else wv_store_bits(s.out, i, 0, s.size);
        s.out_vb[i] = ok;
        return;
    }
    const bool ok = v.c > 0;
    if (s.code == WN_MEAN) {
        const double sum = K == WV_FSUM ? __longlong_as_double((long long)v.x)
                                        : ctype_is_signed_int(s.ct) || s.ct == CT_BOOL ? (double)(int64_t)v.x : (double)v.x;
        ((double*)s.out)[i] = ok ? sum / (double)v.c : 0.0;
    } else if (s.ct == CT_FLOAT32) {
        ((float*)s.out)[i] = ok ? (float)__longlong_as_double((long long)v.x) : 0.0f;
    } else {
        ((uint64_t*)s.out)[i] = ok ? v.x : 0ull;
    }
    s.out_vb[i] = ok;
}
// var = M2 / (m - 1) (NA when m < 2), var_pop = M2 / m (NA when m = 0), std / std_pop their IEEE sqrt; FLOAT64.  A frame holding
// +-inf has a non-finite mean and gives a valid NaN.
template <>
__device__ __forceinline__ void wv_write<WV_MOM>(const WvFunc& s, int64_t i, WvMom v) {
    const bool pop = s.code == WN_VAR_POP || s.code == WN_STD_POP, ok = v.c > (pop ? 0u : 1u);
    // Two branches rather than c - (pop ? 0.0 : 1.0): that constant would be hoisted and held across window_frame_kernel's row loop.
    double r = isfinite(v.mean) ? v.m2 / (pop ? (double)v.c : (double)v.c - 1.0) : __longlong_as_double(0x7FF8000000000000ll);
    if (s.code == WN_STD || s.code == WN_STD_POP) r = sqrt(r);
    ((double*)s.out)[i] = ok ? r : 0.0;
    s.out_vb[i] = ok;
}
// covar_samp = sxy / (m - 1) (NA when m < 2), covar_pop = sxy / m (NA when m = 0), corr = sxy / sqrt(sxx syy) (NA when m < 2,
// sxx = 0 or syy = 0; sxy / (sqrt(sxx) sqrt(syy)) when sxx syy overflows or is subnormal; clamped to [-1, 1]), regr_slope =
// sxy / sxx and regr_intercept = my - slope mx (NA when sxx = 0, which covers m <= 1); FLOAT64.  A frame whose counted pairs hold
// +-inf has a non-finite mean and gives a valid NaN.
template <>
__device__ __forceinline__ void wv_write<WV_CO>(const WvFunc& s, int64_t i, WvCo v) {
    const double m = (double)v.c;
    bool ok;
    double r;
    if (s.code == WN_COVAR_SAMP || s.code == WN_COVAR_POP) {
        const bool pop = s.code == WN_COVAR_POP;
        ok = v.c > (pop ? 0u : 1u);
        r = v.sxy / (m - (pop ? 0.0 : 1.0));
    } else if (s.code == WN_CORR) {
        ok = v.c > 1u && v.sxx != 0.0 && v.syy != 0.0;
        const double p = v.sxx * v.syy;
        r = v.sxy / (p >= DBL_MIN && p <= DBL_MAX ? sqrt(p) : sqrt(v.sxx) * sqrt(v.syy));
        r = r > 1.0 ? 1.0 : r < -1.0 ? -1.0 : r;  // NaN passes
    } else {
        ok = v.sxx != 0.0;
        const double slope = v.sxy / v.sxx;
        r = s.code == WN_REGR_SLOPE ? slope : v.my - slope * v.mx;
    }
    if (!(isfinite(v.mx) && isfinite(v.my))) r = __longlong_as_double(0x7FF8000000000000ll);
    ((double*)s.out)[i] = ok ? r : 0.0;
    s.out_vb[i] = ok;
}

template <int K, bool FINAL>
__global__ void __launch_bounds__(TILE_THREADS) window_vscan_kernel(const __grid_constant__ WvArgs a, const __grid_constant__ WvCol x) {
    const int64_t t = blockIdx.x;
    wv_t<K> v[TILE_ITEMS];
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        v[k] = i < a.n ? wv_value<K>(a.s, x, i, a.flags[i] & WN_PART) : Wv<K>::identity();
    }
    tile_scan<Wv<K>>(FINAL ? wv_buf<K>(a.carry)[t] : Wv<K>::identity(), v);
    if (!FINAL) {  // padding rows hold the identity, so the tile's last slot holds its reduction
        if (threadIdx.x == TILE_THREADS - 1) wv_buf<K>(a.carry)[t] = v[TILE_ITEMS - 1];
        return;
    }
    const uint8_t end_flag = a.s.frame == WF_RANGE ? WN_PEER : WN_PART;
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        if (i >= a.n) break;
        if (a.s.frame == WF_ROWS || i + 1 == a.n || (a.flags[i + 1] & end_flag)) wv_write<K>(a.s, i, v[k]);
    }
}

__global__ void __launch_bounds__(TILE_THREADS) window_veval_kernel(const __grid_constant__ WnArgs w, const __grid_constant__ WvArgs a) {
    wn_for_rows(w.n, w.flags, w.tile, [&](int64_t i, const WnAgg vk) {
        const int64_t P = vk.p, pe = P + w.psize[vk.p];  // the partition is [P, pe)
        for (int fn = 0; fn < a.n_funcs; fn++) {
            const WvFunc& g = a.f[fn];
            const int64_t e = g.frame == WF_ROWS ? i : g.frame == WF_RANGE ? (int64_t)w.pend[vk.q] - 1 : pe - 1;
            int64_t src;
            switch (g.code) {
                case WN_FIRST_VALUE: src = P; break;
                case WN_LAST_VALUE: src = e; break;
                case WN_LAG: src = i - g.k >= P ? i - g.k : -1; break;
                case WN_LEAD: src = i + g.k < pe ? i + g.k : -1; break;
                default:
                    if (g.size == 0) { ((int64_t*)g.out)[i] = e - P + 1; continue; }  // count(*)
                    src = e;  // a scan function: its frame end holds the result
            }
            const bool scanned = wv_aggregate(g.code);
            if (scanned && e == i) continue;
            const char* from = scanned ? g.out : g.data;
            const int sz = scanned ? g.out_size : g.size;
            if (src >= 0) {
                copy_cell(g.out, i, from, src, sz);
                if (g.out_vb) g.out_vb[i] = scanned ? g.out_vb[src] : g.vb ? g.vb[src] : 1;
            } else {
                wv_store_bits(g.out, i, g.dflt, sz);
                g.out_vb[i] = (uint8_t)g.dflt_valid;
            }
        }
    });
}

template <int K>
void launch_wv_scan(const WvArgs& a, const WvCol& x, int64_t n_tiles, cudaStream_t st) {
    window_vscan_kernel<K, false><<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a, x);
    tile_carry_kernel<Wv<K>><<<1, 1024, 0, st>>>((wv_t<K>*)a.carry, n_tiles, nullptr);
    window_vscan_kernel<K, true><<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a, x);
}

// ---- bounded ROWS frames (k PRECEDING / k FOLLOWING) and NTH_VALUE ----
//
// They run after the scans and window_veval_kernel, and only for functions routed here: every function over a bounded frame
// (frame WF_BOUNDED or WF_RANGE_BETWEEN) and NTH_VALUE over any frame.  A row's frame is [lo, hi] (empty when lo > hi), from wf_bounds
// only (frame 5: from its bounds buffer, read by window_range_frame_kernel<K>, the same per-row evaluation without the scan).
//   window_tree_kernel<K>     per aggregate over a bounded frame (sum, count of a column, mean, min, max): a dyadic block tree over
//                             the sorted positions, with no partition reset.  Level l holds the combine of each aligned block
//                             [b 2^l, (b + 1) 2^l) that lies inside [0, n), for l >= 3; levels 0..2 are not stored (the query
//                             reads them from the sorted column).  A launch takes 2048 inputs per block at level `base` (the
//                             sorted column for base 0) and builds levels base + 1 .. base + 11, so n < 2^31 takes at most 3.
//   window_frame_kernel<K>    the ranking scan of the flags (P, Q) again, then per row: the aggregate over [lo, hi] from the tree
//                             (K a scan kind), or every gather function (K = WV_GATHER): count(*) = max(0, hi - lo + 1),
//                             first_value / last_value / nth_value(n) = the cell at lo / hi / lo + n - 1 when that lies in [lo, hi].
// A query combines, left to right, the leaves from lo up to the next multiple of 8 (at most 7), then the largest aligned stored
// block that starts at the current position and ends by the last multiple of 8 in the frame, repeatedly, then the leaves up to hi
// (at most 7).  The order depends only on (lo, hi); a frame of W rows takes at most 14 leaves and 2 log2(W) nodes.
enum { WN_NTH_VALUE = 15 };
enum { WF_BOUNDED = 4, WF_RANGE_BETWEEN = 5 };  // frame 5: bounds per row from window_range_bounds_kernel (below)
constexpr int64_t WF_UNBOUNDED_START = INT64_MIN, WF_UNBOUNDED_END = INT64_MAX;
constexpr int WV_GATHER = 4;            // window_frame_kernel's gather pass (the scan kinds are 0..3, WV_MOM and WV_CO)
constexpr int WT_LOW = 3, WT_LEVELS = 32;  // levels below WT_LOW are not stored; level l < WT_LEVELS

// A function of this path: the value function, its frame bounds (WF_BOUNDED: row offsets or the unbounded sentinels above;
// WF_RANGE_BETWEEN: the bounds buffer of its frame) and, in g.k, nth_value's n.
struct WfFunc {
    WvFunc g;
    union {
        struct { int64_t start, end; };
        const int2* range;  // per row (lo, hi), from window_range_bounds_kernel (below)
    };
};

struct WfArgs {
    int64_t n;
    const uint8_t* flags;
    const WnTile* tile;             // the ranking scan's tile prefixes
    const uint32_t *psize, *pend;
    void* tree;                     // wv_t<K> nodes
    int64_t off[WT_LEVELS];         // level l's first node in `tree` (l >= WT_LOW); level l holds n >> l nodes
    WfFunc s;                       // window_tree_kernel / window_frame_kernel<K != WV_GATHER>: the aggregate
    int n_funcs;                    // window_frame_kernel<WV_GATHER>: the gather functions
    WfFunc f[SORT_MAX_COLS];
};

// Row i's frame [lo, hi] in its partition [P, pe), with qe one past its last peer.
__device__ __forceinline__ void wf_bounds(const WfFunc& g, int64_t i, int64_t P, int64_t pe, int64_t qe, int64_t& lo, int64_t& hi) {
    lo = P;
    hi = g.g.frame == WF_ROWS ? i : g.g.frame == WF_RANGE ? qe - 1 : pe - 1;
    if (g.g.frame == WF_BOUNDED) {
        if (g.start != WF_UNBOUNDED_START) lo = max(P, i + g.start);
        if (g.end != WF_UNBOUNDED_END) hi = min(pe - 1, i + g.end);
    }
}

template <int K>
__device__ __forceinline__ void wt_store(const WfArgs& a, int l, int64_t b, wv_t<K> v) {
    if (l >= WT_LOW && l < WT_LEVELS && b < (a.n >> l)) wv_buf<K>(a.tree)[a.off[l] + b] = v;
}

// Levels base + 1 .. base + 3 of a thread's TILE_ITEMS inputs x, in registers; x[0] ends as their combine.
template <int K>
__device__ __forceinline__ void wt_levels3(const WfArgs& a, int base, int64_t j0, wv_t<K> (&x)[TILE_ITEMS]) {
#pragma unroll
    for (int h = 1, m = TILE_ITEMS / 2; m >= 1; h++, m >>= 1) {
#pragma unroll
        for (int k = 0; k < m; k++) {
            x[k] = Wv<K>::combine(x[2 * k], x[2 * k + 1]);
            wt_store<K>(a, base + h, (j0 >> h) + k, x[k]);
        }
    }
}
// The same with constant trip counts: the loop above leaves the moments' and co-moments' larger combines partly rolled, and x in
// local memory.
template <int K>
__device__ __forceinline__ void wt_levels3_unrolled(const WfArgs& a, int base, int64_t j0, wv_t<K> (&x)[TILE_ITEMS]) {
#pragma unroll
    for (int h = 1; h <= 3; h++) {
#pragma unroll
        for (int k = 0; k < TILE_ITEMS / 2; k++) {
            if (k < (TILE_ITEMS >> h)) {
                x[k] = Wv<K>::combine(x[2 * k], x[2 * k + 1]);
                wt_store<K>(a, base + h, (j0 >> h) + k, x[k]);
            }
        }
    }
}
template <>
__device__ __forceinline__ void wt_levels3<WV_MOM>(const WfArgs& a, int base, int64_t j0, WvMom (&x)[TILE_ITEMS]) {
    wt_levels3_unrolled<WV_MOM>(a, base, j0, x);
}
template <>
__device__ __forceinline__ void wt_levels3<WV_CO>(const WfArgs& a, int base, int64_t j0, WvCo (&x)[TILE_ITEMS]) {
    wt_levels3_unrolled<WV_CO>(a, base, j0, x);
}

template <int K>
__global__ void __launch_bounds__(TILE_THREADS) window_tree_kernel(const __grid_constant__ WfArgs a, int base, const __grid_constant__ WvCol x2) {
    __shared__ wv_t<K> s_node[TILE_THREADS];
    const int64_t n_in = a.n >> base, j0 = (int64_t)blockIdx.x * TILE_ROWS + threadIdx.x * TILE_ITEMS;
    wv_t<K> x[TILE_ITEMS];
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t j = j0 + k;
        x[k] = j >= n_in ? Wv<K>::identity() : base == 0 ? wv_value<K>(a.s.g, x2, j, false) : wv_buf<K>(a.tree)[a.off[base] + j];
    }
    wt_levels3<K>(a, base, j0, x);  // levels base + 1 .. base + 3 in registers
    s_node[threadIdx.x] = x[0];
    __syncthreads();
    for (int h = 4, m = TILE_THREADS / 2; m >= 1; h++, m >>= 1) {  // levels base + 4 .. base + 11 in shared memory
        wv_t<K> y = x[0];
        if (threadIdx.x < m) y = Wv<K>::combine(s_node[2 * threadIdx.x], s_node[2 * threadIdx.x + 1]);
        __syncthreads();
        if (threadIdx.x < m) {
            s_node[threadIdx.x] = y;
            wt_store<K>(a, base + h, (int64_t)blockIdx.x * m + threadIdx.x, y);
        }
        __syncthreads();
    }
}

// The aggregate of the scanned function over [lo, hi]: edge leaves from the sorted column, aligned blocks from the tree.
template <int K>
__device__ __forceinline__ wv_t<K> wt_query(const WfArgs& a, const WvCol& x, int64_t lo, int64_t hi) {
    wv_t<K> acc = Wv<K>::identity();
    const int64_t r = hi + 1, a8 = min(r, (lo + 7) & ~(int64_t)7);
    int64_t j = lo;
    for (; j < a8; j++) acc = Wv<K>::combine(acc, wv_value<K>(a.s.g, x, j, false));
    const int64_t b8 = max(j, r & ~(int64_t)7);
    while (j < b8) {  // j and b8 are multiples of 8, so l >= 3
        const int l = min(j == 0 ? 62 : __ffsll(j) - 1, 63 - __clzll(b8 - j));
        acc = Wv<K>::combine(acc, wv_buf<K>(a.tree)[a.off[l] + (j >> l)]);
        j += (int64_t)1 << l;
    }
    for (; j < r; j++) acc = Wv<K>::combine(acc, wv_value<K>(a.s.g, x, j, false));
    return acc;
}

// Row i's frame functions: the aggregate a.s over its [lo, hi] from the tree (K a scan kind), or every gather function (K =
// WV_GATHER); bounds(g, lo, hi) gives function g's frame.
template <int K, typename Bounds>
__device__ __forceinline__ void wf_eval_row(const WfArgs& a, const WvCol& x, int64_t i, Bounds bounds) {
    constexpr int KQ = K == WV_GATHER ? WV_ISUM : K;  // the scan kind of the aggregate pass
    int64_t lo, hi;
    if (K != WV_GATHER) {
        bounds(a.s, lo, hi);
        wv_write<KQ>(a.s.g, i, wt_query<KQ>(a, x, lo, hi));
    } else for (int fn = 0; fn < a.n_funcs; fn++) {
        const WfFunc& g = a.f[fn];
        bounds(g, lo, hi);
        if (g.g.size == 0) { ((int64_t*)g.g.out)[i] = max(hi - lo + 1, (int64_t)0); continue; }  // count(*)
        const int64_t src = g.g.code == WN_FIRST_VALUE ? lo : g.g.code == WN_LAST_VALUE ? hi : lo + g.g.k - 1;
        const bool in = lo <= hi && src <= hi;
        if (in) copy_cell(g.g.out, i, g.g.data, src, g.g.size);
        else wv_store_bits(g.g.out, i, 0, g.g.size);
        g.g.out_vb[i] = in && (!g.g.vb || g.g.vb[src]);
    }
}

template <int K>
__global__ void __launch_bounds__(TILE_THREADS) window_frame_kernel(const __grid_constant__ WfArgs a, const __grid_constant__ WvCol x) {
    wn_for_rows(a.n, a.flags, a.tile, [&](int64_t i, const WnAgg vk) {
        const int64_t P = vk.p, pe = P + a.psize[vk.p], qe = a.pend[vk.q];
        wf_eval_row<K>(a, x, i, [&](const WfFunc& g, int64_t& lo, int64_t& hi) { wf_bounds(g, i, P, pe, qe, lo, hi); });
    });
}

// The same over frame-5 functions, whose bounds window_range_bounds_kernel wrote: no scan of the flags is needed, so one thread
// per row.  48 registers: at the default budget the compiler holds the double sum in 32 and spills.  The co-moments' 48-byte
// accumulator and leaf spill at 48, so WV_CO takes up to 80 (it uses 68).
template <int K>
__global__ void __maxnreg__(K == WV_CO ? 80 : 48) window_range_frame_kernel(const __grid_constant__ WfArgs a, const __grid_constant__ WvCol x) {
    const int64_t i = (int64_t)blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i >= a.n) return;
    wf_eval_row<K>(a, x, i, [i](const WfFunc& g, int64_t& lo, int64_t& hi) {
        const int2 b = __ldg(g.range + i);
        lo = b.x;
        hi = b.y;
    });
}

// Build the tree of the aggregate a.s (levels WT_LOW.. up to log2 n), then evaluate it at every row.
template <int K>
void launch_wf_tree(const WfArgs& a, const WvCol& x, int64_t n_tiles, cudaStream_t st) {
    for (int base = 0; (a.n >> max(base + 1, WT_LOW)) > 0; base += 11)
        window_tree_kernel<K><<<(unsigned)(((a.n >> base) + TILE_ROWS - 1) / TILE_ROWS), TILE_THREADS, 0, st>>>(a, base, x);
    if (a.s.g.frame == WF_RANGE_BETWEEN) window_range_frame_kernel<K><<<(unsigned)(n_tiles * TILE_ITEMS), TILE_THREADS, 0, st>>>(a, x);
    else window_frame_kernel<K><<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a, x);
}

// ---- RANGE frames with value offsets (RANGE BETWEEN x PRECEDING AND y FOLLOWING): frame 5 ----
//
// A frame-5 function's bounds are a b200_window_range: per side UNBOUNDED, CURRENT ROW (the row's peer group: its first peer Q or
// its last peer qe - 1) or an offset k measured in the single ORDER BY key x.  With the key ascending, a k PRECEDING start is the
// first row of the partition's non-NA run with x_j >= x_i - k and a k FOLLOWING end the last row with x_j <= x_i + k (a PRECEDING
// end and a FOLLOWING start mirror these); descending swaps the signs.  An offset bound at an NA row (null or NaN) is its peer
// group's boundary; at a non-NA row it never reaches an NA row, and one that no row satisfies leaves the frame empty.
//   window_range_bounds_kernel  one launch per distinct frame-5 frame, before that frame's trees and gathers: the ranking scan of
//                               the flags (P, Q) again, psize / pend for pe and qe, then per row and offset side one search of
//                               the sorted key column.  Writes (lo, hi) per row; window_range_frame_kernel<K> reads them.
// Every comparison is exact in an ascending 64-bit order word: integers (DATE in days, DATETIME / TIMEDELTA in ns) as x + 2^63
// (signed) or x (unsigned), so x -+ k is the word -+ k and a carry out of 64 bits means the bound lies past every value of the
// type; floats widened to double and compared against fl(x -+ k) through the sort's double order (-0.0 equals 0.0).
// A state holds at most FS_MAX_ROWS rows: the positions of a non-empty frame fit int32, an empty frame is stored as (0, -1).
static_assert(FS_MAX_ROWS <= (int64_t)INT32_MAX + 1, "window_range_bounds_kernel stores non-empty bounds as int32");
enum { WR_UNBOUNDED_PRECEDING = 0, WR_PRECEDING = 1, WR_CURRENT_ROW = 2, WR_FOLLOWING = 3, WR_UNBOUNDED_FOLLOWING = 4 };

struct WrArgs {
    int64_t n;
    const uint8_t* flags;
    const WnTile* tile;            // the ranking scan's tile prefixes
    const uint32_t *psize, *pend;
    SortKey key;                   // the ORDER BY key (read for offset bounds only)
    const char* data;              // its sorted column and validity bytes (nullptr: numpy)
    const uint8_t* vb;
    int start_kind, end_kind;
    uint64_t start_bits, end_bits; // offset magnitudes: a non-negative integer, or a finite non-negative double's bits
    int2* out;                     // per row: (lo, hi)
};

// Ascending order word of key cell j (load_bits at the key's width, as the sort's encoder reads it); na: null or NaN.
__device__ __forceinline__ uint64_t wr_word(const WrArgs& a, int64_t j, bool& na) {
    const SortKey& k = a.key;
    const uint64_t raw = load_bits(a.data, k.size, j);
    na = a.vb && a.vb[j] == 0;
    if (ctype_is_float(k.ct)) {
        const double d = k.ct == CT_FLOAT64 ? __longlong_as_double((long long)raw) : (double)__uint_as_float((uint32_t)raw);
        na = na || isnan(d);
        return (uint64_t)canon_float_ordered(canon_float_key(d)) ^ 0x8000000000000000ull;
    }
    if (!ctype_is_signed_int(k.ct)) return raw;
    return (uint64_t)((int64_t)(raw << (64 - 8 * k.size)) >> (64 - 8 * k.size)) ^ 0x8000000000000000ull;
}

// Order word of x - k (neg) or x + k for the cell whose word is w; sat = -1 / +1 when an integer result lies below / above every
// word (it then bounds nothing on that side), else 0.
__device__ __forceinline__ uint64_t wr_target(int ct, uint64_t w, bool neg, uint64_t k, int& sat) {
    sat = 0;
    if (ctype_is_float(ct)) {
        const double x = ordered_to_f64(w), d = __longlong_as_double((long long)k), t = neg ? x - d : x + d;
        return (uint64_t)canon_float_ordered(canon_float_key(t)) ^ 0x8000000000000000ull;
    }
    if (neg) { sat = w < k ? -1 : 0; return w - k; }
    sat = w > ~0ull - k ? 1 : 0;
    return w + k;
}

// The first j in [P, pe) with p(j), pe if none, for p false then true over [P, pe): gallop from h in [P, pe) by 1, 2, 4, ...
// rows, then bisect.  O(log d) probes for an answer d rows from h, all near h.
template <typename Pred>
__device__ __forceinline__ int64_t wr_first(int64_t P, int64_t pe, int64_t h, Pred p) {
    int64_t lo, hi;  // p(lo) false or lo = P - 1; p(hi) true or hi = pe
    if (p(h)) {
        hi = h;
        for (int64_t s = 1;; s <<= 1) {
            lo = hi - s;
            if (lo < P) { lo = P - 1; break; }
            if (!p(lo)) break;
            hi = lo;
        }
    } else {
        lo = h;
        for (int64_t s = 1;; s <<= 1) {
            hi = lo + s;
            if (hi >= pe) { hi = pe; break; }
            if (p(hi)) break;
            lo = hi;
        }
    }
    while (hi - lo > 1) {
        const int64_t m = lo + ((hi - lo) >> 1);
        if (p(m)) hi = m;
        else lo = m;
    }
    return hi;
}

// Row i's start (end = false) or end bound of one side.  wi / na: row i's order word and NA flag (read for the offset kinds only).
__device__ __forceinline__ int64_t wr_bound(const WrArgs& a, int kind, uint64_t k, bool end, int64_t P, int64_t pe, int64_t Q,
                                            int64_t qe, uint64_t wi, bool na) {
    if (kind == WR_UNBOUNDED_PRECEDING) return P;
    if (kind == WR_UNBOUNDED_FOLLOWING) return pe - 1;
    if (kind == WR_CURRENT_ROW || na) return end ? qe - 1 : Q;
    // In y = word (ascending) or ~word (descending), y grows with the position over the non-NA run: a start is the first row
    // with y >= Y, an end the last row with y <= Y, i.e. one before the first with y >= Y + 1.  NA rows stand below (NA first)
    // or above (NA last) every y, so the search never needs the run's ends.
    const bool desc = a.key.desc, nl = a.key.na_last;
    int sat;
    uint64_t Y = wr_target(a.key.ct, wi, (kind == WR_PRECEDING) != desc, k, sat);
    if (desc) { Y = ~Y; sat = -sat; }
    if (end) {
        if (sat == 0 && Y == ~0ull) sat = 1;
        Y++;
    }
    const auto p = [&](int64_t j) {
        bool nj;
        const uint64_t wj = wr_word(a, j, nj);
        return nj ? nl : sat < 0 || (sat == 0 && (desc ? ~wj : wj) >= Y);
    };
    const int64_t j = wr_first(P, pe, kind == WR_PRECEDING ? Q : qe - 1, p);
    bool nj = false;
    if (!end) {
        if (j < pe) wr_word(a, j, nj);
        return nj ? pe : j;  // only NA rows satisfy it: empty
    }
    if (j - 1 >= P) wr_word(a, j - 1, nj);
    return nj ? P - 1 : j - 1;
}

__global__ void __launch_bounds__(TILE_THREADS) window_range_bounds_kernel(const __grid_constant__ WrArgs a) {
    const bool offsets = a.start_kind == WR_PRECEDING || a.start_kind == WR_FOLLOWING || a.end_kind == WR_PRECEDING ||
                         a.end_kind == WR_FOLLOWING;
    wn_for_rows(a.n, a.flags, a.tile, [&](int64_t i, const WnAgg vk) {
        const int64_t P = vk.p, pe = P + a.psize[vk.p], Q = vk.q, qe = a.pend[vk.q];
        bool na = false;
        const uint64_t wi = offsets ? wr_word(a, i, na) : 0;
        const int64_t lo = wr_bound(a, a.start_kind, a.start_bits, false, P, pe, Q, qe, wi, na);
        const int64_t hi = wr_bound(a, a.end_kind, a.end_bits, true, P, pe, Q, qe, wi, na);
        // A non-empty frame lies in [0, n) with n <= 2^31, so both bounds fit int32.  An empty one may carry lo = pe = 2^31 (a
        // state of exactly 2^31 rows), so every empty frame is stored as (0, -1): its consumers read nothing for lo > hi.
        a.out[i] = lo <= hi ? make_int2((int)lo, (int)hi) : make_int2(0, -1);
    });
}

// ---- IGNORE NULLS: FIRST_VALUE / LAST_VALUE / NTH_VALUE over every frame, LAG / LEAD ----
//
// A cell is null when count(x) does not count it: its validity byte is 0 or it is a float NaN (RESPECT NULLS first_value keeps
// a NaN as a valid cell; IGNORE NULLS skips it, as pandas' ffill / bfill do).  With v[j] = 1 at the non-null sorted rows, one
// value column gets c[0..n], the exclusive prefix count of v (c[n] = m, the non-null rows), and pos[0..m), their positions:
//   window_nulls_count_kernel    per TILE_ROWS-row tile: its non-null count.
//   tile_carry_kernel            one block: the exclusive scan of the tile counts, and c[n].
//   window_nulls_compact_kernel  per tile again: c[i] from the tile prefix and a ballot per 32 rows; pos[c[i]] = i at non-null i.
// Then each function is index arithmetic on (c, pos) over the frame [lo, hi] or the partition [P, pe) of its RESPECT NULLS form:
//   first_value  j = c[lo], valid iff lo <= hi and j < c[hi + 1]      nth_value(n)  j = c[lo] + n - 1, valid iff j < c[hi + 1]
//   last_value   j = c[hi + 1] - 1, valid iff j >= c[lo]              lag(k)        j = c[i] - k, valid iff j >= c[P]
//   lead(k)      j = c[i + 1] + k - 1, valid iff j < c[pe]            (lo <= hi is tested before c is read: an empty bounded
// frame's lo may lie past n).  The result is the cell at pos[j]; else NA, or lag / lead's default.  lag / lead with k = 0 is the
// row itself, as in RESPECT NULLS.  No arithmetic on the values: the results are exact and depend only on sorted positions.
//   window_nulls_eval_kernel     frames 1..4, lag and lead: the ranking scan of the flags (P, Q) again, then per row every
//                                IGNORE NULLS function of the column whose (c, pos) is built.
//   window_nulls_range_kernel    frame 5: the same, one thread per row, from the bounds window_range_bounds_kernel wrote.
// c and pos are uint32 (n <= 2^31); one buffer of 8 B per row holds them and is rebuilt for each value column.
struct WnlArgs {
    int64_t n;
    const uint8_t* flags;
    const WnTile* tile;             // the ranking scan's tile prefixes
    const uint32_t *psize, *pend;
    WvCol x;                        // the value column of every function below
    uint32_t* tcount;               // per tile: its non-null count, then its exclusive prefix
    uint32_t *c, *pos;
    int n_funcs;
    WfFunc f[SORT_MAX_COLS];        // g.k: nth_value's n or lag / lead's k; frame 5: range
};

__device__ __forceinline__ bool wnl_null(const WvCol& x, int64_t i) {
    if (x.vb && x.vb[i] == 0) return true;
    if (x.ct == CT_FLOAT64) return isnan(__longlong_as_double((long long)load_bits(x.data, 8, i)));
    if (x.ct == CT_FLOAT32) return isnan(__uint_as_float((uint32_t)load_bits(x.data, 4, i)));
    return false;
}

__global__ void __launch_bounds__(TILE_THREADS) window_nulls_count_kernel(const __grid_constant__ WnlArgs a) {
    const int64_t t = blockIdx.x;
    uint32_t cnt = 0;
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        cnt += i < a.n && !wnl_null(a.x, i);
    }
    cnt = block_reduce<SumOf<uint32_t>>(cnt);
    if (threadIdx.x == 0) a.tcount[t] = cnt;
}

__global__ void __launch_bounds__(TILE_THREADS) window_nulls_compact_kernel(const __grid_constant__ WnlArgs a) {
    __shared__ uint32_t s_seg[TILE_ITEMS * TILE_WARPS];  // per (item, warp) segment of 32 rows: its count, then its exclusive prefix
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t t = blockIdx.x;
    uint32_t ball[TILE_ITEMS];
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        ball[k] = __ballot_sync(0xffffffffu, i < a.n && !wnl_null(a.x, i));
        if (lane == 0) s_seg[k * TILE_WARPS + warp] = __popc(ball[k]);
    }
    tile_segment_scan<SumOf<uint32_t>>(s_seg, a.tcount[t]);
    const uint32_t below = (1u << lane) - 1u;
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        const int64_t i = tile_row(t, k);
        if (i >= a.n) break;
        const uint32_t ci = s_seg[k * TILE_WARPS + warp] + __popc(ball[k] & below);
        a.c[i] = ci;
        if ((ball[k] >> lane) & 1u) a.pos[ci] = (uint32_t)i;
    }
}

// Row i's IGNORE NULLS functions; bounds(g, lo, hi) gives a frame function's [lo, hi], and [P, pe) is the row's partition (read
// by lag and lead only).
template <typename Bounds>
__device__ __forceinline__ void wnl_eval_row(const WnlArgs& a, int64_t i, int64_t P, int64_t pe, Bounds bounds) {
    for (int fn = 0; fn < a.n_funcs; fn++) {
        const WfFunc& h = a.f[fn];
        const WvFunc& g = h.g;
        int64_t j = -1;  // the chosen non-null row's index in pos, -1: none
        bool self = false;
        if (g.code == WN_LAG || g.code == WN_LEAD) {
            if (g.k == 0) self = true;
            else if (g.code == WN_LAG) { const int64_t r = (int64_t)a.c[i] - g.k; if (r >= (int64_t)a.c[P]) j = r; }
            else { const int64_t r = (int64_t)a.c[i + 1] + g.k - 1; if (r < (int64_t)a.c[pe]) j = r; }
        } else {
            int64_t lo, hi;
            bounds(h, lo, hi);
            if (lo <= hi) {
                const int64_t c0 = a.c[lo], c1 = a.c[hi + 1];
                const int64_t r = g.code == WN_FIRST_VALUE ? c0 : g.code == WN_LAST_VALUE ? c1 - 1 : c0 + g.k - 1;
                if (r >= c0 && r < c1) j = r;
            }
        }
        if (self) {
            copy_cell(g.out, i, g.data, i, g.size);
            g.out_vb[i] = !g.vb || g.vb[i];
        } else if (j >= 0) {
            copy_cell(g.out, i, g.data, a.pos[j], g.size);
            g.out_vb[i] = 1;
        } else {
            const bool nav = g.code == WN_LAG || g.code == WN_LEAD;
            wv_store_bits(g.out, i, nav ? g.dflt : 0ull, g.size);
            g.out_vb[i] = nav ? (uint8_t)g.dflt_valid : 0;
        }
    }
}

__global__ void __launch_bounds__(TILE_THREADS) window_nulls_eval_kernel(const __grid_constant__ WnlArgs a) {
    wn_for_rows(a.n, a.flags, a.tile, [&](int64_t i, const WnAgg vk) {
        const int64_t P = vk.p, pe = P + a.psize[vk.p], qe = a.pend[vk.q];
        wnl_eval_row(a, i, P, pe, [&](const WfFunc& g, int64_t& lo, int64_t& hi) { wf_bounds(g, i, P, pe, qe, lo, hi); });
    });
}

__global__ void __launch_bounds__(TILE_THREADS) window_nulls_range_kernel(const __grid_constant__ WnlArgs a) {
    const int64_t i = (int64_t)blockIdx.x * TILE_THREADS + threadIdx.x;
    if (i >= a.n) return;
    wnl_eval_row(a, i, 0, 0, [i](const WfFunc& g, int64_t& lo, int64_t& hi) {
        const int2 b = __ldg(g.range + i);
        lo = b.x;
        hi = b.y;
    });
}

// (c, pos) of value column x, then `eval` over a.f (frames 1..4, lag and lead) or `range` (frame 5).
static void launch_wnl(WnlArgs& a, const WvCol& x, int64_t n_tiles, bool range, cudaStream_t st) {
    a.x = x;
    window_nulls_count_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a);
    tile_carry_kernel<SumOf<uint32_t>><<<1, 1024, 0, st>>>(a.tcount, n_tiles, a.c + a.n);
    window_nulls_compact_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a);
    if (range) window_nulls_range_kernel<<<(unsigned)(n_tiles * TILE_ITEMS), TILE_THREADS, 0, st>>>(a);
    else window_nulls_eval_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, st>>>(a);
}

// Calls launch(std::integral_constant<int, K>) with aggregate g's scan kind K, which its scan and its frame tree share.
template <typename Launch>
static void with_wv_kind(const WvFunc& g, Launch launch) {
    if (g.code >= WN_COVAR_SAMP) launch(std::integral_constant<int, WV_CO>());
    else if (g.code >= WN_VAR) launch(std::integral_constant<int, WV_MOM>());
    else if (g.code == WN_MIN) launch(std::integral_constant<int, WV_MIN>());
    else if (g.code == WN_MAX) launch(std::integral_constant<int, WV_MAX>());
    else if (g.code != WN_COUNT && ctype_is_float(g.ct)) launch(std::integral_constant<int, WV_FSUM>());
    else launch(std::integral_constant<int, WV_ISUM>());
}

// Ranking and value window functions over (PARTITION BY the first n_part keys ORDER BY the rest).  The output is the full sort's,
// plus one column per function after the input columns: numpy for the ranking functions and count, nullable for the others.
struct WindowState : FullSortState {
    int n_part, n_funcs;
    b200_window_func fn[SORT_MAX_COLS];  // rows / range hold the unbounded frame unless the function came with frame 4 / 5
    std::vector<DevBuf> fout;
    int64_t n_partitions = 0;  // metric 9

    WindowState(const int8_t* c_types, const int8_t* arr_types, int n_arrs, int n_part_, int n_keys, const int32_t* asc,
                const int32_t* na_last, const b200_window_func* funcs, int n_funcs_, int64_t obs, int dev, cudaStream_t st)
        : FullSortState(c_types, arr_types, n_arrs, n_keys, asc, na_last, obs, dev, st), n_part(n_part_), n_funcs(n_funcs_) {
        for (int f = 0; f < n_funcs; f++) {
            b200_window_func& d = fn[f] = funcs[f];
            // the bounds a function's frame does not read: equal functions then reach the kernels as equal bits
            if (d.frame != WF_BOUNDED) d.rows = b200_window_frame{WF_UNBOUNDED_START, WF_UNBOUNDED_END};
            if (d.frame != WF_RANGE_BETWEEN) d.range = b200_window_range{WR_UNBOUNDED_PRECEDING, WR_UNBOUNDED_FOLLOWING, 0, 0};
            B200_REQUIRE(d.code >= WN_ROW_NUMBER && d.code <= WN_REGR_INTERCEPT, "b200 window: unknown function code");
            B200_REQUIRE(!d.ignore_nulls || (d.code >= WN_FIRST_VALUE && d.code <= WN_NTH_VALUE),
                         "b200 window: IGNORE NULLS takes first_value, last_value, lag, lead and nth_value only (codes 11..15)");
            int ct = CT_INT64, at = ARR_NUMPY;
            if (d.code <= WN_NTILE) {
                B200_REQUIRE(d.col == -1 && d.frame == WF_NONE, "b200 window: a ranking function takes no column and no frame");
                if (d.code == WN_NTILE) B200_REQUIRE(d.arg >= 1, "b200 window: ntile needs n >= 1");
                if (d.code == WN_PERCENT_RANK || d.code == WN_CUME_DIST) ct = CT_FLOAT64;
            } else {
                B200_REQUIRE((d.col >= 0 && d.col < n_arrs) || (d.code == WN_COUNT && d.col == -1),
                             "b200 window: value column index out of range (-1, count(*), is for count only)");
                if (d.code == WN_LAG || d.code == WN_LEAD) {
                    B200_REQUIRE(d.frame == WF_NONE, "b200 window: lag and lead take no frame");
                    B200_REQUIRE(d.arg >= 0 && d.arg <= 0x7FFFFFFF, "b200 window: lag / lead offset k must be in [0, 2^31)");
                    B200_REQUIRE(d.default_valid == 0 || d.default_valid == 1, "b200 window: default_valid must be 0 or 1");
                } else {
                    B200_REQUIRE(d.frame >= WF_RANGE && d.frame <= WF_RANGE_BETWEEN,
                                 "b200 window: unknown frame (1 range, 2 rows, 3 partition, 4 rows between, 5 range between)");
                }
                if (d.frame == WF_RANGE_BETWEEN) check_range(d, n_keys);
                if (d.code == WN_NTH_VALUE) B200_REQUIRE(d.arg >= 1 && d.arg <= 0x7FFFFFFF, "b200 window: nth_value needs n in [1, 2^31)");
                if (d.frame == WF_BOUNDED) {
                    const b200_window_frame b = d.rows;
                    const int64_t lim = 0x7FFFFFFF;
                    B200_REQUIRE((b.start == WF_UNBOUNDED_START || (b.start >= -lim && b.start <= lim)) &&
                                 (b.end == WF_UNBOUNDED_END || (b.end >= -lim && b.end <= lim)),
                                 "b200 window: a frame bound is UNBOUNDED or a row offset in (-2^31, 2^31)");
                    B200_REQUIRE(b.start == WF_UNBOUNDED_START || b.end == WF_UNBOUNDED_END || b.start <= b.end,
                                 "b200 window: frame start after frame end");
                    // the spellings of the unbounded frames: the same frame gives the same bits however it is written
                    if (b.start == WF_UNBOUNDED_START && b.end == 0) d.frame = WF_ROWS;
                    else if (b.start == WF_UNBOUNDED_START && b.end == WF_UNBOUNDED_END) d.frame = WF_PARTITION;
                }
                const int vct = d.col >= 0 ? sc.ctype[d.col] : CT_INT64;
                const auto is_temporal = [](int t) { return t == CT_DATE || t == CT_DATETIME || t == CT_TIMEDELTA; };
                const bool temporal = is_temporal(vct);
                if (d.code == WN_SUM || d.code == WN_MEAN)
                    B200_REQUIRE(!temporal, "b200 window: sum and mean need an integer, bool or float column");
                if (d.code >= WN_VAR && d.code <= WN_STD_POP)
                    B200_REQUIRE(!temporal, "b200 window: var and std need an integer, bool or float column");
                if (d.code >= WN_COVAR_SAMP) {  // arg: the second column (x); frame 0 failed above
                    B200_REQUIRE(d.arg >= 0 && d.arg < n_arrs, "b200 window: covar / corr / regr second column index (arg) out of range");
                    B200_REQUIRE(!temporal && !is_temporal(sc.ctype[d.arg]),
                                 "b200 window: covar, corr and regr need integer, bool or float columns");
                }
                if (d.code == WN_SUM) ct = ctype_is_float(vct) ? vct : ctype_is_signed_int(vct) || vct == CT_BOOL ? CT_INT64 : CT_UINT64;
                else if (d.code == WN_MEAN || d.code >= WN_VAR) ct = CT_FLOAT64;
                else if (d.code != WN_COUNT) ct = vct;
                if (d.code != WN_COUNT) at = ARR_NULLABLE;
            }
            sc.ctype[n_out_cols] = ct;
            arr_type[n_out_cols++] = at;
        }
    }

    // Validates function d's range (frame 5) against the keys and zeroes its unread bits; the unbounded-start spellings become
    // frames 1 and 3, so a frame gives the same bits however it is written.
    void check_range(b200_window_func& d, int n_keys) {
        b200_window_range& r = d.range;
        B200_REQUIRE(r.start_kind >= WR_UNBOUNDED_PRECEDING && r.start_kind <= r.end_kind && r.end_kind <= WR_UNBOUNDED_FOLLOWING &&
                     r.start_kind != WR_UNBOUNDED_FOLLOWING && r.end_kind != WR_UNBOUNDED_PRECEDING,
                     "b200 window: range bound kinds are 0..4 with start_kind <= end_kind, start_kind != 4 and end_kind != 0");
        const auto offset = [](int kind) { return kind == WR_PRECEDING || kind == WR_FOLLOWING; };
        if (offset(r.start_kind) || offset(r.end_kind)) {
            B200_REQUIRE(n_keys - n_part == 1, "b200 window: a range offset (k PRECEDING / FOLLOWING) needs exactly one ORDER BY key");
            const int kct = sc.ctype[n_part];
            const bool flt = ctype_is_float(kct);
            B200_REQUIRE(flt || ctype_is_signed_int(kct) || kct == CT_UINT8 || kct == CT_UINT16 || kct == CT_UINT32 || kct == CT_UINT64,
                         "b200 window: a range offset needs an integer, float or temporal ORDER BY key (not bool)");
            for (const uint64_t k : {offset(r.start_kind) ? r.start_bits : 0ull, offset(r.end_kind) ? r.end_bits : 0ull})
                B200_REQUIRE(flt ? k < 0x7FF0000000000000ull : (int64_t)k >= 0,
                             "b200 window: a range offset is a non-negative int64 (integer keys, DATE days, DATETIME / TIMEDELTA ns) or "
                             "the bits of a finite, non-negative double (float keys)");
            // both offsets on one side: PRECEDING starts at least as far back as it ends, FOLLOWING the other way round (finite,
            // non-negative doubles order as their bits)
            if (r.start_kind == r.end_kind)
                B200_REQUIRE(r.start_kind == WR_PRECEDING ? r.start_bits >= r.end_bits : r.start_bits <= r.end_bits,
                             "b200 window: frame start after frame end");
        }
        if (!offset(r.start_kind)) r.start_bits = 0;  // unread: equal frames then compare equal
        if (!offset(r.end_kind)) r.end_bits = 0;
        if (r.start_kind == WR_UNBOUNDED_PRECEDING && r.end_kind == WR_CURRENT_ROW) d.frame = WF_RANGE;
        else if (r.start_kind == WR_UNBOUNDED_PRECEDING && r.end_kind == WR_UNBOUNDED_FOLLOWING) d.frame = WF_PARTITION;
    }

    // The sort first (its chunks and pair buffers are freed on return), then the window scratch and function columns.
    void finish_rows(std::vector<DevBuf>& vbytes) override {
        FullSortState::finish_rows(vbytes);
        const int64_t n = n_out;
        fout.resize(n_funcs);
        WnArgs a{};
        a.n = n; a.n_part = n_part; a.n_keys = sc.n_keys;
        for (int j = 0; j < sc.n_keys; j++) { a.key[j] = sc.key[j]; a.data[j] = out_data[j]; a.vb[j] = out_vb[j]; }
        WvArgs va{};
        std::vector<WvFunc> scans;
        WfArgs fa{};
        std::vector<WfFunc> trees;
        // the functions of one distinct frame 5 (nulls: its IGNORE NULLS functions)
        struct RangeFrame { b200_window_range r; std::vector<WfFunc> trees, gathers, nulls; };
        std::vector<RangeFrame> ranged;
        const auto range_frame = [&](int f) {
            const b200_window_range& r = fn[f].range;
            auto it = std::find_if(ranged.begin(), ranged.end(), [&](const RangeFrame& x) {
                return x.r.start_kind == r.start_kind && x.r.end_kind == r.end_kind && x.r.start_bits == r.start_bits &&
                       x.r.end_bits == r.end_bits;
            });
            return it == ranged.end() ? ranged.insert(ranged.end(), RangeFrame{r, {}, {}, {}}) : it;
        };
        std::vector<WfFunc> nulls;  // IGNORE NULLS functions over frames 1..4, lag and lead
        bool any_nulls = false;
        bool eval = false;
        for (int f = 0; f < n_funcs; f++) {
            const int c = sc.n_cols + f;
            fout[f].alloc((size_t)n * 8);
            out_data[c] = fout[f].as<char>();
            if (arr_type[c] == ARR_NULLABLE) { vbytes[c].alloc((size_t)n); out_vb[c] = vbytes[c].as<uint8_t>(); }
            const b200_window_func& d = fn[f];
            if (d.code <= WN_NTILE) {
                a.out[a.n_funcs] = out_data[c];
                a.func[a.n_funcs] = d.code; a.farg[a.n_funcs++] = d.arg;
                continue;
            }
            WvFunc g{d.code, d.frame, d.col >= 0 ? sc.ctype[d.col] : CT_INT64, d.col >= 0 ? ctype_size(sc.ctype[d.col]) : 0,
                     ctype_size(sc.ctype[c]), d.default_valid, d.arg, d.default_bits, d.col >= 0 ? out_data[d.col] : nullptr,
                     d.col >= 0 ? out_vb[d.col] : nullptr, out_data[c], out_vb[c]};
            WfFunc h{};
            h.g = g;
            h.start = d.rows.start;
            h.end = d.rows.end;
            if (d.ignore_nulls) {  // the IGNORE NULLS kernels only, never a scan, tree or gather
                (d.frame == WF_RANGE_BETWEEN ? range_frame(f)->nulls : nulls).push_back(h);
                any_nulls = true;
                continue;
            }
            if (d.frame == WF_BOUNDED || d.frame == WF_RANGE_BETWEEN || d.code == WN_NTH_VALUE) {  // the frame path only
                const bool agg = wv_aggregate(d.code) && d.col >= 0;
                if (d.frame == WF_RANGE_BETWEEN) {
                    (agg ? range_frame(f)->trees : range_frame(f)->gathers).push_back(h);
                } else if (agg) {
                    trees.push_back(h);
                } else {
                    fa.f[fa.n_funcs++] = h;
                }
                continue;
            }
            const bool scanned = wv_aggregate(d.code) && d.col >= 0;
            if (scanned) scans.push_back(g);
            if (!scanned || d.frame != WF_ROWS) { va.f[va.n_funcs++] = g; eval = true; }
        }
        if (n == 0) return;
        const int64_t n_tiles = (n + TILE_ROWS - 1) / TILE_ROWS;
        DevBuf flags, tiles, total, ends;
        flags.alloc((size_t)n);
        tiles.alloc((size_t)n_tiles * sizeof(WnTile));
        total.alloc(sizeof(WnTile));
        ends.alloc((size_t)n * 12);
        a.flags = flags.as<uint8_t>(); a.tile = tiles.as<WnTile>(); a.total = total.as<WnTile>();
        a.psize = ends.as<uint32_t>(); a.pend = a.psize + n; a.pdense = a.pend + n;
        window_bounds_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(a);
        tile_carry_kernel<WnTile><<<1, 1024, 0, stream>>>(a.tile, n_tiles, a.total);
        window_ends_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(a);
        if (a.n_funcs > 0) window_eval_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(a);
        B200_CUDA(cudaGetLastError());
        const auto moments = [](int code) { return code >= WN_VAR && code <= WN_STD_POP; };
        const auto bivariate = [](int code) { return code >= WN_COVAR_SAMP; };
        const auto value_bytes = [&](int code) { return bivariate(code) ? sizeof(WvCo) : moments(code) ? sizeof(WvMom) : sizeof(WvAgg); };
        const auto col2 = [&](const WvFunc& g) {  // a bivariate function's second column: its index is in arg (g.k)
            const int j = (int)g.k;
            return WvCol{out_data[j], out_vb[j], sc.ctype[j], ctype_size(sc.ctype[j])};
        };
        DevBuf carry;  // sized for the largest scan value among the scans
        size_t carry_bytes = 0;
        for (const WvFunc& g : scans) carry_bytes = std::max(carry_bytes, value_bytes(g.code));
        if (!scans.empty()) carry.alloc((size_t)n_tiles * carry_bytes);
        va.n = n; va.flags = a.flags; va.psize = a.psize; va.pend = a.pend; va.carry = carry.p;
        for (const WvFunc& g : scans) {
            va.s = g;
            const WvCol x = bivariate(g.code) ? col2(g) : WvCol{};
            with_wv_kind(g, [&](auto k) { launch_wv_scan<decltype(k)::value>(va, x, n_tiles, stream); });
        }
        if (eval) window_veval_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(a, va);
        B200_CUDA(cudaGetLastError());
        // IGNORE NULLS: one (c, pos) buffer of 8 B per row (plus a word per tile), rebuilt for each value column.  It is built once
        // per distinct column of the frame 1..4 / lag / lead functions, then once per distinct (frame 5, column) in the frame
        // loop below, after that frame's bounds.
        DevBuf nb;
        WnlArgs na{};
        const auto launch_nulls = [&](const std::vector<WfFunc>& fs, bool range) {
            for (size_t j = 0; j < fs.size(); j++) {
                const WvFunc& g = fs[j].g;
                bool seen = false;
                for (size_t k = 0; k < j; k++) seen = seen || fs[k].g.data == g.data;
                if (seen) continue;
                na.n_funcs = 0;
                for (size_t k = j; k < fs.size(); k++)
                    if (fs[k].g.data == g.data) na.f[na.n_funcs++] = fs[k];
                launch_wnl(na, WvCol{g.data, g.vb, g.ct, g.size}, n_tiles, range, stream);
            }
            B200_CUDA(cudaGetLastError());
        };
        if (any_nulls) {
            nb.alloc((size_t)(2 * n + 1 + n_tiles) * 4);
            na.n = n; na.flags = a.flags; na.tile = a.tile; na.psize = a.psize; na.pend = a.pend;
            na.c = nb.as<uint32_t>(); na.pos = na.c + n + 1; na.tcount = na.pos + n;
            launch_nulls(nulls, false);
        }
        // one tree buffer, reused by every aggregate over a bounded frame: n / 8 + n / 16 + ... nodes of the largest scan value
        // among them, <= 4 B per row (<= 6 B per row with a moment, <= 12 B per row with a bivariate function)
        DevBuf tree, rb;
        if (!trees.empty() || fa.n_funcs > 0 || !ranged.empty()) {
            fa.n = n; fa.flags = a.flags; fa.tile = a.tile; fa.psize = a.psize; fa.pend = a.pend;
            int64_t nodes = 0;
            for (int l = WT_LOW; l < WT_LEVELS; l++) { fa.off[l] = nodes; nodes += n >> l; }
            size_t tree_bytes = 0;  // 0: no tree
            for (const WfFunc& h : trees) tree_bytes = std::max(tree_bytes, value_bytes(h.g.code));
            for (const RangeFrame& rf : ranged)
                for (const WfFunc& h : rf.trees) tree_bytes = std::max(tree_bytes, value_bytes(h.g.code));
            if (tree_bytes > 0) tree.alloc((size_t)std::max<int64_t>(nodes, 1) * tree_bytes);
            fa.tree = tree.p;
            const auto launch_tree = [&](const WfFunc& h) {
                fa.s = h;
                const WvCol x = bivariate(h.g.code) ? col2(h.g) : WvCol{};
                with_wv_kind(h.g, [&](auto k) { launch_wf_tree<decltype(k)::value>(fa, x, n_tiles, stream); });
            };
            for (const WfFunc& h : trees) launch_tree(h);
            if (fa.n_funcs > 0) window_frame_kernel<WV_GATHER><<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(fa, WvCol{});
            B200_CUDA(cudaGetLastError());
            // frame 5: one 8 B/row bounds buffer, reused frame by frame (its bounds, then its trees, then its gathers)
            if (!ranged.empty()) rb.alloc((size_t)n * sizeof(int2));
            const int ok = std::min(n_part, sc.n_keys - 1);  // the ORDER BY key when there is one (offsets need it)
            WrArgs ra{n, a.flags, a.tile, a.psize, a.pend, sc.key[ok], out_data[ok], out_vb[ok], 0, 0, 0, 0, rb.as<int2>()};
            for (RangeFrame& rf : ranged) {
                ra.start_kind = rf.r.start_kind; ra.end_kind = rf.r.end_kind; ra.start_bits = rf.r.start_bits; ra.end_bits = rf.r.end_bits;
                window_range_bounds_kernel<<<(unsigned)n_tiles, TILE_THREADS, 0, stream>>>(ra);
                for (WfFunc& h : rf.trees) { h.range = ra.out; launch_tree(h); }
                fa.n_funcs = 0;
                for (WfFunc& h : rf.gathers) { h.range = ra.out; fa.f[fa.n_funcs++] = h; }
                if (fa.n_funcs > 0) window_range_frame_kernel<WV_GATHER><<<(unsigned)(n_tiles * TILE_ITEMS), TILE_THREADS, 0, stream>>>(fa, WvCol{});
                B200_CUDA(cudaGetLastError());
                for (WfFunc& h : rf.nulls) h.range = ra.out;
                launch_nulls(rf.nulls, true);
            }
        }
        auto* h = (WnTile*)pinned_acquire(sizeof(WnTile));
        B200_CUDA(cudaMemcpyAsync(h, total.p, sizeof(WnTile), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        n_partitions = h->parts;
        pinned_release(h, sizeof(WnTile));
    }

    int64_t metric(int which) const override { return which == 9 ? n_partitions : FullSortState::metric(which); }
};

// A new state from make() once the device is known to exist; nullptr and the last error on failure.
template <typename Make>
static void* sort_state_new(int32_t device, Make make) {
    try {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
            throw Error("b200 sort: no CUDA device available (this path has no CPU fallback)");
        B200_REQUIRE(device >= 0 && device < ndev, "b200 sort: bad device ordinal");
        return make();
    } catch (const std::exception& e) { set_last_error(e.what()); return nullptr; }
}

}  // namespace b200

using b200::SortState;

extern "C" {

void* b200_sort_state_init(int64_t operator_id, int64_t limit, int64_t offset, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs,
                           int32_t n_keys, const int32_t* ascending, const int32_t* na_last, int64_t output_batch_size, int32_t device,
                           void* stream) {
    (void)operator_id;
    return b200::sort_state_new(device, [&]() -> SortState* {
        B200_REQUIRE(limit >= 0 && offset >= 0, "b200 sort: limit and offset must be non-negative");
        B200_REQUIRE(limit <= b200::TK_MAX_K && offset <= b200::TK_MAX_K - limit, "b200 sort: limit + offset exceeds the top-k cap of 2^26 rows");
        return new b200::TopkState(limit, offset, c_types, arr_types, n_arrs, n_keys, ascending, na_last, output_batch_size, device,
                                   (cudaStream_t)stream);
    });
}

void* b200_sort_state_init_full(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs, int32_t n_keys,
                                const int32_t* ascending, const int32_t* na_last, int64_t output_batch_size, int32_t device, void* stream) {
    (void)operator_id;
    return b200::sort_state_new(device, [&]() -> SortState* {
        return new b200::FullSortState(c_types, arr_types, n_arrs, n_keys, ascending, na_last, output_batch_size, device,
                                       (cudaStream_t)stream);
    });
}

void* b200_sort_state_init_runs(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs, int32_t n_keys,
                                const int32_t* ascending, const int32_t* na_last, const int64_t* run_lengths, int32_t n_runs,
                                int64_t output_batch_size, int32_t device, void* stream) {
    (void)operator_id;
    return b200::sort_state_new(device, [&]() -> SortState* {
        B200_REQUIRE(run_lengths && n_runs >= 1, "b200 sort: at least one run length");
        int64_t total = 0;
        for (int32_t r = 0; r < n_runs; r++) {
            B200_REQUIRE(run_lengths[r] >= 0, "b200 sort: run lengths must be non-negative");
            total += run_lengths[r];
            B200_REQUIRE(total <= b200::FS_MAX_ROWS, "b200 sort: a full sort holds at most 2^31 rows (32-bit row ids)");
        }
        return new b200::MergeSortState(run_lengths, n_runs, c_types, arr_types, n_arrs, n_keys, ascending, na_last, output_batch_size,
                                        device, (cudaStream_t)stream);
    });
}

int b200_sort_sample(void* state, int64_t n_samples, int64_t rank, uint64_t* records) {
    try {
        auto* s = dynamic_cast<b200::FullSortState*>((SortState*)state);
        B200_REQUIRE(s, "b200 sort: samples are taken from a full-sort state");
        b200::scratch_set_stream(s->stream);
        s->sample(n_samples, rank, records);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_sort_count_below(void* state, const uint64_t* splitters, int64_t n_splitters, int64_t rank, int64_t* counts) {
    try {
        auto* s = dynamic_cast<b200::FullSortState*>((SortState*)state);
        B200_REQUIRE(s, "b200 sort: splitters are counted in a full-sort state");
        b200::scratch_set_stream(s->stream);
        s->count_below(splitters, n_splitters, rank, counts);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

void* b200_window_state_init(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs, int32_t n_partition_keys,
                             int32_t n_order_keys, const int32_t* order_ascending, const int32_t* order_na_last,
                             const b200_window_func* funcs, int32_t n_funcs, int64_t output_batch_size, int32_t device, void* stream) {
    (void)operator_id;
    return b200::sort_state_new(device, [&]() -> SortState* {
        const int np = n_partition_keys, no = n_order_keys;
        B200_REQUIRE(np >= 0 && no >= 0 && np + no >= 1 && np + no <= b200::SORT_MAX_KEYS,
                     "b200 window: 1 to 4 keys (PARTITION BY plus ORDER BY), neither count negative");
        B200_REQUIRE(no == 0 || (order_ascending && order_na_last), "b200 window: null ORDER BY direction or NA placement");
        B200_REQUIRE(funcs && n_funcs >= 1, "b200 window: at least one function");
        B200_REQUIRE(n_arrs >= np + no && n_arrs + n_funcs <= b200::SORT_MAX_COLS,
                     "b200 window: the keys are the first n_partition_keys + n_order_keys columns, and input plus function columns are at most 32");
        int32_t asc[b200::SORT_MAX_KEYS], na_last[b200::SORT_MAX_KEYS];
        for (int j = 0; j < np + no; j++) {  // PARTITION BY keys: ascending, NA last
            asc[j] = j < np ? 1 : order_ascending[j - np];
            na_last[j] = j < np ? 1 : order_na_last[j - np];
        }
        return new b200::WindowState(c_types, arr_types, n_arrs, np, np + no, asc, na_last, funcs, n_funcs, output_batch_size, device,
                                     (cudaStream_t)stream);
    });
}

int b200_sort_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last, int32_t* request_input) {
    try {
        B200_REQUIRE(state && in_table, "b200 sort: null state or table");
        auto* s = (SortState*)state;
        s->consume(in_table);
        if (is_last) s->finish();
        if (request_input) *request_input = 1;
        return is_last ? 1 : 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_sort_produce_output_batch(void* state, b200_table* out, int32_t* out_is_last, int32_t produce_output) {
    try {
        B200_REQUIRE(state && out && out_is_last, "b200 sort: null argument");
        return ((SortState*)state)->produce(out, out_is_last, produce_output != 0);
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

void b200_delete_sort_state(void* state) {
    auto* s = (SortState*)state;
    if (s) { cudaSetDevice(s->device); b200::scratch_set_stream(s->stream); }  // the form's buffers go back to this pool
    delete s;
}

int64_t b200_sort_get_metric(void* state, int32_t which) {
    return which >= 0 && which <= 9 ? ((SortState*)state)->metric(which) : -1;
}

}  // extern "C"
