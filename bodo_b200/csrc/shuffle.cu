// shuffle.cu — row -> rank radix partition of a columnar table (sm_90a).
//
// Replaces hash_keys_table(SEED_HASH_PARTITION) + mpi_comm_info::set_send_count + fill_send_array of the
// reference's shuffle_table (bodo/libs/_shuffle.cpp:94-163, 345-368, 477+, 1593-1642) and the
// cudf::hash_partition + contiguous_split pair of its GPU path (bodo/libs/gpu_utils.cpp:96-123, 509-525).
//
// One stable counting-sort pass over the rows:
//   K1 dest_hist   : dest[i] = (uint32) xxh3(key[i]) % n_pes (placement identical to the reference's
//                    hash_to_rank), per-CTA histogram of its contiguous row tile  -> hist[cta][dest]
//   K2 scan        : exclusive scan over (dest-major, cta-minor) -> first output row of every (cta, dest)
//   K3 scatter     : every CTA re-walks its tile in row order; a warp-ballot multi-split gives each row its
//                    stable rank; ALL columns are scattered in the same pass (no contiguous_split copy)
//   K4 pack bitmap : validity bytes of each destination segment are re-packed into a per-destination Arrow
//                    bitmap that starts on a byte boundary (the reference sends one null-bitmap buffer per
//                    destination with byte padding, _shuffle.cpp:661-875).
// Rows keep their input order inside a destination (fill_send_array is stable too), so the result is
// bit-identical to the oracle's oracle_shuffle_partition.
//
// b200_shuffle_partition_classes runs the same pass with K1's key hash swapped for KeyClassHash (common.cuh): every row of
// one key class (NA and NaN one class, -0.0 equal to 0.0, any fixed-width key type) goes to one rank, which is what the
// sharded window and min_row_number_filter need.  K2-K4 only read dest8 and are shared.
#include <vector>

#include "common.cuh"

namespace b200 {

constexpr int PART_THREADS = 256;
constexpr int MAX_PES = 256;
constexpr int MAX_SHUFFLE_COLS = 32;

__global__ void hash_to_rank_kernel(const __grid_constant__ KeySet k, int64_t n, int n_pes, int32_t* dest, uint32_t* hash_out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t h = hash_keys_row(k, i, SEED_HASH_PARTITION);
        if (dest) dest[i] = hash_to_rank_u32(h, n_pes);
        if (hash_out) hash_out[i] = h;
    }
}

// K1: tile = contiguous rows [cta * tile_rows, ...). dest8 holds the destination of every row.  H is the key hash policy
// (common.cuh): ReferenceKeyHash places rows as the reference does, KeyClassHash sends every key class to one rank.
template <class H>
__global__ void __launch_bounds__(PART_THREADS) dest_hist_kernel(const __grid_constant__ KeySet k,
                                                                 int64_t n, int64_t tile_rows, int n_pes, uint8_t* dest8,
                                                                 unsigned int* hist /* [gridDim.x][n_pes] */) {
    __shared__ unsigned int sh[MAX_PES];
    for (int d = threadIdx.x; d < n_pes; d += blockDim.x) sh[d] = 0;
    __syncthreads();
    int64_t r0 = (int64_t)blockIdx.x * tile_rows;
    int64_t r1 = r0 + tile_rows < n ? r0 + tile_rows : n;
    for (int64_t i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
        int d = hash_to_rank_u32(hash_keys_row<H>(k, i, SEED_HASH_PARTITION), n_pes);
        dest8[i] = (uint8_t)d;
        atomicAdd(&sh[d], 1u);
    }
    __syncthreads();
    for (int d = threadIdx.x; d < n_pes; d += blockDim.x) hist[(size_t)blockIdx.x * n_pes + d] = sh[d];
}

// K2: one CTA of 1024 threads. offsets[cta][d] = sum_{d' < d} total[d'] + sum_{cta' < cta} hist[cta'][d]; totals[d] = rows per dest.
// Warp w scans the CTA axis of destinations w, w + 32, ... with shuffles (the histogram has n_ctas x n_pes entries, ~10^4).
__global__ void __launch_bounds__(1024) scan_hist_kernel(const unsigned int* hist, int n_ctas, int n_pes, long long* offsets, long long* totals) {
    __shared__ long long tot[MAX_PES];
    __shared__ long long base[MAX_PES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int d = warp; d < n_pes; d += 32) {
        long long carry = 0;
        for (int c0 = 0; c0 < n_ctas; c0 += 32) {
            const int c = c0 + lane;
            const long long x = c < n_ctas ? (long long)hist[(size_t)c * n_pes + d] : 0;
            long long inc = x;
#pragma unroll
            for (int k = 1; k < 32; k <<= 1) { long long y = __shfl_up_sync(0xffffffffu, inc, k); if (lane >= k) inc += y; }
            if (c < n_ctas) offsets[(size_t)c * n_pes + d] = carry + inc - x;
            carry += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (lane == 0) { tot[d] = carry; totals[d] = carry; }
    }
    __syncthreads();
    if (threadIdx.x == 0) { long long b = 0; for (int d = 0; d < n_pes; d++) { base[d] = b; b += tot[d]; } }
    __syncthreads();
    for (int j = threadIdx.x; j < n_ctas * n_pes; j += blockDim.x) offsets[j] += base[j % n_pes];
}

struct ScatterArgs {
    int64_t n;
    int64_t tile_rows;
    int n_pes;
    int n_cols;
    const uint8_t* dest8;
    const long long* offsets;  // [n_ctas][n_pes]
    const void* in_data[MAX_SHUFFLE_COLS];
    const uint8_t* in_valid[MAX_SHUFFLE_COLS];
    void* out_data[MAX_SHUFFLE_COLS];
    uint8_t* out_valid_bytes[MAX_SHUFFLE_COLS];  // one byte per row (temp), nullptr if the column has no bitmap
    int itemsize[MAX_SHUFFLE_COLS];
    long long* perm_out;  // optional: source row of every output row (tests), may be nullptr
};

// K3: stable multi-split.  A CTA walks its tile in chunks of PART_THREADS * SC_STEPS rows; inside a chunk every warp owns a
// contiguous block of 32 * SC_STEPS rows and ranks them in row order with one MATCH.ANY per 32 rows (rank inside the step +
// rows of that destination the warp saw in earlier steps, kept in the warp's row of wtot); the warps' totals are combined once
// per chunk, so a chunk costs four CTA barriers for 2048 rows.
constexpr int SC_STEPS = 8;
__global__ void __launch_bounds__(PART_THREADS) scatter_kernel(const __grid_constant__ ScatterArgs a) {
    constexpr int NW = PART_THREADS / 32;
    __shared__ long long run[MAX_PES];          // next output row per destination for this CTA
    __shared__ unsigned int wtot[NW * MAX_PES];  // [warp][n_pes] rows of destination d in the warp's block of the current chunk
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, P = a.n_pes;
    for (int d = threadIdx.x; d < P; d += blockDim.x) run[d] = a.offsets[(size_t)blockIdx.x * P + d];
    const int64_t r0 = (int64_t)blockIdx.x * a.tile_rows;
    const int64_t r1 = r0 + a.tile_rows < a.n ? r0 + a.tile_rows : a.n;
    for (int64_t c0 = r0; c0 < r1; c0 += PART_THREADS * SC_STEPS) {
        for (int j = threadIdx.x; j < NW * P; j += blockDim.x) wtot[j] = 0;
        __syncthreads();
        const int64_t b0 = c0 + (int64_t)warp * 32 * SC_STEPS;
        int d[SC_STEPS];
        unsigned int rk[SC_STEPS];
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            const int64_t i = b0 + s * 32 + lane;
            const bool in = i < r1;
            d[s] = in ? (int)a.dest8[i] : -1;
            const unsigned peers = __match_any_sync(0xffffffffu, d[s]);
            const int rank = __popc(peers & ((1u << lane) - 1));
            const bool leader = in && rank == 0;
            unsigned int old = leader ? wtot[warp * P + d[s]] : 0u;
            if (leader) wtot[warp * P + d[s]] = old + (unsigned int)__popc(peers);
            old = __shfl_sync(0xffffffffu, old, __ffs(peers) - 1);
            rk[s] = old + (unsigned int)rank;
            __syncwarp();
        }
        __syncthreads();
        long long pos[SC_STEPS];
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            pos[s] = 0;
            if (d[s] < 0) continue;
            unsigned int before = 0;
            for (int w = 0; w < warp; w++) before += wtot[w * P + d[s]];
            pos[s] = run[d[s]] + before + rk[s];
        }
        __syncthreads();
        for (int e = threadIdx.x; e < P; e += blockDim.x) {  // advance the per-destination cursors by this chunk's totals
            unsigned int t = 0;
            for (int w = 0; w < NW; w++) t += wtot[w * P + e];
            run[e] += t;
        }
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            if (d[s] < 0) continue;
            const int64_t i = b0 + s * 32 + lane;
            const long long p = pos[s];
            if (a.perm_out) a.perm_out[p] = i;
            for (int c = 0; c < a.n_cols; c++) {
                switch (a.itemsize[c]) {
                    case 8: ((uint64_t*)a.out_data[c])[p] = __ldcs((const unsigned long long*)a.in_data[c] + i); break;
                    case 4: ((uint32_t*)a.out_data[c])[p] = __ldcs((const unsigned int*)a.in_data[c] + i); break;
                    case 2: ((uint16_t*)a.out_data[c])[p] = ((const uint16_t*)a.in_data[c])[i]; break;
                    default: ((uint8_t*)a.out_data[c])[p] = ((const uint8_t*)a.in_data[c])[i]; break;
                }
                if (a.out_valid_bytes[c]) a.out_valid_bytes[c][p] = bit_valid(a.in_valid[c], i) ? 1 : 0;
            }
        }
        __syncthreads();
    }
}

// K3, specialised: at most 8 destinations (one NVLink box), NC 8-byte columns without validity bitmaps.  Same row order as
// scatter_kernel, but the stable rank comes from eight ballots per 32 rows and the warp's running per-destination counts live
// in registers (16-bit fields of two 64-bit words, identical in every lane): no shared-memory traffic and no warp barrier in
// the ranking loop, one 16-byte shared store per warp and three CTA barriers per 2048-row chunk.
template <int NC>
__global__ void __launch_bounds__(PART_THREADS) scatter_small_kernel(const __grid_constant__ ScatterArgs a) {
    constexpr int NW = PART_THREADS / 32;
    __shared__ long long run[8];
    __shared__ unsigned long long wtot[NW][2];  // per warp: rows per destination of its block, 16-bit fields
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, P = a.n_pes;
    if (threadIdx.x < 8) run[threadIdx.x] = threadIdx.x < P ? a.offsets[(size_t)blockIdx.x * P + threadIdx.x] : 0;
    const int64_t r0 = (int64_t)blockIdx.x * a.tile_rows;
    const int64_t r1 = r0 + a.tile_rows < a.n ? r0 + a.tile_rows : a.n;
    const unsigned lt = (1u << lane) - 1;
    for (int64_t c0 = r0; c0 < r1; c0 += PART_THREADS * SC_STEPS) {
        const int64_t b0 = c0 + (int64_t)warp * 32 * SC_STEPS;
        int d[SC_STEPS];
        unsigned long long v[NC][SC_STEPS];
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {  // all loads of the chunk are issued before anything depends on them
            const int64_t i = b0 + s * 32 + lane;
            d[s] = i < r1 ? (int)a.dest8[i] : 8;
#pragma unroll
            for (int c = 0; c < NC; c++) v[c][s] = i < r1 ? __ldcs((const unsigned long long*)a.in_data[c] + i) : 0ull;
        }
        unsigned long long cl = 0, ch = 0;  // rows per destination this warp has ranked so far (dests 0-3 / 4-7)
        unsigned int rk[SC_STEPS];
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            unsigned int mine = 0;
            unsigned long long al = 0, ah = 0;
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const unsigned b = __ballot_sync(0xffffffffu, d[s] == e);
                if (d[s] == e) mine = (unsigned int)__popc(b & lt);
                if (e < 4) al += (unsigned long long)__popc(b) << (16 * e);
                else ah += (unsigned long long)__popc(b) << (16 * (e - 4));
            }
            const unsigned long long w = (d[s] & 4) ? ch : cl;
            rk[s] = mine + (unsigned int)((w >> (16 * (d[s] & 3))) & 0xffffu);
            cl += al; ch += ah;
        }
        if (lane == 0) { wtot[warp][0] = cl; wtot[warp][1] = ch; }
        __syncthreads();
        unsigned long long bl = 0, bh = 0;  // rows of the warps before this one
        for (int w = 0; w < warp; w++) { bl += wtot[w][0]; bh += wtot[w][1]; }
        long long pos[SC_STEPS];
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            const unsigned long long w = (d[s] & 4) ? bh : bl;
            pos[s] = d[s] < 8 ? run[d[s]] + (long long)((w >> (16 * (d[s] & 3))) & 0xffffu) + rk[s] : 0;
        }
        __syncthreads();
        if (threadIdx.x < 8) {
            unsigned long long t = 0;
            for (int w = 0; w < NW; w++) t += (wtot[w][threadIdx.x >> 2] >> (16 * (threadIdx.x & 3))) & 0xffffull;
            run[threadIdx.x] += (long long)t;
        }
#pragma unroll
        for (int s = 0; s < SC_STEPS; s++) {
            if (d[s] >= 8) continue;
            if (a.perm_out) a.perm_out[pos[s]] = b0 + s * 32 + lane;
#pragma unroll
            for (int c = 0; c < NC; c++) ((unsigned long long*)a.out_data[c])[pos[s]] = v[c][s];
        }
        __syncthreads();
    }
}

// K4: one thread per output bitmap byte of a destination segment.
__global__ void pack_segment_bitmaps_kernel(const uint8_t* valid_bytes, const long long* totals, int n_pes, uint8_t* out_bitmap) {
    // segment d: rows [row_off[d], row_off[d] + totals[d]) -> bytes [byte_off[d], byte_off[d] + ceil(totals[d] / 8))
    long long row_off = 0, byte_off = 0;
    for (int d = 0; d < n_pes; d++) {
        long long cnt = totals[d];
        long long nbytes = (cnt + 7) >> 3;
        for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < nbytes; b += (long long)gridDim.x * blockDim.x) {
            unsigned v = 0;
            for (int k = 0; k < 8; k++) {
                long long r = b * 8 + k;
                if (r < cnt && valid_bytes[row_off + r]) v |= 1u << k;
            }
            out_bitmap[byte_off + b] = (uint8_t)v;
        }
        row_off += cnt;
        byte_off += nbytes;
    }
}

// Receive side of the shuffle: the per-source validity segments (each padded to a byte boundary, in source-rank order)
// become one contiguous Arrow bitmap for the received rows.
__global__ void merge_segment_bitmaps_kernel(const uint8_t* __restrict__ in, const long long* __restrict__ row_off /* n_src + 1 */,
                                             const long long* __restrict__ byte_off /* n_src */, int n_src, uint32_t* out_words) {
    __shared__ long long s_row[MAX_PES + 1];
    __shared__ long long s_byte[MAX_PES];
    for (int j = threadIdx.x; j <= n_src; j += blockDim.x) s_row[j] = row_off[j];
    for (int j = threadIdx.x; j < n_src; j += blockDim.x) s_byte[j] = byte_off[j];
    __syncthreads();
    const long long n = s_row[n_src];
    const long long n_round = (n + 31) & ~31ll;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_round; i += (long long)gridDim.x * blockDim.x) {
        bool bit = false;
        if (i < n) {
            int lo = 0, hi = n_src - 1;  // last source whose first row is <= i
            while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (s_row[mid] <= i) lo = mid; else hi = mid - 1; }
            long long r = i - s_row[lo];
            bit = (in[s_byte[lo] + (r >> 3)] >> (r & 7)) & 1;
        }
        unsigned m = __ballot_sync(0xffffffffu, bit);
        if ((threadIdx.x & 31) == 0) out_words[i >> 5] = m;
    }
}

struct StreamBuf {  // stream-ordered scratch allocation
    void* p = nullptr;
    cudaStream_t s;
    StreamBuf(size_t n, cudaStream_t st) : s(st) { B200_CUDA(cudaMallocAsync(&p, n ? n : 8, st)); }
    ~StreamBuf() { if (p) cudaFreeAsync(p, s); }
    template <typename T> T* as() { return (T*)p; }
};

static int table_device(const b200_table* t) {
    B200_REQUIRE(t->device >= 0, "b200 shuffle: the table must be device resident");
    return t->device;
}
// the first n_keys columns as a KeySet: 4- / 8-byte integer, date and float columns, and with narrow = true also 1- and 2-byte
// integer and bool columns (the key-class placement)
static KeySet make_keyset(const b200_table* t, int n_keys, bool narrow = false) {
    KeySet k{};
    k.n_keys = n_keys;
    for (int j = 0; j < n_keys; j++) {
        const b200_column& c = t->cols[j];
        if (narrow)
            B200_REQUIRE(ctype_size(c.c_type) >= 1 && ctype_size(c.c_type) <= 8, "b200 shuffle: key columns must be fixed-width integer, bool, date, time or float columns");
        else
            B200_REQUIRE(ctype_size(c.c_type) == 4 || ctype_size(c.c_type) == 8, "b200 shuffle: key columns must be 4- or 8-byte integer, date or float columns");
        k.data[j] = c.data; k.valid[j] = c.validity; k.ctype[j] = c.c_type;
    }
    return k;
}

// classes = false: the reference's placement (ReferenceKeyHash); true: one rank per key class (KeyClassHash).
void shuffle_partition(const b200_table* in, int64_t n_keys, int n_pes, b200_table* out, int64_t* send_counts,
                       long long* perm_out_dev, cudaStream_t st, bool classes = false) {
    B200_REQUIRE(n_keys >= 1 && n_keys <= MAX_HASH_KEYS && n_keys <= in->n_cols, "b200 shuffle: between 1 and 4 key columns are supported");
    B200_REQUIRE(n_pes >= 1 && n_pes <= MAX_PES, "b200 shuffle: n_pes must be in [1, 256]");
    B200_REQUIRE(in->n_cols >= 1 && in->n_cols <= MAX_SHUFFLE_COLS, "b200 shuffle: between 1 and 32 columns are supported");
    B200_REQUIRE(out->n_cols == in->n_cols, "b200 shuffle: out table must have the same number of columns");
    int dev = table_device(in);
    B200_CUDA(cudaSetDevice(dev));
    int64_t n = in->n_rows;
    KeySet ks = make_keyset(in, (int)n_keys, classes);
    for (int d = 0; d < n_pes; d++) send_counts[d] = 0;
    out->n_rows = n;
    if (n == 0) return;
    int sms = num_sms(dev);
    int n_ctas = (int)std::min<int64_t>((int64_t)sms * 8, (n + PART_THREADS - 1) / PART_THREADS);
    const int64_t chunk = (int64_t)PART_THREADS * SC_STEPS;
    int64_t tile_rows = ((n + n_ctas - 1) / n_ctas + chunk - 1) / chunk * chunk;
    n_ctas = (int)((n + tile_rows - 1) / tile_rows);
    StreamBuf dest8((size_t)n, st), hist((size_t)n_ctas * n_pes * 4, st), offsets((size_t)n_ctas * n_pes * 8, st), totals((size_t)n_pes * 8, st);
    if (classes)
        dest_hist_kernel<KeyClassHash><<<n_ctas, PART_THREADS, 0, st>>>(ks, n, tile_rows, n_pes, dest8.as<uint8_t>(), hist.as<unsigned int>());
    else
        dest_hist_kernel<ReferenceKeyHash><<<n_ctas, PART_THREADS, 0, st>>>(ks, n, tile_rows, n_pes, dest8.as<uint8_t>(), hist.as<unsigned int>());
    B200_CUDA(cudaGetLastError());
    scan_hist_kernel<<<1, 1024, 0, st>>>(hist.as<unsigned int>(), n_ctas, n_pes, offsets.as<long long>(), totals.as<long long>());
    B200_CUDA(cudaGetLastError());
    ScatterArgs a{};
    a.n = n; a.tile_rows = tile_rows; a.n_pes = n_pes; a.n_cols = in->n_cols; a.dest8 = dest8.as<uint8_t>();
    a.offsets = offsets.as<long long>(); a.perm_out = perm_out_dev;
    std::vector<StreamBuf*> vbytes(in->n_cols, nullptr);
    for (int c = 0; c < in->n_cols; c++) {
        const b200_column& ic = in->cols[c];
        b200_column& oc = out->cols[c];
        B200_REQUIRE(ctype_size(ic.c_type) > 0, "b200 shuffle: unsupported column dtype");
        B200_REQUIRE(oc.data != nullptr, "b200 shuffle: out column data pointer is null");
        a.in_data[c] = ic.data; a.in_valid[c] = ic.validity; a.out_data[c] = oc.data; a.itemsize[c] = ctype_size(ic.c_type);
        a.out_valid_bytes[c] = nullptr;
        if (ic.validity) {
            B200_REQUIRE(oc.validity != nullptr, "b200 shuffle: out column needs a validity buffer of ceil(n/8) + n_pes bytes");
            vbytes[c] = new StreamBuf((size_t)n, st);
            a.out_valid_bytes[c] = vbytes[c]->as<uint8_t>();
        }
        oc.length = n; oc.c_type = ic.c_type; oc.arr_type = ic.arr_type;
    }
    bool small = n_pes <= 8 && in->n_cols <= 4;
    for (int c = 0; c < in->n_cols; c++) small = small && a.itemsize[c] == 8 && !a.in_valid[c];
    if (small) {
        switch (in->n_cols) {
            case 1: scatter_small_kernel<1><<<n_ctas, PART_THREADS, 0, st>>>(a); break;
            case 2: scatter_small_kernel<2><<<n_ctas, PART_THREADS, 0, st>>>(a); break;
            case 3: scatter_small_kernel<3><<<n_ctas, PART_THREADS, 0, st>>>(a); break;
            default: scatter_small_kernel<4><<<n_ctas, PART_THREADS, 0, st>>>(a); break;
        }
    } else {
        scatter_kernel<<<n_ctas, PART_THREADS, 0, st>>>(a);
    }
    B200_CUDA(cudaGetLastError());
    for (int c = 0; c < in->n_cols; c++) {
        if (!vbytes[c]) continue;
        pack_segment_bitmaps_kernel<<<sms * 4, 256, 0, st>>>(vbytes[c]->as<uint8_t>(), totals.as<long long>(), n_pes, out->cols[c].validity);
        delete vbytes[c];
    }
    B200_CUDA(cudaGetLastError());
    std::vector<long long> h(n_pes);
    B200_CUDA(cudaMemcpyAsync(h.data(), totals.p, (size_t)n_pes * 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (int d = 0; d < n_pes; d++) send_counts[d] = h[d];
}

}  // namespace b200

extern "C" {

int b200_hash_to_rank(const b200_table* in_table, int32_t n_pes, int32_t* dest_out, void* stream) {
    return b200_hash_keys_table(in_table, in_table ? 1 : 0, n_pes, dest_out, nullptr, stream);
}

int b200_hash_keys_table(const b200_table* in_table, int64_t n_keys, int32_t n_pes, int32_t* dest_out, uint32_t* hash_out, void* stream) {
    try {
        B200_REQUIRE(in_table && n_keys >= 1 && n_keys <= b200::MAX_HASH_KEYS && in_table->n_cols >= n_keys && n_pes >= 1 && (dest_out || hash_out),
                     "b200_hash_keys_table: bad arguments");
        int dev = b200::table_device(in_table);
        B200_CUDA(cudaSetDevice(dev));
        if (in_table->n_rows == 0) return 0;
        b200::KeySet ks = b200::make_keyset(in_table, (int)n_keys);
        b200::hash_to_rank_kernel<<<b200::num_sms(dev) * 8, 256, 0, (cudaStream_t)stream>>>(ks, in_table->n_rows, n_pes, dest_out, hash_out);
        B200_CUDA(cudaGetLastError());
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_shuffle_partition(const b200_table* in_table, int64_t n_keys, int32_t n_pes, b200_table* out, int64_t* send_counts,
                           void* stream) {
    try {
        B200_REQUIRE(in_table && out && send_counts, "b200_shuffle_partition: null argument");
        b200::shuffle_partition(in_table, n_keys, n_pes, out, send_counts, nullptr, (cudaStream_t)stream);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_merge_segment_bitmaps(const uint8_t* segments, const int64_t* counts, int32_t n_src, uint8_t* out_bitmap, int32_t device, void* stream) {
    try {
        B200_REQUIRE(segments && counts && out_bitmap && n_src >= 1 && n_src <= b200::MAX_PES, "b200_merge_segment_bitmaps: bad arguments");
        B200_CUDA(cudaSetDevice(device)); b200::scratch_set_stream((cudaStream_t)stream);
        std::vector<long long> row_off(n_src + 1, 0), byte_off(n_src, 0);
        long long bytes = 0;
        for (int j = 0; j < n_src; j++) { row_off[j + 1] = row_off[j] + counts[j]; byte_off[j] = bytes; bytes += (counts[j] + 7) >> 3; }
        if (row_off[n_src] == 0) return 0;
        cudaStream_t st = (cudaStream_t)stream;
        b200::StreamBuf d_row((size_t)(n_src + 1) * 8, st), d_byte((size_t)n_src * 8, st);
        B200_CUDA(cudaMemcpyAsync(d_row.p, row_off.data(), (size_t)(n_src + 1) * 8, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemcpyAsync(d_byte.p, byte_off.data(), (size_t)n_src * 8, cudaMemcpyHostToDevice, st));
        b200::merge_segment_bitmaps_kernel<<<b200::num_sms(device) * 4, 256, 0, st>>>(segments, d_row.as<long long>(), d_byte.as<long long>(), n_src, (uint32_t*)out_bitmap);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(st));  // row_off / byte_off are stack buffers
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_shuffle_partition_perm(const b200_table* in_table, int64_t n_keys, int32_t n_pes, b200_table* out, int64_t* send_counts,
                                int64_t* perm_out_dev, void* stream) {
    try {
        B200_REQUIRE(in_table && out && send_counts, "b200_shuffle_partition_perm: null argument");
        b200::shuffle_partition(in_table, n_keys, n_pes, out, send_counts, (long long*)perm_out_dev, (cudaStream_t)stream);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_shuffle_partition_classes(const b200_table* in_table, int64_t n_keys, int32_t n_pes, b200_table* out, int64_t* send_counts,
                                   int64_t* perm_out_dev, void* stream) {
    try {
        B200_REQUIRE(in_table && out && send_counts, "b200_shuffle_partition_classes: null argument");
        b200::shuffle_partition(in_table, n_keys, n_pes, out, send_counts, (long long*)perm_out_dev, (cudaStream_t)stream, true);
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

}  // extern "C"
