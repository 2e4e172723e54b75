// spg_harness.cu — times an SM-partitioned groupby kernel pair in isolation, outside the operator state machine, so kernel
// variants can be compared with one short GPU run each.  Development tool, not part of the library: it includes groupby.cu to
// reach the kernels and links misc.cu for the buffer pool.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -I bodo_b200/csrc \
//        scratch/spg_harness.cu bodo_b200/csrc/misc.cu -o scratch/spg_harness
//   scratch/spg_harness [pair=n] [log2_rows=28] [groups=1000000] [reps=5] [cnt_stride_pad_bytes=0] [keys=d]
//
// pair n: the narrow-row pair (K1n spgn_partition_kernel + K2n spgn_aggregate_kernel), launched as GroupbyState::consume_spg
//         launches it for the flagship (SpgArgs as the host fills them, 2^28 rows = one launch, first launch with ticket
//         reservation).  pair w: the 16-byte pair (K1 spg_partition_tma_kernel + K2 spg_aggregate_kernel) that the heavy-hitter and
//         wide-row paths run.
// Keys are uniform over `groups`, values uniform in [-500, 500), as bodo_b200/synth.py produces them.  keys=s scrambles them:
// each key k becomes mix64(k) truncated to 31 bits (still narrow), so the buckets see keys that a dense range does not model.  Prints per-kernel
// CUDA-event times (min / median over reps, the first, cold repetition excluded), each kernel's design bytes over its median
// time, a plain device copy (read the 16-byte row, write an 8-byte row) timed in the same process as the practical bandwidth
// ceiling, and checks SUM/COUNT totals against the input (the result must be exact).
// K2n is built with SPGN_PHASE_CLOCKS: the output also gives, per launch, where K2n's CTAs spend their SM clocks (table init,
// row loop, flush; mean and max over CTAs, medians over reps).  Building with -DSPGN_SKIP_FLUSH times K2n without its flush
// (the check then fails by design).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define SPGN_PHASE_CLOCKS
#include "../bodo_b200/csrc/groupby.cu"

using namespace b200;

__global__ void harness_fill_kernel(long long* keys, long long* vals, int64_t n, uint64_t n_groups, bool scramble) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint64_t k = mix64((uint64_t)i ^ 0x9e3779b97f4a7c15ULL) % n_groups;
        keys[i] = (long long)(scramble ? mix64(k) & 0x7fffffffULL : k);
        vals[i] = (long long)(mix64((uint64_t)i ^ 0xd1b54a32d192ed03ULL * 2) % 1000) - 500;
    }
}
__global__ void harness_fill_u64(unsigned long long* p, size_t n, unsigned long long v) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void harness_sum_kernel(const long long* v, int64_t n, unsigned long long* out) {
    unsigned long long s = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) s += (unsigned long long)v[i];
    atomicAdd(out, s);
}
// the copy-rate reference: K1n's design traffic without its work (16-byte loads of two rows' keys and values, one 16-byte store)
__global__ void harness_copy_kernel(const longlong2* __restrict__ keys, const longlong2* __restrict__ vals, int4* __restrict__ out, int64_t n2) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n2; i += (int64_t)gridDim.x * blockDim.x) {
        const longlong2 k = __ldcs(keys + i), v = __ldcs(vals + i);
        __stcs(out + i, make_int4((int)k.x, (int)v.x, (int)k.y, (int)v.y));
    }
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

static float median(std::vector<float> v) { std::sort(v.begin(), v.end()); return v[v.size() / 2]; }
static float minimum(const std::vector<float>& v) { return *std::min_element(v.begin(), v.end()); }

int main(int argc, char** argv) {
    const bool narrow = argc > 1 ? strcmp(argv[1], "w") != 0 : true;
    const int lg = argc > 2 ? atoi(argv[2]) : 28;
    const uint64_t groups = argc > 3 ? strtoull(argv[3], nullptr, 10) : 1000000ull;
    const int reps = argc > 4 ? atoi(argv[4]) : 5;
    const size_t pad = argc > 5 ? strtoull(argv[5], nullptr, 10) : 0;  // shifts the owner row counters inside their allocation
    const bool scramble = argc > 6 && strcmp(argv[6], "s") == 0;
    const int64_t rows = 1ll << lg;
    int dev = 0, sms = 0, max_smem = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const int owners = sms;
    // shared-table sizes and K1 shapes exactly as GroupbyState::spg_probe / consume_spg compute them
    const int spg_ns = ((int)(((size_t)max_smem - 64) / 16) - SPG_STASH) & ~1;
    const int spgn_ns = ((int)(((size_t)max_smem - 256 - SPGN_QUEUE_BYTES) / 12) - SPG_STASH) & ~1;
    const int ns = narrow ? spgn_ns : spg_ns;
    const size_t k2_smem = narrow ? (size_t)(spgn_ns + SPG_STASH) * 12 + SPGN_QUEUE_BYTES + 16 : (size_t)(spg_ns + SPG_STASH) * 16 + 16;
    const size_t k1_smem = narrow ? SpgnK1Smem<false>::bytes : SpgK1Smem<false>::bytes;
    const int tile = narrow ? SPGN_TILE : SPG_TILE, k1_threads = SPG_TTHREADS, k1_ctas = narrow ? SPGN_CTAS : SPG_TCTAS;
    const int g1 = (int)std::min<int64_t>((int64_t)sms * k1_ctas, (rows + tile - 1) / tile);
    const int64_t group_cap = (int64_t)owners * (narrow ? spgn_ns * 7 / 10 : spg_ns * 7 / 10);
    const int n_pass = (int)std::min<int64_t>(24, std::max<int64_t>(1, ((int64_t)groups + group_cap - 1) / group_cap));

    long long *keys, *vals, *tkeys, *counters;
    unsigned long long *acc_sum, *acc_cnt, *bucket_cnt_raw, *retry, *chk;
    longlong2* bucket;
    const uint64_t cap = 1ull << 22;
    CK(cudaMalloc(&keys, rows * 8)); CK(cudaMalloc(&vals, rows * 8));
    CK(cudaMalloc(&tkeys, (cap + 2) * 8)); CK(cudaMalloc(&acc_sum, (cap + 2) * 8)); CK(cudaMalloc(&acc_cnt, (cap + 2) * 8));
    CK(cudaMalloc(&counters, 64)); CK(cudaMalloc(&chk, 16));
    const int64_t bucket_cap = rows / owners + rows / owners / 8 + 4096;
    CK(cudaMalloc(&bucket, (size_t)owners * bucket_cap * 16));
    CK(cudaMalloc(&bucket_cnt_raw, (size_t)owners * SPG_CNT_STRIDE * 8 + pad + 256));
    CK(cudaMalloc(&retry, ((size_t)rows + (size_t)owners * spg_ns) * 32));
    unsigned long long* bucket_cnt = (unsigned long long*)((char*)bucket_cnt_raw + pad);
    harness_fill_kernel<<<sms * 8, 256>>>(keys, vals, rows, groups, scramble);
    harness_fill_u64<<<sms * 8, 256>>>((unsigned long long*)tkeys, cap + 2, (unsigned long long)EMPTY_KEY);
    CK(cudaMemset(acc_sum, 0, (cap + 2) * 8)); CK(cudaMemset(acc_cnt, 0, (cap + 2) * 8)); CK(cudaMemset(counters, 0, 64));
    CK(cudaDeviceSynchronize());

    SpgArgs a{};
    a.keys = keys; a.vals = vals; a.n_rows = rows; a.n_owners = owners;
    a.tkeys = tkeys; a.cap = cap; a.acc_sum = acc_sum; a.acc_cnt = acc_cnt; a.counters = counters; a.group_limit = (long long)(cap / 2);
    a.bucket = bucket; a.bucket_cnt = bucket_cnt; a.bucket_cap = narrow ? bucket_cap & ~1ll : bucket_cap; a.retry = retry; a.retry_ctr = counters + 1;
    a.sum_first = 1; a.ns = ns; a.n_pass = narrow ? n_pass : 1;

    const void* k1 = narrow ? (const void*)spgn_partition_kernel<true, true> : (const void*)spg_partition_tma_kernel<true, true>;
    const void* k2 = narrow ? (const void*)spgn_aggregate_kernel<true, true> : (const void*)spg_aggregate_kernel<true, true>;
    CK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k1_smem));
    CK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k2_smem));

    std::vector<float> t1, t2, tc;
    std::vector<float> ph_mean[3], ph_max[3];  // K2n phase clocks per launch
    std::vector<unsigned long long> ph((size_t)SPG_MAX_OWNERS * 4);
    cudaEvent_t e0, e1, e2;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    for (int r = 0; r < reps + 1; r++) {  // the first repetition (table inserts, cold) is not reported
        // the host reserves group tickets only for the first flush into an empty table
        a.reserve_tickets = narrow && r == 0 && (int64_t)groups + (int64_t)groups / 4 <= (int64_t)(cap / 2) ? 1 : 0;
        CK(cudaMemsetAsync(bucket_cnt, 0, (size_t)owners * SPG_CNT_STRIDE * 8));
        if (narrow) { std::fill(ph.begin(), ph.end(), 0ull); CK(cudaMemcpyToSymbol(spgn_phase_clocks, ph.data(), ph.size() * 8)); }
        CK(cudaEventRecord(e0));
        if (narrow) {
            spgn_partition_kernel<true, true><<<g1, k1_threads, k1_smem>>>(a);
            CK(cudaEventRecord(e1));
            spgn_aggregate_kernel<true, true><<<owners, SPG_THREADS, k2_smem>>>(a);
        } else {
            spg_partition_tma_kernel<true, true><<<g1, k1_threads, k1_smem>>>(a);
            CK(cudaEventRecord(e1));
            spg_aggregate_kernel<true, true><<<owners, SPG_THREADS, k2_smem>>>(a);
        }
        CK(cudaEventRecord(e2));
        CK(cudaEventSynchronize(e2));
        CK(cudaGetLastError());
        float a1 = 0, a2 = 0;
        CK(cudaEventElapsedTime(&a1, e0, e1)); CK(cudaEventElapsedTime(&a2, e1, e2));
        if (r > 0) { t1.push_back(a1); t2.push_back(a2); }
        if (narrow && r > 0) {
            CK(cudaMemcpyFromSymbol(ph.data(), spgn_phase_clocks, ph.size() * 8));
            for (int i = 0; i < 3; i++) {
                double sum = 0, mx = 0;
                for (int c = 0; c < owners; c++) { sum += (double)ph[c * 4 + i]; mx = std::max(mx, (double)ph[c * 4 + i]); }
                ph_mean[i].push_back((float)(sum / owners)); ph_max[i].push_back((float)mx);
            }
        }
    }
    // totals: SUM of sums and SUM of counts over the table must equal (reps + 1) x the input totals
    CK(cudaMemset(chk, 0, 16));
    harness_sum_kernel<<<sms * 4, 256>>>((const long long*)acc_cnt, (int64_t)cap + 2, chk);
    harness_sum_kernel<<<sms * 4, 256>>>((const long long*)acc_sum, (int64_t)cap + 2, chk + 1);
    unsigned long long h[2], hin = 0, *din;
    CK(cudaMemcpy(h, chk, 16, cudaMemcpyDeviceToHost));
    CK(cudaMalloc(&din, 8)); CK(cudaMemset(din, 0, 8));
    harness_sum_kernel<<<sms * 4, 256>>>(vals, rows, din);
    CK(cudaMemcpy(&hin, din, 8, cudaMemcpyDeviceToHost));
    long long hc[8];
    CK(cudaMemcpy(hc, counters, 64, cudaMemcpyDeviceToHost));
    const bool ok = h[0] == (unsigned long long)rows * (reps + 1) && h[1] == hin * (unsigned long long)(reps + 1) && hc[1] == 0 && hc[5] == 0;

    // copy rate into the (now unused) bucket array, same process, same reps
    for (int r = 0; r < reps + 1; r++) {
        CK(cudaEventRecord(e0));
        harness_copy_kernel<<<sms * 8, 512>>>((const longlong2*)keys, (const longlong2*)vals, (int4*)bucket, rows / 2);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float c = 0;
        CK(cudaEventElapsedTime(&c, e0, e1));
        if (r > 0) tc.push_back(c);
    }
    const double b1 = narrow ? 24.0 : 48.0, b2 = narrow ? 8.0 : 16.0;  // design bytes per row: K1 reads the row and writes the bucket row, K2 reads it
    const float m1 = median(t1), m2 = median(t2), mc = median(tc);
    const double gbs1 = rows * b1 / (m1 * 1e-3) / 1e9, gbs2 = rows * b2 / (m2 * 1e-3) / 1e9, gbsc = rows * 24.0 / (mc * 1e-3) / 1e9;
    if (narrow)
        printf("{\"k2n_phase_kclk\": {\"init\": [%.1f, %.1f], \"rows\": [%.1f, %.1f], \"flush\": [%.1f, %.1f]}, \"k2n_phase_note\": \"[mean, max] over CTAs, thousands of SM clocks\"}\n",
               median(ph_mean[0]) / 1e3, median(ph_max[0]) / 1e3, median(ph_mean[1]) / 1e3, median(ph_max[1]) / 1e3, median(ph_mean[2]) / 1e3, median(ph_max[2]) / 1e3);
    printf("{\"pair\": \"%s\", \"keys\": \"%s\", \"rows\": %lld, \"groups\": %llu, \"n_pass\": %d, \"k1_shape\": {\"tile\": %d, \"threads\": %d, \"ctas_per_sm\": %d, \"smem\": %zu}, "
           "\"k1_ms\": {\"min\": %.4f, \"median\": %.4f}, \"k2_ms\": {\"min\": %.4f, \"median\": %.4f}, \"copy_ms\": {\"min\": %.4f, \"median\": %.4f}, "
           "\"k1_gbs\": %.1f, \"k2_gbs\": %.1f, \"copy_gbs\": %.1f, \"k1_of_copy\": %.3f, \"k2_of_copy\": %.3f, "
           "\"pair_grows_per_s\": %.2f, \"table_groups\": %lld, \"retry_rows\": %lld, \"wide_rows\": %lld, \"check\": \"%s\"}\n",
           narrow ? "spgn" : "spg", scramble ? "scrambled" : "dense", (long long)rows, (unsigned long long)groups, a.n_pass, tile, k1_threads, k1_ctas, k1_smem,
           minimum(t1), m1, minimum(t2), m2, minimum(tc), mc, gbs1, gbs2, gbsc, gbs1 / gbsc, gbs2 / gbsc,
           rows / ((m1 + m2) * 1e-3) / 1e9, hc[0], hc[1], hc[5], ok ? "ok" : "MISMATCH");
    return ok ? 0 : 3;
}
