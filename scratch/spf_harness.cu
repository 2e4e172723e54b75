// spf_harness.cu — runs the fused SM-partitioned kernel (spf_groupby_kernel, bodo_b200/csrc/spf.cuh) on synthetic rows outside
// the operator state machine: CUDA-event time per launch, achieved fraction of the 16 B/row roofline, and an EXACT per-group
// check against a dense reference built with plain global atomics.  Development tool, not part of the library.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -I bodo_b200/csrc \
//        scratch/spf_harness.cu bodo_b200/csrc/misc.cu -o scratch/spf_harness
//   scratch/spf_harness [log2_rows=27] [groups=1000000] [reps=3] [extra_rows=0] [zipf=0]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../bodo_b200/csrc/groupby.cu"

using namespace b200;

__global__ void h_fill(long long* keys, long long* vals, int64_t n, uint64_t n_groups, int skew) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint64_t r = mix64((uint64_t)i ^ 0x9e3779b97f4a7c15ULL);
        uint64_t k = r % n_groups;
        if (skew && (r >> 40) % 100 < (uint64_t)skew) k = k % 7;  // `skew` percent of the rows fall on 7 hot keys
        keys[i] = (long long)k * 2654435761ll - 77;                // not dense, negative ones too
        vals[i] = (long long)(mix64((uint64_t)i ^ 0xd1b54a32d192ed03ULL * 2) % 1000) - 500;
        if ((i & 0xfffff) == 12345) vals[i] = (long long)0x7fffffff12345678ll;  // exercise the high-word path
    }
}
__global__ void h_fill_u64(unsigned long long* p, size_t n, unsigned long long v) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
// dense reference: ref[key index] via atomics (key index recovered from the synthetic key)
__global__ void h_ref(const long long* keys, const long long* vals, int64_t n, unsigned long long* rsum, unsigned long long* rcnt) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        long long g = (keys[i] + 77) / 2654435761ll;
        atomicAdd(rsum + g, (unsigned long long)vals[i]);
        atomicAdd(rcnt + g, 1ull);
    }
}
__global__ void h_verify(const long long* tkeys, uint64_t cap, const unsigned long long* asum, const unsigned long long* acnt,
                         const unsigned long long* rsum, const unsigned long long* rcnt, unsigned long long reps, uint64_t n_groups, unsigned long long* out) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < cap; s += (uint64_t)gridDim.x * blockDim.x) {
        long long k = tkeys[s];
        if (k == EMPTY_KEY) continue;
        long long g = (k + 77) / 2654435761ll;
        bool ok = g >= 0 && (uint64_t)g < n_groups && (g * 2654435761ll - 77) == k && asum[s] == rsum[g] * reps && acnt[s] == rcnt[g] * reps;
        atomicAdd(out + (ok ? 0 : 1), 1ull);
    }
}
__global__ void h_count_nonzero(const unsigned long long* rcnt, uint64_t n, unsigned long long* out) {
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < n; s += (uint64_t)gridDim.x * blockDim.x) if (rcnt[s]) atomicAdd(out, 1ull);
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

int main(int argc, char** argv) {
    const int lg = argc > 1 ? atoi(argv[1]) : 27;
    const uint64_t groups = argc > 2 ? strtoull(argv[2], nullptr, 10) : 1000000ull;
    const int reps = argc > 3 ? atoi(argv[3]) : 3;
    const int64_t extra = argc > 4 ? atoll(argv[4]) : 0;  // rows beyond 2^lg (exercises the partial last tile)
    const int skew = argc > 5 ? atoi(argv[5]) : 0;
    const int64_t rows = (1ll << lg) + extra;
    int dev = 0, sms = 0, max_smem = 0, coop = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    const int G = sms;
    const int ns = (int)(((size_t)max_smem - SpfSmemLayout::table) / 16) & ~1;
    const size_t smem = SpfSmemLayout::table + (size_t)ns * 16;
    printf("SMs %d, smem/CTA %zu B, table slots/CTA %d (capacity at 80%% load: %.0f groups), coop %d\n", sms, smem, ns, 0.8 * ns * G, coop);

    long long *keys, *vals, *tkeys, *counters;
    unsigned long long *acc_sum, *acc_cnt, *retry, *chk, *rsum, *rcnt, *tile_ctr;
    longlong2* ring; unsigned int *pub, *cons;
    uint64_t cap = 1ull << 22;
    while (cap < 4 * groups) cap <<= 1;
    CK(cudaMalloc(&keys, rows * 8)); CK(cudaMalloc(&vals, rows * 8));
    CK(cudaMalloc(&tkeys, (cap + 2) * 8)); CK(cudaMalloc(&acc_sum, (cap + 2) * 8)); CK(cudaMalloc(&acc_cnt, (cap + 2) * 8));
    CK(cudaMalloc(&counters, 64)); CK(cudaMalloc(&chk, 32)); CK(cudaMalloc(&tile_ctr, 16));
    CK(cudaMalloc(&rsum, groups * 8)); CK(cudaMalloc(&rcnt, groups * 8));
    CK(cudaMalloc(&ring, (size_t)G * G * SPF_R * 16)); CK(cudaMalloc(&pub, (size_t)G * G * 4)); CK(cudaMalloc(&cons, (size_t)G * G * 4));
    CK(cudaMalloc(&retry, (size_t)SPF_RETRY_HARD * 32));
    h_fill<<<sms * 8, 256>>>(keys, vals, rows, groups, skew);
    h_fill_u64<<<sms * 8, 256>>>((unsigned long long*)tkeys, cap + 2, (unsigned long long)EMPTY_KEY);
    CK(cudaMemset(acc_sum, 0, (cap + 2) * 8)); CK(cudaMemset(acc_cnt, 0, (cap + 2) * 8)); CK(cudaMemset(counters, 0, 64));
    CK(cudaMemset(rsum, 0, groups * 8)); CK(cudaMemset(rcnt, 0, groups * 8));
    h_ref<<<sms * 8, 256>>>(keys, vals, rows, rsum, rcnt);
    CK(cudaDeviceSynchronize());

    SpfArgs fa{};
    SpgArgs& a = fa.g;
    a.keys = keys; a.vals = vals; a.n_rows = rows; a.n_owners = G;
    a.tkeys = tkeys; a.cap = cap; a.acc_sum = acc_sum; a.acc_cnt = acc_cnt; a.counters = counters; a.group_limit = (long long)(cap / 2);
    a.retry = retry; a.retry_ctr = counters + 1; a.sum_first = 1;
    fa.ring = ring; fa.pub = pub; fa.cons = cons; fa.tile_ctr = tile_ctr; fa.ns = ns;
    unsigned long long* stats; CK(cudaMalloc(&stats, 512)); CK(cudaMemset(stats, 0, 512)); fa.stats = stats;
    auto kfn = (const void*)spf_groupby_kernel<true, true>;
    CK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spf_groupby_kernel<true, true>, SPF_THREADS, smem));
    printf("occupancy: %d CTA/SM\n", occ);

    std::vector<float> t;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int r = 0; r < reps + 1; r++) {
        CK(cudaMemsetAsync(pub, 0, (size_t)G * G * 4)); CK(cudaMemsetAsync(cons, 0, (size_t)G * G * 4)); CK(cudaMemsetAsync(tile_ctr, 0, 8)); CK(cudaMemsetAsync(tile_ctr + 1, 0xff, 8));
        CK(cudaEventRecord(e0));
        void* params[] = {(void*)&fa};
        CK(cudaLaunchCooperativeKernel(kfn, dim3(G), dim3(SPF_THREADS), params, smem, 0));
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (r > 0) t.push_back(ms); else printf("first (cold) launch: %.3f ms\n", ms);
    }
    std::sort(t.begin(), t.end());
    CK(cudaMemset(chk, 0, 32));
    h_verify<<<sms * 4, 256>>>(tkeys, cap, acc_sum, acc_cnt, rsum, rcnt, (unsigned long long)(reps + 1), groups, chk);
    h_count_nonzero<<<sms * 4, 256>>>(rcnt, groups, chk + 2);
    unsigned long long h[4]; long long hc[8]; unsigned long long tc[2];
    CK(cudaMemcpy(h, chk, 32, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hc, counters, 64, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tc, tile_ctr, 16, cudaMemcpyDeviceToHost));
    const bool ok = h[1] == 0 && h[0] == h[2] && hc[1] == 0 && (long long)h[0] == hc[0];
    const float med = t[t.size() / 2];
    printf("{\"rows\": %lld, \"groups\": %llu, \"skew_pct\": %d, \"ms\": {\"min\": %.4f, \"median\": %.4f}, \"grows_per_s\": %.2f, \"roofline_frac\": %.4f, "
           "\"groups_ok\": %llu, \"groups_bad\": %llu, \"groups_expected\": %llu, \"table_groups\": %lld, \"retry_rows\": %lld, \"tiles_claimed\": %llu, \"abort\": %llu, \"check\": \"%s\"}\n",
           (long long)rows, (unsigned long long)groups, skew, t[0], med, rows / (med * 1e-3) / 1e9, rows * 16.0 / (med * 1e-3) / 3350e9 /* H100 SXM data-sheet HBM bandwidth */,
           h[0], h[1], h[2], hc[0], hc[1], tc[0], tc[1], ok ? "ok" : "MISMATCH");
#ifdef SPF_STATS
    unsigned long long st[64]; CK(cudaMemcpy(st, stats, 512, cudaMemcpyDeviceToHost));
    const double L = reps + 1, cwn = (double)G * SPF_NCW;
    printf("stats per launch: consumer polls per warp: empty %.0f, with work %.0f (lines per working poll %.2f), kick phases per warp %.1f\n",
           st[6] / L / cwn, st[7] / L / cwn, st[7] ? (double)st[8] / st[7] : 0.0, st[4] / L / cwn);
    printf("  producer slot waits: %.0f events per CTA, %.3f Mcycles per CTA (summed over threads)\n", st[41] / L / G, st[40] / L / G / 1e6);
    printf("  flusher ring-full waits: %.0f events per CTA, %.3f Mcycles per CTA (summed over group leaders)\n", st[43] / L / G, st[42] / L / G / 1e6);
    printf("  publisher: %.0f fence+publish rounds per CTA, %.0f cycles per fence\n", st[45] / L / G, st[45] ? (double)st[44] / st[45] : 0.0);
    printf("  flusher lines per busy iteration %.2f\n", st[11] ? (double)st[10] / st[11] : 0.0);
#endif
    return ok ? 0 : 3;
}
