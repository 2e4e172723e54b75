// What bounds SPG K2?  Variants of a per-CTA shared-memory aggregate loop over an owner-like stream (scratch).
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
__host__ __device__ inline uint64_t mix64(uint64_t x) { x += 0x9e3779b97f4a7c15ull; x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull; x = (x ^ (x >> 27)) * 0x94d049bb133111ebull; return x ^ (x >> 31); }
__global__ void gen(longlong2* rows, int64_t n, uint64_t ng) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) rows[i] = make_longlong2((long long)(mix64(i) % ng), (long long)(mix64(i ^ 0x1234567ull) % 1000) - 500);
}
// MODE bits: 1 = key probe (LDS.64 + compare, linear), 2 = returning atomic + carry, 4 = CAS-insert on empty
template <int MODE, int THREADS>
__global__ void __launch_bounds__(THREADS, 1) agg(const longlong2* __restrict__ rows, int64_t n_per_cta, int ns, unsigned long long* out) {
    extern __shared__ __align__(16) unsigned char smem[];
    long long* skeys = (long long*)smem;
    unsigned int* slo = (unsigned int*)(skeys + ns);
    unsigned int* scnt = slo + ns;
    for (int s = threadIdx.x; s < ns; s += THREADS) { skeys[s] = (long long)0x8000000000000000ull; slo[s] = 0x80000000u; scnt[s] = 0; }
    __syncthreads();
    const longlong2* src = rows + (int64_t)blockIdx.x * n_per_cta;
    unsigned long long extra = 0;
    for (int64_t p0 = threadIdx.x; p0 < n_per_cta; p0 += 4 * THREADS) {
        longlong2 r[4];
#pragma unroll
        for (int u = 0; u < 4; u++) { int64_t p = p0 + u * THREADS; r[u] = p < n_per_cta ? __ldcs(src + p) : make_longlong2(0, 0); }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            long long key = r[u].x, val = r[u].y;
            uint64_t h = ((uint64_t)key ^ ((uint64_t)key >> 29)) * 0x9E3779B97F4A7C15ull;
            unsigned int s = __umulhi((unsigned int)(h >> 20), (unsigned int)ns);
            if (MODE & 1) {
                for (int probes = 0; probes < 256; probes++) {
                    long long kk = skeys[s];
                    if (kk == key) break;
                    if (kk == (long long)0x8000000000000000ull) {
                        if (MODE & 4) { long long prev = (long long)atomicCAS((unsigned long long*)&skeys[s], 0x8000000000000000ull, (unsigned long long)key); if (prev == (long long)0x8000000000000000ull || prev == key) break; }
                        else break;
                    }
                    s = s + 1 == (unsigned int)ns ? 0u : s + 1;
                }
            }
            unsigned int lo = (unsigned int)(unsigned long long)val, hi = (unsigned int)((unsigned long long)val >> 32);
            if (MODE & 2) {
                unsigned int old = atomicAdd(&slo[s], lo);
                hi += (old + lo < old) ? 1u : 0u;
                if (hi) extra += hi;
            } else {
                atomicAdd(&slo[s], lo);
            }
            atomicAdd(&scnt[s], 1u);
        }
    }
    __syncthreads();
    unsigned long long acc = extra;
    for (int s = threadIdx.x; s < ns; s += THREADS) acc += slo[s] + scnt[s];
    if (acc == 0x1234567) atomicAdd(out, acc);
}
template <typename F> float timeit(F f, int reps = 3) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; r++) { cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b)); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; }
    return best;
}
int main() {
    int64_t n = 1ll << 26; uint64_t ng = 6757;  // per CTA the same ~6.7k distinct keys (like one SPG owner)
    longlong2* rows; unsigned long long* out;
    CK(cudaMalloc(&rows, n * 16)); CK(cudaMalloc(&out, 8));
    gen<<<132 * 8, 256>>>(rows, n, ng); CK(cudaDeviceSynchronize());
    int64_t per = n / 132;
    int ns = 14000; size_t smb = (size_t)ns * 16 + 64;
    auto rep = [&](const char* name, float ms) { printf("%-44s %8.3f ms %7.2f Grows/s\n", name, ms, n / (ms * 1e-3) / 1e9); fflush(stdout); };
#define RUN(MODE, T, name) { CK(cudaFuncSetAttribute(agg<MODE, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb)); rep(name, timeit([&] { agg<MODE, T><<<132, T, smb>>>(rows, per, ns, out); })); }
    RUN(0, 1024, "2 atomics, no probe, no return");
    RUN(2, 1024, "2 atomics, returning + carry");
    RUN(1, 1024, "probe (no insert) + 2 atomics");
    RUN(3, 1024, "probe + returning + carry");
    RUN(7, 1024, "probe + CAS insert + returning (= K2)");
    RUN(7, 512, "same, 512 threads");
    RUN(5, 1024, "probe + CAS insert, no return");
    return 0;
}
