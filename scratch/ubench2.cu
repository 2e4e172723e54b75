// Variants of the direct hash-aggregate kernel (scratch): which table-probe load keeps the table L2-resident?
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../bodo_b200/csrc/common.cuh"
using namespace b200;
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
namespace b200 { void set_last_error(const std::string&) {} }
constexpr long long EMPTY = (long long)0x8000000000000000ULL;

__global__ void gen(long long* keys, long long* vals, int64_t n, uint64_t ng) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) { keys[i] = (long long)(mix64(i ^ 0x9e3779b97f4a7c15ULL) % ng); vals[i] = (long long)(mix64(i ^ 0x1234567ull) % 1000) - 500; }
}
template <int MODE> __device__ __forceinline__ void loadb(const long long* t, uint64_t b, long long (&k)[4]) {
    // (sm_90 has no 256-bit load: a 32-byte bucket is two 128-bit loads)
    if (MODE == 1) {
        asm volatile("ld.global.cg.v2.s64 {%0,%1}, [%2];" : "=l"(k[0]), "=l"(k[1]) : "l"(t + 4 * b));
        asm volatile("ld.global.cg.v2.s64 {%0,%1}, [%2];" : "=l"(k[2]), "=l"(k[3]) : "l"(t + 4 * b + 2));
    } else if (MODE == 2) {
        asm volatile("ld.global.ca.v2.s64 {%0,%1}, [%2];" : "=l"(k[0]), "=l"(k[1]) : "l"(t + 4 * b));
        asm volatile("ld.global.ca.v2.s64 {%0,%1}, [%2];" : "=l"(k[2]), "=l"(k[3]) : "l"(t + 4 * b + 2));
    } else {
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
        asm volatile("ld.global.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;" : "=l"(k[0]), "=l"(k[1]) : "l"(t + 4 * b), "l"(pol));
        asm volatile("ld.global.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;" : "=l"(k[2]), "=l"(k[3]) : "l"(t + 4 * b + 2), "l"(pol));
    }
}
template <int MODE> __device__ __forceinline__ uint64_t foi(long long* t, uint64_t cap, long long key) {
    uint64_t nbm = (cap >> 2) - 1, b = (xxh3_64_short((uint64_t)key, 8, SEED_HASH_PARTITION) >> 32) & nbm;
    while (true) {
        long long k[4]; loadb<MODE>(t, b, k);
        int match = -1, empty = -1;
#pragma unroll
        for (int j = 3; j >= 0; j--) { if (k[j] == key) match = j; if (k[j] == EMPTY) empty = j; }
        if (match >= 0) return 4 * b + match;
        if (empty >= 0) {
            long long prev = atomicCAS((unsigned long long*)(t + 4 * b + empty), (unsigned long long)EMPTY, (unsigned long long)key);
            if (prev == EMPTY || prev == key) return 4 * b + empty;
            continue;
        }
        b = (b + 1) & nbm;
    }
}
// STREAM: 0 = __ldcs, 1 = plain, 2 = ld.global.nc.L1::no_allocate.L2::evict_first
template <int MODE, int STREAM>
__global__ void __launch_bounds__(256) agg(const long long* __restrict__ keys, const long long* __restrict__ vals, int64_t n, long long* t, uint64_t cap,
                                           unsigned long long* sum, unsigned long long* cnt) {
    int64_t st = (int64_t)gridDim.x * blockDim.x * 2;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2; i + 1 < n; i += st) {
        longlong2 kk, vv;
        if (STREAM == 0) { kk = __ldcs((const longlong2*)(keys + i)); vv = __ldcs((const longlong2*)(vals + i)); }
        else if (STREAM == 1) { kk = *(const longlong2*)(keys + i); vv = *(const longlong2*)(vals + i); }
        else {
            uint64_t pol;
            asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;" : "=l"(kk.x), "=l"(kk.y) : "l"(keys + i), "l"(pol));
            asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;" : "=l"(vv.x), "=l"(vv.y) : "l"(vals + i), "l"(pol));
        }
        uint64_t s0 = foi<MODE>(t, cap, kk.x), s1 = foi<MODE>(t, cap, kk.y);
        atomicAdd(sum + s0, (unsigned long long)vv.x); atomicAdd(cnt + s0, 1ull);
        atomicAdd(sum + s1, (unsigned long long)vv.y); atomicAdd(cnt + s1, 1ull);
    }
}
// linear probing, 64-bit loads (the first version of the library kernel)
template <int STREAM>
__global__ void __launch_bounds__(256) agg_lin(const long long* __restrict__ keys, const long long* __restrict__ vals, int64_t n, long long* t, uint64_t cap,
                                               unsigned long long* sum, unsigned long long* cnt) {
    int64_t st = (int64_t)gridDim.x * blockDim.x * 2;
    uint64_t mask = cap - 1;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2; i + 1 < n; i += st) {
        longlong2 kk, vv;
        if (STREAM == 0) { kk = __ldcs((const longlong2*)(keys + i)); vv = __ldcs((const longlong2*)(vals + i)); }
        else { kk = *(const longlong2*)(keys + i); vv = *(const longlong2*)(vals + i); }
        long long k2[2] = {kk.x, kk.y}, v2[2] = {vv.x, vv.y};
#pragma unroll
        for (int r = 0; r < 2; r++) {
            uint64_t s = (xxh3_64_short((uint64_t)k2[r], 8, SEED_HASH_PARTITION) >> 32) & mask;
            while (true) {
                long long k = __ldcg(t + s);
                if (k == k2[r]) break;
                if (k == EMPTY) { long long prev = atomicCAS((unsigned long long*)(t + s), (unsigned long long)EMPTY, (unsigned long long)k2[r]); if (prev == EMPTY || prev == k2[r]) break; }
                s = (s + 1) & mask;
            }
            atomicAdd(sum + s, (unsigned long long)v2[r]); atomicAdd(cnt + s, 1ull);
        }
    }
}
template <int HASH, int ILP2>
__global__ void __launch_bounds__(256) agg_lin2(const long long* __restrict__ keys, const long long* __restrict__ vals, int64_t n, long long* t, uint64_t cap,
                                                unsigned long long* sum, unsigned long long* cnt) {
    int64_t st = (int64_t)gridDim.x * blockDim.x * 2;
    uint64_t mask = cap - 1;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2; i + 1 < n; i += st) {
        longlong2 kk = __ldcs((const longlong2*)(keys + i)), vv = __ldcs((const longlong2*)(vals + i));
        long long k2[2] = {kk.x, kk.y}, v2[2] = {vv.x, vv.y};
        uint64_t s[2]; long long f[2];
#pragma unroll
        for (int r = 0; r < 2; r++) {
            s[r] = HASH == 0 ? ((xxh3_64_short((uint64_t)k2[r], 8, SEED_HASH_PARTITION) >> 32) & mask) : ((((uint64_t)k2[r] * 0x9e3779b97f4a7c15ull) >> 32) & mask);
            if (ILP2) f[r] = __ldcg(t + s[r]);
        }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            long long k = ILP2 ? f[r] : __ldcg(t + s[r]);
            while (true) {
                if (k == k2[r]) break;
                if (k == EMPTY) { long long prev = atomicCAS((unsigned long long*)(t + s[r]), (unsigned long long)EMPTY, (unsigned long long)k2[r]); if (prev == EMPTY || prev == k2[r]) break; }
                s[r] = (s[r] + 1) & mask;
                k = __ldcg(t + s[r]);
            }
            atomicAdd(sum + s[r], (unsigned long long)v2[r]); atomicAdd(cnt + s[r], 1ull);
        }
    }
}
// no table at all: slot straight from the hash (pure atomic cost)
template <int HASH>
__global__ void __launch_bounds__(256) agg_nocheck(const long long* __restrict__ keys, const long long* __restrict__ vals, int64_t n, uint64_t cap,
                                                   unsigned long long* sum, unsigned long long* cnt) {
    int64_t st = (int64_t)gridDim.x * blockDim.x * 2;
    uint64_t mask = cap - 1;
    for (int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2; i + 1 < n; i += st) {
        longlong2 kk = __ldcs((const longlong2*)(keys + i)), vv = __ldcs((const longlong2*)(vals + i));
        long long k2[2] = {kk.x, kk.y}, v2[2] = {vv.x, vv.y};
#pragma unroll
        for (int r = 0; r < 2; r++) {
            uint64_t s = HASH == 0 ? ((xxh3_64_short((uint64_t)k2[r], 8, SEED_HASH_PARTITION) >> 32) & mask) : ((((uint64_t)k2[r] * 0x9e3779b97f4a7c15ull) >> 32) & mask);
            atomicAdd(sum + s, (unsigned long long)v2[r]); atomicAdd(cnt + s, 1ull);
        }
    }
}
__global__ void fill(long long* p, uint64_t n, long long v) { for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v; }
template <typename F> float timeit(F f, int reps = 3) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; r++) { cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b)); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; }
    return best;
}
int main(int argc, char** argv) {
    int64_t n = argc > 1 ? atoll(argv[1]) : (1ll << 27);
    uint64_t ng = argc > 2 ? atoll(argv[2]) : 1000000;
    int capmul = argc > 3 ? atoi(argv[3]) : 2;
    long long *keys, *vals, *t; unsigned long long *sum, *cnt;
    CK(cudaMalloc(&keys, n * 8)); CK(cudaMalloc(&vals, n * 8));
    gen<<<132 * 8, 256>>>(keys, vals, n, ng);
    uint64_t cap = 1; while (cap < capmul * ng) cap <<= 1;
    CK(cudaMalloc(&t, cap * 8)); CK(cudaMalloc(&sum, cap * 8)); CK(cudaMalloc(&cnt, cap * 8));
    CK(cudaDeviceSynchronize());
    auto reset = [&] { fill<<<1184, 256>>>(t, cap, EMPTY); cudaMemset(sum, 0, cap * 8); cudaMemset(cnt, 0, cap * 8); };
    auto rep = [&](const char* name, float ms) { printf("%-34s %8.3f ms %7.2f Grows/s\n", name, ms, n / (ms * 1e-3) / 1e9); fflush(stdout); };
    int g = 132 * 8;
    printf("n=%lld groups=%llu cap=%llu\n", (long long)n, (unsigned long long)ng, (unsigned long long)cap);
    reset(); rep("nocheck xxh3 (2 red only)", timeit([&] { agg_nocheck<0><<<g, 256>>>(keys, vals, n, cap, sum, cnt); }));
    reset(); rep("nocheck fib (2 red only)", timeit([&] { agg_nocheck<1><<<g, 256>>>(keys, vals, n, cap, sum, cnt); }));
    reset(); rep("linear xxh3 ilp1", timeit([&] { agg_lin2<0, 0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("linear xxh3 ilp2", timeit([&] { agg_lin2<0, 1><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("linear fib  ilp1", timeit([&] { agg_lin2<1, 0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("linear fib  ilp2", timeit([&] { agg_lin2<1, 1><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("linear 64b, ldcs stream", timeit([&] { agg_lin<0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("linear 64b, plain stream", timeit([&] { agg_lin<1><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b cg, ldcs", timeit([&] { agg<1, 0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b cg, plain", timeit([&] { agg<1, 1><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b ca, ldcs", timeit([&] { agg<2, 0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b evict_last, ldcs", timeit([&] { agg<3, 0><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b evict_last, nc ef", timeit([&] { agg<3, 2><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    reset(); rep("bucket 2x128b cg, nc evict_first", timeit([&] { agg<1, 2><<<g, 256>>>(keys, vals, n, t, cap, sum, cnt); }));
    return 0;
}
