// Calibration microbenchmarks for the hash-aggregate design (scratch; not product code).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o scratch/ubench scratch/ubench.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1);} } while (0)

__host__ __device__ inline uint64_t mix64(uint64_t x) {
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

__global__ void gen(int64_t* keys, int64_t* vals, int64_t n, int64_t ngroups) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        keys[i] = (int64_t)(mix64(i) % (uint64_t)ngroups);
        vals[i] = (int64_t)(mix64(i ^ 0x1234567ull) % 1000) - 500;
    }
}

__device__ __forceinline__ uint32_t hslot(int64_t k, uint32_t mask) {
    uint64_t h = (uint64_t)k * 0x9e3779b97f4a7c15ull;
    return (uint32_t)(h >> 32) & mask;
}

__device__ __forceinline__ void ld2(const int64_t* p, int64_t& a, int64_t& b) {
    longlong2 v = *reinterpret_cast<const longlong2*>(p);
    a = v.x; b = v.y;
}

// A: stream only
__global__ void k_stream(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n, unsigned long long* out) {
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    unsigned long long acc = 0;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        acc += (k0 ^ v0) + (k1 ^ v1);
    }
    if (acc == 0x1234567) atomicAdd(out, acc);
}

// B: SoA direct reds (no key check)
template <int NRED>
__global__ void k_soa(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                      unsigned long long* sum, unsigned long long* cnt, uint32_t mask) {
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        atomicAdd(sum + s0, (unsigned long long)v0);
        atomicAdd(sum + s1, (unsigned long long)v1);
        if (NRED > 1) { atomicAdd(cnt + s0, 1ull); atomicAdd(cnt + s1, 1ull); }
    }
}

// C: AoS 32B slot {key,sum,cnt,pad}: key load + compare + 2 reds
struct __align__(32) Slot32 { long long key; unsigned long long sum; unsigned long long cnt; unsigned long long pad; };
template <int CHECK>
__global__ void k_aos32(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                        Slot32* tab, uint32_t mask) {
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        if (CHECK) {
            long long t0 = __ldcg(&tab[s0].key), t1 = __ldcg(&tab[s1].key);
            if (t0 != k0) { s0 = (s0 + 1) & mask; }
            if (t1 != k1) { s1 = (s1 + 1) & mask; }
        }
        atomicAdd(&tab[s0].sum, (unsigned long long)v0);
        atomicAdd(&tab[s0].cnt, 1ull);
        atomicAdd(&tab[s1].sum, (unsigned long long)v1);
        atomicAdd(&tab[s1].cnt, 1ull);
    }
}

// D: key check against separate key array (SoA keys) + 2 reds SoA
__global__ void k_soa_check(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                            const long long* tkeys, unsigned long long* sum, unsigned long long* cnt, uint32_t mask) {
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        long long t0 = __ldcg(tkeys + s0), t1 = __ldcg(tkeys + s1);
        if (t0 != k0) { s0 = (s0 + 1) & mask; }
        if (t1 != k1) { s1 = (s1 + 1) & mask; }
        atomicAdd(sum + s0, (unsigned long long)v0);
        atomicAdd(cnt + s0, 1ull);
        atomicAdd(sum + s1, (unsigned long long)v1);
        atomicAdd(cnt + s1, 1ull);
    }
}

// E: key check only (random 8B loads from L2-resident table), no atomics
__global__ void k_probe_only(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                             const long long* tkeys, uint32_t mask, unsigned long long* out) {
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    unsigned long long acc = 0;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        long long t0 = __ldcg(tkeys + s0), t1 = __ldcg(tkeys + s1);
        acc += (t0 == k0 ? v0 : 0) + (t1 == k1 ? v1 : 0);
    }
    if (acc == 0x1234567) atomicAdd(out, acc);
}

// F: smem atomics: per-CTA table of SM_SLOTS x {sum,cnt}; keys folded into the smem table
template <int MODE>  // 0: two 64-bit smem atomics, 1: non-atomic LDS/STS RMW (racy; throughput only), 2: one 64-bit atomic
__global__ void k_smem(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                       unsigned long long* out, int smslots) {
    extern __shared__ unsigned long long sm[];
    for (int j = threadIdx.x; j < smslots * 2; j += blockDim.x) sm[j] = 0;
    __syncthreads();
    uint32_t mask = smslots - 1;
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        if (MODE == 0) {
            atomicAdd(&sm[2 * s0], (unsigned long long)v0); atomicAdd(&sm[2 * s0 + 1], 1ull);
            atomicAdd(&sm[2 * s1], (unsigned long long)v1); atomicAdd(&sm[2 * s1 + 1], 1ull);
        } else if (MODE == 1) {
            ulonglong2 a = *reinterpret_cast<ulonglong2*>(&sm[2 * s0]);
            a.x += v0; a.y += 1; *reinterpret_cast<ulonglong2*>(&sm[2 * s0]) = a;
            ulonglong2 b = *reinterpret_cast<ulonglong2*>(&sm[2 * s1]);
            b.x += v1; b.y += 1; *reinterpret_cast<ulonglong2*>(&sm[2 * s1]) = b;
        } else {
            atomicAdd(&sm[2 * s0], (unsigned long long)v0 + (1ull << 40));
            atomicAdd(&sm[2 * s1], (unsigned long long)v1 + (1ull << 40));
        }
    }
    __syncthreads();
    unsigned long long acc = 0;
    for (int j = threadIdx.x; j < smslots * 2; j += blockDim.x) acc += sm[j];
    if (acc == 0x1234567) atomicAdd(out, acc);
}

// G: smem atomics 32-bit pair (sum lo32 + cnt32) to compare native 32-bit ATOMS speed
__global__ void k_smem32(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                         unsigned long long* out, int smslots) {
    extern __shared__ unsigned int sm32[];
    for (int j = threadIdx.x; j < smslots * 2; j += blockDim.x) sm32[j] = 0;
    __syncthreads();
    uint32_t mask = smslots - 1;
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    for (; i < n; i += stride) {
        int64_t k0, k1, v0, v1;
        ld2(keys + i, k0, k1); ld2(vals + i, v0, v1);
        uint32_t s0 = hslot(k0, mask), s1 = hslot(k1, mask);
        atomicAdd(&sm32[2 * s0], (unsigned)v0); atomicAdd(&sm32[2 * s0 + 1], 1u);
        atomicAdd(&sm32[2 * s1], (unsigned)v1); atomicAdd(&sm32[2 * s1 + 1], 1u);
    }
    __syncthreads();
    unsigned long long acc = 0;
    for (int j = threadIdx.x; j < smslots * 2; j += blockDim.x) acc += sm32[j];
    if (acc == 0x1234567) atomicAdd(out, acc);
}

// H: partition-write test: every row written (16B) to one of NB buckets through global atomics cursor per warp-run
//    (simplified: per-CTA smem counting sort of a tile, then coalesced run copy-out). Measures phase-A cost.
template <int TILE, int NB>
__global__ void __launch_bounds__(512) k_partition(const int64_t* __restrict__ keys, const int64_t* __restrict__ vals, int64_t n,
                            longlong2* inbox, unsigned int* cursors, int64_t cap_per_bucket) {
    __shared__ unsigned int hist[NB];
    __shared__ unsigned int base[NB];
    __shared__ unsigned int gbase[NB];
    extern __shared__ longlong2 stage[];  // TILE entries
    __shared__ unsigned short bucket_of[TILE];
    int64_t ntiles = (n + TILE - 1) / TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        for (int j = threadIdx.x; j < NB; j += blockDim.x) hist[j] = 0;
        __syncthreads();
        int64_t t0 = t * TILE;
        // pass 1: histogram (keep rows in registers)
        constexpr int PER = TILE / 512;
        int64_t kk[PER], vv[PER]; unsigned int bb[PER], rk[PER];
#pragma unroll
        for (int r = 0; r < PER; r += 2) {
            int64_t idx = t0 + (int64_t)(r / 2) * 1024 + threadIdx.x * 2;
            if (idx + 1 < n) { ld2(keys + idx, kk[r], kk[r + 1]); ld2(vals + idx, vv[r], vv[r + 1]); }
            else { kk[r] = kk[r + 1] = 0; vv[r] = vv[r + 1] = 0; }
        }
#pragma unroll
        for (int r = 0; r < PER; r++) {
            uint64_t h = (uint64_t)kk[r] * 0x9e3779b97f4a7c15ull;
            bb[r] = (unsigned int)(((h >> 32) * (uint64_t)NB) >> 32);
            rk[r] = atomicAdd(&hist[bb[r]], 1u);
        }
        __syncthreads();
        // exclusive scan of hist (NB <= 512): simple warp-serial by thread 0..NB-1 using smem
        if (threadIdx.x < NB) {
            // reserve global space per bucket
            unsigned int c = hist[threadIdx.x];
            gbase[threadIdx.x] = c ? atomicAdd(&cursors[threadIdx.x], c) : 0;
        }
        if (threadIdx.x == 0) {
            unsigned int s = 0;
            for (int j = 0; j < NB; j++) { base[j] = s; s += hist[j]; }
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < PER; r++) {
            unsigned int p = base[bb[r]] + rk[r];
            stage[p] = make_longlong2(kk[r], vv[r]);
            bucket_of[p] = (unsigned short)bb[r];
        }
        __syncthreads();
        // copy-out: consecutive threads write consecutive staged rows (runs are contiguous per bucket)
        for (int p = threadIdx.x; p < TILE; p += blockDim.x) {
            unsigned int b = bucket_of[p];
            unsigned int off = gbase[b] + (p - base[b]);
            if (off < cap_per_bucket) inbox[(int64_t)b * cap_per_bucket + off] = stage[p];
        }
        __syncthreads();
    }
}

template <typename F>
float timeit(F f, int reps = 3) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; r++) {
        cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b));
        float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
    }
    return best;
}

int main(int argc, char** argv) {
    int64_t n = argc > 1 ? atoll(argv[1]) : (1ll << 28);
    int64_t ng = argc > 2 ? atoll(argv[2]) : 1000000;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    printf("dev %s SMs %d L2 %d MB smem/blk optin %zu clock %d\n", prop.name, prop.multiProcessorCount, prop.l2CacheSize >> 20, prop.sharedMemPerBlockOptin, prop.clockRate);
    int64_t *keys, *vals; CK(cudaMalloc(&keys, n * 8)); CK(cudaMalloc(&vals, n * 8));
    gen<<<132 * 8, 256>>>(keys, vals, n, ng); CK(cudaDeviceSynchronize());
    uint32_t cap = 1; while (cap < 2 * ng) cap <<= 1; uint32_t mask = cap - 1;
    unsigned long long *sum, *cnt, *out; long long* tkeys; Slot32* tab;
    CK(cudaMalloc(&sum, cap * 8ull)); CK(cudaMalloc(&cnt, cap * 8ull)); CK(cudaMalloc(&tkeys, cap * 8ull)); CK(cudaMalloc(&tab, cap * 32ull)); CK(cudaMalloc(&out, 8));
    CK(cudaMemset(sum, 0, cap * 8ull)); CK(cudaMemset(cnt, 0, cap * 8ull)); CK(cudaMemset(tkeys, 0, cap * 8ull)); CK(cudaMemset(tab, 0, cap * 32ull));
    double gb = n * 16.0 / 1e9;
    auto rep = [&](const char* name, float ms) { printf("%-28s %8.3f ms  %8.1f GB/s  %7.2f Grows/s\n", name, ms, gb / (ms * 1e-3), n / (ms * 1e-3) / 1e9); fflush(stdout); };
    for (int bps : {4, 8}) {
        int grid = 132 * bps, blk = 256;
        printf("-- grid %d x %d, n=%lld groups=%lld cap=%u\n", grid, blk, (long long)n, (long long)ng, cap);
        rep("A stream", timeit([&] { k_stream<<<grid, blk>>>(keys, vals, n, out); }));
        rep("B soa 1 red", timeit([&] { k_soa<1><<<grid, blk>>>(keys, vals, n, sum, cnt, mask); }));
        rep("B soa 2 red", timeit([&] { k_soa<2><<<grid, blk>>>(keys, vals, n, sum, cnt, mask); }));
        rep("C aos32 nocheck 2 red", timeit([&] { k_aos32<0><<<grid, blk>>>(keys, vals, n, tab, mask); }));
        rep("C aos32 check 2 red", timeit([&] { k_aos32<1><<<grid, blk>>>(keys, vals, n, tab, mask); }));
        rep("D soa check 2 red", timeit([&] { k_soa_check<<<grid, blk>>>(keys, vals, n, tkeys, sum, cnt, mask); }));
        rep("E probe only", timeit([&] { k_probe_only<<<grid, blk>>>(keys, vals, n, tkeys, mask, out); }));
    }
    {
        int smslots = 8192; size_t smb = smslots * 16;
        CK(cudaFuncSetAttribute(k_smem<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        CK(cudaFuncSetAttribute(k_smem<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        CK(cudaFuncSetAttribute(k_smem<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        CK(cudaFuncSetAttribute(k_smem32, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        for (int blk : {512, 1024}) {
            int grid = 132;
            printf("-- smem table %d slots, grid %d x %d\n", smslots, grid, blk);
            rep("F smem 2x atom64", timeit([&] { k_smem<0><<<grid, blk, smb>>>(keys, vals, n, out, smslots); }));
            rep("F smem ld/st rmw", timeit([&] { k_smem<1><<<grid, blk, smb>>>(keys, vals, n, out, smslots); }));
            rep("F smem 1x atom64", timeit([&] { k_smem<2><<<grid, blk, smb>>>(keys, vals, n, out, smslots); }));
            rep("G smem 2x atom32", timeit([&] { k_smem32<<<grid, blk, smb / 2>>>(keys, vals, n, out, smslots); }));
        }
    }
    {
        constexpr int TILE = 4096, NB = 132;
        int64_t capb = (int64_t)(n / NB * 1.05) + 4096;
        // limit n for partition test so inbox fits: use first 64M rows
        int64_t np = n < (1ll << 26) ? n : (1ll << 26);
        capb = (int64_t)(np / NB * 1.05) + 4096;
        longlong2* inbox; unsigned int* cursors;
        CK(cudaMalloc(&inbox, capb * NB * 16)); CK(cudaMalloc(&cursors, NB * 4));
        size_t smb = TILE * 16;
        CK(cudaFuncSetAttribute(k_partition<TILE, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smb));
        for (int bps : {1, 2}) {
            float ms = timeit([&] { cudaMemsetAsync(cursors, 0, NB * 4); k_partition<TILE, NB><<<132 * bps, 512, smb>>>(keys, vals, np, inbox, cursors, capb); });
            printf("H partition %d/SM  %8.3f ms  %7.2f Grows/s (n=%lld, HBM-sized inbox)\n", bps, ms, np / (ms * 1e-3) / 1e9, (long long)np);
        }
        // L2-sized: 2M rows repeatedly into the same 32MB inbox
        int64_t nl = 1ll << 21; capb = (int64_t)(nl / NB * 1.2) + 1024;
        for (int bps : {1, 2}) {
            float ms = timeit([&] { for (int r = 0; r < 16; r++) { cudaMemsetAsync(cursors, 0, NB * 4); k_partition<TILE, NB><<<132 * bps, 512, smb>>>(keys + r * nl, vals + r * nl, nl, inbox, cursors, capb); } });
            printf("H partition L2 %d/SM  %8.3f ms  %7.2f Grows/s (16 x 2M rows, incl launch gaps)\n", bps, ms, 16 * nl / (ms * 1e-3) / 1e9);
        }
    }
    return 0;
}
