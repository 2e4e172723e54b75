// misc.cu — error reporting, runtime probes, raw memory helpers, the shared bitmap-pack and fill kernels and the
// synthetic-table generator.
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace b200 {
namespace {
// A pooled block carries the event recorded on the releasing thread's scratch stream (scratch_set_stream) when it was
// released: DevBuf::ensure() may hand a block back while kernels that read it are still queued, so whoever acquires the
// block next (possibly another state on another stream) first waits for that event.  The pool is stream-ordered.
struct PoolEntry { void* p; size_t bytes; cudaEvent_t ev; };
std::mutex g_pool_mutex;
std::vector<PoolEntry> g_pool[64];
size_t g_pool_bytes[64] = {0};
thread_local cudaStream_t g_scratch_stream = nullptr;

size_t pool_cap_bytes() {
    static size_t cap = [] {
        const char* e = getenv("B200_POOL_MAX_BYTES");
        return e ? (size_t)strtoull(e, nullptr, 10) : ((size_t)24 << 30);
    }();
    return cap;
}
void wait_and_drop_event(cudaEvent_t ev) {
    if (!ev) return;
    cudaEventSynchronize(ev);
    cudaEventDestroy(ev);
}
// caller holds g_pool_mutex
void trim_locked(int device, size_t keep_bytes) {
    auto& v = g_pool[device & 63];
    while (g_pool_bytes[device & 63] > keep_bytes && !v.empty()) {
        int big = 0;
        for (int i = 1; i < (int)v.size(); i++) if (v[i].bytes > v[big].bytes) big = i;
        wait_and_drop_event(v[big].ev);
        cudaFree(v[big].p);
        g_pool_bytes[device & 63] -= v[big].bytes;
        v.erase(v.begin() + big);
    }
}
}  // namespace

void scratch_set_stream(cudaStream_t s) { g_scratch_stream = s; }

void* scratch_acquire(int device, size_t bytes, size_t* got) {
    if (bytes == 0) bytes = 8;
    {
        std::unique_lock<std::mutex> lk(g_pool_mutex);
        auto& v = g_pool[device & 63];
        // best fit, but never hand out a block more than 2x (+1 MiB) larger than asked for
        size_t limit = bytes * 2 + (1u << 20);
        int best = -1;
        for (int i = 0; i < (int)v.size(); i++)
            if (v[i].bytes >= bytes && v[i].bytes <= limit && (best < 0 || v[i].bytes < v[best].bytes)) best = i;
        if (best >= 0) {
            PoolEntry e = v[best];
            v.erase(v.begin() + best);
            g_pool_bytes[device & 63] -= e.bytes;
            lk.unlock();
            wait_and_drop_event(e.ev);  // work queued on the block before its release has finished
            *got = e.bytes;
            return e.p;
        }
    }
    void* p = nullptr;
    B200_CUDA(cudaSetDevice(device));
    cudaError_t err = cudaMalloc(&p, bytes);
    if (err != cudaSuccess) {
        // out of memory: give the pooled blocks back to the driver and retry once
        cudaGetLastError();
        {
            std::lock_guard<std::mutex> lk(g_pool_mutex);
            trim_locked(device, 0);
        }
        B200_CUDA(cudaMalloc(&p, bytes));
    }
    *got = bytes;
    return p;
}
void scratch_release(int device, void* p, size_t bytes) {
    if (!p) return;
    cudaEvent_t ev = nullptr;
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != device) cudaSetDevice(device);
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess) {
        if (cudaEventRecord(ev, g_scratch_stream) != cudaSuccess) { cudaGetLastError(); cudaEventDestroy(ev); ev = nullptr; cudaDeviceSynchronize(); }
    } else { cudaGetLastError(); ev = nullptr; cudaDeviceSynchronize(); }
    if (cur != device && cur >= 0) cudaSetDevice(cur);
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    g_pool[device & 63].push_back({p, bytes, ev});
    g_pool_bytes[device & 63] += bytes;
    // bounded: blocks beyond the cap go back to the driver (largest first), so a process that also runs torch's caching
    // allocator on the same GPU gets the memory back after the states that needed it are gone
    if (g_pool_bytes[device & 63] > pool_cap_bytes()) trim_locked(device, pool_cap_bytes());
}
void scratch_trim(int device, size_t keep_bytes) {
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    trim_locked(device, keep_bytes);
}

namespace { std::vector<PoolEntry> g_pinned; }
void* pinned_acquire(size_t bytes) {
    {
        std::lock_guard<std::mutex> lk(g_pool_mutex);
        for (size_t i = 0; i < g_pinned.size(); i++)
            if (g_pinned[i].bytes >= bytes) { void* p = g_pinned[i].p; g_pinned.erase(g_pinned.begin() + i); return p; }
    }
    void* p = nullptr;
    B200_CUDA(cudaMallocHost(&p, bytes < 256 ? 256 : bytes));
    return p;
}
void pinned_release(void* p, size_t bytes) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    g_pinned.push_back({p, bytes < 256 ? 256 : bytes});
}

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }

__global__ void pack_bitmap_kernel(const uint8_t* bytes, int64_t n, uint32_t* words) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t n_round = (n + 31) & ~31ll;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_round; i += stride) {
        unsigned m = __ballot_sync(0xffffffffu, i < n && bytes[i]);
        if ((threadIdx.x & 31) == 0) words[i >> 5] = m;
    }
}
void launch_pack_bitmap(const uint8_t* bytes, int64_t n, uint32_t* words, int grid, cudaStream_t st) {
    pack_bitmap_kernel<<<grid, 256, 0, st>>>(bytes, n, words);
}

__global__ void fill_u64_kernel(unsigned long long* p, uint64_t n, unsigned long long v) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}
void launch_fill_u64(void* p, uint64_t n, unsigned long long v, int grid, cudaStream_t st) {
    fill_u64_kernel<<<grid, 256, 0, st>>>((unsigned long long*)p, n, v);
}

// key = mix64(row ^ seed-derived salt) % n_groups ; val = (mix64(...) % 1000) - 500 (INT64) or u01 (FLOAT64).
// Same arithmetic as oracle_synth_fill (oracle/bodo_oracle.c) and bodo_b200/synth.py.
__global__ void synth_fill_kernel(long long* keys, void* vals, int64_t row_start, int64_t n, uint64_t n_groups, uint64_t seed,
                                  int val_ctype) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint64_t salt_k = seed * 0x9e3779b97f4a7c15ULL, salt_v = (seed + 1) * 0xd1b54a32d192ed03ULL;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        uint64_t r = (uint64_t)(row_start + i);
        if (keys) keys[i] = (long long)(mix64(r ^ salt_k) % n_groups);
        if (vals) {
            uint64_t m = mix64(r ^ salt_v);
            if (val_ctype == CT_FLOAT64) ((double*)vals)[i] = (double)(m >> 11) * (1.0 / 9007199254740992.0);
            else ((long long*)vals)[i] = (long long)(m % 1000) - 500;
        }
    }
}
}  // namespace b200

extern "C" {

const char* b200_last_error(void) { return b200::g_last_error.c_str(); }
int b200_abi_version(void) { return 1; }
int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void* b200_device_malloc(int32_t device, int64_t nbytes) {
    try {
        B200_CUDA(cudaSetDevice(device));
        void* p = nullptr;
        B200_CUDA(cudaMalloc(&p, (size_t)(nbytes > 0 ? nbytes : 8)));
        return p;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return nullptr; }
}
int64_t b200_pool_trim(int32_t device, int64_t keep_bytes) {
    b200::scratch_trim(device, keep_bytes > 0 ? (size_t)keep_bytes : 0);
    return 0;
}
void b200_device_free(int32_t device, void* p) {
    if (!p) return;
    cudaSetDevice(device);
    cudaFree(p);
}
int b200_memcpy_d2h(void* dst_host, const void* src_dev, int64_t nbytes, void* stream) {
    try {
        if (nbytes <= 0) return 0;
        B200_CUDA(cudaMemcpyAsync(dst_host, src_dev, (size_t)nbytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
        B200_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}
int b200_memcpy_h2d(void* dst_dev, const void* src_host, int64_t nbytes, void* stream) {
    try {
        if (nbytes <= 0) return 0;
        B200_CUDA(cudaMemcpyAsync(dst_dev, src_host, (size_t)nbytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
        B200_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}
int b200_stream_synchronize(void* stream) {
    try { B200_CUDA(cudaStreamSynchronize((cudaStream_t)stream)); return 0; }
    catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_synth_fill(void* key_out, void* val_out, int64_t row_start, int64_t n_rows, int64_t n_groups, uint64_t seed,
                    int32_t val_c_type, void* stream) {
    try {
        B200_REQUIRE(n_groups > 0, "b200_synth_fill: n_groups must be positive");
        B200_REQUIRE(val_c_type == b200::CT_INT64 || val_c_type == b200::CT_FLOAT64, "b200_synth_fill: value type must be INT64 or FLOAT64");
        if (n_rows <= 0) return 0;
        int dev = 0;
        B200_CUDA(cudaGetDevice(&dev));
        int grid = b200::num_sms(dev) * 8;
        b200::synth_fill_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((long long*)key_out, val_out, row_start, n_rows, (uint64_t)n_groups, seed, val_c_type);
        B200_CUDA(cudaGetLastError());
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

}  // extern "C"
