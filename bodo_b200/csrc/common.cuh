// common.cuh — shared device/host helpers for libbodo_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <stdexcept>
#include <string>

#include "../../include/bodo_b200.h"

namespace b200 {

// Bodo_CTypes / bodo_array_type codes (reference: bodo/libs/_bodo_common.h:331-359, :515-532)
enum CType : int { CT_INT8 = 0, CT_UINT8 = 1, CT_INT32 = 2, CT_UINT32 = 3, CT_INT64 = 4, CT_FLOAT32 = 5, CT_FLOAT64 = 6,
                   CT_UINT64 = 7, CT_INT16 = 8, CT_UINT16 = 9, CT_BOOL = 11, CT_DATE = 13, CT_DATETIME = 15,
                   CT_TIMEDELTA = 16 };
enum ArrType : int { ARR_NUMPY = 0, ARR_NULLABLE = 2 };
// Bodo_FTypes (reference: bodo/libs/groupby/_groupby_ftypes.h:17-110)
// 28..34 and 38..40 continue the enum after skew in the reference's order; they are recalled, not read from a reference checkout
// (17 and 26 are fixed by their neighbours).
enum FType : int { FT_SIZE = 4, FT_SUM = 6, FT_COUNT = 7, FT_NUNIQUE = 8, FT_MEAN = 14, FT_MIN = 15, FT_MAX = 16, FT_PROD = 17, FT_FIRST = 18,
                   FT_LAST = 19, FT_VAR_POP = 22, FT_STD_POP = 23, FT_VAR = 24, FT_STD = 25, FT_KURTOSIS = 26, FT_SKEW = 27,
                   FT_BOOLOR_AGG = 28, FT_BOOLAND_AGG = 29, FT_BOOLXOR_AGG = 30, FT_BITOR_AGG = 31, FT_BITAND_AGG = 32, FT_BITXOR_AGG = 33,
                   FT_COUNT_IF = 34, FT_MODE = 38, FT_PERCENTILE_CONT = 39, FT_PERCENTILE_DISC = 40 };

// hash seeds (reference: bodo/libs/_array_hash.h:8-14)
constexpr uint32_t SEED_HASH_PARTITION = 0xb0d01289u;
constexpr uint32_t SEED_HASH_JOIN = 0xb0d01286u;

void set_last_error(const std::string& msg);

struct Error : std::runtime_error {
    using std::runtime_error::runtime_error;
};

#define B200_CUDA(call)                                                                                       \
    do {                                                                                                      \
        cudaError_t _e = (call);                                                                              \
        if (_e != cudaSuccess)                                                                                \
            throw b200::Error(std::string("CUDA error: ") + cudaGetErrorString(_e) + " in " #call " at " +   \
                              __FILE__ + ":" + std::to_string(__LINE__));                                     \
    } while (0)

#define B200_REQUIRE(cond, msg)                      \
    do {                                             \
        if (!(cond)) throw b200::Error(std::string(msg)); \
    } while (0)

__host__ __device__ inline int ctype_size(int ct) {
    switch (ct) {
        case CT_INT8: case CT_UINT8: case CT_BOOL: return 1;
        case CT_INT16: case CT_UINT16: return 2;
        case CT_INT32: case CT_UINT32: case CT_FLOAT32: case CT_DATE: return 4;
        case CT_INT64: case CT_UINT64: case CT_FLOAT64: case CT_DATETIME: case CT_TIMEDELTA: return 8;
        default: return 0;
    }
}
inline const char* ctype_name(int ct) {
    switch (ct) {
        case CT_INT8: return "int8"; case CT_UINT8: return "uint8"; case CT_INT16: return "int16"; case CT_UINT16: return "uint16";
        case CT_INT32: return "int32"; case CT_UINT32: return "uint32"; case CT_INT64: return "int64"; case CT_UINT64: return "uint64";
        case CT_FLOAT32: return "float32"; case CT_FLOAT64: return "float64"; case CT_BOOL: return "bool"; case CT_DATE: return "date";
        case CT_DATETIME: return "datetime"; case CT_TIMEDELTA: return "timedelta"; default: return "unknown";
    }
}
__host__ __device__ inline bool ctype_is_float(int ct) { return ct == CT_FLOAT32 || ct == CT_FLOAT64; }
__host__ __device__ inline bool ctype_is_temporal(int ct) { return ct == CT_DATE || ct == CT_DATETIME || ct == CT_TIMEDELTA; }
__host__ __device__ inline bool ctype_is_signed_int(int ct) {
    return ct == CT_INT8 || ct == CT_INT16 || ct == CT_INT32 || ct == CT_INT64 || ct == CT_DATE || ct == CT_DATETIME ||
           ct == CT_TIMEDELTA;
}

// ---- device helpers -------------------------------------------------------------------------

__device__ __forceinline__ bool bit_valid(const uint8_t* __restrict__ bm, int64_t i) {
    return bm == nullptr || ((bm[i >> 3] >> (i & 7)) & 1);
}

__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

// XXH3_64bits_withSeed for 4- and 8-byte inputs (XXH3_len_4to8_64b + XXH3_rrmxmx), the function behind the
// reference's hash_inner_32 (bodo/libs/vendored/_murmurhash3.h:59-68, vendored/xxhash.h:4034-4041,4102-4119).
// Restated from the published xxHash algorithm; pinned against the reference's vendored header in
// tests/test_oracle.py (through the oracle) and tests/test_gpu_shuffle.py (this device function).
__host__ __device__ __forceinline__ uint64_t xxh3_64_short(uint64_t raw, int len, uint32_t seed32) {
    uint64_t seed = seed32;
    uint32_t s = (uint32_t)seed;
    uint32_t sw = ((s & 0xffu) << 24) | ((s & 0xff00u) << 8) | ((s >> 8) & 0xff00u) | (s >> 24);
    seed ^= (uint64_t)sw << 32;
    uint32_t in1 = (uint32_t)raw;
    uint32_t in2 = len == 8 ? (uint32_t)(raw >> 32) : (uint32_t)raw;
    const uint64_t bitflip = (0x1cad21f72c81017cULL ^ 0xdb979083e96dd4deULL) - seed;
    uint64_t h = ((uint64_t)in2 + ((uint64_t)in1 << 32)) ^ bitflip;
    h ^= ((h << 49) | (h >> 15)) ^ ((h << 24) | (h >> 40));
    h *= 0x9FB21C651E98DF25ULL;
    h ^= (h >> 35) + (uint64_t)len;
    h *= 0x9FB21C651E98DF25ULL;
    return h ^ (h >> 28);
}

// hash_combine_boost (reference: bodo/libs/_array_hash.cpp:41-56): one 32-bit murmur round folding a further key column's
// hash into the running row hash.
__host__ __device__ __forceinline__ uint32_t hash_combine_boost(uint32_t h1, uint32_t k1) {
    k1 *= 0xcc9e2d51u;
    k1 = (k1 << 15) | (k1 >> 17);
    k1 *= 0x1b873593u;
    h1 ^= k1;
    h1 = (h1 << 13) | (h1 >> 19);
    return h1 * 5u + 0xe6546b64u;
}
// _Py_HashDouble (CPython Python/pyhash.c, what the reference feeds float keys through before hashing the resulting
// Py_hash_t, bodo/libs/_array_hash.cpp:119-170): reduction of the double modulo the Mersenne prime 2^61 - 1; NaN -> 0 (the
// reference passes a NULL identity), +-inf -> +-314159.  Restated from the published algorithm; pinned against the oracle
// (which is pinned against the interpreter's own hash(float)) in tests/test_gpu_shuffle.py.
__host__ __device__ inline int64_t py_hash_double(double v) {
    const int BITS = 61;
    const uint64_t MOD = (1ULL << 61) - 1;
    if (isnan(v)) return 0;
    if (isinf(v)) return v > 0 ? 314159 : -314159;
    int e;
    double m = frexp(v, &e);
    int sign = 1;
    if (m < 0) { sign = -1; m = -m; }
    uint64_t x = 0;
    while (m != 0.0) {
        x = ((x << 28) & MOD) | (x >> (BITS - 28));
        m *= 268435456.0;  // 2^28
        e -= 28;
        uint64_t y = (uint64_t)m;
        m -= (double)y;
        x += y;
        if (x >= MOD) x -= MOD;
    }
    e = e >= 0 ? e % BITS : BITS - 1 - ((-1 - e) % BITS);
    x = ((x << e) & MOD) | (x >> (BITS - e));
    int64_t r = (int64_t)x * sign;
    return r == -1 ? -2 : r;
}

// Float groupby keys live in the int64 tables as this encoding of their double value (a float32 key is widened first,
// exactly): the bit pattern, with -0.0 folded onto +0.0 (one group, as in pandas) and every NaN mapped to INT64_MIN.  INT64_MIN
// is the pattern of -0.0, so no other key produces it, and it is the tables' marker key: NaN keys land in the marker slot,
// one group without a validity bitmap.  Integer equality of two encodings is equality of the keys.
__host__ __device__ __forceinline__ long long canon_float_key(double d) {
    if (isnan(d)) return (long long)0x8000000000000000ULL;
    if (d == 0.0) return 0;
#ifdef __CUDA_ARCH__
    return __double_as_longlong(d);
#else
    long long b; memcpy(&b, &d, 8); return b;
#endif
}
__host__ __device__ __forceinline__ double canon_float_decode(long long k) {
    if (k == (long long)0x8000000000000000ULL) return NAN;
#ifdef __CUDA_ARCH__
    return __longlong_as_double(k);
#else
    double d; memcpy(&d, &k, 8); return d;
#endif
}

// hash_to_rank (reference: bodo/libs/_shuffle.h:5-7): (uint32) hash % n_pes.
__host__ __device__ __forceinline__ int hash_to_rank_u32(uint32_t h, int n_pes) { return (int)(h % (uint32_t)n_pes); }

// Table-slot hash: the same xxh3 value (one hash per row); ranks use the low 32 bits, slots the high 32
// bits, so the two are independent (a rank's keys all share low32 % P).
__device__ __forceinline__ uint64_t key_hash(int64_t key) { return xxh3_64_short((uint64_t)key, 8, SEED_HASH_PARTITION); }
// Owner-rank hash of a valid table key of input c-type ct: the hash shuffle_table gives its rows (hash_key_column).  A float key's
// encoding (canon_float_key) goes through _Py_HashDouble of its value first; NaN hashes as 0, as a NaN row does there.  An integer,
// bool or date key narrower than 8 bytes hashes the 4 low bytes of its widened value, as its column's raw bytes hash there.
__device__ __forceinline__ uint32_t owner_key_hash(int64_t key, int ct) {
    if (ct == CT_FLOAT64 || ct == CT_FLOAT32) return (uint32_t)xxh3_64_short((uint64_t)py_hash_double(canon_float_decode(key)), 8, SEED_HASH_PARTITION);
    if (ctype_size(ct) == 8) return (uint32_t)key_hash(key);
    return (uint32_t)xxh3_64_short((uint64_t)(uint32_t)key, 4, SEED_HASH_PARTITION);
}

__device__ __forceinline__ int64_t load_int_as_i64(const void* __restrict__ p, int ct, int64_t i) {
    switch (ct) {
        case CT_INT64: case CT_DATETIME: case CT_TIMEDELTA: case CT_UINT64: return ((const int64_t*)p)[i];
        case CT_INT32: case CT_DATE: return ((const int32_t*)p)[i];
        case CT_UINT32: return ((const uint32_t*)p)[i];
        case CT_INT16: return ((const int16_t*)p)[i];
        case CT_UINT16: return ((const uint16_t*)p)[i];
        case CT_INT8: return ((const int8_t*)p)[i];
        case CT_UINT8: case CT_BOOL: return ((const uint8_t*)p)[i];
        default: return 0;
    }
}
__device__ __forceinline__ double load_as_f64(const void* __restrict__ p, int ct, int64_t i) {
    switch (ct) {
        case CT_FLOAT64: return ((const double*)p)[i];
        case CT_FLOAT32: return (double)((const float*)p)[i];
        case CT_UINT64: return (double)((const uint64_t*)p)[i];  // (its int64 pattern would read 2^63 and above as negative)
        default: return (double)load_int_as_i64(p, ct, i);
    }
}
// The bits of the `size`-byte cell i, zero-extended.
__device__ __forceinline__ uint64_t load_bits(const void* __restrict__ p, int size, int64_t i) {
    switch (size) {
        case 8: return ((const uint64_t*)p)[i];
        case 4: return ((const uint32_t*)p)[i];
        case 2: return ((const uint16_t*)p)[i];
        default: return ((const uint8_t*)p)[i];
    }
}
// dst[di] = src[si] for cells of `size` bytes.
__device__ __forceinline__ void copy_cell(void* dst, int64_t di, const void* src, int64_t si, int size) {
    switch (size) {
        case 8: ((uint64_t*)dst)[di] = ((const uint64_t*)src)[si]; break;
        case 4: ((uint32_t*)dst)[di] = ((const uint32_t*)src)[si]; break;
        case 2: ((uint16_t*)dst)[di] = ((const uint16_t*)src)[si]; break;
        default: ((uint8_t*)dst)[di] = ((const uint8_t*)src)[si]; break;
    }
}

// hash_keys (reference: bodo/libs/_array_hash.cpp:1599-1621) of one row over 1..MAX_HASH_KEYS key columns: the first column is
// hashed (hash_array_inner: sizeof(T) raw bytes of an integer / date column through XXH3, a float column through
// _Py_HashDouble first; NA -> hash_na_val = hash of int64 1), every further column's hash is folded in with
// hash_combine_boost.  Low 32 bits of the XXH3 value, as hash_inner_32 returns them.
constexpr int MAX_HASH_KEYS = 4;
struct KeySet {
    int n_keys;
    const void* data[MAX_HASH_KEYS];
    const uint8_t* valid[MAX_HASH_KEYS];
    int ctype[MAX_HASH_KEYS];
};
__device__ __forceinline__ uint32_t hash_key_column(const void* data, int ct, const uint8_t* valid, int64_t i, uint32_t seed) {
    if (!bit_valid(valid, i)) return (uint32_t)xxh3_64_short(1ull, 8, seed);
    if (ct == CT_FLOAT64 || ct == CT_FLOAT32) return (uint32_t)xxh3_64_short((uint64_t)py_hash_double(load_as_f64(data, ct, i)), 8, seed);
    if (ctype_size(ct) == 8) return (uint32_t)xxh3_64_short((uint64_t)load_int_as_i64(data, ct, i), 8, seed);
    return (uint32_t)xxh3_64_short((uint64_t)(uint32_t)load_int_as_i64(data, ct, i), 4, seed);  // 4-byte keys hash their 4 raw bytes
}
// Key hash policies of hash_keys_row.  ReferenceKeyHash is hash_key_column: the reference's placement, which hashes a valid
// float NaN as a value.  KeyClassHash hashes every cell of one key class alike, equality being the window's, the sort's and the
// groupby's: NA and a float NaN are one class (both hash as hash_na_val), -0.0 equals 0.0 (_Py_HashDouble gives both 0), and a
// 1- or 2-byte integer or bool key hashes as the 4-byte integer of its value.  On keys without NaN it is hash_key_column.
struct ReferenceKeyHash {
    __device__ __forceinline__ static uint32_t column(const void* data, int ct, const uint8_t* valid, int64_t i, uint32_t seed) {
        return hash_key_column(data, ct, valid, i, seed);
    }
};
struct KeyClassHash {
    __device__ __forceinline__ static uint32_t column(const void* data, int ct, const uint8_t* valid, int64_t i, uint32_t seed) {
        if ((ct == CT_FLOAT64 || ct == CT_FLOAT32) && bit_valid(valid, i) && isnan(load_as_f64(data, ct, i)))
            return (uint32_t)xxh3_64_short(1ull, 8, seed);
        return hash_key_column(data, ct, valid, i, seed);  // (its narrow-integer path reads 1- and 2-byte cells as their value)
    }
};
template <class H = ReferenceKeyHash>
__device__ __forceinline__ uint32_t hash_keys_row(const KeySet& k, int64_t i, uint32_t seed) {
    uint32_t h = H::column(k.data[0], k.ctype[0], k.valid[0], i, seed);
    for (int j = 1; j < k.n_keys; j++) h = hash_combine_boost(h, H::column(k.data[j], k.ctype[j], k.valid[j], i, seed));
    return h;
}

// order-preserving double <-> uint64 encoding (so float min/max are native 64-bit integer atomics)
__host__ __device__ __forceinline__ uint64_t f64_to_ordered(double d) {
#ifdef __CUDA_ARCH__
    uint64_t b = (uint64_t)__double_as_longlong(d);
#else
    uint64_t b; memcpy(&b, &d, 8);
#endif
    return b ^ ((b >> 63) ? 0xFFFFFFFFFFFFFFFFULL : 0x8000000000000000ULL);
}
// order-preserving signed form of a canon_float_key encoding of a non-NaN key (the join's runtime-filter bounds, so they stay
// int64 min / max): a negative double's magnitude bits are flipped.  Its own inverse.
__host__ __device__ __forceinline__ long long canon_float_ordered(long long k) { return k < 0 ? k ^ 0x7FFFFFFFFFFFFFFFLL : k; }
__host__ __device__ __forceinline__ double ordered_to_f64(uint64_t e) {
    uint64_t b = e ^ ((e >> 63) ? 0x8000000000000000ULL : 0xFFFFFFFFFFFFFFFFULL);
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double d; memcpy(&d, &b, 8); return d;
#endif
}

// ---- sort-key encoding: one order for the sort (sort.cu) and the groupby's min_row_number_filter (groupby.cu) ----
// One descriptor per sort key.  A key's width in bytes is held beside its c-type: the kernels' raw loads read it rather than
// derive it from the c-type, which keeps the inlined encoder from being specialised once per load width (smaller, faster filter
// and pass code).
struct SortKey { int ct, size, desc, na_last; };

// Radix word of a key cell whose bits are `raw` (zero-extended).  `na` comes in true for a null cell and leaves true for a null
// or NaN cell, whose word is 0.
__device__ __forceinline__ uint64_t sort_word(const SortKey& k, uint64_t raw, bool& na) {
    uint64_t w;
    int bits;
    if (k.ct == CT_FLOAT64) {
        const double d = __longlong_as_double((long long)raw);
        na = na || isnan(d);
        w = (uint64_t)canon_float_ordered(canon_float_key(d)) ^ 0x8000000000000000ull;
        bits = 64;
    } else if (k.ct == CT_FLOAT32) {
        const float f = __uint_as_float((uint32_t)raw);
        na = na || isnan(f);
        const uint32_t b = f == 0.0f ? 0u : (uint32_t)raw;
        w = b ^ ((b >> 31) ? 0xFFFFFFFFu : 0x80000000u);
        bits = 32;
    } else {
        bits = 8 * k.size;
        w = ctype_is_signed_int(k.ct) ? raw ^ (1ull << (bits - 1)) : raw;
    }
    if (k.desc) w = ~w & (bits == 64 ? ~0ull : (1ull << bits) - 1);
    return na ? 0 : w;
}
// NA-class bit of a key cell (`na`: null or NaN).
__device__ __forceinline__ uint32_t sort_class(const SortKey& k, bool na) { return na ? k.na_last : !k.na_last; }

// counter-based generator of the synthetic workload (SURVEY.md §8d); mirrored in oracle/bodo_oracle.c
// (oracle_synth_fill) and bodo_b200/synth.py.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x += 0x9e3779b97f4a7c15ULL;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ULL;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebULL;
    return x ^ (x >> 31);
}

inline int num_sms(int device) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    return n > 0 ? n : 132;  // H100 SXM
}

// Scratch buffers (bucket / retry / fail lists: up to GBs) come from a process-wide per-device pool and go back to
// it when a state dies, so creating an operator state per query does not pay cudaMalloc / cudaFree of gigabytes
// (cudaFree of multi-GB blocks is synchronous and costs tens of milliseconds).
// The pool is stream-ordered: a released block remembers an event recorded on the releasing thread's scratch stream
// (scratch_set_stream: every state entry point sets it to the state's stream) and is only handed out again once that
// event has completed.  Pooled bytes are capped (B200_POOL_MAX_BYTES, default 24 GiB; scratch_trim frees on request).
void* scratch_acquire(int device, size_t bytes, size_t* got);
void scratch_release(int device, void* p, size_t bytes);
void scratch_set_stream(cudaStream_t s);
void scratch_trim(int device, size_t keep_bytes);
void* pinned_acquire(size_t bytes);   // small pinned host blocks (counter mirrors), pooled for the same reason
void pinned_release(void* p, size_t bytes);

// Kernels every operator uses, launched with `grid` CTAs of 256 threads on `st` (misc.cu).
// words[i / 32] bit (i % 32) = bytes[i] != 0 for i < n; the last word's bits past n are 0.
void launch_pack_bitmap(const uint8_t* bytes, int64_t n, uint32_t* words, int grid, cudaStream_t st);
// n 64-bit words at p set to v
void launch_fill_u64(void* p, uint64_t n, unsigned long long v, int grid, cudaStream_t st);

// RAII device buffer drawn from the pool of the CURRENT device (states call cudaSetDevice first).
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    int device = -1;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes), device(o.device) { o.p = nullptr; o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p = o.p; bytes = o.bytes; device = o.device; o.p = nullptr; o.bytes = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() { if (p) scratch_release(device, p, bytes); p = nullptr; bytes = 0; }
    void alloc(size_t n) {
        release();
        if (n == 0) n = 8;
        B200_CUDA(cudaGetDevice(&device));
        p = scratch_acquire(device, n, &bytes);
    }
    void ensure(size_t n) { if (n > bytes) alloc(n); }
    void ensure(int /*dev*/, size_t n) { ensure(n); }
    template <typename T> T* as() const { return (T*)p; }
};
using PooledBuf = DevBuf;

// Stable ascending radix sort of rows [0, n) by n_keys (1..4) plain device columns without NAs, key j at data[j] encoded by
// keys[j] (sort_word), through the full sort's histogram and pass kernels (sort.cu), on stream `st`.  Returns the permutation in
// ids[0] or ids[1] (mask each entry with 0x7FFFFFFF), or nullptr for the identity (every digit constant, or n == 0).  Adds the
// digit passes it ran to *passes_run unless that is nullptr.
const uint32_t* radix_sort_columns(int n_keys, const void* const* data, const SortKey* keys, int64_t n, DevBuf (&ids)[2], cudaStream_t st,
                                   int64_t* passes_run = nullptr);

// ---- tile scans (join.cu's offsets, sort.cu's window): a tile of 2048 rows, 256 threads x 8 items ----
// A scan runs in three launches: each tile's reduction, tile_carry_kernel over the tile values, then each tile's scan seeded by
// its prefix (tile_scan).  A scan value is a monoid M: M::T the value, M::identity(), and M::combine(a, b) with a covering the
// earlier rows.  Values move between lanes word by word (shfl_up / shfl_xor), so M::T is trivially copyable and 4-byte aligned.
// A value type may supply its own shfl_up(T, int) next to it: the helpers call shfl_up unqualified, so argument-dependent lookup
// at instantiation picks that overload over the word-wise one (sort.cu does so for the window's scan values).
constexpr int TILE_THREADS = 256, TILE_WARPS = TILE_THREADS / 32, TILE_ITEMS = 8, TILE_ROWS = TILE_THREADS * TILE_ITEMS;
// Row of this thread's item k in tile t: items are warp-strided, so every load and store is coalesced.  tile_row(t, k) is
// tile_row(t, 0) + k * TILE_THREADS; a kernel whose item loop only indexes rows takes that form and holds fewer registers.
__device__ __forceinline__ int64_t tile_row(int64_t t, int k) {
    return t * TILE_ROWS + (k * TILE_WARPS + (threadIdx.x >> 5)) * 32 + (threadIdx.x & 31);
}

template <typename U>
struct SumOf {
    using T = U;
    __device__ __forceinline__ static T identity() { return 0; }
    __device__ __forceinline__ static T combine(T a, T b) { return a + b; }
};

template <bool UP, typename T>
__device__ __forceinline__ T shfl_words(T v, int o) {
    static_assert(sizeof(T) % 4 == 0, "a scan value is whole 32-bit words");
    uint32_t w[sizeof(T) / 4];
    memcpy(w, &v, sizeof(T));
#pragma unroll
    for (int j = 0; j < (int)(sizeof(T) / 4); j++) w[j] = UP ? __shfl_up_sync(0xffffffffu, w[j], o) : __shfl_xor_sync(0xffffffffu, w[j], o);
    memcpy(&v, w, sizeof(T));
    return v;
}
template <typename T> __device__ __forceinline__ T shfl_up(T v, int o) { return shfl_words<true>(v, o); }
template <typename T> __device__ __forceinline__ T shfl_xor(T v, int o) { return shfl_words<false>(v, o); }

template <typename M>
__device__ __forceinline__ typename M::T warp_inclusive_scan(typename M::T v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const typename M::T y = shfl_up(v, o);
        if (lane >= o) v = M::combine(y, v);
    }
    return v;
}

// The combine of every thread's v in the tile, in thread 0, for a commutative M: a warp butterfly, then the warps in order.
template <typename M>
__device__ __forceinline__ typename M::T block_reduce(typename M::T v) {
    __shared__ typename M::T s_warp[TILE_WARPS];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = M::combine(v, shfl_xor(v, o));
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < TILE_WARPS; w++) v = M::combine(v, s_warp[w]);
    return v;
}

// s_seg[k * TILE_WARPS + warp] holds the total of segment (item k, warp), 32 rows; each becomes its exclusive prefix seeded by
// `seed`.  Warp 0 scans the 64 segments in row order, two per lane.  Every thread of the tile calls it.  The seed is a reference,
// so a tile prefix in memory is read by warp 0 only, after the barrier, and not held in every thread's registers.
template <typename M>
__device__ __forceinline__ void tile_segment_scan(typename M::T* s_seg, const typename M::T& seed) {
    using T = typename M::T;
    static_assert(TILE_ITEMS * TILE_WARPS == 64, "two segments per lane");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (warp == 0) {
        const T x0 = s_seg[2 * lane], x1 = s_seg[2 * lane + 1];
        const T ex = shfl_up(warp_inclusive_scan<M>(M::combine(x0, x1)), 1);
        T base = seed;
        if (lane > 0) base = M::combine(base, ex);
        s_seg[2 * lane] = base;
        s_seg[2 * lane + 1] = M::combine(base, x0);
    }
    __syncthreads();
}

// Inclusive scan of this thread's TILE_ITEMS values of a tile (v[k] at tile_row(t, k)), seeded by `seed`: a warp scan per item,
// the segment scan, then each segment's prefix combined in.
template <typename M>
__device__ __forceinline__ void tile_scan(const typename M::T& seed, typename M::T (&v)[TILE_ITEMS]) {
    __shared__ typename M::T s_seg[TILE_ITEMS * TILE_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) {
        v[k] = warp_inclusive_scan<M>(v[k]);
        if (lane == 31) s_seg[k * TILE_WARPS + warp] = v[k];
    }
    tile_segment_scan<M>(s_seg, seed);
#pragma unroll
    for (int k = 0; k < TILE_ITEMS; k++) v[k] = M::combine(s_seg[k * TILE_WARPS + warp], v[k]);
}

// One block of 1024 threads, each a contiguous run of the n tile values c: c becomes their exclusive scan and *total (unless
// nullptr) their combine.  A run's prefix starts from the identity, takes the earlier warps in order, then the earlier lanes of
// its warp; the runs are then walked left to right.  The order depends on n only, so float scans are reproducible.
template <typename M>
__global__ void __launch_bounds__(1024) tile_carry_kernel(typename M::T* c, int64_t n, typename M::T* total) {
    using T = typename M::T;
    __shared__ T s_agg[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t per = (n + 1023) / 1024, t0 = threadIdx.x * per, t1 = min(n, t0 + per);
    T acc = M::identity();
    for (int64_t t = t0; t < t1; t++) acc = M::combine(acc, c[t]);
    const T inc = warp_inclusive_scan<M>(acc);
    if (lane == 31) s_agg[warp] = inc;
    __syncthreads();
    T run = M::identity();
    for (int w = 0; w < warp; w++) run = M::combine(run, s_agg[w]);
    const T ex = shfl_up(inc, 1);
    if (lane > 0) run = M::combine(run, ex);
    for (int64_t t = t0; t < t1; t++) {
        const T v = c[t];
        c[t] = run;
        run = M::combine(run, v);
    }
    if (total && threadIdx.x == 1023) *total = run;
}

// Exclusive scan u32 -> u64 (join.cu: offsets_tile_sum_kernel, tile_carry_kernel, offsets_tile_scan_kernel).
struct Scanner {
    DevBuf sums, total;
    unsigned long long* h_total = nullptr;
    ~Scanner();
    // out[i] = sum_{j<i} in[j] on stream st; returns the grand total (synchronises the stream); adds its launches to *launches
    unsigned long long run(const uint32_t* in, int64_t n, unsigned long long* out, cudaStream_t st, int64_t* launches);
};

}  // namespace b200
