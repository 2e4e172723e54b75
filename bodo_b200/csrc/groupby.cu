// groupby.cu — streaming hash groupby/aggregate on one GPU (H100, sm_90a).
//
// Replaces GroupbyState + groupby_agg_build_consume_batch + FinalizeBuild of the reference
// (bodo/libs/streaming/_groupby.cpp:2554-3031, 4325-4457, 4062-4256) and the aggregate kernels of
// bodo/libs/groupby/_groupby_agg_funcs.h.  Design (see DESIGN.md):
//   * one persistent open-addressing table per state (linear probing, load <= 0.5, int64 keys — float keys as
//     canon_float_key, see canon_keys — SoA accumulator columns), instead of the reference's per-batch update table + combine;
//   * the consume kernel fuses hash + find-or-insert + every aggregate update of a row;
//   * rows whose insert would overfill the table are appended to a fail list; the host grows/rehashes
//     the table and replays only those rows (the reference's transactional retry,
//     _groupby.cpp:3309-3341, without the partition split);
//   * finalize compacts occupied slots and evaluates the output columns (mean_eval etc.).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <memory>
#include <vector>

#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>

#include "common.cuh"

namespace b200 {

constexpr long long EMPTY_KEY = (long long)0x8000000000000000ULL;  // INT64_MIN marks a free slot
constexpr int MAX_OPS = 16;
constexpr int64_t CHUNK_ROWS = 1ll << 28;  // rows per consume chunk (bounds the fail list of the direct path at 1 GiB)

// var / std / var_pop / std_pop / skew / kurtosis accumulate the moments of d = x - c about a per-group shift c: K_SHIFT holds c
// (NaN until the group's first non-NA value CASes itself in; c never changes after that), K_MOM1 holds sum d (a0) and the count
// (a1), K_MOM2 sum d^2, K_MOM3 sum d^3, K_MOM4 sum d^4.  They are consecutive primitives, K_SHIFT first: apply_ops and
// combine_apply carry d (or the partial's shift difference) in registers from K_SHIFT to the sums after it.  When the values lie within a factor of 2 of c,
// x - c is exact (Sterbenz), so a large common offset (epoch seconds, prices in cents) costs no digits.
enum OpKind : int { K_SUM_I64 = 0, K_SUM_F64, K_COUNT, K_SIZE, K_MEAN, K_MIN_I64, K_MAX_I64, K_MIN_F64, K_MAX_F64,
                    K_MOM2, K_MOM3,
                    // first / last non-NA value in row order (aggfunc<first / last>, _groupby_agg_funcs.h:594-611): a0 = value
                    // bits, a1 = sequence number of the row that supplied it (see groupby_firstlast_fix_kernel)
                    K_FIRST, K_LAST,
                    K_NUNIQUE,  // number of distinct non-NA values: filled at finalize from a nested (key, value) distinct state
                    // evaluation-only kinds of composite functions (accumulators: K_MOM1 + K_MOM2 (+ K_MOM3))
                    E_VAR, E_STD, E_VAR_POP, E_STD_POP, E_SKEW,
                    K_SHIFT, K_MOM1,
                    K_MRNF,  // one word of a min_row_number_filter winner record (see mrnf_merge_kernel); no consume kernel applies it
                    // prod: a0 = product (uint64 mod 2^64 / double bits), starts at 1; no native atomic (see prod_update)
                    K_PROD_I64, K_PROD_F64,
                    K_MOM4,  // sum d^4 of a moment group (kurtosis), after K_MOM3
                    // 64-bit word ops: bitor / bitand / bitxor of the integer value (AND starts all-ones) and boolor / booland of its
                    // truth (0 or all-ones); a1 (when present) counts the non-NA rows
                    K_OR, K_AND, K_XOR, K_LOR, K_LAND,
                    K_COUNT_IF,  // a0 = rows whose value is true (nonzero); a1 (when present) counts the non-NA rows
                    // evaluation-only kinds: kurtosis (accumulators K_MOM1 .. K_MOM4), boolxor (K_COUNT_IF: exactly one true)
                    E_KURT, E_BOOLXOR,
                    // holistic aggregates (see holistic_append_kernel): K_HID is the group's id word, all-ones until claimed; E_MODE,
                    // E_PCONT and E_PDISC are their result words, written at finalize (a0 = the result's bits, a1 = 0 once it is
                    // valid, all-ones before).  No consume kernel applies any of them: they lie past n_apply()
                    K_HID, E_MODE, E_PCONT, E_PDISC };
constexpr unsigned long long SHIFT_UNSET = 0x7ff8000000000000ull;  // K_SHIFT's initial value (quiet NaN; NaN values are skipped)

struct OpDesc {
    int kind;
    int in_ctype;
    const void* in_data;
    const uint8_t* in_valid;
    void* a0;  // main accumulator column (8 B / slot)
    void* a1;  // second accumulator (mean count, min/max seen-count) or nullptr
};

// The words of a state's device counter block (GroupbyState::d_counters), mirrored to the host by read_counters().
enum CounterSlot : int {
    CTR_GROUPS = 0,         // groups in the table (the tickets find_or_insert takes against the group limit)
    CTR_FAIL = 1,           // rows in the fail list (direct / multi-key / combine), or in the slot-0 retry list (SPG, SPG-G)
    CTR_OUT = 2,            // output cursor of the compaction
    CTR_NA = 3,             // the NA key is present (slot cap)
    CTR_MARKER = 4,         // the marker key EMPTY_KEY is present (slot cap + 1)
    CTR_WIDE = 5,           // SPG-N: rows that did not fit the narrow (int32 key, int32 value) format
    CTR_RETRY1 = 6,         // rows in the slot-1 retry list (SPG)
    CTR_XCHG_OVERFLOW = 7,  // fused exchange: some rank's share overflowed its slab segment, nobody combined
    CTR_RETRY_OVERFLOW = 8, // SPG / SPG-G: an entry did not fit its retry list and was dropped (the host raises an error)
    CTR_DENSE_WIDE = 9,     // SPG-N dense form: rows whose key or value offset did not fit its window
    N_COUNTERS = 10
};

struct ConsumeArgs {
    const void* key_data;
    const uint8_t* key_valid;
    int key_ctype;
    int dropna;
    int64_t n_rows;
    const uint32_t* index_list;  // nullptr: rows [0, n_rows); else replay of the listed rows
    long long* tkeys;
    uint64_t cap;  // power of two; slot cap = NA key, slot cap + 1 = the key equal to EMPTY_KEY
    long long* counters;  // the state's counter block (CounterSlot)
    long long group_limit;
    uint32_t* fail_list;
    unsigned long long seq_base;  // first / last: sequence number of row 0 of this launch, minus 1 (rank << 44 | rows consumed so far)
    int n_ops;
    OpDesc ops[MAX_OPS];
};

// find-or-insert with linear probing over 8-byte key slots; returns the slot, or UINT64_MAX when the table is at
// its group limit (group_limit < 0 disables the limit: rehash into a table that is known to be large enough).
// Bucketed 4-key variants of this probe (scratch/ubench2.cu) issue more L2 requests per row; the L2 random-request rate,
// not probe-chain latency, is what limits this path.
__device__ __forceinline__ uint64_t find_or_insert(long long* __restrict__ tkeys, uint64_t cap, long long key,
                                                   long long* counters, long long group_limit) {
    uint64_t mask = cap - 1;
    uint64_t s = (key_hash(key) >> 32) & mask;
    for (uint64_t probes = 0; probes <= mask; probes++) {
        long long k = __ldcg(tkeys + s);
        if (k == key) return s;
        if (k == EMPTY_KEY) {
            // take a ticket first so the table can never exceed group_limit (probing always terminates).  The lanes of the warp
            // that stand here together take their tickets with ONE atomic (coalesced group): a flush of 10^6 new groups is 10^6
            // tickets on a single address otherwise (measured 0.17 ms per operator state)
            if (group_limit >= 0) {
                const cooperative_groups::coalesced_group cgp = cooperative_groups::coalesced_threads();
                long long t = 0;
                if (cgp.thread_rank() == 0) t = (long long)atomicAdd((unsigned long long*)&counters[CTR_GROUPS], (unsigned long long)cgp.size());
                t = cgp.shfl(t, 0) + (long long)cgp.thread_rank();
                if (t >= group_limit) {
                    atomicAdd((unsigned long long*)&counters[CTR_GROUPS], (unsigned long long)-1ll);
                    return ~0ull;
                }
            }
            long long prev = atomicCAS((unsigned long long*)(tkeys + s), (unsigned long long)EMPTY_KEY,
                                       (unsigned long long)key);
            if (prev == EMPTY_KEY) return s;
            if (group_limit >= 0) atomicAdd((unsigned long long*)&counters[CTR_GROUPS], (unsigned long long)-1ll);  // lost the race
            if (prev == key) return s;
        }
        s = (s + 1) & mask;
    }
    return ~0ull;
}

// lookup only; UINT64_MAX when the key is not in the table
__device__ __forceinline__ uint64_t find_only(const long long* __restrict__ tkeys, uint64_t cap, long long key) {
    uint64_t mask = cap - 1;
    uint64_t s = (key_hash(key) >> 32) & mask;
    for (uint64_t probes = 0; probes <= mask; probes++) {
        long long k = __ldcg(tkeys + s);
        if (k == key) return s;
        if (k == EMPTY_KEY) return ~0ull;
        s = (s + 1) & mask;
    }
    return ~0ull;
}
// value of a first / last input as the 8 bytes kept in the accumulator (integers sign / zero extended, floats as double)
__device__ __forceinline__ bool firstlast_value(const OpDesc& op, int64_t row, unsigned long long& bits) {
    if (op.in_ctype == CT_FLOAT64 || op.in_ctype == CT_FLOAT32) {
        const double v = load_as_f64(op.in_data, op.in_ctype, row);
        bits = (unsigned long long)__double_as_longlong(v);
        return !isnan(v);
    }
    bits = (unsigned long long)load_int_as_i64(op.in_data, op.in_ctype, row);
    return true;
}

// the shift of a var / std / skew group (see K_SHIFT): the slot's c, or v when v is the first value to arrive
__device__ __forceinline__ double group_shift(double* c, double v) {
    const double s = __ldcg(c);  // once set, c never changes: a non-NaN read is final, a stale NaN only costs the CAS
    if (!isnan(s)) return s;
    const unsigned long long prev = atomicCAS((unsigned long long*)c, SHIFT_UNSET, (unsigned long long)__double_as_longlong(v));
    return prev == SHIFT_UNSET ? v : __longlong_as_double((long long)prev);
}

// prod has no native atomic, and a CAS loop on one word completes about one update per round trip to L2, however many warps wait.
// So a batch into few groups is multiplied together on chip first: the lanes of the warp that update the same word multiply their
// values (labeled_partition on the word's address: lanes of different aggregates can run this code together), then the warp's
// leader multiplies that into the CTA's entry for the word (ProdCache, shared memory), and the consume kernel multiplies every
// entry into its word once, at its end (prod_flush).  A word that finds no entry (more distinct words than the cache holds near
// its hash) takes the CAS loop on its global word directly, as the exchange's combine does.  Integers multiply as uint64 (exact
// mod 2^64 in any order), floats as doubles (the order is the only difference from a serial product).
constexpr int PC_SLOTS = 128, PC_PROBES = 8;
constexpr unsigned long long PC_FREE = 0, PC_BUSY = 2;  // entry keys: free, being filled, or word address | 1 for a float word
struct ProdCache {
    unsigned long long key[PC_SLOTS];
    unsigned long long val[PC_SLOTS];
};
template <bool F>
__device__ __forceinline__ unsigned long long prod_mul(unsigned long long a, unsigned long long b) {
    return F ? (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a) * __longlong_as_double((long long)b)) : a * b;
}
// *p *= v by CAS; a failed CAS backs off before it retries, so that a word many CTAs flush into at once is not flooded with CASes
// that carry a stale value
template <bool F>
__device__ __forceinline__ void prod_cas(unsigned long long* p, unsigned long long v, bool shared_word) {
    unsigned long long old = shared_word ? *(volatile unsigned long long*)p : __ldcg(p), seen;
    unsigned int pause = 32;
    for (;;) {
        seen = old;
        const unsigned long long next = prod_mul<F>(seen, v);
        if (next == seen) return;
        old = atomicCAS(p, seen, next);
        if (old == seen) return;
        if (!shared_word) {
            __nanosleep(pause);
            pause = pause < 4096 ? 2 * pause : pause;
        }
    }
}
template <bool F>
__device__ __forceinline__ void prod_update(unsigned long long* p, unsigned long long v, ProdCache* pc) {
    namespace cg = cooperative_groups;
    const cg::coalesced_group same = cg::labeled_partition(cg::coalesced_threads(), (unsigned long long)p);
    if constexpr (F) v = (unsigned long long)__double_as_longlong(cg::reduce(same, __longlong_as_double((long long)v), [](double x, double y) { return x * y; }));
    else v = cg::reduce(same, v, [](unsigned long long x, unsigned long long y) { return x * y; });
    if (same.thread_rank() != 0) return;
    if (pc) {
        const unsigned long long key = (unsigned long long)p | (F ? 1ull : 0ull);
        unsigned int h = (unsigned int)(key_hash((long long)key) >> 32) & (PC_SLOTS - 1);
        for (int probe = 0; probe < PC_PROBES;) {
            const unsigned long long k = *(volatile unsigned long long*)&pc->key[h];
            if (k == key) { prod_cas<F>(&pc->val[h], v, true); return; }
            if (k == PC_BUSY) continue;  // being filled: look again
            if (k == PC_FREE) {
                if (atomicCAS(&pc->key[h], PC_FREE, PC_BUSY) == PC_FREE) {  // the entry starts at this warp's product
                    pc->val[h] = v;
                    __threadfence_block();
                    atomicExch(&pc->key[h], key);
                    return;
                }
                continue;  // somebody else took it: look at it again
            }
            h = (h + 1) & (PC_SLOTS - 1);
            probe++;
        }
    }
    prod_cas<F>(p, v, false);
}
// A consume kernel's cache around its row loop: `on` (some op is a prod; uniform over the CTA) clears it before the loop, then
// multiplies every entry into its word after the loop.
__device__ __forceinline__ void prod_cache_clear(ProdCache& pc, bool on) {
    if (!on) return;
    for (int i = threadIdx.x; i < PC_SLOTS; i += blockDim.x) pc.key[i] = PC_FREE;
    __syncthreads();
}
__device__ __forceinline__ void prod_flush(ProdCache& pc, bool on) {
    if (!on) return;
    __syncthreads();
    for (int i = threadIdx.x; i < PC_SLOTS; i += blockDim.x) {
        const unsigned long long k = pc.key[i];
        if (k == PC_FREE) continue;
        if (k & 1ull) prod_cas<true>((unsigned long long*)(k & ~7ull), pc.val[i], false);
        else prod_cas<false>((unsigned long long*)k, pc.val[i], false);
    }
}
template <typename A>
__host__ __device__ __forceinline__ bool has_prod(const A& a) {
    for (int j = 0; j < a.n_ops; j++) if (a.ops[j].kind == K_PROD_I64 || a.ops[j].kind == K_PROD_F64) return true;
    return false;
}
// the dynamic shared memory of a consume launch: the ProdCache only when it applies a prod, so that other signatures keep the
// whole L1 / shared split they had
template <typename A> size_t prod_smem_bytes(const A& a) { return has_prod(a) ? sizeof(ProdCache) : 0; }
template <typename A> bool has_reduction_kinds(const A& a) {
    for (int j = 0; j < a.n_ops; j++) if (a.ops[j].kind > K_MRNF) return true;
    return false;
}
// The operand of a word op (K_OR .. K_COUNT_IF): the integer for bitor / bitand / bitxor, else the value's truth as 0 or all-ones
// (nonzero is true).  False for an NA value (NaN).
__device__ __forceinline__ bool word_operand(const OpDesc& op, int64_t row, unsigned long long& w) {
    if (ctype_is_float(op.in_ctype)) {
        const double v = load_as_f64(op.in_data, op.in_ctype, row);
        w = v != 0.0 ? ~0ull : 0ull;
        return !isnan(v);
    }
    w = (unsigned long long)load_int_as_i64(op.in_data, op.in_ctype, row);
    if (op.kind != K_OR && op.kind != K_AND && op.kind != K_XOR) w = w ? ~0ull : 0ull;
    return true;
}
// One row's word op on `p`.  An OR / XOR with 0 and an AND with all-ones cannot change the word, so those rows only count.
__device__ __forceinline__ void word_update(int kind, unsigned long long* p, unsigned long long w) {
    switch (kind) {
        case K_AND: case K_LAND: if (w != ~0ull) atomicAnd(p, w); break;
        case K_COUNT_IF: if (w) atomicAdd(p, 1ull); break;
        case K_XOR: if (w) atomicXor(p, w); break;
        default: if (w) atomicOr(p, w); break;  // K_OR, K_LOR
    }
}

// One row's update of prod, a word op or count_if.
__device__ __forceinline__ void apply_reduction_op(const OpDesc& op, uint64_t slot, int64_t row, ProdCache* pc) {
    switch (op.kind) {
        case K_PROD_I64:
            prod_update<false>((unsigned long long*)op.a0 + slot, (unsigned long long)load_int_as_i64(op.in_data, op.in_ctype, row), pc);
            break;
        case K_PROD_F64: {
            const double v = load_as_f64(op.in_data, op.in_ctype, row);
            if (!isnan(v)) prod_update<true>((unsigned long long*)op.a0 + slot, (unsigned long long)__double_as_longlong(v), pc);
            break;
        }
        case K_OR: case K_AND: case K_XOR: case K_LOR: case K_LAND: case K_COUNT_IF: {
            unsigned long long w;
            if (!word_operand(op, row, w)) break;
            word_update(op.kind, (unsigned long long*)op.a0 + slot, w);
            if (op.a1) atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
            break;
        }
    }
}

// RED: the launch applies some kind appended after K_MRNF (prod, kurtosis's K_MOM4, the word ops, count_if).  The consume kernels
// are instantiated for both values and the host picks one per state (has_reduction_kinds), so the other signatures run the row
// loop they ran before these kinds existed.
template <bool RED, typename A>
__device__ __forceinline__ void apply_ops(const A& a, uint64_t slot, int64_t row, ProdCache* pc) {
    double d = 0.0;  // K_SHIFT -> K_MOM*: the row's value minus its group's shift
    bool has_d = false;
#pragma unroll 1
    for (int j = 0; j < a.n_ops; j++) {
        const OpDesc& op = a.ops[j];
        if (op.kind == K_SIZE) {  // size_agg (_groupby_agg_funcs.h:661-669): counts every row
            atomicAdd((unsigned long long*)op.a0 + slot, 1ull);
            continue;
        }
        if (!bit_valid(op.in_valid, row)) continue;  // nullable input: skip NA (do_apply_to_column.cpp:1796-1823)
        switch (op.kind) {
            case K_SUM_I64:  // casted_aggfunc sum: int64 accumulate, wraparound (_groupby_agg_funcs.h:176-190)
                atomicAdd((unsigned long long*)op.a0 + slot, (unsigned long long)load_int_as_i64(op.in_data, op.in_ctype, row));
                break;
            case K_COUNT: {  // count_agg (:644-657): non-NA values (NaN is NA for floats)
                bool ok = true;
                if (op.in_ctype == CT_FLOAT64 || op.in_ctype == CT_FLOAT32) ok = !isnan(load_as_f64(op.in_data, op.in_ctype, row));
                if (ok) atomicAdd((unsigned long long*)op.a0 + slot, 1ull);
                break;
            }
            case K_SUM_F64: {
                double v = load_as_f64(op.in_data, op.in_ctype, row);
                if (!isnan(v)) atomicAdd((double*)op.a0 + slot, v);
                break;
            }
            case K_MEAN: {  // mean_agg (:673-689): double sum + uint64 count
                double v = load_as_f64(op.in_data, op.in_ctype, row);
                if (!isnan(v)) {
                    atomicAdd((double*)op.a0 + slot, v);
                    atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                }
                break;
            }
            case K_SHIFT: {  // (an NA row skips the whole moment group: its ops share the input column)
                const double v = load_as_f64(op.in_data, op.in_ctype, row);
                has_d = !isnan(v);
                if (has_d) d = v - group_shift((double*)op.a0 + slot, v);
                break;
            }
            case K_MOM1:
                if (has_d) {
                    atomicAdd((double*)op.a0 + slot, d);
                    atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                }
                break;
            case K_MOM2: case K_MOM3:
                if (has_d) atomicAdd((double*)op.a0 + slot, op.kind == K_MOM2 ? d * d : d * d * d);
                break;
            default:
                if constexpr (RED) {
                    if (op.kind == K_MOM4) { if (has_d) atomicAdd((double*)op.a0 + slot, (d * d) * (d * d)); }
                    else apply_reduction_op(op, slot, row, pc);  // prod, the word ops, count_if
                }
                break;
            case K_FIRST: case K_LAST: {  // phase 1: which row supplies the value (phase 2 writes it, groupby_firstlast_fix_kernel)
                unsigned long long bits;
                if (firstlast_value(op, row, bits)) {
                    const unsigned long long seq = a.seq_base + (unsigned long long)row + 1ull;
                    if (op.kind == K_FIRST) atomicMin((unsigned long long*)op.a1 + slot, seq);
                    else atomicMax((unsigned long long*)op.a1 + slot, seq);
                }
                break;
            }
            case K_MIN_I64:
                atomicMin((long long*)op.a0 + slot, (long long)load_int_as_i64(op.in_data, op.in_ctype, row));
                if (op.a1) atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                break;
            case K_MAX_I64:
                atomicMax((long long*)op.a0 + slot, (long long)load_int_as_i64(op.in_data, op.in_ctype, row));
                if (op.a1) atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                break;
            case K_MIN_F64: {
                double v = load_as_f64(op.in_data, op.in_ctype, row);
                if (!isnan(v)) {
                    atomicMin((unsigned long long*)op.a0 + slot, f64_to_ordered(v));
                    if (op.a1) atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                }
                break;
            }
            case K_MAX_F64: {
                double v = load_as_f64(op.in_data, op.in_ctype, row);
                if (!isnan(v)) {
                    atomicMax((unsigned long long*)op.a0 + slot, f64_to_ordered(v));
                    if (op.a1) atomicAdd((unsigned long long*)op.a1 + slot, 1ull);
                }
                break;
            }
        }
    }
}

// Generic fused consume kernel: any key/value types, any mix of aggregates, nullable columns.
template <bool RED>
__global__ void __launch_bounds__(256) groupby_consume_kernel(const __grid_constant__ ConsumeArgs a) {
    extern __shared__ __align__(8) unsigned char prod_smem[];  // a ProdCache when some op is a prod (prod_smem_bytes), else empty
    ProdCache& pc = *reinterpret_cast<ProdCache*>(prod_smem);
    const bool prod = RED && has_prod(a);
    prod_cache_clear(pc, prod);
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n_rows; i += stride) {
        int64_t row = a.index_list ? (int64_t)a.index_list[i] : i;
        bool kvalid = bit_valid(a.key_valid, row);
        uint64_t slot;
        if (!kvalid) {
            if (a.dropna) continue;  // filter_na_keys (_groupby.cpp:4278-4309)
            slot = a.cap;
            a.counters[CTR_NA] = 1;
        } else {
            long long key = load_int_as_i64(a.key_data, a.key_ctype, row);
            if (key == EMPTY_KEY) {
                slot = a.cap + 1;
                a.counters[CTR_MARKER] = 1;
            } else {
                slot = find_or_insert(a.tkeys, a.cap, key, a.counters, a.group_limit);
                if (slot == ~0ull) {
                    unsigned long long f = atomicAdd((unsigned long long*)&a.counters[CTR_FAIL], 1ull);
                    a.fail_list[f] = (uint32_t)row;
                    continue;
                }
            }
        }
        apply_ops<RED>(a, slot, row, &pc);
    }
    prod_flush(pc, prod);
}

// first / last, phase 2 (after every row of the launch — replays included — has been applied): the row whose sequence number
// won the atomicMin / atomicMax writes its value.  Two passes because (value, sequence) cannot be updated by one atomic.
__global__ void __launch_bounds__(256) groupby_firstlast_fix_kernel(const __grid_constant__ ConsumeArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < a.n_rows; row += stride) {
        uint64_t slot;
        if (!bit_valid(a.key_valid, row)) { if (a.dropna) continue; slot = a.cap; }
        else {
            const long long key = load_int_as_i64(a.key_data, a.key_ctype, row);
            slot = key == EMPTY_KEY ? a.cap + 1 : find_only(a.tkeys, a.cap, key);
            if (slot == ~0ull) continue;
        }
        const unsigned long long seq = a.seq_base + (unsigned long long)row + 1ull;
#pragma unroll 1
        for (int j = 0; j < a.n_ops; j++) {
            const OpDesc& op = a.ops[j];
            if (op.kind != K_FIRST && op.kind != K_LAST) continue;
            if (!bit_valid(op.in_valid, row)) continue;
            unsigned long long bits;
            if (firstlast_value(op, row, bits) && ((const unsigned long long*)op.a1)[slot] == seq) ((unsigned long long*)op.a0)[slot] = bits;
        }
    }
}

// Specialised consume kernel for the headline shape: non-null int64 key, non-null int64 value,
// aggregates drawn from {sum, count, size} of that one value column (BASELINE.json C1/C2).
// Two rows per thread per iteration through 128-bit loads; the aggregate updates are `red` (no return).
template <bool HAS_SUM, bool HAS_CNT>
__global__ void __launch_bounds__(256) groupby_consume_i64_sumcount_kernel(
    const long long* __restrict__ keys, const long long* __restrict__ vals, int64_t n_rows, long long* tkeys, uint64_t cap,
    unsigned long long* acc_sum, unsigned long long* acc_cnt, long long* counters, long long group_limit,
    uint32_t* fail_list) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x * 2;
    int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 2;
    for (; i < n_rows; i += stride) {
        long long k[2], v[2];
        int m = 2;
        if (i + 1 < n_rows) {
            longlong2 kk = __ldcs(reinterpret_cast<const longlong2*>(keys + i));
            k[0] = kk.x; k[1] = kk.y;
            if (HAS_SUM) { longlong2 vv = __ldcs(reinterpret_cast<const longlong2*>(vals + i)); v[0] = vv.x; v[1] = vv.y; }
        } else {
            k[0] = keys[i]; k[1] = 0; m = 1;
            if (HAS_SUM) { v[0] = vals[i]; v[1] = 0; }
        }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            if (r >= m) break;
            uint64_t sl;
            if (k[r] == EMPTY_KEY) {
                sl = cap + 1;
                counters[CTR_MARKER] = 1;
            } else {
                sl = find_or_insert(tkeys, cap, k[r], counters, group_limit);
                if (sl == ~0ull) {
                    unsigned long long f = atomicAdd((unsigned long long*)&counters[CTR_FAIL], 1ull);
                    fail_list[f] = (uint32_t)(i + r);
                    continue;
                }
            }
            if (HAS_SUM) atomicAdd(acc_sum + sl, (unsigned long long)v[r]);
            if (HAS_CNT) atomicAdd(acc_cnt + sl, 1ull);
        }
    }
}

// Float key column -> its int64 table keys (canon_float_key), before any consume kernel reads the chunk.  A pure stream:
// 8 (float64) or 4 (float32) bytes read and 8 written per row, four rows per thread through 16-byte loads and stores when
// both columns are 16-byte aligned; the rest (or everything, when they are not) goes row by row.
template <typename F>
__global__ void __launch_bounds__(256) canon_float_key_kernel(const F* __restrict__ in, long long* __restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t t0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t n4 = (((uintptr_t)in | (uintptr_t)out) & 15) == 0 ? n / 4 : 0;
    for (int64_t q = t0; q < n4; q += stride) {
        double v[4];
        if constexpr (sizeof(F) == 8) {
            const double2 a = __ldcs(reinterpret_cast<const double2*>(in) + 2 * q), b = __ldcs(reinterpret_cast<const double2*>(in) + 2 * q + 1);
            v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        } else {
            const float4 a = __ldcs(reinterpret_cast<const float4*>(in) + q);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
        }
        longlong2* o = reinterpret_cast<longlong2*>(out) + 2 * q;
        o[0] = make_longlong2(canon_float_key(v[0]), canon_float_key(v[1]));
        o[1] = make_longlong2(canon_float_key(v[2]), canon_float_key(v[3]));
    }
    for (int64_t i = 4 * n4 + t0; i < n; i += stride) out[i] = canon_float_key((double)in[i]);
}

struct RehashArgs {
    const long long* old_keys;
    uint64_t old_cap;
    long long* new_keys;
    uint64_t new_cap;
    int n_acc;
    const unsigned long long* old_acc[2 * MAX_OPS];
    unsigned long long* new_acc[2 * MAX_OPS];
};
// grow: re-insert every occupied slot (and the two special slots) into the new arrays
__global__ void rehash_kernel(const __grid_constant__ RehashArgs a) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < a.old_cap + 2; s += stride) {
        uint64_t ns;
        if (s >= a.old_cap) {
            ns = a.new_cap + (s - a.old_cap);
        } else {
            long long k = a.old_keys[s];
            if (k == EMPTY_KEY) continue;
            ns = find_or_insert(a.new_keys, a.new_cap, k, nullptr, -1);
        }
        for (int j = 0; j < a.n_acc; j++) a.new_acc[j][ns] = a.old_acc[j][s];
    }
}

// ---- finalize: compact occupied slots, then evaluate output columns ----
// n_pes > 1: only the groups this rank OWNS (hash_to_rank(key) == rank) are output — after the exchange the table still
// holds the partial aggregates of groups that were sent to their owners (they are never touched again: received rows only
// carry keys this rank owns).  key_ctype: the key's input type; a float key (canon_float_key) has the NaN group in the marker slot
// and dropna drops it.
__global__ void compact_slots_kernel(const long long* __restrict__ tkeys, uint64_t cap, const long long* counters,
                                     long long* cursor, uint64_t* slot_of_out, int n_pes, int rank, int key_ctype, bool dropna) {
    const bool na_present = counters[CTR_NA] != 0, empty_present = counters[CTR_MARKER] != 0 && !(ctype_is_float(key_ctype) && dropna);
    const uint32_t na_hash = (uint32_t)xxh3_64_short(1ull, 8, SEED_HASH_PARTITION);  // hash_na_val (_array_hash.cpp:22-29)
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s0 = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s0 < ((cap + 2 + 31) & ~31ull); s0 += stride) {
        bool occ = false;
        if (s0 < cap) occ = tkeys[s0] != EMPTY_KEY;
        else if (s0 == cap) occ = na_present;
        else if (s0 == cap + 1) occ = empty_present;
        if (occ && n_pes > 1) {
            const uint32_t h = s0 == cap ? na_hash : owner_key_hash(s0 < cap ? tkeys[s0] : EMPTY_KEY, key_ctype);
            occ = hash_to_rank_u32(h, n_pes) == rank;
        }
        unsigned m = __ballot_sync(0xffffffffu, occ);
        int lane = threadIdx.x & 31;
        long long base = 0;
        if (lane == 0 && m) base = (long long)atomicAdd((unsigned long long*)cursor, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (occ) slot_of_out[base + __popc(m & ((1u << lane) - 1))] = s0;
    }
}

struct OutDesc {
    int kind;       // OpKind
    int out_ctype;  // CType of the output column
    const void* a0;
    const void* a1;
    const void* b0;  // composite functions: sum of squares
    const void* c0;  //                      sum of cubes
    const void* d0;  //                      sum of fourth powers
    void* out_data;
    uint32_t* out_valid;  // validity bitmap as 32-bit words, or nullptr when the column has no nulls
};
struct EvalArgs {
    const long long* tkeys;
    uint64_t cap;
    const uint64_t* slot_of_out;
    const long long* n_out_ptr;  // number of compacted slots (device counter written by compact_slots_kernel)
    int key_ctype;
    void* out_keys;
    uint32_t* out_key_valid;  // nullptr unless the NA-key group can exist
    int n_ops;
    OutDesc ops[MAX_OPS];
};

__device__ __forceinline__ void store_int_typed(void* p, int ct, int64_t i, long long v) {
    switch (ct) {
        case CT_INT64: case CT_UINT64: case CT_DATETIME: case CT_TIMEDELTA: ((long long*)p)[i] = v; break;
        case CT_INT32: case CT_UINT32: case CT_DATE: ((int32_t*)p)[i] = (int32_t)v; break;
        case CT_INT16: case CT_UINT16: ((int16_t*)p)[i] = (int16_t)v; break;
        case CT_INT8: case CT_UINT8: case CT_BOOL: ((int8_t*)p)[i] = (int8_t)v; break;
    }
}
__device__ __forceinline__ void store_f_typed(void* p, int ct, int64_t i, double v) {
    if (ct == CT_FLOAT32) ((float*)p)[i] = (float)v; else ((double*)p)[i] = v;
}

// eval_groupby_funcs_helper (_groupby.cpp:396-457) + output null rules (aggfunc_output_initialize_kernel,
// groupby/_groupby_common.cpp:50-74: sum/count/size valid, min/max/mean NULL when nothing was seen).
__global__ void eval_output_kernel(const __grid_constant__ EvalArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_out = *a.n_out_ptr;
    int64_t n_round = (n_out + 31) & ~31ll;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_round; p += stride) {
        bool in = p < n_out;
        uint64_t s = in ? a.slot_of_out[p] : 0;
        bool key_ok = true;
        if (in && a.tkeys) {  // single-key tables only (multi-key tables write their key columns in eval_mk_keys_kernel)
            long long key = s < a.cap ? a.tkeys[s] : (s == a.cap ? 0 : EMPTY_KEY);
            key_ok = s != a.cap;
            if (ctype_is_float(a.key_ctype)) store_f_typed(a.out_keys, a.key_ctype, p, canon_float_decode(key));
            else store_int_typed(a.out_keys, a.key_ctype, p, key);
        }
        if (a.out_key_valid) {
            unsigned m = __ballot_sync(0xffffffffu, in && key_ok);
            if ((threadIdx.x & 31) == 0) a.out_key_valid[p >> 5] = m;
        }
#pragma unroll 1
        for (int j = 0; j < a.n_ops; j++) {
            const OutDesc& op = a.ops[j];
            bool valid = in;
            if (in) {
                switch (op.kind) {
                    case K_SUM_I64: case K_COUNT: case K_SIZE: case K_NUNIQUE:
                        store_int_typed(op.out_data, op.out_ctype, p, ((const long long*)op.a0)[s]);
                        break;
                    case K_SUM_F64:
                        store_f_typed(op.out_data, op.out_ctype, p, ((const double*)op.a0)[s]);
                        break;
                    case K_MEAN: {  // mean_eval (do_apply_to_column.cpp:880-913)
                        unsigned long long c = ((const unsigned long long*)op.a1)[s];
                        valid = c > 0;
                        store_f_typed(op.out_data, op.out_ctype, p, valid ? ((const double*)op.a0)[s] / (double)c : __longlong_as_double(0x7ff8000000000000ll));
                        break;
                    }
                    case E_VAR: case E_STD: case E_VAR_POP: case E_STD_POP: {
                        // var_eval / std_eval (groupby/_groupby_eval.h:71-95).  The reference carries Welford's (count, mean,
                        // M2); the device carries the power sums of d = x - c (atomics cannot run Welford's recurrence, see
                        // K_SHIFT) and forms M2 = S2 - S1^2 / n, in which c cancels.  Its relative error is O(n u (1 + (mean -
                        // c)^2 / var)), and c is one of the group's values, so it does not grow with |mean| / spread
                        // (tests/test_gpu_groupby_float_values.py derives the bound)
                        const double n = (double)((const unsigned long long*)op.a1)[s];
                        const double s1 = ((const double*)op.a0)[s], s2 = ((const double*)op.b0)[s];
                        const bool pop = op.kind == E_VAR_POP || op.kind == E_STD_POP;
                        valid = pop ? n >= 1 : n >= 2;
                        double m2 = s2 - s1 * s1 / n;
                        if (m2 < 0) m2 = 0;
                        double r = valid ? m2 / (pop ? n : n - 1) : __longlong_as_double(0x7ff8000000000000ll);
                        if (valid && (op.kind == E_STD || op.kind == E_STD_POP)) r = sqrt(r);
                        store_f_typed(op.out_data, op.out_ctype, p, r);
                        break;
                    }
                    case E_SKEW: {  // skew_eval (groupby/_groupby_eval.h:110-137) on the power sums of d = x - c (c cancels)
                        const unsigned long long cnt = ((const unsigned long long*)op.a1)[s];
                        const double n = (double)cnt, m1 = ((const double*)op.a0)[s], m2 = ((const double*)op.b0)[s], m3 = ((const double*)op.c0)[s];
                        valid = cnt >= 3;
                        double r = __longlong_as_double(0x7ff8000000000000ll);
                        if (valid) {
                            const double mean = m1 / n;
                            const double num = m3 - 3.0 * m2 * mean + 2.0 * n * mean * mean * mean;
                            const double den = pow(m2 - mean * m1, 1.5);
                            if (!isfinite(m1) || !isfinite(m2) || !isfinite(m3)) r = __longlong_as_double(0x7ff8000000000000ll);  // a group holding ±inf: NaN, as pandas
                            else if (num == 0.0 || fabs(den) < 1e-14 || isnan(den) || log2(fabs(den)) - log2(fabs(num)) < -20) r = 0.0;
                            else r = (n * pow(n - 1, 1.5) / (n - 2)) * num / den / (n - 1);
                        }
                        store_f_typed(op.out_data, op.out_ctype, p, r);
                        break;
                    }
                    case E_KURT: {  // pandas' nankurt (Fisher's excess kurtosis, bias-corrected) on the power sums of d = x - c
                        const unsigned long long cnt = ((const unsigned long long*)op.a1)[s];
                        const double n = (double)cnt, s1 = ((const double*)op.a0)[s], s2 = ((const double*)op.b0)[s];
                        const double s3 = ((const double*)op.c0)[s], s4 = ((const double*)op.d0)[s];
                        valid = cnt >= 4;
                        double r = __longlong_as_double(0x7ff8000000000000ll);
                        if (valid && isfinite(s1) && isfinite(s2) && isfinite(s3) && isfinite(s4)) {  // (a group holding ±inf: NaN)
                            const double mean = s1 / n;  // central moments, in which c cancels
                            const double m2 = s2 - s1 * mean;
                            const double m4 = s4 - 4.0 * s3 * mean + 6.0 * s2 * mean * mean - 3.0 * s1 * mean * mean * mean;
                            double num = n * (n + 1.0) * (n - 1.0) * m4, den = (n - 2.0) * (n - 3.0) * m2 * m2;
                            if (fabs(num) < 1e-14) num = 0.0;
                            if (fabs(den) < 1e-14) den = 0.0;
                            r = den == 0.0 ? 0.0 : num / den - 3.0 * (n - 1.0) * (n - 1.0) / ((n - 2.0) * (n - 3.0));
                        }
                        store_f_typed(op.out_data, op.out_ctype, p, r);
                        break;
                    }
                    case K_PROD_I64: case K_OR: case K_AND: case K_XOR: {  // (prod: every group valid, 1 when it saw no value)
                        if (op.a1) valid = ((const unsigned long long*)op.a1)[s] > 0;
                        store_int_typed(op.out_data, op.out_ctype, p, ((const long long*)op.a0)[s]);
                        break;
                    }
                    case K_PROD_F64:
                        store_f_typed(op.out_data, op.out_ctype, p, ((const double*)op.a0)[s]);
                        break;
                    case K_LOR: case K_LAND: case E_BOOLXOR: {
                        const unsigned long long w = ((const unsigned long long*)op.a0)[s];
                        if (op.a1) valid = ((const unsigned long long*)op.a1)[s] > 0;
                        store_int_typed(op.out_data, CT_BOOL, p, op.kind == E_BOOLXOR ? w == 1 : w != 0);
                        break;
                    }
                    case K_COUNT_IF:
                        store_int_typed(op.out_data, CT_INT64, p, ((const long long*)op.a0)[s]);
                        break;
                    case K_FIRST: case K_LAST: {  // NA when the group never saw a non-NA value (nullable / float outputs)
                        const unsigned long long q = ((const unsigned long long*)op.a1)[s];
                        const bool seen = op.kind == K_FIRST ? q != ~0ull : q != 0ull;
                        const unsigned long long bits = ((const unsigned long long*)op.a0)[s];
                        valid = seen;
                        if (op.out_ctype == CT_FLOAT32 || op.out_ctype == CT_FLOAT64)
                            store_f_typed(op.out_data, op.out_ctype, p, seen ? __longlong_as_double((long long)bits) : __longlong_as_double(0x7ff8000000000000ll));
                        else store_int_typed(op.out_data, op.out_ctype, p, seen ? (long long)bits : 0);
                        break;
                    }
                    case K_MIN_I64: case K_MAX_I64: {
                        if (op.a1) valid = ((const unsigned long long*)op.a1)[s] > 0;
                        store_int_typed(op.out_data, op.out_ctype, p, valid ? ((const long long*)op.a0)[s] : 0);
                        break;
                    }
                    case K_MIN_F64: case K_MAX_F64: {
                        unsigned long long e = ((const unsigned long long*)op.a0)[s];
                        bool seen = op.kind == K_MIN_F64 ? (e != ~0ull) : (e != 0ull);
                        if (op.a1) valid = seen;
                        store_f_typed(op.out_data, op.out_ctype, p, seen ? ordered_to_f64(e) : __longlong_as_double(0x7ff8000000000000ll));
                        break;
                    }
                }
            }
            if (op.out_valid) {
                unsigned m = __ballot_sync(0xffffffffu, valid);
                if ((threadIdx.x & 31) == 0) op.out_valid[p >> 5] = m;
            }
        }
    }
}

// ---- multi-column keys (2..4 integer / float key columns; SURVEY.md §8f "next" row 1, the reference's select-distinct /
// multi-key groupby: bodo/tests/test_streaming/test_groupby.py:111-177) -----------------------------------------
// A slot is claimed through a 64-bit tag word (hash of the key tuple, bit 63 set; 0 = empty, 1 = being written): the
// claiming thread CASes empty -> locked, writes the key columns + NA mask of the slot, fences and publishes the tag.
// Readers that find their own tag compare the full tuple (so the result is exact, the tag only prunes); readers that
// find `locked` re-read the slot.  Aggregate updates are the single-key kernel's apply_ops.
constexpr int MAX_KEYS = 4;
constexpr unsigned long long TAG_EMPTY = 0ull, TAG_LOCKED = 1ull;

struct MkArgs {
    int nk;
    const void* key_data[MAX_KEYS];
    const uint8_t* key_valid[MAX_KEYS];
    int key_ctype[MAX_KEYS];
    int dropna;
    int64_t n_rows;
    const uint32_t* index_list;
    unsigned long long* tags;
    long long* mk[MAX_KEYS];
    unsigned char* mkmask;  // bit j = key column j is valid (not NA) in this group's key
    uint64_t cap;
    long long* counters;
    long long group_limit;
    uint32_t* fail_list;
    int n_ops;
    OpDesc ops[MAX_OPS];
    unsigned long long seq_base;  // unused (first / last are single-key only); apply_ops reads it
};

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long mk_tag(const long long* keys, unsigned int mask, int nk) {
    unsigned long long h = 0x9E3779B97F4A7C15ULL ^ mask;
    for (int j = 0; j < nk; j++) h = xxh3_64_short((unsigned long long)keys[j] ^ (h * 0xD1B54A32D192ED03ULL), 8, SEED_HASH_PARTITION + j);
    return h | 0x8000000000000000ULL;
}
template <typename A>
__device__ __forceinline__ uint64_t find_or_insert_mk(const A& a, const long long* keys, unsigned int mask, unsigned long long tag) {
    const uint64_t m = a.cap - 1;
    uint64_t s = (tag >> 20) & m;
    for (uint64_t probes = 0; probes <= m;) {
        unsigned long long t = ld_acquire_u64(a.tags + s);
        if (t == tag) {
            bool eq = __ldcg(a.mkmask + s) == (unsigned char)mask;
            for (int j = 0; j < a.nk && eq; j++) eq = __ldcg(a.mk[j] + s) == keys[j];
            if (eq) return s;
        } else if (t == TAG_EMPTY) {
            if (a.group_limit >= 0) {
                long long tk = atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], 1ull);
                if (tk >= a.group_limit) { atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], (unsigned long long)-1ll); return ~0ull; }
            }
            unsigned long long old = atomicCAS(a.tags + s, TAG_EMPTY, TAG_LOCKED);
            if (old == TAG_EMPTY) {
                for (int j = 0; j < a.nk; j++) a.mk[j][s] = keys[j];
                a.mkmask[s] = (unsigned char)mask;
                __threadfence();
                atomicExch(a.tags + s, tag);  // publish
                return s;
            }
            if (a.group_limit >= 0) atomicAdd((unsigned long long*)&a.counters[CTR_GROUPS], (unsigned long long)-1ll);
            continue;  // somebody else took the slot: look at it again
        } else if (t == TAG_LOCKED) {
            continue;  // being written: re-read
        }
        s = (s + 1) & m;
        probes++;
    }
    return ~0ull;
}

template <bool RED>
__global__ void __launch_bounds__(256) groupby_consume_mk_kernel(const __grid_constant__ MkArgs a) {
    extern __shared__ __align__(8) unsigned char prod_smem[];  // a ProdCache when some op is a prod (prod_smem_bytes), else empty
    ProdCache& pc = *reinterpret_cast<ProdCache*>(prod_smem);
    const bool prod = RED && has_prod(a);
    prod_cache_clear(pc, prod);
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n_rows; i += stride) {
        int64_t row = a.index_list ? (int64_t)a.index_list[i] : i;
        long long keys[MAX_KEYS];
        unsigned int mask = 0;
        for (int j = 0; j < a.nk; j++) {
            bool v = bit_valid(a.key_valid[j], row);
            keys[j] = v ? (long long)load_int_as_i64(a.key_data[j], a.key_ctype[j], row) : 0;
            mask |= v ? (1u << j) : 0u;
        }
        if (a.dropna && mask != (1u << a.nk) - 1u) continue;  // any NA key column drops the row (pandas dropna=True)
        uint64_t slot = find_or_insert_mk(a, keys, mask, mk_tag(keys, mask, a.nk));
        if (slot == ~0ull) {
            unsigned long long f = atomicAdd((unsigned long long*)&a.counters[CTR_FAIL], 1ull);
            a.fail_list[f] = (uint32_t)row;
            continue;
        }
        apply_ops<RED>(a, slot, row, &pc);
    }
    prod_flush(pc, prod);
}

struct RehashMkArgs {
    int nk;
    const unsigned long long* old_tags; const long long* old_mk[MAX_KEYS]; const unsigned char* old_mask; uint64_t old_cap;
    unsigned long long* tags; long long* mk[MAX_KEYS]; unsigned char* mkmask; uint64_t cap;
    long long* counters; long long group_limit;  // group_limit < 0: no limit
    int n_acc;
    const unsigned long long* old_acc[2 * MAX_OPS];
    unsigned long long* new_acc[2 * MAX_OPS];
};
__global__ void rehash_mk_kernel(const __grid_constant__ RehashMkArgs a) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < a.old_cap; s += stride) {
        unsigned long long t = a.old_tags[s];
        if (!(t >> 63)) continue;
        long long keys[MAX_KEYS];
        for (int j = 0; j < a.nk; j++) keys[j] = a.old_mk[j][s];
        uint64_t ns = find_or_insert_mk(a, keys, a.old_mask[s], t);
        for (int j = 0; j < a.n_acc; j++) a.new_acc[j][ns] = a.old_acc[j][s];
    }
}
// Ownership of a multi-column key: hash_keys of the tuple exactly as the reference computes it on the original columns
// (sizeof(T) raw bytes per integer column, _Py_HashDouble per float column, NA -> hash_na_val, hash_combine_boost for the
// further columns), from the widened int64 values (float columns: canon_float_key) the table stores.
struct MkOwner {
    int nk, n_pes, rank;
    int own_nk;  // 0: ownership by the hash of all key columns (the reference's hash_keys); 1: by the FIRST key column alone, hashed
                 // like a single-key state's key (nunique's nested (key, value) state: a key's pairs live where the key lives)
    const long long* mk[MAX_KEYS];
    const unsigned char* mkmask;
    int key_ctype[MAX_KEYS];  // the input column types
    unsigned int drop_nan;    // compact_mk_kernel: bit j = drop groups whose float key column j is NaN (dropna)
};
__device__ __forceinline__ uint32_t mk_ref_hash(const long long* keys, unsigned int mask, int nk, const int* ctypes) {
    const uint32_t na_hash = (uint32_t)xxh3_64_short(1ull, 8, SEED_HASH_PARTITION);
    uint32_t h = 0;
    for (int j = 0; j < nk; j++) {
        const uint32_t hj = !((mask >> j) & 1u) ? na_hash
                           : ctype_is_float(ctypes[j]) ? owner_key_hash(keys[j], ctypes[j])
                           : ctype_size(ctypes[j]) == 8 ? (uint32_t)xxh3_64_short((uint64_t)keys[j], 8, SEED_HASH_PARTITION)
                                                        : (uint32_t)xxh3_64_short((uint64_t)(uint32_t)keys[j], 4, SEED_HASH_PARTITION);
        h = j == 0 ? hj : hash_combine_boost(h, hj);
    }
    return h;
}
__device__ __forceinline__ uint32_t mk_owner_hash(const MkOwner& ow, const long long* keys, unsigned int mask) {
    if (ow.own_nk == 1) return (mask & 1u) ? owner_key_hash(keys[0], ow.key_ctype[0]) : (uint32_t)xxh3_64_short(1ull, 8, SEED_HASH_PARTITION);
    return mk_ref_hash(keys, mask, ow.nk, ow.key_ctype);
}
// nunique: one thread per distinct (key, value) pair of the nested state; pairs whose value is NA do not count, nor (float
// value column: canon_float_key) do pairs whose value is NaN, the marker key
struct NuniqueArgs {
    const long long* pk; const long long* pv; const unsigned char* pmask; const uint64_t* slot_of_out; long long n_pairs;
    long long* tkeys; uint64_t cap; long long* counters; int dropna;
    int n_acc; unsigned long long* acc[MAX_OPS];
    int value_float;
};
__global__ void nunique_count_kernel(const __grid_constant__ NuniqueArgs a) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < a.n_pairs; p += (long long)gridDim.x * blockDim.x) {
        const uint64_t s = a.slot_of_out[p];
        const unsigned int m = a.pmask[s];
        if (!(m & 2u)) continue;  // NA value
        if (a.value_float && a.pv[s] == EMPTY_KEY) continue;  // NaN value
        uint64_t slot;
        if (!(m & 1u)) { if (a.dropna) continue; slot = a.cap; a.counters[CTR_NA] = 1; }
        else {
            const long long key = a.pk[s];
            if (key == EMPTY_KEY) { slot = a.cap + 1; a.counters[CTR_MARKER] = 1; }
            else { slot = find_only(a.tkeys, a.cap, key); if (slot == ~0ull) continue; }  // (every key of a pair is a group of the outer table)
        }
        for (int j = 0; j < a.n_acc; j++) atomicAdd(a.acc[j] + slot, 1ull);
    }
}
__global__ void compact_mk_kernel(const unsigned long long* __restrict__ tags, uint64_t cap, long long* cursor, uint64_t* slot_of_out,
                                  const __grid_constant__ MkOwner ow) {
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s0 = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s0 < ((cap + 31) & ~31ull); s0 += stride) {
        bool occ = s0 < cap && (tags[s0] >> 63);
        if (occ && ow.drop_nan) {  // dropna: a NaN in a float key column is NA (it is not in the mask: the table holds the marker)
            const unsigned int mask = ow.mkmask[s0];
            for (int j = 0; j < ow.nk; j++)
                if (((ow.drop_nan & mask) >> j) & 1u) occ = occ && ow.mk[j][s0] != EMPTY_KEY;
        }
        if (occ && ow.n_pes > 1) {  // only the groups this rank owns (see compact_slots_kernel)
            long long keys[MAX_KEYS];
            for (int j = 0; j < ow.nk; j++) keys[j] = ow.mk[j][s0];
            occ = hash_to_rank_u32(mk_owner_hash(ow, keys, ow.mkmask[s0]), ow.n_pes) == ow.rank;
        }
        unsigned m = __ballot_sync(0xffffffffu, occ);
        int lane = threadIdx.x & 31;
        long long base = 0;
        if (lane == 0 && m) base = (long long)atomicAdd((unsigned long long*)cursor, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (occ) slot_of_out[base + __popc(m & ((1u << lane) - 1))] = s0;
    }
}
// ---- multi-rank exchange of partial aggregates ----------------------------------------------------
// Wire format of one partial row (all fields 8 bytes): [key 0 .. key nk-1][NA mask][accumulators in wire order (wire_accs)];
// for a single-column key the NA mask is the flags word [bit0 = key valid].  Every group that another rank owns
// (hash_to_rank of the key, see compact_slots_kernel / mk_owner_hash) travels as one such row; the groups this rank owns stay in
// its table, and finalize's owned-only compaction drops the ones that were sent.
//
// One pack kernel and one combine kernel serve both transports:
//   * fused: every rank owns a receive slab that all peers can store into (symmetric memory over NVLink): XCHG_HDR_BYTES of
//     header (n_pes counts) followed by n_pes segments of cap_rows rows, segment s written by rank s.  xchg_pack_kernel stores
//     every row straight into its owner's slab (no send buffer, no count exchange, no host round trip); xchg_post_counts_kernel
//     tells every peer how many rows it got; after a device-side barrier across the ranks xchg_combine_kernel merges the rows of
//     the own slab.  A sender whose share for some destination exceeds cap_rows flags that in EVERY peer's header; then no rank
//     combines, finalize returns -2, and the host runs the NCCL form (the tables are intact).
//   * NCCL: the pack kernel counts (capacity 0) or packs into one send buffer at the exclusive prefix of those counts; the host
//     moves the rows with an all-to-all-v and the combine kernel reads them back to back, with the receive counts as its header.
constexpr unsigned long long XCHG_OVERFLOW = 1ull << 63;
constexpr int XCHG_HDR_BYTES = 256;

// The two table forms the exchange packs from and combines into; each reads a slot's key tuple and owner hash and finds or inserts
// the key of a wire row.  SlotTable: single-column key, slots [0, cap) plus the NA slot cap and the marker slot cap + 1 (the key
// equal to EMPTY_KEY).  TagTable: multi-column key (tag words, see find_or_insert_mk).
struct SlotTable {
    long long* tkeys;
    uint64_t cap;
    long long* counters;
    long long group_limit;
    int key_ctype;  // the key's input c-type (owner_key_hash)
    struct Key { long long k; bool valid; };
    __host__ __device__ uint64_t n_slots() const { return cap + 2; }
    __device__ int key_words() const { return 2; }
    __device__ bool load(uint64_t s, Key& key) const {
        key.valid = s != cap;
        key.k = s < cap ? tkeys[s] : (s == cap ? 0 : EMPTY_KEY);
        if (s < cap) return key.k != EMPTY_KEY;
        if (s == cap) return counters[CTR_NA] != 0;
        return s == cap + 1 && counters[CTR_MARKER] != 0;
    }
    __device__ uint32_t owner_hash(const Key& key) const {
        return key.valid ? owner_key_hash(key.k, key_ctype) : (uint32_t)xxh3_64_short(1ull, 8, SEED_HASH_PARTITION);  // hash_na_val
    }
    __device__ void store(const Key& key, unsigned long long* o) const { o[0] = (unsigned long long)key.k; o[1] = key.valid ? 1ull : 0ull; }
    __device__ uint64_t insert(const unsigned long long* r) const {
        const long long key = (long long)r[0];
        if (!(r[1] & 1)) { counters[CTR_NA] = 1; return cap; }
        if (key == EMPTY_KEY) { counters[CTR_MARKER] = 1; return cap + 1; }
        return find_or_insert(tkeys, cap, key, counters, group_limit);
    }
    __device__ uint64_t find(const unsigned long long* r) const {
        const long long key = (long long)r[0];
        if (!(r[1] & 1)) return cap;
        if (key == EMPTY_KEY) return cap + 1;
        return find_only(tkeys, cap, key);
    }
};
struct TagTable {
    int nk;
    unsigned long long* tags;
    long long* mk[MAX_KEYS];
    unsigned char* mkmask;
    uint64_t cap;
    long long* counters;
    long long group_limit;
    MkOwner ow;
    struct Key { long long k[MAX_KEYS]; unsigned int mask; };
    __host__ __device__ uint64_t n_slots() const { return cap; }
    __device__ int key_words() const { return nk + 1; }
    __device__ bool load(uint64_t s, Key& key) const {
        if (s >= cap || !(tags[s] >> 63)) return false;
        for (int j = 0; j < nk; j++) key.k[j] = mk[j][s];
        key.mask = mkmask[s];
        return true;
    }
    __device__ uint32_t owner_hash(const Key& key) const { return mk_owner_hash(ow, key.k, key.mask); }
    __device__ void store(const Key& key, unsigned long long* o) const {
        for (int j = 0; j < nk; j++) o[j] = (unsigned long long)key.k[j];
        o[nk] = key.mask;
    }
    __device__ uint64_t insert(const unsigned long long* r) const {
        long long keys[MAX_KEYS];
        for (int j = 0; j < nk; j++) keys[j] = (long long)r[j];
        const unsigned int mask = (unsigned int)r[nk];
        return find_or_insert_mk(*this, keys, mask, mk_tag(keys, mask, nk));
    }
};

struct XchgPackArgs {
    int n_pes, rank;
    int n_acc;
    const unsigned long long* acc[2 * MAX_OPS];
    int row_words;
    unsigned long long* cursors;  // [n_pes] rows per destination (device); the exact counts once the kernel ends, stored or not
    void* const* dest;            // [n_pes] device array: the region of destination d starts dest_offset bytes past dest[d] ...
    long long dest_offset;
    long long cap_rows;           // ... and holds cap_rows rows (0: count only)
};
template <typename T>
__global__ void xchg_pack_kernel(const __grid_constant__ T t, const __grid_constant__ XchgPackArgs a) {
    const int lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; s < ((t.n_slots() + 31) & ~31ull); s += stride) {
        typename T::Key key;
        int d = t.load(s, key) ? hash_to_rank_u32(t.owner_hash(key), a.n_pes) : -1;
        if (d == a.rank) d = -1;  // owned here: stays in the table
        // warp-aggregated cursor: one atomic per (warp, destination)
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        const int rank_in_peers = __popc(peers & ((1u << lane) - 1));
        unsigned long long base = 0;
        if (d >= 0 && lane == leader) base = atomicAdd(&a.cursors[d], (unsigned long long)__popc(peers));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (d >= 0) {
            const unsigned long long pos = base + rank_in_peers;
            if (pos < (unsigned long long)a.cap_rows) {
                unsigned long long* o = (unsigned long long*)((char*)a.dest[d] + a.dest_offset) + pos * a.row_words;
                t.store(key, o);
                const int kw = t.key_words();
                for (int j = 0; j < a.n_acc; j++) o[kw + j] = a.acc[j][s];
            }
        }
    }
}
// fused form: posts the per-source counts of this rank into every peer's slab header
__global__ void xchg_post_counts_kernel(const unsigned long long* cursors, void* const* peer_slabs, int n_pes, int rank, long long cap_rows) {
    const int d = threadIdx.x;
    const unsigned long long c = d < n_pes ? cursors[d] : 0ull;
    const bool any_over = __any_sync(0xffffffffu, c > (unsigned long long)cap_rows);
    if (d < n_pes) ((unsigned long long*)peer_slabs[d])[rank] = (c > (unsigned long long)cap_rows ? (unsigned long long)cap_rows : c) | (any_over ? XCHG_OVERFLOW : 0ull);
}

// The rows a combine reads: n_seg segments, segment s holding hdr[s] rows (| XCHG_OVERFLOW).  A row's flat index (what the fail
// list records) counts from row 0 of segment 0.
struct XchgSource {
    const unsigned long long* rows;  // row 0 of segment 0
    const unsigned long long* hdr;   // [n_seg] counts, device memory
    int n_seg;
    long long seg_rows;              // segment s starts at row s * seg_rows; 0: the segments lie back to back
    const uint32_t* index_list;      // replay: the n_index listed flat row indices instead of the segments
    int64_t n_index;
};
struct CombineArgs {
    XchgSource src;
    int row_words;
    uint32_t* fail_list;
    int n_ops;
    int kinds[MAX_OPS];
    void* a0[MAX_OPS];
    void* a1[MAX_OPS];
};
// calls f(flat row index) for this thread's rows of the source; false (and no call) when a sender flagged an overflow
template <typename F>
__device__ __forceinline__ bool for_each_source_row(const XchgSource& src, F&& f) {
    const int64_t i0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    if (!src.index_list)
        for (int s = 0; s < src.n_seg; s++) if (src.hdr[s] & XCHG_OVERFLOW) return false;
    // (one loop for both cases: the row code is inlined once)
    int64_t first = 0;
    for (int s = 0; s < (src.index_list ? 1 : src.n_seg); s++) {
        const int64_t n = src.index_list ? src.n_index : (int64_t)(src.hdr[s] & ~XCHG_OVERFLOW);
        for (int64_t i = i0; i < n; i += stride) f(src.index_list ? (int64_t)src.index_list[i] : first + i);
        first += src.seg_rows ? src.seg_rows : n;
    }
    return true;
}
// combine step (get_combine_func, groupby/_groupby_update.cpp:41-57): count/size/mean -> sum, min -> min, max -> max
// merges the accumulator words r[0 ...] of one partial row into `slot`
// A moment group (K_SHIFT ...) re-centres the partial's sums about its own shift c_s on the slot's shift c_t: with delta = c_s - c_t,
// sum (d + delta)^k expands to S1 + n delta, S2 + 2 delta S1 + n delta^2, S3 + 3 delta S2 + 3 delta^2 S1 + n delta^3,
// S4 + 4 delta S3 + 6 delta^2 S2 + 4 delta^3 S1 + n delta^4.  A slot without a
// shift takes c_s (delta = 0); a partial without one (every row of the group was NA on that rank) adds nothing.
__device__ __forceinline__ void combine_apply(const CombineArgs& a, uint64_t slot, const unsigned long long* r) {
    {
        int w = 0;
        bool mom = false;
        double delta = 0.0, n_s = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;  // K_SHIFT -> K_MOM*: the partial's moments seen so far
        for (int j = 0; j < a.n_ops; j++) {
            unsigned long long v0 = r[w++];
            unsigned long long v1 = a.a1[j] ? r[w++] : 0;
            const double f0 = __longlong_as_double((long long)v0);
            switch (a.kinds[j]) {
                case K_SUM_I64: case K_COUNT: case K_SIZE: case K_NUNIQUE: atomicAdd((unsigned long long*)a.a0[j] + slot, v0); break;
                case K_SUM_F64: atomicAdd((double*)a.a0[j] + slot, f0); break;
                case K_SHIFT:
                    mom = v0 != SHIFT_UNSET;
                    if (mom) delta = f0 - group_shift((double*)a.a0[j] + slot, f0);
                    break;
                case K_MOM1:
                    if (!mom) break;
                    n_s = (double)v1; s1 = f0;
                    atomicAdd((double*)a.a0[j] + slot, s1 + n_s * delta);
                    atomicAdd((unsigned long long*)a.a1[j] + slot, v1);
                    break;
                case K_MOM2:
                    if (!mom) break;
                    s2 = f0;
                    atomicAdd((double*)a.a0[j] + slot, s2 + 2.0 * delta * s1 + n_s * delta * delta);
                    break;
                case K_MOM3:
                    if (!mom) break;
                    s3 = f0;
                    atomicAdd((double*)a.a0[j] + slot, s3 + 3.0 * delta * s2 + 3.0 * delta * delta * s1 + n_s * delta * delta * delta);
                    break;
                case K_MOM4:
                    if (mom) {
                        const double d2 = delta * delta;
                        atomicAdd((double*)a.a0[j] + slot, f0 + 4.0 * delta * s3 + 6.0 * d2 * s2 + 4.0 * d2 * delta * s1 + n_s * d2 * d2);
                    }
                    break;
                case K_PROD_I64: prod_update<false>((unsigned long long*)a.a0[j] + slot, v0, nullptr); break;
                case K_PROD_F64: prod_update<true>((unsigned long long*)a.a0[j] + slot, v0, nullptr); break;
                // word ops: the partial's word is itself an operand (0 / all-ones for the truth ops); true-counts add
                case K_OR: case K_AND: case K_XOR: case K_LOR: case K_LAND: word_update(a.kinds[j], (unsigned long long*)a.a0[j] + slot, v0); break;
                case K_COUNT_IF: atomicAdd((unsigned long long*)a.a0[j] + slot, v0); break;
                case K_MEAN:
                    atomicAdd((double*)a.a0[j] + slot, __longlong_as_double((long long)v0));
                    atomicAdd((unsigned long long*)a.a1[j] + slot, v1);
                    break;
                case K_MIN_I64: atomicMin((long long*)a.a0[j] + slot, (long long)v0); break;
                case K_MAX_I64: atomicMax((long long*)a.a0[j] + slot, (long long)v0); break;
                case K_MIN_F64: atomicMin((unsigned long long*)a.a0[j] + slot, v0); break;
                case K_MAX_F64: atomicMax((unsigned long long*)a.a0[j] + slot, v0); break;
                // first / last: the partial with the smallest / largest sequence number wins (sequence numbers carry the rank in
                // their high bits: rank order, then row order, as the reference's rank-ordered combine); its value is written by
                // combine_firstlast_fix_kernel once every partial of the batch has been applied
                case K_FIRST: if (v1 != ~0ull) atomicMin((unsigned long long*)a.a1[j] + slot, v1); break;
                case K_LAST: if (v1 != 0ull) atomicMax((unsigned long long*)a.a1[j] + slot, v1); break;
            }
            if (a.a1[j] && a.kinds[j] != K_MEAN && a.kinds[j] != K_MOM1 && a.kinds[j] != K_FIRST && a.kinds[j] != K_LAST) atomicAdd((unsigned long long*)a.a1[j] + slot, v1);
        }
    }
}
// merges the source's rows into the table; a row whose group finds the table at its limit goes to the fail list (flat index)
template <typename T>
__global__ void xchg_combine_kernel(const __grid_constant__ T t, const __grid_constant__ CombineArgs c) {
    const bool combined = for_each_source_row(c.src, [&](int64_t row) {
        const unsigned long long* r = c.src.rows + row * c.row_words;
        const uint64_t slot = t.insert(r);
        if (slot == ~0ull) {
            unsigned long long f = atomicAdd((unsigned long long*)&t.counters[CTR_FAIL], 1ull);
            c.fail_list[f] = (uint32_t)row;
            return;
        }
        combine_apply(c, slot, r + t.key_words());
    });
    // every rank sees the same flags: nobody combines
    if (!combined && blockIdx.x == 0 && threadIdx.x == 0) t.counters[CTR_XCHG_OVERFLOW] = 1;
}
// first / last (single-column keys), phase 2 of the combine step: the partial whose sequence number won writes its value
__global__ void combine_firstlast_fix_kernel(const __grid_constant__ SlotTable t, const __grid_constant__ CombineArgs c) {
    for_each_source_row(c.src, [&](int64_t row) {
        const unsigned long long* r = c.src.rows + row * c.row_words;
        const uint64_t slot = t.find(r);
        if (slot == ~0ull) return;
        int w = t.key_words();
        for (int j = 0; j < c.n_ops; j++) {
            const unsigned long long v0 = r[w++];
            const unsigned long long v1 = c.a1[j] ? r[w++] : 0;
            if ((c.kinds[j] == K_FIRST && v1 != ~0ull) || (c.kinds[j] == K_LAST && v1 != 0ull))
                if (((const unsigned long long*)c.a1[j])[slot] == v1) ((unsigned long long*)c.a0[j])[slot] = v0;
        }
    });
}

struct EvalMkKeysArgs {
    int nk;
    const long long* mk[MAX_KEYS];
    const unsigned char* mkmask;
    const uint64_t* slot_of_out;
    const long long* n_out_ptr;
    int key_ctype[MAX_KEYS];
    void* out_keys[MAX_KEYS];
    uint32_t* out_key_valid[MAX_KEYS];  // nullptr for non-nullable key columns
};
__global__ void eval_mk_keys_kernel(const __grid_constant__ EvalMkKeysArgs a) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_out = *a.n_out_ptr;
    int64_t n_round = (n_out + 31) & ~31ll;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_round; p += stride) {
        bool in = p < n_out;
        uint64_t s = in ? a.slot_of_out[p] : 0;
        unsigned int mask = in ? a.mkmask[s] : 0;
        for (int j = 0; j < a.nk; j++) {
            if (in) {
                if (ctype_is_float(a.key_ctype[j])) store_f_typed(a.out_keys[j], a.key_ctype[j], p, canon_float_decode(a.mk[j][s]));
                else store_int_typed(a.out_keys[j], a.key_ctype[j], p, a.mk[j][s]);
            }
            if (a.out_key_valid[j]) {
                unsigned m = __ballot_sync(0xffffffffu, in && ((mask >> j) & 1));
                if ((threadIdx.x & 31) == 0) a.out_key_valid[j][p >> 5] = m;
            }
        }
    }
}

// ---- min_row_number_filter (MRNF): QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) = 1 ----
// Every group keeps the first row of the stable order by (sort columns, arrival).  A row's rank is the tuple (class_0, word_0,
// ..., class_{n-1}, word_{n-1}, seq) of the sort's key encoding (sort_word / sort_class) and its arrival number seq = rows
// consumed before it + 1.  The tuple is one bit string (fields in that order, each at its own width, seq in MRNF_SEQ_BITS bits)
// cut into big-endian digits of 63 bits; a digit's top bit is always 0, so no digit of a row is all-ones, the value a free
// scratch digit holds.  Comparing digit strings lexicographically is comparing the tuples, and seq makes every row's distinct.
// Per slot the table carries the winner record W (n_digits digits, a validity word with bit j = kept column j valid, one 8-byte
// word per kept column: K_MRNF accumulators, moved by the rehash as any other) and the batch scratch B (n_digits words, all-ones
// between batches).  Per batch, once every row is in the table: digit pass d = 0 .. n_digits-1 (mrnf_min_kernel) takes the
// minimum of digit d over the rows whose digits 0..d-1 equal B's, so B ends as the batch's least tuple per slot; then
// mrnf_merge_kernel lets the one row equal to B compare itself against W, replace it when smaller and reset B.
constexpr int MRNF_MAX_DIGITS = 5;           // 4 keys x (1 + 64) bits + MRNF_SEQ_BITS <= 5 x 63
constexpr int MRNF_SEQ_BITS = 48;
constexpr int MRNF_FIELDS = 2 * MAX_KEYS + 1;  // class and word per sort key, then seq
constexpr int MRNF_MAX_KEEP = 2 * MAX_OPS - MRNF_MAX_DIGITS - 1;  // what the rehash carries besides the digits and validity word
constexpr unsigned long long MRNF_DIGIT_MASK = 0x7FFFFFFFFFFFFFFFull;

struct MrnfArgs {
    int64_t n_rows;
    unsigned long long seq_base;  // rows consumed before this batch
    // the table (single-column: tkeys; multi-column: tags / mk / mkmask) and the batch's key columns (float keys canonical)
    int nk, dropna;
    const void* key_data[MAX_KEYS];
    const uint8_t* key_valid[MAX_KEYS];
    int key_ctype[MAX_KEYS];
    const long long* tkeys;
    const unsigned long long* tags;
    const long long* mk[MAX_KEYS];
    const unsigned char* mkmask;
    uint64_t cap;
    uint64_t* slot;  // per batch row: its slot (pass 0 writes it, later passes read it), ~0 = dropped (NA key, dropna)
    // the order
    int n_sort, n_digits;
    SortKey key[MAX_KEYS];
    const void* sort_data[MAX_KEYS];
    const uint8_t* sort_valid[MAX_KEYS];
    int f_end[MRNF_FIELDS];  // bit position just past each field in the tuple's bit string (fields of absent keys are 0)
    unsigned long long* b;   // B: digit d of slot s at b[d * (cap + 2) + s]
    unsigned long long* w[MRNF_MAX_DIGITS];
    unsigned long long* w_valid;
    // the kept columns as the batch holds them (a kept key column is read here, not from its canonical column)
    int n_keep;
    const void* keep_data[MRNF_MAX_KEEP];
    const uint8_t* keep_valid[MRNF_MAX_KEEP];
    int keep_size[MRNF_MAX_KEEP];
    unsigned long long* keep_w[MRNF_MAX_KEEP];
};

// lookup only in the multi-column table (the key tuple of batch row `row`, NK columns); ~0 when the row was dropped (dropna) or
// its tuple is not in the table.  NK is a template argument so that the tuple stays in registers.
template <int NK>
__device__ __forceinline__ uint64_t find_only_mk(const MrnfArgs& a, int64_t row) {
    long long keys[NK];
    unsigned int mask = 0;
#pragma unroll
    for (int j = 0; j < NK; j++) {
        const bool v = bit_valid(a.key_valid[j], row);
        keys[j] = v ? (long long)load_int_as_i64(a.key_data[j], a.key_ctype[j], row) : 0;
        mask |= v ? (1u << j) : 0u;
    }
    if (a.dropna && mask != (1u << NK) - 1u) return ~0ull;
    const unsigned long long tag = mk_tag(keys, mask, NK);
    const uint64_t m = a.cap - 1;
    uint64_t s = (tag >> 20) & m;
    for (uint64_t probes = 0; probes <= m; probes++) {
        const unsigned long long t = __ldcg(a.tags + s);
        if (t == tag) {
            bool eq = __ldcg(a.mkmask + s) == (unsigned char)mask;
#pragma unroll
            for (int j = 0; j < NK; j++) eq = eq && __ldcg(a.mk[j] + s) == keys[j];
            if (eq) return s;
        } else if (t == TAG_EMPTY) {
            return ~0ull;
        }
        s = (s + 1) & m;
    }
    return ~0ull;
}
// the slot of batch row `row` (every row is in the table), as the consume kernels placed it; ~0 for a row they dropped
__device__ __forceinline__ uint64_t mrnf_find_slot(const MrnfArgs& a, int64_t row) {
    switch (a.nk) {
        case 1: {
            if (!bit_valid(a.key_valid[0], row)) return a.dropna ? ~0ull : a.cap;
            const long long key = load_int_as_i64(a.key_data[0], a.key_ctype[0], row);
            return key == EMPTY_KEY ? a.cap + 1 : find_only(a.tkeys, a.cap, key);
        }
        case 2: return find_only_mk<2>(a, row);
        case 3: return find_only_mk<3>(a, row);
        default: return find_only_mk<4>(a, row);
    }
}
// the tuple's fields of batch row `row`
__device__ __forceinline__ void mrnf_fields(const MrnfArgs& a, int64_t row, unsigned long long* v) {
#pragma unroll
    for (int j = 0; j < MAX_KEYS; j++) {
        v[2 * j] = v[2 * j + 1] = 0;
        if (j < a.n_sort) {
            bool na = !bit_valid(a.sort_valid[j], row);
            v[2 * j + 1] = sort_word(a.key[j], load_bits(a.sort_data[j], a.key[j].size, row), na);
            v[2 * j] = sort_class(a.key[j], na);
        }
    }
    v[2 * MAX_KEYS] = a.seq_base + (unsigned long long)row + 1ull;
}
// digit d: bits [63 d, 63 d + 63) of the bit string; bit i of field f lands at bit i + 63 d + 63 - f_end[f] of the digit
__device__ __forceinline__ unsigned long long mrnf_digit(const MrnfArgs& a, const unsigned long long* v, int d) {
    unsigned long long r = 0;
#pragma unroll
    for (int f = 0; f < MRNF_FIELDS; f++) {
        const int sh = 63 * d + 63 - a.f_end[f];
        if (sh >= 0 && sh < 64) r |= v[f] << sh;
        else if (sh < 0 && sh > -64) r |= v[f] >> -sh;
    }
    return r & MRNF_DIGIT_MASK;
}

// digit pass d: B[d] = min of digit d over the slot's rows whose digits 0..d-1 equal B[0..d-1]
__global__ void __launch_bounds__(256) mrnf_min_kernel(const __grid_constant__ MrnfArgs a, int d) {
    const uint64_t stride_b = a.cap + 2;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < a.n_rows; row += (int64_t)gridDim.x * blockDim.x) {
        uint64_t slot;
        if (d == 0) { slot = mrnf_find_slot(a, row); a.slot[row] = slot; }
        else slot = a.slot[row];
        if (slot == ~0ull) continue;
        unsigned long long v[MRNF_FIELDS];
        mrnf_fields(a, row, v);
        bool in = true;
        for (int e = 0; e < d && in; e++) in = mrnf_digit(a, v, e) == a.b[e * stride_b + slot];
        if (!in) continue;
        unsigned long long* bp = a.b + d * stride_b + slot;
        const unsigned long long x = mrnf_digit(a, v, d);
        if (x < __ldcg(bp)) atomicMin(bp, x);  // (read first: with few groups most rows lose without an atomic)
    }
}
// The row equal to B (one per touched slot: seq differs between rows) replaces W when its tuple is smaller, then resets B.
// Another row of the slot may read B while it is being reset; it sees each digit either as the winner's or as all-ones, which
// no digit of a row equals, so it cannot match.
__global__ void __launch_bounds__(256) mrnf_merge_kernel(const __grid_constant__ MrnfArgs a) {
    const uint64_t stride_b = a.cap + 2;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < a.n_rows; row += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t slot = a.slot[row];
        if (slot == ~0ull) continue;
        unsigned long long v[MRNF_FIELDS];
        mrnf_fields(a, row, v);
        bool win = true;
        for (int e = 0; e < a.n_digits && win; e++) win = mrnf_digit(a, v, e) == __ldcg(a.b + e * stride_b + slot);
        if (!win) continue;
        bool smaller = false;
        for (int e = 0; e < a.n_digits; e++) {
            const unsigned long long x = mrnf_digit(a, v, e), y = a.w[e][slot];
            if (x != y) { smaller = x < y; break; }
        }
        if (smaller) {
            for (int e = 0; e < a.n_digits; e++) a.w[e][slot] = mrnf_digit(a, v, e);
            unsigned long long vw = 0;
            for (int j = 0; j < a.n_keep; j++) {
                a.keep_w[j][slot] = load_bits(a.keep_data[j], a.keep_size[j], row);
                vw |= bit_valid(a.keep_valid[j], row) ? 1ull << j : 0ull;
            }
            a.w_valid[slot] = vw;
        }
        for (int e = 0; e < a.n_digits; e++) a.b[e * stride_b + slot] = ~0ull;
    }
}

struct MrnfOutArgs {
    const uint64_t* slot_of_out;
    const long long* n_out_ptr;
    const unsigned long long* w_valid;
    int n_keep;
    const unsigned long long* keep_w[MRNF_MAX_KEEP];
    int keep_size[MRNF_MAX_KEEP];
    void* out[MRNF_MAX_KEEP];
    uint32_t* out_valid[MRNF_MAX_KEEP];  // validity bitmap as 32-bit words (nullable kept columns), else nullptr
};
// finalize: the winner's cells of every kept column, at the column's width, for the compacted slots
__global__ void mrnf_gather_kernel(const __grid_constant__ MrnfOutArgs a) {
    const int64_t n_out = *a.n_out_ptr;
    const int64_t n_round = (n_out + 31) & ~31ll;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_round; p += (int64_t)gridDim.x * blockDim.x) {
        const bool in = p < n_out;
        const uint64_t s = in ? a.slot_of_out[p] : 0;
        const unsigned long long vw = in ? a.w_valid[s] : 0ull;
        for (int j = 0; j < a.n_keep; j++) {
            if (in) copy_cell(a.out[j], p, a.keep_w[j] + s, 0, a.keep_size[j]);
            if (a.out_valid[j]) {
                const unsigned m = __ballot_sync(0xffffffffu, (vw >> j) & 1ull);
                if ((threadIdx.x & 31) == 0) a.out_valid[j][p >> 5] = m;
            }
        }
    }
}

// ---- min_row_number_filter with a limit n > 1: QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) <= n ----
// Each group keeps its n least rank tuples (the digit strings above).  The table carries one word per slot, the group's dense id
// (a K_MRNF accumulator, all-ones until the group's first candidate claims one), so ids survive growth while slots move.  Per id
// the cutoff C holds the digits of the group's n-th survivor as of the last reduce (all-ones while it had fewer than n).  Per
// batch, once every row is in the table, mrnf_top_filter_kernel appends each row whose digits are below its group's cutoff to the
// candidate store.  A reduce (host-triggered) sorts the store by (id, digits), keeps the first n rows of every id and lowers C.
// Store row layout, one 8-byte column each: id, digits 0 .. n_digits-1, validity word (bit j = kept column j), kept cells.
struct MrnfTopArgs {
    MrnfArgs m;                        // the table, the order and the kept columns (b, w, w_valid, keep_w and slot are unused)
    unsigned long long* gid;           // per slot: the group's id, ~0 = none yet
    unsigned long long* ctr;           // [0] store rows (the append cursor), [1] ids handed out
    const unsigned long long* cutoff;  // digit e of id g at cutoff[g * n_digits + e], for g < n_cut
    unsigned long long n_cut;
    unsigned drop_nan;                 // dropna: key columns (float) whose NaN marker group is dropped, as compact_* drop it
    unsigned long long* store;         // column c of store row r at store[c * store_cap + r]
    unsigned long long store_cap;
};
__global__ void __launch_bounds__(256) mrnf_top_filter_kernel(const __grid_constant__ MrnfTopArgs a) {
    const MrnfArgs& m = a.m;
    const int64_t n_round = (m.n_rows + 31) & ~31ll;
    const int lane = threadIdx.x & 31;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < n_round; row += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t slot = row < m.n_rows ? mrnf_find_slot(m, row) : ~0ull;
        bool in = slot != ~0ull;
        for (int j = 0; j < m.nk && in; j++)
            if (((a.drop_nan >> j) & 1u) && bit_valid(m.key_valid[j], row)) in = load_int_as_i64(m.key_data[j], m.key_ctype[j], row) != EMPTY_KEY;
        unsigned long long v[MRNF_FIELDS];
        unsigned long long id = ~0ull;
        if (in) {
            mrnf_fields(m, row, v);
            id = __ldcg(a.gid + slot);
            if (id < a.n_cut) {  // below the cutoff (a row never equals it: seq differs)
                const unsigned long long* c = a.cutoff + id * m.n_digits;
                for (int e = 0; e < m.n_digits; e++) {
                    const unsigned long long x = mrnf_digit(m, v, e), y = c[e];
                    if (x != y) { in = x < y; break; }
                }
            }
            if (in && id == ~0ull) {  // the group's first candidate: claim an id; a thread that loses the race takes the winner's
                const unsigned long long mine = atomicAdd(a.ctr + 1, 1ull);
                const unsigned long long old = atomicCAS(a.gid + slot, ~0ull, mine);
                id = old == ~0ull ? mine : old;
            }
        }
        const unsigned ball = __ballot_sync(0xffffffffu, in);
        unsigned long long base = 0;
        if (lane == 0 && ball) base = atomicAdd(a.ctr, (unsigned long long)__popc(ball));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (!in) continue;
        unsigned long long* p = a.store + base + __popc(ball & ((1u << lane) - 1));
        p[0] = id;
        for (int e = 0; e < m.n_digits; e++) p[(e + 1) * a.store_cap] = mrnf_digit(m, v, e);
        unsigned long long vw = 0;
        for (int j = 0; j < m.n_keep; j++) {
            p[(m.n_digits + 2 + j) * a.store_cap] = load_bits(m.keep_data[j], m.keep_size[j], row);
            vw |= bit_valid(m.keep_valid[j], row) ? 1ull << j : 0ull;
        }
        p[(m.n_digits + 1) * a.store_cap] = vw;
    }
}

// reduce, on the store sorted by (id, digits) through perm (nullptr: the identity): head[id] = position of the id's first row
__global__ void mrnf_top_head_kernel(const unsigned long long* gid, const uint32_t* perm, int64_t n, uint32_t* head) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long g = gid[perm ? perm[i] & 0x7FFFFFFFu : i];
        if (i == 0 || gid[perm ? perm[i - 1] & 0x7FFFFFFFu : i - 1] != g) head[g] = (uint32_t)i;
    }
}
// keep[i] = the row at sorted position i ranks below `limit` in its id; the row of rank limit - 1 writes its digits as the cutoff
__global__ void mrnf_top_rank_kernel(const unsigned long long* store, uint64_t store_cap, int n_digits, const uint32_t* perm,
                                     int64_t n, const uint32_t* head, long long limit, uint32_t* keep, unsigned long long* cutoff) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = perm ? perm[i] & 0x7FFFFFFFu : i;
        const unsigned long long g = store[r];
        const long long rank = i - (int64_t)head[g];
        keep[i] = rank < limit;
        if (rank == limit - 1)
            for (int e = 0; e < n_digits; e++) cutoff[g * n_digits + e] = store[(e + 1) * store_cap + r];
    }
}
// store row perm[i] (every column) to dst row pos[i], for the rows with keep[i] (all rows when keep is nullptr)
__global__ void mrnf_top_move_kernel(const unsigned long long* src, unsigned long long* dst, uint64_t store_cap, int n_words,
                                     const uint32_t* perm, int64_t n, const uint32_t* keep, const unsigned long long* pos) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (keep && !keep[i]) continue;
        const int64_t r = perm ? perm[i] & 0x7FFFFFFFu : i, d = pos ? (int64_t)pos[i] : i;
        for (int c = 0; c < n_words; c++) dst[c * store_cap + d] = src[c * store_cap + r];
    }
}
// finalize: store rows [0, n_out) (the survivors in (id, rank) order) to the kept columns at their widths
__global__ void mrnf_top_gather_kernel(const unsigned long long* store, uint64_t store_cap, int n_digits, int64_t n_out,
                                       const __grid_constant__ MrnfOutArgs a) {
    const int64_t n_round = (n_out + 31) & ~31ll;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_round; p += (int64_t)gridDim.x * blockDim.x) {
        const bool in = p < n_out;
        const unsigned long long vw = in ? store[(n_digits + 1) * store_cap + p] : 0ull;
        for (int j = 0; j < a.n_keep; j++) {
            if (in) copy_cell(a.out[j], p, store + (n_digits + 2 + j) * store_cap + p, 0, a.keep_size[j]);
            if (a.out_valid[j]) {
                const unsigned m = __ballot_sync(0xffffffffu, (vw >> j) & 1ull);
                if ((threadIdx.x & 31) == 0) a.out_valid[j][p >> 5] = m;
            }
        }
    }
}

// ---- holistic aggregates: mode, percentile_cont, percentile_disc ----
// They need the whole multiset of a group's non-NA values, so the state keeps it.  The table carries one K_HID word per slot, the
// group's id (all-ones until the group's first row claims one; ids survive growth while slots move), and each distinct value
// column has a store of (id, value) rows: a 4-byte id column and a column of the value's own width.  Per batch, once every row
// is in the table, holistic_append_kernel appends each row's non-NA (and non-NaN) values.  Finalize sorts each store by (id,
// sort_word(value)) with radix_sort_columns, marks each id's first and last sorted position (holistic_bounds_kernel) and writes
// every result into its slot's result word (holistic_eval_kernel, one thread per slot): a percentile reads one or two sorted
// positions; mode takes, per id, the longest run of equal values, found from the runs' starts (a flag, the tile scan,
// holistic_run_start_kernel, holistic_run_best_kernel).  No thread walks a group's rows, so one group holding most rows costs
// what a uniform input costs.
struct HoAppendArgs {
    MrnfArgs m;                // the table and the batch's key columns (n_rows, nk, dropna, key_*, tkeys / tags / mk / mkmask, cap)
    unsigned drop_nan;         // dropna: key columns (float) whose NaN marker group is dropped, as compact_* drop it
    unsigned long long* gid;   // per slot: the group's id, ~0 = none yet
    unsigned long long* ctr;   // [0] ids handed out, [1 + i] rows of store i (its append cursor)
    int n_st;
    const void* val[MAX_OPS];  // the batch's value column of store i
    const uint8_t* valid[MAX_OPS];
    int ct[MAX_OPS];
    uint32_t* st_id[MAX_OPS];
    void* st_val[MAX_OPS];
};
__global__ void __launch_bounds__(256) holistic_append_kernel(const __grid_constant__ HoAppendArgs a) {
    const MrnfArgs& m = a.m;
    const int64_t n_round = (m.n_rows + 31) & ~31ll;
    const int lane = threadIdx.x & 31;
    for (int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; row < n_round; row += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t slot = row < m.n_rows ? mrnf_find_slot(m, row) : ~0ull;
        bool in = slot != ~0ull;
        for (int j = 0; j < m.nk && in; j++)
            if (((a.drop_nan >> j) & 1u) && bit_valid(m.key_valid[j], row)) in = load_int_as_i64(m.key_data[j], m.key_ctype[j], row) != EMPTY_KEY;
        unsigned long long id = in ? __ldcg(a.gid + slot) : 0ull;
        // a group without an id: of the warp's lanes that stand on its slot the lowest claims one (a thread that loses the race to
        // another warp takes the winner's), the others take it from that lane
        const bool claim = in && id == ~0ull;
        const unsigned peers = __match_any_sync(0xffffffffu, claim ? slot : ~0ull);
        const int leader = __ffs(peers) - 1;
        if (claim && lane == leader) {
            const unsigned long long mine = atomicAdd(a.ctr, 1ull);
            const unsigned long long old = atomicCAS(a.gid + slot, ~0ull, mine);
            id = old == ~0ull ? mine : old;
        }
        const unsigned long long lead_id = __shfl_sync(0xffffffffu, id, leader);
        if (claim) id = lead_id;
        for (int i = 0; i < a.n_st; i++) {
            bool v = in && bit_valid(a.valid[i], row);
            if (v && ctype_is_float(a.ct[i])) v = !isnan(load_as_f64(a.val[i], a.ct[i], row));
            const unsigned ball = __ballot_sync(0xffffffffu, v);
            unsigned long long base = 0;
            if (lane == 0 && ball) base = atomicAdd(a.ctr + 1 + i, (unsigned long long)__popc(ball));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (!v) continue;
            const unsigned long long r = base + __popc(ball & ((1u << lane) - 1));
            a.st_id[i][r] = (uint32_t)id;
            copy_cell(a.st_val[i], (int64_t)r, a.val[i], row, ctype_size(a.ct[i]));
        }
    }
}

// One store after its sort: sorted position i holds store row row(i).
struct HoSorted {
    const uint32_t* id;
    const void* val;
    SortKey key;  // the value's encoding (ascending)
    const uint32_t* perm;  // nullptr: the identity
    int64_t n;
    __device__ __forceinline__ int64_t row(int64_t i) const { return perm ? (int64_t)(perm[i] & 0x7FFFFFFFu) : i; }
    __device__ __forceinline__ uint64_t word(int64_t r) const {
        bool na = false;
        return sort_word(key, load_bits(val, key.size, r), na);
    }
};
// head[g] = the first sorted position of id g, tail[g] = one past its last (both stay 0 for an id without values); flag[i] = a run
// of equal (id, value) starts at position i (flag nullptr: the store feeds no mode)
__global__ void holistic_bounds_kernel(const __grid_constant__ HoSorted s, uint32_t* head, uint32_t* tail, uint32_t* flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < s.n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = s.row(i);
        const uint32_t g = s.id[r];
        const bool first = i == 0 || s.id[s.row(i - 1)] != g;
        if (first) head[g] = (uint32_t)i;
        if (i + 1 == s.n || s.id[s.row(i + 1)] != g) tail[g] = (uint32_t)(i + 1);
        if (flag) flag[i] = first || s.word(s.row(i - 1)) != s.word(r);
    }
}
// start[pos[i]] = i for every run start i (pos: the exclusive scan of flag)
__global__ void holistic_run_start_kernel(const uint32_t* flag, const unsigned long long* pos, int64_t n, uint32_t* start) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (flag[i]) start[pos[i]] = (uint32_t)i;
}
// Run r covers sorted positions [start[r], start[r + 1]) (the last one ends at n).  best[g] = max over the runs of id g of
// (length << 32 | ~start): the longest run, and of equally long ones the first, which holds the least value.
__global__ void holistic_run_best_kernel(const __grid_constant__ HoSorted s, const uint32_t* start, int64_t n_runs, unsigned long long* best) {
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_runs; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = start[r];
        const int64_t e = r + 1 < n_runs ? (int64_t)start[r + 1] : s.n;
        atomicMax(best + s.id[s.row(b)], ((unsigned long long)(e - b) << 32) | (unsigned long long)(uint32_t)~b);
    }
}

// A store value (raw bits of its width) as a double, -0.0 read as +0.0 (so a result depends on the multiset of sort words only).
__device__ __forceinline__ double ho_f64(int ct, uint64_t raw) {
    double d;
    switch (ct) {
        case CT_FLOAT64: d = __longlong_as_double((long long)raw); break;
        case CT_FLOAT32: d = (double)__uint_as_float((uint32_t)raw); break;
        case CT_UINT64: return (double)raw;
        default: {
            const int sh = 64 - 8 * ctype_size(ct);
            return ctype_is_signed_int(ct) ? (double)((long long)(raw << sh) >> sh) : (double)raw;
        }
    }
    return d == 0.0 ? 0.0 : d;
}
// The result word of a store value as eval_output_kernel's K_FIRST case reads it: a float as its double's bits (+0.0 for a zero),
// an integer, bool or temporal sign- or zero-extended to 64 bits.
__device__ __forceinline__ unsigned long long ho_bits(int ct, uint64_t raw) {
    if (ctype_is_float(ct)) return (unsigned long long)__double_as_longlong(ho_f64(ct, raw));
    const int sh = 64 - 8 * ctype_size(ct);
    return ctype_is_signed_int(ct) ? (unsigned long long)((long long)(raw << sh) >> sh) : raw;
}

struct HoEvalArgs {
    HoSorted s;
    const unsigned long long* gid;  // per slot: the group's id
    uint64_t n_slots;               // cap + 2
    const uint32_t* head;
    const uint32_t* tail;
    const unsigned long long* best;  // mode: see holistic_run_best_kernel
    int n_f;                         // the functions over this store
    int kind[MAX_OPS];               // E_MODE, E_PCONT, E_PDISC
    double q[MAX_OPS];
    unsigned long long* res[MAX_OPS];   // the result word (a0) and its validity word (a1) per slot
    unsigned long long* seen[MAX_OPS];
};
// One thread per slot (one per group: the id's bounds give its m values, v_0 .. v_{m-1} at sorted positions head .. tail - 1).
// percentile_cont: h = q (m - 1), lo = floor(h), f = h - lo; v_lo when f == 0, else a + (b - a) f with a = v_lo and b = v_{lo+1}
// as doubles (pandas' linear group_quantile).  Rounded operations without contraction: the host restatement of the formula gets
// the same bits.  percentile_disc: v_i with i = clamp(ceil(q m) - 1, 0, m - 1).  mode: the value of the id's best run.
__global__ void holistic_eval_kernel(const __grid_constant__ HoEvalArgs a) {
    const HoSorted& s = a.s;
    for (uint64_t slot = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; slot < a.n_slots; slot += (uint64_t)gridDim.x * blockDim.x) {
        const unsigned long long g = a.gid[slot];
        if (g == ~0ull) continue;
        const int64_t h = a.head[g], m = (int64_t)a.tail[g] - h;
        if (m <= 0) continue;
        for (int f = 0; f < a.n_f; f++) {
            unsigned long long bits;
            if (a.kind[f] == E_PCONT) {
                const double hq = __dmul_rn(a.q[f], (double)(m - 1)), lo = floor(hq), fr = __dsub_rn(hq, lo);
                const int64_t i = (int64_t)lo;
                double r = ho_f64(s.key.ct, load_bits(s.val, s.key.size, s.row(h + i)));
                if (fr != 0.0) {
                    const double b = ho_f64(s.key.ct, load_bits(s.val, s.key.size, s.row(h + i + 1)));
                    r = __dadd_rn(r, __dmul_rn(__dsub_rn(b, r), fr));
                }
                bits = (unsigned long long)__double_as_longlong(r);
            } else {
                int64_t p;
                if (a.kind[f] == E_PDISC) {
                    const int64_t i = (int64_t)ceil(__dmul_rn(a.q[f], (double)m)) - 1;
                    p = h + (i < 0 ? 0 : i >= m ? m - 1 : i);
                } else {
                    p = (uint32_t)~(uint32_t)a.best[g];
                }
                bits = ho_bits(s.key.ct, load_bits(s.val, s.key.size, s.row(p)));
            }
            a.res[f][slot] = bits;
            a.seen[f][slot] = 0;
        }
    }
}

// ================================================================================================
// SM-partitioned groupby (SPG): the fast path for cardinalities whose accumulators fit the chip's
// aggregate shared memory (≈ SMs x 10k groups).  Motivation (scratch/ubench*.cu): two global `red`s per
// row cap the direct kernel well below the HBM stream rate and the key probe halves that again (L2 random-request rate), while
// 32-bit shared-memory atomics sustain the full HBM stream rate.  So rows travel to the SM that owns their key:
//
//   K1 spg_partition_tma_kernel : every CTA counting-sorts TILE-row tiles by owner (= mulhi(hash, n_owners)) in
//        shared memory, reserves one run per owner with a single global atomic per (tile, owner) and copies
//        the runs out with coalesced 16-byte stores -> owner buckets of (key, value) rows in HBM.
//   K2 spg_aggregate_kernel : one CTA per owner streams its bucket into a shared-memory hash table (key CAS,
//        SUM = two native 32-bit atomics with carry, COUNT = one), then flushes the table into the state's
//        global table with the ordinary find-or-insert + `red` (each key has one owner: <= n_groups per launch).
//   Algorithmic HBM traffic: 16 B/row read + 16 B/row bucket write + 16 B/row bucket read.
// A persistent single-kernel variant (L2-resident inboxes, inter-CTA barriers) is not used: per-chunk work per SM is
// too small to amortise the barrier latency.
// Rows that do not fit (bucket overflow under skew, shared table full, marker key) take the direct global path
// inside the same kernels; rows that cannot even be inserted there (global table at its limit) are appended to
// a retry list in the partial-aggregate wire format and merged by xchg_combine_kernel after the table grew.
constexpr int SPG_THREADS = 1024;   // K2 (aggregate) threads per CTA
constexpr int SPG_TILE = 2048;
constexpr int SPG_MAX_OWNERS = 256;
// K1 reserves one run per owner per tile with a global atomic on the owner's row counter: ~10^7 atomics per launch.  With
// the per-owner counters packed into a few cache lines K1's speed depended on where the array happened to land (same SASS,
// slower after an unrelated allocation moved it), so every counter gets its own line.
constexpr int SPG_CNT_STRIDE = 16;
constexpr int SPG_STASH = 1024;     // K2: linear-probing stash slots for keys whose two buckets are full
constexpr int SPGN_EMPTY = (int)0x80000000;  // free slot of a shared table with int32 keys (spgn.cuh)

struct SpgArgs {
    const long long* keys;
    const long long* vals;
    int64_t n_rows;
    int n_owners;
    // global table (state)
    long long* tkeys;
    uint64_t cap;
    unsigned long long* acc_sum;
    unsigned long long* acc_cnt;
    long long* counters;  // the state's counter block (CounterSlot); the retry list is counted in retry_ctr
    long long group_limit;
    // owner buckets
    longlong2* bucket;            // [n_owners][bucket_cap]
    unsigned long long* bucket_cnt;  // [n_owners * SPG_CNT_STRIDE] rows appended per owner (may exceed bucket_cap: the excess
                                     // went the direct way); one counter per 128-byte line, see SPG_CNT_STRIDE
    long long bucket_cap;
    unsigned long long* retry;  // partial-aggregate rows [key][1][a0 of func 0][a0 of func 1]
    long long* retry_ctr;       // number of rows in `retry`
    long long retry_cap;        // rows `retry` holds: an entry past it is dropped and raises counters[CTR_RETRY_OVERFLOW]
    int sum_first;              // order of the two accumulators in the wire format
    int ns;                     // shared-memory table slots (K2)
    int n_pass;                 // K2 passes over each owner bucket (pass p keeps the keys of sub-range p): > 1 when the
                                // estimated cardinality exceeds what the shared tables hold at once
    const long long* hot_tab;   // [SPG_HOT_SLOTS] heavy-hitter keys found by spg_hot_sample_kernel (EMPTY_KEY = free), or null
    const int* n_hot;           // number of keys in hot_tab (device memory: K1 reads it, the host never waits for it)
    int reserve_tickets;  // K2n flush: the global table is empty — a CTA reserves the group tickets of all its slots with one atomic
};
// SPG-N dense form (spgn.cuh): key window [kbase, kbase + 2^d_kb), value offsets of d_vb bits above vbase
struct SpgDenseArgs : SpgArgs {
    long long kbase, vbase;
    unsigned int d_kb, d_vb;
    unsigned int d_mul, d_inv;  // odd multiplier of the key scramble, and its inverse mod 2^32
    unsigned int d_gmagic;      // ceil(2^32 / n_owners): x div n_owners = umulhi(x, d_gmagic) for x < 2^21
    int d_slots;                // K2d table slots per owner: ceil(2^d_kb / n_owners)
};

// cheap in-kernel hash for owner / shared-table slot (placement inside one GPU is free to choose; the rank
// placement that must match the reference uses xxh3, see shuffle.cu)
__device__ __forceinline__ uint64_t spg_hash(long long key) {
    uint64_t x = (uint64_t)key;
    return (x ^ (x >> 29)) * 0x9E3779B97F4A7C15ULL;
}
__device__ __forceinline__ unsigned int spg_owner(uint64_t h, int n_owners) { return __umulhi((unsigned int)(h >> 32), (unsigned int)n_owners); }
__device__ __forceinline__ unsigned int spg_slot(uint64_t h, int ns) { return __umulhi((unsigned int)(h >> 20), (unsigned int)ns); }

template <bool HAS_SUM, bool HAS_CNT>
__device__ __forceinline__ void spg_retry_row(const SpgArgs& a, long long key, unsigned long long sum, unsigned long long cnt) {
    unsigned long long f = atomicAdd((unsigned long long*)a.retry_ctr, 1ull);
    if (f >= (unsigned long long)a.retry_cap) { a.counters[CTR_RETRY_OVERFLOW] = 1; return; }
    unsigned long long* r = a.retry + f * 4;
    r[0] = (unsigned long long)key; r[1] = 1ull;
    if (HAS_SUM && HAS_CNT) { r[2] = a.sum_first ? sum : cnt; r[3] = a.sum_first ? cnt : sum; }
    else { r[2] = HAS_SUM ? sum : cnt; r[3] = 0; }
}
template <bool HAS_SUM, bool HAS_CNT>
__device__ __forceinline__ void spg_direct_apply(const SpgArgs& a, long long key, unsigned long long sum, unsigned long long cnt) {
    uint64_t sl;
    if (key == EMPTY_KEY) { sl = a.cap + 1; a.counters[CTR_MARKER] = 1; }
    else {
        sl = find_or_insert(a.tkeys, a.cap, key, a.counters, a.group_limit);
        if (sl == ~0ull) { spg_retry_row<HAS_SUM, HAS_CNT>(a, key, sum, cnt); return; }
    }
    if (HAS_SUM && sum) atomicAdd(a.acc_sum + sl, sum);
    if (HAS_CNT && cnt) atomicAdd(a.acc_cnt + sl, cnt);
}

// ---- heavy hitters (skewed keys) ----------------------------------------------------------------------------
// A key that carries more than ~1/1024 of the rows (Zipf-like inputs: the top key of Zipf(1.1) over 1 M groups carries
// 12 %) would overload its owner: the bucket overflows into the direct path, where every row is a global atomic on ONE
// address (measured 10 Grows/s against 88 uniform).  Such keys are found once per operator state by counting a strided
// sample of the first launch (spg_hot_sample_kernel) and are then aggregated inside K1, in a per-CTA shared-memory
// accumulator table (two-slot buckets: one 16-byte load per row), and never reach the owner buckets.
constexpr int SPG_HOT_SLOTS = 128, SPG_HOT_BUCKETS = SPG_HOT_SLOTS / 2;
constexpr int SPG_HOT_SAMPLE = 1 << 15;  // sampled rows (one CTA counts them: the cost is per operator state, ~0.1 ms)
constexpr int SPG_HOT_TAB = 8192;        // counting-table slots of the sample kernel
constexpr size_t SPG_HOT_SAMPLE_SMEM = (size_t)SPG_HOT_TAB * 12 + SPG_HOT_SLOTS * 8;
__device__ __forceinline__ unsigned int spg_hot_bucket(uint64_t h) { return (unsigned int)(h >> 8) & (SPG_HOT_BUCKETS - 1); }

// Also the SPG-N verdicts: n_hot[1] = sampled rows that do not fit an (int32, int32) bucket row, and range = {min key, max key,
// min value, max value} of the sampled rows (the window of the dense form).
__global__ void __launch_bounds__(1024, 1) spg_hot_sample_kernel(const long long* keys, const long long* vals, int64_t n_rows, long long* hot_tab, int* n_hot,
                                                                 long long* range) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    long long* tk = (long long*)smem_raw;                  // SPG_HOT_TAB keys
    unsigned int* tc = (unsigned int*)(tk + SPG_HOT_TAB);  // their sample counts
    long long* hk = (long long*)(tc + SPG_HOT_TAB);        // SPG_HOT_SLOTS: the hot table being built
    __shared__ unsigned int fill, nh, nwide;
    __shared__ long long rng[4];
    const int tid = threadIdx.x;
    for (int s = tid; s < SPG_HOT_TAB; s += 1024) { tk[s] = EMPTY_KEY; tc[s] = 0; }
    for (int s = tid; s < SPG_HOT_SLOTS; s += 1024) hk[s] = EMPTY_KEY;
    if (tid == 0) { fill = 0; nh = 0; nwide = 0; rng[0] = rng[2] = LLONG_MAX; rng[1] = rng[3] = LLONG_MIN; }
    long long kmin = LLONG_MAX, kmax = LLONG_MIN, vmin = LLONG_MAX, vmax = LLONG_MIN;
    __syncthreads();
    // the sample = 32 evenly spaced blocks of 1024 contiguous rows (one coalesced 8 KB read per block and column: a row-strided
    // sample touched a different DRAM page and TLB entry with every load and took 0.26 ms for 32 Ki rows)
    const int64_t S = n_rows < SPG_HOT_SAMPLE ? n_rows : SPG_HOT_SAMPLE;
    const int64_t block_stride = S == SPG_HOT_SAMPLE ? n_rows / (SPG_HOT_SAMPLE / 1024) : 1024;
    constexpr int ILP = 4;
    for (int64_t i0 = tid; i0 < S; i0 += 1024 * ILP) {
        long long kv[ILP];
#pragma unroll
        for (int u = 0; u < ILP; u++) {
            const int64_t i = i0 + (int64_t)u * 1024;
            const int64_t row = (i >> 10) * block_stride + (i & 1023);
            kv[u] = i < S ? keys[row] : EMPTY_KEY;
            // SPG-N (spgn.cuh): does this sampled row fit an (int32, int32) bucket row?
            if (i < S) {
                const long long v = vals ? vals[row] : 0;
                if (kv[u] != (long long)(int)kv[u] || (int)kv[u] == (int)0x80000000 || v != (long long)(int)v) atomicAdd(&nwide, 1u);
                kmin = min(kmin, kv[u]); kmax = max(kmax, kv[u]); vmin = min(vmin, v); vmax = max(vmax, v);
            }
        }
#pragma unroll
        for (int u = 0; u < ILP; u++) {
            const long long k = kv[u];
            if (k == EMPTY_KEY) continue;
            unsigned int s = (unsigned int)(spg_hash(k) >> 40) & (SPG_HOT_TAB - 1);
            for (int probes = 0; probes < 8; probes++) {  // heavy hitters arrive while the table is empty: short probes suffice
                long long kk = *(volatile long long*)&tk[s];
                if (kk == EMPTY_KEY) {
                    // the table only has to hold the heavy hitters, which show up early: stop admitting keys at 50 % load
                    if (*(volatile unsigned int*)&fill >= SPG_HOT_TAB / 2) break;
                    kk = (long long)atomicCAS((unsigned long long*)&tk[s], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
                    if (kk == EMPTY_KEY) { atomicAdd(&fill, 1u); kk = k; }
                }
                if (kk == k) { atomicAdd(&tc[s], 1u); break; }
                s = (s + 1) & (SPG_HOT_TAB - 1);
            }
        }
    }
    for (int d = 16; d; d >>= 1) {
        kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, d)); kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, d));
        vmin = min(vmin, __shfl_xor_sync(0xffffffffu, vmin, d)); vmax = max(vmax, __shfl_xor_sync(0xffffffffu, vmax, d));
    }
    if ((tid & 31) == 0) { atomicMin(&rng[0], kmin); atomicMax(&rng[1], kmax); atomicMin(&rng[2], vmin); atomicMax(&rng[3], vmax); }
    __syncthreads();
    if (tid < 4) range[tid] = rng[tid];
    const unsigned int T = S >= (16 << 10) ? (unsigned int)(S >> 10) : 16u;  // hot = at least 1/1024 of the sample
    // admit candidates heaviest first (four count bands); a candidate whose two-slot bucket is taken stays an ordinary key
    for (int band = 3; band >= 0; band--) {
        const unsigned int lo = T << band, hi = band == 3 ? 0xffffffffu : (T << (band + 1));
        for (int s = tid; s < SPG_HOT_TAB; s += 1024) {
            const unsigned int c = tc[s];
            if (c < lo || c >= hi) continue;
            const long long k = tk[s];
            const unsigned int hb = spg_hot_bucket(spg_hash(k));
            unsigned long long old = atomicCAS((unsigned long long*)&hk[2 * hb], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
            if (old != (unsigned long long)EMPTY_KEY) old = atomicCAS((unsigned long long*)&hk[2 * hb + 1], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
            if (old == (unsigned long long)EMPTY_KEY) atomicAdd(&nh, 1u);
        }
        __syncthreads();
    }
    for (int s = tid; s < SPG_HOT_SLOTS; s += 1024) hot_tab[s] = hk[s];
    if (tid == 0) { n_hot[0] = (int)nh; n_hot[1] = (int)nwide; }
}

// K1: partition rows into owner buckets. grid = persistent (SPG_TCTAS CTAs / SM), tiles are taken grid-stride.
// The tile's key and value slabs are fetched with cp.async.bulk (TMA, SASS UBLKCP; the inputs must be 16-byte aligned) into
// a shared-memory staging area while the previous tile is being copied out, completion is signalled on an mbarrier
// (expect_tx / complete_tx), so no warp ever stalls on an HBM load and no row lives in registers across a barrier.
// Each tile is counting-sorted by owner in shared memory: hash, shared-memory histogram atomic (a row's rank in its owner's
// run), exclusive scan of the histogram by warp 0, staging of the rows at their sorted positions.  One global atomic per
// (tile, owner) on the owner's row counter reserves a run in its bucket, and the runs are copied out with coalesced 16-byte
// stores; rows past the end of a bucket (skew) take the direct path.  spg_partition_tiles below is this loop for every K1
// form (K1, K1n in spgn.cuh, K1g in spgg.cuh); a form supplies only what it loads, how it classifies and stages a row, and
// how it copies the staged rows out.
constexpr int SPG_TTHREADS = 512;  // threads per CTA of K1 (4 rows per thread per tile)
constexpr int SPG_TCTAS = 3;       // CTAs per SM

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// The shared memory of one K1 shape, as byte offsets: the raw tile (TMA destination: TILE 8-byte keys, TILE 8-byte values),
// TILE staged rows of ROW_BYTES, per class the published run start (gbase), the tile's mbarrier, the class histogram and its
// exclusive scan (lbase), then TAIL bytes the form lays out itself.  Every region is a multiple of 16 bytes (TMA destinations).
// The kernel takes its pointers and the host its launch size (`bytes`) from here.
template <int TILE, int MAX_C, int ROW_BYTES, int TAIL>
struct SpgTileSmem {
    static constexpr size_t raw_k = 0, raw_v = raw_k + (size_t)TILE * 8, stage = raw_v + (size_t)TILE * 8;
    static constexpr size_t gbase = stage + (size_t)TILE * ROW_BYTES, mbar = gbase + (size_t)MAX_C * 8, hist = mbar + 16;
    static constexpr size_t lbase = hist + (size_t)MAX_C * 4, tail = lbase + (size_t)(MAX_C + 4) * 4, bytes = tail + TAIL;
    static_assert(stage % 16 == 0 && gbase % 16 == 0 && lbase % 16 == 0 && tail % 16 == 0, "K1 shared regions stay 16-byte aligned");
};

// The K1 tile loop shared by every form.  C classes (at most the shape's MAX_C, and at most THREADS: the last C threads
// reserve the runs); class c's bucket row counter is cls_cnt[c * SPG_CNT_STRIDE].  The form's part, as callables:
//   load_tma(r0, mbar)    thread 0, full tile at row r0: expect_tx on mbar and the tile's bulk copies
//   load_partial(r0)      every thread, the trailing partial tile: the same slabs with ordinary loads
//   init()                thread 0, once, after the mbarrier's init: the form's own shared state
//   classify(j, w)        tile row j (in range): its class, or -1 when the row was handled here; w is handed on to stage
//   stage(p, j, c, w)     store tile row j of class c at staged position p
//   on_run(c, g0, n)      the run thread of class c, after gbase[c] is published: the run starts at g0 and holds n rows
//   copy_out(n_tile)      copy the n_tile staged rows out: staged row p of class c goes to offset gbase[c] + p of c's bucket
template <int TILE, int THREADS, typename Smem, typename LoadTma, typename LoadPartial, typename Init, typename Classify,
          typename Stage, typename OnRun, typename CopyOut>
__device__ __forceinline__ void spg_partition_tiles(unsigned char* smem, int64_t n_rows, int C, unsigned long long* cls_cnt,
                                                    LoadTma load_tma, LoadPartial load_partial, Init init, Classify classify,
                                                    Stage stage, OnRun on_run, CopyOut copy_out) {
    unsigned long long* gbase = (unsigned long long*)(smem + Smem::gbase);
    uint64_t* mbar = (uint64_t*)(smem + Smem::mbar);
    unsigned int* hist = (unsigned int*)(smem + Smem::hist);
    unsigned int* lbase = (unsigned int*)(smem + Smem::lbase);
    const int tid = threadIdx.x;
    constexpr int ROWS = TILE / THREADS;
    const int64_t n_tiles = (n_rows + TILE - 1) / TILE;
    if (tid == 0) {
        mbar_init(mbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        init();
    }
    for (int j = tid; j < C; j += THREADS) hist[j] = 0;
    __syncthreads();
    // full tiles come in through TMA; a trailing partial tile is loaded with ordinary loads
    auto issue = [&](int64_t t) {
        const int64_t r0 = t * TILE;
        if (r0 + TILE <= n_rows && tid == 0) load_tma(r0, mbar);
    };
    uint32_t phase = 0;
    int64_t t = blockIdx.x;
    if (t < n_tiles) issue(t);
    for (; t < n_tiles; t += gridDim.x) {
        const int64_t r0 = t * TILE;
        const int64_t tn = t + gridDim.x;
        const bool full = r0 + TILE <= n_rows;
        if (full) {
            while (!mbar_try_wait(mbar, phase)) {}
            phase ^= 1;
        } else {
            load_partial(r0);
            __syncthreads();
        }
        int c[ROWS];
        unsigned int rk[ROWS];
        [[maybe_unused]] unsigned int w[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
            const int j = r * THREADS + tid;
            c[r] = -1;
            if (r0 + j >= n_rows) continue;
            c[r] = classify(j, w[r]);
            if (c[r] >= 0) rk[r] = atomicAdd(&hist[c[r]], 1u);
        }
        __syncthreads();
        // reserve one run per class: the global atomic's round trip (~1 us) is kept in a register and only waited for
        // after the staging pass, which needs the local prefix sums but not the global run start
        unsigned long long my_gbase = 0;
        unsigned int my_cnt = 0;
        if (tid >= THREADS - C) { const int cl = tid - (THREADS - C); my_cnt = hist[cl]; if (my_cnt) my_gbase = atomicAdd(&cls_cnt[cl * SPG_CNT_STRIDE], (unsigned long long)my_cnt); }
        if (tid < 32) {
            unsigned int carry = 0;
            for (int base = 0; base < C; base += 32) {
                int j = base + tid;
                unsigned int x = j < C ? hist[j] : 0u, inc = x;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { unsigned int y = __shfl_up_sync(0xffffffffu, inc, d); if (tid >= d) inc += y; }
                if (j < C) lbase[j] = carry + inc - x;
                carry += __shfl_sync(0xffffffffu, inc, 31);
            }
            if (tid == 0) lbase[C] = carry;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
            if (c[r] < 0) continue;
            stage(lbase[c[r]] + rk[r], r * THREADS + tid, c[r], w[r]);
        }
        // publish run start minus local start, so the copy-out computes its destination with one add
        if (tid >= THREADS - C) {
            const int cl = tid - (THREADS - C);
            gbase[cl] = my_gbase - lbase[cl];
            on_run(cl, my_gbase, my_cnt);
        }
        __syncthreads();  // the raw tile is free from here on
        if (tn < n_tiles) issue(tn);  // the next tile streams in during the copy-out
        copy_out(lbase[C]);
        for (int j = tid; j < C; j += THREADS) hist[j] = 0;
        __syncthreads();
    }
}

// K1 (16-byte rows): class = owner.  The marker key takes the direct path; with HOT the heavy hitters are aggregated here.
template <bool HOT>
using SpgK1Smem = SpgTileSmem<SPG_TILE, SPG_MAX_OWNERS, 16, SPG_TILE + (HOT ? SPG_HOT_SLOTS * 20 : 0)>;

template <bool HAS_SUM, bool HAS_CNT, bool HOT = false>
__global__ void __launch_bounds__(SPG_TTHREADS, SPG_TCTAS) spg_partition_tma_kernel(const __grid_constant__ SpgArgs a) {
    extern __shared__ __align__(128) unsigned char smem_tma_raw[];  // own name: the other kernels declare smem_raw with 16-byte alignment
    using L = SpgK1Smem<HOT>;
    long long* raw_k = (long long*)(smem_tma_raw + L::raw_k);
    long long* raw_v = (long long*)(smem_tma_raw + L::raw_v);
    longlong2* stage = (longlong2*)(smem_tma_raw + L::stage);
    const unsigned long long* gbase = (const unsigned long long*)(smem_tma_raw + L::gbase);
    unsigned char* stage_owner = smem_tma_raw + L::tail;                       // SPG_TILE
    long long* hkeys = (long long*)(stage_owner + SPG_TILE);                   // SPG_HOT_SLOTS heavy-hitter keys ...
    unsigned int* hlo = (unsigned int*)(hkeys + SPG_HOT_SLOTS);                // ... and this CTA's partial sums / row counts
    unsigned int* hhi = hlo + SPG_HOT_SLOTS;
    unsigned int* hcnt = hhi + SPG_HOT_SLOTS;
    const int G = a.n_owners, tid = threadIdx.x;
    // HOT is a separate instantiation: the uniform-key kernel carries none of this
    if (HOT)
        for (int s = tid; s < SPG_HOT_SLOTS; s += SPG_TTHREADS) { hkeys[s] = a.hot_tab[s]; hlo[s] = 0; hhi[s] = 0; hcnt[s] = 0; }
    spg_partition_tiles<SPG_TILE, SPG_TTHREADS, L>(
        smem_tma_raw, a.n_rows, G, a.bucket_cnt,
        [&](int64_t r0, uint64_t* mbar) {
            mbar_expect_tx(mbar, (HAS_SUM ? 2u : 1u) * SPG_TILE * 8u);
            tma_load_1d(raw_k, a.keys + r0, SPG_TILE * 8u, mbar);
            if (HAS_SUM) tma_load_1d(raw_v, a.vals + r0, SPG_TILE * 8u, mbar);
        },
        [&](int64_t r0) {
            for (int j = tid; j < SPG_TILE; j += SPG_TTHREADS) {
                const int64_t i = r0 + j;
                raw_k[j] = i < a.n_rows ? a.keys[i] : 0;
                raw_v[j] = (HAS_SUM && i < a.n_rows) ? a.vals[i] : 0;
            }
        },
        [] {},
        [&](int j, unsigned int&) -> int {
            const long long k = raw_k[j];
            if (k == EMPTY_KEY) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, k, HAS_SUM ? (unsigned long long)raw_v[j] : 0ull, 1ull); return -1; }
            const uint64_t h = spg_hash(k);
            if (HOT) {  // heavy hitter: aggregate here, the row never reaches an owner bucket
                const unsigned int hb = spg_hot_bucket(h);
                const ulonglong2 hk2 = *reinterpret_cast<const ulonglong2*>(hkeys + 2 * hb);
                const int hs = hk2.x == (unsigned long long)k ? (int)(2 * hb) : hk2.y == (unsigned long long)k ? (int)(2 * hb + 1) : -1;
                if (hs >= 0) {
                    if (HAS_SUM) {
                        const unsigned long long v = (unsigned long long)raw_v[j];
                        const unsigned int lo = (unsigned int)v;
                        unsigned int hi = (unsigned int)(v >> 32);
                        const unsigned int old = atomicAdd(&hlo[hs], lo);
                        hi += (old + lo < old) ? 1u : 0u;
                        if (hi) atomicAdd(&hhi[hs], hi);
                    }
                    atomicAdd(&hcnt[hs], 1u);  // rows, also when only SUM is asked for: the group has to exist
                    return -1;
                }
            }
            return (int)spg_owner(h, G);
        },
        [&](unsigned int p, int j, int o, unsigned int) {
            stage[p] = make_longlong2(raw_k[j], HAS_SUM ? raw_v[j] : 0);
            stage_owner[p] = (unsigned char)o;
        },
        [](int, unsigned long long, unsigned int) {},
        [&](unsigned int n_tile) {
            for (unsigned int p = tid; p < n_tile; p += SPG_TTHREADS) {
                unsigned int ow = stage_owner[p];
                unsigned long long off = gbase[ow] + p;
                longlong2 row = stage[p];
                if (off < (unsigned long long)a.bucket_cap) a.bucket[(size_t)ow * a.bucket_cap + off] = row;
                else spg_direct_apply<HAS_SUM, HAS_CNT>(a, row.x, (unsigned long long)row.y, 1ull);
            }
        });
    if (HOT) {  // this CTA's heavy-hitter partials -> global table (n_hot atomics per CTA)
        __syncthreads();
        for (int s = tid; s < SPG_HOT_SLOTS; s += SPG_TTHREADS)
            if (hcnt[s]) spg_direct_apply<HAS_SUM, HAS_CNT>(a, hkeys[s], (unsigned long long)hlo[s] | ((unsigned long long)hhi[s] << 32), (unsigned long long)hcnt[s]);
    }
}

// The two-choice shared table of K2, K2n and K2g: every key has two candidate buckets of two slots (one shared load each);
// slots [2 NB, 2 NB + SPG_STASH) are a linear-probing stash.  K is the slot's key word: long long (free = EMPTY_KEY) or int
// (free = SPGN_EMPTY).
template <typename K>
using SpgKeyPair = std::conditional_t<sizeof(K) == 8, longlong2, int2>;
template <typename K>
__device__ __forceinline__ constexpr K spg_free_key() {
    if constexpr (sizeof(K) == 8) return EMPTY_KEY;
    else return SPGN_EMPTY;
}
__device__ __forceinline__ long long spg_cas(long long* p, long long cmp, long long val) {
    return (long long)atomicCAS((unsigned long long*)p, (unsigned long long)cmp, (unsigned long long)val);
}
__device__ __forceinline__ int spg_cas(int* p, int cmp, int val) { return atomicCAS(p, cmp, val); }

// the two candidate buckets of a key with hash h among the NB buckets
__device__ __forceinline__ void spg_buckets(uint64_t h, unsigned int NB, unsigned int& b1, unsigned int& b2) {
    b1 = __umulhi((unsigned int)(h >> 20), NB);
    b2 = __umulhi(((unsigned int)h ^ (unsigned int)(h >> 44)) * 0x9E3779B1u, NB);  // low word of h remixed: independent of b1's bits 20..51 enough
    b2 = b2 == b1 ? (b1 + 1 == NB ? 0u : b1 + 1) : b2;
}

// the slot of `key` among the four candidates, the keys c1 of bucket b1 and c2 of bucket b2, or -1
template <typename K>
__device__ __forceinline__ int spg_match(SpgKeyPair<K> c1, SpgKeyPair<K> c2, unsigned int b1, unsigned int b2, K key) {
    return c1.x == key ? (int)(2 * b1) : c1.y == key ? (int)(2 * b1 + 1) : c2.x == key ? (int)(2 * b2) : c2.y == key ? (int)(2 * b2 + 1) : -1;
}
// the hot lookup: two loads and four compares, no branch
template <typename K>
__device__ __forceinline__ int spg_find(const K* skeys, unsigned int b1, unsigned int b2, K key) {
    return spg_match<K>(*reinterpret_cast<const SpgKeyPair<K>*>(skeys + 2 * b1), *reinterpret_cast<const SpgKeyPair<K>*>(skeys + 2 * b2), b1, b2, key);
}

// The slow path of a key with hash h in a table of NS bucket slots: its slot if one of the four candidates holds it, else a free candidate slot it claims,
// else its find-or-insert slot in the stash; -1 when the stash is full too (the caller takes the direct path).
// Balanced allocation: a new key goes to the EMPTIER of its two buckets (0.9 % of the keys overflow into the stash at 50 %
// load where first-fit left 2.2 % there — every row of a stash-resident key comes through here), and the four CAS attempts
// are skipped when both buckets are full (buckets never lose keys), so a stash-resident key costs two loads and one stash
// probe instead of four failed CAS round trips.
template <typename K>
__device__ __forceinline__ int spg_claim(K* skeys, unsigned int NS, uint64_t h, K key) {
    constexpr K FREE = spg_free_key<K>();
    const unsigned int NB = NS / 2;
    unsigned int b1, b2;
    spg_buckets(h, NB, b1, b2);
    const SpgKeyPair<K> c1 = *reinterpret_cast<const SpgKeyPair<K>*>(skeys + 2 * b1);
    const SpgKeyPair<K> c2 = *reinterpret_cast<const SpgKeyPair<K>*>(skeys + 2 * b2);
    const int f1 = (c1.x == FREE) + (c1.y == FREE), f2 = (c2.x == FREE) + (c2.y == FREE);
    int s = spg_match<K>(c1, c2, b1, b2, key);
    if (s < 0 && f1 + f2 > 0) {
        const unsigned int first = f2 > f1 ? b2 : b1, second = f2 > f1 ? b1 : b2;
        const unsigned int cand[4] = {2 * first, 2 * first + 1, 2 * second, 2 * second + 1};
#pragma unroll
        for (int c = 0; c < 4 && s < 0; c++) {
            const K prev = spg_cas(&skeys[cand[c]], FREE, key);
            if (prev == FREE || prev == key) s = (int)cand[c];
        }
    }
    if (s < 0) {
        unsigned int st = NS + ((unsigned int)(h >> 12) & (SPG_STASH - 1));
        for (int probes = 0; probes < SPG_STASH && s < 0; probes++) {
            K kk = skeys[st];
            if (kk == FREE) {
                const K prev = spg_cas(&skeys[st], FREE, key);
                if (prev == FREE) { s = (int)st; break; }
                kk = prev;
            }
            if (kk == key) { s = (int)st; break; }
            st = st + 1 == NS + SPG_STASH ? NS : st + 1;
        }
    }
    return s;
}

// K2: one CTA per owner aggregates its bucket in shared memory, then flushes into the global table.
//
// Shared table = the two-choice bucketed hash table + stash above (spg_find / spg_claim) with 16-byte candidate loads, so
// the hot lookup is two unconditional loads + four compares, no probe loop and no divergence
// (a linear-probing table spends much of its issue slots on loop control with about half the lanes active; compare a
// collision-free key set with scratch/ubench3.cu).
// Everything else — first appearance of a key (CAS into a free candidate slot), keys whose four candidates are taken
// (~2 % at this load: linear-probing stash behind the buckets), a full stash (direct global path), a non-zero high word
// of the sum — is parked and handled once per iteration behind the hot path.  Two racing inserts may put one key into
// both of its buckets: harmless, both partial sums are flushed into the same global group.
template <bool HAS_SUM, bool HAS_CNT>
__global__ void __launch_bounds__(SPG_THREADS, 1) spg_aggregate_kernel(const __grid_constant__ SpgArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int NS = a.ns, NT = a.ns + SPG_STASH, tid = threadIdx.x, me = blockIdx.x;  // NS bucket slots + stash
    // 16 bytes per slot: key, low 32 bits of the sum (biased by 2^31 so sums of small positive AND negative values stay away
    // from the 32-bit wrap points), count.  The high word of an addition (value bits 32..63 plus the carry out of the low
    // word) is almost always zero; when it is not it is added straight to the global table: SUM stays exact mod 2^64.
    long long* skeys = (long long*)smem_raw;          // NT x 8
    unsigned int* slo = (unsigned int*)(skeys + NT);  // NT x 4
    unsigned int* scnt = slo + NT;
    const unsigned int NB = (unsigned int)NS / 2;
    const unsigned int NP = (unsigned int)a.n_pass, GP = (unsigned int)gridDim.x * NP;

    auto add = [&](int s, long long key, long long val) {
        if (HAS_SUM) {
            unsigned int lo = (unsigned int)(unsigned long long)val, hi = (unsigned int)((unsigned long long)val >> 32);
            unsigned int old = atomicAdd(&slo[s], lo);
            hi += (old + lo < old) ? 1u : 0u;  // carry of this very addition
            if (hi) spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, (unsigned long long)hi << 32, 0ull);
        }
        if (HAS_CNT) atomicAdd(&scnt[s], 1u);
    };
    // slow path: the key's slot, a free candidate slot or a stash slot, else the direct global path
    auto slow_upsert = [&](long long key, long long val) {
        const int s = spg_claim(skeys, (unsigned int)NS, spg_hash(key), key);
        if (s < 0) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, (unsigned long long)val, 1ull); return; }
        add(s, key, val);
    };

    unsigned long long n_in = a.bucket_cnt[me * SPG_CNT_STRIDE];
    if (n_in > (unsigned long long)a.bucket_cap) n_in = (unsigned long long)a.bucket_cap;
    const longlong2* src = a.bucket + (size_t)me * a.bucket_cap;
    constexpr int U = 4;  // independent bucket loads in flight per thread
    // rows of this thread: rsrc[first + u * stride], u = 0..U-1, valid while < limit
    auto process = [&](const longlong2* rsrc, unsigned long long first, unsigned long long stride, unsigned long long limit, unsigned int pass, auto full_tag) {
        constexpr bool FULL = decltype(full_tag)::value;  // FULL: all U rows of every thread are in range (no padding checks)
        longlong2 row[U];
        int sl[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            unsigned long long p = first + (unsigned long long)u * stride;
            row[u] = (FULL || p < limit) ? __ldcs(rsrc + p) : make_longlong2(EMPTY_KEY, 0);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {  // hot lookups: branch-free
            unsigned int b1, b2;
            spg_buckets(spg_hash(row[u].x), NB, b1, b2);
            sl[u] = spg_find(skeys, b1, b2, row[u].x);
            if (!FULL && row[u].x == EMPTY_KEY) sl[u] = -2;  // padding lane
            // multi-pass: owner = mulhi(hash_hi, G) = mulhi(hash_hi, G * NP) / NP; this pass keeps sub-range `pass` only
            if (NP > 1 && __umulhi((unsigned int)(spg_hash(row[u].x) >> 32), GP) - (unsigned int)me * NP != pass) sl[u] = -2;
        }
        long long pk = 0, pv = 0;
        bool parked = false;
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (sl[u] >= 0) add(sl[u], row[u].x, row[u].y);
            else if (sl[u] == -1) {
                if (!parked) { pk = row[u].x; pv = row[u].y; parked = true; }
                else slow_upsert(row[u].x, row[u].y);  // second slow row of this thread in one iteration: rare
            }
        }
        if (parked) slow_upsert(pk, pv);
    };
    const unsigned long long step = (unsigned long long)U * SPG_THREADS;
    const unsigned long long n_full = n_in / step * step;
    for (unsigned int pass = 0; pass < NP; pass++) {
        for (int s = tid; s < NT; s += SPG_THREADS) { skeys[s] = EMPTY_KEY; slo[s] = 0x80000000u; scnt[s] = 0; }
        __syncthreads();
        for (unsigned long long base = 0; base < n_full; base += step) process(src, base + tid, (unsigned long long)SPG_THREADS, n_in, pass, std::true_type{});
        if (n_full < n_in) process(src, n_full + tid, (unsigned long long)SPG_THREADS, n_in, pass, std::false_type{});
        __syncthreads();
        // flush the shared table into the state's global table
        for (int s = tid; s < NT; s += SPG_THREADS) {
            long long key = skeys[s];
            if (key == EMPTY_KEY) continue;
            unsigned long long sum = (unsigned long long)slo[s] - 0x80000000ull;  // remove the bias (wraps mod 2^64)
            spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, sum, (unsigned long long)scnt[s]);
        }
        __syncthreads();
    }
}

#include "spgn.cuh"  // SPG-N: narrow (int32 key, int32 value) bucket rows: 32 instead of 48 B/row of HBM traffic
#include "spgg.cuh"  // SPG-G: the same two kernels for nullable / 4-byte / mean / min / max signatures

// ---- low-cardinality kernel (LC): every CTA keeps a private shared-memory table of ALL groups ----------------
// Used when the (estimated) number of groups fits one CTA's table (<= LC_SLOTS / 2), e.g. BASELINE.json configs[0]
// (20 M rows, 30 groups) where every row of a warp hits one of a handful of hot keys.  Rows are pre-aggregated inside
// the warp when the whole warp holds ONE key (hot key / clustered input): the warp's SUM is formed with four
// __reduce_add_sync (REDUX) over 16-bit limbs (exact: 32 lanes x 65535 < 2^32 per limb, limbs recombined mod 2^64),
// its COUNT is popc(active), and one lane touches the shared table; otherwise each lane updates the CTA-private table
// (CAS-probe + native 32-bit atomics with carry).  One pass over the input: 16 B/row of HBM traffic, no global atomics
// until the final flush.
constexpr int LC_THREADS = 512;
// per-CTA table slots (20 B each); groups beyond LC_SLOTS / 2 take the direct path.  Two instantiations: 1024 slots
// (3 CTAs = 1536 threads per SM, for <= 256 expected groups) and 4096 slots (2 CTAs per SM, <= 1024 expected groups).
constexpr int LC_SLOTS_BIG = 4096, LC_SLOTS_SMALL = 1024;

template <bool HAS_SUM, bool HAS_CNT, int LC_SLOTS, int MIN_CTAS>
__global__ void __launch_bounds__(LC_THREADS, MIN_CTAS) groupby_lowcard_kernel(const __grid_constant__ SpgArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    long long* lkeys = (long long*)smem_raw;                 // LC_SLOTS x 8
    unsigned int* llo = (unsigned int*)(lkeys + LC_SLOTS);  // low / high words of the sum, count
    unsigned int* lhi = llo + LC_SLOTS;
    unsigned int* lcnt = lhi + LC_SLOTS;
    unsigned int* misc = lcnt + LC_SLOTS;
    const int tid = threadIdx.x, lane = tid & 31;
    for (int s = tid; s < LC_SLOTS; s += LC_THREADS) { lkeys[s] = EMPTY_KEY; llo[s] = 0; lhi[s] = 0; lcnt[s] = 0; }
    if (tid == 0) misc[0] = 0;
    __syncthreads();

    auto leader_upsert = [&](long long key, unsigned long long sum, unsigned int cnt) {
        unsigned int s = (unsigned int)(spg_hash(key) >> 32) & (LC_SLOTS - 1);
        bool done = false;
        for (int probes = 0; probes < LC_SLOTS; probes++) {
            long long kk = lkeys[s];
            if (kk == EMPTY_KEY) {
                unsigned int t = atomicAdd(&misc[0], 1u);
                if (t >= LC_SLOTS / 2) { atomicSub(&misc[0], 1u); break; }
                long long prev = (long long)atomicCAS((unsigned long long*)&lkeys[s], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
                if (prev == EMPTY_KEY) { done = true; break; }
                atomicSub(&misc[0], 1u);
                kk = prev;
            }
            if (kk == key) { done = true; break; }
            s = (s + 1) & (LC_SLOTS - 1);
        }
        if (!done) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, sum, (unsigned long long)cnt); return; }
        if (HAS_SUM) {
            unsigned int lo = (unsigned int)sum, hi = (unsigned int)(sum >> 32);
            unsigned int old = atomicAdd(&llo[s], lo);
            hi += (old + lo < old) ? 1u : 0u;
            if (hi) atomicAdd(&lhi[s], hi);
        }
        if (HAS_CNT) atomicAdd(&lcnt[s], cnt);
    };

    // warp-uniform trip count (bounds checked per row): the warp collectives below need converged warps
    const int64_t stride = (int64_t)gridDim.x * LC_THREADS * 2;
    const int64_t n_round = (a.n_rows + 63) & ~63ll;
    for (int64_t i = ((int64_t)blockIdx.x * LC_THREADS + tid) * 2; i < n_round; i += stride) {
        long long k[2] = {0, 0}, v[2] = {0, 0};
        bool ok[2] = {i < a.n_rows, i + 1 < a.n_rows};
        if (ok[1]) {
            longlong2 kk = __ldcs(reinterpret_cast<const longlong2*>(a.keys + i));
            k[0] = kk.x; k[1] = kk.y;
            if (HAS_SUM) { longlong2 vv = __ldcs(reinterpret_cast<const longlong2*>(a.vals + i)); v[0] = vv.x; v[1] = vv.y; }
        } else if (ok[0]) {
            k[0] = a.keys[i];
            if (HAS_SUM) v[0] = a.vals[i];
        }
#pragma unroll
        for (int r = 0; r < 2; r++) {
            if (ok[r] && k[r] == EMPTY_KEY) { spg_direct_apply<HAS_SUM, HAS_CNT>(a, k[r], (unsigned long long)v[r], 1ull); ok[r] = false; }
            const unsigned act = __ballot_sync(0xffffffffu, ok[r]);
            if (!ok[r]) continue;
            // warp-uniform shortcut (one hot key, sorted / clustered input): reduce the whole warp with REDUX and let one
            // lane update the table.  Otherwise every lane updates the CTA table itself: for >= ~30 distinct keys per warp
            // a __match_any_sync based pre-aggregation was measured 3-5x slower (it serialises over the distinct keys).
            const long long k0 = __shfl_sync(act, k[r], __ffs(act) - 1);
            const bool uniform = __all_sync(act, k[r] == k0) && act != (1u << (__ffs(act) - 1));
            if (uniform) {
                unsigned long long sum = 0;
                if (HAS_SUM) {
                    const unsigned long long u = (unsigned long long)v[r];
                    const unsigned int l0 = __reduce_add_sync(act, (unsigned int)(u & 0xffffu));
                    const unsigned int l1 = __reduce_add_sync(act, (unsigned int)((u >> 16) & 0xffffu));
                    const unsigned int l2 = __reduce_add_sync(act, (unsigned int)((u >> 32) & 0xffffu));
                    const unsigned int l3 = __reduce_add_sync(act, (unsigned int)(u >> 48));
                    sum = (unsigned long long)l0 + ((unsigned long long)l1 << 16) + ((unsigned long long)l2 << 32) + ((unsigned long long)l3 << 48);
                }
                if (lane == __ffs(act) - 1) leader_upsert(k0, sum, (unsigned int)__popc(act));
            } else {
                leader_upsert(k[r], (unsigned long long)v[r], 1u);
            }
        }
    }
    __syncthreads();
    for (int s = tid; s < LC_SLOTS; s += LC_THREADS) {
        long long key = lkeys[s];
        if (key == EMPTY_KEY) continue;
        unsigned long long sum = (unsigned long long)llo[s] | ((unsigned long long)lhi[s] << 32);
        spg_direct_apply<HAS_SUM, HAS_CNT>(a, key, sum, (unsigned long long)lcnt[s]);
    }
}

// ================================================================================================
// Host side
// ================================================================================================

// One user-visible aggregate: evaluated from the accumulators of `prim[0..n_prim)` (indices into the primitive list)
struct OutSpec {
    int ftype;
    int kind;        // OpKind used by eval_output_kernel
    int prim[4];
    int n_prim;
    int out_ctype, out_arrtype;
};

struct FuncSpec {
    int ftype;
    int in_col;  // physical input column or -1 (size)
    int in_ctype;
    int in_arrtype;
    int kind;
    int out_ctype;
    int out_arrtype;
    bool has_a1;
    unsigned long long init0;
    unsigned long long init1 = 0;  // initial value of the second accumulator
};

// ---- kernel-variant dispatch ----
// for_each_X(f) calls f once per instantiation of kernel family X that a launch can pick, with its template arguments as
// std::integral_constant values: spg_probe() sets the shared-memory limits through it.  with_X(..., f) calls f for the one
// instantiation the runtime arguments select, found by the same enumeration, so a launch never picks a kernel whose limit
// was not set.
template <bool V> using bool_c = std::bool_constant<V>;
template <int V> using int_c = std::integral_constant<int, V>;
// sum / count kernels <HAS_SUM, HAS_CNT> (LC, K1, K1-hot, K2, K1n, K2n, the direct int64 kernel): <false, false> does not exist
constexpr auto for_each_sum_cnt = [](auto&& f) {
    f(bool_c<true>{}, bool_c<true>{}); f(bool_c<true>{}, bool_c<false>{}); f(bool_c<false>{}, bool_c<true>{});
};
// K1g spgg_partition_kernel<KEY_BYTES, VALUE_BYTES> (0 value bytes: size only)
constexpr auto for_each_spgg_part = [](auto&& f) {
    f(int_c<8>{}, int_c<8>{}); f(int_c<8>{}, int_c<4>{}); f(int_c<8>{}, int_c<0>{});
    f(int_c<4>{}, int_c<8>{}); f(int_c<4>{}, int_c<4>{}); f(int_c<4>{}, int_c<0>{});
};
// K2g spgg_aggregate_kernel<HAS_SUM, HAS_MM, HAS_NN>: all eight
constexpr auto for_each_spgg_agg = [](auto&& f) {
    auto both_sums = [&](auto m, auto n) { f(bool_c<false>{}, m, n); f(bool_c<true>{}, m, n); };
    both_sums(bool_c<false>{}, bool_c<false>{}); both_sums(bool_c<true>{}, bool_c<false>{});
    both_sums(bool_c<false>{}, bool_c<true>{}); both_sums(bool_c<true>{}, bool_c<true>{});
};
template <typename Each, typename F, typename... W>
void with_variant(Each&& each, F&& f, W... want) {
    bool found = false;
    each([&](auto... c) { if (((c == want) && ...)) { found = true; f(c...); } });
    B200_REQUIRE(found, "internal: no kernel instantiation for this aggregate signature");
}
template <typename F> void with_sum_cnt(bool s, bool c, F&& f) { with_variant(for_each_sum_cnt, f, s, c); }
template <typename F> void with_spgg_part(int ks, int vs, F&& f) { with_variant(for_each_spgg_part, f, ks, vs); }
template <typename F> void with_spgg_agg(bool s, bool m, bool n, F&& f) { with_variant(for_each_spgg_agg, f, s, m, n); }

// raises a kernel's dynamic shared-memory limit; false (error cleared) when the device refuses
static bool set_smem_limit(const void* fn, size_t bytes) {
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess) return true;
    cudaGetLastError();
    return false;
}

// The arguments of a min_row_number_filter state (b200_groupby_state_init_mrnf), checked by GroupbyState::setup_mrnf.
struct MrnfSpec {
    int n_sort;
    const int32_t* sort_cols;
    const int32_t* ascending;
    const int32_t* na_last;
    const int32_t* keep;  // one flag per column
    int64_t limit;        // rows kept per group (b200_groupby_state_init_mrnf_limit)
};

class GroupbyState {
   public:
    int device;
    cudaStream_t stream;
    cudaStream_t copy_stream = nullptr;
    int n_cols;
    // Two types per column.  in_types: the caller's (batch validation, output typing, owner hashing).  c_types: what the table
    // and every consume path read — a float key column is consumed as its canonical int64 column (canon_keys), so it is CT_INT64
    // here; every other column has its input type.
    std::vector<int8_t> in_types, c_types, arr_types;
    int n_funcs;                  // primitive accumulator functions (what the kernels, the table and the exchange see)
    std::vector<FuncSpec> funcs;
    int n_outs = 0;               // aggregates the caller asked for (output columns)
    std::vector<OutSpec> outs;
    bool dropna, parallel;
    bool has_firstlast = false;
    int owner_nk = 0;  // see MkOwner::own_nk
    // nunique: one nested distinct state over (key, value) per value column; `prims` = the K_NUNIQUE accumulators it feeds
    struct NuInner { int in_col; std::unique_ptr<GroupbyState> st; std::vector<int> prims; };
    std::vector<NuInner> nu_inner;
    bool nu_applied = false;
    int n_pes, rank;
    int64_t output_batch_size;
    int sms;

    uint64_t cap = 0;
    int nk = 1;  // number of key columns (2..4 = multi-key table: d_tags / d_mk / d_mkmask instead of d_keys)
    DevBuf d_tags, d_mk[MAX_KEYS], d_mkmask;
    DevBuf d_out_mk[MAX_KEYS], d_out_mk_valid[MAX_KEYS];
    DevBuf d_keys;
    std::vector<DevBuf> d_a0, d_a1;
    DevBuf d_counters;
    long long* h_counters = nullptr;  // pinned
    PooledBuf d_fail;
    int64_t n_groups = 0;

    // host-input staging (double buffered, per used column)
    std::vector<DevBuf> stage[2];
    cudaEvent_t stage_free[2] = {nullptr, nullptr}, stage_ready[2] = {nullptr, nullptr};

    // finalize / output
    bool finalized = false;
    int64_t n_out = 0, out_cursor = 0;
    DevBuf d_slot_of_out, d_out_keys, d_out_key_valid;
    std::vector<DevBuf> d_out_data, d_out_valid;
    // host-side time accounting (printed at delete when B200_TRACE is set)
    double t_ctor = 0, t_grow = 0, t_alloc = 0, t_spg = 0, t_finalize = 0;
    static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
    struct ScopedTimer { double& t; double t0 = now(); ~ScopedTimer() { t += now() - t0; } };  // adds its scope's time to t
    // metrics
    int64_t rows_consumed = 0, rebuilds = 0, launches = 0, fail_rows = 0;
    bool build_done = false;
    // optional per-launch timing of the consume kernel (bench.py roofline): CUDA events on `stream`
    bool profiling = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
    int64_t consume_launches = 0;
    double consume_kernel_us() {
        double us = 0;
        for (auto& pr : prof_events) {
            float ms = 0;
            if (cudaEventSynchronize(pr.second) == cudaSuccess && cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) us += ms * 1000.0;
        }
        return us;
    }
    using ProfEvents = std::pair<cudaEvent_t, cudaEvent_t>;
    ProfEvents prof_begin(bool on) {  // (nullptr, nullptr) unless `on`
        ProfEvents ev{nullptr, nullptr};
        if (!on) return ev;
        B200_CUDA(cudaEventCreate(&ev.first)); B200_CUDA(cudaEventCreate(&ev.second));
        B200_CUDA(cudaEventRecord(ev.first, stream));
        return ev;
    }
    void prof_end(ProfEvents ev) {
        if (!ev.first) return;
        B200_CUDA(cudaEventRecord(ev.second, stream));
        prof_events.push_back(ev);
    }

    GroupbyState(const int8_t* ct, const int8_t* at, int n_arrs, const int32_t* ftypes, const int32_t* f_in_offsets,
                 const int32_t* f_in_cols, int n_funcs_, uint64_t n_keys, int64_t out_bs, bool parallel_, bool dropna_,
                 int device_, int n_pes_, int rank_, int64_t expected_groups, cudaStream_t stream_, const MrnfSpec* mrnf = nullptr,
                 const double* fractions = nullptr)
        : device(device_), stream(stream_), n_cols(n_arrs), n_funcs(0), n_outs(n_funcs_), dropna(dropna_), parallel(parallel_),
          n_pes(n_pes_), rank(rank_), output_batch_size(out_bs) {
        B200_REQUIRE(n_keys >= 1 && n_keys <= (uint64_t)MAX_KEYS, "b200 groupby: between 1 and 4 key columns are supported");
        nk = (int)n_keys;
        B200_REQUIRE(n_arrs >= 1, "b200 groupby: empty build schema");
        B200_REQUIRE(n_funcs_ <= 2 * MAX_OPS, "b200 groupby: too many aggregate functions");
        in_types.assign(ct, ct + n_arrs);
        c_types = in_types;
        arr_types.assign(at, at + n_arrs);
        B200_REQUIRE(n_arrs >= nk, "b200 groupby: fewer columns than keys");
        for (int kc = 0; kc < nk; kc++) {
            B200_REQUIRE(ctype_size(in_types[kc]) > 0, "b200 groupby: key columns must be integer, date or float typed");
            B200_REQUIRE(arr_types[kc] == ARR_NUMPY || arr_types[kc] == ARR_NULLABLE, "b200 groupby: unsupported key array type");
            if (ctype_is_float(in_types[kc])) c_types[kc] = CT_INT64;
        }
        if (!parallel) { n_pes = 1; rank = 0; }
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        sms = num_sms(device);
        for (int j = 0; j < n_outs; j++) {
            FuncSpec f{};
            f.ftype = ftypes[j];
            int n_in = f_in_offsets[j + 1] - f_in_offsets[j];
            B200_REQUIRE(n_in <= 1, "b200 groupby: functions with more than one input column are not supported");
            f.in_col = n_in == 1 ? f_in_cols[f_in_offsets[j]] : -1;
            if (f.ftype != FT_SIZE) B200_REQUIRE(f.in_col >= nk && f.in_col < n_arrs, "b200 groupby: bad f_in_cols entry");
            f.in_ctype = f.in_col >= 0 ? c_types[f.in_col] : CT_INT64;
            f.in_arrtype = f.in_col >= 0 ? arr_types[f.in_col] : ARR_NUMPY;
            B200_REQUIRE(f.in_arrtype == ARR_NUMPY || f.in_arrtype == ARR_NULLABLE, "b200 groupby: unsupported value array type");
            B200_REQUIRE(ctype_size(f.in_ctype) > 0, "b200 groupby: unsupported value dtype");
            bool isf = ctype_is_float(f.in_ctype);
            f.has_a1 = false;
            f.init0 = 0;
            // a refusal of the input column's type by the function `name`, which takes `takes`
            auto refuse_type = [&](bool ok, const char* name, const char* takes) {
                B200_REQUIRE(ok, std::string("b200 groupby: ") + name + " does not take a " + ctype_name(f.in_ctype) + " column (column " +
                                     std::to_string(f.in_col) + "; it takes " + takes + ")");
            };
            // output typing: get_groupby_output_dtype (groupby/_groupby_common.cpp:561-668)
            switch (f.ftype) {
                case FT_SIZE: f.kind = K_SIZE; f.out_ctype = CT_INT64; f.out_arrtype = ARR_NUMPY; break;
                case FT_COUNT: f.kind = K_COUNT; f.out_ctype = CT_INT64; f.out_arrtype = ARR_NUMPY; break;
                case FT_SUM: case FT_PROD:
                    if (f.ftype == FT_PROD) refuse_type(!ctype_is_temporal(f.in_ctype), "prod", "integer, bool and float columns");
                    f.kind = f.ftype == FT_SUM ? (isf ? K_SUM_F64 : K_SUM_I64) : (isf ? K_PROD_F64 : K_PROD_I64);
                    f.out_ctype = isf ? f.in_ctype : (ctype_is_signed_int(f.in_ctype) || f.in_ctype == CT_BOOL ? CT_INT64 : CT_UINT64);
                    f.out_arrtype = f.in_ctype == CT_BOOL ? ARR_NULLABLE : f.in_arrtype;
                    if (f.ftype == FT_PROD) f.init0 = isf ? 0x3FF0000000000000ull : 1ull;  // 1.0 / 1: an empty product
                    break;
                case FT_BOOLOR_AGG: case FT_BOOLAND_AGG: case FT_BOOLXOR_AGG: {
                    // nonzero is true; NA (and NaN) rows are skipped; a group without a non-NA value is NA.  boolxor counts the
                    // true values: true iff exactly one is
                    const bool band = f.ftype == FT_BOOLAND_AGG;
                    refuse_type(!ctype_is_temporal(f.in_ctype), band ? "booland_agg" : f.ftype == FT_BOOLOR_AGG ? "boolor_agg" : "boolxor_agg",
                                "bool, integer and float columns");
                    f.kind = band ? K_LAND : f.ftype == FT_BOOLOR_AGG ? K_LOR : K_COUNT_IF;
                    f.out_ctype = CT_BOOL; f.out_arrtype = ARR_NULLABLE;
                    f.has_a1 = f.in_arrtype == ARR_NULLABLE || isf;
                    f.init0 = band ? ~0ull : 0ull;
                    break;
                }
                case FT_BITOR_AGG: case FT_BITAND_AGG: case FT_BITXOR_AGG: {
                    const bool band = f.ftype == FT_BITAND_AGG;
                    refuse_type(!isf && f.in_ctype != CT_BOOL && !ctype_is_temporal(f.in_ctype),
                                band ? "bitand_agg" : f.ftype == FT_BITOR_AGG ? "bitor_agg" : "bitxor_agg", "integer columns");
                    f.kind = band ? K_AND : f.ftype == FT_BITOR_AGG ? K_OR : K_XOR;
                    f.out_ctype = f.in_ctype; f.out_arrtype = ARR_NULLABLE;
                    f.has_a1 = f.in_arrtype == ARR_NULLABLE;
                    f.init0 = band ? ~0ull : 0ull;
                    break;
                }
                case FT_COUNT_IF:
                    refuse_type(f.in_ctype == CT_BOOL, "count_if", "bool columns");
                    f.kind = K_COUNT_IF; f.out_ctype = CT_INT64; f.out_arrtype = ARR_NUMPY;
                    break;
                case FT_MEAN: f.kind = K_MEAN; f.out_ctype = CT_FLOAT64; f.out_arrtype = ARR_NULLABLE; f.has_a1 = true; break;
                case FT_MIN: case FT_MAX: {
                    B200_REQUIRE(f.in_ctype != CT_UINT64, "b200 groupby: min/max of uint64 is not supported");
                    bool mn = f.ftype == FT_MIN;
                    f.kind = isf ? (mn ? K_MIN_F64 : K_MAX_F64) : (mn ? K_MIN_I64 : K_MAX_I64);
                    f.out_ctype = f.in_ctype; f.out_arrtype = f.in_arrtype;
                    f.has_a1 = f.in_arrtype == ARR_NULLABLE;
                    if (isf) f.init0 = mn ? ~0ull : 0ull;
                    else f.init0 = mn ? (unsigned long long)INT64_MAX : (unsigned long long)INT64_MIN;
                    break;
                }
                case FT_NUNIQUE: {
                    // nunique_computation (bodo/libs/groupby/_groupby_col_set.cpp:1771-1810): distinct non-NA values per group
                    B200_REQUIRE(nk == 1, "b200 groupby: nunique is supported for single-column keys");
                    f.kind = K_NUNIQUE; f.out_ctype = CT_INT64; f.out_arrtype = ARR_NUMPY;
                    size_t q = 0;
                    while (q < nu_inner.size() && nu_inner[q].in_col != f.in_col) q++;
                    if (q == nu_inner.size()) { nu_inner.emplace_back(); nu_inner[q].in_col = f.in_col; }
                    nu_inner[q].prims.push_back((int)funcs.size());
                    break;
                }
                case FT_FIRST: case FT_LAST:
                    B200_REQUIRE(nk == 1, "b200 groupby: first / last are supported for single-column keys");
                    f.kind = f.ftype == FT_FIRST ? K_FIRST : K_LAST;
                    f.out_ctype = f.in_ctype; f.out_arrtype = f.in_arrtype;
                    f.has_a1 = true; f.init1 = f.ftype == FT_FIRST ? ~0ull : 0ull;
                    has_firstlast = true;
                    break;
                case FT_VAR: case FT_STD: case FT_VAR_POP: case FT_STD_POP: case FT_SKEW: case FT_KURTOSIS: {
                    // composite: the moment group of its input column (K_SHIFT, K_MOM1, K_MOM2 (, K_MOM3 when some skew or kurtosis
                    // reads the column (, K_MOM4 when some kurtosis does))), shared by every composite over that column
                    OutSpec o{};
                    o.ftype = f.ftype;
                    o.kind = f.ftype == FT_VAR ? E_VAR : f.ftype == FT_STD ? E_STD : f.ftype == FT_VAR_POP ? E_VAR_POP : f.ftype == FT_STD_POP ? E_STD_POP
                           : f.ftype == FT_SKEW ? E_SKEW : E_KURT;
                    o.out_ctype = CT_FLOAT64; o.out_arrtype = ARR_NULLABLE;
                    int g = 0;
                    while (g < (int)funcs.size() && !(funcs[g].kind == K_SHIFT && funcs[g].in_col == f.in_col)) g++;
                    if (g == (int)funcs.size()) {
                        bool skew = false, kurt = false;
                        for (int q = 0; q < n_outs; q++) {
                            if (f_in_offsets[q + 1] == f_in_offsets[q] || f_in_cols[f_in_offsets[q]] != f.in_col) continue;
                            skew |= ftypes[q] == FT_SKEW;
                            kurt |= ftypes[q] == FT_KURTOSIS;
                        }
                        const int kinds[5] = {K_SHIFT, K_MOM1, K_MOM2, K_MOM3, K_MOM4};
                        for (int q = 0; q < (kurt ? 5 : skew ? 4 : 3); q++) {
                            FuncSpec pf = f;
                            pf.kind = kinds[q]; pf.has_a1 = kinds[q] == K_MOM1; pf.out_ctype = CT_FLOAT64; pf.out_arrtype = ARR_NULLABLE;
                            pf.init0 = kinds[q] == K_SHIFT ? SHIFT_UNSET : 0ull;
                            funcs.push_back(pf);
                        }
                    }
                    o.n_prim = f.ftype == FT_KURTOSIS ? 4 : f.ftype == FT_SKEW ? 3 : 2;
                    for (int q = 0; q < o.n_prim; q++) o.prim[q] = g + 1 + q;  // eval reads K_MOM1 (sum, count), K_MOM2 (, K_MOM3 (, K_MOM4))
                    outs.push_back(o);
                    continue;
                }
                case FT_MODE: case FT_PERCENTILE_CONT: case FT_PERCENTILE_DISC: {
                    // holistic: one store per value column; the result word is added after the loop (see Holistic)
                    const bool cont = f.ftype == FT_PERCENTILE_CONT, disc = f.ftype == FT_PERCENTILE_DISC;
                    B200_REQUIRE(n_in == 1, "b200 groupby: mode / percentile_cont / percentile_disc take one input column");
                    if (cont) refuse_type(f.in_ctype != CT_BOOL && !ctype_is_temporal(f.in_ctype), "percentile_cont", "integer and float columns");
                    if (disc) refuse_type(f.in_ctype != CT_BOOL, "percentile_disc", "integer, float, date, datetime and timedelta columns");
                    double q = 0.0;
                    if (cont || disc) {
                        B200_REQUIRE(fractions != nullptr, "b200 groupby: percentile_cont / percentile_disc need a fraction (b200_groupby_state_init_percentiles)");
                        q = fractions[j];
                        B200_REQUIRE(q >= 0.0 && q <= 1.0, "b200 groupby: the fraction of percentile_cont / percentile_disc (function " + std::to_string(j) +
                                                               ") must lie in [0, 1]");
                    }
                    size_t si = 0;
                    while (si < ho.st.size() && ho.st[si].in_col != f.in_col) si++;
                    if (si == ho.st.size()) { ho.st.emplace_back(); ho.st[si].in_col = f.in_col; }
                    ho.on = true;
                    ho.outs.push_back(HoOut{(int)outs.size(), (int)si, cont ? E_PCONT : disc ? E_PDISC : E_MODE, q});
                    OutSpec o{};
                    o.ftype = f.ftype; o.kind = K_FIRST; o.n_prim = 1;  // (prim[0]: the result word, set after the loop)
                    o.out_ctype = cont ? CT_FLOAT64 : f.in_ctype; o.out_arrtype = ARR_NULLABLE;
                    outs.push_back(o);
                    continue;
                }
                default:
                    throw Error("b200 groupby: unsupported aggregate function ftype=" + std::to_string(f.ftype) +
                                " (supported: size, sum, count, nunique, mean, min, max, prod, first, last, var, std, var_pop, std_pop, "
                                "kurtosis, skew, boolor_agg, booland_agg, boolxor_agg, bitor_agg, bitand_agg, bitxor_agg, count_if, mode, "
                                "percentile_cont, percentile_disc)");
            }
            OutSpec o{};
            o.ftype = f.ftype; o.kind = f.ftype == FT_BOOLXOR_AGG ? E_BOOLXOR : f.kind; o.prim[0] = (int)funcs.size(); o.n_prim = 1; o.out_ctype = f.out_ctype; o.out_arrtype = f.out_arrtype;
            outs.push_back(o);
            funcs.push_back(f);
        }
        if (mrnf) setup_mrnf(*mrnf);
        if (ho.on) setup_holistic();
        n_funcs = (int)funcs.size();
        B200_REQUIRE(mr.on || n_funcs <= MAX_OPS, "b200 groupby: too many aggregate functions (composite ones count their accumulator columns)");
        d_a0.resize(n_funcs); d_a1.resize(n_funcs);
        d_out_data.resize(n_outs); d_out_valid.resize(n_outs);
        d_counters.alloc(N_COUNTERS * sizeof(long long));
        B200_CUDA(cudaMemsetAsync(d_counters.p, 0, N_COUNTERS * sizeof(long long), stream));
        h_counters = (long long*)pinned_acquire(N_COUNTERS * sizeof(long long));
        expected_groups_hint = expected_groups > 0 ? expected_groups : 0;
        uint64_t want = 1ull << 16;
        if (expected_groups > 0) { while (want < (uint64_t)expected_groups * 2) want <<= 1; }
        else want = 1ull << 21;
        double t0 = now();
        alloc_table(want, d_keys, d_a0, d_a1);
        if (nk > 1) alloc_mk(want, d_tags, d_mk, d_mkmask);
        cap = want;
        for (auto& ni : nu_inner) {  // nested distinct states over (key, value); their groups are owned where the KEY is owned
            const int8_t ict[2] = {in_types[0], in_types[ni.in_col]}, iat[2] = {arr_types[0], arr_types[ni.in_col]};
            const int32_t no_off[1] = {0};
            ni.st.reset(new GroupbyState(ict, iat, 2, nullptr, no_off, nullptr, 0, 2, 1ll << 40, parallel, /*dropna=*/false, device, n_pes, rank,
                                         expected_groups > 0 ? expected_groups * 4 : 0, stream));
            ni.st->owner_nk = 1;
        }
        t_ctor = now() - t0;
    }

    ~GroupbyState() {
        cudaSetDevice(device);
        scratch_set_stream(stream);
        cudaStreamSynchronize(stream);
        if (getenv("B200_TRACE"))
            fprintf(stderr, "[b200 groupby state] ctor %.3f ms, grow %.3f ms (%lld rebuilds), spg alloc %.3f ms, spg loop %.3f ms, finalize %.3f ms, cap %llu\n",
                    t_ctor * 1e3, t_grow * 1e3, (long long)rebuilds, t_alloc * 1e3, t_spg * 1e3, t_finalize * 1e3, (unsigned long long)cap);
        if (copy_stream) { cudaStreamSynchronize(copy_stream); cudaStreamDestroy(copy_stream); }
        for (int b = 0; b < 2; b++) { if (stage_free[b]) cudaEventDestroy(stage_free[b]); if (stage_ready[b]) cudaEventDestroy(stage_ready[b]); }
        pinned_release(h_counters, N_COUNTERS * sizeof(long long));
        if (mt.h_ctr) pinned_release(mt.h_ctr, 16);
        pinned_release(h_spg, H_SPG_WORDS * sizeof(long long));
        for (int b = 0; b < 2; b++) if (spg_ev[b]) cudaEventDestroy(spg_ev[b]);
        for (auto& pr : prof_events) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    }

    int grid_for(int64_t n, int per_thread = 1, int block = 256) const {
        int64_t want = (n + (int64_t)block * per_thread - 1) / ((int64_t)block * per_thread);
        int64_t maxg = (int64_t)sms * 8;  // 8 resident CTAs of 256 threads per SM
        return (int)std::max<int64_t>(1, std::min(want, maxg));
    }

    void fill(void* p, uint64_t n, unsigned long long v) {
        if (v == 0) { B200_CUDA(cudaMemsetAsync(p, 0, n * 8, stream)); return; }
        launch_fill_u64(p, n, v, grid_for((int64_t)n), stream);
        launches++;
    }

    void alloc_table(uint64_t c, DevBuf& keys, std::vector<DevBuf>& a0, std::vector<DevBuf>& a1) {
        B200_REQUIRE(c <= (1ull << 32), "b200 groupby: hash table would exceed 2^32 slots");
        if (nk == 1) {
            keys.alloc((c + 2) * 8);
            fill(keys.p, c + 2, (unsigned long long)EMPTY_KEY);
        }
        for (int j = 0; j < n_funcs; j++) {
            a0[j].alloc((c + 2) * 8);
            fill(a0[j].p, c + 2, funcs[j].init0);
            if (funcs[j].has_a1) { a1[j].alloc((c + 2) * 8); fill(a1[j].p, c + 2, funcs[j].init1); }
        }
    }

    void read_counters() {
        B200_CUDA(cudaMemcpyAsync(h_counters, d_counters.p, N_COUNTERS * sizeof(long long), cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        n_groups = h_counters[CTR_GROUPS];
    }

    // the accumulator columns in wire order (per function a0, then a1 if it has one) into `out`; returns their number, acc_count()
    template <typename P>
    int wire_accs(const std::vector<DevBuf>& a0, const std::vector<DevBuf>& a1, P* out) const {
        int n = 0;
        for (int j = 0; j < n_funcs; j++) {
            out[n++] = a0[j].as<unsigned long long>();
            if (funcs[j].has_a1) out[n++] = a1[j].as<unsigned long long>();
        }
        return n;
    }

    // next power of two >= 2 x (groups + pending rows + headroom), and at least double
    void grow_to_fit(int64_t pending, int64_t headroom = 0) {
        uint64_t nc = cap;
        while (nc < 2ull * (uint64_t)(n_groups + pending + headroom)) nc <<= 1;
        if (nc == cap) nc <<= 1;
        grow(nc);
    }

    void grow(uint64_t new_cap) {
        ScopedTimer timer{t_grow};
        if (nk > 1) { grow_mk(new_cap); return; }
        DevBuf nkeys; std::vector<DevBuf> na0(n_funcs), na1(n_funcs);
        alloc_table(new_cap, nkeys, na0, na1);
        RehashArgs ra{};
        ra.old_keys = d_keys.as<long long>(); ra.old_cap = cap; ra.new_keys = nkeys.as<long long>(); ra.new_cap = new_cap;
        ra.n_acc = wire_accs(d_a0, d_a1, ra.old_acc);
        wire_accs(na0, na1, ra.new_acc);
        rehash_kernel<<<grid_for((int64_t)cap + 2), 256, 0, stream>>>(ra);
        launches++;
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(stream));  // old arrays are freed below
        d_keys = std::move(nkeys);
        for (int j = 0; j < n_funcs; j++) { d_a0[j] = std::move(na0[j]); d_a1[j] = std::move(na1[j]); }
        cap = new_cap;
        rebuilds++;
    }

    // ---- multi-key table management ----
    void alloc_mk(uint64_t c, DevBuf& tags, DevBuf* mk, DevBuf& mask) {
        tags.alloc(c * 8);
        B200_CUDA(cudaMemsetAsync(tags.p, 0, c * 8, stream));
        for (int j = 0; j < nk; j++) mk[j].alloc(c * 8);
        mask.alloc(c);
    }
    void grow_mk(uint64_t new_cap) {
        DevBuf ntags, nmk[MAX_KEYS], nmask, dummy;
        std::vector<DevBuf> na0(n_funcs), na1(n_funcs);
        alloc_table(new_cap, dummy, na0, na1);
        alloc_mk(new_cap, ntags, nmk, nmask);
        RehashMkArgs ra{};
        ra.nk = nk; ra.old_tags = d_tags.as<unsigned long long>(); ra.old_mask = d_mkmask.as<unsigned char>(); ra.old_cap = cap;
        ra.tags = ntags.as<unsigned long long>(); ra.mkmask = nmask.as<unsigned char>(); ra.cap = new_cap;
        ra.counters = d_counters.as<long long>(); ra.group_limit = -1;
        for (int j = 0; j < nk; j++) { ra.old_mk[j] = d_mk[j].as<long long>(); ra.mk[j] = nmk[j].as<long long>(); }
        ra.n_acc = wire_accs(d_a0, d_a1, ra.old_acc);
        wire_accs(na0, na1, ra.new_acc);
        rehash_mk_kernel<<<grid_for((int64_t)cap), 256, 0, stream>>>(ra);
        launches++;
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(stream));
        d_tags = std::move(ntags); d_mkmask = std::move(nmask);
        for (int j = 0; j < nk; j++) d_mk[j] = std::move(nmk[j]);
        for (int j = 0; j < n_funcs; j++) { d_a0[j] = std::move(na0[j]); d_a1[j] = std::move(na1[j]); }
        cap = new_cap;
        rebuilds++;
    }
    void consume_mk(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n) {
        bool could_fail = (int64_t)(cap / 2) - n_groups_bound < n;
        if (could_fail) d_fail.ensure(device, (size_t)n * 4);
        auto launch = [&](const uint32_t* index_list, int64_t rows) {
            MkArgs a = mk_table_args();
            a.dropna = dropna ? 1 : 0; a.n_rows = rows; a.index_list = index_list;
            for (int j = 0; j < nk; j++) { a.key_data[j] = data[j]; a.key_valid[j] = valid[j]; a.key_ctype[j] = c_types[j]; }
            a.n_ops = n_apply();
            fill_ops(a.ops, data, valid);
            if (has_reduction_kinds(a)) groupby_consume_mk_kernel<true><<<grid_for(rows), 256, prod_smem_bytes(a), stream>>>(a);
            else groupby_consume_mk_kernel<false><<<grid_for(rows), 256, 0, stream>>>(a);
            launches++; consume_launches += index_list == nullptr;
            B200_CUDA(cudaGetLastError());
        };
        launch(nullptr, n);
        if (could_fail) settle<uint32_t>(d_fail, 1, fail_rows, launch);
        if (!could_fail) n_groups_bound += n; else n_groups_bound = n_groups;
        rows_consumed += n;
    }

    // After a launch that may have failed rows: grow + replay until every row is in.  `list` holds counters[CTR_FAIL] entries
    // of `words` T each (row indices, or rows of a wire format); `replayed` counts them.  The replay reads a copy of the list:
    // it appends the entries that fail again to `list` itself.  The grown table has room for every pending entry.
    template <typename T, typename Replay>
    void settle(const DevBuf& list, size_t words, int64_t& replayed, Replay replay) {
        for (read_counters(); h_counters[CTR_FAIL] > 0; read_counters()) {
            B200_REQUIRE(h_counters[CTR_RETRY_OVERFLOW] == 0, "SM-partitioned groupby: a retry list overflowed its buffer (internal sizing error)");
            const int64_t nf = h_counters[CTR_FAIL];
            replayed += nf;
            grow_to_fit(nf);
            DevBuf replay_list;
            replay_list.alloc((size_t)nf * words * sizeof(T));
            B200_CUDA(cudaMemcpyAsync(replay_list.p, list.p, (size_t)nf * words * sizeof(T), cudaMemcpyDeviceToDevice, stream));
            B200_CUDA(cudaMemsetAsync((char*)d_counters.p + CTR_FAIL * 8, 0, 8, stream));
            replay(replay_list.as<T>(), nf);
        }
    }

    // ---- SM-partitioned fast path (SPG) ----
    static constexpr int64_t SPG_LAUNCH_ROWS = 1ll << 27;
    PooledBuf d_bucket;
    DevBuf d_bucket_cnt;
    int spg_owners = 0, spg_ns = 0;
    size_t spg_smem = 0;
    int spg_state = -1;  // -1 not probed, 0 unavailable/disabled, 1 ready
    int64_t spg_launches = 0, spg_retry_rows = 0, lc_launches = 0;
    int64_t expected_groups_hint = 0;

    bool spg_probe() {
        if (spg_state >= 0) return spg_state == 1;
        spg_state = 0;
        const char* env = getenv("B200_SPG");
        if (env && env[0] == '0') return false;
        int max_smem = 0;
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        if (sms > SPG_MAX_OWNERS - 1 || max_smem < 64 * 1024) return false;
        spg_ns = ((int)(((size_t)max_smem - 64) / 16) - SPG_STASH) & ~1;
        spg_smem = (size_t)(spg_ns + SPG_STASH) * 16 + 16;
        // K1 / K1-hot / K2 and the big LC kernel: SPG is off when one of them cannot get its shared memory
        bool ok = true;
        for_each_sum_cnt([&](auto s, auto c) {
            ok = ok && set_smem_limit((const void*)spg_aggregate_kernel<s, c>, spg_smem)
                    && set_smem_limit((const void*)spg_partition_tma_kernel<s, c>, SpgK1Smem<false>::bytes)
                    && set_smem_limit((const void*)spg_partition_tma_kernel<s, c, true>, SpgK1Smem<true>::bytes)
                    && set_smem_limit((const void*)groupby_lowcard_kernel<s, c, LC_SLOTS_BIG, 2>, (size_t)LC_SLOTS_BIG * 20 + 64);
        });
        if (!ok) return false;
        {   // SPG-N (spgn.cuh): narrow bucket rows
            spgn_ns = ((int)(((size_t)max_smem - 256 - SPGN_QUEUE_BYTES) / 12) - SPG_STASH) & ~1;  // (K2n also has a few static shared words)
            spgn_smem = (size_t)(spgn_ns + SPG_STASH) * 12 + SPGN_QUEUE_BYTES + 16;
            spgn_enabled = true;
            spgd_max_smem = (size_t)max_smem - 256;  // (K2d's flush has a few static shared words)
            for_each_sum_cnt([&](auto s, auto c) {
                if (!set_smem_limit((const void*)spgn_partition_kernel<s, c>, SpgnK1Smem<false>::bytes)) spgn_enabled = false;
                if (!set_smem_limit((const void*)spgn_aggregate_kernel<s, c>, spgn_smem)) spgn_enabled = false;
                if (!set_smem_limit((const void*)spgn_partition_kernel<s, c, true>, SpgnK1Smem<true>::bytes)) spgd_max_smem = 0;
                if (!set_smem_limit((const void*)spgn_aggregate_kernel<s, c, true>, spgd_max_smem)) spgd_max_smem = 0;
            });
            const char* e8 = getenv("B200_SPG_NARROW");
            if (e8 && e8[0] == '0') spgn_enabled = false;
            const char* e9 = getenv("B200_SPG_DENSE");
            if ((e9 && e9[0] == '0') || !spgn_enabled || sms < 2) spgd_max_smem = 0;  // (the slot division needs >= 2 owners)
        }
        {   // SPG-G (spgg.cuh): generic signatures
            spgg_enabled = 2 * sms <= GEN_CLS;  // classes of K1g's counting sort: at least owners + owners
            for_each_spgg_part([&](auto ks, auto vs) {
                if (!set_smem_limit((const void*)spgg_partition_kernel<ks, vs>, SpggK1Smem::bytes)) spgg_enabled = false;
            });
            for (int v = 0; v < 4; v++) {  // v = mm + 2 * nn
                const int sb = 16 + ((v & 1) ? 16 : 0) + ((v & 2) ? 4 : 0);
                spgg_ns[v] = ((int)(((size_t)max_smem - 64) / sb) - SPG_STASH) & ~1;
                spgg_smem[v] = (size_t)(spgg_ns[v] + SPG_STASH) * sb + 16;
            }
            for_each_spgg_agg([&](auto s, auto mm, auto nn) {
                if (!set_smem_limit((const void*)spgg_aggregate_kernel<s, mm, nn>, spgg_smem[mm + 2 * nn])) spgg_enabled = false;
            });
            const char* e7 = getenv("B200_SPG_GEN");
            if (e7 && e7[0] == '0') spgg_enabled = false;
        }
        if (!set_smem_limit((const void*)spg_hot_sample_kernel, SPG_HOT_SAMPLE_SMEM)) return false;
        { const char* e4 = getenv("B200_SPG_HOT"); spg_hot_enabled = !(e4 && e4[0] == '0'); }
        d_hot.alloc((size_t)SPG_HOT_SLOTS * 8 + 48);
        { const char* e3 = getenv("B200_LC"); lc_enabled = !(e3 && e3[0] == '0'); }
        spg_owners = sms;  // one owner (bucket + shared table) per SM
        // SPG-G: one counter per class of K1g.  consume_spg_gen clears n_vo + owners counters, and n_vo (owners x passes) may
        // fill all GEN_CLS classes when the value column has no bitmap (e.g. 3 passes x 132 owners on an H100)
        d_bucket_cnt.alloc((size_t)(GEN_CLS + spg_owners) * SPG_CNT_STRIDE * 8);
        spg_state = 1;
        return true;
    }

    bool lc_enabled = true, lowcard_small = false;
    // SPG-N: narrow bucket rows (spgn.cuh)
    int spgn_ns = 0;
    size_t spgn_smem = 0;
    bool spgn_enabled = false;
    int spg_sample_wide = -1;  // sampled rows of the first launch that do NOT fit (int32 key, int32 value); -1 = not sampled
    int64_t spgn_launches = 0, spg16_launches = 0;  // launches of the narrow-row pair (either form), of the 16-byte pair
    // SPG-N dense form (spgn.cuh): chosen once per state from the sample's key and value range
    size_t spgd_max_smem = 0;  // shared memory K2d may use; 0 = the dense form is off (B200_SPG_DENSE=0 or unavailable)
    bool spgd_ok = false;      // the sample fits a dense window: the fields below hold it
    long long spgd_kbase = 0, spgd_vbase = 0;
    unsigned int spgd_kb = 0, spgd_vb = 0;
    int spgd_slots = 0;
    int64_t spgd_wide_rows = 0, spgd_launches = 0;  // rows outside the window so far (counters[CTR_DENSE_WIDE]); dense pairs
    static constexpr unsigned int SPGD_MUL = 0x9E3779B1u;  // odd: the key scramble's multiplier
    static unsigned int odd_inverse(unsigned int m) {       // m^-1 mod 2^32 (Newton: each step doubles the correct low bits)
        unsigned int x = m;                                  // correct to 3 bits for any odd m
        for (int i = 0; i < 4; i++) x *= 2u - m * x;
        return x;
    }
    // The dense window for sampled keys in [kmin, kmax] and values in [vmin, vmax] (DESIGN §3): 1/32 of the key range of head
    // room below and above (none below when the keys start near 0), a power-of-two window of at most 2^21 keys whose K2d table
    // fits the shared memory, and a value window of the bits the slot leaves, centred on the sampled values.
    void spgd_plan(long long kmin, long long kmax, long long vmin, long long vmax, bool has_vals) {
        spgd_ok = false;
        if (spgd_max_smem == 0 || kmin > kmax) return;
        const uint64_t range = (uint64_t)kmax - (uint64_t)kmin;
        if (range >= (1ull << 21)) return;
        const uint64_t pad = range / 32;
        long long kbase;
        if (kmin >= 0 && (uint64_t)kmin <= pad) kbase = 0;
        else if (kmin < LLONG_MIN + (long long)pad + 1) return;  // (the window must not hold EMPTY_KEY, the marker key)
        else kbase = kmin - (long long)pad;
        const uint64_t span = (uint64_t)kmax - (uint64_t)kbase + 1, need = span + span / 32;
        unsigned int kb = 1;
        while ((1ull << kb) < need) kb++;
        if (kb > 21 || kbase > LLONG_MAX - (long long)((1ull << kb) - 1)) return;  // (nor wrap past INT64_MAX)
        const uint64_t slots = ((1ull << kb) + spg_owners - 1) / spg_owners;
        if (slots * 8 > spgd_max_smem) return;
        unsigned int sb = 0;
        while ((1ull << sb) < slots) sb++;
        const unsigned int vb = std::min(32u - sb, 31u);
        long long vbase = 0;
        if (has_vals) {
            const uint64_t vspan = (uint64_t)vmax - (uint64_t)vmin + 1;  // (0 when the sample spans all of int64)
            if (vspan == 0 || vspan > (1ull << vb)) return;
            vbase = (long long)((uint64_t)vmin - ((1ull << vb) - vspan) / 2);
        }
        spgd_ok = true;
        spgd_kbase = kbase; spgd_vbase = vbase; spgd_kb = kb; spgd_vb = vb; spgd_slots = (int)slots;
    }
    int64_t spgn_group_capacity() const { return (int64_t)spg_owners * (spgn_ns * 7 / 10); }
    int spgg_ns[4] = {0, 0, 0, 0};  // K2g table slots, by slot layout v = (min/max fields) + 2 * (NA-value counter)
    size_t spgg_smem[4] = {0, 0, 0, 0};
    bool spgg_enabled = true;      // B200_SPG_GEN=0 disables the generic SM-partitioned path
    int64_t spgg_launches = 0;
    int spg_n_hot = 0;
    bool spg_hot_enabled = true, spg_hot_sampled = false;  // heavy-hitter table: sampled once per state, at its first SPG launch
    DevBuf d_hot;                                           // [SPG_HOT_SLOTS] keys + n_hot (int)
    int spg_passes = 1;
    static constexpr int SPG_MAX_PASSES = 24;
    // K2 passes needed for `est` groups (each pass holds spg_group_capacity() groups); 0 = too many for the SPG path
    int spg_pass_count(int64_t est) const {
        int64_t p = (est + spg_group_capacity() - 1) / spg_group_capacity();
        return p <= 1 ? 1 : (p <= SPG_MAX_PASSES ? (int)p : 0);
    }
    bool lc_pick(int64_t est) { lowcard_small = est <= LC_SLOTS_SMALL / 4; return lc_enabled && est <= LC_SLOTS_BIG / 4; }
    // groups the shared-memory tables of all owners are expected to hold together (two-choice buckets work well up to ~70 %)
    int64_t spg_group_capacity() const { return (int64_t)spg_owners * (spg_ns * 7 / 10); }

    // One SPG launch pair in flight while the host inspects the previous one (two retry lists / counter slots), so
    // the GPU never idles on the host's counter read-back.
    PooledBuf d_retry2[2];
    static constexpr int H_SPG_WORDS = 2 * N_COUNTERS + 5;
    long long* h_spg = nullptr;  // pinned: [slot][N_COUNTERS] counter snapshots, then the two ints of the sample verdict and its key / value range
    cudaEvent_t spg_ev[2] = {nullptr, nullptr};

    int64_t spgn_wide_rows = 0;  // rows that did not fit the narrow format so far (counters[CTR_WIDE])
    static int spg_retry_slot(int slot) { return slot == 0 ? CTR_FAIL : CTR_RETRY1; }  // counter of launch slot `slot`'s retry list
    void spg_finish(int slot, int sum_j, int cnt_j) {
        B200_CUDA(cudaEventSynchronize(spg_ev[slot]));
        const long long* hc = h_spg + slot * N_COUNTERS;
        n_groups = hc[CTR_GROUPS];
        spgn_wide_rows = hc[CTR_WIDE];
        spgd_wide_rows = hc[CTR_DENSE_WIDE];
        const int64_t nr = hc[spg_retry_slot(slot)];  // retry rows of that launch
        if (nr == 0) return;
        // rows / partials that found the global table full: grow, then merge them like received partial rows
        spg_retry_rows += nr;
        B200_CUDA(cudaStreamSynchronize(stream));  // the other in-flight launch uses the table we are about to replace
        read_counters();
        // (the flag is shared by both slots: a list that overflowed has entries, so its own or the other slot's call gets here)
        B200_REQUIRE(h_counters[CTR_RETRY_OVERFLOW] == 0, "SM-partitioned groupby: a retry list overflowed its buffer (internal sizing error)");
        const int64_t pending = h_counters[CTR_FAIL] + h_counters[CTR_RETRY1];
        // the snapshot this call was made on may be stale: the other slot's spg_finish already grew the table and merged
        // BOTH retry lists (their live counters are 0 then) — nothing left to do, and no second grow
        if (pending == 0) return;
        grow_to_fit(pending, (int64_t)spg_owners * spg_ns);
        for (int sl = 0; sl < 2; sl++) {
            int64_t cnt = h_counters[spg_retry_slot(sl)];
            if (cnt == 0) continue;
            B200_CUDA(cudaMemsetAsync((char*)d_counters.p + spg_retry_slot(sl) * 8, 0, 8, stream));
            CombineArgs c{};
            c.src = host_source(d_retry2[sl].p, &cnt, 1); c.row_words = 4;
            d_fail.ensure(device, (size_t)cnt * 4);
            c.fail_list = d_fail.as<uint32_t>(); c.n_ops = 0;  // cannot fail: the table was grown for all pending rows
            // wire order = function order of the (at most two) accumulators
            int order[2] = {sum_j, cnt_j};
            if (sum_j >= 0 && cnt_j >= 0 && cnt_j < sum_j) std::swap(order[0], order[1]);
            if (order[0] < 0) std::swap(order[0], order[1]);
            for (int q = 0; q < 2; q++) if (order[q] >= 0) { c.kinds[c.n_ops] = K_SUM_I64; c.a0[c.n_ops] = d_a0[order[q]].p; c.a1[c.n_ops] = nullptr; c.n_ops++; }
            xchg_combine_kernel<<<grid_for(cnt), 256, 0, stream>>>(slot_table(), c);
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        read_counters();
    }

    void consume_spg(const long long* keys, const long long* vals, int64_t n, int sum_j, int cnt_j, bool lowcard = false, int64_t est_groups = 0) {
        // K1 and K1n fetch their tiles with TMA bulk copies and LC reads row pairs with 16-byte loads: all need aligned columns
        B200_REQUIRE(((uintptr_t)keys & 15) == 0 && ((uintptr_t)vals & 15) == 0, "SM-partitioned groupby: key and value columns must be 16-byte aligned");
        if (!h_spg) {
            h_spg = (long long*)pinned_acquire(H_SPG_WORDS * sizeof(long long));  // [slot][N_COUNTERS] counter snapshots + n_hot read-back
            for (int b = 0; b < 2; b++) B200_CUDA(cudaEventCreateWithFlags(&spg_ev[b], cudaEventDisableTiming));
        }
        ScopedTimer timer{t_spg};
        read_counters();  // exact group count before the first launch
        n_groups_bound = n_groups;
        if (!lowcard && !spg_hot_sampled) {
            // once per state: count a sample of this call's keys (heavy hitters) and test the sampled rows against the narrow-row
            // format; the host reads back both verdicts
            int* d_nhot = (int*)(d_hot.as<long long>() + SPG_HOT_SLOTS);
            spg_hot_sample_kernel<<<1, 1024, SPG_HOT_SAMPLE_SMEM, stream>>>(keys, vals, n, d_hot.as<long long>(), d_nhot, d_hot.as<long long>() + SPG_HOT_SLOTS + 1);
            B200_CUDA(cudaMemcpyAsync(h_spg + 2 * N_COUNTERS, d_nhot, 5 * sizeof(long long), cudaMemcpyDeviceToHost, stream));
            B200_CUDA(cudaStreamSynchronize(stream));
            spg_n_hot = spg_hot_enabled ? ((int*)(h_spg + 2 * N_COUNTERS))[0] : 0;
            spg_sample_wide = ((int*)(h_spg + 2 * N_COUNTERS))[1];
            const long long* rng = h_spg + 2 * N_COUNTERS + 1;
            spgd_plan(rng[0], rng[1], rng[2], rng[3], vals != nullptr);
            spg_hot_sampled = true;
            launches++;
        }
        // SPG-N: no heavy hitters, and the sample found only rows that fit (int32 key, int32 value) — for either form: keys far
        // beyond int32 (2^40 + id) keep the 16-byte pair, whose rare paths tests/test_gpu_spg_row_path.py exercises with them
        const bool narrow_sig = spgn_enabled && !lowcard && spg_n_hot == 0 && spg_sample_wide == 0;
        // narrow bucket rows are half the bytes: twice the rows per launch for the same scratch, half the per-launch flushes
        const int64_t launch_rows = narrow_sig ? 2 * SPG_LAUNCH_ROWS : SPG_LAUNCH_ROWS;
        int64_t li = 0;
        for (int64_t r0 = 0; r0 < n; r0 += launch_rows, li++) {
            int slot = (int)(li & 1);
            int64_t rows = std::min(launch_rows, n - r0);
            // no pre-growing: a flush that finds the global table at its limit lands in the retry list and is merged
            // after the table grew (spg_finish), exactly like rows of the direct path
            // uniform keys put rows / owners rows in every bucket (sd = sqrt of that); 12.5 % + 4096 rows head room,
            // anything beyond (skew) takes the direct path inside K1
            const int64_t bucket_cap = (rows / spg_owners) + (rows / spg_owners) / 8 + 4096;
            const bool small = lowcard_small;
            const int gl = (int)std::min<int64_t>((int64_t)sms * (small ? 3 : 2), (rows + LC_THREADS * 2 - 1) / (LC_THREADS * 2));
            const int g2 = (int)std::min<int64_t>((int64_t)sms * SPG_TCTAS, (rows + SPG_TILE - 1) / SPG_TILE);
            const bool hot = !lowcard && spg_hot_enabled && spg_n_hot > 0;
            // SPG-N: dense when the sample found a window and the rows outside it so far are rare; else the hash form when the rows
            // that did not fit (int32 key, int32 value) so far are rare
            const bool dense = narrow_sig && spgd_ok && spgd_wide_rows * 64 <= rows_consumed;
            const bool narrow = dense || (narrow_sig && spgn_wide_rows * 64 <= rows_consumed);
            const int64_t est_n = std::max<int64_t>(est_groups, 1);
            const int n_pass = dense ? 1 : narrow ? (int)std::min<int64_t>(SPG_MAX_PASSES, std::max<int64_t>(1, (est_n + spgn_group_capacity() - 1) / spgn_group_capacity()))
                                      : spg_passes;
            // retry entries: at most one per row (K1's direct rows; in K2 a carry or a row without a slot), plus one per partial of
            // the per-CTA tables: LC's slots, or every occupied K2 slot (buckets and stash) in every pass and K1's heavy hitters
            const int64_t retry_cap = rows + (lowcard ? (int64_t)gl * (small ? LC_SLOTS_SMALL : LC_SLOTS_BIG)
                                                      : (int64_t)spg_owners * ((narrow ? spgn_ns : spg_ns) + SPG_STASH) * n_pass
                                                        + (hot ? (int64_t)g2 * SPG_HOT_SLOTS : 0));
            double ta = now();
            d_bucket.ensure(device, (size_t)spg_owners * bucket_cap * 16);  // K2 of the previous launch precedes K1 of this one in stream order
            d_retry2[slot].ensure(device, (size_t)retry_cap * 32);
            t_alloc += now() - ta;
            B200_CUDA(cudaMemsetAsync(d_bucket_cnt.p, 0, (size_t)spg_owners * SPG_CNT_STRIDE * 8, stream));
            SpgArgs a{};
            a.keys = keys + r0; a.vals = vals ? vals + r0 : nullptr; a.n_rows = rows; a.n_owners = spg_owners;
            a.tkeys = d_keys.as<long long>(); a.cap = cap;
            a.acc_sum = sum_j >= 0 ? d_a0[sum_j].as<unsigned long long>() : nullptr;
            a.acc_cnt = cnt_j >= 0 ? d_a0[cnt_j].as<unsigned long long>() : nullptr;
            a.counters = d_counters.as<long long>(); a.group_limit = (long long)(cap / 2);
            a.retry_ctr = d_counters.as<long long>() + spg_retry_slot(slot);
            a.bucket = d_bucket.as<longlong2>(); a.bucket_cnt = d_bucket_cnt.as<unsigned long long>(); a.bucket_cap = bucket_cap;
            a.retry = d_retry2[slot].as<unsigned long long>(); a.retry_cap = retry_cap;
            a.sum_first = (sum_j >= 0 && cnt_j >= 0 && sum_j < cnt_j) ? 1 : 0; a.ns = spg_ns; a.n_pass = n_pass;
            const ProfEvents prof = prof_begin(profiling);
            if (lowcard) {
                size_t lsm = (size_t)(small ? LC_SLOTS_SMALL : LC_SLOTS_BIG) * 20 + 64;
                with_sum_cnt(sum_j >= 0, cnt_j >= 0, [&](auto s, auto c) {
                    if (small) groupby_lowcard_kernel<s, c, LC_SLOTS_SMALL, 3><<<gl, LC_THREADS, lsm, stream>>>(a);
                    else groupby_lowcard_kernel<s, c, LC_SLOTS_BIG, 2><<<gl, LC_THREADS, lsm, stream>>>(a);
                });
                lc_launches++;
            } else {
                if (hot) { a.hot_tab = d_hot.as<long long>(); a.n_hot = (const int*)(d_hot.as<long long>() + SPG_HOT_SLOTS); }
                if (narrow) {
                    a.ns = spgn_ns;
                    // first flush into an empty table: per-CTA ticket reservation, but only with >= 25 % head room under the group
                    // limit — a reservation transiently over-counts (slots that hold one key twice), and a CTA that then finds the
                    // limit reached would send its groups to the retry list and make the host grow the table for nothing (seen on
                    // 8 GPUs: 1 M groups against a limit of 2^20 cost 1.4 ms per state in some runs)
                    a.reserve_tickets = (n_groups_bound == 0 && li == 0 && est_groups > 0 && est_groups + est_groups / 4 <= (int64_t)(cap / 2)) ? 1 : 0;
                    a.bucket_cap = bucket_cap & ~1ll;
                    const int gn = (int)std::min<int64_t>((int64_t)sms * SPGN_CTAS, (rows + SPGN_TILE - 1) / SPGN_TILE);
                    if (dense) {
                        a.bucket_cap = bucket_cap & ~3ll;  // 4-byte rows: every owner's bucket starts 16-byte aligned
                        SpgDenseArgs da{};
                        static_cast<SpgArgs&>(da) = a;
                        da.kbase = spgd_kbase; da.vbase = spgd_vbase; da.d_kb = spgd_kb; da.d_vb = spgd_vb;
                        da.d_mul = SPGD_MUL; da.d_inv = odd_inverse(SPGD_MUL);
                        da.d_gmagic = (unsigned int)((0xffffffffull + spg_owners) / spg_owners);  // ceil(2^32 / owners)
                        da.d_slots = spgd_slots;
                        const size_t dsm = (size_t)spgd_slots * 8;
                        with_sum_cnt(sum_j >= 0, cnt_j >= 0, [&](auto s, auto c) {
                            spgn_partition_kernel<s, c, true><<<gn, SPG_TTHREADS, SpgnK1Smem<true>::bytes, stream>>>(da);
                            spgn_aggregate_kernel<s, c, true><<<spg_owners, SPG_THREADS, dsm, stream>>>(da);
                        });
                        spgd_launches++;
                    } else {
                        with_sum_cnt(sum_j >= 0, cnt_j >= 0, [&](auto s, auto c) {
                            spgn_partition_kernel<s, c><<<gn, SPG_TTHREADS, SpgnK1Smem<false>::bytes, stream>>>(a);
                            spgn_aggregate_kernel<s, c><<<spg_owners, SPG_THREADS, spgn_smem, stream>>>(a);
                        });
                    }
                    spgn_launches++;
                } else {
                    with_sum_cnt(sum_j >= 0, cnt_j >= 0, [&](auto s, auto c) {
                        if (hot) spg_partition_tma_kernel<s, c, true><<<g2, SPG_TTHREADS, SpgK1Smem<true>::bytes, stream>>>(a);
                        else spg_partition_tma_kernel<s, c><<<g2, SPG_TTHREADS, SpgK1Smem<false>::bytes, stream>>>(a);
                        spg_aggregate_kernel<s, c><<<spg_owners, SPG_THREADS, spg_smem, stream>>>(a);
                    });
                    spg16_launches++;
                }
            }
            B200_CUDA(cudaGetLastError());
            prof_end(prof);
            B200_CUDA(cudaMemcpyAsync(h_spg + slot * N_COUNTERS, d_counters.p, N_COUNTERS * sizeof(long long), cudaMemcpyDeviceToHost, stream));
            B200_CUDA(cudaEventRecord(spg_ev[slot], stream));
            launches += 2; consume_launches++; spg_launches++;
            rows_consumed += rows;
            if (li > 0) spg_finish(1 - slot, sum_j, cnt_j);  // inspect the previous launch while this one runs
        }
        if (li > 0) spg_finish((int)((li - 1) & 1), sum_j, cnt_j);
        read_counters();
        n_groups_bound = n_groups;
    }

    // ---- SPG-G: the SM-partitioned path for generic signatures (spgg.cuh) ----
    struct GenSig { int vcol = -1; bool has_sum = false, has_mm = false, has_nn = false; int layout = 0; };
    static bool gen_int_ok(int ct) { const int sz = ctype_size(ct); return (sz == 4 || sz == 8) && !ctype_is_float(ct) && ct != CT_UINT64; }
    bool gen_signature(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, GenSig& gs) const {
        if (nk != 1 || n_funcs < 1 || n_funcs > GEN_MAX_F || !gen_int_ok(c_types[0])) return false;
        bool has_size = false;
        for (auto& f : funcs) {
            switch (f.kind) {
                case K_SIZE: has_size = true; continue;
                case K_COUNT: break;
                case K_SUM_I64: case K_MEAN: gs.has_sum = true; break;
                case K_MIN_I64: case K_MAX_I64: gs.has_mm = true; break;
                default: return false;
            }
            if (!gen_int_ok(f.in_ctype)) return false;
            if (gs.vcol >= 0 && gs.vcol != f.in_col) return false;
            gs.vcol = f.in_col;
        }
        // tiles (columns and validity bitmaps) are fetched with TMA bulk copies: 16-byte aligned sources
        if (((uintptr_t)data[0] & 15) || ((uintptr_t)valid[0] & 15)) return false;
        if (gs.vcol >= 0 && (((uintptr_t)data[gs.vcol] & 15) || ((uintptr_t)valid[gs.vcol] & 15))) return false;
        gs.has_nn = gs.vcol >= 0 && valid[gs.vcol] != nullptr && has_size;
        gs.layout = (gs.has_mm ? 1 : 0) + (gs.has_nn ? 2 : 0);
        return true;
    }
    int64_t spgg_group_capacity(int layout) const { return (int64_t)spg_owners * (spgg_ns[layout] * 7 / 10); }
    int spgg_pass_count(int64_t est, int layout) const {
        int64_t p = (est + spgg_group_capacity(layout) - 1) / spgg_group_capacity(layout);
        return p <= 1 ? 1 : (p <= SPG_MAX_PASSES ? (int)p : 0);
    }
    static constexpr int64_t GEN_LAUNCH_ROWS = 1ll << 27;
    PooledBuf d_nbucket;  // key-only buckets of the rows whose value is NA

    void consume_spg_gen(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n, const GenSig& gs, int passes) {
        ScopedTimer timer{t_spg};
        const int kct = c_types[0], vct = gs.vcol >= 0 ? c_types[gs.vcol] : CT_INT64;
        const int ks = ctype_size(kct), vs = gs.vcol >= 0 ? ctype_size(vct) : 0;
        const int mm = gs.layout;
        const bool v_nullable = gs.vcol >= 0 && valid[gs.vcol] != nullptr;
        // multi-pass: K1g partitions straight into owners x passes buckets when its class table has room for them
        const int n_vo = (passes > 1 && spg_owners * passes + (v_nullable ? spg_owners : 0) <= GEN_CLS) ? spg_owners * passes : spg_owners;
        for (int64_t r0 = 0; r0 < n; r0 += GEN_LAUNCH_ROWS) {
            const int64_t rows = std::min(GEN_LAUNCH_ROWS, n - r0);
            // a bucket holds rows / owners rows (NA-value buckets: at most that) however many buckets the valued rows spread over
            const int64_t bucket_cap = (rows / spg_owners) + (rows / spg_owners) / 8 + 4096;
            double ta = now();
            d_bucket.ensure(device, (size_t)n_vo * bucket_cap * 16);
            if (v_nullable) d_nbucket.ensure(device, (size_t)spg_owners * bucket_cap * 8);
            // one entry per row at most (bucket overflow, carry, no room in the shared table), plus one per occupied slot per pass
            const int64_t retry_cap = rows + (int64_t)spg_owners * (spgg_ns[mm] + SPG_STASH) * passes;
            d_retry2[0].ensure(device, (size_t)retry_cap * GEN_RETRY_WORDS * 8);
            t_alloc += now() - ta;
            B200_CUDA(cudaMemsetAsync(d_bucket_cnt.p, 0, (size_t)(n_vo + spg_owners) * SPG_CNT_STRIDE * 8, stream));
            auto make_args = [&]() {
                SpgGenArgs g{};
                g.s.n_rows = rows; g.s.n_owners = spg_owners;
                g.s.tkeys = d_keys.as<long long>(); g.s.cap = cap; g.s.counters = d_counters.as<long long>(); g.s.group_limit = (long long)(cap / 2);
                g.s.retry_ctr = d_counters.as<long long>() + CTR_FAIL; g.s.retry = d_retry2[0].as<unsigned long long>(); g.s.retry_cap = retry_cap;
                g.s.bucket = d_bucket.as<longlong2>(); g.s.bucket_cnt = d_bucket_cnt.as<unsigned long long>(); g.s.bucket_cap = bucket_cap;
                g.s.ns = spgg_ns[mm]; g.s.n_pass = passes;
                g.nbucket = v_nullable ? d_nbucket.as<long long>() : nullptr; g.n_vo = n_vo;
                g.kdata = (const char*)data[0] + r0 * ks; g.kvalid = valid[0] ? valid[0] + r0 / 8 : nullptr;
                g.vdata = gs.vcol >= 0 ? (const char*)data[gs.vcol] + r0 * vs : nullptr;
                g.vvalid = (gs.vcol >= 0 && valid[gs.vcol]) ? valid[gs.vcol] + r0 / 8 : nullptr;
                g.k_signed = ctype_is_signed_int(kct) ? 1 : 0; g.v_signed = ctype_is_signed_int(vct) ? 1 : 0;
                g.dropna = dropna ? 1 : 0;
                g.fl.n = n_funcs;
                for (int j = 0; j < n_funcs; j++) {
                    g.fl.kind[j] = funcs[j].kind; g.fl.a0[j] = d_a0[j].as<unsigned long long>();
                    g.fl.a1[j] = funcs[j].has_a1 ? d_a1[j].as<unsigned long long>() : nullptr;
                }
                return g;
            };
            const SpgGenArgs g = make_args();
            const ProfEvents prof = prof_begin(profiling);
            const int g1 = (int)std::min<int64_t>((int64_t)sms * SPG_TCTAS, (rows + SPG_TILE - 1) / SPG_TILE);
            with_spgg_part(ks, vs, [&](auto k, auto v) { spgg_partition_kernel<k, v><<<g1, SPG_TTHREADS, SpggK1Smem::bytes, stream>>>(g); });
            with_spgg_agg(gs.has_sum, gs.has_mm, gs.has_nn, [&](auto s, auto m, auto nn) {
                spgg_aggregate_kernel<s, m, nn><<<spg_owners, SPG_THREADS, spgg_smem[mm], stream>>>(g);
            });
            B200_CUDA(cudaGetLastError());
            prof_end(prof);
            launches += 2; consume_launches++; spg_launches++; spgg_launches++;
            rows_consumed += rows;
            // partials that found the global table at its limit: grow, replay them
            settle<unsigned long long>(d_retry2[0], GEN_RETRY_WORDS, spg_retry_rows, [&](const unsigned long long* list, int64_t nr) {
                spgg_replay_kernel<<<grid_for(nr), 256, 0, stream>>>(make_args(), list, (long long)nr);
                launches++;
                B200_CUDA(cudaGetLastError());
            });
        }
        n_groups_bound = n_groups;
    }

    // Consume rows [0, n) of device-resident columns.
    void consume_device_chunk(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n) {
        if (n == 0) return;
        if (nk > 1) { consume_mk(data, valid, n); return; }
        // fast path: non-null int64 key + {sum, count/size} over one non-null int64 value column
        bool fast = c_types[0] == CT_INT64 && valid[0] == nullptr && n_funcs >= 1;
        int sum_j = -1, cnt_j = -1, vcol = -1;
        for (int j = 0; j < n_funcs && fast; j++) {
            const FuncSpec& f = funcs[j];
            if (f.kind == K_SUM_I64 && f.in_ctype == CT_INT64 && valid[f.in_col] == nullptr && sum_j < 0) {
                sum_j = j; vcol = f.in_col;
            } else if ((f.kind == K_SIZE || (f.kind == K_COUNT && !ctype_is_float(f.in_ctype) && valid[f.in_col] == nullptr)) && cnt_j < 0) {
                cnt_j = j;
            } else {
                fast = false;
            }
        }
        if (fast && (((uintptr_t)data[0] & 15) || (vcol >= 0 && ((uintptr_t)data[vcol] & 15)))) fast = false;
        // SM-partitioned paths for big batches whose (estimated) cardinality fits the chip's shared memory: SPG for the fast-path
        // signature, SPG-G for generic ones (nullable / 4-byte keys or values / mean / min / max over one integer column)
        const bool spg = n >= (1 << 20) && spg_probe();
        GenSig gs;
        const bool gen = !fast && spg && spgg_enabled && gen_signature(data, valid, gs);
        if (!(fast && spg) && !gen) { consume_direct(data, valid, n, fast, sum_j, cnt_j, vcol, false); return; }
        const char* env = getenv("B200_SPG");
        const bool force = fast && env && env[0] == '1';
        int64_t est = std::max(expected_groups_hint, n_groups);
        std::vector<const void*> d2(data); std::vector<const uint8_t*> v2(valid);
        int64_t left = n;
        const bool learned = !force && est == 0 && rows_consumed == 0;
        if (learned) {  // cardinality unknown: learn it from a prefix through the direct kernel
            const int64_t prefix = std::min<int64_t>(n, 1 << 20);
            consume_direct(data, valid, prefix, fast, sum_j, cnt_j, vcol, /*force_count=*/true);
            est = n_groups;
            if (prefix == n) return;
            for (int c = 0; c < n_cols; c++) {  // (the fast-path signature has no validity bitmaps)
                if (data[c]) d2[c] = (const char*)data[c] + prefix * ctype_size(c_types[c]);
                if (valid[c]) v2[c] = valid[c] + prefix / 8;
            }
            left = n - prefix;
        }
        if (fast) {
            if (force || spg_pass_count(est) > 0) {
                spg_passes = std::max(1, spg_pass_count(est));
                // LC only on an estimate: a hint, groups already in the table, or a prefix (even one that found none)
                const bool lowcard = (learned || est > 0) && lc_pick(est);
                consume_spg((const long long*)d2[0], vcol >= 0 ? (const long long*)d2[vcol] : nullptr, left, sum_j, cnt_j, lowcard, est);
                return;
            }
        } else if (est > LC_SLOTS_BIG / 4 && spgg_pass_count(est, gs.layout) > 0 && left >= (1 << 16)) {
            // (below ~1000 groups the owners are unevenly loaded, and there is no low-cardinality generic kernel: direct path)
            consume_spg_gen(d2, v2, left, gs, spgg_pass_count(est, gs.layout));
            return;
        }
        consume_direct(d2, v2, left, fast, sum_j, cnt_j, vcol, false);
    }

    void consume_direct(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n, bool fast, int sum_j,
                        int cnt_j, int vcol, bool force_count) {
        bool could_fail = force_count || (int64_t)(cap / 2) - n_groups_bound < n;
        if (could_fail) d_fail.ensure(device, (size_t)n * 4);
        // table pointers are looked up at launch time: grow() replaces them between a launch and its replay
        auto launch = [&](const uint32_t* index_list, int64_t rows) {
            const ProfEvents prof = prof_begin(profiling && index_list == nullptr);
            if (fast && index_list == nullptr) {
                const long long* k = (const long long*)data[0];
                const long long* v = vcol >= 0 ? (const long long*)data[vcol] : nullptr;
                unsigned long long* as = sum_j >= 0 ? d_a0[sum_j].as<unsigned long long>() : nullptr;
                unsigned long long* ac = cnt_j >= 0 ? d_a0[cnt_j].as<unsigned long long>() : nullptr;
                with_sum_cnt(sum_j >= 0, cnt_j >= 0, [&](auto s, auto c) {
                    groupby_consume_i64_sumcount_kernel<s, c><<<grid_for(rows, 2), 256, 0, stream>>>(
                        k, v, rows, d_keys.as<long long>(), cap, as, ac, d_counters.as<long long>(), (long long)(cap / 2), d_fail.as<uint32_t>());
                });
            } else {
                ConsumeArgs a = generic_args(data, valid, index_list, rows);
                if (has_reduction_kinds(a)) groupby_consume_kernel<true><<<grid_for(rows), 256, prod_smem_bytes(a), stream>>>(a);
                else groupby_consume_kernel<false><<<grid_for(rows), 256, 0, stream>>>(a);
            }
            launches++;
            if (index_list == nullptr) consume_launches++;
            prof_end(prof);
            B200_CUDA(cudaGetLastError());
        };
        launch(nullptr, n);
        if (could_fail) settle<uint32_t>(d_fail, 1, fail_rows, launch);
        if (has_firstlast) {  // every row is in (replays included): the rows that won first / last write their values
            groupby_firstlast_fix_kernel<<<grid_for(n), 256, 0, stream>>>(generic_args(data, valid, nullptr, n));
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        if (!could_fail) n_groups_bound += n;  // upper bound without a device round trip
        else n_groups_bound = n_groups;
        rows_consumed += n;
    }
    ConsumeArgs generic_args(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, const uint32_t* index_list, int64_t rows) {
        ConsumeArgs a{};
        a.key_data = data[0]; a.key_valid = valid[0]; a.key_ctype = c_types[0]; a.dropna = dropna ? 1 : 0;
        a.n_rows = rows; a.index_list = index_list; a.tkeys = d_keys.as<long long>(); a.cap = cap;
        a.counters = d_counters.as<long long>(); a.group_limit = (long long)(cap / 2); a.fail_list = d_fail.as<uint32_t>(); a.n_ops = n_apply();
        // rank-major sequence numbers: rows of a lower rank come first (the reference's row-block distribution), then row order
        a.seq_base = ((unsigned long long)rank << 44) + (unsigned long long)rows_consumed;
        fill_ops(a.ops, data, valid);
        return a;
    }
    // the aggregate updates a consume launch applies per row: every function's, none for MRNF (its passes run after the launch),
    // none of the holistic words (holistic_append_kernel runs after the launch)
    int n_apply() const { return mr.on ? 0 : ho.on ? ho.p0 : n_funcs; }
    // the n_apply() aggregate updates of a consume launch (ConsumeArgs / MkArgs)
    void fill_ops(OpDesc* ops, const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid) const {
        for (int j = 0; j < n_apply(); j++) {
            const FuncSpec& f = funcs[j];
            ops[j].kind = f.kind; ops[j].in_ctype = f.in_ctype;
            ops[j].in_data = f.in_col >= 0 ? data[f.in_col] : nullptr;
            ops[j].in_valid = f.in_col >= 0 ? valid[f.in_col] : nullptr;
            ops[j].a0 = d_a0[j].p; ops[j].a1 = f.has_a1 ? d_a1[j].p : nullptr;
        }
    }

    int64_t n_groups_bound = 0;  // upper bound on groups in the table known to the host
    bool stage_recorded[2] = {false, false};

    // ---- float keys: canonicalisation pre-pass ----
    bool float_key(int kc) const { return ctype_is_float(in_types[kc]); }
    DevBuf d_canon[MAX_KEYS];  // canonical int64 column of each float key column (pooled: 16-byte aligned, as SPG needs)
    void canon_launch(const void* in, int ct, long long* out, int64_t n) {
        if (n == 0) return;
        const int g = grid_for((n + 3) / 4);
        if (ct == CT_FLOAT64) canon_float_key_kernel<double><<<g, 256, 0, stream>>>((const double*)in, out, n);
        else canon_float_key_kernel<float><<<g, 256, 0, stream>>>((const float*)in, out, n);
        launches++;
        B200_CUDA(cudaGetLastError());
    }
    // points the float key columns of a device-resident chunk at their canonical int64 columns
    void canon_keys(std::vector<const void*>& data, int64_t n) {
        for (int kc = 0; kc < nk; kc++) {
            if (!float_key(kc)) continue;
            d_canon[kc].ensure((size_t)n * 8);
            canon_launch(data[kc], in_types[kc], d_canon[kc].as<long long>(), n);
            data[kc] = d_canon[kc].p;
        }
    }
    // one device-resident chunk of a batch: keys canonicalised, then aggregated (MRNF also reads the batch's own cells)
    void consume_chunk(std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n) {
        const std::vector<const void*> raw = data;
        canon_keys(data, n);
        if (mr.on) consume_mrnf(data, raw, valid, n);
        else if (ho.on) consume_holistic(data, valid, n);
        else consume_device_chunk(data, valid, n);
    }

    // ---- min_row_number_filter (see mrnf_min_kernel) ----
    struct Mrnf {
        bool on = false;
        int n_sort = 0, n_digits = 0;
        int sort_col[MAX_KEYS] = {};
        SortKey key[MAX_KEYS] = {};
        int f_end[MRNF_FIELDS] = {};
        std::vector<int> keep;  // kept columns, in column order
        int w0 = 0;             // funcs[w0 ..): the winner's digits, its validity word, one word per kept column
        DevBuf b, slot;         // B (n_digits x (b_cap + 2) words) and the batch's slot cache
        uint64_t b_cap = 0;
        int64_t limit = 1;      // rows kept per group; > 1: funcs[w0] is the group id word and the rows go through the store
    } mr;

    // ---- limit > 1 (see mrnf_top_filter_kernel) ----
    static constexpr int64_t MRNF_CAND_MAX = 1ll << 31;      // rows radix_sort_columns sorts at once
    static constexpr int64_t MRNF_REDUCE_MIN = 1ll << 22;    // admitted rows that make a reduce worth its sort
    struct MrnfTop {
        DevBuf store[2];        // the candidate store and the reduce's destination, store_words() columns of cap rows each
        int64_t cap = 0;
        int64_t survivors = 0;  // store rows after the last reduce (every id's first `limit` rows, in (id, rank) order)
        int64_t bound = 0;      // upper bound on the store's rows (survivors + rows filtered since)
        int64_t admitted = 0, reduces = 0;  // metrics 18 and 19: candidate rows admitted, reduces run
        DevBuf ctr;             // [0] store rows, [1] ids handed out
        unsigned long long* h_ctr = nullptr;  // pinned mirror of ctr
        DevBuf cutoff, head, keep, pos, ids[2];
        int64_t n_cut = 0;      // ids with a cutoff row (ids handed out at the last reduce)
        Scanner scan;
    } mt;
    int store_words() const { return 2 + mr.n_digits + (int)mr.keep.size(); }

    void setup_mrnf(const MrnfSpec& s) {
        B200_REQUIRE(n_outs == 0, "b200 groupby: min_row_number_filter takes no other aggregate function");
        B200_REQUIRE(s.n_sort >= 1 && s.n_sort <= MAX_KEYS, "b200 groupby: min_row_number_filter takes 1 to 4 sort columns");
        mr.on = true;
        mr.n_sort = s.n_sort;
        int bits = 0;
        for (int j = 0; j < s.n_sort; j++) {
            const int c = s.sort_cols[j];
            const std::string what = "b200 groupby: min_row_number_filter sort column " + std::to_string(j) + " (column " + std::to_string(c) + ")";
            B200_REQUIRE(c >= 0 && c < n_cols, what + " is out of range");
            for (int q = 0; q < j; q++) B200_REQUIRE(s.sort_cols[q] != c, what + " is listed twice");
            B200_REQUIRE(ctype_size(in_types[c]) > 0, what + " is not a fixed-width column");
            B200_REQUIRE(arr_types[c] == ARR_NUMPY || arr_types[c] == ARR_NULLABLE, what + " has an unsupported array type");
            mr.sort_col[j] = c;
            mr.key[j] = SortKey{in_types[c], ctype_size(in_types[c]), s.ascending[j] ? 0 : 1, s.na_last[j] ? 1 : 0};
            mr.f_end[2 * j] = bits += 1;
            mr.f_end[2 * j + 1] = bits += 8 * ctype_size(in_types[c]);
        }
        mr.f_end[2 * MAX_KEYS] = bits += MRNF_SEQ_BITS;
        mr.n_digits = (bits + 62) / 63;
        for (int c = 0; c < n_cols; c++) {
            if (!s.keep[c]) continue;
            const std::string what = "b200 groupby: min_row_number_filter kept column " + std::to_string(c);
            B200_REQUIRE(ctype_size(in_types[c]) > 0, what + " is not a fixed-width column");
            B200_REQUIRE(arr_types[c] == ARR_NUMPY || arr_types[c] == ARR_NULLABLE, what + " has an unsupported array type");
            mr.keep.push_back(c);
        }
        B200_REQUIRE(!mr.keep.empty(), "b200 groupby: min_row_number_filter keeps no column");
        B200_REQUIRE((int)mr.keep.size() <= MRNF_MAX_KEEP, "b200 groupby: min_row_number_filter keeps at most " + std::to_string(MRNF_MAX_KEEP) + " columns");
        B200_REQUIRE(s.limit >= 1 && s.limit < MRNF_CAND_MAX, "b200 groupby: min_row_number_filter rows_per_group must be in [1, 2^31)");
        mr.limit = s.limit;
        mr.w0 = (int)funcs.size();
        if (mr.limit > 1) {  // the group id word, all-ones until claimed
            FuncSpec g{};
            g.in_col = -1; g.in_ctype = CT_INT64; g.in_arrtype = ARR_NUMPY; g.kind = K_MRNF; g.out_ctype = CT_INT64; g.out_arrtype = ARR_NUMPY;
            g.init0 = ~0ull;
            funcs.push_back(g);
            mt.ctr.alloc(16);
            B200_CUDA(cudaMemsetAsync(mt.ctr.p, 0, 16, stream));
            mt.h_ctr = (unsigned long long*)pinned_acquire(16);
            return;
        }
        // the winner record: digits all-ones (above every row's tuple), validity and payload zero
        FuncSpec w{};
        w.in_col = -1; w.in_ctype = CT_INT64; w.in_arrtype = ARR_NUMPY; w.kind = K_MRNF; w.out_ctype = CT_INT64; w.out_arrtype = ARR_NUMPY;
        for (int e = 0; e < mr.n_digits + 1 + (int)mr.keep.size(); e++) {
            w.init0 = e < mr.n_digits ? ~0ull : 0ull;
            funcs.push_back(w);
        }
    }

    void consume_mrnf(const std::vector<const void*>& keys, const std::vector<const void*>& raw, const std::vector<const uint8_t*>& valid, int64_t n) {
        if (n == 0) return;
        B200_REQUIRE(rows_consumed + n < (1ll << MRNF_SEQ_BITS), "b200 groupby: min_row_number_filter takes fewer than 2^48 rows");
        const unsigned long long seq_base = (unsigned long long)rows_consumed;
        // insert the keys (no aggregate: n_apply() is 0); the table grows and the failed rows are replayed until all are in
        if (nk > 1) consume_mk(keys, valid, n);
        else consume_direct(keys, valid, n, false, -1, -1, -1, false);
        if (mr.limit == 1 && mr.b_cap != cap) {  // (B is all-ones whenever the table grows: a fresh B for the new capacity)
            mr.b.alloc((size_t)mr.n_digits * (cap + 2) * 8);
            fill(mr.b.p, (uint64_t)mr.n_digits * (cap + 2), ~0ull);
            mr.b_cap = cap;
        }
        if (mr.limit == 1) mr.slot.ensure((size_t)n * 8);
        MrnfArgs a{};
        a.n_rows = n; a.seq_base = seq_base; a.nk = nk; a.dropna = dropna ? 1 : 0; a.cap = cap;
        for (int j = 0; j < nk; j++) { a.key_data[j] = keys[j]; a.key_valid[j] = valid[j]; a.key_ctype[j] = c_types[j]; }
        if (nk == 1) a.tkeys = d_keys.as<long long>();
        else {
            a.tags = d_tags.as<unsigned long long>(); a.mkmask = d_mkmask.as<unsigned char>();
            for (int j = 0; j < nk; j++) a.mk[j] = d_mk[j].as<long long>();
        }
        a.slot = mr.slot.as<uint64_t>();  // (limit > 1: unused)
        a.n_sort = mr.n_sort; a.n_digits = mr.n_digits;
        for (int j = 0; j < mr.n_sort; j++) { a.key[j] = mr.key[j]; a.sort_data[j] = raw[mr.sort_col[j]]; a.sort_valid[j] = valid[mr.sort_col[j]]; }
        std::copy(mr.f_end, mr.f_end + MRNF_FIELDS, a.f_end);
        a.n_keep = (int)mr.keep.size();
        for (int j = 0; j < a.n_keep; j++) {
            const int c = mr.keep[j];
            a.keep_data[j] = raw[c]; a.keep_valid[j] = valid[c]; a.keep_size[j] = ctype_size(in_types[c]);
        }
        if (mr.limit > 1) { filter_top(a); return; }
        a.b = mr.b.as<unsigned long long>();
        for (int e = 0; e < mr.n_digits; e++) a.w[e] = d_a0[mr.w0 + e].as<unsigned long long>();
        a.w_valid = d_a0[mr.w0 + mr.n_digits].as<unsigned long long>();
        for (int j = 0; j < a.n_keep; j++) a.keep_w[j] = d_a0[mr.w0 + mr.n_digits + 1 + j].as<unsigned long long>();
        for (int d = 0; d < mr.n_digits; d++) mrnf_min_kernel<<<grid_for(n), 256, 0, stream>>>(a, d);
        mrnf_merge_kernel<<<grid_for(n), 256, 0, stream>>>(a);
        launches += mr.n_digits + 1;
        B200_CUDA(cudaGetLastError());
    }

    // ---- limit > 1: the candidate store (see mrnf_top_filter_kernel) ----
    // Filters one chunk (every row is in the table).  Before the launch the host makes room for every row of the chunk in the
    // store, so the kernel never overflows; the store's row count stays on the device, the host keeps an upper bound.
    void filter_top(const MrnfArgs& m) {
        const int64_t n = m.n_rows;
        ensure_candidate_room(n);
        // amortised reduce: once the rows admitted since the last reduce may have reached max(survivors, MRNF_REDUCE_MIN), count them
        const int64_t due = std::max(mt.survivors, MRNF_REDUCE_MIN);
        if (mt.bound - mt.survivors >= due) {
            read_top_counts();
            if (mt.bound - mt.survivors >= due) reduce_top();
        }
        if (mt.bound + n > mt.cap) {  // a larger store, keeping its rows
            const int64_t nc = std::min(MRNF_CAND_MAX, std::max(mt.bound + n, mt.cap + mt.cap / 2));
            const int w = store_words();
            DevBuf g;
            g.alloc((size_t)w * nc * 8);
            if (mt.bound > 0) B200_CUDA(cudaMemcpy2DAsync(g.p, (size_t)nc * 8, mt.store[0].p, (size_t)mt.cap * 8, (size_t)mt.bound * 8, w, cudaMemcpyDeviceToDevice, stream));
            mt.store[0] = std::move(g);
            mt.store[1].alloc((size_t)w * nc * 8);
            mt.cap = nc;
        }
        MrnfTopArgs t{};
        t.m = m;
        t.gid = d_a0[mr.w0].as<unsigned long long>();
        t.ctr = mt.ctr.as<unsigned long long>();
        t.cutoff = mt.cutoff.as<unsigned long long>(); t.n_cut = (unsigned long long)mt.n_cut;
        for (int j = 0; j < nk; j++) if (dropna && float_key(j)) t.drop_nan |= 1u << j;
        t.store = mt.store[0].as<unsigned long long>(); t.store_cap = (unsigned long long)mt.cap;
        mrnf_top_filter_kernel<<<grid_for(n), 256, 0, stream>>>(t);
        launches++;
        B200_CUDA(cudaGetLastError());
        mt.bound += n;
    }
    // Refuses n more rows when the store could pass MRNF_CAND_MAX rows even right after a reduce.
    void ensure_candidate_room(int64_t n) {
        if (mr.limit == 1 || mt.bound + n <= MRNF_CAND_MAX) return;
        read_top_counts();
        reduce_top();
        B200_REQUIRE(mt.survivors + n <= MRNF_CAND_MAX,
                     "b200 groupby: min_row_number_filter with rows_per_group = " + std::to_string(mr.limit) + " sorts its candidates (the " +
                         std::to_string(mt.survivors) + " survivors, at most groups x rows_per_group, plus a batch of " + std::to_string(n) +
                         " rows) in one radix sort of at most 2^31 rows; keep groups x rows_per_group + batch rows below 2^31");
    }
    // the store's exact row count into mt.bound (synchronises the stream)
    void read_top_counts() {
        B200_CUDA(cudaMemcpyAsync(mt.h_ctr, mt.ctr.p, 16, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        mt.bound = (int64_t)mt.h_ctr[0];
    }
    // After read_top_counts: sorts the store by (id, digits), keeps each id's first mr.limit rows, in that order, and writes the
    // cutoff of every id that has mr.limit of them.  Nothing to do when no row came since the last reduce.
    void reduce_top() {
        const int64_t m = mt.bound, n_ids = (int64_t)mt.h_ctr[1];
        if (m == mt.survivors) return;
        mt.admitted += m - mt.survivors;
        mt.reduces++;
        const int nd = mr.n_digits, w = store_words();
        if (n_ids > mt.n_cut) {  // cutoffs for the ids handed out since: all-ones (fewer than limit survivors)
            DevBuf c;
            c.alloc((size_t)n_ids * nd * 8);
            if (mt.n_cut > 0) B200_CUDA(cudaMemcpyAsync(c.p, mt.cutoff.p, (size_t)mt.n_cut * nd * 8, cudaMemcpyDeviceToDevice, stream));
            fill(c.as<unsigned long long>() + mt.n_cut * nd, (uint64_t)(n_ids - mt.n_cut) * nd, ~0ull);
            mt.cutoff = std::move(c);
            mt.n_cut = n_ids;
        }
        const uint64_t sc = (uint64_t)mt.cap;
        const SortKey u64{CT_UINT64, 8, 0, 0};
        const SortKey keys[4] = {u64, u64, u64, u64};
        const void* cols[4];
        auto col = [&](int c) { return (const void*)(mt.store[0].as<unsigned long long>() + c * sc); };
        const uint32_t* perm;
        if (1 + nd > 4) {  // at most four columns per sort: digits 3.. first, then a stable sort by (id, digits 0..2) of that order
            for (int e = 3; e < nd; e++) cols[e - 3] = col(1 + e);
            perm = radix_sort_columns(nd - 3, cols, keys, m, mt.ids, stream);
            if (perm) {
                mrnf_top_move_kernel<<<grid_for(m), 256, 0, stream>>>(mt.store[0].as<unsigned long long>(), mt.store[1].as<unsigned long long>(), sc, w,
                                                                    perm, m, nullptr, nullptr);
                launches++;
                std::swap(mt.store[0], mt.store[1]);
            }
            for (int c = 0; c < 4; c++) cols[c] = col(c);
            perm = radix_sort_columns(4, cols, keys, m, mt.ids, stream);
        } else {
            for (int c = 0; c < 1 + nd; c++) cols[c] = col(c);
            perm = radix_sort_columns(1 + nd, cols, keys, m, mt.ids, stream);
        }
        mt.head.ensure((size_t)n_ids * 4);
        mt.keep.ensure((size_t)m * 4);
        mt.pos.ensure((size_t)m * 8);
        const unsigned long long* st = mt.store[0].as<unsigned long long>();
        mrnf_top_head_kernel<<<grid_for(m), 256, 0, stream>>>(st, perm, m, mt.head.as<uint32_t>());
        mrnf_top_rank_kernel<<<grid_for(m), 256, 0, stream>>>(st, sc, nd, perm, m, mt.head.as<uint32_t>(), (long long)mr.limit,
                                                              mt.keep.as<uint32_t>(), mt.cutoff.as<unsigned long long>());
        launches += 2;
        B200_CUDA(cudaGetLastError());
        const int64_t kept = (int64_t)mt.scan.run(mt.keep.as<uint32_t>(), m, mt.pos.as<unsigned long long>(), stream, &launches);
        mrnf_top_move_kernel<<<grid_for(m), 256, 0, stream>>>(st, mt.store[1].as<unsigned long long>(), sc, w, perm, m, mt.keep.as<uint32_t>(),
                                                            mt.pos.as<unsigned long long>());
        launches++;
        B200_CUDA(cudaGetLastError());
        std::swap(mt.store[0], mt.store[1]);
        mt.survivors = mt.bound = kept;
        fill(mt.ctr.p, 1, (unsigned long long)kept);  // the append cursor
    }
    int64_t finalize_mrnf_top() {
        read_top_counts();
        reduce_top();
        const int64_t max_out = mt.survivors;
        const size_t words = (size_t)((max_out + 31) / 32 + 1);
        const int n_keep = (int)mr.keep.size();
        d_out_data.resize(n_keep); d_out_valid.resize(n_keep);
        MrnfOutArgs o{};
        o.n_keep = n_keep;
        for (int j = 0; j < n_keep; j++) {
            const int c = mr.keep[j];
            o.keep_size[j] = ctype_size(in_types[c]);
            d_out_data[j].ensure((size_t)(max_out + 32) * 8);
            o.out[j] = d_out_data[j].p;
            if (arr_types[c] == ARR_NULLABLE) { d_out_valid[j].ensure(words * 4); o.out_valid[j] = d_out_valid[j].as<uint32_t>(); }
        }
        mrnf_top_gather_kernel<<<grid_for(std::max<int64_t>(max_out, 1)), 256, 0, stream>>>(mt.store[0].as<unsigned long long>(), (uint64_t)mt.cap,
                                                                                            mr.n_digits, max_out, o);
        launches++;
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(stream));
        n_out = max_out;
        finalized = true;
        out_cursor = 0;
        return n_out;
    }

    int64_t finalize_mrnf() {
        if (mr.limit > 1) return finalize_mrnf_top();
        compact();
        const int64_t max_out = max_out_bound();
        const size_t words = (size_t)((max_out + 31) / 32 + 1);
        const int n_keep = (int)mr.keep.size();
        d_out_data.resize(n_keep); d_out_valid.resize(n_keep);
        MrnfOutArgs o{};
        o.slot_of_out = d_slot_of_out.as<uint64_t>(); o.n_out_ptr = d_counters.as<long long>() + CTR_OUT;
        o.w_valid = d_a0[mr.w0 + mr.n_digits].as<unsigned long long>(); o.n_keep = n_keep;
        for (int j = 0; j < n_keep; j++) {
            const int c = mr.keep[j];
            o.keep_w[j] = d_a0[mr.w0 + mr.n_digits + 1 + j].as<unsigned long long>(); o.keep_size[j] = ctype_size(in_types[c]);
            d_out_data[j].ensure((size_t)(max_out + 32) * 8);
            o.out[j] = d_out_data[j].p;
            if (arr_types[c] == ARR_NULLABLE) { d_out_valid[j].ensure(words * 4); o.out_valid[j] = d_out_valid[j].as<uint32_t>(); }
        }
        mrnf_gather_kernel<<<grid_for(max_out), 256, 0, stream>>>(o);
        launches++;
        B200_CUDA(cudaGetLastError());
        read_counters();
        n_out = h_counters[CTR_OUT];
        finalized = true;
        out_cursor = 0;
        return n_out;
    }

    // ---- holistic aggregates (see holistic_append_kernel) ----
    static constexpr int64_t HO_STORE_MAX = 1ll << 31;  // rows radix_sort_columns sorts at once
    static constexpr int64_t HO_MAX_IDS = 1ll << 32;    // store ids are 4 bytes
    struct HoStore {
        int in_col = -1;
        DevBuf id, val;     // cap rows each: the group id (4 bytes) and the value (its width)
        int64_t cap = 0;
        int64_t bound = 0;  // upper bound on the rows (the device cursor ctr[1 + i] is exact)
    };
    struct HoOut { int out, store, kind; double q; };
    struct Holistic {
        bool on = false;
        int p0 = 0;  // funcs[p0]: the group id word (K_HID); funcs[p0 + 1 + k]: the result word of outs[k]
        std::vector<HoStore> st;
        std::vector<HoOut> outs;
        DevBuf ctr;  // [0] ids handed out, [1 + i] rows of store i
        std::vector<unsigned long long> h_ctr;
        int64_t id_bound = 0;  // upper bound on ctr[0]
        int64_t passes = 0;    // metric 21: digit passes of the finalize sorts
        DevBuf perm[2], head, tail, flag, pos, start, best;
        Scanner scan;
    } ho;

    // the id word and one result word per holistic output, after every other accumulator (see n_apply)
    void setup_holistic() {
        B200_REQUIRE(ho.st.size() <= (size_t)MAX_OPS, "b200 groupby: too many value columns for mode / percentiles");
        ho.p0 = (int)funcs.size();
        FuncSpec g{};
        g.in_col = -1; g.in_ctype = CT_INT64; g.in_arrtype = ARR_NUMPY; g.kind = K_HID; g.out_ctype = CT_INT64; g.out_arrtype = ARR_NUMPY;
        g.init0 = ~0ull;
        funcs.push_back(g);
        for (const HoOut& h : ho.outs) {
            FuncSpec r{};
            r.in_col = ho.st[h.store].in_col; r.in_ctype = c_types[r.in_col]; r.in_arrtype = arr_types[r.in_col]; r.kind = h.kind;
            r.out_ctype = outs[h.out].out_ctype; r.out_arrtype = ARR_NULLABLE; r.has_a1 = true; r.init1 = ~0ull;
            outs[h.out].prim[0] = (int)funcs.size();
            funcs.push_back(r);
        }
        ho.ctr.alloc((1 + ho.st.size()) * 8);
        B200_CUDA(cudaMemsetAsync(ho.ctr.p, 0, (1 + ho.st.size()) * 8, stream));
        ho.h_ctr.assign(1 + ho.st.size(), 0);
    }
    // the device counters into ho.h_ctr and the bounds (synchronises the stream)
    void read_holistic_counts() {
        B200_CUDA(cudaMemcpyAsync(ho.h_ctr.data(), ho.ctr.p, ho.h_ctr.size() * 8, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        ho.id_bound = (int64_t)ho.h_ctr[0];
        for (size_t i = 0; i < ho.st.size(); i++) ho.st[i].bound = (int64_t)ho.h_ctr[1 + i];
    }
    int64_t holistic_rows() {  // metric 20: values appended to the stores
        read_holistic_counts();
        int64_t r = 0;
        for (auto& s : ho.st) r += s.bound;
        return r;
    }
    // Refuses a batch of n rows that could take a store past HO_STORE_MAX rows, or the ids past 4 bytes, before anything runs.
    void ensure_holistic_room(int64_t n) {
        bool over = ho.id_bound + n > HO_MAX_IDS;
        for (auto& s : ho.st) over = over || s.bound + n > HO_STORE_MAX;
        if (!over) return;
        read_holistic_counts();
        B200_REQUIRE(ho.id_bound + n <= HO_MAX_IDS, "b200 groupby: mode / percentiles number their groups with 4-byte ids; this batch could "
                                                    "pass 2^32 groups");
        for (auto& s : ho.st)
            B200_REQUIRE(s.bound + n <= HO_STORE_MAX,
                         "b200 groupby: mode / percentile_cont / percentile_disc keep the non-NA values of a column (column " + std::to_string(s.in_col) +
                             ": " + std::to_string(s.bound) + " so far, plus a batch of " + std::to_string(n) +
                             " rows) for one radix sort of at most 2^31 rows; keep them below 2^31 per column");
    }
    void consume_holistic(const std::vector<const void*>& data, const std::vector<const uint8_t*>& valid, int64_t n) {
        if (n == 0) return;
        // every row into the table first (the other aggregates are applied there: n_apply() stops before the holistic words)
        if (nk > 1) consume_mk(data, valid, n);
        else consume_direct(data, valid, n, false, -1, -1, -1, false);
        HoAppendArgs a{};
        MrnfArgs& m = a.m;
        m.n_rows = n; m.nk = nk; m.dropna = dropna ? 1 : 0; m.cap = cap;
        for (int j = 0; j < nk; j++) { m.key_data[j] = data[j]; m.key_valid[j] = valid[j]; m.key_ctype[j] = c_types[j]; }
        if (nk == 1) m.tkeys = d_keys.as<long long>();
        else {
            m.tags = d_tags.as<unsigned long long>(); m.mkmask = d_mkmask.as<unsigned char>();
            for (int j = 0; j < nk; j++) m.mk[j] = d_mk[j].as<long long>();
        }
        for (int j = 0; j < nk; j++) if (dropna && float_key(j)) a.drop_nan |= 1u << j;
        a.gid = d_a0[ho.p0].as<unsigned long long>();
        a.ctr = ho.ctr.as<unsigned long long>();
        a.n_st = (int)ho.st.size();
        for (int i = 0; i < a.n_st; i++) {
            HoStore& s = ho.st[i];
            const int c = s.in_col, w = ctype_size(in_types[c]);
            if (s.bound + n > s.cap) {  // a larger store, keeping its rows (the host makes room: the kernel has no overflow path)
                const int64_t nc = std::min(HO_STORE_MAX, std::max(s.bound + n, s.cap + s.cap / 2));
                DevBuf id, val;
                id.alloc((size_t)nc * 4);
                val.alloc((size_t)nc * w);
                if (s.bound > 0) {
                    B200_CUDA(cudaMemcpyAsync(id.p, s.id.p, (size_t)s.bound * 4, cudaMemcpyDeviceToDevice, stream));
                    B200_CUDA(cudaMemcpyAsync(val.p, s.val.p, (size_t)s.bound * w, cudaMemcpyDeviceToDevice, stream));
                }
                s.id = std::move(id); s.val = std::move(val); s.cap = nc;
            }
            a.val[i] = data[c]; a.valid[i] = valid[c]; a.ct[i] = in_types[c];
            a.st_id[i] = s.id.as<uint32_t>(); a.st_val[i] = s.val.p;
            s.bound += n;
        }
        holistic_append_kernel<<<grid_for(n), 256, 0, stream>>>(a);
        launches++;
        B200_CUDA(cudaGetLastError());
        ho.id_bound += n;
    }
    // Writes every holistic result word (before compaction: eval_output_kernel reads them as first / last words).
    void finalize_holistic() {
        read_holistic_counts();
        const int64_t n_ids = ho.id_bound;
        if (n_ids == 0) return;
        ho.head.ensure((size_t)n_ids * 4);
        ho.tail.ensure((size_t)n_ids * 4);
        for (size_t i = 0; i < ho.st.size(); i++) {
            HoStore& s = ho.st[i];
            const int64_t m = s.bound;
            if (m == 0) continue;  // (every result over this column stays NA)
            const int ct = in_types[s.in_col];
            const SortKey keys[2] = {SortKey{CT_UINT32, 4, 0, 0}, SortKey{ct, ctype_size(ct), 0, 0}};
            const void* cols[2] = {s.id.p, s.val.p};
            HoSorted hs{};
            hs.id = s.id.as<uint32_t>(); hs.val = s.val.p; hs.key = keys[1]; hs.n = m;
            hs.perm = radix_sort_columns(2, cols, keys, m, ho.perm, stream, &ho.passes);
            bool mode = false;
            for (const HoOut& h : ho.outs) mode = mode || (h.store == (int)i && h.kind == E_MODE);
            B200_CUDA(cudaMemsetAsync(ho.head.p, 0, (size_t)n_ids * 4, stream));
            B200_CUDA(cudaMemsetAsync(ho.tail.p, 0, (size_t)n_ids * 4, stream));
            if (mode) ho.flag.ensure((size_t)m * 4);
            holistic_bounds_kernel<<<grid_for(m), 256, 0, stream>>>(hs, ho.head.as<uint32_t>(), ho.tail.as<uint32_t>(), mode ? ho.flag.as<uint32_t>() : nullptr);
            launches++;
            B200_CUDA(cudaGetLastError());
            if (mode) {
                ho.pos.ensure((size_t)m * 8);
                ho.best.ensure((size_t)n_ids * 8);
                B200_CUDA(cudaMemsetAsync(ho.best.p, 0, (size_t)n_ids * 8, stream));
                const int64_t n_runs = (int64_t)ho.scan.run(ho.flag.as<uint32_t>(), m, ho.pos.as<unsigned long long>(), stream, &launches);
                ho.start.ensure((size_t)n_runs * 4);
                holistic_run_start_kernel<<<grid_for(m), 256, 0, stream>>>(ho.flag.as<uint32_t>(), ho.pos.as<unsigned long long>(), m, ho.start.as<uint32_t>());
                holistic_run_best_kernel<<<grid_for(n_runs), 256, 0, stream>>>(hs, ho.start.as<uint32_t>(), n_runs, ho.best.as<unsigned long long>());
                launches += 2;
                B200_CUDA(cudaGetLastError());
            }
            HoEvalArgs e{};
            e.s = hs; e.gid = d_a0[ho.p0].as<unsigned long long>(); e.n_slots = cap + 2;
            e.head = ho.head.as<uint32_t>(); e.tail = ho.tail.as<uint32_t>(); e.best = mode ? ho.best.as<unsigned long long>() : nullptr;
            for (size_t k = 0; k < ho.outs.size(); k++) {
                const HoOut& h = ho.outs[k];
                if (h.store != (int)i) continue;
                const int p = ho.p0 + 1 + (int)k;
                e.kind[e.n_f] = h.kind; e.q[e.n_f] = h.q;
                e.res[e.n_f] = d_a0[p].as<unsigned long long>(); e.seen[e.n_f] = d_a1[p].as<unsigned long long>();
                e.n_f++;
            }
            holistic_eval_kernel<<<grid_for((int64_t)cap + 2), 256, 0, stream>>>(e);
            launches++;
            B200_CUDA(cudaGetLastError());
        }
    }

    void consume(const b200_table* t) {
        B200_REQUIRE(!build_done, "b200 groupby: consume after the build was finished");
        B200_REQUIRE(t->n_cols == n_cols, "b200 groupby: batch has a different number of columns than the build schema");
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        int64_t n = t->n_rows;
        std::vector<bool> used(n_cols, false);
        for (int kc = 0; kc < nk; kc++) used[kc] = true;
        for (auto& f : funcs) if (f.in_col >= 0) used[f.in_col] = true;
        if (mr.on) {
            B200_REQUIRE(n_pes == 1, "b200 groupby: a sharded min_row_number_filter is not supported (n_pes > 1); run it on one rank");
            ensure_candidate_room(n);  // (before anything reads the batch)
            for (int j = 0; j < mr.n_sort; j++) used[mr.sort_col[j]] = true;
            for (int c : mr.keep) used[c] = true;
        }
        if (ho.on) ensure_holistic_room(n);  // (before anything reads the batch)
        for (int c = 0; c < n_cols; c++) {
            if (!used[c]) continue;
            B200_REQUIRE(t->cols[c].c_type == in_types[c], "b200 groupby: batch column dtype differs from the build schema");
            B200_REQUIRE(n == 0 || t->cols[c].data != nullptr, "b200 groupby: null data pointer");
        }
        for (auto& ni : nu_inner) {  // nunique: the (key, value) pairs of this batch go to the nested distinct state
            b200_column pc[2] = {t->cols[0], t->cols[ni.in_col]};
            b200_table pt{};
            pt.n_cols = 2; pt.n_rows = n; pt.cols = pc; pt.device = t->device;
            ni.st->consume(&pt);
            B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        }
        if (coalesce(t, n)) return;  // small batch of the fast-path signature: buffered until a launch is worth it
        flush_coalesced();
        if (t->device >= 0) {
            B200_REQUIRE(t->device == device, "b200 groupby: batch lives on a different device than the state");
            for (int64_t r0 = 0; r0 < n; r0 += CHUNK_ROWS) {
                int64_t rows = std::min(CHUNK_ROWS, n - r0);
                B200_REQUIRE(r0 % 8 == 0, "internal: chunk offset must be byte aligned for validity bitmaps");
                std::vector<const void*> data(n_cols, nullptr);
                std::vector<const uint8_t*> valid(n_cols, nullptr);
                for (int c = 0; c < n_cols; c++) {
                    if (!used[c]) continue;
                    data[c] = (const char*)t->cols[c].data + r0 * ctype_size(in_types[c]);
                    valid[c] = t->cols[c].validity ? t->cols[c].validity + r0 / 8 : nullptr;
                }
                consume_chunk(data, valid, rows);
            }
            return;
        }
        // host batch: pinned or pageable host memory, staged through two device buffers per column so the
        // H2D copy of chunk c+1 overlaps the kernel of chunk c (replaces convertTableToGPU,
        // bodo/pandas/physical/operator.cpp:293-380).
        const int64_t HCHUNK = 1ll << 24;  // 16 Mi rows (128 MiB per 8-byte column)
        if (!copy_stream) {
            B200_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
            for (int b = 0; b < 2; b++) {
                B200_CUDA(cudaEventCreateWithFlags(&stage_free[b], cudaEventDisableTiming));
                B200_CUDA(cudaEventCreateWithFlags(&stage_ready[b], cudaEventDisableTiming));
                stage[b].resize(2 * n_cols);
            }
        }
        int64_t nchunks = (n + HCHUNK - 1) / HCHUNK;
        for (int64_t ci = 0; ci < nchunks; ci++) {
            int b = (int)(ci & 1);
            int64_t r0 = ci * HCHUNK, rows = std::min(HCHUNK, n - r0);
            if (stage_recorded[b]) B200_CUDA(cudaStreamWaitEvent(copy_stream, stage_free[b], 0));
            std::vector<const void*> data(n_cols, nullptr);
            std::vector<const uint8_t*> valid(n_cols, nullptr);
            for (int c = 0; c < n_cols; c++) {
                if (!used[c]) continue;
                size_t isz = ctype_size(in_types[c]);
                stage[b][2 * c].ensure((size_t)std::min(HCHUNK, n) * isz);
                B200_CUDA(cudaMemcpyAsync(stage[b][2 * c].p, (const char*)t->cols[c].data + r0 * isz, rows * isz, cudaMemcpyHostToDevice, copy_stream));
                data[c] = stage[b][2 * c].p;
                if (t->cols[c].validity) {
                    stage[b][2 * c + 1].ensure((size_t)(std::min(HCHUNK, n) + 7) / 8 + 8);
                    B200_CUDA(cudaMemcpyAsync(stage[b][2 * c + 1].p, t->cols[c].validity + r0 / 8, (rows + 7) / 8, cudaMemcpyHostToDevice, copy_stream));
                    valid[c] = stage[b][2 * c + 1].as<uint8_t>();
                }
            }
            B200_CUDA(cudaEventRecord(stage_ready[b], copy_stream));
            B200_CUDA(cudaStreamWaitEvent(stream, stage_ready[b], 0));
            consume_chunk(data, valid, rows);
            B200_CUDA(cudaEventRecord(stage_free[b], stream));
            stage_recorded[b] = true;
        }
    }

    // ---- coalescing of small streaming batches ----
    // The reference streams 32 768-row batches (bodo/libs/streaming/_shuffle.h:27-31); the SM-partitioned and low-cardinality
    // kernels want >= 2^20 rows per launch.  Batches of the fast-path signature (non-null int64 or float key, SUM / COUNT / SIZE over
    // one non-null int64 value column) below that size are appended to a device-side buffer (one D2D or H2D copy per column) and
    // consumed together when the buffer is full, when a batch of another shape arrives, or when the build ends.
    static constexpr int64_t CO_MIN_BATCH = 1ll << 20, CO_ROWS = 1ll << 22;
    DevBuf co_key, co_val;
    int64_t co_n = 0, co_batches = 0;
    int co_vcol = -1;
    bool coalesce(const b200_table* t, int64_t n) {
        if (mr.on || ho.on) return false;
        if (n == 0 || n >= CO_MIN_BATCH || nk != 1 || n_funcs < 1 || c_types[0] != CT_INT64 || t->cols[0].validity != nullptr) return false;
        { const char* e = getenv("B200_COALESCE"); if (e && e[0] == '0') return false; }
        int vcol = -1;
        for (auto& f : funcs) {
            if (f.kind == K_SIZE) continue;
            if (!((f.kind == K_SUM_I64 || f.kind == K_COUNT) && f.in_ctype == CT_INT64 && t->cols[f.in_col].validity == nullptr)) return false;
            if (vcol >= 0 && vcol != f.in_col) return false;
            vcol = f.in_col;
        }
        if (!spg_probe()) return false;
        if (co_n > 0 && (co_vcol != vcol || co_n + n > CO_ROWS)) flush_coalesced();
        co_vcol = vcol;
        co_key.ensure((size_t)CO_ROWS * 8);
        if (vcol >= 0) co_val.ensure((size_t)CO_ROWS * 8);
        const cudaMemcpyKind kind = t->device >= 0 ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if (t->device >= 0) B200_REQUIRE(t->device == device, "b200 groupby: batch lives on a different device than the state");
        if (float_key(0)) {  // the buffer holds canonical keys (a host batch is copied over first)
            const void* k = t->cols[0].data;
            if (kind == cudaMemcpyHostToDevice) {
                const size_t kb = (size_t)n * ctype_size(in_types[0]);
                d_canon[0].ensure(kb);
                B200_CUDA(cudaMemcpyAsync(d_canon[0].p, k, kb, kind, stream));
                k = d_canon[0].p;
            }
            canon_launch(k, in_types[0], co_key.as<long long>() + co_n, n);
        } else
            B200_CUDA(cudaMemcpyAsync(co_key.as<long long>() + co_n, t->cols[0].data, (size_t)n * 8, kind, stream));
        if (vcol >= 0) B200_CUDA(cudaMemcpyAsync(co_val.as<long long>() + co_n, t->cols[vcol].data, (size_t)n * 8, kind, stream));
        if (kind == cudaMemcpyHostToDevice) B200_CUDA(cudaStreamSynchronize(stream));  // the caller may reuse its host batch right away
        co_n += n;
        co_batches++;
        if (co_n + CO_MIN_BATCH > CO_ROWS) flush_coalesced();
        return true;
    }
    void flush_coalesced() {
        if (co_n == 0) return;
        std::vector<const void*> data(n_cols, nullptr);
        std::vector<const uint8_t*> valid(n_cols, nullptr);
        data[0] = co_key.p;
        if (co_vcol >= 0) data[co_vcol] = co_val.p;
        const int64_t n = co_n;
        co_n = 0;
        consume_device_chunk(data, valid, n);
    }

    // ---- finalize ----
    // Compacts the occupied slots (sharded: of the groups this rank owns).  No host synchronisation: the output is sized by
    // the table's group limit (cap / 2 + the two special slots), the count stays on the device (counters[CTR_OUT]).
    int64_t max_out_bound() const { return (int64_t)(cap / 2) + 2; }
    void compact() {
        int64_t max_out = max_out_bound();
        d_slot_of_out.ensure((size_t)max_out * 8);
        B200_CUDA(cudaMemsetAsync((char*)d_counters.p + CTR_OUT * 8, 0, 8, stream));
        if (nk > 1)
            compact_mk_kernel<<<grid_for((int64_t)cap), 256, 0, stream>>>(d_tags.as<unsigned long long>(), cap, d_counters.as<long long>() + CTR_OUT, d_slot_of_out.as<uint64_t>(),
                                                                           mk_owner());
        else
            compact_slots_kernel<<<grid_for((int64_t)cap + 2), 256, 0, stream>>>(d_keys.as<long long>(), cap, d_counters.as<long long>(),
                                                                                      d_counters.as<long long>() + CTR_OUT, d_slot_of_out.as<uint64_t>(),
                                                                                      n_pes, rank, in_types[0], dropna);
        launches++;
        B200_CUDA(cudaGetLastError());
        n_out = -1;  // known on the device (counters[CTR_OUT]); the host learns it with the next counter read-back
    }

    // nunique: count the distinct (key, value) pairs of every nested state into the outer table.  On the sharded path the host
    // has exchanged the nested states first (their pairs are owned where the key is owned) and the outer table already holds
    // the groups this rank owns.
    void apply_nunique() {
        if (nu_applied || nu_inner.empty()) return;
        for (auto& ni : nu_inner) {
            GroupbyState& in = *ni.st;
            // (a holistic state consumes only rows of groups it owns, so its nested states hold only pairs they own: no exchange)
            B200_REQUIRE(n_pes == 1 || in.exchanged || ho.on, "b200 groupby: nunique on the sharded path: exchange the nested states (b200_groupby_inner_state) before the outer finalize");
            const int64_t n_pairs = in.finalize();
            B200_REQUIRE(n_pairs >= 0, "b200 groupby: nunique: the nested state's fused exchange overflowed its slab; exchange it in the NCCL form first");
            B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
            if (n_pairs == 0) continue;
            NuniqueArgs a{};
            a.pk = in.d_mk[0].as<long long>(); a.pv = in.d_mk[1].as<long long>(); a.pmask = in.d_mkmask.as<unsigned char>();
            a.slot_of_out = in.d_slot_of_out.as<uint64_t>(); a.n_pairs = n_pairs;
            a.tkeys = d_keys.as<long long>(); a.cap = cap; a.counters = d_counters.as<long long>(); a.dropna = dropna ? 1 : 0;
            a.n_acc = (int)ni.prims.size();
            for (int j = 0; j < a.n_acc; j++) a.acc[j] = d_a0[ni.prims[j]].as<unsigned long long>();
            a.value_float = in.float_key(1) ? 1 : 0;
            nunique_count_kernel<<<grid_for(n_pairs), 256, 0, stream>>>(a);
            launches++;
            B200_CUDA(cudaGetLastError());
        }
        nu_applied = true;
    }

    int64_t finalize() {
        if (finalized) return n_out;
        ScopedTimer timer{t_finalize};
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        if (mr.on) return finalize_mrnf();
        flush_coalesced();
        // the exchange settles first, so that nunique also counts into the groups it brought
        if (exchanged && !settle_exchange()) return -2;
        apply_nunique();
        if (ho.on) finalize_holistic();
        compact();
        const int64_t max_out = max_out_bound();
        EvalArgs e{};
        e.tkeys = nk == 1 ? d_keys.as<long long>() : nullptr; e.cap = cap; e.slot_of_out = d_slot_of_out.as<uint64_t>(); e.n_out_ptr = d_counters.as<long long>() + CTR_OUT;
        e.key_ctype = in_types[0];
        size_t words = (size_t)((max_out + 31) / 32 + 1);
        if (nk == 1) {
            d_out_keys.ensure((size_t)(max_out + 32) * ctype_size(in_types[0]));
            e.out_keys = d_out_keys.p;
            bool key_nullable = arr_types[0] == ARR_NULLABLE;
            if (key_nullable) { d_out_key_valid.ensure(words * 4); e.out_key_valid = d_out_key_valid.as<uint32_t>(); }
        } else {
            EvalMkKeysArgs k{};
            k.nk = nk; k.mkmask = d_mkmask.as<unsigned char>(); k.slot_of_out = d_slot_of_out.as<uint64_t>(); k.n_out_ptr = d_counters.as<long long>() + CTR_OUT;
            for (int j = 0; j < nk; j++) {
                k.mk[j] = d_mk[j].as<long long>(); k.key_ctype[j] = in_types[j];
                d_out_mk[j].ensure((size_t)(max_out + 32) * ctype_size(in_types[j]));
                k.out_keys[j] = d_out_mk[j].p;
                if (arr_types[j] == ARR_NULLABLE) { d_out_mk_valid[j].ensure(words * 4); k.out_key_valid[j] = d_out_mk_valid[j].as<uint32_t>(); }
            }
            eval_mk_keys_kernel<<<grid_for(max_out), 256, 0, stream>>>(k);
            launches++;
        }
        e.n_ops = n_outs;
        for (int j = 0; j < n_outs; j++) {
            const OutSpec& o = outs[j];
            const int p0 = o.prim[0];
            d_out_data[j].ensure((size_t)(max_out + 32) * 8);
            e.ops[j].kind = o.kind; e.ops[j].out_ctype = o.out_ctype; e.ops[j].a0 = d_a0[p0].p;
            e.ops[j].a1 = funcs[p0].has_a1 ? d_a1[p0].p : nullptr; e.ops[j].out_data = d_out_data[j].p;
            e.ops[j].b0 = o.n_prim > 1 ? d_a0[o.prim[1]].p : nullptr;
            e.ops[j].c0 = o.n_prim > 2 ? d_a0[o.prim[2]].p : nullptr;
            e.ops[j].d0 = o.n_prim > 3 ? d_a0[o.prim[3]].p : nullptr;
            if (o.out_arrtype == ARR_NULLABLE) { d_out_valid[j].ensure(words * 4); e.ops[j].out_valid = d_out_valid[j].as<uint32_t>(); }
        }
        eval_output_kernel<<<grid_for(max_out), 256, 0, stream>>>(e);
        launches++;
        B200_CUDA(cudaGetLastError());
        read_counters();  // one synchronisation: the output is complete and n_out is known
        n_out = h_counters[CTR_OUT];
        finalized = true;
        out_cursor = 0;
        return n_out;
    }

    MkOwner mk_owner() {
        MkOwner o{};
        o.nk = nk; o.n_pes = n_pes; o.rank = rank; o.mkmask = d_mkmask.as<unsigned char>(); o.own_nk = owner_nk;
        for (int j = 0; j < nk; j++) {
            o.mk[j] = d_mk[j].as<long long>(); o.key_ctype[j] = in_types[j];
            if (dropna && float_key(j)) o.drop_nan |= 1u << j;
        }
        return o;
    }
    MkArgs mk_table_args() {
        MkArgs a{};
        a.nk = nk; a.tags = d_tags.as<unsigned long long>(); a.mkmask = d_mkmask.as<unsigned char>(); a.cap = cap;
        for (int j = 0; j < nk; j++) a.mk[j] = d_mk[j].as<long long>();
        a.counters = d_counters.as<long long>(); a.group_limit = (long long)(cap / 2); a.fail_list = d_fail.as<uint32_t>();
        return a;
    }

    // ---- exchange of partial aggregates (see xchg_pack_kernel) ----
    bool exchanged = false;  // a combine ran: finalize settles it from xchg_src, which the caller keeps alive until then
    XchgSource xchg_src{};
    int64_t xchg_max_rows = 0;
    DevBuf d_xchg_cursors, d_xchg_dest, d_xchg_hdr;
    std::vector<int64_t> h_xchg_counts;  // rows per destination of the last pack (exchange_counts)
    SlotTable slot_table() {
        SlotTable t{};
        t.tkeys = d_keys.as<long long>(); t.cap = cap; t.counters = d_counters.as<long long>(); t.group_limit = (long long)(cap / 2);
        t.key_ctype = in_types[0];
        return t;
    }
    TagTable tag_table() {
        TagTable t{};
        t.nk = nk; t.tags = d_tags.as<unsigned long long>(); t.mkmask = d_mkmask.as<unsigned char>(); t.cap = cap;
        for (int j = 0; j < nk; j++) t.mk[j] = d_mk[j].as<long long>();
        t.counters = d_counters.as<long long>(); t.group_limit = (long long)(cap / 2); t.ow = mk_owner();
        return t;
    }
    int acc_count() const { int n = 0; for (auto& f : funcs) n += f.has_a1 ? 2 : 1; return n; }
    int64_t xchg_row_bytes() const { return (int64_t)(nk + 1 + acc_count()) * 8; }
    CombineArgs combine_args(const XchgSource& src) {
        CombineArgs c{};
        c.src = src; c.row_words = (int)(xchg_row_bytes() / 8); c.fail_list = d_fail.as<uint32_t>(); c.n_ops = n_funcs;
        for (int j = 0; j < n_funcs; j++) { c.kinds[j] = funcs[j].kind; c.a0[j] = d_a0[j].p; c.a1[j] = funcs[j].has_a1 ? d_a1[j].p : nullptr; }
        return c;
    }
    // a source of n_seg segments back to back whose counts the host knows (copied into a small device header; a copy from
    // pageable memory is staged before the call returns)
    XchgSource host_source(const void* rows, const int64_t* counts, int n_seg) {
        d_xchg_hdr.ensure((size_t)std::max(n_seg, 32) * 8);
        B200_CUDA(cudaMemcpyAsync(d_xchg_hdr.p, counts, (size_t)n_seg * 8, cudaMemcpyHostToDevice, stream));
        XchgSource src{};
        src.rows = (const unsigned long long*)rows; src.hdr = d_xchg_hdr.as<unsigned long long>(); src.n_seg = n_seg;
        return src;
    }

    // Stores every group another rank owns as one wire row into that rank's region: fused (peer_slabs_dev: the device array of
    // every rank's slab) segment `rank` of the owner's slab, cap_rows rows, then posts the counts into the peers' headers; NCCL
    // (send_buf) the rows of destination d at the exclusive prefix of the counts of the previous pack; neither: count only.
    void exchange_pack(void* const* peer_slabs_dev, int64_t cap_rows, void* send_buf) {
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        B200_REQUIRE(!mr.on, "b200 groupby: a sharded min_row_number_filter is not supported (no exchange of winner records)");
        B200_REQUIRE(!ho.on, "b200 groupby: mode / percentile_cont / percentile_disc do not combine as partial aggregates; a sharded state "
                             "consumes rows hash-partitioned by key (each rank only its own groups) and finalizes without an exchange");
        flush_coalesced();
        build_done = true;
        const size_t cursor_bytes = (size_t)std::max(n_pes, 32) * 8;
        d_xchg_cursors.ensure(cursor_bytes);
        B200_CUDA(cudaMemsetAsync(d_xchg_cursors.p, 0, cursor_bytes, stream));
        XchgPackArgs p{};
        p.n_pes = n_pes; p.rank = rank; p.n_acc = wire_accs(d_a0, d_a1, p.acc); p.row_words = nk + 1 + p.n_acc;
        p.cursors = d_xchg_cursors.as<unsigned long long>();
        if (peer_slabs_dev) {
            p.dest = peer_slabs_dev; p.dest_offset = XCHG_HDR_BYTES + (long long)rank * cap_rows * p.row_words * 8; p.cap_rows = cap_rows;
        } else if (send_buf) {
            B200_REQUIRE((int)h_xchg_counts.size() == n_pes, "b200 groupby: packing into a send buffer needs the counts of a previous pack (b200_groupby_exchange_counts)");
            // the table has not changed since that pack, so destination d gets exactly h_xchg_counts[d] rows again
            std::vector<void*> dest(n_pes);
            int64_t run = 0;
            for (int d = 0; d < n_pes; d++) {
                dest[d] = (char*)send_buf + run * p.row_words * 8;
                run += h_xchg_counts[d];
                p.cap_rows = std::max<long long>(p.cap_rows, h_xchg_counts[d]);
            }
            d_xchg_dest.ensure((size_t)n_pes * 8);
            B200_CUDA(cudaMemcpyAsync(d_xchg_dest.p, dest.data(), (size_t)n_pes * 8, cudaMemcpyHostToDevice, stream));
            p.dest = d_xchg_dest.as<void*>();
        }
        if (nk > 1) xchg_pack_kernel<<<grid_for((int64_t)cap), 256, 0, stream>>>(tag_table(), p);
        else xchg_pack_kernel<<<grid_for((int64_t)cap + 2), 256, 0, stream>>>(slot_table(), p);
        launches++;
        if (peer_slabs_dev) { xchg_post_counts_kernel<<<1, 32, 0, stream>>>(p.cursors, peer_slabs_dev, n_pes, rank, cap_rows); launches++; }
        B200_CUDA(cudaGetLastError());
        if (send_buf) B200_CUDA(cudaStreamSynchronize(stream));  // the caller moves the rows on its own stream
    }
    // exact rows per destination of the last pack (whether or not they fitted)
    void exchange_counts(int64_t* counts) {
        B200_CUDA(cudaSetDevice(device));
        B200_REQUIRE(d_xchg_cursors.p != nullptr, "b200 groupby: exchange counts before any exchange pack");
        h_xchg_counts.resize(n_pes);
        B200_CUDA(cudaMemcpyAsync(h_xchg_counts.data(), d_xchg_cursors.p, (size_t)n_pes * 8, cudaMemcpyDeviceToHost, stream));
        B200_CUDA(cudaStreamSynchronize(stream));
        std::copy(h_xchg_counts.begin(), h_xchg_counts.end(), counts);
    }
    // Merges the received rows: fused (recv_counts == nullptr) the own slab, segment s at row s * cap_rows with its count in the
    // slab header; NCCL the receive buffer, segments back to back with the host's recv_counts.
    void exchange_combine(const void* rows, int64_t cap_rows, const int64_t* recv_counts) {
        B200_CUDA(cudaSetDevice(device)); scratch_set_stream(stream);
        XchgSource src{};
        int64_t max_rows = 0;
        if (recv_counts) {
            for (int s = 0; s < n_pes; s++) max_rows += recv_counts[s];
            src = host_source(rows, recv_counts, n_pes);
        } else {
            src.rows = (const unsigned long long*)((const char*)rows + XCHG_HDR_BYTES); src.hdr = (const unsigned long long*)rows;
            src.n_seg = n_pes; src.seg_rows = cap_rows;
            max_rows = (int64_t)n_pes * cap_rows;
        }
        B200_REQUIRE(max_rows < (1ll << 32), "b200 groupby: too many partial rows in one exchange");
        combine(src, max_rows);
        if (has_firstlast) firstlast_fix(src, max_rows);
        xchg_src = src; xchg_max_rows = max_rows; exchanged = true;
    }
    void combine(const XchgSource& src, int64_t max_rows) {
        d_fail.ensure(device, (size_t)max_rows * 4);
        const CombineArgs c = combine_args(src);
        if (nk > 1) xchg_combine_kernel<<<grid_for(max_rows), 256, 0, stream>>>(tag_table(), c);
        else xchg_combine_kernel<<<grid_for(max_rows), 256, 0, stream>>>(slot_table(), c);
        launches++;
        B200_CUDA(cudaGetLastError());
    }
    void firstlast_fix(const XchgSource& src, int64_t max_rows) {
        combine_firstlast_fix_kernel<<<grid_for(max_rows), 256, 0, stream>>>(slot_table(), combine_args(src));
        launches++;
        B200_CUDA(cudaGetLastError());
    }
    // After a combine: false when some rank's share did not fit its slab segment (nobody combined, the tables are intact: the
    // NCCL form takes over).  Otherwise the rows that found the table at its group limit are merged after it grew.
    bool settle_exchange() {
        read_counters();
        if (h_counters[CTR_XCHG_OVERFLOW] != 0) {
            B200_CUDA(cudaMemsetAsync((char*)d_counters.p + CTR_XCHG_OVERFLOW * 8, 0, 8, stream));
            exchanged = false;
            return false;
        }
        if (h_counters[CTR_FAIL] == 0) return true;
        settle<uint32_t>(d_fail, 1, fail_rows, [&](const uint32_t* list, int64_t nf) {
            XchgSource replay = xchg_src;
            replay.index_list = list; replay.n_index = nf;
            combine(replay, nf);
        });
        if (has_firstlast) firstlast_fix(xchg_src, xchg_max_rows);  // over the whole source again (idempotent): the table moved
        return true;
    }

    int produce(b200_table* out, int32_t* out_is_last, bool produce_output) {
        if (!finalized && finalize() == -2)
            throw Error("b200 groupby: the fused exchange overflowed its slab; run the NCCL form of the exchange (exchange counts, pack into a send buffer, combine) and finalize again before producing output");
        int64_t bs = output_batch_size > 0 ? output_batch_size : n_out;
        if (bs % 32 != 0 && bs < n_out) bs = (bs + 31) & ~31ll;  // validity bitmaps are sliced at word granularity
        int64_t rows = produce_output ? std::min(bs, n_out - out_cursor) : 0;
        B200_REQUIRE(out->cols != nullptr, "b200 groupby: out->cols must point to n_keys + n_funcs descriptors");
        out->n_rows = rows; out->n_cols = nk + n_outs; out->device = device;
        int64_t off = out_cursor;
        if (mr.on) {  // the kept columns only
            out->n_cols = (int32_t)mr.keep.size();
            for (size_t j = 0; j < mr.keep.size(); j++) {
                const int c = mr.keep[j];
                b200_column& k = out->cols[j];
                k.data = (char*)d_out_data[j].p + off * ctype_size(in_types[c]);
                k.validity = arr_types[c] == ARR_NULLABLE ? d_out_valid[j].as<uint8_t>() + off / 8 : nullptr;
                k.length = rows; k.c_type = in_types[c]; k.arr_type = arr_types[c];
            }
            out_cursor += rows;
            *out_is_last = out_cursor >= n_out ? 1 : 0;
            return 0;
        }
        for (int kc = 0; kc < nk; kc++) {
            b200_column& k = out->cols[kc];
            const DevBuf& kd = nk == 1 ? d_out_keys : d_out_mk[kc];
            const DevBuf& kv = nk == 1 ? d_out_key_valid : d_out_mk_valid[kc];
            k.data = (char*)kd.p + off * ctype_size(in_types[kc]);
            k.validity = arr_types[kc] == ARR_NULLABLE ? kv.as<uint8_t>() + off / 8 : nullptr;
            k.length = rows; k.c_type = in_types[kc]; k.arr_type = arr_types[kc];
        }
        for (int j = 0; j < n_outs; j++) {
            b200_column& c = out->cols[nk + j];
            c.data = (char*)d_out_data[j].p + off * ctype_size(outs[j].out_ctype);
            c.validity = outs[j].out_arrtype == ARR_NULLABLE ? d_out_valid[j].as<uint8_t>() + off / 8 : nullptr;
            c.length = rows; c.c_type = outs[j].out_ctype; c.arr_type = outs[j].out_arrtype;
        }
        out_cursor += rows;
        *out_is_last = out_cursor >= n_out ? 1 : 0;
        return 0;
    }
};

}  // namespace b200

using b200::GroupbyState;

#define B200_TRY try {
#define B200_CATCH(retval)                              \
    }                                                   \
    catch (const std::exception& e) {                   \
        b200::set_last_error(e.what());                 \
        return retval;                                  \
    }

extern "C" {

void* b200_groupby_state_init(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                              int32_t n_build_arrs, const int32_t* ftypes, const int32_t* f_in_offsets,
                              const int32_t* f_in_cols, int32_t n_funcs, uint64_t n_keys, int64_t output_batch_size,
                              int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                              int64_t expected_groups, void* stream) {
    return b200_groupby_state_init_percentiles(operator_id, build_arr_c_types, build_arr_array_types, n_build_arrs, ftypes, f_in_offsets,
                                               f_in_cols, n_funcs, n_keys, output_batch_size, parallel, pandas_drop_na, device, n_pes, myrank,
                                               expected_groups, stream, nullptr);
}

void* b200_groupby_state_init_percentiles(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                          int32_t n_build_arrs, const int32_t* ftypes, const int32_t* f_in_offsets,
                                          const int32_t* f_in_cols, int32_t n_funcs, uint64_t n_keys, int64_t output_batch_size,
                                          int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                          int64_t expected_groups, void* stream, const double* fractions) {
    (void)operator_id;
    B200_TRY
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        throw b200::Error("b200 groupby: no CUDA device available (this path has no CPU fallback)");
    B200_REQUIRE(device >= 0 && device < ndev, "b200 groupby: bad device ordinal");
    return new GroupbyState(build_arr_c_types, build_arr_array_types, n_build_arrs, ftypes, f_in_offsets, f_in_cols, n_funcs,
                            n_keys, output_batch_size, parallel != 0, pandas_drop_na != 0, device, n_pes, myrank,
                            expected_groups, (cudaStream_t)stream, nullptr, fractions);
    B200_CATCH(nullptr)
}

void* b200_groupby_state_init_mrnf(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                   int32_t n_build_arrs, uint64_t n_keys, const int32_t* sort_cols, const int32_t* sort_ascending,
                                   const int32_t* sort_na_last, int32_t n_sort, const int32_t* keep, int64_t output_batch_size,
                                   int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                   int64_t expected_groups, void* stream) {
    return b200_groupby_state_init_mrnf_limit(operator_id, build_arr_c_types, build_arr_array_types, n_build_arrs, n_keys, sort_cols, sort_ascending,
                                              sort_na_last, n_sort, keep, output_batch_size, parallel, pandas_drop_na, device, n_pes, myrank,
                                              expected_groups, stream, 1);
}

void* b200_groupby_state_init_mrnf_limit(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                         int32_t n_build_arrs, uint64_t n_keys, const int32_t* sort_cols, const int32_t* sort_ascending,
                                         const int32_t* sort_na_last, int32_t n_sort, const int32_t* keep, int64_t output_batch_size,
                                         int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                         int64_t expected_groups, void* stream, int64_t rows_per_group) {
    (void)operator_id;
    B200_TRY
    B200_REQUIRE(build_arr_c_types && build_arr_array_types && keep && (n_sort <= 0 || (sort_cols && sort_ascending && sort_na_last)),
                 "b200 groupby: null min_row_number_filter argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        throw b200::Error("b200 groupby: no CUDA device available (this path has no CPU fallback)");
    B200_REQUIRE(device >= 0 && device < ndev, "b200 groupby: bad device ordinal");
    const int32_t no_off[1] = {0};
    const b200::MrnfSpec spec{n_sort, sort_cols, sort_ascending, sort_na_last, keep, rows_per_group};
    return new GroupbyState(build_arr_c_types, build_arr_array_types, n_build_arrs, nullptr, no_off, nullptr, 0, n_keys,
                            output_batch_size, parallel != 0, pandas_drop_na != 0, device, n_pes, myrank, expected_groups,
                            (cudaStream_t)stream, &spec);
    B200_CATCH(nullptr)
}

int b200_groupby_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last, int32_t is_final_pipeline,
                                     int32_t* request_input) {
    (void)is_final_pipeline;
    B200_TRY
    B200_REQUIRE(state && in_table, "b200 groupby: null state or table");
    auto* s = (GroupbyState*)state;
    s->consume(in_table);
    if (request_input) *request_input = 1;
    if (is_last && !s->parallel) s->build_done = true;
    return is_last ? 1 : 0;
    B200_CATCH(-1)
}

int64_t b200_groupby_exchange_row_bytes(void* state) { return ((GroupbyState*)state)->xchg_row_bytes(); }
int b200_groupby_exchange_pack(void* state, void* const* peer_slabs_dev, int64_t cap_rows, void* send_buf) {
    B200_TRY
    B200_REQUIRE(state && !(peer_slabs_dev && send_buf) && (!peer_slabs_dev || cap_rows > 0), "b200 groupby: bad exchange pack arguments");
    ((GroupbyState*)state)->exchange_pack(peer_slabs_dev, cap_rows, send_buf);
    return 0;
    B200_CATCH(-1)
}
int b200_groupby_exchange_counts(void* state, int64_t* send_row_counts) {
    B200_TRY
    B200_REQUIRE(state && send_row_counts, "b200 groupby: null argument");
    ((GroupbyState*)state)->exchange_counts(send_row_counts);
    return 0;
    B200_CATCH(-1)
}
int b200_groupby_exchange_combine(void* state, const void* rows, int64_t cap_rows, const int64_t* recv_row_counts) {
    B200_TRY
    B200_REQUIRE(state && (rows || recv_row_counts) && (recv_row_counts || cap_rows > 0), "b200 groupby: bad exchange combine arguments");
    ((GroupbyState*)state)->exchange_combine(rows, cap_rows, recv_row_counts);
    return 0;
    B200_CATCH(-1)
}
int32_t b200_groupby_num_inner_states(void* state) { return state ? (int32_t)((GroupbyState*)state)->nu_inner.size() : 0; }
void* b200_groupby_inner_state(void* state, int32_t i) {
    auto* s = (GroupbyState*)state;
    if (!s || i < 0 || i >= (int32_t)s->nu_inner.size()) { b200::set_last_error("b200_groupby_inner_state: bad arguments"); return nullptr; }
    return s->nu_inner[i].st.get();
}

int64_t b200_groupby_finalize(void* state) {
    B200_TRY
    return ((GroupbyState*)state)->finalize();
    B200_CATCH(-1)
}
int b200_groupby_produce_output_batch(void* state, b200_table* out, int32_t* out_is_last, int32_t produce_output) {
    B200_TRY
    B200_REQUIRE(state && out && out_is_last, "b200 groupby: null argument");
    return ((GroupbyState*)state)->produce(out, out_is_last, produce_output != 0);
    B200_CATCH(-1)
}
void b200_delete_groupby_state(void* state) { delete (GroupbyState*)state; }

int64_t b200_groupby_get_metric(void* state, int32_t which) {
    auto* s = (GroupbyState*)state;
    switch (which) {
        case 0: return s->finalized ? s->n_out : s->n_groups;
        case 1: return (int64_t)s->cap;
        case 2: return s->rows_consumed;
        case 3: return s->rebuilds;
        case 4: return s->launches;
        case 5: return s->fail_rows;
        case 6: return (int64_t)s->consume_kernel_us();
        case 7: return s->consume_launches;
        case 8: return s->spg_launches;
        case 9: return s->spg_retry_rows;
        case 10: return s->lc_launches;
        case 11: return s->co_batches;
        case 12: return s->spgg_launches;
        case 14: return s->spgn_launches;
        case 15: return s->spg16_launches;
        case 16: return s->spg_n_hot;
        case 17: return s->spgd_launches;
        case 18: return s->mt.admitted;
        case 19: return s->mt.reduces;
        case 20: { cudaSetDevice(s->device); return s->ho.on ? s->holistic_rows() : 0; }  // exact (synchronises the stream)
        case 21: return s->ho.passes;
        case 13: { cudaSetDevice(s->device); s->read_counters(); return s->n_groups; }  // exact (synchronises the stream)
        case 100: s->profiling = true; return 0;
        default: return -1;
    }
}

}  // extern "C"
