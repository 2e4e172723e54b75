// expr.cu — fused filter + projection front end of the aggregate / join pipelines (sm_90a).
//
// Replaces PhysicalFilter + PhysicalProjection with their expression trees (bodo/pandas/physical/filter.h, project.h,
// expression.{h,cpp}; GPU twins: cudf::ast expressions + cudf::apply_boolean_mask, gpu_expression.cpp:601+, gpu_filter.h:143)
// for the fixed-width column kinds of this path: ONE kernel evaluates the predicate and every output expression of a row,
// compacts the surviving rows (warp ballot -> CTA scan -> one cursor atomic per 1024-row tile) and writes the output columns
// (pass-through or computed) densely — the filtered intermediate table never exists in HBM.
//
// Expressions are postfix programs over a per-thread value stack (numbers as double or int64 with a validity flag):
// column loads, constants, + - * /, comparisons, and / or / not, casts.  Null semantics are the reference's (Arrow compute /
// pandas nullable): arithmetic and comparisons propagate null, a null predicate drops the row, `and` / `or` are Kleene.
// The same lookup kernel serves dictionary unification (remap_i32: batch-local dictionary indices -> global ids, the
// transpose step of DictionaryBuilder::UnifyDictionaryArray, bodo/libs/_dict_builder.cpp).
#include <vector>

#include "common.cuh"

namespace b200 {

enum ExprOp : int32_t {
    EX_COL = 0,      // push column arg
    EX_CONST_I64,    // push int64 constant (arg bits)
    EX_CONST_F64,    // push double constant (arg bits)
    EX_ADD, EX_SUB, EX_MUL, EX_DIV,
    EX_LT, EX_LE, EX_GT, EX_GE, EX_EQ, EX_NE,
    EX_AND, EX_OR, EX_NOT,
    EX_TO_F64, EX_TO_I64,
    EX_IS_NULL, EX_NEG,
    EX_END
};
constexpr int EX_MAX_INSTR = 64;
constexpr int EX_MAX_STACK = 8;
constexpr int EX_MAX_OUT = 16;
constexpr int EX_MAX_COLS = 32;

struct ExprInstr { int32_t op; int32_t pad; int64_t arg; };

// is_u: the value came straight from a UINT64 column, so `bits` holds it as uint64 (values >= 2^63 read as negative int64).
// Comparisons and conversions to double honour it; arithmetic, negation and casts clear it (uint64 arithmetic wraps as int64).
struct ExprVal { int64_t bits; bool is_f; bool valid; bool is_u; };
__device__ __forceinline__ double ev_f(const ExprVal& v) {
    return v.is_f ? __longlong_as_double(v.bits) : v.is_u ? (double)(unsigned long long)v.bits : (double)v.bits;
}
// Truthiness of a value (and / or / not, the predicate, BOOL stores): value != 0, so a float -0.0 is false and NaN is true.
__device__ __forceinline__ bool ev_true(const ExprVal& v) { return v.is_f ? __longlong_as_double(v.bits) != 0.0 : v.bits != 0; }
// Three-way order of two integer values, exact when either is a uint64 >= 2^63: such a value is above every int64, and two of
// them order like their (top-bit-set) int64 bit patterns.
__device__ __forceinline__ int ev_cmp_int(const ExprVal& x, const ExprVal& y) {
    const bool xbig = x.is_u && x.bits < 0, ybig = y.is_u && y.bits < 0;
    if (xbig != ybig) return xbig ? 1 : -1;
    return x.bits < y.bits ? -1 : x.bits > y.bits ? 1 : 0;
}

struct FilterProjectArgs {
    int64_t n_rows;
    int n_in;
    const void* in_data[EX_MAX_COLS];
    const uint8_t* in_valid[EX_MAX_COLS];
    int in_ctype[EX_MAX_COLS];
    int pred_start;                 // first instruction of the predicate program, -1 = keep every row
    int n_out;
    int out_start[EX_MAX_OUT];      // first instruction of output j's program
    int out_ctype[EX_MAX_OUT];      // CType the value is stored as
    void* out_data[EX_MAX_OUT];
    uint8_t* out_valid_bytes[EX_MAX_OUT];   // one byte per output row (packed into bitmaps afterwards), or nullptr
    unsigned long long* cursor;     // output rows so far
    int n_instr;
    ExprInstr prog[EX_MAX_INSTR];
};

__device__ __forceinline__ ExprVal expr_eval(const FilterProjectArgs& a, int pc, int64_t row) {
    ExprVal st[EX_MAX_STACK];
    int sp = 0;
    for (;; pc++) {
        const ExprInstr in = a.prog[pc];
        if (in.op == EX_END) break;
        switch (in.op) {
            case EX_COL: {
                const int c = (int)in.arg, ct = a.in_ctype[c];
                ExprVal v;
                v.valid = bit_valid(a.in_valid[c], row);
                v.is_f = ctype_is_float(ct);
                v.is_u = ct == CT_UINT64;
                v.bits = v.is_f ? __double_as_longlong(load_as_f64(a.in_data[c], ct, row)) : load_int_as_i64(a.in_data[c], ct, row);
                if (v.is_f && isnan(__longlong_as_double(v.bits))) v.valid = false;  // NaN is NA for float columns (isnan_alltype)
                st[sp++] = v;
                break;
            }
            case EX_CONST_I64: st[sp++] = ExprVal{in.arg, false, true, false}; break;
            case EX_CONST_F64: st[sp++] = ExprVal{in.arg, true, true, false}; break;
            case EX_ADD: case EX_SUB: case EX_MUL: case EX_DIV: {
                const ExprVal b = st[--sp], x = st[--sp];
                ExprVal r;
                r.valid = x.valid && b.valid;
                r.is_u = false;
                r.is_f = x.is_f || b.is_f || in.op == EX_DIV;  // true division, as pandas' `/`
                if (r.is_f) {
                    const double p = ev_f(x), q = ev_f(b);
                    const double v = in.op == EX_ADD ? p + q : in.op == EX_SUB ? p - q : in.op == EX_MUL ? p * q : p / q;
                    r.bits = __double_as_longlong(v);
                } else {
                    const unsigned long long p = (unsigned long long)x.bits, q = (unsigned long long)b.bits;  // wraps like the reference (-fwrapv)
                    r.bits = (int64_t)(in.op == EX_ADD ? p + q : in.op == EX_SUB ? p - q : p * q);
                }
                st[sp++] = r;
                break;
            }
            case EX_LT: case EX_LE: case EX_GT: case EX_GE: case EX_EQ: case EX_NE: {
                const ExprVal b = st[--sp], x = st[--sp];
                bool t;
                if (x.is_f || b.is_f) {
                    const double p = ev_f(x), q = ev_f(b);
                    t = in.op == EX_LT ? p < q : in.op == EX_LE ? p <= q : in.op == EX_GT ? p > q : in.op == EX_GE ? p >= q : in.op == EX_EQ ? p == q : p != q;
                } else {
                    const int c = ev_cmp_int(x, b);
                    t = in.op == EX_LT ? c < 0 : in.op == EX_LE ? c <= 0 : in.op == EX_GT ? c > 0 : in.op == EX_GE ? c >= 0 : in.op == EX_EQ ? c == 0 : c != 0;
                }
                st[sp++] = ExprVal{t ? 1 : 0, false, x.valid && b.valid, false};
                break;
            }
            case EX_AND: case EX_OR: {  // Kleene logic
                const ExprVal b = st[--sp], x = st[--sp];
                const bool xt = x.valid && ev_true(x), xf = x.valid && !ev_true(x), bt = b.valid && ev_true(b), bf = b.valid && !ev_true(b);
                ExprVal r;
                r.is_f = false; r.is_u = false;
                if (in.op == EX_AND) { r.valid = (xf || bf) || (x.valid && b.valid); r.bits = (xt && bt) ? 1 : 0; }
                else { r.valid = (xt || bt) || (x.valid && b.valid); r.bits = (xt || bt) ? 1 : 0; }
                st[sp++] = r;
                break;
            }
            case EX_NOT: { ExprVal& x = st[sp - 1]; x.bits = ev_true(x) ? 0 : 1; x.is_f = false; x.is_u = false; break; }
            case EX_NEG: { ExprVal& x = st[sp - 1]; x.bits = x.is_f ? __double_as_longlong(-__longlong_as_double(x.bits)) : (int64_t)(0ull - (unsigned long long)x.bits); x.is_u = false; break; }
            case EX_TO_F64: { ExprVal& x = st[sp - 1]; if (!x.is_f) { x.bits = __double_as_longlong(ev_f(x)); x.is_f = true; x.is_u = false; } break; }
            // float -> int truncates toward zero; NaN and values outside int64 saturate (numpy leaves those undefined)
            case EX_TO_I64: { ExprVal& x = st[sp - 1]; if (x.is_f) { x.bits = (int64_t)__longlong_as_double(x.bits); x.is_f = false; } x.is_u = false; break; }
            case EX_IS_NULL: { ExprVal& x = st[sp - 1]; x.bits = x.valid ? 0 : 1; x.is_f = false; x.is_u = false; x.valid = true; break; }
            default: break;
        }
    }
    return st[sp - 1];
}

// Stores a value as the output's CType the way numpy's astype converts it (for values the type can hold): a float becomes an
// integer of any width by truncation toward zero (through int64, or uint64 for a UINT64 output), an integer keeps its low
// bytes, an integer becomes FLOAT32 in one rounding, and BOOL stores value != 0.
__device__ __forceinline__ void store_val(void* out, int ct, int64_t i, const ExprVal& v) {
    const double d = __longlong_as_double(v.bits);
    const int64_t iv = !v.is_f ? v.bits : ct == CT_UINT64 ? (int64_t)(unsigned long long)d : (int64_t)d;
    switch (ct) {
        case CT_FLOAT64: ((double*)out)[i] = ev_f(v); break;
        case CT_FLOAT32: ((float*)out)[i] = v.is_f ? (float)d : v.is_u ? (float)(unsigned long long)v.bits : (float)v.bits; break;
        case CT_BOOL: ((uint8_t*)out)[i] = ev_true(v) ? 1 : 0; break;
        case CT_INT64: case CT_UINT64: case CT_DATETIME: case CT_TIMEDELTA: ((int64_t*)out)[i] = iv; break;
        case CT_INT32: case CT_UINT32: case CT_DATE: ((int32_t*)out)[i] = (int32_t)iv; break;
        case CT_INT16: case CT_UINT16: ((int16_t*)out)[i] = (int16_t)iv; break;
        default: ((int8_t*)out)[i] = (int8_t)iv; break;
    }
}

constexpr int FP_THREADS = 256, FP_ROWS = 4, FP_TILE = FP_THREADS * FP_ROWS;

__global__ void __launch_bounds__(FP_THREADS) filter_project_kernel(const __grid_constant__ FilterProjectArgs a) {
    __shared__ unsigned int wsum[FP_ROWS][FP_THREADS / 32];
    __shared__ unsigned long long tile_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t n_tiles = (a.n_rows + FP_TILE - 1) / FP_TILE;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        bool keep[FP_ROWS];
        unsigned int rank[FP_ROWS];
#pragma unroll
        for (int r = 0; r < FP_ROWS; r++) {
            const int64_t row = t * FP_TILE + r * FP_THREADS + threadIdx.x;
            keep[r] = row < a.n_rows;
            if (keep[r] && a.pred_start >= 0) {
                const ExprVal p = expr_eval(a, a.pred_start, row);
                keep[r] = p.valid && ev_true(p);
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep[r]);
            rank[r] = __popc(m & ((1u << lane) - 1));
            if (lane == 0) wsum[r][warp] = __popc(m);
        }
        __syncthreads();
        if (threadIdx.x < 32) {  // exclusive scan of the 32 (row slot, warp) counts in row order; one cursor atomic per tile
            const int r = threadIdx.x >> 3, w = threadIdx.x & 7;
            unsigned int x = wsum[r][w], inc = x;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += y; }
            wsum[r][w] = inc - x;
            if (lane == 31) tile_base = inc ? atomicAdd(a.cursor, (unsigned long long)inc) : 0ull;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < FP_ROWS; r++) {
            if (!keep[r]) continue;
            const int64_t row = t * FP_TILE + r * FP_THREADS + threadIdx.x;
            const int64_t o = (int64_t)(tile_base + wsum[r][warp] + rank[r]);
            for (int j = 0; j < a.n_out; j++) {
                const ExprVal v = expr_eval(a, a.out_start[j], row);
                store_val(a.out_data[j], a.out_ctype[j], o, v);
                if (a.out_valid_bytes[j]) a.out_valid_bytes[j][o] = v.valid ? 1 : 0;
            }
        }
        __syncthreads();
    }
}

__global__ void remap_i32_kernel(const int32_t* in, const uint8_t* valid, int64_t n, const int32_t* map, int32_t map_len, int32_t* out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
        const int32_t v = in[i];
        out[i] = (bit_valid(valid, i) && v >= 0 && v < map_len) ? map[v] : 0;
    }
}

}  // namespace b200

extern "C" {

int64_t b200_filter_project(const b200_table* in_table, const void* program, int32_t n_instr, int32_t pred_start, const int32_t* out_starts,
                            int32_t n_out, b200_table* out, void* stream) {
    try {
        using namespace b200;
        B200_REQUIRE(in_table && program && out && out->cols && (n_out == 0 || out_starts), "b200_filter_project: null argument");
        B200_REQUIRE(in_table->device >= 0, "b200_filter_project: the table must be device resident (this path has no CPU fallback)");
        B200_REQUIRE(in_table->n_cols <= EX_MAX_COLS, "b200_filter_project: the input table has more than 32 columns");
        B200_REQUIRE(n_out >= 0 && n_out <= EX_MAX_OUT, "b200_filter_project: more than 16 output columns");
        B200_REQUIRE(n_instr >= 1 && n_instr <= EX_MAX_INSTR, "b200_filter_project: the program needs 1 to 64 instructions");
        cudaStream_t st = (cudaStream_t)stream;
        B200_CUDA(cudaSetDevice(in_table->device)); scratch_set_stream(st);
        FilterProjectArgs a{};
        a.n_rows = in_table->n_rows; a.n_in = in_table->n_cols;
        for (int c = 0; c < a.n_in; c++) {
            B200_REQUIRE(ctype_size(in_table->cols[c].c_type) > 0, "b200_filter_project: unsupported column dtype");
            a.in_data[c] = in_table->cols[c].data; a.in_valid[c] = in_table->cols[c].validity; a.in_ctype[c] = in_table->cols[c].c_type;
        }
        const ExprInstr* prog = (const ExprInstr*)program;
        a.n_instr = n_instr;
        int depth = 0, max_depth = 0;
        for (int i = 0; i < n_instr; i++) {
            a.prog[i] = prog[i];
            switch (prog[i].op) {  // static validation: column indices and stack depth
                case EX_COL: B200_REQUIRE(prog[i].arg >= 0 && prog[i].arg < a.n_in, "b200_filter_project: bad column index in the program"); depth++; break;
                case EX_CONST_I64: case EX_CONST_F64: depth++; break;
                case EX_ADD: case EX_SUB: case EX_MUL: case EX_DIV: case EX_LT: case EX_LE: case EX_GT: case EX_GE: case EX_EQ: case EX_NE: case EX_AND: case EX_OR:
                    B200_REQUIRE(depth >= 2, "b200_filter_project: malformed program (stack underflow)"); depth--; break;
                case EX_NOT: case EX_NEG: case EX_TO_F64: case EX_TO_I64: case EX_IS_NULL: B200_REQUIRE(depth >= 1, "b200_filter_project: malformed program (stack underflow)"); break;
                case EX_END: B200_REQUIRE(depth == 1, "b200_filter_project: every program must leave exactly one value"); depth = 0; break;
                default: throw Error("b200_filter_project: unknown opcode");
            }
            max_depth = std::max(max_depth, depth);
        }
        B200_REQUIRE(max_depth <= EX_MAX_STACK && prog[n_instr - 1].op == EX_END, "b200_filter_project: program too deep or not terminated");
        // an expression starts at instruction 0 or right after an END; any other start would run the VM off its checked depth
        auto starts_expr = [&](int32_t s) { return s == 0 || (s > 0 && s < n_instr && prog[s - 1].op == EX_END); };
        B200_REQUIRE(pred_start == -1 || starts_expr(pred_start), "b200_filter_project: pred_start does not start an expression");
        for (int j = 0; j < n_out; j++)
            B200_REQUIRE(starts_expr(out_starts[j]), "b200_filter_project: out_starts[j] does not start an expression");
        a.pred_start = pred_start;
        a.n_out = n_out;
        DevBuf cursor;
        cursor.alloc(8);
        B200_CUDA(cudaMemsetAsync(cursor.p, 0, 8, st));
        a.cursor = cursor.as<unsigned long long>();
        std::vector<DevBuf> vbytes(n_out);
        for (int j = 0; j < n_out; j++) {
            b200_column& oc = out->cols[j];
            B200_REQUIRE(oc.data != nullptr && ctype_size(oc.c_type) > 0, "b200_filter_project: out column needs a data buffer of n_rows items and a dtype");
            a.out_start[j] = out_starts[j]; a.out_ctype[j] = oc.c_type; a.out_data[j] = oc.data; a.out_valid_bytes[j] = nullptr;
            if (oc.validity) { vbytes[j].alloc((size_t)std::max<int64_t>(in_table->n_rows, 1)); a.out_valid_bytes[j] = vbytes[j].as<uint8_t>(); }
        }
        int64_t n_keep = 0;
        if (in_table->n_rows > 0) {
            const int sms = num_sms(in_table->device);
            const int64_t n_tiles = (in_table->n_rows + FP_TILE - 1) / FP_TILE;
            filter_project_kernel<<<(int)std::min<int64_t>(n_tiles, (int64_t)sms * 8), FP_THREADS, 0, st>>>(a);
            B200_CUDA(cudaGetLastError());
            unsigned long long* h = (unsigned long long*)pinned_acquire(8);
            B200_CUDA(cudaMemcpyAsync(h, cursor.p, 8, cudaMemcpyDeviceToHost, st));
            B200_CUDA(cudaStreamSynchronize(st));
            n_keep = (int64_t)*h;
            pinned_release(h, 8);
            for (int j = 0; j < n_out; j++)
                if (a.out_valid_bytes[j] && n_keep > 0) launch_pack_bitmap(a.out_valid_bytes[j], n_keep, (uint32_t*)out->cols[j].validity, sms * 4, st);
            B200_CUDA(cudaGetLastError());
            B200_CUDA(cudaStreamSynchronize(st));
        }
        out->n_rows = n_keep; out->n_cols = n_out; out->device = in_table->device;
        for (int j = 0; j < n_out; j++) out->cols[j].length = n_keep;
        return n_keep;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

int b200_remap_i32(const int32_t* in_dev, const uint8_t* valid_dev, int64_t n, const int32_t* map_dev, int32_t map_len, int32_t* out_dev,
                   int32_t device, void* stream) {
    try {
        B200_REQUIRE(in_dev && map_dev && out_dev && n >= 0, "b200_remap_i32: null argument");
        B200_CUDA(cudaSetDevice(device));
        if (n == 0) return 0;
        b200::remap_i32_kernel<<<b200::num_sms(device) * 4, 256, 0, (cudaStream_t)stream>>>(in_dev, valid_dev, n, map_dev, map_len, out_dev);
        B200_CUDA(cudaGetLastError());
        return 0;
    } catch (const std::exception& e) { b200::set_last_error(e.what()); return -1; }
}

}  // extern "C"
