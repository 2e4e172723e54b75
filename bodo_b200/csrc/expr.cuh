// expr.cuh — the postfix expression interpreter shared by the fused filter + projection kernel (expr.cu) and the join's
// non-equi condition (join.cu): instruction encoding, value representation, the evaluation loop and the host-side static
// validation of a program.
//
// Expressions are postfix programs over a per-thread value stack (numbers as double or int64 with a validity flag):
// column loads, constants, + - * /, comparisons, and / or / not, casts.  Null semantics are the reference's (Arrow compute /
// pandas nullable): arithmetic and comparisons propagate null, `and` / `or` are Kleene, isnull is never null.  Where a column
// load reads from is the caller's: the evaluation loop takes a loader `load(arg)` that returns the ExprVal of the cell of the
// column an EX_COL instruction's argument names (the row, or the pair of rows, is the loader's).
#pragma once

#include <algorithm>
#include <string>

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

// The value of cell `row` of a column of CType `ct`; `valid` is the cell's validity.  NaN read from a float column is NA
// (isnan_alltype).
__device__ __forceinline__ ExprVal expr_load(const void* data, int ct, int64_t row, bool valid) {
    ExprVal v;
    v.valid = valid;
    v.is_f = ctype_is_float(ct);
    v.is_u = ct == CT_UINT64;
    v.bits = v.is_f ? __double_as_longlong(load_as_f64(data, ct, row)) : load_int_as_i64(data, ct, row);
    if (v.is_f && isnan(__longlong_as_double(v.bits))) v.valid = false;
    return v;
}

// Evaluates the expression that starts at instruction `pc` of `prog` (it ends at the next EX_END); `load(arg)` is the value of
// the column an EX_COL instruction names.  The program must have passed expr_validate.
template <typename Load>
__device__ __forceinline__ ExprVal expr_run(const ExprInstr* prog, int pc, Load&& load) {
    ExprVal st[EX_MAX_STACK];
    int sp = 0;
    for (;; pc++) {
        const ExprInstr in = prog[pc];
        if (in.op == EX_END) break;
        switch (in.op) {
            case EX_COL: st[sp++] = load(in.arg); break;
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

// Host-side static validation of a program of n_instr (1..64) instructions: every opcode known, every EX_COL argument accepted
// by `col_ok(arg)`, no stack underflow, every expression leaves exactly one value, at most EX_MAX_STACK values live, and the
// last instruction is EX_END.  Errors are thrown with the message prefixed by `who`.
template <typename ColOk>
void expr_validate(const ExprInstr* prog, int n_instr, ColOk&& col_ok, const std::string& who) {
    B200_REQUIRE(n_instr >= 1 && n_instr <= EX_MAX_INSTR, who + ": the program needs 1 to 64 instructions");
    int depth = 0, max_depth = 0;
    for (int i = 0; i < n_instr; i++) {
        switch (prog[i].op) {
            case EX_COL: B200_REQUIRE(col_ok(prog[i].arg), who + ": bad column index in the program"); depth++; break;
            case EX_CONST_I64: case EX_CONST_F64: depth++; break;
            case EX_ADD: case EX_SUB: case EX_MUL: case EX_DIV: case EX_LT: case EX_LE: case EX_GT: case EX_GE: case EX_EQ: case EX_NE: case EX_AND: case EX_OR:
                B200_REQUIRE(depth >= 2, who + ": malformed program (stack underflow)"); depth--; break;
            case EX_NOT: case EX_NEG: case EX_TO_F64: case EX_TO_I64: case EX_IS_NULL: B200_REQUIRE(depth >= 1, who + ": malformed program (stack underflow)"); break;
            case EX_END: B200_REQUIRE(depth == 1, who + ": every program must leave exactly one value"); depth = 0; break;
            default: throw Error(who + ": unknown opcode");
        }
        max_depth = std::max(max_depth, depth);
    }
    B200_REQUIRE(max_depth <= EX_MAX_STACK && prog[n_instr - 1].op == EX_END, who + ": program too deep or not terminated");
}

}  // namespace b200
