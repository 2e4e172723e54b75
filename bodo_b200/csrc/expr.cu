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
// The interpreter and its validation live in expr.cuh, which the join's non-equi condition shares.
// The same lookup kernel serves dictionary unification (remap_i32: batch-local dictionary indices -> global ids, the
// transpose step of DictionaryBuilder::UnifyDictionaryArray, bodo/libs/_dict_builder.cpp).
#include <vector>

#include "expr.cuh"

namespace b200 {

constexpr int EX_MAX_OUT = 16;
constexpr int EX_MAX_COLS = 32;

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
    return expr_run(a.prog, pc, [&](int64_t arg) {
        const int c = (int)arg;
        return expr_load(a.in_data[c], a.in_ctype[c], row, bit_valid(a.in_valid[c], row));
    });
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
        expr_validate(prog, n_instr, [&](int64_t c) { return c >= 0 && c < a.n_in; }, "b200_filter_project");
        a.n_instr = n_instr;
        std::copy(prog, prog + n_instr, a.prog);
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
