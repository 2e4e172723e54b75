/*
 * bodo_b200.h — C ABI of libbodo_b200.so: the CUDA-native (H100) replacement for Bodo's streaming
 * hash groupby / hash join / row->rank shuffle hot path.
 *
 * Every entry point mirrors one reference FFI symbol (cited per function, paths relative to the
 * reference checkout). Differences from the reference ABI, all deliberate:
 *   - tables cross the boundary as `b200_table` (plain column descriptors: data pointer, Arrow
 *     validity bitmap, Bodo_CTypes / bodo_array_type codes) instead of `table_info*`;
 *   - errors are reported by return code + b200_last_error() instead of the CPython error
 *     indicator (reference: PyErr_SetString, bodo/libs/streaming/_groupby.cpp:4669-4675);
 *   - input tables are BORROWED for the duration of the call (the reference steals them).
 * No torch / CUDA types appear in any signature: streams are passed as void* (cudaStream_t).
 *
 * This header is also parsed by cffi (bodo_b200/_lib.py): keep it plain C89 declarations;
 * lines starting with '#' are stripped before parsing.
 */
#ifndef BODO_B200_H
#define BODO_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- data model (reference: bodo/libs/_bodo_common.h:331-359 Bodo_CTypes, :515-532 bodo_array_type,
 *      :927 array_info, :1819 table_info) ---- */

/* b200_column.c_type uses Bodo_CTypes codes: INT8=0 UINT8=1 INT32=2 UINT32=3 INT64=4 FLOAT32=5
 * FLOAT64=6 UINT64=7 INT16=8 UINT16=9 _BOOL=11 DATE=13 DATETIME=15 TIMEDELTA=16.
 * b200_column.arr_type uses bodo_array_type codes: NUMPY=0, NULLABLE_INT_BOOL=2. */
typedef struct b200_column {
    void* data;        /* contiguous values, length * itemsize bytes (host or device, see b200_table.device) */
    uint8_t* validity; /* Arrow validity bitmap (bit i%8 of byte i/8, 1 = valid) or NULL = all valid */
    int64_t length;
    int32_t c_type;
    int32_t arr_type;
} b200_column;

typedef struct b200_table {
    int64_t n_rows;
    int32_t n_cols;
    int32_t device; /* -1: pointers are host memory; >= 0: CUDA device ordinal owning the pointers */
    b200_column* cols;
} b200_table;

/* Last error message of the calling thread ("" if none). Every int-returning entry point returns
 * a negative value on error; pointer-returning ones return NULL. */
const char* b200_last_error(void);

/* Library/runtime probes (used by tests and __graft_entry__). b200_device_count() returns 0 without
 * a GPU and never raises; all compute entry points fail with an error instead of falling back. */
int b200_abi_version(void);
int b200_device_count(void);

/* ---- streaming hash groupby (reference door 1: bodo/libs/streaming/_groupby.cpp) ---- */

/* groupby_state_init_py_entry (_groupby.cpp:4917-4970). Keys are the first n_keys (1..4, integer, date or float typed)
 * columns of every build batch; n_funcs may be 0 (select
 * distinct / drop_duplicates, reference: physical/aggregate.h:198-227); ftypes are Bodo_FTypes (groupby/_groupby_ftypes.h:17-110: size=4 sum=6 count=7 nunique=8 mean=14
 * min=15 max=16 prod=17 first=18 last=19 var_pop=22 std_pop=23 var=24 std=25 kurtosis=26 skew=27 boolor_agg=28 booland_agg=29
 * boolxor_agg=30 bitor_agg=31 bitand_agg=32 bitxor_agg=33 count_if=34; 28..34 are recalled, not read from a reference checkout); f_in_offsets/f_in_cols is the CSR map function -> physical input column
 * (streaming/_groupby.h:1059-1070). Arguments of the reference that only concern window functions,
 * MRNF, sort keys and the host operator pool are dropped (MRNF has its own entry, b200_groupby_state_init_mrnf). `pandas_drop_na`: drop rows with NA keys
 * (filter_na_keys, _groupby.cpp:4278-4309). `parallel`: state is one shard of n_pes; ownership
 * is hash_to_rank(key) (bodo/libs/_shuffle.h:5-7). `expected_groups` is a sizing hint (0 = unknown).
 * `stream` is a cudaStream_t all work is enqueued on (NULL = legacy default stream). */
void* b200_groupby_state_init(int64_t operator_id, const int8_t* build_arr_c_types,
                              const int8_t* build_arr_array_types, int32_t n_build_arrs,
                              const int32_t* ftypes, const int32_t* f_in_offsets,
                              const int32_t* f_in_cols, int32_t n_funcs, uint64_t n_keys,
                              int64_t output_batch_size, int32_t parallel, int32_t pandas_drop_na,
                              int32_t device, int32_t n_pes, int32_t myrank,
                              int64_t expected_groups, void* stream);

/* b200_groupby_state_init with one fraction per function: the holistic aggregates mode=38, percentile_cont=39 and
 * percentile_disc=40 (recalled enum values, not read from a reference checkout) beside any other function.
 * b200_groupby_state_init is this entry with fractions = NULL.
 *   fractions: n_funcs entries; entry j is the q of function j when it is percentile_cont or percentile_disc (0 <= q <= 1, not
 *     NaN) and is ignored otherwise.  NULL is allowed when no function is a percentile.
 *   Each of the three takes exactly one input column (a non-key column).  Per group, V is the multiset of that column's values
 *     with NA cells (and NaN in a float column) skipped, m = |V|, and v_0 <= ... <= v_{m-1} is V in the order of the sort's key
 *     encoding (ascending; -0.0 and 0.0 are one value).  A group with m = 0 gets NA; every output is nullable.
 *   percentile_cont(q): h = q (m - 1), lo = floor(h), f = h - lo (float64); v_lo when f == 0, else a + (b - a) f with a = v_lo and
 *     b = v_{lo+1} as float64, evaluated with rounded operations and no fused multiply-add (pandas' linear group_quantile;
 *     MEDIAN(x) is q = 0.5).  Integer (uint64 included) and float columns; the output is FLOAT64.
 *   percentile_disc(q): v_i with i = clamp(ceil(q m) - 1, 0, m - 1), q m in float64 (numpy's method="inverted_cdf").  Integer,
 *     float, DATE, DATETIME and TIMEDELTA columns; the output has the input's type.
 *   mode: the most frequent value of V, ties to the least value (Series.mode().iloc[0]).  Integer, float, bool, DATE, DATETIME and
 *     TIMEDELTA columns; the output has the input's type.
 *   A result is decoded from the value's encoding (a zero comes back as +0.0), so it depends only on V and is bit-identical across
 *     runs, batch splits, empty batches, table growth and rank counts.
 *   Memory: the state keeps a 4-byte group id and the value (its width) per non-NA value, one store per distinct value column,
 *     sorted at finalize by a radix sort of at most 2^31 rows: a consume call that could take a store past 2^31 rows (or the state
 *     past 2^32 groups) fails before it runs anything and leaves the state usable.
 *   Such a state consumes on the direct (or multi-key) kernels only.  Sharded (parallel, n_pes > 1) it never exchanges partial
 *     aggregates: the caller hash-partitions the rows by key before each consume call, every rank aggregates only the groups it
 *     owns, and b200_groupby_finalize runs without an exchange (the exchange entries refuse the state).
 *   Refused here, naming the argument: a percentile without fractions, a fraction outside [0, 1] or NaN, a function with other
 *     than one input column, a column type the function does not take.
 *   Metrics: 20 the values appended to the stores (exact: synchronises the stream), 21 the digit passes the finalize sorts ran. */
void* b200_groupby_state_init_percentiles(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                          int32_t n_build_arrs, const int32_t* ftypes, const int32_t* f_in_offsets,
                                          const int32_t* f_in_cols, int32_t n_funcs, uint64_t n_keys, int64_t output_batch_size,
                                          int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                          int64_t expected_groups, void* stream, const double* fractions);

/* groupby_state_init_py_entry (_groupby.cpp:4917-4970) with its MRNF arguments (sort_asc / sort_na / n_sort_keys / cols_to_keep):
 * a min_row_number_filter state, QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) = 1, i.e.
 * df.sort_values(sort columns, kind="stable").drop_duplicates(keys, keep="first")[kept columns].
 *   Keys: the first n_keys (1..4) columns, of the key types and with the key equality of b200_groupby_state_init (float keys:
 *     -0.0 equals 0.0 and NaN is the NA key).  pandas_drop_na drops rows with an NA key; otherwise all NA keys form one group.
 *   Sort columns: sort_cols[0 .. n_sort) (1 <= n_sort <= 4, distinct, any column including a key): fixed-width integer, float,
 *     bool, DATE, DATETIME or TIMEDELTA, numpy or nullable.  sort_ascending[j] and sort_na_last[j] (NA last = 1, first = 0) per
 *     column.  A float NaN is NA and -0.0 ties with 0.0: the rules of b200_sort_state_init.
 *   Winner: per group the first row of the stable order by (sort columns, arrival), arrival being batch order, then row order, so
 *     a row that ties on every sort column with an earlier row (of this batch or an earlier one) never wins.  The result is
 *     bit-identical across runs, batch splits and table growth.
 *   Output: one row per group (group order unspecified): the columns c with keep[c] != 0 (keep: one flag per column, at least
 *     one and at most 26 set), in column order, each with the winning row's own cell (bits and validity; a kept float key shows
 *     the winner's -0.0), type and array kind, so `out->cols` of a produce call holds one descriptor per kept column.
 *   Columns that are neither keys, sort columns nor kept are never read.  Every key, sort and kept column is fixed width;
 *   anything else fails here, naming the column.  A state with parallel set and n_pes > 1 fails at its first consume call
 *   (sharded MRNF is not supported); with n_pes == 1 it runs locally.
 * Build-consume, finalize, produce, delete and the metrics are the entries of the ordinary state (metric 0: groups); the exchange
 * entries refuse an MRNF state. */
void* b200_groupby_state_init_mrnf(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                   int32_t n_build_arrs, uint64_t n_keys, const int32_t* sort_cols, const int32_t* sort_ascending,
                                   const int32_t* sort_na_last, int32_t n_sort, const int32_t* keep, int64_t output_batch_size,
                                   int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                   int64_t expected_groups, void* stream);

/* b200_groupby_state_init_mrnf with a limit: QUALIFY ROW_NUMBER() OVER (PARTITION BY keys ORDER BY sort columns) <= rows_per_group,
 * i.e. df.sort_values(sort columns, kind="stable").groupby(keys, sort=False, dropna=...).head(rows_per_group)[kept columns].  The
 * reference's MRNF keeps one row per group; rows_per_group > 1 goes beyond it.
 *   Arguments, keys, sort columns, kept columns (at most 26), dropna and the sharded refusal: as b200_groupby_state_init_mrnf.
 *   rows_per_group: 1 <= rows_per_group < 2^31.  1 is b200_groupby_state_init_mrnf itself (one winner record per group, no store).
 *   Rows: every group keeps the first rows_per_group rows of the stable order by (sort columns, arrival), arrival being batch
 *     order, then row order, so of rows that tie on every sort column the earlier arrival ranks first, even across batches; a group
 *     with fewer rows keeps all of them.  Each row holds its own cells (bits and validity) of the kept columns.
 *   Output order: groups in an unspecified order; a group's rows are consecutive and in rank order, also when the group spans two
 *     output batches, so a cumulative count numbers them.  The rows of every group are bit-identical across runs, batch splits and
 *     table growth.
 *   Limit: rows_per_group > 1 keeps candidate rows in a store that a radix sort of at most 2^31 rows reduces.  A consume call whose
 *     rows, added to the survivors of every group (at most groups x rows_per_group), would pass 2^31 fails, naming the limit;
 *     nothing is truncated.  Fewer than 2^48 rows in all.
 *   Metrics: 0 is the groups while consuming and the output rows after finalize (the groups when rows_per_group == 1); 18 the
 *     candidate rows admitted to the store, 19 the reduces of the store (both 0 when rows_per_group == 1). */
void* b200_groupby_state_init_mrnf_limit(int64_t operator_id, const int8_t* build_arr_c_types, const int8_t* build_arr_array_types,
                                         int32_t n_build_arrs, uint64_t n_keys, const int32_t* sort_cols, const int32_t* sort_ascending,
                                         const int32_t* sort_na_last, int32_t n_sort, const int32_t* keep, int64_t output_batch_size,
                                         int32_t parallel, int32_t pandas_drop_na, int32_t device, int32_t n_pes, int32_t myrank,
                                         int64_t expected_groups, void* stream, int64_t rows_per_group);

/* groupby_build_consume_batch_py_entry (_groupby.cpp:4663-4676). Returns 1 when the build is globally
 * finished (is_last was passed), 0 otherwise, <0 on error. *request_input is always set to 1 (the GPU
 * state sizes its table up front and never back-pressures). */
int b200_groupby_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last,
                                     int32_t is_final_pipeline, int32_t* request_input);

/* Multi-rank exchange of partial aggregates, replacing GroupbyIncrementalShuffleState (streaming/_groupby.cpp:1558-1873)
 * + shuffle_issend/irecv (streaming/_shuffle.cpp:567-652), for any key count.  After the last local batch every group that
 * another rank owns (hash_to_rank of the key, as b200_hash_keys_table computes it) travels to its owner as one partial row of
 * b200_groupby_exchange_row_bytes(state) bytes (layout: DESIGN.md "partial-aggregate wire format"); the groups this rank owns
 * stay in its table.  The owner merges the rows with the combine functions of groupby/_groupby_update.cpp:41-57 (count/size/
 * mean -> sum, min -> min, max -> max).  Two transports, the same pack and combine:
 *   fused: every rank owns a receive slab in memory mapped into all peers (symmetric memory, set up by the host layer): 256
 *     header bytes + n_pes segments of cap_rows rows.
 *       1. b200_groupby_exchange_pack(state, peer_slabs_dev, cap_rows, NULL) stores every row into segment `myrank` of its
 *          owner's slab (peer_slabs_dev = device array of the n_pes slab addresses) and posts the counts into the peers' headers;
 *       2. a barrier across the ranks on the same stream (host layer);
 *       3. b200_groupby_exchange_combine(state, my_slab, cap_rows, NULL) merges the rows received in my_slab.
 *     Nothing here synchronises with the host.  If some rank's share for one destination exceeded cap_rows no rank combines and
 *     b200_groupby_finalize returns -2: run the NCCL form and finalize again (the tables are intact, and the counts of the fused
 *     pack are exact).
 *   NCCL (all-to-all-v):
 *       1. without a fused pack before: b200_groupby_exchange_pack(state, NULL, 0, NULL) counts the rows per destination;
 *       2. b200_groupby_exchange_counts writes them (n_pes, host; synchronises);
 *       3. b200_groupby_exchange_pack(state, NULL, 0, send_buf) packs the rows of destination d at the exclusive prefix of those
 *          counts (send_buf: their sum times the row width, on the state's device) and synchronises;
 *       4. the host exchanges counts and rows;
 *       5. b200_groupby_exchange_combine(state, recv_buf, 0, recv_row_counts) merges the received rows, which lie back to back in
 *          source-rank order (recv_row_counts: n_pes, host).
 * Either combine's rows must stay valid until b200_groupby_finalize returns: rows that found the table full are merged there. */
int64_t b200_groupby_exchange_row_bytes(void* state);
int b200_groupby_exchange_pack(void* state, void* const* peer_slabs_dev, int64_t cap_rows, void* send_buf);
int b200_groupby_exchange_counts(void* state, int64_t* send_row_counts);
int b200_groupby_exchange_combine(void* state, const void* rows, int64_t cap_rows, const int64_t* recv_row_counts);

/* FinalizeBuild (_groupby.cpp:4062-4256): evaluates the output columns (mean_eval etc.). Called
 * implicitly by the first produce call; exposed so the exchange step can be timed separately.
 * Returns the number of output rows (groups owned by this shard), or -2 (see the exchange). */
int64_t b200_groupby_finalize(void* state);

/* groupby_produce_output_batch_py_entry (_groupby.cpp:4772-4783). Fills `out` (caller provides
 * out->cols with room for n_keys + n_funcs descriptors) with pointers to library-owned device
 * columns holding the next <= output_batch_size groups; they stay valid until the next produce call
 * or delete. Sets *out_is_last. Output order of groups is unspecified (as in the reference). */
int b200_groupby_produce_output_batch(void* state, b200_table* out, int32_t* out_is_last,
                                      int32_t produce_output);

/* delete_groupby_state (_groupby.cpp:5246). */
void b200_delete_groupby_state(void* state);

/* Metrics (subset of GroupbyMetrics, streaming/_groupby.h:106-223): 0 n_groups, 1 table capacity,
 * 2 rows consumed, 3 table rebuilds, 4 kernel launches so far, 5 rows replayed from the fail list,
 * 6 accumulated device time of the consume kernel in microseconds (CUDA events on the state's stream;
 * only when profiling was enabled by querying metric 100 first), 7 consume-kernel launches, 8 SM-partitioned
 * (SPG) launches, 9 rows/partials replayed from the SPG retry lists, 10 low-cardinality (LC) launches, 11 small batches
 * that were coalesced on the device before a fast-path launch, 12 SPG launches of the generic signature (SPG-G: nullable /
 * 4-byte keys or values, mean / min / max; included in 8), 13 groups in the table right now (exact: reads the device counter,
 * synchronises the state's stream), 14 SPG launches with narrow (int32 key, int32 value) bucket rows (SPG-N; included in 8),
 * 15 SPG launches with 16-byte (int64 key, int64 value) bucket rows (included in 8), 16 heavy-hitter keys admitted to the
 * partition kernel's hot table (0 when there are none or the table is disabled), 18 / 19 candidate rows admitted / store reduces
 * of a b200_groupby_state_init_mrnf_limit state (0 otherwise), 20 / 21 values appended to the stores / digit passes of the finalize
 * sorts of a state with mode or a percentile (0 otherwise; 20 synchronises the stream). */
/* nunique keeps one nested distinct state over (key, value) per value column (owned by `state`).  A sharded caller exchanges every
 * nested state (the exchange above + b200_groupby_finalize on the handle returned here — a key's pairs are owned where the key is
 * owned) BEFORE it exchanges and finalizes the outer state; single-GPU callers never need these. */
int32_t b200_groupby_num_inner_states(void* state);
void* b200_groupby_inner_state(void* state, int32_t i);

int64_t b200_groupby_get_metric(void* state, int32_t which);

/* ---- streaming hash join (reference: bodo/libs/streaming/_join.cpp) ---- */

/* join_state_init_py_entry (_join.cpp:4087-4136). Inner equi-join on the first n_keys (0..4, 0 = nested loop) columns of each side;
 * build_table_outer / probe_table_outer select right/left/full-outer semantics. `is_na_equal` is the
 * HashJoinState option of the same name: 0 (what join_state_init_py_entry constructs: NA keys never match,
 * _join.cpp:3180) or 1 (what bodo/pandas/physical/join.h:267 passes: NA joins NA, pandas merge semantics).
 * Key columns: integer / date / time types of one width on both sides, or float64 on both sides, or float32 on both sides
 * (a float key against any other key type is an error).  Float keys: -0.0 and 0.0 are one key, and a NaN key is an NA key
 * (is_na_equal decides whether it joins NaN and NA keys); output columns keep the input bits.
 * With n_keys > 1 this rule holds per key position (positions may differ in type from each other) and keys compare column by
 * column: NA is part of the key tuple (is_na_equal: NA equals NA within a column; otherwise a row with any NA key column matches
 * nothing).  Multi-column keys always take the general (CSR) table, never the unique-key tables of metrics 5-7.
 * n_probe_arrs may be 0: the probe schema is then taken from the first probe batch.
 * n_keys 0 is a nested-loop join (the reference's NestedLoopJoinState, bodo/libs/streaming/_nested_loop_join.cpp): every (probe
 * row, build row) pair is a candidate, all of them join without a condition (a cross join) and those that pass it with one
 * (b200_join_set_condition); b200_join_set_kind, the outer flags and metrics 8 / 9 apply as for keys.  Output order is fixed:
 * within a probe call rows follow the probe rows, a probe row's pairs follow the build arrival order, and a NULL-extended, anti or
 * mark row sits in its probe row's place; the build-outer tail follows the last probe call in build order.  One probe call
 * produces at most 2^31 rows: a bigger one fails (before its output is allocated) and the state stays usable.  No as-of form and
 * no runtime filter. */
void* b200_join_state_init(int64_t operator_id, const int8_t* build_arr_c_types,
                           const int8_t* build_arr_array_types, int32_t n_build_arrs,
                           const int8_t* probe_arr_c_types, const int8_t* probe_arr_array_types,
                           int32_t n_probe_arrs, uint64_t n_keys, int32_t build_table_outer,
                           int32_t probe_table_outer, int32_t is_na_equal, int64_t output_batch_size,
                           int32_t device, int64_t expected_build_rows, void* stream);

/* join_build_consume_batch_py_entry (_join.cpp:4149-4185): appends a build batch; on is_last builds the
 * hash table + CSR groups (JoinPartition::BuildHashTable / FinalizeGroups, _join.cpp:381-512). */
int b200_join_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last,
                                  int32_t* request_input);

/* join_probe_consume_batch_py_entry (_join.cpp:4205-4260): probes one batch and materialises the joined
 * rows (kept build columns then kept probe columns, reference order: build table first) into
 * library-owned device columns described by `out` (valid until the next probe call). *total_rows
 * receives the number of output rows of this call. */
int b200_join_probe_consume_batch(void* state, const b200_table* in_table,
                                  const uint64_t* kept_build_cols, int64_t n_kept_build,
                                  const uint64_t* kept_probe_cols, int64_t n_kept_probe,
                                  b200_table* out, int64_t* total_rows, int32_t is_last,
                                  int32_t* out_is_last);

/* delete_join_state (_join.cpp:4429). */
void b200_delete_join_state(void* state);
/* Join kind, to be called between init and the first build batch: mark join (HashJoinState::is_mark_join, _join.h:402 — every
 * probe row goes out once, no build columns, plus one trailing BOOL column "has a match": `out->cols` needs n_kept_probe + 1
 * descriptors) or probe-side anti join (the is_anti_join template argument of the reference's probe, _join.cpp:763-767 — a probe
 * row goes out, with NULL build columns, iff no build row matches).  build_table_outer must be false for both. */
int b200_join_set_kind(void* state, int32_t is_mark_join, int32_t is_anti_join);
/* Non-equi condition (the cond_func argument of join_state_init_py_entry, _join.cpp:4087-4136; bodo/libs/streaming/join.py:991-1100
 * builds it from the `non_equi_condition` string; the GPU path runs cudf::filter_join_indices after the hash join), to be called
 * between init and the first build batch: `program` is n_instr b200_expr_instr (below) forming ONE expression that ends in END.
 * An EX_COL argument c < 32 reads build column c, 32 + c probe column c (physical, keys-first column order of each side).  Build
 * columns are checked here, probe columns when the probe schema is known (here, or at the first probe batch).  A candidate pair
 * (a probe row and a build row with an equal key) joins when the condition is valid and true (b200_filter_project's semantics);
 * the join kinds then apply to the passing pairs: a probe row with none is NULL-extended (probe_table_outer), kept by an anti
 * join, marked false by a mark join; a build row is matched (build_table_outer) only through a passing pair.  The state always
 * takes the general (CSR) table, never the unique-key tables of metrics 5-7. */
int b200_join_set_condition(void* state, const void* program, int32_t n_instr);

/* As-of join, the contract of pandas.merge_asof (the reference's streaming join has no counterpart); call it before the first
 * build batch, like b200_join_set_condition.  build_on_col / probe_on_col are physical, non-key columns of the same c-type: any
 * integer width, FLOAT32, FLOAT64, DATE, DATETIME or TIMEDELTA (not BOOL); the probe side is checked when its schema arrives.
 * For probe row p the candidates are the build rows with equal keys (NA keys as is_na_equal says); with v = p's `on` value and w
 * a candidate's:
 *   direction 0 (backward): the largest w <= v (w < v when allow_exact_matches is 0); among equal w the last in build arrival
 *   order (batch order, then row order).  1 (forward): the smallest w >= v (w > v); among equal w the first.  2 (nearest): the
 *   backward and forward candidates, the one with the smaller |v - w|; a tie goes to the backward one.
 * With has_tolerance the match is dropped when |v - w| > tolerance, in the column's units (ns for DATETIME / TIMEDELTA, days for
 * DATE): tolerance_i64 (>= 0) for integer and temporal columns, where the difference is exact, tolerance_f64 (finite, >= 0) for
 * float columns, where it is computed in float64.  An NA `on` cell (null, or NaN) never matches, on either side; -0.0 equals 0.0.
 * probe_table_outer (the left as-of join, pandas' only form) emits every probe row once, NULL-extended without a match; without
 * it (inner as-of) only matched probe rows go out.  Output rows are in probe order; the probe side need not be sorted.  Fails
 * on a key or out-of-range column, a BOOL or mismatched `on` type, a negative or non-finite tolerance, a build_table_outer
 * state, and a mark, anti or condition join. */
int b200_join_set_asof(void* state, int32_t build_on_col, int32_t probe_on_col, int32_t direction, int32_t allow_exact_matches,
                       int32_t has_tolerance, int64_t tolerance_i64, double tolerance_f64);

/* Runtime join filter (HashJoinState::RuntimeFilter, _join.h:1060-1095; bloom filter bodo/libs/gpu_bloom_filter.cu:60-201; key
 * min / max _join.cpp:3199-3238), available once the build side is complete.  The reference keeps one bloom filter over the whole
 * key and bounds per key column; so does this, for any key count (1..4).
 * b200_join_build_filter builds a split-block bloom filter over the hashes of the build key tuples (n_bloom_blocks 32-byte blocks,
 * 0 = one per 32 build rows) and writes 2 * n_keys bounds (min_0, max_0, min_1, max_1, ...); it returns the device address of the
 * filter words (n_blocks * 8 uint32) so that the ranks of a sharded join can OR their filters together in place (all ranks pass the
 * same n_bloom_blocks; b200_join_set_key_bounds_n installs the reduced bounds, n_keys must be the state's).
 * b200_join_runtime_filter_n writes keep_out[i] = 1 for the rows of a DEVICE-resident table that can still find a partner (inside
 * the bounds, bloom hit): the rows a probe-side scan may drop before they are shuffled or probed (inner and build-outer joins only
 * — an outer probe side must keep its rows).  It takes the table column of every key position (key_cols[j] = -1: absent; the
 * bounds then apply to the present columns — use_min_max[j] per column — and the bloom filter only when every column is present;
 * with no column present every row is kept).  NA (and NaN) key columns: with is_na_equal a row with NA key columns is kept when it
 * can still match (its NA columns skip the bounds and are hashed as the build side hashes them); without it such a row is dropped.
 * Bounds of float keys cover the keys that are neither NA nor NaN, as an order-preserving int64 encoding: the double's bit
 * pattern (a float32 key widened first, -0.0 as +0.0), with bits 0..62 flipped when the sign bit is set.  int64 min / max of
 * encodings is the encoding of the float min / max, so ranks reduce them as they reduce integer bounds. */
int b200_join_build_filter(void* state, int64_t n_bloom_blocks, void** bloom_words_dev, int64_t* n_blocks_out, int64_t* key_min_max);
int b200_join_set_key_bounds_n(void* state, const int64_t* key_min_max, int32_t n_keys);
int b200_join_runtime_filter_n(void* state, const b200_table* in_table, const int32_t* key_cols, int32_t n_keys,
                               const int32_t* use_min_max, int32_t use_bloom, uint8_t* keep_out);

/* Operator metrics (the reference's JoinMetrics, bodo/libs/streaming/_join.h): 0 build rows, 1 hash-table slots, 2 probe rows,
 * 3 output rows, 4 kernel launches, 5 probe batches through a fused (unique-build-key) probe kernel, 6 of those through the
 * inline-payload kernel (key + payload in one 32-byte slot), 7 inline-payload table builds, 8 candidate pairs the non-equi
 * condition evaluated, 9 of those that passed (8 and 9 stay 0 without a condition). */
int64_t b200_join_get_metric(void* state, int32_t which);

/* ---- streaming top-k: ORDER BY ... LIMIT ... OFFSET (reference: bodo/libs/streaming/_sort.cpp) ---- */

/* stream_sort_state_init_py_entry (_sort.cpp), LIMIT form only.  The result is rows [offset, offset + limit) of the input
 * sorted stably (ties keep arrival order: batch order, then row order) by the first n_keys (1..4) of the n_arrs (<= 32) columns;
 * every column is fixed width (integer, float, bool, date, datetime, timedelta; numpy or nullable).  ascending[j] and na_last[j]
 * (na_position "last" = 1, "first" = 0) are per key; a nullable NA and a float NaN are both NA; -0.0 and 0.0 tie.  0 <= limit,
 * 0 <= offset and limit + offset <= 2^26 (the store's uint32 row ids and its two buffers of max(2 (limit + offset), 4 Mi) rows).
 * A dictionary-id key column sorts by id, not by string. */
void* b200_sort_state_init(int64_t operator_id, int64_t limit, int64_t offset, const int8_t* c_types, const int8_t* arr_types,
                           int32_t n_arrs, int32_t n_keys, const int32_t* ascending, const int32_t* na_last,
                           int64_t output_batch_size, int32_t device, void* stream);

/* stream_sort_state_init_py_entry (_sort.cpp), the form without LIMIT: a full sort.  The result is every input row, sorted
 * stably by the same key, type and NA rules as b200_sort_state_init; it equals df.sort_values(by, kind="stable").  The state
 * holds the whole input in device memory (fixed 2^24-row chunks) and sorts it at is_last with an LSD radix sort; at most 2^31
 * rows (32-bit row ids), a consume call past that fails before it launches anything.  The build-consume, produce, delete and
 * metric entries below serve both forms. */
void* b200_sort_state_init_full(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs, int32_t n_keys,
                                const int32_t* ascending, const int32_t* na_last, int64_t output_batch_size, int32_t device,
                                void* stream);

/* The sharded full sort's receive side: a full sort whose input is n_runs (>= 1) runs of run_lengths[r] (>= 0, summing to at
 * most 2^31) rows, consumed back to back in run order, each already sorted by these keys.  is_last merges the runs (ceil(log2
 * n_runs) merge-path rounds) instead of sorting; rows that tie on every key keep their input order, so runs from source ranks
 * 0, 1, ... give the stable sort of the rank inputs concatenated in rank order.  is_last fails when the rows consumed differ
 * from the sum of the lengths.  Unsorted runs give a permutation of the input in an unspecified order. */
void* b200_sort_state_init_runs(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs, int32_t n_keys,
                                const int32_t* ascending, const int32_t* na_last, const int64_t* run_lengths, int32_t n_runs,
                                int64_t output_batch_size, int32_t device, void* stream);

/* Samples a finished full sort (b200_sort_state_init_full or _runs, after is_last): record i (0 <= i < n_samples <= rows) is
 * output row q_i = floor(i * rows / n_samples) as 2 n_keys + 2 uint64 words: per key its NA class (0 or 1, the class that sorts
 * first is 0) and radix word, the sort's own key encoding, then rank and q_i.  Records compare lexicographically word by word
 * in the order of the rows.  `records` is host memory of n_samples * (2 n_keys + 2) words. */
int b200_sort_sample(void* state, int64_t n_samples, int64_t rank, uint64_t* records);

/* counts[k] (host) = the rows of a finished full sort whose record (the words b200_sort_sample would give them, with this rank)
 * is below splitters[k] (host, records of the same layout), 0 <= k < n_splitters: a device binary search over the sorted rows.
 * Rows [counts[k - 1], counts[k]) lie between two nondecreasing splitters. */
int b200_sort_count_below(void* state, const uint64_t* splitters, int64_t n_splitters, int64_t rank, int64_t* counts);

/* Window functions over (PARTITION BY p ORDER BY o), as a third form of the sort state (the reference plans these through its
 * window / MRNF arguments, which the groupby ABI above drops).  The keys are the first n_partition_keys + n_order_keys (0 <= each,
 * 1 <= sum <= 4) of the n_arrs columns, partition keys first; key columns are distinct and of the sort's key types.  PARTITION BY
 * keys sort ascending with NA last; ORDER BY key j takes order_ascending[j] and order_na_last[j].  Two cells of a key are equal
 * when both are NA (a float NaN is NA) or both are valid with equal radix words (-0.0 equals 0.0).  Rows with equal partition
 * keys are a partition; rows of a partition with equal order keys are peers (without ORDER BY every row of a partition is a peer
 * of every other).
 * The ranking functions use codes local to this library: 0 row_number, 1 rank, 2 dense_rank, 3 percent_rank, 4 cume_dist, 5 ntile.
 * With s the partition size and k the row's 0-based position in it: row_number = k + 1 (ties in arrival order); rank = 1 + rows
 * before the row's first peer; dense_rank = 1 + peer groups before the row's; percent_rank = (rank - 1) / (s - 1), 0.0 when
 * s = 1; cume_dist = rows up to and including the row's last peer / s; ntile(n): with q = s / n and r = s % n the first r buckets
 * hold q + 1 rows and the others q (buckets 1..s when n > s).  row_number, rank, dense_rank and ntile are INT64, percent_rank and
 * cume_dist FLOAT64 (one IEEE double division of the two integers); all numpy arrays. */

/* The bounds of a frame 4 (ROWS BETWEEN start AND end): each UNBOUNDED (the sentinels below) or a signed row offset from the
 * current row, -2^31 < offset < 2^31: negative PRECEDING, 0 CURRENT ROW, positive FOLLOWING; start <= end when both are offsets.
 * For row i of the partition [P, pe) (sorted positions) the frame is [lo, hi] with lo = P for an unbounded start, else
 * max(P, i + start), and hi = pe - 1 for an unbounded end, else min(pe - 1, i + end); it is empty when lo > hi.
 * (UNBOUNDED, 0) is frame 2 and (UNBOUNDED, UNBOUNDED) frame 3, with the same results. */
#define B200_WINDOW_UNBOUNDED_PRECEDING INT64_MIN
#define B200_WINDOW_UNBOUNDED_FOLLOWING INT64_MAX
typedef struct b200_window_frame {
    int64_t start, end;
} b200_window_frame;

/* The bounds of a frame 5 (RANGE BETWEEN start AND end), measured in ORDER BY values.  Kinds: 0 UNBOUNDED PRECEDING,
 * 1 PRECEDING, 2 CURRENT ROW, 3 FOLLOWING, 4 UNBOUNDED FOLLOWING, with start_kind <= end_kind, start_kind != 4 and end_kind != 0.
 * The bits of kinds 1 and 3 hold the offset's magnitude k in the key's arithmetic: a non-negative int64 for an integer key, days
 * for DATE, ns for DATETIME and TIMEDELTA, the bits of a finite, non-negative double for a FLOAT32 / FLOAT64 key; the other kinds'
 * bits are not read.  For row i of the partition [P, pe) (sorted positions):
 *   UNBOUNDED is P (start) or pe - 1 (end).  CURRENT ROW is the row's peer group: its first peer (start) or its last peer (end);
 *   it takes any ORDER BY, including none and several keys.
 *   k PRECEDING / k FOLLOWING need exactly one ORDER BY key x, an integer (8 to 64 bits, signed or unsigned), FLOAT32, FLOAT64,
 *   DATE, DATETIME or TIMEDELTA, numpy or nullable (not BOOL).  With x ascending, a k PRECEDING start is the first row of the
 *   partition's non-NA run with x_j >= x_i - k, a k FOLLOWING end the last row with x_j <= x_i + k, a k PRECEDING end the last row
 *   with x_j <= x_i - k and a k FOLLOWING start the first row with x_j >= x_i + k; with x descending PRECEDING means larger
 *   values, so the signs swap.  Integer and temporal keys compare exactly, with no wrap: a bound beyond the type's range reaches
 *   the end of the non-NA run.  Float keys compare against fl(x_i -+ k) in IEEE double (FLOAT32 widened exactly first), so -0.0
 *   equals 0.0 and at x_i = +inf a k PRECEDING start is the first +inf row.
 *   NA and NaN cells are one peer group at one end of the partition (order_na_last).  At an NA row an offset bound is that peer
 *   group's first (start) or last (end) row; at a non-NA row an offset bound never reaches an NA row, and an offset bound that no
 *   non-NA row satisfies leaves the frame empty.
 * The frame is [lo, hi], empty when lo > hi; the definitions of frame 4 over [lo, hi] apply.  (UNBOUNDED PRECEDING, CURRENT ROW)
 * is frame 1 and (UNBOUNDED PRECEDING, UNBOUNDED FOLLOWING) frame 3, with the same results. */
typedef struct b200_window_range {
    int32_t start_kind, end_kind;
    uint64_t start_bits, end_bits;
} b200_window_range;

/* One window function of b200_window_state_init.
 *   code: 0 row_number, 1 rank, 2 dense_rank, 3 percent_rank, 4 cume_dist, 5 ntile (the ranking functions above), then the value
 *         functions 6 sum, 7 count, 8 mean, 9 min, 10 max, 11 first_value, 12 last_value, 13 lag, 14 lead, 15 nth_value,
 *         16 var, 17 std, 18 var_pop, 19 std_pop, 20 covar_samp, 21 covar_pop, 22 corr, 23 regr_slope, 24 regr_intercept.
 *   col: the input column (0 <= col < n_arrs) a value function reads, any column including a key; -1 for a ranking function and
 *        for count(*).
 *   frame: 0 for a ranking function, lag and lead; for the others 1 range (RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW: up
 *          to the row's last peer; the whole partition without ORDER BY), 2 rows (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT
 *          ROW: up to the row itself, ties in arrival order), 3 partition (the whole partition).  Frames 1..3 start at the
 *          partition's first row.  4 rows between: ROWS BETWEEN start AND end of the function's rows.  5 range between: RANGE
 *          BETWEEN start AND end of the function's range.  Every value function other than lag and lead takes frames 1..5.
 *   arg: ntile's n (>= 1); lag / lead's offset k (0 <= k < 2^31; k = 0 is the row itself); nth_value's n (1 <= n < 2^31); the
 *        second column (x, 0 <= arg < n_arrs; any column including a key, and the two may be the same) of codes 20..24, whose
 *        first column (y) is col.  Not read by the other codes.
 *   default_valid, default_bits: lag / lead's value when row i - k / i + k is outside the row's partition: the low bytes of
 *          default_bits in the column's type if default_valid, else NA.
 *   rows: the bounds of frame 4, read only when frame == 4.
 *   range: the bounds of frame 5, read only when frame == 5.
 *   ignore_nulls: non-zero marks the function IGNORE NULLS, 0 RESPECT NULLS; a non-zero flag is accepted for codes 11 first_value,
 *          12 last_value, 13 lag, 14 lead and 15 nth_value only.
 * Over a frame [P, e] (a float NaN is NA for the aggregates):
 *   count     non-NA cells, or e - P + 1 for count(*); INT64, numpy.
 *   sum       sum of the non-NA cells, NA when there are none; integers and bool wrap in 64 bits (INT64 for signed and bool,
 *             UINT64 for unsigned), floats accumulate in double (float32 narrowed once at the end) in an order fixed by the row
 *             count; nullable.  Not for temporal columns.
 *   mean      sum / count in double ((double) of the exact 64-bit sum for integers and bool), NA when count = 0; FLOAT64, nullable.
 *             Not for temporal columns.
 *   min, max  the cell of the earliest row holding the least / greatest non-NA value, compared by the sort's ascending radix
 *             word (-0.0 ties 0.0); NA when the frame has no valid cell; the column's type, nullable.
 *   first_value, last_value  the cell at P / e as it is (bits and validity: a NaN stays a valid NaN); the column's type, nullable.
 *   lag, lead the cell at i - k / i + k when that row is in the row's partition, else the default; the column's type, nullable.
 *   nth_value the cell at P + n - 1 as it is when that row is in the frame, else NA; the column's type, nullable.
 *   var, std, var_pop, std_pop  with m the frame's non-NA cells (integers and bool converted to double, exact up to 2^53) and
 *             M2 = sum (x - mean)^2 over them: 16 var = M2 / (m - 1), NA when m < 2 (VAR_SAMP); 17 std = sqrt(var) (STDDEV_SAMP);
 *             18 var_pop = M2 / m, NA when m = 0, 0.0 when m = 1 (VAR_POP); 19 std_pop = sqrt(var_pop) (STDDEV_POP).  M2 is
 *             combined from (count, mean, M2) triples by Chan's pairwise merge in the scan's or the frame tree's order: never
 *             negative, exactly 0.0 over equal values, a valid NaN when the frame holds +-inf.  FLOAT64, nullable.  Not for
 *             temporal columns.
 *   covar_samp, covar_pop, corr, regr_slope, regr_intercept  with y = col and x = arg, m the frame's rows where both cells are
 *             non-NA (pairwise deletion; integers and bool converted to double, exact up to 2^53), and over them the means
 *             mx, my and Sxx = sum (x - mx)^2, Syy = sum (y - my)^2, Sxy = sum (x - mx)(y - my): 20 covar_samp = Sxy / (m - 1),
 *             NA when m < 2 (COVAR_SAMP(y, x)); 21 covar_pop = Sxy / m, NA when m = 0 (COVAR_POP); 22 corr = Sxy / sqrt(Sxx Syy),
 *             NA when m < 2, Sxx = 0 or Syy = 0, Sxy / (sqrt(Sxx) sqrt(Syy)) when Sxx Syy overflows or is subnormal, clamped
 *             to [-1, 1] (CORR); 23 regr_slope = Sxy / Sxx, NA when Sxx = 0 (REGR_SLOPE(y, x)); 24 regr_intercept =
 *             my - regr_slope mx, NA when Sxx = 0 (REGR_INTERCEPT(y, x)).  (count, mx, my, Sxx, Syy, Sxy) is combined by the
 *             bivariate form of Chan's merge, with no sum of products: covar and corr are bit-symmetric in (x, y), x = y gives
 *             corr 1.0 exactly where Sxx > 0 (and Sxx^2 is normal), equal x gives Sxx = 0 exactly; a valid NaN when the
 *             frame's counted pairs hold +-inf.  FLOAT64, nullable.  Not for temporal columns.
 * Every row that shares a frame end gets a bit-identical result.
 * Over a frame 4 or 5 [lo, hi] the same definitions hold with lo in place of P and hi in place of e; an empty frame (lo > hi)
 * gives NA, and count 0.  Float sums there are combined in an order fixed by (lo, hi) alone, so rows with the same bounds get the
 * same bits, across runs and batch splits.
 * IGNORE NULLS: a cell is null exactly when count does not count it: its validity is clear or it is a float NaN (RESPECT NULLS
 * first_value returns a NaN as a valid cell; IGNORE NULLS skips it, as pandas' ffill / bfill do).  With row i's frame [lo, hi]
 * and partition [P, pe) as RESPECT NULLS computes them (every frame 1..5, the same empty-frame rule):
 *   first_value  the first non-null cell in [lo, hi]; NA if none.
 *   last_value   the last non-null cell in [lo, hi]; NA if none.
 *   nth_value    the n-th non-null cell in [lo, hi] (FROM FIRST); NA if there are fewer than n.
 *   lag          the k-th non-null cell before row i within [P, i); the default if there are fewer than k.
 *   lead         the k-th non-null cell after row i within (i, pe); the default if there are fewer than k.
 * lag / lead with k = 0 are the row itself, as under RESPECT NULLS.  The result keeps the chosen cell's bits (-0.0 stays -0.0);
 * the column's type, nullable.  Results depend only on the sorted positions: bit-identical across runs and batch splits. */
typedef struct b200_window_func {
    int32_t code, col, frame, default_valid;
    int64_t arg;
    uint64_t default_bits;
    b200_window_frame rows;  /* read only when frame == 4 */
    b200_window_range range; /* read only when frame == 5 */
    int32_t ignore_nulls;    /* non-zero: IGNORE NULLS; codes 11..15 only */
} b200_window_func;

/* The window state with n_funcs functions, one descriptor each (n_arrs + n_funcs <= 32).  The output is every input row once,
 * in the stable sort's order by (partition keys, order keys, arrival): the n_arrs input columns, then one column per function
 * in descriptor order, so `out->cols` of a produce call holds n_arrs + n_funcs descriptors.  At most 2^31 rows, as the full
 * sort.  The build-consume, produce, delete and metric entries below serve this form too; metric 9 is the number of partitions.
 * Fails here (NULL, last error set) on: a bad code, column index, frame, ntile n, lag / lead k or nth_value n (outside
 * [1, 2^31)); a frame on a ranking function, lag or lead; a frame 4 bound outside the domain above, or start > end; bad frame 5
 * kinds, an offset without exactly one ORDER BY key, an offset on a BOOL key, a negative or non-finite offset, or start after
 * end; a bad arg of codes 20..24; sum, mean, var, std, var_pop, std_pop or codes 20..24 over a temporal column (either column
 * for 20..24); a non-zero ignore_nulls on a code other than 11..15. */
void* b200_window_state_init(int64_t operator_id, const int8_t* c_types, const int8_t* arr_types, int32_t n_arrs,
                             int32_t n_partition_keys, int32_t n_order_keys, const int32_t* order_ascending,
                             const int32_t* order_na_last, const b200_window_func* funcs, int32_t n_funcs,
                             int64_t output_batch_size, int32_t device, void* stream);

/* The build-consume entry of _sort.cpp: filters a DEVICE-resident batch (same schema as the state) against the current cutoff on
 * the device (full sort: appends it to the chunk store); on is_last reduces to the final rows (full sort: sorts every row).
 * Returns 1 after is_last, 0 otherwise, < 0 on error; *request_input = 1. */
int b200_sort_build_consume_batch(void* state, const b200_table* in_table, int32_t is_last, int32_t* request_input);

/* The produce-output entry of _sort.cpp: fills `out` (out->cols with room for n_arrs descriptors, n_arrs + n_funcs for a window) with library-owned device
 * columns of the next <= output_batch_size result rows, in order; valid until delete.  Sets *out_is_last. */
int b200_sort_produce_output_batch(void* state, b200_table* out, int32_t* out_is_last, int32_t produce_output);

/* delete_stream_sort_state (_sort.cpp). */
void b200_delete_sort_state(void* state);

/* Metrics: 0 rows consumed, 1 rows admitted as candidates, 2 reduce steps, 3 host reads of the candidate count, 4 filter
 * launches, 5 rows admitted while a cutoff existed, 6 store capacity in rows, 7 digit passes run (full sort), 8 digit passes
 * skipped because their digit is constant over all rows (full sort), 9 partitions (window).  A full sort or window reads 0 for
 * metrics 1-5; top-k reads 0 for 7 to 9 and a full sort for 9.  Full-sort passes: per key one per byte of its width, plus one NA-class pass for a nullable or float key. */
int64_t b200_sort_get_metric(void* state, int32_t which);

/* ---- row -> rank shuffle (reference: bodo/libs/_shuffle.cpp) ---- */

/* hash_keys_table(SEED_HASH_PARTITION) + hash_to_rank (bodo/libs/_array_hash.cpp:76-109,
 * _shuffle.h:5-7): dest[i] = (uint32)XXH3_64bits_withSeed(&key[i], 8, 0xb0d01289) % n_pes. Writes
 * per-row destinations (device int32) — exposed for placement-parity tests. */
int b200_hash_to_rank(const b200_table* in_table, int32_t n_pes, int32_t* dest_out, void* stream);
/* hash_keys_table(table, n_keys, SEED_HASH_PARTITION) (bodo/libs/_array_hash.cpp:1599-1621) over the first n_keys (1..4)
 * columns: integer / date columns hash their sizeof(T) raw bytes, float columns go through _Py_HashDouble first
 * (:119-170), NA -> hash_na_val, further columns are folded in with hash_combine_boost (:41-56).  Writes the 32-bit row
 * hashes (hash_out, device uint32, may be NULL) and / or hash % n_pes (dest_out, device int32, may be NULL). */
int b200_hash_keys_table(const b200_table* in_table, int64_t n_keys, int32_t n_pes, int32_t* dest_out,
                         uint32_t* hash_out, void* stream);

/* mpi_comm_info::set_send_count + fill_send_array (bodo/libs/_shuffle.cpp:94-163,345-368,477+) as one
 * radix-partition pass: histogram of destinations, exclusive scan, stable scatter of every column
 * into per-destination contiguous segments. `out` columns (device, same schema/length as the input,
 * provided by the caller) receive the rows grouped by destination; send_counts (host, n_pes) the
 * rows per destination. Validity bitmaps are re-packed per destination segment at byte granularity
 * (segment d starts at byte offset of a fresh bitmap: see DESIGN.md). */
int b200_shuffle_partition(const b200_table* in_table, int64_t n_keys, int32_t n_pes,
                           b200_table* out, int64_t* send_counts, void* stream);
/* Same, and also writes the source row of every output row to perm_out_dev (device int64[n_rows]);
 * used by the parity tests to compare the placement with the oracle row by row. */
int b200_shuffle_partition_perm(const b200_table* in_table, int64_t n_keys, int32_t n_pes,
                                b200_table* out, int64_t* send_counts, int64_t* perm_out_dev,
                                void* stream);
/* The same partition by key class: rows whose keys are equal as the window, the sort and the groupby compare them go to one
 * rank.  NA and a float NaN are one class (both hash as hash_na_val), -0.0 equals 0.0, and every fixed-width key type is
 * accepted: bool, 1-, 2-, 4- and 8-byte integers (a 1- or 2-byte key hashes as the 4-byte integer of its value), float32 /
 * float64, DATE, DATETIME and TIMEDELTA, numpy or nullable.  On keys of 4 or 8 bytes without a valid NaN the placement is
 * b200_shuffle_partition's.  perm_out_dev (device int64[n_rows]) may be NULL. */
int b200_shuffle_partition_classes(const b200_table* in_table, int64_t n_keys, int32_t n_pes,
                                   b200_table* out, int64_t* send_counts, int64_t* perm_out_dev,
                                   void* stream);

/* Receive side of shuffle_table: turns the n_src per-source validity segments (each ceil(counts[j]/8) bytes, back to
 * back, in source-rank order — what the all-to-all-v of the per-destination bitmaps delivers) into one contiguous Arrow
 * bitmap of sum(counts) rows.  out_bitmap must hold 4 * ceil(sum(counts) / 32) bytes on `device`. */
int b200_merge_segment_bitmaps(const uint8_t* segments, const int64_t* counts, int32_t n_src,
                               uint8_t* out_bitmap, int32_t device, void* stream);

/* ---- fused filter + projection front end (reference: bodo/pandas/physical/filter.h, project.h, expression.{h,cpp};
 *      GPU twins gpu_expression.cpp:601+ / gpu_filter.h:143 built on cudf::ast + apply_boolean_mask) ---- */

/* One postfix instruction: op (EX_* below) + 64-bit argument (column index, or the bits of an int64 / double constant).
 * EX_COL=0 CONST_I64=1 CONST_F64=2 ADD=3 SUB=4 MUL=5 DIV=6 LT=7 LE=8 GT=9 GE=10 EQ=11 NE=12 AND=13 OR=14 NOT=15
 * TO_F64=16 TO_I64=17 IS_NULL=18 NEG=19 END=20.  A program is a sequence of expressions, each terminated by END and
 * leaving one value; arithmetic / comparisons propagate NA, AND / OR are Kleene, a NA predicate drops the row.  AND / OR /
 * NOT and the predicate take value != 0 as true (a float -0.0 is false, NaN read from a float column is NA). */
typedef struct b200_expr_instr { int32_t op; int32_t pad; int64_t arg; } b200_expr_instr;

/* Evaluates the predicate (expression starting at instruction pred_start; -1 = keep every row) and the n_out output
 * expressions (starting at out_starts[j]) of every row of a device-resident table in ONE kernel, compacting the surviving
 * rows: out->cols[j] (device buffers of in_table->n_rows items provided by the caller, c_type = storage type, validity =
 * bitmap buffer or NULL) receive the rows that pass, in an unspecified order (each 1024-row tile claims its place with an
 * atomic cursor).  Every start must be 0 or follow an END.  Returns the number of output rows (< 0 on error). */
int64_t b200_filter_project(const b200_table* in_table, const void* program, int32_t n_instr, int32_t pred_start,
                            const int32_t* out_starts, int32_t n_out, b200_table* out, void* stream);

/* out[i] = map[in[i]] (0 where invalid): the transpose step of dictionary unification
 * (DictionaryBuilder::UnifyDictionaryArray, bodo/libs/_dict_builder.cpp): batch-local dictionary indices -> global ids. */
int b200_remap_i32(const int32_t* in_dev, const uint8_t* valid_dev, int64_t n, const int32_t* map_dev, int32_t map_len,
                   int32_t* out_dev, int32_t device, void* stream);

/* ---- helpers for host code that does not link CUDA ---- */
void* b200_device_malloc(int32_t device, int64_t nbytes);
void b200_device_free(int32_t device, void* p);
/* Scratch memory (owner buckets, retry lists, staging) comes from a process-wide, stream-ordered per-device pool that
 * keeps freed blocks for the next operator state; this returns pooled blocks beyond keep_bytes to the driver. */
int64_t b200_pool_trim(int32_t device, int64_t keep_bytes);
int b200_memcpy_d2h(void* dst_host, const void* src_dev, int64_t nbytes, void* stream);
int b200_memcpy_h2d(void* dst_dev, const void* src_host, int64_t nbytes, void* stream);
int b200_stream_synchronize(void* stream);

/* Synthetic table generator used by bench.py (counter-based, seeded; mirrored by the numpy generator
 * in bodo_b200/synth.py so the oracle sees the same rows): key = mix64(seed_k, row) % n_groups,
 * val = (int64)(mix64(seed_v, row) % 1000) - 500 (INT64) or u01 (FLOAT64). */
int b200_synth_fill(void* key_out, void* val_out, int64_t row_start, int64_t n_rows, int64_t n_groups,
                    uint64_t seed, int32_t val_c_type, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BODO_B200_H */
