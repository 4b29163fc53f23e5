/*
 * b200serve.h -- C-ABI of the H100 serving-graph engine (libb200serve.so).
 *
 * The reference (mlrun/mlrun) has no FFI on this path: its hot path is pure Python.  This header is
 * the boundary a maintainer binds (ctypes/cffi) to replace the per-event Python step loop with a batched
 * device plan.  Every entry point names the reference code it replaces (paths relative to the
 * reference root).  Plain pointers and sizes only; no Python / torch types cross it.
 *
 * Conventions
 *   - every call returns 0 on success or a negative b2s_status; the message is thread-local in
 *     b2s_last_error();
 *   - the caller owns host buffers (the library copies on submit); the library owns device memory;
 *   - a "row" is one event's feature vector: n_in_cols 4-byte words (float32, or int32 where the
 *     plan says so), rows `row_stride_bytes` apart;
 *   - outputs are `out_cols` 4-byte words per row (float32 for regression / transform outputs, int32
 *     for class labels), plus an int32 status word per row (0 = ok) so that the Python layer can turn
 *     a bad row into that event's 400 response (mlrun/serving/server.py:278-288) without failing the
 *     whole batch.
 */
#ifndef B200SERVE_H
#define B200SERVE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 100 /* 0.1.0 */

typedef enum b2s_status {
  B2S_OK = 0,
  B2S_ERR_INVALID = -1,   /* bad argument / plan not finalised / schema mismatch */
  B2S_ERR_CUDA = -2,      /* a CUDA runtime call failed (message has the CUDA error string) */
  B2S_ERR_NO_DEVICE = -3, /* no usable GPU: there is NO CPU fallback */
  B2S_ERR_STATE = -4,     /* call sequence error (not initialised, already finalised ...) */
  B2S_ERR_TIMEOUT = -5,
  B2S_ERR_UNSUPPORTED = -6
} b2s_status;

/* per-row status bits written next to each output row */
#define B2S_ROW_OK 0
#define B2S_ROW_NONFINITE_INPUT 1 /* NaN/Inf reached a model input: scikit-learn's predict raises
                                     ValueError there (called from pkl_model_server.py:58) */
#define B2S_ROW_BAD_LABEL 2       /* majority vote saw a negative label (serving/routers.py:717-725
                                     assumes labels 0..max) */
#define B2S_ROW_UNKNOWN_KEY 4     /* b2s_table_enrich_host: the entity key is not in the online table (the reference's
                                     OnlineVectorService.get returns None for it) */

typedef struct b2s_plan_s* b2s_plan_t;

/* output-schema column kinds (b2s_plan_set_output_schema) */
#define B2S_OUT_COPY 0   /* out = value of source column */
#define B2S_OUT_ONEHOT 1 /* out = (value == arg) ? 1 : 0 -- OneHotEncoder._encode, feature_store/steps.py:453-471 */

/* model link functions (what the estimator's predict() does after the raw score) */
#define B2S_LINK_IDENTITY 0   /* regression: out = score[0]                                   */
#define B2S_LINK_BINARY_GT 1  /* classes[score[0] >  0]  (sklearn LogisticRegression.predict) */
#define B2S_LINK_BINARY_GE 2  /* classes[score[0] >= 0]  (sklearn GradientBoostingClassifier) */
#define B2S_LINK_ARGMAX 3     /* classes[argmax_k score[k]], first max wins (np.argmax)       */

/* ensemble vote (VotingEnsemble._apply_logic, serving/routers.py:789-810) */
#define B2S_VOTE_NONE 0     /* emit every model's prediction: out_cols = n_models                 */
#define B2S_VOTE_MEAN 1     /* _mean_vote :732-741   -- sum_m w[m] * pred[m]  (fp64)             */
#define B2S_VOTE_MAJORITY 2 /* _majority_vote :708-730 -- argmax_c sum_m w[m]*[pred[m]==c], first max */

typedef struct b2s_stats {
  int64_t rows;          /* rows in the batch this call rode in                                  */
  float h2d_ms;          /* CUDA-event time of the host->device copy                             */
  float kernel_ms;       /* CUDA-event time of the plan's kernels (b2s_run_host pipelines large  */
  float d2h_ms;          /* pinned batches in chunks: kernel/d2h are then sums over the chunks)   */
  float queue_us;        /* submit -> batch sealed (coalescing wait)                             */
  int32_t kernels;       /* kernel launches in the batch                                         */
  int32_t nonfinite_rows;/* rows flagged B2S_ROW_NONFINITE_INPUT                                 */
} b2s_stats;

typedef struct b2s_devinfo {
  int32_t ordinal, sm_count, cc_major, cc_minor;
  int64_t total_mem, l2_bytes, smem_per_block_optin;
  char name[128];
} b2s_devinfo;

/* ---- library / device ---------------------------------------------------------------------- */
int b2s_version(void);
const char* b2s_last_error(void);
/* Replaces: nothing in the reference (device bring-up).  cfg is "key=value;..." or NULL:
 *   ring_slots (4), max_batch (65536 rows), max_wait_us (0: a coalesced batch leaves as soon as the dispatcher is free, so
 *   batches form while the previous one runs; > 0: the oldest row may wait that long for company).  Idempotent per process. */
int b2s_init(int device_ordinal, const char* cfg);
int b2s_shutdown(void);
int b2s_device_info(b2s_devinfo* out);
/* number of kernels this library has launched since b2s_init (for bench.py's gpu_launches) */
int64_t b2s_launch_count(void);

/* ---- plan construction ---------------------------------------------------------------------
 * A plan is the lowered form of a run of recognised graph steps.  It replaces, for those steps, the
 * reference's per-event loop  FlowStep.run (serving/states.py:1292-1323)  ->  TaskStep.run (:564-599)
 * -> step handler, and the storey Map chain built by _init_async_objects (:1622-1710). */
int b2s_plan_create(int32_t n_in_cols, b2s_plan_t* out);
int b2s_plan_destroy(b2s_plan_t plan);

/* Imputer._impute (feature_store/steps.py:397-406): NaN in column cols[i] -> fills[i]. */
int b2s_plan_set_impute(b2s_plan_t plan, const int32_t* cols, const float* fills, int32_t n);
/* MapValues._map_value exact-match branch (steps.py:200-201): v == keys[i] -> vals[i], else unchanged.
 * Maps are applied after the imputer, in the order they are added. */
int b2s_plan_add_value_map(b2s_plan_t plan, int32_t col, const float* keys, const float* vals, int32_t n);
/* MapValues._map_value range branch (steps.py:193-198): first i with lo[i] <= v < hi[i] -> vals[i]. */
int b2s_plan_add_range_map(b2s_plan_t plan, int32_t col, const float* lo, const float* hi, const float* vals, int32_t n);
/* Output schema after OneHotEncoder._do_storey (steps.py:473-478) / DropFeatures (:721-729):
 * out column j reads source column src_col[j] with kind[j] (B2S_OUT_*) and arg[j]. Default: identity. */
int b2s_plan_set_output_schema(b2s_plan_t plan, const int32_t* src_col, const int32_t* kind, const float* arg, int32_t n_out);

/* Linear scorer = what sklearn's linear estimators compute inside PickleModelServer.predict
 * (frameworks/_ml_common/pkl_model_server.py:52-60): score[k] = b[k] + sum_j W[k][j] * x_out[j] in fp64.
 * W is row-major (n_scores x n_out_cols).  classes: label per class index for the classifier links (may be NULL). */
int b2s_plan_add_linear_model(b2s_plan_t plan, const double* W, const double* b, int32_t n_scores, int32_t link,
                              const int32_t* classes, int32_t n_classes);
/* Tree-ensemble scorer (sklearn GradientBoosting* / RandomForest* / DecisionTree* behind the same
 * predict call).  Trees are concatenated SoA: node i of tree t lives at tree_offset[t] + i.
 *   feature[i] < 0 marks a leaf whose value is leaf_value[i]; otherwise go left when
 *   x[feature[i]] <= threshold[i] (sklearn: float32 x vs float64 threshold; thresholds are passed
 *   already rounded toward -inf to float32, which gives the identical decision).
 *   score[tree_slot[t]] += tree_scale[t] * leaf_value;  score[k] starts at init[k].
 * Scores: 1..32 per model (tree or linear), as for b2s_plan_add_linear_model; a tree plan holds up to 16 such models, so
 * up to 512 scores in all.  Every tree kernel holds one model's scores per row at a time. */
int b2s_plan_add_tree_model(b2s_plan_t plan, int32_t n_trees, const int32_t* tree_offset /* n_trees+1 */,
                            const int32_t* feature, const float* threshold, const int32_t* left,
                            const int32_t* right, const double* leaf_value, const int32_t* tree_slot,
                            const double* tree_scale, const double* init, int32_t n_scores, int32_t link,
                            const int32_t* classes, int32_t n_classes);
/* The same with the tree semantics of the other libraries behind the reference's model servers (XGBoostModelServer is
 * PickleModelServer, frameworks/xgboost/__init__.py:30; LGBMModelServer.predict, frameworks/lgbm/model_server.py:142-159):
 *   cmp_mode       B2S_CMP_LE: left when x <= threshold (scikit-learn, LightGBM);  B2S_CMP_LT: left when x < threshold (xgboost);
 *   default_left   per node (may be NULL = all 0): where a missing value (NaN) goes -- xgboost's "missing" child,
 *                  LightGBM's default_left, scikit-learn's tree_.missing_go_to_left;
 *   nan_mode       B2S_NAN_ERROR: a NaN input flags the row B2S_ROW_NONFINITE_INPUT (estimators whose predict refuses NaN);
 *                  B2S_NAN_DEFAULT_CHILD: NaN follows default_left.  It is honoured when every model of the plan routes
 *                  missing values and the plan runs on the shared-memory tree kernel (b2s_plan_kernel says so); in any
 *                  other plan a NaN row is still flagged -- an error, never a silently different answer.
 * Inf is flagged in both modes (what check_array / DMatrix refuse). */
#define B2S_CMP_LE 0
#define B2S_CMP_LT 1
#define B2S_NAN_ERROR 0
#define B2S_NAN_DEFAULT_CHILD 1
int b2s_plan_add_tree_model_ex(b2s_plan_t plan, int32_t n_trees, const int32_t* tree_offset /* n_trees+1 */,
                               const int32_t* feature, const float* threshold, const int32_t* left, const int32_t* right,
                               const double* leaf_value, const int32_t* tree_slot, const double* tree_scale,
                               const double* init, int32_t n_scores, int32_t link, const int32_t* classes, int32_t n_classes,
                               int32_t cmp_mode, const uint8_t* default_left, int32_t nan_mode);
/* The same with categorical splits (xgboost split_type 1, LightGBM decision_type "=="), in one canonical form the
 * exporters (mlrun_b200/tree_formats.py) normalise both libraries to:
 *   node_cat[i]    -1: a numeric node (the rules above);  s >= 0: node i tests x against set s, whose bitset is
 *                  cat_words[cat_offsets[s] .. cat_offsets[s + 1]) -- code c is bit (c % 32) of word (c / 32);
 *                  `threshold[i]` and `cmp_mode` do not apply to it;
 *   the node sends x RIGHT iff x is a valid code whose bit is set, and LEFT otherwise: an invalid code, a code past the
 *                  end of the set, and a value too large for int32 all go left.  NaN follows default_left[i] under
 *                  B2S_NAN_DEFAULT_CHILD (LightGBM's exporter sets it: NaN takes LightGBM's right child, which it maps to
 *                  the canonical left), and flags the row under B2S_NAN_ERROR, as for numeric nodes;
 *   cat_mode       the model's valid codes: B2S_CAT_NONNEG: x >= 0 (xgboost common::Decision);  B2S_CAT_TRUNC:
 *                  trunc(x) >= 0, i.e. x > -1 (LightGBM Tree::CategoricalDecision, x in (-1, 0) is code 0); the code
 *                  is trunc(x) in both.
 * Sets: n_sets entries, cat_offsets has n_sets + 1 non-decreasing entries from 0 to at most n_cat_words.  Each node's set
 * index must lie in [0, n_sets), and a leaf must have node_cat -1; anything else is B2S_ERR_INVALID.  A model whose
 * node_cat is NULL or all -1 behaves exactly as with b2s_plan_add_tree_model_ex. */
#define B2S_CAT_NONNEG 0
#define B2S_CAT_TRUNC 1
int b2s_plan_add_tree_model_cat(b2s_plan_t plan, int32_t n_trees, const int32_t* tree_offset /* n_trees+1 */,
                                const int32_t* feature, const float* threshold, const int32_t* left, const int32_t* right,
                                const double* leaf_value, const int32_t* tree_slot, const double* tree_scale,
                                const double* init, int32_t n_scores, int32_t link, const int32_t* classes, int32_t n_classes,
                                int32_t cmp_mode, const uint8_t* default_left, int32_t nan_mode,
                                const int32_t* node_cat, const int32_t* cat_offsets /* n_sets+1 */, int32_t n_sets,
                                const uint32_t* cat_words, int32_t n_cat_words, int32_t cat_mode);
/* VotingEnsemble reduce over the plan's models (weights in model order; fp64). */
int b2s_plan_set_vote(b2s_plan_t plan, int32_t vote_kind, const double* weights, int32_t n_weights);
/* Upload tables to HBM, pick kernels, size staging buffers.  After this the plan is immutable. */
int b2s_plan_finalize(b2s_plan_t plan);
/* name + template parameters of the kernel family the plan launches (diagnostics / bench provenance) */
const char* b2s_plan_kernel(b2s_plan_t plan);
/* The kernel family that served the plan's most recent launch (any entry point, any thread), after the run-time
 * demotions b2s_plan_kernel cannot see: rows in mapped host memory (small b2s_run_host batches), rows that are not
 * 16-byte aligned or strided, and a tensor map the driver refuses.  B2S_KERNEL_NONE before the first launch. */
#define B2S_KERNEL_NONE 0
#define B2S_KERNEL_DENSE 1             /* dense_head_kernel (wgmma tf32, TMA tensor-map loads)            */
#define B2S_KERNEL_TREES3_TMAP 2       /* t3_prep_kernel with TMA tensor-map loads + trees3 + vote        */
#define B2S_KERNEL_TREES3 3            /* the same with plain loads                                       */
#define B2S_KERNEL_TREES2_TMAP 4       /* retired (trees_model_kernel, TMA loads): no longer returned     */
#define B2S_KERNEL_TREES2 5            /* retired (trees_model_kernel): no longer returned                */
#define B2S_KERNEL_ROWTHREAD_TMA 6     /* rowthread kernel, TMA tensor-map loads (swizzled 2-D boxes)     */
#define B2S_KERNEL_ROWTHREAD_LDGSTS 7  /* rowthread kernel, cp.async loads from device memory             */
#define B2S_KERNEL_ROWTHREAD_HOST 8    /* rowthread kernel, cp.async loads from mapped host memory        */
#define B2S_KERNEL_ROWWARP 9           /* retired (rowwarp_kernel): no longer returned                    */
#define B2S_KERNEL_ROWS 10             /* generic rows_kernel (fp64, linear or trees)                     */
#define B2S_KERNEL_STORE 11            /* rows_kernel of a transform-only plan                            */
#define B2S_KERNEL_TREES3_CAT_TMAP 12  /* B2S_KERNEL_TREES3_TMAP, walk with categorical splits             */
#define B2S_KERNEL_TREES3_CAT 13       /* B2S_KERNEL_TREES3, walk with categorical splits                  */
#define B2S_KERNEL_ROWS_CAT 14         /* rows_kernel of a tree plan with categorical splits              */
#define B2S_KERNEL_ROWTHREAD_BULK 15   /* rowthread kernel, one TMA bulk copy per row (also the gather)   */
int32_t b2s_plan_last_kernel(b2s_plan_t plan);
/* out_cols 4-byte words per output row; out_is_int != 0 when they are int32 labels */
int b2s_plan_out_info(b2s_plan_t plan, int32_t* out_cols, int32_t* out_is_int);

/* ---- execution -------------------------------------------------------------------------------
 * Replaces GraphServer.run -> graph.run (serving/server.py:252-293) for a batch of events. */

/* Device-resident path: rows and outputs already in HBM (roofline runs, CUDA-graph capture, callers that
 * keep tensors on the GPU).  Asynchronous on `stream` (a cudaStream_t, NULL = the library's stream).
 * d_status may be NULL. */
int b2s_run_device(b2s_plan_t plan, const void* d_rows, int64_t n_rows, int64_t row_stride_bytes, void* d_out,
                   int32_t* d_status, void* stream);
/* Synchronous host call: rows -> kernels -> out.  row_status / stats may be NULL.  Pageable or strided rows are first
 * packed into the plan's pinned staging area; pinned rows are used where they are.  The kernels write votes and status
 * words straight to pinned host memory (no D2H copy), and read a batch of at most 64 KiB of rows from pinned host memory
 * too (no H2D copy: one launch and one synchronisation, the latency path of a serving batch); larger batches are copied
 * to the device first.  Pinned batches of 128 Ki rows and more are pipelined in chunks of 64 Ki rows or more (copy of
 * chunk c + 1 under the kernels of chunk c, results copied back per chunk).  A plan with merge targets or an attached
 * communicator writes no local results: B2S_ERR_UNSUPPORTED, before anything runs (use b2s_run_device). */
int b2s_run_host(b2s_plan_t plan, const void* rows, int64_t n_rows, int64_t row_stride_bytes, void* out,
                 int64_t out_bytes, int32_t* row_status, b2s_stats* stats);
/* Coalescing path (thread-safe, many producers): rows are copied into a pinned ring slot; a dispatcher
 * thread seals a batch when it holds max_batch rows or the oldest row waited max_wait_us (0: as soon as the dispatcher is
 * free -- batches form while the previous one runs), and runs it on its own stream as one b2s_run_host batch that is
 * never pipelined (results straight to the slot's pinned memory, rows read from there up to 64 KiB).  b2s_wait blocks
 * until the ticket's batch completed and copies that ticket's rows out (out_bytes must hold them); a batch that failed,
 * or of a plan with merge targets or an attached communicator (B2S_ERR_UNSUPPORTED), gives every one of its tickets the
 * error.  A ticket is collected once: waiting on it again, or on a ticket that was never issued, is B2S_ERR_INVALID and
 * leaves the other tickets of its batch alone.  This is the replacement of storey's SyncEmitSource.emit / await_result
 * hand-off (serving/states.py:1283-1287).  A ring slot is recycled when every ticket of its batch was collected, and the ring
 * has `ring_slots` (b2s_init cfg, default 4) batches: a producer that keeps submitting without collecting its tickets
 * eventually blocks in b2s_submit -- emit and await per request, as the reference's callers do. */
int b2s_submit(b2s_plan_t plan, const void* rows, int64_t n_rows, int64_t row_stride_bytes, uint64_t* ticket);
int b2s_wait(b2s_plan_t plan, uint64_t ticket, void* out, int64_t out_bytes, int32_t* row_status, b2s_stats* stats);
/* force the open batch out now (drain callback, serving/server.py:353-384) */
int b2s_flush(b2s_plan_t plan);
/* Per-plan ring configuration, before the plan's first b2s_submit: batches in flight, rows per batch and how long the
 * oldest row may wait for company (0 / 0 / negative keep the b2s_init defaults).  This is where a serving function's
 * `spec.parameters["b200"] = {"max_batch": .., "max_wait_us": .., "ring_slots": ..}` lands (runtimes/nuclio/serving.py:
 * 668-724 hands spec.parameters to the GraphServer). */
int b2s_plan_set_ring(b2s_plan_t plan, int32_t ring_slots, int64_t max_batch, int32_t max_wait_us);
/* The ring measured by itself: n_threads native producers, each emitting rows_per_submit rows of `rows` and awaiting them
 * (emit / await_result of one request), for `seconds`.  events = rows served; p50 / p99 of the submit -> wait round trip. */
int b2s_ring_bench(b2s_plan_t plan, const void* rows, int64_t n_src_rows, int64_t row_stride_bytes, int32_t n_threads,
                   int32_t rows_per_submit, double seconds, int64_t* events, double* p50_us, double* p99_us);

/* ---- multi-GPU: fused ensemble-merge ----------------------------------------------------------------
 * One process per GPU, events sharded by rows (they are independent: VotingEnsemble reduces across models,
 * serving/routers.py:797-810).  The only exchange is the merge of every shard's votes into the full
 * response.  Instead of a separate all-gather, a plan can be given the output buffers of all ranks
 * (peer-mapped over NVLink with the IPC calls below); its kernels then store each output row into every
 * target at row `row_offset + row` straight from the epilogue, the same words the plan writes locally (b2s_run_device
 * only: b2s_run_host, the ring and b2s_table_enrich_host / _device refuse the plan with B2S_ERR_UNSUPPORTED).  At most 8
 * targets; row_offset >= 0 needs no alignment.  n_peers = 0 restores local output. */
int b2s_plan_set_merge_targets(b2s_plan_t plan, void* const* peer_out, int32_t n_peers, int64_t row_offset);
int b2s_ipc_export(void* dptr, void* handle64 /* 64 bytes out */);
int b2s_ipc_open(const void* handle64, void** dptr_out);
int b2s_ipc_close(void* dptr);

/* The same exchange as a product object: a communicator owns, per rank, ONE device allocation -- completion flags and the
 * merged response rows in four slots -- that every peer maps over CUDA IPC.  Bootstrap needs any out-of-band channel
 * that can all-gather 64 bytes per rank (torch.distributed, MPI, a file, a socket ...):
 *     b2s_comm_create(rank, world, max_rows_per_rank, out_cols, &c);  b2s_comm_handle(c, mine);
 *     <all-gather the 64-byte handles>;  b2s_comm_connect(c, all);  b2s_plan_attach_comm(plan, c);
 * Every b2s_run_device launch of an attached plan (the host and enrichment entry points refuse it) is then one STEP (epoch
 * e = 1, 2, ...), a launch of 0 rows included: an empty shard stores nothing, but one small kernel still publishes its flag
 * (and runs the fused wait), so that every rank takes every step.  A step is one ensemble-merge
 * (serving/routers.py:414-455 fans the event out to the routes, :789-810 reduces them; here the rows are
 * sharded and the votes merged): the kernels store this rank's votes into slot e & 3 of EVERY rank's merged rows at row
 * block `rank`, and the launch's last CTA publishes e in every rank's flag array (st.release.sys).  b2s_comm_wait enqueues
 * a one-warp kernel that acquires all `world` flags of THIS rank at the current epoch, so work enqueued behind it (a D2H copy,
 * the next kernel) reads a complete response; *d_merged is that response, (world x max_rows_per_rank x out_cols) words, rank
 * r's rows at r * max_rows_per_rank.  Every launch must be followed by a wait on the same stream: b2s_comm_wait (step e,
 * lockstep) or b2s_comm_wait_lag(.., 1, ..) (step e - 1: the votes and flags of step e cross NVLink while step e + 1 is being
 * scored; the response of a step is then available one launch later, and a final b2s_comm_wait drains the last step).
 * Four slots make both safe: before a rank launches step e + 4 (which overwrites slot e & 3 everywhere) it has passed its
 * wait for step e + 2 at the latest, i.e. it has seen every peer's flag of step e + 2 -- and a peer's launch of step e + 2
 * sits behind that peer's wait for (and use of) step e in the peer's own stream.  A peer that never
 * signals makes the wait give up after B2S_COMM_TIMEOUT_MS (default 10 s; b2s_comm_check reports B2S_ERR_TIMEOUT) instead of hanging the GPU. */
typedef struct b2s_comm_s* b2s_comm_t;
int b2s_comm_create(int32_t rank, int32_t world, int64_t max_rows_per_rank, int32_t out_cols, b2s_comm_t* out);
int b2s_comm_handle(b2s_comm_t comm, void* handle64 /* 64 bytes out */);
int b2s_comm_connect(b2s_comm_t comm, const void* all_handles /* world x 64 bytes, in rank order */);
int b2s_plan_attach_comm(b2s_plan_t plan, b2s_comm_t comm /* NULL detaches */);
int b2s_comm_wait(b2s_comm_t comm, void* stream, const void** d_merged, uint32_t* epoch);
/* lag 0 or 1; with fewer than lag + 1 steps launched there is nothing to wait for: *d_merged = NULL, *epoch = 0 */
int b2s_comm_wait_lag(b2s_comm_t comm, void* stream, int32_t lag, const void** d_merged, uint32_t* epoch);
/* Fused wait: lag 0 / 1 makes every launch of an attached plan end by acquiring -- in the launch's last CTA, after it has
 * published its own flag -- this rank's flags of its own step / of the previous step (same timeout as the wait kernel);
 * b2s_comm_wait / b2s_comm_wait_lag then enqueue nothing for a step that is covered.  Saves the wait kernel and its two launch
 * boundaries per step (4.9 us of a 50 us step at 1 Mi events, 2 GPUs).  lag -1 = off (default). */
int b2s_comm_set_fused_wait(b2s_comm_t comm, int32_t lag);
int b2s_comm_check(b2s_comm_t comm);
int b2s_comm_destroy(b2s_comm_t comm);

/* pinned host memory for zero-extra-copy submits and for bench.py's e2e leg */
void* b2s_alloc_pinned(size_t bytes);
int b2s_free_pinned(void* p);
/* plain device memory helpers so that ctypes callers need no other CUDA binding */
void* b2s_device_alloc(size_t bytes);
int b2s_device_free(void* p);
int b2s_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes);
int b2s_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes);
int b2s_device_sync(void);
/* time n_iters back-to-back b2s_run_device launches with CUDA events on the library stream (ms total);
 * used by bench.py so that the timed region contains only the plan's kernels.  d_rows[i % n_bufs]. */
int b2s_time_device(b2s_plan_t plan, const void* const* d_rows, int32_t n_bufs, int64_t n_rows,
                    int64_t row_stride_bytes, void* d_out, int32_t n_iters, float* total_ms);

/* ---- columnar ingest: feature-set transforms over DataFrame-shaped data -------------------------------
 * Replaces the row-at-a-time walk of a feature-set graph by the storey engine
 * (feature_store/ingestion.py:38-127 init_featureset_graph; datastore/sources.py:886-895 DataframeSource emits one
 * dict per row; datastore/targets.py:1856-1868 ReduceToDataFrame re-assembles them).  Data is columnar on both
 * sides, like the DataFrame it comes from: an input/output "slot" is n_rows 4-byte words (float32 / int32); an
 * 8-byte column (datetime64[ns] as int64) takes two adjacent slots.  The plan is a list of column ops; every op
 * reads one input column and writes 0..n output columns; output slots are numbered in the order ops are added.
 * Float sources take an optional Imputer fill first (Imputer._impute, feature_store/steps.py:397-406).
 * `check` bits (1: min, 2: max) attach MinMaxValidator.check (mlrun/features.py:292-321) to the op's result:
 * violating rows are counted (the reference's FeaturesetValidator only prints them, steps.py:117-128). */
typedef struct b2s_cols_s* b2s_cols_t;
#define B2S_COL_F32 0
#define B2S_COL_I32 1
#define B2S_COL_I64 2
/* date parts of DateExtractor._do_storey (steps.py:593-602: getattr(pd.Timestamp(ts), part)) computed on the device */
#define B2S_DATE_YEAR 0
#define B2S_DATE_MONTH 1
#define B2S_DATE_DAY 2
#define B2S_DATE_HOUR 3
#define B2S_DATE_MINUTE 4
#define B2S_DATE_SECOND 5
#define B2S_DATE_DAY_OF_WEEK 6 /* Monday = 0 */
#define B2S_DATE_DAY_OF_YEAR 7
#define B2S_DATE_QUARTER 8
#define B2S_DATE_IS_LEAP_YEAR 9     /* the is_* parts give 0 / 1 */
#define B2S_DATE_DAYS_IN_MONTH 10
#define B2S_DATE_IS_MONTH_START 11
#define B2S_DATE_IS_MONTH_END 12
#define B2S_DATE_IS_QUARTER_START 13
#define B2S_DATE_IS_QUARTER_END 14
#define B2S_DATE_IS_YEAR_START 15
#define B2S_DATE_IS_YEAR_END 16
#define B2S_DATE_WEEK 17             /* ISO 8601 week (pd.Timestamp.week / weekofyear) */

int b2s_cols_create(int32_t n_in_slots, b2s_cols_t* out);
int b2s_cols_destroy(b2s_cols_t plan);
/* pass a column through (keep != 0) and/or validate it; keep == 0 is a column DropFeatures removed
 * (steps.py:721-729) that a validator placed before the drop still sees. */
int b2s_cols_add_copy(b2s_cols_t plan, int32_t src_slot, int32_t kind, int32_t has_fill, float fill, int32_t keep,
                      int32_t check, double cmin, double cmax, int32_t* out_slot, int32_t* check_counter);
/* MapValues._map_value (steps.py:189-201): first i with lo[i] <= v < hi[i] -> vals[i]; no hit: v passes through
 * and counters[miss_counter] counts the row.  The output slot holds int32 when the source is B2S_COL_I32 and every
 * vals[i] is an int32 integer, so every int32 value that passes through stays exact; otherwise it holds float32, which
 * rounds int32 values beyond 2^24 that pass through (mlrun_b200's ingest refuses frames holding such values). */
int b2s_cols_add_range_map(b2s_cols_t plan, int32_t src_slot, int32_t kind, int32_t has_fill, float fill, const double* lo,
                           const double* hi, const double* vals, int32_t n, int32_t check, double cmin, double cmax,
                           int32_t* out_slot, int32_t* miss_counter, int32_t* check_counter);
/* MapValues exact-match branch (steps.py:200-201): v == keys[i] -> vals[i].  Output as for range maps. */
int b2s_cols_add_value_map(b2s_cols_t plan, int32_t src_slot, int32_t kind, int32_t has_fill, float fill, const double* keys,
                           const double* vals, int32_t n, int32_t check, double cmin, double cmax, int32_t* out_slot,
                           int32_t* miss_counter, int32_t* check_counter);
/* OneHotEncoder._encode (steps.py:453-470): n int32 0/1 output slots, in category order; a value matching no
 * category gives all zeros and is counted (the reference logs a warning). */
int b2s_cols_add_onehot(b2s_cols_t plan, int32_t src_slot, int32_t kind, int32_t has_fill, float fill, const double* cats,
                        int32_t n, int32_t* first_out_slot, int32_t* miss_counter);
/* DateExtractor: src_slot is an 8-byte nanosecond timestamp; the int32 output is -1 for NaT (counted). */
int b2s_cols_add_date_part(b2s_cols_t plan, int32_t src_slot, int32_t part, int32_t* out_slot, int32_t* nat_counter);
int b2s_cols_finalize(b2s_cols_t plan);
int b2s_cols_info(b2s_cols_t plan, int32_t* n_out_slots, int32_t* n_counters);
/* Device-resident run: slot s of the input starts at d_in + s * in_slot_stride (bytes, multiple of 8, >= 4 * n_rows);
 * d_counters (n_counters uint64, zeroed by the caller) accumulates.  Asynchronous on `stream`.  Returns B2S_ERR_INVALID,
 * before any launch, when d_in or d_out is NULL (n_rows > 0) or not 4-byte aligned, or not 8-byte aligned while the plan
 * reads (d_in) or writes (d_out) an 8-byte column, or when d_counters is not 8-byte aligned.  Bases and strides that are
 * not multiples of 16 bytes are legal; such runs take the kernel's 4- and 8-byte access paths. */
int b2s_cols_run_device(b2s_cols_t plan, const void* d_in, int64_t in_slot_stride, int64_t n_rows, void* d_out,
                        int64_t out_slot_stride, uint64_t* d_counters, void* stream);
/* Host run: one pointer per input slot the plan reads (an 8-byte column: pointer at its first slot), one per output
 * slot (NULL at the second slot of an 8-byte column): H2D per column -> kernel -> D2H per column. */
int b2s_cols_run_host(b2s_cols_t plan, const void* const* h_in_slots, int64_t n_rows, void* const* h_out_slots,
                      uint64_t* counters, b2s_stats* stats);
/* n_iters back-to-back device runs over rotating inputs, CUDA-event timed (bench.py) */
int b2s_cols_time_device(b2s_cols_t plan, const void* const* d_in, int32_t n_bufs, int64_t in_slot_stride, int64_t n_rows,
                         void* d_out, int64_t out_slot_stride, uint64_t* d_counters, int32_t n_iters, float* total_ms);

/* ---- body codec (host code): the step on either side of the path for HTTP / stream triggers ------------
 * GraphServer.run json-decodes the request body (serving/server.py:262-277) and _process_response json.dumps
 * the result (:298-308).  b2s_json_parse_inputs finds the top-level "inputs" member of a V2 body and converts
 * its numbers straight into float32 rows (row-major; a flat list is one scalar per event): the same values as
 * np.asarray(json.loads(body)["inputs"], dtype=float32) (null counts as NaN).  [value_begin, value_end) is the
 * member's text, so the caller can decode the small remainder of the body (id, model, operation) as usual.
 * B2S_ERR_UNSUPPORTED: not such a body (strings / dicts / ragged rows) -- the caller falls back to json.loads. */
int b2s_json_parse_inputs(const char* body, int64_t len, float* out, int64_t out_cap, int64_t* n_rows, int64_t* n_cols,
                          int64_t* value_begin, int64_t* value_end);
/* text of a result matrix exactly as json.dumps prints it: float32 values widened to double and printed with
 * Python's repr (vals = float32*), or int32 labels (is_int); flat != 0 prints [v0, v1, ...] for n_cols == 1. */
int b2s_json_format_outputs(const void* vals, int32_t is_int, int64_t n_rows, int64_t n_cols, int32_t flat, char* out,
                            int64_t out_cap, int64_t* out_len);

/* ---- online feature table: real-time enrichment on the device -----------------------------------------
 * EnrichmentModelRouter / EnrichmentVotingEnsemble.preprocess (serving/routers.py:1189-1196, 1335-1342) turn entity
 * keys into feature vectors with OnlineVectorService.get (feature_store/feature_vector.py:975-1067): one online-store
 * read per key, then None / NaN / Inf -> the impute policy's value (:1046-1052).  A b2s_table keeps the online table
 * in HBM (64-bit keys -> rows of n_features float32) and resolves a batch of keys in one launch, writing the rows in
 * the layout b2s_run_device reads.  impute[c] = NaN keeps column c as stored; rows of unknown keys are NaN (then
 * imputed) and reported in found[] (the reference returns None for them). */
typedef struct b2s_table_s* b2s_table_t;
int b2s_table_create(const int64_t* keys, int64_t n_keys, const float* values, int32_t n_features, const float* impute,
                     b2s_table_t* out);
int b2s_table_destroy(b2s_table_t table);
int b2s_table_info(b2s_table_t table, int64_t* n_keys, int32_t* n_features, int64_t* capacity);
/* Device keys -> device rows.  row_stride_bytes >= 4 * n_features and a multiple of 4.  B2S_ERR_INVALID, before any
 * launch, when d_keys is NULL (n > 0) or not 8-byte aligned, or d_rows / d_found is not 4-byte aligned.  Rows are
 * stored 16 bytes at a time only when n_features, row_stride_bytes and d_rows all allow it (4-byte words otherwise). */
int b2s_table_lookup_device(b2s_table_t table, const int64_t* d_keys, int64_t n, float* d_rows, int64_t row_stride_bytes,
                            int32_t* d_found, void* stream);
int b2s_table_lookup_host(b2s_table_t table, const int64_t* keys, int64_t n, float* rows, int32_t* found, b2s_stats* stats);
/* Enrichment + predict for a batch of HOST keys in one call (EnrichmentVotingEnsemble.do_event over a batch: preprocess
 * :1335-1342, then the ensemble): keys -> H2D -> gather -> the scoring plan -> D2H of the plan's outputs and status words,
 * nothing else crosses PCIe (one fused launch when b2s_table_enrich_device covers the plan).  row_status (may be NULL) carries the plan's B2S_ROW_* bits plus B2S_ROW_UNKNOWN_KEY.
 * Pinned caller buffers are used directly; pageable ones are staged through the table's pinned block. */
/* The same for device-resident keys, as ONE launch: the scoring kernel's tile loader finds each key in the table and
 * fetches the row from there (one TMA bulk copy per row), so the gathered rows never travel to HBM and back; the table's
 * impute policy folds into the kernel's Imputer operands.  B2S_ERR_UNSUPPORTED for plans the loader does not cover (tree
 * ensembles, MapValues, one-hot sources under an impute policy): use b2s_table_lookup_device + b2s_run_device then.
 * Both enrichment calls refuse a plan with merge targets or an attached communicator (B2S_ERR_UNSUPPORTED, before anything
 * is enqueued and without a step of the communicator): its kernels would store the votes there, not into `out`.
 * B2S_ERR_INVALID, before any launch, when d_keys is not 8-byte aligned or d_out / d_status is not 4-byte aligned. */
int b2s_table_enrich_device(b2s_table_t table, b2s_plan_t plan, const int64_t* d_keys, int64_t n, void* d_out,
                            int32_t* d_status, void* stream);
int b2s_table_enrich_host(b2s_table_t table, b2s_plan_t plan, const int64_t* keys, int64_t n, void* out, int64_t out_bytes,
                          int32_t* row_status, b2s_stats* stats);
int b2s_table_time_device(b2s_table_t table, const int64_t* const* d_keys, int32_t n_bufs, int64_t n, float* d_rows,
                          int64_t row_stride_bytes, int32_t* d_found, int32_t n_iters, float* total_ms);
/* 64-bit FNV-1a of each string of a packed buffer (string i = bytes[offsets[i] .. offsets[i+1])): the key of a
 * string-valued entity.  Host code. */
int b2s_hash_strings(const char* bytes, const int64_t* offsets, int64_t n, int64_t* keys_out);
/* The online table built from columns in memory of the library's device; nothing but the counters and the key of a
 * duplicate crosses to the host.  b2s_table_create_device builds what b2s_table_create builds from the same keys and the
 * same values as float32 (the same capacity, the NaN row, the padded impute vector), so every lookup and enrichment call
 * serves it alike; slot positions may differ, since keys are inserted concurrently.  Feature column c is n_keys values of
 * cols[c] (FLOAT 4 / 8 bytes, INT and UINT 1 / 2 / 4 / 8, BOOL 1), converted as numpy's astype(float32) converts them:
 * round to nearest even, overflow to +-inf, bool to 0 / 1.  Three launches: pack the rows, insert the keys (atomicCAS on
 * the slot's row word), check for duplicates.  A repeated key is B2S_ERR_INVALID with b2s_table_create's message (the
 * key, the first row that repeats an earlier key, and that row).  B2S_ERR_INVALID before any launch for n_keys outside
 * 1 .. 2^31 - 1, a bad kind or width, or keys / columns that are null, misaligned or not on the library's device. */
enum { B2S_TCOL_FLOAT = 0, B2S_TCOL_INT = 1, B2S_TCOL_UINT = 2, B2S_TCOL_BOOL = 3 };
typedef struct b2s_table_col {
  const void* src;
  int32_t bytes;
  int32_t kind; /* B2S_TCOL_* */
} b2s_table_col;
int b2s_table_create_device(const int64_t* d_keys, int64_t n_keys, const b2s_table_col* cols, int32_t n_features,
                            const float* impute, b2s_table_t* out);
/* Feature statistics of n rows of such columns (as float32), over the finite values: stats_out (host, [5][n_features]
 * float32) gets mean, min, max, std (ddof 1) and count, accumulated in float64 and rounded to float32; NaN where a column
 * has no finite value (std: fewer than two).  Three launches; returns when stats_out is filled. */
int b2s_table_stats_device(const b2s_table_col* cols, int32_t n_features, int64_t n, float* stats_out, void* stream);
/* The keys of the rows whose label is truthy (not NaN and not zero), compacted on the device and copied to keys_out
 * (host, room for n) in no particular order; *n_out gets their number.  One launch; returns when they are there. */
int b2s_table_label_keys_device(const int64_t* d_keys, int64_t n, const b2s_table_col* label, int64_t* keys_out, int64_t* n_out,
                                void* stream);
/* status[i] |= B2S_ROW_UNKNOWN_KEY where found[i] is 0: b2s_table_lookup_device + b2s_run_device + this give the status
 * words b2s_table_enrich_device gives.  One launch, asynchronous. */
int b2s_table_mark_unknown_device(const int32_t* d_found, int32_t* d_status, int64_t n, void* stream);

/* Scoring rows held as device columns (a device ingest's result, a mapping of CUDA columns): n_rows rows whose input column
 * c is cols[c] (n_cols must be the plan's n_in; kinds and widths as for b2s_table_create_device, each value converted as
 * numpy's astype(float32) converts it) -> d_out (n_rows x out_cols words) and d_status (may be NULL), as b2s_run_device
 * gives them for the same rows as a contiguous float32 matrix.  The columns are packed into row-major float32 rows at a
 * stride of 4 * n_in bytes in library scratch, then scored by the plan's own launches, so the plan serves them with the
 * kernel it picks for a contiguous host matrix of that width (b2s_plan_last_kernel).  The work runs in ranges of at most
 * 2^20 rows that reuse one scratch buffer of min(n_rows, 2^20) * 4 * n_in bytes, freed on every return; range k's outputs
 * go to d_out + k * 2^20 * out_cols words.  Asynchronous on `stream` (NULL = the library's stream).  stats (may be NULL)
 * gets rows and kernels: per range, 1 pack launch plus the plan's launches; n_rows = 0 launches nothing.
 * B2S_ERR_INVALID, before any launch, for n_cols other than n_in, a bad kind or width, a column that is null, not aligned
 * to its width or not on the library's device, d_out / d_status not 4-byte aligned, a plan that is not finalized and
 * n_rows < 0.  B2S_ERR_UNSUPPORTED, before anything is enqueued, for a plan with merge targets or an attached communicator
 * (each range would be a step of its own). */
int b2s_run_columns_device(b2s_plan_t plan, const b2s_table_col* cols, int32_t n_cols, int64_t n_rows, void* d_out,
                           int32_t* d_status, b2s_stats* stats, void* stream);

/* ---- point-in-time training sets: as-of joins of entity rows onto feature-set indexes ---------------------------
 * get_offline_features on the local engine (feature_store/retrieval/base.py:412-468, local_merger.py:29-81) merges
 * each feature set of a vector onto the entity frame with pandas.merge_asof: equal keys, the set's last row whose
 * timestamp is <= the entity row's (backward, exact matches allowed, no tolerance), NaN / NaT where there is none.
 * A b2s_pit index holds one feature set in HBM: its rows sorted by (64-bit key, int64 nanosecond timestamp), equal
 * pairs in input order, the feature columns as rows of 4-byte words, and each key's run in an open-addressing slot
 * array.  Built once from columns (each 4 or 8 bytes wide; column c takes words [sum of earlier widths / 4, ...)):
 * host arrays for b2s_pit_index_create, which uploads them, or memory of the library's device for
 * b2s_pit_index_create_device, which reads them where they are.  Both refuse n_rows <= 0 (and >= 2^31), more than 64
 * columns and widths other than 4 / 8 with B2S_ERR_INVALID; _device also refuses, before any launch, keys, timestamps
 * (8 bytes) or columns (their width) that are misaligned or not on the library's device.  The build makes 53 launches. */
typedef struct b2s_pit_s* b2s_pit_t;
int b2s_pit_index_create(const int64_t* keys, const int64_t* ts_ns, int64_t n_rows, const void* const* cols,
                         const int32_t* col_bytes, int32_t n_cols, b2s_pit_t* out);
int b2s_pit_index_create_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n_rows, const void* const* d_cols,
                                const int32_t* col_bytes, int32_t n_cols, b2s_pit_t* out);
int b2s_pit_index_destroy(b2s_pit_t index);
/* longest_run 1: every key has one row, so the index can also serve exact-key joins */
int b2s_pit_index_info(b2s_pit_t index, int64_t* n_rows, int64_t* n_keys, int64_t* longest_run, int32_t* row_words,
                       int64_t* capacity);
typedef struct b2s_pit_out {
  int32_t src_word;   /* first word of the column in the index's rows */
  int32_t bytes;      /* 4 or 8 */
  uint64_t miss;      /* bits stored for an entity row without a match (a NaN, NaT or 0) */
  void* out;          /* [n] elements of `bytes` bytes, in sorted order */
} b2s_pit_out;
typedef struct b2s_pit_set {
  b2s_pit_t index;
  const int64_t* keys;   /* [n] the entity rows' keys, input order */
  int32_t asof;          /* 1: as-of join on the entity timestamps; 0: exact key (the index must have one row per key) */
  int32_t n_out;
  const b2s_pit_out* outs;  /* host array of n_out descriptors */
  int64_t* ts_out;       /* [n] the matched row's timestamp, INT64_MIN (NaT) on a miss; may be NULL */
  uint8_t* found;        /* [n] 1 / 0; may be NULL */
} b2s_pit_set;
typedef struct b2s_pit_col {
  const void* src;       /* [n] entity column, input order */
  void* dst;             /* [n] the same column in sorted order */
  int32_t bytes;         /* 1, 2, 4 or 8 */
} b2s_pit_col;
/* Join n entity rows onto n_sets indexes.  With ts (int64 nanoseconds) the rows are ordered by timestamp, ties in input
 * order (a stable radix sort); without it they keep input order (then no set may be as-of).  Every output, the entity
 * columns in `cols` and order[q] (the input row at sorted position q; may be NULL) are written in that order; miss[s]
 * counts the rows without a match in set s.  _device: every array is device memory, miss accumulates (zero it first),
 * asynchronous on `stream`.  _host: host arrays; the join runs in row ranges whose results are copied back while the next
 * range is joined; miss is written; stats->kernels counts every launch: the sort's 24 (with ts) plus, per range, one join
 * launch per set, with the entity columns 64 to a launch (max(1, n_sets, ceil(n_cols / 64))).  B2S_ERR_INVALID before any launch for a misaligned or null array, an output word
 * outside the index's rows, or an exact-key join on an index with more than one row per key. */
int b2s_pit_join_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                        int32_t n_cols, int64_t* d_order, uint64_t* d_miss, void* stream);
int b2s_pit_join_host(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                      int32_t n_cols, int64_t* order, uint64_t* miss, b2s_stats* stats);
/* Training sets: the join above, then only the rows the reference's merged frame keeps after
 * dropna(subset=[label]) (feature_store/retrieval/base.py:343-346): rows every exact-key (inner) join matched and, with a
 * label, rows whose label is present.  The label is output `out` of set `set` (then the set must have matched) or, with
 * set -1, entity column `out`; B2S_PIT_LABEL_NAN also drops NaN values (4- or 8-byte floats), B2S_PIT_LABEL_NAT drops
 * INT64_MIN (8 bytes).  The kept rows of every output, found flag, ts_out, entity column and order are written first, in
 * sorted order, and *kept counts them; the arrays still need room for n rows.  miss[s] counts the rows set s misses among
 * those every earlier exact-key set matched (the frame at the set's place in the merge, before the label filter).  Every
 * set needs its found array.  _device: device arrays, asynchronous on `stream`; miss and *d_kept are written.  _host:
 * host arrays; only the kept rows are copied back, in ranges of 1 Mi rows; phase_ms (may be NULL) gets the sort, join and
 * compaction times; stats->kernels counts every launch: the sort's 24 (with ts), the join's max(1, n_sets,
 * ceil(n_cols / 64)), 2 to find the kept rows and ceil(arrays / 64) to compact them, where arrays counts each set's outputs,
 * ts_out and found, the entity columns and order.  B2S_ERR_INVALID before any launch for what b2s_pit_join_* refuses,
 * more than 64 sets, a set without found flags, a null miss / kept counter, or a label that names no output or does not fit
 * its kind. */
enum { B2S_PIT_LABEL_FOUND = 0, B2S_PIT_LABEL_NAN = 1, B2S_PIT_LABEL_NAT = 2 };
typedef struct b2s_pit_label {
  int32_t set;   /* index of the label's set, or -1: an entity column */
  int32_t out;   /* output of that set, or entity column */
  int32_t kind;  /* B2S_PIT_LABEL_* */
} b2s_pit_label;
int b2s_pit_train_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                         int32_t n_cols, const b2s_pit_label* label, int64_t* d_order, uint64_t* d_miss, int64_t* d_kept,
                         void* stream);
int b2s_pit_train_host(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                       int32_t n_cols, const b2s_pit_label* label, int64_t* order, uint64_t* miss, int64_t* kept,
                       float* phase_ms, b2s_stats* stats);

/* Device arrays the library allocated for its caller (cudaMalloc on the library's device), reference counted: the memory
 * is freed when the last reference goes.  b2s_darray_release drops one.  b2s_darray_dlpack returns a DLPack
 * DLManagedTensor (the unversioned ABI: kDLCUDA, compact row-major, byte_offset 0) that holds one more; its deleter is a
 * function of this library that drops it and frees the struct.  b2s_dlpack_delete calls that deleter, for a producer
 * whose capsule was never consumed.  b2s_darray_live counts the arrays not yet freed. */
typedef struct b2s_darray_s* b2s_darray_t;
int b2s_darray_info(b2s_darray_t a, void** ptr, int64_t* bytes);
int b2s_darray_release(b2s_darray_t a);
void* b2s_darray_dlpack(b2s_darray_t a, int32_t ndim, const int64_t* shape, int32_t code, int32_t bits);
int b2s_dlpack_delete(void* managed);
int64_t b2s_darray_live(void);
/* b2s_darray_alloc: a new array of `bytes` (zero != 0: zeroed on the library stream).  b2s_darray_view: an array over
 * bytes [offset, offset + bytes) of `base`, which it keeps alive; releasing the view drops that reference.  Both refuse a
 * null out, negative sizes and (view) a range outside the base or an offset that is not a multiple of 8 with
 * B2S_ERR_INVALID; the view's address is base + offset. */
int b2s_darray_alloc(int64_t bytes, int32_t zero, b2s_darray_t* out);
int b2s_darray_view(b2s_darray_t base, int64_t offset, int64_t bytes, b2s_darray_t* out);

/* Training sets as device tensors: b2s_pit_train_host's join and kept rows, packed into one row-major matrix in HBM
 * instead of copied back.  Matrix column i is feats[i]: output `out` of set `set`, or with set -1 entity column `out`, a
 * source of `bytes` bytes (the output's or column's own width) of kind B2S_PIT_FEAT_*: a FLOAT of 4 or 8 bytes, an INT
 * (signed) or UINT of 1, 2, 4 or 8, a BOOL of any of those (nonzero is 1).  Each value is converted to x_bytes (4: float32,
 * 8: float64) rounding to nearest; a set's value is NaN where the set found no row.  label_vec (may be NULL) is compacted
 * alongside: a FLOAT keeps its width, an INT / UINT becomes int64, a BOOL one byte 0 / 1.  The library allocates
 * out->features [kept][n_feats], out->order [kept] (int64: the entity row of each matrix row) and out->label [kept] (NULL
 * without label_vec) once it knows kept, and the caller releases each with b2s_darray_release; they are ready when the call
 * returns.  Only the host inputs of `sets` and `cols` are read: every output, found flag, ts_out and entity destination
 * lives in library scratch, so their pointers may be NULL.  phase_ms (may be NULL) gets 4 times: the sort, the join, the
 * compaction (keep, scan and pack) and the pack launch alone; stats->kernels counts every launch: the sort's 24 (with ts), the join's max(1, n_sets,
 * ceil(n_cols / 64)), 2 to find the kept rows and 1 pack launch that writes the matrix, order and label.  B2S_ERR_INVALID
 * before any launch for what b2s_pit_train_host refuses, a feature or label_vec that names no output or column, or whose
 * width or kind does not fit, and x_bytes other than 4 or 8; B2S_ERR_CUDA when an allocation fails (*out is then empty). */
enum { B2S_PIT_FEAT_FLOAT = 0, B2S_PIT_FEAT_INT = 1, B2S_PIT_FEAT_UINT = 2, B2S_PIT_FEAT_BOOL = 3 };
typedef struct b2s_pit_feat {
  int32_t set;    /* index of the set, or -1: an entity column */
  int32_t out;    /* output of that set, or entity column */
  int32_t bytes;  /* the source's width */
  int32_t kind;   /* B2S_PIT_FEAT_* */
} b2s_pit_feat;
typedef struct b2s_pit_tensors {
  b2s_darray_t features;  /* [kept][n_feats] float32 or float64, row-major */
  b2s_darray_t label;     /* [kept], or NULL */
  b2s_darray_t order;     /* [kept] int64 */
  int64_t kept;
} b2s_pit_tensors;
int b2s_pit_train_pack(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                       int32_t n_cols, const b2s_pit_label* label, const b2s_pit_feat* feats, int32_t n_feats,
                       const b2s_pit_feat* label_vec, int32_t x_bytes, b2s_pit_tensors* out, float* phase_ms,
                       b2s_stats* stats);
/* b2s_pit_train_pack with ts, each set's keys and each entity column's src in memory of the library's device: nothing is
 * uploaded (stats->h2d_ms is 0), the launches are the same.  Also B2S_ERR_INVALID, before any launch, for such an input
 * (n > 0) that is misaligned or not on the library's device. */
int b2s_pit_train_pack_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                              int32_t n_cols, const b2s_pit_label* label, const b2s_pit_feat* feats, int32_t n_feats,
                              const b2s_pit_feat* label_vec, int32_t x_bytes, b2s_pit_tensors* out, float* phase_ms,
                              b2s_stats* stats);

/* ---- windowed aggregations at feature-set ingest ------------------------------------------------------------------
 * storey.AggregateByKey as FeatureSet.add_aggregation places it in a feature set's graph (feature_store/feature_set.py:
 * 715-851), emitting every event: row i gains, per (operation, window), the aggregate over the rows j <= i (input order)
 * of its 64-bit key whose timestamps lie in row i's window.  Windows are aligned to the epoch (floor division, so that
 * rows before 1970 are right): sliding (period_ns > 0, dividing every window): b(t) = floor(t / period), row j is in
 * when b(t_j) >= b(t_i) - window / period + 1; fixed (period_ns = 0): floor(t_j / window) == floor(t_i / window).  A
 * window's first timestamp is clamped at INT64_MIN where it would leave the int64 range (near 1677, at any period).
 * Sums accumulate in fp64 over the window's rows alone (a range reduce, never a difference of running sums); stdvar is
 * the sample variance from a pairwise (count, mean, M2) combine, NaN for a window of one row; first is the window's
 * earliest row in input order, last the row itself.  Every output is [n] float64 in input order. */
#define B2S_AGG_COUNT 1
#define B2S_AGG_SUM 2
#define B2S_AGG_SQR 4      /* sum of squares */
#define B2S_AGG_MAX 8
#define B2S_AGG_MIN 16
#define B2S_AGG_FIRST 32
#define B2S_AGG_LAST 64
#define B2S_AGG_AVG 128
#define B2S_AGG_STDVAR 256
#define B2S_AGG_STDDEV 512
typedef struct b2s_agg_spec {
  const void* src;           /* [n] source column in input order, 4-byte words */
  int32_t kind;              /* B2S_COL_F32 or B2S_COL_I32 (both widen exactly to fp64) */
  uint32_t ops;              /* B2S_AGG_* bits */
  int64_t period_ns;         /* sliding period; 0: fixed windows */
  int32_t n_windows;         /* 1 .. 16 */
  const int64_t* windows_ns; /* host array [n_windows] */
  double* const* outs;       /* host array [popcount(ops) * n_windows]: ops in bit order, windows inner; each [n] float64 */
} b2s_agg_spec;
/* n rows: keys and int64 nanosecond timestamps in input order; 1 .. 64 aggregations over at most 16 distinct source
 * columns.  counters[3] count what the semantics refuse, for the caller to raise on: [0] rows whose timestamp is below the
 * previous row of their key (late events), [1] NaT (INT64_MIN) rows, [2] NaN source values; the outputs of such a run
 * are unspecified.  _device: every array is device memory, counters accumulate (zero them first), asynchronous on
 * `stream`.  _host: host arrays (pinned ones copy at full speed, pageable ones are staged by the driver), counters are
 * written; stats->h2d_ms is the copy in, kernel_ms the sort plus the aggregation, kernels every launch: the sort's 24,
 * one prep launch, one per level of each column's range structure (levels with more than 32 elements: about
 * log32(n) of them; none for a column whose aggregations are only count / first / last) and one per aggregation.
 * B2S_ERR_INVALID before any launch for a null or misaligned pointer (keys, timestamps, outputs and counters 8 bytes,
 * sources 4), n >= 2^32 (the sort's 32-bit payload), a period that does not divide a window, a window <= 0, an empty or
 * unknown op mask, or a kind other than F32 / I32. */
int b2s_agg_run_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                       uint64_t* d_counters, void* stream);
int b2s_agg_run_host(const int64_t* keys, const int64_t* ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                     uint64_t* counters, b2s_stats* stats);
/* n_iters device runs on the library stream, CUDA-event timed: the sort alone and the whole run (ms summed over the runs) */
int b2s_agg_time_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                        uint64_t* d_counters, int32_t n_iters, float* sort_ms, float* total_ms);

/* ---- feature-set ingest of device-resident columns -----------------------------------------------------------------
 * What the host ingest does around b2s_cols_run_* and b2s_agg_run_* for columns that already live in device memory.
 * b2s_stream: the library stream (NULL before b2s_init), for producers that order their writes before a consumer's
 * stream (DLPack).  b2s_stream_wait: the library stream waits for the work queued so far on `producer` (a CUDA stream;
 * 1 / 2 are the legacy / per-thread default streams).  b2s_pointer_device: the device that holds `p`, -1 for host memory. */
void* b2s_stream(void);
int b2s_stream_wait(void* producer);
int b2s_pointer_device(const void* p, int32_t* device);
/* b2s_cols_convert_device: n_ops elementwise conversions over n rows in ONE launch, asynchronous on `stream` (NULL: the
 * library stream).  COPY4 / COPY8 and the widenings of 1- and 2-byte ints stage columns into the slot block
 * b2s_cols_run_device reads (bool is U8); the others give result columns the host ingest's dtypes: int32 -> float64,
 * float32 -> int32 (numpy's astype: out of range or NaN gives INT32_MIN), a date part (-1 for NaT) -> float64 with NaN,
 * int32 -> bool (one byte, nonzero is 1).  CHECK_F32 writes nothing: d_counters[counter] (zeroed by the caller) counts
 * the int32 values float32 cannot hold exactly.  B2S_ERR_INVALID before any launch for n < 0, n_ops outside
 * 1 .. 65535, an unknown kind, a null (n > 0) or misaligned source or destination (aligned to its element width), or a
 * CHECK_F32 counter outside [0, n_counters) or without d_counters. */
enum {
  B2S_CONV_COPY4 = 0, B2S_CONV_COPY8 = 1, B2S_CONV_I8_I32 = 2, B2S_CONV_U8_I32 = 3, B2S_CONV_I16_I32 = 4, B2S_CONV_U16_I32 = 5,
  B2S_CONV_I32_F64 = 6, B2S_CONV_F32_I32 = 7, B2S_CONV_DATE_F64 = 8, B2S_CONV_I32_BOOL = 9, B2S_CONV_CHECK_F32 = 10
};
typedef struct b2s_convert {
  const void* src;
  void* dst;        /* unused by CHECK_F32 */
  int32_t kind;     /* B2S_CONV_* */
  int32_t counter;  /* CHECK_F32 only */
} b2s_convert;
int b2s_cols_convert_device(const b2s_convert* ops, int32_t n_ops, int64_t n, uint64_t* d_counters, int32_t n_counters,
                            void* stream);
/* b2s_keys_encode_device: 64-bit entity keys as the point-in-time join and the aggregations encode them, in one launch:
 * one int column (1, 2 or 4 bytes signed or unsigned, 8 bytes signed) widened to int64, or two int32 columns as
 * hi << 32 | (lo & 0xFFFFFFFF).  B2S_ERR_INVALID before any launch for other widths, null (n > 0) or misaligned columns,
 * or d_keys not 8-byte aligned. */
typedef struct b2s_key_col {
  const void* src;
  int32_t bytes;
  int32_t is_signed;
} b2s_key_col;
int b2s_keys_encode_device(const b2s_key_col* cols, int32_t n_cols, int64_t n, int64_t* d_keys, void* stream);
/* b2s_keys_hash_decimal_device: the online table's key of a composite entity, in one launch: FNV-1a (b2s_hash_strings) of
 * the decimal text of each row's values joined by '.', as Python's ".".join(str(v) for v in row), without materialising
 * the text.  1 .. 16 signed int columns of 1, 2, 4 or 8 bytes.  B2S_ERR_INVALID before any launch for other columns, or
 * columns / d_keys that are null (n > 0), misaligned or not on the library's device. */
int b2s_keys_hash_decimal_device(const b2s_key_col* cols, int32_t n_cols, int64_t n, int64_t* d_keys, void* stream);
/* b2s_ts_profile_device: one launch over n int64 nanosecond timestamps in memory of the library's device; counts (host,
 * 4) gets the NaT (INT64_MIN) values and the other values that are not whole multiples of 10^3, 10^6 and 10^9, in one
 * small copy: the call returns when they are there.  n = 0: zeros, no launch.  B2S_ERR_INVALID before any launch for
 * n < 0, a null counts, or d_ts null (n > 0), misaligned or not on the library's device. */
int b2s_ts_profile_device(const int64_t* d_ts, int64_t n, int64_t* counts, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SERVE_H */
