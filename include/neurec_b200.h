/*
 * neurec_b200 -- C ABI of the H100-native (sm_90a) hot path of NeuRec.
 *
 * This header is the drop-in boundary: every entry point replaces one interface of the
 * reference (cited as path:line relative to the reference root).  Signatures use plain
 * pointers and sizes only; no torch / numpy / C++ types.
 *
 * Conventions
 *   - All pointers are DEVICE pointers unless the function name ends in `_host`
 *     (then every buffer is a host buffer and the call does its own staged H2D/D2H).
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Device
 *     entry points are asynchronous on that stream and never free caller memory.
 *   - ids are int32, CSR row pointers are int64, CSR rows are ascending and duplicate-free
 *     (what util/tool.py:56-65 csr_to_user_dict produces).
 *   - Return value: 0 on success, negative NRC_E_* otherwise; nrc_last_error() returns a
 *     thread-local message.  Error codes mirror the Python exceptions the reference raises
 *     at the same place (the Python wrapper re-raises them with the reference's message).
 */
#ifndef NEUREC_B200_H
#define NEUREC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NRC_OK 0
#define NRC_E_VALUE (-1)    /* reference raises ValueError */
#define NRC_E_TYPE (-2)     /* reference raises TypeError */
#define NRC_E_NOTIMPL (-3)  /* reference raises NotImplementedError */
#define NRC_E_CUDA (-4)     /* CUDA runtime failure */
#define NRC_E_LIMIT (-5)    /* argument outside this build's supported range */

/* metric ids, evaluator/backend/cpp/include/metric.h:111-117 (metric_dict) */
#define NRC_METRIC_PRECISION 1
#define NRC_METRIC_RECALL 2
#define NRC_METRIC_MAP 3
#define NRC_METRIC_NDCG 4
#define NRC_METRIC_MRR 5

/* pairwise losses, util/learner.py:18-29; pointwise losses, util/learner.py:31-41 */
#define NRC_LOSS_BPR 0
#define NRC_LOSS_HINGE 1
#define NRC_LOSS_SQUARE 2
#define NRC_LOSS_CROSS_ENTROPY 3

/* optimizers, util/learner.py:2-15 (TensorFlow 1.12 semantics, see DESIGN.md) */
#define NRC_OPT_GD 0
#define NRC_OPT_ADAM 1
#define NRC_OPT_ADAGRAD 2
#define NRC_OPT_RMSPROP 3
#define NRC_OPT_MOMENTUM 4

/* ItemKNN similarity transforms, model/general_recommender/ItemKNN.py:146-181, 476-500 (see nrc_itemknn_similarity) */
#define NRC_ITEMKNN_NORM 0       /* cosine, adjusted, pearson, asymmetric */
#define NRC_ITEMKNN_TANIMOTO 1   /* jaccard, tanimoto */
#define NRC_ITEMKNN_DICE 2
#define NRC_ITEMKNN_TVERSKY 3
#define NRC_ITEMKNN_EUCLIDEAN 4

int nrc_version(void);
const char* nrc_last_error(void);

/* Host <-> device staging of ONE training batch, the analogue of feed_dict / fetches around a
 * sess.run (MF.py:97-101): copy the three host id / label arrays (batch elements of 4 bytes
 * each; pinned memory recommended) to staging[0:batch], [batch:2*batch], [2*batch:3*batch]
 * asynchronously on `stream`; nrc_fetch_host copies `count` floats back and synchronises the
 * stream so the values are valid on return. */
int nrc_stage_batch_host(const void* a_host, const void* b_host, const void* c_host,
                         int64_t batch, void* staging, void* stream);
int nrc_fetch_host(const float* src_dev, float* dst_host, int64_t count, void* stream);

/* Captured training steps (replace the per-batch `sess.run((loss, optimizer), feed_dict)` of
 * MF.py:97-108, NeuMF.py:131-147, MLP.py:104-120, LightGCN.py:170-178).  The reference pays one
 * `sess.run` per batch; the lowest-overhead
 * analogue here is ONE cudaGraphLaunch per batch.  Between nrc_graph_capture_begin and
 * nrc_graph_capture_end every nrc_* device call issued on `stream` is recorded instead of run:
 *   nrc_graph_stage_async   H2D of the pinned staging block (3*batch ids/labels + 1 float lr_t)
 *   nrc_opt_set_lr_source   make the optimizer read lr / Adam's lr_t from that device float
 *   nrc_*_train_epoch       with n = batch (one step)            [adam and gd only: the touched
 *                            stamps are frozen in a graph; TF's adam/gd do not depend on them]
 *   nrc_graph_fetch_async   D2H of the step's loss into pinned memory
 * nrc_graph_step then copies one batch of HOST arrays into the pinned block, stores lr_t after
 * them, launches the graph and synchronises the stream (loss valid on return). */
typedef struct nrc_step_graph nrc_step_graph;
int nrc_graph_capture_begin(void* stream);
int nrc_graph_capture_end(void* stream, nrc_step_graph** out);
int nrc_graph_stage_async(const void* pinned_host, void* staging_dev, int64_t nbytes, void* stream);
int nrc_graph_fetch_async(const float* src_dev, float* pinned_host, int64_t count, void* stream);
int nrc_graph_step(nrc_step_graph* g, const void* a_host, const void* b_host, const void* c_host,
                   int64_t batch, float lr_t, void* pinned_stage, void* stream);
/* to_stream waits for everything issued so far on from_stream.  During a capture this forks /
 * joins the graph: the second stream joins the capture. */
int nrc_graph_depend(void* from_stream, void* to_stream);
/* A run of n_steps steps over consecutive batches of the host arrays with a RING of `ring` pinned
 * blocks (pinned_stage[r], loss slot loss_pinned[r]).  `burst` (may be NULL) is ONE captured graph
 * holding `ring` consecutive steps, captured with nrc_graph_depend so that the H2D of step s+1
 * overlaps the kernels of step s: the host stages `ring` batches, launches it, waits, reads the
 * `ring` losses.  Steps that do not fill a burst (all of them when burst is NULL) use the per-slot
 * single-step graphs `graphs[r]`, launched back to back with one wait per ring wrap.  Every step
 * performs its own H2D and its own loss D2H.  lr_t[s] = learning rate (Adam's lr_t) of step s.
 * *loss_sum = sum of every fetched loss value. */
int nrc_graph_run_steps(nrc_step_graph* burst, nrc_step_graph* const* graphs, int32_t ring,
                        const void* a_host, const void* b_host, const void* c_host, int64_t batch,
                        const float* lr_t, int64_t n_steps, void* const* pinned_stage,
                        const float* const* loss_pinned, int32_t loss_count, double* loss_sum,
                        void* stream);
int nrc_graph_destroy(nrc_step_graph* g);
int nrc_opt_set_lr_source(const float* lr_dev);

/* ======================================================================================
 * Evaluator
 * ==================================================================================== */

/* cpp_evaluate_matrix, evaluator/backend/cpp/include/evaluate.h:53-72, as bound by
 * CPPEvaluator.eval_score_matrix, evaluator/backend/cpp/cpp_evaluator.pyx:28-42.
 *   scores      f32 [num_users, rating_len] row-major (train items already -inf)
 *   test_indptr i64 [num_users+1], test_indices i32: truth set of batch row b
 *   metric      i32 [metric_num] HOST array of ids in 1..5 (it is a std::vector by value
 *               in the reference); results f32 [num_users, metric_num*top_k], metric-major.
 *   ranks       optional i32 [num_users, top_k]: the ranking the metrics were computed on.
 * Selection reproduces std::partial_sort_copy over min(2*top_k, rating_len) slots
 * (evaluate.h:38-42) including its tie order.  `thread_num` of the reference has no
 * meaning on the GPU and is not part of this ABI. */
int nrc_eval_score_matrix(const float* scores, int32_t rating_len, int32_t num_users,
                          const int64_t* test_indptr, const int32_t* test_indices,
                          const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                          float* results, int32_t* ranks, void* stream);

/* Same, every buffer on the HOST (pageable or pinned); rows are streamed to the device in
 * double-buffered chunks.  This is the call a `cdef extern` in cpp_evaluator.pyx binds. */
int nrc_eval_score_matrix_host(const float* scores, int32_t rating_len, int32_t num_users,
                               const int64_t* test_indptr, const int32_t* test_indices,
                               const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                               float* results, int32_t* ranks);

/* arg_top_k_2d, util/cython/include/arg_topk.h:27-45 (arg_topk.pyx:16-35): exactly top_k
 * heap slots (no 2x margin), same tie order. */
int nrc_arg_topk(const float* scores, int32_t rating_len, int32_t rows_num, int32_t top_k,
                 int32_t* results, void* stream);
int nrc_arg_topk_host(const float* scores, int32_t rating_len, int32_t rows_num, int32_t top_k,
                      int32_t* results);

/* Fused UniEvaluator batch body, evaluator/backend/cpp/uni_evaluator.py:132-146 with
 * model.predict = U[users] . V^T (MF.py:120-122, LightGCN.py:187-189): score all items with
 * an fp32 FMA chain over k, mask the user's train items to -inf, select, compute metrics.
 * The [B, num_items] score matrix is never materialised.
 *   user_table f32 [*, dim], item_table f32 [num_items, dim]
 *   users i32 [num_eval_users]; train/test CSR are indexed by USER ID.
 *   results f32 [num_eval_users, metric_num*top_k]; ranks optional.
 * Envelope: the heap-replay kernel keeps 64 user rows, a 64-item tile and 64 heaps in shared
 * memory, so with D4 = dim rounded up to a multiple of 4 and L = min(2*top_k, num_items) a shape
 * is accepted when 256 * (2*D4 + 4 + 2*L + 3*top_k) <= 227 * 1024, i.e. 2*D4 + 2*L + 3*top_k <= 904
 * (dim <= 448; top_k <= 128 at dim 1, 110 at dim 64, 92 at dim 128 when num_items >= 2*top_k).
 * Other shapes return NRC_E_LIMIT and leave the outputs untouched. */
int nrc_eval_mf(const float* user_table, const float* item_table, int32_t dim,
                int32_t num_items, const int32_t* users, int32_t num_eval_users,
                const int64_t* train_indptr, const int32_t* train_indices,
                const int64_t* test_indptr, const int32_t* test_indices,
                const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                float* results, int32_t* ranks, void* stream);

/* nrc_eval_mf normally runs a tie-free fast pass (valid whenever the K+1 largest scores of a
 * user are pairwise distinct) and re-does the remaining users with the exact libstdc++ heap
 * replay; both give the reference's ranking bit for bit.  on != 0 forces the heap replay for
 * every user (test / debugging hook). */
int nrc_eval_force_exact(int32_t on);
/* How many users of the last nrc_eval_mf / nrc_eval_mf_tc call needed a heap replay (host int32 out). */
int nrc_eval_last_undecided(int32_t* count_host);
/* Test hook of the evaluator (it reports and changes nothing; every route is chosen by the shape):
 * HOST bookkeeping written when a call launches, out i32[3], -1 = no such launch yet.  It is one
 * record per process, not per thread: with several host threads it shows whichever launched last.
 *   [0] selection form of the last nrc_eval_mf: 0 heap replay for every user (top_k >= 32 or
 *       nrc_eval_force_exact), 1 fast pass with 2 users per warp (<= 16 users per SM), 2 fast pass
 *       on 128-item tiles, 3 fast pass on 64-item tiles (dim too large for the 128-item tile);
 *       every fast form is followed by the heap replay of the users it could not decide;
 *   [1] 1 when the last eval_rows_kernel launch (nrc_eval_score_matrix[_host], nrc_arg_topk[_host])
 *       ran its fast pass, 0 when it replayed the heap for every row;
 *   [2] that launch's warps per CTA (8, fewer when 2*L + 3*top_k words per warp exceed 12 KB). */
int nrc_eval_last_routes(int32_t* out);

/* nrc_eval_mf for large catalogues (BASELINE config 4) with the score step on the Hopper tensor
 * cores: bf16 copies of the tables, wgmma (64 users x 128 items x k16 per warpgroup, 64 items at
 * dim 192) with fp32 accumulators, a per-user running threshold (the 2*top_k-th best score so far,
 * the reference's heap root, evaluate.h:38-41) with a rigorous error margin to keep every item
 * that can enter the reference's heap, then exact fp32 re-scoring of the candidates, the same
 * tie-aware selection as nrc_eval_mf and -- for users with ties -- the libstdc++ heap replayed
 * over the first 2*top_k items + the candidates.  Results are bit-identical to nrc_eval_mf.
 * dim 64 or 128 with top_k <= 31, or dim 192 with top_k <= 16; cand_cap = entries per candidate
 * list (0 = 1024; users whose list overflows fall back to the full-catalogue heap-replay kernel).
 * Synchronises `stream` once (to size the tie-replay pass): not capturable into a CUDA graph. */
int nrc_eval_mf_tc(const float* user_table, const float* item_table, int32_t dim,
                   int32_t num_items, const int32_t* users, int32_t num_eval_users,
                   const int64_t* train_indptr, const int32_t* train_indices,
                   const int64_t* test_indptr, const int32_t* test_indices,
                   const int32_t* metric_host, int32_t metric_num, int32_t top_k, int32_t cand_cap,
                   float* results, int32_t* ranks, void* stream);
/* nrc_eval_mf_tc keeps a bf16 copy of the item table (and its largest row norm).  By default it is
 * rebuilt on every call; a caller that evaluates ONE fixed model in several calls (user batches) sets
 * a non-zero version first: the copy is then reused while (item_table pointer, shape, version) stay
 * the same.  Change the version (or pass 0) whenever the table's contents change. */
int nrc_eval_tc_items_version(uint64_t version);

/* Epilogue layout of the tensor-core candidate kernel (main pass): 8 warps (one thread per user and
 * item tile) or 16 warps (two threads per user, one per half tile, each with its own threshold and
 * candidate list).  Results are identical; a tuning knob (env NRC_TC_CH=2 selects 16 as well). */
int nrc_eval_tc_epilogue_warps(int32_t warps);

/* Measurement hook: CUDA-event duration (ms, on the launching stream) and algorithmic flops
 * (2 * users * items * dim) of the last candidate-kernel launch made by nrc_eval_mf_tc;
 * waits for that launch.  bench.py derives the tensor-pipe roofline fraction from it. */
int nrc_eval_tc_last_launch(float* kernel_ms, double* flops);

/* Self-test of the wgmma building block used by the tensor-core candidate pass:
 * out f32 [128, 256] = a bf16 [128, k] . b bf16 [256, k]^T (k multiple of 16, <= 256);
 * swizzle = 0: no-swizzle K-major operand layout, 1: SWIZZLE_128B (k % 64 == 0).
 * nrc_tc_gemm_debug issues wgmma m64n128k16 (the instruction of dim <= 128); nrc_tc_gemm_debug_ntile
 * takes the N tile: n_tile = 128 (m64n128k16) or 64 (m64n64k16, the instruction of dim 192). */
int nrc_tc_gemm_debug(const void* a_bf16, const void* b_bf16, int32_t k, int32_t swizzle, float* out,
                      void* stream);
int nrc_tc_gemm_debug_ntile(const void* a_bf16, const void* b_bf16, int32_t k, int32_t swizzle, int32_t n_tile,
                            float* out, void* stream);

/* Test hooks of the tensor-core path (all off by default; they change no result).
 * nrc_eval_tc_force_segments: g = 0 keeps the occupancy heuristic for the number of item segments
 *   (lists per user) of both candidate passes; g >= 1 uses min(g, item tiles) segments.
 * nrc_eval_tc_debug_candidates: runs ONE candidate pass (pass 0: main, 1: tie replay) exactly as
 *   nrc_eval_mf_tc would -- bf16 tables, margin, forced or heuristic segments, 16-warp epilogue
 *   (nrc_eval_tc_epilogue_warps) in pass 0 only -- with threshold rank lq and cap entries per list,
 *   and copies out cand i32 / cand_val f32 (approximate score) [n, nslots, cap], cnt i32 [n, nslots]
 *   (> cap: the list overflowed) and margin f32 [n] into device buffers sized for max_slots lists per
 *   row.  *nslots and *seg_items (items per segment) are HOST outputs; NRC_E_LIMIT when the pass uses
 *   more than max_slots lists.
 * nrc_eval_tc_last_fallbacks: users of the last nrc_eval_mf_tc call re-ranked by the candidate-list
 *   heap replay (ties) and by the full-catalogue heap replay (an overflowed list); HOST outputs,
 *   synchronises the device. */
int nrc_eval_tc_force_segments(int32_t g);
int nrc_eval_tc_debug_candidates(int32_t pass, const float* user_table, const float* item_table, int32_t dim,
                                 int32_t num_items, const int32_t* users, int32_t n, const int64_t* train_indptr,
                                 const int32_t* train_indices, int32_t lq, int32_t cap, int32_t max_slots,
                                 int32_t* cand, float* cand_val, int32_t* cnt, float* margin, int32_t* nslots,
                                 int32_t* seg_items, void* stream);
int nrc_eval_tc_last_fallbacks(int32_t* replayed, int32_t* full_replays);

/* Test hook of the NCF family (it reports and changes nothing; every route is chosen by the shape).
 * nrc_ncf_last_routes: the code paths of the most recent nrc_ncf_grad / nrc_ncf_train_epoch /
 *   nrc_ncf_epoch_fused / nrc_ncf_scores launch, HOST bookkeeping written when the call launches (a call
 *   that returns before launching leaves it as it was).  out i32[7]; -1 = not decided by that call:
 *   [0] per-batch sample kernel: 1 the default-tower kernel (layers [64,32,16]), 0 the generic one;
 *   [1] batch slices of the per-batch weight-gradient kernel (16 from 64 samples, else 1; 0 without layers);
 *   [2] epoch kernel dense gradient: 1 4x4 blocks (every width a multiple of 4), 0 lane quartets;
 *   [3] epoch kernel embedding tables: 1 float4 (widths multiples of 4, 16-byte aligned), 0 scalar;
 *   [4], [5] epoch kernel: bit l set when layer l takes the split forward / split backward form;
 *   [6] scores: 1 the tile kernel (layers [64,32,16], mf_dim <= 64), 0 the warp-per-pair kernel.
 *   nrc_ncf_train_epoch reports its last step. */
int nrc_ncf_last_routes(int32_t* out);

/* MF.predict(user_ids, None), model/general_recommender/MF.py:120-122 (np.matmul(U[users], V.T))
 * and LightGCN.predict, LightGCN.py:187-189, materialised: scores f32 [num_rows, num_items]
 * with the same fp32 FMA chain over k the fused evaluator uses. */
int nrc_mf_scores(const float* user_table, const float* item_table, int32_t dim,
                  int32_t num_items, const int32_t* users, int32_t num_rows, float* scores,
                  void* stream);

/* The train mask of UniEvaluator.evaluate, evaluator/backend/cpp/uni_evaluator.py:140-143:
 * scores[b, train_items(users[b])] = -inf for a materialised [num_rows, rating_len] matrix
 * (train CSR indexed by user id). */
int nrc_mask_rows(float* scores, int32_t rating_len, int32_t num_rows, const int32_t* users,
                  const int64_t* train_indptr, const int32_t* train_indices, void* stream);

/* Item-sharded evaluation (catalogues that exceed one GPU, SURVEY.md 8e): the pieces around the
 * per-shard nrc_eval_mf call.  Replaces MF.predict + cpp_evaluate_matrix (MF.py:120-122,
 * evaluate.h:23-72) when the item table is cut into row blocks over ranks.
 *   nrc_mf_score_pairs        exact fp32 scores (the evaluators' FMA chain) of C candidate items per
 *                             row; user_rows f32 [num_rows, dim] are the batch's gathered user rows,
 *                             items i32 [num_rows, C] index item_table (-1 = none), the train CSR is
 *                             indexed by ROW in the same id space; masked / missing -> -inf
 *   nrc_eval_merge_candidates per row the K best of C (score, GLOBAL id) candidates in (score desc,
 *                             id asc) order + the metrics of metric.h on them; *tie_count += rows
 *                             with equal scores inside their top K+1, fewer than K+1 candidates or a
 *                             NaN candidate (there the reference's order depends on its heap and only
 *                             the score sequence is guaranteed equal); top_k <= 512, C <= 512 */
int nrc_mf_score_pairs(const float* user_rows, const float* item_table, int32_t dim,
                       const int32_t* items, int32_t num_rows, int32_t C, const int64_t* train_indptr,
                       const int32_t* train_indices, float* out, void* stream);
int nrc_eval_merge_candidates(const int32_t* cand_ids, const float* cand_scores, int32_t C,
                              int32_t num_rows, const int64_t* test_indptr, const int32_t* test_indices,
                              const int32_t* metric_host, int32_t metric_num, int32_t top_k,
                              float* results, int32_t* ranks, int32_t* tie_count, void* stream);

/* np.mean(all_user_result, axis=0) in fp32, evaluator/backend/cpp/uni_evaluator.py:150:
 * out[c] = (sequential fp32 sum over rows of results[:, c]) / num_rows, bit-identical to
 * numpy's axis-0 reduction order; a single column is contiguous, and there numpy's (and this
 * call's) sum is pairwise. */
int nrc_mean_rows(const float* results, int64_t num_rows, int32_t num_cols, float* out,
                  void* stream);

/* ======================================================================================
 * Negative sampler
 * ==================================================================================== */

/* _sampling_negative_items, data/sampler.py:71-90 + batch_randint_choice,
 * util/cython/random_choice.pyx:64-89 with replace=True: for positive p (owned by user
 * users[p]) draw neg_num items uniformly from [0, num_items) \ train(users[p]).
 * Counter-based Philox4x32-10: draw (p, s, attempt) depends only on (seed, stream_id) so any
 * partition over GPUs yields the same negatives.  out i32 [n, neg_num].
 * NRC_E_VALUE when neg_num <= 0 (sampler.py:72-73) or a user excludes every item
 * (random_choice.pyx:32-33). */
int nrc_sample_negatives(const int64_t* train_indptr, const int32_t* train_indices,
                         const int32_t* users, int64_t n, int32_t neg_num, int32_t num_items,
                         uint64_t seed, uint64_t stream_id, int64_t first_index,
                         int32_t* out, void* stream);

/* ======================================================================================
 * The device-resident epoch: shuffle + sampling + batching
 * ==================================================================================== */

/* RandomSampler, util/data_iterator.py:45-63 (`np.random.permutation(n)` per epoch): out[p] =
 * index of the sample that lands at shuffled position p.  The order is a keyed bijection of
 * [0, n) (alternating Feistel network + cycle walking, round keys from Philox4x32-10 keyed by
 * (seed, epoch)) evaluated per element: no host permutation, no sort.  shuffle = 0 gives the
 * identity (SequentialSampler, data_iterator.py:33-42).  out i64 [n]. */
int nrc_shuffle_perm(int64_t n, int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t* out,
                     void* stream);

/* One epoch of PairwiseSampler.__iter__ (data/sampler.py:189-206) or PointwiseSampler.__iter__
 * (data/sampler.py:121-147) as device arrays, WITHOUT the per-sample python gather of
 * util/data_iterator.py:147-152: positions [first, first + n_out) of the shuffled epoch.
 *   pos_users / pos_items  the flattened positives of _generate_positive_items (sampler.py:24-39)
 *   pairwise = 1: out_third i32 [n_out, neg_num] negatives of the positive at that position
 *   pairwise = 0: samples are the positives (label 1.0) followed by the k-th negatives of all
 *                 positives, k-major (sampler.py:139-141); out_items holds the item, out_third
 *                 f32 [n_out] the label
 * Negatives are the draws nrc_sample_negatives(seed, stream_id = epoch) makes for the same
 * positive, so the epoch does not depend on how it is cut into calls or GPUs. */
int nrc_epoch_build(const int64_t* train_indptr, const int32_t* train_indices,
                    const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos,
                    int32_t neg_num, int32_t num_items, int32_t pairwise, int32_t shuffle,
                    uint64_t seed, uint64_t epoch, int64_t first, int64_t n_out,
                    int32_t* out_users, int32_t* out_items, void* out_third, void* stream);

/* Steps [first_step, first_step + num_steps) of one epoch of MF.train_model (MF.py:84-108:
 * sampler construction aside, `for batch in data_iter: sess.run((loss, optimizer), feed_dict)`)
 * in ONE persistent cooperative launch: the epoch arrays of nrc_epoch_build (built in the same
 * launch when first_step == 0, into ws_users / ws_items / ws_third, i32 [n_samples] each), then
 * per step the gradient pass and the TensorFlow-1.12 optimizer over both tables with grid-wide
 * barriers in between -- same arithmetic as nrc_mf_train_epoch.
 *   adam_pows   device f32 [2] = {beta1^t, beta2^t} of the next step (TF's beta-power variables,
 *               initialise to {beta1, beta2}); read and advanced by the kernel (adam only)
 *   step_loss   device f32 [steps of the epoch]; zeroed when first_step == 0
 *   drop_last   trims the epoch to a multiple of batch_size (sampler.py:150-155, 208-213)
 * hyper_host = {lr, beta1|rho|momentum, beta2|momentum, eps} as in nrc_opt_apply_rows. */
int nrc_mf_epoch_fused(float* user_table, float* item_table, int32_t num_users, int32_t num_items,
                       int32_t dim, const int64_t* train_indptr, const int32_t* train_indices,
                       const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos,
                       int32_t neg_num, int32_t pairwise, int32_t shuffle, int32_t drop_last,
                       uint64_t seed, uint64_t epoch, int32_t batch_size, int64_t first_step,
                       int64_t num_steps, int32_t loss_kind, float reg, int32_t opt_kind,
                       const float* hyper_host, float* adam_pows, float* grad_user,
                       float* grad_item, int32_t* touched_user, int32_t* touched_item,
                       float* slot0_user, float* slot1_user, float* slot0_item, float* slot1_item,
                       int32_t first_stamp, int32_t* ws_users, int32_t* ws_items, void* ws_third,
                       float* step_loss, void* stream);

/* batch_randint_choice(high, size, replace, p=None, exclusion), random_choice.pyx:64-89.
 * `size` is given as out_indptr i64 [n_rows+1] (prefix sums of the per-row sizes, device) and
 * total_out = out_indptr[n_rows]; exclusion CSR may be NULL.  replace=0 draws without
 * replacement inside a row.  A row whose exclusion covers [0, high) gets -1 entries (the
 * reference raises ValueError, random_choice.pyx:32-33; the Python wrapper checks up front). */
int nrc_batch_randint_choice(int32_t high, const int64_t* out_indptr, int32_t n_rows,
                             int64_t total_out, int32_t replace, const int64_t* excl_indptr,
                             const int32_t* excl_indices, uint64_t seed, uint64_t stream_id,
                             int32_t* out, void* stream);

/* ======================================================================================
 * MF-family training step (BPRMF / pointwise "GMF")
 * ==================================================================================== */

/* Gradient phase of MF._create_loss, model/general_recommender/MF.py:54-69, with
 * learner.pairwise_loss (util/learner.py:18-29) and tool.l2_loss (util/tool.py:216-217):
 *   x = <U[u],V[i]> - <U[u],V[j]>;  loss = sum_b l(x_b) + reg/2 (|U[u]|^2+|V[i]|^2+|V[j]|^2)
 * Reads the tables, adds the row gradients of every triplet into the dense accumulators
 * grad_user/grad_item (duplicate ids sum, as TF's IndexedSlices dedup does), stamps touched
 * rows with `stamp` (> 0, strictly increasing per step; the touched arrays start zeroed and
 * are never cleared), adds the batch loss into *loss.  Tables are NOT modified. */
int nrc_mf_pairwise_grad(const float* user_table, const float* item_table, int32_t dim,
                         const int32_t* users, const int32_t* pos_items,
                         const int32_t* neg_items, int64_t batch, int32_t loss_kind, float reg,
                         float* grad_user, float* grad_item, int32_t* touched_user,
                         int32_t* touched_item, int32_t stamp, float* loss, void* stream);

/* Pointwise branch, MF.py:70-72 with learner.pointwise_loss (util/learner.py:31-41):
 * cross_entropy = MEAN over the batch of max(x,0) - x*z + log1p(exp(-|x|)); square = SUM. */
int nrc_mf_pointwise_grad(const float* user_table, const float* item_table, int32_t dim,
                          const int32_t* users, const int32_t* items, const float* labels,
                          int64_t batch, int32_t loss_kind, float reg, float* grad_user,
                          float* grad_item, int32_t* touched_user, int32_t* touched_item,
                          int32_t stamp, float* loss, void* stream);

/* learner.optimizer, util/learner.py:2-15: apply TensorFlow-1.12 update rules to a table
 * whose gradient arrived as IndexedSlices (embedding rows).
 *   var, grad f32 [rows, dim]; slot0/slot1 optimizer state (adam: m, v; adagrad: accum;
 *   rmsprop: ms, mom; momentum: accum; gd: unused); touched i32 [rows] from the grad phase.
 *   hyper[0..3]: adam {lr_t, beta1, beta2, eps} with lr_t = lr*sqrt(1-b2^t)/(1-b1^t) computed
 *   by the caller in fp32 as TF does; adagrad {lr}; rmsprop {lr, decay, momentum, eps};
 *   momentum {lr, momentum}; gd {lr}.
 * adam moves EVERY row (TF-1.12 _apply_sparse_shared decays m, v densely); the others only
 * rows whose touched stamp equals `stamp`.  Zeroes grad afterwards (ready for the next step). */
int nrc_opt_apply_rows(int32_t opt_kind, float* var, float* grad, float* slot0, float* slot1,
                       const int32_t* touched, int32_t stamp, int64_t rows, int32_t dim,
                       const float* hyper_host, void* stream);

/* Large-table BPR + plain SGD (learner=gd) in ONE HBM pass, for tables too big for a dense
 * gradient accumulator (BASELINE config 5; dim 32 / 64 / 128): per triplet three coalesced row
 * gathers, the two dots, g = -sigmoid(-x), and `row -= lr * grad` applied in place with vector
 * RED.ADD so repeated rows still receive every contribution.  Equals MF.py:62-69 +
 * GradientDescentOptimizer exactly when no row repeats inside the batch; with repeats a triplet
 * may read a row already updated by another triplet of the same batch (documented deviation). */
int nrc_mf_bpr_sgd_fused(float* user_table, float* item_table, int32_t dim, const int32_t* users,
                         const int32_t* pos_items, const int32_t* neg_items, int64_t batch,
                         float lr, float reg, float* loss, void* stream);

/* nrc_mf_bpr_sgd_fused on ROW-SHARDED tables (BASELINE config 5: tables larger than one GPU; the
 * arithmetic is MF.py:54-76 + learner.py:8 `GradientDescentOptimizer`, the reference itself has no
 * multi-device path).
 * Shard r of a table holds global rows [r*rows_per_shard, (r+1)*rows_per_shard); user_shards /
 * item_shards are HOST arrays of `world` device pointers: the caller's own shard plus peer
 * mappings of the other ranks' shards (CUDA IPC; nrc_enable_peer_access first).  Every rank calls
 * it with its own triplets (global ids; the reference partitions by user, so `users` are normally
 * local rows); remote rows are read and updated in place over NVLink by the same kernel -- no
 * all-to-all of ids, rows or gradients (local rows: one vector RED; peer rows: scalar REDs).
 * self_rank = index of the caller's own shard.  world <= 8, global ids must fit int32. */
int nrc_mf_bpr_sgd_sharded(float* const* user_shards, float* const* item_shards, int32_t world,
                           int32_t self_rank, int64_t users_per_shard, int64_t items_per_shard, int32_t dim,
                           const int32_t* users, const int32_t* pos_items, const int32_t* neg_items,
                           int64_t batch, float lr, float reg, float* loss, void* stream);
/* BPR + SGD straight from the train CSR (BASELINE configs[4]; MF.py:54-76 with learner=gd, plus
 * data/sampler.py:71-90,189-206 and util/data_iterator.py:59 fused in): positions
 * [first, first + count) of shuffled epoch `epoch` are sampled (keyed bijection + Philox rejection
 * draw), scored and applied in place by ONE kernel -- no id arrays, no sampler pass.  user_table is
 * this rank's row block and pos_users are LOCAL row ids (the train CSR is partitioned by user
 * owner); item ids are global, item_shards[r] (host array of `world` device pointers) is the row
 * block of rank r: own memory for r == self_rank, peer mappings otherwise (nrc_shard_alloc /
 * nrc_ipc_open), read and RED-updated over NVLink by the same kernel.  world = 1: item_shards[0]
 * is the whole table.  *loss += sum of the triplets' losses.
 * When pos_items == train_indices (the same pointer), pos_users MUST be the row expansion of
 * train_indptr (pos_users[q] = u for q in [train_indptr[u], train_indptr[u+1]), as nrc_csr_row_ids
 * writes it): the kernel then finds the user rows that only one triplet of the call touches from the
 * CSR and the shuffle alone, and writes those with plain stores instead of atomics. */
int nrc_mf_bpr_sgd_epoch(float* user_table, float* const* item_shards, int32_t world,
                         int32_t self_rank, int64_t items_per_shard, int32_t dim,
                         const int64_t* train_indptr, const int32_t* train_indices,
                         const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos,
                         int32_t num_items, int32_t shuffle, uint64_t seed, uint64_t epoch,
                         int64_t first, int64_t count, float lr, float reg, float* loss,
                         void* stream);

/* nrc_mf_bpr_sgd_epoch with a REPLICATED HEAD of the item table (n_hot = 0: identical to it).  Item ids
 * [0, n_hot) -- the loader relabels items by descending train degree (neurec_b200.util.peer.relabel_by_degree),
 * so these are the most popular ones, the rows thousands of triplets of every step land on -- are read from this
 * rank's replica `hot` [n_hot, dim] and their deltas accumulate in this rank's `hot_delta` [n_hot, dim] instead of
 * crossing NVLink as same-address atomics on the owner.  Between steps the caller sums hot_delta over the ranks
 * (one all-reduce of n_hot * dim floats) and calls nrc_mf_hot_apply.  Within a step the replicated rows keep their
 * pre-step values, which is what TF computes for every row (MF.py:54-76: all gradients of a batch are taken at the
 * pre-step variables); the other rows are updated in place. */
int nrc_mf_bpr_sgd_epoch_hot(float* user_table, float* const* item_shards, int32_t world,
                             int32_t self_rank, int64_t items_per_shard, int32_t dim,
                             const int64_t* train_indptr, const int32_t* train_indices,
                             const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos,
                             int32_t num_items, int32_t shuffle, uint64_t seed, uint64_t epoch,
                             int64_t first, int64_t count, float lr, float reg, float* loss,
                             float* hot, float* hot_delta, int32_t n_hot, void* stream);
/* hot[e] += hot_delta[e]; hot_delta[e] = 0 for e < n_floats (a multiple of 4; both 16-byte aligned). */
int nrc_mf_hot_apply(float* hot, float* hot_delta, int64_t n_floats, void* stream);

/* Test hook of the MF training kernels (it reports and changes nothing; every route is chosen by the shape).
 * nrc_mf_last_routes: HOST bookkeeping of the most recent launch of each kernel group, written when a call launches
 * (a call that returns before launching, for a failed check or an empty batch, leaves it as it was); one record per
 * process.  out i32[6 * 7], group k at out[7 * k]; -1 = no such launch yet, or a field the group does not decide.
 *   groups: [0] nrc_mf_pairwise_grad / _pointwise_grad (also inside nrc_mf_train_epoch / _train_step_host);
 *   [1] the id-fed in-place step (nrc_mf_bpr_sgd_fused / _sharded); [2] the CSR-fed in-place step
 *   (nrc_mf_bpr_sgd_epoch / _epoch_hot); [3] nrc_mf_bpr_lazy_adam_epoch; [4] the persistent nrc_mf_epoch_fused;
 *   [5] the multi-tensor optimizer apply (nrc_opt_apply_rows / _multi and the second phase of the per-step paths).
 *   fields of a group:
 *   +0 VEC, floats per lane of a row (dim / 32 for dim 32, 64, 128), 0 the generic any-dim loop;
 *   +1 1 when the kernel's SHARDED form ran (item rows addressed through the shard table), else 0;
 *   +2 CSR-fed step: 1 when user rows touched once by the launch take a plain store (pos_items == train_indices);
 *   +3 CSR-fed step: head rows held in the shared-memory tier, min(n_hot, 8192 / dim);
 *   +4 CTAs launched;
 *   +5 1 when the grid was capped, so a warp (or thread) takes more than one triplet, sample or element: grad and
 *      id-fed step above 64 * SMs triplets, CSR-fed step above 768 per resident CTA, lazy Adam above 2048 * SMs,
 *      persistent epoch when a batch of the launch exceeds its 16 * SMs warps, optimizer apply above 2048 * SMs
 *      elements; else 0;
 *   +6 persistent epoch: 1 the float4 optimizer pass (dim % 4 == 0), 0 the per-element one. */
int nrc_mf_last_routes(int32_t* out);


/* The explicitly-named LAZY-Adam variant of nrc_mf_bpr_sgd_epoch (SURVEY.md 8d, BASELINE configs[4]:
 * "learner=gd for the roofline run plus an explicitly-named lazy-Adam run"; the reference's own
 * learner=adam, util/learner.py:6, is TF's DENSE Adam and is what nrc_opt_apply_* implement).
 * tf.contrib.opt.LazyAdamOptimizer semantics on the rows of each triplet, applied per triplet in one
 * pass without batch-wide de-duplication (rows that repeat inside a batch are updated per occurrence
 * and may overwrite each other).  Single GPU; user / item slots m, v shaped like the tables. */
int nrc_mf_bpr_lazy_adam_epoch(float* user_table, float* user_m, float* user_v, float* item_table,
                               float* item_m, float* item_v, int32_t dim, const int64_t* train_indptr,
                               const int32_t* train_indices, const int32_t* pos_users,
                               const int32_t* pos_items, int64_t n_pos, int32_t num_items,
                               int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t first,
                               int64_t count, float lr_t, float beta1, float beta2, float eps,
                               float reg, float* loss, void* stream);

/* A device allocation of its own (cudaMalloc, never a slice of a caching allocator's block) for a
 * table shard that other ranks map: *dev_ptr_out and its 64-byte CUDA IPC handle.  Peers open the
 * handle with nrc_ipc_open(handle, 0, &ptr) -- one handle per shard, so a mapping is never opened
 * twice in a process -- and close it with nrc_ipc_close(ptr, 0) before the owner frees. */
int nrc_shard_alloc(int64_t nbytes, void** dev_ptr_out, void* handle64_out);
int nrc_shard_free(void* dev_ptr);

/* Let kernels of the current device dereference memory of `peer_device` (idempotent). */
int nrc_enable_peer_access(int32_t peer_device);
/* CUDA IPC for the shards: export = 64-byte handle of the allocation holding dev_ptr + the offset
 * of dev_ptr inside it; open (in ANOTHER process, with the importing device current) maps it with
 * lazy peer access and returns the pointer that corresponds to dev_ptr; close unmaps it. */
int nrc_ipc_export(const void* dev_ptr, void* handle64_out, int64_t* offset_out);
int nrc_ipc_open(const void* handle64, int64_t offset, void** dev_ptr_out);
int nrc_ipc_close(void* dev_ptr, int64_t offset);

/* Same rules for every variable of a model in ONE launch (what `optimizer.minimize(loss)`,
 * util/learner.py:2-16, applies per step).  All arrays are HOST arrays of length n_vars holding device pointers /
 * shapes; dense_var[i] = 1 marks a variable whose gradient is a dense tensor (tf.layers.dense
 * kernel / bias: Apply* functor formulas, every element), 0 an IndexedSlices variable. */
int nrc_opt_apply_multi(int32_t opt_kind, int32_t n_vars, float* const* var, float* const* grad,
                        float* const* slot0, float* const* slot1, const int32_t* const* touched,
                        const int64_t* rows, const int32_t* dims, const int32_t* dense_var,
                        int32_t stamp, const float* hyper_host, void* stream);

/* One epoch of MF.train_model, MF.py:92-108, on device-resident, already shuffled id arrays
 * (n samples, steps = ceil(n / batch_size), last batch smaller, sampler.py:208-213).
 *   third: neg items (pairwise, i32) or labels (pointwise, f32 bits) -- selected by
 *   `pairwise`.  lr_t_host f32 [steps] per-step adam lr_t (ignored for other optimizers
 *   except element 0 = lr).  step_loss f32 [steps] receives each step's loss.  Stamps
 *   first_stamp .. first_stamp+steps-1 are consumed. */
int nrc_mf_train_epoch(float* user_table, float* item_table, int32_t num_users,
                       int32_t num_items, int32_t dim, const int32_t* users,
                       const int32_t* items, const void* third, int64_t n, int32_t batch_size,
                       int32_t pairwise, int32_t loss_kind, float reg, int32_t opt_kind,
                       const float* lr_t_host, const float* hyper_host, float* grad_user,
                       float* grad_item, int32_t* touched_user, int32_t* touched_item,
                       float* slot0_user, float* slot1_user, float* slot0_item,
                       float* slot1_item, int32_t first_stamp, float* step_loss, void* stream);

/* One `sess.run((loss, optimizer), feed_dict)` of MF.train_model (MF.py:97-108): the id /
 * label arrays of ONE batch are HOST buffers (the python lists the reference feeds; pinned
 * memory makes the copies asynchronous), tables and optimizer state stay on the device like TF
 * variables.  Copies the batch H2D into `staging` (device scratch, >= 12*batch+16 bytes), runs
 * both phases, copies the loss back and synchronises the stream: *loss_host is valid on
 * return.  hyper_host[0] must already hold this step's lr_t for adam. */
int nrc_mf_train_step_host(float* user_table, float* item_table, int32_t num_users,
                           int32_t num_items, int32_t dim, const int32_t* users_host,
                           const int32_t* items_host, const void* third_host, int64_t batch,
                           int32_t pairwise, int32_t loss_kind, float reg, int32_t opt_kind,
                           const float* hyper_host, float* grad_user, float* grad_item,
                           int32_t* touched_user, int32_t* touched_item, float* slot0_user,
                           float* slot1_user, float* slot0_item, float* slot1_item,
                           int32_t stamp, void* staging, float* loss_host, void* stream);

/* ======================================================================================
 * NCF family: MLP (model/general_recommender/MLP.py) and NeuMF = GMF + MLP (NeuMF.py)
 * ==================================================================================== */

/* Model shape.  mf_dim = embedding_size (0 for MLP.py); mlp_dim = layers[0]/2, the width of
 * each MLP embedding (NeuMF.py:58-61, MLP.py:48-51); layers = units of the tf.layers.dense
 * stack -- the first layer maps layers[0] -> layers[0] (NeuMF.py:81-82); n_towers = 2 only for
 * pairwise NeuMF, whose negative tower re-instantiates tf.layers.dense (NeuMF.py:90-92).
 * Dense parameters are one packed f32 buffer: for tower t, layer l: kernel [in, out] row-major
 * then bias [out]; towers back to back (nrc_ncf_dense_size floats in total). */
typedef struct nrc_ncf_shape {
    int32_t num_users, num_items;
    int32_t mf_dim, mlp_dim;
    int32_t n_layers;
    int32_t layers[4];
    int32_t n_towers;
} nrc_ncf_shape;

int nrc_ncf_dense_size(const nrc_ncf_shape* shape);

/* Gradient phase of NeuMF._create_loss (NeuMF.py:87-100) / MLP._create_loss (MLP.py:72-82):
 * prediction = sum(mf_user*mf_item) + sum(relu-MLP(concat(mlp_user, mlp_item))) (NeuMF.py:85);
 * pairwise (third = neg items i32) or pointwise (third = labels f32) loss as in util/learner.py;
 * + reg_mf*l2_loss(p1,q2,q1) + reg_mlp*l2_loss(m1,n2,n1).  Adds the gradients of the four
 * tables and of the packed dense parameters into the g_* accumulators (never applies them). */
int nrc_ncf_grad(const nrc_ncf_shape* shape, const float* mf_user, const float* mf_item,
                 const float* mlp_user, const float* mlp_item, const float* dense,
                 const int32_t* users, const int32_t* items, const void* third, int64_t batch,
                 int32_t pairwise, int32_t loss_kind, float reg_mf, float reg_mlp,
                 float* g_mf_user, float* g_mf_item, float* g_mlp_user, float* g_mlp_item,
                 float* g_dense, int32_t* touched_user, int32_t* touched_item, int32_t stamp,
                 float* loss, void* stream);

/* NeuMF.predict / MLP.predict with candidate_items=None (NeuMF.py:163-168): the tower-0 forward
 * of every (users[b], item) pair -> scores f32 [n_users, num_items] (device). */
int nrc_ncf_scores(const nrc_ncf_shape* shape, const float* mf_user, const float* mf_item,
                   const float* mlp_user, const float* mlp_item, const float* dense,
                   const int32_t* users, int32_t n_users, int32_t num_items, float* scores,
                   void* stream);

/* One epoch of NeuMF.train_model (NeuMF.py:126-151) on device-resident shuffled arrays.
 * grads / slot0 / slot1 are HOST arrays of 5 device pointers in the order
 * {mf_user, mf_item, mlp_user, mlp_item, dense}; the four tables get IndexedSlices optimizer
 * semantics, the packed dense parameters dense-gradient semantics (see nrc_opt_apply_multi). */
int nrc_ncf_train_epoch(const nrc_ncf_shape* shape, float* mf_user, float* mf_item,
                        float* mlp_user, float* mlp_item, float* dense, const int32_t* users,
                        const int32_t* items, const void* third, int64_t n, int32_t batch_size,
                        int32_t pairwise, int32_t loss_kind, float reg_mf, float reg_mlp,
                        int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                        float* const* grads, float* const* slot0, float* const* slot1,
                        int32_t* touched_user, int32_t* touched_item, int32_t first_stamp,
                        float* step_loss, void* stream);

/* Steps [first_step, first_step + num_steps) of one epoch of NeuMF.train_model / MLP.train_model
 * (NeuMF.py:126-151, MLP.py:100-120) in ONE persistent cooperative launch: the epoch arrays of
 * nrc_epoch_build (built in the same launch when first_step == 0), then per step the per-sample
 * tower forward / backward out of shared memory, the weight gradients in fixed summation order and
 * the TensorFlow-1.12 optimizer over the four tables and the packed dense parameters, with grid-wide
 * barriers in between.  Arguments as nrc_ncf_train_epoch + the epoch description of
 * nrc_mf_epoch_fused (adam_pows, workspace arrays i32 [n_samples], step_loss zeroed at first_step 0).
 * grads[0..3] are the table accumulators (grads[4] is not used: dW never leaves the chip). */
int nrc_ncf_epoch_fused(const nrc_ncf_shape* shape, float* mf_user, float* mf_item, float* mlp_user,
                        float* mlp_item, float* dense, const int64_t* train_indptr,
                        const int32_t* train_indices, const int32_t* pos_users,
                        const int32_t* pos_items, int64_t n_pos, int32_t neg_num, int32_t pairwise,
                        int32_t shuffle, int32_t drop_last, uint64_t seed, uint64_t epoch,
                        int32_t batch_size, int64_t first_step, int64_t num_steps, int32_t loss_kind,
                        float reg_mf, float reg_mlp, int32_t opt_kind, const float* hyper_host,
                        float* adam_pows, float* const* grads, float* const* slot0,
                        float* const* slot1, int32_t* touched_user, int32_t* touched_item,
                        int32_t first_stamp, int32_t* ws_users, int32_t* ws_items, void* ws_third,
                        float* step_loss, void* stream);

/* ======================================================================================
 * Graph propagation: CSR SpMM and the LightGCN step
 * ==================================================================================== */

/* Accumulation order of every SpMM below.  0 (default): fast order -- several non-zeros per load
 * instruction, FFMA into independent partial sums, long rows split over a CTA; deterministic, within
 * fp32 re-association (<= 1e-6 relative) of the sequential product.  1: each output row is the
 * SEQUENTIAL sum over its non-zeros with separately rounded multiply and add, bit-identical to
 * scipy's csr_matvecs and to TF-1.12's sparse_tensor_dense_matmul CPU kernel (LightGCN.py:140). */
int nrc_spmm_set_exact(int32_t on);

/* tf.sparse_tensor_dense_matmul(adj_mat, ego_embeddings), LightGCN.py:140 / NGCF.py:176:
 *   y[r, :] = sum over the nnz of row r, in CSR order, of values[p] * x[indices[p], :]
 * with separately rounded multiply and add (sequential, TF/scipy CPU order => bit-exact), then
 * the optional epilogue  y = bias[r,:] + y;  Y[r,:] = y;  sum[r,:] = (sum[r,:] + y) [/ div].
 * row_order (optional i32 [n_rows]) is the order rows are dealt to warps (degree-descending
 * for load balance); bias / y / sum may be NULL; div = 0 disables the division. */
int nrc_spmm_csr(const int64_t* indptr, const int32_t* indices, const float* values,
                 const int32_t* row_order, int32_t n_rows, const float* x, int32_t dim,
                 const float* bias, float* y, float* sum, float div, void* stream);

/* _create_lightgcn_embed, LightGCN.py:132-149: e_final = mean(E_0, A E_0, ..., A^L E_0) with
 * E_0 = concat(user_embedding, item_embedding).  work_a / work_b: [n_nodes, dim] scratch. */
int nrc_lightgcn_propagate(const int64_t* indptr, const int32_t* indices, const float* values,
                           const int32_t* row_order, int32_t n_nodes, int32_t dim,
                           int32_t n_layers, const float* e0, float* e_final, float* work_a,
                           float* work_b, void* stream);

/* create_bpr_loss, LightGCN.py:156-166 on the propagated table e_final (users first, then
 * items) with the regulariser on the layer-0 rows e0.  Adds scale * dLoss/dE_final into
 * grad_final and reg * e0[row] into grad_reg (both dense [n_nodes, dim]); loss2 += {mf_loss,
 * emb_loss}.  scale = 1/(n_layers+1) is the reduce_mean factor of LightGCN.py:147. */
int nrc_lightgcn_bpr_grad(const float* e_final, const float* e0, int32_t num_users, int32_t dim,
                          const int32_t* users, const int32_t* pos_items, const int32_t* neg_items,
                          int64_t batch, float reg, float scale, float* grad_final,
                          float* grad_reg, float* loss2, void* stream);

/* One epoch of LightGCN.train_model, LightGCN.py:168-180: per batch the forward propagation
 * (n_layers SpMM), the BPR gradient, the backward propagation (n_layers SpMM with the
 * transposed CSR t_*; pass NULL when A_hat is symmetric, adj_type 'pre') and a dense Adam step
 * over E_0 (TF ApplyAdam formulas; lr_t_host f32 [steps]).  grad_final and grad_e0 must be
 * zero on entry and are zero on return.  step_loss2 f32 [steps, 2] = {mf_loss, emb_loss}. */
int nrc_lightgcn_train_epoch(const int64_t* indptr, const int32_t* indices, const float* values,
                             const int64_t* t_indptr, const int32_t* t_indices,
                             const float* t_values, const int32_t* row_order, int32_t num_users,
                             int32_t num_items, int32_t dim, int32_t n_layers, float* e0,
                             float* adam_m, float* adam_v, const int32_t* users,
                             const int32_t* pos_items, const int32_t* neg_items, int64_t n,
                             int32_t batch_size, float reg, const float* lr_t_host,
                             const float* hyper_host, float* e_final, float* grad_final,
                             float* grad_e0, float* work_a, float* work_b, float* step_loss2,
                             void* stream);

/* Test hook of the graph kernels (it reports and changes nothing; every route is chosen by the shape).
 * nrc_graph_last_routes: HOST bookkeeping of what the most recent calls decided, written when a call launches (a
 * call that returns before launching leaves it as it was); one record per process.  out i32[9]; -1 = no such
 * launch yet, or not decided by the last call of that group:
 *   SpMM (the last nrc_spmm_csr product, also those inside the LightGCN / NGCF calls):
 *   [0] 1 the fast kernel, 0 the exact (sequential) kernel;
 *   [1] fast: lanes per gathered row G = dim / 4 (8, 16, 32); exact: columns per lane V = dim / 32 (1, 2, 4), or 0
 *       for the generic form (any dim up to 256);
 *   [2] 1 when the grid was capped at 8 CTAs per SM, so a CTA (fast) or warp (exact) handles more than one 8-row
 *       unit or row (n_rows > 64 * SMs), else 0;
 *   NGCF (the last nrc_ngcf_forward / nrc_ngcf_grad; a forward sets [4] and [5] to -1):
 *   [3] most rows per warp of the layer forward kernel;
 *   [4] most 32-row tiles per CTA of the layer backward kernel (dW / db accumulated across them);
 *   [5] most triplets per warp of the BPR gradient kernel (0 for an empty batch);
 *   SpectralCF (the last nrc_spectralcf_forward / nrc_spectralcf_grad; 0 = no such product, as with 0 layers;
 *   a forward sets [7] and [8] to -1): number of K slices (gridDim.y) of
 *   [6] the forward products A_hat . E_{k-1}; [7] the backward products A_hat^T . dS; [8] the products dW_k. */
int nrc_graph_last_routes(int32_t* out);

/* ======================================================================================
 * NGCF: dense part of the propagation layer (SURVEY.md 8f rank 1)
 * ==================================================================================== */

/* NGCF.__init__ / _init_weights, NGCF.py:14-44, 262-284 (alg_type 'ngcf').  Weights are one packed
 * f32 buffer: per layer W_gc [d_k, d_k+1] row-major, b_gc [d_k+1], W_bi [d_k, d_k+1], b_bi [d_k+1]
 * (nrc_ngcf_weights_size floats).  Widths up to 64, up to 4 layers. */
typedef struct nrc_ngcf_shape {
    int32_t num_users, num_items;
    int32_t emb_dim;
    int32_t n_layers;
    int32_t layers[4];
} nrc_ngcf_shape;

int nrc_ngcf_weights_size(const nrc_ngcf_shape* shape);
int64_t nrc_ngcf_work_floats(const nrc_ngcf_shape* shape);   /* size of the `work` buffer below */

/* tf.nn.dropout's keep mask (NGCF.py:193, always on): out[e] = 1.0 with probability keep, else 0.0;
 * counter-based Philox4x32-10 keyed by (seed, stream_id).  out f32 [n]. */
int nrc_dropout_mask(int64_t n, float keep, uint64_t seed, uint64_t stream_id, float* out, void* stream);

/* _create_ngcf_embed, NGCF.py:160-202: per layer side = A_hat.ego (the CSR of get_adj_mat, NGCF.py:
 * 299-332; the n_fold slabs of :174-179 are one product), leaky_relu(side W_gc + b_gc) +
 * leaky_relu((ego*side) W_bi + b_bi), dropout with the given masks (f32 0/1, layer k's [N, d_k+1]
 * block after the previous ones; NULL = keep everything), l2_normalize, concatenation.
 * all_emb f32 [N, emb_dim + sum(layers)], users first. */
int nrc_ngcf_forward(const nrc_ngcf_shape* shape, const int64_t* indptr, const int32_t* indices,
                     const float* values, const int32_t* row_order, const float* e0,
                     const float* weights, const float* masks, float keep, float* all_emb,
                     float* work, void* stream);

/* Loss and gradients of one batch, NGCF.py:94-110 + the backward of :160-202: forward as above, then
 * sum softplus(-(pos - neg)) + reg * l2_loss(u, i, j) on the concatenated rows, back through
 * normalise / dropout / leaky-relu / both GEMMs / SpMM (t_* = CSR of A_hat^T, NULL when symmetric).
 * grad_all f32 [N, d_total] must be zero on entry and is zero on return; grad_e0 f32 [N, emb_dim]
 * and grad_weights f32 [weights_size] are overwritten; loss2 f32 [2] += {mf_loss, emb_loss}.
 * Apply them with nrc_opt_apply_multi (dense-gradient formulas, like every variable of NGCF). */
int nrc_ngcf_grad(const nrc_ngcf_shape* shape, const int64_t* indptr, const int32_t* indices,
                  const float* values, const int32_t* row_order, const int64_t* t_indptr,
                  const int32_t* t_indices, const float* t_values, const int32_t* t_row_order,
                  const float* e0, const float* weights, const float* masks, float keep,
                  const int32_t* users, const int32_t* pos_items, const int32_t* neg_items,
                  int64_t batch, float reg, float* all_emb, float* grad_all, float* grad_e0,
                  float* grad_weights, float* work, float* loss2, void* stream);

/* ======================================================================================
 * SURVEY.md 8(f) ranks 3-4: APR, SBPR, time-ordered samplers, interactions -> CSR
 * ==================================================================================== */

/* APR._create_adversarial, model/general_recommender/APR.py:92-118:
 * out[r, :] = tf.nn.l2_normalize(x, 1)[r, :] * scale = (x * rsqrt(max(sum(x^2), 1e-12))) * scale.
 * x, out f32 [rows, dim] (may alias). */
int nrc_l2_normalize_rows(const float* x, int64_t rows, int32_t dim, float scale, float* out, void* stream);

/* out[p, :] = src[index[p] % src_rows, :]; src i32 [src_rows, width], index i64 [n] (nrc_shuffle_perm), out i32
 * [n, width].  The recent-items window of TimeOrderPointwiseSampler / TimeOrderPairwiseSampler
 * (data/sampler.py:216-354) travelling with the shuffled samples (util/data_iterator.py:147-152). */
int nrc_gather_rows_i32(const int32_t* src, int64_t src_rows, int32_t width, const int64_t* index, int64_t n,
                        int32_t* out, void* stream);

/* SBPR._get_pairwise_all_data + DataIterator(shuffle=True), model/social_recommender/SBPR.py:103-149:
 * positions [first, first + count) of the shuffled epoch `epoch`.  For the positive (u, i) at a position:
 * social item k uniform (with replacement) over social_items(u) (np.random.choice, :139), negative j uniform over
 * the items outside train(u) + social_items(u) (randint_choice with exclusion, :135-137),
 * s_uk = 1 + #{f in trust(u): k in train(f)} (:141-145).  CSRs have ascending rows; pos_users / pos_items are the
 * flattened positives of the users with a non-empty social row (:125-131), n_pos of them; max_excluded = the
 * largest train(u) + social(u) size (ValueError when >= num_items, random_choice.pyx:32-33).
 * Outputs i32 [count] x 4 and f32 [count]. */
int nrc_sbpr_epoch_build(const int64_t* train_indptr, const int32_t* train_indices, const int64_t* social_indptr,
                         const int32_t* social_indices, const int64_t* trust_indptr, const int32_t* trust_indices,
                         const int32_t* pos_users, const int32_t* pos_items, int64_t n_pos, int32_t num_items,
                         int32_t max_excluded, int32_t shuffle, uint64_t seed, uint64_t epoch, int64_t first,
                         int64_t count, int32_t* out_users, int32_t* out_pos, int32_t* out_social,
                         int32_t* out_neg, float* out_suk, void* stream);

/* SBPR._create_inference / _create_loss, SBPR.py:66-92: x = <p, q> + b per item; loss =
 * l((x_i - x_k) / s_uk) + l(x_k - x_j) + reg * l2_loss(p, q_k, q_i, q_j, b_i, b_k, b_j) with l = learner.pairwise_loss
 * (util/learner.py:17-29), summed over the batch into *loss.  Row gradients are ADDED into the dense accumulators
 * (grad_bias f32 [num_items]); touched_* get `stamp` (bias shares the items' stamps). */
int nrc_sbpr_grad(const float* user_table, const float* item_table, const float* item_bias, int32_t dim,
                  const int32_t* users, const int32_t* pos_items, const int32_t* social_items,
                  const int32_t* neg_items, const float* suk, int64_t batch, int32_t loss_kind, float reg,
                  float* grad_user, float* grad_item, float* grad_bias, int32_t* touched_user,
                  int32_t* touched_item, int32_t stamp, float* loss, void* stream);

/* SBPR.train_model's batch loop, SBPR.py:111-121, over a device-built epoch of n samples: per batch nrc_sbpr_grad +
 * one TF-1.12 optimizer launch over user table, item table and item bias.  lr_t_host f32 [steps] (adam), hyper_host
 * as nrc_opt_apply_rows; step_loss f32 [steps] receives every batch's loss. */
int nrc_sbpr_train_epoch(float* user_table, float* item_table, float* item_bias, int32_t num_users,
                         int32_t num_items, int32_t dim, const int32_t* users, const int32_t* pos_items,
                         const int32_t* social_items, const int32_t* neg_items, const float* suk, int64_t n,
                         int32_t batch_size, int32_t loss_kind, float reg, int32_t opt_kind,
                         const float* lr_t_host, const float* hyper_host, float* grad_user, float* grad_item,
                         float* grad_bias, int32_t* touched_user, int32_t* touched_item, float* slot0_user,
                         float* slot1_user, float* slot0_item, float* slot1_item, float* slot0_bias,
                         float* slot1_bias, int32_t first_stamp, float* step_loss, void* stream);

/* Interactions (COO, any order, duplicates allowed) -> CSR with ascending duplicate-free rows: what
 * Dataset.to_csr_matrix + csr_to_user_dict (data/dataset.py:288-296, util/tool.py:56-65) hand to samplers and
 * evaluator.  rows, cols i32 [nnz]; out_indptr i64 [num_rows + 1]; out_indices i32 [nnz] (the first
 * out_indptr[num_rows] entries are valid); scratch work_i64 [2 * (num_rows + 1)], work_i32 [2 * nnz];
 * *bad_flag (device i32) = 1 when an id was out of range (those interactions are dropped). */
int nrc_csr_from_coo(const int32_t* rows, const int32_t* cols, int64_t nnz, int32_t num_rows, int32_t num_cols,
                     int64_t* out_indptr, int32_t* out_indices, int64_t* work_i64, int32_t* work_i32,
                     int32_t* bad_flag, void* stream);

/* users_list of _generate_positive_items (data/sampler.py:24-39) expanded on the device: out[e] = row of CSR entry e,
 * out i32 [indptr[num_rows]] -- only (indptr, indices) of the train interactions have to be uploaded. */
int nrc_csr_row_ids(const int64_t* indptr, int64_t num_rows, int32_t* out, void* stream);

/* split_by_ratio / split_by_loo, data/utils.py:59-106, on the device: every user's interactions ordered by `keys`
 * (i64 [n] interaction times, by_time=True) or, when keys is NULL (by_time=False), by a counter-based random word
 * keyed by `seed` (DataFrame.sample(frac=1)); ties by input position; the first ceil(ratio * n_u) (mode 0) or all but
 * the last when n_u > 3 (mode 1, leave-one-out) go to the train set.  users i32 [n] dense ids; is_train i32 [n] <- 1/0.
 * Scratch work_i64 [2 * (num_users + 1)], work_i32 [n]; *bad_flag (device i32) = 1 on an out-of-range user id. */
int nrc_split_interactions(const int32_t* users, const int64_t* keys, int64_t n, int32_t num_users, int32_t mode,
                           double ratio, uint64_t seed, int32_t* is_train, int64_t* work_i64, int32_t* work_i32,
                           int32_t* bad_flag, void* stream);

/* SpectralCF, model/general_recommender/SpectralCF.py:63-91.  a_hat f32 [N, N] (N = users + items, users first) is
 * the constant dense operator U U^T + U diag(lamda) U^T the reference builds with numpy at construction (:37-43,
 * 67-69); filters f32 [num_layers, dim, dim]; activation ids follow util/tool.py:10-33 (softmax is not provided:
 * NRC_E_NOTIMPL, like an unknown name).  dim <= 128, num_layers <= 8. */
#define NRC_ACT_IDENTITY 0
#define NRC_ACT_SIGMOID 1
#define NRC_ACT_TANH 2
#define NRC_ACT_RELU 3
#define NRC_ACT_ELU 4
#define NRC_ACT_SELU 5
int64_t nrc_spectralcf_work_floats(int32_t num_nodes, int32_t dim, int32_t num_layers);
/* _create_inference (:63-83): all_emb f32 [N, dim * (num_layers + 1)] = [E_0 | E_1 | ...], E_k = act((a_hat E_{k-1}) W_k). */
int nrc_spectralcf_forward(int32_t num_nodes, int32_t dim, int32_t num_layers, const float* a_hat, const float* e0,
                           const float* filters, int32_t activation, float* all_emb, float* work, void* stream);
/* One batch of _create_loss (:85-91) and the backward of the whole graph: forward as above, learner.pairwise_loss on
 * the concatenated rows + reg * l2_loss(u, i, j), then back through concat / activation / both products per layer.
 * a_hat_t: a_hat transposed, or NULL (the kernel then reads a_hat with transposed indexing).  grad_all f32
 * [N, dim * (num_layers + 1)] must be zero on entry and is zero on return; touched i32 [N] scratch; grad_e0 f32
 * [N, dim] and grad_filters f32 [num_layers, dim, dim] are overwritten; *loss += the batch loss.  Apply with
 * nrc_opt_apply_multi (dense-gradient formulas: every variable's gradient flows through tf.matmul). */
int nrc_spectralcf_grad(int32_t num_users, int32_t num_items, int32_t dim, int32_t num_layers, const float* a_hat,
                        const float* a_hat_t, const float* e0, const float* filters, int32_t activation,
                        const int32_t* users, const int32_t* pos_items, const int32_t* neg_items, int64_t batch,
                        int32_t loss_kind, float reg, float* all_emb, float* grad_all, int32_t* touched,
                        float* grad_e0, float* grad_filters, float* work, float* loss, void* stream);

/* WRMF, model/general_recommender/WRMF.py:51-61,69-85: one ALS half-step, every row of a CSR solved in one call.
 * For row r with CSR entries J(r) over the fixed table Y (fixed f32 [num_fixed, dim]):
 *   x_r = (Y^T Y + alpha * sum_{j in J(r)} y_j y_j^T + reg * I)^-1 (1 + alpha) sum_{j in J(r)} y_j
 * written to out f32 [num_rows, dim] (out must not alias fixed).  The user half passes the user-major CSR and the
 * item table, the item half the item-major CSR and the user table just written; an empty row gets x = 0.  Y^T Y is
 * summed over fixed slices of num_fixed, then in a fixed order, and made exactly symmetric; each row is factored by
 * Cholesky with one fixed summation order, so the result is bit-reproducible and independent of which other rows
 * are in the call.  row_order i32 [num_rows] (a permutation: the order rows are scheduled in, heaviest first), or
 * NULL for 0 .. num_rows - 1.  work f32 [nrc_wrmf_work_floats(max(num_fixed), dim)].  *not_spd (device i32) is set
 * to the number of rows whose matrix had a pivot that was not positive and finite; those rows are left unchanged
 * (impossible with reg > 0).  NRC_E_LIMIT when dim is outside [1, 128]; NRC_E_VALUE when alpha or reg is negative
 * or not finite (the reference's LU solve would still return a value there).  A rejected call writes nothing. */
int64_t nrc_wrmf_work_floats(int32_t num_rows_max, int32_t dim);
int nrc_wrmf_half_step(const float* fixed, int32_t num_fixed, const int64_t* indptr, const int32_t* indices,
                       const int32_t* row_order, int32_t num_rows, int32_t dim, float alpha, float reg, float* out,
                       float* work, int32_t* not_spd, void* stream);

/* ======================================================================================
 * Sequential recommenders over one recent item: FPMC and TransRec (model/sequential_recommender/), high_order = 1
 * ==================================================================================== */

/* Shared conventions.  One batch is (users, recent, items, third) i32 [batch] each, with `third` the negatives (i32,
 * pairwise = 1) or the labels (f32, pairwise = 0) -- the layout of TimeOrderPairwiseSampler / TimeOrderPointwiseSampler
 * (data/sampler.py:216-354).  Losses are learner.pairwise_loss / pointwise_loss (util/learner.py:17-41); the batch
 * loss is ADDED into *loss; row gradients are ADDED into dense accumulators (duplicate ids sum, as TF's IndexedSlices
 * de-duplication does) and every row that receives one gets `stamp` in its touched array (the rows adagrad, momentum
 * and rmsprop move).  NRC_E_LIMIT when dim is outside [1, 256]; NRC_E_VALUE with "please choose a suitable loss
 * function" for a loss the mode does not define.  A rejected call writes nothing. */

/* FPMC._create_inference / _create_loss, FPMC.py:61-84, tables UI [U, d], IU, IL, LI [I, d]:
 *   x(u, l, i) = <UI_u, IU_i> + <IL_i, LI_l>     (l = the recent item)
 *   pairwise   l(x_i - x_j) + reg * l2_loss(UI_u, IU_i, IL_i, LI_l, IU_j, IL_j)
 *   pointwise  l(z, x_i)    + reg * l2_loss(UI_u, IU_i, IL_i, LI_l)
 * touched_user <- users, touched_item <- items and negatives (IU and IL), touched_recent <- recent (LI). */
int nrc_fpmc_grad(const float* ui, const float* iu, const float* il, const float* li, int32_t dim,
                  const int32_t* users, const int32_t* recent, const int32_t* items, const void* third,
                  int64_t batch, int32_t pairwise, int32_t loss_kind, float reg, float* grad_ui,
                  float* grad_iu, float* grad_il, float* grad_li, int32_t* touched_user,
                  int32_t* touched_item, int32_t* touched_recent, int32_t stamp, float* loss, void* stream);

/* FPMC.train_model's batch loop, FPMC.py:106-131, over a device-built epoch of n samples: per batch nrc_fpmc_grad +
 * one TF-1.12 optimizer launch over UI, IU, IL and LI.  slot0 / slot1: HOST arrays of the four variables' slot
 * pointers in that order (NULL where the optimizer keeps no such slot); lr_t_host f32 [steps] (adam), hyper_host
 * as nrc_opt_apply_rows; step_loss f32 [steps] receives every batch's loss; stamps first_stamp .. + steps - 1. */
int nrc_fpmc_train_epoch(float* ui, float* iu, float* il, float* li, int32_t num_users, int32_t num_items,
                         int32_t dim, const int32_t* users, const int32_t* recent, const int32_t* items,
                         const void* third, int64_t n, int32_t batch_size, int32_t pairwise, int32_t loss_kind,
                         float reg, int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                         float* grad_ui, float* grad_iu, float* grad_il, float* grad_li,
                         int32_t* touched_user, int32_t* touched_item, int32_t* touched_recent,
                         float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                         void* stream);

/* FPMC.predict, FPMC.py:140-165: out f32 [rows, num_items], out[r, j] = <UI_u, IU_j> + <IL_j, LI_l> for
 * (u, l) = (users[r], recent[r]). */
int nrc_fpmc_scores(const float* ui, const float* iu, const float* il, const float* li, int32_t num_items,
                    int32_t dim, const int32_t* users, const int32_t* recent, int64_t rows, float* out,
                    void* stream);

/* Scratch of nrc_transrec_grad / nrc_transrec_train_epoch in floats: per-CTA partial sums of g's gradient and a
 * completion counter.  Zero-fill it once before its first use; every call leaves it ready for the next (calls that
 * share one work buffer must not run concurrently). */
int64_t nrc_transrec_work_floats(int32_t dim);

/* TransRec._create_inference / _create_loss, TransRec.py:66-91, variables P [U, d], Q [I, d], b [I], g [1, d]:
 *   x(u, l, i) = b_i - |(P_u + g) + Q_l - Q_i|^2          (squared)
 *   pairwise   l(x_i - x_j) + reg * l2_loss(P_u, Q_l, Q_j, Q_i, b_i, b_j, g)
 *   pointwise  l(z, x_i)    + reg * l2_loss(P_u, Q_l, Q_i, b_i, g)
 * g's reg term enters once per batch.  grad_global f32 [d] is a dense gradient: it is summed per CTA and then across
 * CTAs in one fixed order (no per-sample atomics) and added into grad_global.  touched_user <- users,
 * touched_item <- recent, items and negatives (Q), touched_bias <- items and negatives only (b). */
int nrc_transrec_grad(const float* user_table, const float* item_table, const float* item_bias,
                      const float* global, int32_t dim, const int32_t* users, const int32_t* recent,
                      const int32_t* items, const void* third, int64_t batch, int32_t pairwise,
                      int32_t loss_kind, float reg, float* grad_user, float* grad_item, float* grad_bias,
                      float* grad_global, int32_t* touched_user, int32_t* touched_item,
                      int32_t* touched_bias, int32_t stamp, float* work, float* loss, void* stream);

/* TransRec.train_model's batch loop, TransRec.py:110-147: per batch nrc_transrec_grad + one optimizer launch over P,
 * Q, b (IndexedSlices rules) and g (dense rules: Adam and RMSProp take the Apply* formulas).  slot0 / slot1: HOST
 * arrays of the four variables' slot pointers in the order P, Q, b, g; the rest as nrc_fpmc_train_epoch. */
int nrc_transrec_train_epoch(float* user_table, float* item_table, float* item_bias, float* global,
                             int32_t num_users, int32_t num_items, int32_t dim, const int32_t* users,
                             const int32_t* recent, const int32_t* items, const void* third, int64_t n,
                             int32_t batch_size, int32_t pairwise, int32_t loss_kind, float reg,
                             int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                             float* grad_user, float* grad_item, float* grad_bias, float* grad_global,
                             int32_t* touched_user, int32_t* touched_item, int32_t* touched_bias,
                             float* const* slot0, float* const* slot1, int32_t first_stamp, float* work,
                             float* step_loss, void* stream);

/* TransRec's prediction graph, TransRec.py:102-107: out f32 [rows, num_items],
 * out[r, j] = b_j - sqrt(sum_k (x_k - Q_jk)^2) with x = (P_u + g) + Q_l -- the distance, NOT squared.  The sum is
 * taken over the differences themselves, so x == Q_j scores exactly b_j. */
int nrc_transrec_scores(const float* user_table, const float* item_table, const float* item_bias,
                        const float* global, int32_t num_items, int32_t dim, const int32_t* users,
                        const int32_t* recent, int64_t rows, float* out, void* stream);

/* ======================================================================================
 * Sequential recommenders over a window of recent items: HRM and NPE (model/sequential_recommender/), pointwise
 * ==================================================================================== */

/* Shared conventions.  One batch is users, items i32 [batch], labels f32 [batch] and recent i32 [batch, window]: each
 * sample's window of the user's previous items, oldest first -- the layout of TimeOrderPointwiseSampler(high_order =
 * window) (data/sampler.py:42-68, 216-294).  The loss is learner.pointwise_loss (cross_entropy: the batch mean, square:
 * the batch sum); the batch loss is ADDED into *loss; row gradients are ADDED into dense accumulators and every row
 * that receives one gets `stamp` in its touched array, as for FPMC.  l2_loss counts every gathered row, window rows
 * included, so an id repeated in a window gets reg * row once per occurrence.  NRC_E_LIMIT when dim is outside
 * [1, 256] or window outside [1, 64]; NRC_E_VALUE with "please choose a suitable loss function" for a loss other than
 * cross_entropy / square.  A rejected call writes nothing.  The *_train_epoch entry points take slot0 / slot1, lr_t_host,
 * hyper_host, step_loss and the stamps as nrc_fpmc_train_epoch, with the slot arrays listing the model's variables in
 * the order given below.
 *
 * Predict: the window of user u is train_dict[u][len - window:] as Python evaluates it, so a user with len < window
 * train items has the shorter window seq[max(0, 2 len - window):].  The query entry points read it from a per-user
 * table recent i32 [num_users, window] (row u padded after its first recent_len[u] entries, recent_len[u] >= 1) and
 * pool over that length; scores are then nrc_mf_scores of the query rows against the item rows. */

/* HRM._create_inference / _create_loss, HRM.py:62-91, variables P [U, d] (user_embeddings), E [I, d]
 * (item_embeddings; window and target share it):
 *   s = pool_S(E[w_0], .., E[w_{window-1}]),  h = pool_P(P_u, s),  x = <h, E_i>
 *   l(z, x) + reg * l2_loss(P_u, E[w], E_i)
 * Pools are elementwise; session_agg / pre_agg = 1 takes the max, 0 the mean (the conf's "max" and anything else).
 * Gradients as TF: the mean passes grad / count, the max passes (1 / n) * grad to each of the n inputs equal to the
 * maximum (ties are split).  At window = 1 this is the reference's concat branch.  touched_user <- users,
 * touched_item <- window items and items (E). */
int nrc_hrm_grad(const float* user_table, const float* item_table, int32_t dim, int32_t window,
                 const int32_t* users, const int32_t* recent, const int32_t* items, const float* labels,
                 int64_t batch, int32_t pre_agg, int32_t session_agg, int32_t loss_kind, float reg,
                 float* grad_user, float* grad_item, int32_t* touched_user, int32_t* touched_item,
                 int32_t stamp, float* loss, void* stream);

/* HRM.train_model's batch loop, HRM.py:104-129: per batch nrc_hrm_grad + one optimizer launch over P and E. */
int nrc_hrm_train_epoch(float* user_table, float* item_table, int32_t num_users, int32_t num_items,
                        int32_t dim, int32_t window, const int32_t* users, const int32_t* recent,
                        const int32_t* items, const float* labels, int64_t n, int32_t batch_size,
                        int32_t pre_agg, int32_t session_agg, int32_t loss_kind, float reg,
                        int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                        float* grad_user, float* grad_item, int32_t* touched_user, int32_t* touched_item,
                        float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                        void* stream);

/* HRM.predict's query, HRM.py:135-163: out f32 [rows, dim], out[r] = h of user users[r] over its table window; the
 * scores of every item are nrc_mf_scores(out, E). */
int nrc_hrm_query(const float* user_table, const float* item_table, int32_t dim, int32_t window,
                  const int32_t* users, int64_t rows, const int32_t* recent, const int32_t* recent_len,
                  int32_t pre_agg, int32_t session_agg, float* out, void* stream);

/* NPE._create_inference / _create_loss, NPE.py:54-71, variables UI [U, d], IU [I, d], IL [I, d]:
 *   c = sum_l IL[w_l],  x = sum_k relu(UI_u)_k relu(IU_i)_k + relu(IU_i)_k relu(c)_k
 *   l(z, x) + reg * l2_loss(UI_u, IU_i, IL[w])
 * relu's gradient is 0 where its input is <= 0 (TF's ReluGrad).  touched_user <- users (UI), touched_item <- items
 * (IU), touched_recent <- window items (IL).  The epoch's slot arrays list UI, IU, IL. */
int nrc_npe_grad(const float* ui, const float* iu, const float* il, int32_t dim, int32_t window,
                 const int32_t* users, const int32_t* recent, const int32_t* items, const float* labels,
                 int64_t batch, int32_t loss_kind, float reg, float* grad_ui, float* grad_iu,
                 float* grad_il, int32_t* touched_user, int32_t* touched_item, int32_t* touched_recent,
                 int32_t stamp, float* loss, void* stream);

/* NPE.train_model's batch loop, NPE.py:84-108: per batch nrc_npe_grad + one optimizer launch over UI, IU and IL. */
int nrc_npe_train_epoch(float* ui, float* iu, float* il, int32_t num_users, int32_t num_items, int32_t dim,
                        int32_t window, const int32_t* users, const int32_t* recent, const int32_t* items,
                        const float* labels, int64_t n, int32_t batch_size, int32_t loss_kind, float reg,
                        int32_t opt_kind, const float* lr_t_host, const float* hyper_host, float* grad_ui,
                        float* grad_iu, float* grad_il, int32_t* touched_user, int32_t* touched_item,
                        int32_t* touched_recent, float* const* slot0, float* const* slot1,
                        int32_t first_stamp, float* step_loss, void* stream);

/* NPE.predict's query, NPE.py:114-142: out f32 [rows, dim], out[r] = relu(UI_u) + relu(c) for user users[r] over its
 * table window, and, when out_items is not NULL, out_items f32 [num_items, dim] = relu(IU).  The scores of every item
 * are nrc_mf_scores(out, out_items): sum_k relu(IU_j)_k (relu(UI_u)_k + relu(c)_k). */
int nrc_npe_query(const float* ui, const float* iu, const float* il, int32_t num_items, int32_t dim,
                  int32_t window, const int32_t* users, int64_t rows, const int32_t* recent,
                  const int32_t* recent_len, float* out, float* out_items, void* stream);

/* ======================================================================================
 * FPMCplus (model/sequential_recommender/FPMCplus.py): attention over a window of recent items, conditioned on the
 * candidate item, pairwise or pointwise
 * ==================================================================================== */

/* FPMCplus._attention_mlp / _create_inference / _create_loss, FPMCplus.py:53-119.  Variables UI [U, d], IU, IL, LI
 * [I, d], W [3d, weight_size] (rows [0, d) for the user, [d, 2d) for the item, [2d, 3d) for the window item), b and h
 * [weight_size].  For user u, window l_1..l_L and item i:
 *   e_k = <h, tanh([UI_u, IL_i, LI_{l_k}] W + b)>,  a_k = exp(e_k) / sum_k exp(e_k)   (no max shift)
 *   x   = <UI_u, IU_i> + <IL_i, sum_k a_k LI_{l_k}>
 *   pairwise   l(x_i - x_j) + reg_mf * l2_loss(UI_u, IU_i, IL_i, LI_w, IU_j, IL_j) + reg_w * l2_loss(W, h)
 *   pointwise  l(z, x_i)    + reg_mf * l2_loss(UI_u, IU_i, IL_i, LI_w)              (reg_w is not used)
 * The batch layout, losses, loss and row-gradient accumulation and touched rules are those of the HRM / NPE section
 * (recent i32 [batch, window]) with `third` as for FPMC: touched_user <- users (UI), touched_item <- items and
 * negatives (IU and IL), touched_recent <- window items (LI).  grad_w, grad_b and grad_h are dense gradients: every
 * sample's factors go to work and are summed over the batch in one fixed order (no atomics onto them), so they are
 * the same bits on every call with the same inputs.  The reg_w term of the loss counts once per batch.
 * NRC_E_LIMIT when dim is outside [1, 256], weight_size outside [1, 128], window outside [1, 64] or batch above
 * 65535 * 32; NRC_E_VALUE for a loss the mode does not define or a NULL table, gradient or work.  A rejected call
 * writes nothing. */

/* Scratch of nrc_fpmcplus_grad / nrc_fpmcplus_train_epoch in floats, for batches of up to batch_size samples:
 * completion counters, per-sample factors of the dense gradients and per-chunk partial sums.  Zero-fill it once
 * before its first use; every call leaves the counters ready for the next (calls that share one work buffer must not
 * run concurrently).  Negative NRC_E_* when an argument is out of range. */
int64_t nrc_fpmcplus_work_floats(int32_t dim, int32_t weight_size, int32_t window, int32_t batch_size);

int nrc_fpmcplus_grad(const float* ui, const float* iu, const float* il, const float* li, const float* w,
                      const float* b, const float* h, int32_t dim, int32_t weight_size, int32_t window,
                      const int32_t* users, const int32_t* recent, const int32_t* items, const void* third,
                      int64_t batch, int32_t pairwise, int32_t loss_kind, float reg_mf, float reg_w,
                      float* grad_ui, float* grad_iu, float* grad_il, float* grad_li, float* grad_w,
                      float* grad_b, float* grad_h, int32_t* touched_user, int32_t* touched_item,
                      int32_t* touched_recent, int32_t stamp, float* work, float* loss, void* stream);

/* FPMCplus.train_model's batch loop, FPMCplus.py:141-171: per batch nrc_fpmcplus_grad + one optimizer launch over
 * UI, IU, IL, LI (IndexedSlices rules) and W, b, h (dense rules).  slot0 / slot1: HOST arrays of the seven variables'
 * slot pointers in that order; the rest as nrc_fpmc_train_epoch. */
int nrc_fpmcplus_train_epoch(float* ui, float* iu, float* il, float* li, float* w, float* b, float* h,
                             int32_t num_users, int32_t num_items, int32_t dim, int32_t weight_size,
                             int32_t window, const int32_t* users, const int32_t* recent, const int32_t* items,
                             const void* third, int64_t n, int32_t batch_size, int32_t pairwise, int32_t loss_kind,
                             float reg_mf, float reg_w, int32_t opt_kind, const float* lr_t_host,
                             const float* hyper_host, float* grad_ui, float* grad_iu, float* grad_il,
                             float* grad_li, float* grad_w, float* grad_b, float* grad_h, int32_t* touched_user,
                             int32_t* touched_item, int32_t* touched_recent, float* const* slot0,
                             float* const* slot1, int32_t first_stamp, float* work, float* step_loss, void* stream);

/* Scratch of nrc_fpmcplus_scores in floats: the item-side projection IL W_I and the transposed IL and IU
 * (num_items * (weight_size + 2 dim)), and every row's UI_u W_U + b and window projections LI W_L
 * (rows * (window + 1) * weight_size).  No initialisation needed. */
int64_t nrc_fpmcplus_score_work_floats(int32_t num_items, int32_t dim, int32_t weight_size, int32_t window,
                                       int64_t rows);

/* FPMCplus.predict, FPMCplus.py:177-205: out f32 [rows, num_items], out[r, j] = x(users[r], window, j) over the user's
 * table window (recent / recent_len as for nrc_hrm_query; a window shorter than `window` takes the softmax over its
 * actual length).  Where sum_k exp(e_k) overflows, the score is NaN if some exp(e_k) overflowed and
 * <UI_u, IU_j> otherwise, as the reference's exp / sum gives it. */
int nrc_fpmcplus_scores(const float* ui, const float* iu, const float* il, const float* li, const float* w,
                        const float* b, const float* h, int32_t num_items, int32_t dim, int32_t weight_size,
                        int32_t window, const int32_t* users, int64_t rows, const int32_t* recent,
                        const int32_t* recent_len, float* work, float* out, void* stream);

/* Test hook of the FPMCplus kernels, as nrc_seq_last_routes: out i32[4 * 6], group k at out[6 * k].
 *   groups: [0] the per-sample gradient kernel, [1] the dense-gradient reduction (both also inside
 *   nrc_fpmcplus_train_epoch), [2] the projection pass of nrc_fpmcplus_scores, [3] its pair kernel.
 *   fields: +0 1 the pairwise form, 0 the pointwise one (gradient groups); +1 gridDim.x (CTAs; the reduction: element
 *   tiles of 256; the pair kernel: row groups); +2 gridDim.y (the reduction: chunks of 32 samples; the pair kernel:
 *   item tiles of 256); +3 1 when the grid was capped (the gradient kernel above 64 * SMs samples, the projection
 *   above 4096 * SMs elements), else 0; +4 the window L; +5 the pair kernel's rows per CTA (at most 8, fewer where
 *   their window rows would not fit in shared memory). */
int nrc_fpmcplus_last_routes(int32_t* out);

/* ======================================================================================
 * Caser (model/sequential_recommender/Caser.py): convolutions over the embeddings of the last L items
 * ==================================================================================== */

/* Caser._create_variable / build_graph, Caser.py:37-122.  Variables P [U, d] (user_embeddings), E [I, d]
 * (seq_item_embeddings; the pad id I reads a zero row), W2 [I, 2d] (item_embeddings), b2 [I] (item_biases) and the
 * dense block: every conv and FC weight in one flat f32 buffer, in TF's creation order and layouts,
 *   Kv [L, 1, 1, nv] (element l nv + f), bv [nv],
 *   for h = 1..L: Kh_h [h, d, 1, nh] (element (l d + k) nh + f), bh_h [nh],
 *   W1 [F, d] (element r d + c), b1 [d],           F = nv d + nh L.
 * One sample is users[b], seqs i32 [batch, L] (the window, oldest first), pos i32 [batch, T] and neg i32 [batch, N]
 * (N = neg_samples); with X the [L, d] image of the window:
 *   out_v[k nv + f] = sum_l X[l, k] Kv[l, f] + bv[f],  out_h[(h-1) nh + f] = max_t relu(conv of height h + bh_h[f])
 *   o = ([out_v, out_h] / keep) * mask (o = [out_v, out_h] when mask is NULL),  z = relu(o W1 + b1)
 *   x_j = <[z, P_u], W2[j]> + b2[j] over pos ++ neg
 *   loss = mean(-log(sigmoid(x_pos) + 1e-24)) + mean(-log(1 - sigmoid(x_neg) + 1e-24))   (means over this batch)
 * A target equal to the pad id I reads a zero row and a zero bias (x = 0): its loss term counts and it gets no
 * gradient.  Gradients as TF: the max passes grad / n to each of the n tied maxima, relu passes where its output is
 * > 0.  NRC_E_LIMIT when dim is outside [1, 256], seq_L outside [1, 16], nv or nh outside [1, 64], seq_T +
 * neg_samples above 64 or batch above 65535 * 32; NRC_E_VALUE when seq_T or neg_samples is below 1, keep is outside
 * (0, 1] or a table, gradient or work is NULL.  A rejected call writes nothing. */

/* Floats of the dense block (layout above); negative NRC_E_* when a size is out of range. */
int64_t nrc_caser_dense_floats(int32_t dim, int32_t seq_L, int32_t nv, int32_t nh);

/* Scratch of nrc_caser_grad / nrc_caser_train_epoch in floats, for batches of up to batch_size samples: completion
 * counters, each sample's layer inputs and output gradients, per-chunk partial sums of the dense gradient and the
 * step's dropout mask.  Zero-fill it once before its first use; every call leaves the counters ready for the next
 * (calls that share one work buffer must not run concurrently). */
int64_t nrc_caser_work_floats(int32_t dim, int32_t seq_L, int32_t nv, int32_t nh, int32_t batch_size);

/* Loss and gradients of one batch.  mask f32 [batch, F] (0 / 1) applies dropout with keep probability keep; NULL
 * means no dropout.  Row gradients are ADDED into grad_user [U, d], grad_seq [I, d] (window rows; pad ids get none),
 * grad_item [I, 2d] and grad_bias [I] (targets) with atomics; grad_dense [dense floats] is OVERWRITTEN with the
 * dense block's gradient, summed over the batch in one fixed order (the same bits on every call).  The batch's data
 * loss (without the l2 term) is ADDED into *loss when loss is not NULL. */
int nrc_caser_grad(const float* user_table, const float* seq_table, const float* item_table, const float* item_bias,
                   const float* dense, int32_t num_items, int32_t dim, int32_t seq_L, int32_t seq_T, int32_t nv,
                   int32_t nh, int32_t neg_samples, const int32_t* users, const int32_t* seqs, const int32_t* pos,
                   const int32_t* neg, int64_t batch, const float* mask, float keep, float* grad_user,
                   float* grad_seq, float* grad_item, float* grad_bias, float* grad_dense, float* work, float* loss,
                   void* stream);

/* Caser.train_model's batch loop, Caser.py:128-139, over an epoch already shuffled and sampled (users, seqs, pos,
 * neg as above, n samples).  Per batch s: the dropout mask nrc_dropout_mask(rows * F, keep, seed, epoch << 32 | s);
 * every table's gradient set to l2_reg * var (0 when l2_reg = 0); nrc_caser_grad; one Adam launch (hyper_host =
 * {lr, beta1, beta2, eps}, lr_t_host [steps]) over P, E, W2, b2 in the IndexedSlices form on every row and the
 * dense block in the dense form.  slot0 / slot1: HOST arrays of the five variables' m and v slots in that order.
 * step_loss f32 [steps] gets each batch's data loss. */
int nrc_caser_train_epoch(float* user_table, float* seq_table, float* item_table, float* item_bias, float* dense,
                          int32_t num_users, int32_t num_items, int32_t dim, int32_t seq_L, int32_t seq_T, int32_t nv,
                          int32_t nh, int32_t neg_samples, const int32_t* users, const int32_t* seqs,
                          const int32_t* pos, const int32_t* neg, int64_t n, int32_t batch_size, float keep,
                          float l2_reg, uint64_t seed, uint64_t epoch, const float* lr_t_host,
                          const float* hyper_host, float* grad_user, float* grad_seq, float* grad_item,
                          float* grad_bias, float* grad_dense, float* const* slot0, float* const* slot1, float* work,
                          float* step_loss, void* stream);

/* Caser.predict's user vectors, Caser.py:194-209: out f32 [rows, 2d] = [z, P_u] of user users[r] without dropout,
 * over its window windows[users[r]] (windows i32 [num_users, L]).  The scores of every item are
 * nrc_mf_scores(out, W2) -- the reference's all_logits, without b2. */
int nrc_caser_query(const float* user_table, const float* seq_table, const float* dense, int32_t num_items,
                    int32_t dim, int32_t seq_L, int32_t nv, int32_t nh, const int32_t* users, int64_t rows,
                    const int32_t* windows, float* out, void* stream);

/* Test hook of the Caser kernels, as nrc_seq_last_routes: out i32[4 * 6], group k at out[6 * k].
 *   groups: [0] the per-sample gradient kernel, [1] the dense-gradient reduction (both also inside
 *   nrc_caser_train_epoch), [2] the query kernel, [3] the per-step reg pass of nrc_caser_train_epoch.
 *   fields: +0 1 when the dense block was staged in shared memory (it fits with the kernel's buffers), 0 when it was
 *   read from global memory; +1 gridDim.x (CTAs; the reduction: element tiles of 256); +2 gridDim.y (the reduction:
 *   chunks of 32 samples); +3 1 when the grid was capped (the gradient and query kernels above 2 * SMs samples or
 *   rows, the reg pass above 4096 * SMs elements), else 0; +4 the window L; +5 1 when a dropout mask was applied. */
int nrc_caser_last_routes(int32_t* out);

/* ======================================================================================
 * FISM (model/general_recommender/FISM.py): a user is the sum of the item rows of its train history
 * ==================================================================================== */

/* FISM._create_variables / _create_inference / _create_loss, FISM.py:55-88.  Variables c1 [I, d], Q [I, d]
 * (embedding_Q) and b [I] (bias).  Histories are rows of a CSR (hist_ptr i64 [rows + 1], hist_idx i32); the
 * reference's pad id (a zero row) is not materialised.  Sample s is (rows[s], excl[s], num[s], items[s], third[s]):
 *   p = sum of c1[h] over h in hist_idx[hist_ptr[r] .. hist_ptr[r + 1]) with h != excl[s] (excl NULL or -1: none)
 *   x = powf(num[s], -alpha) * <p, Q[i]> + b[i]
 *   pointwise (third = labels f32):    l(z, x) + lambda * l2_loss(p) + gamma * l2_loss(Q[i])
 *   pairwise  (third = negatives i32): l(x - x_j) + lambda * l2_loss(p) + gamma * (l2_loss(Q[j]) + l2_loss(Q[i])),
 *     x_j = powf(num_neg[s], -alpha) * <p, Q[j]> + b[j] over the same history p.
 * l2_loss(t) = sum t^2 / 2.  Cross entropy is a batch mean, the other losses are sums.  Every history row h (once per
 * occurrence; once for both sides of a pair) takes dl/dp = g c Q[i] [- g c_j Q[j]] + lambda p.  NRC_E_LIMIT when dim
 * is outside [1, 256]; NRC_E_VALUE when num_items < 1, the loss does not suit the mode, batch < 0, alpha is not
 * finite, or a table, the CSR, the batch, num_neg (pairwise), a gradient or a stamp array is NULL.  A rejected call
 * writes nothing. */

/* Loss and row gradients of one batch.  Gradients are ADDED into grad_c1 [I, d], grad_q [I, d] and grad_bias [I] with
 * atomics; touched_c1[h] = stamp for every history row read, touched_item[i] (and [j]) = stamp for the targets (Q and
 * b share it).  The batch's loss, regularisers included, is ADDED into *loss when loss is not NULL. */
int nrc_fism_grad(const float* c1, const float* q, const float* bias, int32_t num_items, int32_t dim,
                  const int64_t* hist_ptr, const int32_t* hist_idx, const int32_t* rows, const int32_t* excl,
                  const int32_t* num, const int32_t* items, const void* third, const int32_t* num_neg, int64_t batch,
                  int32_t pairwise, int32_t loss_kind, float alpha, float lambda, float gamma, float* grad_c1,
                  float* grad_q, float* grad_bias, int32_t* touched_c1, int32_t* touched_item, int32_t stamp,
                  float* loss, void* stream);

/* FISM.train_model's batch loop, FISM.py:100-144, over an epoch already built and shuffled (n samples as above).  Per
 * batch s (stamp first_stamp + s): nrc_fism_grad, then one optimizer launch over c1, Q and b, all three in the
 * IndexedSlices form (touched rows for adagrad / rmsprop / momentum, Adam's sparse form on every row).  lr_t_host
 * [steps] is Adam's lr_t per step (ignored otherwise); hyper_host = {lr, beta1 | rho | momentum, beta2 | momentum,
 * eps}; slot0 / slot1: HOST arrays of the three variables' slots (NULL entries where the optimizer keeps none).
 * step_loss f32 [steps] gets each batch's loss. */
int nrc_fism_train_epoch(float* c1, float* q, float* bias, int32_t num_items, int32_t dim, const int64_t* hist_ptr,
                         const int32_t* hist_idx, const int32_t* rows, const int32_t* excl, const int32_t* num,
                         const int32_t* items, const void* third, const int32_t* num_neg, int64_t n,
                         int32_t batch_size, int32_t pairwise, int32_t loss_kind, float alpha, float lambda,
                         float gamma, int32_t opt_kind, const float* lr_t_host, const float* hyper_host,
                         float* grad_c1, float* grad_q, float* grad_bias, int32_t* touched_c1, int32_t* touched_item,
                         float* const* slot0, float* const* slot1, int32_t first_stamp, float* step_loss,
                         void* stream);

/* FISM.predict's user rows, FISM.py:154-180: out f32 [rows, d] = the sum of c1 over user users[r]'s whole history
 * row. */
int nrc_fism_query(const float* c1, int32_t num_items, int32_t dim, const int64_t* hist_ptr, const int32_t* hist_idx,
                   const int32_t* users, int64_t rows, float* out, void* stream);

/* Scores of every item: out f32 [rows, I], out[r, j] = powf(n, -alpha) * <query[r], Q[j]> + b[j] with n the length
 * of user users[r]'s history row (query from nrc_fism_query).  NRC_E_LIMIT also when I is above 65535 * 256. */
int nrc_fism_scores(const float* query, const float* q, const float* bias, int32_t num_items, int32_t dim, float alpha,
                    const int64_t* hist_ptr, const int32_t* users, int64_t rows, float* out, void* stream);

/* Test hook of the FISM kernels, as nrc_seq_last_routes: out i32[3 * 6], group k at out[6 * k].
 *   groups: [0] the gradient kernel (also inside nrc_fism_train_epoch), [1] the query kernel, [2] the score kernel.
 *   fields: +0 1 the pairwise form, 0 the pointwise one (gradient); +1 floats per lane load (4 when dim % 4 == 0,
 *   else 1); +2 lanes per history row (gradient and query: a power of two, 32 / lanes rows per warp load); +3
 *   gridDim.x (CTAs of 64 threads, a warp per sample or row; the score kernel: groups of 8 rows); +4 gridDim.y (the
 *   score kernel: item tiles of 256); +5 1 when the grid was capped above 64 * SMs samples or rows, else 0. */
int nrc_fism_last_routes(int32_t* out);

/* ======================================================================================
 * ItemKNN (model/general_recommender/ItemKNN.py): item-item similarity, top-K neighbours, ratings = R . W
 * ==================================================================================== */

/* Bytes of the `work` buffer nrc_itemknn_similarity needs for num_items items: 0 while a CTA's row of num_items x 8 B
 * fits in shared memory (220 KB), else one such row per CTA of the capped grid (4 * SMs CTAs). */
int64_t nrc_itemknn_work_bytes(int32_t num_items);

/* Compute_Similarity(...).compute_similarity(), ItemKNN.py:11-547, as ItemKNN.build_graph calls it (normalize=True).
 * X [num_users, num_items] comes twice, as a CSR (csr_ptr i64 [U + 1], csr_idx i32, csr_val f64) and as its CSC
 * (csc_ptr i64 [I + 1], csc_idx i32 users ascending, csc_val f64), values already centred (adjusted: minus the row
 * average; pearson: minus the column average) or made binary (tanimoto, dice, tversky) by the caller.  va, vb f64 [I]
 * are the per-item vectors the reference computes with numpy: NORM va = vb = sqrt(sum of squares), or (asymmetric)
 * va = s^(2 alpha), vb = s^(2 (1 - alpha)); TANIMOTO / DICE / TVERSKY va = the sum of squares (vb unused);
 * EUCLIDEAN va = the sum of squares, vb = its sqrt.  For column c, w_k = sum over users ascending of X[u,k] X[u,c],
 * w_c = 0, then in the reference's order with correctly rounded f64 operations:
 *   NORM       w * (1 / (va_c * vb_k + shrink + 1e-6))
 *   TANIMOTO   w * (1 / (va_c + va_k - w + shrink + 1e-6))
 *   DICE       w * (1 / (va_c + va_k + shrink + 1e-6))
 *   TVERSKY    w * (1 / (w + (va_c - w) * tversky_alpha + (va_k - w) * tversky_beta + shrink + 1e-6))
 *   EUCLIDEAN  1 / (sqrt((va_k + va_c - 2 w) / (vb_c * vb_k)) + shrink + 1e-9), and 0 at k = c.
 * The top min(neighbor, I) values of the column by (value descending, row ascending, NaN last) are selected and those
 * != 0.0 kept (the row-ascending tie rule is the one deviation: numpy's introselect orders ties its own way).  W is
 * written in padded CSC form, slot-major: column c holds counts[c] entries, entry t at [t * I + c] of rows i32 and vals
 * f32 (the float64 value rounded once), rows ascending; both arrays hold min(neighbor, I) * I entries.  integral != 0
 * vouches that every value is an integer; with gram_bound (an upper bound on every |w_k|) at most 2^31 - 1 the dots
 * are summed as int32, otherwise as f64.  work: nrc_itemknn_work_bytes(num_items) bytes (NULL when 0).  NRC_E_VALUE
 * when num_users < 0, num_items < 1, kind is outside [0, 4], neighbor < 1, shrink or a tversky coefficient is NaN,
 * an array is NULL or work is too small.  A rejected call writes nothing. */
int nrc_itemknn_similarity(int32_t num_users, int32_t num_items, const int64_t* csr_ptr, const int32_t* csr_idx,
                           const double* csr_val, const int64_t* csc_ptr, const int32_t* csc_idx,
                           const double* csc_val, int32_t kind, const double* va, const double* vb, double shrink,
                           double tversky_alpha, double tversky_beta, int32_t neighbor, int32_t integral,
                           double gram_bound, void* work, int64_t work_bytes, int32_t* counts, int32_t* rows,
                           float* vals, void* stream);

/* ItemKNN.predict(users, None), ItemKNN.py:573 and 583-585: out f32 [batch, I], out[b, j] = the f64 sum over column
 * j's entries k of W (ascending) with X[u, k] stored of X[u, k] * W[k, j], u = users[b], rounded once to f32: the
 * order in which scipy's csr_matmat forms train.tocsc().dot(W).  The CSR is X's (the un-centred train values); W is
 * nrc_itemknn_similarity's output at the same neighbor.  NRC_E_LIMIT when num_items is above 220 KB / 8 B * 32;
 * NRC_E_VALUE when num_items < 1, neighbor < 1, batch < 0 or an array is NULL. */
int nrc_itemknn_scores(int32_t num_items, const int64_t* csr_ptr, const int32_t* csr_idx, const double* csr_val,
                       int32_t neighbor, const int32_t* counts, const int32_t* rows, const float* vals,
                       const int32_t* users, int64_t batch, float* out, void* stream);

/* Test hook of the ItemKNN kernels, as nrc_seq_last_routes: out i32[2 * 6], group k at out[6 * k].
 *   groups: [0] the similarity kernel, [1] the score kernel.
 *   fields: +0 0 the int32 accumulator, 1 the f64 one (similarity); +1 the tier: 0 the CTA's row in shared memory,
 *   1 an int32 accumulator in shared memory and the keys in global work, 2 both in global work (similarity); +2
 *   gridDim.x (a CTA per column / per user, grid-strided); +3 1 when that grid was capped (above 4 * SMs columns,
 *   8 * SMs users), else 0; +4 min(neighbor, I); +5 dynamic shared memory in bytes. */
int nrc_itemknn_last_routes(int32_t* out);

/* Test hook of the sequential kernels (it reports and changes nothing; every route is chosen by the shape).
 * nrc_seq_last_routes: HOST bookkeeping of the most recent launch of each kernel group, written when a call launches
 * (a call that returns before launching, for a failed check, an empty batch or no rows, leaves it as it was); one
 * record per process.  out i32[9 * 7], group k at out[7 * k]; -1 = no such launch yet, or a field the group does not
 * decide.
 *   groups: [0] nrc_fpmc_grad, [1] nrc_transrec_grad, [2] nrc_hrm_grad, [3] nrc_npe_grad (each also inside its
 *   *_train_epoch); [4] nrc_fpmc_scores, [5] nrc_transrec_scores; [6] nrc_hrm_query, [7] the query rows of
 *   nrc_npe_query; [8] the relu pass of nrc_npe_query over the items (out_items).
 *   fields of a group:
 *   +0 1 the pairwise form, 0 the pointwise one (gradient kernels);
 *   +1 HRM: 1 when the window pool (session_agg) is the max, 0 the mean;
 *   +2 HRM: 1 when the user pool (pre_agg) is the max, 0 the mean;
 *   +3 CTAs launched (gridDim.x); score kernels: groups of 8 rows;
 *   +4 score kernels: item tiles of 256 (gridDim.y);
 *   +5 1 when the grid was capped, so a warp or thread takes more than one sample or element: FPMC, HRM and NPE
 *      gradients above 64 * SMs samples, TransRec's above 1024 (128 CTAs), the query and relu passes above
 *      4096 * SMs elements; else 0;
 *   +6 the window L (HRM and NPE). */
int nrc_seq_last_routes(int32_t* out);

/* Test hook of the data-side kernels (APR's normaliser, the row gather, SBPR, the CSR / split / row-id builders), the
 * negative samplers and LightGCN's BPR gradient (it reports and changes nothing; every route is chosen by the shape).
 * nrc_extras_last_routes: HOST bookkeeping of the most recent launch of each group, written just before the launch (a
 * call that returns before launching, for a failed check or an empty input, leaves it as it was); one record per
 * process.  out i32[10 * 6], group k at out[6 * k]; -1 = no such launch yet, or a field the group does not decide.
 *   groups: [0] nrc_l2_normalize_rows, [1] nrc_gather_rows_i32, [2] nrc_sbpr_epoch_build, [3] nrc_sbpr_grad (also
 *   inside nrc_sbpr_train_epoch), [4] nrc_csr_from_coo, [5] nrc_split_interactions, [6] nrc_csr_row_ids,
 *   [7] nrc_sample_negatives, [8] nrc_batch_randint_choice, [9] nrc_lightgcn_bpr_grad (also inside
 *   nrc_lightgcn_train_epoch).
 *   fields of a group:
 *   +0 CTAs launched (gridDim.x); [4] and [5]: of the per-entry passes (count, scatter), 0 when there are no entries;
 *   +1 1 when that grid was capped, so a thread or warp takes more than one item, else 0: the per-row kernels ([0],
 *      [3], [6], [9]) above 64 * SMs rows or samples, the per-element kernels ([1], [2], the entry passes of [4] and
 *      [5]) above 2048 * SMs elements, the samplers' per-element kernels above 4096 * SMs; the no-replace form of [8]
 *      (one thread per row) is never capped;
 *   +2 [4], [5]: CTAs of the per-row passes (sort and compaction, split ranks), a warp per row;
 *   +3 [4], [5]: 1 when the per-row grid was capped (above 64 * SMs rows), else 0;
 *   +4 [4], [5]: 1024-row chunks of the single-CTA row-pointer scan, ceil(rows / 1024);
 *   +5 [8]: 1 the replace form, 0 the no-replace form. */
int nrc_extras_last_routes(int32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* NEUREC_B200_H */
