/*
 * include/difacto_b200.h -- the drop-in boundary of difacto-b200.
 *
 * A C-ABI (plain pointers and sizes, no C++/torch types) over the H100-native
 * FM-SGD engine.  Each entry point replaces one interface of the reference
 * (dmlc/difacto @ 78e3562; paths below are relative to that tree).  The reference
 * itself has no C ABI on this path -- it has four C++ abstract classes
 * (include/difacto/{loss,updater,store,learner}.h); INTEGRATION.md shows the
 * adapter classes a maintainer adds there to bind these symbols.
 *
 * Conventions
 *  - every function returns 0 on success or a negative dfb_status; the message is
 *    available from dfb_last_error(h).  Nothing aborts the process (the reference
 *    CHECK()s -> abort(), Makefile:13 -DDMLC_LOG_FATAL_THROW=0; the C++ adapter maps a
 *    non-zero code back to LOG(FATAL)).
 *  - a handle owns one CUDA device, one compute stream and one copy stream.  It is
 *    thread-compatible: at most one call in flight per handle (the reference's Loss is
 *    not re-entrant either: fm_loss.h:202-203 member state).
 *  - "host" pointers are ordinary host memory (pinned memory from dfb_host_alloc makes
 *    the copies asynchronous); "dev" pointers are device memory on the handle's device.
 *  - feature keys are the reference's *reversed* feature ids (ReverseBytes,
 *    include/difacto/base.h:39-51), sorted ascending and unique, exactly what
 *    Localizer::Compact emits (src/data/localizer.cc:36-49).
 *  - all floating point is fp32 (real_t, include/difacto/base.h:16).
 */
#ifndef DIFACTO_B200_H_
#define DIFACTO_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dfb_engine* dfb_handle;

typedef enum {
  DFB_OK = 0,
  DFB_ERR_INVALID = -1,   /* bad argument / a CHECK of the reference would have fired */
  DFB_ERR_CUDA = -2,      /* CUDA runtime error */
  DFB_ERR_CAPACITY = -3,  /* key table or V-row pool exhausted */
  DFB_ERR_PARAM = -4,     /* parameter missing / out of range (dmlc::ParamError in the reference) */
  DFB_ERR_NCCL = -5,
  DFB_ERR_TIMEOUT = -6    /* a rank of the sharded store did not show up within shard_timeout_ms */
} dfb_status;

/* value types of Store::Push / Pull: include/difacto/store.h:33-35 */
enum { DFB_FEA_COUNT = 1, DFB_WEIGHT = 2, DFB_GRADIENT = 3 };

/* sgd::Progress, src/sgd/sgd_utils.h:40-45 (+ device-side counters) */
typedef struct {
  float loss;      /* sum_i log(1+exp(-y_i pred_i))            loss.h:57-66            */
  float penalty;   /* l1|w| + .5 l2 w^2 + .5 V_l2 V^2 (pulled)  sgd_learner.cc:249-273  */
  float auc;       /* AUC * nrows                               bin_class_metric.h:35-56 */
  float nnz_w;     /* unused by the SGD learner (kept for layout compatibility)          */
  float nrows;
  /* extras (not in the reference) */
  uint64_t new_keys;    /* keys inserted by this step                 */
  uint64_t new_vrows;   /* V rows allocated (InitV) by this step      */
} dfb_progress;

/* ---------------------------------------------------------------------------------
 * life cycle.  Replaces SGDUpdater::Init (src/sgd/sgd_updater.cc:9-11) + FMLoss::Init
 * (src/loss/fm_loss.h:37-39) + Store::Init.  Consumes the reference's SGDUpdaterParam
 * keys with the same names, defaults and ranges (src/sgd/sgd_param.h:66-107):
 *   l1 l2 V_l2 lr lr_beta V_lr V_lr_beta V_init_scale V_dim V_threshold seed
 * plus engine-only keys (unknown to the reference, ignored by it with a warning):
 *   device (0)            CUDA device ordinal
 *   table_capacity (1<<20) number of distinct keys this shard can hold at first
 *   V_capacity (=table_capacity) number of keys with an allocated V row at first
 *   table_capacity_max (=table_capacity)  the key capacity may grow to this, in [table_capacity, 2^30]
 *   V_capacity_max (=V_capacity when given, else table_capacity_max)  the V-row capacity may grow to this
 *                         Before every call that can insert keys (training and feature-count steps, dfb_pull,
 *                         dfb_push_*, dfb_dev_feacnt / _pull_rows* / _push_rows, restore) the engine grows the table
 *                         and the V-row pool when the keys it knows of plus an upper bound of that call's insertions
 *                         (nnz of a raw batch, nkeys, n, a snapshot's counts) could exceed them, up to the maxima,
 *                         without waiting for the device.  Capacities stay below about twice the keys plus the bounds
 *                         of the steps in flight.  A growth that cannot get memory keeps the current capacities; a
 *                         call reports DFB_ERR_CAPACITY exactly when it overflows them.  With both maxima at their
 *                         defaults nothing grows.  The fused sharded store refuses an engine that can grow unless
 *                         shard_growth = 1.
 *   shard_growth (0)      0 | 1: 1 lets an engine that can grow (a maximum above its capacity) be a rank of the fused
 *                         sharded store (dfb_shard_init).  Before a training or feature-count step inserts, the owner
 *                         counts on the device the keys every worker's segment brings it (one 1-thread kernel on its
 *                         lookup stream) and grows to max(2 x current, the counts it knows + the keys received in the
 *                         steps in flight), capped at the maxima.  The host waits for that count only when the worst
 *                         case (nranks x seg_keys per step in flight) does not fit -- so a rank waits on every training
 *                         step until its headroom reaches nranks x seg_keys.  The wait covers every worker's phase 0 of
 *                         the step, and the poller in front of it times out after shard_timeout_ms.  A
 *                         rehash runs on the owner stream after the previous step's update, and that step's lookup
 *                         waits for it.  Results are bit-identical to pre-sized ranks; DFB_ERR_CAPACITY comes in the
 *                         same step and rank as on ranks pre-sized to the maxima.  Validation and predict steps never
 *                         grow.  An engine whose capacities equal its maxima launches exactly what a fixed one does.
 *   compute_auc (1)       evaluate AUC on device each step (sgd_learner.cc:150-153)
 *   scatter (sorted)      sorted = gradient reduced per key through a stable radix-sorted CSC view of
 *                         the batch, fused with the FTRL/AdaGrad step (no atomics, bit-reproducible,
 *                         row order per key like SpMM::TransTimes); atomic = fp32 red.global scatter
 *                         into dense gradient rows followed by a separate update kernel
 *   overlap_auc (1)       run the AUC kernels on an auxiliary stream, overlapped with the update
 *   l2_hints (1)          per-access L2 eviction policies: the gather's V rows evict_first, the per-nnz {w, row
 *                         index} view evict_last when it fits in L2; when a step's table rows exceed L2, the fused
 *                         update keeps the per-row p*XV / p evict_last, streams the V rows evict_first and drops
 *                         p*XV / p from L2 afterwards
 *   id_bits (0)           > 0: feature ids are < 2^id_bits; fixes the bit range the GPU localizer's radix sort
 *                         visits.  The range is rounded up to whole nibbles: ids below 2^(4*ceil(id_bits/4)) are
 *                         accepted and sorted correctly.  0: the range is learned from the first raw batch (one
 *                         8-byte sync) and verified on the device afterwards; it widens to a wider batch for the
 *                         batches localized after that batch's key mask is read back (without waiting; at the
 *                         latest after dfb_sync).  The synchronous dfb_train_step_raw of an engine without id_bits
 *                         measures every batch.
 *                         A raw batch with an id outside the range is DROPPED: it changes nothing (table, V rows,
 *                         AdaGrad state, the InitV random stream), adds nothing to any Progress field, and the read
 *                         of its Progress (dfb_train_step_raw, dfb_wait_step, dfb_read_progress) returns
 *                         DFB_ERR_INVALID once, with a message naming the range.  dfb_localize ignores id_bits.
 *   shard_timeout_ms (20000)  how long a rank of the sharded store waits for a peer
 *   hot_split (256)       a key with more occurrences in a minibatch than this has its gradient pre-reduced in
 *                         chunks by separate warps, then finished in chunk order (0: one warp per key)
 *   long_row_nnz (1024)   an example with at least this many nonzeros is walked by a whole CTA in the forward
 *                         kernel, its chunks added in a fixed order (0: one warp per example whatever its length)
 *   force_generic (0)     1 = use the any-V_dim kernels even where a specialised one exists (tests).  Specialised
 *                         kernels exist for 0 <= V_dim <= 128 (the atomic scatter: V_dim in {8,16,32,64,128})
 *   score_only (0)        1 = a scoring-only engine: it loads a model (dfb_restore*, any snapshot, with or without aux
 *                         data, any M parts -> this shard) and scores it (dfb_predict_raw_*).  Its V rows hold V
 *                         alone -- stride dfb_row_stride elements instead of twice that, no AdaGrad accumulators -- so
 *                         the row pool takes half the memory (V_capacity / V_capacity_max count rows as before, and
 *                         a restore grows the engine up to the maxima).  has_aux reads 0.  Also allowed:
 *                         dfb_table_stats, dfb_row_bytes, dfb_id_range_get/set, dfb_sync, dfb_prefetch_raw, the
 *                         Progress reads (dfb_wait_step, dfb_read_progress), dfb_evaluate / dfb_auc, the timing
 *                         calls, dfb_destroy.  It may be a scoring rank of the fused sharded store (dfb_shard_init;
 *                         its predict steps, see there).  Every call that trains, counts features, validates, reads
 *                         or writes rows, saves or prunes returns DFB_ERR_INVALID with a message naming score_only
 *                         and changes nothing: dfb_train_step*, dfb_train_step_raw*, dfb_push_feacnt, dfb_pull,
 *                         dfb_push_grad, dfb_predict, dfb_calc_grad, dfb_read_entries, dfb_dev_*, dfb_snapshot*,
 *                         dfb_prune, dfb_shard_step_*, dfb_shard_begin_dev / _async.  Needs 0 <= V_dim <= 128 and
 *                         force_generic = 0 (DFB_ERR_PARAM
 *                         otherwise): the predict step of other configurations is the validation step.
 *                         The fp32 scoring engine's predictions and Progress are bit-identical to the training
 *                         engine's predict step on the same model.
 *   V_storage (fp32)      fp32 | bf16: the element type of a scoring-only engine's V rows.  bf16 halves the rows
 *                         again (2 bytes per element): restore rounds every V value to the nearest bf16, ties to
 *                         even (NaN and Inf as __float2bfloat16_rn defines them), the forward widens the elements
 *                         back to fp32 (exact) and accumulates in fp32 in the fp32 kernels' order, so its outputs
 *                         are bit-identical to an fp32 scoring engine's on a model whose V values were rounded so
 *                         beforehand.  w stays fp32.  bf16 without score_only = 1 is DFB_ERR_PARAM.
 * Keys that are neither are returned through dfb_unknown_kwarg, mirroring the
 * "return the unconsumed kwargs" convention (updater.h:34, main.cc:25-31).
 * ------------------------------------------------------------------------------- */
int dfb_create(const char* const* keys, const char* const* vals, int n, dfb_handle* out);
int dfb_destroy(dfb_handle h);
const char* dfb_last_error(dfb_handle h);   /* h may be NULL: error of the failed dfb_create */
int dfb_num_unknown_kwargs(dfb_handle h);
int dfb_unknown_kwarg(dfb_handle h, int i, const char** key, const char** val);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
uint64_t dfb_launch_count(dfb_handle h);
/* number of keys / V rows currently stored, and the current (grown) key and V-row capacities */
int dfb_table_stats(dfb_handle h, uint64_t* n_keys, uint64_t* n_vrows, uint64_t* capacity,
                    uint64_t* v_capacity);
/* the bytes one V row takes in the row pool -- dfb_row_stride elements times 8 ([V|cg] of a training engine), 4
 * (score_only, fp32) or 2 (score_only, V_storage = bf16) -- and n_vrows times that (either may be NULL) */
int dfb_row_bytes(dfb_handle h, uint64_t* bytes_per_row, uint64_t* bytes_in_use);
/* calls that grew the table or the V-row pool so far, and how often a sharded step's growth decision waited for the
 * device (shard_growth = 1: the worst case did not fit); either may be NULL */
int dfb_growth_stats(dfb_handle h, uint64_t* growths, uint64_t* host_waits);

/* pinned host memory so that H2D/D2H copies are asynchronous DMA */
int dfb_host_alloc(void** ptr, size_t bytes);
int dfb_host_free(void* ptr);

/* ---------------------------------------------------------------------------------
 * (A) API-faithful path: host buffers in, host buffers out; one call = one reference
 * call.  Used by the adapter classes GpuStore/GpuSGDUpdater/GpuFMLoss (INTEGRATION.md).
 * ------------------------------------------------------------------------------- */

/* Store::Push(keys, kFeaCount, cnt)  store_local.h:24-34 -> SGDUpdater::Update
 * sgd_updater.cc:62-73: fea_cnt += cnt; allocate V when w!=0 && fea_cnt>V_threshold. */
int dfb_push_feacnt(dfb_handle h, const uint64_t* keys, size_t n, const float* cnt);

/* Store::Pull(keys, kWeight, &vals, &lens)  store_local.h:36-44 -> SGDUpdater::Get
 * sgd_updater.cc:32-56.  vals_out (capacity vals_cap floats, n*(1+V_dim) always suffices)
 * receives the ragged [w_i, V_i...] rows; lens_out[n] receives 1 or 1+V_dim;
 * *nlens = 0 when V_dim == 0 (sgd_updater.cc:40), n otherwise. */
int dfb_pull(dfb_handle h, const uint64_t* keys, size_t n, float* vals_out, size_t vals_cap,
             int* lens_out, size_t* nvals, size_t* nlens);

/* Store::Push(keys, kGradient, grads, lens) -> SGDUpdater::Update sgd_updater.cc:74-101:
 * FTRL on w (UpdateW :104-127), AdaGrad on V (UpdateV :129-138), lazy InitV (:140-147).
 * nlens == 0 means w-only (lens.empty()). */
int dfb_push_grad(dfb_handle h, const uint64_t* keys, size_t n, const float* grads,
                  size_t nvals, const int* lens, size_t nlens);

/* FMLoss::Predict  src/loss/fm_loss.h:67-119.  CSR<u32> data (dmlc::RowBlock<unsigned>:
 * offset[nrows+1] of size_t, index, optional value), weights in the pulled ragged layout
 * with w_pos/V_pos (-1 = absent; both NULL = direct indexing, the V_dim==0 path).
 * pred[nrows] is ACCUMULATED into, as in the reference (caller zero-fills). */
int dfb_predict(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index,
                const float* value_or_null, const float* weights, size_t nweights,
                const int* w_pos, const int* V_pos, size_t npos, float* pred);

/* FMLoss::CalcGrad  src/loss/fm_loss.h:148-199.  grad[nweights] (same ragged layout as
 * weights) is ACCUMULATED into.  Unlike the reference it does not depend on member state
 * left behind by Predict (XV_ is recomputed on device). */
int dfb_calc_grad(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index,
                  const float* value_or_null, const float* label, const float* weights,
                  size_t nweights, const int* w_pos, const int* V_pos, size_t npos,
                  const float* pred, float* grad);

/* Loss::Evaluate  include/difacto/loss.h:57-66 */
int dfb_evaluate(dfb_handle h, const float* label, const float* pred, size_t n, float* objv);

/* BinClassMetric::AUC  src/loss/bin_class_metric.h:35-56 (returns AUC * n; ties keep row order) */
int dfb_auc(dfb_handle h, const float* label, const float* pred, size_t n, float* auc_times_n);

/* ---------------------------------------------------------------------------------
 * (B) fused device-resident step: replaces the whole pull_callback of
 * SGDLearner::IterateData (src/sgd/sgd_learner.cc:138-177 + the kFeaCount push :214-217):
 *   [fea_cnt push] -> Pull -> GetPos -> Predict -> Evaluate -> penalty -> AUC ->
 *   [CalcGrad -> Push(kGradient)]
 * on a batch already localized by Localizer::Compact (CSR<u32> + sorted unique reversed
 * keys [+ counts]).  The table never leaves HBM; the host sees only dfb_progress.
 * cnt_or_null != NULL reproduces the epoch-0 feature-count push; is_train == 0 is a
 * validation batch (no CalcGrad/Push, sgd_learner.cc:158-171).
 * pred_out_or_null receives the nrows clamped predictions if not NULL.
 * ------------------------------------------------------------------------------- */
int dfb_train_step(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index,
                   const float* value_or_null, const float* label, const uint64_t* keys,
                   size_t nkeys, const float* cnt_or_null, int is_train, dfb_progress* out,
                   float* pred_out_or_null);

/* same, but every array is already resident in device memory on the handle's device and
 * the call only enqueues work on the handle's stream (no host synchronisation);
 * dfb_sync() / dfb_read_progress() collect the result. */
int dfb_train_step_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset,
                       const uint32_t* d_index, const float* d_value_or_null,
                       const float* d_label, const uint64_t* d_keys, size_t nkeys,
                       const float* d_cnt_or_null, int is_train);
int dfb_sync(dfb_handle h);
/* blocks until enqueued steps are done; returns the Progress ACCUMULATED since the last
 * read (the reference merges per-batch Progress by addition, sgd_utils.h:66-71) */
int dfb_read_progress(dfb_handle h, dfb_progress* out);

/* pipelined host-buffer variant: enqueue H2D (from pinned memory: truly asynchronous)
 * + the step, double-buffered so that the copy of batch t+1 overlaps the compute of
 * batch t (the reference keeps <=2 batches in flight, sgd_learner.cc:220-223). */
int dfb_train_step_async(dfb_handle h, size_t nrows, const uint64_t* offset,
                         const uint32_t* index, const float* value_or_null, const float* label,
                         const uint64_t* keys, size_t nkeys, const float* cnt_or_null,
                         int is_train);

/* ---------------------------------------------------------------------------------
 * raw (un-localized) minibatches: Localizer::Compact on the device (SURVEY.md 8f rank 1).
 * dfb_localize is Localizer(max_index).Compact (src/data/localizer.h:41-51, localizer.cc:11-103)
 * for any input (it measures the id range of every call: neither id_bits nor the learned range apply)
 * with host buffers in and out, bit-exact: index_out[nnz] = rank of every nnz's key, keys_out =
 * ascending unique ReverseBytes(id % max_index), cnt_out = occurrence counts (may be NULL).
 * dfb_train_step_raw* take the CSR<uint64> block the reader produced (BatchReader::Value) and run
 * Localizer(-1).Compact + [kFeaCount push when push_cnt] + the fused step; the CSC view the
 * gradient kernel needs falls out of the same radix sort.
 * ------------------------------------------------------------------------------- */
int dfb_localize(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* index,
                 uint64_t max_index, uint32_t* index_out, uint64_t* keys_out, float* cnt_out,
                 size_t* nkeys);
int dfb_train_step_raw(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                       const float* value_or_null, const float* label, int push_cnt, int is_train,
                       dfb_progress* out, float* pred_out_or_null);
int dfb_train_step_raw_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                             const float* value_or_null, const float* label, int push_cnt,
                             int is_train);
/* optional double-buffering hint: start the H2D copy of the batch the NEXT dfb_train_step_raw_async call
 * (or dfb_predict_raw_async / sharded step) will be given (same pointers, label included; it may be NULL for a
 * predict step), so that the copy overlaps the step submitted before it */
int dfb_prefetch_raw(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                     const float* value_or_null, const float* label);
int dfb_train_step_raw_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset,
                           const uint64_t* d_ids, const float* d_value_or_null, const float* d_label,
                           int push_cnt, int is_train);

/* predict steps on raw ids: the forward pass of a frozen model.  A predict step writes nothing of the model (table,
 * V rows, AdaGrad state, InitV stream) and runs neither the localizer, the key lookup nor the penalty: for
 * 0 <= V_dim <= 128 (and force_generic = 0) it is one forward launch whose kernels look each nonzero's id up in the
 * table themselves; other configurations run the validation step (dfb_train_step_raw with is_train = 0) minus its
 * penalty.  The predictions are bit-identical to those of that validation step.  Progress: loss and AUC (0 without
 * labels) and nrows; penalty, new_keys and new_vrows are 0.  id_bits > 0 keeps its meaning: a batch with an id at or
 * above 2^(4*ceil(id_bits/4)) is dropped (predictions 0, nothing in Progress, DFB_ERR_INVALID once on its read);
 * with id_bits = 0 every id is scored.
 *   dfb_predict_raw_async  host buffers, staged through the double-buffered input sets (dfb_prefetch_raw applies);
 *                          the copy of the nrows predictions into pred_out_or_null is enqueued at the end of the step:
 *                          pinned memory keeps it asynchronous, and it must stay valid until the step is collected
 *                          (dfb_wait_step / dfb_read_progress / dfb_sync).  Takes its place in the Progress ring of the
 *                          other async steps, and sees the updates of the training steps enqueued before it.
 *   dfb_predict_raw_dev    device buffers, enqueue only (the Progress accumulates as for dfb_train_step_raw_dev);
 *                          d_pred_out_or_null receives the predictions in stream order.
 * An engine that is a rank of the sharded store (dfb_shard_init) refuses both: DFB_ERR_INVALID.
 * These are the steps a score_only = 1 engine runs: on fp32 rows the same kernels at the V-only row stride, on bf16
 * rows (V_storage = bf16) instantiations of them that differ in the row load alone. */
int dfb_predict_raw_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                          const float* value_or_null, const float* label_or_null, float* pred_out_or_null);
int dfb_predict_raw_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                        const float* d_value_or_null, const float* d_label_or_null, float* d_pred_out_or_null);

/* blocks until the OLDEST not yet collected dfb_train_step_async step has finished and
 * returns that step's Progress (each async step snapshots its Progress into a pinned ring,
 * so collecting step t does not drain step t+1 from the pipeline).  Up to 8 steps may be outstanding;
 * beyond that the oldest snapshots are folded into the sum dfb_read_progress returns. */
int dfb_wait_step(dfb_handle h, dfb_progress* out);

/* per-stage device timing with CUDA events on the stream each stage runs on (bench.py's roofline):
 * stage 0 = key lookup + pull, 1 = FM forward kernel, 2 = AUC, 3 = CSC sort of the batch,
 * 4 = per-key gradient reduce + FTRL/AdaGrad update (+ InitV pass), 5 = GPU localizer (raw batches);
 * sharded store: 6 = worker: slice the batch + scatter to the owners, 7 = owner: lookup + partial interaction
 * sums of all workers' rows, 8 = worker: reduce the partials (pred / loss / p, p*XV back), 9 = owner: the
 * workers' updates (incl. waiting for their p*XV).
 * dfb_profile_read returns the accumulated milliseconds and launch counts of the DFB_NUM_STAGES
 * stages and resets them.  While profiling, AUC runs on the main stream (otherwise it overlaps
 * the update on an auxiliary stream).
 * dfb_time_mark(h, 0) / (h, 1) bracket a region with CUDA events that cover ALL streams of the handle
 * (mark 1 joins them); dfb_time_elapsed_ms synchronises and returns the device time between the marks. */
#define DFB_NUM_STAGES 10
int dfb_time_mark(dfb_handle h, int which);
int dfb_time_elapsed_ms(dfb_handle h, float* ms);
int dfb_profile(dfb_handle h, int enable);
int dfb_profile_read(dfb_handle h, double* stage_ms, uint64_t* stage_count);

/* ---------------------------------------------------------------------------------
 * model inspection (tests, checkpointing): read entries of the table.
 * scal_out[n][4] = {fea_cnt, w, sqrt_g, z} (SGDEntry, sgd_updater.h:19-29),
 * has_V_out[n] in {-1 absent, 0 no V, 1 V}; V_out/cg_out [n][V_dim] (may be NULL).
 * ------------------------------------------------------------------------------- */
int dfb_read_entries(dfb_handle h, const uint64_t* keys, size_t n, float* scal_out,
                     int* has_V_out, float* V_out, float* cg_out);
/* checkpoint = Updater::Save / Updater::Load (include/difacto/updater.h:40-47; TODO stubs in the
 * reference's SGDUpdater, sgd_updater.h:44-50, so the byte format is this library's).  Format v1, little-endian:
 *   header (40 bytes) { char magic[8] = "DFB200\0\1"; u32 version = 1; i32 V_dim; u64 n_keys; u64 n_vrows;
 *                       u32 seed (the InitV rand_r state); u32 has_aux }
 *   n_keys records in strictly ascending (reversed) key order:
 *     { u64 key; f32 fea_cnt; f32 w; [f32 sqrt_g; f32 z;] i32 has_V (0/1); has_V: f32 V[V_dim] [f32 cg[V_dim]] }
 *   the bracketed fields only with save_aux.  A snapshot without aux data restores a model that can predict but
 *   not train ("no aux data", sgd_updater.cc:75).
 * Streaming: dfb_snapshot_write sorts and packs the records on the device and hands the stream to write_fn in
 * pieces of at most chunk_bytes (0 = 64 MiB; at least 40); host memory is two pinned chunks and an 8 MB
 * histogram, device workspace is allocated for the call (about 4 x chunk_bytes of records, more when the keys
 * that share their top 20 bits need more) and released at its end.  dfb_restore_read pulls the stream from
 * read_fn in chunks of at most chunk_bytes (0 = 64 MiB), validates it on the host (magic, version, V_dim, has_V,
 * ascending keys, truncation, the header's counts) and unpacks it on the device.  Both wait for every stream of
 * the handle first: they run between steps, never while steps are in flight.
 * Re-sharding: the stream is part `part` of `nparts` (a num_gpus = nparts run's rank `part`, or 0 of 1); the engine
 * is shard `shard` of `nshards` and keeps the keys with dfb_key_owner(key, nshards) == shard.  A key outside the
 * part's own ps-lite range is DFB_ERR_INVALID (parts miscounted or mixed up).  Several calls merge several parts
 * into one engine; a key restored twice is DFB_ERR_INVALID.  V rows are appended in stream order.
 * Seed and aux: the InitV state comes from the header of the first stream restored into an empty table, so an
 * nparts == nshards restore gives every rank its own part's stream, exactly as it was saved; after a re-shard
 * (nparts != nshards) each rank continues the InitV stream of the lowest part it read (a convention: the reference
 * has no checkpoint to compare with).  has_aux is the AND over the streams restored.
 * Errors: a failed dfb_restore_read (bad stream, capacity, read_fn error) leaves an EMPTY table behind -- the
 * message says the table was cleared -- so that the caller can retry.  dfb_snapshot_write changes nothing, also
 * when write_fn fails.
 * dfb_snapshot / dfb_restore are the same over one memory buffer (dfb_snapshot_size bytes); dfb_restore needs an
 * empty table (refused without clearing anything otherwise).
 * A score_only = 1 engine restores the same streams into V-only rows (the records' cg and, for the engine's has_aux,
 * their aux data are skipped; V_storage = bf16 rounds V to nearest even) and reports has_aux 0; dfb_snapshot_size,
 * dfb_snapshot, dfb_snapshot_write and dfb_snapshot_begin are refused on it (DFB_ERR_INVALID): it no longer holds
 * what the format stores. */
typedef int (*dfb_write_fn)(void* ctx, const void* buf, size_t bytes);   /* 0 = ok */
typedef size_t (*dfb_read_fn)(void* ctx, void* buf, size_t cap);       /* bytes read, 0 = end, (size_t)-1 = error */
int dfb_snapshot_write(dfb_handle h, int save_aux, size_t chunk_bytes, dfb_write_fn write_fn, void* ctx);
int dfb_restore_read(dfb_handle h, dfb_read_fn read_fn, void* ctx, uint32_t part, uint32_t nparts, uint32_t shard,
                     uint32_t nshards, size_t chunk_bytes, int* has_aux_out);
int dfb_snapshot_size(dfb_handle h, int save_aux, size_t* bytes);
int dfb_snapshot(dfb_handle h, int save_aux, void* buf, size_t bytes);
int dfb_restore(dfb_handle h, const void* buf, size_t bytes, int* has_aux_out);
/* checkpoint while training continues.  dfb_snapshot_begin waits for every stream of the handle, as
 * dfb_snapshot_write does, copies the table's slots, its V rows and its counts and InitV state into fresh device
 * memory, waits for the copy and returns: the handle is free to train from then on.  The copy takes the table's
 * slots (32 bytes each) plus n_vrows V rows (dfb_row_stride floats each); when
 * that memory cannot be had it returns DFB_ERR_CAPACITY and changes nothing.  The copy comes from the device's default
 * memory pool and goes back to the device after its release.  On an engine that can still grow (table_capacity_max /
 * V_capacity_max above the current capacities) begin also returns DFB_ERR_CAPACITY, changing nothing, when the free
 * device memory would not cover the copy and that growth besides, so that a copy never takes the memory a later
 * rehash or row-pool mapping needs.  At most one frozen snapshot per handle
 * (a second begin is DFB_ERR_INVALID); it does not follow the handle's later growth (a rehash frees the old table,
 * not the copy).
 * dfb_frozen_write streams the copy through the same writer as dfb_snapshot_write, byte for byte what
 * dfb_snapshot_write would have written at the moment of begin, on a low-priority stream of its own with its own
 * device workspace, pinned chunks and error message (dfb_frozen_error).  It touches nothing of the handle, so it may
 * run on another host thread while the handle's owning thread keeps enqueuing steps.  It may be called more than
 * once; a write_fn error fails that call only.
 * dfb_frozen_release frees the copy (stream-ordered after the writer's work); call it on the handle's owning thread
 * once no dfb_frozen_write is running.  dfb_destroy releases a copy left behind. */
typedef struct dfb_frozen_s* dfb_frozen;
int dfb_snapshot_begin(dfb_handle h, int save_aux, dfb_frozen* out);
int dfb_frozen_write(dfb_frozen f, size_t chunk_bytes, dfb_write_fn write_fn, void* ctx);
const char* dfb_frozen_error(dfb_frozen f);
int dfb_frozen_release(dfb_frozen f);
/* state of the InitV random stream (SGDUpdaterParam::seed after the rand_r calls so far) */
int dfb_rng_state(dfb_handle h, uint32_t* seed);
/* the id range an engine with id_bits = 0 has learned from its raw batches (see id_bits), as a bit count: the ids
 * seen so far lie below 2^bits (exactly: the byte-reversed keys have no bit set below 64 - bits).  get waits for the
 * key masks still in flight and returns 0 when nothing has been learned yet; set gives an engine that has learned
 * nothing that range (1 <= bits <= 64), and it then sorts, widens and drops batches exactly as the engine that
 * learned it.  Together with a snapshot this is all the engine state a resumed run needs: the InitV state travels in
 * the snapshot header, and the sharded store's per-step stamps (entry pad, in [1, 2^24)) never equal the 0 every
 * restored entry carries. */
int dfb_id_range_get(dfb_handle h, int* bits);
int dfb_id_range_set(dfb_handle h, int bits);
/* Drops every entry with w == 0, no V row and fea_cnt <= max_count; returns how many entries it dropped.
 * Such an entry adds nothing to any prediction: the forward reads a key the table lacks exactly so (w = 0, no V row).
 * Predictions are therefore unchanged; a dropped key that comes back starts its FTRL state (fea_cnt, sqrt_g, z) from
 * zero.  Entries with a V row are never dropped: V rows, n_vrows and the InitV state do not change, and every kept
 * entry keeps its 32 bytes (its pad too).  n_keys drops by *n_dropped; the capacities stay, and the freed slots take
 * new keys.  Like dfb_snapshot_begin it waits for every stream of the handle and runs between steps: during a sharded
 * step (dfb_shard_begin_* .. dfb_shard_phase(4)) it is DFB_ERR_INVALID.  A frozen snapshot is a copy and is not
 * changed.  The table is rebuilt in place with a workspace of 32 bytes per kept entry, taken before the table is
 * touched: DFB_ERR_CAPACITY when it cannot be had, and then nothing has changed.  Refused on a score_only = 1
 * engine (DFB_ERR_INVALID): prune the model where it is trained. */
int dfb_prune(dfb_handle h, float max_count, uint64_t* n_dropped);

/* ---------------------------------------------------------------------------------
 * key-range sharding (multi-GPU).  ps-lite Postoffice::GetServerKeyRanges
 * (ps-lite/src/postoffice.cc:127-136) + KVWorker::DefaultSlicer (kv_app.h:406-460):
 * shard i owns reversed keys in [UINT64_MAX/S*i, UINT64_MAX/S*(i+1)); the tail above
 * UINT64_MAX/S*S is clamped into shard S-1.  Because keys are sorted, every shard's keys
 * are one contiguous segment: bounds_out[S+1] are the segment boundaries.
 * ------------------------------------------------------------------------------- */
uint32_t dfb_key_owner(uint64_t reversed_key, uint32_t num_shards);
int dfb_shard_bounds(const uint64_t* sorted_keys, size_t n, uint32_t num_shards,
                     size_t* bounds_out);

/* device-side building blocks for the sharded store (all pointers are device memory, work is
 * enqueued on the handle's stream; difacto_b200/sharded.py holds the protocol):
 *   dfb_dev_feacnt     owner: Update(kFeaCount) for the keys one worker sent
 *   dfb_dev_pull_rows  owner side of Pull: keys -> dense rows {w[n], has_V[n] (-1/1), V[n][ks]}
 *                      packed for the all-to-all (SGDUpdater::Get, dense instead of ragged)
 *   dfb_dev_fm_step    worker: Predict/Evaluate/penalty/AUC/CalcGrad on the pulled dense buffers;
 *                      writes the COMPLETE gradient rows gw[n], gV[n][ks] (incl. the -V*XXp term
 *                      computed with the pulled V, fm_loss.h:181-188) for the keys with has_V >= 0
 *   dfb_dev_push_rows  owner side of Push(kGradient): FTRL/AdaGrad from the rows one worker sent;
 *                      has_V is the worker's pull-time view (lens[i] > 1, sgd_updater.cc:91)   */
int dfb_row_stride(dfb_handle h);  /* ks: V_dim rounded up to a multiple of 4 floats */
int dfb_dev_feacnt(dfb_handle h, const uint64_t* d_keys, size_t n, const float* d_cnt);
int dfb_dev_pull_rows(dfb_handle h, const uint64_t* d_keys, size_t n, float* d_w_out,
                      int* d_hasv_out, float* d_V_out);
int dfb_dev_fm_step(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset,
                    const uint32_t* d_index, const float* d_value_or_null, const float* d_label,
                    size_t nkeys, const float* d_w, const int* d_hasv, const float* d_V,
                    int is_train, float* d_gw_out, float* d_gV_out);
int dfb_dev_push_rows(dfb_handle h, const uint64_t* d_keys, size_t n, const float* d_gw,
                      const int* d_hasv, const float* d_gV);
/* NVLink peer-store variants (one process per GPU, buffers shared through CUDA IPC):
 *   dfb_peer_alloc / dfb_peer_open   a device buffer + its 64-byte cudaIpcMemHandle_t; a peer process opens
 *                                    the handle and gets a pointer its kernels can store through
 *   dfb_dev_pull_rows_peer           owner: gather {w, has_V, V} for one requester's key segment and store the
 *                                    rows straight into the requester's pull buffer (fused gather + transfer);
 *                                    the pull-time has_V flags are also kept locally for the later push
 *   dfb_dev_fm_step_peer             worker: as dfb_dev_fm_step (training), but the gradient rows of key
 *                                    segment s (keys [seg_bounds[s], seg_bounds[s+1])) are stored straight into
 *                                    owner s's receive buffer (peer_gw[s], peer_gV[s] = where the segment starts) */
int dfb_peer_alloc(dfb_handle h, size_t bytes, void** ptr, unsigned char* handle64);
int dfb_peer_open(dfb_handle h, const unsigned char* handle64, void** ptr);
int dfb_peer_close(dfb_handle h, void* ptr);
int dfb_peer_free(dfb_handle h, void* ptr);
int dfb_dev_pull_rows_peer(dfb_handle h, const uint64_t* d_keys, size_t n, float* peer_w_out,
                           int* peer_hasv_out, float* peer_V_out, int* d_hasv_local_out);
int dfb_dev_fm_step_peer(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset,
                         const uint32_t* d_index, const float* d_value_or_null, const float* d_label,
                         size_t nkeys, const float* d_w, const int* d_hasv, const float* d_V, int nseg,
                         const size_t* seg_bounds, float* const* peer_gw, float* const* peer_gV,
                         int first_seg /* segment to start with (own rank): staggers peer traffic */);

/* ---------------------------------------------------------------------------------
 * The NVLink-sharded store behind the C-ABI: N engines (one per GPU; one process per GPU with CUDA IPC, or
 * all of them in one process with peer access) form one model, rank r owning the r-th range of the reversed key space exactly
 * like ps-lite's servers (postoffice.cc:127-136).  It replaces, for this path, the worker/server exchange of
 * the reference (SGDLearner's workers calling Store::Pull / Push on KVWorker, the servers running
 * SGDUpdater; src/sgd/sgd_learner.cc:78-89,138-177, ps-lite/include/ps/kv_app.h:406-460).
 * Every rank calls dfb_shard_step_* once per minibatch, COLLECTIVELY (same number of calls, same push_cnt /
 * is_train; a rank that ran out of data passes nrows = 0).  A step is bulk-synchronous like the
 * all_to_all protocol of dfb_dev_*: every worker's forward sees the model after all updates of the previous
 * step; an owner applies the workers' gradients as separate Updates in rank order (sgd_updater.cc:74-98),
 * each taken at the V the worker "pulled" at step start.  What crosses NVLink is not the k-wide rows but the
 * per-example partial interaction sums (see csrc/kernels_shard.cu); nothing is synchronised with the host.
 *   dfb_shard_init     allocate this rank's mailbox (capacity: max_rows x max_nnz per minibatch; seg_keys /
 *                      seg_nnz = capacity of one (worker, owner) key segment, 0 = twice the even share).  Needs
 *                      0 <= V_dim <= 128, scatter=sorted and force_generic=0 (DFB_ERR_INVALID otherwise).
 *                      A score_only = 1 engine becomes a scoring rank of a store of nranks >= 2 (nranks = 1:
 *                      DFB_ERR_INVALID naming score_only; alone it scores with dfb_predict_raw_*): its shard is
 *                      V-only rows (fp32 or bf16), it allocates none of the training steps' workspaces (pull-time V rows of shared keys, InitV
 *                      flags, hot-key pre-reduction), and it may grow (up to its maxima, in dfb_restore* only: its
 *                      steps never insert) without shard_growth.  It runs dfb_shard_predict_async and
 *                      dfb_shard_begin_predict_async; dfb_shard_step_* and dfb_shard_begin_dev / _async (training,
 *                      feature counts or validation) return DFB_ERR_INVALID naming score_only before anything is
 *                      enqueued.  Its mailbox is a training rank's (same mailbox_bytes), so one store may mix training
 *                      and scoring ranks for predict steps; fp32 scoring ranks predict bit-identically to training
 *                      ranks holding the same model
 *   dfb_shard_export   the mailbox pointer (peers in the same process) and its CUDA IPC handle (peers in
 *                      other processes open it with dfb_peer_open)
 *   dfb_shard_connect  the peers' mailbox pointers, indexed by rank (entry [rank] is ignored)
 *   dfb_shard_step_dev   one minibatch of raw CSR<uint64> already on the device (enqueue only)
 *   dfb_shard_step_async the same from host buffers (pinned: asynchronous), double-buffered like
 *                        dfb_train_step_raw_async; dfb_prefetch_raw may stage the next batch early
 * Results: dfb_wait_step (per step) / dfb_read_progress (accumulated), as for the other async entry points;
 * Progress is this rank's own minibatch (loss, AUC, penalty of the weights it used).  DFB_ERR_TIMEOUT: a peer
 * did not reach the step within shard_timeout_ms (kwarg, default 20000).
 * A dropped batch: a rank's batch with an id outside the id range (id_bits, or the range learned from earlier
 * batches), or with a key segment larger than seg_keys / seg_nnz, changes nothing on any owner and adds nothing
 * to that rank's loss, penalty, AUC or row count (its new_keys / new_vrows count what this rank inserted as an
 * owner, for the other workers); the other ranks step as if it held an empty batch.  It is reported once,
 * by that rank's read of its own step: DFB_ERR_INVALID (range) or DFB_ERR_CAPACITY (segment).
 * ------------------------------------------------------------------------------- */
int dfb_shard_init(dfb_handle h, int rank, int nranks, size_t max_rows, size_t max_nnz, size_t seg_keys,
                   size_t seg_nnz, size_t* mailbox_bytes_out);
int dfb_shard_export(dfb_handle h, void** mailbox_ptr, unsigned char* handle64);
int dfb_shard_connect(dfb_handle h, void* const* peer_mailbox);
int dfb_shard_step_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                       const float* d_value_or_null, const float* d_label, int push_cnt, int is_train);
int dfb_shard_step_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                         const float* value_or_null, const float* label, int push_cnt, int is_train);
/* The same step split into its five enqueue phases (0 worker: localize + scatter the slices, 1 owner: lookup +
 * partial sums, 2 worker: reduce + p*XV back, 3 owner: updates, 4 finish): dfb_shard_step_* is begin + phases
 * 0..4.  Needed whenever ONE host thread drives several ranks (the C++ CLI's num_gpus = N, the one-device tests):
 * the phases must be interleaved -- phase p of every rank before phase p+1 of any -- so that every device-side
 * wait refers to work that is already enqueued.  With monolithic steps, rank 0's pollers would wait for work
 * the thread has not enqueued yet; on one device that never completes, and on several devices it deadlocks as
 * soon as a driver call in between blocks (a lazily loaded kernel synchronises its context).  Ranks that have a
 * host thread or a process of their own just call dfb_shard_step_*.
 * On the wire every minibatch is valued (x = 1 for a binary one), so the workers of a step may hold any mix of
 * binary, valued and empty minibatches. */
int dfb_shard_begin_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                          const float* value_or_null, const float* label, int push_cnt, int is_train);
int dfb_shard_begin_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                        const float* d_value_or_null, const float* d_label, int push_cnt, int is_train);
int dfb_shard_phase(dfb_handle h, int phase);
/* A predict step of the sharded store: the step with is_train = 0 and push_cnt = 0, except that the owners evaluate no
 * penalty (Progress: loss, AUC, nrows; 0 loss and AUC without labels) and that pred_out_or_null receives this rank's
 * nrows predictions at the end of the step (pinned memory keeps the copy asynchronous; valid until the step is
 * collected).  Collective like every step: every rank calls a predict form in the same step.  The predictions equal
 * those of one engine holding the whole model up to the order of the owners' partial sums.
 * dfb_shard_begin_predict_async is followed by dfb_shard_phase(0..4), as dfb_shard_begin_async. */
int dfb_shard_predict_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                            const float* value_or_null, const float* label_or_null, float* pred_out_or_null);
int dfb_shard_begin_predict_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                                  const float* value_or_null, const float* label_or_null, float* pred_out_or_null);
int dfb_shard_info(dfb_handle h, int* rank, int* nranks, size_t* seg_keys, size_t* seg_nnz, uint64_t* steps);

/* the CUDA stream (cudaStream_t) the handle enqueues on, for event interop with torch */
void* dfb_stream(dfb_handle h);

#ifdef __cplusplus
}
#endif
#endif  /* DIFACTO_B200_H_ */
