// difacto_b200/csrc/engine_internal.cuh -- the engine object behind a dfb_handle and the host-side helpers
// shared by engine.cu (C-ABI, single-GPU step) and shard.cu (the NVLink-sharded store).
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <utility>
#include <vector>

#include "../../include/difacto_b200.h"
#include "dfb_internal.cuh"

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  template <typename T> T* as() const { return static_cast<T*>(p); }
};

struct ShardState;   // shard.cu
struct dfb_frozen_s; // checkpoint.cu

struct dfb_engine {
  dfb::Params prm;
  int device = 0;
  int compute_auc = 1;
  int force_generic = 0;
  int scatter_sorted = 1;   // 1: atomic-free sorted reduction (deterministic); 0: red.global atomics
  int overlap_auc = 1;      // run the AUC kernels on the auxiliary stream, concurrently with the update
  int has_aux = 1;          // false after restoring a snapshot saved without aux data (sgd_updater.h:88)
  int score_only = 0;       // kwarg score_only: V-only rows (tab.vonly), has_aux 0; restore, raw predict and reads only
  int restored_parts = 0;   // snapshot streams merged into the table since it was last empty (checkpoint.cu)
  int l2_hints = 1;         // per-load L2 eviction policies in the gather kernels
  int id_bits = 0;          // > 0: feature ids are < 2^id_bits (fixes the radix-sort bit range of the GPU localizer)
  int loc_begin_bit = -1;   // auto mode: lowest significant bit of the reversed keys seen so far (sticky)
  long long shard_timeout_ms = 20000;
  int long_row_nnz = 1024;  // rows with at least this many nonzeros are walked by a whole CTA (k_fm_long); 0: off
  int hot_split = 256;      // occurrence lists longer than this are pre-reduced in chunks by separate warps (0: off)
  cudaStream_t stream = nullptr, copy_stream = nullptr, aux_stream = nullptr;
  cudaEvent_t ev_fm_done = nullptr, ev_auc_done = nullptr;
  dfb::Table tab;
  std::string err;
  std::vector<std::pair<std::string, std::string>> unknown;
  uint64_t launches = 0;

  // workspaces (grown on demand)
  DevBuf u_wv;
  DevBuf keys, cnt, slot, u_w, u_vrow, flags, pos, lens, cub, gw, gxxp, gV, pred, vals;
  DevBuf auc_k, auc_v, auc_tmp;
  DevBuf pxv, p_row, occ, occ_sorted, lidx_sorted, col_start, col_end;
  DevBuf hot_map, hot_info, hot_part, hot_ps, hot_cnt;
  DevBuf l_rkeys, l_skeys, l_pay, l_spay, l_tmp;
  // outputs of the GPU localizer, double-buffered: the localizer of batch t+1 runs on loc_stream
  // while the step of batch t (which reads set t) runs on the main stream
  struct LocSet {
    DevBuf keys, lidx, cnt, occ_sorted, col_start, col_end;
    DevBuf scal;                          // {OR of all reversed keys, number of unique keys} (u64 x 2)
    cudaEvent_t done = nullptr, consumed = nullptr;
    bool used = false;
    const unsigned long long* dU() const { return scal.as<unsigned long long>() + 1; }
  } loc[2];
  uint64_t loc_seq = 0;
  cudaStream_t loc_stream = nullptr;
  unsigned long long* h_scal = nullptr;   // pinned: {or_all, n_unique} of a synchronous localize
  unsigned long long* h_or = nullptr;     // pinned ring [2]: or_all of earlier asynchronous localizes
  cudaEvent_t ev_or[2] = {nullptr, nullptr};
  bool or_pending[2] = {false, false};
  uint64_t or_seq = 0;
  DevBuf a_off, a_idx, a_val, a_lab, a_w, a_wpos, a_vpos, a_pred, a_grad;
  DevBuf scal, hasv, rV, rcg, nvals;
  DevBuf id_ok;                         // u64: 0 when the raw-id predict step's batch fails its id_bits range check
  // double-buffered inputs of the pipelined step
  struct InSet {
    DevBuf off, idx, val, lab, keys, cnt, ids;
    cudaEvent_t copied = nullptr, consumed = nullptr;
    const void* pre_ids = nullptr;     // host batch already staged by dfb_prefetch_raw (identity check)
    const void* pre_lab = nullptr;
    size_t pre_nrows = 0, pre_nnz = 0;
    bool prefetched(const void* ids, const void* lab, size_t nrows, size_t nnz) const {
      return pre_ids == ids && ids && pre_lab == lab && pre_nrows == nrows && pre_nnz == nnz;
    }
  } in[2];
  uint64_t seq = 0;
  // per-step Progress snapshots of the pipelined path (pinned ring + completion events)
  static constexpr int kRing = 8;
  dfb::DevProgress* h_ring = nullptr;
  cudaEvent_t ring_done[kRing] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  uint64_t submitted = 0, collected = 0;
  dfb::DevProgress backlog;             // snapshots folded in when the ring was full
  // optional per-stage CUDA-event timing (bench.py's roofline numbers)
  // 0 lookup+pull, 1 fm, 2 auc, 3 csc sort, 4 update(+initv), 5 GPU localizer (raw batches),
  // sharded store: 6 worker slice+scatter, 7 owner lookup+partial sums, 8 worker reduce, 9 owner updates
  static constexpr int kStages = DFB_NUM_STAGES;
  static constexpr int kProfRing = 32;
  int profile = 0;
  std::vector<cudaEvent_t> pev;          // [kProfRing][kStages][2]
  std::vector<char> pev_used;            // [kProfRing][kStages]
  uint64_t prof_steps = 0;
  double stage_ms[kStages] = {};
  uint64_t stage_n[kStages] = {};
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr, ev_join = nullptr;   // dfb_time_mark
  dfb::DevProgress* h_prog = nullptr;   // pinned
  unsigned long long* h_nvals = nullptr;  // pinned
  ShardState* shard = nullptr;          // the NVLink-sharded store this engine is a rank of (shard.cu)
  dfb_frozen_s* frozen = nullptr;       // the snapshot dfb_snapshot_begin froze, until dfb_frozen_release

  // capacity growth up to table_capacity_max / V_capacity_max (growth.cu)
  struct Growth {
    uint64_t tab_max = 0, v_max = 0;
    bool on = false;                    // a maximum lies above its initial capacity
    cudaMemPool_t pool = nullptr;       // the table's stream-ordered allocations (release threshold 0)
    // the V-row pool: address space reserved for v_max rows, physical memory mapped at its start
    unsigned long long vbase = 0;
    size_t vreserved = 0, vmapped = 0, gran = 0;
    std::vector<std::pair<unsigned long long, size_t>> vchunks;   // {allocation handle, bytes}, in address order
    // the last table counts the host knows, and the insertion bounds enqueued since: each inserting call enqueues a
    // copy of {n_keys, n_vrows} as they are before it into a pinned ring, read once its event has completed
    static constexpr int kRing = 8;
    unsigned long long* h_st = nullptr;             // pinned [kRing][2]
    cudaEvent_t ev[kRing] = {};
    uint64_t at_k[kRing] = {}, at_v[kRing] = {};    // the bound totals when the copy was enqueued
    uint64_t head = 0, seq = 0;                     // ring entries [head, seq) are in flight
    uint64_t known_k = 0, known_v = 0, known_at_k = 0, known_at_v = 0, total_k = 0, total_v = 0;
    // sharded steps (shard_growth = 1): each one adds its worst case to the totals and is made exact once k_shard_count
    // has stored the keys its owner received.  calls numbers the bounds added, so that a correction reaches exactly
    // the copies whose totals include the corrected bound.
    uint64_t calls = 0, at_call[kRing] = {}, known_at_call = 0;
    unsigned long long* h_rcv = nullptr;            // pinned, mapped [kRing]: the received keys of one sharded step
    unsigned long long* d_rcv = nullptr;            // its device address
    cudaEvent_t rev[kRing] = {};
    uint64_t r_call[kRing] = {}, r_worst[kRing] = {};
    bool r_v[kRing] = {};                           // the step's bound was added to the V rows' total too
    uint64_t rhead = 0, rseq = 0;                   // entries [rhead, rseq) are not yet exact
    // calls that grew the table or the pool; host waits for a sharded step's count (dfb_growth_stats)
    uint64_t n_growths = 0, n_waits = 0;
  } grow;
  int shard_growth = 0;     // kwarg shard_growth: a growing engine may be a rank of the fused sharded store

  // true when a step runs the specialised sorted kernels: the 16-byte-lane forward (0 <= V_dim <= 128) and,
  // when it trains, the atomic-free sorted gradient reduction
  bool sorted_path(bool is_train = true) const {
    return !force_generic && dfb::fm_fast_supported(prm.V_dim) && (!is_train || scatter_sorted);
  }
  int fail(int code, const std::string& msg) { err = msg; return code; }
  // at the top of every entry point that trains, counts features, validates, reads or writes rows, saves or prunes: a
  // scoring-only engine holds neither the AdaGrad half of a row nor, with bf16 rows, the V values a snapshot stores
  int refuse_score_only(const char* call) {
    return fail(DFB_ERR_INVALID, std::string(call) + " is not available on a score_only = 1 engine (it restores a "
                                 "model and scores with dfb_predict_raw_*, or as a rank of the sharded store with "
                                 "dfb_shard_*predict_async)");
  }
  int cuda_fail(cudaError_t e, const char* what) {
    err = std::string(what) + ": " + cudaGetErrorString(e);
    return DFB_ERR_CUDA;
  }
  // grow a workspace; frees/reallocs only after the streams that may still read it have drained
  int ensure(DevBuf& b, size_t bytes);
};

#define DFB_CUDA(h, call)                                                  \
  do {                                                                     \
    cudaError_t _e = (call);                                               \
    if (_e != cudaSuccess) return (h)->cuda_fail(_e, #call);               \
  } while (0)
#define DFB_NOT_SCORE_ONLY(h, call)                                \
  do {                                                             \
    if ((h)->score_only) return (h)->refuse_score_only(call);      \
  } while (0)
#define DFB_TRY(expr)              \
  do {                             \
    int _rc = (expr);              \
    if (_rc != 0) return _rc;      \
  } while (0)

// CUDA-event pair around one stage of a step (only while dfb_profile is on), on the stream the stage runs on
struct StageTimer {
  dfb_engine* h; int st; cudaStream_t s; cudaEvent_t* e = nullptr;
  StageTimer(dfb_engine* h_, int st_, cudaStream_t s_ = nullptr) : h(h_), st(st_), s(s_ ? s_ : h_->stream) {
    if (!h->profile) return;
    const int r = (int)(h->prof_steps % dfb_engine::kProfRing);
    e = &h->pev[(r * dfb_engine::kStages + st) * 2];
    cudaEventRecord(e[0], s);
  }
  void stop() {
    if (!e) return;
    cudaEventRecord(e[1], s);
    h->pev_used[((h->prof_steps % dfb_engine::kProfRing)) * dfb_engine::kStages + st] = 1;
    e = nullptr;
  }
  ~StageTimer() { stop(); }
};

// host-side helpers defined in engine.cu and used by shard.cu
namespace dfbh {
int prof_drain(dfb_engine* h);
// workspaces of the hot-key pre-reduction for a batch of nkeys keys / nnz non-zeros (hot_split > 0)
int hot_ws(dfb_engine* h, size_t nkeys, size_t nnz, dfb::HotWs* ws);
int join_streams(dfb_engine* h);        // make the main stream wait for everything enqueued on the others
int ensure_key_ws(dfb_engine* h, size_t n);
// Localizer::Compact on the device into L (no host synchronisation unless need_host_U):
//   *U_out = the unique-key count when need_host_U, else the capacity (nnz); L.dU() holds the count on the device.
//   A batch whose ids fall outside the sorted range is dropped: 0 keys (nnz > 0), and kErrIdRange is raised into
//   drop_prog when given (otherwise the caller reports it).  standalone (dfb_localize): the range is measured,
//   whatever id_bits or the learned range say, and the learned range is left alone.  need_lidx = false: L.lidx (the
//   remapped CSR index) is not written, for a step that reads the raw ids instead.
int localize_dev(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
                 const float* d_val, uint64_t max_index, dfb_engine::LocSet& L, cudaStream_t s, bool need_host_U,
                 bool exact_range, size_t* U_out, dfb::DevProgress* drop_prog = nullptr, bool standalone = false,
                 bool need_lidx = true);
int check_csr(dfb_engine* h, size_t nrows, const uint64_t* offset);
// (label may be NULL: a predict step without labels)
int stage_raw(dfb_engine* h, dfb_engine::InSet& in, size_t nrows, size_t nnz, const uint64_t* offset,
              const uint64_t* ids, const float* value, const float* label);
int collect_one(dfb_engine* h, dfb::DevProgress* acc);
// growth.cu: the table (h->tab.cap slots) and the V-row pool (h->tab.vcap rows mapped, grow.v_max reserved) at create,
// and their release
int capacity_create(dfb_engine* h);
void capacity_destroy(dfb_engine* h);
// before a call that can insert up to new_keys keys and new_vrows V rows (enqueued next on h->stream): grows the
// table and the pool when the known counts plus every bound enqueued since could exceed their capacities.  Never
// waits for the device, and a failed allocation keeps the current table and pool (a step that really overflows them
// reports DFB_ERR_CAPACITY).  Does nothing on an engine that cannot grow.
int reserve(dfb_engine* h, uint64_t new_keys, uint64_t new_vrows);
// the sharded step's growth (shard_growth = 1), in phase 1 before the lookup.  shard_rcv_slot: where k_shard_count
// stores the keys this owner receives in the step, or NULL when nothing can grow (then nothing below is called).
// reserve_shard, after that count is enqueued on counted_on: grows the table and the pool when the known counts plus
// the bounds in flight -- each step's received keys once counted, `worst` before -- could exceed their capacities,
// waiting for this step's count first when the worst case does not fit.  *rehashed: the table was rebuilt on
// h->stream, which the lookup must wait for.  shard_counts_copy, after the step's InitV: the counts the next
// decision starts from.
int shard_rcv_slot(dfb_engine* h, unsigned long long** slot);
int reserve_shard(dfb_engine* h, cudaStream_t counted_on, uint64_t worst, bool vrows, bool* rehashed);
int shard_counts_copy(dfb_engine* h);
// a copy of the table's slots (cap entries) and of V rows [0, n_vrows) in fresh stream-ordered device memory, made
// on h->stream and waited for; DFB_ERR_CAPACITY with nothing allocated when the memory cannot be had.  The copy keeps
// cap, mask, ks and rs, has vcap = n_vrows and no state or progress: the snapshot writer's view of a table.
int table_copy(dfb_engine* h, uint64_t n_vrows, dfb::Table* out);
void table_copy_free(dfb::Table* t, cudaStream_t s);   // stream-ordered on s
// after a dfb_prune (which waited for every stream): the table holds exactly n_keys keys and n_vrows V rows, and no
// inserting call or sharded step is in flight
void counts_known(dfb_engine* h, uint64_t n_keys, uint64_t n_vrows);
void frozen_destroy(dfb_frozen_s* f);   // checkpoint.cu: frees the copy after its stream's work
int drain(dfb_engine* h);               // checkpoint.cu: wait for everything enqueued on any of the handle's streams
void shard_destroy(dfb_engine* h);      // shard.cu
int shard_sync(dfb_engine* h);          // shard.cu: drain the shard's streams
bool shard_step_open(const dfb_engine* h);   // shard.cu: a sharded step is begun and its phase 4 not yet enqueued
}  // namespace dfbh
