// difacto_b200/csrc/engine.cu -- host side of the engine and the C-ABI of include/difacto_b200.h.
//
// One engine = one shard of the model on one GPU + the workspaces of a minibatch.
// (A) the API-faithful entry points move host buffers in and out around single kernels;
// (B) dfb_train_step* is the fused device-resident minibatch of SGDLearner::IterateData
//     (src/sgd/sgd_learner.cc:138-177 of the reference).
#include <cuda_runtime.h>

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "engine_internal.cuh"

using namespace dfb;  // NOLINT

int dfb_engine::ensure(DevBuf& b, size_t bytes) {
  if (bytes <= b.bytes && b.p) return 0;
  if (bytes == 0) bytes = 16;
  size_t want = bytes + bytes / 4 + 256;
  cudaError_t e;
  if (b.p) {
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return cuda_fail(e, "sync");
    if ((e = cudaStreamSynchronize(copy_stream)) != cudaSuccess) return cuda_fail(e, "sync");
    if (loc_stream && (e = cudaStreamSynchronize(loc_stream)) != cudaSuccess) return cuda_fail(e, "sync");
    if (shard) dfbh::shard_sync(this);
    b.reset();
  }
  if ((e = b.alloc(want)) != cudaSuccess) return cuda_fail(e, "cudaMalloc(workspace)");
  return 0;
}

namespace {

thread_local std::string g_create_error;

uint64_t next_pow2(uint64_t x) {
  uint64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

bool parse_float(const std::string& s, float* out) {
  if (s.empty()) return false;
  char* end = nullptr;
  errno = 0;
  float v = strtof(s.c_str(), &end);
  if (end == s.c_str() || *end != '\0') return false;
  *out = v;
  return true;
}
bool parse_i64(const std::string& s, long long* out) {
  if (s.empty()) return false;
  char* end = nullptr;
  errno = 0;
  long long v = strtoll(s.c_str(), &end, 10);
  if (end == s.c_str() || *end != '\0') return false;
  *out = v;
  return true;
}

// check the sticky device error flag after a synchronisation point
int check_dev_err(dfb_engine* h) {
  int code = h->h_prog->err;
  if (code == 0) return 0;
  switch (code) {
    case DFB_ERR_CAPACITY:
      return h->fail(code, "table_capacity / V_capacity exhausted (raise table_capacity or V_capacity)");
    case DFB_ERR_INVALID:
      return h->fail(code, "invalid input detected on device (a CHECK of the reference would have failed: "
                           "lens[i] != V_dim+1, gradient for a key without V, or key == UINT64_MAX)");
    case kErrIdRange: {
      const std::string range = h->id_bits > 0
          ? "id_bits = " + std::to_string(h->id_bits) + ": ids below 2^" + std::to_string(4 * ((h->id_bits + 3) / 4))
          : std::string("id_bits = 0: the range learned from earlier batches, which widens to these ids for later "
                        "batches");
      return h->fail(DFB_ERR_INVALID, "a raw batch was dropped, untrained: its ids do not fit in the id range the GPU "
                                      "localizer sorts (" + range + ")");
    }
    case DFB_ERR_TIMEOUT:
      return h->fail(code, "a rank of the sharded store did not reach this step within shard_timeout_ms (peer crashed, ran out "
                           "of data without calling the step with nrows = 0, or the ranks' hosts deadlocked)");
    default:
      return h->fail(code, "device-side error " + std::to_string(code));
  }
}

// D2H of the progress block, clearing the device accumulators (err is sticky until read)
int fetch_progress(dfb_engine* h, dfb_progress* out) {
  DFB_CUDA(h, cudaMemcpyAsync(h->h_prog, h->tab.prog, sizeof(DevProgress), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaMemsetAsync(h->tab.prog, 0, sizeof(DevProgress), h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (out) {
    out->loss = (float)h->h_prog->loss;
    out->penalty = (float)h->h_prog->penalty;
    out->auc = (float)h->h_prog->auc;
    out->nnz_w = 0.f;
    out->nrows = (float)h->h_prog->nrows;
    out->new_keys = h->h_prog->new_keys;
    out->new_vrows = h->h_prog->new_vrows;
  }
  return check_dev_err(h);
}

// synchronise and surface a device-side error without disturbing the accumulated Progress
int sync_and_check(dfb_engine* h) {
  DFB_CUDA(h, cudaMemcpyAsync(h->h_prog, h->tab.prog, sizeof(DevProgress), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (h->h_prog->err != 0) {
    DFB_CUDA(h, cudaMemsetAsync(&h->tab.prog->err, 0, sizeof(int), h->stream));
    DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return check_dev_err(h);
}

// read the scratch accumulator block (prog[1]) used by dfb_evaluate / dfb_auc
int fetch_scratch(dfb_engine* h, DevProgress* out) {
  DFB_CUDA(h, cudaMemcpyAsync(h->h_prog, h->tab.prog + 1, sizeof(DevProgress), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  *out = *h->h_prog;
  return 0;
}

}  // namespace
int dfbh::ensure_key_ws(dfb_engine* h, size_t n) {
  DFB_TRY(h->ensure(h->slot, n * sizeof(int)));
  DFB_TRY(h->ensure(h->u_w, n * sizeof(float)));
  DFB_TRY(h->ensure(h->u_vrow, n * sizeof(int)));
  DFB_TRY(h->ensure(h->u_wv, n * sizeof(int2)));
  DFB_TRY(h->ensure(h->flags, n * sizeof(int)));
  DFB_TRY(h->ensure(h->pos, (n + 64) * sizeof(int)));     // also the tile workspace of the InitV pass
  DFB_TRY(h->ensure(h->cub, scan_tmp_bytes(n)));
  return 0;
}
using dfbh::ensure_key_ws;

int dfbh::hot_ws(dfb_engine* h, size_t nkeys, size_t nnz, HotWs* ws) {
  memset(ws, 0, sizeof(*ws));
  if (h->hot_split <= 0) return 0;
  const size_t chunk = h->hot_split / 2 > 32 ? h->hot_split / 2 : 32;
  const size_t cap = nnz / chunk + nnz / (size_t)h->hot_split + 64;
  DFB_TRY(h->ensure(h->hot_map, (nkeys ? nkeys : 1) * sizeof(int)));
  DFB_TRY(h->ensure(h->hot_info, cap * sizeof(int2)));
  DFB_TRY(h->ensure(h->hot_part, cap * (size_t)h->tab.ks * sizeof(float)));
  DFB_TRY(h->ensure(h->hot_ps, cap * sizeof(float2)));
  DFB_TRY(h->ensure(h->hot_cnt, 16));
  ws->hotmap = h->hot_map.as<int>(); ws->info = h->hot_info.as<int2>(); ws->part = h->hot_part.as<float>();
  ws->part_s = h->hot_ps.as<float2>(); ws->counter = h->hot_cnt.as<unsigned long long>(); ws->cap = (int)cap;
  return 0;
}

namespace {

int h2d(dfb_engine* h, DevBuf& b, const void* src, size_t bytes, cudaStream_t s) {
  DFB_TRY(h->ensure(b, bytes));
  if (bytes) DFB_CUDA(h, cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s));
  return 0;
}

void add_prog(DevProgress& a, const DevProgress& b) {
  a.loss += b.loss; a.penalty += b.penalty; a.auc += b.auc;
  a.nrows += b.nrows; a.new_keys += b.new_keys; a.new_vrows += b.new_vrows;
  if (a.err == 0) a.err = b.err;
}

void to_public(const DevProgress& d, dfb_progress* out) {
  out->loss = (float)d.loss; out->penalty = (float)d.penalty; out->auc = (float)d.auc;
  out->nnz_w = 0.f; out->nrows = (float)d.nrows; out->new_keys = d.new_keys; out->new_vrows = d.new_vrows;
}

}  // namespace

int dfbh::prof_drain(dfb_engine* h) {
  if (h->pev.empty()) return 0;
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->loc_stream));
  if (h->shard) DFB_TRY(dfbh::shard_sync(h));
  for (int r = 0; r < dfb_engine::kProfRing; ++r)
    for (int st = 0; st < dfb_engine::kStages; ++st) {
      char& used = h->pev_used[r * dfb_engine::kStages + st];
      if (!used) continue;
      float ms = 0.f;
      const Event* e = &h->pev[(r * dfb_engine::kStages + st) * 2];
      if (cudaEventElapsedTime(&ms, e[0], e[1]) == cudaSuccess) { h->stage_ms[st] += ms; h->stage_n[st]++; }
      used = 0;
    }
  return 0;
}
using dfbh::prof_drain;

// the error of a launch_fm that returned nl < 0
static int fm_launch_fail(dfb_engine* h, int nl, cudaError_t e) {
  if (nl == dfb::kLaunchRefused)
    return h->fail(DFB_ERR_CUDA, std::string("the FM forward launch failed: ") + cudaGetErrorString(e));
  return h->fail(DFB_ERR_INVALID, "unsupported FM configuration");
}

namespace {

// the fused minibatch on device-resident inputs (everything enqueued on h->stream)
int ensure_sorted_ws(dfb_engine* h, size_t nrows, size_t nnz, size_t U, bool valued, bool csc_given = false) {
  DFB_TRY(h->ensure(h->pxv, nrows * (size_t)h->tab.ks * sizeof(float)));
  DFB_TRY(h->ensure(h->p_row, nrows * sizeof(float)));
  if (csc_given) return 0;
  DFB_TRY(h->ensure(h->occ, nnz * (valued ? 8 : 4)));
  DFB_TRY(h->ensure(h->occ_sorted, nnz * (valued ? 8 : 4)));
  DFB_TRY(h->ensure(h->lidx_sorted, nnz * sizeof(uint32_t)));
  DFB_TRY(h->ensure(h->col_start, U * sizeof(int)));
  DFB_TRY(h->ensure(h->col_end, U * sizeof(int)));
  const size_t cb = csc_tmp_bytes(nnz, valued);
  if (cb > h->cub.bytes) DFB_TRY(h->ensure(h->cub, cb));
  return 0;
}

// the keys a batch of n nonzeros can hold: n, or fewer when ids below 2^id_bits bound them
size_t key_bound(const dfb_engine* h, size_t n) {
  return (h->id_bits > 0 && h->id_bits < 40) ? std::min(n, (size_t)1 << h->id_bits) : n;
}

// true when the pulled view {w, vrow} (8 bytes per key) of that many keys fits in half the L2
bool view_fits_l2(size_t keys) { return keys * sizeof(int2) <= l2_bytes() / 2; }

// U is the number of keys, or (dU != nullptr) the capacity of the key arrays with the actual count on the device
// (a batch localized on the GPU never reports its size to the host); d_cnt / cnt_cols: see launch_feacnt.
// predict: a predict step (dfb_predict_raw_* on widths without the raw-id kernels): no penalty; d_lab may be NULL.
// d_ids: the batch's raw ids (a sorted training step on the GPU localizer's CSC view, without a feature-count push):
// no key lookup and no pulled view -- the forward probes the table with each nonzero's id, the update finds or
// inserts the keys itself -- and d_idx is not read.
int step_dev(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint32_t* d_idx,
             const float* d_val, const float* d_lab, const uint64_t* d_keys, size_t U, const float* d_cnt,
             int is_train, const dfb_engine::LocSet* csc = nullptr, const unsigned long long* dU = nullptr,
             const int* cnt_cols = nullptr, bool predict = false, const uint64_t* d_ids = nullptr) {
  const bool csc_ready = csc != nullptr;
  const bool push_cnt = d_cnt != nullptr || cnt_cols != nullptr;
  const bool probe = d_ids != nullptr;
  if (probe && !(is_train && h->sorted_path() && csc_ready && !push_cnt))
    return h->fail(DFB_ERR_INVALID, "the lookup-free step is a sorted training step on the GPU localizer's output");
  if (U > 0x7fffffffULL || nrows > 0x7fffffffULL || nnz > 0x7fffffffULL)
    return h->fail(DFB_ERR_INVALID, "batch too large");
  if (is_train && !h->has_aux) return h->fail(DFB_ERR_INVALID, "no aux data");   // CHECK(has_aux_), sgd_updater.cc:75
  const bool sorted = is_train && h->sorted_path();
  // a training or feature-count step inserts at most U keys (U: the key count or its bound nnz), each with a V row
  if (is_train || push_cnt) DFB_TRY(dfbh::reserve(h, U, U));
  const int ks = h->tab.ks;
  cudaStream_t s = h->stream;
  DFB_TRY(ensure_key_ws(h, U));
  DFB_TRY(h->ensure(h->pred, nrows * sizeof(float)));
  int* slot = h->slot.as<int>();
  float* u_w = h->u_w.as<float>();
  int* u_vrow = h->u_vrow.as<int>();
  int* flags = h->flags.as<int>();
  int* pos = h->pos.as<int>();
  if (h->profile && h->prof_steps && h->prof_steps % dfb_engine::kProfRing == 0) DFB_TRY(prof_drain(h));
  // Push(kFeaCount) then Pull (sgd_learner.cc:214-217, :177).  The lookup-free step has neither: its stage 0 is empty.
  {
  StageTimer tm(h, 0);
  // a validation / prediction batch must not grow the table: a missing entry reads as w = 0, no V
  // (what a default-constructed SGDEntry would give), so nothing needs to be inserted
  const bool insert = is_train || push_cnt;
  if (push_cnt) {
    h->launches += launch_lookup(h->tab, d_keys, U, dU, true, slot, nullptr, nullptr, nullptr, s);
    h->launches += launch_feacnt(h->tab, h->prm, slot, U, dU, d_cnt, cnt_cols, flags, pos, s);
    h->launches += launch_pull_view(h->tab, slot, U, dU, u_w, u_vrow, h->u_wv.as<int2>(), s);
  } else if (!probe) {
    h->launches += launch_lookup(h->tab, d_keys, U, dU, insert, slot, u_w, u_vrow, h->u_wv.as<int2>(), s);
  }
  }
  FmView v;
  memset(&v, 0, sizeof(v));
  v.vbase = h->tab.V; v.vstride = h->tab.rs; v.dense = 0;
  v.l2hint = h->l2_hints;
  const size_t u_bound = key_bound(h, U);      // U is the key count or its bound nnz
  if (probe) {
    v.tab = h->tab.tab; v.tab_mask = h->tab.mask;
  } else {
    v.wbase = u_w; v.w_pos = nullptr;
    v.wv = h->u_wv.as<int2>();
    v.v_pos = u_vrow;
    // the pulled view {w,vrow} (8 bytes per key) is read once per nnz: keep it in L2 only when it fits with room to
    // spare (Criteo-shaped batches: at most 2.6 M keys, 20 MB).  At the flagship shape it can be 52 MB, more than an
    // H100's whole L2, and each key is read about once, so evict_last would only take room from the p*XV rows.
    v.wv_last = h->l2_hints && view_fits_l2(u_bound);
  }
  // the update's L2 plan (p*XV / p kept, the [V|cg] rows streamed past them) pays when the rows a step touches exceed
  // L2.  When they fit (rcv1- and gisette-shaped batches: at most 65536 keys) the default policy is faster: with the
  // plan the rcv1-shaped update took 0.218 ms instead of 0.201 ms (H100 SXM, 700 W).
  const bool l2_plan = h->l2_hints && u_bound * (size_t)h->tab.rs * sizeof(float) > l2_bytes();
  if (dU && !(sorted || !is_train)) return h->fail(DFB_ERR_INVALID, "device-side key count needs the sorted path");
  if (sorted) {
    DFB_TRY(ensure_sorted_ws(h, nrows, nnz, U, d_val != nullptr, csc_ready));
  } else if (is_train) {
    DFB_TRY(h->ensure(h->gw, U * sizeof(float)));
    DFB_CUDA(h, cudaMemsetAsync(h->gw.p, 0, U * sizeof(float), s));
    if (h->prm.V_dim > 0) {
      DFB_TRY(h->ensure(h->gV, U * (size_t)ks * sizeof(float)));
      DFB_CUDA(h, cudaMemsetAsync(h->gV.p, 0, U * (size_t)ks * sizeof(float), s));
      if (d_val) {
        DFB_TRY(h->ensure(h->gxxp, U * sizeof(float)));
        DFB_CUDA(h, cudaMemsetAsync(h->gxxp.p, 0, U * sizeof(float), s));
      }
    }
    v.gwbase = h->gw.as<float>(); v.gw_pos = nullptr;
    v.gvbase = h->gV.as<float>(); v.gv_pos = nullptr; v.gvstride = ks;
    v.gxxp = d_val ? h->gxxp.as<float>() : nullptr;
  }
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.nrows = nrows; b.offset = d_off; b.index = d_idx; b.value = d_val; b.label = d_lab;
  b.pred_in = nullptr; b.pred_io = h->pred.as<float>(); b.pred_acc = 0;
  b.V_dim = h->prm.V_dim; b.train = is_train; b.prog = h->tab.prog;
  b.long_nnz = (unsigned)h->long_row_nnz; b.nnz_hint = nnz;
  b.dev_nkeys = dU;      // 0 keys for nnz > 0: the localizer dropped the batch; every kernel below then does nothing
  b.ids = d_ids;
  if (sorted) {
    b.emit = 1; b.p_out = h->p_row.as<float>(); b.pxv_out = h->pxv.as<float>();
    b.occ_row = csc_ready ? nullptr : h->occ.as<uint32_t>();
    b.occ_rowx = csc_ready ? nullptr : h->occ.as<unsigned long long>();
  }
  if (nrows) {
    StageTimer tm(h, 1);
    cudaError_t le = cudaSuccess;
    const int nl = probe ? launch_fm_raw(b, v, false, s) : launch_fm(b, v, h->force_generic, s, &le);
    if (nl < 0) return fm_launch_fail(h, nl, le);
    h->launches += nl;
  }
  bool auc_pending = false;
  if (h->compute_auc && nrows && d_lab) {
    // AUC depends only on pred: run it on the auxiliary stream, overlapped with the gradient
    // reduction / update below (when profiling, keep it on the main stream so that it is timed)
    DFB_TRY(h->ensure(h->auc_k, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_v, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_tmp, sort_tmp_bytes(nrows)));
    const bool side = h->overlap_auc && !h->profile;
    cudaStream_t as = side ? h->aux_stream : s;
    if (side) {
      DFB_CUDA(h, cudaEventRecord(h->ev_fm_done, s));
      DFB_CUDA(h, cudaStreamWaitEvent(as, h->ev_fm_done, 0));
    }
    StageTimer tm(h, 2);
    h->launches += launch_auc(d_lab, h->pred.as<float>(), nrows, h->auc_k.as<float>(),
                              h->auc_v.as<float>(), h->auc_tmp.p, h->auc_tmp.bytes, &h->tab.prog->auc, dU, as);
    if (side) {
      DFB_CUDA(h, cudaEventRecord(h->ev_auc_done, as));
      auc_pending = true;
    }
  }
  if (sorted) {
    // CalcGrad + Push(kGradient) without materialising the gradient: CSC view of the batch, then
    // per key reduce + FTRL + AdaGrad (+ the -V*XXp term and the penalty of the pulled weights)
    StageTimer tm(h, 3);
    if (!csc_ready) {
      int nl = launch_csc_build(d_idx, h->occ.p, d_val != nullptr, nnz, U, h->lidx_sorted.as<uint32_t>(),
                                h->occ_sorted.p, h->col_start.as<int>(), h->col_end.as<int>(), h->cub.p,
                                h->cub.bytes, h->tab.prog, s);
      if (nl < 0) return h->fail(DFB_ERR_CUDA, "CSC sort of the batch failed (temporary storage)");
      h->launches += nl;
    }
  }
  StageTimer tm_upd(h, 4);
  if (sorted) {
    const int* cs = csc ? csc->col_start.as<int>() : h->col_start.as<int>();
    const int* ce = csc ? csc->col_end.as<int>() : h->col_end.as<int>();
    const void* occs = csc ? csc->occ_sorted.p : h->occ_sorted.p;
    HotWs hws;
    HotPart hp;
    DFB_TRY(dfbh::hot_ws(h, U, nnz, &hws));
    h->launches += launch_hot_prereduce(h->prm.V_dim, U, dU, cs, ce, occs, d_val != nullptr, h->p_row.as<float>(),
                                        h->pxv.as<float>(), h->hot_split, hws, &hp, l2_plan, s);
    // without a lookup the update finds (or inserts) every key itself and leaves its slot for the InitV pass
    int nl = launch_bwd_update(h->tab, h->prm, probe ? d_keys : nullptr, slot, u_vrow, U, dU, cs, ce, occs, d_val != nullptr,
                               h->p_row.as<float>(), h->pxv.as<float>(), flags, 1, nullptr, hp.part ? &hp : nullptr,
                               l2_plan, s);
    if (nl < 0) return h->fail(DFB_ERR_INVALID, "sorted scatter unsupported for this V_dim");
    h->launches += nl;
    if (l2_plan)
      h->launches += launch_l2_discard(h->pxv.p, nrows * (size_t)ks * sizeof(float), h->p_row.p,
                                       nrows * sizeof(float), s);
    h->launches += launch_initv(h->tab, h->prm, slot, U, dU, flags, pos, s);
  } else if (is_train) {
    // Push(kGradient): FTRL + AdaGrad (+ the -V*XXp term and the penalty of the pulled weights)
    h->launches += launch_update_dense(h->tab, h->prm, slot, u_vrow, 0, U, h->gw.as<float>(),
                                       d_val ? h->gxxp.as<float>() : nullptr, h->gV.as<float>(), flags, 1,
                                       d_val ? 1 : 2, s);
    h->launches += launch_initv(h->tab, h->prm, slot, U, nullptr, flags, pos, s);
  } else if (!predict) {
    h->launches += launch_penalty(h->prm, h->tab.prog, u_w, u_vrow, h->tab.V, h->tab.rs, 0, U, dU, s);
  }
  if (h->profile) {
    tm_upd.stop();
    h->prof_steps++;
  }
  if (auc_pending) DFB_CUDA(h, cudaStreamWaitEvent(s, h->ev_auc_done, 0));
  DFB_CUDA(h, cudaGetLastError());
  return 0;
}

}  // namespace

// fold the oldest outstanding snapshot of the pipelined path into *acc
int dfbh::collect_one(dfb_engine* h, DevProgress* acc) {
  const int r = (int)(h->collected % dfb_engine::kRing);
  DFB_CUDA(h, cudaEventSynchronize(h->ring_done[r]));
  add_prog(*acc, h->h_ring[r]);
  h->collected++;
  return 0;
}
using dfbh::collect_one;

namespace {
int lowest_bit(unsigned long long or_all) {
  if (!or_all) return 63;    // every key is 0
  int b = 0;
  while (((or_all >> b) & 1ULL) == 0) ++b;
  return b;
}
}  // namespace

// Localizer::Compact on the device.  Leaves the unique keys, the remapped CSR index and the CSC view
// (occ_sorted / col_start / col_end; col_start has U+1 entries) in L.  The radix sort only visits the key
// bits that are not constant zero; which bits those are is either given (id_bits: ids < 2^id_bits fill the
// top nibbles of the reversed key, rounded up to whole nibbles), or learned: the first batch is measured with one
// 8-byte D2H sync, later batches reuse the range (verified on the device; earlier batches' OR masks are read back
// without waiting and can only widen it); exact_range measures every batch of an engine without id_bits (the
// synchronous entry points, which wait for the step anyway).  A batch the range does not cover is dropped (see
// engine_internal.cuh).  With need_host_U the unique-key count is also synchronised to the host, otherwise it
// stays on the device (L.dU()) and *U_out is the capacity nnz.
int dfbh::localize_dev(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
                       const float* d_val, uint64_t max_index, dfb_engine::LocSet& L, cudaStream_t s,
                       bool need_host_U, bool exact_range, size_t* U_out, DevProgress* drop_prog, bool standalone,
                       bool need_lidx) {
  *U_out = 0;
  if (nnz > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "batch too large");   // localizer.cc:19-20
  if (max_index == 0) return h->fail(DFB_ERR_INVALID, "max_index must be > 0");
  const size_t n1 = nnz ? nnz : 1;
  DFB_TRY(h->ensure(h->l_rkeys, n1 * 8));
  DFB_TRY(h->ensure(h->l_skeys, n1 * 8));
  DFB_TRY(h->ensure(h->l_pay, n1 * 8));
  DFB_TRY(h->ensure(h->l_spay, n1 * 8));
  DFB_TRY(h->ensure(h->l_tmp, localize_sort_tmp_bytes(nnz)));
  DFB_TRY(h->ensure(L.scal, 16));
  DFB_TRY(h->ensure(L.keys, n1 * 8));
  DFB_TRY(h->ensure(L.lidx, n1 * 4));
  DFB_TRY(h->ensure(L.cnt, n1 * 4));
  DFB_TRY(h->ensure(L.occ_sorted, n1 * (d_val ? 8 : 4)));
  DFB_TRY(h->ensure(L.col_start, (n1 + 1) * 4));
  DFB_TRY(h->ensure(L.col_end, n1 * 4));
  unsigned long long* scal = L.scal.as<unsigned long long>();
  if (nnz == 0) {
    DFB_CUDA(h, cudaMemsetAsync(scal, 0, 16, s));
    return 0;
  }
  // ---- the bit range of the sort (known before the keys are produced, unless this batch must be measured) ----
  int begin_bit = -1;
  // dfb_localize (any max_index): measured, never dropped, and the engine's own range is neither used nor learned
  const bool restricted = standalone || max_index != ~0ULL;
  if (h->id_bits > 0 && !restricted) {
    begin_bit = 64 - 4 * ((h->id_bits + 3) / 4);
  } else if (!restricted && !need_host_U && !exact_range) {
    for (int q = 0; q < 2; ++q)                        // masks of earlier batches, if they have arrived
      if (h->or_pending[q] && cudaEventQuery(h->ev_or[q]) == cudaSuccess) {
        h->or_pending[q] = false;
        const int b = lowest_bit(h->h_or[q]);
        if (h->loc_begin_bit < 0 || b < h->loc_begin_bit) h->loc_begin_bit = b;
      }
    begin_bit = h->loc_begin_bit;
  }
  const bool hi32 = begin_bit >= 32;       // only the upper 32 key bits can be set: 32-bit sort keys
  h->launches += launch_localize_keys(d_ids, nnz, max_index, h->l_rkeys.as<unsigned long long>(),
                                      h->l_pay.p, scal, d_off, nrows, hi32, s);
  if (begin_bit < 0) {
    DFB_CUDA(h, cudaMemcpyAsync(h->h_scal, scal, 8, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(h, cudaStreamSynchronize(s));
    begin_bit = lowest_bit(h->h_scal[0]);
    if (!restricted && (h->loc_begin_bit < 0 || begin_bit < h->loc_begin_bit)) h->loc_begin_bit = begin_bit;
  } else if (h->id_bits <= 0 && !restricted) {
    const int q = (int)(h->or_seq++ & 1);
    if (!h->or_pending[q]) {
      DFB_CUDA(h, cudaMemcpyAsync(h->h_or + q, scal, 8, cudaMemcpyDeviceToHost, s));
      DFB_CUDA(h, cudaEventRecord(h->ev_or[q], s));
      h->or_pending[q] = true;
    }
  }
  {
    int nl = launch_localize_sort(h->l_rkeys.as<unsigned long long>(), h->l_pay.p, nnz, begin_bit, hi32,
                                  h->l_skeys.as<unsigned long long>(), h->l_spay.p, h->l_tmp.p, h->l_tmp.bytes, d_val,
                                  L.keys.as<uint64_t>(),
                                  L.col_start.as<int>(), L.col_end.as<int>(),
                                  need_lidx ? L.lidx.as<uint32_t>() : nullptr,
                                  L.occ_sorted.p, scal, drop_prog, s);
    if (nl < 0) return h->fail(DFB_ERR_CUDA, "radix sort / scan of the GPU localizer failed (temporary storage)");
    h->launches += nl;
  }
  if (need_host_U) {
    DFB_CUDA(h, cudaMemcpyAsync(h->h_scal + 1, scal + 1, 8, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(h, cudaStreamSynchronize(s));
    *U_out = (size_t)h->h_scal[1];
  } else {
    *U_out = nnz;
  }
  return 0;
}
using dfbh::localize_dev;

namespace {

// raw (un-localized) CSR<u64> minibatch: Localizer::Compact + the fused step, all on the device.
// The localizer runs on its own stream into one of two output sets, overlapped with the step of the
// previous batch; on the sorted fast path nothing of it is synchronised to the host (the unique-key
// count stays on the device), so a step is one uninterrupted enqueue.
int step_raw_dev(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
                 const float* d_val, const float* d_lab, int push_cnt, int is_train, cudaEvent_t inputs_ready,
                 bool exact_range = false, bool predict = false) {
  dfb_engine::LocSet& L = h->loc[h->loc_seq & 1];
  // while profiling the localizer shares the main stream: per-stage times are then those of kernels running alone
  cudaStream_t ls = h->profile ? h->stream : h->loc_stream;
  if (inputs_ready) DFB_CUDA(h, cudaStreamWaitEvent(ls, inputs_ready, 0));
  if (L.used) DFB_CUDA(h, cudaStreamWaitEvent(ls, L.consumed, 0));
  const bool dev_count_ok = h->sorted_path(is_train);
  // a sorted training step without a feature-count push looks no key up (step_dev's d_ids): nothing reads the ranks.
  // A push_cnt step keeps the lookup: Update(kFeaCount) can start InitV before the Pull, so V rows must exist before
  // the forward; a validation step's penalty reads the pulled view.  So does a batch whose pulled view fits in L2
  // (few keys, many nonzeros each: Criteo-, gisette- and rcv1-shaped batches): there the forward reads each nonzero's
  // metadata from L2, where probing the table costs a chain of round trips per nonzero.  Without the lookup, criteo39
  // steps took 1.02 instead of 0.95 ms and gisette's 1.09 instead of 0.95 ms (H100 80 GB HBM3, 400 W).
  // (The key-finding update exists with the L2 plan only, which such a batch has when V_dim > 0 and l2_hints is on.)
  const bool probe = is_train && !push_cnt && dev_count_ok && !predict && !view_fits_l2(key_bound(h, nnz)) &&
                     h->l2_hints && h->prm.V_dim > 0;
  size_t U = 0;
  if (h->profile && h->prof_steps && h->prof_steps % dfb_engine::kProfRing == 0) DFB_TRY(prof_drain(h));
  {
    StageTimer tm(h, 5, ls);
    DFB_TRY(localize_dev(h, nrows, nnz, d_off, d_ids, d_val, ~0ULL, L, ls, !dev_count_ok, exact_range, &U, nullptr,
                         false, !probe));   // Localizer(-1, ...), sgd_learner.cc:203
  }
  const float* d_cnt = nullptr;
  const int* cnt_cols = nullptr;
  if (push_cnt && U) {
    if (dev_count_ok) {
      cnt_cols = L.col_start.as<int>();       // U+1 column offsets: the counts are their differences
    } else {
      h->launches += launch_cnt_from_cols(L.col_start.as<int>(), L.col_end.as<int>(), U, L.cnt.as<float>(), ls);
      d_cnt = L.cnt.as<float>();
    }
  }
  DFB_CUDA(h, cudaEventRecord(L.done, ls));
  DFB_CUDA(h, cudaStreamWaitEvent(h->stream, L.done, 0));
  int rc = 0;
  if (!dev_count_ok && nnz && U == 0) {
    // the localizer dropped the batch (ids outside the sorted range): no step; the drop is reported in this step's
    // Progress, in stream order.  (With the count on the device, step_dev's kernels see the 0 and do the same.)
    DFB_TRY(h->ensure(h->pred, nrows * sizeof(float)));       // what dfb_train_step_raw's pred_out copies
    h->launches += launch_raise_err(h->tab.prog, kErrIdRange, h->stream);
  } else {
    rc = step_dev(h, nrows, nnz, d_off, probe ? nullptr : L.lidx.as<uint32_t>(), d_val, d_lab, L.keys.as<uint64_t>(),
                  U, d_cnt, is_train, &L, (dev_count_ok && nnz) ? L.dU() : nullptr, cnt_cols, predict,
                  probe ? d_ids : nullptr);
  }
  DFB_CUDA(h, cudaEventRecord(L.consumed, h->stream));
  L.used = true;
  h->loc_seq++;
  return rc;
}

// the predict step on raw ids: the forward pass of a frozen model, written into h->pred.  Nothing of the model is
// written.  Where the specialised kernels exist it is ONE forward launch that probes the table for each nonzero's id
// (no localizer, no key lookup, no penalty: launch_fm_raw), plus the id_bits range check when id_bits > 0 and the
// AUC when labels are given.  Other widths (V_dim > 128, force_generic) run the validation step without its penalty.
int predict_dev(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
                const float* d_val, const float* d_lab, cudaEvent_t inputs_ready) {
  if (h->shard)
    return h->fail(DFB_ERR_INVALID, "this engine holds one shard of a sharded model: predict with dfb_shard_predict_async");
  if (nrows > 0x7fffffffULL || nnz > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "batch too large");
  cudaStream_t s = h->stream;
  DFB_TRY(h->ensure(h->pred, (nrows ? nrows : 1) * sizeof(float)));
  if (!h->sorted_path(false)) {
    // a dropped batch (ids outside id_bits) predicts 0 for every row
    if (nrows) DFB_CUDA(h, cudaMemsetAsync(h->pred.p, 0, nrows * sizeof(float), s));
    return step_raw_dev(h, nrows, nnz, d_off, d_ids, d_val, d_lab, 0, 0, inputs_ready, true, true);
  }
  if (h->profile && h->prof_steps && h->prof_steps % dfb_engine::kProfRing == 0) DFB_TRY(prof_drain(h));
  FmView v;
  memset(&v, 0, sizeof(v));
  v.vbase = h->tab.V; v.vstride = h->tab.rs; v.l2hint = h->l2_hints;
  v.tab = h->tab.tab; v.tab_mask = h->tab.mask;
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.nrows = nrows; b.offset = d_off; b.ids = d_ids; b.value = d_val; b.label = d_lab;
  b.pred_io = h->pred.as<float>(); b.V_dim = h->prm.V_dim; b.train = 0; b.prog = h->tab.prog;
  b.long_nnz = (unsigned)h->long_row_nnz; b.nnz_hint = nnz;
  const int nbits = 4 * ((h->id_bits + 3) / 4);
  if (h->id_bits > 0 && nbits < 64 && nnz) {
    // the range the localizer would sort: a batch outside it is dropped as a training batch would be (0 predictions,
    // nothing in Progress, kErrIdRange raised by the forward kernel)
    DFB_TRY(h->ensure(h->id_ok, sizeof(unsigned long long)));
    DFB_CUDA(h, cudaMemsetAsync(h->id_ok.p, 0xff, sizeof(unsigned long long), s));
    DFB_CUDA(h, cudaMemsetAsync(h->pred.p, 0, nrows * sizeof(float), s));
    h->launches += launch_id_range(d_ids, nnz, nbits, h->id_ok.as<unsigned long long>(), s);
    b.dev_nkeys = h->id_ok.as<unsigned long long>();
  }
  if (nrows) {
    StageTimer tm(h, 1);
    const int nl = launch_fm_raw(b, v, h->tab.vonly == 2, s);
    if (nl < 0) return h->fail(DFB_ERR_INVALID, "unsupported FM configuration");
    h->launches += nl;
  }
  if (h->compute_auc && nrows && d_lab) {
    DFB_TRY(h->ensure(h->auc_k, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_v, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_tmp, sort_tmp_bytes(nrows)));
    StageTimer tm(h, 2);
    h->launches += launch_auc(d_lab, h->pred.as<float>(), nrows, h->auc_k.as<float>(), h->auc_v.as<float>(),
                              h->auc_tmp.p, h->auc_tmp.bytes, &h->tab.prog->auc, b.dev_nkeys, s);
  }
  if (h->profile) h->prof_steps++;
  DFB_CUDA(h, cudaGetLastError());
  return 0;
}

}  // namespace

int dfbh::check_csr(dfb_engine* h, size_t nrows, const uint64_t* offset) {
  if (nrows && !offset) return h->fail(DFB_ERR_INVALID, "offset is NULL");
  if (nrows && offset[0] != 0) return h->fail(DFB_ERR_INVALID, "offset[0] must be 0 (fm_loss.h:88 assumes it)");
  // nnz is offset[nrows]: rows must not run backwards, or the kernels would index outside the nnz arrays
  for (size_t r = 0; r < nrows; ++r)
    if (offset[r + 1] < offset[r]) return h->fail(DFB_ERR_INVALID, "offset must be non-decreasing");
  return 0;
}
using dfbh::check_csr;

extern "C" {

const char* dfb_last_error(dfb_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int dfb_destroy(dfb_handle h);

int dfb_create(const char* const* keys, const char* const* vals, int n, dfb_handle* out) {
  if (!out) { g_create_error = "out is NULL"; return DFB_ERR_INVALID; }
  *out = nullptr;
  dfb_engine* h = new dfb_engine();
  // defaults and ranges: src/sgd/sgd_param.h:94-106
  Params& p = h->prm;
  p.l1 = 1.f; p.l2 = 0.f; p.V_l2 = .01f; p.lr = .01f; p.lr_beta = 1.f; p.V_lr = .01f; p.V_lr_beta = 1.f;
  p.V_init_scale = .01f; p.V_threshold = 10; p.V_dim = -1; p.seed = 0;
  long long table_capacity = 1 << 20, v_capacity = -1, table_capacity_max = -1, v_capacity_max = -1;
  bool v_bf16 = false;
  struct FR { const char* name; float* dst; float lo, hi; };
  FR fr[] = {{"l1", &p.l1, 0, 1e10f}, {"l2", &p.l2, 0, 1e10f}, {"V_l2", &p.V_l2, 0, 1e10f},
             {"lr", &p.lr, 0, 10}, {"lr_beta", &p.lr_beta, 0, 1e10f}, {"V_lr", &p.V_lr, 0, 1e10f},
             {"V_lr_beta", &p.V_lr_beta, 0, 10}, {"V_init_scale", &p.V_init_scale, 0, 10}};
  auto bad = [&](const std::string& m) {
    g_create_error = m;
    delete h;
    return (int)DFB_ERR_PARAM;
  };
  for (int i = 0; i < n; ++i) {
    const std::string k = keys[i] ? keys[i] : "", v = vals[i] ? vals[i] : "";
    bool used = false;
    for (auto& f : fr) {
      if (k == f.name) {
        float x;
        if (!parse_float(v, &x)) return bad("Invalid Parameter format for " + k + " expect float but value='" + v + "'");
        if (!(x >= f.lo && x <= f.hi)) return bad("value " + v + " for Parameter " + k + " exceed bound [" + std::to_string(f.lo) + "," + std::to_string(f.hi) + "]");
        *f.dst = x;
        used = true;
      }
    }
    if (used) continue;
    long long x = 0;
    auto need_int = [&](long long lo, long long hi) {
      if (!parse_i64(v, &x)) { g_create_error = "Invalid Parameter format for " + k + " expect int but value='" + v + "'"; return false; }
      if (x < lo || x > hi) { g_create_error = "value " + v + " for Parameter " + k + " out of range"; return false; }
      return true;
    };
    if (k == "V_dim") { if (!need_int(0, 10000)) { delete h; return DFB_ERR_PARAM; } p.V_dim = (int)x; }
    else if (k == "V_threshold") { if (!need_int(-2147483647LL, 2147483647LL)) { delete h; return DFB_ERR_PARAM; } p.V_threshold = (int)x; }
    else if (k == "seed") { if (!need_int(0, 4294967295LL)) { delete h; return DFB_ERR_PARAM; } p.seed = (unsigned)x; }
    else if (k == "device") { if (!need_int(0, 1023)) { delete h; return DFB_ERR_PARAM; } h->device = (int)x; }
    else if (k == "table_capacity") { if (!need_int(1, 1LL << 30)) { delete h; return DFB_ERR_PARAM; } table_capacity = x; }
    else if (k == "V_capacity") { if (!need_int(0, 1LL << 30)) { delete h; return DFB_ERR_PARAM; } v_capacity = x; }
    else if (k == "table_capacity_max") { if (!need_int(1, 1LL << 30)) { delete h; return DFB_ERR_PARAM; } table_capacity_max = x; }
    else if (k == "V_capacity_max") { if (!need_int(0, 1LL << 30)) { delete h; return DFB_ERR_PARAM; } v_capacity_max = x; }
    else if (k == "compute_auc") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->compute_auc = (int)x; }
    else if (k == "force_generic") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->force_generic = (int)x; }
    else if (k == "overlap_auc") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->overlap_auc = (int)x; }
    else if (k == "long_row_nnz") { if (!need_int(0, 1 << 30)) { delete h; return DFB_ERR_PARAM; } h->long_row_nnz = (int)x; }
    else if (k == "hot_split") { if (!need_int(0, 1 << 30)) { delete h; return DFB_ERR_PARAM; } h->hot_split = (int)x; }
    else if (k == "l2_hints") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->l2_hints = (int)x; }
    else if (k == "id_bits") { if (!need_int(0, 64)) { delete h; return DFB_ERR_PARAM; } h->id_bits = (int)x; }
    else if (k == "shard_timeout_ms") { if (!need_int(1, 3600000)) { delete h; return DFB_ERR_PARAM; } h->shard_timeout_ms = x; }
    else if (k == "shard_growth") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->shard_growth = (int)x; }
    else if (k == "score_only") { if (!need_int(0, 1)) { delete h; return DFB_ERR_PARAM; } h->score_only = (int)x; }
    else if (k == "V_storage") {
      if (v == "fp32") v_bf16 = false;
      else if (v == "bf16") v_bf16 = true;
      else return bad("V_storage must be 'fp32' or 'bf16'");
    }
    else if (k == "scatter") {
      if (v == "sorted") h->scatter_sorted = 1;
      else if (v == "atomic") h->scatter_sorted = 0;
      else return bad("scatter must be 'sorted' or 'atomic'");
    }
    else h->unknown.push_back(std::make_pair(k, v));
  }
  if (p.V_dim < 0) return bad("Required parameter V_dim of int is not presented");   // sgd_param.h:104
  if (v_bf16 && !h->score_only) return bad("V_storage = bf16 needs score_only = 1 (training on 2-byte rows is not offered)");
  // a scoring-only engine predicts with the raw-id forward alone: the other widths' predict step is the validation
  // step, which reads a pulled view the engine does not build
  if (h->score_only && (h->force_generic || !fm_fast_supported(p.V_dim)))
    return bad("score_only = 1 needs 0 <= V_dim <= 128 and force_generic = 0");
  // the initial capacities and the maxima they may grow to (equal by default: nothing grows)
  if (table_capacity_max < 0) table_capacity_max = table_capacity;
  if (table_capacity_max < table_capacity) return bad("table_capacity_max must be >= table_capacity");
  if (v_capacity_max < 0) v_capacity_max = v_capacity >= 0 ? v_capacity : table_capacity_max;
  if (v_capacity < 0) v_capacity = table_capacity;
  if (v_capacity_max < v_capacity) return bad("V_capacity_max must be >= V_capacity");
  if (p.V_dim == 0) v_capacity = v_capacity_max = 0;
  h->grow.tab_max = (uint64_t)table_capacity_max;
  h->grow.v_max = (uint64_t)v_capacity_max;
  h->grow.on = table_capacity_max > table_capacity || v_capacity_max > v_capacity;

  cudaError_t e;
  auto cfail = [&](const char* what) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(e);
    cudaGetLastError();   // clear the sticky error before releasing what was created so far
    dfb_destroy(h);
    return (int)DFB_ERR_CUDA;
  };
  if ((e = cudaSetDevice(h->device)) != cudaSuccess) return cfail("cudaSetDevice");
  // All four at the default priority, the localizer's loc_stream too.  On one GPU a high-priority localizer takes SM
  // slots from the latency-bound lookup / gather kernels of the current step and costs ~4 %, measured.  Holding it
  // back until the update stage starts (HBM-bound, short-lived CTAs) and then giving it the greatest priority put 91 %
  // of its kernel time under the update, but the update grew from 3.05 to 3.75 ms: the two share HBM, and the step
  // got 2.3 % slower (H100 SXM, 700 W).  The sharded store's worker stream does get priority.
  for (Stream* s : {&h->stream, &h->copy_stream, &h->aux_stream, &h->loc_stream})
    if ((e = s->create()) != cudaSuccess) return cfail("cudaStreamCreate");
  for (Event* ev : {&h->loc[0].done, &h->loc[0].consumed, &h->loc[1].done, &h->loc[1].consumed, &h->ev_fm_done,
                    &h->ev_auc_done, &h->in[0].copied, &h->in[0].consumed, &h->in[1].copied, &h->in[1].consumed,
                    &h->ev_or[0], &h->ev_or[1]})
    if ((e = ev->create()) != cudaSuccess) return cfail("cudaEventCreate");
  for (auto& ev : h->ring_done)
    if ((e = ev.create()) != cudaSuccess) return cfail("cudaEventCreate");
  Table& t = h->tab;
  t.max_keys = (uint64_t)table_capacity;
  t.cap = next_pow2(2 * t.max_keys);
  if (t.cap < 1024) t.cap = 1024;
  if (t.cap > (1ULL << 31)) { g_create_error = "table_capacity too large (slots are 31-bit)"; dfb_destroy(h); return DFB_ERR_PARAM; }
  t.mask = t.cap - 1;
  t.ks = (p.V_dim + 3) / 4 * 4;
  t.vcap = (uint64_t)v_capacity;
  t.rs = h->score_only ? t.ks : 2 * t.ks;
  t.vonly = h->score_only ? (v_bf16 ? 2 : 1) : 0;
  if (h->score_only) h->has_aux = 0;
  if (const int rc = dfbh::capacity_create(h)) {
    g_create_error = h->err;
    cudaGetLastError();
    dfb_destroy(h);
    return rc;
  }
  if ((e = h->tab_state.alloc(sizeof(TableState))) != cudaSuccess) return cfail("cudaMalloc(state)");
  if ((e = h->tab_prog.alloc(2 * sizeof(DevProgress))) != cudaSuccess) return cfail("cudaMalloc(prog)");
  t.state = h->tab_state.as<TableState>();
  t.prog = h->tab_prog.as<DevProgress>();
  if ((e = cudaMemset(t.prog, 0, 2 * sizeof(DevProgress))) != cudaSuccess) return cfail("cudaMemset(prog)");
  if ((e = h->h_prog.alloc(1)) != cudaSuccess) return cfail("cudaHostAlloc");
  if ((e = h->h_nvals.alloc(1)) != cudaSuccess) return cfail("cudaHostAlloc");
  memset(h->h_prog, 0, sizeof(DevProgress));
  if ((e = h->h_scal.alloc(2)) != cudaSuccess) return cfail("cudaHostAlloc");
  if ((e = h->h_or.alloc(2)) != cudaSuccess) return cfail("cudaHostAlloc");
  if ((e = h->h_ring.alloc(dfb_engine::kRing)) != cudaSuccess) return cfail("cudaHostAlloc");
  memset(h->h_ring, 0, dfb_engine::kRing * sizeof(DevProgress));
  memset(&h->backlog, 0, sizeof(DevProgress));
  h->launches += launch_table_init(t, p.seed, h->stream);
  if ((e = cudaStreamSynchronize(h->stream)) != cudaSuccess) return cfail("table init");
  *out = h;
  return DFB_OK;
}

int dfb_destroy(dfb_handle h) {
  if (!h) return DFB_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  if (h->frozen) dfbh::frozen_destroy(h->frozen);   // a frozen snapshot not released: its handle dangles from here
  h->frozen = nullptr;
  h->shard.reset();
  dfbh::capacity_destroy(h);
  delete h;
  return DFB_OK;
}

int dfb_num_unknown_kwargs(dfb_handle h) { return h ? (int)h->unknown.size() : 0; }
int dfb_unknown_kwarg(dfb_handle h, int i, const char** key, const char** val) {
  if (!h || i < 0 || i >= (int)h->unknown.size()) return DFB_ERR_INVALID;
  *key = h->unknown[i].first.c_str();
  *val = h->unknown[i].second.c_str();
  return DFB_OK;
}
uint64_t dfb_launch_count(dfb_handle h) { return h ? h->launches : 0; }
void* dfb_stream(dfb_handle h) { return h ? (void*)h->stream : nullptr; }
int dfb_row_stride(dfb_handle h) { return h ? h->tab.ks : 0; }

int dfb_row_bytes(dfb_handle h, uint64_t* bytes_per_row, uint64_t* bytes_in_use) {
  if (!h) return DFB_ERR_INVALID;
  const uint64_t rb = (uint64_t)h->tab.rs * (h->tab.vonly == 2 ? 2 : 4);
  uint64_t n_vrows = 0;
  DFB_TRY(dfb_table_stats(h, nullptr, &n_vrows, nullptr, nullptr));
  if (bytes_per_row) *bytes_per_row = rb;
  if (bytes_in_use) *bytes_in_use = n_vrows * rb;
  return DFB_OK;
}

int dfb_growth_stats(dfb_handle h, uint64_t* growths, uint64_t* host_waits) {
  if (!h) return DFB_ERR_INVALID;
  if (growths) *growths = h->grow.n_growths;
  if (host_waits) *host_waits = h->grow.n_waits;
  return DFB_OK;
}

int dfb_table_stats(dfb_handle h, uint64_t* n_keys, uint64_t* n_vrows, uint64_t* capacity, uint64_t* v_capacity) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  TableState st;
  DFB_CUDA(h, cudaMemcpyAsync(&st, h->tab.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (n_keys) *n_keys = st.n_keys;
  if (n_vrows) *n_vrows = st.n_vrows;
  if (capacity) *capacity = h->tab.max_keys;
  if (v_capacity) *v_capacity = h->tab.vcap;
  return DFB_OK;
}

int dfb_rng_state(dfb_handle h, uint32_t* seed) {
  if (!h || !seed) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  TableState st;
  DFB_CUDA(h, cudaMemcpyAsync(&st, h->tab.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  *seed = st.seed;
  return DFB_OK;
}

int dfb_id_range_get(dfb_handle h, int* bits) {
  if (!h || !bits) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  // the key masks of the batches enqueued so far widen the range once read: wait for them and fold them in
  for (int q = 0; q < 2; ++q)
    if (h->or_pending[q]) {
      DFB_CUDA(h, cudaEventSynchronize(h->ev_or[q]));
      h->or_pending[q] = false;
      const int b = lowest_bit(h->h_or[q]);
      if (h->loc_begin_bit < 0 || b < h->loc_begin_bit) h->loc_begin_bit = b;
    }
  *bits = h->loc_begin_bit < 0 ? 0 : 64 - h->loc_begin_bit;
  return DFB_OK;
}

int dfb_id_range_set(dfb_handle h, int bits) {
  if (!h) return DFB_ERR_INVALID;
  if (bits < 1 || bits > 64) return h->fail(DFB_ERR_INVALID, "id range bits must be in [1, 64]");
  if (h->loc_begin_bit >= 0 || h->or_pending[0] || h->or_pending[1])
    return h->fail(DFB_ERR_INVALID, "the engine has already learned an id range");
  h->loc_begin_bit = 64 - bits;
  return DFB_OK;
}

int dfb_host_alloc(void** ptr, size_t bytes) {
  if (!ptr) return DFB_ERR_INVALID;
  return cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocDefault) == cudaSuccess ? DFB_OK : DFB_ERR_CUDA;
}
int dfb_host_free(void* ptr) { return cudaFreeHost(ptr) == cudaSuccess ? DFB_OK : DFB_ERR_CUDA; }

// ------------------------------------------------------------------------------------------
// (A) API-faithful path
// ------------------------------------------------------------------------------------------
int dfb_push_feacnt(dfb_handle h, const uint64_t* keys, size_t n, const float* cnt) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_push_feacnt");
  if (n && (!keys || !cnt)) return h->fail(DFB_ERR_INVALID, "keys/cnt is NULL");
  if (n > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "too many keys");
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->keys, keys, n * sizeof(uint64_t), s));
  DFB_TRY(h2d(h, h->cnt, cnt, n * sizeof(float), s));
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(dfbh::reserve(h, n, n));
  h->launches += launch_lookup(h->tab, h->keys.as<uint64_t>(), n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_feacnt(h->tab, h->prm, h->slot.as<int>(), n, nullptr, h->cnt.as<float>(), nullptr,
                               h->flags.as<int>(), h->pos.as<int>(), s);
  return sync_and_check(h);
}

int dfb_pull(dfb_handle h, const uint64_t* keys, size_t n, float* vals_out, size_t vals_cap, int* lens_out,
             size_t* nvals, size_t* nlens) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_pull");
  if (!nvals || !nlens) return h->fail(DFB_ERR_INVALID, "nvals/nlens is NULL");
  if (n && (!keys || !vals_out)) return h->fail(DFB_ERR_INVALID, "keys/vals_out is NULL");
  if (n > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "too many keys");
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int k = h->prm.V_dim;
  *nvals = 0; *nlens = 0;
  if (n == 0) return DFB_OK;
  DFB_TRY(h2d(h, h->keys, keys, n * sizeof(uint64_t), s));
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(dfbh::reserve(h, n, 0));     // model_[key] inserts; a pull allocates no V row
  if (k == 0) {
    if (vals_cap < n) return h->fail(DFB_ERR_INVALID, "vals_out too small");
    h->launches += launch_lookup(h->tab, h->keys.as<uint64_t>(), n, nullptr, true, h->slot.as<int>(), h->u_w.as<float>(),
                                 h->u_vrow.as<int>(), nullptr, s);
    DFB_CUDA(h, cudaMemcpyAsync(vals_out, h->u_w.p, n * sizeof(float), cudaMemcpyDeviceToHost, s));
    DFB_TRY(sync_and_check(h));
    *nvals = n; *nlens = 0;   // lens->resize(V_dim == 0 ? 0 : size), sgd_updater.cc:40
    return DFB_OK;
  }
  if (!lens_out) return h->fail(DFB_ERR_INVALID, "lens_out is NULL");
  if ((unsigned long long)n * (unsigned long long)(k + 1) > 0x7fffffffULL)
    return h->fail(DFB_ERR_INVALID, "pull too large for 31-bit positions (the reference's int p overflows too)");
  DFB_TRY(h->ensure(h->lens, n * sizeof(int)));
  DFB_TRY(h->ensure(h->vals, n * (size_t)(k + 1) * sizeof(float)));
  DFB_TRY(h->ensure(h->nvals, sizeof(unsigned long long)));
  h->launches += launch_lookup(h->tab, h->keys.as<uint64_t>(), n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_pack_ragged(h->tab, h->prm, h->slot.as<int>(), n, h->lens.as<int>(), h->pos.as<int>(),
                                    h->vals.as<float>(), h->nvals.as<unsigned long long>(), h->cub.p,
                                    h->cub.bytes, s);
  DFB_CUDA(h, cudaMemcpyAsync(h->h_nvals, h->nvals.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaMemcpyAsync(lens_out, h->lens.p, n * sizeof(int), cudaMemcpyDeviceToHost, s));
  DFB_TRY(sync_and_check(h));
  const size_t nv = (size_t)*h->h_nvals;
  if (nv > vals_cap) return h->fail(DFB_ERR_INVALID, "vals_out too small");
  DFB_CUDA(h, cudaMemcpyAsync(vals_out, h->vals.p, nv * sizeof(float), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaStreamSynchronize(s));
  *nvals = nv; *nlens = n;
  return DFB_OK;
}

int dfb_push_grad(dfb_handle h, const uint64_t* keys, size_t n, const float* grads, size_t nvals,
                  const int* lens, size_t nlens) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_push_grad");
  if (n && (!keys || !grads)) return h->fail(DFB_ERR_INVALID, "keys/grads is NULL");
  if (n > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "too many keys");
  if (!h->has_aux) return h->fail(DFB_ERR_INVALID, "no aux data");   // CHECK(has_aux_), sgd_updater.cc:75
  const bool w_only = nlens == 0;   // sgd_updater.cc:77-82
  if (w_only) { if (nvals != n) return h->fail(DFB_ERR_INVALID, "CHECK_EQ(values.size(), size) failed"); }
  else {
    if (nlens != n || !lens) return h->fail(DFB_ERR_INVALID, "CHECK_EQ(lens.size(), size) failed");
    unsigned long long tot = 0;
    for (size_t i = 0; i < n; ++i) {
      if (lens[i] < 1) return h->fail(DFB_ERR_INVALID, "lens[i] < 1");
      tot += (unsigned long long)lens[i];
    }
    if (tot != nvals) return h->fail(DFB_ERR_INVALID, "CHECK_EQ(p, values.size()) failed");   // :99
    if (tot > 0x7fffffffULL) return h->fail(DFB_ERR_INVALID, "push too large for 31-bit positions");
  }
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  if (n == 0) return DFB_OK;
  DFB_TRY(h2d(h, h->keys, keys, n * sizeof(uint64_t), s));
  DFB_TRY(h2d(h, h->vals, grads, nvals * sizeof(float), s));
  DFB_TRY(ensure_key_ws(h, n));
  const int* d_lens = nullptr;
  if (!w_only) {
    DFB_TRY(h2d(h, h->lens, lens, n * sizeof(int), s));
    d_lens = h->lens.as<int>();
    h->launches += launch_lens_scan(d_lens, n, h->pos.as<int>(), h->cub.p, h->cub.bytes, s);
  }
  DFB_TRY(dfbh::reserve(h, n, n));
  h->launches += launch_lookup(h->tab, h->keys.as<uint64_t>(), n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_update_ragged(h->tab, h->prm, h->slot.as<int>(), n, h->vals.as<float>(), d_lens,
                                      h->pos.as<int>(), h->flags.as<int>(), s);
  h->launches += launch_initv(h->tab, h->prm, h->slot.as<int>(), n, nullptr, h->flags.as<int>(), h->pos.as<int>(), s);
  return sync_and_check(h);
}

static int stage_fm_inputs(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index,
                           const float* value, const float* weights, size_t nweights, const int* w_pos,
                           const int* V_pos, size_t npos, size_t* nnz_out) {
  DFB_TRY(check_csr(h, nrows, offset));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !index) return h->fail(DFB_ERR_INVALID, "index is NULL");
  if (nweights && !weights) return h->fail(DFB_ERR_INVALID, "weights is NULL");
  if ((w_pos == nullptr) != (V_pos == nullptr)) return h->fail(DFB_ERR_INVALID, "w_pos and V_pos must both be given or both be NULL");
  if (h->prm.V_dim > 0 && !V_pos) return h->fail(DFB_ERR_INVALID, "V_pos is required when V_dim > 0");
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->a_off, offset, (nrows + 1) * sizeof(uint64_t), s));
  DFB_TRY(h2d(h, h->a_idx, index, nnz * sizeof(uint32_t), s));
  if (value) DFB_TRY(h2d(h, h->a_val, value, nnz * sizeof(float), s));
  DFB_TRY(h2d(h, h->a_w, weights, nweights * sizeof(float), s));
  if (w_pos) {
    DFB_TRY(h2d(h, h->a_wpos, w_pos, npos * sizeof(int), s));
    DFB_TRY(h2d(h, h->a_vpos, V_pos, npos * sizeof(int), s));
  }
  *nnz_out = nnz;
  return 0;
}

int dfb_predict(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index, const float* value,
                const float* weights, size_t nweights, const int* w_pos, const int* V_pos, size_t npos,
                float* pred) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_predict");
  if (nrows == 0) return DFB_OK;
  if (!pred) return h->fail(DFB_ERR_INVALID, "pred is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  size_t nnz = 0;
  DFB_TRY(stage_fm_inputs(h, nrows, offset, index, value, weights, nweights, w_pos, V_pos, npos, &nnz));
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->a_pred, pred, nrows * sizeof(float), s));   // pred is accumulated into
  FmView v;
  memset(&v, 0, sizeof(v));
  v.wbase = h->a_w.as<float>(); v.w_pos = w_pos ? h->a_wpos.as<int>() : nullptr;
  v.vbase = h->a_w.as<float>(); v.v_pos = V_pos ? h->a_vpos.as<int>() : nullptr; v.vstride = 1;
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.nrows = nrows; b.offset = h->a_off.as<uint64_t>(); b.index = h->a_idx.as<uint32_t>();
  b.value = value ? h->a_val.as<float>() : nullptr;
  b.pred_io = h->a_pred.as<float>(); b.pred_acc = 1; b.V_dim = h->prm.V_dim; b.train = 0;
  cudaError_t le = cudaSuccess;
  int nl = launch_fm(b, v, 1, s, &le);
  if (nl < 0) return fm_launch_fail(h, nl, le);
  h->launches += nl;
  DFB_CUDA(h, cudaMemcpyAsync(pred, h->a_pred.p, nrows * sizeof(float), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaStreamSynchronize(s));
  return DFB_OK;
}

int dfb_calc_grad(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index, const float* value,
                  const float* label, const float* weights, size_t nweights, const int* w_pos, const int* V_pos,
                  size_t npos, const float* pred, float* grad) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_calc_grad");
  if (nrows == 0) return DFB_OK;
  if (!pred || !grad || !label) return h->fail(DFB_ERR_INVALID, "pred/grad/label is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  size_t nnz = 0;
  DFB_TRY(stage_fm_inputs(h, nrows, offset, index, value, weights, nweights, w_pos, V_pos, npos, &nnz));
  cudaStream_t s = h->stream;
  const int k = h->prm.V_dim;
  DFB_TRY(h2d(h, h->a_pred, pred, nrows * sizeof(float), s));
  DFB_TRY(h2d(h, h->a_lab, label, nrows * sizeof(float), s));
  DFB_TRY(h2d(h, h->a_grad, grad, nweights * sizeof(float), s));   // grad is accumulated into
  if (k > 0) {
    DFB_TRY(h->ensure(h->gxxp, npos * sizeof(float)));
    DFB_CUDA(h, cudaMemsetAsync(h->gxxp.p, 0, npos * sizeof(float), s));
  }
  FmView v;
  memset(&v, 0, sizeof(v));
  v.wbase = h->a_w.as<float>(); v.w_pos = w_pos ? h->a_wpos.as<int>() : nullptr;
  v.vbase = h->a_w.as<float>(); v.v_pos = V_pos ? h->a_vpos.as<int>() : nullptr; v.vstride = 1;
  v.gwbase = h->a_grad.as<float>(); v.gw_pos = v.w_pos;
  v.gvbase = h->a_grad.as<float>(); v.gv_pos = v.v_pos; v.gvstride = 1;
  v.gxxp = k > 0 ? h->gxxp.as<float>() : nullptr;
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.nrows = nrows; b.offset = h->a_off.as<uint64_t>(); b.index = h->a_idx.as<uint32_t>();
  b.value = value ? h->a_val.as<float>() : nullptr; b.label = h->a_lab.as<float>();
  b.pred_in = h->a_pred.as<float>(); b.pred_io = nullptr; b.pred_acc = 0; b.V_dim = k; b.train = 1;
  b.prog = nullptr;
  cudaError_t le = cudaSuccess;
  int nl = launch_fm(b, v, 1, s, &le);
  if (nl < 0) return fm_launch_fail(h, nl, le);
  h->launches += nl;
  if (k > 0)
    h->launches += launch_grad_finalize(k, npos, h->a_w.as<float>(), h->a_vpos.as<int>(), h->gxxp.as<float>(),
                                        h->a_grad.as<float>(), s);
  DFB_CUDA(h, cudaMemcpyAsync(grad, h->a_grad.p, nweights * sizeof(float), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaStreamSynchronize(s));
  return DFB_OK;
}

int dfb_evaluate(dfb_handle h, const float* label, const float* pred, size_t n, float* objv) {
  if (!h || !objv) return DFB_ERR_INVALID;
  *objv = 0.f;
  if (n == 0) return DFB_OK;
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->a_lab, label, n * sizeof(float), s));
  DFB_TRY(h2d(h, h->a_pred, pred, n * sizeof(float), s));
  DFB_CUDA(h, cudaMemsetAsync(h->tab.prog + 1, 0, sizeof(DevProgress), s));
  h->launches += launch_evaluate(h->a_lab.as<float>(), h->a_pred.as<float>(), n, &(h->tab.prog + 1)->loss, s);
  DevProgress pr;
  DFB_TRY(fetch_scratch(h, &pr));
  *objv = (float)pr.loss;
  return DFB_OK;
}

int dfb_auc(dfb_handle h, const float* label, const float* pred, size_t n, float* auc_times_n) {
  if (!h || !auc_times_n) return DFB_ERR_INVALID;
  *auc_times_n = 0.f;
  if (n == 0) return DFB_OK;
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->a_lab, label, n * sizeof(float), s));
  DFB_TRY(h2d(h, h->a_pred, pred, n * sizeof(float), s));
  DFB_TRY(h->ensure(h->auc_k, n * sizeof(float)));
  DFB_TRY(h->ensure(h->auc_v, n * sizeof(float)));
  DFB_TRY(h->ensure(h->cub, sort_tmp_bytes(n)));
  DFB_CUDA(h, cudaMemsetAsync(h->tab.prog + 1, 0, sizeof(DevProgress), s));
  h->launches += launch_auc(h->a_lab.as<float>(), h->a_pred.as<float>(), n, h->auc_k.as<float>(),
                            h->auc_v.as<float>(), h->cub.p, h->cub.bytes, &(h->tab.prog + 1)->auc, nullptr, s);
  DevProgress pr;
  DFB_TRY(fetch_scratch(h, &pr));
  *auc_times_n = (float)pr.auc;
  return DFB_OK;
}

// ------------------------------------------------------------------------------------------
// (B) fused step
// ------------------------------------------------------------------------------------------
int dfb_train_step_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint32_t* d_index,
                       const float* d_value_or_null, const float* d_label, const uint64_t* d_keys, size_t nkeys,
                       const float* d_cnt_or_null, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_train_step_dev");
  DFB_CUDA(h, cudaSetDevice(h->device));
  return step_dev(h, nrows, nnz, d_offset, d_index, d_value_or_null, d_label, d_keys, nkeys, d_cnt_or_null,
                  is_train);
}

int dfb_sync(dfb_handle h) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->loc_stream));
  if (h->shard) DFB_TRY(dfbh::shard_sync(h));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  return DFB_OK;
}

int dfb_read_progress(dfb_handle h, dfb_progress* out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  DevProgress acc = h->backlog;
  memset(&h->backlog, 0, sizeof(DevProgress));
  while (h->collected < h->submitted) DFB_TRY(collect_one(h, &acc));
  int rc = fetch_progress(h, nullptr);    // what is still on the device (dfb_train_step_dev steps)
  add_prog(acc, *h->h_prog);
  if (out) to_public(acc, out);
  if (rc != 0) return rc;
  *h->h_prog = acc;
  return check_dev_err(h);
}

static int snapshot_step(dfb_handle h);

int dfb_train_step_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index,
                         const float* value, const float* label, const uint64_t* keys, size_t nkeys,
                         const float* cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_train_step_async");
  DFB_TRY(check_csr(h, nrows, offset));
  if (nrows && !label) return h->fail(DFB_ERR_INVALID, "label is NULL");
  if (nkeys && !keys) return h->fail(DFB_ERR_INVALID, "keys is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !index) return h->fail(DFB_ERR_INVALID, "index is NULL");
  auto& in = h->in[h->seq & 1];
  in.pre = {};
  cudaStream_t cs = h->copy_stream;
  // the copy of batch t+1 may overwrite set b only after batch t-1 (same set) was consumed
  if (h->seq >= 2) DFB_CUDA(h, cudaStreamWaitEvent(cs, in.consumed, 0));
  DFB_TRY(h2d(h, in.off, offset, (nrows + 1) * sizeof(uint64_t), cs));
  DFB_TRY(h2d(h, in.idx, index, nnz * sizeof(uint32_t), cs));
  if (value) DFB_TRY(h2d(h, in.val, value, nnz * sizeof(float), cs));
  DFB_TRY(h2d(h, in.lab, label, nrows * sizeof(float), cs));
  DFB_TRY(h2d(h, in.keys, keys, nkeys * sizeof(uint64_t), cs));
  if (cnt) DFB_TRY(h2d(h, in.cnt, cnt, nkeys * sizeof(float), cs));
  DFB_CUDA(h, cudaEventRecord(in.copied, cs));
  DFB_CUDA(h, cudaStreamWaitEvent(h->stream, in.copied, 0));
  int rc = step_dev(h, nrows, nnz, in.off.as<uint64_t>(), in.idx.as<uint32_t>(), value ? in.val.as<float>() : nullptr,
                    in.lab.as<float>(), in.keys.as<uint64_t>(), nkeys, cnt ? in.cnt.as<float>() : nullptr,
                    is_train);
  DFB_CUDA(h, cudaEventRecord(in.consumed, h->stream));
  h->seq++;
  if (rc != 0) return rc;
  return snapshot_step(h);   // per-step snapshot of the Progress block: D2H into the pinned ring, then clear
}

int dfb_wait_step(dfb_handle h, dfb_progress* out) {
  if (!h) return DFB_ERR_INVALID;
  if (h->submitted == h->collected) return h->fail(DFB_ERR_INVALID, "no outstanding step");
  DFB_CUDA(h, cudaSetDevice(h->device));
  DevProgress one;
  memset(&one, 0, sizeof(one));
  DFB_TRY(collect_one(h, &one));
  if (out) to_public(one, out);
  *h->h_prog = one;
  return check_dev_err(h);
}

}  // extern "C"
int dfbh::join_streams(dfb_engine* h) {
  if (!h->ev_join) DFB_CUDA(h, h->ev_join.create());
  cudaStream_t others[] = {h->copy_stream, h->aux_stream, h->loc_stream};
  for (cudaStream_t o : others) {
    DFB_CUDA(h, cudaEventRecord(h->ev_join, o));
    DFB_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_join, 0));
  }
  return 0;
}
extern "C" {

int dfb_time_mark(dfb_handle h, int which) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (!h->ev_t0) { DFB_CUDA(h, h->ev_t0.create(cudaEventDefault)); DFB_CUDA(h, h->ev_t1.create(cudaEventDefault)); }
  if (which == 0) {
    DFB_CUDA(h, cudaEventRecord(h->ev_t0, h->stream));
  } else {
    if (h->shard) DFB_TRY(dfbh::shard_sync(h));       // the shard's streams: drained (its last event is on another stream)
    DFB_TRY(dfbh::join_streams(h));
    DFB_CUDA(h, cudaEventRecord(h->ev_t1, h->stream));
  }
  return DFB_OK;
}

int dfb_time_elapsed_ms(dfb_handle h, float* ms) {
  if (!h || !ms || !h->ev_t0) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaEventSynchronize(h->ev_t1));
  DFB_CUDA(h, cudaEventElapsedTime(ms, h->ev_t0, h->ev_t1));
  return DFB_OK;
}

int dfb_profile(dfb_handle h, int enable) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (enable && h->pev.empty()) {
    h->pev.resize((size_t)dfb_engine::kProfRing * dfb_engine::kStages * 2);
    h->pev_used.assign((size_t)dfb_engine::kProfRing * dfb_engine::kStages, 0);
    for (auto& ev : h->pev) DFB_CUDA(h, ev.create(cudaEventDefault));
  }
  if (!enable && h->profile) DFB_TRY(prof_drain(h));
  h->profile = enable ? 1 : 0;
  return DFB_OK;
}

int dfb_profile_read(dfb_handle h, double* stage_ms, uint64_t* stage_count) {
  if (!h || !stage_ms || !stage_count) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(prof_drain(h));
  for (int i = 0; i < dfb_engine::kStages; ++i) {
    stage_ms[i] = h->stage_ms[i]; stage_count[i] = h->stage_n[i];
    h->stage_ms[i] = 0; h->stage_n[i] = 0;
  }
  h->prof_steps = 0;
  return DFB_OK;
}

// snapshot of the Progress block into the pinned ring (shared by the async entry points)
static int snapshot_step(dfb_handle h) {
  if (h->submitted - h->collected == (uint64_t)dfb_engine::kRing) DFB_TRY(collect_one(h, &h->backlog));
  const int r = (int)(h->submitted % dfb_engine::kRing);
  DFB_CUDA(h, cudaMemcpyAsync(&h->h_ring[r], h->tab.prog, sizeof(DevProgress), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaMemsetAsync(h->tab.prog, 0, sizeof(DevProgress), h->stream));
  DFB_CUDA(h, cudaEventRecord(h->ring_done[r], h->stream));
  h->submitted++;
  return DFB_OK;
}

int dfb_localize(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* index, uint64_t max_index,
                 uint32_t* index_out, uint64_t* keys_out, float* cnt_out, size_t* nkeys) {
  if (!h || !nkeys) return DFB_ERR_INVALID;
  *nkeys = 0;
  DFB_TRY(check_csr(h, nrows, offset));
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz == 0) return DFB_OK;                       // localizer.cc:16
  if (!index || !index_out || !keys_out) return h->fail(DFB_ERR_INVALID, "NULL argument");
  cudaStream_t s = h->stream;
  DFB_TRY(h2d(h, h->a_off, offset, (nrows + 1) * sizeof(uint64_t), s));
  DFB_TRY(h2d(h, h->keys, index, nnz * sizeof(uint64_t), s));
  size_t U = 0;
  DFB_CUDA(h, cudaStreamSynchronize(h->loc_stream));
  dfb_engine::LocSet& L = h->loc[0];
  DFB_TRY(localize_dev(h, nrows, nnz, h->a_off.as<uint64_t>(), h->keys.as<uint64_t>(), nullptr, max_index, L, s, true, true, &U,
                         nullptr, true));
  DFB_CUDA(h, cudaMemcpyAsync(index_out, L.lidx.p, nnz * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaMemcpyAsync(keys_out, L.keys.p, U * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  if (cnt_out) {
    h->launches += launch_cnt_from_cols(L.col_start.as<int>(), L.col_end.as<int>(), U, L.cnt.as<float>(), s);
    DFB_CUDA(h, cudaMemcpyAsync(cnt_out, L.cnt.p, U * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  DFB_CUDA(h, cudaStreamSynchronize(s));
  *nkeys = U;
  return DFB_OK;
}

int dfb_train_step_raw_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                           const float* d_value_or_null, const float* d_label, int push_cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_train_step_raw_dev");
  DFB_CUDA(h, cudaSetDevice(h->device));
  return step_raw_dev(h, nrows, nnz, d_offset, d_ids, d_value_or_null, d_label, push_cnt, is_train, nullptr);
}

// H2D of one raw batch into the input set the next submission will use (copy stream)
}  // extern "C"
int dfbh::stage_raw(dfb_engine* h, dfb_engine::InSet& in, size_t nrows, size_t nnz, const uint64_t* offset,
                    const uint64_t* ids, const float* value, const float* label) {
  cudaStream_t cs = h->copy_stream;
  if (h->seq >= 2) DFB_CUDA(h, cudaStreamWaitEvent(cs, in.consumed, 0));
  if (nrows) DFB_TRY(h2d(h, in.off, offset, (nrows + 1) * sizeof(uint64_t), cs));     // an empty batch has no offset array
  else DFB_TRY(h->ensure(in.off, 16));
  DFB_TRY(h2d(h, in.ids, ids, nnz * sizeof(uint64_t), cs));
  if (value) DFB_TRY(h2d(h, in.val, value, nnz * sizeof(float), cs));
  if (label) DFB_TRY(h2d(h, in.lab, label, nrows * sizeof(float), cs));
  DFB_CUDA(h, cudaEventRecord(in.copied, cs));
  return 0;
}
int dfbh::stage_host_batch(dfb_engine* h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                           const float* label, bool need_label, dfb_engine::InSet** in_out, size_t* nnz_out) {
  DFB_TRY(check_csr(h, nrows, offset));
  if (need_label && nrows && !label) return h->fail(DFB_ERR_INVALID, "label is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !ids) return h->fail(DFB_ERR_INVALID, "ids is NULL");
  auto& in = h->in[h->seq & 1];
  const bool reuse = in.prefetched(offset, ids, value, label, nrows, nnz);
  in.pre = {};                                // (also when the staging below fails part way)
  if (!reuse) DFB_TRY(stage_raw(h, in, nrows, nnz, offset, ids, value, label));
  *in_out = &in;
  *nnz_out = nnz;
  return 0;
}
using dfbh::stage_raw;
extern "C" {

int dfb_prefetch_raw(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                     const float* label) {
  if (!h) return DFB_ERR_INVALID;
  DFB_TRY(check_csr(h, nrows, offset));       // (label may be NULL: the batch of a predict step)
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !ids) return h->fail(DFB_ERR_INVALID, "ids is NULL");
  auto& in = h->in[h->seq & 1];
  in.pre = {};
  DFB_TRY(stage_raw(h, in, nrows, nnz, offset, ids, value, label));
  in.pre = {offset, ids, value, label, nrows, nnz};
  return DFB_OK;
}

static int raw_async_impl(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                          const float* value, const float* label, int push_cnt, int is_train, bool exact_range) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_train_step_raw");
  dfb_engine::InSet* inp;
  size_t nnz;
  DFB_TRY(dfbh::stage_host_batch(h, nrows, offset, ids, value, label, true, &inp, &nnz));
  dfb_engine::InSet& in = *inp;
  DFB_CUDA(h, cudaStreamWaitEvent(h->stream, in.copied, 0));
  int rc = step_raw_dev(h, nrows, nnz, in.off.as<uint64_t>(), in.ids.as<uint64_t>(),
                        value ? in.val.as<float>() : nullptr, in.lab.as<float>(), push_cnt, is_train, in.copied,
                        exact_range);
  DFB_CUDA(h, cudaEventRecord(in.consumed, h->stream));
  h->seq++;
  if (rc != 0) return rc;
  return snapshot_step(h);
}

int dfb_predict_raw_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                          const float* label, float* pred_out) {
  if (!h) return DFB_ERR_INVALID;
  if (h->shard)
    return h->fail(DFB_ERR_INVALID, "this engine holds one shard of a sharded model: predict with dfb_shard_predict_async");
  dfb_engine::InSet* inp;
  size_t nnz;
  DFB_TRY(dfbh::stage_host_batch(h, nrows, offset, ids, value, label, false, &inp, &nnz));
  dfb_engine::InSet& in = *inp;
  DFB_CUDA(h, cudaStreamWaitEvent(h->stream, in.copied, 0));
  int rc = predict_dev(h, nrows, nnz, in.off.as<uint64_t>(), in.ids.as<uint64_t>(), value ? in.val.as<float>() : nullptr,
                       label ? in.lab.as<float>() : nullptr, in.copied);
  // the predictions leave at the end of the step, in stream order (before the next step rewrites h->pred)
  if (rc == 0 && pred_out && nrows)
    DFB_CUDA(h, cudaMemcpyAsync(pred_out, h->pred.p, nrows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaEventRecord(in.consumed, h->stream));
  h->seq++;
  if (rc != 0) return rc;
  return snapshot_step(h);
}

int dfb_predict_raw_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                        const float* d_value_or_null, const float* d_label_or_null, float* d_pred_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(predict_dev(h, nrows, nnz, d_offset, d_ids, d_value_or_null, d_label_or_null, nullptr));
  if (d_pred_out && nrows)
    DFB_CUDA(h, cudaMemcpyAsync(d_pred_out, h->pred.p, nrows * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  return DFB_OK;
}

int dfb_train_step_raw_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                             const float* value, const float* label, int push_cnt, int is_train) {
  return raw_async_impl(h, nrows, offset, ids, value, label, push_cnt, is_train, false);
}

int dfb_train_step_raw(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                       const float* label, int push_cnt, int is_train, dfb_progress* out, float* pred_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_TRY(raw_async_impl(h, nrows, offset, ids, value, label, push_cnt, is_train, true));
  if (pred_out && nrows)
    DFB_CUDA(h, cudaMemcpyAsync(pred_out, h->pred.p, nrows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return dfb_read_progress(h, out);
}

int dfb_train_step(dfb_handle h, size_t nrows, const uint64_t* offset, const uint32_t* index, const float* value,
                   const float* label, const uint64_t* keys, size_t nkeys, const float* cnt, int is_train,
                   dfb_progress* out, float* pred_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_TRY(dfb_train_step_async(h, nrows, offset, index, value, label, keys, nkeys, cnt, is_train));
  if (pred_out && nrows)
    DFB_CUDA(h, cudaMemcpyAsync(pred_out, h->pred.p, nrows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return dfb_read_progress(h, out);
}

int dfb_read_entries(dfb_handle h, const uint64_t* keys, size_t n, float* scal_out, int* has_V_out, float* V_out,
                     float* cg_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_read_entries");
  if (n == 0) return DFB_OK;
  if (!keys || !scal_out || !has_V_out) return h->fail(DFB_ERR_INVALID, "NULL argument");
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int k = h->prm.V_dim;
  DFB_TRY(h2d(h, h->keys, keys, n * sizeof(uint64_t), s));
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(h->ensure(h->scal, n * 4 * sizeof(float)));
  DFB_TRY(h->ensure(h->hasv, n * sizeof(int)));
  DFB_TRY(h->ensure(h->rV, n * (size_t)(k ? k : 1) * sizeof(float)));
  DFB_TRY(h->ensure(h->rcg, n * (size_t)(k ? k : 1) * sizeof(float)));
  DFB_CUDA(h, cudaMemsetAsync(h->rV.p, 0, n * (size_t)(k ? k : 1) * sizeof(float), s));
  DFB_CUDA(h, cudaMemsetAsync(h->rcg.p, 0, n * (size_t)(k ? k : 1) * sizeof(float), s));
  h->launches += launch_lookup(h->tab, h->keys.as<uint64_t>(), n, nullptr, false, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_read_entries(h->tab, h->slot.as<int>(), n, h->scal.as<float>(), h->hasv.as<int>(),
                                     h->rV.as<float>(), h->rcg.as<float>(), k, s);
  DFB_CUDA(h, cudaMemcpyAsync(scal_out, h->scal.p, n * 4 * sizeof(float), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaMemcpyAsync(has_V_out, h->hasv.p, n * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (V_out && k) DFB_CUDA(h, cudaMemcpyAsync(V_out, h->rV.p, n * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (cg_out && k) DFB_CUDA(h, cudaMemcpyAsync(cg_out, h->rcg.p, n * (size_t)k * sizeof(float), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaStreamSynchronize(s));
  return DFB_OK;
}

// ------------------------------------------------------------------------------------------
// sharding
// ------------------------------------------------------------------------------------------
uint32_t dfb_key_owner(uint64_t key, uint32_t S) {
  if (S == 0) return 0;
  const uint64_t width = UINT64_MAX / (uint64_t)S;   // postoffice.cc:130-134
  const uint64_t o = key / width;
  return (uint32_t)(o >= S ? S - 1 : o);
}

int dfb_shard_bounds(const uint64_t* keys, size_t n, uint32_t S, size_t* bounds) {
  if (!bounds || S == 0 || (n && !keys)) return DFB_ERR_INVALID;
  const uint64_t width = UINT64_MAX / (uint64_t)S;
  bounds[0] = 0;
  for (uint32_t i = 1; i < S; ++i) {
    // first key >= width*i  (lower_bound, like DefaultSlicer kv_app.h:416-429)
    const uint64_t lo_key = width * i;
    size_t lo = bounds[i - 1], hi = n;
    while (lo < hi) {
      size_t mid = lo + (hi - lo) / 2;
      if (keys[mid] < lo_key) lo = mid + 1; else hi = mid;
    }
    bounds[i] = lo;
  }
  bounds[S] = n;
  return DFB_OK;
}

int dfb_dev_feacnt(dfb_handle h, const uint64_t* d_keys, size_t n, const float* d_cnt) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_dev_feacnt");
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (n == 0) return DFB_OK;
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(dfbh::reserve(h, n, n));
  cudaStream_t s = h->stream;
  h->launches += launch_lookup(h->tab, d_keys, n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_feacnt(h->tab, h->prm, h->slot.as<int>(), n, nullptr, d_cnt, nullptr, h->flags.as<int>(),
                               h->pos.as<int>(), s);
  DFB_CUDA(h, cudaGetLastError());
  return DFB_OK;
}

static int dev_pull_rows_impl(dfb_handle h, const uint64_t* d_keys, size_t n, float* d_w_out, int* d_hasv_out,
                              int* d_hasv_out2, float* d_V_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_dev_pull_rows");
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (n == 0) return DFB_OK;
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(dfbh::reserve(h, n, 0));
  cudaStream_t s = h->stream;
  h->launches += launch_lookup(h->tab, d_keys, n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  h->launches += launch_gather_rows(h->tab, h->slot.as<int>(), n, d_w_out, d_hasv_out, d_hasv_out2,
                                    h->prm.V_dim > 0 ? d_V_out : nullptr, s);
  DFB_CUDA(h, cudaGetLastError());
  return DFB_OK;
}

int dfb_dev_pull_rows(dfb_handle h, const uint64_t* d_keys, size_t n, float* d_w_out, int* d_hasv_out,
                      float* d_V_out) {
  return dev_pull_rows_impl(h, d_keys, n, d_w_out, d_hasv_out, nullptr, d_V_out);
}

int dfb_dev_pull_rows_peer(dfb_handle h, const uint64_t* d_keys, size_t n, float* peer_w_out, int* peer_hasv_out,
                           float* peer_V_out, int* d_hasv_local_out) {
  return dev_pull_rows_impl(h, d_keys, n, peer_w_out, peer_hasv_out, d_hasv_local_out, peer_V_out);
}

// ---- peer-accessible buffers (CUDA IPC) for the NVLink store ----
int dfb_peer_alloc(dfb_handle h, size_t bytes, void** ptr, unsigned char* handle64) {
  if (!h || !ptr || !handle64) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaMalloc(ptr, bytes ? bytes : 256));
  cudaIpcMemHandle_t mh;
  static_assert(sizeof(mh) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaError_t e = cudaIpcGetMemHandle(&mh, *ptr);
  if (e != cudaSuccess) { cudaFree(*ptr); *ptr = nullptr; return h->cuda_fail(e, "cudaIpcGetMemHandle"); }
  memcpy(handle64, &mh, 64);
  return DFB_OK;
}

int dfb_peer_open(dfb_handle h, const unsigned char* handle64, void** ptr) {
  if (!h || !ptr || !handle64) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaIpcMemHandle_t mh;
  memcpy(&mh, handle64, 64);
  DFB_CUDA(h, cudaIpcOpenMemHandle(ptr, mh, cudaIpcMemLazyEnablePeerAccess));
  return DFB_OK;
}

int dfb_peer_close(dfb_handle h, void* ptr) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaIpcCloseMemHandle(ptr));
  return DFB_OK;
}

int dfb_peer_free(dfb_handle h, void* ptr) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_CUDA(h, cudaFree(ptr));
  return DFB_OK;
}

static int dev_fm_step_impl(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint32_t* d_index,
                           const float* d_value, const float* d_label, size_t nkeys, const float* d_w,
                           const int* d_hasv, const float* d_V, int is_train, float* d_gw_out, float* d_gV_out,
                           const SegDst* seg);

int dfb_dev_fm_step(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint32_t* d_index,
                    const float* d_value, const float* d_label, size_t nkeys, const float* d_w, const int* d_hasv,
                    const float* d_V, int is_train, float* d_gw_out, float* d_gV_out) {
  return dev_fm_step_impl(h, nrows, nnz, d_offset, d_index, d_value, d_label, nkeys, d_w, d_hasv, d_V, is_train,
                          d_gw_out, d_gV_out, nullptr);
}

int dfb_dev_fm_step_peer(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint32_t* d_index,
                         const float* d_value, const float* d_label, size_t nkeys, const float* d_w,
                         const int* d_hasv, const float* d_V, int nseg, const size_t* seg_bounds,
                         float* const* peer_gw, float* const* peer_gV, int first_seg) {
  if (!h) return DFB_ERR_INVALID;
  if (nseg < 1 || nseg > 8 || !seg_bounds || !peer_gw || !peer_gV)
    return h->fail(DFB_ERR_INVALID, "dfb_dev_fm_step_peer: 1..8 segments with destinations required");
  SegDst sd;
  memset(&sd, 0, sizeof(sd));
  sd.nseg = nseg;
  for (int i = 0; i <= nseg; ++i) sd.bounds[i] = (int)seg_bounds[i];
  for (int i = 0; i < nseg; ++i) { sd.gw[i] = peer_gw[i]; sd.gV[i] = peer_gV[i]; }
  if (first_seg >= 0 && first_seg < nseg) sd.rot = sd.bounds[first_seg] / 32 * 32;
  if ((size_t)sd.bounds[nseg] != nkeys) return h->fail(DFB_ERR_INVALID, "seg_bounds[nseg] must equal nkeys");
  if (!h->sorted_path() || fast_lane_width(h->prm.V_dim) != h->prm.V_dim)
    return h->fail(DFB_ERR_INVALID, "peer gradient stores need the sorted scatter path (V_dim in {8,16,32,64,128})");
  return dev_fm_step_impl(h, nrows, nnz, d_offset, d_index, d_value, d_label, nkeys, d_w, d_hasv, d_V, 1,
                          peer_gw[0], peer_gV[0], &sd);
}

static int dev_fm_step_impl(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint32_t* d_index,
                           const float* d_value, const float* d_label, size_t nkeys, const float* d_w,
                           const int* d_hasv, const float* d_V, int is_train, float* d_gw_out, float* d_gV_out,
                           const SegDst* seg) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_dev_fm_step");
  DFB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int ks = h->tab.ks, k = h->prm.V_dim;
  if (nkeys > 0x7fffffffULL || nrows > 0x7fffffffULL || nnz > 0x7fffffffULL)
    return h->fail(DFB_ERR_INVALID, "batch too large");
  // the worker's dense gradient rows (launch_bwd_dense) exist at the exact widths only
  const bool sorted = is_train && h->sorted_path() && fast_lane_width(k) == k;
  DFB_TRY(h->ensure(h->pred, nrows * sizeof(float)));
  FmView v;
  memset(&v, 0, sizeof(v));
  v.wbase = d_w; v.w_pos = nullptr;
  v.vbase = d_V; v.v_pos = d_hasv; v.vstride = ks; v.dense = 1;
  float* gxxp = nullptr;
  if (is_train) {
    if (!d_gw_out || (k > 0 && !d_gV_out)) return h->fail(DFB_ERR_INVALID, "gradient outputs are NULL");
    if (sorted) {
      DFB_TRY(ensure_sorted_ws(h, nrows, nnz, nkeys, d_value != nullptr));
    } else {
      DFB_CUDA(h, cudaMemsetAsync(d_gw_out, 0, nkeys * sizeof(float), s));
      if (k > 0) DFB_CUDA(h, cudaMemsetAsync(d_gV_out, 0, nkeys * (size_t)ks * sizeof(float), s));
      if (k > 0 && d_value) {
        DFB_TRY(h->ensure(h->gxxp, nkeys * sizeof(float)));
        DFB_CUDA(h, cudaMemsetAsync(h->gxxp.p, 0, nkeys * sizeof(float), s));
        gxxp = h->gxxp.as<float>();
      }
      v.gwbase = d_gw_out; v.gvbase = d_gV_out; v.gvstride = ks; v.gxxp = gxxp;
    }
  }
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.nrows = nrows; b.offset = d_offset; b.index = d_index; b.value = d_value; b.label = d_label;
  b.pred_io = h->pred.as<float>(); b.V_dim = k; b.train = is_train; b.prog = h->tab.prog;
  b.long_nnz = (unsigned)h->long_row_nnz; b.nnz_hint = nnz;
  if (sorted) {
    b.emit = 1; b.p_out = h->p_row.as<float>(); b.pxv_out = h->pxv.as<float>();
    b.occ_row = h->occ.as<uint32_t>(); b.occ_rowx = h->occ.as<unsigned long long>();
  }
  if (nrows) {
    cudaError_t le = cudaSuccess;
    int nl = launch_fm(b, v, h->force_generic, s, &le);
    if (nl < 0) return fm_launch_fail(h, nl, le);
    h->launches += nl;
  }
  if (sorted) {
    {
      int nlc = launch_csc_build(d_index, h->occ.p, d_value != nullptr, nnz, nkeys, h->lidx_sorted.as<uint32_t>(),
                                 h->occ_sorted.p, h->col_start.as<int>(), h->col_end.as<int>(), h->cub.p,
                                 h->cub.bytes, h->tab.prog, s);
      if (nlc < 0) return h->fail(DFB_ERR_CUDA, "CSC sort of the batch failed (temporary storage)");
      h->launches += nlc;
    }
    // the penalty of the pulled weights (sgd_learner.cc:148) is accumulated by the same kernel
    int nl = launch_bwd_dense(h->prm, h->tab.prog, ks, d_w, d_hasv, nkeys, h->col_start.as<int>(),
                              h->col_end.as<int>(), h->occ_sorted.p, d_value != nullptr, h->p_row.as<float>(),
                              h->pxv.as<float>(), d_gw_out, d_V, d_gV_out, 1, seg, s);
    if (nl < 0) return h->fail(DFB_ERR_INVALID, "sorted scatter unsupported for this V_dim");
    h->launches += nl;
  } else if (is_train && k > 0) {
    // grad_V -= V_pulled * XXp (XXp == grad_w for binary data): the worker ships complete gradients
    h->launches += launch_grad_finalize_dense(k, ks, nkeys, d_hasv, d_V, gxxp ? gxxp : d_gw_out, d_gV_out, s);
  }
  if (h->compute_auc && nrows) {
    DFB_TRY(h->ensure(h->auc_k, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_v, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_tmp, sort_tmp_bytes(nrows)));
    h->launches += launch_auc(d_label, h->pred.as<float>(), nrows, h->auc_k.as<float>(),
                              h->auc_v.as<float>(), h->auc_tmp.p, h->auc_tmp.bytes, &h->tab.prog->auc, nullptr, s);
  }
  // the worker evaluates the penalty of what it pulled (sgd_learner.cc:148)
  if (!sorted) h->launches += launch_penalty(h->prm, h->tab.prog, d_w, d_hasv, d_V, ks, 1, nkeys, nullptr, s);
  DFB_CUDA(h, cudaGetLastError());
  return DFB_OK;
}

int dfb_dev_push_rows(dfb_handle h, const uint64_t* d_keys, size_t n, const float* d_gw, const int* d_hasv,
                      const float* d_gV) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_dev_push_rows");
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (n == 0) return DFB_OK;
  DFB_TRY(ensure_key_ws(h, n));
  DFB_TRY(dfbh::reserve(h, n, n));
  cudaStream_t s = h->stream;
  h->launches += launch_lookup(h->tab, d_keys, n, nullptr, true, h->slot.as<int>(), nullptr, nullptr, nullptr, s);
  int nl = h->force_generic ? -1 : launch_update_pushed(h->tab, h->prm, h->slot.as<int>(), d_hasv, n, d_gw, d_gV,
                                                        h->flags.as<int>(), s);
  if (nl < 0)
    nl = launch_update_dense(h->tab, h->prm, h->slot.as<int>(), d_hasv, 1, n, d_gw, nullptr, d_gV,
                             h->flags.as<int>(), 0, 0, s);
  h->launches += nl;
  h->launches += launch_initv(h->tab, h->prm, h->slot.as<int>(), n, nullptr, h->flags.as<int>(), h->pos.as<int>(), s);
  DFB_CUDA(h, cudaGetLastError());
  return DFB_OK;
}

}  // extern "C"
