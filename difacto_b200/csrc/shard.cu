// difacto_b200/csrc/shard.cu -- host side of the NVLink-sharded model store (dfb_shard_* of the C-ABI).
//
// Replaces, for the FM-SGD hot path, the worker/server exchange the reference was written for
// (src/sgd/sgd_learner.cc:78-89 + Store::Push/Pull over ps-lite KVWorker/KVServer,
// ps-lite/include/ps/kv_app.h:406-460; difacto's own distributed Store is LOG(FATAL) "not implemented",
// src/store/store.cc:9-11).  One engine per GPU is at the same time a WORKER (its own minibatch) and the
// OWNER of one contiguous range of the reversed key space (postoffice.cc:127-136).  See kernels_shard.cu
// for what crosses NVLink.  One step of every rank, all asynchronous, no host synchronisation:
//
//   stream W (worker)            stream O (owner = the engine's main stream)            stream F (finish)
//   localize raw ids (GPU)                 [stream L: slots of all workers' key segments (find / insert), beside
//   segment bounds, scatter the             the update of the previous step]
//   CSC/CSR slices -> owners  --struct-->  (feacnt,) pull {w, V row} of all workers' key segments
//                                          partial interaction sums of all workers' rows
//   add partials, pred/loss/p <--part----  (stored into the workers' mailboxes)
//   p, p*XV -> owners         --pxv----->  per worker, rank order: per-key gradient from its
//   AUC (aux stream)                       column lists + FTRL/AdaGrad in place, InitV     --done--> penalties,
//                                                                                          Progress snapshot
// W of step t+1 (localize, scatter) overlaps O of step t (update); mailbox slots are double-buffered by step
// parity.  Dependencies on the SAME GPU are CUDA events, dependencies on other GPUs are step counters in
// peer memory polled by one-warp kernels (with a timeout), so the FIFO order of the host's enqueues is
// deadlock-free whatever the stream-to-hardware-queue mapping is.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "engine_internal.cuh"
#include "shard_layout.cuh"

using namespace dfb;  // NOLINT

struct ShardState {
  int rank = 0, S = 1;
  ShardLayout lay;
  size_t Bcap = 0, Ncap = 0;
  void* mailbox = nullptr;
  void* peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool connected = false;
  cudaStream_t w_stream = nullptr, f_stream = nullptr, l_stream = nullptr;
  cudaEvent_t ev_struct[2] = {}, ev_part[2] = {}, ev_reduce[2] = {}, ev_auc[2] = {}, ev_upd[2] = {}, ev_fin[2] = {},
              ev_lookup[2] = {};
  cudaEvent_t ev_grow = nullptr;     // a rehash on stream O, which the lookup of the same step waits for
  uint64_t step = 0;
  dfb_engine::LocSet L;
  DevBuf wb, rowcnt, pred[2];    // wb: ShardBounds [2] by step parity (the AUC of step t reads it beside step t+1)
  DevBuf slot[2], conf[2];        // by step parity: the lookup of step t+1 runs beside the update of step t
  DevBuf w, vrow, wv, vsave, flags, ws;
  DevProgress* dprog = nullptr;   // device: [0,S) per-worker scratch, [S,S+2) worker Progress by parity, [S+2,S+4) staging
  long long timeout_cycles = 0;
  // the step being enqueued (dfb_shard_begin_* .. dfb_shard_phase(4))
  struct Ctx {
    bool open = false;
    int next_phase = 0;
    size_t nrows = 0, nnz = 0;
    const uint64_t* d_off = nullptr;
    const uint64_t* d_ids = nullptr;
    const float* d_val = nullptr;
    const float* d_lab = nullptr;
    int push_cnt = 0, is_train = 0;
    bool predict = false;            // a predict step (dfb_shard_*predict*): no penalty, label optional
    float* pred_out = nullptr;       // host: this rank's predictions, copied at the end of the step
    cudaEvent_t inputs_ready = nullptr, consumed = nullptr;
    LookupArgs la;
    bool auc = false;
  } cx;
  DevProgress* src_prog(int r) { return dprog + r; }
  DevProgress* prog_w(int d) { return dprog + S + d; }
  DevProgress* stage(int d) { return dprog + S + 2 + d; }
  ShardBounds* bounds(int d) { return wb.as<ShardBounds>() + d; }
};

namespace {

// DFB_DEBUG_SYNC=1: synchronise the device after every launch group of a sharded step and name the first one that
// faulted (debugging aid; the ranks still only wait for work that is already enqueued, see shard_phase)
bool dbg_on() {
  static const bool on = getenv("DFB_DEBUG_SYNC") != nullptr;
  return on;
}
#define DFB_DBG(h, tag)                                                                            \
  do {                                                                                             \
    if (dbg_on()) {                                                                                \
      cudaError_t _e = cudaDeviceSynchronize();                                                    \
      if (_e != cudaSuccess) return (h)->cuda_fail(_e, "sharded step, after " tag);                 \
    }                                                                                              \
  } while (0)

// predict: the step is a predict step (is_train = push_cnt = 0, label may be NULL); pred_out receives the rows'
// predictions at the end of the step
int shard_begin(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
                const float* d_val, const float* d_lab, int push_cnt, int is_train, cudaEvent_t inputs_ready,
                cudaEvent_t consumed, bool predict = false, float* pred_out = nullptr) {
  ShardState* shp = h->shard;
  if (!shp) return h->fail(DFB_ERR_INVALID, "dfb_shard_init was not called");
  ShardState& sh = *shp;
  if (!sh.connected) return h->fail(DFB_ERR_INVALID, "dfb_shard_connect was not called");
  if (sh.cx.open) return h->fail(DFB_ERR_INVALID, "the previous sharded step was not finished (dfb_shard_phase 0..4)");
  if (nrows > sh.Bcap || nnz > sh.Ncap) return h->fail(DFB_ERR_CAPACITY, "batch larger than dfb_shard_init's max_rows / max_nnz");
  if (is_train && !h->has_aux) return h->fail(DFB_ERR_INVALID, "no aux data");   // CHECK(has_aux_), sgd_updater.cc:75
  if (nrows && !d_lab && !predict) return h->fail(DFB_ERR_INVALID, "label is NULL");
  ShardState::Ctx& c = sh.cx;
  c.open = true; c.next_phase = 0;
  c.nrows = nrows; c.nnz = nnz; c.d_off = d_off; c.d_ids = d_ids; c.d_val = d_val; c.d_lab = d_lab;
  c.push_cnt = push_cnt; c.is_train = is_train; c.inputs_ready = inputs_ready; c.consumed = consumed;
  c.predict = predict; c.pred_out = pred_out;
  c.auc = h->compute_auc && nrows && d_lab;
  return DFB_OK;
}

// one of the five enqueue phases of a step (see the file header): 0 = W part 1, 1 = O part 1, 2 = W part 2 (+AUC),
// 3 = O part 2, 4 = F.  A host thread that drives several engines of ONE device must interleave the phases
// (phase p of every engine before phase p+1 of any), so that every wait refers to work enqueued earlier.
int shard_phase(dfb_engine* h, int phase) {
  ShardState* shp = h->shard;
  if (!shp || !shp->cx.open) return h->fail(DFB_ERR_INVALID, "no sharded step in progress (dfb_shard_begin_*)");
  ShardState& sh = *shp;
  ShardState::Ctx& c = sh.cx;
  if (phase != c.next_phase) return h->fail(DFB_ERR_INVALID, "dfb_shard_phase: phases must be called in order 0..4");
  c.next_phase++;
  const size_t nrows = c.nrows, nnz = c.nnz;
  const uint64_t* d_off = c.d_off;
  const uint64_t* d_ids = c.d_ids;
  const float* d_val = c.d_val;
  const float* d_lab = c.d_lab;
  const int push_cnt = c.push_cnt, is_train = c.is_train;
  cudaEvent_t inputs_ready = c.inputs_ready, consumed = c.consumed;
  LookupArgs& la = c.la;
  const ShardLayout& lay = sh.lay;
  const int S = sh.S, me = sh.rank, K = h->prm.V_dim, ks = h->tab.ks;
  const uint64_t t = sh.step;
  const int d = (int)(t & 1);
  const unsigned long long fv = t + 1;
  const bool valued = d_val != nullptr;      // of THIS rank's batch; on the wire every batch is valued (kernels_shard.cu)
  const unsigned remote = ((1u << S) - 1u) & ~(1u << me);
  cudaStream_t W = sh.w_stream, O = h->stream, A = h->aux_stream, F = sh.f_stream, L = sh.l_stream;
  void* mine = sh.mailbox;
  const size_t Kseg = lay.Kseg;

  const ShardHdr* hdr[8];
  for (int r = 0; r < S; ++r) hdr[r] = lay.at<ShardHdr>(mine, lay.off_hdr, lay.str_hdr, d, r);
  int* flags = sh.flags.as<int>();
  int* ws = sh.ws.as<int>();
  const bool auc = c.auc;

  if (phase == 0) {
  // ------------------------------- W part 1: localize, slice, scatter -------------------------------
  if (inputs_ready) DFB_CUDA(h, cudaStreamWaitEvent(W, inputs_ready, 0));
  if (t >= 2) DFB_CUDA(h, cudaStreamWaitEvent(W, sh.ev_fin[d], 0));     // parity slots of step t-2 are free again
  size_t Ucap = 0;
  if (h->profile && h->prof_steps && h->prof_steps % dfb_engine::kProfRing == 0) DFB_TRY(dfbh::prof_drain(h));
  DFB_TRY(h->ensure(sh.rowcnt, (size_t)S * (nrows + 1) * sizeof(int)));
  DFB_TRY(h->ensure(sh.pred[d], (nrows ? nrows : 1) * sizeof(float)));
  // a dropped batch makes no prediction (k_shard_reduce returns at once): its rows read 0
  if (c.pred_out && nrows) DFB_CUDA(h, cudaMemsetAsync(sh.pred[d].p, 0, nrows * sizeof(float), W));
  {
    StageTimer tm(h, 5, W);
    // a dropped batch (range, or a segment over its capacity below) is reported into this step's own Progress slot:
    // the engine-wide one may still be read by the previous step's snapshot, which runs beside this stream
    DFB_TRY(dfbh::localize_dev(h, nrows, nnz, d_off, d_ids, d_val, ~0ULL, sh.L, W, false, false, &Ucap, sh.prog_w(d)));   // Localizer(-1), sgd_learner.cc:203
  }
  DFB_DBG(h, "localize");
  StageTimer tm_slice(h, 6, W);
  ShardBounds* wb = sh.bounds(d);
  h->launches += launch_shard_bounds(sh.L.keys.as<uint64_t>(), sh.L.dU(), Ucap, sh.L.col_start.as<int>(), nnz, S, Kseg,
                                     lay.Nseg, wb, sh.prog_w(d), W);
  {
    ScatterArgs a;
    memset(&a, 0, sizeof(a));
    a.S = S; a.me = me; a.wb = wb; a.keys = sh.L.keys.as<uint64_t>(); a.col_start = sh.L.col_start.as<int>();
    a.occ = sh.L.occ_sorted.p; a.nrows = nrows;
    a.flags = (is_train ? 1ULL : 0ULL) | (push_cnt ? 2ULL : 0ULL) | (valued ? 4ULL : 0ULL);
    a.step = fv;
    RowptrDst rd;
    FillDst fd;
    memset(&rd, 0, sizeof(rd));
    memset(&fd, 0, sizeof(fd));
    for (int s = 0; s < S; ++s) {
      a.hdr_dst[s] = lay.at<ShardHdr>(sh.peer[s], lay.off_hdr, lay.str_hdr, d, me);
      a.keys_dst[s] = lay.at<uint64_t>(sh.peer[s], lay.off_keys, lay.str_keys, d, me);
      a.cstart_dst[s] = lay.at<int>(sh.peer[s], lay.off_cstart, lay.str_cstart, d, me);
      a.occ_dst[s] = lay.at<void>(sh.peer[s], lay.off_occ, lay.str_occ, d, me);
      rd.rowptr_dst[s] = lay.at<uint64_t>(sh.peer[s], lay.off_rowptr, lay.str_rowptr, d, me);
      fd.ridx_dst[s] = lay.at<uint32_t>(sh.peer[s], lay.off_ridx, lay.str_ridx, d, me);
      fd.rval_dst[s] = lay.at<float>(sh.peer[s], lay.off_rval, lay.str_rval, d, me);
    }
    DFB_DBG(h, "bounds");
    h->launches += launch_shard_scatter(a, valued, nnz ? nnz : 1, W);
    DFB_DBG(h, "scatter");
    h->launches += launch_shard_subcsr(d_off, sh.L.lidx.as<uint32_t>(), d_val, nrows, wb, S, sh.rowcnt.as<int>(), rd, fd, W);
  }
  DFB_DBG(h, "subcsr");
  tm_slice.stop();
  {
    SignalDst sd;
    memset(&sd, 0, sizeof(sd));
    sd.n = S;
    for (int s = 0; s < S; ++s) sd.flag[s] = s == me ? nullptr : lay.flag(sh.peer[s], ShardLayout::F_STRUCT, me);
    if (remote) h->launches += launch_shard_signal(sd, fv, W);
  }
  DFB_CUDA(h, cudaEventRecord(sh.ev_struct[d], W));
  }

  if (phase == 1) {
  // ------------------------------- O part 1: lookup, pull, partial interaction sums -------------------------------
  // (a) stream L: the slots of all workers' key segments (find / insert) and which keys several workers share --
  // needs only the workers' structure, so it runs beside the update of the previous step on stream O
  DFB_CUDA(h, cudaStreamWaitEvent(L, sh.ev_struct[d], 0));
  if (t >= 2) DFB_CUDA(h, cudaStreamWaitEvent(L, sh.ev_fin[d], 0));        // slot[d] / conf[d] of step t-2 are free
  h->launches += launch_shard_wait(lay.flag(mine, ShardLayout::F_STRUCT, 0), 8, remote, fv, sh.timeout_cycles, h->tab.prog, L);
  memset(&la, 0, sizeof(la));
  la.S = S; la.Kseg = Kseg;
  la.stamp = (is_train && S > 1) ? (unsigned)((fv & 0xFFFFFFULL) ? (fv & 0xFFFFFFULL) : 1ULL) : 0u;
  la.slot = sh.slot[d].as<int>(); la.w = sh.w.as<float>(); la.vrow = sh.vrow.as<int>(); la.wv = sh.wv.as<int2>();
  for (int r = 0; r < S; ++r) {
    la.hdr[r] = hdr[r];
    la.keys[r] = lay.at<uint64_t>(mine, lay.off_keys, lay.str_keys, d, r);
  }
  if (is_train || push_cnt) {
    // a growing owner: count the keys this step brings (all workers' segments are in place after the poller), grow
    // before they are inserted.  A rehash runs on stream O after the previous step's update, which still addresses
    // the old slots; this step's lookup and everything after it take the new table.
    unsigned long long* rcv = nullptr;
    DFB_TRY(dfbh::shard_rcv_slot(h, &rcv));
    if (rcv) {
      h->launches += launch_shard_count(la, rcv, L);
      bool rehashed = false;
      DFB_TRY(dfbh::reserve_shard(h, L, (uint64_t)S * Kseg, is_train != 0, &rehashed));
      if (rehashed) {
        DFB_CUDA(h, cudaEventRecord(sh.ev_grow, O));
        DFB_CUDA(h, cudaStreamWaitEvent(L, sh.ev_grow, 0));
      }
    }
  }
  {
    StageTimer tm_lk(h, 0, L);
    // a validation / prediction batch must not grow the table (a missing entry reads as w = 0, no V)
    for (int r = 0; r < S; ++r)
      h->launches += launch_shard_lookup(h->tab, la, r, is_train || push_cnt, sh.conf[d].as<unsigned char>(), L);
  }
  DFB_CUDA(h, cudaEventRecord(sh.ev_lookup[d], L));
  DFB_DBG(h, "lookup");
  // (b) stream O, after the previous step's update: Push(kFeaCount) before Pull (sgd_learner.cc:214-217; one Update
  // per worker, rank order), the Pull itself, the partial sums
  DFB_CUDA(h, cudaStreamWaitEvent(O, sh.ev_lookup[d], 0));
  StageTimer tm_fwd(h, 7, O);
  if (push_cnt) {
    for (int r = 0; r < S; ++r)
      h->launches += launch_feacnt(h->tab, h->prm, la.slot + (size_t)r * Kseg, Kseg, &hdr[r]->nkeys, nullptr,
                                   lay.at<int>(mine, lay.off_cstart, lay.str_cstart, d, r), flags, ws, O);
  }
  h->launches += launch_shard_pull(h->tab, la, sh.conf[d].as<unsigned char>(), sh.vsave.as<float>(), O);
  DFB_DBG(h, "feacnt / pull view");
  {
    PartArgs pa;
    memset(&pa, 0, sizeof(pa));
    pa.nsrc = S; pa.rot = me; pa.bcap = sh.Bcap;
    for (int r = 0; r < S; ++r) {
      pa.s[r].rowptr = lay.at<uint64_t>(mine, lay.off_rowptr, lay.str_rowptr, d, r);
      pa.s[r].ridx = lay.at<uint32_t>(mine, lay.off_ridx, lay.str_ridx, d, r);
      pa.s[r].rval = lay.at<float>(mine, lay.off_rval, lay.str_rval, d, r);
      pa.s[r].wv = la.wv + (size_t)r * Kseg;
      pa.s[r].hdr = hdr[r];
      pa.s[r].out_xv = lay.at<float>(sh.peer[r], lay.off_part_xv, lay.str_part_xv, d, me);
      pa.s[r].out_sc = lay.at<float2>(sh.peer[r], lay.off_part_sc, lay.str_part_sc, d, me);
    }
    FmView v;
    memset(&v, 0, sizeof(v));
    v.vbase = h->tab.V; v.vstride = h->tab.rs; v.l2hint = h->l2_hints; v.wv_last = h->l2_hints;
    int nl = launch_fm_partial(K, true, h->tab.vonly == 2, v, pa, O);
    if (nl < 0) return h->fail(DFB_ERR_INVALID, "unsupported V_dim for the sharded store");
    h->launches += nl;
  }
  DFB_DBG(h, "partial sums");
  tm_fwd.stop();
  {
    SignalDst sd;
    memset(&sd, 0, sizeof(sd));
    sd.n = S;
    for (int r = 0; r < S; ++r) sd.flag[r] = r == me ? nullptr : lay.flag(sh.peer[r], ShardLayout::F_PART, me);
    if (remote) h->launches += launch_shard_signal(sd, fv, O);
  }
  DFB_CUDA(h, cudaEventRecord(sh.ev_part[d], O));
  }

  if (phase == 2) {
  // ------------------------------- W part 2: reduce the partials, p and p*XV back -------------------------------
  DFB_CUDA(h, cudaStreamWaitEvent(W, sh.ev_part[d], 0));
  h->launches += launch_shard_wait(lay.flag(mine, ShardLayout::F_PART, 0), 8, remote, fv, sh.timeout_cycles, h->tab.prog, W);
  {
    StageTimer tm_red(h, 8, W);
    ReduceArgs ra;
    memset(&ra, 0, sizeof(ra));
    ra.S = S; ra.me = me; ra.train = is_train ? 1 : 0; ra.V_dim = K; ra.nrows = nrows; ra.wb = sh.bounds(d);
    for (int s = 0; s < S; ++s) {
      ra.part_xv[s] = lay.at<float>(mine, lay.off_part_xv, lay.str_part_xv, d, s);
      ra.part_sc[s] = lay.at<float2>(mine, lay.off_part_sc, lay.str_part_sc, d, s);
      ra.p_dst[s] = lay.at<float>(sh.peer[s], lay.off_p, lay.str_p, d, me);
      ra.pxv_dst[s] = lay.at<float>(sh.peer[s], lay.off_pxv, lay.str_pxv, d, me);
    }
    ra.label = d_lab; ra.pred = sh.pred[d].as<float>(); ra.prog = sh.prog_w(d);
    int nl = launch_shard_reduce(ra, W);
    if (nl < 0) return h->fail(DFB_ERR_INVALID, "unsupported V_dim for the sharded store");
    h->launches += nl;
    DFB_DBG(h, "reduce");
  }
  {
    SignalDst sd;
    memset(&sd, 0, sizeof(sd));
    sd.n = S;
    for (int s = 0; s < S; ++s) sd.flag[s] = s == me ? nullptr : lay.flag(sh.peer[s], ShardLayout::F_PXV, me);
    if (remote) h->launches += launch_shard_signal(sd, fv, W);
  }
  DFB_CUDA(h, cudaEventRecord(sh.ev_reduce[d], W));
  if (auc) {
    DFB_TRY(h->ensure(h->auc_k, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_v, nrows * sizeof(float)));
    DFB_TRY(h->ensure(h->auc_tmp, sort_tmp_bytes(nrows)));
    DFB_CUDA(h, cudaStreamWaitEvent(A, sh.ev_reduce[d], 0));
    // a dropped batch made no prediction: ShardBounds::valid == 0 makes the AUC add nothing
    h->launches += launch_auc(d_lab, sh.pred[d].as<float>(), nrows, h->auc_k.as<float>(), h->auc_v.as<float>(),
                              h->auc_tmp.p, h->auc_tmp.bytes, &sh.prog_w(d)->auc, &sh.bounds(d)->valid, A);
    DFB_CUDA(h, cudaEventRecord(sh.ev_auc[d], A));
  }
  }

  if (phase == 3) {
  // ------------------------------- O part 2: one Update per worker, rank order -------------------------------
  StageTimer tm_upd(h, 9, O);
  // the InitV requests of all workers' updates: flags[S][Kseg], zero where no key is (one pass after the last update)
  if (is_train) DFB_CUDA(h, cudaMemsetAsync(flags, 0, (size_t)S * Kseg * sizeof(int), O));
  DFB_DBG(h, "flags memset");
  for (int r = 0; r < S; ++r) {
    if (r == me) DFB_CUDA(h, cudaStreamWaitEvent(O, sh.ev_reduce[d], 0));
    else h->launches += launch_shard_wait(lay.flag(mine, ShardLayout::F_PXV, r), 8, 1u, fv, sh.timeout_cycles, h->tab.prog, O);
    DFB_DBG(h, "wait for a worker's p*XV");
    const size_t o = (size_t)r * Kseg;
    const int* cstart = lay.at<int>(mine, lay.off_cstart, lay.str_cstart, d, r);
    if (is_train) {
      Table tt = h->tab;
      tt.prog = sh.src_prog(r);
      ShardApply ap;
      ap.w_pulled = la.w + o;
      ap.conf = la.stamp ? sh.conf[d].as<unsigned char>() + o : nullptr;
      ap.vsave = sh.vsave.as<float>() + o * (size_t)ks;
      const void* occ_r = lay.at<void>(mine, lay.off_occ, lay.str_occ, d, r);
      const float* p_r = lay.at<float>(mine, lay.off_p, lay.str_p, d, r);
      const float* pxv_r = lay.at<float>(mine, lay.off_pxv, lay.str_pxv, d, r);
      HotWs hws;
      HotPart hp;
      DFB_TRY(dfbh::hot_ws(h, Kseg, lay.Nseg, &hws));
      h->launches += launch_hot_prereduce(K, Kseg, &hdr[r]->nkeys, cstart, cstart + 1, occ_r, true, p_r, pxv_r,
                                          h->hot_split, hws, &hp, 0, O);
      DFB_DBG(h, "hot-key pre-reduction");
      int nl = launch_bwd_update(tt, h->prm, nullptr, la.slot + o, la.vrow + o, Kseg, &hdr[r]->nkeys, cstart, cstart + 1,
                                 occ_r, true, p_r, pxv_r, flags + o, 1, &ap, hp.part ? &hp : nullptr, 0, O);
      if (nl < 0) return h->fail(DFB_ERR_INVALID, "unsupported V_dim for the sharded store");
      h->launches += nl;
    } else if (!c.predict) {      // (a predict step is collective: every worker's Progress has penalty 0)
      h->launches += launch_penalty(h->prm, sh.src_prog(r), la.w + o, la.vrow + o, h->tab.V, h->tab.rs, 0, Kseg,
                                    &hdr[r]->nkeys, O);
    }
    DFB_DBG(h, "update of one worker");
    h->launches += launch_shard_done(sh.src_prog(r), h->tab.prog, lay.at<double>(sh.peer[r], lay.off_pen, lay.str_pen, d, me),
                                     lay.flag(sh.peer[r], ShardLayout::F_DONE, me), fv, O);
    DFB_DBG(h, "done signal");
  }
  // InitV (sgd_updater.cc:121-126,140-147) for the keys whose w left zero, in worker-major key order -- the order in
  // which the reference's server would have met them
  if (is_train) h->launches += launch_initv(h->tab, h->prm, la.slot, (size_t)S * Kseg, nullptr, flags, ws, O);
  DFB_DBG(h, "InitV");
  if (is_train || push_cnt) DFB_TRY(dfbh::shard_counts_copy(h));
  tm_upd.stop();
  DFB_CUDA(h, cudaEventRecord(sh.ev_upd[d], O));
  }

  if (phase == 4) {
  // ------------------------------- F: penalties back, Progress snapshot -------------------------------
  DFB_CUDA(h, cudaStreamWaitEvent(F, sh.ev_reduce[d], 0));
  if (auc) DFB_CUDA(h, cudaStreamWaitEvent(F, sh.ev_auc[d], 0));
  DFB_CUDA(h, cudaStreamWaitEvent(F, sh.ev_upd[d], 0));
  h->launches += launch_shard_wait(lay.flag(mine, ShardLayout::F_DONE, 0), 8, remote, fv, sh.timeout_cycles, h->tab.prog, F);
  DFB_DBG(h, "done flags");
  h->launches += launch_shard_collect(lay.at<double>(mine, lay.off_pen, lay.str_pen, d, 0), (int)(lay.str_pen / 8), S,
                                      sh.prog_w(d), h->tab.prog, sh.stage(d), F);
  if (h->submitted - h->collected == (uint64_t)dfb_engine::kRing) DFB_TRY(dfbh::collect_one(h, &h->backlog));
  const int rs = (int)(h->submitted % dfb_engine::kRing);
  DFB_CUDA(h, cudaMemcpyAsync(&h->h_ring[rs], sh.stage(d), sizeof(DevProgress), cudaMemcpyDeviceToHost, F));
  if (c.pred_out && nrows)
    DFB_CUDA(h, cudaMemcpyAsync(c.pred_out, sh.pred[d].p, nrows * sizeof(float), cudaMemcpyDeviceToHost, F));
  DFB_CUDA(h, cudaEventRecord(h->ring_done[rs], F));
  h->submitted++;
  DFB_CUDA(h, cudaEventRecord(sh.ev_fin[d], F));
  if (consumed) DFB_CUDA(h, cudaEventRecord(consumed, F));
  sh.step++;
  c.open = false;
  if (h->profile) h->prof_steps++;
  }
  DFB_CUDA(h, cudaGetLastError());
  return DFB_OK;
}

int shard_step(dfb_engine* h, size_t nrows, size_t nnz, const uint64_t* d_off, const uint64_t* d_ids,
               const float* d_val, const float* d_lab, int push_cnt, int is_train, cudaEvent_t inputs_ready,
               cudaEvent_t consumed) {
  DFB_TRY(shard_begin(h, nrows, nnz, d_off, d_ids, d_val, d_lab, push_cnt, is_train, inputs_ready, consumed));
  for (int ph = 0; ph < 5; ++ph) {
    int rc = shard_phase(h, ph);
    if (rc != 0) { h->shard->cx.open = false; return rc; }
  }
  return DFB_OK;
}

}  // namespace

void dfbh::shard_destroy(dfb_engine* h) {
  ShardState* sh = h->shard;
  if (!sh) return;
  if (sh->w_stream) cudaStreamDestroy(sh->w_stream);
  if (sh->f_stream) cudaStreamDestroy(sh->f_stream);
  if (sh->l_stream) cudaStreamDestroy(sh->l_stream);
  if (sh->ev_grow) cudaEventDestroy(sh->ev_grow);
  cudaEvent_t* evs[] = {sh->ev_struct, sh->ev_part, sh->ev_reduce, sh->ev_auc, sh->ev_upd, sh->ev_fin, sh->ev_lookup};
  for (auto* e : evs) for (int i = 0; i < 2; ++i) if (e[i]) cudaEventDestroy(e[i]);
  DevBuf* bufs[] = {&sh->L.keys, &sh->L.lidx, &sh->L.cnt, &sh->L.occ_sorted, &sh->L.col_start, &sh->L.col_end, &sh->L.scal,
                    &sh->wb, &sh->rowcnt, &sh->pred[0], &sh->pred[1], &sh->slot[0], &sh->slot[1], &sh->w, &sh->vrow, &sh->wv, &sh->conf[0],
                    &sh->conf[1],
                    &sh->vsave, &sh->flags, &sh->ws};
  for (auto* b : bufs) if (b->p) cudaFree(b->p);
  if (sh->dprog) cudaFree(sh->dprog);
  if (sh->mailbox) cudaFree(sh->mailbox);
  delete sh;
  h->shard = nullptr;
}

int dfbh::shard_sync(dfb_engine* h) {
  ShardState* sh = h->shard;
  if (!sh) return DFB_OK;
  DFB_CUDA(h, cudaStreamSynchronize(sh->w_stream));
  DFB_CUDA(h, cudaStreamSynchronize(sh->l_stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->aux_stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(sh->f_stream));
  return DFB_OK;
}

bool dfbh::shard_step_open(const dfb_engine* h) { return h->shard && h->shard->cx.open; }

extern "C" {

int dfb_shard_init(dfb_handle h, int rank, int nranks, size_t max_rows, size_t max_nnz, size_t seg_keys,
                   size_t seg_nnz, size_t* mailbox_bytes) {
  if (!h) return DFB_ERR_INVALID;
  if (h->shard) return h->fail(DFB_ERR_INVALID, "dfb_shard_init was already called");
  if (nranks < 1 || nranks > 8 || rank < 0 || rank >= nranks) return h->fail(DFB_ERR_INVALID, "1 <= nranks <= 8, 0 <= rank < nranks");
  if (max_rows == 0 || max_nnz == 0 || max_nnz > 0x7fffffffULL || max_rows > 0x7fffffffULL)
    return h->fail(DFB_ERR_INVALID, "max_rows / max_nnz out of range");
  // a scoring engine on its own already scores its whole model with dfb_predict_raw_*: a one-rank store would only add
  // the store's workspaces
  if (h->score_only && nranks < 2)
    return h->fail(DFB_ERR_INVALID, "dfb_shard_init: a score_only = 1 engine is a rank of a store of nranks >= 2 (on "
                                    "its own it scores with dfb_predict_raw_*)");
  const int ks = h->tab.ks;
  if (!h->sorted_path())
    return h->fail(DFB_ERR_INVALID, "the fused sharded store needs V_dim in 0..128, scatter=sorted and no force_generic "
                                    "(other configurations: the all_to_all ShardedStore)");
  // a growing rank bounds each step's insertions by the keys its owner received, counted on the device
  // (shard_growth = 1, growth.cu); without that opt-in the store keeps fixed capacities.  A scoring rank's predict
  // steps never insert: it grows only in dfb_restore*, which runs between steps.
  if (h->grow.on && !h->shard_growth && !h->score_only)
    return h->fail(DFB_ERR_INVALID, "the fused sharded store does not grow its shards: create the engine with "
                                    "table_capacity_max = table_capacity and V_capacity_max = V_capacity, or with "
                                    "shard_growth = 1");
  DFB_CUDA(h, cudaSetDevice(h->device));
  ShardState* sh = new ShardState();
  h->shard = sh;
  sh->rank = rank; sh->S = nranks; sh->Bcap = max_rows; sh->Ncap = max_nnz;
  // capacity of one (worker, owner) segment: everything for one rank, else twice the even share (skew margin)
  auto seg_default = [&](size_t total) { return nranks == 1 ? total : std::min(total, 2 * total / (size_t)nranks + 4096); };
  const size_t Kseg = seg_keys ? std::min(seg_keys, max_nnz) : seg_default(max_nnz);
  const size_t Nseg = seg_nnz ? std::min(seg_nnz, max_nnz) : seg_default(max_nnz);
  sh->lay.compute(nranks, ks, max_rows, Kseg, Nseg);
  sh->timeout_cycles = h->shard_timeout_ms * 2000000LL;
  auto fail = [&](int rc) { dfbh::shard_destroy(h); return rc; };
  cudaError_t e;
  if ((e = cudaMalloc(&sh->mailbox, sh->lay.total)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaMalloc(shard mailbox)"));
  if ((e = cudaMemset(sh->mailbox, 0, sh->lay.total)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaMemset(shard mailbox)"));
  sh->peer[rank] = sh->mailbox;
  // the worker stream (localize / scatter of the NEXT step) and the lookup stream run beside the owner's update of
  // the current step on the engine's main stream: give them the higher priority, or the update's CTAs (queued
  // first) would take every SM slot that frees up and the overlap would not happen
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if ((e = cudaStreamCreateWithPriority(&sh->w_stream, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaStreamCreate"));
  if ((e = cudaStreamCreateWithFlags(&sh->f_stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaStreamCreate"));
  if ((e = cudaStreamCreateWithPriority(&sh->l_stream, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaStreamCreate"));
  cudaEvent_t* evs[] = {sh->ev_struct, sh->ev_part, sh->ev_reduce, sh->ev_auc, sh->ev_upd, sh->ev_fin, sh->ev_lookup};
  for (auto* ev : evs)
    for (int i = 0; i < 2; ++i)
      if ((e = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaEventCreate"));
  if ((e = cudaEventCreateWithFlags(&sh->ev_grow, cudaEventDisableTiming)) != cudaSuccess) return fail(h->cuda_fail(e, "cudaEventCreate"));
  const size_t tot = (size_t)nranks * Kseg;
  // a scoring rank (score_only = 1) runs predict steps only: it has no InitV requests (flags, ws), no pull-time V rows
  // to save for the updates (conf, vsave) and no hot keys to pre-reduce.  Its mailbox is a training rank's: the peers
  // address it without knowing which kind it is.
  const bool train = !h->score_only;
  int rc = 0;
  if ((rc = h->ensure(sh->wb, 2 * sizeof(ShardBounds))) || (rc = h->ensure(sh->slot[0], tot * 4)) || (rc = h->ensure(sh->slot[1], tot * 4)) || (rc = h->ensure(sh->w, tot * 4)) ||
      (rc = h->ensure(sh->vrow, tot * 4)) || (rc = h->ensure(sh->wv, tot * 8)))
    return fail(rc);
  if (train && ((rc = h->ensure(sh->flags, tot * 4)) || (rc = h->ensure(sh->ws, (tot / 32 + 64) * 4))))
    return fail(rc);
  if (train && nranks > 1 && ((rc = h->ensure(sh->conf[0], tot)) || (rc = h->ensure(sh->conf[1], tot)) ||
                              (rc = h->ensure(sh->vsave, tot * (size_t)ks * 4))))
    return fail(rc);
  // Every workspace a step can touch is allocated NOW, for the declared capacities: a cudaMalloc / cudaFree in the
  // middle of a step is not just slow -- with peer access enabled it synchronises the peer devices, whose pollers
  // may be waiting for the very step this rank has not finished enqueuing (ranks that are threads of one process).
  {
    const size_t n1 = max_nnz, B = max_rows;
    DevBuf* nnz8[] = {&h->l_rkeys, &h->l_skeys, &h->l_pay, &h->l_spay, &sh->L.keys, &sh->L.occ_sorted};
    DevBuf* nnz4[] = {&sh->L.lidx, &sh->L.cnt, &sh->L.col_end};
    for (auto* b : nnz8) if ((rc = h->ensure(*b, n1 * 8))) return fail(rc);
    for (auto* b : nnz4) if ((rc = h->ensure(*b, n1 * 4))) return fail(rc);
    HotWs hws;
    if ((rc = h->ensure(sh->L.col_start, (n1 + 1) * 4)) || (rc = h->ensure(sh->L.scal, 16)) ||
        (rc = h->ensure(h->l_tmp, localize_sort_tmp_bytes(n1))) || (rc = h->ensure(sh->rowcnt, (size_t)nranks * (B + 1) * 4)) ||
        (rc = h->ensure(sh->pred[0], B * 4)) || (rc = h->ensure(sh->pred[1], B * 4)) || (rc = h->ensure(h->auc_k, B * 4)) ||
        (rc = h->ensure(h->auc_v, B * 4)) || (rc = h->ensure(h->auc_tmp, sort_tmp_bytes(B))) ||
        (train && (rc = dfbh::hot_ws(h, Kseg, Nseg, &hws))))
      return fail(rc);
    for (auto& in : h->in)
      if ((rc = h->ensure(in.off, (B + 1) * 8)) || (rc = h->ensure(in.ids, n1 * 8)) || (rc = h->ensure(in.val, n1 * 4)) ||
          (rc = h->ensure(in.lab, B * 4)))
        return fail(rc);
  }
  const size_t np = (size_t)nranks + 4;
  if ((e = cudaMalloc(&sh->dprog, np * sizeof(DevProgress))) != cudaSuccess) return fail(h->cuda_fail(e, "cudaMalloc"));
  if ((e = cudaMemset(sh->dprog, 0, np * sizeof(DevProgress))) != cudaSuccess) return fail(h->cuda_fail(e, "cudaMemset"));
  sh->connected = nranks == 1;
  if (mailbox_bytes) *mailbox_bytes = sh->lay.total;
  // cudaMemset of device memory is asynchronous: the zeroed mailbox must be in place before any peer may store into it
  if ((e = cudaDeviceSynchronize()) != cudaSuccess) return fail(h->cuda_fail(e, "cudaDeviceSynchronize"));
  return DFB_OK;
}

int dfb_shard_export(dfb_handle h, void** mailbox_ptr, unsigned char* handle64) {
  if (!h || !h->shard) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (mailbox_ptr) *mailbox_ptr = h->shard->mailbox;
  if (handle64) {
    cudaIpcMemHandle_t mh;
    DFB_CUDA(h, cudaIpcGetMemHandle(&mh, h->shard->mailbox));
    memcpy(handle64, &mh, 64);
  }
  return DFB_OK;
}

int dfb_shard_connect(dfb_handle h, void* const* peer_mailbox) {
  if (!h || !h->shard || !peer_mailbox) return DFB_ERR_INVALID;
  ShardState& sh = *h->shard;
  DFB_CUDA(h, cudaSetDevice(h->device));
  for (int s = 0; s < sh.S; ++s) {
    if (s == sh.rank) continue;
    if (!peer_mailbox[s]) return h->fail(DFB_ERR_INVALID, "peer mailbox pointer is NULL");
    sh.peer[s] = peer_mailbox[s];
    cudaPointerAttributes at;
    cudaError_t pe = cudaPointerGetAttributes(&at, peer_mailbox[s]);
    if (pe != cudaSuccess) return h->cuda_fail(pe, "cudaPointerGetAttributes(peer mailbox)");
    if (at.type != cudaMemoryTypeDevice) return h->fail(DFB_ERR_INVALID, "peer mailbox is not device memory");
    if (at.device != h->device) {
      int can = 0;
      DFB_CUDA(h, cudaDeviceCanAccessPeer(&can, h->device, at.device));
      if (!can) return h->fail(DFB_ERR_INVALID, "this GPU cannot access the peer GPU's memory");
      cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);     // same-process peers; IPC mappings enabled it already
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return h->cuda_fail(e, "cudaDeviceEnablePeerAccess");
      cudaGetLastError();
    }
  }
  sh.connected = true;
  DFB_CUDA(h, cudaDeviceSynchronize());
  return DFB_OK;
}

int dfb_shard_step_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                       const float* d_value_or_null, const float* d_label, int push_cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_shard_step_dev");
  DFB_CUDA(h, cudaSetDevice(h->device));
  return shard_step(h, nrows, nnz, d_offset, d_ids, d_value_or_null, d_label, push_cnt, is_train, nullptr, nullptr);
}

int dfb_shard_step_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                         const float* label, int push_cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_shard_step_async");
  DFB_TRY(dfbh::check_csr(h, nrows, offset));
  if (nrows && !label) return h->fail(DFB_ERR_INVALID, "label is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !ids) return h->fail(DFB_ERR_INVALID, "ids is NULL");
  auto& in = h->in[h->seq & 1];
  if (!in.prefetched(ids, label, nrows, nnz)) DFB_TRY(dfbh::stage_raw(h, in, nrows, nnz, offset, ids, value, label));
  in.pre_ids = nullptr;
  int rc = shard_step(h, nrows, nnz, in.off.as<uint64_t>(), in.ids.as<uint64_t>(), value ? in.val.as<float>() : nullptr,
                      in.lab.as<float>(), push_cnt, is_train, in.copied, in.consumed);
  h->seq++;
  return rc;
}

int dfb_shard_begin_dev(dfb_handle h, size_t nrows, size_t nnz, const uint64_t* d_offset, const uint64_t* d_ids,
                        const float* d_value_or_null, const float* d_label, int push_cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_shard_begin_dev");
  DFB_CUDA(h, cudaSetDevice(h->device));
  return shard_begin(h, nrows, nnz, d_offset, d_ids, d_value_or_null, d_label, push_cnt, is_train, nullptr, nullptr);
}

int dfb_shard_begin_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                          const float* label, int push_cnt, int is_train) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_shard_begin_async");
  DFB_TRY(dfbh::check_csr(h, nrows, offset));
  if (nrows && !label) return h->fail(DFB_ERR_INVALID, "label is NULL");
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !ids) return h->fail(DFB_ERR_INVALID, "ids is NULL");
  auto& in = h->in[h->seq & 1];
  if (!(in.pre_ids == ids && ids && in.pre_nrows == nrows && in.pre_nnz == nnz))
    DFB_TRY(dfbh::stage_raw(h, in, nrows, nnz, offset, ids, value, label));
  in.pre_ids = nullptr;
  int rc = shard_begin(h, nrows, nnz, in.off.as<uint64_t>(), in.ids.as<uint64_t>(), value ? in.val.as<float>() : nullptr,
                       in.lab.as<float>(), push_cnt, is_train, in.copied, in.consumed);
  h->seq++;
  return rc;
}

}  // extern "C"

namespace {
// the host-buffer predict step: staged through the double-buffered input sets like dfb_shard_begin_async
int shard_begin_predict(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                        const float* label, float* pred_out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_TRY(dfbh::check_csr(h, nrows, offset));
  DFB_CUDA(h, cudaSetDevice(h->device));
  const size_t nnz = nrows ? (size_t)offset[nrows] : 0;
  if (nnz && !ids) return h->fail(DFB_ERR_INVALID, "ids is NULL");
  auto& in = h->in[h->seq & 1];
  if (!in.prefetched(ids, label, nrows, nnz)) DFB_TRY(dfbh::stage_raw(h, in, nrows, nnz, offset, ids, value, label));
  in.pre_ids = nullptr;
  int rc = shard_begin(h, nrows, nnz, in.off.as<uint64_t>(), in.ids.as<uint64_t>(), value ? in.val.as<float>() : nullptr,
                       label ? in.lab.as<float>() : nullptr, 0, 0, in.copied, in.consumed, true, pred_out);
  h->seq++;
  return rc;
}
}  // namespace

extern "C" {

int dfb_shard_begin_predict_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids,
                                  const float* value, const float* label, float* pred_out) {
  return shard_begin_predict(h, nrows, offset, ids, value, label, pred_out);
}

int dfb_shard_predict_async(dfb_handle h, size_t nrows, const uint64_t* offset, const uint64_t* ids, const float* value,
                            const float* label, float* pred_out) {
  DFB_TRY(shard_begin_predict(h, nrows, offset, ids, value, label, pred_out));
  for (int ph = 0; ph < 5; ++ph) {
    int rc = shard_phase(h, ph);
    if (rc != 0) { h->shard->cx.open = false; return rc; }
  }
  return DFB_OK;
}

int dfb_shard_phase(dfb_handle h, int phase) {
  if (!h) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  return shard_phase(h, phase);
}

int dfb_shard_info(dfb_handle h, int* rank, int* nranks, size_t* seg_keys, size_t* seg_nnz, uint64_t* steps) {
  if (!h || !h->shard) return DFB_ERR_INVALID;
  if (rank) *rank = h->shard->rank;
  if (nranks) *nranks = h->shard->S;
  if (seg_keys) *seg_keys = h->shard->lay.Kseg;
  if (seg_nnz) *seg_nnz = h->shard->lay.Nseg;
  if (steps) *steps = h->shard->step;
  return DFB_OK;
}

}  // extern "C"
