// difacto_b200/host/src/sgd_learner.cc -- see sgd_learner.h.  Control flow follows
// src/sgd/sgd_learner.cc of the reference (cited per function); the arithmetic lives on the GPU.
#include "difacto_b200/sgd_learner.h"

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <thread>

namespace difacto {

Loss* Loss::Create(const std::string& type, int nthreads) {   // src/loss/loss.cc:13-26
  if (type != "fm") throw Error("unknown loss type: " + type + " (the GPU engine provides \"fm\")");
  Loss* l = new GpuFMLoss();
  l->set_nthreads(nthreads);
  return l;
}

Store* Store::Create() { return new GpuStore(); }   // src/store/store.cc:8-15

Learner* Learner::Create(const std::string& type) {   // src/learner.cc:15-26
  if (type == "sgd") return new SGDLearner();
  throw Error("unknown learner type: " + type + " (the GPU engine accelerates the sgd learner)");
}

// SGDLearner::Init, sgd_learner.cc:229-246
KWArgs SGDLearner::Init(const KWArgs& kwargs) {
  KWArgs remain = param_.InitAllowUnknown(kwargs);
  auto* updater = new GpuSGDUpdater();
  std::shared_ptr<Updater> holder(updater);
  remain = updater->Init(remain);
  remain.push_back(std::make_pair("V_dim", std::to_string(updater->param().V_dim)));   // :236
  store_ = Store::Create();
  store_->SetUpdater(holder);
  remain = store_->Init(remain);
  loss_ = Loss::Create(param_.loss, 2);
  static_cast<GpuFMLoss*>(loss_)->AttachEngine(updater->engine());
  remain = loss_->Init(remain);
  if (param_.num_gpus > 1) {
    // one engine (= one shard of the model) per GPU, the same hyper-parameters everywhere; wire the mailboxes
    if (param_.fused != 1) throw ParamError("num_gpus > 1 needs fused = 1 (raw blocks through the sharded store)");
    if (param_.num_gpus > 8) throw ParamError("num_gpus must be <= 8");
    for (int r = 1; r < param_.num_gpus; ++r) {
      KWArgs kw;
      for (const auto& kv : kwargs) if (kv.first != "device") kw.push_back(kv);
      kw.push_back(std::make_pair("device", std::to_string(r)));
      KWArgs engine_kw;     // only what dfb_create knows: drop the learner's keys (it would report them as unknown)
      SGDLearnerParam tmp;
      engine_kw = tmp.InitAllowUnknown(kw);
      shard_engines_.push_back(std::make_shared<GpuEngine>(engine_kw));
    }
    const int N = param_.num_gpus;
    const size_t max_rows = static_cast<size_t>(std::max(param_.batch_size, 65536));     // validation reads 65536-row chunks
    const size_t max_nnz = param_.shard_max_nnz > 0 ? static_cast<size_t>(param_.shard_max_nnz) : max_rows * 256;
    std::vector<void*> boxes(N, nullptr);
    for (int r = 0; r < N; ++r) {
      const auto& e = ShardEngine(r);
      e->Check(dfb_shard_init(e->handle(), r, N, max_rows, max_nnz, 0, 0, nullptr), "dfb_shard_init");
      unsigned char ipc_handle[64];      // unused here (same process); other processes would open it with dfb_peer_open
      e->Check(dfb_shard_export(e->handle(), &boxes[r], getenv("DFB_NO_IPC_EXPORT") ? nullptr : ipc_handle), "dfb_shard_export");
    }
    for (int r = 0; r < N; ++r) ShardEngine(r)->Check(dfb_shard_connect(ShardEngine(r)->handle(), boxes.data()), "dfb_shard_connect");
  }
  return remain;
}

namespace {
bool FileExists(const std::string& fn) { return static_cast<bool>(std::ifstream(fn, std::ios::binary)); }

// ps-lite's key range of shard r of S (postoffice.cc:127-136; the tail above UINT64_MAX/S*S belongs to S-1), as
// an inclusive [lo, hi]
void KeyRange(uint32_t r, uint32_t S, uint64_t* lo, uint64_t* hi) {
  const uint64_t width = UINT64_MAX / S;
  *lo = width * r;
  *hi = r + 1 == S ? UINT64_MAX : width * (r + 1) - 1;
}
}  // namespace

// model_in = X -> the engine(s).  The model is one file X (a num_gpus = 1 run) or the parts X_part-0 .. X_part-(M-1)
// of a num_gpus = M run.  num_gpus = 1 reads X when it exists, otherwise the parts; num_gpus = N > 1 reads the parts
// when X_part-0 exists, otherwise X.  Rank r of N restores every part whose key range overlaps its own and keeps its
// keys (dfb_restore_read), so M parts load into any number of GPUs; M = N is part r alone.
void SGDLearner::LoadShards() {
  const std::string& base = param_.model_in;
  auto part_name = [&](int p) { return base + "_part-" + std::to_string(p); };
  const bool parts = param_.num_gpus > 1 ? FileExists(part_name(0)) : !FileExists(base);
  std::vector<std::string> files;
  if (parts) {
    for (int p = 0; FileExists(part_name(p)); ++p) files.push_back(part_name(p));
  } else if (FileExists(base)) {
    files.push_back(base);
  }
  if (files.empty()) throw Error("failed to open model_in " + base + " (nor " + part_name(0) + ")");
  const uint32_t M = static_cast<uint32_t>(files.size()), N = static_cast<uint32_t>(param_.num_gpus);
  for (uint32_t r = 0; r < N; ++r) {
    uint64_t rlo, rhi;
    KeyRange(r, N, &rlo, &rhi);
    bool aux = true;
    int read = 0;
    for (uint32_t p = 0; p < M; ++p) {
      uint64_t plo, phi;
      KeyRange(p, M, &plo, &phi);
      if (plo > rhi || rlo > phi) continue;      // part p cannot hold keys of rank r
      std::ifstream fi(files[p], std::ios::binary);
      if (!fi) throw Error("failed to open model_in " + files[p]);
      aux = RestoreEngine(*ShardEngine(r), &fi, p, M, r, N) && aux;
      ++read;
    }
    if (verbose) {
      printf("Loaded model from %s (%u part%s", base.c_str(), M, M > 1 ? "s" : "");
      if (N > 1) printf(", %d read by GPU %u", read, r);
      printf(", %s aux data)\n", aux ? "with" : "without");
    }
  }
}

// SGDLearner::RunScheduler, sgd_learner.cc:31-68 (+ model_in / model_out, declared in
// sgd_param.h:53-54 but never acted on by the reference: Job::kLoadModel/kSaveModel are not issued)
void SGDLearner::RunScheduler() {
  // num_gpus = N > 1: one snapshot per shard, <name>_part-<r> (the format of Updater::Save per shard)
  auto shard_name = [&](const std::string& base, int r) { return param_.num_gpus > 1 ? base + "_part-" + std::to_string(r) : base; };
  if (!param_.model_in.empty()) LoadShards();
  RunEpochs();
  if (!param_.model_out.empty()) {
    for (int r = 0; r < param_.num_gpus; ++r) {
      const std::string fn = shard_name(param_.model_out, r);
      std::ofstream fo(fn, std::ios::binary);
      if (!fo) throw Error("failed to open model_out " + fn);
      SaveEngine(*ShardEngine(r), true, &fo);
      if (verbose) printf("Saved model to %s\n", fn.c_str());
    }
  }
}

namespace {
// a pinned host buffer from dfb_host_alloc (asynchronous copies), grown on demand
class PinnedBuf {
 public:
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  ~PinnedBuf() { if (p_) dfb_host_free(p_); }
  template <typename T> T* get(size_t n) {
    const size_t bytes = n * sizeof(T);
    if (bytes > cap_) {
      if (p_) dfb_host_free(p_);
      p_ = nullptr; cap_ = 0;
      const size_t want = bytes + bytes / 4 + 256;
      if (dfb_host_alloc(&p_, want) != DFB_OK) throw Error("dfb_host_alloc failed");
      cap_ = want;
    }
    return static_cast<T*>(p_);
  }

 private:
  void* p_ = nullptr;
  size_t cap_ = 0;
};

void AddProgress(const dfb_progress& pr, sgd::Progress* prog) {
  prog->loss += pr.loss; prog->penalty += pr.penalty; prog->auc += pr.auc; prog->nrows += pr.nrows;
}

void WritePreds(FILE* fo, const real_t* pred, size_t n) {
  for (size_t i = 0; i < n; ++i) fprintf(fo, "%.9g\n", pred[i]);
}
}  // namespace

sgd::Progress SGDLearner::Predict() {
  if (param_.model_in.empty()) throw Error("task=predict needs model_in");
  if (param_.num_gpus > 1) {
    // the model (one file or any number of parts), re-sharded over and scored by N GPUs
    LoadShards();
    sgd::Progress prog;
    param_.data_val = param_.data_in;
    RunEpochSharded(0, sgd::Job::kValidation, &prog, param_.pred_out.empty() ? nullptr : &param_.pred_out);
    if (verbose) printf(" - Prediction: %s, rows = %g\n", prog.TextString().c_str(), prog.nrows);
    return prog;
  }
  LoadShards();      // one file, or all parts of a num_gpus = M model merged into this GPU
  FILE* fo = param_.pred_out.empty() ? nullptr : fopen(param_.pred_out.c_str(), "w");
  if (!param_.pred_out.empty() && !fo) throw Error("failed to open pred_out " + param_.pred_out);
  sgd::Progress prog;
  const auto& eng = GetUpdater()->engine();
  BatchReader reader(param_.data_in, param_.data_format, 0, 1, 65536u);
  // predict steps, two in flight: chunk t is on the GPU while the reader parses chunk t+1 and the file receives the
  // predictions of chunk t-1.  Two pinned input sets and two pinned prediction buffers; set t & 1 is refilled only
  // after step t-2, which used it, has been collected.
  struct Set { PinnedBuf off, ids, val, lab, pred; size_t nrows = 0; };
  Set sets[2];
  uint64_t t = 0;
  auto collect = [&](uint64_t step) {
    dfb_progress pr;
    eng->Check(dfb_wait_step(eng->handle(), &pr), "dfb_predict_raw_async");
    AddProgress(pr, &prog);
    Set& s = sets[step & 1];
    if (fo) WritePreds(fo, s.pred.get<real_t>(s.nrows), s.nrows);
  };
  while (reader.Next()) {
    const auto blk = reader.Value();
    Set& s = sets[t & 1];
    const size_t n = blk.size, nnz = blk.offset[blk.size];
    s.nrows = n;
    uint64_t* off = s.off.get<uint64_t>(n + 1);
    uint64_t* ids = s.ids.get<uint64_t>(nnz);
    real_t* lab = s.lab.get<real_t>(n);
    real_t* val = blk.value ? s.val.get<real_t>(nnz) : nullptr;
    memcpy(off, blk.offset, (n + 1) * sizeof(uint64_t));
    memcpy(ids, blk.index, nnz * sizeof(uint64_t));
    memcpy(lab, blk.label, n * sizeof(real_t));
    if (val) memcpy(val, blk.value, nnz * sizeof(real_t));
    eng->Check(dfb_predict_raw_async(eng->handle(), n, off, ids, val, lab, fo ? s.pred.get<real_t>(n) : nullptr),
               "dfb_predict_raw_async");
    if (t >= 1) collect(t - 1);
    ++t;
  }
  if (t >= 1) collect(t - 1);
  if (fo) fclose(fo);
  if (verbose) printf(" - Prediction: %s, rows = %g\n", prog.TextString().c_str(), prog.nrows);
  return prog;
}

void SGDLearner::RunEpochs() {
  real_t pre_loss = 0, pre_val_auc = 0;
  for (int k = 0; k < param_.max_num_epochs; ++k) {
    sgd::Progress train_prog, val_prog;
    if (verbose) printf("Start epoch %d\n", k);
    RunEpoch(k, sgd::Job::kTraining, &train_prog);
    if (verbose) printf(" - Training: %s\n", train_prog.TextString().c_str());
    if (!param_.data_val.empty()) {
      RunEpoch(k, sgd::Job::kValidation, &val_prog);
      if (verbose) printf(" - Validation: %s\n", val_prog.TextString().c_str());
    }
    for (const auto& cb : epoch_end_callback_) cb(k, train_prog, val_prog);
    real_t eps = std::fabs(train_prog.loss - pre_loss) / pre_loss;
    if (eps < param_.stop_rel_objv) {
      if (verbose) printf("Change of loss [%g] < stop_rel_objv [%g]\n", eps, param_.stop_rel_objv);
      break;
    }
    if (val_prog.auc > 0) {
      eps = (val_prog.auc - pre_val_auc) / val_prog.nrows;
      if (eps < param_.stop_val_auc) {
        if (verbose) printf("Change of validation AUC [%g] < stop_val_auc [%g]\n", eps, param_.stop_val_auc);
        break;
      }
    }
    if (k + 1 >= param_.max_num_epochs && verbose) printf("Reach maximal number of epochs\n");
    pre_loss = train_prog.loss;
    pre_val_auc = val_prog.auc;
    if (verbose) fflush(stdout);
  }
}

// SGDLearner::RunEpoch, sgd_learner.cc:70-111: n = NumWorkers * num_jobs_per_epoch file parts,
// executed in order (the reference's LocalTracker runs them serially on one thread too)
void SGDLearner::RunEpoch(int epoch, int job_type, sgd::Progress* prog) {
  if (param_.num_gpus > 1) { RunEpochSharded(epoch, job_type, prog); return; }
  const int n = store_->NumWorkers() * param_.num_jobs_per_epoch;
  for (int i = 0; i < n; ++i) {
    sgd::Job job;
    job.type = job_type; job.epoch = epoch; job.num_parts = n; job.part_idx = i;
    sgd::Progress p;
    IterateData(job, &p);
    prog->Merge(p);
  }
}

// num_gpus = N > 1: the epoch of sgd_learner.cc:70-111 with N workers.  File part i of the N * num_jobs_per_epoch
// parts goes to worker i % N (the reference's tracker hands parts to whichever worker is free; the assignment is fixed
// here so that runs are reproducible).  Every round each worker contributes its next minibatch (or an empty one when
// its parts are exhausted) to ONE collective sharded step.  One host thread drives all N engines and interleaves
// the five enqueue phases of the step (dfb_shard_begin_async + dfb_shard_phase): nothing in a step waits for
// the host, so the GPUs run concurrently; the readers parse their next batches on helper threads meanwhile.
//
// pred_out: the rows of part i go to a temporary file <pred_out>.part-<i> (host memory stays bounded), which are
// concatenated in part order into pred_out at the end and removed.
void SGDLearner::RunEpochSharded(int epoch, int job_type, sgd::Progress* prog, const std::string* pred_out) {
  const int N = param_.num_gpus;
  const int nparts = N * param_.num_jobs_per_epoch;
  const bool train = job_type == sgd::Job::kTraining;
  const bool push_cnt = train && epoch == 0;      // sgd_learner.cc:201-202
  const bool predict = pred_out != nullptr;
  auto tmp_name = [&](int part) { return *pred_out + ".part-" + std::to_string(part); };
  std::vector<FILE*> part_files(predict ? nparts : 0, nullptr);
  std::vector<PinnedBuf> pred_bufs(predict ? N : 0);
  std::vector<int> step_part(N, -1);
  auto close_parts = [&]() {
    for (auto& f : part_files) if (f) { fclose(f); f = nullptr; }
  };
  struct Worker {
    int part = 0;
    std::unique_ptr<BatchReader> reader;
    bool has = false;
    std::string error;
  };
  std::vector<Worker> w(N);
  for (int r = 0; r < N; ++r) w[r].part = r;
  auto next = [&](int r) {          // host only (file parsing): runs on a helper thread per worker
    Worker& me = w[r];
    me.has = false;
    try {
      for (;;) {
        if (!me.reader) {
          if (me.part >= nparts) return;
          me.reader.reset(new BatchReader(train ? param_.data_in : param_.data_val, param_.data_format,
                                          static_cast<unsigned>(me.part), static_cast<unsigned>(nparts),
                                          train ? static_cast<unsigned>(param_.batch_size) : 65536u,
                                          train ? static_cast<unsigned>(param_.batch_size) * static_cast<unsigned>(param_.shuffle) : 0u,
                                          train ? param_.neg_sampling : 1.0f, static_cast<unsigned>(epoch)));
        }
        if (me.reader->Next()) { me.has = true; return; }
        me.reader.reset();
        me.part += N;
      }
    } catch (const std::exception& e) {
      me.error = e.what();
    }
  };
  for (;;) {
    {
      std::vector<std::thread> th;
      for (int r = 0; r < N; ++r) th.emplace_back(next, r);
      for (auto& t : th) t.join();
    }
    bool any = false;
    for (int r = 0; r < N; ++r) {
      if (!w[r].error.empty()) { close_parts(); throw Error("worker " + std::to_string(r) + ": " + w[r].error); }
      any = any || w[r].has;
    }
    if (!any) break;
    for (int r = 0; r < N; ++r) {
      const auto& eng = ShardEngine(r);
      dmlc::RowBlock<feaid_t> blk;
      if (w[r].has) blk = w[r].reader->Value();
      step_part[r] = w[r].has ? w[r].part : -1;
      const uint64_t* off = blk.size ? reinterpret_cast<const uint64_t*>(blk.offset) : nullptr;
      if (predict) {       // every rank predicts in the same step (the step is collective)
        eng->Check(dfb_shard_begin_predict_async(eng->handle(), blk.size, off, blk.index, blk.value, blk.label,
                                                 pred_bufs[r].get<real_t>(blk.size ? blk.size : 1)),
                   "dfb_shard_begin_predict_async");
      } else {
        eng->Check(dfb_shard_begin_async(eng->handle(), blk.size, off, blk.index, blk.value, blk.label, push_cnt ? 1 : 0,
                                         train ? 1 : 0), "dfb_shard_begin_async");
      }
    }
    for (int ph = 0; ph < 5; ++ph)
      for (int r = 0; r < N; ++r) ShardEngine(r)->Check(dfb_shard_phase(ShardEngine(r)->handle(), ph), "dfb_shard_phase");
    for (int r = 0; r < N; ++r) {
      dfb_progress pr;
      ShardEngine(r)->Check(dfb_wait_step(ShardEngine(r)->handle(), &pr), "dfb_wait_step");
      prog->loss += pr.loss; prog->penalty += pr.penalty; prog->auc += pr.auc; prog->nrows += pr.nrows;
      if (predict && step_part[r] >= 0) {
        FILE*& f = part_files[step_part[r]];
        if (!f && !(f = fopen(tmp_name(step_part[r]).c_str(), "w"))) {
          close_parts();
          throw Error("failed to open " + tmp_name(step_part[r]));
        }
        const size_t n = w[r].reader->Value().size;
        WritePreds(f, pred_bufs[r].get<real_t>(n ? n : 1), n);
      }
    }
  }
  if (!predict) return;
  close_parts();
  FILE* fo = fopen(pred_out->c_str(), "w");
  if (!fo) throw Error("failed to open pred_out " + *pred_out);
  std::vector<char> buf(1 << 20);
  for (int i = 0; i < nparts; ++i) {
    FILE* fi = fopen(tmp_name(i).c_str(), "r");
    if (!fi) continue;        // a part without rows
    size_t n;
    while ((n = fread(buf.data(), 1, buf.size(), fi)) > 0) fwrite(buf.data(), 1, n, fo);
    fclose(fi);
    std::remove(tmp_name(i).c_str());
  }
  fclose(fo);
}

// SGDLearner::GetPos, sgd_learner.cc:113-127
void SGDLearner::GetPos(const SArray<int>& len, SArray<int>* w_pos, SArray<int>* V_pos) {
  const size_t n = len.size();
  w_pos->resize(n);
  V_pos->resize(n);
  int p = 0;
  for (size_t i = 0; i < n; ++i) {
    const int l = len[i];
    (*w_pos)[i] = l == 0 ? -1 : p;
    (*V_pos)[i] = l > 1 ? p + 1 : -1;
    p += l;
  }
}

// SGDLearner::EvaluatePenalty, sgd_learner.cc:249-273
real_t SGDLearner::EvaluatePenalty(const SArray<real_t>& weights, const SArray<int>& w_pos,
                                   const SArray<int>& V_pos) {
  const auto& param = GetUpdater()->param();
  real_t objv = 0;
  if (w_pos.size()) {
    for (int p : w_pos) {
      if (p == -1) continue;
      const real_t w = weights[p];
      objv += param.l1 * std::fabs(w) + .5 * param.l2 * w * w;
    }
    for (int p : V_pos) {
      if (p == -1) continue;
      for (int i = 0; i < param.V_dim; ++i) {
        const real_t V = weights[p + i];
        objv += .5 * param.V_l2 * V * V;
      }
    }
  } else {
    for (real_t w : weights) objv += param.l1 * std::fabs(w) + .5 * param.l2 * w * w;
  }
  return objv;
}

// the pull_callback of IterateData (sgd_learner.cc:138-177) as ONE fused device step
void SGDLearner::BatchFused(const RowBlockContainer<unsigned>& data, const std::vector<feaid_t>& keys,
                            const std::vector<real_t>* cnt, bool train, sgd::Progress* prog) {
  const auto& eng = GetUpdater()->engine();
  dfb_progress pr;
  eng->Check(dfb_train_step(eng->handle(), data.Size(), reinterpret_cast<const uint64_t*>(data.offset.data()),
                            data.index.data(), data.value.empty() ? nullptr : data.value.data(), data.label.data(),
                            keys.data(), keys.size(), cnt ? cnt->data() : nullptr, train ? 1 : 0, &pr, nullptr),
             "dfb_train_step");
  prog->loss += pr.loss; prog->penalty += pr.penalty; prog->auc += pr.auc; prog->nrows += pr.nrows;
}

// the same minibatch through the reference's own plugin calls (sgd_learner.cc:138-177, :214-217)
void SGDLearner::BatchPluginCalls(const RowBlockContainer<unsigned>& data_c, const std::vector<feaid_t>& keys,
                                  const std::vector<real_t>* cnt, bool train, sgd::Progress* prog) {
  SArray<feaid_t> feaids(const_cast<feaid_t*>(keys.data()), keys.size());
  if (cnt) {
    SArray<real_t> feacnt(const_cast<real_t*>(cnt->data()), cnt->size());
    store_->Wait(store_->Push(feaids, Store::kFeaCount, feacnt, SArray<int>()));
  }
  SArray<real_t> values;
  SArray<int> lengths;
  store_->Pull(feaids, Store::kWeight, &values, &lengths);
  auto data = data_c.GetBlock();
  prog->nrows += data.size;
  SArray<real_t> pred(data.size);
  SArray<int> w_pos, V_pos;
  GetPos(lengths, &w_pos, &V_pos);
  std::vector<SArray<char>> inputs = {SArray<char>(values), SArray<char>(w_pos), SArray<char>(V_pos)};
  loss_->Predict(data, inputs, &pred);
  prog->loss += loss_->Evaluate(data.label, pred);
  prog->penalty += EvaluatePenalty(values, w_pos, V_pos);
  prog->auc += static_cast<GpuFMLoss*>(loss_)->AUC(data.label, pred);
  if (train) {
    SArray<real_t> grads(values.size());
    inputs.push_back(SArray<char>(pred));
    loss_->CalcGrad(data, inputs, &grads);
    store_->Push(feaids, Store::kGradient, grads, lengths);
  }
}

// SGDLearner::IterateData, sgd_learner.cc:129-227
void SGDLearner::IterateData(const sgd::Job& job, sgd::Progress* progress) {
  const bool train = job.type == sgd::Job::kTraining;
  // training: BatchReader(batch_size, shuffle window = batch_size*shuffle, neg_sampling) (:182-188);
  // validation: plain reader, here in chunks of 65536 rows (:190-194 reads 256 MB chunks)
  BatchReader reader(train ? param_.data_in : param_.data_val, param_.data_format,
                     static_cast<unsigned>(job.part_idx), static_cast<unsigned>(job.num_parts),
                     train ? static_cast<unsigned>(param_.batch_size) : 65536u,
                     train ? static_cast<unsigned>(param_.batch_size) * static_cast<unsigned>(param_.shuffle) : 0u,
                     train ? param_.neg_sampling : 1.0f, static_cast<unsigned>(job.epoch), 0,
                     ShuffleOrder::kReference);      // one reader at a time: the reference's own shuffle order
  while (reader.Next()) {
    const bool push_cnt = train && job.epoch == 0;   // :201-202
    if (param_.fused == 1) {
      // Localizer::Compact + [kFeaCount push] + Pull/Predict/.../Push in one device call on the raw block
      const auto blk = reader.Value();
      const auto& eng = GetUpdater()->engine();
      dfb_progress pr;
      eng->Check(dfb_train_step_raw(eng->handle(), blk.size, reinterpret_cast<const uint64_t*>(blk.offset),
                                    blk.index, blk.value, blk.label, push_cnt ? 1 : 0, train ? 1 : 0, &pr, nullptr),
                 "dfb_train_step_raw");
      progress->loss += pr.loss; progress->penalty += pr.penalty; progress->auc += pr.auc; progress->nrows += pr.nrows;
      continue;
    }
    RowBlockContainer<unsigned> data;
    std::vector<feaid_t> feaids;
    std::vector<real_t> feacnt;
    Localizer lc(-1, 2);
    lc.Compact(reader.Value(), &data, &feaids, push_cnt ? &feacnt : nullptr);
    if (param_.fused == 2) BatchFused(data, feaids, push_cnt ? &feacnt : nullptr, train, progress);
    else BatchPluginCalls(data, feaids, push_cnt ? &feacnt : nullptr, train, progress);
  }
}

}  // namespace difacto
