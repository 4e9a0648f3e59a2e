// difacto_b200/host/src/sgd_learner.cc -- see sgd_learner.h.  Control flow follows
// src/sgd/sgd_learner.cc of the reference (cited per function); the arithmetic lives on the GPU.
#include "difacto_b200/sgd_learner.h"

#include <errno.h>
#include <fcntl.h>
#include <unistd.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
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

namespace {
// a setting as the engine parses it: a float as the float it parses to (%.9g tells every float apart), an integer as
// that integer.  Anything else as given (the engine refuses it).
std::string FloatSetting(float f) {
  char b[64];
  snprintf(b, sizeof(b), "%.9g", f);
  return b;
}
std::string FloatSetting(const std::string& v) {
  char* end = nullptr;
  const float f = strtof(v.c_str(), &end);
  if (v.empty() || *end) return v;
  return FloatSetting(f);
}
bool FileExists(const std::string& fn) { return static_cast<bool>(std::ifstream(fn, std::ios::binary)); }
std::string IntSetting(const std::string& v) {
  char* end = nullptr;
  const long long x = strtoll(v.c_str(), &end, 10);
  if (v.empty() || *end) return v;
  return std::to_string(x);
}
}  // namespace

SGDLearner::~SGDLearner() {
  if (ckpt_thread_.joinable()) ckpt_thread_.join();
  for (dfb_frozen f : frozen_) if (f) dfb_frozen_release(f);
  delete loss_;
  delete store_;
}

std::vector<std::pair<std::string, std::string>> SGDLearner::Settings(const SGDLearnerParam& p, const KWArgs& kwargs) {
  std::vector<std::pair<std::string, std::string>> s = {
      {"data_in", p.data_in}, {"data_val", p.data_val}, {"data_format", p.data_format}, {"loss", p.loss},
      {"num_gpus", std::to_string(p.num_gpus)}, {"num_jobs_per_epoch", std::to_string(p.num_jobs_per_epoch)},
      {"batch_size", std::to_string(p.batch_size)}, {"shuffle", std::to_string(p.shuffle)},
      {"neg_sampling", FloatSetting(p.neg_sampling)}, {"prune_period", std::to_string(p.prune_period)},
      {"prune_count", FloatSetting(p.prune_count)}};
  // SGDUpdaterParam (sgd_param.h:94-106) and id_bits, with the engine's defaults for the keys not given
  struct Key { const char* name; const char* dflt; bool is_float; };
  const Key keys[] = {{"l1", "1", true}, {"l2", "0", true}, {"V_l2", ".01", true}, {"lr", ".01", true},
                      {"lr_beta", "1", true}, {"V_lr", ".01", true}, {"V_lr_beta", "1", true},
                      {"V_init_scale", ".01", true}, {"V_dim", "-1", false}, {"V_threshold", "10", false},
                      {"seed", "0", false}, {"id_bits", "0", false}};
  for (const Key& k : keys) {
    std::string v = k.dflt;
    for (const auto& kv : kwargs) if (kv.first == k.name) v = kv.second;
    s.push_back(std::make_pair(std::string(k.name), k.is_float ? FloatSetting(v) : IntSetting(v)));
  }
  return s;
}

// SGDLearner::Init, sgd_learner.cc:229-246
KWArgs SGDLearner::Init(const KWArgs& kwargs) {
  KWArgs remain = param_.InitAllowUnknown(kwargs);
  // score_only / V_storage are engine keys and reach dfb_create with the rest (every GPU's engine: with num_gpus > 1
  // each rank of the sharded store holds its shard in V-only rows)
  for (const auto& kv : kwargs)
    if (kv.first == "score_only") score_only_ = kv.second != "0";
  // N scoring GPUs load the parts of a model a num_gpus run saved.  A one-file model was trained on one GPU, so its
  // scoring-only layout (half or a quarter of the rows) fits one GPU: it is scored there, without the store's workspaces
  if (score_only_ && param_.num_gpus > 1 && !FileExists(param_.model_in + "_part-0"))
    throw ParamError("score_only = 1 with num_gpus > 1 scores the parts of a model saved by a num_gpus run (model_in = X "
                     "reads X_part-0 ...); score a one-file model with num_gpus = 1");
  settings_ = Settings(param_, kwargs);
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
void SGDLearner::LoadShards(const std::string& base) {
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
  if (!param_.checkpoint_in.empty()) {
    if (!param_.model_in.empty()) throw ParamError("checkpoint_in and model_in both load a model: give one of them");
    LoadCheckpoint();
  } else if (!param_.model_in.empty()) {
    LoadShards(param_.model_in);
  }
  RunEpochs();
  WaitCheckpoint();
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
    LoadShards(param_.model_in);
    sgd::Progress prog;
    param_.data_val = param_.data_in;
    // a scoring-only store runs predict steps only (its ranks refuse validation steps); a training-layout one predicts
    // when it writes the predictions, and otherwise validates (Progress with the penalty)
    const bool write = !param_.pred_out.empty();
    RunEpochSharded(0, sgd::Job::kValidation, &prog, write || score_only_, write ? &param_.pred_out : nullptr);
    if (verbose) printf(" - Prediction: %s, rows = %g\n", prog.TextString().c_str(), prog.nrows);
    return prog;
  }
  LoadShards(param_.model_in);      // one file, or all parts of a num_gpus = M model merged into this GPU
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

namespace {
void ToBits(const sgd::Progress& p, float* out) {
  out[0] = p.loss; out[1] = p.penalty; out[2] = p.auc; out[3] = p.nnz_w; out[4] = p.nrows;
}
sgd::Progress FromBits(const float* in) {
  sgd::Progress p;
  p.loss = in[0]; p.penalty = in[1]; p.auc = in[2]; p.nnz_w = in[3]; p.nrows = in[4];
  return p;
}
}  // namespace

void SGDLearner::RunEpochs() {
  real_t& pre_loss = pos_.pre_loss;
  real_t& pre_val_auc = pos_.pre_val_auc;
  pre_loss = 0; pre_val_auc = 0;
  int k0 = 0;
  if (resume_) {        // the epoch the checkpoint was taken in, and what the finished part of it added up to
    k0 = resume_->epoch;
    pre_loss = resume_->pre_loss;
    pre_val_auc = resume_->pre_val_auc;
  }
  for (int k = k0; k < param_.max_num_epochs; ++k) {
    sgd::Progress train_prog, val_prog;
    if (resume_) train_prog = FromBits(resume_->epoch_prog);
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
  const bool train = job_type == sgd::Job::kTraining;
  int i0 = 0;
  sgd::Progress p0;
  if (train && resume_) {      // resumed: from the part the checkpoint was taken in, with its Progress so far
    i0 = resume_->workers[0].part;
    p0 = FromBits(resume_->part_prog);
  }
  for (int i = i0; i < n; ++i) {
    sgd::Job job;
    job.type = job_type; job.epoch = epoch; job.num_parts = n; job.part_idx = i;
    sgd::Progress p = i == i0 ? p0 : sgd::Progress();
    epoch_prog_ = prog;
    part_prog_ = &p;
    IterateData(job, &p);
    prog->Merge(p);
  }
  epoch_prog_ = part_prog_ = nullptr;
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
void SGDLearner::RunEpochSharded(int epoch, int job_type, sgd::Progress* prog, bool predict, const std::string* pred_out) {
  const int N = param_.num_gpus;
  const int nparts = N * param_.num_jobs_per_epoch;
  const bool train = job_type == sgd::Job::kTraining;
  const bool push_cnt = train && epoch == 0;      // sgd_learner.cc:201-202
  const bool write = pred_out != nullptr;
  auto tmp_name = [&](int part) { return *pred_out + ".part-" + std::to_string(part); };
  std::vector<FILE*> part_files(write ? nparts : 0, nullptr);
  std::vector<PinnedBuf> pred_bufs(write ? N : 0);
  std::vector<int> step_part(N, -1);
  auto close_parts = [&]() {
    for (auto& f : part_files) if (f) { fclose(f); f = nullptr; }
  };
  struct Worker {
    int part = 0;
    uint64_t consumed = 0, skip = 0;     // minibatches read from the part; and still to be replayed on a resume
    std::unique_ptr<BatchReader> reader;
    bool has = false;
    std::string error;
  };
  std::vector<Worker> w(N);
  for (int r = 0; r < N; ++r) w[r].part = r;
  if (train && resume_) {      // resumed: each worker on its part, past the minibatches it had read
    for (int r = 0; r < N; ++r) { w[r].part = resume_->workers[r].part; w[r].skip = resume_->workers[r].consumed; }
    resume_.reset();
  }
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
          me.consumed = 0;
          for (; me.skip; --me.skip, ++me.consumed)    // read and dropped on the host: the GPUs had them
            if (!me.reader->Next()) throw Error("checkpoint_in: file part " + std::to_string(me.part) + " is shorter than the checkpoint says");
        }
        if (me.reader->Next()) { me.has = true; ++me.consumed; return; }
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
                                                 write ? pred_bufs[r].get<real_t>(blk.size ? blk.size : 1) : nullptr),
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
      if (write && step_part[r] >= 0) {
        FILE*& f = part_files[step_part[r]];
        if (!f && !(f = fopen(tmp_name(step_part[r]).c_str(), "w"))) {
          close_parts();
          throw Error("failed to open " + tmp_name(step_part[r]));
        }
        const size_t n = w[r].reader->Value().size;
        WritePreds(f, pred_bufs[r].get<real_t>(n ? n : 1), n);
      }
    }
    if (train) {     // every rank's checkpoint after the same collected round
      pos_.epoch = epoch;
      pos_.has_rand = false;
      pos_.workers.resize(N);
      for (int r = 0; r < N; ++r) { pos_.workers[r].part = w[r].part; pos_.workers[r].consumed = w[r].consumed; }
      epoch_prog_ = prog;
      part_prog_ = nullptr;
      EndMinibatch();
      epoch_prog_ = nullptr;
    }
  }
  if (!write) return;
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
  // the reader draws its shuffle from rand(): a resume restores it as it was at the start of the part, and every
  // checkpoint records it so
  if (train && resume_ && resume_->has_rand) resume_->rand.Restore();
  RandState rand_at_start;
  if (train && param_.checkpoint_period > 0) rand_at_start = RandState::Save();
  // training: BatchReader(batch_size, shuffle window = batch_size*shuffle, neg_sampling) (:182-188);
  // validation: plain reader, here in chunks of 65536 rows (:190-194 reads 256 MB chunks)
  BatchReader reader(train ? param_.data_in : param_.data_val, param_.data_format,
                     static_cast<unsigned>(job.part_idx), static_cast<unsigned>(job.num_parts),
                     train ? static_cast<unsigned>(param_.batch_size) : 65536u,
                     train ? static_cast<unsigned>(param_.batch_size) * static_cast<unsigned>(param_.shuffle) : 0u,
                     train ? param_.neg_sampling : 1.0f, static_cast<unsigned>(job.epoch), 0,
                     ShuffleOrder::kReference);      // one reader at a time: the reference's own shuffle order
  uint64_t skip = 0;
  if (train) {
    pos_.epoch = job.epoch;
    pos_.workers.assign(1, CheckpointState::Worker());
    pos_.workers[0].part = job.part_idx;
    pos_.has_rand = param_.checkpoint_period > 0;
    pos_.rand = rand_at_start;
  }
  if (train && resume_) {
    skip = resume_->workers[0].consumed;
    resume_.reset();
  }
  while (reader.Next()) {
    if (skip) {        // resumed: the minibatches the checkpoint had trained, read and dropped on the host
      --skip;
      ++pos_.workers[0].consumed;
      continue;
    }
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
    } else {
      RowBlockContainer<unsigned> data;
      std::vector<feaid_t> feaids;
      std::vector<real_t> feacnt;
      Localizer lc(-1, 2);
      lc.Compact(reader.Value(), &data, &feaids, push_cnt ? &feacnt : nullptr);
      if (param_.fused == 2) BatchFused(data, feaids, push_cnt ? &feacnt : nullptr, train, progress);
      else BatchPluginCalls(data, feaids, push_cnt ? &feacnt : nullptr, train, progress);
    }
    if (train) {
      ++pos_.workers[0].consumed;
      EndMinibatch();
    }
  }
}

namespace {
// dfb_write_fn into a file descriptor
int FdSink(void* ctx, const void* buf, size_t bytes) {
  const int fd = *static_cast<const int*>(ctx);
  const char* p = static_cast<const char*>(buf);
  while (bytes) {
    const ssize_t n = ::write(fd, p, bytes);
    if (n < 0) {
      if (errno == EINTR) continue;
      return 1;
    }
    p += n;
    bytes -= static_cast<size_t>(n);
  }
  return 0;
}

// path, filled by fill(fd), then flushed to the disk
void WriteSynced(const std::string& path, const std::function<void(int)>& fill) {
  const int fd = ::open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) throw Error("failed to open " + path + ": " + strerror(errno));
  try {
    fill(fd);
  } catch (...) {
    ::close(fd);
    throw;
  }
  const bool synced = ::fsync(fd) == 0;
  if (::close(fd) != 0 || !synced) throw Error("failed to write " + path + ": " + strerror(errno));
}

void WriteBytes(const std::string& path, const std::string& bytes) {
  WriteSynced(path, [&](int fd) {
    if (FdSink(&fd, bytes.data(), bytes.size())) throw Error("failed to write " + path + ": " + strerror(errno));
  });
}

// the directory entry of a rename, flushed to the disk
void SyncDir(const std::string& path) {
  const size_t slash = path.rfind('/');
  const std::string dir = slash == std::string::npos ? "." : (slash == 0 ? "/" : path.substr(0, slash));
  const int fd = ::open(dir.c_str(), O_RDONLY | O_DIRECTORY);
  if (fd < 0) return;
  ::fsync(fd);
  ::close(fd);
}

// the model file of rank r in checkpoint `base` (= P.<c>): the names model_out / model_in use
std::string CkptModel(const std::string& base, int N, int r) {
  return N > 1 ? base + ".model_part-" + std::to_string(r) : base + ".model";
}

void RemoveCheckpoint(const std::string& P, int c, int N) {
  const std::string base = P + "." + std::to_string(c);
  for (int r = 0; r < N; ++r) std::remove(CkptModel(base, N, r).c_str());
  std::remove((base + ".state").c_str());
}
}  // namespace

// checkpoint c: P.<c>.model (P.<c>.model_part-<r>), P.<c>.state, then P names c.  Until the rename, P names c - 1,
// which stays complete on the disk; it is removed after.
void SGDLearner::EndMinibatch() {
  ++pos_.minibatches;
  MaybePrune();
  MaybeCheckpoint();
}

// every rank's table at the same boundary, after all ranks' steps: the prune waits for each engine's streams
void SGDLearner::MaybePrune() {
  if (param_.prune_period <= 0 || pos_.minibatches % static_cast<uint64_t>(param_.prune_period) != 0) return;
  uint64_t dropped = 0, n_keys = 0;
  for (int r = 0; r < param_.num_gpus; ++r) {
    const auto& e = ShardEngine(r);
    uint64_t d = 0, k = 0;
    int rc = dfb_prune(e->handle(), param_.prune_count, &d);
    if (rc == DFB_ERR_CAPACITY && !frozen_.empty()) {    // no room for the workspace beside a checkpoint's device copy
      WaitCheckpoint();
      rc = dfb_prune(e->handle(), param_.prune_count, &d);
    }
    e->Check(rc, "dfb_prune");
    e->Check(dfb_table_stats(e->handle(), &k, nullptr, nullptr, nullptr), "dfb_table_stats");
    dropped += d;
    n_keys += k;
  }
  if (verbose)
    printf("Prune: minibatch %llu, dropped %llu, n_keys %llu\n", static_cast<unsigned long long>(pos_.minibatches),
           static_cast<unsigned long long>(dropped), static_cast<unsigned long long>(n_keys));
}

void SGDLearner::MaybeCheckpoint() {
  if (param_.checkpoint_period <= 0 || pos_.minibatches % static_cast<uint64_t>(param_.checkpoint_period) != 0) return;
  WaitCheckpoint();
  const int N = param_.num_gpus;
  const int c = ckpt_seq_++;
  const std::string P = param_.checkpoint_out, base = P + "." + std::to_string(c);
  CheckpointState st = pos_;
  st.settings = settings_;
  ToBits(*epoch_prog_, st.epoch_prog);
  if (part_prog_) ToBits(*part_prog_, st.part_prog);
  st.id_ranges.assign(N, 0);
  for (int r = 0; r < N; ++r) ShardEngine(r)->Check(dfb_id_range_get(ShardEngine(r)->handle(), &st.id_ranges[r]), "dfb_id_range_get");
  // freeze every rank's model on its GPU; where there is no room for the copy, write that rank's model now
  frozen_.assign(N, nullptr);
  for (int r = 0; r < N; ++r) {
    const auto& e = ShardEngine(r);
    const int rc = dfb_snapshot_begin(e->handle(), 1, &frozen_[r]);
    if (rc == DFB_ERR_CAPACITY) {
      frozen_[r] = nullptr;
      WriteSynced(CkptModel(base, N, r), [&](int fd) {
        e->Check(dfb_snapshot_write(e->handle(), 1, 0, FdSink, &fd), "dfb_snapshot_write");
      });
    } else {
      e->Check(rc, "dfb_snapshot_begin");
    }
  }
  const std::string rec = st.Serialize();
  if (verbose) {
    printf("Checkpoint %d: minibatch %llu, epoch %d, part:minibatches", c, static_cast<unsigned long long>(st.minibatches),
           st.epoch);
    for (const auto& w : st.workers) printf(" %d:%llu", w.part, static_cast<unsigned long long>(w.consumed));
    printf("\n");
  }
  const int prev = ckpt_prev_;
  ckpt_prev_ = c;
  const std::vector<dfb_frozen> fr = frozen_;
  ckpt_thread_ = std::thread([this, fr, rec, P, base, c, prev, N]() {
    try {
      for (int r = 0; r < N; ++r) {
        if (!fr[r]) continue;
        WriteSynced(CkptModel(base, N, r), [&](int fd) {
          if (dfb_frozen_write(fr[r], 0, FdSink, &fd) != DFB_OK)
            throw Error(std::string("dfb_frozen_write: ") + dfb_frozen_error(fr[r]));
        });
      }
      WriteBytes(base + ".state", rec);
      const std::string tmp = P + ".tmp";
      WriteBytes(tmp, std::to_string(c) + "\n");
      if (std::rename(tmp.c_str(), P.c_str()) != 0) throw Error("failed to rename " + tmp + " to " + P);
      SyncDir(P);
      if (prev >= 0) RemoveCheckpoint(P, prev, N);
    } catch (const std::exception& e) {
      ckpt_error_ = e.what();
    }
  });
}

void SGDLearner::WaitCheckpoint() {
  if (ckpt_thread_.joinable()) ckpt_thread_.join();
  for (dfb_frozen f : frozen_) if (f) dfb_frozen_release(f);
  frozen_.clear();
  if (!ckpt_error_.empty()) {
    std::string e;
    e.swap(ckpt_error_);
    throw Error("checkpoint: " + e);
  }
}

void SGDLearner::LoadCheckpoint() {
  const std::string& P = param_.checkpoint_in;
  std::ifstream fp(P);
  if (!fp) throw Error("checkpoint_in: failed to open " + P);
  long long c = -1;
  fp >> c;
  if (!fp || c < 0) throw Error("checkpoint_in: " + P + " does not name a checkpoint");
  const std::string base = P + "." + std::to_string(c);
  std::ifstream fs(base + ".state", std::ios::binary);
  if (!fs) throw Error("checkpoint_in: checkpoint " + std::to_string(c) + " that " + P + " names is missing (" + base + ".state)");
  std::stringstream ss;
  ss << fs.rdbuf();
  std::unique_ptr<CheckpointState> st(new CheckpointState(CheckpointState::Parse(ss.str())));
  st->CheckSettings(settings_, SettingsAddedLater());
  const int N = param_.num_gpus;
  if (static_cast<int>(st->workers.size()) != N || static_cast<int>(st->id_ranges.size()) != N)
    throw Error("checkpoint_in: " + base + ".state does not hold " + std::to_string(N) + " workers");
  for (int r = 0; r < N; ++r)
    if (!FileExists(CkptModel(base, N, r)))
      throw Error("checkpoint_in: checkpoint " + std::to_string(c) + " that " + P + " names is missing " + CkptModel(base, N, r));
  LoadShards(base + ".model");
  for (int r = 0; r < N; ++r)
    if (st->id_ranges[r] > 0) ShardEngine(r)->Check(dfb_id_range_set(ShardEngine(r)->handle(), st->id_ranges[r]), "dfb_id_range_set");
  pos_.minibatches = st->minibatches;
  ckpt_seq_ = static_cast<int>(c) + 1;
  ckpt_prev_ = param_.checkpoint_out == P ? static_cast<int>(c) : -1;
  if (verbose) printf("Resuming from checkpoint %lld of %s: epoch %d, minibatch %llu\n", c, P.c_str(), st->epoch,
                      static_cast<unsigned long long>(st->minibatches));
  resume_ = std::move(st);
}

}  // namespace difacto
