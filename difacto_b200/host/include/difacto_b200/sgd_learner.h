// difacto_b200/host/include/difacto_b200/sgd_learner.h -- SGDLearner over the GPU engine.
// Mirrors src/sgd/sgd_learner.{h,cc} + sgd_utils.h of the reference: epochs -> jobs (file parts) ->
// minibatches; per-epoch Progress, epoch-end callbacks and the two stop criteria are identical.
// The minibatch itself (the pull_callback of IterateData, sgd_learner.cc:138-177) is either
//   fused = 1 (default): one dfb_train_step_raw per batch on the reader's raw block (Localizer::Compact
//              on the device too), the model never leaves HBM;
//   fused = 2: host Localizer::Compact, then one dfb_train_step per batch;
//   fused = 0: the reference's own sequence of plugin calls Store::Pull -> GetPos -> Loss::Predict ->
//              Evaluate -> penalty -> AUC -> Loss::CalcGrad -> Store::Push through the adapter classes.
// num_gpus = N > 1 (with fused = 1): the worker/server split SGDLearner::RunEpoch was written for
// (sgd_learner.cc:78-89): N workers, each reading its own file parts (parsed on helper threads) and owning GPU
// r's shard of the model, one collective sharded step per round of minibatches, enqueued by one host thread in
// interleaved phases (dfb_shard_begin_async + dfb_shard_phase; the NVLink-sharded store, csrc/shard.cu).
#pragma once
#include <cmath>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "api.h"
#include "checkpoint_state.h"
#include "config.h"
#include "data.h"
#include "engine_adapters.h"

namespace difacto {
namespace sgd {

/** sgd::Job, src/sgd/sgd_utils.h:16-38 */
struct Job {
  static const int kLoadModel = 1, kSaveModel = 2, kTraining = 3, kValidation = 4, kEvaluation = 5;
  int type = kTraining, num_parts = 1, part_idx = 0, epoch = 0;
};

/** sgd::Progress, src/sgd/sgd_utils.h:40-75 */
struct Progress {
  real_t loss = 0, penalty = 0, auc = 0, nnz_w = 0, nrows = 0;
  std::string TextString() const {
    std::stringstream ss;
    ss << "loss = " << loss << ", AUC = " << auc / nrows;
    return ss.str();
  }
  void Merge(const Progress& o) {
    loss += o.loss; penalty += o.penalty; auc += o.auc; nnz_w += o.nnz_w; nrows += o.nrows;
  }
};

}  // namespace sgd

class SGDLearner : public Learner {
 public:
  typedef std::function<void(int epoch, const sgd::Progress& train, const sgd::Progress& val)> EpochCallback;
  SGDLearner() {}
  ~SGDLearner() override;
  KWArgs Init(const KWArgs& kwargs) override;
  void AddEpochEndCallback(const EpochCallback& cb) { epoch_end_callback_.push_back(cb); }
  GpuSGDUpdater* GetUpdater() { return static_cast<GpuSGDUpdater*>(store_->updater().get()); }
  /** task=predict (a `LOG(FATAL) << "TODO"` in the reference, main.cc:61-62): load model_in, run the forward pass
   * over data_in in file order and write one prediction (the clamped FM score, fm_loss.h:118) per row to pred_out;
   * returns the Progress (loss, AUC*n, nrows) of the pass */
  sgd::Progress Predict();
  /** set false to silence the per-epoch log lines */
  bool verbose = true;
  /** the settings that fix the minibatches and the model, as parsed values (the engine's defaults for the keys not
   * given): a checkpoint resumes only under the same settings */
  static std::vector<std::pair<std::string, std::string>> Settings(const SGDLearnerParam& p, const KWArgs& kwargs);
  /** the settings a checkpoint written before they existed does not record, with the value it ran under: the
   * default, so such a checkpoint resumes under the defaults and is refused under anything else */
  static std::vector<std::pair<std::string, std::string>> SettingsAddedLater() {
    return {{"prune_period", "0"}, {"prune_count", "0"}};
  }

 protected:
  void RunScheduler() override;

 private:
  void RunEpochs();
  void RunEpoch(int epoch, int job_type, sgd::Progress* prog);
  void IterateData(const sgd::Job& job, sgd::Progress* prog);
  /** num_gpus > 1: one epoch over all N * num_jobs_per_epoch file parts, part i handled by worker i % N.
   * predict (task=predict): predict steps instead of validation steps (penalty 0); pred_out: the predictions of every
   * row to that file, in file order */
  void RunEpochSharded(int epoch, int job_type, sgd::Progress* prog, bool predict = false,
                       const std::string* pred_out = nullptr);
  /** the model X (one file) or X_part-0 .. of a num_gpus = M run into the engines (model_in, checkpoint_in) */
  void LoadShards(const std::string& base);
  /** checkpoint_in: the model, the id ranges and the position in the run of the checkpoint the pointer file names */
  void LoadCheckpoint();
  /** after a training minibatch per worker (every rank's step collected): counts it, then prunes and checkpoints
   * when their periods have come round, the prune first */
  void EndMinibatch();
  /** prune_period: every rank drops its entries with w == 0, no V row and fea_cnt <= prune_count (dfb_prune) */
  void MaybePrune();
  /** a checkpoint when the period has come round.  The model is frozen on every GPU now; a helper thread writes it,
   * then the state record, then renames the pointer file */
  void MaybeCheckpoint();
  /** waits for the checkpoint write in flight and releases its device copies; throws what it failed with */
  void WaitCheckpoint();
  /** engine of GPU r (r = 0: the updater's own) */
  const std::shared_ptr<GpuEngine>& ShardEngine(int r) { return r == 0 ? GetUpdater()->engine() : shard_engines_[r - 1]; }
  void BatchFused(const RowBlockContainer<unsigned>& data, const std::vector<feaid_t>& keys,
                  const std::vector<real_t>* cnt, bool train, sgd::Progress* prog);
  void BatchPluginCalls(const RowBlockContainer<unsigned>& data, const std::vector<feaid_t>& keys,
                        const std::vector<real_t>* cnt, bool train, sgd::Progress* prog);
  static void GetPos(const SArray<int>& len, SArray<int>* w_pos, SArray<int>* V_pos);
  real_t EvaluatePenalty(const SArray<real_t>& weights, const SArray<int>& w_pos, const SArray<int>& V_pos);

  Store* store_ = nullptr;
  Loss* loss_ = nullptr;
  SGDLearnerParam param_;
  std::vector<EpochCallback> epoch_end_callback_;
  std::vector<std::shared_ptr<GpuEngine>> shard_engines_;     // GPUs 1..N-1 (num_gpus > 1)
  bool score_only_ = false;     // the engine key score_only = 1: scoring-only engines, which run predict steps only

  // checkpoints: the settings the state record fingerprints, the run's position (kept current by the drivers), the
  // state to resume from, and the write in flight
  std::vector<std::pair<std::string, std::string>> settings_;
  CheckpointState pos_;
  sgd::Progress* epoch_prog_ = nullptr;   // the Progress of the epoch being trained, and (num_gpus = 1) of its part
  sgd::Progress* part_prog_ = nullptr;
  std::unique_ptr<CheckpointState> resume_;
  int ckpt_seq_ = 0, ckpt_prev_ = -1;
  std::thread ckpt_thread_;
  std::string ckpt_error_;
  std::vector<dfb_frozen> frozen_;
};

}  // namespace difacto
