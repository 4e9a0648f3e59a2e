// difacto_b200/host/include/difacto_b200/engine_adapters.h
//
// The three plugin classes of the SGD path, implemented over the C-ABI (include/difacto_b200.h):
//   GpuSGDUpdater : Updater   replaces SGDUpdater   (src/sgd/sgd_updater.{h,cc})
//   GpuFMLoss     : Loss      replaces FMLoss       (src/loss/fm_loss.h), registered as "fm"
//   GpuStore      : Store     replaces StoreLocal   (src/store/store_local.h)
// A non-zero C-ABI status becomes a difacto::Error carrying dfb_last_error() (the reference would
// LOG(FATAL) -> abort()).
#pragma once
#include <istream>
#include <iterator>
#include <memory>
#include <ostream>
#include <string>
#include <vector>

#include "../../../../include/difacto_b200.h"
#include "api.h"

namespace difacto {

/** RAII owner of one dfb_handle (one table shard on one GPU), shared by updater and loss */
class GpuEngine {
 public:
  explicit GpuEngine(const KWArgs& kwargs) {
    std::vector<const char*> k, v;
    for (const auto& kv : kwargs) { k.push_back(kv.first.c_str()); v.push_back(kv.second.c_str()); }
    int rc = dfb_create(k.data(), v.data(), static_cast<int>(k.size()), &h_);
    if (rc == DFB_ERR_PARAM) throw ParamError(dfb_last_error(nullptr));
    if (rc != DFB_OK) throw Error(std::string("dfb_create: ") + dfb_last_error(nullptr));
    for (int i = 0; i < dfb_num_unknown_kwargs(h_); ++i) {
      const char *key, *val;
      dfb_unknown_kwarg(h_, i, &key, &val);
      remain_.push_back(std::make_pair(std::string(key), std::string(val)));
    }
  }
  ~GpuEngine() { dfb_destroy(h_); }
  GpuEngine(const GpuEngine&) = delete;
  GpuEngine& operator=(const GpuEngine&) = delete;
  dfb_handle handle() const { return h_; }
  const KWArgs& remain() const { return remain_; }
  void Check(int rc, const char* what) const {
    if (rc != DFB_OK) throw Error(std::string(what) + ": " + dfb_last_error(h_));
  }

 private:
  dfb_handle h_ = nullptr;
  KWArgs remain_;
};

/** the streamed checkpoint over std::ostream / std::istream (dfb_snapshot_write / dfb_restore_read) */
inline int OstreamSink(void* ctx, const void* buf, size_t bytes) {
  auto* fo = static_cast<std::ostream*>(ctx);
  fo->write(static_cast<const char*>(buf), static_cast<std::streamsize>(bytes));
  return fo->good() ? 0 : 1;
}
inline size_t IstreamSource(void* ctx, void* buf, size_t cap) {
  auto* fi = static_cast<std::istream*>(ctx);
  if (fi->bad()) return static_cast<size_t>(-1);
  if (fi->eof()) return 0;
  fi->read(static_cast<char*>(buf), static_cast<std::streamsize>(cap));
  if (fi->bad()) return static_cast<size_t>(-1);
  return static_cast<size_t>(fi->gcount());
}
/** save engine e's model to fo, one chunk at a time */
inline void SaveEngine(const GpuEngine& e, bool save_aux, std::ostream* fo) {
  e.Check(dfb_snapshot_write(e.handle(), save_aux ? 1 : 0, 0, OstreamSink, fo), "dfb_snapshot_write");
  fo->flush();
  if (!fo->good()) throw Error("failed to write the model");
}
/** restore (merge) part `part` of `nparts` read from fi into engine e, shard `shard` of `nshards`; returns has_aux */
inline bool RestoreEngine(const GpuEngine& e, std::istream* fi, uint32_t part, uint32_t nparts, uint32_t shard,
                          uint32_t nshards) {
  int aux = 0;
  e.Check(dfb_restore_read(e.handle(), IstreamSource, fi, part, nparts, shard, nshards, 0, &aux), "dfb_restore_read");
  return aux != 0;
}

/** the reference's SGDUpdaterParam fields the host needs to see (src/sgd/sgd_param.h:66-107) */
struct SGDUpdaterParamView {
  float l1 = 1, l2 = 0, V_l2 = .01f;
  int V_dim = 0;
};

class GpuSGDUpdater : public Updater {
 public:
  KWArgs Init(const KWArgs& kwargs) override {
    engine_ = std::make_shared<GpuEngine>(kwargs);
    for (const auto& kv : kwargs) {
      if (kv.first == "V_dim") param_.V_dim = std::stoi(kv.second);
      else if (kv.first == "l1") param_.l1 = std::stof(kv.second);
      else if (kv.first == "l2") param_.l2 = std::stof(kv.second);
      else if (kv.first == "V_l2") param_.V_l2 = std::stof(kv.second);
    }
    return engine_->remain();
  }
  /** Updater::Load / Save (updater.h:40-47).  TODO stubs in the reference's SGDUpdater
   * (sgd_updater.h:44-50); here a snapshot of the table in the format of dfb_snapshot, streamed through the GPU
   * in bounded host memory.  Load needs an empty table, like dfb_restore. */
  void Load(std::istream* fi, bool* has_aux) override {
    uint64_t n_keys = 0;
    engine_->Check(dfb_table_stats(engine_->handle(), &n_keys, nullptr, nullptr, nullptr), "dfb_table_stats");
    if (n_keys != 0) throw Error("Load needs an empty table");
    const bool aux = RestoreEngine(*engine_, fi, 0, 1, 0, 1);
    if (has_aux) *has_aux = aux;
  }
  void Save(bool save_aux, std::ostream* fo) const override { SaveEngine(*engine_, save_aux, fo); }

  /** SGDUpdater::Get, sgd_updater.cc:32-56 */
  void Get(const SArray<feaid_t>& fea_ids, int val_type, SArray<real_t>* weights, SArray<int>* lens) override {
    DFB_CHECK(val_type == Store::kWeight);
    const size_t n = fea_ids.size();
    weights->resize(n * (1 + static_cast<size_t>(param_.V_dim)));
    lens->resize(n);
    size_t nvals = 0, nlens = 0;
    engine_->Check(dfb_pull(engine_->handle(), fea_ids.data(), n, weights->data(), weights->size(), lens->data(),
                            &nvals, &nlens), "dfb_pull");
    weights->resize(nvals);
    lens->resize(nlens);
  }

  /** SGDUpdater::Update, sgd_updater.cc:58-101 */
  void Update(const SArray<feaid_t>& fea_ids, int value_type, const SArray<real_t>& values,
              const SArray<int>& lens) override {
    if (value_type == Store::kFeaCount) {
      DFB_CHECK(fea_ids.size() == values.size());
      engine_->Check(dfb_push_feacnt(engine_->handle(), fea_ids.data(), fea_ids.size(), values.data()),
                     "dfb_push_feacnt");
    } else if (value_type == Store::kGradient) {
      engine_->Check(dfb_push_grad(engine_->handle(), fea_ids.data(), fea_ids.size(), values.data(), values.size(),
                                   lens.data(), lens.size()), "dfb_push_grad");
    } else {
      throw Error("unknown value type");
    }
  }
  const SGDUpdaterParamView& param() const { return param_; }
  const std::shared_ptr<GpuEngine>& engine() const { return engine_; }

 private:
  std::shared_ptr<GpuEngine> engine_;
  SGDUpdaterParamView param_;
};

class GpuFMLoss : public Loss {
 public:
  /** FMLossParam: V_dim (fm_loss.h:19-27).  Stand-alone use (as in the reference's fm_loss_test.cc)
   * creates a private engine; inside SGDLearner the updater's engine is attached instead. */
  KWArgs Init(const KWArgs& kwargs) override {
    KWArgs remain;
    for (const auto& kv : kwargs) {
      if (kv.first == "V_dim") V_dim_ = std::stoi(kv.second);
      else remain.push_back(kv);
    }
    if (V_dim_ < 0 || V_dim_ > 10000) throw ParamError("value for Parameter V_dim exceed bound [0,10000]");
    if (!engine_) engine_ = std::make_shared<GpuEngine>(KWArgs{{"V_dim", std::to_string(V_dim_)}, {"table_capacity", "1024"}});
    return remain;
  }
  void AttachEngine(const std::shared_ptr<GpuEngine>& e) { engine_ = e; }

  void Predict(const dmlc::RowBlock<unsigned>& data, const std::vector<SArray<char>>& param,
               SArray<real_t>* pred) override {
    DFB_CHECK(param.size() == 3);
    Predict(data, SArray<real_t>(param[0]), SArray<int>(param[1]), SArray<int>(param[2]), pred);
  }
  /** FMLoss::Predict (fm_loss.h:67-119): pred += X w + .5 sum((XV)^2 - (X.X)(V.V)), clamped */
  void Predict(const dmlc::RowBlock<unsigned>& data, const SArray<real_t>& weights, const SArray<int>& w_pos,
               const SArray<int>& V_pos, SArray<real_t>* pred) {
    DFB_CHECK(pred->size() == data.size);
    DFB_CHECK(w_pos.size() == V_pos.size());
    engine_->Check(dfb_predict(engine_->handle(), data.size, reinterpret_cast<const uint64_t*>(data.offset),
                               data.index, data.value, weights.data(), weights.size(),
                               w_pos.empty() ? nullptr : w_pos.data(), V_pos.empty() ? nullptr : V_pos.data(),
                               w_pos.size(), pred->data()), "dfb_predict");
  }
  /** Loss::Evaluate (loss.h:57-66) */
  real_t Evaluate(dmlc::real_t const* label, const SArray<real_t>& pred) const override {
    float objv = 0;
    engine_->Check(dfb_evaluate(engine_->handle(), label, pred.data(), pred.size(), &objv), "dfb_evaluate");
    return objv;
  }
  void CalcGrad(const dmlc::RowBlock<unsigned>& data, const std::vector<SArray<char>>& param,
                SArray<real_t>* grad) override {
    DFB_CHECK(param.size() == 4);
    CalcGrad(data, SArray<real_t>(param[0]), SArray<int>(param[1]), SArray<int>(param[2]),
             SArray<real_t>(param[3]), grad);
  }
  /** FMLoss::CalcGrad (fm_loss.h:148-199) */
  void CalcGrad(const dmlc::RowBlock<unsigned>& data, const SArray<real_t>& weights, const SArray<int>& w_pos,
                const SArray<int>& V_pos, const SArray<real_t>& pred, SArray<real_t>* grad) {
    DFB_CHECK(pred.size() == data.size);
    DFB_CHECK(grad->size() == weights.size());
    engine_->Check(dfb_calc_grad(engine_->handle(), data.size, reinterpret_cast<const uint64_t*>(data.offset),
                                 data.index, data.value, data.label, weights.data(), weights.size(),
                                 w_pos.empty() ? nullptr : w_pos.data(), V_pos.empty() ? nullptr : V_pos.data(),
                                 w_pos.size(), pred.data(), grad->data()), "dfb_calc_grad");
  }
  /** BinClassMetric::AUC (bin_class_metric.h:35-56), returns AUC * n */
  real_t AUC(dmlc::real_t const* label, const SArray<real_t>& pred) const {
    float a = 0;
    engine_->Check(dfb_auc(engine_->handle(), label, pred.data(), pred.size(), &a), "dfb_auc");
    return a;
  }
  const std::shared_ptr<GpuEngine>& engine() const { return engine_; }

 private:
  std::shared_ptr<GpuEngine> engine_;
  int V_dim_ = 0;
};

/** StoreLocal (store_local.h:19-49): synchronous passthrough to the updater */
class GpuStore : public Store {
 public:
  KWArgs Init(const KWArgs& kwargs) override { return kwargs; }
  int Push(const SArray<feaid_t>& fea_ids, int val_type, const SArray<real_t>& vals, const SArray<int>& lens,
           const std::function<void()>& on_complete = nullptr) override {
    updater_->Update(fea_ids, val_type, vals, lens);   // the C-ABI copies its inputs to the device
    if (on_complete) on_complete();
    return time_++;
  }
  int Pull(const SArray<feaid_t>& fea_ids, int val_type, SArray<real_t>* vals, SArray<int>* lens,
           const std::function<void()>& on_complete = nullptr) override {
    updater_->Get(fea_ids, val_type, vals, lens);
    if (on_complete) on_complete();
    return time_++;
  }
  void Wait(int) override {}
  int Rank() override { return 0; }
  int NumWorkers() override { return 1; }
  int NumServers() override { return 1; }

 private:
  int time_ = 0;
};

}  // namespace difacto
