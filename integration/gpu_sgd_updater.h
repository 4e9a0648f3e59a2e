/**
 * integration/gpu_sgd_updater.h -- the Updater a difacto maintainer drops into the REFERENCE tree (next to
 * src/sgd/sgd_updater.h) to run SGDUpdater's job on the GPU engine.  Compiled against the unmodified
 * reference headers (include/difacto/updater.h, src/sgd/sgd_updater.h, src/sgd/sgd_param.h of dmlc/difacto
 * @ 78e3562) by oracle/Makefile (target ref_gpu) and exercised under the reference's own SGDLearner by
 * tests/test_gpu_reference_binding.py.
 *
 * It derives from the reference's SGDUpdater so that SGDLearner::GetUpdater()'s static cast
 * (src/sgd/sgd_learner.h:33-36) and `updater->param().V_dim` (src/sgd/sgd_learner.cc:235) keep working; the
 * inherited unordered_map stays empty -- the model lives in HBM behind the C-ABI of include/difacto_b200.h.
 */
#ifndef INTEGRATION_GPU_SGD_UPDATER_H_
#define INTEGRATION_GPU_SGD_UPDATER_H_
#include <mutex>
#include <string>
#include <vector>
#include "sgd/sgd_updater.h"
#include "difacto/store.h"
#include "difacto_b200.h"
namespace difacto {

class GpuSGDUpdater : public SGDUpdater {
 public:
  GpuSGDUpdater() {}
  virtual ~GpuSGDUpdater() { if (h_) dfb_destroy(h_); }

  /** SGDUpdater::Init (sgd_updater.cc:9-11) parses SGDUpdaterParam; the same values create the engine.
   *  Engine-only keys (device, table_capacity, ...) are consumed here; the rest is returned like any Init. */
  KWArgs Init(const KWArgs& kwargs) override {
    KWArgs remain = SGDUpdater::Init(kwargs);
    const SGDUpdaterParam& p = param();
    std::vector<std::pair<std::string, std::string>> kv = {
      {"l1", std::to_string(p.l1)}, {"l2", std::to_string(p.l2)}, {"V_l2", std::to_string(p.V_l2)},
      {"lr", std::to_string(p.lr)}, {"lr_beta", std::to_string(p.lr_beta)}, {"V_lr", std::to_string(p.V_lr)},
      {"V_lr_beta", std::to_string(p.V_lr_beta)}, {"V_init_scale", std::to_string(p.V_init_scale)},
      {"V_dim", std::to_string(p.V_dim)}, {"V_threshold", std::to_string(p.V_threshold)},
      {"seed", std::to_string(p.seed)}};
    KWArgs rest;
    for (const auto& a : remain) {
      if (a.first == "device" || a.first == "table_capacity" || a.first == "V_capacity" ||
          a.first == "table_capacity_max" || a.first == "V_capacity_max" || a.first == "scatter")
        kv.push_back(a);
      else
        rest.push_back(a);
    }
    std::vector<const char*> k, v;
    for (const auto& a : kv) { k.push_back(a.first.c_str()); v.push_back(a.second.c_str()); }
    CHECK_EQ(dfb_create(k.data(), v.data(), static_cast<int>(k.size()), &h_), 0) << dfb_last_error(nullptr);
    V_dim_ = p.V_dim;
    return rest;
  }

  void Get(const SArray<feaid_t>& fea_ids, int value_type, SArray<real_t>* weights, SArray<int>* val_lens) override {
    CHECK_EQ(value_type, Store::kWeight);
    // a dfb_handle takes one call at a time; SGDLearner pushes feature counts from the job thread while the
    // batch thread pulls / pushes gradients (sgd_learner.cc:214-217 vs :177) -- SGDUpdater holds a mutex too (cc:41,61)
    std::lock_guard<std::mutex> lk(gpu_mu_);
    const size_t n = fea_ids.size();
    weights->resize(n * (1 + V_dim_));
    val_lens->resize(n);
    size_t nv = 0, nl = 0;
    CHECK_EQ(dfb_pull(h_, fea_ids.data(), n, weights->data(), weights->size(), val_lens->data(), &nv, &nl), 0)
        << dfb_last_error(h_);
    weights->resize(nv);
    val_lens->resize(nl);     // empty when V_dim == 0, like sgd_updater.cc:40
  }

  void Update(const SArray<feaid_t>& fea_ids, int value_type, const SArray<real_t>& values,
              const SArray<int>& val_lens) override {
    std::lock_guard<std::mutex> lk(gpu_mu_);
    int rc;
    if (value_type == Store::kFeaCount) {
      CHECK_EQ(fea_ids.size(), values.size());
      rc = dfb_push_feacnt(h_, fea_ids.data(), fea_ids.size(), values.data());
    } else {
      CHECK_EQ(value_type, Store::kGradient);
      rc = dfb_push_grad(h_, fea_ids.data(), fea_ids.size(), values.data(), values.size(), val_lens.data(),
                         val_lens.size());
    }
    CHECK_EQ(rc, 0) << dfb_last_error(h_);    // LOG(FATAL), like every CHECK of the reference
  }

  dfb_handle handle() const { return h_; }

 private:
  dfb_handle h_ = nullptr;
  int V_dim_ = 0;
  std::mutex gpu_mu_;
};

}  // namespace difacto
#endif  // INTEGRATION_GPU_SGD_UPDATER_H_
