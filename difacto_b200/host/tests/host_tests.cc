// difacto_b200/host/tests/host_tests.cc -- the reference's hot-path gtest cases, re-expressed
// against the host mirror API (same test names, inputs and golden values):
//   tests/cpp/fm_loss_test.cc      FMLoss.NoV / FMLoss.HasV
//   tests/cpp/localizer_test.cc    Localizer.Base / BaseHash / ReverseBytes
//   tests/cpp/sgd_learner_test.cc  SGDLearner.Basic (stop_rel_objv=0 so that all 20 epochs run)
// plus SGDLearner.PluginCallsEqualFused (fused=0 vs fused=1).  No gtest in this image: a 30-line
// harness.  Data: $DFB_TEST_DATA = the reference's 100-row fixture written as libsvm text.
// Usage: host_tests [filter]; tests whose name starts with "Gpu" need a device.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "difacto_b200/sgd_learner.h"

using namespace difacto;   // NOLINT

static int g_fail = 0;
#define EXPECT_TRUE(c) do { if (!(c)) { printf("  EXPECT failed: %s (%s:%d)\n", #c, __FILE__, __LINE__); ++g_fail; } } while (0)
#define EXPECT_LT(a, b) do { double _a = (a), _b = (b); if (!(_a < _b)) { printf("  EXPECT_LT failed: %s = %.9g !< %s = %.9g (%s:%d)\n", #a, _a, #b, _b, __FILE__, __LINE__); ++g_fail; } } while (0)
#define EXPECT_EQ(a, b) do { if (!((a) == (b))) { printf("  EXPECT_EQ failed: %s vs %s (%s:%d)\n", #a, #b, __FILE__, __LINE__); ++g_fail; } } while (0)

static std::string DataPath() {
  const char* p = getenv("DFB_TEST_DATA");
  return p ? p : "../tests/data";
}

template <typename T>
double norm1(const T* d, size_t n) { double s = 0; for (size_t i = 0; i < n; ++i) s += std::fabs(static_cast<double>(d[i])); return s; }
template <typename T>
double norm2(const T* d, size_t n) { double s = 0; for (size_t i = 0; i < n; ++i) s += static_cast<double>(d[i]) * d[i]; return s; }

// tests/cpp/utils.h:126-136
static void load_data(RowBlockContainer<unsigned>* data, std::vector<feaid_t>* uidx) {
  BatchReader reader(DataPath(), "libsvm", 0, 1, 100);
  DFB_CHECK(reader.Next());
  Localizer lc;
  lc.Compact(reader.Value(), data, uidx);
  if (uidx) for (auto& i : *uidx) i = ReverseBytes(i);
}

static void Localizer_Base() {
  BatchReader reader(DataPath(), "libsvm", 0, 1, 100);
  DFB_CHECK(reader.Next());
  RowBlockContainer<unsigned> compact;
  std::vector<feaid_t> uidx;
  std::vector<real_t> freq;
  Localizer lc;
  lc.Compact(reader.Value(), &compact, &uidx, &freq);
  for (auto& i : uidx) i = ReverseBytes(i);
  EXPECT_EQ(static_cast<uint64_t>(norm1(uidx.data(), uidx.size())), 65111856ull);   // localizer_test.cc:26
  EXPECT_EQ(norm1(freq.data(), freq.size()), 9648.0);                               // :27
  auto blk = reader.Value();
  EXPECT_EQ(norm1(blk.offset, 101), norm1(compact.offset.data(), 101));
  EXPECT_EQ(norm2(blk.value, blk.offset[100]), norm2(compact.value.data(), compact.offset[100]));
}

static void Localizer_BaseHash() {
  BatchReader reader(DataPath(), "libsvm", 0, 1, 100);
  DFB_CHECK(reader.Next());
  RowBlockContainer<unsigned> compact;
  std::vector<feaid_t> uidx;
  std::vector<real_t> freq;
  Localizer lc(1000);
  lc.Compact(reader.Value(), &compact, &uidx, &freq);
  for (auto& i : uidx) i = ReverseBytes(i);
  EXPECT_EQ(static_cast<uint64_t>(norm1(uidx.data(), uidx.size())), 478817ull);     // localizer_test.cc:48
  EXPECT_EQ(norm1(freq.data(), freq.size()), 9648.0);
}

static void Localizer_ReverseBytes() {
  feaid_t max = static_cast<feaid_t>(-1);
  const int n = 1000000;
  for (int i = 0; i < n; i += 7) {
    feaid_t j = (max / n) * i;
    EXPECT_TRUE(j == ReverseBytes(ReverseBytes(j)));
  }
}

// tests/cpp/batch_reader_test.cc:9-57 (same goldens)
static const int kBatch = 37;
static const int kLabelSum[] = {11, 15, 10};
static const int kLen[] = {37, 37, 26};
static const size_t kOffSum[] = {85035, 63968, 31323};
static const uint64_t kIdxSum[] = {95285478, 70504854, 62972349};
static const float kValNorm[] = {37.0f, 37.0f, 26.0f};

static void BatchReader_Read() {
  BatchReader reader(DataPath(), "libsvm", 0, 1, kBatch);
  int i = 0;
  while (reader.Next() && i < 3) {
    auto b = reader.Value();
    double ls = 0;
    for (size_t r = 0; r < b.size; ++r) ls += b.label[r];
    EXPECT_EQ(static_cast<int>(ls), kLabelSum[i]);
    EXPECT_EQ(static_cast<int>(b.size), kLen[i]);
    EXPECT_EQ(static_cast<size_t>(norm1(b.offset, b.size + 1)), kOffSum[i]);
    EXPECT_EQ(static_cast<uint64_t>(norm1(b.index, b.offset[b.size])), kIdxSum[i]);
    EXPECT_LT(std::fabs(kValNorm[i] - norm2(b.value, b.offset[b.size])), 1e-4);
    ++i;
  }
  EXPECT_EQ(i, 3);
}

static void BatchReader_RandRead() {
  BatchReader reader(DataPath(), "libsvm", 0, 1, kBatch, kBatch);
  int i = 0;
  while (reader.Next() && i < 3) {
    auto b = reader.Value();
    double ls = 0;
    for (size_t r = 0; r < b.size; ++r) ls += b.label[r];
    EXPECT_EQ(static_cast<int>(ls), kLabelSum[i]);
    EXPECT_EQ(static_cast<int>(b.size), kLen[i]);
    EXPECT_TRUE(static_cast<size_t>(norm1(b.offset, b.size + 1)) != kOffSum[i]);   // shuffled rows
    EXPECT_EQ(static_cast<uint64_t>(norm1(b.index, b.offset[b.size])), kIdxSum[i]);
    EXPECT_LT(std::fabs(kValNorm[i] - norm2(b.value, b.offset[b.size])), 1e-4);
    ++i;
  }
  EXPECT_EQ(i, 3);
}

static void BatchReader_PartRead() {
  BatchReader reader(DataPath(), "libsvm", 1, 2, kBatch);
  int ttl = 0;
  while (reader.Next()) {
    auto b = reader.Value();
    EXPECT_LT(std::fabs(static_cast<double>(b.size) - norm2(b.value, b.offset[b.size])), 1e-4);
    ttl += static_cast<int>(b.size);
  }
  EXPECT_TRUE(ttl <= 60 && ttl >= 40);
  // the two halves partition the file: no row lost or duplicated
  BatchReader other(DataPath(), "libsvm", 0, 2, kBatch);
  int ttl0 = 0;
  while (other.Next()) ttl0 += static_cast<int>(other.Value().size);
  EXPECT_EQ(ttl + ttl0, 100);
}

// the part is streamed in chunks: any chunk size (here: smaller than one line, and a few lines) gives the rows of
// the one-chunk read, for whole files and for parts, with and without a shuffle window
static void BatchReader_StreamedChunks() {
  for (unsigned nparts : {1u, 3u}) {
    for (unsigned part = 0; part < nparts; ++part) {
      for (unsigned shuf : {0u, 50u}) {
        for (size_t chunk : {size_t(7), size_t(1000), size_t(4096)}) {
          BatchReader whole2(DataPath(), "libsvm", part, nparts, kBatch, shuf, 1.0f, 2);
          BatchReader piece(DataPath(), "libsvm", part, nparts, kBatch, shuf, 1.0f, 2, chunk);
          for (;;) {
            const bool a = whole2.Next(), b = piece.Next();
            EXPECT_TRUE(a == b);
            if (!a || !b) break;
            auto x = whole2.Value(), y = piece.Value();
            EXPECT_EQ(x.size, y.size);
            EXPECT_EQ(x.offset[x.size], y.offset[y.size]);
            EXPECT_TRUE(memcmp(x.index, y.index, sizeof(feaid_t) * x.offset[x.size]) == 0);
            EXPECT_TRUE(memcmp(x.label, y.label, sizeof(real_t) * x.size) == 0);
            EXPECT_TRUE((x.value == nullptr) == (y.value == nullptr));
            if (x.value && y.value) EXPECT_TRUE(memcmp(x.value, y.value, sizeof(real_t) * x.offset[x.size]) == 0);
          }
        }
      }
    }
  }
}

// the state record of a mid-epoch checkpoint reads back as it was written, float bits and all
static void CheckpointState_RoundTrip() {
  CheckpointState st;
  st.settings = {{"data_in", "a b.libsvm"}, {"batch_size", "100"}, {"id_bits", ""}};
  st.epoch = 3;
  st.workers = {{2, 17}, {5, 0}};
  st.has_rand = true;
  for (size_t i = 0; i < RandState::kBytes; ++i) st.rand.bytes[i] = static_cast<unsigned char>(i * 7 + 1);
  const float odd[5] = {1.0f / 3, -0.0f, 1e-38f, 123456.789f, 42.f};
  for (int i = 0; i < 5; ++i) { st.epoch_prog[i] = odd[i]; st.part_prog[i] = odd[4 - i] * 3; }
  st.pre_loss = 0.1f; st.pre_val_auc = 77.5f;
  st.minibatches = (1ULL << 40) + 3;
  st.id_ranges = {0, 37};
  const std::string rec = st.Serialize();
  const CheckpointState back = CheckpointState::Parse(rec);
  EXPECT_TRUE(back.Serialize() == rec);
  EXPECT_TRUE(back.settings == st.settings);
  EXPECT_EQ(back.epoch, 3);
  EXPECT_EQ(back.workers.size(), size_t(2));
  EXPECT_EQ(back.workers[0].part, 2);
  EXPECT_EQ(back.workers[0].consumed, uint64_t(17));
  EXPECT_TRUE(memcmp(back.epoch_prog, st.epoch_prog, sizeof(st.epoch_prog)) == 0);
  EXPECT_TRUE(memcmp(back.part_prog, st.part_prog, sizeof(st.part_prog)) == 0);
  EXPECT_TRUE(memcmp(back.rand.bytes, st.rand.bytes, RandState::kBytes) == 0);
  EXPECT_EQ(back.minibatches, st.minibatches);
  EXPECT_TRUE(back.id_ranges == st.id_ranges);
  // a different setting is refused by name; a truncated record is refused
  bool named = false;
  try {
    back.CheckSettings({{"batch_size", "200"}});
  } catch (const Error& e) {
    named = std::string(e.what()).find("batch_size") != std::string::npos;
  }
  EXPECT_TRUE(named);
  bool truncated = false;
  try {
    CheckpointState::Parse(rec.substr(0, rec.size() - 3));
  } catch (const Error&) {
    truncated = true;
  }
  EXPECT_TRUE(truncated);
}

// rand() saved before a reference-order reader starts and restored later gives that reader's batches again, whatever
// was drawn in between
static void CheckpointState_RandRestoresTheReader() {
  auto dump = [](std::vector<std::vector<feaid_t>>* out) {
    BatchReader r(DataPath(), "libsvm", 0, 1, 10, 30, 0.5f, 0, 0, ShuffleOrder::kReference);
    while (r.Next()) {
      auto b = r.Value();
      out->push_back(std::vector<feaid_t>(b.index, b.index + b.offset[b.size]));
      out->back().push_back(static_cast<feaid_t>(b.size));
    }
  };
  const RandState at = RandState::Save();
  std::vector<std::vector<feaid_t>> first, again, moved;
  dump(&first);
  dump(&moved);                // rand() has moved on: another order
  at.Restore();
  dump(&again);
  EXPECT_TRUE(first.size() >= 3);
  EXPECT_TRUE(first == again);
  EXPECT_TRUE(first != moved);
  for (int i = 0; i < 1000; ++i) rand();
  at.Restore();
  const int x = rand();
  at.Restore();
  EXPECT_EQ(rand(), x);
}

static void ArgParser_LastValueWins() {
  ArgParser p;
  p.AddArg("V_dim=64");
  p.AddArg("l1 = 2");
  p.AddArg("V_dim=10");
  KWArgs kw = p.GetKWArgs();
  EXPECT_EQ(kw.size(), 2u);
  EXPECT_TRUE(kw[0].first == "l1" && kw[0].second == "2");
  EXPECT_TRUE(kw[1].first == "V_dim" && kw[1].second == "10");
  bool threw = false;
  try { SGDLearnerParam sp; sp.InitAllowUnknown({{"data_in", "x"}}); } catch (const ParamError&) { threw = true; }
  EXPECT_TRUE(threw);   // batch_size is required (sgd_param.h:58)
}

static void GpuFMLoss_NoV() {
  SArray<real_t> weight(47149);
  for (size_t i = 0; i < weight.size(); ++i) weight[i] = i / 5e4;
  RowBlockContainer<unsigned> rowblk;
  std::vector<feaid_t> uidx;
  load_data(&rowblk, &uidx);
  SArray<real_t> w(uidx.size());
  for (size_t i = 0; i < uidx.size(); ++i) w[i] = weight[uidx[i]];
  KWArgs args = {{"V_dim", "0"}};
  GpuFMLoss loss;
  loss.Init(args);
  auto data = rowblk.GetBlock();
  SArray<real_t> pred(data.size);
  loss.Predict(data, w, SArray<int>(), SArray<int>(), &pred);
  EXPECT_LT(std::fabs(loss.Evaluate(data.label, pred) - 147.4672), 1e-3);           // fm_loss_test.cc:35
  SArray<real_t> grad(w.size());
  loss.CalcGrad(data, w, SArray<int>(), SArray<int>(), pred, &grad);
  EXPECT_LT(std::fabs(norm2(grad.data(), grad.size()) - 90.5817), 1e-3);            // :39
}

static void GpuFMLoss_HasV() {
  const int V_dim = 5, n = 47149;
  std::vector<real_t> weight(static_cast<size_t>(n) * (V_dim + 1));
  for (int i = 0; i < n; ++i) {
    weight[i * (V_dim + 1)] = i / 5e4;
    for (int j = 1; j <= V_dim; ++j) weight[i * (V_dim + 1) + j] = i * j / 5e5;
  }
  RowBlockContainer<unsigned> rowblk;
  std::vector<feaid_t> uidx;
  load_data(&rowblk, &uidx);
  SArray<int> w_pos(uidx.size()), V_pos(uidx.size());
  SArray<real_t> w(uidx.size() * (V_dim + 1));
  int p = 0;
  for (size_t i = 0; i < uidx.size(); ++i) {
    for (int j = 0; j < V_dim + 1; ++j) w[i * (V_dim + 1) + j] = weight[uidx[i] * (V_dim + 1) + j];
    w_pos[i] = p; V_pos[i] = p + 1; p += V_dim + 1;
  }
  KWArgs args = {{"V_dim", std::to_string(V_dim)}};
  GpuFMLoss loss;
  loss.Init(args);
  auto data = rowblk.GetBlock();
  SArray<real_t> pred(data.size);
  loss.Predict(data, w, w_pos, V_pos, &pred);
  EXPECT_LT(std::fabs(loss.Evaluate(data.label, pred) - 330.628), 1e-3);            // fm_loss_test.cc:78
  SArray<real_t> grad(w.size());
  loss.CalcGrad(data, w, w_pos, V_pos, pred, &grad);
  EXPECT_LT(std::fabs(norm2(grad.data(), grad.size()) - 1.2378e+03), 1e-1);         // :82
}

static const double kSgdGolden[20] = {69.314718, 69.314718, 67.151912, 61.414778, 56.244989, 53.218700, 51.248737,
                                      49.846688, 48.650164, 47.698351, 46.924038, 46.388223, 45.970721, 45.499307,
                                      45.102245, 44.798413, 44.565211, 44.386417, 44.240657, 44.109764};

static std::vector<double> RunBasic(const char* fused, const char* V_dim, std::vector<double>* pen) {
  SGDLearner learner;
  learner.verbose = false;
  KWArgs args = {{"data_in", DataPath()}, {"V_dim", V_dim}, {"l2", "1"}, {"l1", "1"}, {"lr", "1"},
                 {"num_jobs_per_epoch", "1"}, {"batch_size", "100"}, {"max_num_epochs", "20"},
                 {"stop_rel_objv", "0"}, {"fused", fused}, {"V_threshold", "2"}, {"table_capacity", "8192"}};
  auto remain = learner.Init(args);
  EXPECT_EQ(remain.size(), 0u);
  std::vector<double> losses;
  learner.AddEpochEndCallback([&](int, const sgd::Progress& train, const sgd::Progress&) {
    losses.push_back(train.loss);
    if (pen) pen->push_back(train.penalty);
  });
  learner.Run();
  return losses;
}

static void GpuSGDLearner_Basic() {   // sgd_learner_test.cc:9-49, tolerance 5e-5 there; 2e-4 here (fp32 sum order)
  auto losses = RunBasic("1", "0", nullptr);
  EXPECT_EQ(losses.size(), 20u);
  for (size_t e = 0; e < losses.size() && e < 20; ++e) EXPECT_LT(std::fabs(losses[e] - kSgdGolden[e]), 2e-4);
}

static void GpuSGDUpdater_SaveLoad() {
  // train 5 epochs, save, load into a fresh updater: identical Get() for every key
  KWArgs args = {{"V_dim", "8"}, {"l1", "0.1"}, {"lr", "0.5"}, {"V_threshold", "1"}, {"table_capacity", "8192"}};
  GpuSGDUpdater a, b;
  a.Init(args);
  b.Init(args);
  RowBlockContainer<unsigned> data;
  std::vector<feaid_t> keys;
  std::vector<real_t> cnt;
  {
    BatchReader reader(DataPath(), "libsvm", 0, 1, 100);
    DFB_CHECK(reader.Next());
    Localizer lc;
    lc.Compact(reader.Value(), &data, &keys, &cnt);
  }
  for (int ep = 0; ep < 5; ++ep) {
    dfb_progress pr;
    a.engine()->Check(dfb_train_step(a.engine()->handle(), data.Size(), reinterpret_cast<const uint64_t*>(data.offset.data()),
                                     data.index.data(), data.value.data(), data.label.data(), keys.data(), keys.size(),
                                     ep == 0 ? cnt.data() : nullptr, 1, &pr, nullptr), "step");
  }
  std::stringstream ss;
  a.Save(true, &ss);
  bool has_aux = false;
  b.Load(&ss, &has_aux);
  EXPECT_TRUE(has_aux);
  SArray<feaid_t> ids(keys.data(), keys.size());
  SArray<real_t> wa, wb;
  SArray<int> la, lb;
  a.Get(ids, Store::kWeight, &wa, &la);
  b.Get(ids, Store::kWeight, &wb, &lb);
  EXPECT_EQ(wa.size(), wb.size());
  EXPECT_TRUE(wa.size() == wb.size() && memcmp(wa.data(), wb.data(), wa.size() * sizeof(real_t)) == 0);
  EXPECT_TRUE(la.size() == lb.size() && memcmp(la.data(), lb.data(), la.size() * sizeof(int)) == 0);
  size_t nv = 0;
  for (int l : la) nv += l > 1;
  EXPECT_TRUE(nv > 100);
}

static void GpuSGDLearner_PluginCallsEqualFused() {
  for (const char* vd : {"0", "8"}) {
    std::vector<double> p1, p0, p2;
    auto fused = RunBasic("1", vd, &p1);
    auto plugin = RunBasic("0", vd, &p0);
    auto fused2 = RunBasic("2", vd, &p2);
    EXPECT_EQ(fused.size(), fused2.size());
    for (size_t e = 0; e < fused.size() && e < fused2.size(); ++e)
      EXPECT_LT(std::fabs(fused[e] - fused2[e]), 1e-3 * std::fabs(fused2[e]) + 1e-4);
    EXPECT_EQ(fused.size(), plugin.size());
    for (size_t e = 0; e < fused.size() && e < plugin.size(); ++e) {
      EXPECT_LT(std::fabs(fused[e] - plugin[e]), 1e-3 * std::fabs(plugin[e]) + 1e-4);
      EXPECT_LT(std::fabs(p1[e] - p0[e]), 1e-3 * std::fabs(p0[e]) + 1e-4);
    }
  }
}

struct Case { const char* name; void (*fn)(); };
static const Case kCases[] = {
    {"Localizer.Base", Localizer_Base}, {"Localizer.BaseHash", Localizer_BaseHash},
    {"Localizer.ReverseBytes", Localizer_ReverseBytes}, {"ArgParser.LastValueWins", ArgParser_LastValueWins},
    {"BatchReader.Read", BatchReader_Read}, {"BatchReader.RandRead", BatchReader_RandRead},
    {"BatchReader.PartRead", BatchReader_PartRead},
    {"BatchReader.StreamedChunks", BatchReader_StreamedChunks},
    {"CheckpointState.RoundTrip", CheckpointState_RoundTrip},
    {"CheckpointState.RandRestoresTheReader", CheckpointState_RandRestoresTheReader},
    {"GpuFMLoss.NoV", GpuFMLoss_NoV}, {"GpuFMLoss.HasV", GpuFMLoss_HasV},
    {"GpuSGDLearner.Basic", GpuSGDLearner_Basic}, {"GpuSGDUpdater.SaveLoad", GpuSGDUpdater_SaveLoad},
    {"GpuSGDLearner.PluginCallsEqualFused", GpuSGDLearner_PluginCallsEqualFused}};

int main(int argc, char** argv) {
  const char* filter = argc > 1 ? argv[1] : "";
  const bool exclude = filter[0] == '-';
  if (exclude) ++filter;
  int ran = 0, failed = 0;
  for (const auto& c : kCases) {
    const bool match = strstr(c.name, filter) != nullptr;
    if (*filter && (exclude ? match : !match)) continue;
    printf("[ RUN  ] %s\n", c.name);
    const int before = g_fail;
    try { c.fn(); } catch (const std::exception& e) { printf("  exception: %s\n", e.what()); ++g_fail; }
    const bool ok = g_fail == before;
    printf("[ %s ] %s\n", ok ? " OK " : "FAIL", c.name);
    ++ran;
    failed += !ok;
  }
  printf("%d tests ran, %d failed\n", ran, failed);
  return failed ? 1 : 0;
}
