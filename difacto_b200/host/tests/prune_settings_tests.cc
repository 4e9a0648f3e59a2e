// difacto_b200/host/tests/prune_settings_tests.cc -- the prune_period / prune_count keys (no device needed): how
// they parse, their checks, and that the checkpoint fingerprint records them so that a resume under other prune
// settings is refused by name.  Prints "ok" and exits 0 when every check holds.
#include <cstdio>
#include <string>

#include "difacto_b200/sgd_learner.h"

using namespace difacto;   // NOLINT

static int g_fail = 0;
#define EXPECT_TRUE(c) do { if (!(c)) { printf("  EXPECT failed: %s (%s:%d)\n", #c, __FILE__, __LINE__); ++g_fail; } } while (0)

static std::string Setting(const std::vector<std::pair<std::string, std::string>>& s, const std::string& k) {
  for (const auto& kv : s) if (kv.first == k) return kv.second;
  return "<missing>";
}

static bool Throws(const KWArgs& kw) {
  try {
    SGDLearnerParam p;
    p.InitAllowUnknown(kw);
  } catch (const ParamError&) {
    return true;
  }
  return false;
}

// the message CheckSettings refuses `now` with ("" when it accepts)
static std::string Refusal(const CheckpointState& saved, const std::vector<std::pair<std::string, std::string>>& now) {
  try {
    saved.CheckSettings(now, SGDLearner::SettingsAddedLater());
  } catch (const Error& e) {
    return e.what();
  }
  return "";
}

int main() {
  const KWArgs base = {{"data_in", "x"}, {"batch_size", "100"}};
  // defaults: off
  SGDLearnerParam p;
  KWArgs rest = p.InitAllowUnknown(base);
  EXPECT_TRUE(p.prune_period == 0 && p.prune_count == 0.f && rest.empty());
  // parsed as learner keys: never passed on to the engine
  KWArgs kw = base;
  kw.push_back({"prune_period", "25"});
  kw.push_back({"prune_count", "2.5"});
  kw.push_back({"l1", "3"});
  SGDLearnerParam q;
  rest = q.InitAllowUnknown(kw);
  EXPECT_TRUE(q.prune_period == 25 && q.prune_count == 2.5f);
  EXPECT_TRUE(rest.size() == 1 && rest[0].first == "l1");
  // checks
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_period", "-1"}}));
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_period", "often"}}));
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_count", "nan"}}));
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_count", "few"}}));
  // the fingerprint: parsed values, defaults when not given
  const auto s0 = SGDLearner::Settings(p, base);
  EXPECT_TRUE(Setting(s0, "prune_period") == "0" && Setting(s0, "prune_count") == "0");
  const auto s1 = SGDLearner::Settings(q, kw);
  EXPECT_TRUE(Setting(s1, "prune_period") == "25" && Setting(s1, "prune_count") == "2.5");
  KWArgs spelled = base;
  spelled.push_back({"prune_period", "+25"});
  spelled.push_back({"prune_count", "2.50"});
  spelled.push_back({"l1", "3.0"});
  SGDLearnerParam q2;
  q2.InitAllowUnknown(spelled);
  EXPECT_TRUE(SGDLearner::Settings(q2, spelled) == s1);    // the same settings spelled otherwise
  // a checkpoint taken under s1 resumes under s1 only; the refusal names the key
  CheckpointState saved;
  saved.settings = s1;
  const CheckpointState back = CheckpointState::Parse(saved.Serialize());
  EXPECT_TRUE(Refusal(back, s1).empty());
  EXPECT_TRUE(Refusal(back, s0).find("prune_period") != std::string::npos);
  KWArgs other = kw;
  other[3].second = "3";
  SGDLearnerParam q3;
  q3.InitAllowUnknown(other);
  EXPECT_TRUE(Refusal(back, SGDLearner::Settings(q3, other)).find("prune_count") != std::string::npos);
  // a checkpoint written before the prune keys existed records neither: it ran without pruning, so it resumes under
  // the defaults and is refused, by name, under pruning
  CheckpointState old;
  for (const auto& kv : s0) if (kv.first != "prune_period" && kv.first != "prune_count") old.settings.push_back(kv);
  EXPECT_TRUE(old.settings.size() + 2 == s0.size());
  const CheckpointState old_back = CheckpointState::Parse(old.Serialize());
  EXPECT_TRUE(Refusal(old_back, s0).empty());
  EXPECT_TRUE(Refusal(old_back, s1).find("prune_period") != std::string::npos);
  SGDLearnerParam q4;
  KWArgs count_only = base;
  count_only.push_back({"prune_count", "1"});
  q4.InitAllowUnknown(count_only);
  EXPECT_TRUE(Refusal(old_back, SGDLearner::Settings(q4, count_only)).find("prune_count") != std::string::npos);
  printf(g_fail ? "%d failed\n" : "ok\n", g_fail);
  return g_fail ? 1 : 0;
}
