// difacto_b200/host/tests/prune_rare_settings_tests.cc -- the prune_rare key (no device needed): how it parses, that
// the checkpoint fingerprint records it only when it is set (so the fingerprint at the defaults, and every checkpoint
// written before the key existed, stay as they were), and that a resume under another value is refused by name.
// Prints "ok" and exits 0 when every check holds.
#include <cstdio>
#include <string>

#include "difacto_b200/sgd_learner.h"

using namespace difacto;   // NOLINT

static int g_fail = 0;
#define EXPECT_TRUE(c) do { if (!(c)) { printf("  EXPECT failed: %s (%s:%d)\n", #c, __FILE__, __LINE__); ++g_fail; } } while (0)

typedef std::vector<std::pair<std::string, std::string>> SettingList;

static std::string Setting(const SettingList& s, const std::string& k) {
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
static std::string Refusal(const CheckpointState& saved, const SettingList& now) {
  try {
    saved.CheckSettings(now, SGDLearner::SettingsAddedLater());
  } catch (const Error& e) {
    return e.what();
  }
  return "";
}

static SettingList SettingsOf(const KWArgs& kw) {
  SGDLearnerParam p;
  p.InitAllowUnknown(kw);
  return SGDLearner::Settings(p, kw);
}

static CheckpointState Saved(const SettingList& s) {
  CheckpointState st;
  st.settings = s;
  return CheckpointState::Parse(st.Serialize());
}

int main() {
  const KWArgs base = {{"data_in", "x"}, {"batch_size", "100"}, {"prune_period", "10"}, {"prune_count", "1"}};
  KWArgs rare = base;
  rare.push_back({"prune_rare", "1"});
  // parsing: off by default, a learner key (never passed on to the engine), 0 or 1 only
  SGDLearnerParam p;
  KWArgs rest = p.InitAllowUnknown(base);
  EXPECT_TRUE(p.prune_rare == 0 && rest.empty());
  SGDLearnerParam q;
  rest = q.InitAllowUnknown(rare);
  EXPECT_TRUE(q.prune_rare == 1 && rest.empty());
  KWArgs zero = base;
  zero.push_back({"prune_rare", "0"});
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_rare", "2"}}));
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_rare", "-1"}}));
  EXPECT_TRUE(Throws({{"data_in", "x"}, {"batch_size", "1"}, {"prune_rare", "yes"}}));
  // the fingerprint: unchanged at the default, whether the key is given as 0 or not given; recorded when set
  const SettingList s0 = SettingsOf(base), sz = SettingsOf(zero), s1 = SettingsOf(rare);
  EXPECT_TRUE(Setting(s0, "prune_rare") == "<missing>" && sz == s0);
  EXPECT_TRUE(Setting(s1, "prune_rare") == "1" && s1.size() == s0.size() + 1);
  KWArgs spelled = base;
  spelled.push_back({"prune_rare", "+1"});
  EXPECT_TRUE(SettingsOf(spelled) == s1);
  // a checkpoint under prune_rare = 1 resumes under it only, and the refusal names the key
  EXPECT_TRUE(Refusal(Saved(s1), s1).empty());
  EXPECT_TRUE(Refusal(Saved(s1), s0).find("prune_rare") != std::string::npos);
  EXPECT_TRUE(Refusal(Saved(s1), sz).find("prune_rare") != std::string::npos);
  // a checkpoint under the default (and every one written before the key existed) records no prune_rare: it resumes
  // under the default and is refused, by name, under prune_rare = 1
  EXPECT_TRUE(Refusal(Saved(s0), s0).empty());
  EXPECT_TRUE(Refusal(Saved(s0), s1).find("prune_rare") != std::string::npos);
  // one written before any prune key existed
  SettingList old;
  for (const auto& kv : SettingsOf({{"data_in", "x"}, {"batch_size", "100"}}))
    if (kv.first != "prune_period" && kv.first != "prune_count") old.push_back(kv);
  const SettingList now_default = SettingsOf({{"data_in", "x"}, {"batch_size", "100"}});
  EXPECT_TRUE(Refusal(Saved(old), now_default).empty());
  KWArgs old_rare = {{"data_in", "x"}, {"batch_size", "100"}, {"prune_rare", "1"}};
  EXPECT_TRUE(Refusal(Saved(old), SettingsOf(old_rare)).find("prune_rare") != std::string::npos);
  // another setting that differs is still named first
  KWArgs other = rare;
  other[3].second = "2";
  EXPECT_TRUE(Refusal(Saved(s1), SettingsOf(other)).find("prune_count") != std::string::npos);
  printf(g_fail ? "%d failed\n" : "ok\n", g_fail);
  return g_fail ? 1 : 0;
}
