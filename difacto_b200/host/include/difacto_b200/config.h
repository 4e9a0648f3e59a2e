// difacto_b200/host/include/difacto_b200/config.h -- the key=value .conf surface.
// ArgParser restates src/common/arg_parser.h + dmlc::Config's tokenizer (dmlc-core/src/config.cc):
// tokens are [^\s=]+ | "quoted" | = ; '#' starts a comment; `argfile=path` inlines a file AFTER the
// command-line arguments and, as in dmlc::Config, the LAST occurrence of a key wins -- so values in
// the argfile override the command line, exactly like the reference.
#pragma once
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "api.h"

namespace difacto {

class ArgParser {
 public:
  void AddArg(const char* argv) { data_.append(argv); data_.append(" "); }
  KWArgs GetKWArgs() {
    KWArgs kw = Tokenize(data_);
    for (const auto& it : kw) {
      if (it.first == "argfile") {
        std::ifstream f(it.second);
        if (!f) throw Error("failed to open " + it.second);
        std::stringstream ss;
        ss << f.rdbuf();
        data_.append(ss.str());
        kw = Tokenize(data_);
        break;
      }
    }
    KWArgs out;
    for (const auto& it : kw) if (it.first != "argfile") out.push_back(it);
    return out;
  }

 private:
  static KWArgs Tokenize(const std::string& s) {
    std::vector<std::string> tok;
    size_t i = 0;
    const size_t n = s.size();
    while (i < n) {
      const char c = s[i];
      if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { ++i; continue; }
      if (c == '#') { while (i < n && s[i] != '\n' && s[i] != '\r') ++i; continue; }
      if (c == '=') { tok.push_back("="); ++i; continue; }
      if (c == '"') {
        std::string t;
        ++i;
        while (i < n && s[i] != '"') {
          if (s[i] == '\\' && i + 1 < n && s[i + 1] == '"') { t += '"'; i += 2; continue; }
          t += s[i++];
        }
        ++i;
        tok.push_back(t);
        continue;
      }
      std::string t;
      while (i < n && s[i] != ' ' && s[i] != '\t' && s[i] != '\n' && s[i] != '\r' && s[i] != '=' && s[i] != '#') t += s[i++];
      tok.push_back(t);
    }
    // k = v triples; the last occurrence of a key wins and keeps its (last) position
    std::vector<std::pair<std::string, std::string>> all;
    if (tok.size() % 3 != 0) throw Error("Parsing error: expect format \"k = v\"");
    for (size_t t = 0; t + 3 <= tok.size(); t += 3) {
      if (tok[t + 1] != "=") throw Error("Parsing error: expect format \"k = v\" near \"" + tok[t] + "\"");
      all.push_back(std::make_pair(tok[t], tok[t + 2]));
    }
    KWArgs out;
    for (size_t a = 0; a < all.size(); ++a) {
      bool later = false;
      for (size_t b = a + 1; b < all.size(); ++b) if (all[b].first == all[a].first) { later = true; break; }
      if (!later) out.push_back(all[a]);
    }
    return out;
  }
  std::string data_;
};

/** SGDLearnerParam, src/sgd/sgd_param.h:12-64: same keys, defaults and required fields */
struct SGDLearnerParam {
  std::string data_in, data_val, data_format = "libsvm", model_out, model_in, loss = "fm";
  std::string pred_out;   // engine-only: where task=predict writes one prediction per input row
                          // (task=predict also takes the engine keys score_only = 1 and V_storage = bf16: the model
                          // is loaded without its AdaGrad state, V rows in fp32 or bf16, on one GPU or -- the parts of
                          // a num_gpus run, num_gpus = N -- into N scoring ranks of the sharded store, which run predict
                          // steps with or without pred_out)
  int max_num_epochs = 20, num_jobs_per_epoch = 10, batch_size = -1, shuffle = 10;
  float neg_sampling = 1, stop_rel_objv = 1e-5f, stop_val_auc = 1e-5f;
  int fused = 1;   // engine-only: 1 = raw block -> one device call, 2 = host localizer + one device call,
                   // 0 = the reference's Pull/Predict/CalcGrad/Push plugin calls
  int num_gpus = 1;          // engine-only: > 1 = the NVLink-sharded store over GPUs 0..num_gpus-1 (one worker thread
                             // and one table shard per GPU, dfb_shard_*; needs fused = 1)
  long long shard_max_nnz = 0;   // engine-only: capacity (non-zeros) of one minibatch in the sharded store;
                                 // 0 = batch_size * 256
  // engine-only: a checkpoint every checkpoint_period training minibatches per worker (0: none) into
  // checkpoint_out.<c>.* and the pointer file checkpoint_out; checkpoint_in resumes the run a pointer file names
  std::string checkpoint_out, checkpoint_in;
  long long checkpoint_period = 0;
  // engine-only: every prune_period training minibatches per worker (0: never) drop the table entries with w == 0, no
  // V row and fea_cnt <= prune_count (dfb_prune)
  long long prune_period = 0;
  float prune_count = 0;
  // 1: the periodic prune drops every entry with fea_cnt <= prune_count, V rows included, and compacts the V-row pool
  // (dfb_prune_rare); 0: only the entries that carry no weight (dfb_prune)
  int prune_rare = 0;

  KWArgs InitAllowUnknown(const KWArgs& kwargs) {
    KWArgs remain;
    bool has_data_in = false;
    for (const auto& kv : kwargs) {
      const std::string &k = kv.first, &v = kv.second;
      try {
        if (k == "data_in") { data_in = v; has_data_in = true; }
        else if (k == "data_val") data_val = v;
        else if (k == "data_format") data_format = v;
        else if (k == "model_out") model_out = v;
        else if (k == "model_in") model_in = v;
        else if (k == "pred_out") pred_out = v;
        else if (k == "loss") loss = v;
        else if (k == "max_num_epochs") max_num_epochs = std::stoi(v);
        else if (k == "num_jobs_per_epoch") num_jobs_per_epoch = std::stoi(v);
        else if (k == "batch_size") batch_size = std::stoi(v);
        else if (k == "shuffle") shuffle = std::stoi(v);
        else if (k == "neg_sampling") neg_sampling = std::stof(v);
        else if (k == "stop_rel_objv") stop_rel_objv = std::stof(v);
        else if (k == "stop_val_auc") stop_val_auc = std::stof(v);
        else if (k == "fused") fused = std::stoi(v);
        else if (k == "num_gpus") num_gpus = std::stoi(v);
        else if (k == "shard_max_nnz") shard_max_nnz = std::stoll(v);
        else if (k == "checkpoint_out") checkpoint_out = v;
        else if (k == "checkpoint_in") checkpoint_in = v;
        else if (k == "checkpoint_period") checkpoint_period = std::stoll(v);
        else if (k == "prune_period") prune_period = std::stoll(v);
        else if (k == "prune_count") prune_count = std::stof(v);
        else if (k == "prune_rare") prune_rare = std::stoi(v);
        else remain.push_back(kv);
      } catch (const std::logic_error&) {
        throw ParamError("Invalid Parameter format for " + k + " value='" + v + "'");
      }
    }
    if (!has_data_in) throw ParamError("Required parameter data_in of string is not presented");
    if (batch_size < 0) throw ParamError("Required parameter batch_size of int is not presented");   // sgd_param.h:58
    if (checkpoint_period < 0) throw ParamError("checkpoint_period must be >= 0");
    if (checkpoint_period > 0 && checkpoint_out.empty()) throw ParamError("checkpoint_period needs checkpoint_out");
    if (prune_period < 0) throw ParamError("prune_period must be >= 0");
    if (prune_count != prune_count) throw ParamError("prune_count must be a number");
    if (prune_rare != 0 && prune_rare != 1) throw ParamError("prune_rare must be 0 or 1");
    return remain;
  }
};

}  // namespace difacto
