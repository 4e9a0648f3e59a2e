// difacto_b200/host/src/main.cc -- the `difacto` command line for the SGD path on H100.
//   difacto_b200 key1=val1 key2=val2 ... [argfile=example.conf]
// Same surface as src/main.cc of the reference: task = train (default) | predict | convert,
// learner = sgd (default); unknown keys are warned about, not fatal (main.cc:25-31).
#include <cstdio>
#include <exception>

#include "difacto_b200/config.h"
#include "difacto_b200/sgd_learner.h"

int main(int argc, char* argv[]) {
  using namespace difacto;   // NOLINT
  if (argc < 2) {
    fprintf(stderr, "usage: difacto_b200 key1=val1 key2=val2 ...\n");
    fprintf(stderr, "  task=predict model_in=M data_in=D [pred_out=P] [num_gpus=N] [score_only=1 [V_storage=bf16]]:\n"
                    "  score a saved model (one file or the parts of a num_gpus run) on N GPUs (score_only=1: the parts only);\n"
                    "  score_only=1 loads it without its AdaGrad state (half the V-row memory, the same predictions),\n"
                    "  V_storage=bf16 also stores V in bf16 (a quarter; predictions differ by bf16 rounding of V)\n");
    return 0;
  }
  try {
    ArgParser parser;
    for (int i = 1; i < argc; ++i) parser.AddArg(argv[i]);
    KWArgs kwargs = parser.GetKWArgs();
    std::string task = "train", learner_type = "sgd";
    KWArgs remain;
    bool dry_run = false;
    for (const auto& kv : kwargs) {
      if (kv.first == "task") task = kv.second;
      else if (kv.first == "learner") learner_type = kv.second;
      else if (kv.first == "dry_run") dry_run = kv.second != "0";
      else remain.push_back(kv);
    }
    if (dry_run) {   // print the parsed configuration and stop (no GPU needed)
      printf("task = %s\nlearner = %s\n", task.c_str(), learner_type.c_str());
      for (const auto& kv : remain) printf("%s = %s\n", kv.first.c_str(), kv.second.c_str());
      SGDLearnerParam p;
      p.InitAllowUnknown(remain);
      return 0;
    }
    if (task == "train") {
      Learner* learner = Learner::Create(learner_type);
      KWArgs unknown = learner->Init(remain);
      if (!unknown.empty()) {
        fprintf(stderr, "Unrecognized keyword argument for task = %s\n", task.c_str());
        for (const auto& kv : unknown) fprintf(stderr, " - %s = %s\n", kv.first.c_str(), kv.second.c_str());
      }
      learner->Run();
      delete learner;
    } else if (task == "predict") {
      // a TODO in the reference (main.cc:61-62): forward pass of a saved model over data_in
      if (learner_type != "sgd") throw Error("task=predict is implemented for learner=sgd");
      SGDLearner learner;
      KWArgs unknown = learner.Init(remain);
      for (const auto& kv : unknown) fprintf(stderr, " - unrecognized %s = %s\n", kv.first.c_str(), kv.second.c_str());
      learner.Predict();
    } else if (task == "convert") {
      throw Error("task=convert (data format conversion) is host I/O outside the accelerated path");
    } else {
      throw Error("unknown task: " + task);
    }
  } catch (const std::exception& e) {
    fprintf(stderr, "difacto_b200: %s\n", e.what());
    return 1;
  }
  return 0;
}
