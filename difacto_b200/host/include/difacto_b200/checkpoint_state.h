// difacto_b200/host/include/difacto_b200/checkpoint_state.h -- what a mid-epoch checkpoint stores beside the model
// (checkpoint_out / checkpoint_in of SGDLearner), and the process-wide rand() state the reference-order reader draws
// its shuffle from.  Host only.
#pragma once
#include <stdlib.h>

#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "api.h"

namespace difacto {

/** glibc's rand() state: the 128-byte TYPE_3 table rand() draws from (the default, as after srand), its read
 * position encoded in its first word.  Saving switches to a scratch table for a moment, which makes glibc encode the
 * position into the table in use, and switches back; restoring overwrites the table in use the same way. */
struct RandState {
  static constexpr size_t kBytes = 128;
  unsigned char bytes[kBytes] = {};

  static RandState Save() {
    RandState s;
    char* cur = Swap();
    memcpy(s.bytes, cur, kBytes);
    setstate(cur);
    return s;
  }
  void Restore() const {
    char* cur = Swap();
    memcpy(cur, bytes, kBytes);
    setstate(cur);
  }

 private:
  // makes a scratch table current and returns the one that was, with its position written into its first word
  static char* Swap() {
    alignas(8) static char scratch[kBytes];
    char* cur = initstate(1, scratch, kBytes);
    int32_t w0;
    memcpy(&w0, cur, 4);
    if (w0 % 5 != 3) {       // MAX_TYPES = 5; TYPE_3 is rand()'s default table (128 bytes)
      setstate(cur);
      throw Error("rand() does not run on its default 128-byte table: its state cannot be checkpointed");
    }
    return cur;
  }
};

/** the record P.<c>.state of checkpoint c: everything an exact resume needs beyond the model */
struct CheckpointState {
  static constexpr uint32_t kVersion = 1;
  struct Worker {
    int32_t part = 0;          // the file part the worker reads (>= num_parts: its parts are exhausted)
    uint64_t consumed = 0;     // minibatches it has read from that part
  };
  std::vector<std::pair<std::string, std::string>> settings;   // the settings that fix the batches and the model
  int32_t epoch = 0;
  std::vector<Worker> workers;
  bool has_rand = false;       // num_gpus = 1: rand() at the start of the worker's part
  RandState rand;
  float epoch_prog[5] = {};    // Progress {loss, penalty, auc, nnz_w, nrows} of the epoch's finished parts / rounds
  float part_prog[5] = {};     // num_gpus = 1: the Progress of the current part so far
  float pre_loss = 0, pre_val_auc = 0;
  uint64_t minibatches = 0;    // training minibatches per worker since the run began
  std::vector<int32_t> id_ranges;   // per engine: dfb_id_range_get

  std::string Serialize() const {
    std::string o("DFBCKST\0", 8);
    Put(&o, kVersion);
    Put(&o, static_cast<uint32_t>(settings.size()));
    for (const auto& kv : settings) { PutStr(&o, kv.first); PutStr(&o, kv.second); }
    Put(&o, epoch);
    Put(&o, static_cast<uint32_t>(workers.size()));
    for (const auto& w : workers) { Put(&o, w.part); Put(&o, w.consumed); }
    Put(&o, static_cast<uint32_t>(has_rand ? 1 : 0));
    o.append(reinterpret_cast<const char*>(rand.bytes), RandState::kBytes);
    for (float f : epoch_prog) Put(&o, f);
    for (float f : part_prog) Put(&o, f);
    Put(&o, pre_loss); Put(&o, pre_val_auc);
    Put(&o, minibatches);
    Put(&o, static_cast<uint32_t>(id_ranges.size()));
    for (int32_t b : id_ranges) Put(&o, b);
    return o;
  }
  static CheckpointState Parse(const std::string& s) {
    CheckpointState st;
    size_t p = 0;
    if (s.size() < 8 || s.compare(0, 8, std::string("DFBCKST\0", 8)) != 0) throw Error("not a checkpoint state record");
    p = 8;
    if (Get<uint32_t>(s, &p) != kVersion) throw Error("unknown checkpoint state version");
    const uint32_t ns = Get<uint32_t>(s, &p);
    for (uint32_t i = 0; i < ns; ++i) {
      std::string k = GetStr(s, &p);
      st.settings.emplace_back(k, GetStr(s, &p));
    }
    st.epoch = Get<int32_t>(s, &p);
    const uint32_t nw = Get<uint32_t>(s, &p);
    if (nw > 64) throw Error("checkpoint state corrupt (workers)");
    st.workers.resize(nw);
    for (auto& w : st.workers) { w.part = Get<int32_t>(s, &p); w.consumed = Get<uint64_t>(s, &p); }
    st.has_rand = Get<uint32_t>(s, &p) != 0;
    if (p + RandState::kBytes > s.size()) throw Error("checkpoint state truncated");
    memcpy(st.rand.bytes, s.data() + p, RandState::kBytes);
    p += RandState::kBytes;
    for (float& f : st.epoch_prog) f = Get<float>(s, &p);
    for (float& f : st.part_prog) f = Get<float>(s, &p);
    st.pre_loss = Get<float>(s, &p);
    st.pre_val_auc = Get<float>(s, &p);
    st.minibatches = Get<uint64_t>(s, &p);
    const uint32_t ne = Get<uint32_t>(s, &p);
    if (ne > 64) throw Error("checkpoint state corrupt (engines)");
    for (uint32_t i = 0; i < ne; ++i) st.id_ranges.push_back(Get<int32_t>(s, &p));
    if (p != s.size()) throw Error("checkpoint state corrupt (trailing bytes)");
    return st;
  }
  /** throws naming the first setting that differs from `now`.  `later`: settings the record format gained after
   * checkpoints were first written, with the value a record that lacks one stands for (the setting's default).  A
   * setting of `later` may also be left out of `now` (it is recorded only away from its default): a checkpoint that
   * records it at another value is refused by its name too */
  void CheckSettings(const std::vector<std::pair<std::string, std::string>>& now,
                     const std::vector<std::pair<std::string, std::string>>& later = {}) const {
    for (const auto& kv : now) {
      const std::string* saved = nullptr;
      for (const auto& s : settings) if (s.first == kv.first) saved = &s.second;
      if (!saved) for (const auto& s : later) if (s.first == kv.first) saved = &s.second;
      if (!saved) throw Error("checkpoint_in: the checkpoint does not record " + kv.first);
      if (*saved != kv.second)
        throw Error("checkpoint_in: " + kv.first + " differs from the checkpoint's (" + kv.first + " = " + *saved +
                    " there, " + kv.second + " here)");
    }
    for (const auto& d : later) {
      bool given = false;
      for (const auto& kv : now) given = given || kv.first == d.first;
      if (given) continue;
      for (const auto& s : settings)
        if (s.first == d.first && s.second != d.second)
          throw Error("checkpoint_in: " + d.first + " differs from the checkpoint's (" + d.first + " = " + s.second +
                      " there, " + d.second + " here)");
    }
  }

 private:
  template <typename T> static void Put(std::string* o, T v) { o->append(reinterpret_cast<const char*>(&v), sizeof(T)); }
  static void PutStr(std::string* o, const std::string& v) {
    Put(o, static_cast<uint32_t>(v.size()));
    o->append(v);
  }
  template <typename T> static T Get(const std::string& s, size_t* p) {
    if (*p + sizeof(T) > s.size()) throw Error("checkpoint state truncated");
    T v;
    memcpy(&v, s.data() + *p, sizeof(T));
    *p += sizeof(T);
    return v;
  }
  static std::string GetStr(const std::string& s, size_t* p) {
    const uint32_t n = Get<uint32_t>(s, p);
    if (*p + n > s.size()) throw Error("checkpoint state truncated");
    std::string v = s.substr(*p, n);
    *p += n;
    return v;
  }
};

}  // namespace difacto
