// difacto_b200/csrc/prune.cu -- dfb_prune: drop the table entries that carry no weight (DESIGN.md section 10), and
// dfb_prune_rare: drop the rarely seen entries with their V rows (section 10.1).
//
// Between steps: every stream of the handle is drained first.  The kept entries are counted, a workspace of exactly
// that many entries is taken from the engine's stream-ordered pool -- before anything of the table changes -- and the
// table is rebuilt in place (kernels_prune.cu).  Capacity, V rows, the InitV state and every kept entry's 32 bytes are
// unchanged; n_keys drops by the entries dropped.  dfb_prune_rare also takes the pool compaction's workspaces first,
// and then moves the kept V rows above the new n_vrows into the dropped rows' places below it.
#include <cuda_runtime.h>

#include <string>

#include "engine_internal.cuh"

using namespace dfb;  // NOLINT

namespace {

// device memory from the engine's pool on h->stream, freed in stream order when the call returns
struct PoolBuf {
  dfb_engine* h;
  void* p = nullptr;
  explicit PoolBuf(dfb_engine* h_) : h(h_) {}
  ~PoolBuf() {
    if (p) cudaFreeAsync(p, h->stream);
  }
  bool alloc(size_t bytes) {
    if (cudaMallocFromPoolAsync(&p, bytes, h->grow.pool, h->stream) == cudaSuccess) return true;
    cudaGetLastError();
    p = nullptr;
    return false;
  }
};

int prune(dfb_engine* h, float max_count, uint64_t* n_dropped) {
  TableState st;
  DFB_CUDA(h, cudaMemcpyAsync(&st, h->tab.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  const int grid = prune_grid(h->tab.cap);
  PoolBuf small(h);                      // {kept, dropped}, then the kept entries of every block
  if (!small.alloc(2 * sizeof(unsigned long long) + (size_t)grid * sizeof(unsigned)))
    return h->fail(DFB_ERR_CAPACITY, "dfb_prune: no device memory for its counters");
  unsigned long long* tot = static_cast<unsigned long long*>(small.p);
  unsigned* blk_kept = reinterpret_cast<unsigned*>(tot + 2);
  DFB_CUDA(h, cudaMemsetAsync(small.p, 0, 2 * sizeof(unsigned long long) + (size_t)grid * sizeof(unsigned), h->stream));
  h->launches += launch_prune_count(h->tab, max_count, grid, tot, blk_kept, h->stream);
  unsigned long long cnt[2];
  DFB_CUDA(h, cudaMemcpyAsync(cnt, tot, sizeof(cnt), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  const uint64_t n_kept = cnt[0], dropped = cnt[1];
  if (n_kept + dropped != st.n_keys)
    return h->fail(DFB_ERR_INVALID, "dfb_prune: the table holds " + std::to_string(n_kept + dropped) +
                                        " entries but counts " + std::to_string(st.n_keys));
  if (dropped == 0) return DFB_OK;
  PoolBuf kept(h);
  if (n_kept && !kept.alloc(n_kept * sizeof(Entry)))
    return h->fail(DFB_ERR_CAPACITY, "dfb_prune: no device memory for the " + std::to_string(n_kept) +
                                         " kept entries (" + std::to_string(n_kept * sizeof(Entry)) + " bytes)");
  h->launches += launch_prune_rebuild(h->tab, max_count, grid, tot, blk_kept, static_cast<Entry*>(kept.p), n_kept,
                                      h->stream);
  DFB_CUDA(h, cudaGetLastError());
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (h->grow.on) dfbh::counts_known(h, n_kept, st.n_vrows);
  *n_dropped = dropped;
  return DFB_OK;
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

int prune_rare(dfb_engine* h, float max_count, uint64_t* n_dropped, uint64_t* n_vrows_freed) {
  TableState st;
  DFB_CUDA(h, cudaMemcpyAsync(&st, h->tab.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  const int grid = prune_grid(h->tab.cap);
  // {kept, dropped, kept V rows, dropped V rows}, the broken-pool flag, then the kept entries of every block
  const size_t small_bytes = 4 * sizeof(unsigned long long) + sizeof(unsigned) + (size_t)grid * sizeof(unsigned);
  PoolBuf small(h);
  if (!small.alloc(small_bytes)) return h->fail(DFB_ERR_CAPACITY, "dfb_prune_rare: no device memory for its counters");
  unsigned long long* tot = static_cast<unsigned long long*>(small.p);
  unsigned* bad = reinterpret_cast<unsigned*>(tot + 4);
  unsigned* blk_kept = bad + 1;
  DFB_CUDA(h, cudaMemsetAsync(small.p, 0, small_bytes, h->stream));
  h->launches += launch_prune_count(h->tab, max_count, grid, tot, blk_kept, h->stream, true);
  unsigned long long cnt[4];
  DFB_CUDA(h, cudaMemcpyAsync(cnt, tot, sizeof(cnt), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  const uint64_t n_kept = cnt[0], dropped = cnt[1], kept_v = cnt[2], dropped_v = cnt[3];
  if (n_kept + dropped != st.n_keys)
    return h->fail(DFB_ERR_INVALID, "dfb_prune_rare: the table holds " + std::to_string(n_kept + dropped) +
                                        " entries but counts " + std::to_string(st.n_keys));
  if (kept_v + dropped_v != st.n_vrows)
    return h->fail(DFB_ERR_INVALID, "dfb_prune_rare: the table's entries own " + std::to_string(kept_v + dropped_v) +
                                        " V rows but it counts " + std::to_string(st.n_vrows));
  if (dropped == 0) return DFB_OK;
  const uint64_t n_vkeep = st.n_vrows - dropped_v;
  // every workspace before anything of the table or the pool changes
  PoolBuf kept(h);
  if (n_kept && !kept.alloc(n_kept * sizeof(Entry)))
    return h->fail(DFB_ERR_CAPACITY, "dfb_prune_rare: no device memory for the " + std::to_string(n_kept) +
                                         " kept entries (" + std::to_string(n_kept * sizeof(Entry)) + " bytes)");
  RareWs ws = {};
  PoolBuf pool_ws(h);
  if (dropped_v) {
    const size_t W = (st.n_vrows + 31) / 32;
    ws.n_list = 2 * dropped_v;
    ws.tmp_bytes = rare_scan_tmp_bytes(W);
    const size_t o_owner = align256(W * sizeof(unsigned)), o_cnt = o_owner + align256(dropped_v * sizeof(int));
    const size_t o_at = o_cnt + align256(2 * W * sizeof(unsigned)), o_list = o_at + align256(2 * W * sizeof(unsigned));
    const size_t o_tmp = o_list + align256(ws.n_list * sizeof(int)), bytes = o_tmp + ws.tmp_bytes;
    if (!pool_ws.alloc(bytes))
      return h->fail(DFB_ERR_CAPACITY, "dfb_prune_rare: no device memory for the V-row pool's compaction (" +
                                           std::to_string(bytes) + " bytes)");
    char* b = static_cast<char*>(pool_ws.p);
    ws.bits = reinterpret_cast<unsigned*>(b);
    ws.owner = reinterpret_cast<int*>(b + o_owner);
    ws.cnt = reinterpret_cast<unsigned*>(b + o_cnt);
    ws.at = reinterpret_cast<unsigned*>(b + o_at);
    ws.list = reinterpret_cast<int*>(b + o_list);
    ws.tmp = b + o_tmp;
    DFB_CUDA(h, cudaMemsetAsync(ws.bits, 0, W * sizeof(unsigned), h->stream));
  }
  ws.bad = bad;
  h->launches += launch_prune_rare(h->tab, max_count, grid, tot, blk_kept, static_cast<Entry*>(kept.p), n_kept,
                                   st.n_vrows, n_vkeep, ws, h->stream);
  DFB_CUDA(h, cudaGetLastError());
  unsigned broken = 0;
  DFB_CUDA(h, cudaMemcpyAsync(&broken, bad, sizeof(broken), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (h->grow.on) dfbh::counts_known(h, n_kept, broken ? st.n_vrows : n_vkeep);
  *n_dropped = dropped;
  if (broken)
    return h->fail(DFB_ERR_INVALID, "dfb_prune_rare: a V row is owned by two entries, or lies outside [0, n_vrows): "
                                    "the entries were pruned, the V rows left where they were");
  *n_vrows_freed = dropped_v;
  return DFB_OK;
}

}  // namespace

extern "C" {

int dfb_prune(dfb_handle h, float max_count, uint64_t* n_dropped) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_prune");
  if (!n_dropped) return h->fail(DFB_ERR_INVALID, "n_dropped is NULL");
  *n_dropped = 0;
  if (max_count != max_count) return h->fail(DFB_ERR_INVALID, "dfb_prune: max_count is NaN");
  if (dfbh::shard_step_open(h))
    return h->fail(DFB_ERR_INVALID, "dfb_prune during a sharded step (call it after dfb_shard_phase(4))");
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(dfbh::drain(h));
  const int rc = prune(h, max_count, n_dropped);
  cudaStreamSynchronize(h->stream);      // the workspaces are back in the pool
  return rc;
}

int dfb_prune_rare(dfb_handle h, float max_count, uint64_t* n_dropped, uint64_t* n_vrows_freed) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_prune_rare");
  if (!n_dropped || !n_vrows_freed) return h->fail(DFB_ERR_INVALID, "n_dropped or n_vrows_freed is NULL");
  *n_dropped = 0;
  *n_vrows_freed = 0;
  if (max_count != max_count) return h->fail(DFB_ERR_INVALID, "dfb_prune_rare: max_count is NaN");
  if (dfbh::shard_step_open(h))
    return h->fail(DFB_ERR_INVALID, "dfb_prune_rare during a sharded step (call it after dfb_shard_phase(4))");
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(dfbh::drain(h));
  const int rc = prune_rare(h, max_count, n_dropped, n_vrows_freed);
  cudaStreamSynchronize(h->stream);      // the workspaces are back in the pool
  return rc;
}

}  // extern "C"
