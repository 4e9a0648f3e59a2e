// difacto_b200/csrc/prune.cu -- dfb_prune: drop the table entries that carry no weight (DESIGN.md section 10).
//
// Between steps: every stream of the handle is drained first.  The kept entries are counted, a workspace of exactly
// that many entries is taken from the engine's stream-ordered pool -- before anything of the table changes -- and the
// table is rebuilt in place (kernels_prune.cu).  Capacity, V rows, the InitV state and every kept entry's 32 bytes are
// unchanged; n_keys drops by the entries dropped.
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

}  // extern "C"
