// difacto_b200/csrc/kernels_shard.cu -- device side of the NVLink-sharded model store.
//
// The reference shards the model over ps-lite servers by contiguous ranges of the reversed key
// (ps-lite/src/postoffice.cc:127-136) and a worker's sorted key list is sliced per server
// (ps-lite/include/ps/kv_app.h:406-460); Pull ships the k-wide rows of the minibatch's keys to the worker
// and Push ships as many gradient rows back.  At V_dim = 64 that is 2 x 1.7 GB per GPU per step over NVLink,
// more than the step's HBM time.  Here the rows never leave their owner: the FM interaction is linear in
// the rows up to one square,
//     XV_i = sum_s XV_i^(s),  XV_i^(s) = sum_{j owned by s} x_ij V_j      (fm_loss.h:81-83, spmm.h:94-122)
// so every owner computes the partial sums of EVERY worker's rows over its own keys and ships (k+2) floats
// per row instead of k floats per key; the worker adds the S partials, finishes pred / loss / p
// (fm_loss.h:108-118,155-161) and sends p_i * XV_i back (k floats per row); the owner then reduces the
// per-key gradient from the worker's column lists and applies FTRL/AdaGrad in place
// (sgd_updater.cc:74-147), one Update per worker in rank order like the reference's server.
// Per GPU and step ~0.3 GB crosses NVLink instead of ~6 GB, and the path is HBM-bound again.
//
// All cross-GPU traffic is plain stores into peer memory (CUDA IPC / peer access) issued by the producing
// kernels; completion is signalled by monotonically increasing step counters in the consumer's mailbox
// (st.release.sys after a system fence / ld.acquire.sys polling with a timeout) -- no NCCL call, no host
// synchronisation inside a step.
#include "dfb_device.cuh"
#include "shard_layout.cuh"

namespace dfb {

namespace {

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// poll up to 8 step counters in this GPU's own mailbox until each reaches `target`
__global__ void k_shard_wait(const unsigned long long* flags, int stride_u64, unsigned mask, unsigned long long target,
                             long long timeout_cycles, DevProgress* prog) {
  const int lane = threadIdx.x;
  if (lane >= 8 || !((mask >> lane) & 1u)) return;
  const unsigned long long* f = flags + (size_t)lane * stride_u64;
  const long long t0 = clock64();
  unsigned ns = 32;
  while (ld_acquire_sys(f) < target) {
    if (clock64() - t0 > timeout_cycles) { raise_err(prog, DFB_ERR_TIMEOUT); return; }
    __nanosleep(ns);
    if (ns < 1024) ns <<= 1;
  }
}

// publish a step counter to up to 8 mailboxes (peer memory).  Everything the previous kernels of this stream
// stored is ordered before it (kernel boundary + system fence).
__global__ void k_shard_signal(SignalDst d, unsigned long long value) {
  const int lane = threadIdx.x;
  if (lane >= d.n || d.flag[lane] == nullptr) return;
  __threadfence_system();
  st_release_sys(d.flag[lane], value);
}

// ------------------------------------------------------------------------------------------------------
// worker side
// ------------------------------------------------------------------------------------------------------
// segment boundaries of the sorted key list (DefaultSlicer, kv_app.h:416-429) and of the CSC view
__global__ void k_shard_bounds(const uint64_t* __restrict__ keys, const unsigned long long* __restrict__ dU,
                               size_t U_cap, const int* __restrict__ col_start, size_t nnz, int S, size_t Kseg,
                               size_t Nseg, ShardBounds* wb, DevProgress* prog) {
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  const size_t U = dev_count(U_cap, dU);
  const uint64_t width = ~0ULL / (uint64_t)S;     // postoffice.cc:130-134
  // lane s finds the first key of owner s: S - 1 independent binary searches side by side
  const int lane = threadIdx.x;
  size_t lo = 0, hi = (lane >= 1 && lane < S) ? U : 0;
  const uint64_t lo_key = width * (uint64_t)lane;
  while (__any_sync(kFullMask, lo < hi)) {
    if (lo < hi) {
      const size_t mid = lo + (hi - lo) / 2;
      if (keys[mid] < lo_key) lo = mid + 1; else hi = mid;
    }
  }
  ShardBounds b;
  for (int s = 0; s < S; ++s) b.kb[s] = (int)__shfl_sync(kFullMask, (unsigned long long)lo, s);
  if (lane != 0) return;
  b.kb[0] = 0;
  b.kb[S] = (int)U;
  for (int s = 0; s <= S; ++s) b.nb[s] = (U == 0) ? 0 : ((size_t)b.kb[s] < U ? col_start[b.kb[s]] : (int)nnz);
  // no keys for non-zeros: the localizer dropped the batch (ids outside the sorted range) and reported it.  A batch
  // without non-zeros is not dropped: its rows still count, with the bias-free prediction 0.
  b.valid = (U > 0 || nnz == 0) ? 1 : 0;
  for (int s = 0; s < S; ++s)
    if ((size_t)(b.kb[s + 1] - b.kb[s]) > Kseg || (size_t)(b.nb[s + 1] - b.nb[s]) > Nseg) {
      // a key segment larger than the mailbox slot (skewed key distribution): drop the batch, report
      raise_err(prog, DFB_ERR_CAPACITY);
      b.valid = 0;
    }
  if (!b.valid) for (int s = 0; s <= S; ++s) { b.kb[s] = 0; b.nb[s] = 0; }
  for (int s = S + 1; s < 9; ++s) { b.kb[s] = b.kb[S]; b.nb[s] = b.nb[S]; }
  *wb = b;
}

// keys, column offsets and column payload of every owner's segment -> that owner's mailbox.
// On the wire every minibatch is VALUED ((row << 32) | bits(x) per occurrence, x = 1 for a binary batch): an owner
// consumes the slices of all workers with one kernel flavour, whatever mix of binary and valued batches (or empty
// ones) the workers happen to hold in a step.
template <bool HAS_VAL>
__global__ void __launch_bounds__(256) k_shard_scatter(ScatterArgs a) {
  __shared__ ShardBounds b;
  if (threadIdx.x == 0) b = *a.wb;
  __syncthreads();
  const int S = a.S;
  const unsigned U = (unsigned)b.kb[S], N = (unsigned)b.nb[S];
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  // start at this rank's own segment and go round, so that the ranks write into different owners at a time
  const unsigned rot_k = (unsigned)b.kb[a.me], rot_n = (unsigned)b.nb[a.me];
  for (unsigned i0 = tid; i0 < U; i0 += nth) {
    unsigned i = i0 + rot_k;
    if (i >= U) i -= U;
    int s = 0;
    while ((int)i >= b.kb[s + 1]) ++s;
    const unsigned r = i - (unsigned)b.kb[s];
    a.keys_dst[s][r] = a.keys[i];
    a.cstart_dst[s][r] = a.col_start[i] - b.nb[s];
  }
  for (unsigned j0 = tid; j0 < N; j0 += nth) {
    unsigned j = j0 + rot_n;
    if (j >= N) j -= N;
    int s = 0;
    while ((int)j >= b.nb[s + 1]) ++s;
    const unsigned r = j - (unsigned)b.nb[s];
    reinterpret_cast<unsigned long long*>(a.occ_dst[s])[r] =
        HAS_VAL ? reinterpret_cast<const unsigned long long*>(a.occ)[j]
                : (((unsigned long long)reinterpret_cast<const uint32_t*>(a.occ)[j] << 32) | 0x3f800000ULL);
  }
  if (blockIdx.x == 0 && threadIdx.x < (unsigned)S) {
    const int s = threadIdx.x;
    const unsigned nk = (unsigned)(b.kb[s + 1] - b.kb[s]), nn = (unsigned)(b.nb[s + 1] - b.nb[s]);
    a.cstart_dst[s][nk] = (int)nn;      // nk + 1 column offsets
    ShardHdr h;
    h.nkeys = nk; h.nnz = nn; h.nrows = b.valid ? a.nrows : 0; h.flags = a.flags; h.step = a.step;
    h.pad[0] = h.pad[1] = h.pad[2] = 0;
    *a.hdr_dst[s] = h;
  }
}

__device__ __forceinline__ int owner_of(const ShardBounds& b, int S, uint32_t lidx) {
  int s = 0;
  while (s + 1 < S && (int)lidx >= b.kb[s + 1]) ++s;
  return s;
}

// the rows of the worker's CSR, split by owner of the column: per (owner, row) counts ...
// (one __match_any per 32-nnz chunk groups the lanes by owner; the lowest lane of a group adds the group's size)
__global__ void __launch_bounds__(256) k_shard_rowcount(const uint64_t* __restrict__ offset,
                                                        const uint32_t* __restrict__ lidx, size_t nrows,
                                                        const ShardBounds* __restrict__ wb, int S,
                                                        int* __restrict__ cnt /* [S][nrows+1] */) {
  __shared__ ShardBounds b;
  __shared__ int s_cnt[8][8];          // [warp][owner]
  if (threadIdx.x == 0) b = *wb;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t row = warp0; row < nrows; row += nwarps) {
    const uint64_t o0 = offset[row], o1 = offset[row + 1];
    if (lane < 8) s_cnt[wid][lane] = 0;
    __syncwarp();
    if (b.valid) {
      for (uint64_t cc = o0; cc < o1; cc += 32) {
        const uint64_t j = cc + lane;
        const int own = j < o1 ? owner_of(b, S, __ldg(lidx + j)) : 8 + (lane & 7);   // inactive lanes: groups that are ignored
        const unsigned peers = __match_any_sync(kFullMask, own);
        if (own < 8 && lane == __ffs(peers) - 1) s_cnt[wid][own] += __popc(peers);
        __syncwarp();
      }
    }
    if (lane < S) cnt[(size_t)lane * (nrows + 1) + row] = s_cnt[wid][lane];
    __syncwarp();
  }
}

// ... exclusive scan per owner (one CTA each) = the row pointers of the owner's sub-CSR, kept locally (int) and
// stored into the owner's mailbox (u64, the offset type of dmlc::RowBlock)
__global__ void __launch_bounds__(1024) k_shard_rowscan(int* __restrict__ cnt, size_t nrows, RowptrDst d) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int s = blockIdx.x;
  int* c = cnt + (size_t)s * (nrows + 1);
  uint64_t* dst = d.rowptr_dst[s];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (size_t b0 = 0; b0 < nrows; b0 += (size_t)blockDim.x * 8) {     // 8 consecutive rows per thread
    const size_t i0 = b0 + (size_t)threadIdx.x * 8;
    int v[8], sum = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) { v[q] = i0 + q < nrows ? c[i0 + q] : 0; sum += v[q]; }
    int x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(kFullMask, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int wv = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(kFullMask, wv, o);
        if (lane >= o) wv += y;
      }
      s_warp[lane] = wv;
    }
    __syncthreads();
    const int carry = s_carry;
    int run = carry + (wid ? s_warp[wid - 1] : 0) + (x - sum);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (i0 + q < nrows) { c[i0 + q] = run; dst[i0 + q] = (uint64_t)run; }
      run += v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + s_warp[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) { c[nrows] = s_carry; dst[nrows] = (uint64_t)s_carry; }
}

// ... and the column indices (relative to the owner's segment) [+ values], CSR order kept inside a row
template <bool HAS_VAL>
__global__ void __launch_bounds__(256) k_shard_fill(const uint64_t* __restrict__ offset,
                                                    const uint32_t* __restrict__ lidx,
                                                    const float* __restrict__ value, size_t nrows,
                                                    const ShardBounds* __restrict__ wb, int S,
                                                    const int* __restrict__ rowptr /* [S][nrows+1] */, FillDst d) {
  __shared__ ShardBounds b;
  __shared__ int s_pos[8][8];          // [warp][owner]: next free slot of the owner's sub-row
  if (threadIdx.x == 0) b = *wb;
  __syncthreads();
  if (!b.valid) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t row = warp0; row < nrows; row += nwarps) {
    const uint64_t o0 = offset[row], o1 = offset[row + 1];
    if (lane < S) s_pos[wid][lane] = rowptr[(size_t)lane * (nrows + 1) + row];
    __syncwarp();
    for (uint64_t cc = o0; cc < o1; cc += 32) {
      const uint64_t j = cc + lane;
      uint32_t u = 0;
      float x = 0.f;
      int own = 8 + (lane & 7);
      if (j < o1) {
        u = __ldg(lidx + j);
        if (HAS_VAL) x = __ldg(value + j);
        own = owner_of(b, S, u);
      }
      const unsigned peers = __match_any_sync(kFullMask, own);
      if (own < 8) {
        const int at = s_pos[wid][own] + __popc(peers & ((1u << lane) - 1u));
        d.ridx_dst[own][at] = u - (uint32_t)b.kb[own];
        d.rval_dst[own][at] = HAS_VAL ? x : 1.f;
      }
      __syncwarp();
      if (own < 8 && lane == __ffs(peers) - 1) s_pos[wid][own] += __popc(peers);
      __syncwarp();
    }
  }
}

// add the owners' partials, finish Predict / Evaluate / p (fm_loss.h:108-118,155-161; loss.h:57-66) and send
// p_i and p_i * XV_i to every owner.  LPR lanes (one float4 each) per row, G rows per warp.  PAD: rows of stride
// ks < K, the lanes beyond it idle, no clamp at V_dim 0 (fm_loss.h:77)
template <int K, bool PAD = false>
__global__ void __launch_bounds__(256) k_shard_reduce(ReduceArgs a) {
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  __shared__ float red_s[8];
  // a dropped batch: the owners sent no partials (their slots hold an older step's), so nothing is predicted, stored
  // or added to Progress
  if (!a.wb->valid) return;
  const int lane = threadIdx.x & 31, sub = lane % LPR, grp = lane / LPR;
  const int ks = PAD ? (a.V_dim + 3) / 4 * 4 : K;
  const bool act = !PAD || sub * 4 < ks;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const size_t ntiles = (a.nrows + G - 1) / G;
  float loss_acc = 0.f;
  for (size_t tl = warp0; tl < ntiles; tl += nwarps) {
    const size_t row = tl * G + grp;
    const bool ok = row < a.nrows;
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc2 = 0.f, wsum = 0.f;
    if (ok) {
      for (int s = 0; s < a.S; ++s) {      // fixed order: bit-reproducible
        if (act) {
          const float4 t = *reinterpret_cast<const float4*>(a.part_xv[s] + row * (size_t)ks + sub * 4);
          xv.x += t.x; xv.y += t.y; xv.z += t.z; xv.w += t.w;
        }
        if (sub == 0) { const float2 sc = a.part_sc[s][row]; acc2 += sc.x; wsum += sc.y; }
      }
    }
    float s1 = xv.x * xv.x + xv.y * xv.y + xv.z * xv.z + xv.w * xv.w;
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) s1 += __shfl_xor_sync(kFullMask, s1, o);
    acc2 = __shfl_sync(kFullMask, acc2, grp * LPR);
    wsum = __shfl_sync(kFullMask, wsum, grp * LPR);
    float pred = wsum + 0.5f * (s1 - acc2);
    if (!PAD || a.V_dim > 0) pred = pred > 20.f ? 20.f : (pred < -20.f ? -20.f : pred);   // fm_loss.h:77,118
    if (!ok) continue;
    // (no label: a predict step without labels -- the predictions are stored, the loss stays 0)
    const float label = a.label ? __ldg(a.label + row) : 0.f;
    const float y = label > 0.f ? 1.f : -1.f;
    if (sub == 0) {
      a.pred[row] = pred;
      if (a.label) loss_acc += logf(1.f + expf(-y * pred));
    }
    if (a.train) {
      const float p = -y / (1.f + expf(y * pred));
      const float4 g = make_float4(p * xv.x, p * xv.y, p * xv.z, p * xv.w);
      for (int q = 0; q < a.S; ++q) {
        int s = q + a.me;
        if (s >= a.S) s -= a.S;
        if (act) *reinterpret_cast<float4*>(a.pxv_dst[s] + row * (size_t)ks + sub * 4) = g;
        if (sub == 0) a.p_dst[s][row] = p;
      }
    }
  }
  loss_acc = warp_sum_f(loss_acc);
  if (lane == 0) red_s[threadIdx.x >> 5] = loss_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red_s[w];
    atomicAdd(&a.prog->loss, (double)v);
    if (blockIdx.x == 0) atomicAdd(&a.prog->nrows, (unsigned long long)a.nrows);
  }
}

// ------------------------------------------------------------------------------------------------------
// owner side
// ------------------------------------------------------------------------------------------------------
// model_[key] for the key segment ONE worker sent (SGDUpdater::Get, sgd_updater.cc:32-56): slots only (find or
// default-construct); the owner runs it once per worker, in rank order, on its lookup stream -- beside the previous
// step's update, which addresses entries by slot and is not disturbed by inserts.  With stamp != 0 every touched
// entry also records which workers hold it in this step (entry.pad = stamp << 8 | worker bitmask).  A key that a
// lower-rank worker also holds will already have been updated by that worker's push when this worker's push is
// applied, but the gradient a worker pushes is taken at the V it pulled (fm_loss.h:181-188): such keys are
// flagged (conf); k_shard_pull saves their pull-time V row.
template <bool INSERT>
__global__ void __launch_bounds__(256) k_shard_lookup(Table t, LookupArgs a, int r, unsigned char* __restrict__ conf) {
  constexpr int ILP = 2;
  const size_t n = (size_t)a.hdr[r]->nkeys < a.Kseg ? (size_t)a.hdr[r]->nkeys : a.Kseg;
  const uint64_t* __restrict__ keys = a.keys[r];
  const size_t o = (size_t)r * a.Kseg;
  const size_t tile = (size_t)blockDim.x * ILP;
  for (size_t base = (size_t)blockIdx.x * tile; base < n; base += (size_t)gridDim.x * tile) {
    unsigned long long key[ILP];
    uint64_t h[ILP];
    Entry256 e[ILP];
#pragma unroll
    for (int q = 0; q < ILP; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      key[q] = i < n ? keys[i] : 0ULL;
      h[q] = hash64(key[q]) & t.mask;
    }
#pragma unroll
    for (int q = 0; q < ILP; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      if (i < n) e[q] = load_entry(&t.tab[h[q]]);
    }
#pragma unroll
    for (int q = 0; q < ILP; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      if (i >= n) continue;
      int slot = -1, old = 0;
      if (key[q] == kEmptyKey) {
        raise_err(t.prog, DFB_ERR_INVALID);
      } else if (e[q].key == key[q]) {
        slot = (int)h[q]; old = (int)(unsigned)(e[q].q1 >> 32);
      } else {
        slot = table_find<INSERT>(t, key[q], h[q]);
        if (slot >= 0) old = *reinterpret_cast<volatile int*>(&t.tab[slot].pad);
      }
      const size_t v = o + i;
      a.slot[v] = slot;
      if (a.stamp != 0) {
        // the keys of one worker are distinct and the workers' lookups are separate launches in rank order, so the
        // stamp word of an entry has one writer at a time: plain read (it came with the entry) - modify - write
        int c = 0;
        if (slot >= 0) {
          const bool cur = (((unsigned)old) >> 8) == a.stamp;
          t.tab[slot].pad = (cur ? old : (int)(a.stamp << 8)) | (1 << r);
          c = (cur && (old & ((1 << r) - 1) & 0xff) != 0) ? 1 : 0;
        }
        conf[v] = (unsigned char)c;
      }
    }
  }
}

// the keys this owner received in one step: the sum over the workers' segments (each as k_shard_lookup reads it),
// stored to host memory.  A growing owner bounds the step's new keys and new V rows by it (growth.cu, reserve_shard).
__global__ void k_shard_count(LookupArgs a, unsigned long long* out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  unsigned long long n = 0;
  for (int r = 0; r < a.S; ++r) {
    const unsigned long long k = a.hdr[r]->nkeys;
    n += k < a.Kseg ? k : a.Kseg;
  }
  *out = n;
}

// Pull (Store::Pull -> SGDUpdater::Get, sgd_updater.cc:41-62) of all workers' key segments at once: {w, V-row index} of
// every resolved slot -- taken AFTER the previous step's updates and this step's Update(kFeaCount), while the slots
// themselves were resolved earlier (k_shard_lookup runs beside the previous step's update: open addressing without
// deletes keeps slots stable).  For a key a lower-rank worker of this step holds too (conf), the pull-time V row is
// saved: that worker's push will have changed the table row by the time this worker's gradient needs it.
__global__ void __launch_bounds__(256) k_shard_pull(Table t, LookupArgs a, const unsigned char* __restrict__ conf,
                                                    float* __restrict__ vsave, int ks) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const size_t total = (size_t)a.S * a.Kseg;
  for (size_t base = warp0 * 32; base < total; base += nwarps * 32) {
    const size_t v = base + lane;
    int vr_save = -1;
    if (v < total) {
      const int r = (int)(v / a.Kseg);
      const size_t i = v - (size_t)r * a.Kseg;
      if (i < (size_t)a.hdr[r]->nkeys) {
        const int s = a.slot[v];
        float w = 0.f;
        int vr = -1;
        if (s >= 0) {
          const Entry256 e = load_entry(&t.tab[s]);
          w = e.w(); vr = e.vrow();
        }
        a.w[v] = w;
        a.vrow[v] = vr;
        a.wv[v] = make_int2(__float_as_int(w), vr);
        if (a.stamp != 0 && conf[v]) vr_save = vr;
      }
    }
    unsigned m = __ballot_sync(kFullMask, vr_save >= 0);
    while (m) {
      const int b = __ffs(m) - 1;
      m &= m - 1;
      const int vrb = __shfl_sync(kFullMask, vr_save, b);
      const float4* src = reinterpret_cast<const float4*>(t.V + (size_t)vrb * t.rs);
      float4* dst = reinterpret_cast<float4*>(vsave + (base + b) * (size_t)ks);
      for (int l = lane; l < ks / 4; l += 32) dst[l] = src[l];
    }
  }
}

// end of one worker's Update on this owner: hand the penalty of what that worker pulled back to it, forward
// a device-side error, publish "done"
__global__ void k_shard_done(DevProgress* src_prog, DevProgress* main_prog, double* pen_dst,
                             unsigned long long* flag_dst, unsigned long long value) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const double pen = src_prog->penalty;
  const int err = src_prog->err;
  src_prog->penalty = 0.0;
  src_prog->err = 0;
  if (err) raise_err(main_prog, err);
  *pen_dst = pen;
  __threadfence_system();
  st_release_sys(flag_dst, value);
}

// worker: fold the owners' penalties into this step's Progress, stage it for the D2H snapshot, reset
__global__ void k_shard_collect(const double* pen_in, int stride_f64, int S, DevProgress* prog_w,
                                DevProgress* main_prog, DevProgress* stage) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  DevProgress o = *prog_w;
  for (int s = 0; s < S; ++s) o.penalty += pen_in[(size_t)s * stride_f64];
  // the owner-side counters / sticky error of this engine travel with the snapshot (the owner stream may be
  // adding to them concurrently: exchange, do not read-then-clear)
  o.new_keys = atomicExch(&main_prog->new_keys, 0ULL);
  o.new_vrows = atomicExch(&main_prog->new_vrows, 0ULL);
  const int merr = atomicExch(&main_prog->err, 0);
  o.err = prog_w->err ? prog_w->err : merr;
  *stage = o;
  DevProgress z;
  z.loss = 0; z.penalty = 0; z.auc = 0; z.nrows = 0; z.new_keys = 0; z.new_vrows = 0; z.err = 0; z.pad = 0;
  *prog_w = z;
}

inline int grid_cap(size_t n, int per_block, int cap) {
  size_t g = (n + per_block - 1) / per_block;
  if (g == 0) g = 1;
  return (int)(g < (size_t)cap ? g : (size_t)cap);
}

}  // namespace

int launch_shard_wait(const unsigned long long* flags, int stride_u64, unsigned mask, unsigned long long target,
                      long long timeout_cycles, DevProgress* prog, cudaStream_t s) {
  if (mask == 0) return 0;
  k_shard_wait<<<1, 32, 0, s>>>(flags, stride_u64, mask, target, timeout_cycles, prog);
  return 1;
}

int launch_shard_signal(const SignalDst& d, unsigned long long value, cudaStream_t s) {
  if (d.n == 0) return 0;
  k_shard_signal<<<1, 32, 0, s>>>(d, value);
  return 1;
}

int launch_shard_bounds(const uint64_t* keys, const unsigned long long* dU, size_t U_cap, const int* col_start,
                        size_t nnz, int S, size_t Kseg, size_t Nseg, ShardBounds* wb, DevProgress* prog,
                        cudaStream_t s) {
  k_shard_bounds<<<1, 32, 0, s>>>(keys, dU, U_cap, col_start, nnz, S, Kseg, Nseg, wb, prog);
  return 1;
}

int launch_shard_scatter(const ScatterArgs& a, bool valued, size_t work_cap, cudaStream_t s) {
  const int grid = grid_cap(work_cap, 256, num_sms() * 8);
  if (valued) k_shard_scatter<true><<<grid, 256, 0, s>>>(a);
  else        k_shard_scatter<false><<<grid, 256, 0, s>>>(a);
  return 1;
}

int launch_shard_subcsr(const uint64_t* offset, const uint32_t* lidx, const float* value, size_t nrows,
                        const ShardBounds* wb, int S, int* rowcnt, const RowptrDst& rd, const FillDst& fd,
                        cudaStream_t s) {
  const int grid = grid_cap(nrows ? nrows : 1, 8, num_sms() * 8);
  k_shard_rowcount<<<grid, 256, 0, s>>>(offset, lidx, nrows, wb, S, rowcnt);
  k_shard_rowscan<<<S, 1024, 0, s>>>(rowcnt, nrows, rd);
  if (value) k_shard_fill<true><<<grid, 256, 0, s>>>(offset, lidx, value, nrows, wb, S, rowcnt, fd);
  else       k_shard_fill<false><<<grid, 256, 0, s>>>(offset, lidx, value, nrows, wb, S, rowcnt, fd);
  return 3;
}

int launch_shard_reduce(const ReduceArgs& a, cudaStream_t s) {
  if (a.nrows == 0) return 0;
  return with_lane_width(a.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    const size_t tiles = (a.nrows + (32 / (K / 4)) - 1) / (32 / (K / 4));
    if (a.V_dim == K) k_shard_reduce<K><<<grid_cap(tiles, 8, num_sms() * 8), 256, 0, s>>>(a);
    else              k_shard_reduce<K, true><<<grid_cap(tiles, 8, num_sms() * 8), 256, 0, s>>>(a);
    return 1;
  });
}

int launch_shard_lookup(Table& t, const LookupArgs& a, int r, bool insert, unsigned char* conf, cudaStream_t s) {
  const int grid = grid_cap(a.Kseg, 256 * 2, num_sms() * 64);
  if (insert) k_shard_lookup<true><<<grid, 256, 0, s>>>(t, a, r, conf);
  else        k_shard_lookup<false><<<grid, 256, 0, s>>>(t, a, r, conf);
  return 1;
}

int launch_shard_count(const LookupArgs& a, unsigned long long* out, cudaStream_t s) {
  k_shard_count<<<1, 32, 0, s>>>(a, out);
  return 1;
}

int launch_shard_pull(Table& t, const LookupArgs& a, const unsigned char* conf, float* vsave, cudaStream_t s) {
  const size_t total = (size_t)a.S * a.Kseg;
  k_shard_pull<<<grid_cap((total + 31) / 32, 8, num_sms() * 16), 256, 0, s>>>(t, a, conf, vsave, t.ks);
  return 1;
}

int launch_shard_done(DevProgress* src_prog, DevProgress* main_prog, double* pen_dst, unsigned long long* flag_dst,
                      unsigned long long value, cudaStream_t s) {
  k_shard_done<<<1, 32, 0, s>>>(src_prog, main_prog, pen_dst, flag_dst, value);
  return 1;
}

int launch_shard_collect(const double* pen_in, int stride_f64, int S, DevProgress* prog_w, DevProgress* main_prog,
                         DevProgress* stage, cudaStream_t s) {
  k_shard_collect<<<1, 32, 0, s>>>(pen_in, stride_f64, S, prog_w, main_prog, stage);
  return 1;
}

}  // namespace dfb
