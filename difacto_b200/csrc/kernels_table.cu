// difacto_b200/csrc/kernels_table.cu -- the HBM-resident model table and its per-key kernels.
//
// GPU restatement of SGDUpdater (src/sgd/sgd_updater.{h,cc} of the reference):
//   model_[key]            -> open-addressing hash of 32-byte entries (k_lookup)
//   Get        cc:32-56    -> k_lookup(+pull) / k_pack_ragged / k_gather_rows
//   Update(kFeaCount) :62-73 -> k_feacnt (+ InitV pass)
//   Update(kGradient) :74-98 -> k_update_dense / k_update_ragged
//   UpdateW (FTRL)   :104-127, UpdateV (AdaGrad) :129-138 -> ftrl_step / adagrad_step, written
//                       with explicit round-to-nearest intrinsics (no FMA contraction) so that,
//                       given identical gradients, the state is bit-identical to the reference
//   InitV            :140-147 -> k_initv: glibc rand_r restated with LCG jump-ahead so that new
//                       rows consume the random stream in ascending key order like the reference
// plus Loss::Evaluate (loss.h:57-66), BinClassMetric::AUC (bin_class_metric.h:35-56) and
// SGDLearner::EvaluatePenalty (sgd_learner.cc:249-273).
#include "dfb_device.cuh"

#include <cub/cub.cuh>

#include <atomic>

namespace dfb {

namespace {

constexpr unsigned kFull = kFullMask;

__device__ __forceinline__ float warp_sum(float v) { return warp_sum_f(v); }

__device__ __forceinline__ void raise(DevProgress* prog, int code) { raise_err(prog, code); }

__global__ void k_table_init(Entry* tab, uint64_t cap, TableState* st, DevProgress* prog, unsigned seed) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = i0; i < cap; i += stride) {
    Entry e;
    e.key = kEmptyKey; e.vrow = -1; e.pad = 0;
    e.fea_cnt = 0.f; e.w = 0.f; e.sqrt_g = 0.f; e.z = 0.f;
    tab[i] = e;
  }
  if (i0 == 0) {
    st->n_keys = 0; st->n_vrows = 0; st->seed = seed; st->pad = 0;
    prog->loss = 0; prog->penalty = 0; prog->auc = 0;
    prog->nrows = 0; prog->new_keys = 0; prog->new_vrows = 0; prog->err = 0; prog->pad = 0;
  }
}

// model_[key] (sgd_updater.cc:43-45,65-67,86-88): find or default-construct, and the Pull of the
// fused path (w and the V-row index of every key).  Random 32-byte sectors: the kernel is latency
// bound, so every thread keeps kLookupIlp = 2 independent first probes in flight (both halves of the
// entry are fetched with the probe; a hit needs no second round trip) and only collisions fall back to
// the serial probe loop.
constexpr int kLookupIlp = 2;
template <bool INSERT>
__global__ void __launch_bounds__(256) k_lookup(Table t, const uint64_t* __restrict__ keys, size_t n_cap,
                                                const unsigned long long* __restrict__ dn,
                                                int* __restrict__ slot_out, float* __restrict__ w_out,
                                                int* __restrict__ vrow_out, int2* __restrict__ wv_out) {
  const size_t n = dev_count(n_cap, dn);
  const size_t tile = (size_t)blockDim.x * kLookupIlp;
  for (size_t base = (size_t)blockIdx.x * tile; base < n; base += (size_t)gridDim.x * tile) {
    unsigned long long key[kLookupIlp];
    uint64_t h[kLookupIlp];
    Entry256 e[kLookupIlp];
#pragma unroll
    for (int q = 0; q < kLookupIlp; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      key[q] = i < n ? keys[i] : 0ULL;
      h[q] = hash64(key[q]) & t.mask;
    }
#pragma unroll
    for (int q = 0; q < kLookupIlp; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      if (i < n) e[q] = load_entry(&t.tab[h[q]]);
    }
#pragma unroll
    for (int q = 0; q < kLookupIlp; ++q) {
      const size_t i = base + (size_t)q * blockDim.x + threadIdx.x;
      if (i >= n) continue;
      int slot = -1, vr = -1;
      float w = 0.f;
      if (key[q] == kEmptyKey) {
        raise(t.prog, DFB_ERR_INVALID);
      } else {
        if (e[q].key == key[q]) {
          slot = (int)h[q]; w = e[q].w(); vr = e[q].vrow();
        } else {
          slot = table_find<INSERT>(t, key[q], h[q]);
          if (slot >= 0 && w_out) { w = t.tab[slot].w; vr = t.tab[slot].vrow; }
        }
      }
      slot_out[i] = slot;
      if (w_out) {
        w_out[i] = w;
        vrow_out[i] = vr;
        if (wv_out) wv_out[i] = make_int2(__float_as_int(w), vr);
      }
    }
  }
}

// SGDUpdater::Update(kFeaCount), sgd_updater.cc:62-73
__global__ void k_feacnt(Table t, Params p, const int* __restrict__ slot, size_t n_cap,
                         const unsigned long long* __restrict__ dn, const float* __restrict__ cnt,
                         const int* __restrict__ cnt_cols, int* __restrict__ flags) {
  const size_t n = dev_count(n_cap, dn);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int s = slot[i];
    int f = 0;
    if (s >= 0) {
      Entry* e = &t.tab[s];
      // counts either given, or the column lengths of the batch's CSC view (idx_frq, localizer.cc:41-46)
      const float c = cnt ? cnt[i] : (float)(cnt_cols[i + 1] - cnt_cols[i]);
      const float fc = __fadd_rn(e->fea_cnt, c);
      e->fea_cnt = fc;
      if (p.V_dim > 0 && e->vrow < 0 && e->w != 0.f && fc > (float)p.V_threshold) f = 1;
    }
    flags[i] = f;
  }
}

// ---- glibc rand_r restated: next = next*1103515245 + 12345 three times per draw ----
struct Affine { unsigned a, c; };   // x -> a*x + c  (mod 2^32)
__device__ __forceinline__ Affine compose(Affine f, Affine g) {   // g after f
  Affine r; r.a = g.a * f.a; r.c = g.a * f.c + g.c; return r;
}
__device__ __forceinline__ unsigned lcg_jump(unsigned x, unsigned long long steps) {
  Affine acc = {1u, 0u};
  Affine cur = {1103515245u, 12345u};
  unsigned m = (unsigned)steps;   // the LCG has period 2^32
  while (m) {
    if (m & 1u) acc = compose(acc, cur);
    cur = compose(cur, cur);
    m >>= 1;
  }
  return acc.a * x + acc.c;
}
__device__ __forceinline__ int rand_r_dev(unsigned* seed) {
  unsigned next = *seed, result;
  next = next * 1103515245u + 12345u; result = (next >> 16) & 2047u;
  next = next * 1103515245u + 12345u; result = (result << 10) ^ ((next >> 16) & 1023u);
  next = next * 1103515245u + 12345u; result = (result << 10) ^ ((next >> 16) & 1023u);
  *seed = next;
  return (int)result;
}

// ---- ranks of the flagged keys without a host-known count: counts per tile of 32 keys, one-CTA
// exclusive scan over the tiles, rank inside the tile from a ballot.
// ws[0..1] = total (u64), ws[2] = "any flag set" (the usual answer is no: everything after the count is skipped),
// ws[4 + t] = tile t ----
constexpr int kTileBase = 4;
__global__ void k_flag_tiles(const int* __restrict__ flags, size_t n_cap, const unsigned long long* __restrict__ dn,
                             int* __restrict__ ws) {
  const size_t n = dev_count(n_cap, dn);
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const size_t ntiles = (n + 31) / 32;
  for (size_t tl = warp0; tl < ntiles; tl += nwarps) {
    const size_t i = tl * 32 + lane;
    const unsigned m = __ballot_sync(kFull, i < n && flags[i] != 0);
    if (lane == 0) {
      ws[kTileBase + tl] = __popc(m);
      if (m) atomicOr(&ws[2], 1);
    }
  }
}

// 8 consecutive tiles per thread, 8192 per iteration of the block
__global__ void __launch_bounds__(1024) k_tile_scan(int* __restrict__ ws, size_t n_cap,
                                                    const unsigned long long* __restrict__ dn) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  if (ws[2] == 0) return;          // nothing flagged: total stays 0
  const size_t n = dev_count(n_cap, dn);
  const size_t ntiles = (n + 31) / 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int* tiles = ws + kTileBase;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (size_t b0 = 0; b0 < ntiles; b0 += (size_t)blockDim.x * 8) {
    const size_t i0 = b0 + (size_t)threadIdx.x * 8;
    int v[8], sum = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) { v[q] = i0 + q < ntiles ? tiles[i0 + q] : 0; sum += v[q]; }
    int x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(kFull, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int wv = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(kFull, wv, o);
        if (lane >= o) wv += y;
      }
      s_warp[lane] = wv;     // inclusive over warps
    }
    __syncthreads();
    const int carry = s_carry;
    int run = carry + (wid ? s_warp[wid - 1] : 0) + (x - sum);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (i0 + q < ntiles) tiles[i0 + q] = run;
      run += v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry = carry + s_warp[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *reinterpret_cast<unsigned long long*>(ws) = (unsigned long long)s_carry;
}

// InitV (sgd_updater.cc:140-147) for the flagged keys, in ascending key order of the random stream.
// A warp scans 32 flags at a time (almost always all zero) and cooperates on each set one.
__global__ void k_initv(Table t, Params p, const int* __restrict__ slot, size_t n_cap,
                        const unsigned long long* __restrict__ dn, const int* __restrict__ flags,
                        const int* __restrict__ ws) {
  if (ws[2] == 0) return;          // no key was flagged
  const size_t n = dev_count(n_cap, dn);
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int k = p.V_dim;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t mine = base + lane;
    const unsigned m0 = __ballot_sync(kFull, mine < n && flags[mine] != 0);
    if (m0 == 0) continue;
    unsigned m = m0;
    const unsigned long long vbase = t.state->n_vrows;
    const unsigned seed0 = t.state->seed;
    const unsigned long long tile_first = (unsigned long long)ws[kTileBase + (base >> 5)];
    while (m) {
      const int b = __ffs(m) - 1;
      m &= m - 1;
      const size_t i = base + b;
      const unsigned long long rank = tile_first + (unsigned long long)__popc(m0 & ((1u << b) - 1u));
      const unsigned long long r = vbase + rank;
      if (r >= t.vcap) { if (lane == 0) raise(t.prog, DFB_ERR_CAPACITY); continue; }
      float* Vr = t.V + r * t.rs;
      float* Cr = t.Vcg + r * t.rs;
      for (int l = lane; l < t.ks; l += 32) {
        float val = 0.f;
        if (l < k) {
          unsigned sd = lcg_jump(seed0, 3ULL * (rank * k + l));
          const int rr = rand_r_dev(&sd);
          // (rand_r / (real_t)RAND_MAX - 0.5) * V_init_scale: float division, then double
          const float u01 = __fdiv_rn((float)rr, 2147483648.0f);
          val = __double2float_rn(__dmul_rn(__dsub_rn((double)u01, 0.5), (double)p.V_init_scale));
        }
        Vr[l] = val;
        Cr[l] = 0.f;
      }
      if (lane == 0) t.tab[slot[i]].vrow = (int)r;
    }
  }
}

__global__ void k_initv_finalize(Table t, Params p, const int* ws) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const unsigned long long total = *reinterpret_cast<const unsigned long long*>(ws);
  if (total == 0) return;
  t.state->n_vrows += total;
  t.state->seed = lcg_jump(t.state->seed, 3ULL * total * (unsigned long long)p.V_dim);
  t.prog->new_vrows += total;
}

// fused scatter-finalize + FTRL + AdaGrad over dense per-key gradient rows.
// One group of LPR lanes (float4 each) per key.
template <int K>
__global__ void __launch_bounds__(256) k_update_fast(Table t, Params p, const int* __restrict__ slot,
                                                     const int* __restrict__ pull_vrow, int vrow_is_flag,
                                                     size_t n, const float* __restrict__ gw,
                                                     const float* __restrict__ gxxp,
                                                     const float* __restrict__ gV, int* __restrict__ flags,
                                                     int acc_pen, int xxp_mode) {
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, grp = lane / LPR;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  float pen = 0.f;
  for (size_t base = warp0 * G; base < n; base += nwarps * G) {
    const size_t i = base + grp;
    if (i >= n) continue;
    const int s = slot[i];
    if (s < 0) { if (sub == 0) flags[i] = 0; continue; }
    int vr = pull_vrow[i];
    Entry* e = &t.tab[s];
    if (vrow_is_flag && vr >= 0) vr = e->vrow;
    const float g_w = gw[i];
    if (sub == 0) {
      float4 sc = *reinterpret_cast<const float4*>(&e->fea_cnt);   // {fea_cnt, w, sqrt_g, z}
      if (acc_pen) pen += pen_w(p, sc.y);
      const bool became_nz = ftrl_step(p, g_w, sc.y, sc.z, sc.w);
      *reinterpret_cast<float4*>(&e->fea_cnt) = sc;
      flags[i] = (became_nz && p.V_dim > 0 && e->vrow < 0 && sc.x > (float)p.V_threshold) ? 1 : 0;
    }
    if (vr >= 0) {
      const float xxp = xxp_mode == 0 ? 0.f : (xxp_mode == 1 ? gxxp[i] : g_w);
      float* Vr = t.V + (size_t)vr * t.rs + sub * 4;
      float* Cr = t.Vcg + (size_t)vr * t.rs + sub * 4;
      float4 v = *reinterpret_cast<const float4*>(Vr);
      float4 c = *reinterpret_cast<const float4*>(Cr);
      const float4 g = __ldg(reinterpret_cast<const float4*>(gV + i * (size_t)t.ks + sub * 4));
      if (acc_pen) pen += 0.5f * p.V_l2 * (v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w);
      // grad_V = sum_i x p XV_i  -  V * XXp   (fm_loss.h:181-198)
      adagrad_step(p, __fsub_rn(g.x, __fmul_rn(v.x, xxp)), v.x, c.x);
      adagrad_step(p, __fsub_rn(g.y, __fmul_rn(v.y, xxp)), v.y, c.y);
      adagrad_step(p, __fsub_rn(g.z, __fmul_rn(v.z, xxp)), v.z, c.z);
      adagrad_step(p, __fsub_rn(g.w, __fmul_rn(v.w, xxp)), v.w, c.w);
      *reinterpret_cast<float4*>(Vr) = v;
      *reinterpret_cast<float4*>(Cr) = c;
    }
  }
  if (acc_pen) {
    pen = warp_sum(pen);
    if (lane == 0 && pen != 0.f) atomicAdd(&t.prog->penalty, (double)pen);
  }
}

// any V_dim: one warp per key, dense gradient rows of stride ks
__global__ void __launch_bounds__(256) k_update_dense_generic(Table t, Params p, const int* __restrict__ slot,
                                                              const int* __restrict__ pull_vrow,
                                                              int vrow_is_flag, size_t n,
                                                              const float* __restrict__ gw,
                                                              const float* __restrict__ gxxp,
                                                              const float* __restrict__ gV,
                                                              int* __restrict__ flags, int acc_pen, int xxp_mode) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int k = p.V_dim;
  float pen = 0.f;
  for (size_t i = warp0; i < n; i += nwarps) {
    const int s = slot[i];
    if (s < 0) { if (lane == 0) flags[i] = 0; continue; }
    Entry* e = &t.tab[s];
    int vr = k > 0 ? pull_vrow[i] : -1;
    if (vrow_is_flag && vr >= 0) vr = e->vrow;
    const float g_w = gw[i];
    if (lane == 0) {
      float4 sc = *reinterpret_cast<const float4*>(&e->fea_cnt);
      if (acc_pen) pen += pen_w(p, sc.y);
      const bool became_nz = ftrl_step(p, g_w, sc.y, sc.z, sc.w);
      *reinterpret_cast<float4*>(&e->fea_cnt) = sc;
      flags[i] = (became_nz && k > 0 && e->vrow < 0 && sc.x > (float)p.V_threshold) ? 1 : 0;
    }
    if (vr >= 0) {
      const float xxp = xxp_mode == 0 ? 0.f : (xxp_mode == 1 ? gxxp[i] : g_w);
      float* Vr = t.V + (size_t)vr * t.rs;
      float* Cr = t.Vcg + (size_t)vr * t.rs;
      const float* g = gV + i * (size_t)t.ks;
      for (int l = lane; l < k; l += 32) {
        float v = Vr[l], c = Cr[l];
        if (acc_pen) pen += 0.5f * p.V_l2 * v * v;
        adagrad_step(p, __fsub_rn(g[l], __fmul_rn(v, xxp)), v, c);
        Vr[l] = v; Cr[l] = c;
      }
    }
  }
  if (acc_pen) {
    pen = warp_sum(pen);
    if (lane == 0 && pen != 0.f) atomicAdd(&t.prog->penalty, (double)pen);
  }
}

// the reference's ragged layout: grads = [gw_0,(gV_0..)][gw_1,...], lens[i] in {1, k+1}
// (sgd_updater.cc:74-98).  lens == nullptr: w-only.
__global__ void __launch_bounds__(256) k_update_ragged(Table t, Params p, const int* __restrict__ slot,
                                                       size_t n, const float* __restrict__ grads,
                                                       const int* __restrict__ lens,
                                                       const int* __restrict__ pos, int* __restrict__ flags) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int k = p.V_dim;
  for (size_t i = warp0; i < n; i += nwarps) {
    const int s = slot[i];
    if (s < 0) { if (lane == 0) flags[i] = 0; continue; }
    Entry* e = &t.tab[s];
    const size_t off = lens ? (size_t)pos[i] : i;
    const int len = lens ? lens[i] : 1;
    const int vr = e->vrow;
    if (lane == 0) {
      float4 sc = *reinterpret_cast<const float4*>(&e->fea_cnt);
      const bool became_nz = ftrl_step(p, grads[off], sc.y, sc.z, sc.w);
      *reinterpret_cast<float4*>(&e->fea_cnt) = sc;
      flags[i] = (became_nz && k > 0 && vr < 0 && sc.x > (float)p.V_threshold) ? 1 : 0;
    }
    if (len > 1) {
      // CHECK_EQ(lens[i], V_dim+1); CHECK(e.V != nullptr)  (sgd_updater.cc:92-93)
      if (len != k + 1 || vr < 0) { if (lane == 0) raise(t.prog, DFB_ERR_INVALID); continue; }
      float* Vr = t.V + (size_t)vr * t.rs;
      float* Cr = t.Vcg + (size_t)vr * t.rs;
      const float* g = grads + off + 1;
      for (int l = lane; l < k; l += 32) {
        float v = Vr[l], c = Cr[l];
        adagrad_step(p, g[l], v, c);
        Vr[l] = v; Cr[l] = c;
      }
    }
  }
}

// penalty over pulled rows without updating (validation batches and the sharded worker;
// sgd_learner.cc:249-273).  w_arr[i] is the pulled w; the V row is V + vrow[i]*ks, or
// V + i*ks when dense (a pulled [n][ks] buffer with vrow[i] >= 0 meaning "present").
__global__ void __launch_bounds__(256) k_penalty(Params p, DevProgress* prog, const float* __restrict__ w_arr,
                                                 const int* __restrict__ vrow, const float* __restrict__ V,
                                                 int ks, int dense, size_t n_cap,
                                                 const unsigned long long* __restrict__ dn) {
  const size_t n = dev_count(n_cap, dn);
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int k = p.V_dim;
  float pen = 0.f;
  for (size_t i = warp0; i < n; i += nwarps) {
    if (lane == 0) pen += pen_w(p, w_arr[i]);
    const int vr = k > 0 ? vrow[i] : -1;
    if (vr >= 0) {
      const float* Vr = V + (dense ? i : (size_t)vr) * (size_t)ks;
      for (int l = lane; l < k; l += 32) pen += 0.5f * p.V_l2 * Vr[l] * Vr[l];
    }
  }
  pen = warp_sum(pen);
  if (lane == 0 && pen != 0.f) atomicAdd(&prog->penalty, (double)pen);
}

// w and vrow of already-located entries (the Pull of the fused path after a feature-count push)
__global__ void k_pull_view(Table t, const int* __restrict__ slot, size_t n_cap,
                            const unsigned long long* __restrict__ dn, float* __restrict__ w_out,
                            int* __restrict__ vrow_out, int2* __restrict__ wv_out) {
  const size_t n = dev_count(n_cap, dn);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int s = slot[i];
    const float w = s >= 0 ? t.tab[s].w : 0.f;
    const int vr = s >= 0 ? t.tab[s].vrow : -1;
    w_out[i] = w;
    vrow_out[i] = vr;
    if (wv_out) wv_out[i] = make_int2(__float_as_int(w), vr);
  }
}

// SGDUpdater::Get: lens (sgd_updater.cc:46-53)
__global__ void k_lens(Table t, Params p, const int* __restrict__ slot, size_t n, int* __restrict__ lens) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slot[i];
  int len = 1;
  if (p.V_dim > 0 && s >= 0 && t.tab[s].vrow >= 0) len = p.V_dim + 1;
  lens[i] = len;
}

__global__ void k_pack_ragged(Table t, Params p, const int* __restrict__ slot, size_t n,
                              const int* __restrict__ lens, const int* __restrict__ pos,
                              float* __restrict__ vals, unsigned long long* nvals_out) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int k = p.V_dim;
  for (size_t i = warp0; i < n; i += nwarps) {
    const int s = slot[i];
    const size_t off = (size_t)pos[i];
    if (lane == 0) vals[off] = s >= 0 ? t.tab[s].w : 0.f;
    if (lens[i] > 1) {
      const float* Vr = t.V + (size_t)t.tab[s].vrow * t.rs;
      for (int l = lane; l < k; l += 32) vals[off + 1 + l] = Vr[l];
    }
    if (i == n - 1 && lane == 0) *nvals_out = (unsigned long long)pos[i] + (unsigned long long)lens[i];
  }
}

__global__ void __launch_bounds__(256) k_gather_rows(Table t, const int* __restrict__ slot, size_t n,
                                                     float* __restrict__ w_out, int* __restrict__ hasv_out,
                                                     int* __restrict__ hasv_out2, float* __restrict__ V_out) {
  const int lane = threadIdx.x & 31, sub = lane & 15, grp = lane >> 4;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int nv4 = t.ks / 4;
  for (size_t base = warp0 * 32; base < n; base += nwarps * 32) {
    const size_t i = base + lane;
    int vr = -1;
    if (i < n) {
      const int s = slot[i];
      float w = 0.f;
      if (s >= 0) { w = t.tab[s].w; vr = t.tab[s].vrow; }
      w_out[i] = w;
      hasv_out[i] = vr >= 0 ? 1 : -1;
      if (hasv_out2) hasv_out2[i] = vr >= 0 ? 1 : -1;
    }
    if (!V_out) continue;
    // two rows per pass (16 lanes each), four passes in flight
#pragma unroll 1
    for (int pass = 0; pass < 16; pass += 4) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int kk = (pass + q) * 2 + grp;
        const int vr_k = __shfl_sync(kFull, vr, kk);
        if (vr_k < 0) continue;
        const float4* src = reinterpret_cast<const float4*>(t.V + (size_t)vr_k * t.rs);
        float4* dst = reinterpret_cast<float4*>(V_out + (base + kk) * (size_t)t.ks);
        for (int l = sub; l < nv4; l += 16) dst[l] = src[l];
      }
    }
  }
}

__global__ void k_read_entries(Table t, const int* __restrict__ slot, size_t n, float* scal, int* hasv,
                               float* V, float* cg, int k) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = slot[i];
  if (s < 0) {
    hasv[i] = -1;
    for (int j = 0; j < 4; ++j) scal[i * 4 + j] = 0.f;
    return;
  }
  const Entry e = t.tab[s];
  scal[i * 4 + 0] = e.fea_cnt; scal[i * 4 + 1] = e.w; scal[i * 4 + 2] = e.sqrt_g; scal[i * 4 + 3] = e.z;
  hasv[i] = e.vrow >= 0 ? 1 : 0;
  if (e.vrow >= 0) {
    for (int l = 0; l < k; ++l) {
      if (V) V[i * (size_t)k + l] = t.V[(size_t)e.vrow * t.rs + l];
      if (cg) cg[i * (size_t)k + l] = t.Vcg[(size_t)e.vrow * t.rs + l];
    }
  }
}

// checkpoint restore: insert the saved keys and write their scalar state / row index
__global__ void k_restore(Table t, const uint64_t* __restrict__ keys, size_t n, const float* __restrict__ scal,
                          const int* __restrict__ vrow) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = keys[i];
  uint64_t h = hash64(key) & t.mask;
  for (uint64_t probe = 0; probe <= t.mask; ++probe) {
    const unsigned long long prev = atomicCAS(&t.tab[h].key, kEmptyKey, key);
    if (prev == kEmptyKey || prev == key) {
      Entry* e = &t.tab[h];
      e->vrow = vrow[i];
      e->fea_cnt = scal[i * 4 + 0]; e->w = scal[i * 4 + 1]; e->sqrt_g = scal[i * 4 + 2]; e->z = scal[i * 4 + 3];
      return;
    }
    h = (h + 1) & t.mask;
  }
  raise(t.prog, DFB_ERR_CAPACITY);
}

__global__ void k_set_state(TableState* st, unsigned long long n_keys, unsigned long long n_vrows, unsigned seed) {
  st->n_keys = n_keys; st->n_vrows = n_vrows; st->seed = seed;
}

// table growth, two launches of one kernel: phase 0 writes the empty entry into every slot of the new table, phase 1
// re-inserts every occupied entry of the old one -- all 32 bytes as they are -- with table_find's hash and linear
// probing.  The keys are unique, so a claimed slot is always an empty one.  TableState is not touched.
__global__ void __launch_bounds__(256) k_table_rehash(const Entry* __restrict__ old_tab, uint64_t old_cap, Entry* nw,
                                                      uint64_t nw_mask, int phase) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  ulonglong2* out = reinterpret_cast<ulonglong2*>(nw);
  if (phase == 0) {
    for (size_t i = i0; i <= nw_mask; i += stride) {
      out[2 * i] = make_ulonglong2(kEmptyKey, 0x00000000ffffffffULL);    // {key, vrow -1 | pad 0}
      out[2 * i + 1] = make_ulonglong2(0ULL, 0ULL);                      // fea_cnt, w, sqrt_g, z
    }
    return;
  }
  const ulonglong2* in = reinterpret_cast<const ulonglong2*>(old_tab);
  for (size_t i = i0; i < old_cap; i += stride) {
    const ulonglong2 a = in[2 * i];
    if (a.x == kEmptyKey) continue;
    const ulonglong2 b = in[2 * i + 1];
    uint64_t h = hash64(a.x) & nw_mask;
    for (uint64_t probe = 0; probe <= nw_mask; ++probe) {
      if (atomicCAS(&nw[h].key, kEmptyKey, a.x) == kEmptyKey) {
        out[2 * h] = a;
        out[2 * h + 1] = b;
        break;
      }
      h = (h + 1) & nw_mask;
    }
  }
}

// Loss::Evaluate, loss.h:57-66
__global__ void k_evaluate(const float* __restrict__ label, const float* __restrict__ pred, size_t n, double* out) {
  __shared__ float red_s[32];
  float acc = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float y = label[i] > 0.f ? 1.f : -1.f;
    acc += logf(1.f + expf(-y * pred[i]));
  }
  acc = warp_sum(acc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red_s[wid] = acc;
  __syncthreads();
  if (wid == 0) {
    float v = lane < (int)(blockDim.x >> 5) ? red_s[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0) atomicAdd(out, (double)v);
  }
}

// BinClassMetric::AUC (bin_class_metric.h:35-56) on (pred ascending, label) pairs
__global__ void __launch_bounds__(1024) k_auc_area(const float* __restrict__ sorted_label, size_t n, double* out_add,
                                                   const unsigned long long* __restrict__ dev_nkeys) {
  if (dev_nkeys && *dev_nkeys == 0ULL) return;     // a batch the GPU localizer dropped: no prediction was made
  __shared__ unsigned long long s_tp[1024];
  __shared__ unsigned long long s_area[1024];
  const int tid = threadIdx.x;
  const size_t per = (n + blockDim.x - 1) / blockDim.x;
  const size_t b = (size_t)tid * per, e = b + per < n ? b + per : n;
  unsigned long long tp = 0;
  for (size_t i = b; i < e; ++i) tp += sorted_label[i] > 0.f ? 1 : 0;
  s_tp[tid] = tp;
  __syncthreads();
  // exclusive prefix of positives before this thread's chunk (serial over 1024 in thread 0: tiny)
  if (tid == 0) {
    unsigned long long run = 0;
    for (int i = 0; i < (int)blockDim.x; ++i) { const unsigned long long c = s_tp[i]; s_tp[i] = run; run += c; }
    s_area[0] = run;   // total positives, stashed
  }
  __syncthreads();
  const unsigned long long total_tp = s_area[0];
  __syncthreads();
  unsigned long long cum = s_tp[tid], area = 0;
  for (size_t i = b; i < e; ++i) {
    if (sorted_label[i] > 0.f) cum += 1; else area += cum;
  }
  s_area[tid] = area;
  __syncthreads();
  if (tid == 0) {
    unsigned long long a = 0;
    for (int i = 0; i < (int)blockDim.x; ++i) a += s_area[i];
    double res;
    if (total_tp == 0 || total_tp == n) {
      res = 1.0;   // bin_class_metric.h:52
    } else {
      double ar = (double)a / ((double)total_tp * (double)(n - total_tp));
      res = (ar < 0.5 ? 1.0 - ar : ar) * (double)n;
    }
    *out_add += res;
  }
}


// ---------------------------------------------------------------------------------------
// sorted (atomic-free) gradient reduction
// ---------------------------------------------------------------------------------------
// boundaries of the runs of equal key ids in the sorted id list
__global__ void k_col_bounds(const uint32_t* __restrict__ sorted, size_t n, size_t nkeys, int* __restrict__ col_start,
                             int* __restrict__ col_end, DevProgress* prog) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t cur = sorted[j];
  // a caller-provided local index outside [0, nkeys) would write out of bounds: report it instead (the sort
  // only looks at ceil(log2 nkeys) bits, so such an index shows up here as a value >= nkeys or out of order)
  if (cur >= nkeys || (j > 0 && sorted[j - 1] > cur)) { if (prog) raise(prog, DFB_ERR_INVALID); return; }
  if (j == 0) col_start[cur] = 0;
  else {
    const uint32_t prev = sorted[j - 1];
    if (prev != cur) { col_start[cur] = (int)j; col_end[prev] = (int)j; }
  }
  if (j == n - 1) col_end[cur] = (int)n;
}

// HINT: with the L2 policy pol (the occurrence lists are read once per step)
template <bool HAS_VAL, bool HINT = false>
__device__ __forceinline__ void load_occ(const void* occ, int o, uint32_t& row, float& x, uint64_t pol = 0) {
  if (HAS_VAL) {
    const unsigned long long* q = reinterpret_cast<const unsigned long long*>(occ) + o;
    const unsigned long long rx = HINT ? ldg_u64_pol(q, pol) : __ldg(q);
    row = (uint32_t)(rx >> 32);
    x = __uint_as_float((uint32_t)rx);
  } else {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(occ) + o;
    row = HINT ? ldg_u32_pol(q, pol) : __ldg(q);
    x = 1.f;
  }
}

// Per unique key: grad_w = sum x p_i, XXp = sum x^2 p_i, grad_V = sum x (p XV)_i - V XXp
// (fm_loss.h:164-198, summed in row order like SpMM::TransTimes), immediately consumed by
// FTRL (w) and AdaGrad (V): the gradient never exists in HBM.  APPLY=false writes the dense
// gradient rows instead (worker side of the sharded store).
//
// A warp owns 32 consecutive keys.  Phase A is lane-parallel (one key per lane): coalesced
// metadata loads, 32 independent entry sectors in flight, the scalar reductions and FTRL.
// Phase B walks the 32 keys G at a time with LPR lanes (one float4 each) per 8K-byte table row,
// UNRB row-groups in flight; the first occurrence's p*XV row is fetched together with V|cg.
// SRC 0: gradient reduced from the occurrence lists (fused step / worker).  SRC 1: gradient read
// from dense rows gw_in[n], gV_in[n][K] that a worker pushed (owner side of the sharded store).
// SRC 0 with APPLY (the single-GPU step) and keys != nullptr finds or inserts every key itself: lane i reads keys[i],
// loads the entry at its hash (the whole 32-byte sector, as k_lookup does) and walks the probe chain only when that is
// not the key; the slot goes to slot_out[i] for the InitV pass.  The keys of a batch are unique, so one lane inserts
// each of them.  Otherwise (a step that ran k_lookup; SRC 1 / 2) the slots and pulled V-row indices of the earlier
// lookup come in slot / pull_vrow.
// PAD (V_dim < K, single-GPU step and SRC 2 only): lanes at or beyond ks = t.ks touch nothing, the per-row buffers
// (p*XV, hot-key partials, vsave) have stride ks, and the pad columns [V_dim, ks) of the last float4 are not updated.
// 3 CTAs/SM (80 registers): at 4 (64 registers) sm_90 spills ~100 bytes per thread and the update stage of the
// V_dim = 64 training step takes 3.54 ms instead of 3.34 ms (H100 SXM, 700 W)
#ifndef DFB_BU_MINBLOCKS
#define DFB_BU_MINBLOCKS 3
#endif
#ifndef DFB_BU_UNRB
#define DFB_BU_UNRB 2
#endif
template <int K, bool HAS_VAL, bool APPLY, int SRC = 0, bool HINT = false, bool PAD = false, bool FIND = false>
__global__ void __launch_bounds__(256, DFB_BU_MINBLOCKS) k_bwd_update(Table t, Params p, const int* __restrict__ slot,
                                                    const int* __restrict__ pull_vrow, size_t n_cap,
                                                    const unsigned long long* __restrict__ dn,
                                                    const int* __restrict__ col_start,
                                                    const int* __restrict__ col_end,
                                                    const void* __restrict__ occ,
                                                    const float* __restrict__ p_row,
                                                    const float* __restrict__ pxv, int* __restrict__ flags,
                                                    int acc_pen, float* __restrict__ gw_out,
                                                    const float* __restrict__ V_pulled,
                                                    float* __restrict__ gV_out, SegDst seg, ShardApply sa,
                                                    HotPart hp, const unsigned long long* __restrict__ keys,
                                                    int* __restrict__ slot_out) {
  const unsigned n = (unsigned)dev_count(n_cap, dn);     // < 2^31 (checked by the host): 32-bit index math
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  constexpr int NPASS = 32 / G;
  constexpr int UNRB = NPASS >= DFB_BU_UNRB ? DFB_BU_UNRB : 1;
  constexpr int kHeavy = 64;     // occurrence-list length above which a key is reduced cooperatively
  static_assert(!PAD || (APPLY && SRC != 1), "padded rows: the table-applying update of the fused paths only");
  // FIND: the single-GPU step without an earlier lookup, keys in, slots out (its own instantiations, so that the
  // slot-taking ones stay as they were)
  static_assert(!FIND || (SRC == 0 && APPLY), "the key-finding update is the single-GPU step's");
  const int lane = threadIdx.x & 31, sub = lane % LPR, grp = lane / LPR;
  const int ks = PAD ? t.ks : K;                  // stride of the per-row buffers
  const bool act = !PAD || sub * 4 < ks;          // this lane's float4 holds V columns
  const int nact = PAD ? min(4, p.V_dim - sub * 4) : 4;
  const unsigned warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  // L2 plan of the single-GPU step (dfb_device.cuh): this batch's p*XV rows and p (16.8 MB at the flagship shape) are
  // read once per nnz and kept (evict_last); the [V|cg] rows and the per-key metadata are touched once and stream
  // past them (evict_first).  The 32-byte entry keeps the default policy: it is half-written and its other half read
  // again after the store, and evict_first on it made the update 0.26 ms slower (V_dim 64, H100 SXM, 700 W).
  // HINT = false is the default policy: the sharded kernels (SRC 1 / 2, APPLY = false), which read p*XV of up to 8
  // workers (more than L2 holds), and steps whose table rows fit in L2 (the host decides: step_dev in engine.cu).
  static_assert(!HINT || (SRC == 0 && APPLY), "the L2 plan is the single-GPU fused step's");
  const uint64_t pol_keep = HINT ? l2_policy(kL2EvictLast) : 0;
  const uint64_t pol_once = HINT ? l2_policy(kL2EvictFirst) : 0;
  auto ld_meta = [&](const int* a) { return HINT ? ldg_s32_pol(a, pol_once) : __ldg(a); };
  auto ld_p = [&](const float* a) { return HINT ? ldg_f32_pol(a, pol_keep) : __ldg(a); };
  auto ld_pxv = [&](const float* a) {
    return HINT ? ldg128_pol(a, pol_keep) : __ldg(reinterpret_cast<const float4*>(a));
  };
  auto ld_row = [&](const float* a) { return HINT ? ld128_pol(a, pol_once) : *reinterpret_cast<const float4*>(a); };
  auto st_row = [&](float* a, float4 v) {
    if (HINT) st128_pol(a, v, pol_once); else *reinterpret_cast<float4*>(a) = v;
  };
  float pen = 0.f;
  const unsigned npad = (n + 31u) / 32u * 32u;
  for (unsigned b0 = warp0 * 32u; b0 < n; b0 += nwarps * 32u) {
    // start at this rank's own key segment and go round: at any moment the ranks of a sharded
    // step store into different peers (seg.rot == 0 outside the peer-store path)
    unsigned base = b0 + (unsigned)seg.rot;
    if (base >= npad) base -= npad;
    // ---------------- phase A: one key per lane ----------------
    const unsigned i = base + lane;
    const bool active = i < n;
    int s = -1, vr = -1, o0 = 0, o1 = 0;
    unsigned long long key = 0;
    if (active) {
      if (FIND) key = HINT ? ldg_u64_pol(keys + i, pol_once) : __ldg(keys + i);
      else vr = ld_meta(pull_vrow + i);
      if (SRC != 1) { o0 = ld_meta(col_start + i); o1 = ld_meta(col_end + i); }
      if (APPLY && !FIND) s = ld_meta(slot + i);
    }
    // SRC 2 (owner side of the fused sharded store): this key was already updated in this step by a
    // lower-rank worker's push, so the pull-time V row is the saved copy, not the table row
    const int cf = (SRC == 2 && active && sa.conf != nullptr) ? (int)sa.conf[i] : 0;
    Entry* e = nullptr;
    float4 sc = make_float4(0.f, 0.f, 0.f, 0.f);
    // FIND: the entry sector at the key's hash is loaded here and looked at only after the scalar reduction below, so
    // that its DRAM latency overlaps the occurrence-list loads instead of stalling the lane in front of them
    Entry256 en;
    if (FIND && active && key != kEmptyKey) en = load_entry(t.tab + (hash64(key) & t.mask));
    if (!FIND && APPLY && s >= 0) {
      e = &t.tab[s];
      sc = *reinterpret_cast<const float4*>(&e->fea_cnt);
    }
    float gw = 0.f, xxp = 0.f, x0 = 0.f;
    uint32_t row0 = 0;
    if (SRC == 1 && active) gw = p_row[i];      // dense source: p_row aliases gw_in
    // keys with at most kHeavy occurrences: this lane sums them strictly in row order (the
    // reference's order, spmv.h:162-164), four loads in flight; longer lists ("hot" features of a
    // skewed batch) are reduced by the whole warp below (fixed tree: still bit-reproducible)
    const bool heavy = (o1 - o0) > kHeavy;
    if (o0 < o1) load_occ<HAS_VAL, HINT>(occ, o0, row0, x0, pol_once);
    if (!heavy) {
      for (int o = o0; o < o1; o += 4) {
        uint32_t rw[4]; float xs[4], pr[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          rw[q] = 0; xs[q] = 0.f; pr[q] = 0.f;
          if (o + q < o1) { load_occ<HAS_VAL, HINT>(occ, o + q, rw[q], xs[q], pol_once); pr[q] = ld_p(p_row + rw[q]); }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (o + q < o1) {
            gw = __fadd_rn(gw, __fmul_rn(pr[q], xs[q]));
            if (HAS_VAL) xxp = __fadd_rn(xxp, __fmul_rn(pr[q], __fmul_rn(xs[q], xs[q])));
          }
        }
      }
    }
    if (SRC != 1) {
      unsigned hm = __ballot_sync(kFull, heavy);
      while (hm) {
        const int hl = __ffs(hm) - 1;
        hm &= hm - 1;
        const int ho0 = __shfl_sync(kFull, o0, hl), ho1 = __shfl_sync(kFull, o1, hl);
        float a = 0.f, b2 = 0.f;
        int first = -1;
        if (hp.part != nullptr && ho1 - ho0 > hp.split) first = hp.hotmap[base + (unsigned)hl];
        if (first >= 0) {      // pre-reduced in chunks (k_hot_reduce): add the chunk partials in chunk order
          if (lane == 0) {
            const int nch = (ho1 - ho0 + hp.chunk - 1) / hp.chunk;
            for (int c = 0; c < nch; ++c) { const float2 ps = hp.part_s[first + c]; a += ps.x; b2 += ps.y; }
          }
        } else
        for (int o = ho0 + lane; o < ho1; o += 32) {
          uint32_t row; float x;
          load_occ<HAS_VAL, HINT>(occ, o, row, x, pol_once);
          const float pr = ld_p(p_row + row);
          a = fmaf(pr, x, a);
          if (HAS_VAL) b2 = fmaf(pr, x * x, b2);
        }
        a = warp_sum(a);
        if (HAS_VAL) b2 = warp_sum(b2);
        if (lane == hl) { gw = a; xxp = b2; }
      }
    }
    if (!HAS_VAL) xxp = gw;
    if (SRC == 1) xxp = 0.f;                    // pushed rows are complete gradients
    if (FIND && active) {
      if (key == kEmptyKey) {
        raise(t.prog, DFB_ERR_INVALID);         // the empty marker is no key (k_lookup reports it the same way)
      } else {
        s = find_insert_entry(t, key, hash64(key) & t.mask, en);
        if (s >= 0) { vr = en.vrow(); sc = en.scalars(); e = &t.tab[s]; }
      }
      slot_out[i] = s;
    }
    if (APPLY) {
      if (s >= 0) {
        if (vr >= 0) vr = SRC == 1 ? e->vrow : vr;   // SRC 1: pull_vrow is the worker's has_V flag
        if (acc_pen) pen += pen_w(p, SRC == 2 ? sa.w_pulled[i] : sc.y);   // penalty of the PULLED weights (sgd_learner.cc:148)
        const bool became_nz = ftrl_step(p, gw, sc.y, sc.z, sc.w);
        *reinterpret_cast<float4*>(&e->fea_cnt) = sc;
        if (SRC == 2) {
          // sharded store: InitV of all workers' updates runs once after the last one (same order of the random
          // stream: worker-major, key order); vrow = -2 marks "row pending" so that a later worker's update in
          // the same step neither uses nor re-requests it
          const bool fl = became_nz && p.V_dim > 0 && e->vrow == -1 && sc.x > (float)p.V_threshold;
          if (fl) e->vrow = -2;
          flags[i] = fl ? 1 : 0;
        } else {
          flags[i] = (became_nz && p.V_dim > 0 && (FIND ? vr : e->vrow) < 0 && sc.x > (float)p.V_threshold) ? 1 : 0;
        }
      } else if (active) {
        flags[i] = 0;
      }
      if (s < 0) vr = -1;
    } else if (active) {
      if (seg.nseg == 0) {
        gw_out[i] = gw;
      } else {   // the owner's receive buffer (peer memory over NVLink)
        int sg = 0;
        while (sg + 1 < seg.nseg && (int)i >= seg.bounds[sg + 1]) ++sg;
        seg.gw[sg][i - (unsigned)seg.bounds[sg]] = gw;
      }
      if (acc_pen) pen += pen_w(p, slot ? __int_as_float(slot[i]) : 0.f);   // worker: slot aliases the pulled w
    }
    // ---------------- phase B: the table rows, G keys per pass ----------------
#pragma unroll 1
    for (int pass = 0; pass < NPASS; pass += UNRB) {
      float4 v[UNRB], c[UNRB], g[UNRB];
      int vrk[UNRB], o0k[UNRB], o1k[UNRB], cfk[UNRB];
      float xxpk[UNRB];
#pragma unroll
      for (int q = 0; q < UNRB; ++q) {
        const int kk = (pass + q) * G + grp;
        vrk[q] = __shfl_sync(kFull, vr, kk);
        o0k[q] = __shfl_sync(kFull, o0, kk);
        o1k[q] = __shfl_sync(kFull, o1, kk);
        xxpk[q] = __shfl_sync(kFull, xxp, kk);
        cfk[q] = SRC == 2 ? __shfl_sync(kFull, cf, kk) : 0;
        const uint32_t r0 = __shfl_sync(kFull, row0, kk);
        const float xx0 = __shfl_sync(kFull, x0, kk);
        v[q] = c[q] = g[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (o1k[q] - o0k[q] > kHeavy) vrk[q] = -1;      // handled by the whole warp after the passes
        if (vrk[q] >= 0 && act) {
          if (APPLY) {
            const float* Vr = t.V + (size_t)vrk[q] * t.rs + sub * 4;
            v[q] = ld_row(Vr);
            c[q] = ld_row(Vr + t.ks);
          } else {
            // the pulled row (dense [n][K] buffer): the worker applies "- V * XXp" itself (fm_loss.h:181-188)
            const size_t ik = base + (unsigned)((pass + q) * G + grp);
            v[q] = __ldg(reinterpret_cast<const float4*>(V_pulled + ik * (size_t)K + sub * 4));
          }
          if (SRC == 1) {
            const size_t ik = base + (unsigned)((pass + q) * G + grp);
            g[q] = __ldg(reinterpret_cast<const float4*>(pxv + ik * (size_t)K + sub * 4));   // pxv aliases gV_in
          } else if (o1k[q] > o0k[q]) {
            const float4 tt = ld_pxv(pxv + (size_t)r0 * ks + sub * 4);
            g[q] = make_float4(__fmul_rn(tt.x, xx0), __fmul_rn(tt.y, xx0), __fmul_rn(tt.z, xx0),
                               __fmul_rn(tt.w, xx0));                                   // spmm.h:152-154
          }
        }
      }
#pragma unroll
      for (int q = 0; q < UNRB; ++q) {
        if (vrk[q] < 0 || !act) continue;
        for (int o = o0k[q] + 1; o < o1k[q]; o += 4) {   // further occurrences: loads 4 ahead, sums in row order
          float4 tt[4]; float xs[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            xs[r] = 0.f; tt[r] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (o + r < o1k[q]) {
              uint32_t row;
              load_occ<HAS_VAL, HINT>(occ, o + r, row, xs[r], pol_once);
              tt[r] = ld_pxv(pxv + (size_t)row * ks + sub * 4);
            }
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            if (o + r < o1k[q]) {
              g[q].x = __fadd_rn(g[q].x, __fmul_rn(tt[r].x, xs[r])); g[q].y = __fadd_rn(g[q].y, __fmul_rn(tt[r].y, xs[r]));
              g[q].z = __fadd_rn(g[q].z, __fmul_rn(tt[r].z, xs[r])); g[q].w = __fadd_rn(g[q].w, __fmul_rn(tt[r].w, xs[r]));
            }
          }
        }
        if (APPLY) {
          // the worker's gradient is taken at the PULLED V (fm_loss.h:181-188); it differs from the table row
          // only for a key a lower-rank worker's push has already updated in this step (SRC 2)
          float4 vp = v[q];
          if (SRC == 2 && cfk[q])
            vp = __ldg(reinterpret_cast<const float4*>(sa.vsave + (size_t)(base + (unsigned)((pass + q) * G + grp)) * (size_t)ks + sub * 4));
          if (acc_pen) pen += 0.5f * p.V_l2 * (vp.x * vp.x + vp.y * vp.y + vp.z * vp.z + vp.w * vp.w);
          adagrad4<PAD>(p, g[q], vp, xxpk[q], v[q], c[q], nact);
          float* Vr = t.V + (size_t)vrk[q] * t.rs + sub * 4;
          st_row(Vr, v[q]);
          st_row(Vr + t.ks, c[q]);
        } else {
          const size_t ik = base + (unsigned)((pass + q) * G + grp);
          const float xp = xxpk[q];
          if (acc_pen) pen += 0.5f * p.V_l2 * (v[q].x * v[q].x + v[q].y * v[q].y + v[q].z * v[q].z + v[q].w * v[q].w);
          float* grow = gV_out + ik * (size_t)K;
          if (seg.nseg != 0) {
            int sg = 0;
            while (sg + 1 < seg.nseg && (int)ik >= seg.bounds[sg + 1]) ++sg;
            grow = seg.gV[sg] + (ik - (size_t)seg.bounds[sg]) * (size_t)K;
          }
          *reinterpret_cast<float4*>(grow + sub * 4) =
              make_float4(__fsub_rn(g[q].x, __fmul_rn(v[q].x, xp)), __fsub_rn(g[q].y, __fmul_rn(v[q].y, xp)),
                          __fsub_rn(g[q].z, __fmul_rn(v[q].z, xp)), __fsub_rn(g[q].w, __fmul_rn(v[q].w, xp)));
        }
      }
    }
    // ---------------- hot keys: the whole warp reduces one occurrence list ----------------
    if (SRC != 1) {
      unsigned hm = __ballot_sync(kFull, active && (o1 - o0) > kHeavy && vr >= 0);
      while (hm) {
        const int hl = __ffs(hm) - 1;
        hm &= hm - 1;
        const int hvr = __shfl_sync(kFull, vr, hl);
        const int ho0 = __shfl_sync(kFull, o0, hl), ho1 = __shfl_sync(kFull, o1, hl);
        const float hxp = __shfl_sync(kFull, xxp, hl);
        const int hcf = SRC == 2 ? __shfl_sync(kFull, cf, hl) : 0;
        const size_t ik = base + (unsigned)hl;
        float4 hv = make_float4(0.f, 0.f, 0.f, 0.f), hc = hv;
        float* Vr = nullptr;
        if (grp == 0 && act) {
          if (APPLY) {
            Vr = t.V + (size_t)hvr * t.rs + sub * 4;
            hv = ld_row(Vr);
            hc = ld_row(Vr + t.ks);
          } else {
            hv = __ldg(reinterpret_cast<const float4*>(V_pulled + ik * (size_t)K + sub * 4));
          }
        }
        float4 acc[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        int first = -1;
        if (hp.part != nullptr && ho1 - ho0 > hp.split) first = hp.hotmap[ik];
        if (first >= 0) {      // pre-reduced in chunks: chunk partials in chunk order
          if (grp == 0 && act) {
            const int nch = (ho1 - ho0 + hp.chunk - 1) / hp.chunk;
            for (int c = 0; c < nch; ++c) {
              const float4 tp = __ldg(reinterpret_cast<const float4*>(hp.part + (size_t)(first + c) * ks + sub * 4));
              acc[0].x += tp.x; acc[0].y += tp.y; acc[0].z += tp.z; acc[0].w += tp.w;
            }
          }
        } else
        for (int o = ho0 + grp; o < ho1; o += 4 * G) {    // G row-groups x 4 rows in flight
          float4 tt[4]; float xs[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            xs[r] = 0.f; tt[r] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (o + r * G < ho1 && act) {
              uint32_t row;
              load_occ<HAS_VAL, HINT>(occ, o + r * G, row, xs[r], pol_once);
              tt[r] = ld_pxv(pxv + (size_t)row * ks + sub * 4);
            }
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            acc[r].x = fmaf(tt[r].x, xs[r], acc[r].x); acc[r].y = fmaf(tt[r].y, xs[r], acc[r].y);
            acc[r].z = fmaf(tt[r].z, xs[r], acc[r].z); acc[r].w = fmaf(tt[r].w, xs[r], acc[r].w);
          }
        }
        float4 hg = make_float4((acc[0].x + acc[1].x) + (acc[2].x + acc[3].x), (acc[0].y + acc[1].y) + (acc[2].y + acc[3].y),
                                (acc[0].z + acc[1].z) + (acc[2].z + acc[3].z), (acc[0].w + acc[1].w) + (acc[2].w + acc[3].w));
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) {
          hg.x += __shfl_xor_sync(kFull, hg.x, o); hg.y += __shfl_xor_sync(kFull, hg.y, o);
          hg.z += __shfl_xor_sync(kFull, hg.z, o); hg.w += __shfl_xor_sync(kFull, hg.w, o);
        }
        if (grp == 0 && act) {
          float4 hp = hv;      // the pulled row (see phase B)
          if (SRC == 2 && hcf)
            hp = __ldg(reinterpret_cast<const float4*>(sa.vsave + ik * (size_t)ks + sub * 4));
          if (acc_pen) pen += 0.5f * p.V_l2 * (hp.x * hp.x + hp.y * hp.y + hp.z * hp.z + hp.w * hp.w);
          if (APPLY) {
            adagrad4<PAD>(p, hg, hp, hxp, hv, hc, nact);
            st_row(Vr, hv);
            st_row(Vr + t.ks, hc);
          } else {
            float* grow = gV_out + ik * (size_t)K;
            if (seg.nseg != 0) {
              int sg = 0;
              while (sg + 1 < seg.nseg && (int)ik >= seg.bounds[sg + 1]) ++sg;
              grow = seg.gV[sg] + (ik - (size_t)seg.bounds[sg]) * (size_t)K;
            }
            *reinterpret_cast<float4*>(grow + sub * 4) =
                make_float4(__fsub_rn(hg.x, __fmul_rn(hv.x, hxp)), __fsub_rn(hg.y, __fmul_rn(hv.y, hxp)),
                            __fsub_rn(hg.z, __fmul_rn(hv.z, hxp)), __fsub_rn(hg.w, __fmul_rn(hv.w, hxp)));
          }
        }
      }
    }
  }
  if (acc_pen) {
    pen = warp_sum(pen);
    if (lane == 0 && pen != 0.f) atomicAdd(&t.prog->penalty, (double)pen);
  }
}

// ---- pre-reduction of the very hot keys (see HotPart) ----
__global__ void k_hot_find(const int* __restrict__ col_start, const int* __restrict__ col_end, size_t n_cap,
                           const unsigned long long* __restrict__ dn, int split, int chunk, HotWs ws) {
  const size_t n = dev_count(n_cap, dn);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int o0 = col_start[i], o1 = col_end[i];
    if (o1 - o0 <= split) continue;
    const int nch = (o1 - o0 + chunk - 1) / chunk;
    const unsigned long long first = atomicAdd(ws.counter, (unsigned long long)nch);
    if (first + (unsigned long long)nch > (unsigned long long)ws.cap) { ws.hotmap[i] = -1; continue; }   // falls back to one warp
    ws.hotmap[i] = (int)first;
    for (int c = 0; c < nch; ++c) {
      const int b = o0 + c * chunk;
      ws.info[first + c] = make_int2(b, b + chunk < o1 ? b + chunk : o1);
    }
  }
}

// PAD: rows of stride ks < K (see k_bwd_update)
template <int K, bool HAS_VAL, bool PAD = false>
__global__ void __launch_bounds__(256) k_hot_reduce(const void* __restrict__ occ, const float* __restrict__ p_row,
                                                    const float* __restrict__ pxv, HotWs ws, int l2hint, int ks_pad) {
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, grp = lane / LPR;
  const int ks = PAD ? ks_pad : K;
  const bool act = !PAD || sub * 4 < ks;
  const unsigned warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  // the L2 plan of k_bwd_update: p*XV / p kept for the update that follows, the occurrence lists streamed
  const uint64_t pol_keep = l2_policy(l2hint ? kL2EvictLast : kL2Normal);
  const uint64_t pol_once = l2_policy(l2hint ? kL2EvictFirst : kL2Normal);
  unsigned long long nch = *ws.counter;
  if (nch > (unsigned long long)ws.cap) nch = 0;     // overflow: nothing was registered consistently beyond cap
  for (unsigned c = warp0; c < (unsigned)nch; c += nwarps) {
    const int2 be = ws.info[c];
    float a = 0.f, b2 = 0.f;
    for (int o = be.x + lane; o < be.y; o += 32) {
      uint32_t row; float x;
      load_occ<HAS_VAL, true>(occ, o, row, x, pol_once);
      const float pr = ldg_f32_pol(p_row + row, pol_keep);
      a = fmaf(pr, x, a);
      if (HAS_VAL) b2 = fmaf(pr, x * x, b2);
    }
    a = warp_sum(a);
    if (HAS_VAL) b2 = warp_sum(b2);
    float4 acc[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int o = be.x + grp; o < be.y; o += 4 * G) {
      float4 tt[4]; float xs[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        xs[r] = 0.f; tt[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (o + r * G < be.y && act) {
          uint32_t row;
          load_occ<HAS_VAL, true>(occ, o + r * G, row, xs[r], pol_once);
          tt[r] = ldg128_pol(pxv + (size_t)row * ks + sub * 4, pol_keep);
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        acc[r].x = fmaf(tt[r].x, xs[r], acc[r].x); acc[r].y = fmaf(tt[r].y, xs[r], acc[r].y);
        acc[r].z = fmaf(tt[r].z, xs[r], acc[r].z); acc[r].w = fmaf(tt[r].w, xs[r], acc[r].w);
      }
    }
    float4 hg = make_float4((acc[0].x + acc[1].x) + (acc[2].x + acc[3].x), (acc[0].y + acc[1].y) + (acc[2].y + acc[3].y),
                            (acc[0].z + acc[1].z) + (acc[2].z + acc[3].z), (acc[0].w + acc[1].w) + (acc[2].w + acc[3].w));
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
      hg.x += __shfl_xor_sync(kFull, hg.x, o); hg.y += __shfl_xor_sync(kFull, hg.y, o);
      hg.z += __shfl_xor_sync(kFull, hg.z, o); hg.w += __shfl_xor_sync(kFull, hg.w, o);
    }
    if (grp == 0 && act) *reinterpret_cast<float4*>(ws.part + (size_t)c * ks + sub * 4) = hg;
    if (lane == 0) ws.part_s[c] = make_float2(a, HAS_VAL ? b2 : a);
  }
}

// the step's p*XV rows and p are dead once the update has read them: drop their L2 lines without writing them back,
// so that they (kept evict_last by the update) do not hold L2 into the next step and cost no DRAM write
__global__ void k_l2_discard(char* a, size_t na, char* b, size_t nb) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < na + nb; i += (size_t)gridDim.x * blockDim.x) {
    char* line = i < na ? a + i * 128 : b + (i - na) * 128;
    asm volatile("discard.global.L2 [%0], 128;" ::"l"(line) : "memory");
  }
}

inline int bits_for(size_t n) {
  int b = 1;
  while (b < 32 && ((size_t)1 << b) < n) ++b;
  return b;
}

inline int grid_for(size_t n, int threads, int cap) {
  size_t g = (n + threads - 1) / threads;
  if (g == 0) g = 1;
  return (int)(g < (size_t)cap ? g : (size_t)cap);
}
inline int grid_warps(size_t nwarps_needed, int warps_per_block, int cap) {
  size_t g = (nwarps_needed + warps_per_block - 1) / warps_per_block;
  if (g == 0) g = 1;
  return (int)(g < (size_t)cap ? g : (size_t)cap);
}

}  // namespace

namespace {
constexpr int kMaxDevices = 64;
// a device attribute of the current device, queried once per device (fallback: the H100 SXM's value)
int cached_attr(std::atomic<int>* cache, cudaDeviceAttr attr, int fallback) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, attr, dev) != cudaSuccess || n <= 0) n = fallback;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
}  // namespace

int num_sms() {
  static std::atomic<int> cache[kMaxDevices];
  return cached_attr(cache, cudaDevAttrMultiProcessorCount, 132);
}

size_t l2_bytes() {
  static std::atomic<int> cache[kMaxDevices];
  return (size_t)cached_attr(cache, cudaDevAttrL2CacheSize, 50 << 20);
}

int launch_table_init(Table& t, unsigned seed, cudaStream_t s) {
  k_table_init<<<num_sms() * 8, 256, 0, s>>>(t.tab, t.cap, t.state, t.prog, seed);
  return 1;
}

int launch_table_rehash(const Table& old_t, const Table& new_t, cudaStream_t s) {
  k_table_rehash<<<num_sms() * 8, 256, 0, s>>>(old_t.tab, old_t.cap, new_t.tab, new_t.mask, 0);
  k_table_rehash<<<num_sms() * 8, 256, 0, s>>>(old_t.tab, old_t.cap, new_t.tab, new_t.mask, 1);
  return 2;
}

int launch_table_insert(const Entry* src, uint64_t n, const Table& t, cudaStream_t s) {
  if (n == 0) return 0;
  k_table_rehash<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>(src, n, t.tab, t.mask, 1);
  return 1;
}

int launch_lookup(Table& t, const uint64_t* keys, size_t n, const unsigned long long* dn, bool insert,
                  int* slot_out, float* w_out, int* vrow_out, int2* wv_out, cudaStream_t s) {
  if (n == 0) return 0;
  const int grid = grid_for(n, 256 * kLookupIlp, num_sms() * 64);
  if (insert) k_lookup<true><<<grid, 256, 0, s>>>(t, keys, n, dn, slot_out, w_out, vrow_out, wv_out);
  else        k_lookup<false><<<grid, 256, 0, s>>>(t, keys, n, dn, slot_out, w_out, vrow_out, wv_out);
  return 1;
}

size_t scan_tmp_bytes(size_t n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const int*)nullptr, (int*)nullptr, (int)(n ? n : 1));
  return bytes;
}

size_t sort_tmp_bytes(size_t n) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const float*)nullptr, (float*)nullptr,
                                  (const float*)nullptr, (float*)nullptr, (int)(n ? n : 1));
  return bytes;
}

int launch_initv(Table& t, const Params& p, const int* slot, size_t n, const unsigned long long* dn, int* flags,
                 int* ws, cudaStream_t s) {
  if (n == 0 || p.V_dim == 0) return 0;
  const int grid = grid_warps((n + 31) / 32, 8, num_sms() * 8);
  cudaMemsetAsync(ws, 0, 16, s);
  k_flag_tiles<<<grid, 256, 0, s>>>(flags, n, dn, ws);
  k_tile_scan<<<1, 1024, 0, s>>>(ws, n, dn);
  k_initv<<<grid, 256, 0, s>>>(t, p, slot, n, dn, flags, ws);
  k_initv_finalize<<<1, 32, 0, s>>>(t, p, ws);
  return 4;
}

int launch_feacnt(Table& t, const Params& p, const int* slot, size_t n, const unsigned long long* dn,
                  const float* cnt, const int* cnt_cols, int* flags, int* ws, cudaStream_t s) {
  if (n == 0) return 0;
  k_feacnt<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>(t, p, slot, n, dn, cnt, cnt_cols, flags);
  return 1 + launch_initv(t, p, slot, n, dn, flags, ws, s);
}

int launch_lens_scan(const int* lens, size_t n, int* pos, void* cub_tmp, size_t cub_bytes, cudaStream_t s) {
  if (n == 0) return 0;
  cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, lens, pos, (int)n, s);
  return 2;
}

int launch_pack_ragged(Table& t, const Params& p, const int* slot, size_t n, int* lens, int* pos, float* vals,
                       unsigned long long* nvals_out, void* cub_tmp, size_t cub_bytes, cudaStream_t s) {
  if (n == 0) return 0;
  k_lens<<<(int)((n + 255) / 256), 256, 0, s>>>(t, p, slot, n, lens);
  cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, lens, pos, (int)n, s);
  k_pack_ragged<<<grid_warps(n, 8, num_sms() * 8), 256, 0, s>>>(t, p, slot, n, lens, pos, vals, nvals_out);
  return 4;
}

int launch_gather_rows(Table& t, const int* slot, size_t n, float* w_out, int* hasv_out, int* hasv_out2,
                       float* V_out, cudaStream_t s) {
  if (n == 0) return 0;
  k_gather_rows<<<grid_warps((n + 31) / 32, 8, num_sms() * 8), 256, 0, s>>>(t, slot, n, w_out, hasv_out, hasv_out2, V_out);
  return 1;
}

int launch_update_dense(Table& t, const Params& p, const int* slot, const int* pull_vrow, int vrow_is_flag,
                        size_t n, const float* gw, const float* gxxp, const float* gV, int* flags,
                        int acc_pen, int xxp_mode, cudaStream_t s) {
  if (n == 0) return 0;
  // the specialised kernel at the exact widths only (the atomic scatter's update)
  const int nl = with_lane_width(p.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (p.V_dim != K) return -1;
    k_update_fast<K><<<grid_warps((n + (32 / (K / 4)) - 1) / (32 / (K / 4)), 8, num_sms() * 8), 256, 0, s>>>(
        t, p, slot, pull_vrow, vrow_is_flag, n, gw, gxxp, gV, flags, acc_pen, xxp_mode);
    return 1;
  });
  if (nl > 0) return nl;
  k_update_dense_generic<<<grid_warps(n, 8, num_sms() * 8), 256, 0, s>>>(t, p, slot, pull_vrow, vrow_is_flag, n, gw,
                                                                  gxxp, gV, flags, acc_pen, xxp_mode);
  return 1;
}

int launch_update_ragged(Table& t, const Params& p, const int* slot, size_t n, const float* grads,
                         const int* lens_or_null, const int* pos, int* flags, cudaStream_t s) {
  if (n == 0) return 0;
  k_update_ragged<<<grid_warps(n, 8, num_sms() * 8), 256, 0, s>>>(t, p, slot, n, grads, lens_or_null, pos, flags);
  return 1;
}

int launch_penalty(const Params& p, DevProgress* prog, const float* w_arr, const int* vrow, const float* V,
                   int ks, int dense, size_t n, const unsigned long long* dn, cudaStream_t s) {
  if (n == 0) return 0;
  k_penalty<<<grid_warps(n, 8, num_sms() * 8), 256, 0, s>>>(p, prog, w_arr, vrow, V, ks, dense, n, dn);
  return 1;
}

int launch_pull_view(Table& t, const int* slot, size_t n, const unsigned long long* dn, float* w_out,
                     int* vrow_out, int2* wv_out, cudaStream_t s) {
  if (n == 0) return 0;
  k_pull_view<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>(t, slot, n, dn, w_out, vrow_out, wv_out);
  return 1;
}

int launch_evaluate(const float* label, const float* pred, size_t n, double* out, cudaStream_t s) {
  if (n == 0) return 0;
  k_evaluate<<<grid_for(n, 256, num_sms() * 4), 256, 0, s>>>(label, pred, n, out);
  return 1;
}

int launch_auc(const float* label, const float* pred, size_t n, float* key_tmp2, float* val_tmp2, void* cub_tmp,
               size_t cub_bytes, double* out_add, const unsigned long long* dev_nkeys, cudaStream_t s) {
  if (n == 0) return 0;
  // stable ascending radix sort by pred: ties keep original row order
  if (cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, pred, key_tmp2, label, val_tmp2, (int)n, 0, 32, s) != cudaSuccess)
    return -1;
  k_auc_area<<<1, 1024, 0, s>>>(val_tmp2, n, out_add, dev_nkeys);
  return 4;
}


size_t csc_tmp_bytes(size_t nnz, bool valued) {
  size_t bytes = 0;
  const int n = (int)(nnz ? nnz : 1);
  if (valued)
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);
  else
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, n);
  return bytes;
}

int launch_csc_build(const uint32_t* lidx, const void* occ, bool valued, size_t nnz, size_t nkeys,
                     uint32_t* lidx_sorted, void* occ_sorted, int* col_start, int* col_end, void* cub_tmp,
                     size_t cub_bytes, DevProgress* prog, cudaStream_t s) {
  if (nkeys == 0) return 0;
  if (cudaMemsetAsync(col_start, 0, nkeys * sizeof(int), s) != cudaSuccess) return -1;
  if (cudaMemsetAsync(col_end, 0, nkeys * sizeof(int), s) != cudaSuccess) return -1;
  if (nnz == 0) return 0;
  // all 32 bits take part when an index could be out of range; the common case sorts ceil(log2 nkeys) bits and
  // k_col_bounds verifies the result (sortedness + range)
  const int eb = bits_for(nkeys);
  cudaError_t e;
  if (valued)
    e = cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, lidx, lidx_sorted,
                                        reinterpret_cast<const unsigned long long*>(occ),
                                        reinterpret_cast<unsigned long long*>(occ_sorted), (int)nnz, 0, eb, s);
  else
    e = cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, lidx, lidx_sorted,
                                        reinterpret_cast<const uint32_t*>(occ),
                                        reinterpret_cast<uint32_t*>(occ_sorted), (int)nnz, 0, eb, s);
  if (e != cudaSuccess) return -1;
  k_col_bounds<<<(int)((nnz + 255) / 256), 256, 0, s>>>(lidx_sorted, nnz, nkeys, col_start, col_end, prog);
  return 2 + (eb + 7) / 8;   // histogram + one onesweep pass per 8 key bits + bounds
}

int launch_bwd_update(Table& t, const Params& p, const uint64_t* keys, int* slot, const int* pull_vrow, size_t n,
                      const unsigned long long* dn, const int* col_start, const int* col_end,
                      const void* occ_sorted, bool valued, const float* p_row, const float* pxv, int* flags,
                      int acc_pen, const ShardApply* shard, const HotPart* hot, int l2hint, cudaStream_t s) {
  if (n == 0) return 0;
  const unsigned long long* k64 = reinterpret_cast<const unsigned long long*>(keys);
  SegDst noseg;
  memset(&noseg, 0, sizeof(noseg));
  ShardApply sa;
  memset(&sa, 0, sizeof(sa));
  if (shard) sa = *shard;
  HotPart hp;
  memset(&hp, 0, sizeof(hp));
  if (hot) hp = *hot;
#define DFB_BU_(K, VAL, SRC, HINT, PAD, FIND)                                                                  \
  k_bwd_update<K, VAL, true, SRC, HINT, PAD, FIND><<<grid, 256, 0, s>>>(t, p, slot, pull_vrow, n, dn, col_start,     \
                                                             col_end, occ_sorted, p_row, pxv, flags, acc_pen, nullptr, \
                                                             nullptr, nullptr, noseg, sa, hp, k64, slot)
  // the single-GPU step: finding the keys (keys != nullptr; only with the L2 plan, which every batch too large for the
  // lookup has) or taking the slots of k_lookup
#define DFB_BU0_(K, PAD)                                                                                       \
  do {                                                                                                         \
    if (keys) {                                                                                                \
      if (!l2hint) return -1;                                                                                  \
      if (valued) DFB_BU_(K, true, 0, true, PAD, true); else DFB_BU_(K, false, 0, true, PAD, true);            \
    } else if (l2hint) {                                                                                       \
      if (valued) DFB_BU_(K, true, 0, true, PAD, false); else DFB_BU_(K, false, 0, true, PAD, false);          \
    } else {                                                                                                   \
      if (valued) DFB_BU_(K, true, 0, false, PAD, false); else DFB_BU_(K, false, 0, false, PAD, false);        \
    }                                                                                                          \
  } while (0)
  // one short-lived CTA per 256 keys, so that the higher-priority streams working on the NEXT step (localizer;
  // worker / lookup streams of the sharded store) get SM slots as CTAs retire -- a grid-stride grid holds every
  // slot until the kernel ends
  const int grid = grid_warps((n + 31) / 32, 8, 1 << 22);
  return with_lane_width(p.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (p.V_dim == K) {
      if (shard) { if (valued) DFB_BU_(K, true, 2, false, false, false); else DFB_BU_(K, false, 2, false, false, false); }
      else DFB_BU0_(K, false);
    } else {
      if (shard) {
        if (!valued) return -1;         // the owners' wire format is always valued (kernels_shard.cu)
        DFB_BU_(K, true, 2, false, true, false);
      }
      else DFB_BU0_(K, true);
    }
    return 1;
  });
#undef DFB_BU0_
#undef DFB_BU_
}

int launch_l2_discard(void* a, size_t a_bytes, void* b, size_t b_bytes, cudaStream_t s) {
  const size_t na = a_bytes / 128, nb = b_bytes / 128;      // whole lines only: the buffers are 256-byte aligned
  if (na + nb == 0) return 0;
  k_l2_discard<<<grid_for(na + nb, 256, num_sms() * 4), 256, 0, s>>>(static_cast<char*>(a), na, static_cast<char*>(b), nb);
  return 1;
}

int launch_hot_prereduce(int V_dim, size_t n, const unsigned long long* dn, const int* col_start, const int* col_end,
                         const void* occ_sorted, bool valued, const float* p_row, const float* pxv, int split,
                         const HotWs& ws, HotPart* hp, int l2hint, cudaStream_t s) {
  memset(hp, 0, sizeof(*hp));
  if (n == 0 || split <= 0) return 0;
  const int chunk = split / 2 > 32 ? split / 2 : 32;
  cudaMemsetAsync(ws.counter, 0, sizeof(unsigned long long), s);
  k_hot_find<<<grid_for(n, 256, num_sms() * 8), 256, 0, s>>>(col_start, col_end, n, dn, split, chunk, ws);
  const int grid = num_sms() * 4;
  const int ks = (V_dim + 3) / 4 * 4;
  const int nl = with_lane_width(V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (V_dim == K) {
      if (valued) k_hot_reduce<K, true><<<grid, 256, 0, s>>>(occ_sorted, p_row, pxv, ws, l2hint, ks);
      else        k_hot_reduce<K, false><<<grid, 256, 0, s>>>(occ_sorted, p_row, pxv, ws, l2hint, ks);
    } else {
      if (valued) k_hot_reduce<K, true, true><<<grid, 256, 0, s>>>(occ_sorted, p_row, pxv, ws, l2hint, ks);
      else        k_hot_reduce<K, false, true><<<grid, 256, 0, s>>>(occ_sorted, p_row, pxv, ws, l2hint, ks);
    }
    return 1;
  });
  if (nl < 0) return 0;
  hp->hotmap = ws.hotmap; hp->part = ws.part; hp->part_s = ws.part_s; hp->split = split; hp->chunk = chunk;
  return 2;
}

int launch_bwd_dense(const Params& p, DevProgress* prog, int ks, const float* w_pulled, const int* hasv, size_t n,
                     const int* col_start, const int* col_end, const void* occ_sorted, bool valued,
                     const float* p_row, const float* pxv, float* gw_out, const float* V_pulled, float* gV_out,
                     int acc_pen, const SegDst* seg, cudaStream_t s) {
  if (n == 0) return 0;
  if (ks != p.V_dim) return -1;
  Table t;
  t.prog = prog;
  SegDst sd;
  if (seg) sd = *seg; else memset(&sd, 0, sizeof(sd));
  const int* w_alias = reinterpret_cast<const int*>(w_pulled);
  ShardApply nosa;
  memset(&nosa, 0, sizeof(nosa));
  HotPart nohp;
  memset(&nohp, 0, sizeof(nohp));
  return with_lane_width(p.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (p.V_dim != K) return -1;        // exact widths only
    const int grid = grid_warps((n + 31) / 32, 8, num_sms() * 8);
    if (valued) k_bwd_update<K, true, false><<<grid, 256, 0, s>>>(t, p, w_alias, hasv, n, nullptr, col_start, col_end,
                   occ_sorted, p_row, pxv, nullptr, acc_pen, gw_out, V_pulled, gV_out, sd, nosa, nohp, nullptr, nullptr);
    else k_bwd_update<K, false, false><<<grid, 256, 0, s>>>(t, p, w_alias, hasv, n, nullptr, col_start, col_end,
                   occ_sorted, p_row, pxv, nullptr, acc_pen, gw_out, V_pulled, gV_out, sd, nosa, nohp, nullptr, nullptr);
    return 1;
  });
}

// owner side of Push(kGradient) for the specialised V_dims: same phase A/B kernel, gradient read
// from the dense rows a worker sent
int launch_update_pushed(Table& t, const Params& p, const int* slot, const int* hasv, size_t n, const float* gw,
                         const float* gV, int* flags, cudaStream_t s) {
  if (n == 0) return 0;
  SegDst noseg;
  memset(&noseg, 0, sizeof(noseg));
  ShardApply nosa;
  memset(&nosa, 0, sizeof(nosa));
  HotPart nohp;
  memset(&nohp, 0, sizeof(nohp));
  return with_lane_width(p.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (p.V_dim != K) return -1;        // exact widths only
    const int grid = grid_warps((n + 31) / 32, 8, num_sms() * 8);
    k_bwd_update<K, false, true, 1><<<grid, 256, 0, s>>>(t, p, slot, hasv, n, nullptr, nullptr, nullptr, nullptr, gw,
                                                          gV, flags, 0, nullptr, nullptr, nullptr, noseg, nosa, nohp,
                                                          nullptr, nullptr);
    return 1;
  });
}

int launch_restore(Table& t, const uint64_t* keys, size_t n, const float* scal, const int* vrow,
                   unsigned long long n_vrows, unsigned seed, cudaStream_t s) {
  if (n) k_restore<<<(int)((n + 255) / 256), 256, 0, s>>>(t, keys, n, scal, vrow);
  k_set_state<<<1, 1, 0, s>>>(t.state, (unsigned long long)n, n_vrows, seed);
  return 2;
}

int launch_read_entries(Table& t, const int* slot, size_t n, float* scal, int* hasv, float* V, float* cg,
                        int k, cudaStream_t s) {
  if (n == 0) return 0;
  k_read_entries<<<(int)((n + 127) / 128), 128, 0, s>>>(t, slot, n, scal, hasv, V, cg, k);
  return 1;
}

}  // namespace dfb
