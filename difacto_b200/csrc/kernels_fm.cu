// difacto_b200/csrc/kernels_fm.cu -- FM forward (+ fused backward scatter) for sm_90a.
//
// Restates, for the GPU, FMLoss::Predict (src/loss/fm_loss.h:67-119: SpMV::Times,
// 2x SpMM::Times, row reduce, clamp), Loss::Evaluate (include/difacto/loss.h:57-66) and
// FMLoss::CalcGrad (fm_loss.h:148-199: p = -y/(1+exp(y pred)), SpMV::TransTimes,
// SpMM::TransTimes) of the reference as ONE pass per CSR row:
//
//   phase 1  gather the k-wide V rows of the row's active features (coalesced 16-byte lanes,
//            UNR independent loads in flight per lane), accumulate XV = sum x V and
//            sum (x V)^2 in registers, warp-shuffle reduce over k -> pred, logloss
//   phase 2  (training) p from the clamped pred, then scatter x p XV into the per-key gradient
//            rows with vector fp32 reductions (red.global.add.v4.f32), x p into grad_w and
//            x^2 p into XXp.  The "- V_j XXp_j" term (fm_loss.h:181-188) needs V once per
//            unique key, not per nnz, so it is applied where V is read anyway: in the fused
//            FTRL/AdaGrad kernel (kernels_table.cu) or in grad_finalize below.
//
// The whole path is HBM-bound (about 0.5 FLOP/B): no tensor cores on purpose.
#include "dfb_device.cuh"

#include <math.h>
#include <string.h>

namespace dfb {

namespace {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float4 ldg128(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
               "f"(d)
               : "memory");
}

__device__ __forceinline__ void red_add(float* p, float a) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// logloss of one row: log(1 + exp(-y pred)), y = label > 0 ? 1 : -1 (loss.h:62-63)
__device__ __forceinline__ float row_logloss(float label, float pred) {
  float y = label > 0.f ? 1.f : -1.f;
  return logf(1.f + expf(-y * pred));
}

// p = -y / (1 + exp(y pred))  (fm_loss.h:157-161)
__device__ __forceinline__ float row_p(float label, float pred) {
  float y = label > 0.f ? 1.f : -1.f;
  return -y / (1.f + expf(y * pred));
}

// true when the GPU localizer dropped this batch (FmBatch::dev_nkeys): its ranks index nothing, so the kernel must
// return before it reads them.  Block-uniform.  raise: this kernel reports the drop (one per forward launch).
__device__ __forceinline__ bool batch_dropped(const FmBatch& b, bool raise) {
  if (b.dev_nkeys == nullptr || *b.dev_nkeys != 0ULL) return false;
  if (raise && blockIdx.x == 0 && threadIdx.x == 0 && b.prog) raise_err(b.prog, kErrIdRange);
  return true;
}

// the raw-id forward: {w, V-row index} of the entry of a raw id, found the way the validation step's find-only
// k_lookup finds it (the whole 32-byte entry with the first probe, the probe loop only on a collision).  A missing
// key reads as w = 0 and no V row, what that lookup leaves in the pulled view.
__device__ __forceinline__ void probe_raw(const FmView& v, unsigned long long id, float& w, int& vr) {
  const unsigned long long key = raw_key(id);
  const uint64_t h = hash64(key) & v.tab_mask;
  const Entry256 e = load_entry(v.tab + h);
  if (e.key == key) {
    w = e.w(); vr = e.vrow();
  } else if (e.key != kEmptyKey) {
    Table t;
    t.tab = const_cast<Entry*>(v.tab); t.mask = v.tab_mask;
    const int s = table_find<false>(t, key, h);
    if (s >= 0) { w = v.tab[s].w; vr = v.tab[s].vrow; }
  }
}

// a lane's 4 columns of a V row, at element offset `at` from the rows' base: one 16-byte load of fp32 elements, or
// (BF16: a scoring-only engine's 2-byte rows) one 8-byte load widened to fp32
template <bool BF16>
__device__ __forceinline__ float4 load_vrow4(const float* base, long long at, uint64_t pol) {
  if constexpr (BF16) return ldg_bf16x4_pol(reinterpret_cast<const unsigned short*>(base) + at, pol);
  else return ldg128_pol(base + at, pol);
}

__device__ __forceinline__ void block_add_loss(float loss_acc, size_t nrows, DevProgress* prog) {
  __shared__ float red_s[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // lane 0 of each warp holds that warp's partial
  if (lane == 0) red_s[wid] = loss_acc;
  __syncthreads();
  if (wid == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    float v = lane < nw ? red_s[lane] : 0.f;
    v = warp_sum(v);
    if (lane == 0 && prog) {
      atomicAdd(&prog->loss, (double)v);
      if (blockIdx.x == 0) atomicAdd(&prog->nrows, (unsigned long long)nrows);
    }
  }
}

// ---------------------------------------------------------------------------------------
// fast path: K in {8,16,32,64,128}, 16-byte aligned rows
// ---------------------------------------------------------------------------------------
// PAD (V_dim < K, see fast_lane_width): the rows have stride ks = V_dim rounded up to 4, lanes whose float4 starts at
// or beyond ks load and store nothing, and V_dim 0 leaves the prediction unclamped (fm_loss.h:77)
// MODE 0: predict only.  MODE 1: training with fp32 red.global scatter into dense gradient rows.
// MODE 2: training, "emit": writes p_i, p_i*XV_i and the (row[,x]) payload of every nnz so that
//         the gradient can be reduced per key without atomics (kernels_table.cu: k_bwd_update).
// MODE 3: owner side of the fused sharded store: partial sums of every worker's rows over this owner's
//         key segment, stored into the workers' mailboxes (see PartArgs).
// RAW (MODE 0 and 2): the nonzeros carry raw feature ids (b.ids); the metadata of each is probed in the table
//         (probe_raw) instead of being read from a pulled view through a localized index.  Everything after the
//         metadata is the same code, so the predictions (and p, p*XV) are bit-identical to those of the steps that
//         look the keys up first.  MODE 2 needs the CSC view of the GPU localizer (b.occ_row == nullptr).
#ifndef DFB_FM_MINBLOCKS
#define DFB_FM_MINBLOCKS 4
#endif
// The raw-id kernels use the same rule although their metadata chain is longer: prefetching at every K made the K >= 32
// instantiations spill 130-220 bytes and the flagship predict forward (K = 64) 17 % slower, 0.703 against 0.599 ms
// (H100 SXM, 700 W).
#ifndef DFB_FM_PF_MAXK
#define DFB_FM_PF_MAXK 16       // metadata prefetch (one chunk ahead) for V_dim <= this
#endif
#ifndef DFB_FM_MINBLOCKS32
#define DFB_FM_MINBLOCKS32 DFB_FM_MINBLOCKS     // V_dim = 32 (tuning builds: 3 removes its ~130-byte spills)
#endif
template <int K, int MODE, bool HAS_VAL, bool PAD = false, bool RAW = false, bool BF16 = false>
__global__ void __launch_bounds__(256, K == 32 ? DFB_FM_MINBLOCKS32 : DFB_FM_MINBLOCKS) k_fm_fast(FmBatch b, FmView v, PartArgs pa) {
  constexpr bool TRAIN = MODE == 1;
  static_assert(!BF16 || (RAW && MODE == 0), "bf16 rows: the raw-id predict step only");
  static_assert(!(PAD && TRAIN), "the atomic scatter runs the exact widths only");
  static_assert(!RAW || MODE == 0 || MODE == 2, "raw ids: predict and emit only");
  constexpr int LPR = K / 4;                 // lanes per V row, one float4 each
  constexpr int G = 32 / LPR;                // V rows fetched by one warp-wide load
  constexpr int UNR = (32 / G) < 8 ? (32 / G) : 8;   // independent loads in flight per lane
  constexpr bool PF = K <= DFB_FM_PF_MAXK;
  if (MODE != 3 && batch_dropped(b, true)) return;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR, grp = lane / LPR;
  const int ks = PAD ? (b.V_dim + 3) / 4 * 4 : K;
  const bool act = !PAD || sub * 4 < ks;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  float loss_acc = 0.f;
  const uint64_t pol_v = l2_policy(v.l2hint ? kL2EvictFirst : kL2Normal);
  const uint64_t pol_wv = l2_policy(v.wv_last ? kL2EvictLast : kL2Normal);
  const size_t total_rows = MODE == 3 ? (size_t)pa.nsrc * (size_t)pa.bcap : b.nrows;

  for (size_t vrow_id = warp0; vrow_id < total_rows; vrow_id += nwarps) {
    size_t row = vrow_id;
    const uint64_t* offp = b.offset;
    const uint32_t* idxp = b.index;
    const float* valp = b.value;
    const int2* wvp = v.wv;
    int src = 0;
    if (MODE == 3) {
      const int s0 = (int)(vrow_id / pa.bcap);
      row = vrow_id - (size_t)s0 * pa.bcap;
      src = s0 + pa.rot;
      if (src >= pa.nsrc) src -= pa.nsrc;
      if (row >= (size_t)shard_hdr_nrows(pa.s[src].hdr)) continue;
      offp = pa.s[src].rowptr; idxp = pa.s[src].ridx; valp = pa.s[src].rval; wvp = pa.s[src].wv;
    }
    const uint64_t o0 = offp[row], o1 = offp[row + 1];
    if ((MODE == 0 || MODE == 2) && b.long_nnz && o1 - o0 >= b.long_nnz) continue;   // k_fm_long's row
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc2 = 0.f, wsum = 0.f;

    // the per-nnz metadata {x, w, V-row index} of a 32-nnz chunk hangs on a dependent chain (index -> pulled view);
    // it is fetched one chunk ahead, so that chain overlaps the V-row gathers of the current chunk
    auto load_meta = [&](uint64_t c, float& x, float& w, int& vr) {
      const uint64_t j = c + lane;
      x = 0.f; w = 0.f; vr = -1;
      if (RAW && j < o1) {
        const unsigned long long id = __ldg(reinterpret_cast<const unsigned long long*>(b.ids) + j);
        x = HAS_VAL ? __ldg(valp + j) : 1.f;
        probe_raw(v, id, w, vr);
      } else if (j < o1) {
        const uint32_t u = __ldg(idxp + j);
        x = HAS_VAL ? __ldg(valp + j) : 1.f;
        if (wvp) {
          const int2 t = ldg64_pol(wvp + u, pol_wv);
          w = __int_as_float(t.x);
          vr = t.y;
        } else {
          const int wp = v.w_pos ? __ldg(v.w_pos + u) : (int)u;
          w = wp >= 0 ? __ldg(v.wbase + wp) : 0.f;
          vr = __ldg(v.v_pos + u);
          if (v.dense && vr >= 0) vr = (int)u;
        }
        if (MODE == 2 && b.occ_row != nullptr) {   // nullptr: the CSC view already exists (GPU localizer)
          if (HAS_VAL) b.occ_rowx[j] = ((unsigned long long)row << 32) | (unsigned long long)__float_as_uint(x);
          else b.occ_row[j] = (uint32_t)row;
        }
      }
    };
    float x_n = 0.f, w_n = 0.f;
    int vr_n = -1;
    if (PF) load_meta(o0, x_n, w_n, vr_n);
    for (uint64_t c = o0; c < o1; c += 32) {
      float x, w;
      int vr;
      if (PF) {
        x = x_n; w = w_n; vr = vr_n;
        if (c + 32 < o1) load_meta(c + 32, x_n, w_n, vr_n);
      } else {
        load_meta(c, x, w, vr);
      }
      wsum = fmaf(x, w, wsum);
      const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
      for (int t0 = 0; t0 < cnt; t0 += G * UNR) {
        float4 vv[UNR];
        float xs[UNR];
#pragma unroll
        for (int q = 0; q < UNR; ++q) {
          const int t = t0 + q * G + grp;
          const int vr_t = __shfl_sync(kFull, vr, t & 31);
          const float x_t = __shfl_sync(kFull, x, t & 31);
          const bool ok = (t < cnt) && (vr_t >= 0) && act;
          xs[q] = ok ? x_t : 0.f;
          vv[q] = ok ? load_vrow4<BF16>(v.vbase, (long long)vr_t * v.vstride + sub * 4, pol_v)
                     : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int q = 0; q < UNR; ++q) {
          const float a0 = xs[q] * vv[q].x, a1 = xs[q] * vv[q].y;
          const float a2 = xs[q] * vv[q].z, a3 = xs[q] * vv[q].w;
          xv.x += a0; xv.y += a1; xv.z += a2; xv.w += a3;
          acc2 = fmaf(a0, a0, acc2); acc2 = fmaf(a1, a1, acc2);
          acc2 = fmaf(a2, a2, acc2); acc2 = fmaf(a3, a3, acc2);
        }
      }
    }
    // combine the G row-groups: afterwards every group holds the full XV for its 4 dims
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
      xv.x += __shfl_xor_sync(kFull, xv.x, o);
      xv.y += __shfl_xor_sync(kFull, xv.y, o);
      xv.z += __shfl_xor_sync(kFull, xv.z, o);
      xv.w += __shfl_xor_sync(kFull, xv.w, o);
    }
    acc2 = warp_sum(acc2);
    wsum = warp_sum(wsum);
    if (MODE == 3) {
      // ||XV||^2 is not linear in the rows: the worker squares the SUM of the owners' partials
      if (grp == 0 && act) *reinterpret_cast<float4*>(pa.s[src].out_xv + row * (size_t)ks + sub * 4) = xv;
      if (lane == 0) pa.s[src].out_sc[row] = make_float2(acc2, wsum);
      continue;
    }
    float s1 = grp == 0 ? (xv.x * xv.x + xv.y * xv.y + xv.z * xv.z + xv.w * xv.w) : 0.f;
    s1 = warp_sum(s1);
    float pred = (b.pred_acc ? b.pred_io[row] : 0.f) + wsum;
    pred += 0.5f * (s1 - acc2);
    if (!PAD || b.V_dim > 0) pred = pred > 20.f ? 20.f : (pred < -20.f ? -20.f : pred);   // fm_loss.h:77,118
    const float label = b.label ? __ldg(b.label + row) : 0.f;
    if (lane == 0) {
      if (b.pred_io) b.pred_io[row] = pred;
      if (b.label) loss_acc += row_logloss(label, pred);
    }
    if (MODE == 2) {
      const float p = row_p(label, pred);
      if (lane == 0) b.p_out[row] = p;
      // XV_ *= p (fm_loss.h:191-195), one coalesced 4ks-byte row
      if (grp == 0 && act)
        *reinterpret_cast<float4*>(b.pxv_out + row * (size_t)ks + sub * 4) =
            make_float4(p * xv.x, p * xv.y, p * xv.z, p * xv.w);
    }

    if (TRAIN) {
      const float p = row_p(label, b.pred_in ? __ldg(b.pred_in + row) : pred);
      const float4 gx = make_float4(p * xv.x, p * xv.y, p * xv.z, p * xv.w);
      for (uint64_t c = o0; c < o1; c += 32) {
        const uint64_t j = c + lane;
        const bool valid = j < o1;
        uint32_t u = 0;
        float x = 0.f;
        int vr = -1;
        if (valid) {
          u = __ldg(b.index + j);
          x = HAS_VAL ? __ldg(b.value + j) : 1.f;
          vr = __ldg(v.v_pos + u);
          const int gp = v.gw_pos ? __ldg(v.gw_pos + u) : (int)u;
          if (gp >= 0) red_add(v.gwbase + gp, x * p);
          if (HAS_VAL && vr >= 0) red_add(v.gxxp + u, x * x * p);
        }
        const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
        for (int t0 = 0; t0 < cnt; t0 += G) {
          const int t = t0 + grp;
          const int vr_t = __shfl_sync(kFull, vr, t & 31);
          const float x_t = __shfl_sync(kFull, x, t & 31);
          const uint32_t u_t = __shfl_sync(kFull, u, t & 31);
          if (t < cnt && vr_t >= 0) {
            const long long r = v.gv_pos ? (long long)__ldg(v.gv_pos + u_t) : (long long)u_t;
            red_add_v4(v.gvbase + r * v.gvstride + sub * 4, x_t * gx.x, x_t * gx.y, x_t * gx.z,
                       x_t * gx.w);
          }
        }
      }
    }
  }
  if (MODE != 3) block_add_loss(loss_acc, b.nrows, b.prog);
}

// ---------------------------------------------------------------------------------------
// long rows (gisette: ~5000 nonzeros per example): one CTA per row.  A single warp would walk such a row as
// ~nnz/16 dependent gather rounds with 32 lanes of loads in flight; here the 8 warps of a CTA take the row's
// 32-nnz chunks round-robin, and their partial (XV, sum (xV)^2, sum xw) are added in warp order through shared
// memory (fixed order: bit-reproducible).  Rows shorter than b.long_nnz are k_fm_fast's.  MODE 0 / 2 as above.
// ---------------------------------------------------------------------------------------
constexpr int kLongWarps = 8;

template <int K, int MODE, bool HAS_VAL, bool PAD = false, bool RAW = false, bool BF16 = false>
__global__ void __launch_bounds__(kLongWarps * 32) k_fm_long(FmBatch b, FmView v, int scan_rows) {
  static_assert(!RAW || MODE == 0 || MODE == 2, "raw ids: predict and emit only");
  static_assert(!BF16 || (RAW && MODE == 0), "bf16 rows: the raw-id predict step only");
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  constexpr int UNR = (32 / G) < 8 ? (32 / G) : 8;
  __shared__ float4 s_xv[kLongWarps][LPR];
  __shared__ float2 s_sc[kLongWarps];
  if (batch_dropped(b, false)) return;                // k_fm_fast reports it
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  const int ks = PAD ? (b.V_dim + 3) / 4 * 4 : K;
  const bool act = !PAD || sub * 4 < ks;
  const uint64_t pol_v = l2_policy(v.l2hint ? kL2EvictFirst : kL2Normal);
  const uint64_t pol_wv = l2_policy(v.wv_last ? kL2EvictLast : kL2Normal);
  float loss_acc = 0.f;                       // thread 0 only

  // a CTA looks at scan_rows (<= 256, one per thread) row lengths at a time: with many rows per CTA the scan is one
  // coalesced load (and almost always finds nothing); with few rows (a batch of long rows only) scan_rows is 1 and
  // every CTA gets its own row
  __shared__ unsigned char s_long[kLongWarps * 32];
  for (size_t base = (size_t)blockIdx.x * scan_rows; base < b.nrows; base += (size_t)gridDim.x * scan_rows) {
    const size_t mine = base + threadIdx.x;
    bool is_long = false;
    if ((int)threadIdx.x < scan_rows && mine < b.nrows) is_long = b.offset[mine + 1] - b.offset[mine] >= b.long_nnz;
    s_long[threadIdx.x] = is_long ? 1 : 0;
    if (!__syncthreads_or(is_long)) continue;
    for (int r = 0; r < scan_rows; ++r) {                // in row order (the loss sum stays reproducible)
      if (!s_long[r]) continue;                          // CTA-uniform
      const size_t row = base + r;
      const uint64_t o0 = b.offset[row], o1 = b.offset[row + 1];
      float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
      float acc2 = 0.f, wsum = 0.f;
      for (uint64_t c = o0 + 32u * wid; c < o1; c += 32u * kLongWarps) {
        const uint64_t j = c + lane;
        float x = 0.f, w = 0.f;
        int vr = -1;
        if (RAW && j < o1) {
          const unsigned long long id = __ldg(reinterpret_cast<const unsigned long long*>(b.ids) + j);
          x = HAS_VAL ? __ldg(b.value + j) : 1.f;
          probe_raw(v, id, w, vr);
        } else if (j < o1) {
          const uint32_t u = __ldg(b.index + j);
          x = HAS_VAL ? __ldg(b.value + j) : 1.f;
          if (v.wv) {
            const int2 t = ldg64_pol(v.wv + u, pol_wv);
            w = __int_as_float(t.x);
            vr = t.y;
          } else {
            const int wp = v.w_pos ? __ldg(v.w_pos + u) : (int)u;
            w = wp >= 0 ? __ldg(v.wbase + wp) : 0.f;
            vr = __ldg(v.v_pos + u);
            if (v.dense && vr >= 0) vr = (int)u;
          }
          if (MODE == 2 && b.occ_row != nullptr) {
            if (HAS_VAL) b.occ_rowx[j] = ((unsigned long long)row << 32) | (unsigned long long)__float_as_uint(x);
            else b.occ_row[j] = (uint32_t)row;
          }
        }
        wsum = fmaf(x, w, wsum);
        const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
        for (int t0 = 0; t0 < cnt; t0 += G * UNR) {
          float4 vv[UNR];
          float xs[UNR];
  #pragma unroll
          for (int q = 0; q < UNR; ++q) {
            const int t = t0 + q * G + grp;
            const int vr_t = __shfl_sync(kFull, vr, t & 31);
            const float x_t = __shfl_sync(kFull, x, t & 31);
            const bool ok = (t < cnt) && (vr_t >= 0) && act;
            xs[q] = ok ? x_t : 0.f;
            vv[q] = ok ? load_vrow4<BF16>(v.vbase, (long long)vr_t * v.vstride + sub * 4, pol_v)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
          }
  #pragma unroll
          for (int q = 0; q < UNR; ++q) {
            const float a0 = xs[q] * vv[q].x, a1 = xs[q] * vv[q].y;
            const float a2 = xs[q] * vv[q].z, a3 = xs[q] * vv[q].w;
            xv.x += a0; xv.y += a1; xv.z += a2; xv.w += a3;
            acc2 = fmaf(a0, a0, acc2); acc2 = fmaf(a1, a1, acc2);
            acc2 = fmaf(a2, a2, acc2); acc2 = fmaf(a3, a3, acc2);
          }
        }
      }
  #pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        xv.x += __shfl_xor_sync(kFull, xv.x, o);
        xv.y += __shfl_xor_sync(kFull, xv.y, o);
        xv.z += __shfl_xor_sync(kFull, xv.z, o);
        xv.w += __shfl_xor_sync(kFull, xv.w, o);
      }
      acc2 = warp_sum(acc2);
      wsum = warp_sum(wsum);
      if (grp == 0) s_xv[wid][sub] = xv;
      if (lane == 0) s_sc[wid] = make_float2(acc2, wsum);
      __syncthreads();
      if (wid == 0) {
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        float a2 = 0.f, ws = 0.f;
  #pragma unroll
        for (int q = 0; q < kLongWarps; ++q) {
          const float4 e = s_xv[q][sub];
          t.x += e.x; t.y += e.y; t.z += e.z; t.w += e.w;
          a2 += s_sc[q].x; ws += s_sc[q].y;
        }
        float s1 = grp == 0 ? (t.x * t.x + t.y * t.y + t.z * t.z + t.w * t.w) : 0.f;
        s1 = warp_sum(s1);
        float pred = (b.pred_acc ? b.pred_io[row] : 0.f) + ws;
        pred += 0.5f * (s1 - a2);
        if (!PAD || b.V_dim > 0) pred = pred > 20.f ? 20.f : (pred < -20.f ? -20.f : pred);   // fm_loss.h:77,118
        const float label = b.label ? __ldg(b.label + row) : 0.f;
        if (lane == 0) {
          if (b.pred_io) b.pred_io[row] = pred;
          if (b.label) loss_acc += row_logloss(label, pred);
        }
        if (MODE == 2) {
          const float p = row_p(label, pred);
          if (lane == 0) b.p_out[row] = p;
          if (grp == 0 && act)
            *reinterpret_cast<float4*>(b.pxv_out + row * (size_t)ks + sub * 4) = make_float4(p * t.x, p * t.y, p * t.z, p * t.w);
        }
      }
      __syncthreads();
    }
    __syncthreads();                                      // s_long is rewritten by the next scan
  }
  // (nrows is counted by k_fm_fast)
  if (threadIdx.x == 0 && b.prog && loss_acc != 0.f) atomicAdd(&b.prog->loss, (double)loss_acc);
}

// ---------------------------------------------------------------------------------------
// generic path: any V_dim (including 0), unaligned / ragged rows (the pulled layout of the
// reference: [w_0,(V_0..)][w_1,(V_1..)] with w_pos/V_pos, sgd_updater.cc:46-53)
// ---------------------------------------------------------------------------------------
template <bool TRAIN>
__global__ void __launch_bounds__(128) k_fm_generic(FmBatch b, FmView v) {
  extern __shared__ float smem[];
  if (batch_dropped(b, true)) return;
  const int k = b.V_dim;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float* xv = smem + (size_t)wid * k;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const bool has_val = b.value != nullptr;
  float loss_acc = 0.f;

  for (size_t row = warp0; row < b.nrows; row += nwarps) {
    const uint64_t o0 = b.offset[row], o1 = b.offset[row + 1];
    for (int l = lane; l < k; l += 32) xv[l] = 0.f;
    float acc2 = 0.f, wsum = 0.f;
    for (uint64_t c = o0; c < o1; c += 32) {
      const uint64_t j = c + lane;
      const bool valid = j < o1;
      uint32_t u = 0;
      float x = 0.f, w = 0.f;
      long long vr = -1;
      if (valid) {
        u = b.index[j];
        x = has_val ? b.value[j] : 1.f;
        const int wp = v.w_pos ? v.w_pos[u] : (int)u;
        w = wp >= 0 ? v.wbase[wp] : 0.f;
        if (k > 0 && v.v_pos) {
          vr = v.v_pos[u];
          if (v.dense && vr >= 0) vr = u;
        }
      }
      wsum = fmaf(x, w, wsum);
      if (k > 0) {
        const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
        for (int t = 0; t < cnt; ++t) {
          const long long vr_t = __shfl_sync(kFull, vr, t);
          const float x_t = __shfl_sync(kFull, x, t);
          if (vr_t < 0) continue;   // warp-uniform
          const float* rowp = v.vbase + vr_t * v.vstride;
          for (int l = lane; l < k; l += 32) {
            const float a = x_t * rowp[l];
            xv[l] += a;
            acc2 = fmaf(a, a, acc2);
          }
        }
      }
    }
    float pred = (b.pred_acc ? b.pred_io[row] : 0.f);
    wsum = warp_sum(wsum);
    pred += wsum;
    if (k > 0) {   // V_dim == 0 returns before the clamp (fm_loss.h:77)
      float s1 = 0.f;
      for (int l = lane; l < k; l += 32) s1 = fmaf(xv[l], xv[l], s1);
      s1 = warp_sum(s1);
      acc2 = warp_sum(acc2);
      pred += 0.5f * (s1 - acc2);
      pred = pred > 20.f ? 20.f : (pred < -20.f ? -20.f : pred);
    }
    const float label = b.label ? b.label[row] : 0.f;
    if (lane == 0) {
      if (b.pred_io) b.pred_io[row] = pred;
      if (b.label) loss_acc += row_logloss(label, pred);
    }
    if (TRAIN) {
      const float p = row_p(label, b.pred_in ? b.pred_in[row] : pred);
      for (uint64_t c = o0; c < o1; c += 32) {
        const uint64_t j = c + lane;
        const bool valid = j < o1;
        uint32_t u = 0;
        float x = 0.f;
        long long gr = -1;
        if (valid) {
          u = b.index[j];
          x = has_val ? b.value[j] : 1.f;
          const int gp = v.gw_pos ? v.gw_pos[u] : (int)u;
          if (gp >= 0) red_add(v.gwbase + gp, x * p);
          if (k > 0 && v.v_pos && v.v_pos[u] >= 0) {
            gr = v.gv_pos ? (long long)v.gv_pos[u] : (long long)u;
            if (v.gxxp) red_add(v.gxxp + u, (has_val ? x * x : 1.f) * p);
          }
        }
        if (k > 0) {
          const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
          for (int t = 0; t < cnt; ++t) {
            const long long gr_t = __shfl_sync(kFull, gr, t);
            const float x_t = __shfl_sync(kFull, x, t);
            if (gr_t < 0) continue;
            float* g = v.gvbase + gr_t * v.gvstride;
            const float xp = x_t * p;
            for (int l = lane; l < k; l += 32) red_add(g + l, xp * xv[l]);
          }
        }
      }
    }
  }
  block_add_loss(loss_acc, b.nrows, b.prog);
}

// grad_V -= diag(XXp) V for the ragged layout (fm_loss.h:181-188)
__global__ void k_grad_finalize(int k, size_t nkeys, const float* weights, const int* V_pos,
                                const float* xxp, float* grad) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t u = warp0; u < nkeys; u += nwarps) {
    const int p = V_pos[u];
    if (p < 0) continue;
    const float s = xxp[u];
    for (int l = lane; l < k; l += 32) grad[p + l] -= weights[p + l] * s;
  }
}

// dense pulled layout: gV[u][ks] -= V[u][ks] * xxp[u] for keys with a V row (fm_loss.h:181-188)
__global__ void k_grad_finalize_dense(int k, int ks, size_t nkeys, const int* hasv, const float* V,
                                      const float* xxp, float* gV) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t u = warp0; u < nkeys; u += nwarps) {
    if (hasv[u] < 0) continue;
    const float s = xxp[u];
    for (int l = lane; l < k; l += 32) gV[u * (size_t)ks + l] -= V[u * (size_t)ks + l] * s;
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// RAW: the raw-id kernels (launch_fm_raw): predict (MODE 0) or, in a training step, emit (MODE 2).
// BF16 (RAW predict only): the rows are a scoring-only engine's bf16 V rows
template <int K, bool PAD, bool RAW = false, bool BF16 = false>
int launch_fast_k(const FmBatch& b, const FmView& v, cudaStream_t s) {
  const int threads = 256;
  size_t need = (b.nrows + 7) / 8;
  int grid = (int)(need < (size_t)(num_sms() * 8) ? (need ? need : 1) : (size_t)(num_sms() * 8));
  const bool hv = b.value != nullptr;
  PartArgs pa;
  memset(&pa, 0, sizeof(pa));
  if constexpr (BF16) {
    if (b.train) return -1;
    if (hv) k_fm_fast<K, 0, true, PAD, true, true><<<grid, threads, 0, s>>>(b, v, pa);
    else    k_fm_fast<K, 0, false, PAD, true, true><<<grid, threads, 0, s>>>(b, v, pa);
  } else if constexpr (RAW) {
    if (b.train) {
      if (hv) k_fm_fast<K, 2, true, PAD, true><<<grid, threads, 0, s>>>(b, v, pa);
      else    k_fm_fast<K, 2, false, PAD, true><<<grid, threads, 0, s>>>(b, v, pa);
    } else {
      if (hv) k_fm_fast<K, 0, true, PAD, true><<<grid, threads, 0, s>>>(b, v, pa);
      else    k_fm_fast<K, 0, false, PAD, true><<<grid, threads, 0, s>>>(b, v, pa);
    }
  } else if (b.train && b.emit) {
    if (hv) k_fm_fast<K, 2, true, PAD><<<grid, threads, 0, s>>>(b, v, pa);
    else    k_fm_fast<K, 2, false, PAD><<<grid, threads, 0, s>>>(b, v, pa);
  } else if (b.train) {
    if constexpr (PAD) return -1;      // (launch_fm sends the atomic scatter to the generic kernel)
    else if (hv) k_fm_fast<K, 1, true><<<grid, threads, 0, s>>>(b, v, pa);
    else         k_fm_fast<K, 1, false><<<grid, threads, 0, s>>>(b, v, pa);
  } else {
    if (hv) k_fm_fast<K, 0, true, PAD><<<grid, threads, 0, s>>>(b, v, pa);
    else    k_fm_fast<K, 0, false, PAD><<<grid, threads, 0, s>>>(b, v, pa);
  }
  // rows of >= long_nnz nonzeros: one CTA each (the scan over the offsets costs ~1 us when there is none)
  if (b.long_nnz && (!b.train || b.emit) && (b.nnz_hint == 0 || b.nnz_hint >= b.long_nnz)) {
    const int lgrid = (int)(b.nrows < (size_t)(num_sms() * 4) ? b.nrows : (size_t)(num_sms() * 4));
    int scan = 1;
    while (scan < kLongWarps * 32 && (size_t)lgrid * scan * 2 <= b.nrows) scan *= 2;
    if constexpr (BF16) {
      if (hv) k_fm_long<K, 0, true, PAD, true, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
      else    k_fm_long<K, 0, false, PAD, true, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
    } else if constexpr (RAW) {
      if (b.train) {
        if (hv) k_fm_long<K, 2, true, PAD, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
        else    k_fm_long<K, 2, false, PAD, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
      } else {
        if (hv) k_fm_long<K, 0, true, PAD, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
        else    k_fm_long<K, 0, false, PAD, true><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
      }
    } else if (b.train) {
      if (hv) k_fm_long<K, 2, true, PAD><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
      else    k_fm_long<K, 2, false, PAD><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
    } else {
      if (hv) k_fm_long<K, 0, true, PAD><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
      else    k_fm_long<K, 0, false, PAD><<<lgrid, kLongWarps * 32, 0, s>>>(b, v, scan);
    }
    return 2;
  }
  return 1;
}

template <int K, bool PAD>
int launch_partial_k(int V_dim, bool valued, const FmView& v, const PartArgs& pa, cudaStream_t s) {
  FmBatch b;
  memset(&b, 0, sizeof(b));
  b.V_dim = V_dim;
  const int grid = num_sms() * 8;
  if constexpr (PAD) {
    if (!valued) return -1;       // the owners' wire format is always valued (kernels_shard.cu)
    k_fm_fast<K, 3, true, true><<<grid, 256, 0, s>>>(b, v, pa);
  } else {
    if (valued) k_fm_fast<K, 3, true><<<grid, 256, 0, s>>>(b, v, pa);
    else        k_fm_fast<K, 3, false><<<grid, 256, 0, s>>>(b, v, pa);
  }
  return 1;
}

}  // namespace

bool fm_fast_supported(int k) { return fast_lane_width(k) != 0; }

int launch_fm_partial(int V_dim, bool valued, const FmView& v, const PartArgs& pa, cudaStream_t s) {
  return with_lane_width(V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    return V_dim == K ? launch_partial_k<K, false>(V_dim, valued, v, pa, s)
                      : launch_partial_k<K, true>(V_dim, valued, v, pa, s);
  });
}

int launch_fm_raw(const FmBatch& b, const FmView& v, bool bf16_rows, cudaStream_t s) {
  // training: the emit mode over the CSC view the GPU localizer already wrote
  if (b.train && (bf16_rows || !b.emit || b.occ_row != nullptr || b.occ_rowx != nullptr)) return -1;
  if (!aligned16(v.vbase) || v.vstride % 4 != 0) return -1;
  return with_lane_width(b.V_dim, [&](auto kc) {
    constexpr int K = decltype(kc)::value;
    if (bf16_rows)
      return b.V_dim == K ? launch_fast_k<K, false, true, true>(b, v, s) : launch_fast_k<K, true, true, true>(b, v, s);
    return b.V_dim == K ? launch_fast_k<K, false, true>(b, v, s) : launch_fast_k<K, true, true>(b, v, s);
  });
}

// dynamic shared memory above the default 48 KB per block needs the opt-in, and the limit counts the kernel's static
// shared memory too (block_add_loss's 128 bytes): at V_dim 3072 the row of XV per warp is exactly 48 KB, and without
// the opt-in the launch was refused
template <typename Kern>
void generic_smem_opt_in(Kern kern, size_t smem) {
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, kern) == cudaSuccess && smem + fa.sharedSizeBytes > 48 * 1024)
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

int launch_fm(const FmBatch& b, const FmView& v, int force_generic, cudaStream_t s, cudaError_t* launch_err) {
  const int k = b.V_dim;
  bool fast = !force_generic && fm_fast_supported(k) &&
              v.v_pos != nullptr && aligned16(v.vbase) && (v.vstride % 4 == 0);
  if (fast && b.train && !b.emit) {      // the atomic scatter: exact widths only
    fast = fast_lane_width(k) == k && aligned16(v.gvbase) && (v.gvstride % 4 == 0) &&
           (b.value == nullptr || v.gxxp != nullptr);
  }
  if (b.train && b.emit && !fast) return -1;   // the emit mode exists only on the fast path
  if (fast) {
    return with_lane_width(k, [&](auto kc) {
      constexpr int K = decltype(kc)::value;
      return k == K ? launch_fast_k<K, false>(b, v, s) : launch_fast_k<K, true>(b, v, s);
    });
  }
  if (k > 0 && v.v_pos == nullptr) return -1;   // V_pos is required when V_dim > 0
  const int threads = 128;
  const size_t smem = (size_t)4 * k * sizeof(float);
  if (smem > 200 * 1024) return -1;
  size_t need = (b.nrows + 3) / 4;
  int grid = (int)(need < (size_t)(num_sms() * 16) ? (need ? need : 1) : (size_t)(num_sms() * 16));
  if (b.train) {
    generic_smem_opt_in(k_fm_generic<true>, smem);
    k_fm_generic<true><<<grid, threads, smem, s>>>(b, v);
  } else {
    generic_smem_opt_in(k_fm_generic<false>, smem);
    k_fm_generic<false><<<grid, threads, smem, s>>>(b, v);
  }
  // a launch the device refuses must fail the step, not leave it without a forward: its status, taken (and cleared)
  // here, so that it fails this step and not the next
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (launch_err) *launch_err = e;
    return kLaunchRefused;
  }
  return 1;
}

int launch_grad_finalize_dense(int V_dim, int ks, size_t nkeys, const int* hasv, const float* V,
                               const float* xxp, float* gV, cudaStream_t s) {
  if (V_dim == 0 || nkeys == 0) return 0;
  size_t need = (nkeys + 7) / 8;
  int grid = (int)(need < (size_t)(num_sms() * 8) ? need : (size_t)(num_sms() * 8));
  k_grad_finalize_dense<<<grid, 256, 0, s>>>(V_dim, ks, nkeys, hasv, V, xxp, gV);
  return 1;
}

int launch_grad_finalize(int V_dim, size_t nkeys, const float* weights, const int* V_pos,
                         const float* xxp, float* grad, cudaStream_t s) {
  if (V_dim == 0 || nkeys == 0) return 0;
  size_t need = (nkeys + 7) / 8;
  int grid = (int)(need < (size_t)(num_sms() * 8) ? need : (size_t)(num_sms() * 8));
  k_grad_finalize<<<grid, 256, 0, s>>>(V_dim, nkeys, weights, V_pos, xxp, grad);
  return 1;
}

}  // namespace dfb
