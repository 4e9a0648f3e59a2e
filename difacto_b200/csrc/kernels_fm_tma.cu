// difacto_b200/csrc/kernels_fm_tma.cu -- the gather+interaction kernel (K1) with the V rows staged through shared
// memory by the bulk-copy engine: an A/B against k_fm_fast's register-staged LDG.128 gather (kernels_fm.cu).
//
// The gathered rows are not a tile (every nnz names another 4k-byte row of the table), so the tensor-map form of
// TMA has nothing to describe; what the hardware (sm_90) does offer is the 1-D bulk copy `cp.async.bulk.shared.global`
// (UBLKCP in SASS) completing on an mbarrier.  Here every lane of a warp issues one bulk copy per nnz (one table row -> the warp's shared-memory
// stage), two 32-row stages per warp are in flight, and the FM arithmetic reads the rows from shared memory.
// Compared with k_fm_fast this frees the 32 registers that hold 8 x float4 in flight and lets the copy engine
// keep up to 16 KB per warp outstanding.  Predict only (MODE 0); engine kwarg k1_tma=1 selects it for
// validation batches; the register-staged kernel stays the default.
#include "dfb_internal.cuh"

#include <math.h>
#include <string.h>

namespace dfb {

namespace {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
// one table row -> shared memory, completion counted in bytes on the mbarrier (UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

constexpr int kTmaWarps = 4;      // per CTA: 4 warps x 2 stages x 32 rows x 4K bytes

template <int K, bool HAS_VAL>
__global__ void __launch_bounds__(kTmaWarps * 32) k_fm_tma(FmBatch b, FmView v) {
  constexpr int LPR = K / 4;
  constexpr int G = 32 / LPR;
  constexpr int ROWB = K * 4;
  constexpr int STAGEB = 32 * ROWB;
  extern __shared__ __align__(128) unsigned char smem[];
  if (b.dev_nkeys && *b.dev_nkeys == 0ULL) {          // dropped by the GPU localizer: see FmBatch::dev_nkeys
    if (blockIdx.x == 0 && threadIdx.x == 0 && b.prog) atomicCAS(&b.prog->err, 0, kErrIdRange);
    return;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int sub = lane % LPR, grp = lane / LPR;
  unsigned char* stage0 = smem + (size_t)wid * 2 * STAGEB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)kTmaWarps * 2 * STAGEB);
  const uint32_t bar0 = smem_u32(&bars[wid * 2]), bar1 = smem_u32(&bars[wid * 2 + 1]);
  if (threadIdx.x == 0) {
    for (int i = 0; i < kTmaWarps * 2; ++i) mbar_init(smem_u32(&bars[i]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  uint32_t ph0 = 0, ph1 = 0;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  float loss_acc = 0.f;

  for (size_t row = warp0; row < b.nrows; row += nwarps) {
    const uint64_t o0 = b.offset[row], o1 = b.offset[row + 1];
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc2 = 0.f, wsum = 0.f;
    // metadata of a chunk + the bulk copies of its rows into stage st
    auto issue = [&](uint64_t c, int st, float& x, int& vr) {
      const uint64_t j = c + lane;
      x = 0.f; vr = -1;
      float w = 0.f;
      if (j < o1) {
        const uint32_t u = __ldg(b.index + j);
        x = HAS_VAL ? __ldg(b.value + j) : 1.f;
        const int2 t = __ldg(v.wv + u);
        w = __int_as_float(t.x);
        vr = t.y;
      }
      wsum = fmaf(x, w, wsum);
      const unsigned m = __ballot_sync(kFull, vr >= 0);
      const uint32_t bar = st ? bar1 : bar0;
      // reads of this stage by the generic proxy (two chunks ago) are ordered before the async-proxy writes
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      if (lane == 0) mbar_expect_tx(bar, (uint32_t)__popc(m) * ROWB);
      __syncwarp();
      if (vr >= 0)
        bulk_g2s(smem_u32(stage0 + (size_t)st * STAGEB + (size_t)lane * ROWB), v.vbase + (long long)vr * v.vstride, ROWB, bar);
    };
    float x_c, x_n = 0.f;
    int vr_c, vr_n = -1;
    if (o0 < o1) issue(o0, 0, x_n, vr_n);
    int st = 0;
    for (uint64_t c = o0; c < o1; c += 32, st ^= 1) {
      x_c = x_n; vr_c = vr_n;
      if (c + 32 < o1) issue(c + 32, st ^ 1, x_n, vr_n);
      if (st) { mbar_wait(bar1, ph1); ph1 ^= 1; } else { mbar_wait(bar0, ph0); ph0 ^= 1; }
      const unsigned char* sb = stage0 + (size_t)st * STAGEB;
      const int cnt = (int)((o1 - c) < 32 ? (o1 - c) : 32);
#pragma unroll 4
      for (int t0 = 0; t0 < cnt; t0 += G) {
        const int t = t0 + grp;
        const int vr_t = __shfl_sync(kFull, vr_c, t & 31);
        const float x_t = __shfl_sync(kFull, x_c, t & 31);
        if (t < cnt && vr_t >= 0) {
          const float4 vv = *reinterpret_cast<const float4*>(sb + (size_t)t * ROWB + sub * 16);
          const float a0 = x_t * vv.x, a1 = x_t * vv.y, a2 = x_t * vv.z, a3 = x_t * vv.w;
          xv.x += a0; xv.y += a1; xv.z += a2; xv.w += a3;
          acc2 = fmaf(a0, a0, acc2); acc2 = fmaf(a1, a1, acc2);
          acc2 = fmaf(a2, a2, acc2); acc2 = fmaf(a3, a3, acc2);
        }
      }
      __syncwarp();
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
    float s1 = grp == 0 ? (xv.x * xv.x + xv.y * xv.y + xv.z * xv.z + xv.w * xv.w) : 0.f;
    s1 = warp_sum(s1);
    float pred = wsum + 0.5f * (s1 - acc2);
    pred = pred > 20.f ? 20.f : (pred < -20.f ? -20.f : pred);   // fm_loss.h:118
    if (lane == 0) {
      if (b.pred_io) b.pred_io[row] = pred;
      if (b.label) {
        const float y = __ldg(b.label + row) > 0.f ? 1.f : -1.f;
        loss_acc += logf(1.f + expf(-y * pred));
      }
    }
  }
  // logloss: one atomic per warp (the kernel is an experiment; k_fm_fast block-reduces)
  if (b.prog) {
    loss_acc = warp_sum(loss_acc);
    if (lane == 0) {
      atomicAdd(&b.prog->loss, (double)loss_acc);
      if (warp0 == 0) atomicAdd(&b.prog->nrows, (unsigned long long)b.nrows);
    }
  }
}

}  // namespace

// returns 1 when launched, 0 when the configuration is not covered by the experiment (caller uses k_fm_fast)
int launch_fm_tma_predict(const FmBatch& b, const FmView& v, cudaStream_t s) {
  if (b.V_dim != 64 || b.train || v.wv == nullptr || b.pred_acc || b.nrows == 0) return 0;
  if ((reinterpret_cast<uintptr_t>(v.vbase) & 15u) != 0 || (v.vstride % 4) != 0) return 0;
  const size_t smem = (size_t)kTmaWarps * 2 * 32 * 64 * 4 + kTmaWarps * 2 * sizeof(uint64_t);
  const int grid = num_sms() * 3;
  if (b.value) {
    cudaFuncSetAttribute(k_fm_tma<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_fm_tma<64, true><<<grid, kTmaWarps * 32, smem, s>>>(b, v);
  } else {
    cudaFuncSetAttribute(k_fm_tma<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    k_fm_tma<64, false><<<grid, kTmaWarps * 32, smem, s>>>(b, v);
  }
  return 1;
}

}  // namespace dfb
