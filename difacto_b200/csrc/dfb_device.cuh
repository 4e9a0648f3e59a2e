// difacto_b200/csrc/dfb_device.cuh -- device-side helpers shared by the table and shard kernels.
//
// The per-key arithmetic of SGDUpdater (src/sgd/sgd_updater.cc of the reference) lives here so that
// the fused single-GPU kernels (kernels_table.cu) and the owner side of the NVLink-sharded store
// (kernels_shard.cu) run literally the same code.
#pragma once
#include "dfb_internal.cuh"

#include "../../include/difacto_b200.h"

namespace dfb {

constexpr unsigned kFullMask = 0xffffffffu;

__device__ __forceinline__ uint64_t hash64(uint64_t h) {
  h ^= h >> 33; h *= 0xff51afd7ed558ccdULL;
  h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL;
  h ^= h >> 33;
  return h;
}

__device__ __forceinline__ unsigned long long reverse_nibbles(unsigned long long x) {
  // byte reversal, then swap the two nibbles of every byte  == reversing the 16 nibbles
  x = ((unsigned long long)__byte_perm((unsigned)(x & 0xffffffffULL), 0, 0x0123) << 32) |
      (unsigned long long)__byte_perm((unsigned)(x >> 32), 0, 0x0123);
  return ((x & 0x0F0F0F0F0F0F0F0FULL) << 4) | ((x & 0xF0F0F0F0F0F0F0F0ULL) >> 4);
}

// the table key of a raw feature id as Localizer(-1) forms it: ReverseBytes(id % (2^64-1)) (localizer.cc:22-26)
__device__ __forceinline__ unsigned long long raw_key(unsigned long long id) {
  return reverse_nibbles(id == ~0ULL ? 0ULL : id);
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
  return v;
}

__device__ __forceinline__ void raise_err(DevProgress* prog, int code) { atomicCAS(&prog->err, 0, code); }

// ---- per-access L2 eviction policies (createpolicy + the .L2::cache_hint forms of ld / st) ----
// The step's L2 plan (DESIGN.md section 2): the per-row p*XV / p that the update re-reads per nnz are kept
// (evict_last); the [V|cg] rows and per-key metadata touched once per step stream past them (evict_first).
// Engine kwarg l2_hints=0 turns all of them off.
enum L2Kind { kL2Normal = 0, kL2EvictFirst = 1, kL2EvictLast = 2 };
__device__ __forceinline__ uint64_t l2_policy(int kind) {
  uint64_t pol;
  if (kind == kL2EvictFirst) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  else if (kind == kL2EvictLast) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// read-only for the lifetime of the kernel: the non-coherent path (ld.global.nc)
__device__ __forceinline__ float4 ldg128_pol(const float* p, uint64_t pol) {
  float4 r;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
// 4 bf16 columns of a scoring-only engine's V row (one 8-byte load), widened to fp32: exact, a 16-bit shift
__device__ __forceinline__ float4 ldg_bf16x4_pol(const void* p, uint64_t pol) {
  unsigned lo, hi;
  asm volatile("ld.global.nc.L2::cache_hint.v2.b32 {%0, %1}, [%2], %3;" : "=r"(lo), "=r"(hi) : "l"(p), "l"(pol));
  return make_float4(__uint_as_float(lo << 16), __uint_as_float(lo & 0xffff0000u),
                     __uint_as_float(hi << 16), __uint_as_float(hi & 0xffff0000u));
}
__device__ __forceinline__ int2 ldg64_pol(const int2* p, uint64_t pol) {
  int2 r;
  asm volatile("ld.global.nc.L2::cache_hint.v2.s32 {%0, %1}, [%2], %3;" : "=r"(r.x), "=r"(r.y) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ unsigned long long ldg_u64_pol(const unsigned long long* p, uint64_t pol) {
  unsigned long long r;
  asm volatile("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ unsigned ldg_u32_pol(const void* p, uint64_t pol) {
  unsigned r;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ int ldg_s32_pol(const int* p, uint64_t pol) { return (int)ldg_u32_pol(p, pol); }
__device__ __forceinline__ float ldg_f32_pol(const float* p, uint64_t pol) { return __uint_as_float(ldg_u32_pol(p, pol)); }
// rows the same kernel writes back: the coherent path (ld.global / st.global)
__device__ __forceinline__ float4 ld128_pol(const float* p, uint64_t pol) {
  float4 r;
  asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void st128_pol(float* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
               ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}

// the count of a launch: a host value, or (when dn != nullptr) a value a previous kernel left on the
// device -- the sizes of a localized batch never visit the host (no synchronisation inside a step)
__device__ __forceinline__ size_t dev_count(size_t n_host, const unsigned long long* dn) {
  if (dn == nullptr) return n_host;
  const unsigned long long v = *dn;
  return v < (unsigned long long)n_host ? (size_t)v : n_host;   // n_host is the capacity the buffers were sized for
}

// ---- FTRL-proximal on w: SGDUpdater::UpdateW, sgd_updater.cc:104-127 ----
// returns true when w went 0 -> nonzero (the InitV trigger :121-126)
__device__ __forceinline__ bool ftrl_step(const Params& p, float gw, float& w, float& sqrt_g, float& z) {
  const float sg = sqrt_g, w0 = w;
  gw = __fadd_rn(gw, __fmul_rn(w0, p.l2));
  sqrt_g = __fsqrt_rn(__fadd_rn(__fmul_rn(sg, sg), __fmul_rn(gw, gw)));
  // z -= gw - (sqrt_g' - sg) / lr * w
  z = __fsub_rn(z, __fsub_rn(gw, __fmul_rn(__fdiv_rn(__fsub_rn(sqrt_g, sg), p.lr), w0)));
  const float l1 = p.l1;
  if (z <= l1 && z >= -l1) {
    w = 0.f;
  } else {
    const float eta = __fdiv_rn(__fadd_rn(p.lr_beta, sqrt_g), p.lr);
    w = __fdiv_rn(z > 0.f ? __fsub_rn(z, l1) : __fadd_rn(z, l1), eta);
  }
  return w0 == 0.f && w != 0.f;
}

// ---- AdaGrad on one V component: SGDUpdater::UpdateV, sgd_updater.cc:129-138 ----
__device__ __forceinline__ void adagrad_step(const Params& p, float gV, float& v, float& cg) {
  const float g = __fadd_rn(gV, __fmul_rn(p.V_l2, v));
  cg = __fsqrt_rn(__fadd_rn(__fmul_rn(cg, cg), __fmul_rn(g, g)));
  const float eta = __fdiv_rn(p.V_lr, __fadd_rn(cg, p.V_lr_beta));
  v = __fsub_rn(v, __fmul_rn(eta, g));
}

// AdaGrad on one float4 of a V row, grad = g - vp * xp (fm_loss.h:181-198).  PAD: only the first nact (>= 1) columns
// are V_dim's; the pad columns after them stay as they are (0) -- with V_lr_beta = 0 the step would divide by cg = 0
template <bool PAD>
__device__ __forceinline__ void adagrad4(const Params& p, float4 g, float4 vp, float xp, float4& v, float4& c, int nact) {
  adagrad_step(p, __fsub_rn(g.x, __fmul_rn(vp.x, xp)), v.x, c.x);
  if (!PAD || nact > 1) adagrad_step(p, __fsub_rn(g.y, __fmul_rn(vp.y, xp)), v.y, c.y);
  if (!PAD || nact > 2) adagrad_step(p, __fsub_rn(g.z, __fmul_rn(vp.z, xp)), v.z, c.z);
  if (!PAD || nact > 3) adagrad_step(p, __fsub_rn(g.w, __fmul_rn(vp.w, xp)), v.w, c.w);
}

// penalty of one w (sgd_learner.cc:257 ; evaluated in fp32 here, double there)
__device__ __forceinline__ float pen_w(const Params& p, float w) {
  return p.l1 * fabsf(w) + 0.5f * p.l2 * w * w;
}

// one 32-byte table entry (one DRAM sector) fetched with two independent 128-bit requests issued back to back
// (sm_90 has no 256-bit load), L2-only so that an entry another thread of the same launch just inserted is never
// served stale from L1
struct Entry256 {
  unsigned long long key, q1, q2, q3;      // {key | vrow, pad | fea_cnt, w | sqrt_g, z}
  __device__ __forceinline__ int vrow() const { return (int)(unsigned)(q1 & 0xffffffffULL); }
  __device__ __forceinline__ float w() const { return __uint_as_float((unsigned)(q2 >> 32)); }
  __device__ __forceinline__ float4 scalars() const {    // {fea_cnt, w, sqrt_g, z}
    return make_float4(__uint_as_float((unsigned)q2), __uint_as_float((unsigned)(q2 >> 32)),
                       __uint_as_float((unsigned)q3), __uint_as_float((unsigned)(q3 >> 32)));
  }
};
__device__ __forceinline__ Entry256 load_entry(const Entry* p) {
  Entry256 e;
  const unsigned long long* q = reinterpret_cast<const unsigned long long*>(p);
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(e.key), "=l"(e.q1) : "l"(q));
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(e.q2), "=l"(e.q3) : "l"(q + 2));
  return e;
}

// model_[key] (sgd_updater.cc:43-45,65-67,86-88): find or default-construct.  Returns the slot or -1.
// On a hit (or a fresh insert) *lo receives the first half of the entry {key, vrow, pad} as loaded.
template <bool INSERT>
__device__ __forceinline__ int table_find(const Table& t, unsigned long long key, uint64_t h) {
  for (uint64_t probe = 0; probe <= t.mask; ++probe) {
    unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(&t.tab[h].key);
    if (cur == key) return (int)h;
    if (cur == kEmptyKey) {
      if (!INSERT) return -1;
      const unsigned long long prev = atomicCAS(&t.tab[h].key, kEmptyKey, key);
      if (prev == kEmptyKey) {
        const unsigned long long nk = atomicAdd(&t.state->n_keys, 1ULL) + 1;
        atomicAdd(&t.prog->new_keys, 1ULL);
        if (nk > t.max_keys) raise_err(t.prog, DFB_ERR_CAPACITY);
        return (int)h;
      }
      if (prev == key) return (int)h;
    }
    h = (h + 1) & t.mask;
  }
  if (INSERT) raise_err(t.prog, DFB_ERR_CAPACITY);
  return -1;
}

// model_[key] for a key whose home entry e (at h, loaded with load_entry) is in hand -- the update's find / insert in
// the single-GPU step, counted, inserted and raised exactly as table_find<true>.  Returns the slot with its entry in e,
// or -1.
// A key away from its home slot costs a probe chain, and a warp waits for the longest chain of its 32 lanes: the
// keys of the next 4 slots are loaded at once (one round trip instead of up to 4), and only the hit's entry is loaded
// again.  (The flagship update took 3.47 ms so; probing one slot at a time 3.92 ms, and 4.17 ms when the home slot and
// the hit were also read again; H100 80 GB HBM3, 400 W.)  An empty slot
// holds the default entry (vrow -1, zeros), so a fresh insert is that entry with its key.
__device__ __forceinline__ int find_insert_entry(const Table& t, unsigned long long key, uint64_t h, Entry256& e) {
  if (e.key == key) return (int)h;
  uint64_t probe = 0;
  for (;;) {
    if (e.key == kEmptyKey) {
      const unsigned long long prev = atomicCAS(&t.tab[h].key, kEmptyKey, key);
      if (prev == kEmptyKey) {
        const unsigned long long nk = atomicAdd(&t.state->n_keys, 1ULL) + 1;
        atomicAdd(&t.prog->new_keys, 1ULL);
        if (nk > t.max_keys) raise_err(t.prog, DFB_ERR_CAPACITY);
        e.key = key;
        return (int)h;
      }
      if (prev == key) { e = load_entry(t.tab + h); return (int)h; }
    }
    unsigned long long k4[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(k4[q]) : "l"(&t.tab[(h + 1 + q) & t.mask].key));
    int q = 0;
    for (; q < 4; ++q) {
      h = (h + 1) & t.mask;
      if (++probe > t.mask) { raise_err(t.prog, DFB_ERR_CAPACITY); return -1; }   // every slot visited
      if (k4[q] == key) { e = load_entry(t.tab + h); return (int)h; }
      if (k4[q] == kEmptyKey) break;
    }
    if (q < 4) { e.key = kEmptyKey; e.q1 = 0x00000000ffffffffULL; e.q2 = 0ULL; e.q3 = 0ULL; }   // the default entry
    else e.key = k4[3];                        // another key: go on after it
  }
}

}  // namespace dfb
