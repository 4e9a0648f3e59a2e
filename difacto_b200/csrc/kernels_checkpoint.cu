// difacto_b200/csrc/kernels_checkpoint.cu -- the device side of the streamed checkpoint (checkpoint.cu).
//
// Writer: a histogram of the occupied table entries by the top 20 bits of the reversed key (k_ckpt_hist) lets the
// host cut the key space into passes of consecutive bins; per pass k_ckpt_select collects the (key, slot) pairs
// of the pass's bins, a CUB radix sort orders them, k_ckpt_hasv + an exclusive scan give every record the V rows
// before it, and k_ckpt_pack writes the v1 records, word by word, at their byte offsets.
// Reader: the host has found the record offsets of a chunk; k_rst_mark checks every key's source part and picks
// this shard's records, a scan ranks them, and k_rst_insert puts them into the table and the row pool.
#include "dfb_device.cuh"

#include <cuda_bf16.h>

#include <cub/cub.cuh>

namespace dfb {

namespace {

constexpr int kBinShift = 64 - kCkptBinBits;

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }

__global__ void k_ckpt_hist(const Entry* __restrict__ tab, uint64_t cap, unsigned* __restrict__ nk,
                            unsigned* __restrict__ nv) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  // cap is a multiple of 1024 and stride of 32: every warp runs the loop with all its lanes
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i - lane_id() < cap; i += stride) {
    unsigned long long key = kEmptyKey;
    int vrow = -1;
    if (i < cap) {
      const ulonglong2 q = *reinterpret_cast<const ulonglong2*>(&tab[i]);
      key = q.x; vrow = (int)(unsigned)(q.y & 0xffffffffULL);
    }
    const bool used = key != kEmptyKey;
    const unsigned bin = used ? (unsigned)(key >> kBinShift) : 0xffffffffu;
    // Criteo-shaped keys crowd into few bins: one atomic per distinct bin of the warp
    const unsigned peers = __match_any_sync(kFullMask, bin);
    const unsigned withv = __ballot_sync(kFullMask, used && vrow >= 0) & peers;
    if (used && lane_id() == (unsigned)(__ffs(peers) - 1)) {
      atomicAdd(&nk[bin], (unsigned)__popc(peers));
      if (withv) atomicAdd(&nv[bin], (unsigned)__popc(withv));
    }
  }
}

__global__ void k_ckpt_select(const Entry* __restrict__ tab, uint64_t cap, unsigned b0, unsigned b1,
                              unsigned long long* __restrict__ keys, unsigned* __restrict__ slots,
                              unsigned long long* __restrict__ counter) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i - lane_id() < cap; i += stride) {
    unsigned long long key = kEmptyKey;
    if (i < cap) key = tab[i].key;
    const unsigned bin = (unsigned)(key >> kBinShift);
    const bool take = key != kEmptyKey && bin >= b0 && bin < b1;
    const unsigned m = __ballot_sync(kFullMask, take);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane_id() == 0) base = atomicAdd(counter, (unsigned long long)__popc(m));
    base = __shfl_sync(kFullMask, base, 0);
    if (take) {
      const unsigned long long at = base + __popc(m & ((1u << lane_id()) - 1u));
      keys[at] = key;
      slots[at] = (unsigned)i;
    }
  }
}

__global__ void k_ckpt_hasv(const Entry* __restrict__ tab, const unsigned* __restrict__ slots, size_t n,
                            unsigned* __restrict__ hv) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    hv[i] = tab[slots[i]].vrow >= 0 ? 1u : 0u;
}

// one warp per record: {u64 key, f32 fea_cnt, f32 w, [f32 sqrt_g, f32 z], i32 has_V, [V[k], [cg[k]]]}
__global__ void k_ckpt_pack(Table t, const unsigned long long* __restrict__ keys, const unsigned* __restrict__ slots,
                            const unsigned* __restrict__ vbefore, size_t n, int aux, int k,
                            unsigned* __restrict__ out) {
  const int fixw = aux ? 7 : 5;
  const size_t roww = (size_t)k * (aux ? 2 : 1);
  const size_t warps = (size_t)gridDim.x * blockDim.x / 32;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < n; i += warps) {
    const Entry e = t.tab[slots[i]];
    const unsigned long long key = keys[i];
    unsigned* o = out + i * fixw + (size_t)vbefore[i] * roww;
    const unsigned l = lane_id();
    if (l < (unsigned)fixw) {
      unsigned wd;
      const int hv = e.vrow >= 0 ? 1 : 0;
      if (l == 0) wd = (unsigned)key;
      else if (l == 1) wd = (unsigned)(key >> 32);
      else if (l == 2) wd = __float_as_uint(e.fea_cnt);
      else if (l == 3) wd = __float_as_uint(e.w);
      else if (l == (unsigned)fixw - 1) wd = (unsigned)hv;
      else if (l == 4) wd = __float_as_uint(e.sqrt_g);
      else wd = __float_as_uint(e.z);
      o[l] = wd;
    }
    if (e.vrow >= 0) {
      const float* row = t.V + (size_t)e.vrow * t.rs;
      o += fixw;
      for (int j = (int)l; j < k; j += 32) o[j] = __float_as_uint(row[j]);
      if (aux)
        for (int j = (int)l; j < k; j += 32) o[k + j] = __float_as_uint(row[t.ks + j]);
    }
  }
}

__device__ __forceinline__ unsigned key_owner_dev(unsigned long long key, unsigned S) {
  const unsigned long long width = ~0ULL / (unsigned long long)S;   // ps-lite postoffice.cc:130-134
  const unsigned long long o = key / width;
  return o >= S ? S - 1 : (unsigned)o;
}

__device__ __forceinline__ unsigned long long rec_key(const unsigned* rec) {
  return (unsigned long long)rec[0] | ((unsigned long long)rec[1] << 32);
}

// flags[i] = kept | (kept && has_V) << 32; a key outside the source part's range raises kErrCkptRange
__global__ void k_rst_mark(const unsigned* __restrict__ buf, const unsigned* __restrict__ roff, size_t n, int aux,
                           unsigned part, unsigned nparts, unsigned shard, unsigned nshards,
                           unsigned long long* __restrict__ flags, DevProgress* prog) {
  const int fixw = aux ? 7 : 5;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned* rec = buf + roff[i];
    const unsigned long long key = rec_key(rec);
    if (key_owner_dev(key, nparts) != part) raise_err(prog, kErrCkptRange);
    const unsigned long long keep = key_owner_dev(key, nshards) == shard ? 1ULL : 0ULL;
    flags[i] = keep | ((keep && rec[fixw - 1] != 0u) ? (1ULL << 32) : 0ULL);
  }
}

// one warp per kept record: insert the key (a key already present raises kErrCkptDup), write its scalars, and its
// V / cg row at n_vrows + rank with the pad columns [V_dim, ks) zero in both halves.
// VONLY (a scoring-only engine's table): the row is V alone at stride ks, 1 = fp32, 2 = bf16 rounded to nearest even
// (NaN and Inf as __float2bfloat16_rn defines them); the record's cg words are not read.
template <int VONLY>
__global__ void k_rst_insert(Table t, const unsigned* __restrict__ buf, const unsigned* __restrict__ roff, size_t n,
                             int aux, int k, const unsigned long long* __restrict__ flags,
                             const unsigned long long* __restrict__ rank) {
  const int fixw = aux ? 7 : 5;
  const unsigned long long base_k = t.state->n_keys, base_v = t.state->n_vrows;
  const size_t warps = (size_t)gridDim.x * blockDim.x / 32;
  const unsigned l = lane_id();
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < n; i += warps) {
    const unsigned long long f = flags[i];
    if (!(f & 1ULL)) continue;
    const unsigned long long r = rank[i];
    const unsigned long long rk = r & 0xffffffffULL, rv = r >> 32;
    const bool hv = (f >> 32) != 0;
    if (base_k + rk >= t.max_keys || (hv && base_v + rv >= t.vcap)) {
      if (l == 0) raise_err(t.prog, DFB_ERR_CAPACITY);
      continue;
    }
    const unsigned* rec = buf + roff[i];
    const long long vrow = hv ? (long long)(base_v + rv) : -1;
    if (l == 0) {
      const unsigned long long key = rec_key(rec);
      uint64_t h = hash64(key) & t.mask;
      bool done = false;
      for (uint64_t probe = 0; probe <= t.mask && !done; ++probe) {
        const unsigned long long prev = atomicCAS(&t.tab[h].key, kEmptyKey, key);
        if (prev == kEmptyKey) {
          Entry* e = &t.tab[h];
          e->vrow = (int)vrow;
          e->fea_cnt = __uint_as_float(rec[2]); e->w = __uint_as_float(rec[3]);
          e->sqrt_g = aux ? __uint_as_float(rec[4]) : 0.f; e->z = aux ? __uint_as_float(rec[5]) : 0.f;
          done = true;
        } else if (prev == key) {
          raise_err(t.prog, kErrCkptDup);
          done = true;
        }
        h = (h + 1) & t.mask;
      }
      if (!done) raise_err(t.prog, DFB_ERR_CAPACITY);
    }
    if (hv) {
      const unsigned* src = rec + fixw;
      if (VONLY == 2) {
        __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(t.V) + (size_t)vrow * t.rs;
        for (int j = (int)l; j < t.ks; j += 32) row[j] = __float2bfloat16_rn(j < k ? __uint_as_float(src[j]) : 0.f);
      } else {
        float* row = t.V + (size_t)vrow * t.rs;
        for (int j = (int)l; j < t.ks; j += 32) {
          row[j] = j < k ? __uint_as_float(src[j]) : 0.f;
          if (VONLY == 0) row[t.ks + j] = (aux && j < k) ? __uint_as_float(src[k + j]) : 0.f;
        }
      }
    }
  }
}

__global__ void k_rst_count(TableState* st, const unsigned long long* __restrict__ flags,
                            const unsigned long long* __restrict__ rank, size_t n) {
  const unsigned long long tot = rank[n - 1] + flags[n - 1];
  st->n_keys += tot & 0xffffffffULL;
  st->n_vrows += tot >> 32;
}

__global__ void k_rst_seed(TableState* st, unsigned seed) { st->seed = seed; }

int grid_cap(size_t n, int per_block, int max_blocks) {
  const size_t g = (n + per_block - 1) / per_block;
  return (int)(g < 1 ? 1 : (g > (size_t)max_blocks ? (size_t)max_blocks : g));
}

}  // namespace

int launch_ckpt_hist(const Table& t, unsigned* nk, unsigned* nv, cudaStream_t s) {
  k_ckpt_hist<<<grid_cap(t.cap, 256, num_sms() * 8), 256, 0, s>>>(t.tab, t.cap, nk, nv);
  return 1;
}

size_t ckpt_sort_tmp_bytes(size_t n) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const unsigned*)nullptr, (unsigned*)nullptr, (int)(n ? n : 1));
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (int)(n ? n : 1));
  return a > b ? a : b;
}

int launch_ckpt_pass(const Table& t, unsigned b0, unsigned b1, size_t n, int aux, int k, const CkptWs& ws,
                     cudaStream_t s) {
  if (n == 0) return 0;
  int nl = 0;
  if (cudaMemsetAsync(ws.counter, 0, sizeof(unsigned long long), s) != cudaSuccess) return -1;
  k_ckpt_select<<<grid_cap(t.cap, 256, num_sms() * 8), 256, 0, s>>>(t.tab, t.cap, b0, b1, ws.keys_in, ws.slots_in,
                                                                     ws.counter);
  ++nl;
  size_t tb = ws.tmp_bytes;
  if (cub::DeviceRadixSort::SortPairs(ws.tmp, tb, ws.keys_in, ws.keys_out, ws.slots_in, ws.slots_out, (int)n, 0, 64,
                                      s) != cudaSuccess)
    return -1;
  ++nl;
  k_ckpt_hasv<<<grid_cap(n, 256, num_sms() * 8), 256, 0, s>>>(t.tab, ws.slots_out, n, ws.hv);
  ++nl;
  tb = ws.tmp_bytes;
  if (cub::DeviceScan::ExclusiveSum(ws.tmp, tb, ws.hv, ws.vbefore, (int)n, s) != cudaSuccess) return -1;
  ++nl;
  k_ckpt_pack<<<grid_cap(n, 8, num_sms() * 16), 256, 0, s>>>(t, ws.keys_out, ws.slots_out, ws.vbefore, n, aux, k,
                                                              ws.out);
  return nl + 1;
}

size_t rst_scan_tmp_bytes(size_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                (int)(n ? n : 1));
  return b;
}

int launch_rst_chunk(Table& t, const unsigned* buf, const unsigned* roff, size_t n, int aux, int k, unsigned part,
                     unsigned nparts, unsigned shard, unsigned nshards, unsigned long long* flags,
                     unsigned long long* rank, void* tmp, size_t tmp_bytes, cudaStream_t s) {
  if (n == 0) return 0;
  k_rst_mark<<<grid_cap(n, 256, num_sms() * 8), 256, 0, s>>>(buf, roff, n, aux, part, nparts, shard, nshards, flags,
                                                              t.prog);
  size_t tb = tmp_bytes;
  if (cub::DeviceScan::ExclusiveSum(tmp, tb, flags, rank, (int)n, s) != cudaSuccess) return -1;
  const int grid = grid_cap(n, 8, num_sms() * 16);
  if (t.vonly == 2) k_rst_insert<2><<<grid, 256, 0, s>>>(t, buf, roff, n, aux, k, flags, rank);
  else if (t.vonly == 1) k_rst_insert<1><<<grid, 256, 0, s>>>(t, buf, roff, n, aux, k, flags, rank);
  else k_rst_insert<0><<<grid, 256, 0, s>>>(t, buf, roff, n, aux, k, flags, rank);
  k_rst_count<<<1, 1, 0, s>>>(t.state, flags, rank, n);
  return 4;
}

int launch_rst_seed(Table& t, unsigned seed, cudaStream_t s) {
  k_rst_seed<<<1, 1, 0, s>>>(t.state, seed);
  return 1;
}

}  // namespace dfb
