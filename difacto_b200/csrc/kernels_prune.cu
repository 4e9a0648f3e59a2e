// difacto_b200/csrc/kernels_prune.cu -- the device side of dfb_prune (prune.cu, DESIGN.md section 10).
//
// An entry is dropped when it carries no weight: w == 0, no V row, fea_cnt <= max_count.  Open addressing cannot blank
// a slot in the middle of a probe chain, so the table is rebuilt in place:
//   k_prune_count    counts the kept and the dropped entries (warp-aggregated atomics), and the kept ones per block;
//   k_prune_compact  copies the kept entries, all 32 bytes, into a workspace of n_kept entries (in slot order: block b
//                    writes after the kept entries of blocks 0..b-1) and writes the empty entry into every occupied
//                    slot; an empty slot already holds it;
// then k_table_rehash (kernels_table.cu) re-inserts the workspace unchanged, and k_prune_commit lowers n_keys.
// Both passes walk the slots in the same tiles (kPruneTile slots, kPruneSub per thread with their loads in flight
// together), so a block's count is exactly what it compacts.
//
// dfb_prune_rare (DESIGN.md section 10.1) runs the same two passes under the rare predicate (fea_cnt <= max_count,
// whatever w and V hold; the count pass also counts the kept and the dropped V rows), then compacts the V-row pool in
// place, n_vkeep = n_vrows - dropped V rows:
//   k_rare_mark   sets bit vrow of a bitmap over [0, n_vrows) for every kept entry of the workspace, and records the
//                 entry of every row at or above n_vkeep in owner[vrow - n_vkeep];
//   k_rare_count  per bitmap word: the holes (clear bits below n_vkeep) and the movers (set bits from n_vkeep on),
//                 scanned over [holes of words 0..W) ++ [movers of words 0..W), so hole i and mover i land at i and H + i;
//   k_rare_list   writes each hole's and each mover's row there, in ascending row order;
//   k_rare_move   one warp per pair: the mover's whole [V | cg] row into the hole, and the new row into its entry.
// Holes lie below n_vkeep and movers at or above it, so no copy overlaps another.  Nothing is sorted and no result
// depends on the order of atomics: the layout is the same on every run.
#include <cub/cub.cuh>

#include "dfb_device.cuh"

namespace dfb {

namespace {

constexpr int kPruneThreads = 256;
constexpr int kPruneWarps = kPruneThreads / 32;
// slots per thread per tile, their loads issued together: a tile is kPruneSub sub-tiles of kPruneThreads slots, slot
// base + j * kPruneThreads + threadIdx.x is sub-tile j's
constexpr int kPruneSub = 4;
constexpr int kPruneTile = kPruneThreads * kPruneSub;

__device__ __forceinline__ unsigned prune_lane() { return threadIdx.x & 31; }

// the slot's entry as {key | vrow, pad}, {fea_cnt | w, sqrt_g | z}; 1: kept, 2: dropped, 0: empty.  RARE: dropped
// when fea_cnt <= max_count alone (dfb_prune_rare); otherwise also w == 0 and no V row (dfb_prune)
template <bool RARE>
__device__ __forceinline__ int prune_kind(const ulonglong2& a, const ulonglong2& b, float max_count) {
  if (a.x == kEmptyKey) return 0;
  const int vrow = (int)(unsigned)(a.y & 0xffffffffULL);
  const float fea_cnt = __uint_as_float((unsigned)(b.x & 0xffffffffULL));
  const float w = __uint_as_float((unsigned)(b.x >> 32));
  if (RARE) return fea_cnt <= max_count ? 2 : 1;
  return (vrow < 0 && w == 0.f && fea_cnt <= max_count) ? 2 : 1;
}

__device__ __forceinline__ bool has_vrow(const ulonglong2& a) { return (int)(unsigned)(a.y & 0xffffffffULL) >= 0; }

// tot = {kept, dropped} (RARE: {kept, dropped, kept V rows, dropped V rows}); blk_kept[b] = the entries block b keeps
// (both zeroed by the caller)
template <bool RARE>
__global__ void __launch_bounds__(kPruneThreads) k_prune_count(const Entry* __restrict__ tab, uint64_t cap,
                                                               float max_count, unsigned long long* __restrict__ tot,
                                                               unsigned* __restrict__ blk_kept) {
  const ulonglong2* in = reinterpret_cast<const ulonglong2*>(tab);
  unsigned kept = 0, dropped = 0, kept_v = 0, dropped_v = 0;
  for (size_t base = (size_t)blockIdx.x * kPruneTile; base < cap; base += (size_t)gridDim.x * kPruneTile) {
    ulonglong2 a[kPruneSub], b[kPruneSub];
#pragma unroll
    for (int j = 0; j < kPruneSub; ++j) {
      const size_t i = base + (size_t)j * kPruneThreads + threadIdx.x;
      a[j] = make_ulonglong2(kEmptyKey, 0ULL); b[j] = make_ulonglong2(0ULL, 0ULL);
      if (i < cap) { a[j] = in[2 * i]; b[j] = in[2 * i + 1]; }
    }
#pragma unroll
    for (int j = 0; j < kPruneSub; ++j) {
      const int k = prune_kind<RARE>(a[j], b[j], max_count);
      kept += k == 1;
      dropped += k == 2;
      if (RARE) {
        kept_v += k == 1 && has_vrow(a[j]);
        dropped_v += k == 2 && has_vrow(a[j]);
      }
    }
  }
  kept = __reduce_add_sync(kFullMask, kept);
  dropped = __reduce_add_sync(kFullMask, dropped);
  if (RARE) {
    kept_v = __reduce_add_sync(kFullMask, kept_v);
    dropped_v = __reduce_add_sync(kFullMask, dropped_v);
  }
  if (prune_lane() == 0) {
    if (kept) {
      atomicAdd(&tot[0], (unsigned long long)kept);
      atomicAdd(&blk_kept[blockIdx.x], kept);
    }
    if (dropped) atomicAdd(&tot[1], (unsigned long long)dropped);
    if (RARE && kept_v) atomicAdd(&tot[2], (unsigned long long)kept_v);
    if (RARE && dropped_v) atomicAdd(&tot[3], (unsigned long long)dropped_v);
  }
}

template <bool RARE>
__global__ void __launch_bounds__(kPruneThreads) k_prune_compact(Entry* tab, uint64_t cap, float max_count,
                                                                 const unsigned* __restrict__ blk_kept,
                                                                 Entry* __restrict__ out) {
  __shared__ unsigned long long s_part[kPruneWarps];
  __shared__ unsigned s_warp[kPruneSub][kPruneWarps];
  const unsigned lane = prune_lane(), wid = threadIdx.x >> 5;
  // where this block's kept entries start: the kept entries of the blocks before it
  unsigned long long before = 0;
  for (unsigned b = threadIdx.x; b < blockIdx.x; b += kPruneThreads) before += blk_kept[b];
  before = __reduce_add_sync(kFullMask, (unsigned)before);   // < 2^32: the table holds at most 2^31 slots
  if (lane == 0) s_part[wid] = before;
  __syncthreads();
  unsigned long long at = 0;
  for (int w = 0; w < kPruneWarps; ++w) at += s_part[w];
  ulonglong2* slots = reinterpret_cast<ulonglong2*>(tab);
  ulonglong2* dst = reinterpret_cast<ulonglong2*>(out);
  for (size_t base = (size_t)blockIdx.x * kPruneTile; base < cap; base += (size_t)gridDim.x * kPruneTile) {
    ulonglong2 a[kPruneSub], b[kPruneSub];
    int k[kPruneSub];
    unsigned m[kPruneSub];
#pragma unroll
    for (int j = 0; j < kPruneSub; ++j) {
      const size_t i = base + (size_t)j * kPruneThreads + threadIdx.x;
      a[j] = make_ulonglong2(kEmptyKey, 0ULL); b[j] = make_ulonglong2(0ULL, 0ULL);
      if (i < cap) { a[j] = slots[2 * i]; b[j] = slots[2 * i + 1]; }
    }
#pragma unroll
    for (int j = 0; j < kPruneSub; ++j) {
      k[j] = prune_kind<RARE>(a[j], b[j], max_count);
      m[j] = __ballot_sync(kFullMask, k[j] == 1);
    }
    __syncthreads();                      // the previous tile's s_warp has been read
    if (lane == 0)
#pragma unroll
      for (int j = 0; j < kPruneSub; ++j) s_warp[j][wid] = __popc(m[j]);
    __syncthreads();
    // the kept entries before each of this thread's slots, in slot order: sub-tile, then warp, then lane
    unsigned run = 0;
#pragma unroll
    for (int j = 0; j < kPruneSub; ++j) {
      unsigned off = 0, sub = 0;
      for (int w = 0; w < kPruneWarps; ++w) {
        const unsigned c = s_warp[j][w];
        off += (unsigned)w < wid ? c : 0u;
        sub += c;
      }
      const size_t i = base + (size_t)j * kPruneThreads + threadIdx.x;
      if (k[j] == 1) {
        const unsigned long long p = at + run + off + __popc(m[j] & ((1u << lane) - 1u));
        dst[2 * p] = a[j];
        dst[2 * p + 1] = b[j];
      }
      if (k[j] != 0) {
        slots[2 * i] = make_ulonglong2(kEmptyKey, 0x00000000ffffffffULL);   // {key, vrow -1 | pad 0}
        slots[2 * i + 1] = make_ulonglong2(0ULL, 0ULL);                     // fea_cnt, w, sqrt_g, z
      }
      run += sub;
    }
    at += run;
  }
}

__global__ void k_prune_commit(TableState* st, const unsigned long long* __restrict__ tot) { st->n_keys -= tot[1]; }

// ---- dfb_prune_rare: the V-row pool's compaction ----
constexpr int kRareThreads = 256;

// raised when a kept row is owned twice or lies outside [0, n_vrows): the pool is then left as it is
__device__ __forceinline__ void rare_broken(DevProgress* prog, unsigned* bad) {
  raise_err(prog, DFB_ERR_INVALID);
  atomicOr(bad, 1u);
}

__global__ void __launch_bounds__(kRareThreads) k_rare_mark(const Entry* __restrict__ kept, uint64_t n_kept,
                                                            unsigned long long n_vrows, unsigned long long n_vkeep,
                                                            unsigned* __restrict__ bits, int* __restrict__ owner,
                                                            DevProgress* prog, unsigned* bad) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_kept; i += (size_t)gridDim.x * blockDim.x) {
    const int vrow = kept[i].vrow;
    if (vrow < 0) continue;
    if ((unsigned long long)vrow >= n_vrows) { rare_broken(prog, bad); continue; }
    const unsigned bit = 1u << (vrow & 31);
    if (atomicOr(&bits[vrow >> 5], bit) & bit) { rare_broken(prog, bad); continue; }
    if ((unsigned long long)vrow >= n_vkeep) owner[vrow - n_vkeep] = (int)i;
  }
}

// the bits of word w that stand for rows below n_vkeep (lo) and for rows in [n_vkeep, n_vrows) (hi)
__device__ __forceinline__ void rare_masks(size_t w, unsigned long long n_vrows, unsigned long long n_vkeep,
                                           unsigned& lo, unsigned& hi) {
  const unsigned long long p0 = (unsigned long long)w * 32;
  auto below = [p0](unsigned long long n) -> unsigned {
    return n >= p0 + 32 ? ~0u : n <= p0 ? 0u : (1u << (unsigned)(n - p0)) - 1u;
  };
  lo = below(n_vkeep);
  hi = below(n_vrows) & ~lo;
}

// cnt[w] = the holes of word w, cnt[W + w] = its movers
__global__ void __launch_bounds__(kRareThreads) k_rare_count(const unsigned* __restrict__ bits, size_t W,
                                                             unsigned long long n_vrows, unsigned long long n_vkeep,
                                                             unsigned* __restrict__ cnt) {
  for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (size_t)gridDim.x * blockDim.x) {
    unsigned lo, hi;
    rare_masks(w, n_vrows, n_vkeep, lo, hi);
    const unsigned b = bits[w];
    cnt[w] = __popc(~b & lo);
    cnt[W + w] = __popc(b & hi);
  }
}

// at[] = the exclusive scan of cnt[]: hole i's row into list[i], mover i's into list[H + i] (at[W] == H); list holds
// n_list ints (a broken pool may count more than fit: those are not written, and k_rare_move does nothing)
__global__ void __launch_bounds__(kRareThreads) k_rare_list(const unsigned* __restrict__ bits, size_t W,
                                                            unsigned long long n_vrows, unsigned long long n_vkeep,
                                                            const unsigned* __restrict__ at, int* __restrict__ list,
                                                            size_t n_list) {
  for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (size_t)gridDim.x * blockDim.x) {
    unsigned lo, hi;
    rare_masks(w, n_vrows, n_vkeep, lo, hi);
    const unsigned b = bits[w];
    unsigned m = ~b & lo;
    for (size_t o = at[w]; m; m &= m - 1, ++o)
      if (o < n_list) list[o] = (int)(w * 32 + __ffs(m) - 1);
    m = b & hi;
    for (size_t o = at[W + w]; m; m &= m - 1, ++o)
      if (o < n_list) list[o] = (int)(w * 32 + __ffs(m) - 1);
  }
}

// one warp per pair: row list[H + i] -> row list[i], rs floats (a multiple of 4: [V | cg] with its pad columns) with
// 16-byte accesses; then the mover's entry in the workspace takes the new row
__global__ void __launch_bounds__(kRareThreads) k_rare_move(float* V, int rs, const unsigned* __restrict__ at, size_t W,
                                                            const int* __restrict__ list, const int* __restrict__ owner,
                                                            unsigned long long n_vkeep, Entry* kept,
                                                            const unsigned* __restrict__ bad) {
  if (*bad) return;
  const size_t H = at[W];
  const unsigned lane = threadIdx.x & 31;
  const int n4 = rs / 4;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < H;
       i += ((size_t)gridDim.x * blockDim.x) >> 5) {
    const int dst = list[i], src = list[H + i];
    const float4* from = reinterpret_cast<const float4*>(V + (size_t)src * rs);
    float4* to = reinterpret_cast<float4*>(V + (size_t)dst * rs);
    for (int c = lane; c < n4; c += 32) to[c] = from[c];
    if (lane == 0) kept[owner[src - n_vkeep]].vrow = dst;
  }
}

// n_keys and n_vrows lowered by the dropped entries and rows (n_vrows kept as it was when the pool was found broken)
__global__ void k_rare_commit(TableState* st, const unsigned long long* __restrict__ tot, const unsigned* __restrict__ bad) {
  st->n_keys -= tot[1];
  if (!*bad) st->n_vrows -= tot[3];
}

int rare_grid(size_t n) {
  const size_t b = (n + kRareThreads - 1) / kRareThreads;
  const size_t g = (size_t)num_sms() * 8;
  return (int)(b < g ? (b ? b : 1) : g);
}

}  // namespace

int prune_grid(uint64_t cap) {
  const uint64_t tiles = (cap + kPruneTile - 1) / kPruneTile;
  const uint64_t g = (uint64_t)num_sms() * 8;
  return (int)(tiles < g ? (tiles ? tiles : 1) : g);
}

int launch_prune_count(const Table& t, float max_count, int grid, unsigned long long* tot, unsigned* blk_kept,
                       cudaStream_t s, bool rare) {
  if (rare) k_prune_count<true><<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, tot, blk_kept);
  else k_prune_count<false><<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, tot, blk_kept);
  return 1;
}

int launch_prune_rebuild(Table& t, float max_count, int grid, const unsigned long long* tot, const unsigned* blk_kept,
                         Entry* kept, uint64_t n_kept, cudaStream_t s) {
  k_prune_compact<false><<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, blk_kept, kept);
  int nl = 1 + launch_table_insert(kept, n_kept, t, s);
  k_prune_commit<<<1, 1, 0, s>>>(t.state, tot);
  return nl + 1;
}

size_t rare_scan_tmp_bytes(size_t W) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (int)(W ? 2 * W : 1));
  return bytes;
}

int launch_prune_rare(Table& t, float max_count, int grid, const unsigned long long* tot, const unsigned* blk_kept,
                      Entry* kept, uint64_t n_kept, uint64_t n_vrows, uint64_t n_vkeep, const RareWs& ws,
                      cudaStream_t s) {
  int nl = 0;
  k_prune_compact<true><<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, blk_kept, kept);
  ++nl;
  const size_t W = (n_vrows + 31) / 32;
  if (n_vkeep < n_vrows) {
    k_rare_mark<<<rare_grid(n_kept), kRareThreads, 0, s>>>(kept, n_kept, n_vrows, n_vkeep, ws.bits, ws.owner, t.prog,
                                                           ws.bad);
    k_rare_count<<<rare_grid(W), kRareThreads, 0, s>>>(ws.bits, W, n_vrows, n_vkeep, ws.cnt);
    size_t tmp_bytes = ws.tmp_bytes;
    cub::DeviceScan::ExclusiveSum(ws.tmp, tmp_bytes, ws.cnt, ws.at, (int)(2 * W), s);
    k_rare_list<<<rare_grid(W), kRareThreads, 0, s>>>(ws.bits, W, n_vrows, n_vkeep, ws.at, ws.list, ws.n_list);
    if (t.rs > 0)
      k_rare_move<<<num_sms() * 8, kRareThreads, 0, s>>>(t.V, t.rs, ws.at, W, ws.list, ws.owner, n_vkeep, kept,
                                                         ws.bad);
    nl += 4 + (t.rs > 0);
  }
  nl += launch_table_insert(kept, n_kept, t, s);
  k_rare_commit<<<1, 1, 0, s>>>(t.state, tot, ws.bad);
  return nl + 1;
}

}  // namespace dfb
