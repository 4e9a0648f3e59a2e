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

// the slot's entry as {key | vrow, pad}, {fea_cnt | w, sqrt_g | z}; 1: kept, 2: dropped, 0: empty
__device__ __forceinline__ int prune_kind(const ulonglong2& a, const ulonglong2& b, float max_count) {
  if (a.x == kEmptyKey) return 0;
  const int vrow = (int)(unsigned)(a.y & 0xffffffffULL);
  const float fea_cnt = __uint_as_float((unsigned)(b.x & 0xffffffffULL));
  const float w = __uint_as_float((unsigned)(b.x >> 32));
  return (vrow < 0 && w == 0.f && fea_cnt <= max_count) ? 2 : 1;
}

// tot = {kept, dropped}; blk_kept[b] = the entries block b keeps (both zeroed by the caller)
__global__ void __launch_bounds__(kPruneThreads) k_prune_count(const Entry* __restrict__ tab, uint64_t cap,
                                                               float max_count, unsigned long long* __restrict__ tot,
                                                               unsigned* __restrict__ blk_kept) {
  const ulonglong2* in = reinterpret_cast<const ulonglong2*>(tab);
  unsigned kept = 0, dropped = 0;
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
      const int k = prune_kind(a[j], b[j], max_count);
      kept += k == 1;
      dropped += k == 2;
    }
  }
  kept = __reduce_add_sync(kFullMask, kept);
  dropped = __reduce_add_sync(kFullMask, dropped);
  if (prune_lane() == 0) {
    if (kept) {
      atomicAdd(&tot[0], (unsigned long long)kept);
      atomicAdd(&blk_kept[blockIdx.x], kept);
    }
    if (dropped) atomicAdd(&tot[1], (unsigned long long)dropped);
  }
}

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
      k[j] = prune_kind(a[j], b[j], max_count);
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

}  // namespace

int prune_grid(uint64_t cap) {
  const uint64_t tiles = (cap + kPruneTile - 1) / kPruneTile;
  const uint64_t g = (uint64_t)num_sms() * 8;
  return (int)(tiles < g ? (tiles ? tiles : 1) : g);
}

int launch_prune_count(const Table& t, float max_count, int grid, unsigned long long* tot, unsigned* blk_kept,
                       cudaStream_t s) {
  k_prune_count<<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, tot, blk_kept);
  return 1;
}

int launch_prune_rebuild(Table& t, float max_count, int grid, const unsigned long long* tot, const unsigned* blk_kept,
                         Entry* kept, uint64_t n_kept, cudaStream_t s) {
  k_prune_compact<<<grid, kPruneThreads, 0, s>>>(t.tab, t.cap, max_count, blk_kept, kept);
  int nl = 1 + launch_table_insert(kept, n_kept, t, s);
  k_prune_commit<<<1, 1, 0, s>>>(t.state, tot);
  return nl + 1;
}

}  // namespace dfb
