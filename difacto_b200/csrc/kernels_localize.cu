// difacto_b200/csrc/kernels_localize.cu -- Localizer::Compact on the GPU (SURVEY.md 8f rank 1).
//
// GPU restatement of src/data/localizer.cc:11-103 of the reference:
//   key_j = ReverseBytes(id_j % max_index)                (CountUniqIndex :22-26, base.h:39-51)
//   sort (key, position) pairs by key                      (:28-29; here a stable LSD radix sort)
//   unique keys ascending + occurrence counts              (:36-49)
//   index_j = rank of key_j among the unique keys          (RemapIndex :53-103)
// Integer work only: bit-exact by construction (tests compare with the oracle and the reference).
//
// The same sort also yields the CSC view of the batch (per key: the rows that contain it, in row
// order) that the atomic-free gradient kernel needs, so a raw-id step skips the separate CSC sort.
#include "dfb_device.cuh"

#include <cub/cub.cuh>

namespace dfb {

namespace {

// HI32: the caller knows that only the upper 32 bits of the reversed keys can be non-zero (ids < 2^32): the sort
// then runs on 32-bit keys (a third less traffic per radix pass); the OR mask still covers all 64 bits, so a wrong
// assumption is detected by k_emit like any other range violation.
// One warp per row (coalesced).  The sort payload (Payload<KT>) depends on the key width:
//  - 32-bit keys: (row << 32) | j.  The emit reads each occurrence's row from the sorted payload: at the flagship
//    shape a per-nnz row array (26 MB) has left L2 by the time the emit gathers it at random.
//  - 64-bit keys: the position j, and the row goes to nnz_row[j].  These sorts run up to 8 passes, each of which
//    would carry 4 more payload bytes per pair both ways, while Criteo-sized batches (2.6 M nnz, row array 10 MB)
//    find the gathered rows in L2.
// Positions outside [0, n) (an offset array that does not describe n nonzeros) are skipped.
template <typename KT> struct PayloadT { using type = unsigned long long; };
template <> struct PayloadT<unsigned long long> { using type = uint32_t; };
template <typename KT> using Payload = typename PayloadT<KT>::type;

template <bool HI32>
__global__ void k_rev_keys(const uint64_t* __restrict__ ids, size_t n, const uint64_t* __restrict__ offset,
                           size_t nrows, unsigned long long max_index, unsigned long long* __restrict__ rkeys,
                           void* __restrict__ pay, uint32_t* __restrict__ nnz_row,
                           unsigned long long* __restrict__ or_all) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  unsigned long long acc = 0;
  for (size_t r = warp0; r < nrows; r += nwarps) {
    const uint64_t o0 = offset[r], o1 = offset[r + 1] < n ? offset[r + 1] : n;
    for (uint64_t j = o0 + lane; j < o1; j += 32) {
      unsigned long long x = ids[j];
      if (max_index == ~0ULL) x = (x == ~0ULL) ? 0ULL : x;   // x % (2^64-1)
      else x = x % max_index;
      const unsigned long long k = reverse_nibbles(x);
      acc |= k;
      if (HI32) {
        reinterpret_cast<uint32_t*>(rkeys)[j] = (uint32_t)(k >> 32);
        static_cast<unsigned long long*>(pay)[j] = ((unsigned long long)r << 32) | j;
      } else {
        rkeys[j] = k;
        static_cast<uint32_t*>(pay)[j] = (uint32_t)j;
        nnz_row[j] = (uint32_t)r;
      }
    }
  }
  // OR of all keys: the radix sort only needs the bit range that is not constant zero
  // (warp shuffle -> shared memory -> one atomic per block)
  __shared__ unsigned long long s_or[8];
  for (int o = 16; o > 0; o >>= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) s_or[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long a = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) a |= s_or[w];
    if (a) atomicOr(or_all, a);
  }
}

// Single-pass emit over the sorted (key, payload) pairs.  Each CTA owns one tile of kEmitTile pairs; warp w of the
// CTA owns the kEmitItems * 32 consecutive pairs starting at tile + w * 32 * kEmitItems, read 32 at a time (coalesced).
// A pair is a head when its key differs from its predecessor's; the rank of a key is the number of heads up to and
// including its first pair, minus one.  Heads are counted by warp ballots, the warp counts are scanned in the CTA, and
// the tile's offset comes from the tiles before it by decoupled look-back (CUB's ScanTileState).
constexpr int kEmitThreads = 256;
constexpr int kEmitItems = 8;
constexpr int kEmitTile = kEmitThreads * kEmitItems;
using EmitTileState = cub::ScanTileState<int>;

__global__ void k_emit_init(EmitTileState ts, int ntiles) { ts.InitializeStatus(ntiles); }

// Emits unique keys, per-key segment bounds, the remapped CSR index and the per-occurrence payload (row [, x]) in
// key-then-row order.  RANKS = false: no remapped index (lidx_out is not written; the step that follows probes the
// table with the raw ids instead), which saves the random 4-byte scatter of the inverse permutation.
template <typename KT, bool RANKS>
__global__ void __launch_bounds__(kEmitThreads)
k_emit(const KT* __restrict__ skeys, const Payload<KT>* __restrict__ spay, const uint32_t* __restrict__ nnz_row,
       size_t n, const float* __restrict__ value, uint64_t* __restrict__ keys_out, int* __restrict__ col_start,
       int* __restrict__ col_end, uint32_t* __restrict__ lidx_out, uint32_t* __restrict__ occ_row,
       unsigned long long* __restrict__ occ_rowx, unsigned long long* __restrict__ scal, int begin_bit,
       DevProgress* prog, EmitTileState ts) {
  using PrefixOp = cub::TilePrefixCallbackOp<int, ::cuda::std::plus<int>, EmitTileState>;
  __shared__ typename PrefixOp::TempStorage s_prefix;
  __shared__ int s_warp[kEmitThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tile = blockIdx.x;
  const size_t base = (size_t)tile * kEmitTile + (size_t)warp * (32 * kEmitItems) + lane;
  Payload<KT> pay[kEmitItems];
  int before[kEmitItems];     // heads of this warp's pairs before pair i
  unsigned heads = 0;         // bit i: pair i is a head
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < kEmitItems; ++i) {
    const size_t j = base + (size_t)i * 32;
    bool h = false;
    pay[i] = 0;
    if (j < n) {
      pay[i] = spay[j];
      h = j == 0 || skeys[j] != skeys[j - 1];
    }
    const unsigned b = __ballot_sync(0xffffffffu, h);
    before[i] = cnt + __popc(b & ((1u << lane) - 1u));
    cnt += __popc(b);
    heads |= (unsigned)h << i;
  }
  if (lane == 0) s_warp[warp] = cnt;
  __syncthreads();
  if (warp == 0) {
    const int c = lane < kEmitThreads / 32 ? s_warp[lane] : 0;
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    int prefix = 0;
    if (tile == 0) {
      if (lane == 0) ts.SetInclusive(0, total);
    } else {
      PrefixOp op(ts, s_prefix, ::cuda::std::plus<int>(), tile);
      prefix = __shfl_sync(0xffffffffu, op(total), 0);   // valid in lane 0
    }
    __syncwarp();
    if (lane < kEmitThreads / 32) s_warp[lane] = prefix + incl - c;
  }
  __syncthreads();
  const int off = s_warp[warp] - 1;
#pragma unroll
  for (int i = 0; i < kEmitItems; ++i) {
    const size_t j = base + (size_t)i * 32;
    if (j >= n) break;
    const bool h = (heads >> i) & 1u;
    const int r = off + before[i] + (h ? 1 : 0);
    const uint32_t p = (uint32_t)pay[i];
    const bool in = p < n;          // false only for a pair k_rev_keys skipped (its payload is stale)
    uint32_t row = 0;
    if (sizeof(KT) == 4) row = (uint32_t)((unsigned long long)pay[i] >> 32);
    else if (in) row = nnz_row[p];
    if (RANKS && in) lidx_out[p] = (uint32_t)r;
    if (value) occ_rowx[j] = ((unsigned long long)row << 32) | (unsigned long long)__float_as_uint(in ? value[p] : 0.f);
    else occ_row[j] = row;
    if (h) {
      const KT k = skeys[j];    // read in the first pass: a cache hit
      keys_out[r] = sizeof(KT) == 4 ? ((uint64_t)k << 32) : (uint64_t)k;
      col_start[r] = (int)j;
      if (j > 0) col_end[r - 1] = (int)j;
    }
    if (j == n - 1) {
      col_end[r] = (int)n;
      col_start[r + 1] = (int)n;      // col_start doubles as the U+1 column offsets of the CSC view
      // scal = {OR of all keys, number of unique keys}.  A key bit below the sorted range means the range was
      // assumed too narrow (id_bits / the range learned from earlier batches): the batch is NOT sorted, so it is
      // dropped (zero keys).  The single-GPU step sees the zero and reports the drop in stream order (prog ==
      // nullptr here: this kernel runs on the localizer's stream, concurrently with the previous step's Progress).
      const unsigned long long low = begin_bit > 0 ? (scal[0] & ((1ULL << begin_bit) - 1ULL)) : 0ULL;
      if (low != 0ULL) {
        scal[1] = 0ULL;
        if (prog) raise_err(prog, kErrIdRange);
      } else {
        scal[1] = (unsigned long long)(r + 1);
      }
    }
  }
}

__global__ void k_cnt_from_cols(const int* __restrict__ col_start, const int* __restrict__ col_end, size_t n,
                                float* __restrict__ cnt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cnt[i] = (float)(col_end[i] - col_start[i]);   // idx_frq, localizer.cc:41-46
}

}  // namespace

// temporary storage of the localizer: the emit's tile states, then the radix sort's workspace
static size_t emit_state_bytes(size_t nnz) {
  size_t b = 0;
  EmitTileState::AllocationSize((int)((nnz + kEmitTile - 1) / kEmitTile), b);
  return (b + 255) & ~(size_t)255;
}

size_t localize_sort_tmp_bytes(size_t nnz) {
  size_t b1 = 0, b2 = 0;
  const int n = (int)(nnz ? nnz : 1);
  cub::DeviceRadixSort::SortPairs(nullptr, b1, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, n);
  cub::DeviceRadixSort::SortPairs(nullptr, b2, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);
  return emit_state_bytes(n) + (b1 > b2 ? b1 : b2);
}

// pay (8 bytes per nnz): hi32: the (row << 32) | position payload; otherwise the u32 position payload in its first
// half and the u32 row array in its second half
int launch_localize_keys(const uint64_t* ids, size_t nnz, uint64_t max_index, unsigned long long* rkeys, void* pay,
                         unsigned long long* or_all, const uint64_t* offset, size_t nrows, bool hi32, cudaStream_t s) {
  cudaMemsetAsync(or_all, 0, sizeof(unsigned long long), s);
  if (nnz == 0) return 0;
  size_t need = (nrows + 7) / 8;
  int grid = (int)(need < (size_t)(num_sms() * 8) ? (need ? need : 1) : (size_t)(num_sms() * 8));
  uint32_t* nnz_row = static_cast<uint32_t*>(pay) + nnz;
  if (hi32) k_rev_keys<true><<<grid, 256, 0, s>>>(ids, nnz, offset, nrows, max_index, rkeys, pay, nullptr, or_all);
  else      k_rev_keys<false><<<grid, 256, 0, s>>>(ids, nnz, offset, nrows, max_index, rkeys, pay, nnz_row, or_all);
  return 1;
}

// hi32 must be what launch_localize_keys was given (it implies begin_bit >= 32); pay is what it wrote
int launch_localize_sort(const unsigned long long* rkeys, const void* pay, size_t nnz, int begin_bit, bool hi32,
                         unsigned long long* skeys, void* spay, void* tmp, size_t tmp_bytes, const float* value,
                         uint64_t* keys_out, int* col_start, int* col_end, uint32_t* lidx_out, void* occ_sorted,
                         unsigned long long* scal, DevProgress* prog, cudaStream_t s) {
  cudaMemsetAsync(scal + 1, 0, sizeof(unsigned long long), s);
  if (nnz == 0) return 0;
  const int ntiles = (int)((nnz + kEmitTile - 1) / kEmitTile);
  const size_t ts_bytes = emit_state_bytes(nnz);
  if (tmp_bytes < ts_bytes) return -1;
  EmitTileState ts;
  if (ts.Init(ntiles, tmp, ts_bytes) != cudaSuccess) return -1;
  void* sort_tmp = static_cast<char*>(tmp) + ts_bytes;
  size_t sort_bytes = tmp_bytes - ts_bytes;
  uint32_t* occ_row = reinterpret_cast<uint32_t*>(occ_sorted);
  unsigned long long* occ_rowx = reinterpret_cast<unsigned long long*>(occ_sorted);
  int passes;
  if (hi32) {
    const uint32_t* rk = reinterpret_cast<const uint32_t*>(rkeys);
    uint32_t* sk = reinterpret_cast<uint32_t*>(skeys);
    const auto* pv = static_cast<const unsigned long long*>(pay);
    auto* spv = static_cast<unsigned long long*>(spay);
    const int bb = begin_bit >= 32 ? begin_bit - 32 : 0;
    if (cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, rk, sk, pv, spv, (int)nnz, bb, 32, s) != cudaSuccess) return -1;
    k_emit_init<<<(ntiles + 255) / 256, 256, 0, s>>>(ts, ntiles);
    auto emit = lidx_out ? k_emit<uint32_t, true> : k_emit<uint32_t, false>;
    emit<<<ntiles, kEmitThreads, 0, s>>>(sk, spv, nullptr, nnz, value, keys_out, col_start, col_end, lidx_out, occ_row,
                                         occ_rowx, scal, begin_bit >= 32 ? begin_bit : 32, prog, ts);
    passes = (32 - bb + 7) / 8;
  } else {
    const auto* pv = static_cast<const uint32_t*>(pay);
    auto* spv = static_cast<uint32_t*>(spay);
    if (cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, rkeys, skeys, pv, spv, (int)nnz, begin_bit, 64, s) != cudaSuccess) return -1;
    k_emit_init<<<(ntiles + 255) / 256, 256, 0, s>>>(ts, ntiles);
    auto emit = lidx_out ? k_emit<unsigned long long, true> : k_emit<unsigned long long, false>;
    emit<<<ntiles, kEmitThreads, 0, s>>>(skeys, spv, pv + nnz, nnz, value, keys_out, col_start, col_end, lidx_out,
                                         occ_row, occ_rowx, scal, begin_bit, prog, ts);
    passes = (64 - begin_bit + 7) / 8;
  }
  return 3 + passes;
}

__global__ void k_raise_err(DevProgress* prog, int code) { raise_err(prog, code); }

int launch_raise_err(DevProgress* prog, int code, cudaStream_t s) {
  k_raise_err<<<1, 1, 0, s>>>(prog, code);
  return 1;
}

// the range check of a batch that is scored without the localizer: clears *ok when an id (as Localizer(-1) maps it)
// is not below 2^nbits, i.e. when the localizer's sort over the same range would have dropped the batch
__global__ void __launch_bounds__(256) k_id_range(const unsigned long long* __restrict__ ids, size_t n, int nbits,
                                                  unsigned long long* ok) {
  unsigned long long acc = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long x = __ldg(ids + i);
    acc |= x == ~0ULL ? 0ULL : x;
  }
  if (__any_sync(0xffffffffu, (acc >> nbits) != 0ULL) && (threadIdx.x & 31) == 0) *ok = 0ULL;
}

int launch_id_range(const uint64_t* ids, size_t n, int nbits, unsigned long long* ok, cudaStream_t s) {
  if (n == 0 || nbits >= 64) return 0;
  const size_t need = (n + 255) / 256;
  const int grid = (int)(need < (size_t)num_sms() * 8 ? need : (size_t)num_sms() * 8);
  k_id_range<<<grid, 256, 0, s>>>(reinterpret_cast<const unsigned long long*>(ids), n, nbits, ok);
  return 1;
}

int launch_cnt_from_cols(const int* col_start, const int* col_end, size_t n, float* cnt, cudaStream_t s) {
  if (n == 0) return 0;
  k_cnt_from_cols<<<(int)((n + 255) / 256), 256, 0, s>>>(col_start, col_end, n, cnt);
  return 1;
}

}  // namespace dfb
