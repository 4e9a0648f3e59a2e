// difacto_b200/csrc/shard_layout.cuh -- mailbox layout and kernel argument blocks of the NVLink-sharded store.
//
// Every rank owns ONE device allocation (the "mailbox"), exported through CUDA IPC (or used directly by peers of
// the same process).  All ranks use the same capacities, so the layout is identical everywhere and a rank
// addresses a peer's mailbox as peer_base + offset.  Everything in it is double-buffered by step parity
// (the structure exchange of step t+1 overlaps the update of step t); the step counters are not.
//
//   written by worker r into owner s's mailbox, slot [parity][r]:
//     hdr      ShardHdr                         counts of the segment
//     keys     u64 [Kseg]                       the worker's unique keys that fall into s's range (sorted)
//     cstart   i32 [Kseg+1]                     CSC column offsets of those keys (row lists in occ)
//     occ      u32|u64 [Nseg]                   per column: the rows that contain it, in row order (+ value bits)
//     rowptr   u64 [Bcap+1], ridx u32 [Nseg], rval f32 [Nseg]    the same non-zeros as a CSR over the worker's rows
//     p        f32 [Bcap], pxv f32 [Bcap][ks]   after the worker's reduce: p_i and p_i * XV_i   (fm_loss.h:155-195)
//   written by owner s into worker r's mailbox, slot [parity][s]:
//     part_xv  f32 [Bcap][ks], part_sc float2 [Bcap]    partial XV / {sum (xV)^2, sum x w} over s's keys
//   (ks = V_dim rounded up to 4 floats, the stride of the table rows)
//     pen      f64                                       penalty of the weights r "pulled" from s (sgd_learner.cc:249-273)
//   step counters (u64, one 64-byte line each): f_struct[r], f_pxv[r] (worker r -> me as owner),
//                                               f_part[s], f_done[s] (owner s -> me as worker)
#pragma once
#include "dfb_internal.cuh"

namespace dfb {

struct ShardBounds {
  int kb[9];     // key index boundaries of the owners' segments in the worker's sorted key list
  int nb[9];     // the same boundaries in the CSC payload (non-zeros)
  // 0: the batch is dropped (error raised into the step's Progress): every segment is sent empty, and the worker's
  // reduce and AUC add nothing.  A u64, so that k_auc_area can take it as its "dropped when 0" count.
  unsigned long long valid;
};

struct ShardLayout {
  int S = 1, ks = 0;
  size_t Bcap = 0, Kseg = 0, Nseg = 0;
  size_t off_hdr = 0, off_keys = 0, off_cstart = 0, off_occ = 0, off_rowptr = 0, off_ridx = 0, off_rval = 0,
         off_p = 0, off_pxv = 0, off_part_xv = 0, off_part_sc = 0, off_pen = 0, off_flags = 0, total = 0;
  size_t str_hdr = 0, str_keys = 0, str_cstart = 0, str_occ = 0, str_rowptr = 0, str_ridx = 0, str_rval = 0,
         str_p = 0, str_pxv = 0, str_part_xv = 0, str_part_sc = 0, str_pen = 0;
  // slot [parity d][index i] of a region
  template <typename T> T* at(void* base, size_t off, size_t stride, int d, int i) const {
    return reinterpret_cast<T*>(static_cast<char*>(base) + off + ((size_t)d * S + i) * stride);
  }
  enum { F_STRUCT = 0, F_PXV = 1, F_PART = 2, F_DONE = 3 };
  unsigned long long* flag(void* base, int kind, int i) const {
    return reinterpret_cast<unsigned long long*>(static_cast<char*>(base) + off_flags + ((size_t)kind * 8 + i) * 64);
  }
  static size_t al(size_t n) { return (n + 255) / 256 * 256; }
  void compute(int S_, int ks_, size_t Bcap_, size_t Kseg_, size_t Nseg_) {
    S = S_; ks = ks_; Bcap = Bcap_; Kseg = Kseg_; Nseg = Nseg_;
    size_t o = 0;
    auto region = [&](size_t& off, size_t& str, size_t bytes) { off = o; str = al(bytes); o += 2 * (size_t)S * str; };
    region(off_hdr, str_hdr, sizeof(ShardHdr));
    region(off_keys, str_keys, Kseg * 8);
    region(off_cstart, str_cstart, (Kseg + 1) * 4);
    region(off_occ, str_occ, Nseg * 8);
    region(off_rowptr, str_rowptr, (Bcap + 1) * 8);
    region(off_ridx, str_ridx, Nseg * 4);
    region(off_rval, str_rval, Nseg * 4);
    region(off_p, str_p, Bcap * 4);
    region(off_pxv, str_pxv, Bcap * (size_t)ks * 4);
    region(off_part_xv, str_part_xv, Bcap * (size_t)ks * 4);
    region(off_part_sc, str_part_sc, Bcap * 8);
    region(off_pen, str_pen, 8);
    off_flags = o;
    o += 4 * 8 * 64;
    total = al(o);
  }
};

struct SignalDst { int n; unsigned long long* flag[8]; };

struct ScatterArgs {
  int S, me;
  const ShardBounds* wb;
  const uint64_t* keys;
  const int* col_start;
  const void* occ;
  unsigned long long nrows, flags, step;
  ShardHdr* hdr_dst[8];
  uint64_t* keys_dst[8];
  int* cstart_dst[8];
  void* occ_dst[8];
};
struct RowptrDst { uint64_t* rowptr_dst[8]; };
struct FillDst { uint32_t* ridx_dst[8]; float* rval_dst[8]; };

struct ReduceArgs {
  int S, me, train, V_dim;
  size_t nrows;
  const ShardBounds* wb;       // !wb->valid: the batch was dropped, the owners computed no partials for it
  const float* part_xv[8];
  const float2* part_sc[8];
  float* p_dst[8];
  float* pxv_dst[8];
  const float* label;          // nullptr (predict steps only): no loss
  float* pred;
  DevProgress* prog;
};

struct LookupArgs {
  int S;
  size_t Kseg;
  unsigned stamp;              // 0: no sharing bookkeeping (validation steps, S == 1)
  const uint64_t* keys[8];
  const ShardHdr* hdr[8];
  int* slot;                   // [S][Kseg]
  float* w;
  int* vrow;
  int2* wv;
};

int launch_shard_wait(const unsigned long long* flags, int stride_u64, unsigned mask, unsigned long long target,
                      long long timeout_cycles, DevProgress* prog, cudaStream_t s);
int launch_shard_signal(const SignalDst& d, unsigned long long value, cudaStream_t s);
int launch_shard_bounds(const uint64_t* keys, const unsigned long long* dU, size_t U_cap, const int* col_start,
                        size_t nnz, int S, size_t Kseg, size_t Nseg, ShardBounds* wb, DevProgress* prog,
                        cudaStream_t s);
int launch_shard_scatter(const ScatterArgs& a, bool valued, size_t work_cap, cudaStream_t s);
int launch_shard_subcsr(const uint64_t* offset, const uint32_t* lidx, const float* value, size_t nrows,
                        const ShardBounds* wb, int S, int* rowcnt, const RowptrDst& rd, const FillDst& fd,
                        cudaStream_t s);
int launch_shard_reduce(const ReduceArgs& a, cudaStream_t s);
// one launch per worker, in rank order (conf / vsave: [S][Kseg] flags and [S][Kseg][ks] saved rows; unused when stamp == 0)
int launch_shard_lookup(Table& t, const LookupArgs& a, int r, bool insert, unsigned char* conf, cudaStream_t s);
// the keys all workers' segments of this step bring (the sum of min(nkeys, Kseg)) -> *out (host-mapped memory)
int launch_shard_count(const LookupArgs& a, unsigned long long* out, cudaStream_t s);
int launch_shard_pull(Table& t, const LookupArgs& a, const unsigned char* conf, float* vsave, cudaStream_t s);
int launch_shard_done(DevProgress* src_prog, DevProgress* main_prog, double* pen_dst, unsigned long long* flag_dst,
                      unsigned long long value, cudaStream_t s);
int launch_shard_collect(const double* pen_in, int stride_f64, int S, DevProgress* prog_w, DevProgress* main_prog,
                         DevProgress* stage, cudaStream_t s);

}  // namespace dfb
