// difacto_b200/csrc/dfb_internal.cuh -- shared declarations of the sm_90a engine.
//
// Data layout in HBM (one shard = one GPU):
//   Entry tab[cap]        32-byte open-addressing hash entries, one DRAM sector each:
//                         {u64 reversed key, i32 vrow, i32 pad, f32 fea_cnt, w, sqrt_g, z}
//                         == the reference's unordered_map<feaid_t,SGDEntry> (sgd_updater.h:19-29,84)
//   float VV[vcap][2*ks]  one row per key with an embedding: [V (ks) | AdaGrad accumulators (ks)],
//                         ks = V_dim rounded up to 4 floats -- the reference's `new real_t[2n]`
//                         (sgd_updater.cc:142).  The gather reads the first half (one contiguous
//                         4k-byte chunk); the update reads and writes the whole 8k-byte row.
//                         A scoring-only engine (score_only = 1) holds V only: VV[vcap][ks] of fp32 or bf16 elements
//                         (Table::rs == ks, Table::vonly), and nothing that trains or saves runs on it.
// V rows are allocated lazily from a bump pool, exactly when the reference calls InitV.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace dfb {

struct __align__(32) Entry {
  unsigned long long key;
  int vrow;       // -1: no V allocated (SGDEntry::V == nullptr)
  int pad;
  float fea_cnt, w, sqrt_g, z;
};
static_assert(sizeof(Entry) == 32, "Entry must be one 32-byte sector");

constexpr unsigned long long kEmptyKey = ~0ULL;  // ReverseBytes(id % (2^64-1)) never yields it

// SGDUpdaterParam (src/sgd/sgd_param.h:66-107)
struct Params {
  float l1, l2, V_l2, lr, lr_beta, V_lr, V_lr_beta, V_init_scale;
  int V_dim, V_threshold;
  unsigned seed;
};

// accumulated on device, read back by dfb_read_progress
struct DevProgress {
  double loss, penalty, auc;
  unsigned long long nrows, new_keys, new_vrows;
  int err;        // sticky dfb_status raised by a kernel (capacity, invalid lens ...), or kErrIdRange
  int pad;
};
// DevProgress::err of a raw batch the GPU localizer dropped because its ids fall outside the sorted bit range;
// reported to the caller as DFB_ERR_INVALID with a message that names the range
constexpr int kErrIdRange = -100;

// device-resident mutable scalars of the table
struct TableState {
  unsigned long long n_keys;
  unsigned long long n_vrows;
  unsigned int seed;     // SGDUpdaterParam::seed as advanced by rand_r (sgd_updater.cc:144)
  unsigned int pad;
};

struct Table {
  Entry* tab = nullptr;
  uint64_t cap = 0, mask = 0, max_keys = 0;   // slots (power of 2, >= 2 max_keys), cap - 1, keys it may hold
  float* V = nullptr;
  float* Vcg = nullptr;
  uint64_t vcap = 0;
  int ks = 0;  // V_dim rounded up to a multiple of 4 floats
  int rs = 0;  // stride between table rows in elements: 2*ks floats, Vcg == V + ks; a scoring-only engine: ks, no Vcg
  int vonly = 0;   // a scoring-only engine's rows: 1 = fp32 V, 2 = bf16 V (V then points at 2-byte elements; only the
                   // restore's scoring insert and the bf16 raw forward touch them).  0: the training layout
  TableState* state = nullptr;
  DevProgress* prog = nullptr;
};

// how a kernel finds w / V (and where it puts the gradient) for local key u of a batch
struct FmView {
  // w = wbase[w_pos ? w_pos[u] : u]; w_pos[u] == -1 -> 0
  const float* wbase;
  const int* w_pos;
  // optional packed pulled view {bits(w), vrow} per key: one 8-byte load per nnz instead of two
  // 4-byte loads from different arrays (fast kernel only; overrides wbase/w_pos/v_pos when set)
  const int2* wv;
  // V row = vbase + (int64)r * vstride, r = v_pos[u] (or u when dense && v_pos[u] >= 0); -1 -> absent
  const float* vbase;
  const int* v_pos;
  long long vstride;
  int dense;
  // gradient destinations (TRAIN): gw[gw_pos ? gw_pos[u] : u], gV row = gvbase + r' * gvstride with
  // r' = (gv_pos ? gv_pos[u] : u); gxxp[u] (only when values are present)
  float* gwbase;
  const int* gw_pos;
  float* gvbase;
  const int* gv_pos;
  long long gvstride;
  float* gxxp;
  // 1: per-load L2 policies -- the V rows are touched once (evict_first)
  int l2hint;
  // 1: the pulled view {w,vrow} is re-read per nnz and fits in L2 with room to spare (evict_last); 0: normal policy
  int wv_last;
  // the raw-id forward (launch_fm_raw): the hash table that each nonzero's id is looked up in, find only
  const Entry* tab;
  unsigned long long tab_mask;
};

// where the worker's gradient rows go: locally contiguous (nseg == 0) or, per owner segment of the
// sorted key list, straight into that owner's receive buffer over NVLink (peer pointers)
struct SegDst {
  int nseg;
  int rot;            // first key (multiple of 32) this rank starts with: staggers the peers' inbound traffic
  int bounds[9];      // key index boundaries of the segments (nseg + 1 used)
  float* gw[8];       // per segment: destination of gw for the segment's first key
  float* gV[8];       // per segment: destination row of gV for the segment's first key
};

// owner side of the fused sharded store (SRC 2 of k_bwd_update): what differs from the single-GPU update
struct ShardApply {
  const float* w_pulled;        // w of every key as pulled at step start (penalty of the pulled weights)
  const unsigned char* conf;    // != 0: a lower-rank worker's push already updated this key in this step ...
  const float* vsave;           // ... and this is its V row as pulled at step start ([n][ks])
};

// very hot keys (a Criteo feature that occurs in most rows of a batch): their occurrence lists are cut into chunks
// that are reduced by separate warps beforehand (k_hot_reduce), in a fixed order, so that no single warp walks a
// 65536-row list; k_bwd_update then adds the chunk partials in chunk order (bit-reproducible)
struct HotPart {
  const int* hotmap;        // per key: first chunk id (only valid for keys longer than `split`), < 0: not pre-reduced
  const float* part;        // [chunks][ks] partial sum_occ x * pXV[row]
  const float2* part_s;     // [chunks] partial {sum x p, sum x^2 p}
  int split, chunk;         // lists longer than split are cut into chunks of `chunk` occurrences; part == nullptr: off
};
struct HotWs {              // device workspaces of the pre-reduction
  int* hotmap; int2* info; float* part; float2* part_s; unsigned long long* counter; int cap;
};

// forward "partials" of the fused sharded store (MODE 3 of k_fm_fast): the owner of a key segment computes,
// for every row of every worker's minibatch, the part of the FM interaction that is linear in ITS rows
//   XV_i^(s) = sum_{j in segment s} x_ij V_j,  sum_j (x_ij V_j)^2,  sum_j x_ij w_j
// and stores it straight into that worker's mailbox (peer memory over NVLink).
// what a worker tells the owner of a key segment about its minibatch (written into the owner's mailbox)
struct ShardHdr {
  unsigned long long nkeys;   // keys of the worker's batch that fall into this owner's range
  unsigned long long nnz;     // non-zeros over those keys
  unsigned long long nrows;   // rows of the worker's batch
  unsigned long long flags;   // bit 0: is_train, bit 1: push_cnt, bit 2: valued
  unsigned long long step;
  unsigned long long pad[3];
};
static_assert(sizeof(ShardHdr) == 64, "ShardHdr is one 64-byte record");
__host__ __device__ inline unsigned long long shard_hdr_nrows(const ShardHdr* h) { return h->nrows; }

struct PartSrc {
  const uint64_t* rowptr;   // [nrows+1] offsets into ridx (this worker's rows restricted to my key segment)
  const uint32_t* ridx;     // key index relative to the segment
  const float* rval;        // values (nullptr: binary)
  const int2* wv;           // pulled view {bits(w), vrow} of the segment's keys
  const ShardHdr* hdr;      // nrows of the worker's batch
  float* out_xv;            // [nrows][ks]   (peer memory)
  float2* out_sc;           // [nrows] {sum (xV)^2, sum x w}
};
struct PartArgs {
  int nsrc, rot;            // rot: first source this owner starts with (staggers the peers' inbound traffic)
  unsigned long long bcap;  // rows are enumerated as src * bcap + row
  PartSrc s[8];
};

struct FmBatch {
  size_t nrows;
  const uint64_t* offset;   // size_t offsets, as in dmlc::RowBlock (dmlc/data.h:141)
  const uint32_t* index;
  const float* value;       // nullptr: binary features
  const float* label;
  const float* pred_in;     // CalcGrad with a caller-provided pred (fm_loss.h:155-161), else nullptr
  float* pred_io;           // output; accumulated into when pred_acc
  int pred_acc;
  int V_dim;
  int train;
  DevProgress* prog;        // loss / nrows accumulated here when non-null
  // emit mode (train && emit): instead of scattering with atomics the kernel writes
  int emit;
  float* p_out;             //   p_i = -y/(1+exp(y pred_i))            [nrows]
  float* pxv_out;           //   p_i * XV_i                             [nrows][ks]
  uint32_t* occ_row;        //   row of every nnz (binary data)         [nnz]
  unsigned long long* occ_rowx;  // (row << 32 | bits(x)) (valued data) [nnz]
  // long rows (predict / emit on the fast path): rows of >= long_nnz nonzeros are left to k_fm_long, where a whole
  // CTA walks one row (0 = one warp per row whatever its length); nnz_hint = the batch's nnz when the host knows it
  unsigned long_nnz;
  size_t nnz_hint;
  // the device-side key count of a batch the GPU localizer produced (nullptr: none).  0 there (with nnz > 0) means
  // the localizer dropped the batch: the kernels then return at once, without reading the batch's ranks, and the
  // forward raises kErrIdRange into prog
  const unsigned long long* dev_nkeys;
  // the raw feature id of every nnz (launch_fm_raw: replaces index)
  const uint64_t* ids;
};

// true when the specialised (16-byte-lane) kernels serve this V_dim: 0 <= V_dim <= 128
bool fm_fast_supported(int V_dim);

// The specialised kernels' lane-group width for a V_dim: the smallest K in {8,16,32,64,128} with K >= V_dim (V_dim 0:
// 8), 0 above 128.  A row is handled by K/4 lanes of one float4 each; every per-row buffer has the stride
// ks = V_dim rounded up to 4 <= K, and the lanes whose float4 starts at or beyond ks load and store nothing.  The
// kernels take that predicate as a template flag PAD = (V_dim != K): their PAD = false instantiations are the
// exact-width code.
inline int fast_lane_width(int V_dim) {
  if (V_dim < 0 || V_dim > 128) return 0;
  int K = 8;
  while (K < V_dim) K *= 2;
  return K;
}
// f(std::integral_constant<int, K>{}) for K = fast_lane_width(V_dim); -1 when V_dim has no fast kernels
template <typename F>
int with_lane_width(int V_dim, F&& f) {
  switch (fast_lane_width(V_dim)) {
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 128: return f(std::integral_constant<int, 128>{});
  }
  return -1;
}

// streaming multiprocessors of the current device (cached per device); the grid-stride kernels cap their
// grids at a multiple of it
int num_sms();
// L2 cache of the current device in bytes (cached per device)
size_t l2_bytes();

// ---- launchers (kernels_fm.cu) ----
// returns number of kernel launches performed, or <0 on invalid configuration
// kLaunchRefused: the device refused the generic kernel's launch (its error in *launch_err when given)
constexpr int kLaunchRefused = -2;
int launch_fm(const FmBatch& b, const FmView& v, int force_generic, cudaStream_t s,
              cudaError_t* launch_err = nullptr);
// predict only, on raw ids (b.ids): the specialised kernels probe the table (v.tab) for each nonzero's key instead of
// reading a pulled view; v.vbase / vstride = the table rows.  -1 when V_dim has no specialised kernels.
// bf16_rows (predict only; a scoring-only engine with V_storage = bf16): v.vbase points at bf16 elements and vstride
// counts them; each lane widens its 4 columns to fp32 and everything after the load is the fp32 kernels' code
int launch_fm_raw(const FmBatch& b, const FmView& v, bool bf16_rows, cudaStream_t s);
// MODE 3: partial interaction sums of every source's rows (see PartArgs); v.vbase/vstride = the table rows.
// bf16_rows: a scoring-only owner's bf16 V rows, widened in the row load as in launch_fm_raw
int launch_fm_partial(int V_dim, bool valued, bool bf16_rows, const FmView& v, const PartArgs& pa, cudaStream_t s);
int launch_grad_finalize(int V_dim, size_t nkeys, const float* weights, const int* V_pos,
                         const float* xxp, float* grad, cudaStream_t s);

int launch_grad_finalize_dense(int V_dim, int ks, size_t nkeys, const int* hasv, const float* V,
                               const float* xxp, float* gV, cudaStream_t s);

// ---- launchers (kernels_table.cu) ----
int launch_table_init(Table& t, unsigned seed, cudaStream_t s);
// empties new_t (new_t.cap >= old_t.cap slots) and re-inserts every entry of old_t into it, bytes unchanged
int launch_table_rehash(const Table& old_t, const Table& new_t, cudaStream_t s);
// inserts the n entries src[n] (distinct keys, none in t), all 32 bytes as they are, into t: k_table_rehash's insert
int launch_table_insert(const Entry* src, uint64_t n, const Table& t, cudaStream_t s);
// find (or insert) keys; slot_out[i] = hash position or -1.  When pull outputs are non-null also
// emits w and vrow of each entry.
// n is a host count, or (dn != nullptr) the capacity with the actual count read from the device
int launch_lookup(Table& t, const uint64_t* keys, size_t n, const unsigned long long* dn, bool insert,
                  int* slot_out, float* w_out, int* vrow_out, int2* wv_out, cudaStream_t s);
// SGDUpdater::Update(kFeaCount) incl. the InitV pass.  flags/pos/cub_tmp are workspaces of n ints.
// counts: cnt[n], or (cnt == nullptr) the differences of cnt_cols[n+1].  ws: (n+31)/32 + 2 ints.
int launch_feacnt(Table& t, const Params& p, const int* slot, size_t n, const unsigned long long* dn,
                  const float* cnt, const int* cnt_cols, int* flags, int* ws, cudaStream_t s);
size_t scan_tmp_bytes(size_t n);
size_t sort_tmp_bytes(size_t n);
// InitV for flagged keys, consuming the rand_r stream in key order (sgd_updater.cc:140-147)
int launch_initv(Table& t, const Params& p, const int* slot, size_t n, const unsigned long long* dn,
                 int* flags, int* ws, cudaStream_t s);
// SGDUpdater::Get packing: lens -> scan -> ragged [w, V...] (sgd_updater.cc:32-56)
int launch_pack_ragged(Table& t, const Params& p, const int* slot, size_t n, int* lens, int* pos,
                       float* vals, unsigned long long* nvals_out, void* cub_tmp, size_t cub_bytes,
                       cudaStream_t s);
// dense rows for the sharded store: w[n], hasv[n] (-1/1), V[n][ks]
int launch_gather_rows(Table& t, const int* slot, size_t n, float* w_out, int* hasv_out,
                       int* hasv_out2, float* V_out, cudaStream_t s);
// FTRL/AdaGrad from per-key dense gradient rows (fused path and sharded push).
//   pull_vrow[i] >= 0 <=> the worker saw a V row at pull time (lens[i] > 1); when
//   vrow_is_flag the actual row is taken from the entry.
//   xxp_mode 0: gV is the complete gradient; 1: grad_V = gV - V*gxxp[i]; 2: grad_V = gV - V*gw[i]
//   (binary data, where XXp == grad_w).
int launch_update_dense(Table& t, const Params& p, const int* slot, const int* pull_vrow,
                        int vrow_is_flag, size_t n, const float* gw, const float* gxxp,
                        const float* gV, int* flags, int accumulate_penalty, int xxp_mode,
                        cudaStream_t s);
// FTRL/AdaGrad from the reference's ragged gradient layout (sgd_updater.cc:74-98)
int launch_update_ragged(Table& t, const Params& p, const int* slot, size_t n, const float* grads,
                         const int* lens_or_null, const int* pos, int* flags, cudaStream_t s);
// penalty over a pulled view without updating (validation batches, sharded worker)
int launch_penalty(const Params& p, DevProgress* prog, const float* w_arr, const int* vrow,
                   const float* V, int ks, int dense, size_t n, const unsigned long long* dn, cudaStream_t s);
int launch_pull_view(Table& t, const int* slot, size_t n, const unsigned long long* dn, float* w_out,
                     int* vrow_out, int2* wv_out, cudaStream_t s);
int launch_lens_scan(const int* lens, size_t n, int* pos, void* cub_tmp, size_t cub_bytes,
                     cudaStream_t s);
// Loss::Evaluate / BinClassMetric::AUC on device; results added to prog (or written to out)
int launch_evaluate(const float* label, const float* pred, size_t n, double* out, cudaStream_t s);
// dev_nkeys: as FmBatch::dev_nkeys (a dropped batch adds nothing), or nullptr
int launch_auc(const float* label, const float* pred, size_t n, float* key_tmp2, float* val_tmp2,
               void* cub_tmp, size_t cub_bytes, double* out_add, const unsigned long long* dev_nkeys, cudaStream_t s);
// raises a dfb_status (or kErrIdRange) into prog, in stream order
int launch_raise_err(DevProgress* prog, int code, cudaStream_t s);
int launch_restore(Table& t, const uint64_t* keys, size_t n, const float* scal, const int* vrow,
                   unsigned long long n_vrows, unsigned seed, cudaStream_t s);
int launch_read_entries(Table& t, const int* slot, size_t n, float* scal, int* hasv, float* V,
                        float* cg, int k, cudaStream_t s);

// ---- streamed checkpoint (kernels_checkpoint.cu, host side in checkpoint.cu) ----
// the writer histograms the table by the top kCkptBinBits bits of the reversed key: [2^20] keys and V rows per bin
constexpr int kCkptBinBits = 20;
// DevProgress::err codes of the reader, mapped to messages by checkpoint.cu (the table is cleared on either)
constexpr int kErrCkptDup = -101;     // a restored key was already in the table
constexpr int kErrCkptRange = -102;   // a key outside the declared source part's range
// the workspace of one writer pass of n records
struct CkptWs {
  unsigned long long *keys_in, *keys_out, *counter;
  unsigned *slots_in, *slots_out, *hv, *vbefore;
  void* tmp;
  size_t tmp_bytes;
  unsigned* out;      // the pass's packed records
};
int launch_ckpt_hist(const Table& t, unsigned* nk, unsigned* nv, cudaStream_t s);
size_t ckpt_sort_tmp_bytes(size_t n);
// the v1 records of the keys whose bin lies in [b0, b1) (n of them), in ascending key order, packed into ws.out
int launch_ckpt_pass(const Table& t, unsigned b0, unsigned b1, size_t n, int aux, int k, const CkptWs& ws,
                     cudaStream_t s);
size_t rst_scan_tmp_bytes(size_t n);
// n records of a chunk (roff: word offset of each record in buf): keep this shard's keys and insert them.  A table of
// V-only rows (t.vonly) gets V alone, rounded to nearest even when the rows are bf16; the records' cg is skipped
int launch_rst_chunk(Table& t, const unsigned* buf, const unsigned* roff, size_t n, int aux, int k, unsigned part,
                     unsigned nparts, unsigned shard, unsigned nshards, unsigned long long* flags,
                     unsigned long long* rank, void* tmp, size_t tmp_bytes, cudaStream_t s);
int launch_rst_seed(Table& t, unsigned seed, cudaStream_t s);

// ---- dfb_prune (kernels_prune.cu, host side in prune.cu) ----
// an entry is dropped when w == 0, it has no V row and fea_cnt <= max_count.  Both launches run prune_grid(t.cap)
// blocks.  count: tot[2] = {kept, dropped} and blk_kept[grid] (zeroed by the caller).  rebuild: the kept entries into
// kept[n_kept] (n_kept = tot[0]), the slots emptied, the kept entries re-inserted, n_keys lowered by tot[1].
int prune_grid(uint64_t cap);
// rare (dfb_prune_rare): an entry is dropped when fea_cnt <= max_count alone, and tot[4] = {kept, dropped, kept V rows,
// dropped V rows}
int launch_prune_count(const Table& t, float max_count, int grid, unsigned long long* tot, unsigned* blk_kept,
                       cudaStream_t s, bool rare = false);
int launch_prune_rebuild(Table& t, float max_count, int grid, const unsigned long long* tot, const unsigned* blk_kept,
                         Entry* kept, uint64_t n_kept, cudaStream_t s);
// ---- dfb_prune_rare: the V-row pool's compaction over W = ceil(n_vrows / 32) bitmap words (DESIGN.md section 10.1)
struct RareWs {
  unsigned* bits;        // [W], zeroed by the caller
  int* owner;            // [n_vrows - n_vkeep]: the workspace entry of each kept row at or above n_vkeep
  unsigned *cnt, *at;    // [2W] each: holes and movers per word, and their exclusive scan
  int* list;             // [n_list]: the holes' rows, then the movers' rows
  size_t n_list;
  void* tmp;             // rare_scan_tmp_bytes(W)
  size_t tmp_bytes;
  unsigned* bad;         // zeroed by the caller; set (and DFB_ERR_INVALID raised into t.prog) when a kept row is owned
                         // twice or lies outside [0, n_vrows): then no row moves and n_vrows is not lowered
};
size_t rare_scan_tmp_bytes(size_t W);
// the rare rebuild: the kept entries into kept[n_kept] and the slots emptied (as launch_prune_rebuild), then, when rows
// were dropped (n_vkeep < n_vrows), every kept row at or above n_vkeep moved into a hole below it and its workspace
// entry pointed there; the kept entries re-inserted; n_keys lowered by tot[1] and n_vrows by tot[3]
int launch_prune_rare(Table& t, float max_count, int grid, const unsigned long long* tot, const unsigned* blk_kept,
                      Entry* kept, uint64_t n_kept, uint64_t n_vrows, uint64_t n_vkeep, const RareWs& ws,
                      cudaStream_t s);

// ---- GPU localizer (kernels_localize.cu): Localizer::Compact + the CSC view from one radix sort ----
size_t localize_sort_tmp_bytes(size_t nnz);
// hi32: sort on the upper 32 key bits only (the caller knows the lower 32 are zero: ids < 2^32); verified on the device
// pay / spay: 8 bytes per nnz, the sort payload (and on the 64-bit-key path the row of every nnz); see
// kernels_localize.cu.  offset must describe the nnz ids as CSR: positions no row covers are not localized.
// lidx_out may be nullptr when nothing reads the remapped CSR index.
int launch_localize_keys(const uint64_t* ids, size_t nnz, uint64_t max_index, unsigned long long* rkeys, void* pay,
                         unsigned long long* or_all, const uint64_t* offset, size_t nrows, bool hi32, cudaStream_t s);
int launch_localize_sort(const unsigned long long* rkeys, const void* pay, size_t nnz, int begin_bit,
                         bool hi32, unsigned long long* skeys, void* spay, void* tmp, size_t tmp_bytes,
                         const float* value, uint64_t* keys_out, int* col_start, int* col_end, uint32_t* lidx_out,
                         void* occ_sorted, unsigned long long* scal /* {or_all, n_unique} */,
                         DevProgress* prog /* nullptr: a dropped batch (n_unique = 0) is the caller's to report */,
                         cudaStream_t s);
int launch_cnt_from_cols(const int* col_start, const int* col_end, size_t n, float* cnt, cudaStream_t s);
// *ok (set non-zero by the caller) is cleared when an id of the n, mapped as Localizer(-1) maps it, is >= 2^nbits
int launch_id_range(const uint64_t* ids, size_t n, int nbits, unsigned long long* ok, cudaStream_t s);

// ---- sorted (atomic-free, deterministic) gradient reduction ----
// CSC view of the batch: stable radix sort of (local key id -> occurrence payload); afterwards
// key u owns occ_sorted[col_start[u] .. col_end[u]) in row order (the reference's summation
// order per column, spmm.h:140-156).
size_t csc_tmp_bytes(size_t nnz, bool valued);
int launch_csc_build(const uint32_t* lidx, const void* occ, bool valued, size_t nnz, size_t nkeys,
                     uint32_t* lidx_sorted, void* occ_sorted, int* col_start, int* col_end,
                     void* cub_tmp, size_t cub_bytes, DevProgress* prog, cudaStream_t s);
// per key: grad = sum_occ x * pXV[row] - V * XXp, then either FTRL/AdaGrad in place (apply) or
// complete dense gradient rows out (gw_out, gV_out = sum - V_pulled*XXp; the sharded worker).
// l2hint: the L2 plan of the single-GPU step (p*XV / p kept, [V|cg] rows streamed); ignored when shard != nullptr.
// keys != nullptr (the single-GPU step without a lookup): the kernel finds or inserts every key of keys[n] itself and
// writes its slot (or -1) into slot[n], what the InitV pass reads.  keys == nullptr (a step that ran k_lookup, and the
// owner side of the sharded store): the slots and pulled V-row indices of that lookup come in slot / pull_vrow.
int launch_bwd_update(Table& t, const Params& p, const uint64_t* keys, int* slot, const int* pull_vrow, size_t n,
                      const unsigned long long* dn, const int* col_start, const int* col_end,
                      const void* occ_sorted, bool valued, const float* p_row, const float* pxv, int* flags,
                      int accumulate_penalty, const ShardApply* shard, const HotPart* hot, int l2hint, cudaStream_t s);
// drops the L2 lines of two dead device buffers without writing them back (discard.global.L2; contents undefined after)
int launch_l2_discard(void* a, size_t a_bytes, void* b, size_t b_bytes, cudaStream_t s);
// pre-reduction of the very hot keys' occurrence lists (split > 0); fills *hp for launch_bwd_update
int launch_hot_prereduce(int V_dim, size_t n, const unsigned long long* dn, const int* col_start, const int* col_end,
                         const void* occ_sorted, bool valued, const float* p_row, const float* pxv, int split,
                         const HotWs& ws, HotPart* hp, int l2hint, cudaStream_t s);
int launch_bwd_dense(const Params& p, DevProgress* prog, int ks, const float* w_pulled,
                     const int* hasv, size_t n, const int* col_start, const int* col_end,
                     const void* occ_sorted, bool valued, const float* p_row, const float* pxv,
                     float* gw_out, const float* V_pulled, float* gV_out, int accumulate_penalty,
                     const SegDst* seg, cudaStream_t s);
// owner side of the sharded Push for V_dim in {8,16,32,64,128}: FTRL/AdaGrad from complete dense
// gradient rows; returns -1 for other V_dim (use launch_update_dense)
int launch_update_pushed(Table& t, const Params& p, const int* slot, const int* hasv, size_t n,
                         const float* gw, const float* gV, int* flags, cudaStream_t s);

}  // namespace dfb
