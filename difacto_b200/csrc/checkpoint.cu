// difacto_b200/csrc/checkpoint.cu -- Updater::Save / Load (include/difacto/updater.h:40-47; TODO stubs in the
// reference's SGDUpdater, sgd_updater.h:44-50, so the byte format is ours), streamed through the GPU.
//   header { char magic[8] "DFB200\0\1"; u32 version; i32 V_dim; u64 n_keys; u64 n_vrows; u32 seed; u32 has_aux }
//   n_keys records in ascending key order:
//     u64 key; f32 fea_cnt; f32 w; [aux: f32 sqrt_g; f32 z;] i32 has_V; has_V ? f32 V[V_dim] [aux: f32 cg[V_dim]]
// The writer sorts and packs the records on the device, pass by pass (kernels_checkpoint.cu), and hands them to the
// caller's sink through two pinned chunks; the reader walks the record chain of each chunk on the host (validation),
// and the device keeps, inserts and unpacks the records of its shard.  Neither holds the table, the row pool or the
// file on the host.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "engine_internal.cuh"

using namespace dfb;  // NOLINT

// a checkpoint runs between steps: wait for everything enqueued on any of the handle's streams
int dfbh::drain(dfb_engine* h) {
  DFB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->loc_stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->aux_stream));
  if (h->shard) DFB_TRY(dfbh::shard_sync(h));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  return 0;
}

namespace {

struct SnapHeader {
  char magic[8];
  uint32_t version;
  int32_t V_dim;
  uint64_t n_keys, n_vrows;
  uint32_t seed, has_aux;
};
static_assert(sizeof(SnapHeader) == 40, "v1 header is 40 bytes");
const char kSnapMagic[8] = {'D', 'F', 'B', '2', '0', '0', 0, 1};
constexpr size_t kDefaultChunk = size_t(64) << 20;
constexpr size_t kMaxChunk = size_t(1) << 30;      // record offsets within a chunk are 32-bit word offsets

size_t fixed_bytes(bool aux) { return 8 + 4 + 4 + (aux ? 8 : 0) + 4; }
size_t row_bytes(int k, bool aux) { return (size_t)k * 4 * (aux ? 2 : 1); }

// where a routine reports its errors: the handle's message, or a frozen copy's own (dfb_frozen_write runs beside
// the handle's owning thread and must not touch the handle)
struct ErrSink {
  std::string* err;
  int fail(int code, const std::string& msg) { *err = msg; return code; }
  int cuda_fail(cudaError_t e, const char* what) {
    *err = std::string(what) + ": " + cudaGetErrorString(e);
    return DFB_ERR_CUDA;
  }
};

// everything a streamed checkpoint allocates, released on every path out of the call (after the stream drained).
// Device memory is stream-ordered on s, so a writer beside training steps never synchronises the device.
struct Scratch {
  ErrSink* es;
  cudaStream_t s;
  std::vector<void*> dev, host;
  std::vector<cudaEvent_t> ev;
  Scratch(ErrSink* es_, cudaStream_t s_) : es(es_), s(s_) {}
  ~Scratch() {
    for (void* p : dev) cudaFreeAsync(p, s);
    cudaStreamSynchronize(s);
    for (void* p : host) cudaFreeHost(p);
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
  template <typename T> int dalloc(T** p, size_t bytes) {
    void* q = nullptr;
    DFB_CUDA(es, cudaMallocAsync(&q, bytes ? bytes : 16, s));
    dev.push_back(q);
    *p = static_cast<T*>(q);
    return 0;
  }
  template <typename T> int halloc(T** p, size_t bytes) {
    void* q = nullptr;
    DFB_CUDA(es, cudaHostAlloc(&q, bytes ? bytes : 16, cudaHostAllocDefault));
    host.push_back(q);
    *p = static_cast<T*>(q);
    return 0;
  }
  int event(cudaEvent_t* e) {
    DFB_CUDA(es, cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    ev.push_back(*e);
    return 0;
  }
};

// the writer's two pinned chunks and their events: a call's own (dfb_snapshot_write), or kept by a frozen copy
// across its writes and freed at its release, off the writer thread
struct PinnedChunks {
  PinnedHost<char> pin[2];
  Event ev[2];
  size_t bytes = 0;
  int ensure(ErrSink* es, size_t chunk) {
    if (chunk <= bytes) return 0;
    bytes = 0;
    for (auto& p : pin) p.reset();      // both before the larger ones are allocated
    for (int i = 0; i < 2; ++i) {
      DFB_CUDA(es, pin[i].alloc(chunk));
      DFB_CUDA(es, ev[i].create());
    }
    bytes = chunk;
    return 0;
  }
};

using dfbh::drain;

int read_state(dfb_engine* h, TableState* st) {
  DFB_CUDA(h, cudaMemcpyAsync(st, h->tab.state, sizeof(TableState), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA(h, cudaStreamSynchronize(h->stream));
  return 0;
}

struct Pass {
  unsigned b0, b1;
  size_t nk, bytes;
};

// the v1 stream of table t (whose counts and InitV state are st) to fn, every pass on stream s.  Reads t and
// nothing else of an engine: dfb_snapshot_write runs it over the live table between steps, dfb_frozen_write over a
// frozen copy while steps run.  launches counts the kernels it ran.
int write_records(const Table& t, const TableState& st, int k, bool aux, size_t chunk, dfb_write_fn fn, void* ctx,
                  cudaStream_t s, PinnedChunks& pc, ErrSink* es, uint64_t* launches) {
  Scratch sc(es, s);
  // ---- histogram: keys and V rows per bin of the top kCkptBinBits key bits ----
  const size_t nbins = size_t(1) << kCkptBinBits;
  unsigned *d_nk, *d_nv;
  DFB_TRY(sc.dalloc(&d_nk, nbins * 4));
  DFB_TRY(sc.dalloc(&d_nv, nbins * 4));
  DFB_CUDA(es, cudaMemsetAsync(d_nk, 0, nbins * 4, s));
  DFB_CUDA(es, cudaMemsetAsync(d_nv, 0, nbins * 4, s));
  *launches += launch_ckpt_hist(t, d_nk, d_nv, s);
  std::vector<unsigned> nk(nbins), nv(nbins);
  DFB_CUDA(es, cudaMemcpyAsync(nk.data(), d_nk, nbins * 4, cudaMemcpyDeviceToHost, s));
  DFB_CUDA(es, cudaMemcpyAsync(nv.data(), d_nv, nbins * 4, cudaMemcpyDeviceToHost, s));
  DFB_CUDA(es, cudaStreamSynchronize(s));
  // ---- passes: runs of consecutive bins whose records fit the staging budget (a larger single bin: one pass) ----
  const size_t fixed = fixed_bytes(aux), rowb = row_bytes(k, aux);
  const size_t budget = 4 * chunk;
  std::vector<Pass> passes;
  uint64_t tk = 0, tv = 0;
  Pass cur{0, 0, 0, 0};
  for (size_t b = 0; b < nbins; ++b) {
    tk += nk[b]; tv += nv[b];
    const size_t bytes = (size_t)nk[b] * fixed + (size_t)nv[b] * rowb;
    if (cur.nk && cur.bytes + bytes > budget) {
      passes.push_back(cur);
      cur = Pass{(unsigned)b, (unsigned)b, 0, 0};
    }
    if (!cur.nk) cur.b0 = (unsigned)b;
    cur.b1 = (unsigned)b + 1;
    cur.nk += nk[b]; cur.bytes += bytes;
  }
  if (cur.nk) passes.push_back(cur);
  if (tk != st.n_keys || tv != st.n_vrows)
    return es->fail(DFB_ERR_INVALID, "table changed while taking the snapshot");
  size_t max_n = 0, max_bytes = 0;
  for (const Pass& p : passes) { max_n = std::max(max_n, p.nk); max_bytes = std::max(max_bytes, p.bytes); }
  // ---- header ----
  SnapHeader hd;
  memcpy(hd.magic, kSnapMagic, 8);
  hd.version = 1; hd.V_dim = k; hd.n_keys = st.n_keys; hd.n_vrows = st.n_vrows; hd.seed = st.seed;
  hd.has_aux = aux ? 1 : 0;
  if (int rc = fn(ctx, &hd, sizeof(hd))) return es->fail(DFB_ERR_INVALID, "snapshot sink failed (" + std::to_string(rc) + ")");
  if (passes.empty()) return 0;
  // ---- workspace of the largest pass, two pinned chunks ----
  CkptWs ws;
  DFB_TRY(sc.dalloc(&ws.keys_in, max_n * 8));
  DFB_TRY(sc.dalloc(&ws.keys_out, max_n * 8));
  DFB_TRY(sc.dalloc(&ws.slots_in, max_n * 4));
  DFB_TRY(sc.dalloc(&ws.slots_out, max_n * 4));
  DFB_TRY(sc.dalloc(&ws.hv, max_n * 4));
  DFB_TRY(sc.dalloc(&ws.vbefore, max_n * 4));
  DFB_TRY(sc.dalloc(&ws.counter, 8));
  ws.tmp_bytes = ckpt_sort_tmp_bytes(max_n);
  DFB_TRY(sc.dalloc(&ws.tmp, ws.tmp_bytes));
  DFB_TRY(sc.dalloc(&ws.out, max_bytes));
  DFB_TRY(pc.ensure(es, chunk));
  const PinnedHost<char>* pin = pc.pin;
  const Event* ev = pc.ev;
  for (const Pass& p : passes) {
    const int nl = launch_ckpt_pass(t, p.b0, p.b1, p.nk, aux, k, ws, s);
    if (nl < 0) return es->fail(DFB_ERR_CUDA, "snapshot pass failed (radix sort / scan)");
    *launches += nl;
    // D2H of chunk c + 1 overlaps the sink call of chunk c
    const char* src = reinterpret_cast<const char*>(ws.out);
    const size_t nch = (p.bytes + chunk - 1) / chunk;
    auto issue = [&](size_t c) {
      const size_t len = std::min(chunk, p.bytes - c * chunk);
      cudaMemcpyAsync(pin[c & 1], src + c * chunk, len, cudaMemcpyDeviceToHost, s);
      return cudaEventRecord(ev[c & 1], s);
    };
    DFB_CUDA(es, issue(0));
    for (size_t c = 0; c < nch; ++c) {
      if (c + 1 < nch) DFB_CUDA(es, issue(c + 1));
      DFB_CUDA(es, cudaEventSynchronize(ev[c & 1]));
      const size_t len = std::min(chunk, p.bytes - c * chunk);
      if (int rc = fn(ctx, pin[c & 1], len))
        return es->fail(DFB_ERR_INVALID, "snapshot sink failed (" + std::to_string(rc) + ")");
    }
  }
  DFB_CUDA(es, cudaGetLastError());
  return 0;
}

int check_chunk(size_t* chunk, ErrSink* es) {
  if (*chunk == 0) *chunk = kDefaultChunk;
  if (*chunk < sizeof(SnapHeader) || *chunk > kMaxChunk)
    return es->fail(DFB_ERR_INVALID, "chunk_bytes must be 0 or in [40, 2^30]");
  return 0;
}

// the record chain of one chunk, validated (input from outside the program)
struct Walk {
  bool have_hdr = false, aux = false, have_last = false;
  SnapHeader hd;
  uint64_t keys = 0, vrows = 0, last = 0;
};

int restore_read(dfb_engine* h, dfb_read_fn fn, void* ctx, uint32_t part, uint32_t nparts, uint32_t shard,
                 uint32_t nshards, size_t chunk, int* has_aux_out) {
  const int k = h->prm.V_dim;
  TableState st;
  DFB_TRY(read_state(h, &st));
  const bool first = st.n_keys == 0 && h->restored_parts == 0;   // this stream's header seeds the InitV stream
  cudaStream_t s = h->stream;
  ErrSink es{&h->err};
  Scratch sc(&es, s);
  const size_t max_rec = std::max(fixed_bytes(true) + row_bytes(k, true), sizeof(SnapHeader));
  const size_t cap = chunk + max_rec;              // a chunk plus the carried-over start of a record
  const size_t max_n = cap / fixed_bytes(false) + 1;
  char* pin[2];
  unsigned* proff[2];
  cudaEvent_t ev[2];
  bool pending[2] = {false, false};
  for (int i = 0; i < 2; ++i) {
    DFB_TRY(sc.halloc(&pin[i], cap));
    DFB_TRY(sc.halloc(&proff[i], max_n * 4));
    DFB_TRY(sc.event(&ev[i]));
  }
  unsigned *d_buf, *d_roff;
  unsigned long long *d_flags, *d_rank;
  DFB_TRY(sc.dalloc(&d_buf, cap));
  DFB_TRY(sc.dalloc(&d_roff, max_n * 4));
  DFB_TRY(sc.dalloc(&d_flags, max_n * 8));
  DFB_TRY(sc.dalloc(&d_rank, max_n * 8));
  const size_t tmp_bytes = rst_scan_tmp_bytes(max_n);
  void* d_tmp = nullptr;
  DFB_TRY(sc.dalloc(&d_tmp, tmp_bytes));
  Walk wk;
  size_t carry = 0;
  int b = 0;
  for (bool eof = false; !eof;) {
    if (pending[b]) { DFB_CUDA(h, cudaEventSynchronize(ev[b])); pending[b] = false; }
    const size_t got = fn(ctx, pin[b] + carry, chunk);
    if (got == (size_t)-1) return h->fail(DFB_ERR_INVALID, "snapshot source failed");
    if (got > chunk) return h->fail(DFB_ERR_INVALID, "snapshot source returned more than it was asked for");
    eof = got == 0;
    const size_t len = carry + got;
    const char* p = pin[b];
    size_t pos = 0;
    if (!wk.have_hdr) {
      if (len < sizeof(SnapHeader)) {
        if (eof) return h->fail(DFB_ERR_INVALID, "snapshot truncated (header)");
        carry = len;      // stays at the start of this buffer
        continue;
      }
      memcpy(&wk.hd, p, sizeof(SnapHeader));
      if (memcmp(wk.hd.magic, kSnapMagic, 8) != 0 || wk.hd.version != 1)
        return h->fail(DFB_ERR_INVALID, "not a difacto_b200 snapshot");
      if (wk.hd.V_dim != k) return h->fail(DFB_ERR_INVALID, "snapshot V_dim differs from the engine's V_dim");
      if (wk.hd.has_aux > 1) return h->fail(DFB_ERR_INVALID, "snapshot corrupt (has_aux)");
      wk.have_hdr = true;
      wk.aux = wk.hd.has_aux != 0;
      pos = sizeof(SnapHeader);
      // room for the whole stream before the first record is inserted (an engine below its maximum grows)
      DFB_TRY(dfbh::reserve(h, wk.hd.n_keys, wk.hd.n_vrows));
    }
    const size_t fixed = fixed_bytes(wk.aux), rowb = row_bytes(k, wk.aux);
    const size_t start = pos;
    size_t n = 0;
    while (pos + fixed <= len) {
      int32_t hv;
      memcpy(&hv, p + pos + fixed - 4, 4);
      if (hv != 0 && hv != 1) return h->fail(DFB_ERR_INVALID, "snapshot corrupt (has_V is neither 0 nor 1)");
      const size_t rec = fixed + (hv ? rowb : 0);
      if (pos + rec > len) break;
      uint64_t key;
      memcpy(&key, p + pos, 8);
      if (wk.have_last && key <= wk.last) return h->fail(DFB_ERR_INVALID, "snapshot corrupt (keys not ascending)");
      if (++wk.keys > wk.hd.n_keys) return h->fail(DFB_ERR_INVALID, "snapshot corrupt (more records than n_keys)");
      if (hv && ++wk.vrows > wk.hd.n_vrows) return h->fail(DFB_ERR_INVALID, "snapshot corrupt (more V rows than n_vrows)");
      wk.last = key; wk.have_last = true;
      proff[b][n++] = (unsigned)((pos - start) / 4);
      pos += rec;
    }
    if (n) {
      DFB_CUDA(h, cudaMemcpyAsync(d_buf, p + start, pos - start, cudaMemcpyHostToDevice, s));
      DFB_CUDA(h, cudaMemcpyAsync(d_roff, proff[b], n * 4, cudaMemcpyHostToDevice, s));
      DFB_CUDA(h, cudaEventRecord(ev[b], s));
      pending[b] = true;
      const int nl = launch_rst_chunk(h->tab, d_buf, d_roff, n, wk.aux, k, part, nparts, shard, nshards, d_flags,
                                      d_rank, d_tmp, tmp_bytes, s);
      if (nl < 0) return h->fail(DFB_ERR_CUDA, "restore chunk failed (scan)");
      h->launches += nl;
    }
    carry = len - pos;
    if (eof) break;
    // the start of a record that straddles the chunk boundary moves to the head of the other buffer, once the
    // H2D copy that last read that buffer has finished
    b ^= 1;
    if (pending[b]) { DFB_CUDA(h, cudaEventSynchronize(ev[b])); pending[b] = false; }
    if (carry) memcpy(pin[b], p + pos, carry);
  }
  if (!wk.have_hdr) return h->fail(DFB_ERR_INVALID, "snapshot truncated (header)");
  if (carry || wk.keys < wk.hd.n_keys) return h->fail(DFB_ERR_INVALID, "snapshot truncated");
  if (first) h->launches += launch_rst_seed(h->tab, wk.hd.seed, s);
  DFB_CUDA(h, cudaGetLastError());
  DFB_CUDA(h, cudaMemcpyAsync(h->h_prog, h->tab.prog, sizeof(DevProgress), cudaMemcpyDeviceToHost, s));
  DFB_CUDA(h, cudaStreamSynchronize(s));
  switch (h->h_prog->err) {
    case 0: break;
    case kErrCkptDup: return h->fail(DFB_ERR_INVALID, "a restored key is already in the table (the same part restored twice?)");
    case kErrCkptRange:
      return h->fail(DFB_ERR_INVALID, "a key lies outside part " + std::to_string(part) + " of " + std::to_string(nparts) +
                                      " (parts miscounted or mixed up)");
    case DFB_ERR_CAPACITY:
      return h->fail(DFB_ERR_CAPACITY, "snapshot larger than table_capacity / V_capacity");
    default: return h->fail(DFB_ERR_INVALID, "device-side error " + std::to_string(h->h_prog->err) + " while restoring");
  }
  h->has_aux = first ? (wk.aux ? 1 : 0) : (h->has_aux && wk.aux ? 1 : 0);
  if (h->score_only) h->has_aux = 0;    // V-only rows: the streams' aux data, if any, was not kept
  h->restored_parts++;
  if (has_aux_out) *has_aux_out = h->has_aux;
  return 0;
}

// a failed restore leaves a half-merged table behind: clear it, so that the caller can retry
int clear_table(dfb_engine* h, int rc) {
  const std::string msg = h->err;
  cudaGetLastError();
  cudaStreamSynchronize(h->stream);
  h->launches += launch_table_init(h->tab, h->prm.seed, h->stream);
  const cudaError_t e = cudaStreamSynchronize(h->stream);
  h->restored_parts = 0;
  h->has_aux = h->score_only ? 0 : 1;
  h->err = msg + "; the table was cleared";
  if (e != cudaSuccess) h->err += std::string(" (clearing failed: ") + cudaGetErrorString(e) + ")";
  return rc;
}

struct MemSink {
  char* p;
  size_t left;
};
int mem_write(void* ctx, const void* buf, size_t bytes) {
  MemSink* m = static_cast<MemSink*>(ctx);
  if (bytes > m->left) return 1;
  memcpy(m->p, buf, bytes);
  m->p += bytes; m->left -= bytes;
  return 0;
}
struct MemSource {
  const char* p;
  size_t left;
};
size_t mem_read(void* ctx, void* buf, size_t cap) {
  MemSource* m = static_cast<MemSource*>(ctx);
  const size_t n = std::min(cap, m->left);
  memcpy(buf, m->p, n);
  m->p += n; m->left -= n;
  return n;
}

}  // namespace

// a snapshot frozen by dfb_snapshot_begin: a device copy of the table's slots and of its V rows, the table state at
// that moment, and the writer's own low-priority stream, pinned chunks and error message
struct dfb_frozen_s {
  dfb_engine* h = nullptr;
  int device = 0, V_dim = 0;
  bool aux = false;
  Table tab;
  TableState st;
  cudaStream_t stream = nullptr;
  PinnedChunks chunks;
  std::string err;
  uint64_t launches = 0;
};

void dfbh::frozen_destroy(dfb_frozen_s* f) {
  if (f->stream) {
    dfbh::table_copy_free(&f->tab, f->stream);    // after the writer's last pass, without a device-wide wait
    cudaStreamSynchronize(f->stream);
    cudaStreamDestroy(f->stream);
  }
  delete f;
}

extern "C" {

int dfb_snapshot_size(dfb_handle h, int save_aux, size_t* bytes) {
  if (!h || !bytes) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_snapshot_size");
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(drain(h));
  TableState st;
  DFB_TRY(read_state(h, &st));
  *bytes = sizeof(SnapHeader) + st.n_keys * (fixed_bytes(save_aux != 0)) +
           st.n_vrows * row_bytes(h->prm.V_dim, save_aux != 0);
  return DFB_OK;
}

int dfb_snapshot_write(dfb_handle h, int save_aux, size_t chunk_bytes, dfb_write_fn fn, void* ctx) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_snapshot_write");
  if (!fn) return h->fail(DFB_ERR_INVALID, "write callback is NULL");
  ErrSink es{&h->err};
  DFB_TRY(check_chunk(&chunk_bytes, &es));
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (save_aux && !h->has_aux) return h->fail(DFB_ERR_INVALID, "no aux data to save");
  DFB_TRY(drain(h));
  TableState st;
  DFB_TRY(read_state(h, &st));
  PinnedChunks pc;
  return write_records(h->tab, st, h->prm.V_dim, save_aux != 0, chunk_bytes, fn, ctx, h->stream, pc, &es,
                       &h->launches);
}

int dfb_snapshot_begin(dfb_handle h, int save_aux, dfb_frozen* out) {
  if (!h) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_snapshot_begin");
  if (!out) return h->fail(DFB_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (h->frozen) return h->fail(DFB_ERR_INVALID, "the handle already has a frozen snapshot (release it first)");
  DFB_CUDA(h, cudaSetDevice(h->device));
  if (save_aux && !h->has_aux) return h->fail(DFB_ERR_INVALID, "no aux data to save");
  DFB_TRY(drain(h));
  dfb_frozen_s* f = new dfb_frozen_s();
  f->h = h; f->device = h->device; f->V_dim = h->prm.V_dim; f->aux = save_aux != 0;
  if (int rc = read_state(h, &f->st)) { delete f; return rc; }
  if (int rc = dfbh::table_copy(h, f->st.n_vrows, &f->tab)) { delete f; return rc; }
  int least = 0, greatest = 0;
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&f->stream, cudaStreamNonBlocking, least);
  if (e != cudaSuccess) {
    dfbh::table_copy_free(&f->tab, h->stream);
    delete f;
    return h->cuda_fail(e, "cudaStreamCreateWithPriority(frozen snapshot)");
  }
  h->frozen = f;
  *out = f;
  return DFB_OK;
}

int dfb_frozen_write(dfb_frozen f, size_t chunk_bytes, dfb_write_fn fn, void* ctx) {
  if (!f) return DFB_ERR_INVALID;
  ErrSink es{&f->err};
  if (!fn) return es.fail(DFB_ERR_INVALID, "write callback is NULL");
  DFB_TRY(check_chunk(&chunk_bytes, &es));
  DFB_CUDA(&es, cudaSetDevice(f->device));
  return write_records(f->tab, f->st, f->V_dim, f->aux, chunk_bytes, fn, ctx, f->stream, f->chunks, &es,
                       &f->launches);
}

const char* dfb_frozen_error(dfb_frozen f) { return f ? f->err.c_str() : "frozen snapshot is NULL"; }

int dfb_frozen_release(dfb_frozen f) {
  if (!f) return DFB_OK;
  cudaSetDevice(f->device);
  f->h->frozen = nullptr;
  dfbh::frozen_destroy(f);
  return DFB_OK;
}

int dfb_restore_read(dfb_handle h, dfb_read_fn fn, void* ctx, uint32_t part, uint32_t nparts, uint32_t shard,
                     uint32_t nshards, size_t chunk_bytes, int* has_aux_out) {
  if (!h) return DFB_ERR_INVALID;
  if (!fn) return h->fail(DFB_ERR_INVALID, "read callback is NULL");
  if (nparts == 0 || part >= nparts || nshards == 0 || shard >= nshards)
    return h->fail(DFB_ERR_INVALID, "need part < nparts and shard < nshards");
  if (chunk_bytes == 0) chunk_bytes = kDefaultChunk;
  if (chunk_bytes > kMaxChunk) return h->fail(DFB_ERR_INVALID, "chunk_bytes must be 0 or at most 2^30");
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(drain(h));
  const int rc = restore_read(h, fn, ctx, part, nparts, shard, nshards, chunk_bytes, has_aux_out);
  return rc ? clear_table(h, rc) : DFB_OK;
}

int dfb_snapshot(dfb_handle h, int save_aux, void* buf, size_t bytes) {
  if (!h || !buf) return DFB_ERR_INVALID;
  DFB_NOT_SCORE_ONLY(h, "dfb_snapshot");
  size_t need = 0;
  DFB_TRY(dfb_snapshot_size(h, save_aux, &need));
  if (bytes < need) return h->fail(DFB_ERR_INVALID, "snapshot buffer too small");
  MemSink m{static_cast<char*>(buf), bytes};
  return dfb_snapshot_write(h, save_aux, 0, mem_write, &m);
}

int dfb_restore(dfb_handle h, const void* buf, size_t bytes, int* has_aux) {
  if (!h || !buf) return DFB_ERR_INVALID;
  DFB_CUDA(h, cudaSetDevice(h->device));
  DFB_TRY(drain(h));
  TableState st;
  DFB_TRY(read_state(h, &st));
  if (st.n_keys != 0) return h->fail(DFB_ERR_INVALID, "dfb_restore needs an empty table");
  MemSource m{static_cast<const char*>(buf), bytes};
  return dfb_restore_read(h, mem_read, &m, 0, 1, 0, 1, 0, has_aux);
}

}  // extern "C"
