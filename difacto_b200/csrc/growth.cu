// difacto_b200/csrc/growth.cu -- the engine's hash table and V-row pool, and their growth on demand up to
// table_capacity_max / V_capacity_max (DESIGN.md section 2).
//
// The table is reallocated (stream-ordered, from an engine-owned memory pool) and rehashed on h->stream, so the
// kernels enqueued before see the old table and those enqueued after the new one: every table-touching kernel runs on
// h->stream and takes the Table by value.  The V-row pool is a reserved address range for V_capacity_max rows with
// physical memory mapped at its start; growing it maps more after the last mapping, so rows never move.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>

#include "engine_internal.cuh"

using namespace dfb;  // NOLINT

namespace {

// the driver's virtual memory management, through the runtime's entry-point query (the library links cudart only)
struct Vmm {
  PFN_cuMemAddressReserve reserve = nullptr;
  PFN_cuMemAddressFree addr_free = nullptr;
  PFN_cuMemCreate create = nullptr;
  PFN_cuMemRelease release = nullptr;
  PFN_cuMemMap map = nullptr;
  PFN_cuMemUnmap unmap = nullptr;
  PFN_cuMemSetAccess set_access = nullptr;
  PFN_cuMemGetAllocationGranularity granularity = nullptr;
  bool ok = false;
};

const Vmm& vmm() {
  static const Vmm v = [] {
    Vmm x;
    auto get = [](const char* name, void* fn) {
      cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
      void** p = static_cast<void**>(fn);
      return cudaGetDriverEntryPointByVersion(name, p, 12000, cudaEnableDefault, &q) == cudaSuccess &&
             q == cudaDriverEntryPointSuccess && *p != nullptr;
    };
    x.ok = get("cuMemAddressReserve", &x.reserve) && get("cuMemAddressFree", &x.addr_free) &&
           get("cuMemCreate", &x.create) && get("cuMemRelease", &x.release) && get("cuMemMap", &x.map) &&
           get("cuMemUnmap", &x.unmap) && get("cuMemSetAccess", &x.set_access) &&
           get("cuMemGetAllocationGranularity", &x.granularity);
    return x;
  }();
  return v;
}

CUmemAllocationProp pool_prop(int device) {
  CUmemAllocationProp p;
  memset(&p, 0, sizeof(p));
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = device;
  return p;
}

uint64_t next_pow2(uint64_t x) {
  uint64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

size_t round_up(size_t x, size_t g) { return (x + g - 1) / g * g; }

// rs elements of 4 bytes, or of 2 in a scoring-only engine's bf16 rows
size_t row_bytes(const dfb_engine* h) { return (size_t)h->tab.rs * (h->tab.vonly == 2 ? 2 : 4); }

// maps physical memory up to `bytes` (a multiple of the granularity, at most the reservation) of the V-row pool;
// false (nothing changed) when the memory cannot be had
bool vpool_map(dfb_engine* h, size_t bytes) {
  dfb_engine::Growth& g = h->grow;
  if (bytes <= g.vmapped) return true;
  const Vmm& d = vmm();
  const size_t add = bytes - g.vmapped;
  const CUdeviceptr at = (CUdeviceptr)(g.vbase + g.vmapped);
  const CUmemAllocationProp prop = pool_prop(h->device);
  CUmemGenericAllocationHandle mh;
  if (d.create(&mh, add, &prop, 0) != CUDA_SUCCESS) return false;
  if (d.map(at, add, 0, mh, 0) != CUDA_SUCCESS) {
    d.release(mh);
    return false;
  }
  CUmemAccessDesc acc;
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (d.set_access(at, add, &acc, 1) != CUDA_SUCCESS) {
    d.unmap(at, add);
    d.release(mh);
    return false;
  }
  g.vchunks.push_back(std::make_pair((unsigned long long)mh, add));
  g.vmapped = bytes;
  return true;
}

// a table for new_max keys, filled from the current one on h->stream; the old one is freed in stream order.  A
// failed allocation keeps the current table.
int grow_table(dfb_engine* h, uint64_t new_max) {
  Table& t = h->tab;
  Table nt = t;
  nt.max_keys = new_max;
  nt.cap = std::max<uint64_t>(t.cap, next_pow2(2 * new_max));
  if (nt.cap == t.cap) {       // the slots already allow it (load factor <= 0.5)
    t.max_keys = new_max;
    return 0;
  }
  nt.mask = nt.cap - 1;
  cudaStream_t s = h->stream;
  if (cudaMallocFromPoolAsync(reinterpret_cast<void**>(&nt.tab), nt.cap * sizeof(Entry), h->grow.pool, s) !=
      cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  h->launches += launch_table_rehash(t, nt, s);
  DFB_CUDA(h, cudaFreeAsync(t.tab, s));
  t.tab = nt.tab; t.cap = nt.cap; t.mask = nt.mask; t.max_keys = nt.max_keys;
  return 0;
}

// maps memory for new_rows V rows (rounded up to the granularity); a failed mapping keeps the current pool
void grow_pool(dfb_engine* h, uint64_t new_rows) {
  dfb_engine::Growth& g = h->grow;
  const size_t rb = row_bytes(h);
  if (!vpool_map(h, std::min(round_up((size_t)new_rows * rb, g.gran), g.vreserved))) return;
  h->tab.vcap = std::min<uint64_t>(g.v_max, g.vmapped / rb);
}

}  // namespace

int dfbh::capacity_create(dfb_engine* h) {
  Table& t = h->tab;
  dfb_engine::Growth& g = h->grow;
  cudaMemPoolProps pp;
  memset(&pp, 0, sizeof(pp));
  pp.allocType = cudaMemAllocationTypePinned;
  pp.location.type = cudaMemLocationTypeDevice;
  pp.location.id = h->device;
  DFB_CUDA(h, cudaMemPoolCreate(&g.pool, &pp));
  uint64_t keep = 0;     // a freed table goes back to the device at the next synchronisation
  DFB_CUDA(h, cudaMemPoolSetAttribute(g.pool, cudaMemPoolAttrReleaseThreshold, &keep));
  DFB_CUDA(h, cudaMallocFromPoolAsync(reinterpret_cast<void**>(&t.tab), t.cap * sizeof(Entry), g.pool, h->stream));
  if (g.v_max && t.ks) {
    const Vmm& d = vmm();
    if (!d.ok) return h->fail(DFB_ERR_CUDA, "the driver's virtual memory management functions are not available");
    const CUmemAllocationProp prop = pool_prop(h->device);
    if (d.granularity(&g.gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || g.gran == 0)
      return h->fail(DFB_ERR_CUDA, "cuMemGetAllocationGranularity failed");
    g.vreserved = round_up((size_t)g.v_max * row_bytes(h), g.gran);
    CUdeviceptr base = 0;
    if (d.reserve(&base, g.vreserved, 0, 0, 0) != CUDA_SUCCESS)
      return h->fail(DFB_ERR_CUDA, "cuMemAddressReserve(V rows) failed: V_capacity_max too large for the address space");
    g.vbase = (unsigned long long)base;
    if (!vpool_map(h, round_up((size_t)t.vcap * row_bytes(h), g.gran)))
      return h->fail(DFB_ERR_CUDA, "out of device memory for V_capacity V rows");
    t.V = reinterpret_cast<float*>(g.vbase);
    t.Vcg = t.vonly ? nullptr : t.V + t.ks;
  }
  if (g.on) {
    DFB_CUDA(h, g.h_st.alloc(2 * dfb_engine::Growth::kRing));
    for (auto& ev : g.ev) DFB_CUDA(h, ev.create());
  }
  if (g.on && h->shard_growth) {
    DFB_CUDA(h, g.h_rcv.alloc(dfb_engine::Growth::kRing, cudaHostAllocMapped));
    DFB_CUDA(h, cudaHostGetDevicePointer(reinterpret_cast<void**>(&g.d_rcv), g.h_rcv, 0));
    for (auto& ev : g.rev) DFB_CUDA(h, ev.create());
  }
  return 0;
}

void dfbh::capacity_destroy(dfb_engine* h) {
  dfb_engine::Growth& g = h->grow;
  if (h->tab.tab) {
    cudaFreeAsync(h->tab.tab, h->stream);
    cudaStreamSynchronize(h->stream);
    h->tab.tab = nullptr;
  }
  if (g.pool) cudaMemPoolDestroy(g.pool);
  if (g.vbase) {
    const Vmm& d = vmm();
    size_t off = 0;
    for (const auto& c : g.vchunks) {
      d.unmap((CUdeviceptr)(g.vbase + off), c.second);
      d.release((CUmemGenericAllocationHandle)c.first);
      off += c.second;
    }
    d.addr_free((CUdeviceptr)g.vbase, g.vreserved);
  }
  g.vchunks.clear();
  g.vbase = 0; g.vmapped = 0;
  h->tab.V = h->tab.Vcg = nullptr;
}

namespace {

bool can_grow(const dfb_engine* h) {
  const dfb_engine::Growth& g = h->grow;
  const Table& t = h->tab;
  return g.on && (t.max_keys < g.tab_max || (g.vbase && t.vcap < g.v_max));
}

// takes in what the device has finished: the received-key counts of sharded steps (each replaces its step's worst case
// in the totals, and in every copy taken after that bound was added), then the newest completed copy of the counts
int fold(dfb_engine* h) {
  dfb_engine::Growth& g = h->grow;
  constexpr int R = dfb_engine::Growth::kRing;
  while (g.rhead < g.rseq) {
    const int r = (int)(g.rhead % R);
    const cudaError_t e = cudaEventQuery(g.rev[r]);
    if (e == cudaErrorNotReady) break;
    if (e != cudaSuccess) return h->cuda_fail(e, "cudaEventQuery(received keys)");
    const uint64_t d = g.r_worst[r] - std::min<uint64_t>(g.h_rcv[r], g.r_worst[r]);
    const uint64_t dv = g.r_v[r] ? d : 0;
    g.total_k -= d; g.total_v -= dv;
    for (uint64_t i = g.head; i < g.seq; ++i) {
      const int c = (int)(i % R);
      if (g.at_call[c] > g.r_call[r]) { g.at_k[c] -= d; g.at_v[c] -= dv; }
    }
    if (g.known_at_call > g.r_call[r]) { g.known_at_k -= d; g.known_at_v -= dv; }
    g.rhead++;
  }
  // the copies complete in stream order: take the newest one that has
  while (g.head < g.seq) {
    const int r = (int)(g.head % R);
    const cudaError_t e = cudaEventQuery(g.ev[r]);
    if (e == cudaErrorNotReady) break;
    if (e != cudaSuccess) return h->cuda_fail(e, "cudaEventQuery(table counts)");
    g.known_k = g.h_st[2 * r]; g.known_v = g.h_st[2 * r + 1];
    g.known_at_k = g.at_k[r]; g.known_at_v = g.at_v[r]; g.known_at_call = g.at_call[r];
    g.head++;
  }
  return 0;
}

// the counts the table may reach: the last known ones plus every bound added since (and new_* not added yet)
uint64_t need_keys(const dfb_engine::Growth& g, uint64_t new_keys = 0) { return g.known_k + (g.total_k - g.known_at_k) + new_keys; }
uint64_t need_vrows(const dfb_engine::Growth& g, uint64_t new_vrows = 0) { return g.known_v + (g.total_v - g.known_at_v) + new_vrows; }

bool short_of(const dfb_engine* h) {
  const dfb_engine::Growth& g = h->grow;
  const Table& t = h->tab;
  return (need_keys(g) > t.max_keys && t.max_keys < g.tab_max) ||
         (g.vbase && need_vrows(g) > t.vcap && t.vcap < g.v_max);
}

// geometric: at least double, and at least the need -- so a capacity stays below twice what it had to hold
int grow_to_need(dfb_engine* h, uint64_t new_keys = 0, uint64_t new_vrows = 0) {
  dfb_engine::Growth& g = h->grow;
  Table& t = h->tab;
  const uint64_t need_k = need_keys(g, new_keys), need_v = need_vrows(g, new_vrows);
  const uint64_t k0 = t.max_keys, v0 = t.vcap;
  if (need_k > t.max_keys && t.max_keys < g.tab_max)
    DFB_TRY(grow_table(h, std::min(g.tab_max, std::max(need_k, 2 * t.max_keys))));
  if (g.vbase && need_v > t.vcap && t.vcap < g.v_max) grow_pool(h, std::min(g.v_max, std::max(need_v, 2 * t.vcap)));
  if (t.max_keys != k0 || t.vcap != v0) g.n_growths++;
  return 0;
}

// a copy of {n_keys, n_vrows} as they are at this point of h->stream, with the bound totals it corresponds to
int enqueue_copy(dfb_engine* h) {
  dfb_engine::Growth& g = h->grow;
  constexpr int R = dfb_engine::Growth::kRing;
  if (g.seq - g.head >= (uint64_t)R) return 0;
  const int r = (int)(g.seq % R);
  DFB_CUDA(h, cudaMemcpyAsync(g.h_st + 2 * r, h->tab.state, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                              h->stream));
  DFB_CUDA(h, cudaEventRecord(g.ev[r], h->stream));
  g.at_k[r] = g.total_k; g.at_v[r] = g.total_v; g.at_call[r] = g.calls;
  g.seq++;
  return 0;
}

}  // namespace

int dfbh::reserve(dfb_engine* h, uint64_t new_keys, uint64_t new_vrows) {
  if (!can_grow(h)) return 0;
  dfb_engine::Growth& g = h->grow;
  new_keys = std::min<uint64_t>(new_keys, 1ULL << 32);    // above any capacity (a snapshot header is outside input)
  new_vrows = std::min<uint64_t>(new_vrows, 1ULL << 32);
  DFB_TRY(fold(h));
  DFB_TRY(grow_to_need(h, new_keys, new_vrows));
  DFB_TRY(enqueue_copy(h));
  g.total_k += new_keys;
  g.total_v += new_vrows;
  g.calls++;
  return 0;
}

int dfbh::shard_rcv_slot(dfb_engine* h, unsigned long long** slot) {
  *slot = nullptr;
  if (!h->shard_growth || !can_grow(h)) return 0;
  dfb_engine::Growth& g = h->grow;
  constexpr int R = dfb_engine::Growth::kRing;
  // a full ring: the oldest count is that of a step kRing steps back, whose phase 0 every rank has enqueued
  if (g.rseq - g.rhead >= (uint64_t)R) {
    DFB_CUDA(h, cudaEventSynchronize(g.rev[g.rhead % R]));
    g.n_waits++;
    DFB_TRY(fold(h));
  }
  *slot = g.d_rcv + g.rseq % R;
  return 0;
}

int dfbh::reserve_shard(dfb_engine* h, cudaStream_t counted_on, uint64_t worst, bool vrows, bool* rehashed) {
  dfb_engine::Growth& g = h->grow;
  constexpr int R = dfb_engine::Growth::kRing;
  const int r = (int)(g.rseq % R);
  DFB_CUDA(h, cudaEventRecord(g.rev[r], counted_on));
  g.r_call[r] = g.calls++; g.r_worst[r] = worst; g.r_v[r] = vrows;
  g.rseq++;
  g.total_k += worst;
  if (vrows) g.total_v += worst;
  DFB_TRY(fold(h));
  // the worst case does not fit: wait for this step's count.  It waits only for every worker's structure of this step
  // (phase 0, enqueued by each rank before its phase 1) and for the poller in front of it, which times out.
  if (short_of(h) && g.rhead < g.rseq) {
    DFB_CUDA(h, cudaEventSynchronize(g.rev[r]));
    g.n_waits++;
    DFB_TRY(fold(h));
  }
  const Entry* before = h->tab.tab;
  DFB_TRY(grow_to_need(h));
  *rehashed = h->tab.tab != before;
  return 0;
}

int dfbh::shard_counts_copy(dfb_engine* h) {
  if (!h->shard_growth || !can_grow(h)) return 0;
  return enqueue_copy(h);
}

void dfbh::counts_known(dfb_engine* h, uint64_t n_keys, uint64_t n_vrows) {
  dfb_engine::Growth& g = h->grow;
  g.head = g.seq;                       // the copies and counts in flight are complete, and older than these counts
  g.rhead = g.rseq;
  g.known_k = n_keys; g.known_v = n_vrows;
  g.known_at_k = g.total_k; g.known_at_v = g.total_v; g.known_at_call = g.calls;
}

int dfbh::table_copy(dfb_engine* h, uint64_t n_vrows, Table* out) {
  const Table& t = h->tab;
  Table c = t;
  c.V = c.Vcg = nullptr;
  c.vcap = n_vrows;
  c.state = nullptr; c.prog = nullptr;
  const size_t vbytes = (size_t)n_vrows * row_bytes(h);
  cudaStream_t s = h->stream;
  // an engine that can still grow keeps room for that growth: the copy is refused (the caller falls back to the
  // blocking writer) rather than starving a later rehash or pool mapping into DFB_ERR_CAPACITY
  const dfb_engine::Growth& g = h->grow;
  if (g.on) {
    size_t need = t.cap * sizeof(Entry) + vbytes;
    if (t.max_keys < g.tab_max) need += next_pow2(2 * g.tab_max) * sizeof(Entry) * 3 / 2;  // the last rehash: new + old
    if (g.vbase) need += std::min(round_up((size_t)g.v_max * row_bytes(h), g.gran), g.vreserved) - g.vmapped;
    size_t free_b = 0, total_b = 0;
    DFB_CUDA(h, cudaMemGetInfo(&free_b, &total_b));
    if (free_b < need)
      return h->fail(DFB_ERR_CAPACITY, "no device memory for a copy of the table beside the growth up to "
                                       "table_capacity_max / V_capacity_max");
  }
  if (cudaMallocAsync(reinterpret_cast<void**>(&c.tab), t.cap * sizeof(Entry), s) != cudaSuccess) {
    cudaGetLastError();
    return h->fail(DFB_ERR_CAPACITY, "no device memory for a copy of the table");
  }
  if (vbytes && cudaMallocAsync(reinterpret_cast<void**>(&c.V), vbytes, s) != cudaSuccess) {
    cudaGetLastError();
    cudaFreeAsync(c.tab, s);
    cudaStreamSynchronize(s);
    return h->fail(DFB_ERR_CAPACITY, "no device memory for a copy of the V rows");
  }
  if (c.V) c.Vcg = c.V + t.ks;
  DFB_CUDA(h, cudaMemcpyAsync(c.tab, t.tab, t.cap * sizeof(Entry), cudaMemcpyDeviceToDevice, s));
  if (vbytes) DFB_CUDA(h, cudaMemcpyAsync(c.V, t.V, vbytes, cudaMemcpyDeviceToDevice, s));
  // the sharded store inserts on streams of its own: the copy is complete before any later step may run
  DFB_CUDA(h, cudaStreamSynchronize(s));
  *out = c;
  return 0;
}

void dfbh::table_copy_free(Table* t, cudaStream_t s) {
  if (t->tab) cudaFreeAsync(t->tab, s);
  if (t->V) cudaFreeAsync(t->V, s);
  t->tab = nullptr; t->V = t->Vcg = nullptr;
}
