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
    DFB_CUDA(h, cudaHostAlloc(&g.h_st, 2 * dfb_engine::Growth::kRing * sizeof(unsigned long long), cudaHostAllocDefault));
    for (auto& ev : g.ev) DFB_CUDA(h, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
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
  if (g.h_st) cudaFreeHost(g.h_st);
  for (auto& ev : g.ev) if (ev) cudaEventDestroy(ev);
}

int dfbh::reserve(dfb_engine* h, uint64_t new_keys, uint64_t new_vrows) {
  dfb_engine::Growth& g = h->grow;
  Table& t = h->tab;
  if (!g.on || (t.max_keys >= g.tab_max && (t.vcap >= g.v_max || !g.vbase))) return 0;   // nothing can grow
  constexpr int R = dfb_engine::Growth::kRing;
  new_keys = std::min<uint64_t>(new_keys, 1ULL << 32);    // above any capacity (a snapshot header is outside input)
  new_vrows = std::min<uint64_t>(new_vrows, 1ULL << 32);
  // the copies complete in stream order: take the newest one that has
  while (g.head < g.seq) {
    const int r = (int)(g.head % R);
    const cudaError_t e = cudaEventQuery(g.ev[r]);
    if (e == cudaErrorNotReady) break;
    if (e != cudaSuccess) return h->cuda_fail(e, "cudaEventQuery(table counts)");
    g.known_k = g.h_st[2 * r]; g.known_v = g.h_st[2 * r + 1];
    g.known_at_k = g.at_k[r]; g.known_at_v = g.at_v[r];
    g.head++;
  }
  const uint64_t need_k = g.known_k + (g.total_k - g.known_at_k) + new_keys;
  const uint64_t need_v = g.known_v + (g.total_v - g.known_at_v) + new_vrows;
  // geometric: at least double, and at least the bound -- so a capacity stays below twice what it had to hold
  if (need_k > t.max_keys && t.max_keys < g.tab_max)
    DFB_TRY(grow_table(h, std::min(g.tab_max, std::max(need_k, 2 * t.max_keys))));
  if (g.vbase && need_v > t.vcap && t.vcap < g.v_max) grow_pool(h, std::min(g.v_max, std::max(need_v, 2 * t.vcap)));
  if (g.seq - g.head < (uint64_t)R) {
    const int r = (int)(g.seq % R);
    DFB_CUDA(h, cudaMemcpyAsync(g.h_st + 2 * r, t.state, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                                h->stream));
    DFB_CUDA(h, cudaEventRecord(g.ev[r], h->stream));
    g.at_k[r] = g.total_k; g.at_v[r] = g.total_v;
    g.seq++;
  }
  g.total_k += new_keys;
  g.total_v += new_vrows;
  return 0;
}

void dfbh::counts_known(dfb_engine* h, uint64_t n_keys, uint64_t n_vrows) {
  dfb_engine::Growth& g = h->grow;
  g.head = g.seq;                       // the copies in flight are complete, and older than these counts
  g.known_k = n_keys; g.known_v = n_vrows;
  g.known_at_k = g.total_k; g.known_at_v = g.total_v;
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
