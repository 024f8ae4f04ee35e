// Runtime core of libedb.so: process state, symmetric heap, CUDA-IPC peer mapping, groups.
//
// Replaces (natively on the GPU) what the reference gets from ProcessGroupNCCL + _expand_group
// (easydist/torch/passes/sharding.py:95) and the DeviceMesh rank bookkeeping
// (easydist/torch/device_mesh.py:129-150): instead of NCCL communicators we keep one
// cudaMalloc'd slab per rank, mapped into every peer of the NVSwitch domain with CUDA IPC, and
// per-group flag blocks inside that slab.
#include <stdarg.h>

#include <atomic>

#include "edb_internal.cuh"

namespace edb {

static Runtime g_rt;
static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

Runtime& rt() { return g_rt; }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

bool gemm2_enabled() {
  if (g_rt.gemm2 < 0) {
    const char* e = getenv("EDB_GEMM2");
    g_rt.gemm2 = (e && !strcmp(e, "0")) ? 0 : 1;
  }
  return g_rt.gemm2 != 0;
}

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int cuda_check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  return set_error(EDB_E_CUDA, "CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
}

}  // namespace edb

using namespace edb;

extern "C" {

int edb_version(void) { return EDB_VERSION; }
const char* edb_last_error(void) { return g_err; }
uint64_t edb_launch_count(void) { return g_launches.load(); }
int edb_is_initialized(void) { return g_rt.inited ? 1 : 0; }

int edb_init(int rank, int world, int device, size_t heap_bytes) {
  Runtime& r = g_rt;
  if (r.inited) return set_error(EDB_E_STATE, "edb_init: already initialised");
  EDB_REQUIRE(world >= 1 && world <= kMaxWorld, "edb_init: world %d out of range", world);
  EDB_REQUIRE(rank >= 0 && rank < world, "edb_init: rank %d out of range", rank);
  const size_t two_mb = 2u << 20;
  heap_bytes = (heap_bytes + two_mb - 1) / two_mb * two_mb;
  EDB_REQUIRE(heap_bytes >= kUserOffset + two_mb, "edb_init: heap of %zu bytes is too small",
              heap_bytes);
  EDB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  EDB_CUDA(cudaGetDeviceProperties(&prop, device));
  void* p = nullptr;
  EDB_CUDA(cudaMalloc(&p, heap_bytes));
  EDB_CUDA(cudaMemset(p, 0, kUserOffset));
  // pinned host error record, visible to the kernels through word F_ERRHOST of every flag block
  // (fatal_timeout writes it before trapping; edb_health reads it from the host)
  if (!r.host_err) {
    void* h = nullptr;
    EDB_CUDA(cudaHostAlloc(&h, 64, cudaHostAllocMapped));
    memset(h, 0, 64);
    void* d = nullptr;
    EDB_CUDA(cudaHostGetDevicePointer(&d, h, 0));
    r.host_err = static_cast<uint64_t*>(h);
    r.host_err_dev = static_cast<uint64_t*>(d);
  }
  for (int slot = 0; slot < kMaxGroups; ++slot) {
    const uint64_t v = (uint64_t)(uintptr_t)r.host_err_dev;
    EDB_CUDA(cudaMemcpy(flag_block(static_cast<char*>(p), slot) + F_ERRHOST, &v, sizeof(v),
                        cudaMemcpyHostToDevice));
  }
  EDB_CUDA(cudaDeviceSynchronize());
  r.rank = rank;
  r.world = world;
  r.device = device;
  r.sm_count = prop.multiProcessorCount;
  r.heap = static_cast<char*>(p);
  r.heap_bytes = heap_bytes;
  r.bump = kUserOffset;
  for (int i = 0; i < kMaxWorld; ++i) {
    r.peer_heap[i] = nullptr;
    r.peer_is_ipc[i] = false;
  }
  r.peer_heap[rank] = r.heap;
  r.ngroups = 0;
  r.inited = true;
  return EDB_OK;
}

int edb_finalize(void) {
  Runtime& r = g_rt;
  if (!r.inited) return EDB_OK;
  cudaSetDevice(r.device);
  cudaDeviceSynchronize();
  for (int i = 0; i < kMaxWorld; ++i) {
    if (r.peer_is_ipc[i] && r.peer_heap[i]) cudaIpcCloseMemHandle(r.peer_heap[i]);
    r.peer_heap[i] = nullptr;
    r.peer_is_ipc[i] = false;
  }
  cudaFree(r.heap);
  if (r.host_err) cudaFreeHost(r.host_err);
  r = Runtime();
  return EDB_OK;
}

int edb_health(void) {
  Runtime& r = g_rt;
  if (!r.inited || !r.host_err) return EDB_OK;
  volatile uint64_t* h = r.host_err;
  if (h[0] == 0) return EDB_OK;
  static const char* kinds[] = {"?", "flag wait", "epoch barrier", "low-latency packet"};
  const uint64_t kind = h[2] < 4 ? h[2] : 0;
  return set_error(EDB_E_STATE,
                   "a collective on rank %d timed out waiting for a peer (%s, op/epoch %llu, timeout "
                   "%lld ms): a peer is lost or too far behind; the kernel trapped and this process's "
                   "CUDA context is unusable",
                   r.rank, kinds[kind], (unsigned long long)h[1], (long long)r.spin_timeout_ms);
}

int edb_heap_info(void** base, size_t* bytes, size_t* user_offset) {
  if (!g_rt.inited) return set_error(EDB_E_STATE, "edb_heap_info: not initialised");
  if (base) *base = g_rt.heap;
  if (bytes) *bytes = g_rt.heap_bytes;
  if (user_offset) *user_offset = kUserOffset;
  return EDB_OK;
}

int edb_ipc_export(void* handle_out) {
  if (!g_rt.inited) return set_error(EDB_E_STATE, "edb_ipc_export: not initialised");
  static_assert(sizeof(cudaIpcMemHandle_t) == EDB_IPC_HANDLE_BYTES, "ipc handle size");
  cudaIpcMemHandle_t h;
  EDB_CUDA(cudaIpcGetMemHandle(&h, g_rt.heap));
  memcpy(handle_out, &h, sizeof(h));
  return EDB_OK;
}

int edb_ipc_attach(int peer_rank, const void* handle) {
  Runtime& r = g_rt;
  if (!r.inited) return set_error(EDB_E_STATE, "edb_ipc_attach: not initialised");
  EDB_REQUIRE(peer_rank >= 0 && peer_rank < r.world, "edb_ipc_attach: bad peer %d", peer_rank);
  if (peer_rank == r.rank) return EDB_OK;
  if (r.peer_heap[peer_rank]) return EDB_OK;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  EDB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  r.peer_heap[peer_rank] = static_cast<char*>(p);
  r.peer_is_ipc[peer_rank] = true;
  return EDB_OK;
}

int edb_attach_local(int peer_rank, void* base) {
  Runtime& r = g_rt;
  if (!r.inited) return set_error(EDB_E_STATE, "edb_attach_local: not initialised");
  EDB_REQUIRE(peer_rank >= 0 && peer_rank < r.world, "edb_attach_local: bad peer %d", peer_rank);
  r.peer_heap[peer_rank] = static_cast<char*>(base);
  r.peer_is_ipc[peer_rank] = false;
  return EDB_OK;
}

int edb_group_create(const int* ranks, int n, int slot, int* gid_out) {
  Runtime& r = g_rt;
  if (!r.inited) return set_error(EDB_E_STATE, "edb_group_create: not initialised");
  EDB_REQUIRE(n >= 1 && n <= kMaxGroup, "edb_group_create: group size %d not in [1,%d]", n,
              kMaxGroup);
  EDB_REQUIRE(slot >= 0 && slot < kMaxGroups, "edb_group_create: slot %d out of range", slot);
  EDB_REQUIRE(r.ngroups < kMaxGroups, "edb_group_create: too many groups");
  int me = -1;
  for (int i = 0; i < n; ++i) {
    EDB_REQUIRE(ranks[i] >= 0 && ranks[i] < r.world, "edb_group_create: rank %d out of range",
                ranks[i]);
    for (int j = 0; j < i; ++j)
      EDB_REQUIRE(ranks[j] != ranks[i], "edb_group_create: duplicate rank %d", ranks[i]);
    if (ranks[i] == r.rank) me = i;
  }
  EDB_REQUIRE(me >= 0, "edb_group_create: calling rank %d is not a member", r.rank);
  for (int g = 0; g < r.ngroups; ++g)
    EDB_REQUIRE(r.groups[g].slot != slot, "edb_group_create: slot %d already in use", slot);
  for (int i = 0; i < n; ++i)
    if (!r.peer_heap[ranks[i]])
      return set_error(EDB_E_STATE, "edb_group_create: peer %d not attached", ranks[i]);
  Group& g = r.groups[r.ngroups];
  g.n = n;
  g.me = me;
  g.slot = slot;
  for (int i = 0; i < n; ++i) g.ranks[i] = ranks[i];
  *gid_out = r.ngroups++;
  return EDB_OK;
}

int edb_group_info(int gid, int* n_out, int* my_index_out) {
  Runtime& r = g_rt;
  EDB_REQUIRE(r.inited && gid >= 0 && gid < r.ngroups, "edb_group_info: bad gid %d", gid);
  if (n_out) *n_out = r.groups[gid].n;
  if (my_index_out) *my_index_out = r.groups[gid].me;
  return EDB_OK;
}

int edb_symm_alloc(size_t bytes, size_t align, uint64_t* offset_out) {
  Runtime& r = g_rt;
  if (!r.inited) return set_error(EDB_E_STATE, "edb_symm_alloc: not initialised");
  if (align < 256) align = 256;
  EDB_REQUIRE((align & (align - 1)) == 0, "edb_symm_alloc: align %zu not a power of two", align);
  size_t off = (r.bump + align - 1) & ~(align - 1);
  if (off + bytes > r.heap_bytes)
    return set_error(EDB_E_STATE,
                     "edb_symm_alloc: symmetric heap exhausted (%zu + %zu > %zu); raise "
                     "EDB_HEAP_BYTES",
                     off, bytes, r.heap_bytes);
  r.bump = off + bytes;
  *offset_out = off;
  return EDB_OK;
}

int edb_symm_mark(uint64_t* mark_out) {
  if (!g_rt.inited) return set_error(EDB_E_STATE, "edb_symm_mark: not initialised");
  *mark_out = g_rt.bump;
  return EDB_OK;
}

int edb_symm_reset(uint64_t mark) {
  Runtime& r = g_rt;
  if (!r.inited) return set_error(EDB_E_STATE, "edb_symm_reset: not initialised");
  EDB_REQUIRE(mark >= kUserOffset && mark <= r.heap_bytes, "edb_symm_reset: bad mark");
  r.bump = mark;
  return EDB_OK;
}

int edb_set_option(const char* name, int64_t value) {
  Runtime& r = g_rt;
  if (!strcmp(name, "allreduce_oneshot_bytes")) r.allreduce_oneshot_bytes = value;
  else if (!strcmp(name, "copy_ctas_per_sm")) r.copy_ctas_per_sm = value;
  else if (!strcmp(name, "comm_ctas")) r.comm_ctas = value;
  else if (!strcmp(name, "spin_timeout_ms")) r.spin_timeout_ms = value;
  else if (!strcmp(name, "gemm_splitk")) r.gemm_splitk = value;
  else if (!strcmp(name, "gemm_force_bn")) r.gemm_force_bn = value;
  else if (!strcmp(name, "gemm2")) {
    if (value != 0 && value != 1) return set_error(EDB_E_INVALID, "edb_set_option: gemm2 must be 0 or 1");
    r.gemm2 = value;
  }
  else if (!strcmp(name, "ll_max_bytes")) r.ll_max_bytes = value;
  else if (!strcmp(name, "push_sync")) r.push_sync = value;
  else return set_error(EDB_E_INVALID, "edb_set_option: unknown option '%s'", name);
  return EDB_OK;
}

int edb_get_option(const char* name, int64_t* out) {
  Runtime& r = g_rt;
  if (!strcmp(name, "allreduce_oneshot_bytes")) *out = r.allreduce_oneshot_bytes;
  else if (!strcmp(name, "copy_ctas_per_sm")) *out = r.copy_ctas_per_sm;
  else if (!strcmp(name, "comm_ctas")) *out = r.comm_ctas;
  else if (!strcmp(name, "spin_timeout_ms")) *out = r.spin_timeout_ms;
  else if (!strcmp(name, "gemm_splitk")) *out = r.gemm_splitk;
  else if (!strcmp(name, "gemm_force_bn")) *out = r.gemm_force_bn;
  else if (!strcmp(name, "gemm2")) *out = gemm2_enabled() ? 1 : 0;
  else if (!strcmp(name, "ll_max_bytes")) *out = r.ll_max_bytes;
  else if (!strcmp(name, "push_sync")) *out = r.push_sync;
  else if (!strcmp(name, "sm_count")) *out = r.sm_count;
  else if (!strcmp(name, "rank")) *out = r.rank;
  else if (!strcmp(name, "world")) *out = r.world;
  else return set_error(EDB_E_INVALID, "edb_get_option: unknown option '%s'", name);
  return EDB_OK;
}

}  // extern "C"
