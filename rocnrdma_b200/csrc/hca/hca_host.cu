// Host side of the software HCA: verbs-shaped object model (HCA context, MR, CQ,
// QP with the RC state machine, connect) + engine lifecycle + host-posted verbs,
// exported as a flat C ABI (rn_*) for ctypes and the C++ tools.
//
// Reference parity:
//   rn_reg_mr / rn_dereg_mr  ~ acquire + get_pages + dma_map / dma_unmap + put_pages + release
//                              (amdp2p.c:112-167, :169-216, :219-264, :266-313, :345-360)
//   rn_mr_revoke             ~ free_callback -> invalidate (amdp2p.c:88-109); here an explicit
//                              state machine (PINNED -> REVOKED -> RELEASED), not a bare flag
//   rn_hca_open failure modes~ amd_peer_bridge_init (amdp2p.c:374-399)
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>

#include "engine.cuh"
#include "hca_types.h"

using namespace rn;

#define RN_API extern "C" __attribute__((visibility("default")))

namespace {

thread_local char g_err[512] = "";
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}
#define CU_OK(call)                                                                        \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess) return fail(-(int)e_ - 1000, "%s: %s", #call, cudaGetErrorString(e_)); \
  } while (0)

enum MrState : int { MR_FREE = 0, MR_PINNED = 1, MR_REVOKED = 2 };

struct Mr {
  int state = MR_FREE;
  uint64_t base = 0, len = 0;
  uint32_t key = 0, access = 0, kind = 0;
  bool host_registered_by_us = false;
  int dmabuf_fd = -1;
  uint8_t tag = 0;
  uint64_t buffer_id = 0;     // CUDA allocation identity at registration (device memory); 0 = not tracked
  bool driver_revoked = false;
};

struct Cq {
  struct Hca* hca;
  CqDev h;            // host shadow
  CqDev* d;           // device struct
  uint32_t mem;       // MemKind of ring
  uint8_t* ring_host; // valid when mem == MEM_HOST_PINNED (same VA on device under UVA)
  uint32_t h_ci = 0;  // host consumer index
};

struct Qp {
  struct Hca* hca;
  QpDev h;            // host shadow of static part
  QpDev* d;
  uint32_t sq_mem;
  Cq *scq, *rcq;
  Qp* peer_local = nullptr;
  uint64_t h_sq_pi = 0, h_rq_pi = 0;   // host poster indices
  uint64_t h_sq_done = 0;              // send WQEs known complete (from polled CQEs, or the engine's retire head)
  uint64_t h_rq_done = 0;              // receive WQEs known consumed (from polled responder CQEs)
  bool in_engine_table = false;
  bool adopted = false;                // queues belong to a real HCA (mlx5dv): the engine never sees this QP
};

struct Hca {
  int dev = 0;
  cudaStream_t ctl = nullptr, eng = nullptr, work = nullptr, aux = nullptr;
  cudaStream_t pool[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // extra pre-created poster streams
  uint8_t *arena = nullptr, *harena = nullptr;
  size_t arena_size = 0, arena_off = 0, harena_size = 0, harena_off = 0;
  uint32_t max_mkeys = 0;
  MKeyEntry* d_mkeys = nullptr;
  std::vector<Mr> mrs;
  EngineCtl* d_ctl = nullptr;
  volatile uint32_t* h_stop = nullptr;
  uint8_t* scratch = nullptr;          // mapped pinned result area (kernels write, host reads)
  size_t scratch_size = 0;
  uint8_t* dscratch = nullptr;         // zeroed device scratch for kernel counters (kernels self-clean)
  size_t dscratch_size = 0;
  QpDev** d_qptab = nullptr;
  uint32_t max_qps = 0;
  std::vector<Qp*> qps;
  std::vector<Cq*> cqs;
  uint32_t next_qpn = 0x100, next_cqn = 1;
  int engine_ctas = 0;
  bool engine_launched = false;
  int oneshot = 0;
  uint64_t idle_timeout_ns = 5ull * 1000000000ull, rnr_timeout_ns = 500ull * 1000000ull;
  std::mutex mu;
};

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

void* arena_alloc(Hca* h, size_t bytes, bool host) {
  size_t& off = host ? h->harena_off : h->arena_off;
  size_t cap = host ? h->harena_size : h->arena_size;
  size_t o = align_up(off, 256);
  if (o + bytes > cap) return nullptr;
  off = o + bytes;
  return (host ? h->harena : h->arena) + o;
}

int push(Hca* h, void* dst, const void* src, size_t n) {
  CU_OK(cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, h->ctl));
  CU_OK(cudaStreamSynchronize(h->ctl));
  return 0;
}
int pull(Hca* h, void* dst, const void* src, size_t n) { return push(h, dst, src, n); }

int log2_exact(uint32_t v) {
  if (v == 0 || (v & (v - 1))) return -1;
  int l = 0;
  while ((1u << l) < v) ++l;
  return l;
}

bool legal_transition(uint32_t from, uint32_t to) {
  if (to == QPS_RESET || to == QPS_ERR) return true;
  if (from == QPS_RESET && to == QPS_INIT) return true;
  if (from == QPS_INIT && (to == QPS_INIT || to == QPS_RTR)) return true;
  if (from == QPS_RTR && to == QPS_RTS) return true;
  if (from == QPS_RTS && (to == QPS_RTS || to == QPS_SQD)) return true;
  if (from == QPS_SQD && to == QPS_RTS) return true;
  if (from == QPS_SQE && to == QPS_RTS) return true;
  return false;
}

}  // namespace

// Every translation unit with kernels exports rn_preload_<tu>(): it touches each
// kernel with cudaFuncGetAttributes so the driver loads the code NOW.  With CUDA's
// default lazy module loading the first launch of a kernel loads it, and that load is
// serialised behind a resident persistent kernel -- a poster launched for the first
// time while the engine runs would only start after the engine's watchdog exit
// (observed with driver 580.159; see DESIGN.md "engine residency rules").
extern "C" {
uint64_t rn_gemm_workspace_bytes() __attribute__((weak));
void rn_gemm_set_workspace(int dev, uint64_t ptr) __attribute__((weak));
void rn_preload_rdma_ops() __attribute__((weak));
void rn_preload_pack() __attribute__((weak));
void rn_preload_gemm() __attribute__((weak));
void rn_preload_gemm_mx() __attribute__((weak));
}
static void preload_all_kernels() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, eng::engine_kernel);
  if (rn_preload_rdma_ops) rn_preload_rdma_ops();
  if (rn_preload_pack) rn_preload_pack();
  if (rn_preload_gemm) rn_preload_gemm();
  if (rn_preload_gemm_mx) rn_preload_gemm_mx();
  cudaGetLastError();
}

RN_API const char* rn_last_error() { return g_err; }

RN_API int rn_abi_sizes(uint32_t* out, int n) {
  uint32_t v[] = {(uint32_t)sizeof(Wqe64),    (uint32_t)sizeof(Cqe64), (uint32_t)sizeof(MKeyEntry),
                  (uint32_t)sizeof(Resolved), (uint32_t)sizeof(QpDev), (uint32_t)sizeof(CqDev),
                  (uint32_t)sizeof(EngineCtl), (uint32_t)sizeof(RemoteView)};
  for (int i = 0; i < n && i < (int)(sizeof v / sizeof v[0]); ++i) out[i] = v[i];
  return (int)(sizeof v / sizeof v[0]);
}

// ------------------------------------------------------------------ context
RN_API int rn_hca_open(int dev, uint32_t max_mkeys, uint32_t max_qps, uint64_t arena_bytes,
                       uint64_t host_arena_bytes, void** out) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail(-1, "no CUDA device: %s", cudaGetErrorString(e));
  if (dev < 0 || dev >= ndev) return fail(-2, "device %d out of range (%d devices)", dev, ndev);
  CU_OK(cudaSetDevice(dev));
  Hca* h = new Hca();
  h->dev = dev;
  int lo, hi;
  CU_OK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  CU_OK(cudaStreamCreateWithPriority(&h->ctl, cudaStreamNonBlocking, hi));
  CU_OK(cudaStreamCreateWithPriority(&h->eng, cudaStreamNonBlocking, hi));
  // Work stream for posters: created now because creating a stream (like any allocation)
  // is serialised behind a running persistent kernel by the driver.
  CU_OK(cudaStreamCreateWithFlags(&h->work, cudaStreamNonBlocking));
  CU_OK(cudaStreamCreateWithFlags(&h->aux, cudaStreamNonBlocking));
  for (auto& st : h->pool) CU_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  h->arena_size = arena_bytes ? arena_bytes : (64ull << 20);
  h->harena_size = host_arena_bytes ? host_arena_bytes : (16ull << 20);
  CU_OK(cudaMalloc(&h->arena, h->arena_size));
  CU_OK(cudaMemsetAsync(h->arena, 0, h->arena_size, h->ctl));
  CU_OK(cudaHostAlloc(&h->harena, h->harena_size, cudaHostAllocMapped | cudaHostAllocPortable));
  memset(h->harena, 0, h->harena_size);
  h->max_mkeys = max_mkeys ? max_mkeys : 1024;
  h->max_qps = max_qps ? max_qps : 256;
  h->d_mkeys = (MKeyEntry*)arena_alloc(h, sizeof(MKeyEntry) * h->max_mkeys, false);
  h->d_ctl = (EngineCtl*)arena_alloc(h, sizeof(EngineCtl), false);
  h->d_qptab = (QpDev**)arena_alloc(h, sizeof(QpDev*) * h->max_qps, false);
  h->h_stop = (volatile uint32_t*)arena_alloc(h, 64, true);
  h->scratch_size = 256 << 10;
  h->scratch = (uint8_t*)arena_alloc(h, h->scratch_size, true);
  h->dscratch_size = 1 << 20;
  h->dscratch = (uint8_t*)arena_alloc(h, h->dscratch_size, false);
  h->mrs.resize(h->max_mkeys);
  if (rn_gemm_workspace_bytes && rn_gemm_set_workspace) {
    // stream-K workspace of the wide GEMM kernel (one per device, shared by every context on it; never freed: a
    // later context may still be launching GEMMs that use it)
    static void* ws_by_dev[16] = {};
    if (dev < 16 && !ws_by_dev[dev]) {
      const size_t n = (size_t)rn_gemm_workspace_bytes();
      if (cudaMalloc(&ws_by_dev[dev], n) == cudaSuccess) cudaMemsetAsync(ws_by_dev[dev], 0, n, h->ctl);
      else { ws_by_dev[dev] = nullptr; cudaGetLastError(); }
    }
    if (dev < 16) rn_gemm_set_workspace(dev, (uint64_t)ws_by_dev[dev]);
  }
  preload_all_kernels();
  CU_OK(cudaStreamSynchronize(h->ctl));
  *out = h;
  return 0;
}

RN_API int rn_engine_stop(void* hca);

RN_API int rn_hca_close(void* hca) {
  Hca* h = (Hca*)hca;
  if (!h) return 0;
  cudaSetDevice(h->dev);
  rn_engine_stop(h);
  for (auto& m : h->mrs)
    if (m.state != MR_FREE && m.host_registered_by_us) cudaHostUnregister((void*)m.base);
  for (auto* q : h->qps) delete q;
  for (auto* c : h->cqs) delete c;
  cudaFree(h->arena);
  cudaFreeHost(h->harena);
  cudaStreamDestroy(h->ctl);
  cudaStreamDestroy(h->eng);
  // work/aux are handed to PyTorch as ExternalStreams; its allocators may still record events on
  // them when tensors that were used there die (after close()), so they live for the process.
  cudaStreamSynchronize(h->work);
  cudaStreamSynchronize(h->aux);
  delete h;
  return 0;
}

RN_API uint64_t rn_hca_dev_scratch(void* hca, uint64_t* size) {
  Hca* h = (Hca*)hca;
  if (size) *size = h->dscratch_size;
  return (uint64_t)h->dscratch;
}
// Let this HCA's GPU (its engine, its posters) reach memory of `peer_dev` over NVLink: MKey tables,
// receive rings and CQs of a peer HCA live there when two GPUs are connected.
RN_API int rn_hca_enable_peer(void* hca, int peer_dev) {
  Hca* h = (Hca*)hca;
  CU_OK(cudaSetDevice(h->dev));
  if (peer_dev == h->dev) return 0;
  int can = 0;
  CU_OK(cudaDeviceCanAccessPeer(&can, h->dev, peer_dev));
  if (!can) return fail(-13, "device %d cannot access device %d", h->dev, peer_dev);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_dev, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(-13, "enable peer access: %s", cudaGetErrorString(e));
  cudaGetLastError();
  return 0;
}
RN_API int rn_set_device(int dev) { return cudaSetDevice(dev) == cudaSuccess ? 0 : -19; }
RN_API uint64_t rn_hca_work_stream(void* hca) { return (uint64_t)((Hca*)hca)->work; }
RN_API uint64_t rn_hca_aux_stream(void* hca) { return (uint64_t)((Hca*)hca)->aux; }
// stream i of the pre-created set: 0 = work, 1 = aux, 2..7 = pool
RN_API uint64_t rn_hca_stream(void* hca, int i) {
  Hca* h = (Hca*)hca;
  if (i == 0) return (uint64_t)h->work;
  if (i == 1) return (uint64_t)h->aux;
  if (i >= 2 && i < 8) return (uint64_t)h->pool[i - 2];
  return 0;
}
RN_API uint64_t rn_hca_scratch(void* hca, uint64_t* size) {
  Hca* h = (Hca*)hca;
  if (size) *size = h->scratch_size;
  return (uint64_t)h->scratch;
}
RN_API uint64_t rn_hca_mkey_table(void* hca) { return (uint64_t)((Hca*)hca)->d_mkeys; }
RN_API uint64_t rn_hca_arena(void* hca, uint64_t* size) {
  Hca* h = (Hca*)hca;
  if (size) *size = h->arena_size;
  return (uint64_t)h->arena;
}

// ------------------------------------------------------------------ memory regions
// classify: 0 = not CUDA-known host memory, 1 = device memory, 2 = pinned/registered host
RN_API int rn_classify_ptr(uint64_t ptr, int* device_out) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, (void*)ptr);
  if (e != cudaSuccess) { cudaGetLastError(); return 0; }
  if (device_out) *device_out = a.device;
  if (a.type == cudaMemoryTypeDevice) return 1;
  if (a.type == cudaMemoryTypeHost) return 2;
  if (a.type == cudaMemoryTypeManaged) return 3;
  return 0;
}

extern "C" int rn_buffer_id(uint64_t ptr, uint64_t* id) __attribute__((weak));
extern "C" int rn_dmabuf_export(uint64_t ptr, uint64_t len, int* cu_err_out) __attribute__((weak));
extern "C" int rn_dmabuf_close(int fd) __attribute__((weak));

RN_API int rn_reg_mr(void* hca, uint64_t ptr, uint64_t len, uint32_t access, uint32_t* key_out);

// Registration modes (SURVEY.md N1): 0 = direct (software HCA translates the VA itself),
// 1 = dmabuf (additionally export the 4 KiB-aligned range as a dma-buf fd -- the pin an HCA would be
// given through ibv_reg_dmabuf_mr; the fd is the pin's owner and is closed on dereg / revoke).
RN_API int rn_reg_mr_mode(void* hca, uint64_t ptr, uint64_t len, uint32_t access, uint32_t mode, uint32_t* key_out,
                          int* dmabuf_fd_out) {
  Hca* h = (Hca*)hca;
  if (dmabuf_fd_out) *dmabuf_fd_out = -1;
  int fd = -1;
  if (mode == 1) {
    if (!rn_dmabuf_export) return fail(-38, "reg_mr: dma-buf support not built");
    CU_OK(cudaSetDevice(h->dev));
    uint64_t lo = ptr & ~4095ull, hi = (ptr + len + 4095) & ~4095ull;
    int cu = 0;
    fd = rn_dmabuf_export(lo, hi - lo, &cu);
    if (fd < 0) return fail(fd, "reg_mr: dma-buf export of [0x%llx, +0x%llx) failed (CUresult %d)", (unsigned long long)lo,
                            (unsigned long long)(hi - lo), cu);
  }
  int rc = rn_reg_mr(hca, ptr, len, access, key_out);
  if (rc) { if (fd >= 0) rn_dmabuf_close(fd); return rc; }
  if (fd >= 0) {
    std::lock_guard<std::mutex> g(h->mu);
    h->mrs[*key_out >> 8].dmabuf_fd = fd;
  }
  if (dmabuf_fd_out) *dmabuf_fd_out = fd;
  return 0;
}

RN_API int rn_reg_mr(void* hca, uint64_t ptr, uint64_t len, uint32_t access, uint32_t* key_out) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  if (len == 0 || ptr == 0) return fail(-22, "reg_mr: null or empty range");
  if (ptr + len < ptr) return fail(-22, "reg_mr: range wraps");
  int pdev = -1;
  int cls = rn_classify_ptr(ptr, &pdev);
  Mr m;
  if (cls == 1) {
    m.kind = (pdev == h->dev) ? MEM_DEVICE : MEM_PEER;
    if (pdev != h->dev) {
      int can = 0;
      cudaDeviceCanAccessPeer(&can, h->dev, pdev);
      if (!can) return fail(-13, "reg_mr: device %d memory is not peer-accessible from device %d", pdev, h->dev);
      cudaError_t e = cudaDeviceEnablePeerAccess(pdev, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
        return fail(-13, "enable peer access: %s", cudaGetErrorString(e));
      cudaGetLastError();
    }
  } else if (cls == 2) {
    m.kind = MEM_HOST_PINNED;
  } else if (cls == 0) {
    // plain host memory: pin it, as ibv_reg_mr would
    cudaError_t e = cudaHostRegister((void*)ptr, len, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(-14, "reg_mr: cannot pin host range: %s", cudaGetErrorString(e)); }
    m.kind = MEM_HOST_PINNED;
    m.host_registered_by_us = true;
  } else {
    return fail(-95, "reg_mr: managed memory is not registrable");
  }
  uint32_t idx = 0;
  for (; idx < h->max_mkeys; ++idx)
    if (h->mrs[idx].state == MR_FREE) break;
  if (idx == h->max_mkeys) return fail(-12, "reg_mr: MKey table full (%u)", h->max_mkeys);
  if (cls == 1 && rn_buffer_id) rn_buffer_id(ptr, &m.buffer_id);
  m.tag = (uint8_t)(h->mrs[idx].tag + 1);  // a recycled index never yields the old key
  m.state = MR_PINNED;
  m.base = ptr; m.len = len; m.access = access;
  m.key = (idx << 8) | m.tag;
  MKeyEntry e{};
  e.base = ptr; e.len = len; e.map_base = ptr; e.key = m.key; e.access = access; e.valid = 1; e.kind = m.kind;
  int rc = push(h, h->d_mkeys + idx, &e, sizeof e);
  if (rc) return rc;
  h->mrs[idx] = m;
  *key_out = m.key;
  return 0;
}

static int mr_lookup(Hca* h, uint32_t key, uint32_t* idx) {
  uint32_t i = key >> 8;
  if (i >= h->max_mkeys || h->mrs[i].state == MR_FREE || h->mrs[i].key != key) return fail(-22, "unknown MKey 0x%x", key);
  *idx = i;
  return 0;
}

// Revocation: the memory is going away under a live MR (cudaFree while registered).
// The MKey stops translating immediately; dereg afterwards only releases the slot.
RN_API int rn_mr_revoke(void* hca, uint32_t key) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  uint32_t i = 0;
  int rc = mr_lookup(h, key, &i);
  if (rc) return rc;
  if (h->mrs[i].state == MR_REVOKED) return 0;
  uint32_t zero = 0;
  rc = push(h, &h->d_mkeys[i].valid, &zero, sizeof zero);
  if (rc) return rc;
  h->mrs[i].state = MR_REVOKED;
  if (h->mrs[i].dmabuf_fd >= 0 && rn_dmabuf_close) { rn_dmabuf_close(h->mrs[i].dmabuf_fd); h->mrs[i].dmabuf_fd = -1; }   // the pin goes with the memory
  return 0;
}

// Driver-originated revocation.  The kernel bridge learns that pinned memory is going away through the GPU
// driver's free callback (kmod/b200p2p.c: b200_free_callback; reference amdp2p.c:88-109).  A userspace HCA has no
// such upcall, so it asks the driver: every device-memory registration remembers the CUDA allocation id it was
// made on; a registration whose pointer the driver no longer knows, or that now belongs to a different
// allocation, is revoked exactly as if the callback had fired (MKey stops translating, the dma-buf pin is
// dropped).  Called by the host-side post path and the kernel launch wrappers, by Context.sweep_revoked(), and by
// the optional watcher thread.  Returns the number of registrations revoked by this call.
RN_API int rn_hca_sweep_revoked(void* hca) {
  Hca* h = (Hca*)hca;
  if (!rn_buffer_id) return 0;
  std::lock_guard<std::mutex> g(h->mu);
  cudaSetDevice(h->dev);
  int n = 0;
  for (uint32_t i = 0; i < h->max_mkeys; ++i) {
    Mr& m = h->mrs[i];
    if (m.state != MR_PINNED || !m.buffer_id) continue;
    uint64_t now = 0;
    const int rc = rn_buffer_id(m.base, &now);
    if (rc == 0 && now == m.buffer_id) continue;
    uint32_t zero = 0;
    if (push(h, &h->d_mkeys[i].valid, &zero, sizeof zero)) continue;
    m.state = MR_REVOKED;
    m.driver_revoked = true;
    if (m.dmabuf_fd >= 0 && rn_dmabuf_close) { rn_dmabuf_close(m.dmabuf_fd); m.dmabuf_fd = -1; }
    ++n;
  }
  return n;
}
RN_API int rn_mr_driver_revoked(void* hca, uint32_t key) {
  Hca* h = (Hca*)hca;
  uint32_t i = key >> 8;
  return i < h->max_mkeys && h->mrs[i].key == key && h->mrs[i].driver_revoked ? 1 : 0;
}

RN_API int rn_dereg_mr(void* hca, uint32_t key) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  uint32_t i = 0;
  int rc = mr_lookup(h, key, &i);
  if (rc) return rc;
  Mr& m = h->mrs[i];
  if (m.state == MR_PINNED) {
    uint32_t zero = 0;
    rc = push(h, &h->d_mkeys[i].valid, &zero, sizeof zero);
    if (rc) return rc;
    if (m.host_registered_by_us) cudaHostUnregister((void*)m.base);
  }
  if (m.dmabuf_fd >= 0 && rn_dmabuf_close) rn_dmabuf_close(m.dmabuf_fd);
  uint8_t tag = m.tag;
  m = Mr();
  m.tag = tag;
  return 0;
}

RN_API int rn_mr_state(void* hca, uint32_t key) {
  Hca* h = (Hca*)hca;
  uint32_t i = key >> 8;
  if (i >= h->max_mkeys || h->mrs[i].key != key) return MR_FREE;
  return h->mrs[i].state;
}

// ------------------------------------------------------------------ completion queues
RN_API int rn_create_cq(void* hca, uint32_t ncqe, uint32_t mem, void** out) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  int lg = log2_exact(ncqe);
  if (lg < 1 || lg > 20) return fail(-22, "create_cq: ncqe must be a power of two in [2, 2^20]");
  bool host = mem == MEM_HOST_PINNED;
  Cq* c = new Cq();
  c->hca = h;
  c->mem = mem;
  uint8_t* ring = (uint8_t*)arena_alloc(h, (size_t)ncqe * 64, host);
  uint32_t* dbrec = (uint32_t*)arena_alloc(h, 64, host);
  c->d = (CqDev*)arena_alloc(h, sizeof(CqDev), false);
  if (!ring || !dbrec || !c->d) { delete c; return fail(-12, "create_cq: control arena exhausted"); }
  // every CQE starts INVALID with owner = 1 (the first hardware pass writes owner 0)
  std::vector<uint8_t> init((size_t)ncqe * 64, 0);
  for (uint32_t i = 0; i < ncqe; ++i) init[(size_t)i * 64 + 63] = cqe_op_own(CQE_INVALID, 1);
  if (host) memcpy(ring, init.data(), init.size());
  else { int rc = push(h, ring, init.data(), init.size()); if (rc) { delete c; return rc; } }
  c->ring_host = host ? ring : nullptr;
  c->h.buf = ring; c->h.dbrec = dbrec; c->h.log_n = (uint32_t)lg; c->h.cqn = h->next_cqn++;
  c->h.pi = 0; c->h.ci = 0; c->h.overruns = 0;
  int rc = push(h, c->d, &c->h, sizeof(CqDev));
  if (rc) { delete c; return rc; }
  h->cqs.push_back(c);
  *out = c;
  return 0;
}
RN_API uint64_t rn_cq_dev(void* cq) { return (uint64_t)((Cq*)cq)->d; }

struct RnWc {          // host-visible work completion
  uint32_t qpn, byte_cnt, imm;
  uint16_t wqe_counter;
  uint8_t opcode, syndrome, wqe_opcode, is_error;
};

RN_API int rn_poll_cq(void* cq, int max, RnWc* out) {
  Cq* c = (Cq*)cq;
  Hca* h = c->hca;
  int n = 0;
  while (n < max) {
    Cqe64 cqe;
    size_t off = (size_t)(c->h_ci & ((1u << c->h.log_n) - 1)) << 6;
    if (c->ring_host) {
      volatile uint8_t* p = c->ring_host + off;
      uint8_t oo = p[63];
      if (!cqe_valid(oo, c->h_ci, c->h.log_n)) break;
      __sync_synchronize();
      memcpy(&cqe, (const void*)p, 64);
    } else {
      cudaSetDevice(h->dev);
      if (pull(h, &cqe, c->h.buf + off, 64)) return -5;
      if (!cqe_valid(cqe.op_own, c->h_ci, c->h.log_n)) break;
    }
    CqeView v;
    decode_cqe(&cqe, &v);
    out[n].qpn = v.qpn; out[n].byte_cnt = v.byte_cnt; out[n].imm = v.imm;
    out[n].wqe_counter = v.wqe_counter; out[n].opcode = v.opcode; out[n].syndrome = v.syndrome;
    out[n].wqe_opcode = v.wqe_opcode; out[n].is_error = v.is_error;
    // flow-control credit for the host poster (rn_post_send / rn_post_recv refuse a full queue)
    for (auto* q : h->qps) {
      if (q->h.qpn != v.qpn) continue;
      if (v.opcode == CQE_REQ || v.opcode == CQE_REQ_ERR) {
        uint64_t done = q->h_sq_done + (uint16_t)(v.wqe_counter + 1 - (uint16_t)q->h_sq_done);
        if (done <= q->h_sq_pi) q->h_sq_done = done;
      } else if (q->rcq == c) {
        uint64_t done = q->h_rq_done + (uint16_t)(v.wqe_counter + 1 - (uint16_t)q->h_rq_done);
        if (done <= q->h_rq_pi) q->h_rq_done = done;
      }
      break;
    }
    ++n;
    ++c->h_ci;
  }
  if (n) {
    uint32_t rec = be32(c->h_ci & 0xffffff);
    if (c->ring_host) *(volatile uint32_t*)c->h.dbrec = rec;
    else push(h, c->h.dbrec, &rec, 4);
  }
  return n;
}

// ------------------------------------------------------------------ queue pairs
RN_API int rn_create_qp(void* hca, void* scq, void* rcq, uint32_t nsq, uint32_t nrq, uint32_t sq_mem,
                        uint32_t chunk_bytes, void** out) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  int ls = log2_exact(nsq), lr = log2_exact(nrq);
  // 16384, not 32768: the doorbell carries a 16-bit index and the engine tells "pending" from "wrapped" by
  // a signed 16-bit distance, so at most 2^15 - 1 WQEs may ever be outstanding.
  if (ls < 1 || ls > 14 || lr < 1 || lr > 14) return fail(-22, "create_qp: queue depths must be powers of two in [2, 16384]");
  if (!scq || !rcq) return fail(-22, "create_qp: CQs required");
  if (h->qps.size() >= h->max_qps) return fail(-12, "create_qp: QP table full");
  if (chunk_bytes == 0) chunk_bytes = 512u << 10;
  if (chunk_bytes & 15) return fail(-22, "create_qp: chunk_bytes must be a multiple of 16");
  bool host = sq_mem == MEM_HOST_PINNED;
  Qp* q = new Qp();
  q->hca = h; q->sq_mem = sq_mem; q->scq = (Cq*)scq; q->rcq = (Cq*)rcq;
  uint8_t* sq = (uint8_t*)arena_alloc(h, (size_t)nsq * 64, host);
  uint8_t* rq = (uint8_t*)arena_alloc(h, (size_t)nrq * 16, host);
  uint32_t* dbr = (uint32_t*)arena_alloc(h, 64, host);
  unsigned long long* bf = (unsigned long long*)arena_alloc(h, 64, host);
  Resolved* res = (Resolved*)arena_alloc(h, (size_t)nsq * sizeof(Resolved), false);
  unsigned long long* trace = (unsigned long long*)arena_alloc(h, (size_t)nsq * 64, false);
  uint32_t* flags = (uint32_t*)arena_alloc(h, (size_t)nsq * 4, false);
  q->d = (QpDev*)arena_alloc(h, sizeof(QpDev), false);
  if (!sq || !rq || !dbr || !bf || !res || !trace || !flags || !q->d) { delete q; return fail(-12, "create_qp: control arena exhausted"); }
  memset(&q->h, 0, sizeof q->h);
  q->h.qpn = h->next_qpn++;
  q->h.state = QPS_RESET;
  q->h.sq = sq; q->h.sq_log = (uint32_t)ls; q->h.rq = rq; q->h.rq_log = (uint32_t)lr;
  q->h.dbr = dbr; q->h.bf = bf;
  q->h.scq = q->scq->d; q->h.rcq = q->rcq->d;
  q->h.lkeys = h->d_mkeys; q->h.n_lkeys = h->max_mkeys;
  q->h.chunk_bytes = chunk_bytes;
  q->h.resolved = res;
  q->h.trace = trace;
  q->h.ready_flags = flags;
  q->h.trace_on = 0;
  q->h.sq_in_device = host ? 0 : 1;
  q->h.sys_scope = (host || q->scq->mem == MEM_HOST_PINNED || q->rcq->mem == MEM_HOST_PINNED) ? 1 : 0;
  // doorbell register idle value: "last posted index = 0xffff" <=> nothing posted
  unsigned long long bf0 = (unsigned long long)ctrl_word0(OP_NOP, 0xffff) | ((unsigned long long)ctrl_word1(q->h.qpn, 0) << 32);
  int rc = 0;
  if (host) *bf = bf0; else rc = push(h, bf, &bf0, 8);
  if (!rc) rc = push(h, q->d, &q->h, sizeof(QpDev));
  if (rc) { delete q; return rc; }
  h->qps.push_back(q);
  *out = q;
  return 0;
}
RN_API uint64_t rn_qp_dev(void* qp) { return (uint64_t)((Qp*)qp)->d; }
// Force system-scope fences (peer-GPU or real-NIC connections) / toggle lifecycle tracing.
RN_API int rn_qp_set_flags(void* qp, int sys_scope, int trace_on) {
  Qp* q = (Qp*)qp;
  cudaSetDevice(q->hca->dev);
  int rc = 0;
  if (sys_scope >= 0) { q->h.sys_scope = (uint32_t)sys_scope; rc = push(q->hca, &q->d->sys_scope, &q->h.sys_scope, 4); }
  if (!rc && trace_on >= 0) { q->h.trace_on = (uint32_t)trace_on; rc = push(q->hca, &q->d->trace_on, &q->h.trace_on, 4); }
  return rc;
}
// Copy out the lifecycle stamps of SQ slots [0, n): 8 u64 per slot.
RN_API int rn_qp_read_trace(void* qp, uint64_t* out, uint32_t nslots) {
  Qp* q = (Qp*)qp;
  cudaSetDevice(q->hca->dev);
  uint32_t depth = 1u << q->h.sq_log;
  if (nslots > depth) nslots = depth;
  return pull(q->hca, out, q->h.trace, (size_t)nslots * 64);
}
RN_API uint32_t rn_qp_num(void* qp) { return ((Qp*)qp)->h.qpn; }
RN_API uint32_t rn_qp_state(void* qp) {
  Qp* q = (Qp*)qp;
  uint32_t s = 0;
  cudaSetDevice(q->hca->dev);
  pull(q->hca, &s, (const void*)&q->d->state, 4);
  q->h.state = s;
  return s;
}

struct RnRemote {       // everything a requester needs about the responder, pre-translated
  uint64_t rkeys; uint32_t n_rkeys; uint32_t qpn;
  uint64_t rq; uint64_t rq_dbr; uint32_t rq_log; uint32_t pad;
  uint64_t rcq; uint64_t rcq_buf;
};

RN_API int rn_qp_describe(void* qp, RnRemote* out) {
  Qp* q = (Qp*)qp;
  out->rkeys = (uint64_t)q->hca->d_mkeys; out->n_rkeys = q->hca->max_mkeys; out->qpn = q->h.qpn;
  out->rq = (uint64_t)q->h.rq; out->rq_dbr = (uint64_t)q->h.dbr; out->rq_log = q->h.rq_log;
  out->pad = 1;   // flags, bit 0: pointers are in the describer's own address space (a cross-process translation clears it)
  out->rcq = (uint64_t)q->rcq->d; out->rcq_buf = (uint64_t)q->rcq->h.buf;
  return 0;
}

RN_API int rn_qp_connect(void* qp, const RnRemote* r) {
  Qp* q = (Qp*)qp;
  Hca* h = q->hca;
  std::lock_guard<std::mutex> g(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  uint32_t st = rn_qp_state(q);
  if (st != QPS_INIT) return fail(-22, "connect: QP must be in INIT (is %u)", st);
  q->h.r.rkeys = (MKeyEntry*)r->rkeys; q->h.r.n_rkeys = r->n_rkeys; q->h.r.qpn = r->qpn;
  q->h.r.rq = (uint8_t*)r->rq; q->h.r.rq_dbr = (uint32_t*)r->rq_dbr; q->h.r.rq_log = r->rq_log;
  q->h.r.rcq = (CqDev*)r->rcq; q->h.r.rcq_buf = (uint8_t*)r->rcq_buf;
  q->h.r.connected = 1u | ((r->pad & 1u) ? 2u : 0u);   // bit 1: the responder's CQ consumer record is addressable as is
  return push(h, &q->d->r, &q->h.r, sizeof(RemoteView));
}

RN_API int rn_modify_qp(void* qp, uint32_t new_state) {
  Qp* q = (Qp*)qp;
  Hca* h = q->hca;
  std::lock_guard<std::mutex> g(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  if (q->adopted) return fail(-95, "modify_qp: this QP belongs to a real HCA; change its state through the verbs backend");
  uint32_t st = rn_qp_state(q);
  if (!legal_transition(st, new_state)) return fail(-22, "modify_qp: illegal transition %u -> %u", st, new_state);
  if (new_state == QPS_RTR && !q->h.r.connected) return fail(-22, "modify_qp: RTR requires a connected peer");
  if (new_state == QPS_RESET) {
    // back to a pristine queue: indices, cursor and doorbell all rewind
    QpDev fresh = q->h;
    memset(&fresh.resv_head, 0, sizeof(QpDev) - offsetof(QpDev, resv_head));
    fresh.r = RemoteView{};
    fresh.state = QPS_RESET;
    q->h = fresh;
    q->h_sq_pi = q->h_rq_pi = 0;
    unsigned long long bf0 = (unsigned long long)ctrl_word0(OP_NOP, 0xffff) | ((unsigned long long)ctrl_word1(q->h.qpn, 0) << 32);
    int rc = push(h, q->h.bf, &bf0, 8);
    uint32_t z[2] = {0, 0};
    if (!rc) rc = push(h, q->h.dbr, z, 8);
    if (!rc) rc = cudaMemsetAsync(q->h.resolved, 0, sizeof(Resolved) << q->h.sq_log, h->ctl) == cudaSuccess ? 0 : -5;
    // Ready flags are generation-tagged with idx + 1 and indices restart at 0: a flag left from the previous
    // life would make the shared submit ring the doorbell over a WQE nobody has written yet, and the stale WQE
    // bytes (matching index and qpn) would be executed again.  Clear both.
    if (!rc) rc = cudaMemsetAsync(q->h.ready_flags, 0, sizeof(uint32_t) << q->h.sq_log, h->ctl) == cudaSuccess ? 0 : -5;
    if (!rc) {
      if (q->sq_mem == MEM_HOST_PINNED) memset(q->h.sq, 0, (size_t)64 << q->h.sq_log);
      else rc = cudaMemsetAsync(q->h.sq, 0, (size_t)64 << q->h.sq_log, h->ctl) == cudaSuccess ? 0 : -5;
    }
    q->h_sq_done = q->h_rq_done = 0;
    if (!rc) rc = push(h, q->d, &q->h, sizeof(QpDev));
    return rc;
  }
  q->h.state = new_state;
  int rc = push(h, (void*)&q->d->state, &new_state, 4);
  if (rc) return rc;
  if (new_state == QPS_RTS && !q->in_engine_table) {
    uint32_t slot = 0;
    for (auto* o : h->qps) if (o->in_engine_table) ++slot;
    QpDev* dptr = q->d;
    rc = push(h, h->d_qptab + slot, &dptr, sizeof dptr);
    uint32_t n = slot + 1;
    if (!rc) rc = push(h, (void*)&h->d_ctl->n_qps, &n, 4);
    if (!rc) q->in_engine_table = true;
  }
  return rc;
}

// Loopback / in-process helper: INIT both, cross-connect, RTR, RTS.
RN_API int rn_qp_connect_pair(void* a, void* b) {
  Qp *qa = (Qp*)a, *qb = (Qp*)b;
  int rc;
  RnRemote ra, rb;
  if ((rc = rn_modify_qp(qa, QPS_INIT))) return rc;
  if (qb != qa && (rc = rn_modify_qp(qb, QPS_INIT))) return rc;
  rn_qp_describe(qa, &ra);
  rn_qp_describe(qb, &rb);
  if ((rc = rn_qp_connect(qa, &rb))) return rc;
  if (qb != qa && (rc = rn_qp_connect(qb, &ra))) return rc;
  qa->peer_local = qb; qb->peer_local = qa;
  if ((rc = rn_modify_qp(qa, QPS_RTR)) || (rc = rn_modify_qp(qa, QPS_RTS))) return rc;
  if (qb != qa && ((rc = rn_modify_qp(qb, QPS_RTR)) || (rc = rn_modify_qp(qb, QPS_RTS)))) return rc;
  return 0;
}

struct RnQpCounters {
  uint64_t n_wqe, n_cqe, n_err, n_db_order_violations, n_bytes, n_rnr;
  uint64_t resv_head, ready_head, sq_cons, cursor, retire_head;
  uint32_t state, pad;
};
RN_API int rn_qp_query(void* qp, RnQpCounters* out) {
  Qp* q = (Qp*)qp;
  QpDev d;
  cudaSetDevice(q->hca->dev);
  int rc = pull(q->hca, &d, q->d, sizeof d);
  if (rc) return rc;
  out->n_wqe = d.n_wqe; out->n_cqe = d.n_cqe; out->n_err = d.n_err;
  out->n_db_order_violations = d.n_db_order_violations; out->n_bytes = d.n_bytes; out->n_rnr = d.n_rnr;
  out->resv_head = d.resv_head; out->ready_head = d.ready_head; out->sq_cons = d.sq_cons;
  out->cursor = d.cursor; out->retire_head = d.retire_head;  // cursor = claim head
  out->state = d.state; out->pad = 0;
  return 0;
}

// ------------------------------------------------------------------ adoption of a real HCA's queues (N3)
// verbs_dl.cc (rn_verbs_map_qp_to_gpu) maps an mlx5 QP's send / receive rings, doorbell record, BlueFlame
// register and completion queues into this GPU's address space; this wraps them in the QpDev / CqDev the
// device-side poster (hca/post.cuh) already speaks, so rdma_stream_kernel, pack_fp8_write_kernel and the
// GEMM epilogue drive a ConnectX with the code that drives the software HCA.  What differs from a softhca QP:
//   * every ring lives outside the GPU (host memory the NIC reads over PCIe; the register is MMIO), so
//     sq_in_device = 0 and the poster's doorbell release is system scope;
//   * geometry comes from the provider: wqe_cnt / cqe_cnt are powers of two but not ours to choose;
//   * the engine never sees the QP (no MKey table, no resolved[] slots): the NIC executes the WQEs.
// The QP must be fresh (nothing posted or polled through libibverbs): the producer / consumer indices start
// at 0 here, as they do in the hardware.
struct RnGpuQp {
  uint64_t sq_dev, rq_dev, dbrec_dev, bf_dev, cq_dev, cq_dbrec_dev, rcq_dev, rcq_dbrec_dev;
  uint32_t sq_wqe_cnt, rq_wqe_cnt, cq_cqe_cnt, rcq_cqe_cnt, qpn, cqn, rcqn, flags;
};
RN_API int rn_qp_adopt(void* hca, const RnGpuQp* g, void** out) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> lk(h->mu);
  CU_OK(cudaSetDevice(h->dev));
  const int ls = log2_exact(g->sq_wqe_cnt), lr = log2_exact(g->rq_wqe_cnt), lc = log2_exact(g->cq_cqe_cnt), lrc = log2_exact(g->rcq_cqe_cnt);
  if (ls < 0 || lr < 0 || lc < 0 || lrc < 0) return fail(-22, "adopt: queue sizes must be powers of two (sq %u rq %u cq %u rcq %u)",
                                                         g->sq_wqe_cnt, g->rq_wqe_cnt, g->cq_cqe_cnt, g->rcq_cqe_cnt);
  if (ls > 15) return fail(-22, "adopt: send queue of %u WQEBBs exceeds the 16-bit doorbell window", g->sq_wqe_cnt);
  if (!g->sq_dev || !g->dbrec_dev || !g->bf_dev || !g->cq_dev || !g->cq_dbrec_dev) return fail(-22, "adopt: unmapped queue");
  auto make_cq = [&](uint64_t buf, uint64_t dbrec, int lg, uint32_t cqn) -> Cq* {
    Cq* c = new Cq();
    c->hca = h; c->mem = MEM_HOST_PINNED; c->ring_host = nullptr;     // polled on the device, never by rn_poll_cq
    c->d = (CqDev*)arena_alloc(h, sizeof(CqDev), false);
    if (!c->d) { delete c; return nullptr; }
    memset(&c->h, 0, sizeof c->h);
    c->h.buf = (uint8_t*)buf; c->h.dbrec = (uint32_t*)dbrec; c->h.log_n = (uint32_t)lg; c->h.cqn = cqn;
    if (push(h, c->d, &c->h, sizeof(CqDev))) { delete c; return nullptr; }
    h->cqs.push_back(c);
    return c;
  };
  Cq* scq = make_cq(g->cq_dev, g->cq_dbrec_dev, lc, g->cqn);
  Cq* rcq = (g->rcq_dev && g->rcq_dev != g->cq_dev) ? make_cq(g->rcq_dev, g->rcq_dbrec_dev, lrc, g->rcqn) : scq;
  if (!scq || !rcq) return fail(-12, "adopt: control arena exhausted");
  Qp* q = new Qp();
  q->hca = h; q->sq_mem = MEM_HOST_PINNED; q->scq = scq; q->rcq = rcq; q->adopted = true;
  const uint32_t nsq = g->sq_wqe_cnt;
  unsigned long long* trace = (unsigned long long*)arena_alloc(h, (size_t)nsq * 64, false);
  uint32_t* flags = (uint32_t*)arena_alloc(h, (size_t)nsq * 4, false);
  q->d = (QpDev*)arena_alloc(h, sizeof(QpDev), false);
  if (!trace || !flags || !q->d) { delete q; return fail(-12, "adopt: control arena exhausted"); }
  memset(&q->h, 0, sizeof q->h);
  q->h.qpn = g->qpn;
  q->h.state = QPS_RTS;
  q->h.sq = (uint8_t*)g->sq_dev; q->h.sq_log = (uint32_t)ls;
  q->h.rq = (uint8_t*)g->rq_dev; q->h.rq_log = (uint32_t)lr;
  q->h.dbr = (uint32_t*)g->dbrec_dev; q->h.bf = (unsigned long long*)g->bf_dev;
  q->h.scq = scq->d; q->h.rcq = rcq->d;
  q->h.lkeys = nullptr; q->h.n_lkeys = 0; q->h.chunk_bytes = 0;
  q->h.sys_scope = 1; q->h.sq_in_device = 0;
  q->h.trace = trace; q->h.ready_flags = flags; q->h.resolved = nullptr;
  int rc = push(h, q->d, &q->h, sizeof(QpDev));
  if (rc) { delete q; return rc; }
  h->qps.push_back(q);
  *out = q;
  return 0;
}
RN_API int rn_qp_is_adopted(void* qp) { return ((Qp*)qp)->adopted ? 1 : 0; }

// ------------------------------------------------------------------ host-posted verbs
static int host_store(Qp* q, void* dst, const void* src, size_t n) {
  if (q->sq_mem == MEM_HOST_PINNED) { memcpy(dst, src, n); return 0; }
  return push(q->hca, dst, src, n);
}

RN_API int rn_post_send(void* qp, uint32_t opcode, uint64_t laddr, uint32_t lkey, uint64_t raddr, uint32_t rkey,
                        uint32_t bytes, uint32_t flags, uint32_t imm, uint64_t* idx_out) {
  Qp* q = (Qp*)qp;
  if (q->adopted) return fail(-95, "post_send: adopted QPs are posted to by device kernels only");
  cudaSetDevice(q->hca->dev);
  uint64_t idx = q->h_sq_pi;
  const uint64_t depth = 1ull << q->h.sq_log;
  if (idx - q->h_sq_done >= depth) {
    // Unsignaled WQEs produce no CQE: before refusing, ask the engine how far it has retired.
    unsigned long long rh = 0;
    if (!pull(q->hca, &rh, &q->d->retire_head, 8) && rh > q->h_sq_done && rh <= idx) q->h_sq_done = rh;
    if (idx - q->h_sq_done >= depth)
      return fail(-12, "post_send: send queue full (%llu posted, %llu complete, depth %llu): poll the CQ first",
                  (unsigned long long)idx, (unsigned long long)q->h_sq_done, (unsigned long long)depth);
  }
  Wqe64 w;
  memset(&w, 0, sizeof w);
  switch (opcode) {
    case OP_RDMA_WRITE: case OP_RDMA_WRITE_IMM: case OP_RDMA_READ:
      build_rdma_wqe(&w, (uint8_t)opcode, (uint16_t)idx, q->h.qpn, laddr, lkey, raddr, rkey, bytes, (uint8_t)flags, imm);
      break;
    case OP_SEND: case OP_SEND_IMM:
      build_send_wqe(&w, (uint8_t)opcode, (uint16_t)idx, q->h.qpn, laddr, lkey, bytes, (uint8_t)flags, imm);
      break;
    case OP_NOP:
      encode_ctrl(&w.ctrl, OP_NOP, (uint16_t)idx, q->h.qpn, 1, (uint8_t)flags, 0);
      break;
    default:
      // deliberately still posted: lets tests drive the engine's bad-opcode path
      encode_ctrl(&w.ctrl, (uint8_t)opcode, (uint16_t)idx, q->h.qpn, 1, (uint8_t)flags, 0);
  }
  uint8_t* slot = q->h.sq + ((idx & ((1ull << q->h.sq_log) - 1)) << 6);
  int rc = host_store(q, slot, &w, 64);
  if (rc) return rc;
  __sync_synchronize();
  uint32_t rec = be32((uint32_t)((idx + 1) & 0xffff));
  rc = host_store(q, &q->h.dbr[DBR_SND], &rec, 4);
  if (rc) return rc;
  __sync_synchronize();
  unsigned long long db = (unsigned long long)ctrl_word0(OP_NOP, (uint16_t)idx) | ((unsigned long long)ctrl_word1(q->h.qpn, 0) << 32);
  rc = host_store(q, q->h.bf, &db, 8);
  if (rc) return rc;
  q->h_sq_pi = idx + 1;
  if (idx_out) *idx_out = idx;
  return 0;
}

RN_API int rn_post_recv(void* qp, uint64_t addr, uint32_t lkey, uint32_t bytes) {
  Qp* q = (Qp*)qp;
  cudaSetDevice(q->hca->dev);
  uint64_t i = q->h_rq_pi;
  if (i - q->h_rq_done >= (1ull << q->h.rq_log)) {
    // Consumption is only visible to the host through polled responder CQEs; when a kernel consumes the
    // receive CQ instead, ask the requester's engine state (possible when the peer QP is in this process).
    unsigned long long taken = 0;
    if (q->peer_local && !pull(q->hca, &taken, &q->peer_local->d->rq_head, 8) && taken > q->h_rq_done && taken <= i)
      q->h_rq_done = taken;
    const bool can_know = q->peer_local || q->rcq->ring_host;
    if (can_know && i - q->h_rq_done >= (1ull << q->h.rq_log))
      return fail(-12, "post_recv: receive queue full (%llu posted, %llu consumed): poll the receive CQ first",
                  (unsigned long long)i, (unsigned long long)q->h_rq_done);
  }
  RecvWqe w;
  encode_data(&w.data, addr, lkey, bytes);
  int rc = host_store(q, q->h.rq + ((i & ((1ull << q->h.rq_log) - 1)) << 4), &w, 16);
  if (rc) return rc;
  __sync_synchronize();
  uint32_t rec = be32((uint32_t)((i + 1) & 0xffff));
  rc = host_store(q, &q->h.dbr[DBR_RCV], &rec, 4);
  if (rc) return rc;
  q->h_rq_pi = i + 1;
  // keep the device poster's view coherent if a kernel later posts receives too
  unsigned long long pi = i + 1;
  return push(q->hca, &q->d->rq_pi, &pi, 8);
}

// ------------------------------------------------------------------ engine lifecycle
RN_API int rn_engine_running(void* hca) {
  Hca* h = (Hca*)hca;
  if (!h->engine_launched) return 0;
  cudaSetDevice(h->dev);
  cudaError_t e = cudaStreamQuery(h->eng);
  if (e == cudaErrorNotReady) return 1;
  cudaGetLastError();
  h->engine_launched = false;
  return 0;
}

RN_API int rn_engine_set_oneshot(void* hca, int on) { ((Hca*)hca)->oneshot = on; return 0; }
RN_API int rn_engine_wait(void* hca) {
  Hca* h = (Hca*)hca;
  if (!h->engine_launched) return 0;
  cudaSetDevice(h->dev);
  cudaError_t e = cudaStreamSynchronize(h->eng);
  h->engine_launched = false;
  return e == cudaSuccess ? 0 : fail(-5, "engine wait: %s", cudaGetErrorString(e));
}

RN_API int rn_engine_start(void* hca, int n_ctas, uint64_t idle_timeout_ms, uint64_t rnr_timeout_ms) {
  Hca* h = (Hca*)hca;
  CU_OK(cudaSetDevice(h->dev));
  if (rn_engine_running(h)) {
    if (n_ctas == h->engine_ctas || n_ctas <= 0) return 0;
    rn_engine_stop(h);
  }
  // Anything the caller queued on the legacy default stream (torch.zeros / randn / copies initialising the buffers it is
  // about to post) must have RUN before the engine becomes resident: legacy-stream work that has not started by then is
  // held behind the persistent kernel (DESIGN.md 3.2) and would execute after the transfers it was meant to precede --
  // compute-sanitizer's slow launches showed exactly that (zero-fills landing on top of delivered data).  Free when idle.
  CU_OK(cudaStreamSynchronize(cudaStreamLegacy));
  cudaDeviceProp prop;
  CU_OK(cudaGetDeviceProperties(&prop, h->dev));
  if (n_ctas <= 0) n_ctas = h->engine_ctas > 0 ? h->engine_ctas : 32;
  if (n_ctas > prop.multiProcessorCount) n_ctas = prop.multiProcessorCount;
  if (idle_timeout_ms) h->idle_timeout_ns = idle_timeout_ms * 1000000ull;
  if (rnr_timeout_ms) h->rnr_timeout_ns = rnr_timeout_ms * 1000000ull;
  *h->h_stop = 0;
  EngineCtl c;
  memset(&c, 0, sizeof c);
  uint32_t nq = 0;
  for (auto* q : h->qps) if (q->in_engine_table) ++nq;
  c.stop = h->h_stop; c.qps = h->d_qptab; c.n_qps = nq; c.max_qps = h->max_qps;
  c.idle_timeout_ns = h->idle_timeout_ns; c.rnr_timeout_ns = h->rnr_timeout_ns;
  c.oneshot = h->oneshot;
  {
    const char* e = getenv("RN_ENGINE_STORES_IN_FLIGHT");
    int v = e ? atoi(e) : 0;
    c.stores_in_flight = (v == 4 || v == 6 || v == 8) ? (unsigned)v : 4u;
  }
  int rc = push(h, h->d_ctl, &c, sizeof c);
  if (rc) return rc;
  size_t smem = eng::engine_smem_bytes();
  CU_OK(cudaFuncSetAttribute(eng::engine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eng::engine_kernel<<<n_ctas, eng::kThreads, smem, h->eng>>>(h->d_ctl);
  CU_OK(cudaGetLastError());
  h->engine_ctas = n_ctas;
  h->engine_launched = true;
  return 0;
}

RN_API int rn_engine_stop(void* hca) {
  Hca* h = (Hca*)hca;
  if (!h->engine_launched) return 0;
  cudaSetDevice(h->dev);
  *h->h_stop = 1;
  __sync_synchronize();
  cudaError_t e = cudaStreamSynchronize(h->eng);
  *h->h_stop = 0;
  h->engine_launched = false;
  if (e != cudaSuccess) return fail(-5, "engine stop: %s", cudaGetErrorString(e));
  return 0;
}

struct RnEngineStats { uint64_t n_bulk_chunks, t_start, t_exit; uint32_t running_ctas, exited_idle, fatal, n_qps, ctas, pad; };
RN_API int rn_engine_stats(void* hca, RnEngineStats* out) {
  Hca* h = (Hca*)hca;
  EngineCtl c;
  cudaSetDevice(h->dev);
  int rc = pull(h, &c, h->d_ctl, sizeof c);
  if (rc) return rc;
  out->n_bulk_chunks = c.n_bulk_chunks; out->t_start = c.t_start; out->t_exit = c.t_exit; out->fatal = c.fatal; out->pad = 0;
  out->running_ctas = c.running_ctas; out->exited_idle = c.exited_idle; out->n_qps = c.n_qps;
  out->ctas = (uint32_t)h->engine_ctas;
  return 0;
}

// ------------------------------------------------------------------ test hooks (tier-0, no GPU)
RN_API void rn_wire_build_wqe(uint8_t* out64, uint32_t opcode, uint32_t idx, uint32_t qpn, uint64_t laddr,
                              uint32_t lkey, uint64_t raddr, uint32_t rkey, uint32_t bytes, uint32_t flags,
                              uint32_t imm) {
  Wqe64 w;
  memset(&w, 0, sizeof w);
  if (opcode == OP_SEND || opcode == OP_SEND_IMM)
    build_send_wqe(&w, (uint8_t)opcode, (uint16_t)idx, qpn, laddr, lkey, bytes, (uint8_t)flags, imm);
  else
    build_rdma_wqe(&w, (uint8_t)opcode, (uint16_t)idx, qpn, laddr, lkey, raddr, rkey, bytes, (uint8_t)flags, imm);
  memcpy(out64, &w, 64);
}
RN_API int rn_wire_decode_cqe(const uint8_t* cqe64, RnWc* out) {
  Cqe64 c;
  memcpy(&c, cqe64, 64);
  CqeView v;
  decode_cqe(&c, &v);
  out->qpn = v.qpn; out->byte_cnt = v.byte_cnt; out->imm = v.imm; out->wqe_counter = v.wqe_counter;
  out->opcode = v.opcode; out->syndrome = v.syndrome; out->wqe_opcode = v.wqe_opcode; out->is_error = v.is_error;
  return 0;
}

// ------------------------------------------------------------------ host-driven baselines (B1 / B2 of BASELINE.md)
#include <chrono>
static inline uint64_t now_ns() {
  return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// B2: the host posts (like ib_write_bw on a peermem MR): window-limited stream of `iters` work requests on a QP
// whose rings live in pinned host memory, CQ polled by the CPU.  Returns elapsed ns through *ns_out.
RN_API int rn_host_stream(void* qp, uint32_t opcode, uint64_t laddr, uint32_t lkey, uint64_t raddr, uint32_t rkey,
                          uint32_t bytes, uint32_t iters, uint32_t window, uint64_t slot_stride, uint32_t nslots,
                          uint64_t timeout_ms, uint64_t* ns_out, uint32_t* errors_out) {
  Qp* q = (Qp*)qp;
  if (q->sq_mem != MEM_HOST_PINNED || !q->scq->ring_host) return fail(-22, "host_stream: QP and CQ rings must be in pinned host memory");
  if (!window || window > (1u << q->h.sq_log)) window = 1u << q->h.sq_log;
  if (!nslots) nslots = 1;
  uint32_t posted = 0, done = 0, errors = 0;
  RnWc wc[32];
  const uint64_t t0 = now_ns(), deadline = t0 + (timeout_ms ? timeout_ms : 5000) * 1000000ull;
  while (done < iters) {
    while (posted < iters && posted - done < window) {
      uint64_t off = (uint64_t)(posted % nslots) * slot_stride;
      int rc = rn_post_send(qp, opcode, laddr + off, lkey, raddr + off, rkey, bytes, CTRL_CQ_UPDATE, 0, nullptr);
      if (rc) return rc;
      ++posted;
    }
    int n = rn_poll_cq(q->scq, 32, wc);
    if (n < 0) return n;
    for (int i = 0; i < n; ++i) errors += wc[i].is_error;
    done += (uint32_t)n;
    if (!n && now_ns() > deadline) return fail(-110, "host_stream: timed out with %u/%u completions", done, iters);
  }
  *ns_out = now_ns() - t0;
  if (errors_out) *errors_out = errors;
  return 0;
}

// B1: host-staged.  Per message: cudaMemcpy D2H into a pinned bounce buffer, host-posted RDMA write between two
// host MRs, cudaMemcpy H2D out of the second bounce buffer.  Everything the GPU-direct path exists to avoid.
RN_API int rn_host_staged_stream(void* qp, uint64_t dev_src, uint64_t dev_dst, uint64_t host_a, uint32_t lkey_a,
                                 uint64_t host_b, uint32_t rkey_b, uint32_t bytes, uint32_t iters, uint64_t slot_stride,
                                 uint32_t nslots, uint64_t timeout_ms, uint64_t* ns_out) {
  Qp* q = (Qp*)qp;
  Hca* h = q->hca;
  if (q->sq_mem != MEM_HOST_PINNED || !q->scq->ring_host) return fail(-22, "host_staged: QP and CQ rings must be in pinned host memory");
  CU_OK(cudaSetDevice(h->dev));
  if (!nslots) nslots = 1;
  RnWc wc;
  const uint64_t t0 = now_ns();
  for (uint32_t i = 0; i < iters; ++i) {
    uint64_t off = (uint64_t)(i % nslots) * slot_stride;
    CU_OK(cudaMemcpyAsync((void*)host_a, (const void*)(dev_src + off), bytes, cudaMemcpyDeviceToHost, h->ctl));
    CU_OK(cudaStreamSynchronize(h->ctl));
    int rc = rn_post_send(qp, OP_RDMA_WRITE, host_a, lkey_a, host_b, rkey_b, bytes, CTRL_CQ_UPDATE, 0, nullptr);
    if (rc) return rc;
    const uint64_t deadline = now_ns() + (timeout_ms ? timeout_ms : 5000) * 1000000ull;
    int n = 0;
    while ((n = rn_poll_cq(q->scq, 1, &wc)) == 0)
      if (now_ns() > deadline) return fail(-110, "host_staged: completion timed out");
    if (n < 0 || wc.is_error) return fail(-5, "host_staged: error completion (syndrome 0x%x)", wc.syndrome);
    CU_OK(cudaMemcpyAsync((void*)(dev_dst + off), (const void*)host_b, bytes, cudaMemcpyHostToDevice, h->ctl));
    CU_OK(cudaStreamSynchronize(h->ctl));
  }
  *ns_out = now_ns() - t0;
  return 0;
}

// ------------------------------------------------------------------ cross-process peers (CUDA IPC over NVLink)
extern "C" int rn_alloc_range(uint64_t ptr, uint64_t* base, uint64_t* size) __attribute__((weak));

// Export the cudaMalloc allocation that contains ptr: 64-byte IPC handle + where ptr sits inside it.
RN_API int rn_ipc_export(uint64_t ptr, uint8_t* handle64, uint64_t* alloc_base, uint64_t* alloc_size) {
  uint64_t base = ptr, size = 0;
  if (rn_alloc_range && rn_alloc_range(ptr, &base, &size)) return fail(-22, "ipc_export: 0x%llx is not inside a CUDA allocation", (unsigned long long)ptr);
  cudaIpcMemHandle_t h;
  CU_OK(cudaIpcGetMemHandle(&h, (void*)base));
  static_assert(sizeof(h) == 64, "IPC handle size");
  memcpy(handle64, &h, 64);
  *alloc_base = base;
  *alloc_size = size;
  return 0;
}
RN_API int rn_ipc_open(void* hca, const uint8_t* handle64, uint64_t* mapped_base) {
  Hca* hh = (Hca*)hca;
  CU_OK(cudaSetDevice(hh->dev));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  CU_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *mapped_base = (uint64_t)p;
  return 0;
}
RN_API int rn_ipc_close(uint64_t mapped_base) { return cudaIpcCloseMemHandle((void*)mapped_base) == cudaSuccess ? 0 : -5; }

// A local mirror of a peer HCA's MKey table whose map_base fields point at OUR mappings of the peer's memory.
RN_API uint64_t rn_hca_alloc_remote_table(void* hca, uint32_t n) {
  Hca* h = (Hca*)hca;
  std::lock_guard<std::mutex> g(h->mu);
  return (uint64_t)arena_alloc(h, sizeof(MKeyEntry) * (size_t)n, false);
}
RN_API int rn_hca_set_remote_mkey(void* hca, uint64_t table, uint32_t idx, uint64_t base, uint64_t len, uint64_t map_base,
                                  uint32_t key, uint32_t access) {
  Hca* h = (Hca*)hca;
  CU_OK(cudaSetDevice(h->dev));
  MKeyEntry e{};
  e.base = base; e.len = len; e.map_base = map_base; e.key = key; e.access = access; e.valid = 1; e.kind = MEM_PEER;
  return push(h, (MKeyEntry*)table + idx, &e, sizeof e);
}
