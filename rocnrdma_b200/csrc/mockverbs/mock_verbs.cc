// Mock rdma-core provider: a libibverbs.so.1 / libmlx5.so.1 look-alike whose "ConnectX" is a host
// thread.  It exists for the same reason kmod/shim mocks nvidia.ko and ib_core: the sandbox exposes no
// /dev/infiniband and ships no rdma-core, so without it the real-NIC backend (verbs/verbs_dl.cc), the
// mlx5dv queue adoption (hca/hca_host.cu: rn_qp_adopt) and the GPU-initiated posting code would never
// execute against anything that is shaped like a NIC.  The backend dlopen()s this exactly like the real
// libraries (ROCNRDMA_VERBS_LIBDIR points at lib/mock); nothing in the backend knows it is a mock.
//
// What is modelled, faithfully to the mlx5 programming interface:
//   * ibv_device / ibv_context (fast path through context->ops, as in the real library), PD, MR table
//     (lkey == rkey == index<<8 | tag, bounds + access checks), CQ, RC QP with the IB state machine and
//     the modify_qp attribute masks an mlx5 device insists on;
//   * queue memory exactly as rdma-core lays it out: one buffer [RQ | SQ] of 16-byte receive strides and
//     64-byte WQEBBs, a doorbell record {rcv, snd} of big-endian counters, a UAR page with two
//     alternating BlueFlame registers, CQEs of 64 bytes with the owner-bit protocol -- all in ordinary
//     host memory, which is where a real NIC's queues live too (the NIC reads them over PCIe);
//   * ibv_post_send builds real mlx5 WQEs (ctrl / raddr / data segments, big-endian) and rings the
//     doorbell; ibv_poll_cq parses real CQE64s.  mlx5dv_init_obj() exposes the raw queues, so a GPU
//     kernel can write WQEs and ring the doorbell itself (IBGDA) -- the "NIC" does not care who posted;
//   * the NIC: one thread that watches doorbell registers (a GPU store to a UAR page does not trap),
//     fetches WQEs, translates keys, moves the bytes (memcpy for host memory, cuMemcpyAsync through the
//     CUDA driver for device memory: the PCIe peer-to-peer DMA), writes CQEs, handles RNR, errors and
//     flushes.  Two mock devices share one "fabric", so NIC0 -> NIC1 transfers work.
//   * GPU memory registration the way ib_core does it: get_user_pages cannot pin a device pointer, so
//     ibv_reg_mr() asks the peer-memory clients.  ROCNRDMA_MOCK_PEERMEM selects who answers:
//       "1" (default)  a stock client is present (nvidia-peermem): device pointers register;
//       "0"            none: ibv_reg_mr(gpu_ptr) fails with EFAULT, as on a box without peermem;
//       "b200p2p"      the in-tree bridge: kmod/b200p2p.c compiled against kmod/shim runs its real
//                      acquire / get_pages / dma_map callbacks, the MR's translation table holds the BUS
//                      addresses it returned, and the NIC DMAs through them; freeing the memory fires the
//                      module's free callback -> invalidate -> the MR stops translating
//                      (reference: amdp2p.c:88-109, :112-264).
//     ibv_reg_dmabuf_mr() takes a dma-buf fd (CUDA-exported for HBM; a memfd is accepted as a host
//     "dma-buf" so the path is testable without a GPU).
//
// Send scatter-gather lists of up to two entries are modelled (one WQEBB per WQE); receive WQEs keep one.
// Not modelled: UD/UC, SRQ, events/completion channels, path MTU segmentation, retransmission.
#include <dlfcn.h>
#include <errno.h>
#include <fcntl.h>
#include <limits.h>
#include <sched.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <atomic>
#include <mutex>
#include <thread>
#include <vector>

#include "../verbs/abi/verbs_abi.h"
#include "../wire/mlx5_wire.h"

using namespace rnabi;
using rn::be32;
using rn::be64;

#define MOCK_API extern "C" __attribute__((visibility("default")))

namespace {

// ------------------------------------------------------------------ CUDA driver, loaded lazily (absent on CPU-only boxes)
typedef int CUresult;
typedef unsigned long long CUdeviceptr;
typedef void* CUcontext;
typedef void* CUstream;
struct Cuda {
  void* lib = nullptr;
  bool ok = false;
  CUresult (*init)(unsigned) = nullptr;
  CUresult (*pointer_attr)(void*, int, CUdeviceptr) = nullptr;
  CUresult (*ctx_set)(CUcontext) = nullptr;
  CUresult (*stream_create)(CUstream*, unsigned) = nullptr;
  CUresult (*stream_sync)(CUstream) = nullptr;
  CUresult (*memcpy_async)(CUdeviceptr, CUdeviceptr, size_t, CUstream) = nullptr;
  CUresult (*addr_range)(CUdeviceptr*, size_t*, CUdeviceptr) = nullptr;
};
enum { CU_ATTR_CONTEXT = 1, CU_ATTR_MEMORY_TYPE = 2, CU_MEMTYPE_DEVICE = 2 };
Cuda& cuda() {
  static Cuda c;
  static std::once_flag once;
  std::call_once(once, [] {
    if (getenv("ROCNRDMA_MOCK_NO_CUDA")) return;
    c.lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!c.lib) return;
#define CU(field, name) c.field = (decltype(c.field))dlsym(c.lib, name)
    CU(init, "cuInit"); CU(pointer_attr, "cuPointerGetAttribute"); CU(ctx_set, "cuCtxSetCurrent");
    CU(stream_create, "cuStreamCreate"); CU(stream_sync, "cuStreamSynchronize"); CU(memcpy_async, "cuMemcpyAsync");
    CU(addr_range, "cuMemGetAddressRange_v2");
#undef CU
    c.ok = c.init && c.pointer_attr && c.ctx_set && c.stream_create && c.stream_sync && c.memcpy_async && c.init(0) == 0;
  });
  return c;
}
// Device memory as the CUDA driver sees it (the only authority on what a "GPU address" is).
bool cuda_is_device_ptr(uint64_t p, CUcontext* ctx_out) {
  Cuda& c = cuda();
  if (!c.ok) return false;
  unsigned type = 0;
  if (c.pointer_attr(&type, CU_ATTR_MEMORY_TYPE, (CUdeviceptr)p) != 0 || type != CU_MEMTYPE_DEVICE) return false;
  if (ctx_out) { CUcontext x = nullptr; if (c.pointer_attr(&x, CU_ATTR_CONTEXT, (CUdeviceptr)p) == 0) *ctx_out = x; }
  return true;
}

// ------------------------------------------------------------------ b200p2p bridge (kmod sim), loaded lazily
struct Bridge {
  void* lib = nullptr;
  bool ok = false;
  int (*load)() = nullptr;
  int (*gpu_alloc)(uint64_t, uint64_t) = nullptr;
  int (*gpu_free)(uint64_t) = nullptr;
  uint64_t (*bus_addr)(uint64_t) = nullptr;
  long (*reg_mr)(uint64_t, uint64_t, int) = nullptr;
  int (*dereg_mr)(long) = nullptr;
  int (*mr_dma)(long, int, uint64_t*, uint64_t*) = nullptr;
  int (*mr_nmap)(long) = nullptr;
  int (*mr_invalidated)(long) = nullptr;
  uint64_t (*mr_page_size)(long) = nullptr;
  char why[256] = "";
};
Bridge& bridge() {
  static Bridge b;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* path = getenv("ROCNRDMA_KMOD_SIM");
    char buf[PATH_MAX];
    if (!path) {
      Dl_info di;
      if (dladdr((void*)&bridge, &di) && di.dli_fname) {   // <repo>/rocnrdma_b200/lib/mock/libibverbs.so.1 -> <repo>/kmod/...
        snprintf(buf, sizeof buf, "%s", di.dli_fname);
        for (int up = 0; up < 4; ++up) { char* s = strrchr(buf, '/'); if (s) *s = 0; }
        strncat(buf, "/kmod/libb200p2p_sim.so", sizeof buf - strlen(buf) - 1);
        path = buf;
      }
    }
    b.lib = path ? dlopen(path, RTLD_NOW | RTLD_LOCAL) : nullptr;
    if (!b.lib) { snprintf(b.why, sizeof b.why, "kmod simulation not loadable (%s): build it with tools/build_kmod_sim.py", path ? path : "?"); return; }
#define SIM(field, name) b.field = (decltype(b.field))dlsym(b.lib, name)
    SIM(load, "sim_b200p2p_load"); SIM(gpu_alloc, "sim_gpu_alloc"); SIM(gpu_free, "sim_gpu_free"); SIM(bus_addr, "sim_gpu_bus_addr");
    SIM(reg_mr, "sim_ib_reg_mr"); SIM(dereg_mr, "sim_ib_dereg_mr"); SIM(mr_dma, "sim_ib_mr_dma"); SIM(mr_nmap, "sim_ib_mr_nmap");
    SIM(mr_invalidated, "sim_ib_mr_invalidated"); SIM(mr_page_size, "sim_ib_mr_page_size");
#undef SIM
    if (!(b.load && b.gpu_alloc && b.gpu_free && b.bus_addr && b.reg_mr && b.dereg_mr && b.mr_dma && b.mr_nmap && b.mr_invalidated)) {
      snprintf(b.why, sizeof b.why, "kmod simulation lacks expected symbols");
      return;
    }
    int rc = b.load();          // insmod b200p2p: registers the peer-memory client with the mock ib_core
    if (rc) { snprintf(b.why, sizeof b.why, "b200p2p module init failed (%d)", rc); return; }
    b.ok = true;
  });
  return b;
}

// ------------------------------------------------------------------ object model
constexpr uint32_t kMaxMkeys = 4096, kMaxQps = 1024, kMaxCqs = 1024;
constexpr uint32_t kBfSize = 256, kBfOffset = 0x800;   // BlueFlame registers at page + 0x800 and + 0x900, like a UAR

enum MrKind { MR_HOST = 0, MR_DEVICE = 1, MR_DMABUF_MAPPED = 2, MR_BRIDGED = 3 };
struct MockMr {
  ibv_mr v;                // must be first: handed out as ibv_mr*
  bool live = false;
  int kind = MR_HOST;
  uint64_t iova = 0, len = 0;
  uint64_t map_base = 0;   // where the NIC reaches iova (identity except for an mmapped dma-buf)
  unsigned access = 0;
  uint8_t tag = 0;
  int dmabuf_fd = -1;
  void* mapping = nullptr; size_t mapping_len = 0;
  CUcontext cu_ctx = nullptr;
  // bridged registration: the translation table the peer-memory client produced
  long bridge_id = -1;
  int bridge_hca = 0;      // which HCA the client's dma_map was made for (the mapping is per device)
  uint64_t pin_va = 0;     // 64 KiB-aligned start of the pinned range
  std::vector<std::pair<uint64_t, uint64_t>> sg;   // (bus address, length)
};

struct MockCq {
  ibv_cq v;
  uint8_t* buf = nullptr;
  uint32_t* dbrec = nullptr;
  uint32_t log_n = 0, cqn = 0;
  std::atomic<uint32_t> pi{0};   // NIC producer
  uint32_t ci = 0;               // host consumer (ibv_poll_cq)
  uint64_t overruns = 0;
  struct MockCtx* ctx = nullptr;
};

struct MockQp {
  ibv_qp v;
  struct MockCtx* ctx = nullptr;
  MockCq *scq = nullptr, *rcq = nullptr;
  uint8_t* buf = nullptr;        // [RQ | SQ]
  size_t buf_len = 0;
  uint8_t *sq = nullptr, *rq = nullptr;
  uint32_t sq_cnt = 0, rq_cnt = 0;
  uint32_t* dbrec = nullptr;     // [0] rcv, [1] snd
  uint8_t* uar = nullptr;        // one page
  int sq_sig_all = 0;
  uint32_t max_sge = 1;          // send scatter-gather entries granted at create (1..MAX_SGE)
  // host poster (ibv_post_send / ibv_post_recv) state
  std::mutex post_mu;
  uint64_t sq_head = 0, sq_tail = 0, rq_head = 0, rq_tail = 0;
  uint32_t bf_off = 0;
  std::vector<uint64_t> sq_wrid, rq_wrid;
  // connection
  uint32_t dest_qpn = 0; uint16_t dlid = 0; uint8_t port = 1;
  unsigned access_flags = 0;
  // NIC state
  uint64_t hw_sq_cons = 0;       // next WQE index to execute
  uint64_t hw_rq_cons = 0;       // next receive WQE of THIS qp to consume (as responder)
  unsigned long long bf_seen[2] = {0, 0};
  uint64_t rnr_since_ns = 0;
  bool hw_err = false;
  // counters
  uint64_t n_wqe = 0, n_cqe = 0, n_err = 0, n_bytes = 0, n_rnr = 0, n_db_no_progress = 0, n_doorbells = 0;
};

struct MockDev {
  ibv_device v;
  int index = 0;
  uint16_t lid = 0;
  MockMr* mkeys[kMaxMkeys] = {};
  uint8_t mkey_tag[kMaxMkeys] = {};
  MockQp* qps[kMaxQps] = {};
  MockCq* cqs[kMaxCqs] = {};
};

struct MockCtx {
  ibv_context v;
  MockDev* dev = nullptr;
};
struct MockPd { ibv_pd v; };

constexpr int kMaxDevs = 8;
MockDev g_devs[kMaxDevs];
int g_ndev = 0;
std::recursive_mutex g_mu;               // object tables + NIC sweeps
std::thread g_nic;
std::atomic<bool> g_nic_run{false}, g_nic_stop{false};
std::atomic<uint64_t> g_rnr_timeout_ns{500ull * 1000000ull};
struct FakeGpuRange { uint64_t va, len; bool live; };
std::vector<FakeGpuRange> g_fake_gpu;    // host ranges a test declared to be "GPU memory" (CPU-only CI of the peer-memory path)

uint64_t now_ns() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}
uint32_t roundup_pow2(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }
uint32_t log2u(uint32_t v) { uint32_t l = 0; while ((1u << l) < v) ++l; return l; }
void* page_alloc(size_t n) {
  void* p = nullptr;
  n = (n + 4095) & ~(size_t)4095;
  if (posix_memalign(&p, 4096, n)) return nullptr;
  memset(p, 0, n);
  return p;
}

void init_devices() {
  static std::once_flag once;
  std::call_once(once, [] {
    const char* e = getenv("ROCNRDMA_MOCK_NDEV");
    g_ndev = e ? atoi(e) : 2;
    if (g_ndev < 1) g_ndev = 1;
    if (g_ndev > kMaxDevs) g_ndev = kMaxDevs;
    for (int i = 0; i < g_ndev; ++i) {
      MockDev& d = g_devs[i];
      memset(&d.v, 0, sizeof d.v);
      d.index = i; d.lid = (uint16_t)(i + 1);
      d.v.node_type = IBV_NODE_CA; d.v.transport_type = IBV_TRANSPORT_IB;
      snprintf(d.v.name, sizeof d.v.name, "mock_mlx5_%d", i);
      snprintf(d.v.dev_name, sizeof d.v.dev_name, "uverbs%d", i);
      snprintf(d.v.dev_path, sizeof d.v.dev_path, "/sys/class/infiniband_verbs/uverbs%d", i);
      snprintf(d.v.ibdev_path, sizeof d.v.ibdev_path, "/sys/class/infiniband/mock_mlx5_%d", i);
    }
  });
}

bool fake_gpu_range(uint64_t p, uint64_t n) {
  for (auto& r : g_fake_gpu) if (r.live && p >= r.va && p + n <= r.va + r.len) return true;
  return false;
}

// ------------------------------------------------------------------ key translation (what the HCA's MTT does)
// Returns the address through which the NIC reaches [addr, addr+n) of key, or 0 with *syn set.
uint64_t translate(MockDev* d, uint32_t key, uint64_t addr, uint64_t n, unsigned need, bool remote, uint8_t* syn, MockMr** mr_out) {
  const uint32_t idx = key >> 8;
  MockMr* m = idx < kMaxMkeys ? d->mkeys[idx] : nullptr;
  const uint8_t bad = remote ? rn::SYN_REMOTE_ACCESS_ERR : rn::SYN_LOCAL_PROT_ERR;
  if (!m || !m->live || m->v.lkey != key) { *syn = bad; return 0; }
  if (addr < m->iova || addr + n < addr || addr + n > m->iova + m->len) { *syn = bad; return 0; }
  if ((m->access & need) != need) { *syn = remote ? rn::SYN_REMOTE_ACCESS_ERR : rn::SYN_LOCAL_ACCESS_ERR; return 0; }
  if (mr_out) *mr_out = m;
  if (m->kind == MR_BRIDGED) {
    // The peer-memory client revoked the pages (GPU memory freed under the MR): ib_core invalidated the MR.
    if (bridge().mr_invalidated(m->bridge_id)) { *syn = bad; return 0; }
    // Walk the scatterlist the client's dma_map produced: bus address of the page that holds `addr`.
    uint64_t off = addr - m->pin_va;
    for (auto& e : m->sg) {
      if (off < e.second) {
        if (off + n > e.second && &e != &m->sg.back()) {
          // crosses an sg entry: entries of one pin are bus-contiguous in the simulation, checked here
          const auto& nx = *(&e + 1);
          if (nx.first != e.first + e.second) { *syn = bad; return 0; }
        }
        // This HCA's IOMMU window (the simulation folds the device id into bits 52+ so that a mapping made for
        // one HCA is useless to another), then the "PCIe fabric": bus address -> the memory the DMA lands on.
        const uint64_t iova = e.first + off;
        if ((iova >> 52) != (uint64_t)m->bridge_hca || d->index != m->bridge_hca) { *syn = bad; return 0; }
        return bridge().bus_addr(iova - ((uint64_t)m->bridge_hca << 52));
      }
      off -= e.second;
    }
    *syn = bad;
    return 0;
  }
  return m->map_base + (addr - m->iova);
}

// ------------------------------------------------------------------ DMA (the PCIe transfers of the NIC)
struct DmaStream { CUcontext ctx; CUstream st; };
std::vector<DmaStream> g_dma_streams;
CUstream dma_stream_for(CUcontext ctx) {
  for (auto& s : g_dma_streams) if (s.ctx == ctx) return s.st;
  Cuda& c = cuda();
  if (c.ctx_set(ctx) != 0) return nullptr;
  CUstream st = nullptr;
  if (c.stream_create(&st, 1 /* CU_STREAM_NON_BLOCKING */) != 0) return nullptr;
  g_dma_streams.push_back({ctx, st});
  return st;
}
// Copy n bytes; either side may be device memory.  Returns false when the transfer could not be made.
bool dma_copy(uint64_t dst, MockMr* dmr, uint64_t src, MockMr* smr, uint64_t n) {
  if (n == 0) return true;
  CUcontext cctx = nullptr;
  if (dmr && dmr->cu_ctx) cctx = dmr->cu_ctx;
  if (smr && smr->cu_ctx) cctx = smr->cu_ctx;
  if (!cctx) { memcpy((void*)dst, (const void*)src, n); return true; }
  Cuda& c = cuda();
  CUstream st = dma_stream_for(cctx);
  if (!st || c.ctx_set(cctx) != 0) return false;
  if (c.memcpy_async((CUdeviceptr)dst, (CUdeviceptr)src, n, st) != 0) return false;
  return c.stream_sync(st) == 0;
}

// 8-byte atomic on the responder's memory; *old = the value before.  Host memory: a __atomic builtin.  CUDA memory:
// read-modify-write through the DMA stream.  That is atomic with respect to this NIC only -- the NIC thread executes
// one WQE at a time -- which is what a ConnectX promises under IBV_ATOMIC_HCA (the GPU's own atomics on the word are
// not coordinated with it).
bool nic_atomic(uint8_t opcode, uint64_t tgt, MockMr* mr, uint64_t swap_add, uint64_t compare, uint64_t* old) {
  if (!mr || !mr->cu_ctx) {
    uint64_t* p = (uint64_t*)tgt;
    if (opcode == rn::OP_ATOMIC_FA) {
      *old = __atomic_fetch_add(p, swap_add, __ATOMIC_SEQ_CST);
    } else {
      uint64_t expect = compare;
      __atomic_compare_exchange_n(p, &expect, swap_add, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
      *old = expect;
    }
    return true;
  }
  uint64_t v = 0;
  if (!dma_copy((uint64_t)&v, nullptr, tgt, mr, 8)) return false;
  *old = v;
  const uint64_t nv = opcode == rn::OP_ATOMIC_FA ? v + swap_add : (v == compare ? swap_add : v);
  if (nv == v) return true;
  return dma_copy(tgt, mr, (uint64_t)&nv, nullptr, 8);
}

// ------------------------------------------------------------------ CQE writer
void write_cqe(MockCq* cq, uint8_t opcode, uint8_t wqe_opcode, uint32_t qpn, uint16_t counter, uint32_t bytes, uint32_t imm,
               uint8_t syndrome) {
  const uint32_t depth = 1u << cq->log_n;
  const uint32_t slot = cq->pi.load(std::memory_order_relaxed);
  const uint32_t ci = rn::cq_dbr_index(*(volatile uint32_t*)&cq->dbrec[0]);
  if (((slot - ci) & 0xffffffu) >= depth) {   // the record holds 24 bits of ci: distance mod 2^24
    // CQ overrun: the consumer has not freed the slot.  A ConnectX raises a CQ error; the mock counts it and
    // drops the completion (the consumer's bounded wait then reports the loss) rather than corrupting the ring.
    cq->overruns++;
    return;
  }
  uint8_t* p = cq->buf + ((size_t)(slot & (depth - 1)) << 6);
  rn::Cqe64 c;
  rn::encode_cqe(&c, opcode, (uint8_t)((slot >> cq->log_n) & 1u), counter, qpn, wqe_opcode, bytes, imm, syndrome, 0x5a, now_ns());
  memcpy(p, &c, rn::CQE_OP_OWN_OFF);
  // owner bit last, released: a poller (host, or a GPU reading this page over PCIe) that sees it sees the body
  __atomic_store_n(p + rn::CQE_OP_OWN_OFF, c.op_own, __ATOMIC_RELEASE);
  cq->pi.store(slot + 1, std::memory_order_release);
}

// A receive-consuming request (SEND, SEND_IMM, WRITE_IMM) that passed its own checks waits for the responder to post a
// receive, up to the RNR timeout.  Returns 1 when a receive is there, 0 while the WQE must be retried later, -1 once the
// timeout has passed.
int recv_wait(MockQp* qp, MockQp* peer) {
  const uint16_t rpi = rn::wq_dbr_index(*(volatile uint32_t*)&peer->dbrec[rn::DBR_RCV]);
  if ((uint16_t)(rpi - (uint16_t)peer->hw_rq_cons) != 0) return 1;
  const uint64_t t = now_ns();
  if (!qp->rnr_since_ns) { qp->rnr_since_ns = t; qp->n_rnr++; }
  return t - qp->rnr_since_ns < g_rnr_timeout_ns.load() ? 0 : -1;
}

MockQp* find_qp(uint16_t lid, uint32_t qpn) {
  if (lid < 1 || lid > g_ndev) return nullptr;
  MockDev& d = g_devs[lid - 1];
  return qpn < kMaxQps ? d.qps[qpn] : nullptr;
}

// A WQE's local entries: one, or the two of a gather / scatter list, each checked over its own range in list order.
struct Local { uint64_t a[2]; MockMr* mr[2]; uint32_t len[2]; int n; };
bool local_entries(MockDev* d, const rn::WqeView& v, unsigned need, uint8_t* syn, Local* L) {
  L->n = v.nsge == 2 ? 2 : 1;
  L->len[0] = L->n == 2 ? v.len0 : v.bytes;
  L->len[1] = v.bytes - L->len[0];
  L->mr[0] = L->mr[1] = nullptr;
  L->a[0] = translate(d, v.lkey, v.laddr, L->len[0], need, false, syn, &L->mr[0]);
  if (!L->a[0]) return false;
  if (L->n == 2) L->a[1] = translate(d, v.lkey1, v.laddr1, L->len[1], need, false, syn, &L->mr[1]);
  return L->n == 1 || L->a[1] != 0;
}
// The message is the entries in list order: gather them to [remote, remote + bytes), or scatter that range into them.
bool dma_entries(const Local& L, uint64_t remote, MockMr* rmr, bool scatter) {
  uint64_t off = 0;
  for (int i = 0; i < L.n; off += L.len[i], ++i)
    if (!(scatter ? dma_copy(L.a[i], L.mr[i], remote + off, rmr, L.len[i]) : dma_copy(remote + off, rmr, L.a[i], L.mr[i], L.len[i])))
      return false;
  return true;
}

// ------------------------------------------------------------------ the NIC: execute one WQE of `qp`
// Returns false when it must be retried later (receiver not ready).
bool nic_execute(MockQp* qp, uint64_t w) {
  const uint8_t* slot = qp->sq + ((w & (qp->sq_cnt - 1)) << 6);
  rn::Wqe64 wqe;
  memcpy(&wqe, slot, 64);
  rn::WqeView v;
  uint8_t syn = rn::SYN_OK;
  const bool ok = rn::decode_wqe(&wqe, &v);
  MockQp* peer = find_qp(qp->dlid, qp->dest_qpn);
  MockDev* ldev = qp->ctx->dev;
  bool consumed_rq = false;
  uint16_t rq_index = 0;
  uint32_t moved = 0;
  if (qp->hw_err) {
    syn = rn::SYN_WR_FLUSH_ERR;
  } else if (!ok || v.qpn != qp->v.qp_num || v.wqe_idx != (uint16_t)w) {
    syn = rn::SYN_LOCAL_QP_OP_ERR;
  } else if (v.bytes > rn::MAX_MSG) {            // the max_msg_sz ibv_query_port reports
    syn = rn::SYN_LOCAL_LENGTH_ERR;                // over-long message, before any key or the peer (DESIGN.md 3.1)
  } else if (v.opcode == rn::OP_NOP) {
  } else if (!peer || (peer->v.state != IBV_QPS_RTR && peer->v.state != IBV_QPS_RTS)) {
    syn = rn::SYN_TRANSPORT_RETRY_EXC_ERR;        // nobody answers: what a dead peer looks like on RC
  } else {
    MockDev* rdev = peer->ctx->dev;
    MockMr *lmr = nullptr, *rmr = nullptr;
    switch (v.opcode) {
      case rn::OP_RDMA_WRITE: case rn::OP_RDMA_WRITE_IMM: {
        // Zero length: no key is looked at and nothing moves (DESIGN.md 3.1).  Otherwise the keys are checked before the
        // receive wait, so a WRITE_IMM that fails them never takes a receive.  Inline: the payload is in the WQE (no
        // local key); else it is gathered through the lkeys of its entries.
        uint64_t dst = 0;
        Local L;
        if (v.bytes) {
          const bool lok = v.inl_off || local_entries(ldev, v, 0, &syn, &L);
          dst = lok ? translate(rdev, v.rkey, v.raddr, v.bytes, IBV_ACCESS_REMOTE_WRITE, true, &syn, &rmr) : 0;
        }
        if (syn == rn::SYN_OK && !(peer->access_flags & IBV_ACCESS_REMOTE_WRITE)) syn = rn::SYN_REMOTE_ACCESS_ERR;
        if (syn == rn::SYN_OK && v.opcode == rn::OP_RDMA_WRITE_IMM) {
          const int r = recv_wait(qp, peer);
          if (r == 0) return false;
          if (r < 0) { syn = rn::SYN_RNR_RETRY_EXC_ERR; break; }
        }
        if (syn == rn::SYN_OK && v.bytes &&
            !(v.inl_off ? dma_copy(dst, rmr, (uint64_t)(uintptr_t)((const uint8_t*)&wqe + v.inl_off), nullptr, v.bytes)
                        : dma_entries(L, dst, rmr, false)))
          syn = rn::SYN_LOCAL_PROT_ERR;
        if (syn == rn::SYN_OK) {
          moved = v.bytes;
          if (v.opcode == rn::OP_RDMA_WRITE_IMM) { consumed_rq = true; rq_index = (uint16_t)peer->hw_rq_cons++; }
        }
        break;
      }
      case rn::OP_RDMA_READ: {
        uint64_t src = 0;
        Local L;
        if (v.bytes) {   // zero length: no key is looked at, as for WRITE; the fetched bytes scatter over the entries
          const bool lok = local_entries(ldev, v, IBV_ACCESS_LOCAL_WRITE, &syn, &L);
          src = lok ? translate(rdev, v.rkey, v.raddr, v.bytes, IBV_ACCESS_REMOTE_READ, true, &syn, &rmr) : 0;
        }
        if (syn == rn::SYN_OK && !(peer->access_flags & IBV_ACCESS_REMOTE_READ)) syn = rn::SYN_REMOTE_ACCESS_ERR;
        if (syn == rn::SYN_OK && v.bytes && !dma_entries(L, src, rmr, true)) syn = rn::SYN_LOCAL_PROT_ERR;
        if (syn == rn::SYN_OK) moved = v.bytes;
        break;
      }
      case rn::OP_SEND: case rn::OP_SEND_IMM: {
        // The requester's own check comes first: a SEND whose lkey fails never reaches the responder, so it neither
        // waits for nor consumes a receive.
        Local L;
        if (!v.inl_off && !local_entries(ldev, v, 0, &syn, &L)) break;
        const int r = recv_wait(qp, peer);
        if (r == 0) return false;
        if (r < 0) { syn = rn::SYN_RNR_RETRY_EXC_ERR; break; }
        std::atomic_thread_fence(std::memory_order_acquire);
        const uint8_t* rs = peer->rq + ((peer->hw_rq_cons & (peer->rq_cnt - 1)) << 4);
        rn::Words16 rw;
        memcpy(&rw, rs, 16);
        consumed_rq = true; rq_index = (uint16_t)peer->hw_rq_cons++;
        if (rn::recv_wqe_bytes(rw) < v.bytes) syn = rn::SYN_REMOTE_INVAL_REQ_ERR;
        uint64_t dst = syn == rn::SYN_OK ? translate(rdev, rn::recv_wqe_lkey(rw), rn::recv_wqe_addr(rw), v.bytes, IBV_ACCESS_LOCAL_WRITE,
                                                     true, &syn, &rmr) : 0;
        if (syn == rn::SYN_OK && v.bytes &&
            !(v.inl_off ? dma_copy(dst, rmr, (uint64_t)(uintptr_t)((const uint8_t*)&wqe + v.inl_off), nullptr, v.bytes)
                        : dma_entries(L, dst, rmr, false)))
          syn = rn::SYN_LOCAL_PROT_ERR;
        if (syn == rn::SYN_OK) moved = v.bytes;
        break;
      }
      case rn::OP_ATOMIC_CS: case rn::OP_ATOMIC_FA: {
        if (v.bytes != 8) { syn = rn::SYN_LOCAL_LENGTH_ERR; break; }
        uint64_t dst = translate(ldev, v.lkey, v.laddr, 8, IBV_ACCESS_LOCAL_WRITE, false, &syn, &lmr);
        if (dst && (v.raddr & 7)) { syn = rn::SYN_REMOTE_INVAL_REQ_ERR; break; }
        uint64_t tgt = dst ? translate(rdev, v.rkey, v.raddr, 8, IBV_ACCESS_REMOTE_ATOMIC, true, &syn, &rmr) : 0;
        if (syn == rn::SYN_OK && !(peer->access_flags & IBV_ACCESS_REMOTE_ATOMIC)) syn = rn::SYN_REMOTE_ACCESS_ERR;
        uint64_t old = 0;
        if (syn == rn::SYN_OK && !nic_atomic(v.opcode, tgt, rmr, v.swap_add, v.compare, &old)) syn = rn::SYN_REMOTE_OP_ERR;
        if (syn == rn::SYN_OK && !dma_copy(dst, lmr, (uint64_t)&old, nullptr, 8)) syn = rn::SYN_LOCAL_PROT_ERR;
        if (syn == rn::SYN_OK) moved = 8;
        break;
      }
      default: syn = rn::SYN_LOCAL_QP_OP_ERR;
    }
  }
  qp->rnr_since_ns = 0;
  const bool err = syn != rn::SYN_OK;
  const uint8_t opc = ok ? v.opcode : 0;
  if (consumed_rq && peer && peer->rcq) {
    const uint8_t rop = err ? rn::CQE_RESP_ERR
                            : (opc == rn::OP_SEND ? rn::CQE_RESP_SEND : (opc == rn::OP_SEND_IMM ? rn::CQE_RESP_SEND_IMM : rn::CQE_RESP_WR_IMM));
    write_cqe(peer->rcq, rop, 0, peer->v.qp_num, rq_index, moved, be32(wqe.ctrl.imm), err ? syn : 0);
  }
  if (err || (ok && (v.fm_ce_se & rn::CTRL_CQ_UPDATE)) || qp->sq_sig_all) {
    write_cqe(qp->scq, err ? rn::CQE_REQ_ERR : rn::CQE_REQ, opc, qp->v.qp_num, (uint16_t)w, moved, 0, err ? syn : 0);
    qp->n_cqe++;
  }
  qp->n_wqe++;
  qp->n_bytes += moved;
  if (err) {
    qp->n_err++;
    if (!qp->hw_err) { qp->hw_err = true; qp->v.state = IBV_QPS_ERR; }
  }
  return true;
}

// One sweep over every QP that can send.  Returns true if anything happened.
bool nic_sweep() {
  bool busy = false;
  std::lock_guard<std::recursive_mutex> g(g_mu);
  for (int di = 0; di < g_ndev; ++di) {
    for (uint32_t qi = 0; qi < kMaxQps; ++qi) {
      MockQp* qp = g_devs[di].qps[qi];
      if (!qp || (qp->v.state != IBV_QPS_RTS && qp->v.state != IBV_QPS_ERR && qp->v.state != IBV_QPS_SQD)) continue;
      // A doorbell is a store to either BlueFlame register; its value is the first 8 bytes of a ctrl segment.
      bool rung = false;
      unsigned long long rung_val = 0;
      for (int r = 0; r < 2; ++r) {
        const unsigned long long val = __atomic_load_n((unsigned long long*)(qp->uar + kBfOffset + r * kBfSize), __ATOMIC_ACQUIRE);
        if (val != qp->bf_seen[r]) { qp->bf_seen[r] = val; rung = true; rung_val = val; }
      }
      const uint16_t pi16 = rn::wq_dbr_index(*(volatile uint32_t*)&qp->dbrec[rn::DBR_SND]);
      uint16_t pending = (uint16_t)(pi16 - (uint16_t)qp->hw_sq_cons);
      if (rung) {
        qp->n_doorbells++;
        // The doorbell value is the first 8 bytes of a ctrl segment, i.e. it names a WQE index; the record, read AFTER the
        // register, must already cover that WQE -- otherwise the register store overtook the record store (ordering bug in
        // the poster).  ("Nothing pending" is not the test: an earlier sweep may already have executed this WQE off a
        // record that was ahead of its doorbell, which is legal.)
        const uint16_t bell_idx = rn::doorbell_index(rung_val);
        if ((uint16_t)(pi16 - (uint16_t)(bell_idx + 1)) >= 0x8000u) qp->n_db_no_progress++;
      }
      // Work is only fetched on a doorbell (a real NIC does not look at the record unprompted); a WQE that had
      // to wait for a receive buffer stays pending and is retried without one.
      if (!rung && !(pending && qp->rnr_since_ns)) continue;
      if (pending > qp->sq_cnt) pending = (uint16_t)qp->sq_cnt;
      std::atomic_thread_fence(std::memory_order_acquire);
      while (pending) {
        if (!nic_execute(qp, qp->hw_sq_cons)) break;
        qp->hw_sq_cons++;
        --pending;
        busy = true;
      }
      if (pending && qp->rnr_since_ns) busy = true;
    }
  }
  return busy;
}

void nic_main() {
  uint64_t idle_since = 0;
  while (!g_nic_stop.load(std::memory_order_relaxed)) {
    if (nic_sweep()) { idle_since = 0; continue; }
    const uint64_t t = now_ns();
    if (!idle_since) idle_since = t;
    if (t - idle_since > 2000000ull) { struct timespec ts = {0, 50000}; nanosleep(&ts, nullptr); }
    else sched_yield();
  }
}
void nic_start() {
  bool expect = false;
  if (!g_nic_run.compare_exchange_strong(expect, true)) return;
  g_nic_stop = false;
  g_nic = std::thread(nic_main);
  atexit([] { g_nic_stop = true; if (g_nic.joinable()) g_nic.join(); });
}

// ------------------------------------------------------------------ fast path: ops table
// Publish the WQEs up to `head` (the caller holds post_mu): doorbell record, then the doorbell -- the first 8 bytes of the
// last WQE's ctrl segment into the BlueFlame register, alternating between the two registers as libmlx5 does.
void ring_sq(MockQp* qp, uint64_t head) {
  std::atomic_thread_fence(std::memory_order_release);
  *(volatile uint32_t*)&qp->dbrec[rn::DBR_SND] = rn::wq_dbr_word(head);
  std::atomic_thread_fence(std::memory_order_release);
  unsigned long long db;
  memcpy(&db, qp->sq + (((head - 1) & (qp->sq_cnt - 1)) << 6), 8);
  __atomic_store_n((unsigned long long*)(qp->uar + kBfOffset + qp->bf_off), db, __ATOMIC_RELEASE);
  qp->bf_off ^= kBfSize;
  qp->sq_head = head;
}

int mock_post_send(ibv_qp* q, ibv_send_wr* wr, ibv_send_wr** bad) {
  MockQp* qp = reinterpret_cast<MockQp*>(q);
  std::lock_guard<std::mutex> g(qp->post_mu);
  if (q->state != IBV_QPS_RTS && q->state != IBV_QPS_ERR && q->state != IBV_QPS_SQD) { if (bad) *bad = wr; return EINVAL; }
  uint64_t head = qp->sq_head;
  const uint64_t first = head;
  for (; wr; wr = wr->next) {
    if (head - qp->sq_tail >= qp->sq_cnt) { if (bad) *bad = wr; errno = ENOMEM; break; }
    if (wr->num_sge > (int)qp->max_sge || wr->num_sge < 0) { if (bad) *bad = wr; errno = EINVAL; break; }
    uint8_t opc;
    switch (wr->opcode) {
      case IBV_WR_RDMA_WRITE: opc = rn::OP_RDMA_WRITE; break;
      case IBV_WR_RDMA_WRITE_WITH_IMM: opc = rn::OP_RDMA_WRITE_IMM; break;
      case IBV_WR_SEND: opc = rn::OP_SEND; break;
      case IBV_WR_SEND_WITH_IMM: opc = rn::OP_SEND_IMM; break;
      case IBV_WR_RDMA_READ: opc = rn::OP_RDMA_READ; break;
      case IBV_WR_ATOMIC_CMP_AND_SWP: opc = rn::OP_ATOMIC_CS; break;
      case IBV_WR_ATOMIC_FETCH_AND_ADD: opc = rn::OP_ATOMIC_FA; break;
      default: opc = 0xff;
    }
    if (opc == 0xff) { if (bad) *bad = wr; errno = EOPNOTSUPP; break; }
    const uint8_t fm = (uint8_t)(((wr->send_flags & IBV_SEND_SIGNALED) || qp->sq_sig_all ? rn::CTRL_CQ_UPDATE : 0) |
                                 ((wr->send_flags & IBV_SEND_SOLICITED) ? rn::CTRL_SOLICITED : 0) |
                                 ((wr->send_flags & IBV_SEND_FENCE) ? rn::CTRL_FENCE : 0));
    if (rn::is_atomic(opc) && wr->num_sge != 1) { if (bad) *bad = wr; errno = EINVAL; break; }   // exactly one 8-byte SGE
    rn::Sge sg[rn::MAX_SGE] = {};
    for (int i = 0; i < wr->num_sge; ++i) sg[i] = rn::Sge{wr->sg_list[i].addr, wr->sg_list[i].lkey, wr->sg_list[i].length};
    const int nsg = wr->num_sge;
    const uint64_t laddr = sg[0].addr;
    const uint32_t lkey = sg[0].lkey, len = sg[0].bytes;
    rn::Wqe64 w;
    memset(&w, 0, sizeof w);
    const uint32_t imm = be32(wr->imm_data);       // imm_data is already big-endian; build_* swaps it back onto the wire
    const bool inl = (wr->send_flags & IBV_SEND_INLINE) != 0;
    // Inline: the entries' bytes are concatenated into the WQE now, from their host addresses (libmlx5's set_data_inl_seg);
    // the lkeys are not looked at.
    uint8_t inl_buf[rn::MAX_INLINE];
    uint64_t inl_len = 0;
    bool inl_ok = inl && opc != rn::OP_RDMA_READ && !rn::is_atomic(opc);
    for (int i = 0; inl_ok && i < nsg; ++i) {
      if (inl_len + sg[i].bytes > rn::MAX_INLINE) { inl_ok = false; break; }
      memcpy(inl_buf + inl_len, (const void*)(uintptr_t)sg[i].addr, sg[i].bytes);
      inl_len += sg[i].bytes;
    }
    if (inl && (!inl_ok || inl_len == 0)) {
      if (bad) *bad = wr;
      errno = EINVAL;
      break;
    }
    if (inl)
      rn::build_inline_wqe(&w, opc, (uint16_t)head, q->qp_num, wr->wr.rdma.remote_addr, wr->wr.rdma.rkey,
                           inl_buf, (uint32_t)inl_len, fm, imm);
    else if (opc == rn::OP_SEND || opc == rn::OP_SEND_IMM)   // zero-length entries dropped, as libmlx5 does
      rn::build_send_sg_wqe(&w, opc, (uint16_t)head, q->qp_num, sg, nsg, fm, imm);
    else if (rn::is_atomic(opc))   // libmlx5: FA carries compare_add as the addend, CS carries swap + compare
      rn::build_atomic_wqe(&w, opc, (uint16_t)head, q->qp_num, laddr, lkey, wr->wr.atomic.remote_addr, wr->wr.atomic.rkey,
                           opc == rn::OP_ATOMIC_FA ? wr->wr.atomic.compare_add : wr->wr.atomic.swap, wr->wr.atomic.compare_add, fm, len);
    else
      rn::build_rdma_sg_wqe(&w, opc, (uint16_t)head, q->qp_num, sg, nsg, wr->wr.rdma.remote_addr, wr->wr.rdma.rkey, fm, imm);
    memcpy(qp->sq + ((head & (qp->sq_cnt - 1)) << 6), &w, 64);
    qp->sq_wrid[head & (qp->sq_cnt - 1)] = wr->wr_id;
    ++head;
  }
  int rc = wr ? errno : 0;
  if (head != first) ring_sq(qp, head);
  return rc;
}

int mock_post_recv(ibv_qp* q, ibv_recv_wr* wr, ibv_recv_wr** bad) {
  MockQp* qp = reinterpret_cast<MockQp*>(q);
  std::lock_guard<std::mutex> g(qp->post_mu);
  if (q->state == IBV_QPS_RESET) { if (bad) *bad = wr; return EINVAL; }
  uint64_t head = qp->rq_head;
  int rc = 0;
  for (; wr; wr = wr->next) {
    if (head - qp->rq_tail >= qp->rq_cnt) { if (bad) *bad = wr; rc = ENOMEM; break; }
    if (wr->num_sge != 1) { if (bad) *bad = wr; rc = EINVAL; break; }
    const rn::Words16 r = rn::recv_wqe_words(wr->sg_list[0].addr, wr->sg_list[0].lkey, wr->sg_list[0].length);
    memcpy(qp->rq + ((head & (qp->rq_cnt - 1)) << 4), &r, 16);
    qp->rq_wrid[head & (qp->rq_cnt - 1)] = wr->wr_id;
    ++head;
  }
  if (head != qp->rq_head) {
    std::atomic_thread_fence(std::memory_order_release);
    *(volatile uint32_t*)&qp->dbrec[rn::DBR_RCV] = rn::wq_dbr_word(head);
    qp->rq_head = head;
  }
  return rc;
}

enum ibv_wc_status wc_status_of(uint8_t syn) {
  switch (syn) {
    case rn::SYN_OK: return IBV_WC_SUCCESS;
    case rn::SYN_LOCAL_LENGTH_ERR: return IBV_WC_LOC_LEN_ERR;
    case rn::SYN_LOCAL_QP_OP_ERR: return IBV_WC_LOC_QP_OP_ERR;
    case rn::SYN_LOCAL_PROT_ERR: return IBV_WC_LOC_PROT_ERR;
    case rn::SYN_WR_FLUSH_ERR: return IBV_WC_WR_FLUSH_ERR;
    case rn::SYN_MW_BIND_ERR: return IBV_WC_MW_BIND_ERR;
    case rn::SYN_BAD_RESP_ERR: return IBV_WC_BAD_RESP_ERR;
    case rn::SYN_LOCAL_ACCESS_ERR: return IBV_WC_LOC_ACCESS_ERR;
    case rn::SYN_REMOTE_INVAL_REQ_ERR: return IBV_WC_REM_INV_REQ_ERR;
    case rn::SYN_REMOTE_ACCESS_ERR: return IBV_WC_REM_ACCESS_ERR;
    case rn::SYN_REMOTE_OP_ERR: return IBV_WC_REM_OP_ERR;
    case rn::SYN_TRANSPORT_RETRY_EXC_ERR: return IBV_WC_RETRY_EXC_ERR;
    case rn::SYN_RNR_RETRY_EXC_ERR: return IBV_WC_RNR_RETRY_EXC_ERR;
    case rn::SYN_REMOTE_ABORTED_ERR: return IBV_WC_REM_ABORT_ERR;
    default: return IBV_WC_GENERAL_ERR;
  }
}

int mock_poll_cq(ibv_cq* c, int n, ibv_wc* wc) {
  MockCq* cq = reinterpret_cast<MockCq*>(c);
  MockDev* dev = cq->ctx->dev;
  int got = 0;
  while (got < n) {
    const uint8_t* p = cq->buf + ((size_t)(cq->ci & ((1u << cq->log_n) - 1)) << 6);
    const uint8_t oo = __atomic_load_n(p + rn::CQE_OP_OWN_OFF, __ATOMIC_ACQUIRE);
    if (!rn::cqe_valid(oo, cq->ci, cq->log_n)) break;
    rn::Cqe64 e;
    memcpy(&e, p, 64);
    rn::CqeView v;
    rn::decode_cqe(&e, &v);
    ibv_wc& o = wc[got];
    memset(&o, 0, sizeof o);
    o.status = wc_status_of(v.syndrome);
    o.vendor_err = v.vendor_synd;
    o.byte_len = v.byte_cnt;
    o.qp_num = v.qpn;
    MockQp* qp = v.qpn < kMaxQps ? dev->qps[v.qpn] : nullptr;
    const bool req = v.opcode == rn::CQE_REQ || v.opcode == rn::CQE_REQ_ERR;
    if (qp) {
      std::lock_guard<std::mutex> g(qp->post_mu);
      if (req) {
        o.wr_id = qp->sq_wrid[v.wqe_counter & (qp->sq_cnt - 1)];
        const uint64_t done = rn::expand16(v.wqe_counter + 1u, qp->sq_tail);
        if (done <= qp->sq_head) qp->sq_tail = done;     // unsignaled predecessors are complete too (RC is in order)
      } else {
        o.wr_id = qp->rq_wrid[v.wqe_counter & (qp->rq_cnt - 1)];
        const uint64_t done = rn::expand16(v.wqe_counter + 1u, qp->rq_tail);
        if (done <= qp->rq_head) qp->rq_tail = done;
      }
    }
    if (req) {
      switch (v.wqe_opcode) {
        case rn::OP_RDMA_READ: o.opcode = IBV_WC_RDMA_READ; break;
        case rn::OP_SEND: case rn::OP_SEND_IMM: o.opcode = IBV_WC_SEND; break;
        default: o.opcode = IBV_WC_RDMA_WRITE;
      }
    } else {
      o.opcode = v.opcode == rn::CQE_RESP_WR_IMM ? IBV_WC_RECV_RDMA_WITH_IMM : IBV_WC_RECV;
      if (v.opcode == rn::CQE_RESP_WR_IMM || v.opcode == rn::CQE_RESP_SEND_IMM) { o.wc_flags |= IBV_WC_WITH_IMM; o.imm_data = e.imm_inval_pkey; }
    }
    ++cq->ci;
    ++got;
  }
  if (got) *(volatile uint32_t*)&cq->dbrec[0] = rn::cq_dbr_word(cq->ci);
  // A real NIC needs no CPU; this one is a thread.  A caller that spins on an empty CQ from the core the NIC
  // thread was placed on would starve it for a scheduler tick at a time, so an empty poll gives the core away
  // now and then.
  static thread_local unsigned empties = 0;
  if (got) empties = 0;
  else if ((++empties & 31u) == 0) sched_yield();
  return got;
}

int mock_req_notify_cq(ibv_cq*, int) { return 0; }

}  // namespace

// ====================================================================== exported libibverbs surface
MOCK_API ibv_device** ibv_get_device_list(int* num) {
  init_devices();
  ibv_device** l = (ibv_device**)calloc((size_t)g_ndev + 1, sizeof(ibv_device*));
  if (!l) { errno = ENOMEM; return nullptr; }
  for (int i = 0; i < g_ndev; ++i) l[i] = &g_devs[i].v;
  if (num) *num = g_ndev;
  return l;
}
MOCK_API void ibv_free_device_list(ibv_device** l) { free(l); }
MOCK_API const char* ibv_get_device_name(ibv_device* d) { return d ? d->name : nullptr; }
MOCK_API uint64_t ibv_get_device_guid(ibv_device* d) { return be64(0x0002c90300b20000ull | (uint64_t)reinterpret_cast<MockDev*>(d)->index); }

MOCK_API ibv_context* ibv_open_device(ibv_device* d) {
  init_devices();
  MockDev* dev = reinterpret_cast<MockDev*>(d);
  if (dev < g_devs || dev >= g_devs + g_ndev) { errno = ENODEV; return nullptr; }
  MockCtx* c = new MockCtx();
  memset(&c->v, 0, sizeof c->v);
  c->dev = dev;
  c->v.device = d;
  c->v.ops.poll_cq = mock_poll_cq;
  c->v.ops.req_notify_cq = mock_req_notify_cq;
  c->v.ops.post_send = mock_post_send;
  c->v.ops.post_recv = mock_post_recv;
  c->v.cmd_fd = -1; c->v.async_fd = -1; c->v.num_comp_vectors = 1;
  pthread_mutex_init(&c->v.mutex, nullptr);
  return &c->v;
}
MOCK_API int ibv_close_device(ibv_context* c) {
  delete reinterpret_cast<MockCtx*>(c);
  return 0;
}

// IBVERBS_1.1 compat entry point: fills the leading fields of ibv_port_attr (what verbs_dl.cc reads).
MOCK_API int ibv_query_port(ibv_context* c, uint8_t port, ibv_port_attr* a) {
  if (port != 1) return EINVAL;
  MockDev* dev = reinterpret_cast<MockCtx*>(c)->dev;
  a->state = IBV_PORT_ACTIVE; a->max_mtu = IBV_MTU_4096; a->active_mtu = IBV_MTU_4096; a->gid_tbl_len = 8;
  a->port_cap_flags = 0; a->max_msg_sz = rn::MAX_MSG; a->bad_pkey_cntr = 0; a->qkey_viol_cntr = 0; a->pkey_tbl_len = 1;
  a->lid = dev->lid; a->sm_lid = 1; a->lmc = 0; a->max_vl_num = 4; a->sm_sl = 0; a->subnet_timeout = 18; a->init_type_reply = 0;
  a->active_width = 2 /* 4x */; a->active_speed = 128 /* NDR */; a->phys_state = 5 /* LinkUp */;
  a->link_layer = IBV_LINK_LAYER_INFINIBAND; a->flags = 0;
  return 0;
}
MOCK_API int ibv_query_gid(ibv_context* c, uint8_t port, int index, ibv_gid* gid) {
  if (port != 1 || index < 0 || index >= 8) return EINVAL;
  MockDev* dev = reinterpret_cast<MockCtx*>(c)->dev;
  memset(gid, 0, sizeof *gid);
  gid->raw[0] = 0xfe; gid->raw[1] = 0x80;
  gid->raw[8] = 0x00; gid->raw[9] = 0x02; gid->raw[10] = 0xc9; gid->raw[11] = 0x03; gid->raw[14] = (uint8_t)index; gid->raw[15] = (uint8_t)dev->lid;
  return 0;
}

MOCK_API ibv_pd* ibv_alloc_pd(ibv_context* c) {
  MockPd* p = new MockPd();
  p->v.context = c; p->v.handle = 1;
  return &p->v;
}
MOCK_API int ibv_dealloc_pd(ibv_pd* p) { delete reinterpret_cast<MockPd*>(p); return 0; }

namespace {
MockMr* mr_install(ibv_pd* pd, MockMr* m) {
  std::lock_guard<std::recursive_mutex> g(g_mu);
  MockDev* dev = reinterpret_cast<MockCtx*>(pd->context)->dev;
  uint32_t idx = 1;
  for (; idx < kMaxMkeys; ++idx) if (!dev->mkeys[idx]) break;
  if (idx == kMaxMkeys) { errno = ENOMEM; return nullptr; }
  m->tag = ++dev->mkey_tag[idx];
  m->v.context = pd->context; m->v.pd = pd; m->v.addr = (void*)m->iova; m->v.length = m->len;
  m->v.handle = idx; m->v.lkey = m->v.rkey = (idx << 8) | m->tag;
  m->live = true;
  dev->mkeys[idx] = m;
  return m;
}
}  // namespace

MOCK_API ibv_mr* ibv_reg_mr(ibv_pd* pd, void* addr, size_t len, int access) {
  if (!pd || !addr || !len) { errno = EINVAL; return nullptr; }
  const uint64_t p = (uint64_t)addr;
  MockMr* m = new MockMr();
  m->iova = p; m->len = len; m->map_base = p; m->access = (unsigned)access;
  CUcontext cctx = nullptr;
  const bool fake_gpu = fake_gpu_range(p, len);
  const bool is_dev = fake_gpu || cuda_is_device_ptr(p, &cctx);
  if (is_dev) {
    // get_user_pages() cannot pin this range: ib_core walks its peer-memory clients (amdp2p.c:112-167 is one).
    const char* mode = getenv("ROCNRDMA_MOCK_PEERMEM");
    if (mode && !strcmp(mode, "0")) { delete m; errno = EFAULT; return nullptr; }
    m->cu_ctx = fake_gpu ? nullptr : cctx;
    m->kind = MR_DEVICE;
    if (mode && !strcmp(mode, "b200p2p")) {
      Bridge& b = bridge();
      if (!b.ok) { delete m; errno = ENODEV; return nullptr; }
      std::lock_guard<std::recursive_mutex> g(g_mu);
      // The GPU driver knows the allocation that contains the range (the simulation is told about it here; on
      // hardware nvidia.ko already knows).  Idempotent per allocation.
      uint64_t abase = p & ~65535ull, asize = ((p + len + 65535) & ~65535ull) - abase;
      if (!fake_gpu && cuda().addr_range) {
        CUdeviceptr ab = 0; size_t as = 0;
        if (cuda().addr_range(&ab, &as, (CUdeviceptr)p) == 0) { abase = ab & ~65535ull; asize = (((uint64_t)ab + as + 65535) & ~65535ull) - abase; }
      } else if (fake_gpu) {
        for (auto& r : g_fake_gpu) if (r.live && p >= r.va && p + len <= r.va + r.len) { abase = r.va; asize = r.len; }
      }
      b.gpu_alloc(abase, asize);                      // -ENOMEM/-EINVAL only matter if the pin then fails
      const int hca = reinterpret_cast<MockCtx*>(pd->context)->dev->index;
      long id = b.reg_mr(p, len, hca);               // acquire -> get_page_size -> get_pages -> dma_map, as ib_core orders them
      if (id < 0) { delete m; errno = id == -95 ? EFAULT : (int)-id; return nullptr; }
      m->kind = MR_BRIDGED;
      m->bridge_id = id;
      m->bridge_hca = hca;
      m->pin_va = p & ~65535ull;
      const int n = b.mr_nmap(id);
      for (int i = 0; i < n; ++i) {
        uint64_t a = 0, l = 0;
        if (b.mr_dma(id, i, &a, &l)) break;
        m->sg.emplace_back(a, l);
      }
      if (m->sg.empty()) { b.dereg_mr(id); delete m; errno = EFAULT; return nullptr; }
    }
  }
  if (!mr_install(pd, m)) { if (m->kind == MR_BRIDGED) bridge().dereg_mr(m->bridge_id); delete m; return nullptr; }
  return &m->v;
}
MOCK_API ibv_mr* ibv_reg_mr_iova2(ibv_pd* pd, void* addr, size_t len, uint64_t iova, unsigned access) {
  if ((uint64_t)addr != iova) { errno = EOPNOTSUPP; return nullptr; }
  return ibv_reg_mr(pd, addr, len, (int)access);
}

MOCK_API ibv_mr* ibv_reg_dmabuf_mr(ibv_pd* pd, uint64_t offset, size_t len, uint64_t iova, int fd, int access) {
  if (!pd || !len || fd < 0) { errno = EINVAL; return nullptr; }
  struct stat st;
  if (fstat(fd, &st)) { errno = EBADF; return nullptr; }
  char link[64], target[256] = "";
  snprintf(link, sizeof link, "/proc/self/fd/%d", fd);
  ssize_t tl = readlink(link, target, sizeof target - 1);
  if (tl > 0) target[tl] = 0;
  const off_t size = lseek(fd, 0, SEEK_END);
  if (size >= 0 && (uint64_t)size < offset + len) { errno = EINVAL; return nullptr; }
  MockMr* m = new MockMr();
  m->iova = iova; m->len = len; m->access = (unsigned)access; m->dmabuf_fd = dup(fd);
  void* map = mmap(nullptr, offset + len, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  if (map != MAP_FAILED) {
    // a CPU-mappable exporter (memfd / udmabuf): the NIC reaches the pages through this mapping
    m->kind = MR_DMABUF_MAPPED; m->mapping = map; m->mapping_len = offset + len; m->map_base = (uint64_t)map + offset;
  } else {
    // a device exporter (CUDA's dma-buf of an HBM range): not CPU-mappable; its pages are the ones iova names
    CUcontext cctx = nullptr;
    if (!strstr(target, "dmabuf") || !cuda_is_device_ptr(iova, &cctx)) { if (m->dmabuf_fd >= 0) close(m->dmabuf_fd); delete m; errno = EINVAL; return nullptr; }
    m->kind = MR_DEVICE; m->cu_ctx = cctx; m->map_base = iova;
  }
  if (!mr_install(pd, m)) { if (m->mapping) munmap(m->mapping, m->mapping_len); if (m->dmabuf_fd >= 0) close(m->dmabuf_fd); delete m; return nullptr; }
  return &m->v;
}

MOCK_API int ibv_dereg_mr(ibv_mr* mr) {
  MockMr* m = reinterpret_cast<MockMr*>(mr);
  std::lock_guard<std::recursive_mutex> g(g_mu);
  MockDev* dev = reinterpret_cast<MockCtx*>(mr->context)->dev;
  if (mr->handle >= kMaxMkeys || dev->mkeys[mr->handle] != m) return EINVAL;
  dev->mkeys[mr->handle] = nullptr;
  if (m->kind == MR_BRIDGED) bridge().dereg_mr(m->bridge_id);      // dma_unmap -> put_pages -> release
  if (m->mapping) munmap(m->mapping, m->mapping_len);
  if (m->dmabuf_fd >= 0) close(m->dmabuf_fd);
  delete m;
  return 0;
}

MOCK_API ibv_cq* ibv_create_cq(ibv_context* c, int cqe, void* cq_context, ibv_comp_channel* ch, int) {
  if (cqe < 1 || cqe > (1 << 22)) { errno = EINVAL; return nullptr; }
  std::lock_guard<std::recursive_mutex> g(g_mu);
  MockDev* dev = reinterpret_cast<MockCtx*>(c)->dev;
  uint32_t cqn = 1;
  for (; cqn < kMaxCqs; ++cqn) if (!dev->cqs[cqn]) break;
  if (cqn == kMaxCqs) { errno = ENOMEM; return nullptr; }
  MockCq* q = new MockCq();
  memset(&q->v, 0, sizeof q->v);
  const uint32_t n = roundup_pow2((uint32_t)cqe + 1);   // rdma-core rounds cqe + 1 up to a power of two
  q->log_n = log2u(n); q->cqn = cqn; q->ctx = reinterpret_cast<MockCtx*>(c);
  q->buf = (uint8_t*)page_alloc((size_t)n * 64);
  q->dbrec = (uint32_t*)page_alloc(64);
  if (!q->buf || !q->dbrec) { free(q->buf); free(q->dbrec); delete q; errno = ENOMEM; return nullptr; }
  rn::init_cq_ring(q->buf, n);
  q->v.context = c; q->v.channel = ch; q->v.cq_context = cq_context; q->v.handle = cqn; q->v.cqe = (int)n - 1;
  pthread_mutex_init(&q->v.mutex, nullptr);
  pthread_cond_init(&q->v.cond, nullptr);
  dev->cqs[cqn] = q;
  return &q->v;
}
MOCK_API int ibv_destroy_cq(ibv_cq* c) {
  MockCq* q = reinterpret_cast<MockCq*>(c);
  std::lock_guard<std::recursive_mutex> g(g_mu);
  MockDev* dev = q->ctx->dev;
  for (uint32_t i = 0; i < kMaxQps; ++i)
    if (dev->qps[i] && (dev->qps[i]->scq == q || dev->qps[i]->rcq == q)) return EBUSY;
  dev->cqs[q->cqn] = nullptr;
  free(q->buf); free(q->dbrec);
  delete q;
  return 0;
}

MOCK_API ibv_qp* ibv_create_qp(ibv_pd* pd, ibv_qp_init_attr* a) {
  if (!pd || !a || !a->send_cq || !a->recv_cq) { errno = EINVAL; return nullptr; }
  if (a->qp_type != IBV_QPT_RC) { errno = EOPNOTSUPP; return nullptr; }
  if (a->cap.max_send_wr < 1 || a->cap.max_send_wr > 16384 || a->cap.max_recv_wr > 16384 || a->cap.max_send_sge > rn::MAX_SGE || a->cap.max_recv_sge > 1 ||
      a->cap.max_inline_data > rn::MAX_INLINE) {
    errno = EINVAL;
    return nullptr;
  }
  std::lock_guard<std::recursive_mutex> g(g_mu);
  MockCtx* ctx = reinterpret_cast<MockCtx*>(pd->context);
  MockDev* dev = ctx->dev;
  uint32_t qpn = 0x40 + (uint32_t)dev->index;    // distinct number spaces make a mis-routed WQE visible
  for (; qpn < kMaxQps; ++qpn) if (!dev->qps[qpn]) break;
  if (qpn >= kMaxQps) { errno = ENOMEM; return nullptr; }
  MockQp* q = new MockQp();
  memset(&q->v, 0, sizeof q->v);
  q->ctx = ctx; q->scq = reinterpret_cast<MockCq*>(a->send_cq); q->rcq = reinterpret_cast<MockCq*>(a->recv_cq);
  q->sq_cnt = roundup_pow2(a->cap.max_send_wr);
  q->rq_cnt = roundup_pow2(a->cap.max_recv_wr ? a->cap.max_recv_wr : 1);
  const size_t rq_bytes = ((size_t)q->rq_cnt * 16 + 63) & ~(size_t)63;
  q->buf_len = rq_bytes + (size_t)q->sq_cnt * 64;
  q->buf = (uint8_t*)page_alloc(q->buf_len);
  q->dbrec = (uint32_t*)page_alloc(64);
  q->uar = (uint8_t*)page_alloc(4096);
  if (!q->buf || !q->dbrec || !q->uar) { free(q->buf); free(q->dbrec); free(q->uar); delete q; errno = ENOMEM; return nullptr; }
  q->rq = q->buf; q->sq = q->buf + rq_bytes;
  q->sq_wrid.assign(q->sq_cnt, 0); q->rq_wrid.assign(q->rq_cnt, 0);
  q->sq_sig_all = a->sq_sig_all;
  q->max_sge = a->cap.max_send_sge ? a->cap.max_send_sge : 1;   // what was asked for: ctrl + raddr + two data segments fit one WQEBB
  q->v.context = pd->context; q->v.qp_context = a->qp_context; q->v.pd = pd; q->v.send_cq = a->send_cq; q->v.recv_cq = a->recv_cq;
  q->v.handle = qpn; q->v.qp_num = qpn; q->v.state = IBV_QPS_RESET; q->v.qp_type = IBV_QPT_RC;
  pthread_mutex_init(&q->v.mutex, nullptr);
  pthread_cond_init(&q->v.cond, nullptr);
  a->cap.max_send_wr = q->sq_cnt; a->cap.max_recv_wr = q->rq_cnt; a->cap.max_inline_data = rn::MAX_INLINE;
  a->cap.max_send_sge = q->max_sge; a->cap.max_recv_sge = 1;
  dev->qps[qpn] = q;
  return &q->v;
}
MOCK_API int ibv_destroy_qp(ibv_qp* qq) {
  MockQp* q = reinterpret_cast<MockQp*>(qq);
  std::lock_guard<std::recursive_mutex> g(g_mu);
  q->ctx->dev->qps[q->v.qp_num] = nullptr;
  free(q->buf); free(q->dbrec); free(q->uar);
  delete q;
  return 0;
}

MOCK_API int ibv_modify_qp(ibv_qp* qq, ibv_qp_attr* a, int mask) {
  MockQp* q = reinterpret_cast<MockQp*>(qq);
  if (!(mask & IBV_QP_STATE)) return EINVAL;
  std::lock_guard<std::recursive_mutex> g(g_mu);
  const ibv_qp_state from = qq->state, to = a->qp_state;
  auto need = [&](int m) { return (mask & m) == m; };
  if (to == IBV_QPS_RESET) {
    std::lock_guard<std::mutex> pg(q->post_mu);
    memset(q->buf, 0, q->buf_len);
    q->dbrec[0] = q->dbrec[1] = 0;
    memset(q->uar, 0, 4096);
    q->sq_head = q->sq_tail = q->rq_head = q->rq_tail = 0; q->bf_off = 0;
    q->hw_sq_cons = q->hw_rq_cons = 0; q->bf_seen[0] = q->bf_seen[1] = 0; q->hw_err = false; q->rnr_since_ns = 0;
    q->dest_qpn = 0; q->dlid = 0;
    qq->state = IBV_QPS_RESET;
    return 0;
  }
  if (to == IBV_QPS_ERR) { q->hw_err = true; qq->state = IBV_QPS_ERR; return 0; }
  if (from == IBV_QPS_RESET && to == IBV_QPS_INIT) {
    if (!need(IBV_QP_PKEY_INDEX | IBV_QP_PORT | IBV_QP_ACCESS_FLAGS)) return EINVAL;
    if (a->port_num != 1) return EINVAL;
    q->port = a->port_num; q->access_flags = a->qp_access_flags;
  } else if (from == IBV_QPS_INIT && to == IBV_QPS_INIT) {
    if (mask & IBV_QP_ACCESS_FLAGS) q->access_flags = a->qp_access_flags;
  } else if (from == IBV_QPS_INIT && to == IBV_QPS_RTR) {
    if (!need(IBV_QP_AV | IBV_QP_PATH_MTU | IBV_QP_DEST_QPN | IBV_QP_RQ_PSN | IBV_QP_MAX_DEST_RD_ATOMIC | IBV_QP_MIN_RNR_TIMER)) return EINVAL;
    if (a->path_mtu < IBV_MTU_256 || a->path_mtu > IBV_MTU_4096) return EINVAL;
    uint16_t dlid = a->ah_attr.dlid;
    if (a->ah_attr.is_global && !dlid) dlid = a->ah_attr.grh.dgid.raw[15];     // RoCE-style addressing: the mock GID carries the port id
    if (dlid < 1 || dlid > g_ndev) return ENETUNREACH;
    q->dlid = dlid; q->dest_qpn = a->dest_qp_num;
  } else if (from == IBV_QPS_RTR && to == IBV_QPS_RTS) {
    if (!need(IBV_QP_TIMEOUT | IBV_QP_RETRY_CNT | IBV_QP_RNR_RETRY | IBV_QP_SQ_PSN | IBV_QP_MAX_QP_RD_ATOMIC)) return EINVAL;
    nic_start();
  } else if ((from == IBV_QPS_RTS && (to == IBV_QPS_RTS || to == IBV_QPS_SQD)) || (from == IBV_QPS_SQD && to == IBV_QPS_RTS) ||
             (from == IBV_QPS_SQE && to == IBV_QPS_RTS)) {
  } else {
    return EINVAL;
  }
  qq->state = to;
  return 0;
}

// ====================================================================== libmlx5 surface (exported from here; libmlx5.so.1 forwards)
MOCK_API int mock_mlx5dv_init_obj(mlx5dv_obj* obj, uint64_t type) {
  if (!obj) return EINVAL;
  if (type & MLX5DV_OBJ_QP) {
    MockQp* q = reinterpret_cast<MockQp*>(obj->qp.in);
    mlx5dv_qp* o = obj->qp.out;
    if (!q || !o) return EINVAL;
    o->dbrec = q->dbrec;
    o->sq.buf = q->sq; o->sq.wqe_cnt = q->sq_cnt; o->sq.stride = 64;
    o->rq.buf = q->rq; o->rq.wqe_cnt = q->rq_cnt; o->rq.stride = 16;
    o->bf.reg = q->uar + kBfOffset; o->bf.size = kBfSize;
    o->comp_mask = 0; o->uar_mmap_offset = 0;
    o->tirn = o->tisn = o->rqn = 0; o->sqn = q->v.qp_num; o->tir_icm_addr = 0;
  }
  if (type & MLX5DV_OBJ_CQ) {
    MockCq* c = reinterpret_cast<MockCq*>(obj->cq.in);
    mlx5dv_cq* o = obj->cq.out;
    if (!c || !o) return EINVAL;
    o->buf = c->buf; o->dbrec = c->dbrec; o->cqe_cnt = 1u << c->log_n; o->cqe_size = 64; o->cq_uar = nullptr; o->cqn = c->cqn; o->comp_mask = 0;
  }
  if (type & ~(uint64_t)(MLX5DV_OBJ_QP | MLX5DV_OBJ_CQ)) return EOPNOTSUPP;
  return 0;
}
MOCK_API bool mock_mlx5dv_is_supported(ibv_device* d) {
  init_devices();
  return reinterpret_cast<MockDev*>(d) >= g_devs && reinterpret_cast<MockDev*>(d) < g_devs + g_ndev;
}

// ====================================================================== mock control plane (tests, counters)
MOCK_API int mock_verbs_is_mock() { return 1; }
MOCK_API void mock_set_rnr_timeout_ms(uint64_t ms) { g_rnr_timeout_ns = ms * 1000000ull; }
struct MockQpStats { uint64_t n_wqe, n_cqe, n_err, n_bytes, n_rnr, n_db_no_progress, n_doorbells, hw_sq_cons, sq_cq_overruns; };
MOCK_API int mock_qp_stats(ibv_qp* qq, MockQpStats* o) {
  MockQp* q = reinterpret_cast<MockQp*>(qq);
  std::lock_guard<std::recursive_mutex> g(g_mu);
  o->n_wqe = q->n_wqe; o->n_cqe = q->n_cqe; o->n_err = q->n_err; o->n_bytes = q->n_bytes; o->n_rnr = q->n_rnr;
  o->n_db_no_progress = q->n_db_no_progress; o->n_doorbells = q->n_doorbells; o->hw_sq_cons = q->hw_sq_cons; o->sq_cq_overruns = q->scq->overruns;
  return 0;
}
// Test hook: post a caller-built WQE the way mock_post_send posts the ones it builds -- its 64 bytes as given, with this
// QP's number and the next index written into the ctrl segment.  It hands the NIC WQEs no poster makes (a two-segment
// list with a zero-length segment).
MOCK_API int mock_post_wqe(ibv_qp* q, const uint8_t* wqe64, uint64_t wr_id) {
  MockQp* qp = reinterpret_cast<MockQp*>(q);
  std::lock_guard<std::mutex> g(qp->post_mu);
  if (q->state != IBV_QPS_RTS && q->state != IBV_QPS_ERR && q->state != IBV_QPS_SQD) return EINVAL;   // as mock_post_send
  const uint64_t head = qp->sq_head;
  if (head - qp->sq_tail >= qp->sq_cnt) return ENOMEM;
  rn::Wqe64 w;
  memcpy(&w, wqe64, 64);
  const uint32_t w0 = be32(w.ctrl.opmod_idx_opcode), w1 = be32(w.ctrl.qpn_ds);
  w.ctrl.opmod_idx_opcode = rn::ctrl_word0((uint8_t)w0, (uint16_t)head, (uint8_t)(w0 >> 24));
  w.ctrl.qpn_ds = rn::ctrl_word1(q->qp_num, (uint8_t)(w1 & 0x3f));
  memcpy(qp->sq + ((head & (qp->sq_cnt - 1)) << 6), &w, 64);
  qp->sq_wrid[head & (qp->sq_cnt - 1)] = wr_id;
  ring_sq(qp, head + 1);
  return 0;
}
// CPU-only CI of the peer-memory path: declare a host range to be "GPU memory" (ib_core cannot pin it; a peer
// client must claim it), and "cudaFree" it (the GPU driver revokes every pin on it).
MOCK_API int mock_declare_gpu_range(uint64_t va, uint64_t len) {
  if ((va | len) & 65535ull || !len) return -EINVAL;
  std::lock_guard<std::recursive_mutex> g(g_mu);
  g_fake_gpu.push_back({va, len, true});
  return 0;
}
MOCK_API int mock_gpu_free(uint64_t va) {
  std::lock_guard<std::recursive_mutex> g(g_mu);
  int rc = -ENOENT;
  for (auto& r : g_fake_gpu) if (r.live && r.va == va) { r.live = false; rc = 0; }
  const char* mode = getenv("ROCNRDMA_MOCK_PEERMEM");
  if (mode && !strcmp(mode, "b200p2p") && bridge().ok) {
    int n = bridge().gpu_free(va & ~65535ull);     // nvidia.ko revokes: free callbacks -> invalidate_peer_memory
    if (n >= 0) rc = n;
  }
  return rc;
}
MOCK_API const char* mock_bridge_status() { Bridge& b = bridge(); return b.ok ? "ok" : b.why; }
