// K1 / K2 / K6 (SURVEY.md section 2.3): GPU-initiated RDMA write / read / send driver
// kernels, plus the verification + device-timing helpers.
//
//   rdma_stream_kernel  one CTA per QP; lane 0 posts `iters` work requests with a
//                       bounded window, polls the CQ on the device, stamps
//                       %globaltimer around the whole exchange.  This is the
//                       "ib_write_bw / ib_read_bw, but the poster is an SM" loop.
//   fill / checksum / compare   random payloads and byte-exact verification.
//
// No counterpart in the reference (it has no data path: SURVEY.md section 3.2).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../hca/post.cuh"

using namespace rn;
using namespace rn::dev;

#define RN_API extern "C" __attribute__((visibility("default")))

constexpr int kMaxStreamQps = 64;
struct StreamArgs {
  QpDev* qps[kMaxStreamQps];   // one per CTA, by value: no device allocation on the hot path
  uint32_t opcode;         // OP_RDMA_WRITE / OP_RDMA_READ / OP_SEND
  uint64_t laddr, raddr;   // base addresses (per-CTA stride added)
  uint64_t stride;         // address stride between CTAs' buffers
  uint32_t lkey, rkey;
  uint32_t bytes;          // message size
  uint32_t iters;
  uint32_t window;         // max outstanding WQEs per QP
  uint32_t signal_every;   // 1 = every WQE signaled
  uint32_t burst;          // WQEs per doorbell (1..32)
  uint32_t post_only;      // 1: do not wait for the last completion (the caller reaps it: profilers serialise kernels, so the
                           //    engine / NIC cannot make progress while this kernel is resident)
  uint64_t slot_stride;    // each iteration i uses offset (i % nslots) * slot_stride
  uint32_t nslots;
  uint32_t fence_every;    // 0: no WR fenced; k: WRs k-1, 2k-1, ... of each QP carry CTRL_FENCE
  uint64_t timeout_ns;
  unsigned long long* out; // per CTA: [status, t_start, t_end, done, first_idx, last_idx, 0, 0]
};

// The streaming kernels' windowed burst loop.  One warp per QP: the warp owns the QP and its send CQ for the whole
// kernel, so queue state lives in lane 0's registers (dev::Poster), no atomics, and the CQ is only read when the window
// is full.  Messages of k WQEs each (k = 1, or 2: a WRITE and its signal) go out in bursts of n (perftest's --post_list):
// lane 0 reserves the burst's k * n slots at once, lane j builds WQE j of the burst, lane 0 publishes it with ONE
// doorbell and, when the window (counted in messages) is full, polls the CQ for the oldest burst.  With burst = 1 this is
// the plain post-one / poll-one loop (5-6 dependent L2 round trips per message, ~3.7 us measured); bursts amortise the
// reservation, the fences, the doorbell and -- with signal_every (perftest's --cq-mod) -- the completion polling over up
// to 32 WQEs.  A message's last WQE is signaled when the message is (every signal_every-th message, and the last one);
// its other WQEs never are.
//   build(uint8_t* slot, uint16_t wqe_idx, uint32_t qpn, uint32_t i, uint32_t part, uint8_t fm_ce_se): builds WQE `part` of
//   message i with an mlx5_wire.h builder and stores it to its SQ slot (store_wqe)
//   out: [status, t_start, t_end, messages done, first_idx, last_idx, cons, 0]
template <typename Build>
__device__ __forceinline__ void stream_post(QpDev* qp, uint32_t k, uint32_t iters, uint32_t window, uint32_t burst,
                                            uint32_t signal_every, bool post_only, unsigned long long timeout_ns,
                                            unsigned long long* out, Build build) {
  const uint32_t lane = threadIdx.x;
  int status = WAIT_OK;
  unsigned long long first = ~0ull, last = 0;
  uint32_t done = 0;                                  // messages
  Poster p = poster_open(qp);
  if (qp->state == QPS_ERR) status = WAIT_QP_ERROR;
  const unsigned long long t0 = globaltimer_ns();
  while (done < iters && status != WAIT_QP_ERROR) {
    const uint32_t n = min(burst, iters - done);
    // this lane's WQE of the burst, worked out before the window wait so that it stays off the path from a completion
    // to the next doorbell
    const uint32_t i = done + lane / k, part = lane % k;
    const bool sig = part == k - 1 && ((signal_every <= 1) || ((i + 1) % signal_every == 0) || (i + 1 == iters));
    unsigned long long idx = 0;
    int rc = WAIT_OK;
    if (lane == 0) {
      // leaves <= window - n messages outstanding: the last WQE of message done + n - window - 1 has completed
      if (window && done + n > window) rc = poster_wait(p, last + (unsigned long long)k * n - (unsigned long long)k * window, timeout_ns);
      if (rc != WAIT_TIMEOUT) {
        idx = poster_reserve(p, k * n, timeout_ns);
        if (idx == ~0ull) rc = WAIT_TIMEOUT;
      }
    }
    rc = __shfl_sync(0xffffffffu, rc, 0);
    idx = __shfl_sync(0xffffffffu, idx, 0);
    if (rc != WAIT_OK) status = rc;
    if (rc == WAIT_TIMEOUT) break;
    if (first == ~0ull) first = idx;
    if (lane < k * n) build(poster_slot(p, idx + lane), (uint16_t)(idx + lane), p.qpn, i, part, sig ? CTRL_CQ_UPDATE : 0);
    if (k * n > 1) __syncwarp();                     // the burst's WQE bytes happen-before lane 0's release
    if (lane == 0) {
      // overlap the completion poll with the doorbell release: the CQE load is in flight while the fence in
      // front of the doorbell waits for the WQE stores (one exposed round trip per post instead of two)
      const bool outstanding = p.head > p.cons;
      uint4 tail = make_uint4(0, 0, 0, 0);
      if (outstanding) tail = poster_peek(p);
      poster_ring(p, idx + k * n);
      if (outstanding && poster_take(p, tail) < 0) status = WAIT_CQE_ERROR;
    }
    last = idx + k * n - 1;
    done += n;
  }
  if (lane != 0) return;
  if (done && !post_only) {
    const int rc = poster_wait(p, last, timeout_ns);
    if (rc != WAIT_OK) status = rc;
  }
  const unsigned long long t1 = globaltimer_ns();
  poster_close(p);
  out[0] = (unsigned long long)(long long)status;
  out[1] = t0; out[2] = t1; out[3] = done; out[4] = first; out[5] = last;
  out[6] = p.cons;
  out[7] = 0;
}

__global__ void __launch_bounds__(32, 1) rdma_stream_kernel(StreamArgs a) {
  const uint64_t lbase = a.laddr + blockIdx.x * a.stride, rbase = a.raddr + blockIdx.x * a.stride;
  stream_post(a.qps[blockIdx.x], 1, a.iters, a.window, a.burst, a.signal_every, a.post_only, a.timeout_ns,
              a.out + (size_t)blockIdx.x * 8,
              [&](uint8_t* slot, uint16_t idx, uint32_t qpn, uint32_t i, uint32_t, uint8_t flags) {
                const uint64_t off = (uint64_t)(i % a.nslots) * a.slot_stride;
                if (a.fence_every && (i + 1) % a.fence_every == 0) flags |= CTRL_FENCE;
                Wqe64 w;
                if (a.opcode == OP_SEND) {
                  build_send_wqe(&w, OP_SEND, idx, qpn, lbase + off, a.lkey, a.bytes, flags, 0);
                  store_wqe(slot, w);
                } else {
                  build_rdma_wqe(&w, (uint8_t)a.opcode, idx, qpn, lbase + off, a.lkey, rbase + off, a.rkey, a.bytes, flags, 0);
                  store_wqe(slot, w);
                }
              });
}

// Posting parameters that can always make progress (pure host function, unit-tested on the CPU):
// burst in 1..32 and at most half the window; the window wait targets a WQE `window - burst` behind the
// newest one, so a signaled WQE must already sit at or after it: signal_every <= window - burst + 1.
RN_API void rn_stream_clamp(uint32_t window, uint32_t* burst, uint32_t* signal_every) {
  uint32_t b = *burst ? (*burst > 32 ? 32 : *burst) : 1, s = *signal_every ? *signal_every : 1;
  if (window) {
    if (b > (window + 1) / 2) b = (window + 1) / 2;
    if (s > window - b + 1) s = window - b + 1;
  }
  *burst = b; *signal_every = s;
}

RN_API int rn_k_rdma_stream(uint64_t stream, const uint64_t* qps_host, uint32_t nqp, uint32_t opcode, uint64_t laddr,
                            uint32_t lkey, uint64_t raddr, uint32_t rkey, uint64_t stride, uint32_t bytes,
                            uint32_t iters, uint32_t window, uint32_t signal_every, uint32_t burst, uint64_t slot_stride,
                            uint32_t nslots, uint64_t timeout_ms, uint64_t out_dev, uint32_t fence_every) {
  StreamArgs a;
  if (!copy_qps(a.qps, qps_host, nqp)) return -22;
  a.post_only = (opcode >> 31) & 1u; opcode &= 0x7fffffffu;
  a.opcode = opcode; a.laddr = laddr; a.raddr = raddr; a.stride = stride;
  a.lkey = lkey; a.rkey = rkey; a.bytes = bytes; a.iters = iters; a.window = window;
  rn_stream_clamp(window, &burst, &signal_every);
  a.signal_every = signal_every; a.burst = burst;
  a.slot_stride = slot_stride; a.nslots = nslots ? nslots : 1;
  a.fence_every = fence_every;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  rdma_stream_kernel<<<nqp, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- a WRITE and a dependent READ
// One thread, `iters` times: an RDMA WRITE of `bytes` from laddr to raddr, then an RDMA READ of those bytes back from raddr
// into back, and wait for the READ's completion.  How the READ is kept behind the WRITE:
//   mode 0  the READ is fenced; both WQEs go out under ONE doorbell (exclusive poster)
//   mode 1  the WRITE is signaled and its CQE awaited before the READ is posted (what ordering costs without the fence)
//   mode 2  dev::rdma_write, then dev::rdma_read(..., fence = true) through the shared submit, then sq_wait
// out: [status, t_start, t_end, pairs done, sum of pair ns, min pair ns, 0, 0]
__global__ void __launch_bounds__(32, 1) write_read_kernel(QpDev* qp, uint64_t laddr, uint32_t lkey, uint64_t raddr, uint32_t rkey,
                                                           uint64_t back, uint32_t back_lkey, uint32_t bytes, uint32_t iters,
                                                           uint32_t mode, unsigned long long timeout_ns, unsigned long long* out) {
  if (threadIdx.x != 0) return;
  int status = qp->state == QPS_ERR ? WAIT_QP_ERROR : WAIT_OK;
  unsigned long long sum = 0, mn = ~0ull;
  uint32_t done = 0;
  const unsigned long long t0 = globaltimer_ns();
  if (mode == 2) {
    for (; done < iters && status == WAIT_OK; ++done) {
      const unsigned long long ts = globaltimer_ns();
      const unsigned long long i0 = rdma_write(qp, laddr, lkey, raddr, rkey, bytes, false);
      const unsigned long long i1 = i0 == ~0ull ? ~0ull : rdma_read(qp, back, back_lkey, raddr, rkey, bytes, true, true);
      if (i1 == ~0ull) { status = WAIT_TIMEOUT; break; }
      status = sq_wait(qp, i1, timeout_ns);
      const unsigned long long dt = globaltimer_ns() - ts;
      sum += dt; mn = dt < mn ? dt : mn;
    }
  } else {
    Poster p = poster_open(qp);
    for (; done < iters && status == WAIT_OK; ++done) {
      const unsigned long long ts = globaltimer_ns();
      Wqe64 w;
      unsigned long long idx = poster_reserve(p, 2, timeout_ns);
      if (idx == ~0ull) { status = WAIT_TIMEOUT; break; }
      build_rdma_wqe(&w, OP_RDMA_WRITE, (uint16_t)idx, p.qpn, laddr, lkey, raddr, rkey, bytes, mode == 0 ? 0 : CTRL_CQ_UPDATE, 0);
      store_wqe(poster_slot(p, idx), w);
      if (mode == 1) {
        poster_ring(p, idx + 1);
        if ((status = poster_wait(p, idx, timeout_ns)) != WAIT_OK) break;
      }
      build_rdma_wqe(&w, OP_RDMA_READ, (uint16_t)(idx + 1), p.qpn, back, back_lkey, raddr, rkey, bytes,
                     mode == 0 ? (CTRL_CQ_UPDATE | CTRL_FENCE) : CTRL_CQ_UPDATE, 0);
      store_wqe(poster_slot(p, idx + 1), w);
      poster_ring(p, idx + 2);
      if ((status = poster_wait(p, idx + 1, timeout_ns)) != WAIT_OK) break;
      const unsigned long long dt = globaltimer_ns() - ts;
      sum += dt; mn = dt < mn ? dt : mn;
    }
    poster_close(p);
  }
  out[0] = (unsigned long long)(long long)status;
  out[1] = t0; out[2] = globaltimer_ns(); out[3] = done; out[4] = sum; out[5] = mn;
}
RN_API int rn_k_write_read(uint64_t stream, uint64_t qp_dev, uint64_t laddr, uint32_t lkey, uint64_t raddr, uint32_t rkey,
                           uint64_t back, uint32_t back_lkey, uint32_t bytes, uint32_t iters, uint32_t mode, uint64_t timeout_ms,
                           uint64_t out_dev) {
  if (mode > 2) return -22;
  write_read_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((QpDev*)qp_dev, laddr, lkey, raddr, rkey, back, back_lkey, bytes, iters, mode,
                                                        timeout_ns(timeout_ms), (unsigned long long*)out_dev);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- shared-SQ stress (SURVEY.md section 5: "many CTAs, one SQ")
// Every CTA posts `per_cta` small RDMA writes to ONE QP through the shared (non-blocking) submit, each to
// its own 64-byte cell; the last CTA posts the flush and waits.  Exercises slot reservation, the ready-flag
// doorbell hand-off and in-order retirement under maximum contention.
__global__ void __launch_bounds__(32) shared_post_stress_kernel(QpDev* qp, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                                                uint32_t rkey, uint32_t per_cta, unsigned int* done_ctas,
                                                                unsigned long long* out, unsigned long long timeout_ns) {
  if (threadIdx.x != 0) return;
  const unsigned long long t0 = globaltimer_ns();
  int status = WAIT_OK;
  for (uint32_t i = 0; i < per_cta; ++i) {
    const uint64_t cell = ((uint64_t)blockIdx.x * per_cta + i) * 64;
    const unsigned long long idx = post_one(qp, [&](Wqe64* w, unsigned long long j) {
      build_rdma_wqe(w, OP_RDMA_WRITE, (uint16_t)j, qp->qpn, laddr + cell, lkey, raddr + cell, rkey, 64,
                     ((j & 7) == 7) ? CTRL_CQ_UPDATE : 0, 0);
    }, timeout_ns);
    if (idx == ~0ull) { status = WAIT_TIMEOUT; break; }
  }
  if (status != WAIT_OK) out[0] = (unsigned long long)(long long)status;
  fence_gpu();
  if (atomicAdd(done_ctas, 1u) + 1 == gridDim.x) {
    const int rc = post_flush(qp, false, timeout_ns);
    if (rc != WAIT_OK) out[0] = (unsigned long long)(long long)rc;
    out[1] = t0; out[2] = globaltimer_ns(); out[3] = (unsigned long long)gridDim.x * per_cta;
    *done_ctas = 0;
  }
}
RN_API int rn_k_shared_post_stress(uint64_t stream, uint64_t qp_dev, int ctas, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                   uint32_t rkey, uint32_t per_cta, uint64_t counter_dev, uint64_t out_dev, uint64_t timeout_ms) {
  unsigned long long* o = clear_record(out_dev);
  shared_post_stress_kernel<<<ctas, 32, 0, (cudaStream_t)stream>>>((QpDev*)qp_dev, laddr, lkey, raddr, rkey, per_cta,
                                                                   (unsigned int*)counter_dev, o, timeout_ns(timeout_ms));
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- receive-side consumer
// Waits on the QP's receive CQ for `n` arrivals (SEND or RDMA_WRITE_IMM), stamps each by its immediate.
// out: [status, t_start, t_end, seen, bytes_total, 0,0,0] ; stamps[imm] = %globaltimer at observation.
// With prepost_bytes != ~0 the kernel first posts its own `n` receive WQEs from the device (dev::post_recv):
// buffer i is [prepost_addr + i * prepost_bytes, +prepost_bytes).
__global__ void __launch_bounds__(32, 1) recv_consume_kernel(QpDev* qp, uint32_t n, uint32_t max_imm, unsigned long long* stamps,
                                                             unsigned long long* out, unsigned long long timeout_ns,
                                                             uint64_t prepost_addr, uint32_t prepost_lkey, uint32_t prepost_bytes) {
  if (threadIdx.x != 0) return;
  const unsigned long long t0 = globaltimer_ns();
  if (prepost_bytes != ~0u)
    for (uint32_t i = 0; i < n; ++i) post_recv(qp, prepost_addr + (uint64_t)i * prepost_bytes, prepost_lkey, prepost_bytes);
  unsigned long long bytes = 0;
  uint32_t seen = 0;
  int status = WAIT_OK;
  while (seen < n) {
    uint32_t imm = 0;
    long long got = recv_wait(qp, &imm, timeout_ns);
    if (got < 0) { status = (int)got; break; }
    // release: whoever acquires the stamp (a GEMM waiting for this panel: gemm_mxfp8.cu) also sees the panel the completion announced
    if (stamps && imm < max_imm) asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(stamps + imm), "l"(globaltimer_ns()) : "memory");
    bytes += (unsigned long long)got;
    ++seen;
  }
  out[0] = (unsigned long long)(long long)status;
  out[1] = t0; out[2] = globaltimer_ns(); out[3] = seen; out[4] = bytes;
}
RN_API int rn_k_recv_consume(uint64_t stream, uint64_t qp_dev, uint32_t n, uint32_t max_imm, uint64_t stamps_dev,
                             uint64_t out_dev, uint64_t timeout_ms, uint64_t prepost_addr, uint32_t prepost_lkey,
                             uint32_t prepost_bytes) {
  recv_consume_kernel<<<1, 32, 0, (cudaStream_t)stream>>>((QpDev*)qp_dev, n, max_imm, (unsigned long long*)stamps_dev,
                                                          (unsigned long long*)out_dev, timeout_ns(timeout_ms),
                                                          prepost_addr, prepost_lkey, prepost_bytes);
  return (int)cudaGetLastError();
}

// The consumer of a mesh: up to kMaxRecvQps receive QPs, one per source, that share one receive CQ.  The kernel first
// posts prepost[i] zero-length receive WQEs on qps[i] (RDMA_WRITE_IMM ignores the buffer), then takes `n` completions
// from the shared CQ and stamps each by its immediate, as recv_consume_kernel does.  recv_wait ignores the QP number of
// a receive completion and the engine claims the CQ's producer index atomically, so completions of every QP arrive on
// the one CQ in the order the engine claimed them.  out: as recv_consume_kernel's.
constexpr int kMaxRecvQps = 7;
struct RecvQpsArgs {
  QpDev* qps[kMaxRecvQps];
  uint32_t prepost[kMaxRecvQps];
  uint32_t nqp, n, max_imm;
  uint64_t prepost_addr;
  uint32_t prepost_lkey;
  unsigned long long* stamps;
  unsigned long long* out;
  unsigned long long timeout_ns;
};

__global__ void __launch_bounds__(32, 1) recv_consume_qps_kernel(RecvQpsArgs a) {
  if (threadIdx.x != 0) return;
  const unsigned long long t0 = globaltimer_ns();
  for (uint32_t q = 0; q < a.nqp; ++q)
    for (uint32_t i = 0; i < a.prepost[q]; ++i) post_recv(a.qps[q], a.prepost_addr, a.prepost_lkey, 0);
  unsigned long long bytes = 0;
  uint32_t seen = 0;
  int status = WAIT_OK;
  while (seen < a.n) {
    uint32_t imm = 0;
    long long got = recv_wait(a.qps[0], &imm, a.timeout_ns);
    if (got < 0) { status = (int)got; break; }
    if (a.stamps && imm < a.max_imm)
      asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(a.stamps + imm), "l"(globaltimer_ns()) : "memory");
    bytes += (unsigned long long)got;
    ++seen;
  }
  a.out[0] = (unsigned long long)(long long)status;
  a.out[1] = t0; a.out[2] = globaltimer_ns(); a.out[3] = seen; a.out[4] = bytes;
}
// qps_host / prepost_host: nqp (1..7) queue pairs and the receive WQEs to post on each.  The caller guarantees that
// they share one receive CQ.
RN_API int rn_k_recv_consume_qps(uint64_t stream, const uint64_t* qps_host, const uint32_t* prepost_host, uint32_t nqp,
                                 uint32_t n, uint32_t max_imm, uint64_t stamps_dev, uint64_t out_dev, uint64_t timeout_ms,
                                 uint64_t prepost_addr, uint32_t prepost_lkey) {
  RecvQpsArgs a;
  if (!copy_qps(a.qps, qps_host, nqp)) return -22;
  for (uint32_t i = 0; i < nqp; ++i) a.prepost[i] = prepost_host[i];
  a.nqp = nqp; a.n = n; a.max_imm = max_imm;
  a.prepost_addr = prepost_addr; a.prepost_lkey = prepost_lkey;
  a.stamps = (unsigned long long*)stamps_dev;
  a.out = clear_record(out_dev);
  a.timeout_ns = timeout_ns(timeout_ms);
  recv_consume_qps_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- remote atomics (device-posted)
// One warp per QP, posting CS / FA work requests with the exclusive Poster exactly like rdma_stream_kernel: bursts
// share one reservation and one doorbell, the window bounds the outstanding WQEs.  Op i of CTA c targets the word at
// target + c * target_stride and has its fetched (original) value written to fetch + (c * iters + i) * 8, so every
// value an atomic returned can be checked afterwards (exactly-once under contention, in-order execution of a chain).
struct AtomicArgs {
  QpDev* qps[kMaxStreamQps];
  uint32_t opcode;           // OP_ATOMIC_FA / OP_ATOMIC_CS
  uint32_t chain;            // CS only: op i is CS(compare = i, swap = i + 1)
  uint64_t target, target_stride, fetch;
  uint32_t rkey, lkey;
  uint64_t add, compare, swap;
  uint32_t iters, window, signal_every, burst;
  uint64_t timeout_ns;
  unsigned long long* out;   // per CTA: [status, t_start, t_end, done, first_idx, last_idx, cons, 0]
};

__global__ void __launch_bounds__(32, 1) atomic_stream_kernel(AtomicArgs a) {
  const uint64_t tgt = a.target + blockIdx.x * a.target_stride;
  const uint64_t fbase = a.fetch + (uint64_t)blockIdx.x * a.iters * 8;
  stream_post(a.qps[blockIdx.x], 1, a.iters, a.window, a.burst, a.signal_every, false, a.timeout_ns,
              a.out + (size_t)blockIdx.x * 8,
              [&](uint8_t* slot, uint16_t idx, uint32_t qpn, uint32_t i, uint32_t, uint8_t flags) {
                const uint64_t cmp = a.chain ? (uint64_t)i : a.compare, swp = a.chain ? (uint64_t)i + 1 : a.swap;
                Wqe64 w;
                build_atomic_wqe(&w, (uint8_t)a.opcode, idx, qpn, fbase + (uint64_t)i * 8, a.lkey, tgt, a.rkey,
                                 a.opcode == OP_ATOMIC_FA ? a.add : swp, cmp, flags);
                store_wqe(slot, w);
              });
}

RN_API int rn_k_atomic_stream(uint64_t stream, const uint64_t* qps_host, uint32_t nqp, uint32_t opcode, uint32_t chain,
                              uint64_t target, uint32_t rkey, uint64_t target_stride, uint64_t fetch, uint32_t lkey,
                              uint64_t add, uint64_t compare, uint64_t swap, uint32_t iters, uint32_t window,
                              uint32_t signal_every, uint32_t burst, uint64_t timeout_ms, uint64_t out_dev) {
  AtomicArgs a;
  if (!copy_qps(a.qps, qps_host, nqp)) return -22;
  if (opcode != OP_ATOMIC_FA && opcode != OP_ATOMIC_CS) return -22;
  a.opcode = opcode; a.chain = chain && opcode == OP_ATOMIC_CS;
  a.target = target; a.target_stride = target_stride; a.fetch = fetch; a.rkey = rkey; a.lkey = lkey;
  a.add = add; a.compare = compare; a.swap = swap;
  a.iters = iters; a.window = window;
  rn_stream_clamp(window, &burst, &signal_every);
  a.signal_every = signal_every; a.burst = burst;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  atomic_stream_kernel<<<nqp, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- put-with-signal
// Each message is an RDMA WRITE of `nbytes` (unsignaled) followed by a fetch-and-add of `add` on the remote signal
// word (signaled), built by lanes 0 and 1 and published with ONE doorbell.  The engine executes the atomic only once
// the WRITE before it on the QP has landed, so a receiver that sees the signal reach k may read messages 0..k-1.
// Message i writes slot (i % nslots) * slot_stride; its fetched value goes to fetch + (i % fetch_slots) * 8.
struct PutSignalArgs {
  QpDev* qp;
  uint64_t src, dst;
  uint32_t lkey, rkey, nbytes, nslots;
  uint64_t slot_stride;
  uint64_t sig;
  uint32_t sig_rkey, fetch_lkey;
  uint64_t fetch;
  uint32_t fetch_slots, iters, window, pad;
  uint64_t add;
  uint64_t timeout_ns;
  unsigned long long* out;   // [status, t_start, t_end, done, first_idx, last_idx, cons, 0]
};

__global__ void __launch_bounds__(32, 1) put_signal_kernel(PutSignalArgs a) {
  stream_post(a.qp, 2, a.iters, a.window, 1, 1, false, a.timeout_ns, a.out,
              [&](uint8_t* slot, uint16_t idx, uint32_t qpn, uint32_t i, uint32_t part, uint8_t flags) {
                Wqe64 w;
                if (part == 0) {
                  const uint64_t off = (uint64_t)(i % a.nslots) * a.slot_stride;
                  build_rdma_wqe(&w, OP_RDMA_WRITE, idx, qpn, a.src + off, a.lkey, a.dst + off, a.rkey, a.nbytes, flags, 0);
                  store_wqe(slot, w);
                } else {
                  build_atomic_wqe(&w, OP_ATOMIC_FA, idx, qpn, a.fetch + (uint64_t)(i % a.fetch_slots) * 8, a.fetch_lkey, a.sig,
                                   a.sig_rkey, a.add, 0, flags);
                  store_wqe(slot, w);
                }
              });
}

RN_API int rn_k_put_signal(uint64_t stream, uint64_t qp_dev, uint64_t src, uint32_t lkey, uint64_t dst, uint32_t rkey,
                           uint32_t nbytes, uint64_t slot_stride, uint32_t nslots, uint64_t sig, uint32_t sig_rkey,
                           uint64_t fetch, uint32_t fetch_lkey, uint32_t fetch_slots, uint64_t add, uint32_t iters,
                           uint32_t window, uint64_t timeout_ms, uint64_t out_dev) {
  PutSignalArgs a;
  a.qp = (QpDev*)qp_dev;
  a.src = src; a.dst = dst; a.lkey = lkey; a.rkey = rkey; a.nbytes = nbytes;
  a.nslots = nslots ? nslots : 1; a.slot_stride = slot_stride;
  a.sig = sig; a.sig_rkey = sig_rkey; a.fetch = fetch; a.fetch_lkey = fetch_lkey; a.fetch_slots = fetch_slots ? fetch_slots : 1;
  a.iters = iters; a.window = window; a.pad = 0; a.add = add;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  put_signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- inline puts (DOCA p / p_signal, nvshmem_p)
// One warp per QP, windowed and bursted like rdma_stream_kernel.  Message i of CTA c (m = c * iters + i) is an inline
// RDMA WRITE of nbytes (1..MAX_INLINE) read into registers from row m % rows of `values` -- plain device memory, never
// registered -- to dst + (m % nslots) * slot_stride.  With a signal word (sig != 0) each message is that WRITE plus a
// FETCH_AND_ADD of `add` on sig + c * 8, built by two lanes (window and burst then count messages, 2 WQEs each); the
// engine executes the atomic only after the WRITE has landed, so ops.signal_wait works unchanged on the receiver.
struct PutInlineArgs {
  QpDev* qps[kMaxStreamQps];
  const uint8_t* values;
  uint64_t row_bytes;
  uint32_t rows, nbytes;
  uint64_t dst, slot_stride;
  uint32_t rkey, nslots;
  uint64_t sig, fetch, add;           // sig == 0: plain inline puts
  uint32_t sig_rkey, fetch_lkey, fetch_slots;
  uint32_t iters, window, signal_every, burst;
  uint64_t timeout_ns;
  unsigned long long* out;            // per CTA: [status, t_start, t_end, done, first_idx, last_idx, cons, 0]
};

__global__ void __launch_bounds__(32, 1) put_inline_kernel(PutInlineArgs a) {
  const uint64_t sig = a.sig + (uint64_t)blockIdx.x * 8;
  const uint32_t m0 = blockIdx.x * a.iters;
  stream_post(a.qps[blockIdx.x], a.sig ? 2u : 1u, a.iters, a.window, a.burst, a.signal_every, false, a.timeout_ns,
              a.out + (size_t)blockIdx.x * 8,
              [&](uint8_t* slot, uint16_t idx, uint32_t qpn, uint32_t i, uint32_t part, uint8_t flags) {
                const uint32_t m = m0 + i;
                Wqe64 w;
                if (part == 1) {
                  build_atomic_wqe(&w, OP_ATOMIC_FA, idx, qpn, a.fetch + (uint64_t)(m % a.fetch_slots) * 8, a.fetch_lkey, sig,
                                   a.sig_rkey, a.add, 0, flags);
                  store_wqe(slot, w);
                } else {
                  const InlinePayload d = inline_load(a.values + (uint64_t)(m % a.rows) * a.row_bytes, a.nbytes);
                  build_inline_wqe(&w, OP_RDMA_WRITE, idx, qpn, a.dst + (uint64_t)(m % a.nslots) * a.slot_stride, a.rkey, d,
                                   a.nbytes, flags, 0);
                  store_wqe(slot, w);
                }
              });
}

RN_API int rn_k_put_inline(uint64_t stream, const uint64_t* qps_host, uint32_t nqp, uint64_t values, uint64_t row_bytes,
                           uint32_t rows, uint64_t dst, uint32_t rkey, uint32_t nbytes, uint64_t slot_stride, uint32_t nslots,
                           uint64_t sig, uint32_t sig_rkey, uint64_t fetch, uint32_t fetch_lkey, uint32_t fetch_slots,
                           uint64_t add, uint32_t iters, uint32_t window, uint32_t signal_every, uint32_t burst,
                           uint64_t timeout_ms, uint64_t out_dev) {
  PutInlineArgs a;
  if (!copy_qps(a.qps, qps_host, nqp)) return -22;
  if (nbytes == 0 || nbytes > MAX_INLINE || rows == 0 || (uint64_t)nqp * iters > 0xffffffffull) return -22;
  a.values = (const uint8_t*)values; a.row_bytes = row_bytes; a.rows = rows; a.nbytes = nbytes;
  a.dst = dst; a.slot_stride = slot_stride; a.rkey = rkey; a.nslots = nslots ? nslots : 1;
  a.sig = sig; a.fetch = fetch; a.add = add;
  a.sig_rkey = sig_rkey; a.fetch_lkey = fetch_lkey; a.fetch_slots = fetch_slots ? fetch_slots : 1;
  a.iters = iters; a.window = window;
  if (sig && burst > 16) burst = 16;                  // two WQEs per message, one lane each
  rn_stream_clamp(window, &burst, &signal_every);
  a.signal_every = signal_every; a.burst = burst;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  put_inline_kernel<<<nqp, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- two-entry gathers and scatters
// One warp per QP.  Message i of CTA c uses slot offset off = (i % nslots) * slot_stride and is cut at `split` bytes:
// entry 0 is the first `split` bytes at laddr + c * stride + off, entry 1 the other bytes - split at
// laddr1 + c * stride + off (the same slot of a second MR), and the remote side is [raddr + c * stride + off, + bytes).
// WRITE and SEND gather the two entries into it (a SEND into the responder's next receive), READ scatters it into them.
//   via 0: the windowed, bursted exclusive Poster of rdma_stream_kernel (stream_post)
//   via 1: lane 0 posts each message with dev::rdma_write_sg / rdma_read_sg / rdma_send_sg (shared submit) and keeps at
//          most `window` messages in flight with sq_wait
struct GatherArgs {
  QpDev* qps[kMaxStreamQps];
  uint32_t opcode;
  uint64_t laddr, laddr1, raddr, stride, slot_stride;
  uint32_t lkey, lkey1, rkey;
  uint32_t bytes, split, nslots;
  uint32_t iters, window, signal_every, burst, via;
  uint64_t timeout_ns;
  unsigned long long* out;            // per CTA: [status, t_start, t_end, done, first_idx, last_idx, cons, 0]
};

__global__ void __launch_bounds__(32, 1) gather_stream_kernel(GatherArgs a) {
  const uint64_t cta = (uint64_t)blockIdx.x * a.stride;
  const uint64_t l0 = a.laddr + cta, l1 = a.laddr1 + cta, r = a.raddr + cta;
  const uint8_t opc = (uint8_t)a.opcode;
  auto entries = [&](uint32_t i, Sge (&sg)[MAX_SGE]) -> uint64_t {
    const uint64_t off = (uint64_t)(i % a.nslots) * a.slot_stride;
    sg[0] = Sge{l0 + off, a.lkey, a.split};
    sg[1] = Sge{l1 + off, a.lkey1, a.bytes - a.split};
    return r + off;
  };
  QpDev* qp = a.qps[blockIdx.x];
  unsigned long long* out = a.out + (size_t)blockIdx.x * 8;
  if (a.via == 0) {
    stream_post(qp, 1, a.iters, a.window, a.burst, a.signal_every, false, a.timeout_ns, out,
                [&](uint8_t* slot, uint16_t idx, uint32_t qpn, uint32_t i, uint32_t, uint8_t flags) {
                  Sge sg[MAX_SGE];
                  const uint64_t raddr = entries(i, sg);
                  Wqe64 w;
                  if (opc == OP_SEND) build_send_sg_wqe(&w, OP_SEND, idx, qpn, sg, MAX_SGE, flags, 0);
                  else build_rdma_sg_wqe(&w, opc, idx, qpn, sg, MAX_SGE, raddr, a.rkey, flags, 0);
                  store_wqe(slot, w);
                });
    return;
  }
  if (threadIdx.x != 0) return;
  int status = qp->state == QPS_ERR ? WAIT_QP_ERROR : WAIT_OK;
  unsigned long long first = ~0ull, last = 0;
  uint32_t done = 0;
  const unsigned long long t0 = globaltimer_ns();
  for (; done < a.iters && status == WAIT_OK; ++done) {
    const uint32_t i = done;
    const bool sig = a.signal_every <= 1 || (i + 1) % a.signal_every == 0 || i + 1 == a.iters;
    // at most `window` messages in flight: message i - window has completed (a signaled WQE lies within the window)
    if (a.window && i >= a.window && (status = sq_wait(qp, first + i - a.window, a.timeout_ns)) != WAIT_OK) break;
    Sge sg[MAX_SGE];
    const uint64_t raddr = entries(i, sg);
    const unsigned long long idx = opc == OP_SEND ? rdma_send_sg(qp, sg, sig)
                                   : opc == OP_RDMA_READ ? rdma_read_sg(qp, sg, raddr, a.rkey, sig)
                                                         : rdma_write_sg(qp, sg, raddr, a.rkey, sig);
    if (idx == ~0ull) { status = WAIT_TIMEOUT; break; }
    if (first == ~0ull) first = idx;
    last = idx;
  }
  if (done && status == WAIT_OK) status = sq_wait(qp, last, a.timeout_ns);
  out[0] = (unsigned long long)(long long)status;
  out[1] = t0; out[2] = globaltimer_ns(); out[3] = done; out[4] = first; out[5] = last;
  out[6] = ld_u64_volatile(&qp->sq_cons);
  out[7] = 0;
}

RN_API int rn_k_gather_stream(uint64_t stream, const uint64_t* qps_host, uint32_t nqp, uint32_t opcode, uint64_t laddr,
                              uint32_t lkey, uint64_t laddr1, uint32_t lkey1, uint64_t raddr, uint32_t rkey, uint64_t stride,
                              uint32_t bytes, uint32_t split, uint64_t slot_stride, uint32_t nslots, uint32_t iters,
                              uint32_t window, uint32_t signal_every, uint32_t burst, uint32_t via, uint64_t timeout_ms,
                              uint64_t out_dev) {
  GatherArgs a;
  if (!copy_qps(a.qps, qps_host, nqp) || split > bytes || via > 1) return -22;
  if (opcode != OP_RDMA_WRITE && opcode != OP_RDMA_READ && opcode != OP_SEND) return -22;
  a.opcode = opcode; a.laddr = laddr; a.laddr1 = laddr1; a.raddr = raddr; a.stride = stride; a.slot_stride = slot_stride;
  a.lkey = lkey; a.lkey1 = lkey1; a.rkey = rkey; a.bytes = bytes; a.split = split; a.nslots = nslots ? nslots : 1;
  a.iters = iters; a.window = window; a.via = via;
  rn_stream_clamp(window, &burst, &signal_every);
  a.signal_every = signal_every; a.burst = burst;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  gather_stream_kernel<<<nqp, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- pulled records with arrival words
// One warp owns the QP and its send CQ (dev::Poster) and pulls n fixed-size records: record r is one RDMA READ of
// rec_bytes from raddr + j * src_stride (j = indices[r], or r) into laddr + r * rec_bytes.  Record r is WQE base + r.
// Word r of `ready` gets %globaltimer (st.release.gpu) once record r has landed, the same arrival word recv_consume writes
// for pushed records, so unpack_fp8(ready=) and gemm_mxfp8(a_ready=) consume pulls and pushes alike.  RC completes in
// order: a requester CQE covers its own WQE and every earlier one, a failed one only the earlier ones.  So one CQE stamps
// up to signal_every records, all with one value, and after a failure nothing more is stamped.  The loop is stream_post's
// (window, bursts, peek before the doorbell), but every completion is taken one at a time and stamped as it is taken,
// the final drain included, so a record is stamped by the first CQ poll that sees its completion.
struct ReadRecordsArgs {
  QpDev* qp;
  uint64_t laddr, raddr;             // dst_mr.addr + dst_off, src_mr.addr + src_off
  uint64_t src_stride;
  const int32_t* indices;            // nullptr: record r reads source record r
  unsigned long long* ready;         // nullptr: no arrival words
  uint32_t lkey, rkey, rec_bytes, n;
  uint32_t window, burst, signal_every;
  uint64_t timeout_ns;
  unsigned long long* out;           // [status, t_start, t_end, records landed, first_idx, last_idx, cons, 0]
};

// Take the CQE whose tail poster_peek loaded, if it is ready and ours, and stamp the records it completes.  1 / 0 / WAIT_CQE_ERROR.
__device__ __forceinline__ int read_records_take(Poster& p, const uint4 tail, unsigned long long base, uint32_t& landed,
                                                 unsigned long long* ready) {
  const int rc = poster_take(p, tail);   // its __threadfence is the acquire of everything the CQE announces
  if (rc == 0) return 0;
  const unsigned long long upto = p.cons - (rc < 0 ? 1 : 0);   // a failed WQE has not landed
  if (upto > base + landed) {
    const unsigned long long now = globaltimer_ns();
    for (; base + landed < upto; ++landed)
      if (ready) asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(ready + landed), "l"(now) : "memory");
  }
  return rc;
}
// Take completions one at a time until every WQE below `until` has completed.  WAIT_OK / WAIT_CQE_ERROR / WAIT_TIMEOUT.
__device__ __forceinline__ int read_records_reap(Poster& p, unsigned long long base, uint32_t& landed, unsigned long long* ready,
                                                 unsigned long long until, unsigned long long timeout_ns) {
  unsigned long long t0 = 0;
  for (unsigned it = 0; p.cons < until; ++it) {
    const int rc = read_records_take(p, poster_peek(p), base, landed, ready);
    if (rc < 0) return rc;
    if (rc == 0) {
      if (t0 == 0) t0 = globaltimer_ns();
      else if ((it & 15) == 0 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
    }
  }
  return WAIT_OK;
}

__global__ void __launch_bounds__(32, 1) read_records_kernel(ReadRecordsArgs a) {
  const uint32_t lane = threadIdx.x;
  int status = WAIT_OK;
  uint32_t posted = 0, landed = 0;
  Poster p = poster_open(a.qp);
  const unsigned long long base = p.head, depth = (unsigned long long)p.sq_mask + 1;
  if (a.qp->state == QPS_ERR) status = WAIT_QP_ERROR;
  const unsigned long long t0 = globaltimer_ns();
  while (posted < a.n && status == WAIT_OK) {
    const uint32_t m = min(a.burst, a.n - posted), r = posted + lane;
    // this lane's record, worked out before the window wait so that it stays off the path from a completion to the doorbell
    uint64_t src = 0;
    bool sig = false;
    if (lane < m) {
      src = a.raddr + (uint64_t)(uint32_t)(a.indices ? __ldg(a.indices + r) : (int32_t)r) * a.src_stride;
      sig = a.signal_every <= 1 || (r + 1) % a.signal_every == 0 || r + 1 == a.n;
    }
    int rc = WAIT_OK;
    if (lane == 0) {
      // at most window - m records outstanding, and room for m WQEs, before the burst is built: taken here, with stamps,
      // so that poster_reserve never has to consume a completion itself
      unsigned long long until = p.head + m > depth ? p.head + m - depth : 0;
      if (a.window && posted + m > a.window && base + posted + m - a.window > until) until = base + posted + m - a.window;
      rc = read_records_reap(p, base, landed, a.ready, until, a.timeout_ns);
      if (rc == WAIT_OK && poster_reserve(p, m, a.timeout_ns) == ~0ull) rc = WAIT_TIMEOUT;
    }
    rc = __shfl_sync(0xffffffffu, rc, 0);
    if (rc != WAIT_OK) { status = rc; break; }
    if (lane < m) {
      Wqe64 w;
      build_rdma_wqe(&w, OP_RDMA_READ, (uint16_t)(base + r), p.qpn, a.laddr + (uint64_t)r * a.rec_bytes, a.lkey, src, a.rkey,
                     a.rec_bytes, sig ? CTRL_CQ_UPDATE : 0, 0);
      store_wqe(poster_slot(p, base + r), w);
    }
    if (m > 1) __syncwarp();                          // the burst's WQE bytes happen-before lane 0's release
    if (lane == 0) {
      const bool outstanding = p.head > p.cons;
      uint4 tail = make_uint4(0, 0, 0, 0);
      if (outstanding) tail = poster_peek(p);        // in flight while the doorbell's release waits for the WQE stores
      poster_ring(p, base + posted + m);
      if (outstanding && read_records_take(p, tail, base, landed, a.ready) < 0) status = WAIT_CQE_ERROR;
    }
    status = __shfl_sync(0xffffffffu, status, 0);
    posted += m;
  }
  if (lane != 0) return;
  if (status == WAIT_OK && posted) status = read_records_reap(p, base, landed, a.ready, base + posted, a.timeout_ns);
  // after a failure the QP is in ERR and every later WQE completes flushed: take those completions (nothing is stamped)
  // so that the queue state published below is whole
  if (status == WAIT_CQE_ERROR && p.head > p.cons) poster_wait(p, p.head - 1, a.timeout_ns);
  const unsigned long long t1 = globaltimer_ns();
  poster_close(p);
  a.out[0] = (unsigned long long)(long long)status;
  a.out[1] = t0; a.out[2] = t1; a.out[3] = landed;
  a.out[4] = posted ? base : ~0ull; a.out[5] = posted ? base + posted - 1 : 0;
  a.out[6] = p.cons;
  a.out[7] = 0;
}

RN_API int rn_k_read_records(uint64_t stream, uint64_t qp_dev, uint64_t laddr, uint32_t lkey, uint64_t raddr, uint32_t rkey,
                             uint64_t src_stride, uint32_t rec_bytes, uint32_t n, uint64_t indices_dev, uint64_t ready_dev,
                             uint32_t window, uint32_t burst, uint32_t signal_every, uint64_t timeout_ms, uint64_t out_dev) {
  if (rec_bytes == 0) return -22;
  ReadRecordsArgs a;
  a.qp = (QpDev*)qp_dev;
  a.laddr = laddr; a.raddr = raddr; a.src_stride = src_stride;
  a.indices = (const int32_t*)indices_dev; a.ready = (unsigned long long*)ready_dev;
  a.lkey = lkey; a.rkey = rkey; a.rec_bytes = rec_bytes; a.n = n;
  rn_stream_clamp(window, &burst, &signal_every);
  a.window = window; a.burst = burst; a.signal_every = signal_every;
  a.timeout_ns = timeout_ns(timeout_ms);
  a.out = (unsigned long long*)out_dev;
  read_records_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- signal wait (receiver side)
// Runs on the GPU that holds the signal word.  Thread 0 polls it with system-scope acquire loads until it reaches
// `until`; every value 1..until is stamped (%globaltimer) when first seen.  Each wait for the next arrival is bounded
// by timeout_ns.  With check_bytes != 0, as soon as the signal covers message k the whole CTA compares slot k of
// check_dst with check_src (slot k at k * check_stride, check_bytes long) and counts mismatching 16-byte words.
// out: [status, t_start, t_end, last value seen, mismatches, 0, 0, 0]
constexpr int kSignalWaitThreads = 1024;
__global__ void __launch_bounds__(kSignalWaitThreads, 1) signal_wait_kernel(const unsigned long long* signal, uint64_t until,
                                                                            unsigned long long* stamps, unsigned long long* out,
                                                                            unsigned long long timeout_ns, const uint8_t* check_dst,
                                                                            const uint8_t* check_src, uint64_t check_bytes,
                                                                            uint64_t check_stride) {
  __shared__ unsigned long long s_seen, s_bad;
  __shared__ int s_status;
  unsigned long long seen = 0, bad = 0;
  const unsigned long long t0 = globaltimer_ns();
  if (threadIdx.x == 0) { s_seen = 0; s_bad = 0; s_status = WAIT_OK; }
  __syncthreads();
  while (seen < until) {
    if (threadIdx.x == 0) {
      unsigned long long v = ld_u64_acquire(signal), tw = globaltimer_ns();
      while (v <= seen) {
        const unsigned long long now = globaltimer_ns();
        if (now - tw > timeout_ns) { s_status = WAIT_TIMEOUT; break; }
        __nanosleep(64);
        v = ld_u64_acquire(signal);
      }
      if (v > seen) {
        const unsigned long long now = globaltimer_ns();
        if (stamps)
          for (unsigned long long k = seen; k < v && k < until; ++k) stamps[k] = now;
        s_seen = v;
      }
    }
    __syncthreads();   // thread 0's acquire, then the barrier: every thread's loads below see the messages it covers
    const unsigned long long v = s_seen;
    const int st = s_status;
    if (check_bytes) {
      const unsigned long long hi = v < until ? v : until;
      for (unsigned long long k = seen; k < hi; ++k) {
        const uint8_t* d = check_dst + k * check_stride;
        const uint8_t* s = check_src + k * check_stride;
        for (uint64_t o = (uint64_t)threadIdx.x * 16; o + 16 <= check_bytes; o += (uint64_t)kSignalWaitThreads * 16) {
          const uint4 x = ld_v4_volatile(d + o), y = ld_v4_volatile(s + o);
          if (x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w) ++bad;
        }
      }
    }
    seen = v;
    __syncthreads();
    if (st != WAIT_OK) break;
  }
  for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(&s_bad, bad);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = (unsigned long long)(long long)s_status;
    out[1] = t0; out[2] = globaltimer_ns(); out[3] = s_seen; out[4] = s_bad;
  }
}

RN_API int rn_k_signal_wait(uint64_t stream, uint64_t signal, uint64_t until, uint64_t stamps_dev, uint64_t out_dev,
                            uint64_t timeout_ms, uint64_t check_dst, uint64_t check_src, uint64_t check_bytes,
                            uint64_t check_stride) {
  if (check_bytes & 15) return -22;
  unsigned long long* o = clear_record(out_dev);
  signal_wait_kernel<<<1, kSignalWaitThreads, 0, (cudaStream_t)stream>>>(
      (const unsigned long long*)signal, until, (unsigned long long*)stamps_dev, o, timeout_ns(timeout_ms),
      (const uint8_t*)check_dst, (const uint8_t*)check_src, check_bytes, check_stride);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- CQ watch (receiver-side payload check)
// Watches a send CQ without consuming it (the poster that owns the CQ keeps reaping it; the ring must hold all n CQEs, so
// no slot is reused while this runs).  Thread 0 waits for CQE k (k = 0 .. n-1) with a relaxed load of its owner byte and
// a system-scope fence (acquire); then the whole CTA compares, at once, the message the CQE names (wqe_counter c: bytes
// at (c % nslots) * stride of dst and src).  Of each `piece` bytes of a message only the last `tail` are compared --
// what a chunk of `piece` bytes stores last -- so the check keeps up with a full-rate stream.  Each wait is bounded by
// timeout_ns.  out: [status, t_start, t_end, CQEs seen, mismatching 16-byte words, error CQEs, 0, 0]
constexpr int kCqWatchThreads = 1024;
__global__ void __launch_bounds__(kCqWatchThreads, 1) cq_watch_kernel(const CqDev* cq, uint32_t n, const uint8_t* dst,
                                                                      const uint8_t* src, uint64_t stride, uint32_t nslots,
                                                                      uint64_t msg_bytes, uint64_t piece, uint64_t tail,
                                                                      unsigned long long timeout_ns, unsigned long long* out) {
  __shared__ unsigned long long s_bad;
  __shared__ uint32_t s_counter, s_errs;
  __shared__ int s_status;
  const unsigned long long t0 = globaltimer_ns();
  const uint8_t* buf = cq->buf;
  const uint32_t log_n = cq->log_n;
  unsigned long long bad = 0;
  if (threadIdx.x == 0) { s_bad = 0; s_errs = 0; s_status = WAIT_OK; }
  __syncthreads();
  uint32_t k = 0;
  for (; k < n; ++k) {
    if (threadIdx.x == 0) {
      const uint8_t* cqe = buf + ((size_t)(k & ((1u << log_n) - 1)) << 6);
      const unsigned long long tw = globaltimer_ns();
      uint4 t = ld_v4_volatile(cqe + CQE_TAIL_OFF);
      while (!cqe_valid(cqe_tail_op_own(t), k, log_n)) {
        if (globaltimer_ns() - tw > timeout_ns) { s_status = WAIT_TIMEOUT; break; }
        t = ld_v4_volatile(cqe + CQE_TAIL_OFF);
      }
      fence_sys();   // acquire: the payload the CQE announces
      s_counter = cqe_tail_counter(t);
      if (cqe_tail_opcode(t) == CQE_REQ_ERR) ++s_errs;
    }
    __syncthreads();   // thread 0's acquire, then the barrier: every thread's loads below see the message
    if (s_status != WAIT_OK) break;
    const uint64_t base = (uint64_t)(s_counter % nslots) * stride;
    for (uint64_t p = 0; p < msg_bytes; p += piece) {
      const uint64_t end = p + piece < msg_bytes ? p + piece : msg_bytes;
      const uint64_t beg = end - (end - p < tail ? end - p : tail);
      for (uint64_t o = beg + (uint64_t)threadIdx.x * 16; o + 16 <= end; o += (uint64_t)kCqWatchThreads * 16) {
        const uint4 x = ld_v4_volatile(dst + base + o), y = ld_v4_volatile(src + base + o);
        if (x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w) ++bad;
      }
    }
    __syncthreads();   // s_counter is rewritten next round
  }
  for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(&s_bad, bad);
  __syncthreads();
  if (threadIdx.x == 0) {
    out[0] = (unsigned long long)(long long)s_status;
    out[1] = t0; out[2] = globaltimer_ns(); out[3] = k; out[4] = s_bad; out[5] = s_errs;
  }
}

RN_API int rn_k_cq_watch(uint64_t stream, uint64_t cq_dev, uint32_t n, uint64_t dst, uint64_t src, uint64_t stride,
                         uint32_t nslots, uint64_t msg_bytes, uint64_t piece, uint64_t tail, uint64_t timeout_ms,
                         uint64_t out_dev) {
  if (!nslots || !piece || !tail || ((dst | src | stride | piece | tail) & 15)) return -22;
  unsigned long long* o = clear_record(out_dev);
  cq_watch_kernel<<<1, kCqWatchThreads, 0, (cudaStream_t)stream>>>(
      (const CqDev*)cq_dev, n, (const uint8_t*)dst, (const uint8_t*)src, stride, nslots, msg_bytes, piece, tail,
      timeout_ns(timeout_ms), o);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------- K6: verification
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

__global__ void fill_random_kernel(uint64_t* p, size_t n64, uint8_t* tail, uint32_t ntail, uint64_t seed) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n64; i += step) p[i] = splitmix64(seed + i);
  if (blockIdx.x == 0 && threadIdx.x < ntail) tail[threadIdx.x] = (uint8_t)splitmix64(seed + n64 + threadIdx.x);
}

// bf16 payload with a controlled dynamic range (for the fp8 pack tests/bench)
__global__ void fill_bf16_kernel(uint16_t* p, size_t n, uint64_t seed, float scale) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += step) {
    uint64_t r = splitmix64(seed + i);
    // roughly normal via sum of 4 uniforms, times a per-32-block scale spread
    float u = ((r & 0xffff) + ((r >> 16) & 0xffff) + ((r >> 32) & 0xffff) + ((r >> 48) & 0xffff)) * (1.0f / 65536.0f) - 2.0f;
    float blk = 1.0f + (float)(splitmix64(seed ^ (i >> 5)) & 7);
    float v = u * scale * blk;
    uint32_t b = __float_as_uint(v);
    b += 0x7fffu + ((b >> 16) & 1u);
    p[i] = (uint16_t)(b >> 16);
  }
}

__global__ void checksum_kernel(const uint64_t* p, size_t n64, const uint8_t* tail, uint32_t ntail,
                                unsigned long long* out) {
  unsigned long long acc = 0;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n64; i += step) acc += splitmix64(p[i] ^ i);
  if (blockIdx.x == 0 && threadIdx.x < ntail) acc += splitmix64((uint64_t)tail[threadIdx.x] ^ (n64 + threadIdx.x));
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

__global__ void compare_kernel(const uint8_t* a, const uint8_t* b, size_t n, unsigned long long* out) {
  unsigned long long bad = 0;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  if ((((uintptr_t)a | (uintptr_t)b) & 15) == 0) {
    const uint4 *a4 = (const uint4*)a, *b4 = (const uint4*)b;
    size_t n4 = n / 16;
    for (size_t k = i; k < n4; k += step) {
      uint4 x = a4[k], y = b4[k];
      if (x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w) ++bad;
    }
    for (size_t k = n4 * 16 + i; k < n; k += step) bad += a[k] != b[k];
  } else {
    for (size_t k = i; k < n; k += step) bad += a[k] != b[k];
  }
  for (int o = 16; o; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(out, bad);
}

RN_API int rn_k_fill_random(uint64_t stream, uint64_t ptr, uint64_t bytes, uint64_t seed) {
  size_t n64 = bytes / 8;
  uint32_t ntail = (uint32_t)(bytes % 8);
  int grid = (int)((n64 + 255) / 256);
  if (grid > device_sms() * 16) grid = device_sms() * 16;
  if (grid < 1) grid = 1;
  fill_random_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint64_t*)ptr, n64, (uint8_t*)ptr + n64 * 8, ntail, seed);
  return (int)cudaGetLastError();
}
RN_API int rn_k_fill_bf16(uint64_t stream, uint64_t ptr, uint64_t n, uint64_t seed, float scale) {
  int grid = (int)((n + 255) / 256);
  if (grid > device_sms() * 16) grid = device_sms() * 16;
  if (grid < 1) grid = 1;
  fill_bf16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint16_t*)ptr, n, seed, scale);
  return (int)cudaGetLastError();
}
RN_API int rn_k_checksum(uint64_t stream, uint64_t ptr, uint64_t bytes, uint64_t out_dev) {
  size_t n64 = bytes / 8;
  uint32_t ntail = (uint32_t)(bytes % 8);
  int grid = (int)((n64 + 255) / 256);
  if (grid > device_sms() * 8) grid = device_sms() * 8;
  if (grid < 1) grid = 1;
  cudaMemsetAsync((void*)out_dev, 0, 8, (cudaStream_t)stream);
  checksum_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint64_t*)ptr, n64, (const uint8_t*)ptr + n64 * 8, ntail,
                                                          (unsigned long long*)out_dev);
  return (int)cudaGetLastError();
}
RN_API int rn_k_compare(uint64_t stream, uint64_t a, uint64_t b, uint64_t bytes, uint64_t out_dev) {
  int grid = (int)((bytes / 16 + 255) / 256);
  if (grid > device_sms() * 8) grid = device_sms() * 8;
  if (grid < 1) grid = 1;
  cudaMemsetAsync((void*)out_dev, 0, 8, (cudaStream_t)stream);
  compare_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)a, (const uint8_t*)b, bytes,
                                                         (unsigned long long*)out_dev);
  return (int)cudaGetLastError();
}

// L2 flush between timed iterations: stream a buffer larger than the L2 (50 MB on H100).
__global__ void l2_flush_kernel(uint4* p, size_t n4, uint32_t v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (; i < n4; i += step) p[i] = make_uint4(v, v, v, v);
}
RN_API int rn_k_l2_flush(uint64_t stream, uint64_t ptr, uint64_t bytes, uint32_t v) {
  l2_flush_kernel<<<device_sms() * 8, 256, 0, (cudaStream_t)stream>>>((uint4*)ptr, bytes / 16, v);
  return (int)cudaGetLastError();
}

extern "C" __attribute__((visibility("default"))) void rn_preload_rdma_ops() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, rdma_stream_kernel);
  cudaFuncGetAttributes(&a, recv_consume_kernel);
  cudaFuncGetAttributes(&a, recv_consume_qps_kernel);
  cudaFuncGetAttributes(&a, shared_post_stress_kernel);
  cudaFuncGetAttributes(&a, write_read_kernel);
  cudaFuncGetAttributes(&a, atomic_stream_kernel);
  cudaFuncGetAttributes(&a, put_signal_kernel);
  cudaFuncGetAttributes(&a, put_inline_kernel);
  cudaFuncGetAttributes(&a, gather_stream_kernel);
  cudaFuncGetAttributes(&a, read_records_kernel);
  cudaFuncGetAttributes(&a, signal_wait_kernel);
  cudaFuncGetAttributes(&a, cq_watch_kernel);
  cudaFuncGetAttributes(&a, fill_random_kernel);
  cudaFuncGetAttributes(&a, fill_bf16_kernel);
  cudaFuncGetAttributes(&a, checksum_kernel);
  cudaFuncGetAttributes(&a, compare_kernel);
  cudaFuncGetAttributes(&a, l2_flush_kernel);
}
