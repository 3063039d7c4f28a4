// GPU-initiated posting: reserve an SQ slot, write the 64-byte WQE, publish the
// doorbell record, ring the doorbell, poll the completion queue -- all from an
// GPU thread, no host in the loop (SURVEY.md N3, kernels K1/K2).
//
// Ordering contract (what a ConnectX requires, and what the softhca engine checks
// and counts violations of in QpDev::n_db_order_violations):
//     WQE bytes, doorbell record  --release (gpu scope on a device-local QP, sys otherwise)-->
//     doorbell register
// Multi-poster scheme: resv_head hands out indices, ready_head serialises the
// doorbell so the register never runs ahead of a WQE that is still being written
// (three-counter scheme: resv_head / ready_head / sq_cons).
//
// The reference leaves posting to host ibv_post_send (README.md:67); this file is
// the part of the new build that has no counterpart there.
#pragma once
#include <cuda_runtime.h>
#include "hca_types.h"

namespace rn {
namespace dev {

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void st_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_v4_volatile(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_u64_volatile(const void* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_u64_acquire(const void* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_u64_release(void* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_u32_volatile(const void* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_u32_volatile(void* p, uint32_t v) {
  asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
// System scope only when something on the path lives outside this GPU (host-resident
// rings, a peer GPU, a real NIC); a device-local QP pays the much cheaper gpu scope.
__device__ __forceinline__ void fence_scope(bool sys) { if (sys) fence_sys(); else fence_gpu(); }
__device__ __forceinline__ void st_u64_relaxed(void* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
enum TraceSlot : int { TR_POST = 0, TR_CLAIM = 1, TR_PARSED = 2, TR_COPIED = 3, TR_CQE = 4, TR_SEEN = 5 };
__device__ __forceinline__ void trace_stamp(QpDev* qp, unsigned long long idx, int which) {
  if (qp->trace_on) qp->trace[((idx & ((1ull << qp->sq_log) - 1)) << 3) + which] = globaltimer_ns();
}

// -------------------------------------------------------------- slot reservation
// Returns the 64-bit index of the first of `n` consecutive WQEs, or ~0ull if the
// queue stayed full past `timeout_ns` (the CQ is polled while waiting so that a
// poster that never calls wait() still makes progress).
__device__ int cq_poll_once(QpDev* qp);

__device__ __forceinline__ unsigned long long sq_reserve(QpDev* qp, uint32_t n,
                                                         unsigned long long timeout_ns = 2000000000ull) {
  if (qp->state == QPS_ERR) return ~0ull;          // like ibv_post_send on an errored QP: refuse, reserve nothing
  unsigned long long idx = atomicAdd(&qp->resv_head, (unsigned long long)n);
  const unsigned long long depth = 1ull << qp->sq_log;
  if (idx + n - ld_u64_volatile(&qp->sq_cons) <= depth) return idx;
  unsigned long long t0 = globaltimer_ns();
  while (idx + n - ld_u64_volatile(&qp->sq_cons) > depth) {
    cq_poll_once(qp);
    if (globaltimer_ns() - t0 > timeout_ns) {
      // The indices [idx, idx+n) are handed out and can never be filled (their ring slots still hold
      // unfinished WQEs), so the ready-run scan of the shared submit would stall behind this hole
      // forever.  Fail the QP instead: every later reserve returns at once, the host sees ERR and
      // resets the QP (which rewinds resv_head and clears the flags).
      qp->state = QPS_ERR;
      __threadfence();
      return ~0ull;
    }
  }
  return idx;
}

// -------------------------------------------------------------- WQE store
__device__ __forceinline__ uint8_t* sq_slot(const QpDev* qp, unsigned long long idx) {
  return qp->sq + ((idx & ((1ull << qp->sq_log) - 1)) << 6);
}
// One WQEBB as four 16-byte stores.  The bytes come from the mlx5_wire.h builders, built into a local Wqe64.
__device__ __forceinline__ void store_wqe(uint8_t* dst, const Wqe64& w) {
  const uint4* v = reinterpret_cast<const uint4*>(&w);
#pragma unroll
  for (int i = 0; i < 4; ++i) st_v4(dst + 16 * i, v[i].x, v[i].y, v[i].z, v[i].w);
}

// Read n (1..MAX_INLINE) bytes at p into registers.  Any address works (the memory need not be registered); word loads
// when p and n are 4-byte multiples, byte loads otherwise -- nothing past p + n is read.
__device__ __forceinline__ InlinePayload inline_load(const void* p, uint32_t n) {
  InlinePayload d;
  const uint8_t* b = static_cast<const uint8_t*>(p);
  if ((((uintptr_t)b | n) & 3u) == 0) {
#pragma unroll
    for (uint32_t j = 0; j < 7; ++j) d.w[j] = 4 * j < n ? reinterpret_cast<const uint32_t*>(b)[j] : 0u;
  } else {
#pragma unroll
    for (uint32_t j = 0; j < 7; ++j) {
      uint32_t x = 0;
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
        if (4 * j + k < n) x |= (uint32_t)b[4 * j + k] << (8 * k);
      d.w[j] = x;
    }
  }
  return d;
}

// -------------------------------------------------------------- doorbell
// Publish WQEs [idx, idx+n): in index order, update the doorbell record, then ring
// the doorbell register with the first 8 bytes of the last WQE's ctrl segment.
// `shared` = other threads may post to this QP concurrently (then the ready_head hand-off
// needs acquire/release); a QP driven by a single thread skips both.
__device__ __forceinline__ void st_u64_release_scope(void* p, unsigned long long v, bool sys) {
  if (sys) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  else asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Ring the doorbell for every WQE below `to`: record, then register.
__device__ __forceinline__ void ring_doorbell(uint32_t* dbr, unsigned long long* bf, uint32_t qpn, unsigned long long to,
                                              bool sys) {
  st_u32_volatile(&dbr[DBR_SND], wq_dbr_word(to));
  // The doorbell register store is a RELEASE: WQE bytes and the doorbell record are visible before
  // it (what the engine audits, and what a ConnectX requires: it may fetch the record and the WQE as
  // soon as the MMIO write lands).
  st_u64_release_scope(bf, doorbell_word(qpn, (uint16_t)(to - 1)), sys);
}

// Single-poster submit: the calling thread is the only one posting to this QP.
// Scope of the POSTER's fences: system scope only when the send queue / doorbell are outside this GPU
// (host-resident rings, a real NIC).  A device-resident queue is consumed by the engine on the same
// GPU, so gpu scope is enough even if the responder is another GPU -- publishing remotely-visible
// bytes is the engine's job (QpDev::sys_scope).  (Using system scope here stretched a 230 us GEMM to
// 470 us when its panels went over NVLink: each MEMBAR.SYS stalled an epilogue.)
__device__ __forceinline__ bool poster_sys(const QpDev* qp) { return qp->sq_in_device == 0; }

__device__ __forceinline__ int sq_submit_exclusive(QpDev* qp, unsigned long long idx, uint32_t n) {
  ring_doorbell(qp->dbr, qp->bf, qp->qpn, idx + n, poster_sys(qp));
  trace_stamp(qp, idx, TR_POST);
  st_u64_relaxed(&qp->ready_head, idx + n);
  return WAIT_OK;
}

// Shared submit: any number of threads post concurrently and NOBODY waits for a predecessor.
//   1. publish "WQE idx is complete" in its slot flag (generation-tagged with idx + 1);
//   2. try-lock db_lock; the holder scans the run of consecutive ready slots from ready_head, rings ONE
//      doorbell for the whole run, unlocks and re-checks.  A poster that finds the lock taken just
//      leaves: the holder's re-check (after unlock) or a later poster covers its WQE.
// The in-order variant (wait until ready_head == idx, then ring) serialised one doorbell per WQE --
// ~2 us each at gpu scope, ~10 us at system scope -- and a waiting poster stalls its CTA: with 64
// panel posts it stretched a 262 us GEMM to 629 us over NVLink.
// The flag store / lock and unlock / flag load pairs form a store-buffering pattern, hence the
// sequentially-consistent fences (__threadfence*), not acq_rel ones.
__device__ __forceinline__ int sq_submit_shared(QpDev* qp, unsigned long long idx, uint32_t n) {
  const bool sys = poster_sys(qp);
  const unsigned long long mask = (1ull << qp->sq_log) - 1;
  if (sys) __threadfence_system(); else __threadfence();          // WQE bytes before the flag
  for (uint32_t i = 0; i < n; ++i) st_u32_volatile(&qp->ready_flags[(idx + i) & mask], (uint32_t)(idx + i + 1));
  trace_stamp(qp, idx, TR_POST);
  for (;;) {
    __threadfence();                                               // flag store before the lock attempt (SC)
    if (atomicCAS(&qp->db_lock, 0u, 1u) != 0u) return WAIT_OK;
    __threadfence();
    unsigned long long h = ld_u64_volatile(&qp->ready_head), to = h;
    while (to - h <= mask && ld_u32_volatile(&qp->ready_flags[to & mask]) == (uint32_t)(to + 1)) ++to;
    if (to > h) {
      if (sys) __threadfence_system(); else __threadfence();      // other posters' WQE bytes (seen via their flags) before the doorbell
      ring_doorbell(qp->dbr, qp->bf, qp->qpn, to, sys);
      st_u64_relaxed(&qp->ready_head, to);
    }
    __threadfence();
    atomicExch(&qp->db_lock, 0u);
    __threadfence();                                               // unlock before the re-check load (SC)
    if (ld_u32_volatile(&qp->ready_flags[to & mask]) != (uint32_t)(to + 1)) return WAIT_OK;
  }
}

__device__ __forceinline__ int sq_submit(QpDev* qp, unsigned long long idx, uint32_t n, bool shared = true) {
  return shared ? sq_submit_shared(qp, idx, n) : sq_submit_exclusive(qp, idx, n);
}

// -------------------------------------------------------------- completion queue
// Every send-CQ consumer reads a CQE's last 16 bytes (timestamp_l | sop_drop_qpn | wqe_counter,sig,op_own) and, once
// cqe_valid holds, asks whether it is a requester completion of its QP; a failed one also sets rc = WAIT_CQE_ERROR.
// A CQ may be shared (send + receive side of a loopback QP, or several QPs): a responder completion, or a
// requester completion of another QP, is NOT ours -- its wqe_counter is an index into another queue, so crediting it to
// sq_cons would hand out SQ slots that have not executed yet.  Leave it at the head for its own consumer (recv_wait /
// the other QP's poller).
__device__ __forceinline__ bool req_cqe(const uint4& tail, uint32_t qpn, int& rc) {
  const uint8_t opc = cqe_tail_opcode(tail);
  if ((opc != CQE_REQ && opc != CQE_REQ_ERR) || cqe_tail_qpn(tail) != qpn) return false;
  if (opc == CQE_REQ_ERR) rc = WAIT_CQE_ERROR;
  return true;
}
// The completed index after an accepted CQE: its 16-bit wqe_counter + 1 expanded against the consumer position `cons`.
__device__ __forceinline__ unsigned long long req_cqe_done(const uint4& tail, unsigned long long cons) {
  return expand16(cqe_tail_counter(tail) + 1u, cons);
}

// Consume at most one CQE of the QP's send CQ.  Returns 1 if one was consumed, 0 if
// none was ready, <0 on an error CQE (which also moves the QP to ERR).
__device__ __forceinline__ int cq_poll_once(QpDev* qp) {
  CqDev* cq = qp->scq;
  unsigned int ci = *(volatile unsigned int*)&cq->ci;
  const uint8_t* cqe = cq->buf + ((size_t)(ci & ((1u << cq->log_n) - 1)) << 6);
  const uint4 tail = ld_v4_volatile(cqe + CQE_TAIL_OFF);
  if (!cqe_valid(cqe_tail_op_own(tail), ci, cq->log_n)) return 0;
  __threadfence();  // acquire: payload and the rest of the CQE are visible past this point
  int rc = 1;
  if (!req_cqe(tail, qp->qpn, rc)) return 0;
  unsigned long long done = req_cqe_done(tail, ld_u64_volatile(&qp->sq_cons));
  if (atomicCAS(&cq->ci, ci, ci + 1) == ci) {
    trace_stamp(qp, done - 1, TR_SEEN);
    atomicMax(&qp->sq_cons, done);
    st_u32_volatile(&cq->dbrec[0], cq_dbr_word(ci + 1));
  }
  return rc;
}

// Wait until WQE `idx` (and, RC being in-order, everything before it) completed.
__device__ __forceinline__ int sq_wait(QpDev* qp, unsigned long long idx,
                                       unsigned long long timeout_ns = 2000000000ull) {
  unsigned long long t0 = 0;
  int err = WAIT_OK;
  for (unsigned it = 0;; ++it) {
    if (ld_u64_volatile(&qp->sq_cons) > idx) return err;
    int rc = cq_poll_once(qp);
    if (rc < 0) err = rc;
    if (rc == 0) {
      if (t0 == 0) t0 = globaltimer_ns();
      else if ((it & 15) == 0 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
    }
  }
}

// -------------------------------------------------------------- exclusive poster (fast path)
// When ONE thread owns a QP and its send CQ for the duration of a kernel (the stream poster, a fused
// kernel's posting warp), nothing about the queue needs an atomic or a re-read: the producer index, the
// completed index and the CQ consumer index live in registers, the QpDev / CqDev words are only written
// (fire-and-forget stores, for the host and for later kernels), and the completion queue is consulted
// only when the window is actually full.  Per message that leaves ONE dependent wait on the critical
// path -- the release in front of the doorbell -- instead of the 5-6 round trips of reserve (atomic) /
// submit / poll (CAS + atomicMax): 3.7 us -> ~1 us per single post on the device-local wire, and on a
// ConnectX the same structure is what keeps the SM off the PCIe round trip.
struct Poster {
  QpDev* qp;
  uint8_t* sq;
  const uint8_t* cq_buf;
  CqDev* cq;
  uint32_t* dbr;
  unsigned long long* bf;
  unsigned long long head;     // next WQE index to build
  unsigned long long cons;     // every index below this is complete
  unsigned int ci;             // CQ consumer index
  uint32_t sq_mask, cq_log, qpn;
  bool sys, trace;
};

__device__ __forceinline__ Poster poster_open(QpDev* qp) {
  Poster p;
  p.qp = qp; p.sq = qp->sq; p.cq = qp->scq; p.cq_buf = p.cq->buf; p.cq_log = p.cq->log_n;
  p.dbr = qp->dbr; p.bf = qp->bf; p.qpn = qp->qpn; p.sq_mask = (1u << qp->sq_log) - 1;
  p.head = ld_u64_volatile(&qp->resv_head);
  p.cons = ld_u64_volatile(&qp->sq_cons);
  p.ci = *(volatile unsigned int*)&p.cq->ci;
  p.sys = poster_sys(qp);
  p.trace = qp->trace_on != 0;
  return p;
}
// Publish the register state (so the host, the shared-submit path and later kernels continue from it).
__device__ __forceinline__ void poster_close(Poster& p) {
  st_u64_relaxed(&p.qp->resv_head, p.head);
  st_u64_relaxed(&p.qp->ready_head, p.head);
  st_u64_relaxed(&p.qp->sq_cons, p.cons);
  *(volatile unsigned int*)&p.cq->ci = p.ci;
  st_u32_volatile(&p.cq->dbrec[0], cq_dbr_word(p.ci));
}
// Consume CQEs that are ready now.  Returns <0 on an error completion (the rest of the run is still
// consumed), else the number consumed.  A CQE that is not a requester completion of this QP stops the
// scan (shared CQ: not ours to take).
__device__ __forceinline__ int poster_poll(Poster& p, int max_cqes = 8) {
  int n = 0, rc = 0;
  while (n < max_cqes) {
    const uint8_t* cqe = p.cq_buf + ((size_t)(p.ci & ((1u << p.cq_log) - 1)) << 6);
    const uint4 tail = ld_v4_volatile(cqe + CQE_TAIL_OFF);
    if (!cqe_valid(cqe_tail_op_own(tail), p.ci, p.cq_log)) break;
    if (!req_cqe(tail, p.qpn, rc)) break;
    p.cons = req_cqe_done(tail, p.cons);
    if (p.trace) trace_stamp(p.qp, p.cons - 1, TR_SEEN);
    ++p.ci;
    ++n;
  }
  if (n) {
    __threadfence();                                              // acquire: payload behind the CQEs just seen
    st_u32_volatile(&p.cq->dbrec[0], cq_dbr_word(p.ci));          // consumer record (what a NIC checks for overrun)
    *(volatile unsigned int*)&p.cq->ci = p.ci;
  }
  return rc < 0 ? rc : n;
}
// Split poll: issue the load of the next CQE's tail now, look at it later.  A poster that interleaves
//     build WQE -> poster_peek -> poster_ring (release + doorbell) -> poster_take
// has the CQE load in flight while the release in front of the doorbell waits for the WQE stores to be acknowledged:
// the two L2 round trips of a post-one / poll-one iteration overlap instead of adding up.
__device__ __forceinline__ uint4 poster_peek(const Poster& p) {
  return ld_v4_volatile(p.cq_buf + ((size_t)(p.ci & ((1u << p.cq_log) - 1)) << 6) + CQE_TAIL_OFF);
}
// Consume the CQE whose tail was loaded by poster_peek, if it was ready and ours.  Returns 1 / 0 / WAIT_CQE_ERROR.
__device__ __forceinline__ int poster_take(Poster& p, const uint4 tail) {
  if (!cqe_valid(cqe_tail_op_own(tail), p.ci, p.cq_log)) return 0;
  int rc = 1;
  if (!req_cqe(tail, p.qpn, rc)) return 0;
  p.cons = req_cqe_done(tail, p.cons);
  if (p.trace) trace_stamp(p.qp, p.cons - 1, TR_SEEN);
  ++p.ci;
  __threadfence();                                                // acquire: payload behind the CQE
  st_u32_volatile(&p.cq->dbrec[0], cq_dbr_word(p.ci));
  return rc;
}

// Block until WQE `idx` completed (or timeout / error).
__device__ __forceinline__ int poster_wait(Poster& p, unsigned long long idx, unsigned long long timeout_ns) {
  int err = WAIT_OK;
  unsigned long long t0 = 0;
  for (unsigned it = 0; p.cons <= idx; ++it) {
    const int rc = poster_poll(p);
    if (rc < 0) err = rc;
    if (rc == 0) {
      if (t0 == 0) t0 = globaltimer_ns();
      else if ((it & 15) == 0 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
    }
  }
  return err;
}
// Make room for n more WQEs; returns the first index or ~0ull on timeout (nothing was reserved: the
// producer index only moves when the WQEs are built, so a timeout leaves no hole).
__device__ __forceinline__ unsigned long long poster_reserve(Poster& p, uint32_t n, unsigned long long timeout_ns) {
  const unsigned long long depth = (unsigned long long)p.sq_mask + 1;
  if (p.head + n - p.cons > depth) {
    const int rc = poster_wait(p, p.head + n - depth - 1, timeout_ns);
    if (rc == WAIT_TIMEOUT) return ~0ull;
  }
  return p.head;
}
__device__ __forceinline__ uint8_t* poster_slot(const Poster& p, unsigned long long idx) {
  return p.sq + ((idx & p.sq_mask) << 6);
}
// Ring ONE doorbell for everything built in [p.head, to).
__device__ __forceinline__ void poster_ring(Poster& p, unsigned long long to) {
  ring_doorbell(p.dbr, p.bf, p.qpn, to, p.sys);
  if (p.trace) for (unsigned long long i = p.head; i < to; ++i) trace_stamp(p.qp, i, TR_POST);
  p.head = to;
}

// -------------------------------------------------------------- one WQE through the shared submit
// Reserve a slot, let build(Wqe64*, idx) encode WQE idx (an mlx5_wire.h builder), store it, submit.  Returns the WQE
// index, or ~0ull when the queue stayed full or the QP is in ERR.
template <typename Build>
__device__ __forceinline__ unsigned long long post_one(QpDev* qp, Build build,
                                                       unsigned long long timeout_ns = 2000000000ull) {
  const unsigned long long idx = sq_reserve(qp, 1, timeout_ns);
  if (idx == ~0ull) return idx;
  Wqe64 w;
  build(&w, idx);
  store_wqe(sq_slot(qp, idx), w);
  if (sq_submit(qp, idx, 1) != WAIT_OK) return ~0ull;
  return idx;
}

// -------------------------------------------------------------- one-call verbs
// Every one-call verb takes `signaled` (a CQE on success) and, last, `fence` (IBV_SEND_FENCE: the WR moves no byte, and
// its atomic does not execute, before every earlier WR of the QP has finished -- DESIGN.md 3.1).
__device__ __forceinline__ uint8_t wr_flags(bool signaled, bool fence) {
  return (uint8_t)((signaled ? CTRL_CQ_UPDATE : 0) | (fence ? CTRL_FENCE : 0));
}
__device__ __forceinline__ unsigned long long rdma_write(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                         uint64_t raddr, uint32_t rkey, uint32_t bytes,
                                                         bool signaled = true, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_rdma_wqe(w, OP_RDMA_WRITE, (uint16_t)idx, qp->qpn, laddr, lkey, raddr, rkey, bytes, wr_flags(signaled, fence), 0);
  });
}
__device__ __forceinline__ unsigned long long rdma_read(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                        uint64_t raddr, uint32_t rkey, uint32_t bytes,
                                                        bool signaled = true, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_rdma_wqe(w, OP_RDMA_READ, (uint16_t)idx, qp->qpn, laddr, lkey, raddr, rkey, bytes, wr_flags(signaled, fence), 0);
  });
}
__device__ __forceinline__ unsigned long long rdma_send(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                        uint32_t bytes, bool signaled = true,
                                                        uint32_t imm = 0, bool with_imm = false, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_send_wqe(w, with_imm ? OP_SEND_IMM : OP_SEND, (uint16_t)idx, qp->qpn, laddr, lkey, bytes,
                   wr_flags(signaled, fence), imm);
  });
}

// Two-entry scatter-gather verbs through the shared submit: the message is sg[0] then sg[1] (zero-length entries dropped;
// with at most one left, the WQE is the one-entry verb's).  WRITE: gathered to [raddr, raddr + total).  READ: that range
// scattered into sg[0] then sg[1].  SEND: the concatenation into the responder's next receive.
__device__ __forceinline__ unsigned long long rdma_write_sg(QpDev* qp, const Sge (&sg)[MAX_SGE], uint64_t raddr, uint32_t rkey,
                                                            bool signaled = true, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_rdma_sg_wqe(w, OP_RDMA_WRITE, (uint16_t)idx, qp->qpn, sg, MAX_SGE, raddr, rkey, wr_flags(signaled, fence), 0);
  });
}
__device__ __forceinline__ unsigned long long rdma_read_sg(QpDev* qp, const Sge (&sg)[MAX_SGE], uint64_t raddr, uint32_t rkey,
                                                           bool signaled = true, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_rdma_sg_wqe(w, OP_RDMA_READ, (uint16_t)idx, qp->qpn, sg, MAX_SGE, raddr, rkey, wr_flags(signaled, fence), 0);
  });
}
__device__ __forceinline__ unsigned long long rdma_send_sg(QpDev* qp, const Sge (&sg)[MAX_SGE], bool signaled = true,
                                                           uint32_t imm = 0, bool with_imm = false, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_send_sg_wqe(w, with_imm ? OP_SEND_IMM : OP_SEND, (uint16_t)idx, qp->qpn, sg, MAX_SGE, wr_flags(signaled, fence), imm);
  });
}

// Remote 8-byte atomics through the shared submit: any thread of any kernel may call them (a producer signalling
// "data landed" after its RDMA WRITEs: the engine executes the atomic only after every earlier WQE of the QP).
// The original remote value lands in the 8 local bytes at laddr.
__device__ __forceinline__ unsigned long long rdma_fetch_add(QpDev* qp, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                                             uint32_t rkey, uint64_t add, bool signaled = true,
                                                             bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_atomic_wqe(w, OP_ATOMIC_FA, (uint16_t)idx, qp->qpn, laddr, lkey, raddr, rkey, add, 0, wr_flags(signaled, fence));
  });
}
__device__ __forceinline__ unsigned long long rdma_cmp_swap(QpDev* qp, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                                            uint32_t rkey, uint64_t compare, uint64_t swap,
                                                            bool signaled = true, bool fence = false) {
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_atomic_wqe(w, OP_ATOMIC_CS, (uint16_t)idx, qp->qpn, laddr, lkey, raddr, rkey, swap, compare,
                     wr_flags(signaled, fence));
  });
}

// Inline puts through the shared submit: an RDMA WRITE whose 1..MAX_INLINE payload bytes travel in the WQE.  No local
// buffer and no lkey: `data` may be any memory the calling thread can read (or a register, with rdma_p), and it may be
// reused as soon as the call returns.  Returns the WQE index, or ~0ull when n is out of range or the queue stayed full.
__device__ __forceinline__ unsigned long long rdma_put_inline(QpDev* qp, uint64_t raddr, uint32_t rkey, const void* data,
                                                              uint32_t n, bool signaled = true, bool fence = false) {
  if (n == 0 || n > MAX_INLINE) return ~0ull;
  const InlinePayload d = inline_load(data, n);
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_inline_wqe(w, OP_RDMA_WRITE, (uint16_t)idx, qp->qpn, raddr, rkey, d, n, wr_flags(signaled, fence), 0);
  });
}
// nvshmem_p / doca_gpu_dev_verbs_p: one 1-, 2-, 4- or 8-byte value straight from a register.
template <typename T>
__device__ __forceinline__ unsigned long long rdma_p(QpDev* qp, uint64_t raddr, uint32_t rkey, T value, bool signaled = true,
                                                     bool fence = false) {
  static_assert(sizeof(T) == 1 || sizeof(T) == 2 || sizeof(T) == 4 || sizeof(T) == 8, "rdma_p: 1, 2, 4 or 8 bytes");
  InlinePayload d = {};
  memcpy(d.w, &value, sizeof(T));
  return post_one(qp, [&](Wqe64* w, unsigned long long idx) {
    build_inline_wqe(w, OP_RDMA_WRITE, (uint16_t)idx, qp->qpn, raddr, rkey, d, (uint32_t)sizeof(T),
                     wr_flags(signaled, fence), 0);
  });
}

// -------------------------------------------------------------- fused kernels' posts
// One record WRITE (or WRITE_IMM, carrying `imm`), posted by whichever CTA finishes the record.  Records go out in
// completion order, not record order, so they are signaled by WQE index (every signal_every-th slot): the CQ keeps
// freeing the send queue.  A posted record is counted in acc = [highest index + 1, records posted, ~earliest post time];
// a failed post sets out[0] = WAIT_TIMEOUT.
__device__ __forceinline__ void post_record(QpDev* qp, uint8_t opcode, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                            uint32_t rkey, uint32_t bytes, uint32_t imm, uint32_t signal_every,
                                            unsigned long long* acc, unsigned long long* out,
                                            unsigned long long timeout_ns) {
  const unsigned long long idx = post_one(qp, [&](Wqe64* w, unsigned long long i) {
    const bool sig = signal_every <= 1 || ((i + 1) % signal_every == 0);
    build_rdma_wqe(w, opcode, (uint16_t)i, qp->qpn, laddr, lkey, raddr, rkey, bytes, sig ? CTRL_CQ_UPDATE : 0, imm);
  }, timeout_ns);
  if (idx == ~0ull) {
    out[0] = (unsigned long long)(long long)WAIT_TIMEOUT;
    return;
  }
  atomicMax(&acc[0], idx + 1);
  atomicAdd(&acc[1], 1ull);
  atomicMax(&acc[2], ~globaltimer_ns());
}
// Flush: one signaled NOP behind everything posted so far.  RC completes in order, so its CQE shows that every earlier
// WQE of the QP has completed.  Waits for it unless post_only (then the caller reaps it).  Returns a WAIT_* status.
__device__ __forceinline__ int post_flush(QpDev* qp, bool post_only, unsigned long long timeout_ns) {
  const unsigned long long idx = post_one(qp, [&](Wqe64* w, unsigned long long i) {
    build_nop_wqe(w, (uint16_t)i, qp->qpn, CTRL_CQ_UPDATE);
  }, timeout_ns);
  if (idx == ~0ull) return WAIT_TIMEOUT;
  return post_only ? WAIT_OK : sq_wait(qp, idx, timeout_ns);
}

// Post one receive WQE on the QP's own RQ (single poster per RQ).
__device__ __forceinline__ void post_recv(QpDev* qp, uint64_t addr, uint32_t lkey, uint32_t bytes) {
  unsigned long long i = qp->rq_pi;
  uint8_t* slot = qp->rq + ((i & ((1ull << qp->rq_log) - 1)) << 4);
  const uint4 r = recv_wqe_words(addr, lkey, bytes);
  st_v4(slot, r.x, r.y, r.z, r.w);
  fence_sys();
  qp->rq_pi = i + 1;
  st_u32_volatile(&qp->dbr[DBR_RCV], wq_dbr_word(i + 1));
  fence_sys();
}

// Poll the receive CQ for one completion.  Returns bytes received (>=0) and the
// immediate through *imm, WAIT_TIMEOUT, or WAIT_CQE_ERROR.
__device__ __forceinline__ long long recv_wait(QpDev* qp, uint32_t* imm, unsigned long long timeout_ns) {
  CqDev* cq = qp->rcq;
  unsigned long long t0 = globaltimer_ns();
  for (unsigned it = 0;; ++it) {
    unsigned int ci = *(volatile unsigned int*)&cq->ci;
    const uint8_t* cqe = cq->buf + ((size_t)(ci & ((1u << cq->log_n) - 1)) << 6);
    const uint4 tail = ld_v4_volatile(cqe + CQE_TAIL_OFF);
    if (cqe_valid(cqe_tail_op_own(tail), ci, cq->log_n)) {
      __threadfence();
      const uint4 mid = ld_v4_volatile(cqe + CQE_MID_OFF);
      const uint8_t opc = cqe_tail_opcode(tail);
      if (opc == CQE_REQ || opc == CQE_REQ_ERR) {      // shared CQ: a send completion is at the head; its poller takes it
        if ((it & 15) == 15 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
        continue;
      }
      if (atomicCAS(&cq->ci, ci, ci + 1) != ci) continue;
      st_u32_volatile(&cq->dbrec[0], cq_dbr_word(ci + 1));
      if (cqe_is_error(opc)) return WAIT_CQE_ERROR;
      if (imm) *imm = cqe_mid_imm(mid);
      return (long long)cqe_mid_byte_cnt(mid);
    }
    if ((it & 15) == 15 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
  }
}

}  // namespace dev

// SM count of the current device (launch sizing of the persistent and grid-stride kernels)
static inline int device_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  return n;
}

// What the ops launchers share on the host.
// A wait bound in ns from the timeout_ms every entry point takes (0: 2 s).
static inline unsigned long long timeout_ns(uint64_t timeout_ms) { return (timeout_ms ? timeout_ms : 2000) * 1000000ull; }

// Zero a launch's 8-word result record: mapped pinned memory, so the host writes it directly (no memset kernel).
static inline unsigned long long* clear_record(uint64_t out_dev) {
  unsigned long long* o = (unsigned long long*)out_dev;
  for (int i = 0; i < 8; ++i) o[i] = 0;
  return o;
}

// Copy a multi-QP launch's queue pairs, one per CTA, into its by-value argument array; false unless 1 <= nqp <= kMax.
template <int kMax>
static inline bool copy_qps(QpDev* (&qps)[kMax], const uint64_t* qps_host, uint32_t nqp) {
  if (nqp == 0 || nqp > (uint32_t)kMax) return false;
  for (uint32_t i = 0; i < nqp; ++i) qps[i] = (QpDev*)qps_host[i];
  return true;
}
}  // namespace rn
