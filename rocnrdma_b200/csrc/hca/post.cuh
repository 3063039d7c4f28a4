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

// -------------------------------------------------------------- WQE writers
// Four 16-byte stores = one WQEBB.  Fields are big-endian on the wire.
__device__ __forceinline__ void write_rdma_wqe(QpDev* qp, unsigned long long idx, uint8_t opcode,
                                               uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                               uint32_t rkey, uint32_t bytes, uint8_t fm_ce_se,
                                               uint32_t imm = 0) {
  uint8_t* slot = qp->sq + ((idx & ((1ull << qp->sq_log) - 1)) << 6);
  // ctrl: opmod_idx_opcode | qpn_ds | sig,rsvd,fm_ce_se | imm
  st_v4(slot + 0, ctrl_word0(opcode, (uint16_t)idx), ctrl_word1(qp->qpn, 3), (uint32_t)fm_ce_se << 24,
        be32(imm));
  // raddr: be64 raddr | be32 rkey | 0      (be64 in memory = be32(hi), be32(lo))
  st_v4(slot + 16, be32((uint32_t)(raddr >> 32)), be32((uint32_t)raddr), be32(rkey), 0u);
  // data: be32 byte_count | be32 lkey | be64 addr
  st_v4(slot + 32, be32(bytes & 0x7fffffffu), be32(lkey), be32((uint32_t)(laddr >> 32)), be32((uint32_t)laddr));
  st_v4(slot + 48, 0u, 0u, 0u, 0u);
}
__device__ __forceinline__ void write_send_wqe(QpDev* qp, unsigned long long idx, uint8_t opcode,
                                               uint64_t laddr, uint32_t lkey, uint32_t bytes,
                                               uint8_t fm_ce_se, uint32_t imm = 0) {
  uint8_t* slot = qp->sq + ((idx & ((1ull << qp->sq_log) - 1)) << 6);
  st_v4(slot + 0, ctrl_word0(opcode, (uint16_t)idx), ctrl_word1(qp->qpn, 2), (uint32_t)fm_ce_se << 24,
        be32(imm));
  st_v4(slot + 16, be32(bytes & 0x7fffffffu), be32(lkey), be32((uint32_t)(laddr >> 32)), be32((uint32_t)laddr));
  st_v4(slot + 32, 0u, 0u, 0u, 0u);
  st_v4(slot + 48, 0u, 0u, 0u, 0u);
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
// Ring the doorbell for WQEs [from, to): record, then register (a release store), then ready_head.
__device__ __forceinline__ void ring_doorbell(QpDev* qp, unsigned long long to, bool sys) {
  const unsigned long long last = to - 1;
  st_u32_volatile(&qp->dbr[DBR_SND], be32((uint32_t)(to & 0xffff)));
  unsigned long long db = (unsigned long long)ctrl_word0(OP_NOP, (uint16_t)last) |
                          ((unsigned long long)ctrl_word1(qp->qpn, 0) << 32);
  // The doorbell register store is a RELEASE: WQE bytes and the doorbell record are visible before
  // it (what the engine audits, and what a ConnectX requires: it may fetch the record and the WQE as
  // soon as the MMIO write lands).
  st_u64_release_scope(qp->bf, db, sys);
}

// Single-poster submit: the calling thread is the only one posting to this QP.
// Scope of the POSTER's fences: system scope only when the send queue / doorbell are outside this GPU
// (host-resident rings, a real NIC).  A device-resident queue is consumed by the engine on the same
// GPU, so gpu scope is enough even if the responder is another GPU -- publishing remotely-visible
// bytes is the engine's job (QpDev::sys_scope).  (Using system scope here stretched a 230 us GEMM to
// 470 us when its panels went over NVLink: each MEMBAR.SYS stalled an epilogue.)
__device__ __forceinline__ bool poster_sys(const QpDev* qp) { return qp->sq_in_device == 0; }

__device__ __forceinline__ int sq_submit_exclusive(QpDev* qp, unsigned long long idx, uint32_t n) {
  const bool sys = poster_sys(qp);
  ring_doorbell(qp, idx + n, sys);
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
      ring_doorbell(qp, to, sys);
      st_u64_relaxed(&qp->ready_head, to);
    }
    __threadfence();
    atomicExch(&qp->db_lock, 0u);
    __threadfence();                                               // unlock before the re-check load (SC)
    if (ld_u32_volatile(&qp->ready_flags[to & mask]) != (uint32_t)(to + 1)) return WAIT_OK;
  }
}

__device__ __forceinline__ int sq_submit(QpDev* qp, unsigned long long idx, uint32_t n,
                                         unsigned long long timeout_ns = 2000000000ull, bool shared = true) {
  (void)timeout_ns;
  return shared ? sq_submit_shared(qp, idx, n) : sq_submit_exclusive(qp, idx, n);
}

// -------------------------------------------------------------- completion queue
// Consume at most one CQE of the QP's send CQ.  Returns 1 if one was consumed, 0 if
// none was ready, <0 on an error CQE (which also moves the QP to ERR).
__device__ __forceinline__ int cq_poll_once(QpDev* qp) {
  CqDev* cq = qp->scq;
  unsigned int ci = *(volatile unsigned int*)&cq->ci;
  const uint8_t* cqe = cq->buf + ((size_t)(ci & ((1u << cq->log_n) - 1)) << 6);
  uint4 tail = ld_v4_volatile(cqe + 48);  // timestamp_l | sop_drop_qpn | wqe_counter,sig,op_own
  uint8_t op_own = (uint8_t)(tail.w >> 24);
  if (!cqe_valid(op_own, ci, cq->log_n)) return 0;
  __threadfence();  // acquire: payload and the rest of the CQE are visible past this point
  uint16_t wqe_counter = be16((uint16_t)(tail.w & 0xffff));
  int rc = 1;
  uint8_t opc = cqe_opcode(op_own);
  // A CQ may be shared (send + receive side of a loopback QP, or several QPs): a responder completion,
  // or a requester completion of another QP, is NOT ours -- its wqe_counter is an index into another
  // queue, so crediting it to sq_cons would hand out SQ slots that have not executed yet.  Leave it at
  // the head for its own consumer (recv_wait / the other QP's poller).
  if ((opc != CQE_REQ && opc != CQE_REQ_ERR) || (be32(tail.z) & 0xffffffu) != qp->qpn) return 0;
  if (opc == CQE_REQ_ERR) rc = WAIT_CQE_ERROR;
  // Expand the 16-bit counter against the current consumer position.
  unsigned long long cons = ld_u64_volatile(&qp->sq_cons);
  unsigned long long done = cons + (unsigned long long)((uint16_t)(wqe_counter + 1 - (uint16_t)cons));
  if (atomicCAS(&cq->ci, ci, ci + 1) == ci) {
    trace_stamp(qp, done - 1, TR_SEEN);
    atomicMax(&qp->sq_cons, done);
    st_u32_volatile(&cq->dbrec[0], be32((ci + 1) & 0xffffff));
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
      if (qp->state == QPS_ERR && ld_u64_volatile(&qp->sq_cons) <= idx && it > 64) {
        // keep draining: flushed WQEs still produce error CQEs
      }
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
  st_u32_volatile(&p.cq->dbrec[0], be32(p.ci & 0xffffff));
}
// Consume CQEs that are ready now.  Returns <0 on an error completion (the rest of the run is still
// consumed), else the number consumed.  A CQE that is not a requester completion of this QP stops the
// scan (shared CQ: not ours to take).
__device__ __forceinline__ int poster_poll(Poster& p, int max_cqes = 8) {
  int n = 0, rc = 0;
  while (n < max_cqes) {
    const uint8_t* cqe = p.cq_buf + ((size_t)(p.ci & ((1u << p.cq_log) - 1)) << 6);
    const uint4 tail = ld_v4_volatile(cqe + 48);
    const uint8_t op_own = (uint8_t)(tail.w >> 24);
    if (!cqe_valid(op_own, p.ci, p.cq_log)) break;
    const uint8_t opc = cqe_opcode(op_own);
    if ((opc != CQE_REQ && opc != CQE_REQ_ERR) || (be32(tail.z) & 0xffffffu) != p.qpn) break;
    if (opc == CQE_REQ_ERR) rc = WAIT_CQE_ERROR;
    const uint16_t wqe_counter = be16((uint16_t)(tail.w & 0xffff));
    p.cons += (unsigned long long)((uint16_t)(wqe_counter + 1 - (uint16_t)p.cons));
    if (p.trace) trace_stamp(p.qp, p.cons - 1, TR_SEEN);
    ++p.ci;
    ++n;
  }
  if (n) {
    __threadfence();                                              // acquire: payload behind the CQEs just seen
    st_u32_volatile(&p.cq->dbrec[0], be32(p.ci & 0xffffff));      // consumer record (what a NIC checks for overrun)
    *(volatile unsigned int*)&p.cq->ci = p.ci;
  }
  return rc < 0 ? rc : n;
}
// Split poll: issue the load of the next CQE's tail now, look at it later.  A poster that interleaves
//     build WQE -> poster_peek -> poster_ring (release + doorbell) -> poster_take
// has the CQE load in flight while the release in front of the doorbell waits for the WQE stores to be acknowledged:
// the two L2 round trips of a post-one / poll-one iteration overlap instead of adding up.
__device__ __forceinline__ uint4 poster_peek(const Poster& p) {
  return ld_v4_volatile(p.cq_buf + ((size_t)(p.ci & ((1u << p.cq_log) - 1)) << 6) + 48);
}
// Consume the CQE whose tail was loaded by poster_peek, if it was ready and ours.  Returns 1 / 0 / WAIT_CQE_ERROR.
__device__ __forceinline__ int poster_take(Poster& p, const uint4 tail) {
  const uint8_t op_own = (uint8_t)(tail.w >> 24);
  if (!cqe_valid(op_own, p.ci, p.cq_log)) return 0;
  const uint8_t opc = cqe_opcode(op_own);
  if ((opc != CQE_REQ && opc != CQE_REQ_ERR) || (be32(tail.z) & 0xffffffu) != p.qpn) return 0;
  const uint16_t wqe_counter = be16((uint16_t)(tail.w & 0xffff));
  p.cons += (unsigned long long)((uint16_t)(wqe_counter + 1 - (uint16_t)p.cons));
  if (p.trace) trace_stamp(p.qp, p.cons - 1, TR_SEEN);
  ++p.ci;
  __threadfence();                                                // acquire: payload behind the CQE
  st_u32_volatile(&p.cq->dbrec[0], be32(p.ci & 0xffffff));
  return opc == CQE_REQ_ERR ? WAIT_CQE_ERROR : 1;
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
__device__ __forceinline__ void poster_build_rdma(const Poster& p, unsigned long long idx, uint8_t opcode, uint64_t laddr,
                                                  uint32_t lkey, uint64_t raddr, uint32_t rkey, uint32_t bytes,
                                                  uint8_t fm_ce_se, uint32_t imm = 0) {
  uint8_t* slot = poster_slot(p, idx);
  st_v4(slot + 0, ctrl_word0(opcode, (uint16_t)idx), ctrl_word1(p.qpn, 3), (uint32_t)fm_ce_se << 24, be32(imm));
  st_v4(slot + 16, be32((uint32_t)(raddr >> 32)), be32((uint32_t)raddr), be32(rkey), 0u);
  st_v4(slot + 32, be32(bytes & 0x7fffffffu), be32(lkey), be32((uint32_t)(laddr >> 32)), be32((uint32_t)laddr));
  st_v4(slot + 48, 0u, 0u, 0u, 0u);
}
__device__ __forceinline__ void poster_build_send(const Poster& p, unsigned long long idx, uint8_t opcode, uint64_t laddr,
                                                  uint32_t lkey, uint32_t bytes, uint8_t fm_ce_se, uint32_t imm = 0) {
  uint8_t* slot = poster_slot(p, idx);
  st_v4(slot + 0, ctrl_word0(opcode, (uint16_t)idx), ctrl_word1(p.qpn, 2), (uint32_t)fm_ce_se << 24, be32(imm));
  st_v4(slot + 16, be32(bytes & 0x7fffffffu), be32(lkey), be32((uint32_t)(laddr >> 32)), be32((uint32_t)laddr));
  st_v4(slot + 32, 0u, 0u, 0u, 0u);
  st_v4(slot + 48, 0u, 0u, 0u, 0u);
}
// Ring ONE doorbell for everything built in [p.head, to): record, release, register.
__device__ __forceinline__ void poster_ring(Poster& p, unsigned long long to) {
  const unsigned long long last = to - 1;
  st_u32_volatile(&p.dbr[DBR_SND], be32((uint32_t)(to & 0xffff)));
  const unsigned long long db = (unsigned long long)ctrl_word0(OP_NOP, (uint16_t)last) |
                                ((unsigned long long)ctrl_word1(p.qpn, 0) << 32);
  st_u64_release_scope(p.bf, db, p.sys);
  if (p.trace) for (unsigned long long i = p.head; i < to; ++i) trace_stamp(p.qp, i, TR_POST);
  p.head = to;
}

// -------------------------------------------------------------- one-call verbs
__device__ __forceinline__ unsigned long long rdma_write(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                         uint64_t raddr, uint32_t rkey, uint32_t bytes,
                                                         bool signaled = true) {
  unsigned long long idx = sq_reserve(qp, 1);
  if (idx == ~0ull) return idx;
  write_rdma_wqe(qp, idx, OP_RDMA_WRITE, laddr, lkey, raddr, rkey, bytes, signaled ? CTRL_CQ_UPDATE : 0);
  if (sq_submit(qp, idx, 1) != WAIT_OK) return ~0ull;
  return idx;
}
__device__ __forceinline__ unsigned long long rdma_read(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                        uint64_t raddr, uint32_t rkey, uint32_t bytes,
                                                        bool signaled = true) {
  unsigned long long idx = sq_reserve(qp, 1);
  if (idx == ~0ull) return idx;
  write_rdma_wqe(qp, idx, OP_RDMA_READ, laddr, lkey, raddr, rkey, bytes, signaled ? CTRL_CQ_UPDATE : 0);
  if (sq_submit(qp, idx, 1) != WAIT_OK) return ~0ull;
  return idx;
}
__device__ __forceinline__ unsigned long long rdma_send(QpDev* qp, uint64_t laddr, uint32_t lkey,
                                                        uint32_t bytes, bool signaled = true,
                                                        uint32_t imm = 0, bool with_imm = false) {
  unsigned long long idx = sq_reserve(qp, 1);
  if (idx == ~0ull) return idx;
  write_send_wqe(qp, idx, with_imm ? OP_SEND_IMM : OP_SEND, laddr, lkey, bytes,
                 signaled ? CTRL_CQ_UPDATE : 0, imm);
  if (sq_submit(qp, idx, 1) != WAIT_OK) return ~0ull;
  return idx;
}

// Post one receive WQE on the QP's own RQ (single poster per RQ).
__device__ __forceinline__ void post_recv(QpDev* qp, uint64_t addr, uint32_t lkey, uint32_t bytes) {
  unsigned long long i = qp->rq_pi;
  uint8_t* slot = qp->rq + ((i & ((1ull << qp->rq_log) - 1)) << 4);
  st_v4(slot, be32(bytes & 0x7fffffffu), be32(lkey), be32((uint32_t)(addr >> 32)), be32((uint32_t)addr));
  fence_sys();
  qp->rq_pi = i + 1;
  st_u32_volatile(&qp->dbr[DBR_RCV], be32((uint32_t)((i + 1) & 0xffff)));
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
    uint4 tail = ld_v4_volatile(cqe + 48);
    uint8_t op_own = (uint8_t)(tail.w >> 24);
    if (cqe_valid(op_own, ci, cq->log_n)) {
      __threadfence();
      uint4 mid = ld_v4_volatile(cqe + 32);  // srqn | imm | rsvd | byte_cnt
      uint8_t opc = cqe_opcode(op_own);
      if (opc == CQE_REQ || opc == CQE_REQ_ERR) {      // shared CQ: a send completion is at the head; its poller takes it
        if ((it & 15) == 15 && globaltimer_ns() - t0 > timeout_ns) return WAIT_TIMEOUT;
        continue;
      }
      if (atomicCAS(&cq->ci, ci, ci + 1) != ci) continue;
      st_u32_volatile(&cq->dbrec[0], be32((ci + 1) & 0xffffff));
      if (opc == CQE_RESP_ERR || opc == CQE_REQ_ERR) return WAIT_CQE_ERROR;
      if (imm) *imm = be32(mid.y);
      return (long long)be32(mid.w);
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
}  // namespace rn
