// The softhca DMA engine: a persistent sm_90a kernel that plays the HCA.
//
// Pipeline per QP (every stage can be on a different CTA, many WQEs in flight):
//   claim    one CAS on the claim head hands WQE w -- or, with a backlog visible, up to 16 WQEs -- to a
//            CTA (the doorbell bounds it)
//   parse    that CTA reads + decodes the WQE and translates both MKeys -- in parallel
//            with the CTAs parsing w-1, w+1, ...
//   commit   a short ordered section (parse_seq turn): QP-error flush, receive-WQE
//            matching for SEND / WRITE_IMM, publish resolved[w], arm the chunk ticket
//   move     TMA bulk-copy pipeline (cp.async.bulk global->shared->global, one issuing
//            thread, mbarrier-tracked, no LSU traffic); a multi-chunk WQE is offered to
//            idle CTAs through a fetch-add ticket, its owner keeps drawing from it too
//   retire   strictly in order, warp-collective: one CAS on retire_word = (head << 1) | locked takes the
//            per-QP lock and proves the turn, lane i publishes the mlx5 CQEs of WQE head + i
// Large transfers fan out over every engine CTA (HBM / NVLink speed); small messages
// cost one claim + one ordered hand-off each and pipeline across CTAs.
//
// Failure handling mirrors an RC QP: a bad key / bounds / opcode produces an error
// CQE with an IB syndrome, moves the QP to ERR and flushes later WQEs; a missing
// receive WQE is retried until rnr_timeout_ns, then fails with RNR_RETRY_EXC.
// Nothing spins unbounded: the engine leaves when *stop is set or when no doorbell
// has moved for idle_timeout_ns (watchdog), so a forgotten engine cannot wedge a
// GPU (SURVEY.md section 5, "bounded spin + status word").
//
// Reference parity: this is the role the Mellanox HCA itself plays below
// amdp2p's dma_map (amdp2p.c:219-264): consuming bus addresses and moving bytes.
#pragma once
#include <cuda_runtime.h>
#include "hca_types.h"
#include "post.cuh"

namespace rn {
namespace eng {

using namespace rn::dev;

constexpr int kThreads = 128;
constexpr uint32_t kSub = 16384;        // bytes per TMA bulk transaction
constexpr int kStages = 12;             // smem ring: 12 x 16 KiB
// ring split: EngineCtl::stores_in_flight stages (default 4) may hold a TMA store that is still reading smem,
// the others hold loads in flight (copy_bulk<kSif>)
constexpr uint32_t kBulkMin = 4096;     // below this the generic path is as fast

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------ MKey lookup
// Returns the engine-reachable pointer for [addr, addr+len) under `key`, or 0 with
// *syn set.  need = access bits that must all be present.
struct MKeyRaw { uint4 a, b, c; bool in_range; };
// The three 16-byte loads of one entry, issued without looking at them: a WQE's local and remote key
// are fetched back to back (one round trip for both; the remote table may sit across NVLink).
__device__ __forceinline__ MKeyRaw mkey_load(const MKeyEntry* tab, uint32_t n, uint32_t key) {
  MKeyRaw r;
  const uint32_t idx = key >> 8;
  r.in_range = idx < n;
  const uint8_t* e = reinterpret_cast<const uint8_t*>(tab + (r.in_range ? idx : 0));
  r.a = ld_v4_volatile(e);        // base, len
  r.b = ld_v4_volatile(e + 16);   // map_base, key, access
  r.c = ld_v4_volatile(e + 32);   // valid, kind
  return r;
}
__device__ __forceinline__ uint64_t mkey_check(const MKeyRaw& r, uint32_t key, uint64_t addr, uint32_t len, uint32_t need,
                                               bool remote, uint8_t* syn) {
  if (!r.in_range) { *syn = remote ? SYN_REMOTE_ACCESS_ERR : SYN_LOCAL_PROT_ERR; return 0; }
  const uint64_t base = ((uint64_t)r.a.y << 32) | r.a.x, mlen = ((uint64_t)r.a.w << 32) | r.a.z;
  const uint64_t map_base = ((uint64_t)r.b.y << 32) | r.b.x;
  const uint32_t ekey = r.b.z, acc = r.b.w, valid = r.c.x;
  if (!valid || ekey != key) { *syn = remote ? SYN_REMOTE_ACCESS_ERR : SYN_LOCAL_PROT_ERR; return 0; }
  if ((acc & need) != need) { *syn = remote ? SYN_REMOTE_ACCESS_ERR : SYN_LOCAL_ACCESS_ERR; return 0; }
  if (addr < base || addr + len > base + mlen || addr + len < addr) {
    *syn = remote ? SYN_REMOTE_ACCESS_ERR : SYN_LOCAL_PROT_ERR;
    return 0;
  }
  if (len == 0) return map_base ? map_base : 1;  // zero-length: any non-null token
  return map_base + (addr - base);
}
__device__ __forceinline__ uint64_t translate(const MKeyEntry* tab, uint32_t n, uint32_t key, uint64_t addr,
                                              uint32_t len, uint32_t need, bool remote, uint8_t* syn) {
  const MKeyRaw r = mkey_load(tab, n, key);
  return mkey_check(r, key, addr, len, need, remote, syn);
}

// ------------------------------------------------------------------ CQE writer
// A CQE is published in two steps so that a whole run of completions shares one fence: the body
// (first 48 bytes) of every CQE of the run, ONE fence, then the 16-byte tails that carry the owner bit
// (the only word a consumer tests).  Slots are reserved with one atomic per CQ per run.
__device__ __forceinline__ uint8_t* cqe_slot(uint8_t* ring, uint32_t log_n, unsigned int slot) {
  return ring + ((size_t)(slot & ((1u << log_n) - 1)) << 6);
}
__device__ __forceinline__ void cqe_body(uint8_t* cqe, uint8_t opcode, uint32_t byte_cnt, uint32_t imm) {
  const bool err = (opcode == CQE_REQ_ERR || opcode == CQE_RESP_ERR);
  st_v4(cqe + 0, 0u, 0u, 0u, 0u);
  st_v4(cqe + 16, 0u, 0u, 0u, 0u);
  if (!err) st_v4(cqe + 32, 0u, be32(imm), 0u, be32(byte_cnt));
  else st_v4(cqe + 32, 0u, 0u, 0u, 0u);
}
__device__ __forceinline__ void cqe_tail(uint8_t* cqe, uint32_t log_n, unsigned int slot, uint8_t opcode, uint8_t wqe_opcode,
                                         uint32_t qpn, uint16_t wqe_counter, uint8_t syndrome, unsigned long long now) {
  const bool err = (opcode == CQE_REQ_ERR || opcode == CQE_RESP_ERR);
  const uint8_t owner = (uint8_t)((slot >> log_n) & 1u);
  // err view: byte 54 = vendor_err_synd, byte 55 = syndrome (top byte of the word at 52)
  uint32_t w48 = err ? 0u : be32((uint32_t)(now >> 32));
  uint32_t w52 = err ? ((uint32_t)syndrome << 24) : be32((uint32_t)now);
  uint32_t w56 = be32(((uint32_t)wqe_opcode << 24) | (qpn & 0xffffff));
  uint32_t w60 = (uint32_t)be16(wqe_counter) | ((uint32_t)cqe_op_own(opcode, owner) << 24);
  st_v4(cqe + 48, w48, w52, w56, w60);
}

// ------------------------------------------------------------------ chunk copy
struct Smem {
  alignas(128) uint8_t ring[kStages][kSub];
  alignas(8) uint64_t full[kStages];
  // work descriptor broadcast from thread 0
  uint64_t src, dst;
  uint32_t len, nch;
  int have_work;
  uint32_t phase_bits;   // per-stage parity of the next wait
};

// Bulk path: thread 0 keeps kStages - kSif loads and kSif stores in flight.
// (With a single store in flight every 16 KiB step exposed the store's smem-read latency,
// ~0.35 us, which capped a CTA near 45 GB/s.)  Requires 16-byte aligned src, dst and len.
template <int kSif>
__device__ __forceinline__ bool copy_bulk(Smem& s, uint64_t src, uint64_t dst, uint32_t len) {
  const uint32_t nsub = (len + kSub - 1) / kSub;
  uint32_t phase_bits = s.phase_bits;
  constexpr int P = kStages - kSif;
  auto sub_len = [&](uint32_t i) { return (i + 1 == nsub) ? (len - i * kSub) : kSub; };
  uint32_t issued = 0;
  for (; issued < nsub && issued < (uint32_t)P; ++issued) {
    int st = issued % kStages;
    mbar_expect_tx(&s.full[st], sub_len(issued));
    bulk_g2s(s.ring[st], (const void*)(src + (uint64_t)issued * kSub), sub_len(issued), &s.full[st]);
  }
  for (uint32_t i = 0; i < nsub; ++i) {
    int st = i % kStages;
    if (!mbar_try_wait(&s.full[st], (phase_bits >> st) & 1u)) {
      // bounded: a bulk load that never lands (bad mapping) must not wedge the SM
      unsigned long long t0 = globaltimer_ns();
      while (!mbar_try_wait(&s.full[st], (phase_bits >> st) & 1u)) {
        if (globaltimer_ns() - t0 > 1000000000ull) { s.phase_bits = phase_bits; return false; }
      }
    }
    phase_bits ^= 1u << st;
    bulk_s2g((void*)(dst + (uint64_t)i * kSub), s.ring[st], sub_len(i));
    bulk_commit();
    if (issued < nsub) {
      // the stage of load `issued` (= i + P) was last read by store i - kSif:
      // stores i .. i - kSif + 1 may still be pending
      bulk_wait_read<kSif>();
      int ls = issued % kStages;
      mbar_expect_tx(&s.full[ls], sub_len(issued));
      bulk_g2s(s.ring[ls], (const void*)(src + (uint64_t)issued * kSub), sub_len(issued), &s.full[ls]);
      ++issued;
    }
  }
  bulk_wait_all();  // writes complete and visible to this thread
  s.phase_bits = phase_bits;
  return true;
}

// Generic path: any alignment, whole CTA.
__device__ __forceinline__ void copy_generic(uint64_t src, uint64_t dst, uint32_t len) {
  const uint8_t* s = (const uint8_t*)src;
  uint8_t* d = (uint8_t*)dst;
  if ((((src ^ dst) & 15) == 0) && len >= 64) {
    uint32_t head = (uint32_t)((16 - (src & 15)) & 15);
    if (head > len) head = len;
    for (uint32_t i = threadIdx.x; i < head; i += kThreads) d[i] = s[i];
    uint32_t body = (len - head) & ~15u;
    const uint4* s4 = (const uint4*)(s + head);
    uint4* d4 = (uint4*)(d + head);
    for (uint32_t i = threadIdx.x; i < body / 16; i += kThreads) d4[i] = s4[i];
    for (uint32_t i = head + body + threadIdx.x; i < len; i += kThreads) d[i] = s[i];
  } else {
    for (uint32_t i = threadIdx.x; i < len; i += kThreads) d[i] = s[i];
  }
}

// ------------------------------------------------------------------ parse + commit
struct Parsed {
  WqeView v;
  uint64_t src, dst;
  uint8_t syn;
};

// Parallel part: runs concurrently for neighbouring WQEs of the same QP.
__device__ __forceinline__ void parse_wqe(QpDev* qp, unsigned long long w, Parsed* p) {
  const uint32_t mask = (1u << qp->sq_log) - 1;
  const uint8_t* slot = qp->sq + ((w & mask) << 6);
  Wqe64 wqe;
  uint4* wv = reinterpret_cast<uint4*>(&wqe);
  wv[0] = ld_v4_volatile(slot);
  wv[1] = ld_v4_volatile(slot + 16);
  wv[2] = ld_v4_volatile(slot + 32);
  wv[3] = ld_v4_volatile(slot + 48);
  p->syn = SYN_OK;
  p->src = p->dst = 0;
  bool ok = decode_wqe(&wqe, &p->v);
  WqeView& v = p->v;
  if (!ok || v.qpn != qp->qpn || v.wqe_idx != (uint16_t)w) {
    p->syn = SYN_LOCAL_QP_OP_ERR;
  } else if (!qp->r.connected && v.opcode != OP_NOP) {
    p->syn = SYN_LOCAL_QP_OP_ERR;
  } else {
    switch (v.opcode) {
      case OP_NOP: v.bytes = 0; break;
      case OP_RDMA_WRITE:
      case OP_RDMA_WRITE_IMM: {
        const MKeyRaw lk = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), rk = mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey);
        p->src = mkey_check(lk, v.lkey, v.laddr, v.bytes, 0, false, &p->syn);
        if (p->src) p->dst = mkey_check(rk, v.rkey, v.raddr, v.bytes, ACC_REMOTE_WRITE, true, &p->syn);
        break;
      }
      case OP_RDMA_READ: {
        const MKeyRaw lk = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), rk = mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey);
        p->dst = mkey_check(lk, v.lkey, v.laddr, v.bytes, ACC_LOCAL_WRITE, false, &p->syn);
        if (p->dst) p->src = mkey_check(rk, v.rkey, v.raddr, v.bytes, ACC_REMOTE_READ, true, &p->syn);
        break;
      }
      case OP_SEND:
      case OP_SEND_IMM:
        p->src = translate(qp->lkeys, qp->n_lkeys, v.lkey, v.laddr, v.bytes, 0, false, &p->syn);
        break;
      default: p->syn = SYN_LOCAL_QP_OP_ERR;
    }
  }
}

__device__ __forceinline__ bool needs_recv_wqe(uint8_t opcode) {
  return opcode == OP_SEND || opcode == OP_SEND_IMM || opcode == OP_RDMA_WRITE_IMM;
}

// Publish resolved[w].  Runs in the parallel part for plain RDMA WRITE / READ / NOP and in
// the ordered part for receive-consuming opcodes.  Returns the number of chunks.
__device__ __forceinline__ uint32_t write_resolved(QpDev* qp, unsigned long long w, const WqeView& v, uint8_t syn,
                                                   uint64_t src, uint64_t dst, uint64_t rq_idx, uint8_t rq_taken,
                                                   uint32_t* chunk_out = nullptr) {
  Resolved* r = qp->resolved + (w & ((1u << qp->sq_log) - 1));
  // Work granule: at least the QP's chunk_bytes, grown so that a very large message is cut
  // into ~8 claims per engine CTA (bounded claim traffic, still balances the tail).
  uint32_t chunk = qp->chunk_bytes;
  {
    uint32_t target = 8u * gridDim.x;
    uint32_t want = (uint32_t)(((uint64_t)v.bytes + target - 1) / target);
    want = (want + kSub - 1) / kSub * kSub;
    if (want > chunk) chunk = want;
  }
  uint32_t nchunks = (syn == SYN_OK && v.bytes > 0) ? (v.bytes + chunk - 1) / chunk : 1;
  r->chunk = chunk;
  if (chunk_out) *chunk_out = chunk;
  r->src = src; r->dst = dst;
  r->bytes = (syn == SYN_OK) ? v.bytes : 0;
  r->nchunks = nchunks;
  r->imm = v.imm;
  r->opcode = v.opcode; r->fm_ce_se = v.fm_ce_se; r->syndrome = syn; r->rq_consumed = rq_taken;
  r->rq_idx = rq_idx;
  r->done = 0;
  *(volatile unsigned long long*)&r->state = (w << 2) | 1ull;
  return nchunks;
}

// Receive matching: only ever executed by the turn holder, i.e. in WQE order.  May block
// (bounded by rnr_timeout_ns) on a receiver that has not posted a buffer yet -- which is
// exactly what RC does to the WQEs queued behind it.
__device__ __forceinline__ void match_recv(EngineCtl* ctl, QpDev* qp, const WqeView& v, uint8_t* syn, uint64_t* dst,
                                           uint64_t* rq_idx, uint8_t* rq_taken) {
  unsigned long long head = qp->rq_head;
  unsigned long long t0 = 0;
  // The responder's doorbell record and receive ring live wherever the responder does (another GPU
  // over NVLink: ~3 us per dependent read, and this runs inside the ordered section).  So the
  // producer count is cached and only re-read when the cache says "empty", and the receive WQE body
  // is only fetched when the opcode actually needs the buffer it names (SEND, not WRITE_IMM).
  bool have = head < qp->rq_cached_pi;
  while (!have) {
    uint32_t rpi16 = be32(ld_u32_volatile(&qp->r.rq_dbr[DBR_RCV])) & 0xffff;
    qp->rq_cached_pi = head + ((rpi16 - (uint32_t)head) & 0xffff);
    if (head < qp->rq_cached_pi) { have = true; break; }
    unsigned long long now = globaltimer_ns();
    if (t0 == 0) { t0 = now; atomicAdd(&qp->n_rnr, 1ull); }
    if (now - t0 > ctl->rnr_timeout_ns || *ctl->stop) break;
    __nanosleep(500);
  }
  if (!have) { *syn = SYN_RNR_RETRY_EXC_ERR; return; }
  if (v.opcode == OP_RDMA_WRITE_IMM) {       // consumes the slot, ignores its contents
    *rq_idx = head;
    *rq_taken = 1;
    qp->rq_head = head + 1;
    return;
  }
  fence_scope(qp->sys_scope != 0);
  const uint8_t* rs = qp->r.rq + ((head & ((1ull << qp->r.rq_log) - 1)) << 4);
  uint4 d = ld_v4_volatile(rs);
  uint32_t rbytes = be32(d.x) & 0x7fffffffu, rlkey = be32(d.y);
  uint64_t raddr = ((uint64_t)be32(d.z) << 32) | be32(d.w);
  *rq_idx = head;
  *rq_taken = 1;
  qp->rq_head = head + 1;
  if (rbytes < v.bytes) *syn = SYN_REMOTE_INVAL_REQ_ERR;
  else *dst = translate(qp->r.rkeys, qp->r.n_rkeys, rlkey, raddr, v.bytes, ACC_LOCAL_WRITE, true, syn);
}

// ------------------------------------------------------------------ retire
// Warp-collective, strictly in order, under the per-QP retire try-lock.  Lane i looks at WQE h + i: one
// round trip tells the warp how long the run of finished WQEs is (ballot), one more fetches every lane's
// record, lane 0 reserves the CQ slots of the whole run with ONE atomic per CQ (a remote CQ costs a link
// round trip), prefix popcounts hand each lane its slots, and every lane publishes its own CQEs: body,
// its own fence (acquire of the payload chain + release of the body), owner-bit tail.  A run of 32
// completions costs the same ~6 round trips as a run of one.  (The first version walked the run with
// dependent loads in one thread: ~0.85 us per WQE, which was the engine's message-rate ceiling.)
constexpr int kRetireBatch = 32;

__device__ __forceinline__ uint8_t recv_cqe_opcode(uint8_t opc, bool err) {
  return err ? CQE_RESP_ERR : (opc == OP_SEND ? CQE_RESP_SEND : (opc == OP_SEND_IMM ? CQE_RESP_SEND_IMM : CQE_RESP_WR_IMM));
}

// CQ overrun (what a ConnectX reports as a CQ error): the producer is about to wrap onto CQEs the consumer has
// not taken.  The consumer index is the consumer's doorbell record (be32, 24 bits) -- possibly host memory, a
// slow read -- so it is cached in the CqDev and only refreshed when the cached value says "full".
__device__ __forceinline__ bool cq_would_overrun(CqDev* cq, unsigned int end_pi, uint32_t log_n) {
  const unsigned int depth = 1u << log_n;
  unsigned int ci = *(volatile unsigned int*)&cq->ci_seen;
  if (end_pi - ci <= depth) return false;
  const unsigned int ci24 = be32(ld_u32_volatile(cq->dbrec)) & 0xffffffu;
  ci = end_pi - ((end_pi - ci24) & 0xffffffu);
  *(volatile unsigned int*)&cq->ci_seen = ci;
  return end_pi - ci > depth;
}

__device__ __forceinline__ void retire(QpDev* qp, uint32_t lane, unsigned long long w_finished) {
  const uint32_t mask = (1u << qp->sq_log) - 1;
  const bool sys = qp->sys_scope != 0;
  const uint32_t lt = (1u << lane) - 1;
  // The caller just finished WQE w_finished.  retire_word = (head << 1) | locked, so one CAS answers both
  // "is it this WQE's turn" and "did I get the lock".  A failed CAS needs no follow-up: either a holder
  // exists (it re-checks the head slot after unlocking) or an earlier WQE is still unfinished (its
  // finisher will find this one in its run).
  unsigned long long h = __shfl_sync(0xffffffffu, w_finished, 0);
  for (;;) {
    // the state words of the next 32 WQEs travel together with the lock attempt (a stale "not finished"
    // only shortens the run; the state names its own index, so it can never be stale-positive)
    unsigned long long st = ld_u64_volatile(&(qp->resolved + ((h + lane) & mask))->state);
    int locked = 0;
    if (lane == 0) locked = atomicCAS(&qp->retire_word, h << 1, (h << 1) | 1ull) == (h << 1);
    if (!__shfl_sync(0xffffffffu, locked, 0)) return;
    bool first = true;
    for (;;) {
      // ---- pass 1: the run of finished WQEs starting at the head (a lane that wrapped around a short ring
      //      sees a state word that names another index, i.e. "not mine")
      const unsigned long long w = h + lane;
      Resolved* r = qp->resolved + (w & mask);
      if (!first) st = ld_u64_volatile(&r->state);
      first = false;
      const bool fin = st == ((w << 2) | 2ull);
      const uint32_t finmask = __ballot_sync(0xffffffffu, fin);
      const int n = finmask == 0xffffffffu ? 32 : __ffs((int)~finmask) - 1;   // leading run
      if (n == 0) break;
      const bool active = (int)lane < n;
      // ---- pass 2: my record (only touched once its state said "finished")
      uint32_t bytes = 0, imm = 0;
      uint8_t opc = 0, syn = 0;
      bool want_recv = false, want_send = false;
      uint64_t rq_idx = 0;
      if (active) {
        const uint4 f = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r) + 16);   // bytes | nchunks | imm | opcode,fm_ce_se,syndrome,rq_consumed
        bytes = f.x; imm = f.z;
        opc = (uint8_t)f.w; syn = (uint8_t)(f.w >> 16);
        const uint8_t fm = (uint8_t)(f.w >> 8), rqc = (uint8_t)(f.w >> 24);
        want_recv = rqc && qp->r.rcq;
        want_send = syn != SYN_OK || (fm & CTRL_CQ_UPDATE);
        if (want_recv) rq_idx = ld_u64_volatile(&r->rq_idx);
      }
      const bool err = active && syn != SYN_OK;
      const uint32_t smask = __ballot_sync(0xffffffffu, want_send), rmask = __ballot_sync(0xffffffffu, want_recv);
      const int n_send = __popc(smask), n_recv = __popc(rmask);
      // ---- one slot reservation per CQ for the whole run
      CqDev* scq = qp->scq;
      unsigned int s_slot = 0, r_slot = 0;
      const uint32_t s_log = scq->log_n, r_log = qp->r.rcq ? qp->r.rcq->log_n : 0;
      int over = 0;
      if (lane == 0) {
        if (n_send) {
          s_slot = sys ? atomicAdd_system(&scq->pi, (unsigned)n_send) : atomicAdd(&scq->pi, (unsigned)n_send);
          if (cq_would_overrun(scq, s_slot + (unsigned)n_send, s_log)) over |= 1;
        }
        if (n_recv) {
          r_slot = atomicAdd_system(&qp->r.rcq->pi, (unsigned)n_recv);
          // the responder's consumer record is only addressable when its CQ was not re-mapped (same process)
          if ((qp->r.connected & 2u) && cq_would_overrun(qp->r.rcq, r_slot + (unsigned)n_recv, r_log)) over |= 2;
        }
        if (over) {
          if (over & 1) atomicAdd(&scq->overruns, 1u);
          if (over & 2) atomicAdd(&qp->r.rcq->overruns, 1u);
          qp->state = QPS_ERR;     // CQ error is fatal for the QPs attached to it; nothing more is written to the full ring
        }
      }
      over = __shfl_sync(0xffffffffu, over, 0);
      if (over & 1) want_send = false;
      if (over & 2) want_recv = false;
      s_slot = __shfl_sync(0xffffffffu, s_slot, 0) + __popc(smask & lt);
      r_slot = __shfl_sync(0xffffffffu, r_slot, 0) + __popc(rmask & lt);
      // ---- bodies, fence, tails: every lane for its own WQE
      if (want_recv) cqe_body(cqe_slot(qp->r.rcq_buf, r_log, r_slot), recv_cqe_opcode(opc, err), bytes, imm);
      if (want_send) cqe_body(cqe_slot(scq->buf, s_log, s_slot), err ? CQE_REQ_ERR : CQE_REQ, bytes, 0);
      if (want_recv || want_send) {
        fence_scope(sys);  // payload (cumulative over every chunk's release, observed through the state word) + body before the owner bit
        const unsigned long long now = globaltimer_ns();
        if (want_recv) cqe_tail(cqe_slot(qp->r.rcq_buf, r_log, r_slot), r_log, r_slot, recv_cqe_opcode(opc, err), 0, qp->r.qpn, (uint16_t)rq_idx, syn, now);
        if (want_send) {
          cqe_tail(cqe_slot(scq->buf, s_log, s_slot), s_log, s_slot, err ? CQE_REQ_ERR : CQE_REQ, opc, qp->qpn, (uint16_t)w, syn, now);
          trace_stamp(qp, w, TR_CQE);
        }
      }
      // ---- counters: fire-and-forget reductions (nobody waits for them, no stale-line hazard)
      unsigned long long run_bytes = bytes;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) run_bytes += __shfl_xor_sync(0xffffffffu, run_bytes, o);
      const uint32_t n_err = __popc(__ballot_sync(0xffffffffu, err));
      if (lane == 0) {
        if (n_send) atomicAdd(&qp->n_cqe, (unsigned long long)n_send);
        if (n_err) atomicAdd(&qp->n_err, (unsigned long long)n_err);
        atomicAdd(&qp->n_wqe, (unsigned long long)n);
        if (run_bytes) atomicAdd(&qp->n_bytes, run_bytes);
      }
      h += (unsigned)n;
      if (n < kRetireBatch) break;
    }
    __syncwarp();   // every lane's tails are ordered before lane 0's release below
    int again = 0;
    if (lane == 0) {
      *(volatile unsigned long long*)&qp->retire_head = h;   // for observers (idle detection, host queries)
      fence_gpu();  // release
      atomicExch(&qp->retire_word, h << 1);
      __threadfence();  // SC: unlock before re-checking the next slot (store-buffering pattern with finishers)
      again = ld_u64_volatile(&(qp->resolved + (h & mask))->state) == ((h << 2) | 2ull);
    }
    if (!__shfl_sync(0xffffffffu, again, 0)) return;
    h = __shfl_sync(0xffffffffu, h, 0);
  }
}

// ------------------------------------------------------------------ claim
struct Work {
  QpDev* qp;
  unsigned long long w;
  uint32_t chunk;
  // filled by a direct (single-WQE) claim, which has just computed them: saves re-reading resolved[w]
  uint32_t have_desc, len, nch;
  uint64_t src, dst;
};

// Draw one chunk from the ticket of the WQE in slot `res`.  `w_hint` is any index whose
// low 20 bits are close to the real one (used to rebuild the full index).
__device__ __forceinline__ bool draw_chunk(QpDev* qp, Resolved* res, unsigned long long w_hint, Work* out) {
  unsigned long long peek = ld_u64_volatile(&res->ticket);
  if ((uint32_t)(peek >> 40) >= (uint32_t)(peek & TICKET_FIELD_MASK)) return false;   // exhausted: no atomic
  unsigned long long t = atomicAdd(&res->ticket, (unsigned long long)TICKET_ONE);
  uint32_t c = (uint32_t)(t >> 40), gen = (uint32_t)((t >> TICKET_GEN_SHIFT) & TICKET_FIELD_MASK);
  uint32_t n = (uint32_t)(t & TICKET_FIELD_MASK);
  if (c >= n) return false;
  // the ticket names its own WQE (generation), so a draw on a recycled slot is still a
  // valid claim on whatever WQE lives there now
  long long delta = (long long)((gen - (uint32_t)w_hint) & TICKET_FIELD_MASK);
  if (delta >= (long long)(TICKET_FIELD_MASK + 1) / 2) delta -= (long long)(TICKET_FIELD_MASK + 1);
  fence_gpu();  // acquire: resolved[] fields of that generation
  out->qp = qp; out->w = (unsigned long long)((long long)w_hint + delta); out->chunk = c; out->have_desc = 0;
  return true;
}

// Returns 0: nothing, 1: *out is a chunk to move, 2: a BATCH of out->chunk WQEs starting at out->w was
// claimed and still has to be parsed (claim_batch, warp-collective).
constexpr uint32_t kClaimBatch = 16;
__device__ __forceinline__ int try_claim(EngineCtl* ctl, QpDev* qp, Work* out, bool* saw_pending, bool host_watcher) {
  const uint32_t st = qp->state;
  if (st != QPS_RTS && st != QPS_ERR) return 0;
  const bool sys = qp->sys_scope != 0;
  const uint32_t mask = (1u << qp->sq_log) - 1;
  // independent loads, one round trip (the doorbell of a host-resident queue is a PCIe read: only
  // the designated watcher pays it)
  const bool look_at_doorbell = !sys || host_watcher || qp->sq_in_device;
  unsigned long long c = ld_u64_volatile(&qp->cursor);
  unsigned long long db = look_at_doorbell ? ld_u64_volatile(qp->bf) : 0ull;
  unsigned long long off = ld_u64_volatile(&qp->offer);
  unsigned long long ps = ld_u64_volatile(&qp->parse_seq) & ~PARSE_ERR_BIT;
  uint32_t idx16 = (be32((uint32_t)db) >> 8) & 0xffff;
  uint32_t pending = look_at_doorbell ? ((idx16 + 1 - (uint32_t)c) & 0xffff) : 0u;
  if (pending != 0 && pending < 0x8000) {
    *saw_pending = true;
    // Every engine CTA races for the same word with a value it loaded one L2 round trip ago, so only
    // about one CAS per round trip wins (measured: 0.85 us per message however many CTAs run).  When a
    // backlog is visible the winner therefore takes several WQEs at once and parses them as a warp.
    const uint32_t take = pending < kClaimBatch ? pending : kClaimBatch;
    if (take > 1) {
      if (atomicCAS(&qp->cursor, c, c + take) == c) {
        fence_scope(sys);  // acquire: WQE bytes the doorbell announced
        out->qp = qp; out->w = c; out->chunk = take;
        return 2;
      }
    } else if (atomicCAS(&qp->cursor, c, c + 1) == c) {
      const unsigned long long w = c;
      fence_scope(sys);  // acquire: WQE bytes the doorbell announced
      trace_stamp(qp, w, TR_CLAIM);
      // ordering audit: the doorbell record must already cover what the register announced
      uint32_t dbr16 = be32(ld_u32_volatile(&qp->dbr[DBR_SND])) & 0xffff;
      if (((dbr16 - (uint32_t)w) & 0xffff) < pending && ((dbr16 - (uint32_t)w) & 0xffff) < 0x8000)
        atomicAdd(&qp->n_db_order_violations, 1ull);
      // ---- parallel part
      Parsed p;
      parse_wqe(qp, w, &p);
      const bool recv = p.syn == SYN_OK && needs_recv_wqe(p.v.opcode);
      uint32_t n = 1, chunk_sz = 0;
      uint64_t fsrc = p.src, fdst = p.dst;
      if (!recv) n = write_resolved(qp, w, p.v, p.syn, p.src, p.dst, 0, 0, &chunk_sz);
      // ---- ordered part: wait for the turn.  The turn word also carries "QP already failed",
      //      so the common path is one poll + one store, no fence.
      unsigned long long turn = ld_u64_volatile(&qp->parse_seq);
      if ((turn & ~PARSE_ERR_BIT) != w) {
        unsigned long long t0 = globaltimer_ns();
        while (((turn = ld_u64_volatile(&qp->parse_seq)) & ~PARSE_ERR_BIT) != w) {
          if (globaltimer_ns() - t0 > 4000000000ull) { ctl->fatal = 2; break; }   // predecessor died
        }
      }
      bool err = (turn & PARSE_ERR_BIT) != 0 || st == QPS_ERR;
      uint8_t syn = p.syn;
      if (err) {
        // flushed: nothing moves, whatever the parse said
        syn = SYN_WR_FLUSH_ERR;
        n = write_resolved(qp, w, p.v, syn, 0, 0, 0, 0, &chunk_sz);
      } else if (recv) {
        fence_gpu();  // acquire rq_head from the previous receive-consuming WQE
        uint64_t dst = p.dst, rq_idx = 0;
        uint8_t rq_taken = 0;
        match_recv(ctl, qp, p.v, &syn, &dst, &rq_idx, &rq_taken);
        n = write_resolved(qp, w, p.v, syn, p.src, dst, rq_idx, rq_taken, &chunk_sz);
        fdst = dst;
        fence_gpu();  // release rq_head
      }
      if (syn != SYN_OK && !err) { qp->state = QPS_ERR; err = true; }
      Resolved* res = qp->resolved + (w & mask);
      const unsigned long long next = (w + 1) | (err ? (unsigned long long)PARSE_ERR_BIT : 0ull);
      if (n > 1) {
        fence_gpu();  // release resolved[w] before the ticket that lets helpers read it
        st_u64_relaxed(&res->ticket, TICKET_ONE | ((w & TICKET_FIELD_MASK) << TICKET_GEN_SHIFT) | n);
        st_u64_release_scope(&qp->parse_seq, next, false);   // helpers trust: committed => ticket armed
      } else {
        st_u64_relaxed(&qp->parse_seq, next);
      }
      trace_stamp(qp, w, TR_PARSED);
      out->qp = qp; out->w = w; out->chunk = 0;
      {
        const uint32_t bytes = syn == SYN_OK ? p.v.bytes : 0;
        out->have_desc = 1; out->nch = n; out->src = fsrc; out->dst = fdst;
        out->len = bytes < chunk_sz ? bytes : chunk_sz;     // chunk 0
      }
      return 1;
    }
  }
  // ---- help.  The tickets of the 8 oldest committed WQEs are peeked with independent loads (one round
  // trip).  Retirement is in order, so the head WQE's chunks matter most: a WQE with many chunks left
  // absorbs every CTA; a run of single-chunk WQEs (a parsed batch) is spread over the CTAs by block index
  // instead of all of them hammering the oldest ticket.
  if (off < ps) {
    const uint32_t cnt = (ps - off) < 8 ? (uint32_t)(ps - off) : 8u;
    unsigned long long t[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) t[k] = (uint32_t)k < cnt ? ld_u64_volatile(&(qp->resolved + ((off + k) & mask))->ticket) : 0ull;
    uint32_t avail[8], total = 0, lead = 0;
    bool leading = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const bool mine = (uint32_t)((t[k] >> TICKET_GEN_SHIFT) & TICKET_FIELD_MASK) == (uint32_t)((off + k) & TICKET_FIELD_MASK);
      const uint32_t cc = (uint32_t)(t[k] >> 40), nn = (uint32_t)(t[k] & TICKET_FIELD_MASK);
      avail[k] = ((uint32_t)k < cnt && mine && cc < nn) ? nn - cc : 0u;   // single-chunk WQE taken by its claimer, or fully drawn: 0
      total += avail[k];
      if (leading && (uint32_t)k < cnt && avail[k] == 0) ++lead; else leading = false;
    }
    if (lead) atomicMax(&qp->offer, off + lead);
    if (total) {
      *saw_pending = true;
      uint32_t pick = blockIdx.x % (total < gridDim.x ? total : gridDim.x), sel = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (pick < avail[k]) { sel = k; break; }
        pick -= avail[k];
      }
      if (draw_chunk(qp, qp->resolved + ((off + sel) & mask), off + sel, out)) return 1;
    }
  }
  if (ld_u64_volatile(&qp->retire_head) != c) *saw_pending = true;   // work in flight somewhere
  return 0;
}

// Warp-collective: parse and commit the `k` WQEs [w0, w0 + k) that lane 0 claimed with one CAS.
// Lane i parses WQE w0 + i (the round trips for the WQE bytes and both MKeys overlap across lanes);
// the ordered section is entered ONCE for the batch -- lane 0 waits for the turn, lanes commit one after
// another (receive matching, error flush), one fence publishes everything and one store passes the turn
// k WQEs on.  Every WQE gets a ticket that starts at chunk 0: nobody owns any of them, all engine CTAs
// (this one included) draw the chunks through the normal oldest-first offer path.
__device__ __forceinline__ void claim_batch(EngineCtl* ctl, QpDev* qp, unsigned long long w0, uint32_t k, uint32_t lane) {
  const uint32_t mask = (1u << qp->sq_log) - 1;
  const unsigned long long w = w0 + lane;
  Parsed p;
  uint32_t n = 1;
  bool recv = false;
  if (lane < k) {
    trace_stamp(qp, w, TR_CLAIM);
    parse_wqe(qp, w, &p);
    recv = p.syn == SYN_OK && needs_recv_wqe(p.v.opcode);
    if (!recv) n = write_resolved(qp, w, p.v, p.syn, p.src, p.dst, 0, 0);
  }
  __syncwarp();
  unsigned long long turn = 0;
  if (lane == 0) {
    turn = ld_u64_volatile(&qp->parse_seq);
    if ((turn & ~PARSE_ERR_BIT) != w0) {
      unsigned long long t0 = globaltimer_ns();
      while (((turn = ld_u64_volatile(&qp->parse_seq)) & ~PARSE_ERR_BIT) != w0) {
        if (globaltimer_ns() - t0 > 4000000000ull) { ctl->fatal = 2; break; }   // predecessor died
      }
    }
  }
  turn = __shfl_sync(0xffffffffu, turn, 0);
  int err = ((turn & PARSE_ERR_BIT) != 0 || *(volatile uint32_t*)&qp->state == QPS_ERR) ? 1 : 0;
  for (uint32_t i = 0; i < k; ++i) {
    if (lane == i) {
      uint8_t syn = p.syn;
      if (err) {
        syn = SYN_WR_FLUSH_ERR;
        n = write_resolved(qp, w, p.v, syn, 0, 0, 0, 0);
      } else if (recv) {
        fence_gpu();  // acquire rq_head from the previous receive-consuming WQE
        uint64_t dst = p.dst, rq_idx = 0;
        uint8_t rq_taken = 0;
        match_recv(ctl, qp, p.v, &syn, &dst, &rq_idx, &rq_taken);
        n = write_resolved(qp, w, p.v, syn, p.src, dst, rq_idx, rq_taken);
      }
      if (syn != SYN_OK && !err) { qp->state = QPS_ERR; err = 1; }
      Resolved* res = qp->resolved + (w & mask);
      st_u64_relaxed(&res->ticket, ((w & TICKET_FIELD_MASK) << TICKET_GEN_SHIFT) | n);    // chunk counter starts at 0
      trace_stamp(qp, w, TR_PARSED);
    }
    __syncwarp();
    err = __shfl_sync(0xffffffffu, err, i);
  }
  if (lane == 0) {
    fence_gpu();  // release: every lane's resolved[] / ticket / rq_head (ordered before this by the __syncwarp chain)
    st_u64_release_scope(&qp->parse_seq, (w0 + k) | (err ? (unsigned long long)PARSE_ERR_BIT : 0ull), false);
  }
}

// ------------------------------------------------------------------ the kernel
__global__ void __launch_bounds__(kThreads, 1) engine_kernel(EngineCtl* ctl) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  __shared__ Work work, next_work;   // next_work: the following chunk of the same WQE, drawn by a second thread while this one is copied
  __shared__ int quit, next_valid;
  if (threadIdx.x == 0) {
    next_valid = 0;
    for (int i = 0; i < kStages; ++i) mbar_init(&s.full[i], 1);
    s.phase_bits = 0;
    quit = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    atomicAdd(&ctl->running_ctas, 1u);
    if (blockIdx.x == 0) ctl->t_start = globaltimer_ns();
  }
  __syncthreads();
  unsigned long long last_activity = globaltimer_ns();
  uint32_t rr = blockIdx.x;
  unsigned spins = 0;
  QpDev* sticky_qp = nullptr;        // multi-chunk WQE this CTA last worked on: keep drawing from it
  unsigned long long sticky_w = 0;
  // Host-resident queues are polled for NEW work by one designated CTA only.  A GPU load from pinned
  // host memory costs tens of microseconds on this platform; when every CTA paid it in every sweep, a
  // device-resident QP sharing the engine saw its latency go from 11 us to 85 us, and 96 CTAs polling
  // over PCIe starved a concurrent cudaMemcpy (0.9 GB/s).  Helping with an already-parsed WQE only
  // touches device memory, so everybody still does that.
  const bool host_watcher = blockIdx.x == gridDim.x - 1;
  uint32_t n_qps_cached = ctl->n_qps;
  unsigned iter = 0, rot = blockIdx.x;
  for (;;) {
    int batch_k = 0;
    if (threadIdx.x == 0) {
      s.have_work = 0;
      // "everybody leaves" travels with the queue scan (its latency hides behind try_claim's loads); the QP
      // count is re-read every 64 iterations together with the fence that drops stale L1 lines, so host-side
      // updates (new QPs, reconnects) become visible within ~100 us without a dependent load per iteration
      const unsigned quit_all_seen = *(volatile unsigned int*)&ctl->quit_all;
      if ((iter++ & 63u) == 0) { fence_gpu(); n_qps_cached = ctl->n_qps; }
      const uint32_t n = n_qps_cached;
      bool pending = false;
      if (next_valid) {              // drawn (and therefore owed) during the previous chunk's copy
        work = next_work;
        next_valid = 0;
        s.have_work = 1;
      } else if (sticky_qp) {
        Resolved* sr = sticky_qp->resolved + (sticky_w & ((1u << sticky_qp->sq_log) - 1));
        // a successful draw is a claim that MUST be executed, whichever generation it names
        if (draw_chunk(sticky_qp, sr, sticky_w, &work)) s.have_work = 1;
        else sticky_qp = nullptr;
      }
      // Every probe of a QP is at least one L2 round trip, so a CTA does not walk the whole table each
      // iteration (with 8 QPs registered, one active QP ran at half its solo message rate): it looks at the QP
      // that last gave it work and at ONE other, rotating.  CTAs start at different offsets, so every QP is
      // still probed by many CTAs per round trip.  The host watcher keeps the full scan: it alone decides
      // "idle" / "drained" and it is the only one that reads host-resident doorbells.
      const uint32_t n_scan = host_watcher ? n : (n < 2 ? n : 2u);
      for (uint32_t k = 0; k < n_scan && !s.have_work && !batch_k; ++k) {
        const uint32_t qi = (host_watcher || k == 0) ? (rr + k) % n : (rr + 1 + rot % (n - 1)) % n;
        QpDev* qp = *(QpDev* volatile*)&ctl->qps[qi];   // table grows while we run
        if (!qp) continue;
        const int got = try_claim(ctl, qp, &work, &pending, host_watcher);
        if (got == 1) s.have_work = 1;
        else if (got == 2) { batch_k = (int)work.chunk; pending = true; }
        if (got) rr = qi;
      }
      ++rot;
      if (s.have_work) {
        if (work.have_desc) {
          s.len = work.len; s.src = work.src; s.dst = work.dst; s.nch = work.nch;
        } else {
          Resolved* r = work.qp->resolved + (work.w & ((1u << work.qp->sq_log) - 1));
          const uint4 f = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r) + 16);   // bytes | nchunks | imm | flags
          const uint4 a = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r));        // src | dst
          const uint32_t chunk = *(volatile uint32_t*)&r->chunk;
          const uint64_t off = (uint64_t)work.chunk * chunk;
          const uint32_t bytes = f.x;
          s.len = bytes == 0 ? 0 : (uint32_t)((bytes - off < chunk) ? (bytes - off) : chunk);
          s.src = (((uint64_t)a.y << 32) | a.x) + off;
          s.dst = (((uint64_t)a.w << 32) | a.z) + off;
          s.nch = f.y;
        }
        if (s.nch > 1) { sticky_qp = work.qp; sticky_w = work.w; }
        last_activity = globaltimer_ns();
        spins = 0;
      } else {
        ++spins;
        // The host watcher is the only CTA that sees host-resident doorbells, so it alone may declare
        // the engine idle or drained; everybody else follows quit_all.
        if (pending) last_activity = globaltimer_ns();
        else if (host_watcher && ctl->oneshot && spins > 4) { quit = 1; ctl->quit_all = 1; }   // drained: every posted WQE has retired
        if (quit_all_seen) quit = 1;
        if ((spins & 63) == 0) {
          if (*ctl->stop) quit = 1;   // mapped host word: a PCIe read, hence only every 64 idle spins
          else if (host_watcher && globaltimer_ns() - last_activity > ctl->idle_timeout_ns) { quit = 1; ctl->exited_idle = 1; ctl->quit_all = 1; }
        }
        if (spins > 256) __nanosleep(200);
      }
    }
    if (threadIdx.x < 32) {
      // a batch claim is parsed by the whole first warp; its chunks are then drawn like anybody else's
      batch_k = __shfl_sync(0xffffffffu, batch_k, 0);
      if (batch_k) {
        // only lane 0 reads the (shared-memory) work record it wrote; the other lanes' operand is ignored by the shuffle
        unsigned long long wq0 = 0, ww0 = 0;
        if (threadIdx.x == 0) { wq0 = (unsigned long long)*(QpDev* volatile*)&work.qp; ww0 = *(volatile unsigned long long*)&work.w; }
        QpDev* bqp = (QpDev*)__shfl_sync(0xffffffffu, wq0, 0);
        unsigned long long bw = __shfl_sync(0xffffffffu, ww0, 0);
        claim_batch(ctl, bqp, bw, (uint32_t)batch_k, threadIdx.x);
      }
    }
    __syncthreads();
    const int q = quit, hw = s.have_work;
    const uint32_t len = s.len;
    const uint64_t csrc = s.src, cdst = s.dst;
    __syncthreads();  // every thread holds the broadcast in registers before thread 0 reuses smem
    if (q) break;
    if (!hw) continue;
    if (len > 0) {
      const bool bulk = len >= kBulkMin && (((csrc | cdst) & 15) == 0) && ((len & 15) == 0);
      if (bulk && threadIdx.x == 32 && s.nch > 1) {
        // While thread 0 runs the copy pipeline, draw the NEXT chunk of the same WQE and fetch its descriptor:
        // takes the ticket round trips, the fence and the descriptor loads (~2 us) off the per-chunk path.
        Work nw;
        if (draw_chunk(work.qp, work.qp->resolved + (work.w & ((1u << work.qp->sq_log) - 1)), work.w, &nw)) {
          Resolved* r2 = nw.qp->resolved + (nw.w & ((1u << nw.qp->sq_log) - 1));   // the ticket names its own WQE
          const uint4 f = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r2) + 16);
          const uint4 a = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r2));
          const uint32_t chunk = *(volatile uint32_t*)&r2->chunk;
          const uint64_t off = (uint64_t)nw.chunk * chunk;
          nw.have_desc = 1;
          nw.len = f.x == 0 ? 0 : (uint32_t)((f.x - off < chunk) ? (f.x - off) : chunk);
          nw.src = (((uint64_t)a.y << 32) | a.x) + off;
          nw.dst = (((uint64_t)a.w << 32) | a.z) + off;
          nw.nch = f.y;
          next_work = nw;
          next_valid = 1;
        }
      }
      if (bulk) {
        if (threadIdx.x == 0) {
          const unsigned sif = ctl->stores_in_flight;
          const bool okc = sif == 8 ? copy_bulk<8>(s, csrc, cdst, len) : (sif == 6 ? copy_bulk<6>(s, csrc, cdst, len) : copy_bulk<4>(s, csrc, cdst, len));
          if (!okc) { ctl->fatal = 1; quit = 1; }
          atomicAdd(&ctl->n_bulk_chunks, 1ull);
        }
      } else {
        copy_generic(csrc, cdst, len);
      }
    }
    __syncthreads();
    if (quit) break;   // fatal DMA fault: leave without completing (host sees ctl->fatal)
    int finished = 0;
    if (threadIdx.x == 0) {
      QpDev* qp = work.qp;
      Resolved* r = qp->resolved + (work.w & ((1u << qp->sq_log) - 1));
      // This chunk's bytes before the count that may complete the WQE.  gpu scope is enough even
      // when the CQ or the payload lives in host / peer memory: the retirer's system-scope
      // fence in write_cqe() is cumulative over everything this chain of gpu-scope releases made
      // visible to it (a sys fence per chunk cost ~2x on host-resident queues, measured).
      const uint32_t nch = s.nch;
      if (nch > 1) fence_gpu();   // this chunk's bytes before the count that may complete the WQE
      if (nch == 1 || atomicAdd(&r->done, 1u) + 1 == nch) {
        trace_stamp(qp, work.w, TR_COPIED);
        fence_gpu();  // single chunk: its bytes before "finished"; else observe every other chunk's count -> their bytes precede our CQE
        *(volatile unsigned long long*)&r->state = (work.w << 2) | 2ull;
        __threadfence();  // SC: "finished" store before the retire try-lock (pairs with the unlock / re-check below)
        finished = 1;
      }
    }
    if (threadIdx.x < 32) {
      if (__shfl_sync(0xffffffffu, finished, 0)) {
        unsigned long long wq0 = 0, ww0 = 0;
        if (threadIdx.x == 0) { wq0 = (unsigned long long)*(QpDev* volatile*)&work.qp; ww0 = *(volatile unsigned long long*)&work.w; }
        retire((QpDev*)__shfl_sync(0xffffffffu, wq0, 0), threadIdx.x, ww0);
      }
    }
  }
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) ctl->t_exit = globaltimer_ns();
    atomicSub(&ctl->running_ctas, 1u);
  }
}

inline size_t engine_smem_bytes() { return sizeof(Smem) + 128; }

}  // namespace eng
}  // namespace rn
