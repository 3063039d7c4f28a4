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
//            thread fed by a chunk queue so it streams across chunk boundaries, mbarrier-tracked,
//            no LSU traffic); a multi-chunk WQE is offered to idle CTAs through a fetch-add
//            ticket, its owner keeps drawing from it too
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
#include "kernels/sm90.cuh"

namespace rn {
namespace eng {

using namespace rn::dev;
using namespace rn::sm90;

constexpr int kThreads = 128;
constexpr uint32_t kSub = 16384;        // bytes per TMA bulk transaction
constexpr int kStages = 12;             // smem ring: 12 x 16 KiB
// Ring split: kSif stages may hold a TMA store that is still reading smem, the other kStages - kSif hold loads in flight.
// 10 loads + 2 stores: as fast as 1 or 3 stores, faster than 4 (DESIGN.md 3.1).
constexpr int kSif = 2;
constexpr uint32_t kBulkMin = 4096;     // below this the generic path is as fast
// A queued chunk of at most this many bytes is waited for before control scans again (DESIGN.md 3.1).
constexpr uint32_t kSmallChunk = 64 * 1024;

// ------------------------------------------------------------------ PTX helpers (the rest are sm90's)
// try_wait without a suspend-time hint (sm90::mbar_try passes one)
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          s32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(s32(bar))
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(s32(smem_src)), "r"(bytes)
               : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

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
  const uint4 mid = encode_cqe_mid(opcode, byte_cnt, imm);
  st_v4(cqe + 0, 0u, 0u, 0u, 0u);
  st_v4(cqe + 16, 0u, 0u, 0u, 0u);
  st_v4(cqe + CQE_MID_OFF, mid.x, mid.y, mid.z, mid.w);
}
// The engine's vendor syndrome is 0.
__device__ __forceinline__ void cqe_tail(uint8_t* cqe, uint32_t log_n, unsigned int slot, uint8_t opcode, uint8_t wqe_opcode,
                                         uint32_t qpn, uint16_t wqe_counter, uint8_t syndrome, unsigned long long now) {
  const uint4 t = encode_cqe_tail(opcode, (uint8_t)((slot >> log_n) & 1u), wqe_counter, qpn, wqe_opcode, syndrome, 0, now);
  st_v4(cqe + CQE_TAIL_OFF, t.x, t.y, t.z, t.w);
}

// ------------------------------------------------------------------ chunk copy
// An engine CTA is split by role.  Warp 0 is control: it finds, claims and parses work, hands bulk chunks to the mover
// through a small queue and does each chunk's completion accounting.  One lane of warp 1 is the mover: it runs ONE TMA
// pipeline over that queue, so the ring keeps streaming across chunk boundaries.  Warps 0, 2 and 3 run the generic
// (unaligned / small) copies.
constexpr int kQueue = 3;                // chunk descriptors between control and the mover
constexpr uint32_t kQuitLen = 0xffffffffu;
constexpr uint32_t kGenericThreads = kThreads - 32;   // warps 0, 2, 3

struct Chunk { uint64_t src, dst; uint32_t len; };   // len == kQuitLen: the mover leaves
struct Owed { QpDev* qp; unsigned long long w; uint32_t nch; };   // control's record of a queued chunk

struct Smem {
  alignas(128) uint8_t ring[kStages][kSub];
  alignas(8) uint64_t full[kStages];     // ring stage landed (TMA complete_tx)
  uint64_t qfull[kQueue];                // control -> mover: entry holds a chunk
  uint64_t qdone[kQueue];                // mover -> control: that chunk's bulk stores are complete; entry free
  Chunk q[kQueue];
  Owed owed[kQueue];                     // control only
  uint32_t end[kQueue];                  // mover only: store groups committed up to and including the chunk's last
  uint64_t gsrc, gdst;                   // generic copy, control -> warps 2, 3
  uint32_t glen;
  int gquit;
  int mover_fatal;
};

__device__ __forceinline__ void init_barriers(Smem& s) {
  for (int i = 0; i < kStages; ++i) mbar_init(&s.full[i], 1);
  for (int i = 0; i < kQueue; ++i) { mbar_init(&s.qfull[i], 1); mbar_init(&s.qdone[i], 1); }
  s.gquit = 0;
  s.mover_fatal = 0;
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Non-blocking probe (try_wait may suspend the thread for a while; a probe between other work must not).
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void generic_bar() { asm volatile("bar.sync 1, %0;" ::"n"(kGenericThreads) : "memory"); }

// The mover (one thread): kStages - kSif loads and kSif stores in flight, one store group per 16 KiB step.  (With a
// single store in flight every step exposed the store's smem-read latency, ~0.35 us, which capped a CTA near 45 GB/s.)
// Loads for the next queued chunk are issued as ring stages free up, while the current chunk's stores are still in
// flight.  A chunk is written once kSif groups have been committed after its last store: that step waits for the full
// completion (wait_group kSif) instead of the smem read, then reports the chunk to control (mbarrier arrive: release at
// CTA scope).  No fence here: control's gpu-scope fence is cumulative over what this hand-off carries (DESIGN.md 3.1).
// When nothing more is queued the ring drains at once (wait_group 0), so a lone chunk is not held back waiting for work.
// Chunks need 16-byte aligned src, dst and len.  Returns false when a load never landed (bad mapping: bounded, the SM is
// not wedged); true when control queued the quit entry.
// kProf: add %globaltimer ns per wait to prof[MoverProf] (this CTA's row), written once on exit.
template <bool kProf>
__device__ __noinline__ bool move_chunks(Smem& s, unsigned long long* prof) {
  constexpr uint32_t P = kStages - kSif;
  uint32_t ring_ph = 0, q_ph = 0;            // parity of the next wait, per ring stage / per queue entry
  uint32_t n_ld = 0, n_st = 0;               // steps loaded / stored (= store groups committed)
  uint32_t ld_limit = kStages;               // loads below this index have a free stage
  int ld_stage = 0, st_stage = 0, e_ld = 0, e_st = 0, e_wr = 0;
  uint32_t ld_off = 0, st_off = 0, ld_len = 0, st_len = 0;
  uint64_t ld_src = 0, st_dst = 0;
  int unwritten = 0;                         // chunks whose stores are all issued, not yet reported
  bool ld_have = false, quit = false;
  unsigned long long acc[MOVER_PROF_N] = {}, t_in = 0, t_idle = 0;   // kProf only
  if constexpr (kProf) t_in = globaltimer_ns();
  auto stamp = [&]() -> unsigned long long { return kProf ? globaltimer_ns() : 0ull; };
  auto charge = [&](int b, unsigned long long t0) { if constexpr (kProf) acc[b] += globaltimer_ns() - t0; };
  auto leave = [&](bool ok) {
    if constexpr (kProf) {
      acc[MP_TOTAL] = globaltimer_ns() - t_in;
      for (int b = 0; b < MOVER_PROF_N; ++b) prof[b] = acc[b];
    }
    return ok;
  };
  auto next_stage = [](int i) { return i + 1 == kStages ? 0 : i + 1; };
  auto next_entry = [](int i) { return i + 1 == kQueue ? 0 : i + 1; };
  auto report = [&](bool all) {
    const unsigned long long t0 = stamp();
    do {
      mbar_arrive(&s.qdone[e_wr]);
      e_wr = next_entry(e_wr);
      if constexpr (kProf) ++acc[MP_CHUNKS];
    } while (--unwritten && (all || n_st - s.end[e_wr] >= (uint32_t)kSif));
    charge(MP_REPORT, t0);
  };
  for (;;) {
    if (!ld_have && !quit) {
      // idle (nothing in the ring, nothing owed): this wait may suspend; otherwise only probe
      const bool idle = n_st == n_ld && unwritten == 0;
      const uint32_t par = (q_ph >> e_ld) & 1u;
      if constexpr (kProf) if (idle && !t_idle) t_idle = globaltimer_ns();
      if (idle ? mbar_try_wait(&s.qfull[e_ld], par) : mbar_test_wait(&s.qfull[e_ld], par)) {
        q_ph ^= 1u << e_ld;
        ld_len = s.q[e_ld].len;
        if (ld_len == kQuitLen) quit = true;
        else { ld_have = true; ld_src = s.q[e_ld].src; ld_off = 0; }
        if constexpr (kProf) if (t_idle) { charge(MP_QFULL_IDLE, t_idle); t_idle = 0; }
      }
    }
    while (ld_have && n_ld - n_st < P) {
      if ((int32_t)(n_ld - ld_limit) >= 0) {
        // the stage of load n_ld was last read by store n_ld - kStages <= n_st - 1 - kSif
        const unsigned long long t0 = stamp();
        bulk_wait_read<kSif>();
        charge(MP_WAIT_READ, t0);
        ld_limit = n_st + P;
      }
      const uint32_t len = ld_len - ld_off < kSub ? ld_len - ld_off : kSub;
      mbar_expect_tx(&s.full[ld_stage], len);
      bulk_g2s(s.ring[ld_stage], (const void*)(ld_src + ld_off), len, &s.full[ld_stage]);
      ++n_ld;
      ld_stage = next_stage(ld_stage);
      ld_off += len;
      if (ld_off == ld_len) { ld_have = false; e_ld = next_entry(e_ld); }
    }
    if (n_st != n_ld) {
      const uint32_t par = (ring_ph >> st_stage) & 1u;
      if (!mbar_try_wait(&s.full[st_stage], par)) {
        const unsigned long long t0 = globaltimer_ns();
        while (!mbar_try_wait(&s.full[st_stage], par))
          if (globaltimer_ns() - t0 > 1000000000ull) return leave(false);
        charge(MP_FULL, t0);
      }
      ring_ph ^= 1u << st_stage;
      if (st_off == 0) { st_dst = s.q[e_st].dst; st_len = s.q[e_st].len; }
      const uint32_t len = st_len - st_off < kSub ? st_len - st_off : kSub;
      bulk_s2g((void*)(st_dst + st_off), s.ring[st_stage], len);
      bulk_commit();
      ++n_st;
      st_stage = next_stage(st_stage);
      st_off += len;
      if (st_off == st_len) { s.end[e_st] = n_st; e_st = next_entry(e_st); st_off = 0; ++unwritten; }
      if (unwritten && n_st - s.end[e_wr] >= (uint32_t)kSif) {
        const unsigned long long t0 = stamp();
        bulk_wait<kSif>();   // this step only: every group but the last kSif has landed in global memory
        charge(MP_CHUNK_WAIT, t0);
        ld_limit = n_st + P;
        report(false);
      }
    } else if (unwritten && !ld_have) {
      const unsigned long long t0 = stamp();
      bulk_wait<0>();        // the queue ran dry: finish now
      charge(MP_DRY_WAIT, t0);
      ld_limit = n_st + P;
      report(true);
    } else if (quit && !unwritten) {
      return leave(true);
    }
  }
}

// The profiled mover when EngineCtl::mover_prof is set.
__device__ __forceinline__ bool run_mover(Smem& s, unsigned long long* prof) {
  return prof ? move_chunks<true>(s, prof) : move_chunks<false>(s, nullptr);
}

// Generic path: any alignment; thread t of the n threads of warps 0, 2 and 3.
__device__ __forceinline__ void copy_generic(uint64_t src, uint64_t dst, uint32_t len, uint32_t t, uint32_t n) {
  const uint8_t* s = (const uint8_t*)src;
  uint8_t* d = (uint8_t*)dst;
  if ((((src ^ dst) & 15) == 0) && len >= 64) {
    uint32_t head = (uint32_t)((16 - (src & 15)) & 15);
    if (head > len) head = len;
    for (uint32_t i = t; i < head; i += n) d[i] = s[i];
    uint32_t body = (len - head) & ~15u;
    const uint4* s4 = (const uint4*)(s + head);
    uint4* d4 = (uint4*)(d + head);
    for (uint32_t i = t; i < body / 16; i += n) d4[i] = s4[i];
    for (uint32_t i = head + body + t; i < len; i += n) d[i] = s[i];
  } else {
    for (uint32_t i = t; i < len; i += n) d[i] = s[i];
  }
}

// ------------------------------------------------------------------ parse + commit
struct Parsed {
  WqeView v;
  uint64_t src, dst;
  uint64_t local1;        // two-entry WQE: entry 1, translated
  uint8_t syn;
};

// A clean two-entry WQE that moves bytes: its chunks map through the slot's SgSide record.
__device__ __forceinline__ bool is_sg(const WqeView& v, uint8_t syn) { return v.nsge == 2 && syn == SYN_OK && v.bytes != 0; }

// Keys of a two-entry WQE (its total already passed the MAX_MSG check): each local entry over its own range, in list
// order, with `lneed`; then, unless it is a SEND (whose remote side is the receive matched at commit), the remote key over
// the whole message with `rneed`.  The three entries are loaded back to back (one round trip).  Returns the remote side;
// *local0 and p->local1 receive the translated entries.
__device__ __forceinline__ uint64_t parse_sg_keys(const QpDev* qp, Parsed* p, uint32_t lneed, uint32_t rneed, bool remote,
                                                  uint64_t* local0) {
  const WqeView& v = p->v;
  const MKeyRaw l0 = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), l1 = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey1);
  const MKeyRaw rk = remote ? mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey) : MKeyRaw{};
  *local0 = mkey_check(l0, v.lkey, v.laddr, v.len0, lneed, false, &p->syn);
  if (*local0) p->local1 = mkey_check(l1, v.lkey1, v.laddr1, v.bytes - v.len0, lneed, false, &p->syn);
  if (!p->local1 || !remote) return 0;
  return mkey_check(rk, v.rkey, v.raddr, v.bytes, rneed, true, &p->syn);
}

// Atomic (CS / FA): both keys are checked here, nothing is moved; the retirer executes it in WQE order
// (retire_atomics).  On success src = target word, dst = local fetch buffer, v.imm = RESOLVED_ATOMIC_* flags
// and v.bytes = 0 (no chunks).
__device__ __forceinline__ void parse_atomic(const EngineCtl* ctl, const QpDev* qp, Parsed* p) {
  WqeView& v = p->v;
  const MKeyRaw lk = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), rk = mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey);
  if (v.bytes != 8) {
    p->syn = SYN_LOCAL_LENGTH_ERR;
  } else {
    p->dst = mkey_check(lk, v.lkey, v.laddr, 8, ACC_LOCAL_WRITE, false, &p->syn);
    if (p->dst && (v.raddr & 7)) p->syn = SYN_REMOTE_INVAL_REQ_ERR;
    else if (p->dst) p->src = mkey_check(rk, v.rkey, v.raddr, 8, ACC_REMOTE_ATOMIC, true, &p->syn);
    // A GPU atomic on pinned host memory is only atomic with respect to the CPU where the platform says so.
    if (p->src && rk.c.y == MEM_HOST_PINNED && !ctl->host_native_atomics) p->syn = SYN_REMOTE_OP_ERR;
    const bool sys = rk.c.y != MEM_DEVICE || lk.c.y != MEM_DEVICE || qp->sys_scope != 0;
    v.imm = sys ? RESOLVED_ATOMIC_SYS : 0u;
  }
  if (p->syn != SYN_OK) p->src = p->dst = 0;
  v.bytes = 0;
}

// Parallel part: runs concurrently for neighbouring WQEs of the same QP.
__device__ __forceinline__ void parse_wqe(const EngineCtl* ctl, QpDev* qp, unsigned long long w, Parsed* p) {
  const uint32_t mask = (1u << qp->sq_log) - 1;
  const uint8_t* slot = qp->sq + ((w & mask) << 6);
  Wqe64 wqe;
  uint4* wv = reinterpret_cast<uint4*>(&wqe);
  wv[0] = ld_v4_volatile(slot);
  wv[1] = ld_v4_volatile(slot + 16);
  wv[2] = ld_v4_volatile(slot + 32);
  wv[3] = ld_v4_volatile(slot + 48);
  p->syn = SYN_OK;
  p->src = p->dst = p->local1 = 0;
  bool ok = decode_wqe(&wqe, &p->v);
  WqeView& v = p->v;
  if (!ok || v.qpn != qp->qpn || v.wqe_idx != (uint16_t)w) {
    p->syn = SYN_LOCAL_QP_OP_ERR;
  } else if (!qp->r.connected && v.opcode != OP_NOP) {
    p->syn = SYN_LOCAL_QP_OP_ERR;
  } else if (v.bytes > MAX_MSG) {
    // over-long message, before any key is looked at (DESIGN.md 3.1); a NOP decodes to 0 bytes and an atomic of more
    // than 8 bytes fails with this syndrome anyway
    p->syn = SYN_LOCAL_LENGTH_ERR;
  } else {
    switch (v.opcode) {
      case OP_NOP: v.bytes = 0; break;
      case OP_RDMA_WRITE:
      case OP_RDMA_WRITE_IMM: {
        if (v.bytes == 0) { p->src = p->dst = 1; break; }   // zero length: no key is looked at, nothing moves (DESIGN.md 3.1)
        if (v.inl_off) {
          // Inline: only the remote key is checked, and the source is the payload in this SQ slot.  It is read after
          // commit (a flushed WQE copies nothing), and the slot is not reused before the WQE retires (DESIGN.md 3.1).
          p->dst = translate(qp->r.rkeys, qp->r.n_rkeys, v.rkey, v.raddr, v.bytes, ACC_REMOTE_WRITE, true, &p->syn);
          if (p->dst) p->src = (uint64_t)(slot + v.inl_off);
          break;
        }
        if (v.nsge == 2) { p->dst = parse_sg_keys(qp, p, 0, ACC_REMOTE_WRITE, true, &p->src); break; }
        const MKeyRaw lk = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), rk = mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey);
        p->src = mkey_check(lk, v.lkey, v.laddr, v.bytes, 0, false, &p->syn);
        if (p->src) p->dst = mkey_check(rk, v.rkey, v.raddr, v.bytes, ACC_REMOTE_WRITE, true, &p->syn);
        break;
      }
      case OP_RDMA_READ: {
        if (v.bytes == 0) { p->src = p->dst = 1; break; }
        if (v.nsge == 2) { p->src = parse_sg_keys(qp, p, ACC_LOCAL_WRITE, ACC_REMOTE_READ, true, &p->dst); break; }
        const MKeyRaw lk = mkey_load(qp->lkeys, qp->n_lkeys, v.lkey), rk = mkey_load(qp->r.rkeys, qp->r.n_rkeys, v.rkey);
        p->dst = mkey_check(lk, v.lkey, v.laddr, v.bytes, ACC_LOCAL_WRITE, false, &p->syn);
        if (p->dst) p->src = mkey_check(rk, v.rkey, v.raddr, v.bytes, ACC_REMOTE_READ, true, &p->syn);
        break;
      }
      case OP_SEND:
      case OP_SEND_IMM:
        if (v.nsge == 2) { parse_sg_keys(qp, p, 0, 0, false, &p->src); break; }
        p->src = v.inl_off ? (uint64_t)(slot + v.inl_off) : translate(qp->lkeys, qp->n_lkeys, v.lkey, v.laddr, v.bytes, 0, false, &p->syn);
        break;
      case OP_ATOMIC_CS:
      case OP_ATOMIC_FA: parse_atomic(ctl, qp, p); break;
      default: p->syn = SYN_LOCAL_QP_OP_ERR;
    }
  }
}

__device__ __forceinline__ bool needs_recv_wqe(uint8_t opcode) {
  return opcode == OP_SEND || opcode == OP_SEND_IMM || opcode == OP_RDMA_WRITE_IMM;
}

// Publish resolved[w].  Runs in the parallel part for plain RDMA WRITE / READ / NOP and in
// the ordered part for receive-consuming opcodes.  Returns the number of chunks.
// local1: a two-entry WQE's translated entry 1 (is_sg), which goes to the slot's SgSide record.
__device__ __forceinline__ uint32_t write_resolved(QpDev* qp, unsigned long long w, const WqeView& v, uint8_t syn,
                                                   uint64_t src, uint64_t dst, uint64_t rq_idx, uint8_t rq_taken,
                                                   uint64_t local1, uint32_t* chunk_out = nullptr) {
  const uint32_t slot = (uint32_t)(w & ((1u << qp->sq_log) - 1));
  Resolved* r = qp->resolved + slot;
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
  const bool sg = is_sg(v, syn);
  if (sg) {
    // chunks never straddle an entry (SgSide)
    const uint32_t n0 = (v.len0 + chunk - 1) / chunk;
    nchunks = n0 + (v.bytes - v.len0 + chunk - 1) / chunk;
    st_v4(qp->sg + slot, (uint32_t)local1, (uint32_t)(local1 >> 32), v.len0, n0);
  }
  // a clean atomic keeps its operands where a chunked copy / a receive keeps its bookkeeping (hca_types.h)
  const bool atom = syn == SYN_OK && is_atomic(v.opcode);
  r->chunk = atom ? (uint32_t)(v.compare >> 32) : chunk;
  if (chunk_out) *chunk_out = chunk;
  r->src = src; r->dst = dst;
  r->bytes = (syn == SYN_OK) ? v.bytes : 0;
  r->nchunks = nchunks;
  r->imm = v.imm;
  r->opcode = v.opcode; r->syndrome = syn; r->rq_consumed = rq_taken;
  r->fm_ce_se = (uint8_t)((v.fm_ce_se & ~RESOLVED_SG) | (sg ? RESOLVED_SG : 0));
  r->rq_idx = atom ? v.swap_add : rq_idx;
  r->done = atom ? (uint32_t)v.compare : 0u;
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
    qp->rq_cached_pi = expand16(wq_dbr_index(ld_u32_volatile(&qp->r.rq_dbr[DBR_RCV])), head);
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
  const uint4 d = ld_v4_volatile(rs);
  *rq_idx = head;
  *rq_taken = 1;
  qp->rq_head = head + 1;
  if (recv_wqe_bytes(d) < v.bytes) *syn = SYN_REMOTE_INVAL_REQ_ERR;
  else *dst = translate(qp->r.rkeys, qp->r.n_rkeys, recv_wqe_lkey(d), recv_wqe_addr(d), v.bytes, ACC_LOCAL_WRITE, true, syn);
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
  // the record holds 24 bits of ci: the consumer is (end_pi - ci24) mod 2^24 behind the producer
  ci = end_pi - ((end_pi - cq_dbr_index(ld_u32_volatile(cq->dbrec))) & 0xffffffu);
  *(volatile unsigned int*)&cq->ci_seen = ci;
  return end_pi - ci > depth;
}

// Warp-collective part of retire for a run that holds atomics (amask: the lanes whose WQE is a clean CS / FA).
// They execute one at a time in WQE order.  Each takes the fence a CQE owner bit takes -- cumulative over the
// payload of every earlier WQE of the QP, observed through their "finished" state words (the __syncwarp carries
// the other lanes' observations to the executing lane) -- then one 64-bit atom on the target, then stores the
// original value to the local fetch buffer.  The caller publishes the run's CQEs afterwards, behind its own
// fence, so a completion implies both the atomic and its fetched value.
__device__ __forceinline__ void retire_atomics(const Resolved* r, bool mine, uint32_t amask, uint32_t lane, uint8_t opc,
                                               uint32_t flags) {
  uint4 a = make_uint4(0, 0, 0, 0), o = make_uint4(0, 0, 0, 0);
  if (mine) {
    a = ld_v4_volatile(r);                                         // target | fetch buffer
    o = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r) + 32);  // compare (done | chunk) | swap_add (rq_idx)
  }
  __syncwarp();
  for (uint32_t m = amask; m; m &= m - 1) {
    if ((int)lane == __ffs((int)m) - 1) {
      unsigned long long* tgt = reinterpret_cast<unsigned long long*>(((uint64_t)a.y << 32) | a.x);
      uint8_t* fetch = reinterpret_cast<uint8_t*>(((uint64_t)a.w << 32) | a.z);
      const unsigned long long cmp = ((unsigned long long)o.y << 32) | o.x, swp = ((unsigned long long)o.w << 32) | o.z;
      const bool sys = (flags & RESOLVED_ATOMIC_SYS) != 0;
      fence_scope(sys);
      unsigned long long old;
      if (opc == OP_ATOMIC_FA) old = sys ? atomicAdd_system(tgt, swp) : atomicAdd(tgt, swp);
      else old = sys ? atomicCAS_system(tgt, cmp, swp) : atomicCAS(tgt, cmp, swp);
      if (((uintptr_t)fetch & 7) == 0) *reinterpret_cast<volatile unsigned long long*>(fetch) = old;
      else for (int i = 0; i < 8; ++i) reinterpret_cast<volatile uint8_t*>(fetch)[i] = (uint8_t)(old >> (8 * i));
    }
    __syncwarp();
  }
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
      // ---- atomics of the run execute here, in WQE order, before any CQE of the run is published
      const bool atom = active && syn == SYN_OK && is_atomic(opc);
      const uint32_t amask = __ballot_sync(0xffffffffu, atom);
      if (amask) {
        retire_atomics(r, atom, amask, lane, opc, imm);
        if (atom) bytes = 8;
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

// ------------------------------------------------------------------ fence gate
// A WQE posted with CTRL_FENCE (fm = 4; the other fm values gate nothing) moves no byte before every earlier WQE of its
// QP has finished (DESIGN.md 3.1).  Only a clean WQE that moves bytes is gated: an atomic executes at retirement, which
// is in order already, and a flushed or zero-length WQE has nothing to hold back.  Tested on the decoded WQE, so an
// unfenced one pays a bit test.
__device__ __forceinline__ bool fence_gated(const WqeView& v, uint8_t syn) {
  return (v.fm_ce_se & 0xe0u) == CTRL_FENCE && syn == SYN_OK && v.bytes != 0;
}
// Has every WQE before w finished?  Retirement is in order and a WQE retires only once its chunks are written and its
// atomic executed, so "the retirer has reached w" is exactly that.  It is read from retire_word, not retire_head: the
// retirer unlocks with (w << 1) behind its release fence, and nobody can lock at head w before w itself finished, so the
// word reads exactly (w << 1) from then until w retires.  On true, the fence acquires every earlier WQE's bytes for the
// loads of w's chunks (and releases the ticket the caller arms or opens next).
__device__ __forceinline__ bool gate_open(QpDev* qp, unsigned long long w) {
  if (ld_u64_volatile(&qp->retire_word) != (w << 1)) return false;
  fence_gpu();
  return true;
}
// Generic-proxy writes (and what the acquire above carried) before this CTA's later TMA loads (the async proxy).
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ------------------------------------------------------------------ claim
struct Work {
  QpDev* qp;
  unsigned long long w;
  uint32_t chunk;
  // filled by a direct (single-WQE) claim, which has just computed them: saves re-reading resolved[w]
  uint32_t have_desc, len, nch, fenced;
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

// ---- the ordered section, entered in WQE order by the parse_seq turn
// Wait until parse_seq names w and return it.  The turn word also carries "QP already failed" (PARSE_ERR_BIT), so the
// common path is one poll, no fence.
__device__ __forceinline__ unsigned long long wait_turn(EngineCtl* ctl, QpDev* qp, unsigned long long w) {
  unsigned long long turn = ld_u64_volatile(&qp->parse_seq);
  if ((turn & ~PARSE_ERR_BIT) != w) {
    unsigned long long t0 = globaltimer_ns();
    while (((turn = ld_u64_volatile(&qp->parse_seq)) & ~PARSE_ERR_BIT) != w) {
      if (globaltimer_ns() - t0 > 4000000000ull) { ctl->fatal = 2; break; }   // predecessor died
    }
  }
  return turn;
}

struct Committed {
  uint8_t syn;            // final syndrome
  uint32_t n, chunk;      // chunk count and granule of resolved[w]
  uint64_t dst;           // the destination (a SEND's is the receive buffer matched here)
  bool fenced, closed;    // fence_gated, and its gate still closed
};

// Commit WQE w, holding the turn.  The parallel part already published resolved[w] (n chunks of `chunk` bytes) unless
// the WQE needs a receive.  err: the QP has failed; a WQE that fails here sets it.  The caller arms the ticket and passes
// the turn on.  release_rq: release rq_head here, because the single path passes the turn of a one-chunk WQE with a
// relaxed store (the batch path's closing fence releases it instead).
__device__ __forceinline__ Committed commit_wqe(EngineCtl* ctl, QpDev* qp, unsigned long long w, const Parsed& p, bool recv,
                                                uint32_t n, uint32_t chunk, bool& err, bool release_rq) {
  Committed c{p.syn, n, chunk, p.dst, false, false};
  if (err) {
    // flushed: nothing moves, whatever the parse said
    c.syn = SYN_WR_FLUSH_ERR;
    c.n = write_resolved(qp, w, p.v, c.syn, 0, 0, 0, 0, 0, &c.chunk);
  } else if (recv) {
    fence_gpu();  // acquire rq_head from the previous receive-consuming WQE
    uint64_t rq_idx = 0;
    uint8_t rq_taken = 0;
    match_recv(ctl, qp, p.v, &c.syn, &c.dst, &rq_idx, &rq_taken);
    c.n = write_resolved(qp, w, p.v, c.syn, p.src, c.dst, rq_idx, rq_taken, p.local1, &c.chunk);
    if (release_rq) fence_gpu();  // release rq_head
  }
  if (c.syn != SYN_OK && !err) { qp->state = QPS_ERR; err = true; }
  // A fenced WQE whose gate is still closed is not moved by its claimer: even with one chunk it gets a gated ticket,
  // which the helpers' offer scan stops at and opens once the retirer reaches it.  An open gate's fence orders the
  // ticket after it.
  c.fenced = fence_gated(p.v, c.syn);
  c.closed = c.fenced && !gate_open(qp, w);
  if (c.closed) atomicAdd(&qp->n_fence_waits, 1ull);
  return c;
}

// Single claim of WQE w (the caller won the cursor CAS and took its acquire).  st: the QP state try_claim loaded.  The
// claimer moves chunk 0 itself with the descriptor computed here, so only a WQE with more chunks, or a closed gate, gets a
// ticket for the helpers.  Returns 1 with *out = chunk 0, or 0 when the gate is closed.
__device__ __forceinline__ int claim_one(EngineCtl* ctl, QpDev* qp, unsigned long long w, uint32_t st, uint32_t pending,
                                         Work* out, bool* saw_pending) {
  trace_stamp(qp, w, TR_CLAIM);
  // ordering audit: the doorbell record must already cover what the register announced
  const uint16_t ahead = (uint16_t)(wq_dbr_index(ld_u32_volatile(&qp->dbr[DBR_SND])) - (uint16_t)w);
  if (ahead < pending && ahead < 0x8000)
    atomicAdd(&qp->n_db_order_violations, 1ull);
  // ---- parallel part
  Parsed p;
  parse_wqe(ctl, qp, w, &p);
  const bool recv = p.syn == SYN_OK && needs_recv_wqe(p.v.opcode);
  uint32_t n = 1, chunk_sz = 0;
  if (!recv) n = write_resolved(qp, w, p.v, p.syn, p.src, p.dst, 0, 0, p.local1, &chunk_sz);
  // ---- ordered part
  const unsigned long long turn = wait_turn(ctl, qp, w);
  bool err = (turn & PARSE_ERR_BIT) != 0 || st == QPS_ERR;
  const Committed c = commit_wqe(ctl, qp, w, p, recv, n, chunk_sz, err, true);
  Resolved* res = qp->resolved + (w & ((1u << qp->sq_log) - 1));
  const unsigned long long next = (w + 1) | (err ? (unsigned long long)PARSE_ERR_BIT : 0ull);
  if (c.n > 1 || c.closed) {
    fence_gpu();  // release resolved[w] before the ticket that lets helpers read it
    st_u64_relaxed(&res->ticket, (c.closed ? TICKET_GATED : TICKET_ONE) | ((w & TICKET_FIELD_MASK) << TICKET_GEN_SHIFT) | c.n);
    st_u64_release_scope(&qp->parse_seq, next, false);   // helpers trust: committed => ticket armed
  } else {
    st_u64_relaxed(&qp->parse_seq, next);
  }
  trace_stamp(qp, w, TR_PARSED);
  if (c.closed) {
    *saw_pending = true;
    return 0;
  }
  uint32_t bytes = c.syn == SYN_OK ? p.v.bytes : 0;
  uint64_t src = p.src, dst = c.dst;
  if (is_sg(p.v, c.syn)) {
    // two entries: chunk 0 starts entry 0, or entry 1 when entry 0 is empty; the remote side starts at 0 either way
    if (p.v.len0) bytes = p.v.len0;
    else if (p.v.opcode == OP_RDMA_READ) dst = p.local1;
    else src = p.local1;
  }
  out->qp = qp; out->w = w; out->chunk = 0;
  out->have_desc = 1; out->nch = c.n; out->src = src; out->dst = dst; out->fenced = c.fenced;
  out->len = bytes < c.chunk ? bytes : c.chunk;     // chunk 0
  return 1;
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
  uint32_t pending = look_at_doorbell ? (uint16_t)(doorbell_index(db) + 1 - (uint16_t)c) : 0u;
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
      fence_scope(sys);  // acquire: WQE bytes the doorbell announced
      return claim_one(ctl, qp, c, st, pending, out, saw_pending);
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
    uint32_t avail[8], total = 0, lead = 0, gk = 8;
    unsigned long long gt = 0;
    bool leading = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const bool mine = (uint32_t)((t[k] >> TICKET_GEN_SHIFT) & TICKET_FIELD_MASK) == (uint32_t)((off + k) & TICKET_FIELD_MASK);
      const uint32_t cc = (uint32_t)(t[k] >> 40), nn = (uint32_t)(t[k] & TICKET_FIELD_MASK);
      // gated (a fenced WQE waiting for its gate): nothing to draw yet, but the offer must not pass it
      const bool gated = (uint32_t)k < cnt && mine && (t[k] & TICKET_GATED);
      if (gated && gk == 8) { gk = k; gt = t[k]; }
      avail[k] = ((uint32_t)k < cnt && mine && cc < nn) ? nn - cc : 0u;   // single-chunk WQE taken by its claimer, or fully drawn: 0
      total += avail[k];
      if (leading && (uint32_t)k < cnt && avail[k] == 0 && !gated) ++lead; else leading = false;
    }
    if (lead) atomicMax(&qp->offer, off + lead);
    // The gate is polled here: every CTA that scans the QP re-checks it, so it cannot be missed and nobody blocks on it.
    // Only the oldest gated WQE can be at the retire head.  Opening resets the chunk counter (one CAS: a second opener, or
    // a stray draw that bumped the gated counter, makes it fail and the next scan looks again).
    if (gk < 8) {
      *saw_pending = true;
      const unsigned long long gw = off + gk;
      Resolved* gr = qp->resolved + (gw & mask);
      if (gate_open(qp, gw)) {
        atomicCAS(&gr->ticket, gt, gt & TICKET_LOW_MASK);
        if (draw_chunk(qp, gr, gw, out)) return 1;
      }
    }
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
  uint32_t n = 1, chunk = 0;
  bool recv = false;
  if (lane < k) {
    trace_stamp(qp, w, TR_CLAIM);
    parse_wqe(ctl, qp, w, &p);
    recv = p.syn == SYN_OK && needs_recv_wqe(p.v.opcode);
    if (!recv) n = write_resolved(qp, w, p.v, p.syn, p.src, p.dst, 0, 0, p.local1, &chunk);
  }
  __syncwarp();
  unsigned long long turn = 0;
  if (lane == 0) turn = wait_turn(ctl, qp, w0);
  turn = __shfl_sync(0xffffffffu, turn, 0);
  bool err = (turn & PARSE_ERR_BIT) != 0 || *(volatile uint32_t*)&qp->state == QPS_ERR;
  for (uint32_t i = 0; i < k; ++i) {
    if (lane == i) {
      const Committed c = commit_wqe(ctl, qp, w, p, recv, n, chunk, err, false);
      Resolved* res = qp->resolved + (w & mask);
      st_u64_relaxed(&res->ticket, (c.closed ? TICKET_GATED : 0ull) | ((w & TICKET_FIELD_MASK) << TICKET_GEN_SHIFT) | c.n);    // chunk counter starts at 0
      trace_stamp(qp, w, TR_PARSED);
    }
    __syncwarp();
    err = __shfl_sync(0xffffffffu, (int)err, i) != 0;
  }
  if (lane == 0) {
    fence_gpu();  // release: every lane's resolved[] / ticket / rq_head (ordered before this by the __syncwarp chain)
    st_u64_release_scope(&qp->parse_seq, (w0 + k) | (err ? (unsigned long long)PARSE_ERR_BIT : 0ull), false);
  }
}

// ------------------------------------------------------------------ the kernel
// Control, lane 0: has the mover reported queue entry e written?  With `block` it waits, bounded by the mover, which
// reports every chunk or sets mover_fatal within its own bound.  1: written, 0: not yet, -1: the mover failed.
__device__ __forceinline__ int chunk_written(Smem& s, int e, uint32_t& ph, bool block) {
  for (;;) {
    if (mbar_test_wait(&s.qdone[e], (ph >> e) & 1u)) { ph ^= 1u << e; return 1; }
    if (*(volatile int*)&s.mover_fatal) return -1;
    if (!block) return 0;
  }
}

// Control, lane 0: a chunk's bytes are written, and this thread has observed that through a CTA-scope synchronisation
// with the threads that wrote them (the mover's qdone arrive, or the generic copy's named barrier).  Count it; true when
// that finished its WQE.
__device__ __forceinline__ bool complete_chunk(QpDev* qp, unsigned long long w, uint32_t nch) {
  Resolved* r = qp->resolved + (w & ((1u << qp->sq_log) - 1));
  // This chunk's bytes before the count that may complete the WQE: the fence is cumulative over every write this thread
  // has observed, so it releases the mover's and the generic threads' stores as well as its own.  gpu scope is enough even
  // when the CQ or the payload lives in host / peer memory: the retirer's system-scope
  // fence in write_cqe() is cumulative over everything this chain of gpu-scope releases made
  // visible to it (a sys fence per chunk cost ~2x on host-resident queues, measured).
  if (nch > 1) fence_gpu();
  if (nch == 1 || atomicAdd(&r->done, 1u) + 1 == nch) {
    trace_stamp(qp, w, TR_COPIED);
    fence_gpu();  // single chunk: its bytes before "finished"; else observe every other chunk's count -> their bytes precede our CQE
    *(volatile unsigned long long*)&r->state = (w << 2) | 2ull;
    __threadfence();  // SC: "finished" store before the retire try-lock (pairs with the unlock / re-check below)
    return true;
  }
  return false;
}

// What control's lane 0 found to do in one iteration; the whole warp acts on it.
enum Act : int {
  ACT_LEAVE = -1,
  ACT_NONE = 0,          // nothing claimed
  ACT_QUEUED,            // a chunk queued for the mover
  ACT_GENERIC,           // a generic copy for warps 0, 2 and 3
  ACT_NO_BYTES,          // a claimed chunk with nothing to move
  ACT_QUEUED_SMALL,      // queued, at most kSmallChunk: wait for it before scanning again
};

__global__ void __launch_bounds__(kThreads, 1) engine_kernel(EngineCtl* ctl) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  if (threadIdx.x == 0) {
    init_barriers(s);
    atomicAdd(&ctl->running_ctas, 1u);
    if (blockIdx.x == 0) ctl->t_start = globaltimer_ns();
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (warp == 1) {
    if (lane == 0) {
      unsigned long long* prof = ctl->mover_prof;
      const bool ok = run_mover(s, prof ? prof + (size_t)blockIdx.x * MOVER_PROF_N : nullptr);
      if (!ok) { ctl->fatal = 1; *(volatile int*)&s.mover_fatal = 1; }
    }
    return;
  }
  if (warp != 0) {
    // warps 2 and 3: the generic copies control hands out, until control leaves
    for (;;) {
      generic_bar();
      if (s.gquit) return;
      copy_generic(s.gsrc, s.gdst, s.glen, threadIdx.x - 32, kGenericThreads);
      generic_bar();
    }
  }
  // ---- warp 0: control.  Lane 0 finds the work; the warp parses batches and retires.
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
  // lane 0's side of the chunk queue: entries e_done .. e_done + outstanding - 1 are with the mover
  int e_push = 0, e_done = 0, outstanding = 0;
  uint32_t done_ph = 0;
  bool fatal = false;
  // A counted chunk that finished its WQE is retired by the whole warp (lane 0's arguments count).
  auto finish = [&](QpDev* qp, unsigned long long w, uint32_t nch) {
    const int fin = lane == 0 ? (int)complete_chunk(qp, w, nch) : 0;
    if (__shfl_sync(0xffffffffu, fin, 0))
      retire((QpDev*)__shfl_sync(0xffffffffu, (unsigned long long)qp, 0), lane, __shfl_sync(0xffffffffu, w, 0));
  };
  // Count every chunk the mover has written, oldest first; wait while the queue is full, or for all of them.
  auto reap = [&](bool all) -> bool {   // false: the mover failed
    for (;;) {
      int got = 0;
      if (lane == 0 && outstanding) got = chunk_written(s, e_done, done_ph, all || outstanding == kQueue);
      got = __shfl_sync(0xffffffffu, got, 0);
      if (got <= 0) return got == 0;
      Owed o{};
      if (lane == 0) {
        o = s.owed[e_done];
        e_done = e_done + 1 == kQueue ? 0 : e_done + 1;
        --outstanding;
      }
      finish(o.qp, o.w, o.nch);
    }
  };
  for (;;) {
    if (!reap(false)) { fatal = true; break; }
    int batch_k = 0;
    Act act = ACT_NONE;
    Work work;
    uint32_t nch = 0;
    if (lane == 0) {
      bool have = false, quit = false;
      // "everybody leaves" travels with the queue scan (its latency hides behind try_claim's loads); the QP
      // count is re-read every 64 iterations together with the fence that drops stale L1 lines, so host-side
      // updates (new QPs, reconnects) become visible within ~100 us without a dependent load per iteration
      const unsigned quit_all_seen = *(volatile unsigned int*)&ctl->quit_all;
      if ((iter++ & 63u) == 0) { fence_gpu(); n_qps_cached = ctl->n_qps; }
      const uint32_t n = n_qps_cached;
      bool pending = false;
      if (sticky_qp) {
        Resolved* sr = sticky_qp->resolved + (sticky_w & ((1u << sticky_qp->sq_log) - 1));
        // a successful draw is a claim that MUST be executed, whichever generation it names
        if (draw_chunk(sticky_qp, sr, sticky_w, &work)) have = true;
        else sticky_qp = nullptr;
      }
      // Every probe of a QP is at least one L2 round trip, so a CTA does not walk the whole table each
      // iteration (with 8 QPs registered, one active QP ran at half its solo message rate): it looks at the QP
      // that last gave it work and at ONE other, rotating.  CTAs start at different offsets, so every QP is
      // still probed by many CTAs per round trip.  The host watcher keeps the full scan: it alone decides
      // "idle" / "drained" and it is the only one that reads host-resident doorbells.
      const uint32_t n_scan = host_watcher ? n : (n < 2 ? n : 2u);
      for (uint32_t k = 0; k < n_scan && !have && !batch_k; ++k) {
        const uint32_t qi = (host_watcher || k == 0) ? (rr + k) % n : (rr + 1 + rot % (n - 1)) % n;
        QpDev* qp = *(QpDev* volatile*)&ctl->qps[qi];   // table grows while we run
        if (!qp) continue;
        const int got = try_claim(ctl, qp, &work, &pending, host_watcher);
        if (got == 1) have = true;
        else if (got == 2) { batch_k = (int)work.chunk; pending = true; }
        if (got) rr = qi;
      }
      ++rot;
      if (have) {
        uint32_t len;
        uint64_t csrc, cdst;
        bool fenced;
        if (work.have_desc) {
          len = work.len; csrc = work.src; cdst = work.dst; nch = work.nch; fenced = work.fenced != 0;
        } else {
          Resolved* r = work.qp->resolved + (work.w & ((1u << work.qp->sq_log) - 1));
          const uint4 f = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r) + 16);   // bytes | nchunks | imm | flags
          const uint4 a = ld_v4_volatile(reinterpret_cast<const uint8_t*>(r));        // src | dst
          const uint32_t chunk = *(volatile uint32_t*)&r->chunk;
          uint32_t c = work.chunk, bytes = f.x;
          csrc = ((uint64_t)a.y << 32) | a.x;
          cdst = ((uint64_t)a.w << 32) | a.z;
          if ((f.w >> 8) & RESOLVED_SG) {
            // two entries: rebase onto the entry chunk c lies in (SgSide)
            const uint4 g = ld_v4_volatile(work.qp->sg + (work.w & ((1u << work.qp->sq_log) - 1)));   // local1 | len0 | n0
            if (c < g.w) {
              bytes = g.z;
            } else {
              const uint64_t local1 = ((uint64_t)g.y << 32) | g.x;
              c -= g.w;
              bytes -= g.z;
              if ((uint8_t)f.w == OP_RDMA_READ) { csrc += g.z; cdst = local1; }
              else { csrc = local1; cdst += g.z; }
            }
          }
          const uint64_t off = (uint64_t)c * chunk;
          len = bytes == 0 ? 0 : (uint32_t)((bytes - off < chunk) ? (bytes - off) : chunk);
          csrc += off;
          cdst += off;
          nch = f.y;
          fenced = ((f.w >> 8) & 0xe0u) == CTRL_FENCE;
        }
        if (nch > 1) { sticky_qp = work.qp; sticky_w = work.w; }
        last_activity = globaltimer_ns();
        spins = 0;
        if (len == 0) {
          act = ACT_NO_BYTES;
        } else if (len >= kBulkMin && (((csrc | cdst) & 15) == 0) && ((len & 15) == 0)) {
          // reap() left room: outstanding < kQueue
          if (fenced) fence_proxy_async_global();   // the mover's TMA loads see what the gate's acquire made visible
          s.q[e_push] = Chunk{csrc, cdst, len};
          s.owed[e_push] = Owed{work.qp, work.w, nch};
          mbar_arrive(&s.qfull[e_push]);
          e_push = e_push + 1 == kQueue ? 0 : e_push + 1;
          ++outstanding;
          atomicAdd(&ctl->n_bulk_chunks, 1ull);
          // A chunk the ring holds at once gains nothing from streaming; finishing it before the next scan keeps
          // small-message latency what it was (a 4 KiB WQE otherwise waits for the scan to be counted).
          act = len <= kSmallChunk ? ACT_QUEUED_SMALL : ACT_QUEUED;
        } else {
          s.gsrc = csrc; s.gdst = cdst; s.glen = len;
          act = ACT_GENERIC;
        }
      } else {
        ++spins;
        // The host watcher is the only CTA that sees host-resident doorbells, so it alone may declare
        // the engine idle or drained; everybody else follows quit_all.
        if (pending) last_activity = globaltimer_ns();
        else if (host_watcher && ctl->oneshot && spins > 4) { quit = true; ctl->quit_all = 1; }   // drained: every posted WQE has retired
        if (quit_all_seen) quit = true;
        if ((spins & 63) == 0) {
          if (*ctl->stop) quit = true;   // mapped host word: a PCIe read, hence only every 64 idle spins
          else if (host_watcher && globaltimer_ns() - last_activity > ctl->idle_timeout_ns) { quit = true; ctl->exited_idle = 1; ctl->quit_all = 1; }
        }
        if (spins > 256) __nanosleep(200);
        if (quit) act = ACT_LEAVE;
      }
    }
    // a batch claim is parsed by the whole warp; its chunks are then drawn like anybody else's
    batch_k = __shfl_sync(0xffffffffu, batch_k, 0);
    if (batch_k) {
      QpDev* bqp = (QpDev*)__shfl_sync(0xffffffffu, (unsigned long long)work.qp, 0);
      claim_batch(ctl, bqp, __shfl_sync(0xffffffffu, work.w, 0), (uint32_t)batch_k, lane);
    }
    act = (Act)__shfl_sync(0xffffffffu, (int)act, 0);
    if (act == ACT_LEAVE) break;
    if (act == ACT_GENERIC) {
      generic_bar();
      copy_generic(s.gsrc, s.gdst, s.glen, lane, kGenericThreads);
      generic_bar();   // every generic thread's stores before lane 0's release in complete_chunk
    }
    if (act == ACT_QUEUED_SMALL && !reap(true)) { fatal = true; break; }
    if (act == ACT_GENERIC || act == ACT_NO_BYTES) finish(work.qp, work.w, nch);
  }
  // Leaving.  Every chunk handed to the mover is a claim that must be completed; after a mover fault nothing is
  // completed (the host sees ctl->fatal).
  if (!fatal && !reap(true)) fatal = true;
  if (lane == 0) {
    if (!fatal) {
      s.q[e_push].len = kQuitLen;
      mbar_arrive(&s.qfull[e_push]);
    }
    s.gquit = 1;
  }
  generic_bar();
  if (lane == 0) {
    if (blockIdx.x == 0) ctl->t_exit = globaltimer_ns();
    atomicSub(&ctl->running_ctas, 1u);
  }
}

// ------------------------------------------------------------------ ceiling
// What the engine's copy loop reaches with nothing around it: CTA b streams span bytes from src + b * span to
// dst + b * span as ONE queued chunk -- no claims, no chunk boundaries, no completion bookkeeping.  The distance between
// this and the engine on the same CTA count is what the per-chunk work costs (tools/engine_pipeline.py).
// prof (may be null): the mover's stall profile, MOVER_PROF_N counters per CTA, as the engine's.
__global__ void __launch_bounds__(kThreads, 1) engine_ceiling_kernel(uint64_t src, uint64_t dst, uint32_t span,
                                                                    unsigned int* fatal, unsigned long long* prof) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  if (threadIdx.x == 0) init_barriers(s);
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint64_t off = (uint64_t)blockIdx.x * span;
    s.q[0] = Chunk{src + off, dst + off, span};
    mbar_arrive(&s.qfull[0]);
    s.q[1].len = kQuitLen;
    mbar_arrive(&s.qfull[1]);
  } else if (threadIdx.x == 32) {
    const bool ok = run_mover(s, prof ? prof + (size_t)blockIdx.x * MOVER_PROF_N : nullptr);
    if (!ok && fatal) atomicAdd(fatal, 1u);
  }
}

inline size_t engine_smem_bytes() { return sizeof(Smem) + 128; }

}  // namespace eng
}  // namespace rn
