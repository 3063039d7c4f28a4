// Device-visible state of the software HCA ("softhca").
//
// The softhca keeps the exact contract a ConnectX exposes to an IBGDA-style
// poster -- a send queue of 64-byte WQEBBs, a doorbell record, a doorbell
// register, a completion queue of 64-byte CQEs with an owner bit, and an MKey
// table that turns (key, VA, length) into something the DMA engine may touch --
// but the "NIC" is a persistent CUDA kernel (hca/engine.cu) that moves the bytes
// over HBM / NVLink with TMA bulk copies.  It exists because the GPU box exposes
// no /dev/infiniband to the container (gpurun probe, DESIGN.md section 2); the verbs
// backend (verbs/verbs_dl.cc) drives a real mlx5 QP through the same poster code.
//
// Reference parity: amd_mem_context (amdp2p.c:73-85) is the per-registration
// record there; MKeyEntry is its analogue here (VA, size, owner, pin handle).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../wire/mlx5_wire.h"

namespace rn {

enum MemKind : uint32_t { MEM_DEVICE = 0, MEM_HOST_PINNED = 1, MEM_PEER = 2 };

enum Access : uint32_t {
  ACC_LOCAL_WRITE = 1u << 0,
  ACC_REMOTE_WRITE = 1u << 1,
  ACC_REMOTE_READ = 1u << 2,
  ACC_REMOTE_ATOMIC = 1u << 3,
};

enum QpState : uint32_t {
  QPS_RESET = 0, QPS_INIT = 1, QPS_RTR = 2, QPS_RTS = 3, QPS_SQD = 4, QPS_SQE = 5, QPS_ERR = 6,
};

// One registered memory region.  `base` is the VA the application registered and
// puts into WQEs; `map_base` is the address through which the engine's GPU reaches
// the same bytes (identical for local HBM and pinned host memory under UVA, an
// IPC/VMM mapping for a peer GPU's HBM).
struct alignas(16) MKeyEntry {
  uint64_t base;
  uint64_t len;
  uint64_t map_base;
  uint32_t key;       // (index << 8) | 8-bit variant tag ; lkey == rkey, as on mlx5
  uint32_t access;
  uint32_t valid;     // 0 = free or revoked
  uint32_t kind;      // MemKind
  uint64_t pad;
};
static_assert(sizeof(MKeyEntry) == 48, "engine reads an MKey as three 16-byte loads");

struct CqDev {
  uint8_t* buf;              // 2^log_n CQEs of 64 bytes
  uint32_t* dbrec;           // [0] = be32(ci & 0xffffff), written by the consumer
  uint32_t log_n;
  uint32_t cqn;
  unsigned int pi;           // producer index, claimed by engines with atomicAdd (system scope)
  unsigned int ci;           // device consumer index (device pollers)
  unsigned int overruns;     // completions that found the ring full of unconsumed CQEs (the QP that hit it goes to ERR)
  unsigned int ci_seen;      // consumer index as last read from dbrec by a producer (refreshed only when the ring looks full)
};

// Per-SQ-slot record written by the WQE prologue (address translation, checks)
// and shared by every engine CTA that copies a chunk of that WQE.
// An atomic (CS / FA) that parsed cleanly moves no chunks (bytes = 0, nchunks = 1) and is executed by the
// retirer, so the fields a chunk copy or a receive would use carry its operands instead (a union in effect):
//   src = target word, dst = local fetch buffer (both translated), imm = RESOLVED_ATOMIC_* flags,
//   done | chunk = compare (low | high 32 bits), rq_idx = swap_add.
// done | chunk | rq_idx are then one 16-byte load at offset 32.
struct alignas(64) Resolved {
  uint64_t src, dst;
  uint32_t bytes, nchunks;
  uint32_t imm;
  uint8_t opcode, fm_ce_se, syndrome, rq_consumed;
  unsigned int done;          // chunks finished (atomic)
  uint32_t chunk;             // bytes per claim for this WQE (sized so ~4 claims per engine CTA)
  uint64_t rq_idx;            // receive WQE consumed (SEND / WRITE_IMM)
  unsigned long long state;   // (wqe_index << 2) | 1 resolved | 2 finished
  unsigned long long ticket;  // [63:40] next chunk | [39:20] wqe_index mod 2^20 | [19:0] nchunks
};
static_assert(sizeof(Resolved) == 64, "Resolved is one cache-line pair slot");
static_assert(offsetof(Resolved, done) == 32 && offsetof(Resolved, chunk) == 36 && offsetof(Resolved, rq_idx) == 40,
              "atomic operands are read back as one 16-byte load at offset 32");
enum : uint32_t { RESOLVED_ATOMIC_SYS = 1u };   // Resolved::imm of an atomic: execute (and fence) at system scope
// Resolved::fm_ce_se of a clean two-entry WQE (a bit the wire's fm_ce_se leaves reserved): its chunks map through the
// slot's SgSide record.
enum : uint8_t { RESOLVED_SG = 0x10 };

// Per-SQ-slot side record of a two-entry WQE (gather WRITE / WRITE_IMM / SEND, scatter READ), written with its Resolved
// record and read only when that record carries RESOLVED_SG.  Chunks never straddle an entry: chunk c < n0 covers entry
// 0 at offset c * chunk (Resolved's local address), chunk c >= n0 covers entry 1 at local1 + (c - n0) * chunk, and the
// remote side at len0 + (c - n0) * chunk.  One 16-byte load.
struct alignas(16) SgSide {
  uint64_t local1;            // entry 1, translated
  uint32_t len0;              // entry 0's length
  uint32_t n0;                // entry 0's chunks: ceil(len0 / chunk)
};
static_assert(sizeof(SgSide) == 16, "SgSide is one 16-byte load");

// What a requester's engine needs to know about the connected responder QP.  All
// pointers are already translated into the engine GPU's address space.
struct RemoteView {
  MKeyEntry* rkeys;           // responder's MKey table
  uint32_t n_rkeys;
  uint32_t qpn;
  uint8_t* rq;                // responder receive ring (16-byte receive WQEs)
  uint32_t* rq_dbr;           // responder doorbell record ([DBR_RCV] = be32 count)
  uint32_t rq_log;
  uint32_t connected;         // bit 0: connected; bit 1: responder CQ's consumer record addressable (same process)
  CqDev* rcq;                 // responder's receive CQ
  uint8_t* rcq_buf;           // its ring, translated
};

struct QpDev {
  // ---- static after creation
  uint32_t qpn;
  volatile uint32_t state;    // QpState
  uint8_t* sq;                // 2^sq_log WQEBBs
  uint32_t sq_log;
  uint32_t rq_log;
  uint32_t* dbr;              // doorbell record: [DBR_RCV], [DBR_SND], be32 16-bit counters
  unsigned long long* bf;     // doorbell register: first 8 bytes of the last ctrl segment
  uint8_t* rq;                // own receive ring
  CqDev* scq;                 // send CQ
  CqDev* rcq;                 // receive CQ
  MKeyEntry* lkeys;
  uint32_t n_lkeys;
  uint32_t chunk_bytes;       // engine work granule for this QP
  uint32_t sys_scope;         // 1: some ring/peer of this QP is outside this GPU -> system-scope fences
  uint32_t sq_in_device;      // 1: SQ / doorbell live in this GPU's memory (cheap to poll from every CTA)
  uint32_t pad1;
  uint32_t trace_on;          // 1: stamp the WQE lifecycle into trace[]
  unsigned long long* trace;  // 8 x u64 per SQ slot: post, claim, parsed, copied, cqe, seen, -, -
  RemoteView r;
  Resolved* resolved;         // one per SQ slot
  uint32_t* ready_flags;      // one per SQ slot: (index + 1) once the WQE bytes are complete (shared posters)
  SgSide* sg;                 // one per SQ slot: the second entry of a two-entry WQE
  // ---- device poster state
  unsigned long long resv_head;    // next WQE index to hand out
  unsigned long long ready_head;   // every index below this has rung its doorbell
  unsigned long long sq_cons;      // every index below this is complete (from CQEs)
  unsigned long long rq_pi;        // receive WQEs posted
  unsigned int db_lock;            // try-lock: its holder rings one doorbell for every ready WQE
  unsigned int pad2;
  // ---- engine state
  unsigned long long cursor;       // claim head: next WQE index nobody owns yet (claimed by CAS)
  unsigned long long parse_seq;    // ordered-commit turn: WQE index allowed to commit; bit 63 = QP already in error
  unsigned long long offer;        // oldest WQE index that may still have undrawn chunks (helpers go oldest-first)
  unsigned long long retire_head;  // next WQE index to retire in order
  unsigned long long retire_word;  // (retire_head << 1) | locked: ONE compare-and-swap both takes the retire lock and proves whose turn it is
  unsigned long long rq_head;      // next receive WQE of the *peer* to consume
  unsigned long long rq_cached_pi; // responder receive-producer count as last read (a remote read: refreshed only when exhausted)
  // ---- counters (readable from the host; SURVEY.md section 5 "metrics")
  unsigned long long n_wqe, n_cqe, n_err, n_db_order_violations, n_bytes, n_rnr;
  unsigned long long n_fence_waits;  // fenced WQEs whose gate was still closed when they committed
};

// Chunk tickets: one atomicAdd(TICKET_ONE) hands out a self-describing claim.
enum : unsigned long long { PARSE_ERR_BIT = 1ull << 63 };
enum : unsigned long long { TICKET_ONE = 1ull << 40, TICKET_GEN_SHIFT = 20, TICKET_FIELD_MASK = 0xfffffull };
// A fenced WQE's ticket before its gate opens: the top bit of the chunk counter.  The counter then reads >= 2^23, above
// any chunk count, so every existing "next chunk < nchunks" test sees nothing to draw (a stray draw only bumps it).  The
// gate is opened by resetting the counter to 0 (eng::try_claim), which also drops this bit.
enum : unsigned long long { TICKET_GATED = 1ull << 63, TICKET_LOW_MASK = TICKET_ONE - 1 };

struct EngineCtl {
  volatile uint32_t* stop;         // mapped pinned host word: nonzero = exit
  QpDev** qps;                     // device array of QP pointers
  volatile uint32_t n_qps;
  uint32_t max_qps;
  unsigned long long idle_timeout_ns;   // exit when no doorbell moved for this long
  unsigned long long rnr_timeout_ns;
  unsigned int running_ctas;       // CTAs alive (atomic)
  unsigned int exited_idle;        // set when the watchdog ended the engine
  unsigned int fatal;              // a DMA never completed; engine bailed out
  unsigned int quit_all;           // the host-doorbell watcher found the engine idle / drained: everybody leaves
  unsigned int oneshot;            // exit as soon as every queue is drained (profiling under ncu: kernels are serialised there)
  unsigned int host_native_atomics;  // cudaDevAttrHostNativeAtomicSupported: a GPU atomic on pinned host memory is atomic there
  unsigned long long n_bulk_chunks;     // chunks moved through the TMA bulk path
  unsigned long long t_start, t_exit;   // %globaltimer of engine start / exit (CTA 0)
  unsigned long long* mover_prof;       // RN_ENGINE_PROFILE=1: MOVER_PROF_N counters per CTA (eng::move_chunks), else null
};

// The mover's stall profile, one row of MOVER_PROF_N u64 per CTA: %globaltimer ns spent in each wait, the mover's whole
// run, and the chunks it reported.  Order shared with api.MOVER_PROFILE_FIELDS.
enum MoverProf : int {
  MP_WAIT_READ = 0,   // bulk_wait_read: no free ring stage for the next load
  MP_FULL,            // full[] mbarrier: the next stage's load has not landed
  MP_CHUNK_WAIT,      // bulk_wait<kSif>: a chunk's stores completing before it is reported
  MP_REPORT,          // reporting written chunks to control (qdone arrive)
  MP_DRY_WAIT,        // bulk_wait<0>: the queue ran dry, the ring drains
  MP_QFULL_IDLE,      // ring empty, nothing owed: waiting for control to queue a chunk
  MP_TOTAL,           // entry to exit
  MP_CHUNKS,          // chunks reported
  MOVER_PROF_N
};
constexpr int kMaxEngineCtas = 256;     // rows of the profile array

// Status codes returned by device-side waits (never spin forever: SURVEY.md section 5).
enum WaitStatus : int { WAIT_OK = 0, WAIT_TIMEOUT = -1, WAIT_CQE_ERROR = -2, WAIT_QP_ERROR = -3 };

}  // namespace rn
