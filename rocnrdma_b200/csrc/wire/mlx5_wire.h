// mlx5 work-queue wire format: WQE segments, receive WQEs, CQE64, doorbell and CQ consumer records.
//
// Everything a ConnectX HCA reads or writes in a send queue / completion queue,
// byte-exact and big-endian, usable from host C++, CUDA device code and (through
// the C API) the Python unit tests.  The same encoders feed a real mlx5 QP (verbs
// backend) and the software HCA (softhca backend), so the device-side posting code
// is identical on both wires.
//
// Role in the reference: none of this exists there -- amdp2p only makes
// ibv_reg_mr() succeed (amdp2p.c:363-371) and leaves posting to "IB verbs"
// (README.md:67).  SURVEY.md N3/K1 asks for the GPU to build these itself.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define RN_HD __host__ __device__ __forceinline__
#else
#define RN_HD inline
#endif

namespace rn {

// ---------------------------------------------------------------- byte order
RN_HD uint32_t bswap32(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(v, 0, 0x0123);
#else
  return __builtin_bswap32(v);
#endif
}
RN_HD uint16_t bswap16(uint16_t v) { return (uint16_t)((v >> 8) | (v << 8)); }
RN_HD uint64_t bswap64(uint64_t v) {
  return ((uint64_t)bswap32((uint32_t)v) << 32) | bswap32((uint32_t)(v >> 32));
}
// The build only targets little-endian hosts (x86-64) and GPUs.
RN_HD uint32_t be32(uint32_t v) { return bswap32(v); }
RN_HD uint16_t be16(uint16_t v) { return bswap16(v); }
RN_HD uint64_t be64(uint64_t v) { return bswap64(v); }

// ---------------------------------------------------------------- constants
enum : uint32_t {
  WQEBB = 64,        // basic block of the send queue
  WQE_SEG = 16,      // every segment is 16 bytes; ctrl.ds counts these
  CQE_SIZE = 64,
  MAX_INLINE = 28,   // largest inline payload: ctrl + raddr + a 4-byte inline header + 28 bytes fill one WQEBB
  INLINE_SEG = 0x80000000u,   // byte_count flag: the payload follows in the WQE itself
  MAX_BYTE_COUNT = 0x7fffffffu,   // largest byte count a gather data segment carries (bit 31 is INLINE_SEG)
  MAX_MSG = 1u << 30,         // longest message, inclusive (DESIGN.md 3.1); longer WRITE / READ / SEND: LOCAL_LENGTH_ERR
  MAX_SGE = 2,                // scatter-gather entries per WRITE / READ / SEND: ctrl + raddr + two data segments fill one WQEBB
};

enum Opcode : uint8_t {  // ctrl.opmod_idx_opcode[7:0]
  OP_NOP = 0x00,
  OP_SEND_INVAL = 0x01,
  OP_RDMA_WRITE = 0x08,
  OP_RDMA_WRITE_IMM = 0x09,
  OP_SEND = 0x0a,
  OP_SEND_IMM = 0x0b,
  OP_RDMA_READ = 0x10,
  OP_ATOMIC_CS = 0x11,
  OP_ATOMIC_FA = 0x12,
};

enum CtrlFlags : uint8_t {  // ctrl.fm_ce_se
  CTRL_SOLICITED = 1 << 1,
  CTRL_CQ_UPDATE = 2 << 2,     // 0x08: generate a CQE for this WQE
  CTRL_FENCE = 4 << 5,         // 0x80: wait for prior reads before starting
  CTRL_INITIATOR_SMALL_FENCE = 1 << 5,
};

enum CqeOpcode : uint8_t {  // cqe.op_own[7:4]
  CQE_REQ = 0x0,
  CQE_RESP_WR_IMM = 0x1,
  CQE_RESP_SEND = 0x2,
  CQE_RESP_SEND_IMM = 0x3,
  CQE_RESP_SEND_INV = 0x4,
  CQE_RESIZE_CQ = 0x5,
  CQE_REQ_ERR = 0xd,
  CQE_RESP_ERR = 0xe,
  CQE_INVALID = 0xf,
};

enum CqeSyndrome : uint8_t {  // err_cqe.syndrome
  SYN_OK = 0x00,
  SYN_LOCAL_LENGTH_ERR = 0x01,
  SYN_LOCAL_QP_OP_ERR = 0x02,
  SYN_LOCAL_PROT_ERR = 0x04,
  SYN_WR_FLUSH_ERR = 0x05,
  SYN_MW_BIND_ERR = 0x06,
  SYN_BAD_RESP_ERR = 0x10,
  SYN_LOCAL_ACCESS_ERR = 0x11,
  SYN_REMOTE_INVAL_REQ_ERR = 0x12,
  SYN_REMOTE_ACCESS_ERR = 0x13,
  SYN_REMOTE_OP_ERR = 0x14,
  SYN_TRANSPORT_RETRY_EXC_ERR = 0x15,
  SYN_RNR_RETRY_EXC_ERR = 0x16,
  SYN_REMOTE_ABORTED_ERR = 0x22,
};

enum DbrIndex : uint32_t { DBR_RCV = 0, DBR_SND = 1 };

// ---------------------------------------------------------------- segments
struct alignas(16) CtrlSeg {     // mlx5_wqe_ctrl_seg
  uint32_t opmod_idx_opcode;     // be32: opmod[31:24] | wqe_index[23:8] | opcode[7:0]
  uint32_t qpn_ds;               // be32: qpn[31:8] | ds[5:0]  (ds = #16-byte segments)
  uint8_t signature;
  uint8_t rsvd[2];
  uint8_t fm_ce_se;
  uint32_t imm;                  // be32 immediate / invalidation key
};
struct alignas(16) RaddrSeg {    // mlx5_wqe_raddr_seg
  uint64_t raddr;                // be64
  uint32_t rkey;                 // be32
  uint32_t reserved;
};
struct alignas(16) DataSeg {     // mlx5_wqe_data_seg
  uint32_t byte_count;           // be32 (bit 31 = inline)
  uint32_t lkey;                 // be32
  uint64_t addr;                 // be64
};
struct alignas(16) AtomicSeg {   // mlx5_wqe_atomic_seg
  uint64_t swap_add;             // be64
  uint64_t compare;              // be64
};
struct InlineSeg {               // mlx5_wqe_inl_data_seg: the payload follows, zero padded to a 16-byte boundary
  uint32_t byte_count;           // be32 (n | INLINE_SEG)
};
// An inline payload: up to MAX_INLINE bytes in memory order (little-endian words), zero past its length.  Whole words,
// so device code can keep it in registers.
struct InlinePayload { uint32_t w[7]; };
// One WQEBB holding ctrl + raddr + one data segment (RDMA write / read), or
// ctrl + data (send: raddr slot left zero and ds=2 with data in slot 1).
struct alignas(64) Wqe64 {
  CtrlSeg ctrl;
  union {
    struct { RaddrSeg raddr; DataSeg data; uint8_t pad[16]; } rdma;
    struct { DataSeg data; uint8_t pad[32]; } send;
    // two-entry gather / scatter list: RDMA ds = 4 (exactly one WQEBB), SEND ds = 3
    struct { RaddrSeg raddr; DataSeg data[2]; } rdma_sg;
    struct { DataSeg data[2]; uint8_t pad[16]; } send_sg;
    struct { RaddrSeg raddr; AtomicSeg atomic; DataSeg data; } atom;
    // inline: the payload travels in the WQE (ds = 2 + ceil((4 + n) / 16) for RDMA, 1 + ... for SEND)
    struct { RaddrSeg raddr; InlineSeg inl; InlinePayload data; } rdma_inl;
    struct { InlineSeg inl; InlinePayload data; uint32_t pad[4]; } send_inl;
    struct { uint32_t pad[12]; } nop;
  };
};
static_assert(sizeof(CtrlSeg) == 16, "ctrl seg");
static_assert(sizeof(RaddrSeg) == 16, "raddr seg");
static_assert(sizeof(DataSeg) == 16, "data seg");
static_assert(sizeof(InlineSeg) == 4, "inline seg");
static_assert(sizeof(InlinePayload) == MAX_INLINE, "inline payload");
static_assert(sizeof(Wqe64) == 64, "wqebb");
// where the inline payload starts within the WQEBB (the engine copies it from there)
enum : uint32_t { INLINE_OFF_RDMA = 36, INLINE_OFF_SEND = 20 };
static_assert(__builtin_offsetof(Wqe64, rdma_inl.data) == INLINE_OFF_RDMA, "rdma inline payload");
static_assert(__builtin_offsetof(Wqe64, send_inl.data) == INLINE_OFF_SEND, "send inline payload");

struct alignas(64) Cqe64 {       // mlx5_cqe64
  uint8_t outer_l3_tunneled;
  uint8_t rsvd0;
  uint16_t wqe_id;               // be16
  uint8_t lro_tcppsh_abort_dupack;
  uint8_t lro_min_ttl;
  uint16_t lro_tcp_win;
  uint32_t lro_ack_seq_num;
  uint32_t rss_hash_result;
  uint8_t rss_hash_type;
  uint8_t ml_path;
  uint8_t rsvd20[2];
  uint16_t check_sum;
  uint16_t slid;
  uint32_t flags_rqpn;           // be32
  uint8_t hds_ip_ext;
  uint8_t l4_l3_hdr_type;
  uint16_t vlan_info;
  uint32_t srqn;                 // be32
  uint32_t imm_inval_pkey;       // be32
  uint8_t rsvd40[4];
  uint32_t byte_cnt;             // be32
  uint32_t timestamp_h;          // be32
  uint32_t timestamp_l;          // be32
  uint32_t sop_drop_qpn;         // be32: send opcode[31:24] | qpn[23:0]
  uint16_t wqe_counter;          // be16
  uint8_t signature;
  uint8_t op_own;                // opcode[7:4] | se[1] | owner[0]
};
struct alignas(64) ErrCqe {      // mlx5_err_cqe (same 64 bytes, error view)
  uint8_t rsvd0[32];
  uint32_t srqn;
  uint8_t rsvd1[18];
  uint8_t vendor_err_synd;
  uint8_t syndrome;
  uint32_t s_wqe_opcode_qpn;     // be32: wqe opcode[31:24] | qpn[23:0]
  uint16_t wqe_counter;          // be16
  uint8_t signature;
  uint8_t op_own;
};
static_assert(sizeof(Cqe64) == 64, "cqe64");
static_assert(sizeof(ErrCqe) == 64, "err cqe");

// ---------------------------------------------------------------- encoders
RN_HD uint32_t ctrl_word0(uint8_t opcode, uint16_t wqe_idx, uint8_t opmod = 0) {
  return be32(((uint32_t)opmod << 24) | ((uint32_t)wqe_idx << 8) | opcode);
}
RN_HD uint32_t ctrl_word1(uint32_t qpn, uint8_t ds) { return be32((qpn << 8) | (ds & 0x3f)); }
// The doorbell register word: the first 8 bytes of a ctrl segment naming the QP and the last WQE posted (opcode NOP, ds 0).
RN_HD uint64_t doorbell_word(uint32_t qpn, uint16_t last) {
  return (uint64_t)ctrl_word0(OP_NOP, last) | ((uint64_t)ctrl_word1(qpn, 0) << 32);
}
// The last WQE index a doorbell register word names.
RN_HD uint16_t doorbell_index(uint64_t db) { return (uint16_t)(be32((uint32_t)db) >> 8); }

RN_HD void encode_ctrl(CtrlSeg* c, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint8_t ds,
                       uint8_t fm_ce_se, uint32_t imm) {
  c->opmod_idx_opcode = ctrl_word0(opcode, wqe_idx);
  c->qpn_ds = ctrl_word1(qpn, ds);
  c->signature = 0;
  c->rsvd[0] = c->rsvd[1] = 0;
  c->fm_ce_se = fm_ce_se;
  c->imm = be32(imm);
}
RN_HD void encode_raddr(RaddrSeg* r, uint64_t raddr, uint32_t rkey) {
  r->raddr = be64(raddr);
  r->rkey = be32(rkey);
  r->reserved = 0;
}
// A byte count the segment cannot carry saturates, so it reaches the HCA as longer than MAX_MSG and fails there; masking
// it would post a shorter, valid message.
RN_HD uint32_t data_byte_count(uint32_t bytes) { return bytes > MAX_BYTE_COUNT ? MAX_BYTE_COUNT : bytes; }
RN_HD void encode_data(DataSeg* d, uint64_t addr, uint32_t lkey, uint32_t bytes) {
  d->byte_count = be32(data_byte_count(bytes));
  d->lkey = be32(lkey);
  d->addr = be64(addr);
}

// Full WQE builders, each writing all 64 bytes.  Device code builds into a local Wqe64 (registers) and stores it
// with four 16-byte vector stores (dev::store_wqe in hca/post.cuh).
RN_HD void build_rdma_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint64_t laddr,
                          uint32_t lkey, uint64_t raddr, uint32_t rkey, uint32_t bytes,
                          uint8_t fm_ce_se, uint32_t imm) {
  encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, 3, fm_ce_se, imm);
  encode_raddr(&w->rdma.raddr, raddr, rkey);
  encode_data(&w->rdma.data, laddr, lkey, bytes);
  for (int i = 0; i < 16; ++i) w->rdma.pad[i] = 0;
}
RN_HD void build_send_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint64_t laddr,
                          uint32_t lkey, uint32_t bytes, uint8_t fm_ce_se, uint32_t imm) {
  encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, 2, fm_ce_se, imm);
  encode_data(&w->send.data, laddr, lkey, bytes);
  for (int i = 0; i < 32; ++i) w->send.pad[i] = 0;
}
RN_HD void encode_atomic(AtomicSeg* a, uint64_t swap_add, uint64_t compare) {
  a->swap_add = be64(swap_add);
  a->compare = be64(compare);
}
// 8-byte atomic (ds = 4): ctrl + raddr + atomic + data.  Operand placement as in libmlx5: fetch-and-add
// carries the addend in swap_add (compare is zero); compare-and-swap carries the swap value in swap_add and
// the compare value in compare.  The data segment names the local 8 bytes that receive the original remote
// value.  The remote word and the fetched value are native (little-endian) u64s (DESIGN.md section 3.1).
RN_HD void build_atomic_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint64_t laddr, uint32_t lkey,
                            uint64_t raddr, uint32_t rkey, uint64_t swap_add, uint64_t compare, uint8_t fm_ce_se,
                            uint32_t bytes = 8) {
  encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, 4, fm_ce_se, 0);
  encode_raddr(&w->atom.raddr, raddr, rkey);
  encode_atomic(&w->atom.atomic, swap_add, opcode == OP_ATOMIC_CS ? compare : 0);
  encode_data(&w->atom.data, laddr, lkey, bytes);
}
// Segments an inline payload of n bytes takes together with its 4-byte header.
RN_HD constexpr uint8_t inline_segs(uint32_t n) { return (uint8_t)((4 + n + WQE_SEG - 1) / WQE_SEG); }
// Inline WQE (1 <= n <= MAX_INLINE; the caller checks): RDMA_WRITE / WRITE_IMM carry ctrl + raddr + the inline segment
// (ds 3 up to 12 bytes, else 4), SEND / SEND_IMM ctrl + the inline segment (ds 2 up to 12 bytes, else 3).  No lkey, no
// local address: the payload's n bytes travel in the WQE, and the rest of the WQEBB is zero.
RN_HD void build_inline_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint64_t raddr, uint32_t rkey,
                            const InlinePayload& d, uint32_t n, uint8_t fm_ce_se, uint32_t imm) {
  if (opcode == OP_SEND || opcode == OP_SEND_IMM) {
    encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, (uint8_t)(1 + inline_segs(n)), fm_ce_se, imm);
    w->send_inl.inl.byte_count = be32(n | INLINE_SEG);
    w->send_inl.data = d;
    for (int i = 0; i < 4; ++i) w->send_inl.pad[i] = 0;
  } else {
    encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, (uint8_t)(2 + inline_segs(n)), fm_ce_se, imm);
    encode_raddr(&w->rdma_inl.raddr, raddr, rkey);
    w->rdma_inl.inl.byte_count = be32(n | INLINE_SEG);
    w->rdma_inl.data = d;
  }
}
// The same WQE with its payload taken from the n bytes at `data` (host callers; device code loads the payload into
// registers with dev::inline_load).
RN_HD void build_inline_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, uint64_t raddr, uint32_t rkey,
                            const void* data, uint32_t n, uint8_t fm_ce_se, uint32_t imm) {
  InlinePayload d = {};
  for (uint32_t i = 0; i < n; ++i) d.w[i / 4] |= (uint32_t)static_cast<const uint8_t*>(data)[i] << (8 * (i % 4));
  build_inline_wqe(w, opcode, wqe_idx, qpn, raddr, rkey, d, n, fm_ce_se, imm);
}
// One scatter-gather entry: `bytes` at `addr` under `lkey`.
struct Sge { uint64_t addr; uint32_t lkey; uint32_t bytes; };
// Drop zero-length entries, as libmlx5 does; returns how many remain (entries past MAX_SGE are the caller's to refuse).
RN_HD int sg_compact(const Sge* in, int n, Sge* out) {
  int k = 0;
  for (int i = 0; i < n && i < (int)MAX_SGE; ++i)
    if (in[i].bytes) out[k++] = in[i];
  return k;
}
// Gather WRITE / WRITE_IMM or scatter READ of up to MAX_SGE entries: the message is the entries concatenated in list
// order, at [raddr, raddr + sum).  Two non-empty entries: ctrl + raddr + two data segments (ds = 4, one WQEBB).  At most
// one: exactly build_rdma_wqe's WQE, of that entry (of entry 0 with 0 bytes when every entry is empty).
RN_HD void build_rdma_sg_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, const Sge* sg, int n,
                             uint64_t raddr, uint32_t rkey, uint8_t fm_ce_se, uint32_t imm) {
  Sge e[MAX_SGE];
  const int k = sg_compact(sg, n, e);
  if (k < 2) {
    const Sge one = k ? e[0] : Sge{n ? sg[0].addr : 0, n ? sg[0].lkey : 0, 0};
    build_rdma_wqe(w, opcode, wqe_idx, qpn, one.addr, one.lkey, raddr, rkey, one.bytes, fm_ce_se, imm);
    return;
  }
  encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, 4, fm_ce_se, imm);
  encode_raddr(&w->rdma_sg.raddr, raddr, rkey);
  encode_data(&w->rdma_sg.data[0], e[0].addr, e[0].lkey, e[0].bytes);
  encode_data(&w->rdma_sg.data[1], e[1].addr, e[1].lkey, e[1].bytes);
}
// Gather SEND / SEND_IMM: ctrl + two data segments (ds = 3); at most one non-empty entry: build_send_wqe's WQE.
RN_HD void build_send_sg_wqe(Wqe64* w, uint8_t opcode, uint16_t wqe_idx, uint32_t qpn, const Sge* sg, int n,
                             uint8_t fm_ce_se, uint32_t imm) {
  Sge e[MAX_SGE];
  const int k = sg_compact(sg, n, e);
  if (k < 2) {
    const Sge one = k ? e[0] : Sge{n ? sg[0].addr : 0, n ? sg[0].lkey : 0, 0};
    build_send_wqe(w, opcode, wqe_idx, qpn, one.addr, one.lkey, one.bytes, fm_ce_se, imm);
    return;
  }
  encode_ctrl(&w->ctrl, opcode, wqe_idx, qpn, 3, fm_ce_se, imm);
  encode_data(&w->send_sg.data[0], e[0].addr, e[0].lkey, e[0].bytes);
  encode_data(&w->send_sg.data[1], e[1].addr, e[1].lkey, e[1].bytes);
  for (int i = 0; i < 16; ++i) w->send_sg.pad[i] = 0;
}
// NOP (ds = 1): a ctrl segment and nothing else.  Signaled, its CQE shows that every earlier WQE of the QP completed.
RN_HD void build_nop_wqe(Wqe64* w, uint16_t wqe_idx, uint32_t qpn, uint8_t fm_ce_se) {
  encode_ctrl(&w->ctrl, OP_NOP, wqe_idx, qpn, 1, fm_ce_se, 0);
  for (int i = 0; i < 12; ++i) w->nop.pad[i] = 0;
}

// ---------------------------------------------------------------- decoders
struct WqeView {
  uint8_t opcode, opmod, ds, fm_ce_se;
  uint16_t wqe_idx;
  uint32_t qpn, imm;
  uint64_t raddr, laddr;
  uint32_t rkey, lkey, bytes;
  uint64_t swap_add, compare;    // atomics only (native byte order)
  uint8_t inl_off;               // inline WQE: offset of its `bytes` payload bytes in the WQEBB; 0: gather (laddr / lkey)
  uint8_t nsge;                  // gather entries: 2 for a two-entry list (then bytes = len0 + the second entry's), else 1
  uint32_t len0;                 // nsge == 2 only: entry 0's length, and entry 1 (bytes - len0 at laddr1 / lkey1)
  uint64_t laddr1;
  uint32_t lkey1;
};
// A data segment that names a second gather entry: its byte count without the inline flag, else false.
RN_HD bool sg_second(const DataSeg& d, WqeView* v) {
  const uint32_t bc = be32(d.byte_count);
  if (bc & INLINE_SEG) return false;
  v->nsge = 2;
  v->len0 = v->bytes;
  v->laddr1 = be64(d.addr);
  v->lkey1 = be32(d.lkey);
  v->bytes += bc;                // each count is below 2^31: the sum fits
  return true;
}
RN_HD bool is_atomic(uint8_t opcode) { return opcode == OP_ATOMIC_CS || opcode == OP_ATOMIC_FA; }
// An inline byte count is well formed when 1 <= n <= MAX_INLINE and ds counts exactly its segments.
RN_HD bool inline_ok(uint32_t n, uint8_t ds, uint8_t head_segs) {
  return n >= 1 && n <= MAX_INLINE && ds == head_segs + inline_segs(n);
}
RN_HD bool decode_wqe(const Wqe64* w, WqeView* v) {
  uint32_t w0 = be32(w->ctrl.opmod_idx_opcode), w1 = be32(w->ctrl.qpn_ds);
  v->opcode = (uint8_t)(w0 & 0xff);
  v->wqe_idx = (uint16_t)((w0 >> 8) & 0xffff);
  v->opmod = (uint8_t)(w0 >> 24);
  v->qpn = w1 >> 8;
  v->ds = (uint8_t)(w1 & 0x3f);
  v->fm_ce_se = w->ctrl.fm_ce_se;
  v->imm = be32(w->ctrl.imm);
  v->raddr = 0; v->rkey = 0; v->laddr = 0; v->lkey = 0; v->bytes = 0;
  v->swap_add = 0; v->compare = 0; v->inl_off = 0;
  v->nsge = 1; v->len0 = 0; v->laddr1 = 0; v->lkey1 = 0;
  switch (v->opcode) {
    case OP_ATOMIC_CS: case OP_ATOMIC_FA:
      if (v->ds != 4 || (be32(w->atom.data.byte_count) & INLINE_SEG)) return false;
      v->raddr = be64(w->atom.raddr.raddr);
      v->rkey = be32(w->atom.raddr.rkey);
      v->swap_add = be64(w->atom.atomic.swap_add);
      v->compare = be64(w->atom.atomic.compare);
      v->laddr = be64(w->atom.data.addr);
      v->lkey = be32(w->atom.data.lkey);
      v->bytes = be32(w->atom.data.byte_count);
      return true;
    case OP_RDMA_WRITE: case OP_RDMA_WRITE_IMM: case OP_RDMA_READ: {
      const uint32_t bc = be32(w->rdma.data.byte_count);
      if (bc & INLINE_SEG) {   // a READ has nothing to carry inline
        v->bytes = bc & ~INLINE_SEG;
        if (v->opcode == OP_RDMA_READ || !inline_ok(v->bytes, v->ds, 2)) return false;
        v->inl_off = INLINE_OFF_RDMA;
      } else {
        // ds 3: one entry; ds 4: two (the inline flag above already told a 13-28-byte inline WRITE apart)
        if (v->ds != 3 && v->ds != 4) return false;
        v->laddr = be64(w->rdma.data.addr);
        v->lkey = be32(w->rdma.data.lkey);
        v->bytes = bc;
        if (v->ds == 4 && !sg_second(w->rdma_sg.data[1], v)) return false;
      }
      v->raddr = be64(w->rdma.raddr.raddr);
      v->rkey = be32(w->rdma.raddr.rkey);
      return true;
    }
    case OP_SEND: case OP_SEND_IMM: {
      const uint32_t bc = be32(w->send.data.byte_count);
      if (bc & INLINE_SEG) {
        v->bytes = bc & ~INLINE_SEG;
        if (!inline_ok(v->bytes, v->ds, 1)) return false;
        v->inl_off = INLINE_OFF_SEND;
        return true;
      }
      if (v->ds != 2 && v->ds != 3) return false;
      v->laddr = be64(w->send.data.addr);
      v->lkey = be32(w->send.data.lkey);
      v->bytes = bc;
      return v->ds == 2 || sg_second(w->send_sg.data[1], v);
    }
    case OP_NOP:
      return v->ds == 1;
    default:
      return false;
  }
}

RN_HD uint8_t cqe_op_own(uint8_t opcode, uint8_t owner) { return (uint8_t)((opcode << 4) | (owner & 1)); }
RN_HD uint8_t cqe_opcode(uint8_t op_own) { return op_own >> 4; }
RN_HD uint8_t cqe_owner(uint8_t op_own) { return op_own & 1; }
RN_HD bool cqe_is_error(uint8_t opcode) { return opcode == CQE_REQ_ERR || opcode == CQE_RESP_ERR; }

// ---------------------------------------------------------------- CQEs as 16-byte parts
// A CQE is written and read as 16-byte parts of four words in memory order (a uint4 in CUDA code); bytes 0-31 are zero.
//   mid  = bytes 32-47: srqn | imm | reserved | byte_cnt   (imm and byte_cnt are reserved, so zero, in an error CQE)
//   tail = bytes 48-63: timestamp_h | timestamp_l | sop_drop_qpn | wqe_counter, signature, op_own.  An error CQE has
//          zero, then reserved[2], vendor_err_synd, syndrome for the timestamp.  op_own holds the owner bit: tail last.
#if defined(__CUDACC__)
typedef uint4 Words16;
#else
struct alignas(16) Words16 { uint32_t x, y, z, w; };
#endif
enum : uint32_t { CQE_MID_OFF = 32, CQE_TAIL_OFF = 48, CQE_OP_OWN_OFF = 63 };
static_assert(__builtin_offsetof(Cqe64, srqn) == CQE_MID_OFF, "cqe mid");
static_assert(__builtin_offsetof(Cqe64, timestamp_h) == CQE_TAIL_OFF, "cqe tail");
static_assert(__builtin_offsetof(Cqe64, op_own) == CQE_OP_OWN_OFF, "cqe op_own");
static_assert(__builtin_offsetof(ErrCqe, vendor_err_synd) == CQE_TAIL_OFF + 6, "err cqe syndromes");

RN_HD Words16 encode_cqe_mid(uint8_t opcode, uint32_t byte_cnt, uint32_t imm) {
  const bool err = cqe_is_error(opcode);
  return Words16{0u, err ? 0u : be32(imm), 0u, err ? 0u : be32(byte_cnt)};
}
// vendor_synd: the vendor syndrome of an error CQE (bits of no meaning to a consumer).
RN_HD Words16 encode_cqe_tail(uint8_t opcode, uint8_t owner, uint16_t wqe_counter, uint32_t qpn, uint8_t wqe_opcode,
                              uint8_t syndrome, uint8_t vendor_synd, uint64_t timestamp) {
  const bool err = cqe_is_error(opcode);
  return Words16{err ? 0u : be32((uint32_t)(timestamp >> 32)),
                 err ? ((uint32_t)syndrome << 24) | ((uint32_t)vendor_synd << 16) : be32((uint32_t)timestamp),
                 be32(((uint32_t)wqe_opcode << 24) | (qpn & 0xffffff)),
                 (uint32_t)be16(wqe_counter) | ((uint32_t)cqe_op_own(opcode, owner) << 24)};
}
// The whole CQE (host producers and the test hook).
RN_HD void encode_cqe(Cqe64* c, uint8_t opcode, uint8_t owner, uint16_t wqe_counter, uint32_t qpn, uint8_t wqe_opcode,
                      uint32_t byte_cnt, uint32_t imm, uint8_t syndrome, uint8_t vendor_synd, uint64_t timestamp) {
  const Words16 mid = encode_cqe_mid(opcode, byte_cnt, imm);
  const Words16 tail = encode_cqe_tail(opcode, owner, wqe_counter, qpn, wqe_opcode, syndrome, vendor_synd, timestamp);
  memset(c, 0, CQE_MID_OFF);
  memcpy(reinterpret_cast<uint8_t*>(c) + CQE_MID_OFF, &mid, 16);
  memcpy(reinterpret_cast<uint8_t*>(c) + CQE_TAIL_OFF, &tail, 16);
}
// Every slot of a new CQ ring: zero, opcode INVALID, owner 1 (the producer's first pass writes owner 0).
RN_HD void init_cq_ring(uint8_t* ring, uint32_t ncqe) {
  memset(ring, 0, (size_t)ncqe * CQE_SIZE);
  for (uint32_t i = 0; i < ncqe; ++i) ring[(size_t)i * CQE_SIZE + CQE_OP_OWN_OFF] = cqe_op_own(CQE_INVALID, 1);
}

RN_HD uint8_t cqe_tail_op_own(const Words16& tail) { return (uint8_t)(tail.w >> 24); }
RN_HD uint8_t cqe_tail_opcode(const Words16& tail) { return cqe_opcode(cqe_tail_op_own(tail)); }
RN_HD uint16_t cqe_tail_counter(const Words16& tail) { return be16((uint16_t)tail.w); }
RN_HD uint32_t cqe_tail_qpn(const Words16& tail) { return be32(tail.z) & 0xffffff; }
RN_HD uint8_t cqe_tail_wqe_opcode(const Words16& tail) { return (uint8_t)(be32(tail.z) >> 24); }
RN_HD uint8_t cqe_tail_syndrome(const Words16& tail) { return (uint8_t)(tail.y >> 24); }         // error CQEs only
RN_HD uint8_t cqe_tail_vendor_synd(const Words16& tail) { return (uint8_t)(tail.y >> 16); }      // error CQEs only
RN_HD uint32_t cqe_mid_imm(const Words16& mid) { return be32(mid.y); }
RN_HD uint32_t cqe_mid_byte_cnt(const Words16& mid) { return be32(mid.w); }

struct CqeView {
  uint8_t opcode, owner, syndrome, vendor_synd, wqe_opcode;
  uint16_t wqe_counter;
  uint32_t qpn, byte_cnt, imm;
  bool is_error;
};
RN_HD void decode_cqe(const Cqe64* c, CqeView* v) {
  Words16 mid, tail;
  memcpy(&mid, reinterpret_cast<const uint8_t*>(c) + CQE_MID_OFF, 16);
  memcpy(&tail, reinterpret_cast<const uint8_t*>(c) + CQE_TAIL_OFF, 16);
  v->opcode = cqe_tail_opcode(tail);
  v->owner = cqe_owner(cqe_tail_op_own(tail));
  v->wqe_counter = cqe_tail_counter(tail);
  v->qpn = cqe_tail_qpn(tail);
  v->wqe_opcode = cqe_tail_wqe_opcode(tail);
  v->byte_cnt = cqe_mid_byte_cnt(mid);
  v->imm = cqe_mid_imm(mid);
  v->is_error = cqe_is_error(v->opcode);
  v->syndrome = v->is_error ? cqe_tail_syndrome(tail) : 0;
  v->vendor_synd = v->is_error ? cqe_tail_vendor_synd(tail) : 0;
}

// A CQE at consumer index `ci` of a 2^log_n ring is valid when its opcode is not INVALID and its owner bit is ci's pass parity.
RN_HD bool cqe_valid(uint8_t op_own, uint32_t ci, uint32_t log_n) {
  return cqe_opcode(op_own) != CQE_INVALID && cqe_owner(op_own) == ((ci >> log_n) & 1u);
}

// ---------------------------------------------------------------- index records and counters
// A 16-bit wire counter (a CQE's wqe_counter, a doorbell record) expanded to the 64-bit index at or above `near` that
// it names (wire.expand16).  Only the low 16 bits of `counter` count, so a caller may pass wqe_counter + 1 unwrapped.
RN_HD uint64_t expand16(uint32_t counter, uint64_t near) { return near + ((counter - (uint32_t)near) & 0xffffu); }
// SQ / RQ doorbell record: be32 of the producer index's low 16 bits.
RN_HD uint32_t wq_dbr_word(uint64_t pi) { return be32((uint32_t)(pi & 0xffff)); }
RN_HD uint16_t wq_dbr_index(uint32_t rec) { return (uint16_t)be32(rec); }
// CQ consumer record: be32 of the consumer index's low 24 bits.
RN_HD uint32_t cq_dbr_word(uint32_t ci) { return be32(ci & 0xffffff); }
RN_HD uint32_t cq_dbr_index(uint32_t rec) { return be32(rec) & 0xffffff; }

// A receive WQE: one data segment (what encode_data writes) per 16-byte stride.  A buffer longer than the segment can
// say saturates too: it still holds any message.
RN_HD Words16 recv_wqe_words(uint64_t addr, uint32_t lkey, uint32_t bytes) {
  return Words16{be32(data_byte_count(bytes)), be32(lkey), be32((uint32_t)(addr >> 32)), be32((uint32_t)addr)};
}
RN_HD uint32_t recv_wqe_bytes(const Words16& d) { return be32(d.x) & 0x7fffffffu; }
RN_HD uint32_t recv_wqe_lkey(const Words16& d) { return be32(d.y); }
RN_HD uint64_t recv_wqe_addr(const Words16& d) { return ((uint64_t)be32(d.z) << 32) | be32(d.w); }

}  // namespace rn
