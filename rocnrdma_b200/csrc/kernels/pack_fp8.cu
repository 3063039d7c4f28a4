// K3 / K5 (SURVEY.md section 2.3): payload pack fused with GPU-initiated networking, and the reduce of several sources.
//
//  pack_fp8_write_kernel   bf16 -> fp8 e4m3 with one UE8M0 scale per 32 elements (MX-style
//                          block scaling) written into a registered staging region as
//                          self-contained chunk records; the CTA that finishes the last
//                          tile of a chunk builds the RDMA WRITE(_IMM) WQE for that record
//                          and rings the doorbell, so the wire starts moving chunk i while
//                          chunks i+1.. are still being packed.  The kernel ends only when
//                          the last CQE has been seen: its device time is the whole
//                          pack+transfer pipeline.
//  pack_fp8_scatter_kernel K3 of an all-to-all: every shard of x in one launch, in phase order, each record posted
//                          to its own rank's queue pair as it completes; the own shard's records stay in place and
//                          get their arrival words stamped.
//  unpack_fp8_kernel       consumer: optionally waits for each record's arrival (receive
//                          CQE carrying the chunk id as immediate), then fp8 -> bf16; <true> also
//                          forwards each record unchanged, from where it landed, as soon as it is seen.
//  relay_records_kernel    one thread that forwards given records, in a given order, each once its arrival word is set
//                          (the forwarding unpack's per-record gate without the unpack: a ring all-gather's hop).
//  reduce_fp8_kernel       the sum of P sources of records (plus a bf16 addend) as each record's sources land,
//                          as bf16 and / or re-quantised records; the CTA that completes a record of the sum
//                          posts its RDMA WRITE(_IMM), as K3 does.
//
// Record layout for a chunk of C elements (C % 8192 == 0):
//     [ C bytes fp8 e4m3 ][ C/32 bytes UE8M0 scales ][ pad to 64 B ]
// Quantisation (mx_scale.cuh; bit-exact reference: ops/pack.py, quantize_blocks / ref_pack_fp8 / ref_unpack_fp8 /
// ref_reduce_fp8):
//     e = the smallest integer with amax / 2^e <= 448, clamped to [-127, 127], from the fp32 bits of v = amax * (1/448):
//         -127 when v <= 2^-127, else exponent(v) + (mantissa(v) != 0), at most 127
//     y = x * 2^-e ; at e = 120 only, |y| > 240 becomes +-240 (codes 248 and 256 would decode to 2^128 = Inf in fp32)
//     q = cvt.rn.satfinite.e4m3(y) ; scale byte = e + 127
//     so every finite input decodes finite, and the saturation's relative error stays under 2^-4 (worst: 255.99 -> 240)
// Non-finite input:
//     NaN   amax is an fmaxf reduction, which drops NaN: a NaN stays in its own element, its neighbours quantise
//           as if it were absent (an all-NaN block gets scale byte 0 and NaN codes)
//     +-Inf e clamps to 127 (scale byte 254) and 2^-127 is 0.0 here: the Inf becomes NaN, its neighbours +-0
//           (a finite sum that overflows fp32 in a reduce without error feedback is such an Inf)
// Decode: scale byte 0x00 is 2^-127 (the OCP MX value, fp32 0x00400000), as in the block-scaled GEMM; 0xFF is Inf.
// Error feedback (K3 and the reduce with a residual, EF = true): an fp32 residual of n_elems, read and written in place
// by the thread that quantises the element.  K3 quantises v = x + r_in, the reduce v = (its sum) + r_in, the residual
// added last; then r_out = v - d, d = code * ue8m0(scale byte) as the decoders make it, exact in fp32 wherever v and d
// are finite (|d| <= 2|v|, same sign: Sterbenz), and 0 wherever either is not (NaN, a block holding Inf), so one bad
// step cannot poison the residual for good.  Every add of an EF kernel (K3's x + r_in; the reduce's addend + d0, + d1
// and + r_in) saturates (ef_add): finite operands whose sum overflows give +-FLT_MAX instead of +-Inf.  The e = 120
// saturation leaves up to FLT_MAX - 240 * 2^120 in the residual, and without this the next call's x + r_in, or a later
// hop's sum of the records it enlarged, would overflow and turn a finite input into NaN.  So with error feedback finite
// inputs always give finite records and residuals, and |r_out| <= FLT_MAX - 240 * 2^120.  A NaN or Inf operand, and a
// decode that overflows (code 448 under scale byte 254), still propagate as above.
//
// No counterpart in the reference (it moves no payload: SURVEY.md section 3.2).
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../hca/post.cuh"
#include "mx_scale.cuh"

using namespace rn;
using namespace rn::dev;

#define RN_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int kPackThreads = 256;
constexpr int kBlockElems = 32;                            // elements per scale
constexpr int kTileElems = kPackThreads * kBlockElems;     // 8192 elements per CTA iteration

__host__ __device__ inline uint64_t record_bytes(uint64_t chunk_elems) {
  uint64_t b = chunk_elems + chunk_elems / kBlockElems;
  return (b + 63) / 64 * 64;
}

struct PackArgs {
  const __nv_bfloat16* src;
  uint8_t* staging;          // registered; records laid out back to back
  uint64_t n_elems;          // multiple of kTileElems
  uint32_t chunk_elems;      // multiple of kTileElems
  uint32_t n_chunks;
  QpDev* qp;                 // nullptr = pack only (numerics tests)
  uint64_t staging_va;       // VA of `staging` as registered (what goes into the WQE)
  uint32_t lkey;
  uint32_t rkey;
  uint64_t remote_va;        // destination of record 0; records keep their stride remotely
  uint32_t with_imm;         // 1: RDMA_WRITE_IMM carrying the chunk id (wakes a device consumer)
  uint32_t post_only;        // 1: post everything (incl. the flush) but do not wait for the wire to drain -- for profilers that
                             //    serialise kernels (the NIC / engine cannot run while this kernel is resident) and for callers
                             //    that overlap the drain with other work and reap the flush CQE later
  uint32_t direct;           // 1: `staging` IS the peer's registered buffer (NVLink-mapped): the pack's own coalesced stores are the
                             //    transfer; each finished record is announced by a zero-length RDMA_WRITE_IMM posted after a cumulative
                             //    system-scope fence (as gemm_send.cu's direct mode; no engine / NIC moves the payload)
  uint32_t signal_every;     // CQE every k-th chunk (the last one is always signaled)
  unsigned int* counters;    // [0..n_chunks): groups done per chunk ; [n_chunks]: CTAs done
  unsigned long long* acc;   // device accumulators: [0] max WQE index+1, [1] WQEs posted, [2] ~first post time
                             // (atomics stay in device memory; `out` is mapped host memory, plain stores only)
  unsigned long long* out;   // [status, t_start, t_end, wqes_posted, t_first_post, t_pack_end, 0, 0]
  uint64_t timeout_ns;
  float* residual;           // pack_fp8_write_kernel<true> only: n_elems fp32, read and written in place
};

// The quantiser of one MX block (K3's, and the reduce kernel's): 32 fp32 values in element order -> 32 e4m3 codes (q[i]
// holds elements 4i..4i+3, lowest byte first) and the returned UE8M0 scale byte.  The rule is the header's.
__device__ __forceinline__ uint32_t quantize_block32(const float (&x)[32], uint32_t (&q)[8]) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fmaxf(fabsf(x[2 * i]), fabsf(x[2 * i + 1])));
  const int e = mx_scale_exponent(amax);
  const float inv = __uint_as_float((uint32_t)(127 - e) << 23);   // 2^-e, exact (biased exponent 0..254)
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(x[4 * i] * inv, x[4 * i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
    uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(x[4 * i + 2] * inv, x[4 * i + 3] * inv), __NV_SATFINITE, __NV_E4M3);
    q[i] = mx_saturate_codes(lo | (hi << 16), e);
  }
  return (uint32_t)(e + 127);
}

// 32 contiguous bytes per thread, streaming (evict-first): a thread's 32 bytes of fp8 in, and its 64 bytes of bf16 out as two
// whole 32-byte sectors.  Hopper's widest global access is 128 bits, so each is a pair of adjacent 16-byte accesses.
__device__ __forceinline__ void ld256_cs(const void* p, uint32_t* r) {
  asm volatile("ld.global.cs.v4.b32 {%0,%1,%2,%3}, [%8];\n\tld.global.cs.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]) : "l"(p));
}
__device__ __forceinline__ void st256_cs(void* p, const uint32_t* r) {
  asm volatile("st.global.cs.v4.b32 [%0], {%1,%2,%3,%4};\n\tst.global.cs.v4.b32 [%0+16], {%5,%6,%7,%8};"
               ::"l"(p), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]), "r"(r[4]), "r"(r[5]), "r"(r[6]), "r"(r[7]) : "memory");
}

// A thread's 32 fp32 residuals (128 contiguous bytes) in and out, as four 32-byte pairs of accesses.
__device__ __forceinline__ void ld_residual(const float* p, uint32_t (&r)[32]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) ld256_cs(p + 8 * j, r + 8 * j);
}
__device__ __forceinline__ void st_residual(float* p, const float (&r)[32]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) st256_cs(p + 8 * j, reinterpret_cast<const uint32_t*>(r + 8 * j));
}

// A thread's block of tile t: the offset of its first element in a tensor (bf16 data, an fp32 residual), and of its
// first code byte in a record (one byte per element).  Record-major flattened tile T of a launch's records is also tile
// T of its tensors.
__device__ __forceinline__ uint64_t block_off(uint64_t t) { return t * kTileElems + (uint64_t)threadIdx.x * kBlockElems; }
// ... and of its scale byte in a record, after the record's chunk_elems codes.
__device__ __forceinline__ uint64_t scale_off(uint32_t chunk_elems, uint32_t t) {
  return chunk_elems + (uint64_t)t * kPackThreads + threadIdx.x;
}

// Store one quantised block (quantize_block32's codes and scale byte) as tile t of the record at recp.
__device__ __forceinline__ void store_block(uint8_t* recp, uint32_t chunk_elems, uint32_t t, const uint32_t (&q)[8],
                                            uint32_t scale) {
  uint4* o = reinterpret_cast<uint4*>(recp + block_off(t));
  o[0] = make_uint4(q[0], q[1], q[2], q[3]);
  o[1] = make_uint4(q[4], q[5], q[6], q[7]);
  recp[scale_off(chunk_elems, t)] = (uint8_t)scale;
}

// 32 bf16 (w[i] holds elements 2i and 2i+1, lowest half first) -> fp32, exact.
__device__ __forceinline__ void widen_bf16x32(const uint32_t (&w)[16], float (&x)[32]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) { x[2 * i] = __uint_as_float(w[i] << 16); x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u); }
}

// 32 fp32 -> bf16 (round to nearest even), stored at dst as two whole 32-byte sectors.
__device__ __forceinline__ void st_bf16x32(__nv_bfloat16* dst, const float (&x)[32]) {
  uint32_t o[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    __nv_bfloat162 b = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    o[i] = *reinterpret_cast<uint32_t*>(&b);
  }
  st256_cs(dst, o);
  st256_cs(dst + 16, o + 8);
}

// Error feedback's fp32 add: round to nearest, but a sum of finite operands that overflows is +-FLT_MAX, which is what
// round-toward-zero gives there; with a NaN or Inf operand both give the same NaN or Inf.
__device__ __forceinline__ float ef_add(float a, float b) {
  const float s = __fadd_rn(a, b);
  return isinf(s) ? __fadd_rz(a, b) : s;
}

// Error feedback after quantize_block32: v[i] becomes r_out = v - d, d = the block's decode as every decoder makes it
// (mx_decode_block32).  The difference is exact where v and d are finite, and non-finite exactly where one of them is
// not: then r_out = 0.
__device__ __forceinline__ void ef_residual(float (&v)[32], const uint32_t (&q)[8], uint32_t scale) {
  mx_decode_block32(q, scale, [&](int i, float d) {
    const float r = __fsub_rn(v[i], d);
    v[i] = (__float_as_uint(r) & 0x7f800000u) != 0x7f800000u ? r : 0.f;
  });
}

template <int G, bool EF>
__device__ __forceinline__ void pack_group(const PackArgs& a, uint64_t first_tile, uint32_t tiles_per_chunk, uint64_t rec) {
  // G tiles (G x 16 KiB of bf16) per step: all 4G 16-byte loads are issued before the first
  // use, so each thread keeps G x 64 B in flight (the single-tile version left HBM idle:
  // 16 KiB in flight per CTA measured ~2.7 TB/s aggregate at best).  With EF, G x 128 B of residual more.
  uint4 v[G][4];
  uint32_t rv[G][EF ? 32 : 1];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4* p = reinterpret_cast<const uint4*>(a.src + block_off(first_tile + g));
    v[g][0] = __ldcs(p); v[g][1] = __ldcs(p + 1); v[g][2] = __ldcs(p + 2); v[g][3] = __ldcs(p + 3);
    if constexpr (EF) ld_residual(a.residual + block_off(first_tile + g), rv[g]);
  }
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint64_t tile = first_tile + g;
    const uint32_t chunk = (uint32_t)(tile / tiles_per_chunk);
    const uint32_t tile_in_chunk = (uint32_t)(tile % tiles_per_chunk);
    const uint32_t w[16] = {v[g][0].x, v[g][0].y, v[g][0].z, v[g][0].w, v[g][1].x, v[g][1].y, v[g][1].z, v[g][1].w,
                            v[g][2].x, v[g][2].y, v[g][2].z, v[g][2].w, v[g][3].x, v[g][3].y, v[g][3].z, v[g][3].w};
    float x[32];
    widen_bf16x32(w, x);
    if constexpr (EF) {
#pragma unroll
      for (int i = 0; i < 32; ++i) x[i] = ef_add(x[i], __uint_as_float(rv[g][i]));
    }
    uint32_t q[8];
    const uint32_t scale = quantize_block32(x, q);
    store_block(a.staging + (uint64_t)chunk * rec, a.chunk_elems, tile_in_chunk, q, scale);
    if constexpr (EF) {
      ef_residual(x, q, scale);
      st_residual(a.residual + block_off(tile), x);
    }
  }
}

// Thread 0, once this CTA's stores of n units (tiles, or K3's groups of tiles) of a record are released (a barrier, then
// fence_gpu): add them to the record's count.  The arriver that brings it to all `units` counts the record in `done`
// (when given), acquires every other CTA's part of it with one fence -- fences are cumulative, so on a NIC-facing QP
// (`sys`) one system-scope fence here covers the whole record without a sys fence per step -- posts it through post()
// when there is a qp, and re-arms the count for the next launch.
template <class Post>
__device__ __forceinline__ void complete_run(unsigned int* count, uint32_t n, uint32_t units, unsigned int* done,
                                             const QpDev* qp, bool sys, Post post) {
  if (atomicAdd(count, n) + n != units) return;
  if (done) atomicAdd(done, 1u);
  if (qp) {
    fence_scope(sys);
    post();
  }
  *count = 0;
}

// After a CTA's last step: true in thread 0 of the CTA that arrives last, false everywhere else.  The barrier and the
// fence release all of this CTA's work before its arrival.
__device__ __forceinline__ bool last_cta(unsigned int* ctas_done) {
  __syncthreads();
  if (threadIdx.x != 0) return false;
  fence_gpu();
  return atomicAdd(ctas_done, 1u) + 1 == gridDim.x;
}

// The last CTA of a launch that posts records: one flush behind them, whose CQE proves that every record the launch
// posted has landed (waited for unless post_only).  Fewer than `expected` records posted ends the launch TIMEOUT: a
// record whose inputs never came is never posted, and the posted ones still drain.  Re-arms post_record's accumulators
// for the next launch.  Returns the records posted, and in `first` ~acc[2], the time of the first post (all ones when
// nothing was posted).
__device__ __forceinline__ unsigned long long flush_records(QpDev* qp, uint32_t post_only, uint64_t timeout_ns, uint32_t expected,
                                                            unsigned long long* acc, unsigned long long* out,
                                                            unsigned long long& first) {
  const unsigned long long posted = ld_u64_volatile(&acc[1]);
  first = ~ld_u64_volatile(&acc[2]);
  int rc = post_flush(qp, post_only, timeout_ns);
  if (posted != expected && rc == WAIT_OK) rc = WAIT_TIMEOUT;
  if (rc != WAIT_OK) out[0] = (unsigned long long)(long long)rc;
  acc[0] = 0; acc[1] = 0; acc[2] = 0;
  return posted;
}

// EF = true quantises x + residual and writes the new residual back (pack_group's EF); everything else is the same.
template <bool EF>
__global__ void __launch_bounds__(kPackThreads) pack_fp8_write_kernel(PackArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint64_t n_tiles = a.n_elems / kTileElems;
  const uint32_t tiles_per_chunk = a.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.chunk_elems);
  // group = G consecutive tiles of one chunk; G is the largest of {4,2,1} dividing tiles_per_chunk ({2,1} with EF: its
  // residual triples a tile's loads)
  const uint32_t G = (!EF && tiles_per_chunk % 4 == 0) ? 4 : ((tiles_per_chunk % 2 == 0) ? 2 : 1);
  const uint64_t n_groups = n_tiles / G;
  const uint32_t groups_per_chunk = tiles_per_chunk / G;
  const bool sys = a.qp != nullptr && poster_sys(a.qp);
  for (uint64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const uint64_t first_tile = grp * G;
    const uint32_t chunk = (uint32_t)(first_tile / tiles_per_chunk);
    if constexpr (EF) {
      if (G == 2) pack_group<2, true>(a, first_tile, tiles_per_chunk, rec);
      else pack_group<1, true>(a, first_tile, tiles_per_chunk, rec);
    } else {
      if (G == 4) pack_group<4, false>(a, first_tile, tiles_per_chunk, rec);
      else if (G == 2) pack_group<2, false>(a, first_tile, tiles_per_chunk, rec);
      else pack_group<1, false>(a, first_tile, tiles_per_chunk, rec);
    }
    if (a.qp == nullptr) continue;
    // ---- the last arriver of the chunk posts its record.  Counted in groups: counted in tiles (G per group, the same
    // protocol) the <true> kernel takes 130 registers instead of 128, which halves its residency.
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_gpu();   // release this group's record bytes (all threads, via the barrier) before the count
      complete_run(&a.counters[chunk], 1, groups_per_chunk, nullptr, a.qp, sys || a.direct, [&] {
        post_record(a.qp, a.with_imm ? OP_RDMA_WRITE_IMM : OP_RDMA_WRITE, a.staging_va + (uint64_t)chunk * rec, a.lkey,
                    a.remote_va + (uint64_t)chunk * rec, a.rkey, a.direct ? 0u : (uint32_t)rec, chunk, a.signal_every, a.acc,
                    a.out, a.timeout_ns);
      });
    }
  }
  if (a.qp == nullptr) return;
  // ---- the CTA that finishes last waits for the wire to drain
  if (last_cta(&a.counters[a.n_chunks])) {
    const unsigned long long t_pack_end = globaltimer_ns();
    fence_gpu();
    unsigned long long first;
    const unsigned long long posted = flush_records(a.qp, a.post_only, a.timeout_ns, a.n_chunks, a.acc, a.out, first);
    a.out[1] = t_start;                 // this CTA's start: within a launch skew of the grid's
    a.out[2] = globaltimer_ns();
    a.out[3] = posted;
    a.out[4] = first;
    a.out[5] = t_pack_end;
    a.counters[a.n_chunks] = 0;
  }
}

// ---- scatter: K3 of an all-to-all.  x holds `world` shards of `p.n_elems` elements, R = p.n_chunks records each; shard
// d goes to rank d.  One launch packs every shard, in phase order: phase j is shard (rank + j) mod world, so phase 0 is
// the own shard and at each phase every rank of a mesh sends to one peer.  Record r of shard d != rank is packed into the
// send staging at (d R + r) * rec and posted on qps[d] to remote_va[d] + (rank R + r) * rec -- slot `rank` of rank d's
// landing region -- with immediate rank R + r, as soon as it is complete.  The own shard's records are written into the
// plan's own landing slot (`own`) and nothing is posted for them: their arriver stamps own_words[r] with the same
// st.release.gpu the receive consumer uses, so a reader gated on the words starts on them while the pack still runs.
constexpr int kMaxScatter = 8;
struct ScatterArgs {
  PackArgs p;                // src, staging, n_elems (one shard), chunk_elems, n_chunks (R), staging_va, lkey, with_imm,
                             // post_only, signal_every, counters ([world R] groups per record ; CTAs done), out,
                             // timeout_ns; acc: 3 words per destination.  p.qp, p.rkey, p.remote_va, p.direct and
                             // p.residual are unused.
  QpDev* qps[kMaxScatter];   // qps[d]: the send QP to rank d (qps[rank] unused)
  uint64_t remote_va[kMaxScatter];   // rank d's landing region
  uint32_t rkey[kMaxScatter];
  uint8_t* own;              // this rank's landing slot `rank`: R records
  unsigned long long* own_words;     // its R arrival words
  uint32_t rank, world;
  unsigned long long* counts;        // second result record: word d = records posted to rank d
};

__global__ void __launch_bounds__(kPackThreads) pack_fp8_scatter_kernel(ScatterArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint32_t tiles_per_chunk = a.p.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.p.chunk_elems);
  const uint32_t G = tiles_per_chunk % 4 == 0 ? 4 : (tiles_per_chunk % 2 == 0 ? 2 : 1);   // as pack_fp8_write_kernel<false>
  const uint32_t R = a.p.n_chunks, groups_per_chunk = tiles_per_chunk / G;
  const uint64_t groups_per_shard = (uint64_t)R * groups_per_chunk, n_groups = groups_per_shard * a.world;
  for (uint64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const uint32_t d = (uint32_t)((a.rank + grp / groups_per_shard) % a.world);
    const uint64_t first_tile = grp % groups_per_shard * G;
    const uint32_t chunk = (uint32_t)(first_tile / tiles_per_chunk);
    PackArgs p = a.p;
    p.src = a.p.src + (uint64_t)d * a.p.n_elems;
    p.staging = d == a.rank ? a.own : a.p.staging + (uint64_t)d * R * rec;
    if (G == 4) pack_group<4, false>(p, first_tile, tiles_per_chunk, rec);
    else if (G == 2) pack_group<2, false>(p, first_tile, tiles_per_chunk, rec);
    else pack_group<1, false>(p, first_tile, tiles_per_chunk, rec);
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_gpu();   // release this group's record bytes (all threads, via the barrier) before the count
      unsigned int* count = &a.p.counters[(uint64_t)d * R + chunk];
      if (d == a.rank) {
        // complete_run posts when its queue pair is non-null: the own slot has none, so it gets the words as its
        // stand-in, and its "post" is the arrival stamp behind a gpu-scope fence
        complete_run(count, 1, groups_per_chunk, nullptr, reinterpret_cast<const QpDev*>(a.own_words), false, [&] {
          asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(a.own_words + chunk), "l"(globaltimer_ns()) : "memory");
        });
      } else {
        QpDev* qp = a.qps[d];
        complete_run(count, 1, groups_per_chunk, nullptr, qp, poster_sys(qp), [&] {
          post_record(qp, a.p.with_imm ? OP_RDMA_WRITE_IMM : OP_RDMA_WRITE, a.p.staging_va + ((uint64_t)d * R + chunk) * rec,
                      a.p.lkey, a.remote_va[d] + ((uint64_t)a.rank * R + chunk) * rec, a.rkey[d], (uint32_t)rec,
                      a.rank * R + chunk, a.p.signal_every, a.p.acc + 3 * d, a.p.out, a.p.timeout_ns);
        });
      }
    }
  }
  // ---- the CTA that finishes last flushes every destination's queue pair
  if (last_cta(&a.p.counters[(uint64_t)a.world * R])) {
    const unsigned long long t_pack_end = globaltimer_ns();
    fence_gpu();
    unsigned long long total = 0, first_all = ~0ull;
    for (uint32_t d = 0; d < a.world; ++d) {
      if (d == a.rank) continue;
      unsigned long long first;
      const unsigned long long posted = flush_records(a.qps[d], a.p.post_only, a.p.timeout_ns, R, a.p.acc + 3 * d, a.p.out, first);
      a.counts[d] = posted;
      total += posted;
      if (posted && first < first_all) first_all = first;
    }
    a.p.out[1] = t_start;
    a.p.out[2] = globaltimer_ns();
    a.p.out[3] = total;
    a.p.out[4] = total ? first_all : 0;
    a.p.out[5] = t_pack_end;
    a.p.counters[(uint64_t)a.world * R] = 0;
  }
}

// Wait for an arrival word (recv_consume, read_records): an acquire load until it is nonzero.  Returns false when the
// abort flag is raised first, or when timeout_ns passes -- then this waiter writes TIMEOUT to out[0] and raises the flag.
__device__ __forceinline__ bool wait_word(const unsigned long long* w, unsigned int* abort_flag, unsigned long long* out,
                                          uint64_t timeout_ns) {
  unsigned long long v, t0 = 0;
  for (unsigned n = 0;; ++n) {
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(w) : "memory");
    if (v) return true;
    if (*(volatile unsigned int*)abort_flag) return false;
    const unsigned long long now = globaltimer_ns();
    if (!t0) t0 = now;
    else if (now - t0 > timeout_ns) {
      out[0] = (unsigned long long)(long long)WAIT_TIMEOUT; atomicExch(abort_flag, 1u); return false;
    }
    __nanosleep(n < 64 ? 50 : 400);
  }
}

// Before a step reads its records: thread 0 runs wait(r) once for each distinct record r of the step's G tiles (`stride`
// apart from T0 in the flattened record-major order, below `total`), stops at the first that returns false, and fences;
// then every thread gets the outcome.  DIV32 divides in 32 bits, for a caller whose total is below 2^32: a 64-bit
// division is a call.
template <int G, bool DIV32, class Wait>
__device__ __forceinline__ bool step_gate(uint64_t T0, uint32_t stride, uint64_t total, uint32_t tpc, Wait wait) {
  __shared__ int ok;
  if (threadIdx.x == 0) {
    int good = 1;
    uint32_t last = ~0u;
#pragma unroll 1
    for (int g = 0; g < G; ++g) {
      const uint64_t T = T0 + (uint64_t)g * stride;
      if (T >= total) break;
      const uint32_t r = DIV32 ? (uint32_t)T / tpc : (uint32_t)(T / tpc);
      if (r == last) continue;
      last = r;
      if (!wait(r)) { good = 0; break; }
    }
    fence_gpu();
    ok = good;
  }
  __syncthreads();
  const int good = ok;
  __syncthreads();          // everybody has read `ok` before thread 0 re-arms it for the next step
  return good;
}

// Pass record r on unchanged: one RDMA WRITE (WRITE_IMM carrying imm) of rec bytes from src_va + r * rec to
// remote_va + r * rec, after one fence of the poster's scope that releases the record to the wire.  The caller has
// acquired the record (its arrival word, or stream order).  The forwarding unpack's and the relay's per-record post.
__device__ __forceinline__ void forward_record(QpDev* qp, uint32_t with_imm, uint64_t src_va, uint32_t lkey, uint64_t remote_va,
                                               uint32_t rkey, uint64_t rec, uint32_t r, uint32_t imm, uint32_t signal_every,
                                               unsigned long long* acc, unsigned long long* out, uint64_t timeout_ns) {
  fence_scope(poster_sys(qp));
  post_record(qp, with_imm ? OP_RDMA_WRITE_IMM : OP_RDMA_WRITE, src_va + (uint64_t)r * rec, lkey, remote_va + (uint64_t)r * rec,
              rkey, (uint32_t)rec, imm, signal_every, acc, out, timeout_ns);
}

struct UnpackArgs {
  const uint8_t* staging;    // records, back to back
  __nv_bfloat16* dst;
  uint64_t n_elems;
  uint32_t chunk_elems;
  uint32_t n_chunks;
  QpDev* qp;                 // receiver QP whose recv CQ announces records (nullptr: data already there)
  unsigned int* arrived;     // [n_chunks] flags ; [n_chunks] CTAs done ; [n_chunks+1] records seen (self-cleaned)
  const unsigned long long* ready;   // one arrival word per record, nonzero once it has landed (read_records, recv_consume);
                                     // nullptr: no words.  Never together with qp.
  unsigned long long* out;   // [status, t_start, t_end, records_seen, records_forwarded, t_first_post, 0, 0]
  uint64_t timeout_ns;
  // forwarding (unpack_fp8_kernel<true> only): record r is posted unchanged from the landing buffer, from fwd_src_va +
  // r * rec to fwd_remote_va + r * rec, by the CTA that claims it first (arrived[r] is then the claim flag: forwarding
  // never runs with the CQ poller, which owns those flags)
  QpDev* fwd_qp;
  uint64_t fwd_src_va;       // VA of `staging` as registered
  uint64_t fwd_remote_va;
  uint32_t fwd_lkey, fwd_rkey;
  uint32_t with_imm, post_only, signal_every, imm_base;   // WRITE_IMM carries imm_base + r
  unsigned long long* acc;   // post_record's [max WQE index + 1, records posted, ~first post time]
};

// FWD = false is the plain consumer.  FWD = true also forwards each record, once, as soon as its word is seen (or at
// the first step that reads it, with no words), before the record is unpacked; the last CTA posts the flush.  Its
// minimum of 3 CTAs per SM lets ptxas take the 80 registers it needs instead of spilling at 64.
template <bool FWD>
__global__ void __launch_bounds__(kPackThreads, FWD ? 3 : 0) unpack_fp8_kernel(UnpackArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint32_t tiles_per_chunk = a.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.chunk_elems);
  // With a QP, CTA 0 is the receive-CQ poller and nothing else: it turns every RDMA_WRITE_IMM completion into an arrival flag.
  // (The first version let every CTA poll the CQ for "its" record: hundreds of pollers contending for one consumer index made
  // the consumer, not the wire, the tail of the pack -> NVLink -> unpack chain.)  The other CTAs unpack, chunk-major, so that
  // every worker is on the oldest record not yet unpacked, and wait on the flag of the record they are about to read.
  // With arrival words there is no poller: every worker waits on the word of the record it is about to read, each wait
  // bounded by timeout_ns, and a worker that times out stops the others through abort_flag.
  const bool polled = a.qp != nullptr, gated = polled || a.ready != nullptr;
  unsigned int* abort_flag = a.arrived + a.n_chunks + 2;
  if (polled && blockIdx.x == 0) {
    if (threadIdx.x == 0) {
      const unsigned long long t0 = globaltimer_ns();
      uint32_t seen = 0;
      while (seen < a.n_chunks) {
        uint32_t imm = 0;
        long long got = recv_wait(a.qp, &imm, 2000);
        if (got >= 0 && imm < a.n_chunks) {
          fence_gpu();                                        // the record (ordered before its completion) before the flag
          atomicExch(&a.arrived[imm], 1u);
          ++seen;
        } else if (got == WAIT_CQE_ERROR) {
          a.out[0] = (unsigned long long)(long long)WAIT_CQE_ERROR; atomicExch(abort_flag, 1u); break;
        }
        if (globaltimer_ns() - t0 > a.timeout_ns) { a.out[0] = (unsigned long long)(long long)WAIT_TIMEOUT; atomicExch(abort_flag, 1u); break; }
      }
      atomicAdd(&a.arrived[a.n_chunks + 1], seen);
    }
  } else {
    // Workers walk the tiles of ALL records in one flattened, record-major order (so everybody is on the oldest records
    // first, but nobody is held to a record-by-record lockstep: with 64-tile records that left most of the grid idle).
    // Four tiles per step: all loads (4 x 32 bytes of fp8 + the scale bytes) are issued before the first use -- one tile at
    // a time left HBM half idle (3.4 TB/s of traffic; the pack kernel, which already worked this way, reaches 6.3).
    const uint32_t first = polled ? blockIdx.x - 1 : blockIdx.x, stride = polled ? gridDim.x - 1 : gridDim.x;
    const uint64_t total = (uint64_t)a.n_chunks * tiles_per_chunk;
    constexpr int G = 4;
    for (uint64_t T0 = first; T0 < total; T0 += (uint64_t)stride * G) {
      if constexpr (FWD) {
        // wait for, claim and forward the step's records: the word's acquire (or, with no words, the stream order) makes
        // the record visible to thread 0; the CTA that claims it first releases it to the wire with one fence of the
        // poster's scope and posts it.  32-bit divisions: the host keeps total tiles below 2^32.
        if (!step_gate<G, true>(T0, stride, total, tiles_per_chunk, [&](uint32_t r) {
              if (a.ready && !wait_word(a.ready + r, abort_flag, a.out, a.timeout_ns)) return false;
              if (atomicExch(&a.arrived[r], 1u) == 0u)
                forward_record(a.fwd_qp, a.with_imm, a.fwd_src_va, a.fwd_lkey, a.fwd_remote_va, a.fwd_rkey, rec, r,
                               a.imm_base + r, a.signal_every, a.acc, a.out, a.timeout_ns);
              return true;
            }))
          break;
      } else if (gated) {
        // the records this step reads have arrived: their words, or the poller's flags
        if (!step_gate<G, false>(T0, stride, total, tiles_per_chunk, [&](uint32_t r) {
              if (a.ready) return wait_word(a.ready + r, abort_flag, a.out, a.timeout_ns);
              for (unsigned n = 0; *(volatile unsigned int*)&a.arrived[r] == 0; ++n) {
                if (*(volatile unsigned int*)abort_flag) return false;
                __nanosleep(n < 64 ? 50 : 400);
              }
              return true;
            }))
          break;
      }
      uint32_t qv[G][8];
      uint32_t e[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint64_t T = T0 + (uint64_t)g * stride;
        if (T < total) {
          // <true> divides in 32 bits (the host keeps total tiles below 2^32): a 64-bit division is a call
          const uint32_t chunk = FWD ? (uint32_t)T / tiles_per_chunk : (uint32_t)(T / tiles_per_chunk);
          const uint32_t t = FWD ? (uint32_t)T % tiles_per_chunk : (uint32_t)(T % tiles_per_chunk);
          const uint8_t* recp = a.staging + (uint64_t)chunk * rec;
          ld256_cs(recp + block_off(t), qv[g]);
          e[g] = __ldcs(recp + scale_off(a.chunk_elems, t));
        }
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint64_t T = T0 + (uint64_t)g * stride;
        if (T >= total) break;
        float x[32];
        mx_decode_block32(qv[g], e[g], [&](int i, float d) { x[i] = d; });
        st_bf16x32(a.dst + block_off(T), x);
      }
    }
  }
  if (last_cta(&a.arrived[a.n_chunks])) {
    fence_gpu();
    if (FWD) {
      // a record whose word never came was never posted
      unsigned long long first;
      const unsigned long long posted = flush_records(a.fwd_qp, a.post_only, a.timeout_ns, a.n_chunks, a.acc, a.out, first);
      a.out[4] = posted;
      a.out[5] = posted ? first : 0;
    }
    a.out[1] = t_start;
    a.out[2] = globaltimer_ns();
    uint32_t seen = *(volatile unsigned int*)&a.arrived[a.n_chunks + 1];
    if (a.ready)                                                        // records whose word is set by now
      for (uint32_t c = 0; c < a.n_chunks; ++c) seen += ld_u64_volatile(a.ready + c) != 0;
    a.out[3] = seen;
    for (uint32_t c = 0; c <= a.n_chunks + 2; ++c) a.arrived[c] = 0;   // self-clean (the claim flags included)
  }
}

// ---- relay: pass records on, in a given order, each as soon as its arrival word is set -- the forwarding unpack's
// per-record gate without the unpack (a ring all-gather's hop, whose receiver reads the records where they land).
struct RelayArgs {
  QpDev* qp;
  const int32_t* ids;        // record ids, in posting order
  uint32_t n_ids, n_rec;     // ids must lie below n_rec: the records src and dst hold
  const unsigned long long* ready;   // n_rec arrival words (nullptr: the records are in place)
  uint64_t src_va, remote_va;        // record r: src_va + r * rec -> remote_va + r * rec
  uint32_t lkey, rkey;
  uint64_t rec;
  uint32_t with_imm, post_only, signal_every;   // WRITE_IMM carries r
  unsigned int* abort_flag;  // wait_word's (self-cleaned)
  unsigned long long* acc;   // post_record's [max WQE index + 1, records posted, ~first post time]
  unsigned long long* out;   // [status, t_start, t_end, records_posted, t_first_post, 0, 0, 0]
  uint64_t timeout_ns;
};

// One thread: for each id r in order, wait for ready[r], then post record r (forward_record); then one flush, waited for
// unless post_only.  A word that never comes ends the kernel TIMEOUT within timeout_ns, and neither that record nor any
// after it is posted; an id out of range ends it -22 the same way.
__global__ void __launch_bounds__(32) relay_records_kernel(RelayArgs a) {
  if (threadIdx.x != 0) return;
  const unsigned long long t_start = globaltimer_ns();
  bool bad_id = false;
#pragma unroll 1
  for (uint32_t i = 0; i < a.n_ids; ++i) {
    const uint32_t r = (uint32_t)a.ids[i];
    if (r >= a.n_rec) { bad_id = true; break; }
    if (a.ready && !wait_word(a.ready + r, a.abort_flag, a.out, a.timeout_ns)) break;
    forward_record(a.qp, a.with_imm, a.src_va, a.lkey, a.remote_va, a.rkey, a.rec, r, r, a.signal_every, a.acc, a.out,
                   a.timeout_ns);
  }
  unsigned long long first;
  const unsigned long long posted = flush_records(a.qp, a.post_only, a.timeout_ns, a.n_ids, a.acc, a.out, first);
  if (bad_id) a.out[0] = (unsigned long long)(long long)-22;
  a.out[1] = t_start;
  a.out[2] = globaltimer_ns();
  a.out[3] = posted;
  a.out[4] = posted ? first : 0;
  *a.abort_flag = 0;
}

// ---- reduce: the sum of P sources of K3 records (plus an optional bf16 addend) as bf16 and / or as K3 records, each
// finished record posted as it completes.  One rule for the arithmetic: every decoded element is q * 2^(byte - 127) in
// fp32 (exact, or +-Inf where it overflows), the sum starts from `local` (or from source 0) and adds the other sources in
// source order, one __fadd_rn each.  __fmul_rn / __fadd_rn keep the compiler from contracting them into an FMA, which
// would round once where the reference rounds twice.
struct ReduceArgs {
  const uint8_t* src;                // n_src x n_rec records, source-major
  const __nv_bfloat16* local;        // optional addend of n_elems (nullptr: the sum starts from source 0)
  __nv_bfloat16* out;                // optional bf16 sum
  uint8_t* out_rec;                  // optional K3 records of the sum (registered when they are posted)
  uint32_t chunk_elems, n_rec, n_src;
  const unsigned long long* ready;   // optional: word s * n_rec + r is nonzero once record r of source s has landed
  QpDev* qp;                         // nullptr: nothing is posted
  uint64_t out_va;                   // VA of out_rec as registered
  uint32_t lkey, rkey;
  uint64_t remote_va;                // destination of record 0; records keep their stride remotely
  uint32_t with_imm, post_only, signal_every;
  unsigned int* counters;            // [0, n_rec) tiles done per record ; [n_rec] CTAs done ; [n_rec + 1] abort flag ;
                                     // [n_rec + 2] records reduced (self-cleaned)
  unsigned long long* acc;           // post_record's [max WQE index + 1, records posted, ~first post time]
  unsigned long long* res;           // [status, t_start, t_end, records_reduced, records_posted, t_first_post, t_reduce_end, 0]
  uint64_t timeout_ns;
  uint32_t imm_base;                 // WRITE_IMM carries imm_base + r (the record's id in a larger numbering: a ring's slots)
  float* residual;                   // reduce_fp8_kernel<.., true> only: n_elems fp32, read and written in place
};

// One step of G tiles, `stride` apart in the flattened record-major order, of up to PMAX sources: every load (PMAX x 32
// bytes of fp8 and a scale byte per tile, 64 bytes of the addend, and with EF 128 bytes of residual) is issued before the
// first use.  EF adds the residual to the sum last, and `out` and the records then hold that value.
template <int G, int PMAX, bool LOCAL, bool EF>
__device__ __forceinline__ void reduce_step(const ReduceArgs& a, uint64_t T0, uint32_t stride, uint64_t total, uint32_t tpc,
                                            uint64_t rec) {
  uint32_t qv[G][PMAX][8];
  uint32_t e[G][PMAX];
  uint32_t lv[G][LOCAL ? 16 : 1];
  uint32_t rv[G][EF ? 32 : 1];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint64_t T = T0 + (uint64_t)g * stride;
    if (T < total) {
      const uint32_t r = (uint32_t)(T / tpc), t = (uint32_t)(T % tpc);
#pragma unroll
      for (int s = 0; s < PMAX; ++s) {
        if (s < (int)a.n_src) {
          const uint8_t* recp = a.src + ((uint64_t)s * a.n_rec + r) * rec;
          ld256_cs(recp + block_off(t), qv[g][s]);
          e[g][s] = __ldcs(recp + scale_off(a.chunk_elems, t));
        }
      }
      if constexpr (LOCAL) {
        const __nv_bfloat16* lp = a.local + block_off(T);
        ld256_cs(lp, lv[g]);
        ld256_cs(lp + 16, lv[g] + 8);
      }
      if constexpr (EF) ld_residual(a.residual + block_off(T), rv[g]);
    }
  }
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint64_t T = T0 + (uint64_t)g * stride;
    if (T >= total) break;
    float x[32];
    if constexpr (LOCAL) widen_bf16x32(lv[g], x);
#pragma unroll
    for (int s = 0; s < PMAX; ++s) {
      if (s < (int)a.n_src) {
        mx_decode_block32(qv[g][s], e[g][s], [&](int i, float d) {
          x[i] = (!LOCAL && s == 0) ? d : EF ? ef_add(x[i], d) : __fadd_rn(x[i], d);
        });
      }
    }
    if constexpr (EF) {
#pragma unroll
      for (int i = 0; i < 32; ++i) x[i] = ef_add(x[i], __uint_as_float(rv[g][i]));
    }
    if (a.out) st_bf16x32(a.out + block_off(T), x);
    if (a.out_rec) {
      uint32_t q[8];
      const uint32_t scale = quantize_block32(x, q);
      const uint32_t r = (uint32_t)(T / tpc), t = (uint32_t)(T % tpc);
      store_block(a.out_rec + (uint64_t)r * rec, a.chunk_elems, t, q, scale);
      if constexpr (EF) {                                      // EF always has out_rec (the host refuses it without)
        ef_residual(x, q, scale);
        st_residual(a.residual + block_off(T), x);
      }
    }
  }
}

// Workers walk the tiles of all records in K5's flattened record-major order, G tiles per step, so the oldest records
// finish (and are forwarded) first.  With arrival words there is no poller: before each step thread 0 waits for the
// words of every source of every record the step reads.  The CTA whose tiles complete a record posts it, as in K3.
template <int G, int PMAX, bool LOCAL, bool EF>
__global__ void __launch_bounds__(kPackThreads) reduce_fp8_kernel(ReduceArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint32_t tpc = a.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.chunk_elems);
  const uint64_t total = (uint64_t)a.n_rec * tpc;
  unsigned int* abort_flag = a.counters + a.n_rec + 1;
  const bool gated = a.ready != nullptr, counted = gated || a.qp != nullptr;
  const bool sys = a.qp != nullptr && poster_sys(a.qp);
  for (uint64_t T0 = blockIdx.x; T0 < total; T0 += (uint64_t)gridDim.x * G) {
    // every source of every record this step reads has landed
    if (gated && !step_gate<G, false>(T0, gridDim.x, total, tpc, [&](uint32_t r) {
          for (uint32_t s = 0; s < a.n_src; ++s)
            if (!wait_word(a.ready + (uint64_t)s * a.n_rec + r, abort_flag, a.res, a.timeout_ns)) return false;
          return true;
        }))
      break;
    reduce_step<G, PMAX, LOCAL, EF>(a, T0, gridDim.x, total, tpc, rec);
    if (!counted) continue;
    // ---- count the step's tiles per record, one run of consecutive tiles of a record at a time
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_gpu();   // release this step's stores (all threads, via the barrier) before the counts
      for (int g = 0; g < G;) {
        const uint64_t T = T0 + (uint64_t)g * gridDim.x;
        if (T >= total) break;
        const uint32_t r = (uint32_t)(T / tpc);
        uint32_t n = 0;
        while (g < G && T0 + (uint64_t)g * gridDim.x < total && (T0 + (uint64_t)g * gridDim.x) / tpc == r) { ++n; ++g; }
        complete_run(&a.counters[r], n, tpc, &a.counters[a.n_rec + 2], a.qp, sys, [&] {
          post_record(a.qp, a.with_imm ? OP_RDMA_WRITE_IMM : OP_RDMA_WRITE, a.out_va + (uint64_t)r * rec, a.lkey,
                      a.remote_va + (uint64_t)r * rec, a.rkey, (uint32_t)rec, a.imm_base + r, a.signal_every, a.acc, a.res,
                      a.timeout_ns);
        });
      }
    }
  }
  // ---- the CTA that finishes last posts the flush
  if (last_cta(&a.counters[a.n_rec])) {
    const unsigned long long t_reduce_end = globaltimer_ns();
    fence_gpu();
    // with no words to wait on and nothing to post every tile is reduced: nothing counts them
    const uint32_t reduced = counted ? ld_u32_volatile(&a.counters[a.n_rec + 2]) : a.n_rec;
    unsigned long long posted = 0, first = 0;
    if (a.qp) {
      posted = flush_records(a.qp, a.post_only, a.timeout_ns, a.n_rec, a.acc, a.res, first);
      if (!posted) first = 0;
    }
    a.res[1] = t_start;
    a.res[2] = globaltimer_ns();
    a.res[3] = reduced;
    a.res[4] = posted;
    a.res[5] = first;
    a.res[6] = t_reduce_end;
    for (uint32_t r = 0; r <= a.n_rec + 2; ++r) a.counters[r] = 0;   // self-clean, records left unfinished included
  }
}

// (G, PMAX, LOCAL, EF): tiles per step and sources a variant holds, chosen from P and the addend so that every load of a
// step fits in registers (about 72 per thread, as K3's four tiles of bf16) and P = 8 with an addend does not spill.
// With a residual (EF): P = 1 without the addend, and P <= 2 with it (the ring's hops), one tile per step: its 128
// bytes per tile keep a step's loads near the others' (at two tiles P = 1 took 245 registers, one CTA per SM).
#define RN_REDUCE_VARIANTS(X)                                                                                           \
  X(4, 1, false, false) X(4, 2, false, false) X(2, 4, false, false) X(1, 8, false, false) X(2, 2, true, false)          \
  X(1, 8, true, false) X(1, 1, false, true) X(1, 2, true, true)

// What every entry point does once its own checks pass: refuse (-22) a geometry the kernels cannot walk, zero the result
// record, turn the timeout into ns, and pick the grid: `ctas_per_sm` per SM when grid <= 0, at most one CTA per tile.
int launch_setup(uint64_t n_elems, uint32_t chunk_elems, uint64_t out_dev, uint64_t timeout_ms, int ctas_per_sm, int& grid,
                 uint64_t& wait_ns) {
  if (n_elems == 0 || chunk_elems == 0 || n_elems % kTileElems || chunk_elems % kTileElems || n_elems % chunk_elems)
    return -22;
  clear_record(out_dev);
  wait_ns = timeout_ns(timeout_ms);
  if (grid <= 0) grid = device_sms() * ctas_per_sm;
  if ((uint64_t)grid > n_elems / kTileElems) grid = (int)(n_elems / kTileElems);
  return 0;
}

// post_record's three accumulators, after a launch's n_words 32-bit counters rounded up to 8 bytes.
unsigned long long* acc_after(uint64_t counters_dev, uint64_t n_words) {
  return (unsigned long long*)(counters_dev + (n_words * 4 + 7) / 8 * 8);
}

}  // namespace

RN_API uint64_t rn_pack_record_bytes(uint64_t chunk_elems) { return record_bytes(chunk_elems); }
RN_API uint32_t rn_pack_tile_elems() { return kTileElems; }

// counters_dev: >= (n_chunks + 1) * 4 bytes (rounded up to 8) + 24 of zero-initialised device memory that the
// kernel cleans up after itself (no memset on the hot path: see Context.stream docs).
RN_API int rn_k_pack_fp8_write(uint64_t stream, int grid, uint64_t src, uint64_t staging, uint64_t n_elems,
                               uint32_t chunk_elems, uint64_t qp_dev, uint64_t staging_va, uint32_t lkey,
                               uint64_t remote_va, uint32_t rkey, uint32_t with_imm, uint32_t signal_every,
                               uint64_t counters_dev, uint64_t out_dev, uint64_t timeout_ms, uint64_t residual) {
  if (residual & 31) return -22;                               // 256-bit loads / stores
  PackArgs a;
  if (int rc = launch_setup(n_elems, chunk_elems, out_dev, timeout_ms, 4, grid, a.timeout_ns)) return rc;
  a.src = (const __nv_bfloat16*)src; a.staging = (uint8_t*)staging; a.n_elems = n_elems; a.chunk_elems = chunk_elems;
  a.n_chunks = (uint32_t)(n_elems / chunk_elems); a.qp = (QpDev*)qp_dev; a.staging_va = staging_va; a.lkey = lkey;
  a.rkey = rkey; a.remote_va = remote_va; a.with_imm = with_imm & 1u; a.post_only = (with_imm >> 1) & 1u; a.direct = (with_imm >> 2) & 1u; a.signal_every = signal_every ? signal_every : 1;
  a.counters = (unsigned int*)counters_dev;
  a.acc = acc_after(counters_dev, (uint64_t)a.n_chunks + 1);
  a.out = (unsigned long long*)out_dev;
  a.residual = (float*)residual;
  if (residual) pack_fp8_write_kernel<true><<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  else pack_fp8_write_kernel<false><<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// src: world shards of shard_elems bf16; staging: world * R records (shard d's at d * R; the own shard's are unused),
// registered at staging_va / lkey; own: R records, own_words: R arrival words.  qps_host / remote_va_host / rkeys_host:
// world entries, entry `rank` ignored.  counters_dev: >= (world * R + 1) * 4 bytes (rounded up to 8) + 24 * world of
// zeroed device memory, cleaned by the kernel.  out_dev: two result records.  flags: bit 0 RDMA_WRITE_IMM, bit 1 post_only.
RN_API int rn_k_pack_fp8_scatter(uint64_t stream, int grid, uint64_t src, uint64_t staging, uint64_t shard_elems,
                                 uint32_t chunk_elems, uint32_t rank, uint32_t world, const uint64_t* qps_host,
                                 const uint64_t* remote_va_host, const uint32_t* rkeys_host, uint64_t staging_va,
                                 uint32_t lkey, uint64_t own, uint64_t own_words, uint32_t flags, uint32_t signal_every,
                                 uint64_t counters_dev, uint64_t out_dev, uint64_t timeout_ms) {
  if (world < 2 || world > (uint32_t)kMaxScatter || rank >= world || !own_words || !shard_elems) return -22;
  if ((src | staging | own) & 31) return -22;                  // 256-bit loads, 128-bit stores
  ScatterArgs a;
  for (uint32_t d = 0; d < world; ++d) {
    a.qps[d] = d == rank ? nullptr : (QpDev*)qps_host[d];
    if (d != rank && !a.qps[d]) return -22;
    a.remote_va[d] = remote_va_host[d];
    a.rkey[d] = rkeys_host[d];
  }
  if (shard_elems % chunk_elems) return -22;
  if (int rc = launch_setup(world * shard_elems, chunk_elems, out_dev, timeout_ms, 4, grid, a.p.timeout_ns)) return rc;
  a.counts = clear_record(out_dev + 64);
  a.p.src = (const __nv_bfloat16*)src; a.p.staging = (uint8_t*)staging; a.p.n_elems = shard_elems;
  a.p.chunk_elems = chunk_elems; a.p.n_chunks = (uint32_t)(shard_elems / chunk_elems); a.p.qp = nullptr;
  a.p.staging_va = staging_va; a.p.lkey = lkey; a.p.rkey = 0; a.p.remote_va = 0;
  a.p.with_imm = flags & 1u; a.p.post_only = (flags >> 1) & 1u; a.p.direct = 0;
  a.p.signal_every = signal_every ? signal_every : 1;
  a.p.counters = (unsigned int*)counters_dev;
  a.p.acc = acc_after(counters_dev, (uint64_t)world * a.p.n_chunks + 1);
  a.p.out = (unsigned long long*)out_dev;
  a.p.residual = nullptr;
  a.own = (uint8_t*)own; a.own_words = (unsigned long long*)own_words;
  a.rank = rank; a.world = world;
  pack_fp8_scatter_kernel<<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// arrived_dev: >= (n_chunks + 3) * 4 bytes of zeroed device memory, and with fwd_qp (rounded up to 8) + 24 more.
// fwd_flags: bit 0 RDMA_WRITE_IMM (immediate = imm_base + record id), bit 1 post_only.
RN_API int rn_k_unpack_fp8(uint64_t stream, int grid, uint64_t staging, uint64_t dst, uint64_t n_elems,
                           uint32_t chunk_elems, uint64_t qp_dev, uint64_t arrived_dev, uint64_t out_dev,
                           uint64_t timeout_ms, uint64_t ready_dev, uint64_t fwd_qp, uint64_t fwd_src_va, uint32_t fwd_lkey,
                           uint64_t fwd_remote_va, uint32_t fwd_rkey, uint32_t fwd_flags, uint32_t imm_base,
                           uint32_t signal_every) {
  if (qp_dev && ready_dev) return -22;
  if (qp_dev && fwd_qp) return -22;                            // the CQ poller owns the flags the forwarders claim
  if ((staging | dst) & 31) return -22;                        // 256-bit loads / stores: records and output must be 32-byte aligned
  if (fwd_qp && n_elems / kTileElems >= (1ull << 32)) return -22;
  UnpackArgs a;
  // waiting for arrivals the kernel shares the GPU with whatever produces them (a pack kernel, an engine): one CTA per SM then
  if (int rc = launch_setup(n_elems, chunk_elems, out_dev, timeout_ms, (qp_dev || ready_dev || fwd_qp) ? 1 : 4, grid,
                            a.timeout_ns))
    return rc;
  a.staging = (const uint8_t*)staging; a.dst = (__nv_bfloat16*)dst; a.n_elems = n_elems; a.chunk_elems = chunk_elems;
  a.n_chunks = (uint32_t)(n_elems / chunk_elems); a.qp = (QpDev*)qp_dev; a.arrived = (unsigned int*)arrived_dev;
  a.out = (unsigned long long*)out_dev;
  a.ready = (const unsigned long long*)ready_dev;
  a.fwd_qp = (QpDev*)fwd_qp; a.fwd_src_va = fwd_src_va; a.fwd_remote_va = fwd_remote_va; a.fwd_lkey = fwd_lkey;
  a.fwd_rkey = fwd_rkey; a.with_imm = fwd_flags & 1u; a.post_only = (fwd_flags >> 1) & 1u;
  a.signal_every = signal_every ? signal_every : 1; a.imm_base = imm_base;
  a.acc = acc_after(arrived_dev, (uint64_t)a.n_chunks + 3);
  if (qp_dev) grid += 1;                                      // CTA 0 polls the receive CQ, the others unpack
  if (fwd_qp) unpack_fp8_kernel<true><<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  else unpack_fp8_kernel<false><<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// ids_dev: n_ids int32 record ids below n_rec, in posting order; ready_dev: n_rec arrival words, or 0.  Record r goes
// from src_va + r * rec_bytes to remote_va + r * rec_bytes.  counters_dev: 8 + 24 bytes of zeroed device memory, cleaned
// by the kernel.  flags: bit 0 RDMA_WRITE_IMM (immediate = record id), bit 1 post_only.
RN_API int rn_k_relay_records(uint64_t stream, uint64_t qp_dev, uint64_t ids_dev, uint32_t n_ids, uint32_t n_rec,
                              uint64_t ready_dev, uint64_t src_va, uint32_t lkey, uint64_t remote_va, uint32_t rkey,
                              uint64_t rec_bytes, uint32_t flags, uint32_t signal_every, uint64_t counters_dev,
                              uint64_t out_dev, uint64_t timeout_ms) {
  if (!qp_dev || !ids_dev || !counters_dev || !n_ids || !n_rec || !rec_bytes || rec_bytes >= (1ull << 32)) return -22;
  RelayArgs a;
  a.qp = (QpDev*)qp_dev; a.ids = (const int32_t*)ids_dev; a.n_ids = n_ids; a.n_rec = n_rec;
  a.ready = (const unsigned long long*)ready_dev; a.src_va = src_va; a.remote_va = remote_va; a.lkey = lkey; a.rkey = rkey;
  a.rec = rec_bytes; a.with_imm = flags & 1u; a.post_only = (flags >> 1) & 1u; a.signal_every = signal_every ? signal_every : 1;
  a.abort_flag = (unsigned int*)counters_dev;
  a.acc = acc_after(counters_dev, 1);
  a.out = clear_record(out_dev);
  a.timeout_ns = timeout_ns(timeout_ms);
  relay_records_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

// counters_dev: >= (n_rec + 3) * 4 bytes (rounded up to 8) + 24 of zero-initialised device memory, cleaned by the kernel.
// flags: bit 0 RDMA_WRITE_IMM (immediate = record id), bit 1 post_only.  residual: n_elems fp32 of error feedback (0: none);
// it needs out_rec, and P = 1, or P = 2 with the addend.
RN_API int rn_k_reduce_fp8(uint64_t stream, int grid, uint64_t src, uint32_t n_src, uint64_t local, uint64_t out,
                           uint64_t out_rec, uint64_t n_elems, uint32_t chunk_elems, uint64_t ready_dev, uint64_t qp_dev,
                           uint64_t out_va, uint32_t lkey, uint64_t remote_va, uint32_t rkey, uint32_t flags,
                           uint32_t signal_every, uint64_t counters_dev, uint64_t out_dev, uint64_t timeout_ms,
                           uint32_t imm_base, uint64_t residual) {
  if (n_src < 1 || n_src > 8) return -22;
  if ((src | local | out | out_rec) & 31) return -22;          // 256-bit loads / stores
  if (!out && !out_rec) return -22;
  if (qp_dev && !out_rec) return -22;
  if (residual & 31) return -22;
  if (residual && (!out_rec || n_src > (local ? 2u : 1u))) return -22;
  ReduceArgs a;
  // waiting for arrivals the kernel shares the GPU with whatever produces them: one CTA per SM then (as K5)
  if (int rc = launch_setup(n_elems, chunk_elems, out_dev, timeout_ms, ready_dev ? 1 : 4, grid, a.timeout_ns)) return rc;
  a.src = (const uint8_t*)src; a.local = (const __nv_bfloat16*)local; a.out = (__nv_bfloat16*)out; a.out_rec = (uint8_t*)out_rec;
  a.chunk_elems = chunk_elems; a.n_rec = (uint32_t)(n_elems / chunk_elems); a.n_src = n_src;
  a.ready = (const unsigned long long*)ready_dev; a.qp = (QpDev*)qp_dev; a.out_va = out_va; a.lkey = lkey; a.rkey = rkey;
  a.remote_va = remote_va; a.with_imm = flags & 1u; a.post_only = (flags >> 1) & 1u; a.signal_every = signal_every ? signal_every : 1;
  a.counters = (unsigned int*)counters_dev;
  a.acc = acc_after(counters_dev, (uint64_t)a.n_rec + 3);
  a.res = (unsigned long long*)out_dev;
  a.imm_base = imm_base;
  a.residual = (float*)residual;
  const int pmax = local ? (n_src <= 2 ? 2 : 8) : (n_src == 1 ? 1 : n_src <= 2 ? 2 : n_src <= 4 ? 4 : 8);
#define RN_LAUNCH(G, PMAX, LOCAL, EF)                                                   \
  if (pmax == PMAX && (local != 0) == LOCAL && (residual != 0) == EF)                 \
    reduce_fp8_kernel<G, PMAX, LOCAL, EF><<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  RN_REDUCE_VARIANTS(RN_LAUNCH)
#undef RN_LAUNCH
  return (int)cudaGetLastError();
}

extern "C" __attribute__((visibility("default"))) void rn_preload_pack() {
  cudaFuncAttributes at;
  cudaFuncGetAttributes(&at, pack_fp8_write_kernel<false>);
  cudaFuncGetAttributes(&at, pack_fp8_write_kernel<true>);
  cudaFuncGetAttributes(&at, pack_fp8_scatter_kernel);
  cudaFuncGetAttributes(&at, unpack_fp8_kernel<false>);
  cudaFuncGetAttributes(&at, unpack_fp8_kernel<true>);
  cudaFuncGetAttributes(&at, relay_records_kernel);
#define RN_PRELOAD(G, PMAX, LOCAL, EF) cudaFuncGetAttributes(&at, reduce_fp8_kernel<G, PMAX, LOCAL, EF>);
  RN_REDUCE_VARIANTS(RN_PRELOAD)
#undef RN_PRELOAD
}
