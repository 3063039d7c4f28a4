// K3 / K5 (SURVEY.md section 2.3): payload pack fused with GPU-initiated networking.
//
//  pack_fp8_write_kernel   bf16 -> fp8 e4m3 with one UE8M0 scale per 32 elements (MX-style
//                          block scaling) written into a registered staging region as
//                          self-contained chunk records; the CTA that finishes the last
//                          tile of a chunk builds the RDMA WRITE(_IMM) WQE for that record
//                          and rings the doorbell, so the wire starts moving chunk i while
//                          chunks i+1.. are still being packed.  The kernel ends only when
//                          the last CQE has been seen: its device time is the whole
//                          pack+transfer pipeline.
//  unpack_fp8_kernel       consumer: optionally waits for each record's arrival (receive
//                          CQE carrying the chunk id as immediate), then fp8 -> bf16.
//
// Record layout for a chunk of C elements (C % 8192 == 0):
//     [ C bytes fp8 e4m3 ][ C/32 bytes UE8M0 scales ][ pad to 64 B ]
// Quantisation (bit-exact reference in tests/test_pack_fp8.py):
//     v = amax * (1/448)  (fp32) ; e = exponent(v) + (mantissa(v) != 0), clamped to [-127, 127]
//     q = cvt.rn.satfinite.e4m3(x * 2^-e) ; scale byte = e + 127
//
// No counterpart in the reference (it moves no payload: SURVEY.md section 3.2).
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../hca/post.cuh"

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
  unsigned int* counters;    // [0..n_chunks): tiles done per chunk ; [n_chunks]: CTAs done
  unsigned long long* acc;   // device accumulators: [0] max WQE index+1, [1] WQEs posted, [2] ~first post time
                             // (atomics stay in device memory; `out` is mapped host memory, plain stores only)
  unsigned long long* out;   // [status, t_start, t_end, wqes_posted, t_first_post, t_pack_end, 0, 0]
  uint64_t timeout_ns;
};

__device__ __forceinline__ float bf16_bits_to_float(uint32_t hi16) { return __uint_as_float(hi16 << 16); }

template <int G>
__device__ __forceinline__ void pack_group(const PackArgs& a, uint64_t first_tile, uint32_t tiles_per_chunk, uint64_t rec) {
  // G tiles (G x 16 KiB of bf16) per step: all 4G 16-byte loads are issued before the first
  // use, so each thread keeps G x 64 B in flight (the single-tile version left HBM idle:
  // 16 KiB in flight per CTA measured ~2.7 TB/s aggregate at best).
  uint4 v[G][4];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4* p = reinterpret_cast<const uint4*>(a.src + (first_tile + g) * kTileElems + (uint64_t)threadIdx.x * kBlockElems);
    v[g][0] = __ldcs(p); v[g][1] = __ldcs(p + 1); v[g][2] = __ldcs(p + 2); v[g][3] = __ldcs(p + 3);
  }
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint64_t tile = first_tile + g;
    const uint32_t chunk = (uint32_t)(tile / tiles_per_chunk);
    const uint32_t tile_in_chunk = (uint32_t)(tile % tiles_per_chunk);
    const uint32_t w[16] = {v[g][0].x, v[g][0].y, v[g][0].z, v[g][0].w, v[g][1].x, v[g][1].y, v[g][1].z, v[g][1].w,
                            v[g][2].x, v[g][2].y, v[g][2].z, v[g][2].w, v[g][3].x, v[g][3].y, v[g][3].z, v[g][3].w};
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      amax = fmaxf(amax, fmaxf(fabsf(bf16_bits_to_float(w[i] & 0xffffu)), fabsf(bf16_bits_to_float(w[i] >> 16))));
    // UE8M0 scale: smallest power of two 2^e with amax / 2^e <= 448
    const uint32_t vb = __float_as_uint(amax * (1.0f / 448.0f));
    int e = (int)((vb >> 23) & 0xff) - 127 + ((vb & 0x7fffffu) ? 1 : 0);
    e = max(-127, min(127, e));
    const float inv = __uint_as_float((uint32_t)(127 - e) << 23);   // 2^-e, exact (biased exponent 0..254)
    uint32_t q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float s0 = bf16_bits_to_float(w[2 * i] & 0xffffu) * inv, s1 = bf16_bits_to_float(w[2 * i] >> 16) * inv;
      float s2 = bf16_bits_to_float(w[2 * i + 1] & 0xffffu) * inv, s3 = bf16_bits_to_float(w[2 * i + 1] >> 16) * inv;
      uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(s0, s1), __NV_SATFINITE, __NV_E4M3);
      uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(s2, s3), __NV_SATFINITE, __NV_E4M3);
      q[i] = lo | (hi << 16);
    }
    uint8_t* recp = a.staging + (uint64_t)chunk * rec;
    uint4* out = reinterpret_cast<uint4*>(recp + (uint64_t)tile_in_chunk * kTileElems + (uint64_t)threadIdx.x * kBlockElems);
    out[0] = make_uint4(q[0], q[1], q[2], q[3]);
    out[1] = make_uint4(q[4], q[5], q[6], q[7]);
    recp[a.chunk_elems + (uint64_t)tile_in_chunk * kPackThreads + threadIdx.x] = (uint8_t)(e + 127);
  }
}

__global__ void __launch_bounds__(kPackThreads) pack_fp8_write_kernel(PackArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint64_t n_tiles = a.n_elems / kTileElems;
  const uint32_t tiles_per_chunk = a.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.chunk_elems);
  // group = G consecutive tiles of one chunk; G is the largest of {4,2,1} dividing tiles_per_chunk
  const uint32_t G = (tiles_per_chunk % 4 == 0) ? 4 : ((tiles_per_chunk % 2 == 0) ? 2 : 1);
  const uint64_t n_groups = n_tiles / G;
  const uint32_t groups_per_chunk = tiles_per_chunk / G;
  const bool sys = a.qp != nullptr && poster_sys(a.qp);
  for (uint64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    const uint64_t first_tile = grp * G;
    const uint32_t chunk = (uint32_t)(first_tile / tiles_per_chunk);
    if (G == 4) pack_group<4>(a, first_tile, tiles_per_chunk, rec);
    else if (G == 2) pack_group<2>(a, first_tile, tiles_per_chunk, rec);
    else pack_group<1>(a, first_tile, tiles_per_chunk, rec);
    if (a.qp == nullptr) continue;
    // ---- last arriver of the chunk posts its record
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_gpu();   // release this group's record bytes (all threads, via the barrier) before the count
      unsigned int old = atomicAdd(&a.counters[chunk], 1u);
      if (old + 1 == groups_per_chunk) {
        // acquire every other group's bytes; fences are cumulative, so on a NIC-facing QP one
        // system-scope fence here covers the whole record without a sys fence per group
        fence_scope(sys || a.direct);
        unsigned long long idx = sq_reserve(a.qp, 1, a.timeout_ns);
        // Chunks are posted by whichever CTA finishes them, so WQE order != chunk order:
        // signal by WQE index (every k-th slot) so the CQ keeps freeing the send queue.
        const bool sig = a.signal_every <= 1 || ((idx + 1) % a.signal_every == 0);
        if (idx != ~0ull) {
          write_rdma_wqe(a.qp, idx, a.with_imm ? OP_RDMA_WRITE_IMM : OP_RDMA_WRITE, a.staging_va + (uint64_t)chunk * rec,
                         a.lkey, a.remote_va + (uint64_t)chunk * rec, a.rkey, a.direct ? 0u : (uint32_t)rec,
                         sig ? CTRL_CQ_UPDATE : 0, chunk);
          if (sq_submit(a.qp, idx, 1, a.timeout_ns, /*shared=*/true) == WAIT_OK) {
            atomicMax(&a.acc[0], idx + 1);
            atomicAdd(&a.acc[1], 1ull);
            atomicMax(&a.acc[2], ~globaltimer_ns());
          } else {
            a.out[0] = (unsigned long long)(long long)WAIT_TIMEOUT;
          }
        } else {
          a.out[0] = (unsigned long long)(long long)WAIT_TIMEOUT;
        }
        a.counters[chunk] = 0;   // self-clean for the next launch
      }
    }
  }
  if (a.qp == nullptr) return;
  // ---- the CTA that finishes last waits for the wire to drain
  __syncthreads();
  if (threadIdx.x == 0) {
    fence_gpu();
    unsigned int old = atomicAdd(&a.counters[a.n_chunks], 1u);
    if (old + 1 == gridDim.x) {
      const unsigned long long t_pack_end = globaltimer_ns();
      fence_gpu();
      unsigned long long posted = ld_u64_volatile(&a.acc[1]);
      // Flush: one signaled zero-length NOP behind everything this launch posted.  RC
      // completes in order, so its CQE proves every record has landed.
      int rc = WAIT_TIMEOUT;
      unsigned long long fidx = sq_reserve(a.qp, 1, a.timeout_ns);
      if (fidx != ~0ull) {
        uint8_t* slot = a.qp->sq + ((fidx & ((1ull << a.qp->sq_log) - 1)) << 6);
        st_v4(slot + 0, ctrl_word0(OP_NOP, (uint16_t)fidx), ctrl_word1(a.qp->qpn, 1), (uint32_t)CTRL_CQ_UPDATE << 24, 0u);
        st_v4(slot + 16, 0u, 0u, 0u, 0u);
        st_v4(slot + 32, 0u, 0u, 0u, 0u);
        st_v4(slot + 48, 0u, 0u, 0u, 0u);
        if (sq_submit(a.qp, fidx, 1, a.timeout_ns, /*shared=*/true) == WAIT_OK) rc = a.post_only ? WAIT_OK : sq_wait(a.qp, fidx, a.timeout_ns);
      }
      if (posted != a.n_chunks && rc == WAIT_OK) rc = WAIT_TIMEOUT;
      if (rc != WAIT_OK) a.out[0] = (unsigned long long)(long long)rc;
      a.out[1] = t_start;                 // this CTA's start: within a launch skew of the grid's
      a.out[2] = globaltimer_ns();
      a.out[3] = posted;
      a.out[4] = ~ld_u64_volatile(&a.acc[2]);
      a.out[5] = t_pack_end;
      a.counters[a.n_chunks] = 0;
      a.acc[0] = 0; a.acc[1] = 0; a.acc[2] = 0;
    }
  }
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

struct UnpackArgs {
  const uint8_t* staging;    // records, back to back
  __nv_bfloat16* dst;
  uint64_t n_elems;
  uint32_t chunk_elems;
  uint32_t n_chunks;
  QpDev* qp;                 // receiver QP whose recv CQ announces records (nullptr: data already there)
  unsigned int* arrived;     // [n_chunks] flags ; [n_chunks] CTAs done ; [n_chunks+1] records seen (self-cleaned)
  unsigned long long* out;   // [status, t_start, t_end, records_seen]
  uint64_t timeout_ns;
};

__global__ void __launch_bounds__(kPackThreads) unpack_fp8_kernel(UnpackArgs a) {
  const unsigned long long t_start = globaltimer_ns();
  const uint32_t tiles_per_chunk = a.chunk_elems / kTileElems;
  const uint64_t rec = record_bytes(a.chunk_elems);
  __shared__ int ok;
  // With a QP, CTA 0 is the receive-CQ poller and nothing else: it turns every RDMA_WRITE_IMM completion into an arrival flag.
  // (The first version let every CTA poll the CQ for "its" record: hundreds of pollers contending for one consumer index made
  // the consumer, not the wire, the tail of the pack -> NVLink -> unpack chain.)  The other CTAs unpack, chunk-major, so that
  // every worker is on the oldest record not yet unpacked, and wait on the flag of the record they are about to read.
  const bool polled = a.qp != nullptr;
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
      if (polled) {
        if (threadIdx.x == 0) {                                  // the records this step reads have arrived
          ok = 1;
          uint32_t last = ~0u;
          for (int g = 0; g < G && ok; ++g) {
            const uint64_t T = T0 + (uint64_t)g * stride;
            if (T >= total) break;
            const uint32_t chunk = (uint32_t)(T / tiles_per_chunk);
            if (chunk == last) continue;
            last = chunk;
            for (unsigned n = 0; *(volatile unsigned int*)&a.arrived[chunk] == 0; ++n) {
              if (*(volatile unsigned int*)abort_flag) { ok = 0; break; }
              __nanosleep(n < 64 ? 50 : 400);
            }
          }
          fence_gpu();
        }
        __syncthreads();
        const int good = ok;
        __syncthreads();          // everybody has read `ok` before thread 0 re-arms it for the next step
        if (!good) break;
      }
      uint32_t qv[G][8];
      int e[G];
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint64_t T = T0 + (uint64_t)g * stride;
        if (T < total) {
          const uint32_t chunk = (uint32_t)(T / tiles_per_chunk), t = (uint32_t)(T % tiles_per_chunk);
          const uint8_t* recp = a.staging + (uint64_t)chunk * rec;
          ld256_cs(recp + (uint64_t)t * kTileElems + (uint64_t)threadIdx.x * kBlockElems, qv[g]);
          e[g] = (int)__ldcs(recp + a.chunk_elems + (uint64_t)t * kPackThreads + threadIdx.x) - 127;
        }
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const uint64_t T = T0 + (uint64_t)g * stride;
        if (T >= total) break;
        const float s = __uint_as_float((uint32_t)(e[g] + 127) << 23);
        const uint32_t* q = qv[g];
        uint32_t o[16];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          __half2_raw h0 = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(q[i] & 0xffff), __NV_E4M3);
          __half2_raw h1 = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(q[i] >> 16), __NV_E4M3);
          float2 f0 = __half22float2(*reinterpret_cast<__half2*>(&h0));
          float2 f1 = __half22float2(*reinterpret_cast<__half2*>(&h1));
          __nv_bfloat162 b0 = __floats2bfloat162_rn(f0.x * s, f0.y * s);
          __nv_bfloat162 b1 = __floats2bfloat162_rn(f1.x * s, f1.y * s);
          o[2 * i] = *reinterpret_cast<uint32_t*>(&b0);
          o[2 * i + 1] = *reinterpret_cast<uint32_t*>(&b1);
        }
        // record-major flattened tile T is also tile T of the output: chunk * chunk_elems + t * kTileElems
        __nv_bfloat16* dst = a.dst + T * kTileElems + (uint64_t)threadIdx.x * kBlockElems;
        st256_cs(dst, o);
        st256_cs(dst + 16, o + 8);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    fence_gpu();
    unsigned int old = atomicAdd(&a.arrived[a.n_chunks], 1u);
    if (old + 1 == gridDim.x) {
      fence_gpu();
      a.out[1] = t_start;
      a.out[2] = globaltimer_ns();
      a.out[3] = *(volatile unsigned int*)&a.arrived[a.n_chunks + 1];
      for (uint32_t c = 0; c <= a.n_chunks + 2; ++c) a.arrived[c] = 0;   // self-clean
    }
  }
}

}  // namespace

RN_API uint64_t rn_pack_record_bytes(uint64_t chunk_elems) { return record_bytes(chunk_elems); }
RN_API uint32_t rn_pack_tile_elems() { return kTileElems; }

// counters_dev: >= (n_chunks + 1) * 4 + 8 bytes of zero-initialised device memory that the
// kernel cleans up after itself (no memset on the hot path: see Context.stream docs).
RN_API int rn_k_pack_fp8_write(uint64_t stream, int grid, uint64_t src, uint64_t staging, uint64_t n_elems,
                               uint32_t chunk_elems, uint64_t qp_dev, uint64_t staging_va, uint32_t lkey,
                               uint64_t remote_va, uint32_t rkey, uint32_t with_imm, uint32_t signal_every,
                               uint64_t counters_dev, uint64_t out_dev, uint64_t timeout_ms) {
  if (n_elems == 0 || chunk_elems == 0 || n_elems % kTileElems || chunk_elems % kTileElems || n_elems % chunk_elems)
    return -22;
  PackArgs a;
  a.src = (const __nv_bfloat16*)src; a.staging = (uint8_t*)staging; a.n_elems = n_elems; a.chunk_elems = chunk_elems;
  a.n_chunks = (uint32_t)(n_elems / chunk_elems); a.qp = (QpDev*)qp_dev; a.staging_va = staging_va; a.lkey = lkey;
  a.rkey = rkey; a.remote_va = remote_va; a.with_imm = with_imm & 1u; a.post_only = (with_imm >> 1) & 1u; a.direct = (with_imm >> 2) & 1u; a.signal_every = signal_every ? signal_every : 1;
  a.counters = (unsigned int*)counters_dev;
  a.acc = (unsigned long long*)(counters_dev + (((uint64_t)a.n_chunks + 1) * 4 + 7) / 8 * 8);
  a.out = (unsigned long long*)out_dev;
  a.timeout_ns = (timeout_ms ? timeout_ms : 2000) * 1000000ull;
  // out[] lives in mapped pinned memory: the host zeroes it directly (no memset kernel)
  unsigned long long* o = (unsigned long long*)out_dev;
  for (int i = 0; i < 8; ++i) o[i] = 0;
  uint64_t n_tiles = n_elems / kTileElems;
  if (grid <= 0) grid = device_sms() * 4;
  if ((uint64_t)grid > n_tiles) grid = (int)n_tiles;
  pack_fp8_write_kernel<<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

RN_API int rn_k_unpack_fp8(uint64_t stream, int grid, uint64_t staging, uint64_t dst, uint64_t n_elems,
                           uint32_t chunk_elems, uint64_t qp_dev, uint64_t arrived_dev, uint64_t out_dev,
                           uint64_t timeout_ms) {
  if (n_elems == 0 || chunk_elems == 0 || n_elems % kTileElems || chunk_elems % kTileElems || n_elems % chunk_elems)
    return -22;
  if ((staging | dst) & 31) return -22;                        // 256-bit loads / stores: records and output must be 32-byte aligned
  UnpackArgs a;
  a.staging = (const uint8_t*)staging; a.dst = (__nv_bfloat16*)dst; a.n_elems = n_elems; a.chunk_elems = chunk_elems;
  a.n_chunks = (uint32_t)(n_elems / chunk_elems); a.qp = (QpDev*)qp_dev; a.arrived = (unsigned int*)arrived_dev;
  a.out = (unsigned long long*)out_dev; a.timeout_ns = (timeout_ms ? timeout_ms : 2000) * 1000000ull;
  unsigned long long* o = (unsigned long long*)out_dev;
  for (int i = 0; i < 8; ++i) o[i] = 0;
  // waiting for arrivals the kernel shares the GPU with whatever produces them (a pack kernel, an engine): one CTA per SM then
  if (grid <= 0) grid = qp_dev ? device_sms() : device_sms() * 4;
  {
    const uint64_t total_tiles = n_elems / kTileElems;
    if ((uint64_t)grid > total_tiles) grid = (int)total_tiles;
  }
  if (qp_dev) grid += 1;                                      // CTA 0 polls the receive CQ, the others unpack
  unpack_fp8_kernel<<<grid, kPackThreads, 0, (cudaStream_t)stream>>>(a);
  return (int)cudaGetLastError();
}

extern "C" __attribute__((visibility("default"))) void rn_preload_pack() {
  cudaFuncAttributes at;
  cudaFuncGetAttributes(&at, pack_fp8_write_kernel);
  cudaFuncGetAttributes(&at, unpack_fp8_kernel);
}
