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
  uint64_t timeout_ns;
  unsigned long long* out; // per CTA: [status, t_start, t_end, done, first_idx, last_idx, 0, 0]
};

// One warp per QP.  Work requests go out in bursts (perftest's --post_list): lane 0 reserves `burst`
// slots with ONE atomic, lanes 0..n-1 each build one 64-byte WQE, lane 0 publishes the burst with ONE
// doorbell and, when the window is full, polls the CQ for the oldest burst.  With burst = 1 this is the
// plain post-one / poll-one loop (5-6 dependent L2 round trips per message, ~3.7 us measured); bursts
// amortise the reservation, the fences, the doorbell and -- with signal_every (perftest's --cq-mod) --
// the completion polling over up to 32 messages.
__global__ void __launch_bounds__(32, 1) rdma_stream_kernel(StreamArgs a) {
  const uint32_t lane = threadIdx.x;
  QpDev* qp = a.qps[blockIdx.x];
  unsigned long long* out = a.out + (size_t)blockIdx.x * 8;
  const uint64_t lbase = a.laddr + blockIdx.x * a.stride, rbase = a.raddr + blockIdx.x * a.stride;
  int status = WAIT_OK;
  unsigned long long first = ~0ull, last = 0;
  uint32_t done = 0;
  // The warp owns this QP and its send CQ for the whole kernel: queue state lives in lane 0's registers
  // (dev::Poster), no atomics, the CQ is only read when the window is full.
  Poster p = poster_open(qp);
  if (qp->state == QPS_ERR) status = WAIT_QP_ERROR;
  const unsigned long long t0 = globaltimer_ns();
  while (done < a.iters && status != WAIT_QP_ERROR) {
    const uint32_t n = min(a.burst, a.iters - done);
    unsigned long long idx = 0;
    int rc = WAIT_OK;
    if (lane == 0) {
      if (a.window && done + n > a.window) rc = poster_wait(p, last + n - a.window, a.timeout_ns);   // leaves <= window - n outstanding
      if (rc != WAIT_TIMEOUT) {
        idx = poster_reserve(p, n, a.timeout_ns);
        if (idx == ~0ull) rc = WAIT_TIMEOUT;
      }
    }
    rc = __shfl_sync(0xffffffffu, rc, 0);
    idx = __shfl_sync(0xffffffffu, idx, 0);
    if (rc != WAIT_OK) status = rc;
    if (rc == WAIT_TIMEOUT) break;
    if (first == ~0ull) first = idx;
    if (lane < n) {
      const uint32_t i = done + lane;
      const uint64_t off = (uint64_t)(i % a.nslots) * a.slot_stride;
      const bool sig = (a.signal_every <= 1) || ((i + 1) % a.signal_every == 0) || (i + 1 == a.iters);
      const uint8_t flags = sig ? CTRL_CQ_UPDATE : 0;
      if (a.opcode == OP_SEND)
        poster_build_send(p, idx + lane, OP_SEND, lbase + off, a.lkey, a.bytes, flags);
      else
        poster_build_rdma(p, idx + lane, (uint8_t)a.opcode, lbase + off, a.lkey, rbase + off, a.rkey, a.bytes, flags);
    }
    if (n > 1) __syncwarp();                         // the burst's WQE bytes happen-before lane 0's release
    if (lane == 0) {
      // overlap the completion poll with the doorbell release: the CQE load is in flight while the fence in
      // front of the doorbell waits for the WQE stores (one exposed round trip per post instead of two)
      const bool outstanding = p.head > p.cons;
      uint4 tail = make_uint4(0, 0, 0, 0);
      if (outstanding) tail = poster_peek(p);
      poster_ring(p, idx + n);
      if (outstanding && poster_take(p, tail) < 0) status = WAIT_CQE_ERROR;
    }
    last = idx + n - 1;
    done += n;
  }
  if (lane != 0) return;
  if (done && !a.post_only) {
    int rc = poster_wait(p, last, a.timeout_ns);
    if (rc != WAIT_OK) status = rc;
  }
  const unsigned long long t1 = globaltimer_ns();
  poster_close(p);
  out[0] = (unsigned long long)(long long)status;
  out[1] = t0; out[2] = t1; out[3] = done; out[4] = first; out[5] = last;
  out[6] = p.cons;
  out[7] = 0;
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
                            uint32_t nslots, uint64_t timeout_ms, uint64_t out_dev) {
  StreamArgs a;
  if (nqp == 0 || nqp > (uint32_t)kMaxStreamQps) return -22;
  for (uint32_t i = 0; i < nqp; ++i) a.qps[i] = (QpDev*)qps_host[i];
  a.post_only = (opcode >> 31) & 1u; opcode &= 0x7fffffffu;
  a.opcode = opcode; a.laddr = laddr; a.raddr = raddr; a.stride = stride;
  a.lkey = lkey; a.rkey = rkey; a.bytes = bytes; a.iters = iters; a.window = window;
  rn_stream_clamp(window, &burst, &signal_every);
  a.signal_every = signal_every; a.burst = burst;
  a.slot_stride = slot_stride; a.nslots = nslots ? nslots : 1;
  a.timeout_ns = (timeout_ms ? timeout_ms : 2000) * 1000000ull;
  a.out = (unsigned long long*)out_dev;
  rdma_stream_kernel<<<nqp, 32, 0, (cudaStream_t)stream>>>(a);
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
    unsigned long long idx = sq_reserve(qp, 1, timeout_ns);
    if (idx == ~0ull) { status = WAIT_TIMEOUT; break; }
    write_rdma_wqe(qp, idx, OP_RDMA_WRITE, laddr + cell, lkey, raddr + cell, rkey, 64, ((idx & 7) == 7) ? CTRL_CQ_UPDATE : 0);
    sq_submit_shared(qp, idx, 1);
  }
  if (status != WAIT_OK) out[0] = (unsigned long long)(long long)status;
  fence_gpu();
  if (atomicAdd(done_ctas, 1u) + 1 == gridDim.x) {
    unsigned long long fidx = sq_reserve(qp, 1, timeout_ns);
    int rc = WAIT_TIMEOUT;
    if (fidx != ~0ull) {
      uint8_t* slot = qp->sq + ((fidx & ((1ull << qp->sq_log) - 1)) << 6);
      st_v4(slot + 0, ctrl_word0(OP_NOP, (uint16_t)fidx), ctrl_word1(qp->qpn, 1), (uint32_t)CTRL_CQ_UPDATE << 24, 0u);
      st_v4(slot + 16, 0u, 0u, 0u, 0u); st_v4(slot + 32, 0u, 0u, 0u, 0u); st_v4(slot + 48, 0u, 0u, 0u, 0u);
      sq_submit_shared(qp, fidx, 1);
      rc = sq_wait(qp, fidx, timeout_ns);
    }
    if (rc != WAIT_OK) out[0] = (unsigned long long)(long long)rc;
    out[1] = t0; out[2] = globaltimer_ns(); out[3] = (unsigned long long)gridDim.x * per_cta;
    *done_ctas = 0;
  }
}
RN_API int rn_k_shared_post_stress(uint64_t stream, uint64_t qp_dev, int ctas, uint64_t laddr, uint32_t lkey, uint64_t raddr,
                                   uint32_t rkey, uint32_t per_cta, uint64_t counter_dev, uint64_t out_dev, uint64_t timeout_ms) {
  unsigned long long* o = (unsigned long long*)out_dev;
  for (int i = 0; i < 8; ++i) o[i] = 0;
  shared_post_stress_kernel<<<ctas, 32, 0, (cudaStream_t)stream>>>((QpDev*)qp_dev, laddr, lkey, raddr, rkey, per_cta,
                                                                   (unsigned int*)counter_dev, (unsigned long long*)out_dev,
                                                                   (timeout_ms ? timeout_ms : 2000) * 1000000ull);
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
                                                          (unsigned long long*)out_dev, (timeout_ms ? timeout_ms : 2000) * 1000000ull,
                                                          prepost_addr, prepost_lkey, prepost_bytes);
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
  cudaFuncGetAttributes(&a, shared_post_stress_kernel);
  cudaFuncGetAttributes(&a, fill_random_kernel);
  cudaFuncGetAttributes(&a, fill_bf16_kernel);
  cudaFuncGetAttributes(&a, checksum_kernel);
  cudaFuncGetAttributes(&a, compare_kernel);
  cudaFuncGetAttributes(&a, l2_flush_kernel);
}
