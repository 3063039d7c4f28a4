// K7: block-scaled fp8 GEMM that CONSUMES what K3 / K4 put on the wire.
//
//   C[M,N] (bf16) = dequant(A) * dequant(B)^T,   A = (A_q [M,K] e4m3, A_s [M,K/32] UE8M0),  B likewise [N,K]
//
// The operands are exactly the self-contained records the send side produces -- pack_fp8.cu chunk records
// ([elems fp8][elems/32 scales]) and gemm_send.cu panel records ([128 x N fp8][128 x N/32 scales]) -- so a receiver
// can multiply straight out of its registered receive buffer: no dequantisation pass and half the HBM bytes of bf16
// operands.  Hopper's tensor cores multiply e4m3 but do not apply block scales, so the scaling happens in registers:
// per 32-deep MX block of K one wgmma.m64n128k32 (e4m3 x e4m3 -> fp32) produces that block's partial product, and the
// warpgroup adds it into the fp32 accumulator multiplied by 2^(scale_a - 127) * 2^(scale_b - 127) of its row and column.
// Two partial register sets alternate, so the MMA of block k + 1 runs while block k is being scaled.
//
// Persistent, one CTA (384 threads) per SM, 128 x 128 tile per CTA:
//   warpgroup 0    loaders: one thread issues the TMA loads (3-D tensor maps (K, rows-in-record, record), so an operand
//                  may live inside records; 128-byte boxes, SWIZZLE_128B, out-of-bounds rows / K zero-filled); every
//                  thread fetches the four scale bytes of one row of A and one row of B per 128-deep k-block into
//                  shared memory (layout [MX block][row])
//   warpgroups 1-2 each owns 64 rows of the tile: MMA, scaling, then bounds-checked bf16 stores from registers
// gemm_mxfp8_kernel runs one CTA per tile; gemm_mxfp8_pair_kernel a 2-CTA cluster per 256 x 128 tile, each CTA loading
// half of the B tile and multicasting it to both (half the B traffic per FLOP).
// No counterpart in the reference.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../hca/post.cuh"
#include "sm90.cuh"

using namespace rn;
using namespace rn::dev;
using namespace rn::sm90;

#define RN_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int BM = 128, BN = 128, BK = 128, STAGES = 4;
constexpr int A_STAGE = BM * BK, B_STAGE = BN * BK;            // 16 KiB each (one byte per element)
constexpr int kThreads = 384;
constexpr unsigned long long kWaitNs = 2000000000ull;

struct alignas(1024) Smem {
  uint8_t a[STAGES][A_STAGE];
  uint8_t b[STAGES][B_STAGE];
  uint8_t sfa[STAGES][4][BM];                                  // scale bytes of the stage's four MX blocks, [block][row]
  uint8_t sfb[STAGES][4][BN];
  alignas(8) uint64_t full[STAGES], empty[STAGES];
  volatile int abort;
};

struct MxArgs {
  const uint8_t* a_s;        // scales of A: row r of record i at a_s + i * a_rec_stride + r * (K / 32)
  const uint8_t* b_s;
  uint64_t a_rec_stride, b_rec_stride;   // bytes between records (fp8 block and scale block move together)
  uint32_t a_rows_per_rec, b_rows_per_rec;
  __nv_bfloat16* c;
  uint32_t M, N, K;
  unsigned long long* out;   // [status, t_start, t_end, tiles, 0...]: mapped pinned HOST memory -- written by the last CTA only
  unsigned int* done;        // device scratch (zeroed, self-cleaning): CTAs finished
  // Receive-side fusion ("the panel arrives -> its tiles start"): one word per 128-row panel of A, nonzero once the panel's
  // record has landed in this GPU's memory (recv_consume_kernel stamps it when the panel's receive completion shows up).
  // nullptr: A is complete before the launch.  The TMA producer and the scale loaders wait for the word of the panel
  // they are about to read; every wait is bounded.
  const unsigned long long* a_ready;
  uint64_t ready_timeout_ns;
};
// bounded wait for a panel's arrival word; the acquire orders it before the loads of the panel, the proxy fence extends
// that to the async proxy (TMA reads the panel)
__device__ __forceinline__ bool wait_panel(const unsigned long long* ready, uint32_t panel, uint64_t timeout_ns, volatile int* abort) {
  if (!ready) return true;
  unsigned long long v, t0 = 0;
  for (unsigned n = 0;; ++n) {
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ready + panel) : "memory");
    if (v) break;
    if (*abort) return false;
    if ((n & 63) == 63) {
      if (!t0) t0 = globaltimer_ns();
      else if (globaltimer_ns() - t0 > timeout_ns) { *abort = 1; return false; }
      __nanosleep(200);
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");
  return true;
}
// Result words live in host memory: one atomic per CTA there (the first version's atomicMax of the end time) is a PCIe
// round trip each -- one per CTA, serialised, cost ~150 us per launch, more than a 4096^3 product.  Count in device memory,
// let the last CTA write.
__device__ __forceinline__ void mx_finish(const MxArgs& g, bool aborted, unsigned long long t_start, uint32_t n_tiles, uint32_t variant) {
  if (aborted) g.out[0] = (unsigned long long)(long long)WAIT_TIMEOUT;
  __threadfence();
  if (atomicAdd(g.done, 1u) + 1 != gridDim.x) return;
  g.out[1] = t_start; g.out[3] = n_tiles; g.out[6] = variant;
  g.out[2] = globaltimer_ns();
  *g.done = 0;
}
// the four UE8M0 bytes of k-block kb for global row `row` of an operand (127 = 2^0 beyond the matrix: the data
// there is zero-filled by TMA, so any finite scale gives 0)
__device__ __forceinline__ uint32_t load_scales(const uint8_t* base, uint64_t rec_stride, uint32_t rows_per_rec, uint32_t rows, uint32_t ks,
                                                uint32_t row, uint32_t kb) {
  if (row >= rows) return 0x7f7f7f7fu;
  const uint8_t* p = base + (uint64_t)(row / rows_per_rec) * rec_stride + (uint64_t)(row % rows_per_rec) * ks + (uint64_t)kb * 4;
  if (kb * 4 + 4 <= ks && ((uintptr_t)p & 3) == 0) return *reinterpret_cast<const uint32_t*>(p);
  uint32_t v = 0;
#pragma unroll
  for (uint32_t i = 0; i < 4; ++i) v |= (uint32_t)(kb * 4 + i < ks ? p[i] : 0x7f) << (8 * i);
  return v;
}

__device__ __forceinline__ float ue8m0(uint32_t e) { return e ? __uint_as_float(e << 23) : __uint_as_float(0x00400000u); }   // 2^(e - 127)

template <int CTAS>
__device__ __forceinline__ void mx_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const MxArgs& g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CTAS == 2 ? cluster_rank() : 0u;
  const unsigned long long t_start = globaltimer_ns();
  const uint32_t m_tiles = (g.M + CTAS * BM - 1) / (CTAS * BM), n_blks = (g.N + BN - 1) / BN, k_blks = (g.K + BK - 1) / BK;
  const uint32_t n_tiles = m_tiles * n_blks, n_units = gridDim.x / CTAS, unit = blockIdx.x / CTAS;
  const uint32_t ks = g.K / 32;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&s.full[i], 1 + 128); mbar_init(&s.empty[i], 2 * CTAS); }
    s.abort = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if constexpr (CTAS == 2) cluster_sync_all();

  if (warp < 4) {
    // ===================== loaders: thread t fetches the scales of tile row t of A and of B; thread 0 also issues the TMA
    reg_dealloc<40>();
    const uint32_t t = threadIdx.x;
    uint32_t stage = 0, phase = 0;
    for (uint32_t tile = unit; tile < n_tiles && !s.abort; tile += n_units) {
      const uint32_t m_blk = (tile / n_blks) * CTAS + rank, n_blk = tile % n_blks;
      if (!wait_panel(g.a_ready, m_blk, g.ready_timeout_ns, &s.abort)) break;   // the scales travel in the same record
      const uint32_t ar = m_blk * BM, br = n_blk * BN;                       // rows of a tile never straddle records
      for (uint32_t kb = 0; kb < k_blks; ++kb) {
        const uint32_t sa = load_scales(g.a_s, g.a_rec_stride, g.a_rows_per_rec, g.M, ks, ar + t, kb);
        const uint32_t sb = load_scales(g.b_s, g.b_rec_stride, g.b_rows_per_rec, g.N, ks, br + t, kb);
        if (!mbar_wait(&s.abort, &s.empty[stage], phase ^ 1, kWaitNs)) goto loader_done;
        if (t == 0) {
          mbar_expect_tx(&s.full[stage], A_STAGE + B_STAGE);
          tma_load_3d(s.a[stage], &tmap_a, &s.full[stage], (int)(kb * BK), (int)(ar % g.a_rows_per_rec), (int)(ar / g.a_rows_per_rec));
          if constexpr (CTAS == 2) {
            const uint32_t bh = br + rank * (BN / 2);
            tma_load_3d_mc(s.b[stage] + rank * (B_STAGE / 2), &tmap_b, &s.full[stage], (int)(kb * BK), (int)(bh % g.b_rows_per_rec),
                           (int)(bh / g.b_rows_per_rec), (uint16_t)3);
          } else {
            tma_load_3d(s.b[stage], &tmap_b, &s.full[stage], (int)(kb * BK), (int)(br % g.b_rows_per_rec), (int)(br / g.b_rows_per_rec));
          }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) { s.sfa[stage][k][t] = (uint8_t)(sa >> (8 * k)); s.sfb[stage][k][t] = (uint8_t)(sb >> (8 * k)); }
        mbar_arrive(&s.full[stage]);                                           // release: the scale bytes before the arrival
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  loader_done:;
  } else {
    // ===================== MMA + scaling + epilogue: warpgroup wg owns rows wg * 64 .. wg * 64 + 63 of the tile
    reg_alloc<232>();
    const uint32_t wg = (uint32_t)(warp - 4) >> 2, t = threadIdx.x - 128 * (1 + wg), wq = t >> 5;
    const uint32_t rl0 = wg * 64 + wq * 16 + (lane >> 2);                    // fragment rows rl0, rl0 + 8 of the tile
    const bool even = (g.N % 2 == 0) && ((uintptr_t)g.c & 3) == 0;
    uint32_t stage = 0, phase = 0;
    float acc[64], p0[64], p1[64];
    for (uint32_t tile = unit; tile < n_tiles; tile += n_units) {
      const uint32_t m_blk = (tile / n_blks) * CTAS + rank, n_blk = tile % n_blks;
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      bool ok = true;
      for (uint32_t kb = 0; kb < k_blks; ++kb) {
        if (named_sync_or(2 + wg, 128, !mbar_wait(&s.abort, &s.full[stage], phase, kWaitNs))) { ok = false; break; }
        const uint64_t da = wg_desc(s.a[stage] + wg * 64 * BK), db = wg_desc(s.b[stage]);
        wg_fence();
        wgmma_e4m3_n128(p0, da, db, 0u);
        wg_commit();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float* p = (k & 1) ? p1 : p0;
          if (k < 3) {
            wg_fence();
            wgmma_e4m3_n128((k & 1) ? p0 : p1, da + (uint64_t)(2 * (k + 1)), db + (uint64_t)(2 * (k + 1)), 0u);
            wg_commit();
            wg_wait<1>();
          } else {
            wg_wait<0>();
          }
          reg_fence<64>(p);
          const float sa0 = ue8m0(s.sfa[stage][k][rl0]), sa1 = ue8m0(s.sfa[stage][k][rl0 + 8]);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const uint32_t col = 8 * j + 2 * (lane & 3);
            const uint16_t sb = *reinterpret_cast<const uint16_t*>(&s.sfb[stage][k][col]);
            const float sb0 = ue8m0(sb & 0xff), sb1 = ue8m0(sb >> 8);
            acc[4 * j] = fmaf(p[4 * j], sa0 * sb0, acc[4 * j]);
            acc[4 * j + 1] = fmaf(p[4 * j + 1], sa0 * sb1, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(p[4 * j + 2], sa1 * sb0, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(p[4 * j + 3], sa1 * sb1, acc[4 * j + 3]);
          }
        }
        // every warp of the warpgroup has read this stage's scale bytes (wgmma.wait_group orders only the warp's own MMAs,
        // and the loaders rewrite the scales the moment the stage is released)
        named_sync(2 + wg, 128);
        if (t == 0) {                                                          // operands and scales of this stage are consumed
          if constexpr (CTAS == 2) { mbar_arrive_cluster(&s.empty[stage], 0); mbar_arrive_cluster(&s.empty[stage], 1); }
          else mbar_arrive(&s.empty[stage]);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (!ok) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t row = m_blk * BM + rl0 + 8 * h;
        if (row >= g.M) continue;
        __nv_bfloat16* crow = g.c + (size_t)row * g.N;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const uint32_t col = n_blk * BN + 8 * j + 2 * (lane & 3);
          const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (even && col + 1 < g.N) {
            __nv_bfloat162 v = __floats2bfloat162_rn(v0, v1);
            *reinterpret_cast<__nv_bfloat162*>(crow + col) = v;
          } else {
            if (col < g.N) crow[col] = __float2bfloat16_rn(v0);
            if (col + 1 < g.N) crow[col + 1] = __float2bfloat16_rn(v1);
          }
        }
      }
    }
  }

  __syncthreads();
  if constexpr (CTAS == 2) cluster_sync_all();      // no CTA exits while its partner may still multicast into it or arrive on it
  if (threadIdx.x == 128) mx_finish(g, s.abort != 0, t_start, n_tiles, (uint32_t)CTAS);
}

__global__ void __launch_bounds__(kThreads, 1) gemm_mxfp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                                                 const __grid_constant__ MxArgs g) {
  mx_body<1>(tmap_a, tmap_b, g);
}
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kThreads, 1)
gemm_mxfp8_pair_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ MxArgs g) {
  mx_body<2>(tmap_a, tmap_b, g);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// fp8 operand [rows, K] held in n_rec records of rows_per_rec rows, rec_stride bytes apart: a 3-D map (K, row, record)
int make_map3(CUtensorMap* m, const void* base, uint64_t rows, uint64_t K, uint64_t rows_per_rec, uint64_t rec_stride, uint32_t box_rows = BM) {
  EncodeTiledFn fn = encode_tiled();
  if (!fn) return -38;
  const uint64_t n_rec = (rows + rows_per_rec - 1) / rows_per_rec;
  cuuint64_t dims[3] = {K, rows_per_rec < rows ? rows_per_rec : rows, n_rec};
  cuuint64_t strides[2] = {K, rec_stride};
  cuuint32_t box[3] = {BK, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 2000;
}

}  // namespace

// a_q / b_q: fp8 e4m3 bytes; a_s / b_s: UE8M0 scale bytes (one per 32 elements of K); *_rows_per_rec / *_rec_stride
// describe operands that live inside K3 chunk records or K4 panel records (rows_per_rec = rows and any stride for a
// plain matrix).  K % 32 == 0, K % 16 == 0 for the TMA row stride; M and N are free (bf16 C rows of N elements).
RN_API int rn_k_gemm_mxfp8(uint64_t stream, int grid, uint64_t a_q, uint64_t a_s, uint32_t a_rows_per_rec, uint64_t a_rec_stride, uint64_t b_q,
                           uint64_t b_s, uint32_t b_rows_per_rec, uint64_t b_rec_stride, uint64_t c, uint32_t M, uint32_t N, uint32_t K,
                           uint64_t out_dev, uint32_t cta_group, uint64_t done_dev, uint64_t a_ready_dev, uint64_t ready_timeout_ms) {
  if (!M || !N || !K || (K % 32) || (K % 16)) return -22;
  if ((a_q | b_q) & 15 || (c & 1)) return -22;
  if (!a_rows_per_rec) a_rows_per_rec = M;
  if (!b_rows_per_rec) b_rows_per_rec = N;
  if ((a_rows_per_rec < M && a_rows_per_rec % BM) || (b_rows_per_rec < N && b_rows_per_rec % BN)) return -22;   // tiles must not straddle records
  if ((a_rows_per_rec < M && (a_rec_stride % 16 || a_rec_stride < (uint64_t)a_rows_per_rec * K)) ||
      (b_rows_per_rec < N && (b_rec_stride % 16 || b_rec_stride < (uint64_t)b_rows_per_rec * K))) return -22;
  if (a_rows_per_rec >= M) a_rec_stride = (uint64_t)M * K;
  if (b_rows_per_rec >= N) b_rec_stride = (uint64_t)N * K;
  CUtensorMap ma, mb;
  int rc = make_map3(&ma, (const void*)a_q, M, K, a_rows_per_rec, a_rec_stride >= 16 ? (a_rec_stride + 15) / 16 * 16 : 16);
  if (rc) return rc;
  MxArgs g;
  g.a_s = (const uint8_t*)a_s; g.b_s = (const uint8_t*)b_s;
  g.a_rec_stride = a_rec_stride; g.b_rec_stride = b_rec_stride; g.a_rows_per_rec = a_rows_per_rec; g.b_rows_per_rec = b_rows_per_rec;
  g.c = (__nv_bfloat16*)c; g.M = M; g.N = N; g.K = K;
  g.a_ready = (const unsigned long long*)a_ready_dev; g.ready_timeout_ns = (ready_timeout_ms ? ready_timeout_ms : 2000) * 1000000ull;
  g.out = (unsigned long long*)out_dev;
  g.done = (unsigned int*)done_dev;
  if (!done_dev) return -22;
  unsigned long long* o = (unsigned long long*)out_dev;
  for (int i = 0; i < 8; ++i) o[i] = 0;
  // persistent kernels, one CTA per SM
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) return -19;
  if (grid <= 0 || grid > sms) grid = sms;
  const size_t smem = sizeof(Smem) + 1024;
  // cta_group: 2 = 2-CTA cluster per 256 x 128 tile, 1 = one CTA per 128 x 128 tile, 0 = the cluster when the matrix has more
  // than one 128-row block (a cluster tile hanging over the last rows computes zeros: correct, wasted)
  if ((cta_group == 2 || (cta_group == 0 && M > BM)) && grid >= 2) {
    rc = make_map3(&mb, (const void*)b_q, N, K, b_rows_per_rec, b_rec_stride >= 16 ? (b_rec_stride + 15) / 16 * 16 : 16, BN / 2);
    if (rc) return rc;
    const uint32_t n_tiles = ((M + 2 * BM - 1) / (2 * BM)) * ((N + BN - 1) / BN);
    grid &= ~1;
    if ((uint32_t)grid > 2 * n_tiles) grid = (int)(2 * n_tiles);
    cudaError_t e = cudaFuncSetAttribute(gemm_mxfp8_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -(int)e - 1000;
    gemm_mxfp8_pair_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(ma, mb, g);
    return (int)cudaGetLastError();
  }
  rc = make_map3(&mb, (const void*)b_q, N, K, b_rows_per_rec, b_rec_stride >= 16 ? (b_rec_stride + 15) / 16 * 16 : 16);
  if (rc) return rc;
  const uint32_t n_tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  if ((uint32_t)grid > n_tiles) grid = (int)n_tiles;
  cudaError_t e = cudaFuncSetAttribute(gemm_mxfp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return -(int)e - 1000;
  gemm_mxfp8_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(ma, mb, g);
  return (int)cudaGetLastError();
}

extern "C" __attribute__((visibility("default"))) void rn_preload_gemm_mx() {
  cudaFuncAttributes at;
  cudaFuncGetAttributes(&at, gemm_mxfp8_kernel);
  cudaFuncSetAttribute(gemm_mxfp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(Smem) + 1024));
  cudaFuncGetAttributes(&at, gemm_mxfp8_pair_kernel);
  cudaFuncSetAttribute(gemm_mxfp8_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(Smem) + 1024));
  encode_tiled();
}
