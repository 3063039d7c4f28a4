// The inline WQE against DOCA GPUNetIO's definitions (doca_gpunetio_verbs_def.h, shipped in the NCCL wheel): the largest
// inline payload, the inline segment's size and flag, and the segment count the encoder writes at both ends of the range.
// Every layout assertion is a static_assert: compiling is the test (tests/test_inline_crosscheck.py).
#include <stddef.h>
#include <stdint.h>

#include DOCA_VERBS_DEF_H          // -DDOCA_VERBS_DEF_H='"<...>/doca_gpunetio_verbs_def.h"'
#include "wire/mlx5_wire.h"

using namespace rn;

static_assert(MAX_INLINE == DOCA_GPUNETIO_VERBS_MAX_INLINE_SIZE, "largest inline payload");
static_assert(sizeof(InlineSeg) == sizeof(doca_gpunetio_ib_mlx5_wqe_inl_data_seg), "inline segment size");
static_assert(INLINE_SEG == (uint32_t)DOCA_GPUNETIO_IB_MLX5_INLINE_SEG, "inline flag");
// ctrl | raddr | inline header + payload: the payload starts right after the inline header
static_assert(offsetof(Wqe64, rdma_inl.inl) == sizeof(doca_gpunetio_ib_mlx5_wqe_ctrl_seg) + sizeof(doca_gpunetio_ib_mlx5_wqe_raddr_seg),
              "inline segment follows raddr");
static_assert(INLINE_OFF_RDMA == offsetof(Wqe64, rdma_inl.inl) + sizeof(doca_gpunetio_ib_mlx5_wqe_inl_data_seg), "payload offset");
// DOCA: ds = INL_MIN while the payload fits the rest of one data segment (16 - 4 bytes), INL_MAX above
static_assert(2 + inline_segs(12) == DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MIN, "ds of a 12-byte inline WRITE");
static_assert(2 + inline_segs(13) == DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MAX, "ds of a 13-byte inline WRITE");
static_assert(2 + inline_segs(DOCA_GPUNETIO_VERBS_MAX_INLINE_SIZE) == DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MAX,
              "ds of a 28-byte inline WRITE");
static_assert(DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MAX * WQE_SEG == WQEBB, "the largest inline WRITE fills one WQEBB");

int main() {
  // run-time half: the encoder really writes those ds values, and the decoder reads them back
  static const uint8_t data[MAX_INLINE] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28};
  const uint32_t sizes[2] = {12, MAX_INLINE};
  const uint8_t want[2] = {DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MIN, DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_RDMA_WRITE_INL_MAX};
  for (int i = 0; i < 2; ++i) {
    Wqe64 w;
    build_inline_wqe(&w, OP_RDMA_WRITE, 1, 2, 0x1000, 3, data, sizes[i], CTRL_CQ_UPDATE, 0);
    WqeView v;
    if (!decode_wqe(&w, &v) || v.ds != want[i] || v.bytes != sizes[i] || v.inl_off != INLINE_OFF_RDMA) return 1;
    if (be32(w.rdma_inl.inl.byte_count) != (sizes[i] | (uint32_t)DOCA_GPUNETIO_IB_MLX5_INLINE_SEG)) return 1;
  }
  return 0;
}
