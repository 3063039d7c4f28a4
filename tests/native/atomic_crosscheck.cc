// The atomic WQE against DOCA GPUNetIO's definitions (doca_gpunetio_verbs_def.h, shipped in the NCCL wheel): the atomic
// segment's size and field offsets, its place in the WQE, and the segment count of an FA / CS WQE.  Every assertion is
// a static_assert: compiling is the test (tests/test_atomic_crosscheck.py).
#include <stddef.h>
#include <stdint.h>

#include DOCA_VERBS_DEF_H          // -DDOCA_VERBS_DEF_H='"<...>/doca_gpunetio_verbs_def.h"'
#include "wire/mlx5_wire.h"

using namespace rn;

static_assert(sizeof(AtomicSeg) == sizeof(doca_gpunetio_ib_mlx5_wqe_atomic_seg), "atomic segment size");
static_assert(offsetof(AtomicSeg, swap_add) == offsetof(doca_gpunetio_ib_mlx5_wqe_atomic_seg, swap_add), "swap_add offset");
static_assert(offsetof(AtomicSeg, compare) == offsetof(doca_gpunetio_ib_mlx5_wqe_atomic_seg, compare), "compare offset");
// ctrl | raddr | atomic | data, one 16-byte segment each
static_assert(offsetof(Wqe64, atom.raddr) == sizeof(doca_gpunetio_ib_mlx5_wqe_ctrl_seg), "raddr follows ctrl");
static_assert(offsetof(Wqe64, atom.atomic) == offsetof(Wqe64, atom.raddr) + sizeof(doca_gpunetio_ib_mlx5_wqe_raddr_seg),
              "atomic follows raddr");
static_assert(offsetof(Wqe64, atom.data) == offsetof(Wqe64, atom.atomic) + sizeof(doca_gpunetio_ib_mlx5_wqe_atomic_seg),
              "data follows atomic");
static_assert(sizeof(Wqe64) == offsetof(Wqe64, atom.data) + sizeof(doca_gpunetio_ib_mlx5_wqe_data_seg), "one WQEBB");

// ds of an FA / CS WQE (build_atomic_wqe writes it; main() reads it back through the decoder)
constexpr uint8_t kAtomicDs = 4;
static_assert(kAtomicDs == DOCA_GPUNETIO_VERBS_WQE_SEG_CNT_ATOMIC_FA_CAS, "segment count of an FA / CS WQE");
static_assert(kAtomicDs * WQE_SEG == WQEBB, "an atomic fills exactly one WQEBB");
static_assert(OP_ATOMIC_CS == DOCA_GPUNETIO_IB_MLX5_OPCODE_ATOMIC_CS && OP_ATOMIC_FA == DOCA_GPUNETIO_IB_MLX5_OPCODE_ATOMIC_FA,
              "opcodes");

int main() {
  // run-time half (built and executed when a host compiler is there): the encoder really writes ds = 4
  Wqe64 w;
  build_atomic_wqe(&w, OP_ATOMIC_FA, 1, 2, 8, 1, 8, 1, 1, 0, 0);
  WqeView v;
  return (decode_wqe(&w, &v) && v.ds == kAtomicDs && v.bytes == 8) ? 0 : 1;
}
