// The two-entry WQE against DOCA GPUNetIO's definitions (doca_gpunetio_verbs_def.h, shipped in the NCCL wheel): the data
// segment's size and field offsets, and the segment counts a two-entry RDMA WQE and SEND get when built from DOCA's own
// segment sizes.  Every layout assertion is a static_assert: compiling is the test (tests/test_wire_sgl.py).
#include <stddef.h>
#include <stdint.h>

#include DOCA_VERBS_DEF_H          // -DDOCA_VERBS_DEF_H='"<...>/doca_gpunetio_verbs_def.h"'
#include "wire/mlx5_wire.h"

using namespace rn;

typedef doca_gpunetio_ib_mlx5_wqe_data_seg DocaData;
static_assert(sizeof(DataSeg) == sizeof(DocaData), "data segment size");
static_assert(offsetof(DataSeg, byte_count) == offsetof(DocaData, byte_count), "data segment byte_count");
static_assert(offsetof(DataSeg, lkey) == offsetof(DocaData, lkey), "data segment lkey");
static_assert(offsetof(DataSeg, addr) == offsetof(DocaData, addr), "data segment addr");
constexpr size_t kCtrl = sizeof(doca_gpunetio_ib_mlx5_wqe_ctrl_seg), kRaddr = sizeof(doca_gpunetio_ib_mlx5_wqe_raddr_seg);
// ctrl | raddr | data | data: the second entry follows the first, and the whole WQE is one WQEBB
constexpr uint8_t kRdmaDs = (uint8_t)((kCtrl + kRaddr + MAX_SGE * sizeof(DocaData)) / WQE_SEG);
constexpr uint8_t kSendDs = (uint8_t)((kCtrl + MAX_SGE * sizeof(DocaData)) / WQE_SEG);
static_assert(offsetof(Wqe64, rdma_sg.data) == kCtrl + kRaddr, "entry 0 follows raddr");
static_assert(offsetof(Wqe64, rdma_sg.data) + sizeof(DataSeg) == kCtrl + kRaddr + sizeof(DocaData), "entry 1 follows entry 0");
static_assert(offsetof(Wqe64, send_sg.data) == kCtrl, "a SEND's entry 0 follows ctrl");
static_assert(kRdmaDs * WQE_SEG == WQEBB, "a two-entry RDMA WQE fills one WQEBB");
static_assert(kRdmaDs == 4 && kSendDs == 3, "segment counts of two-entry WQEs");

int main() {
  // run-time half: the encoders write those ds values, and the decoder reads both entries back
  const Sge sg[MAX_SGE] = {{0x1000, 0x101, 7}, {0x9000, 0x202, 9}};
  Wqe64 w;
  WqeView v;
  build_rdma_sg_wqe(&w, OP_RDMA_WRITE, 1, 2, sg, MAX_SGE, 0x5000, 3, CTRL_CQ_UPDATE, 0);
  if (!decode_wqe(&w, &v) || v.ds != kRdmaDs || v.nsge != 2 || v.bytes != 16 || v.len0 != 7 || v.laddr1 != 0x9000) return 1;
  if (be32(reinterpret_cast<const DocaData*>(&w.rdma_sg.data[1])->lkey) != 0x202) return 1;
  build_send_sg_wqe(&w, OP_SEND, 1, 2, sg, MAX_SGE, CTRL_CQ_UPDATE, 0);
  if (!decode_wqe(&w, &v) || v.ds != kSendDs || v.nsge != 2 || v.bytes != 16 || v.lkey1 != 0x202) return 1;
  return 0;
}
