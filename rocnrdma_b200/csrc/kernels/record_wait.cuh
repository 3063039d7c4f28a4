// The arrival gate of the GEMMs that read records as they land (gemm_mxfp8.cu's K7 on arrival, gemm_send.cu's K4 with a
// landed addend): one word per record, nonzero once recv_consume has stamped the record's arrival.
#pragma once
#include <stdint.h>

#include "../hca/post.cuh"

namespace rn {
namespace sm90 {

// bounded wait for a record's arrival word; the acquire orders it before the loads of the record, the proxy fence extends
// that to the async proxy (TMA reads the record)
__device__ __forceinline__ bool wait_record(const unsigned long long* ready, uint32_t rec, uint64_t timeout_ns, volatile int* abort) {
  if (!ready) return true;
  unsigned long long v, t0 = 0;
  for (unsigned n = 0;; ++n) {
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ready + rec) : "memory");
    if (v) break;
    if (*abort) return false;
    if ((n & 63) == 63) {
      if (!t0) t0 = rn::dev::globaltimer_ns();
      else if (rn::dev::globaltimer_ns() - t0 > timeout_ns) { *abort = 1; return false; }
      __nanosleep(200);
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");
  return true;
}

}  // namespace sm90
}  // namespace rn
