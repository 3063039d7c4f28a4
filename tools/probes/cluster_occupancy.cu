// How many thread-block clusters of size 1/2/4/8 with one ~200 KiB CTA per SM can be resident at once on this GPU?
// (GPC sizes decide: a cluster never spans GPCs.)  nvcc -arch=sm_90a -o cluster_occupancy cluster_occupancy.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(int* p) { extern __shared__ char s[]; if (p && threadIdx.x == 9999) p[0] = s[0]; }
int main() {
  cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
  printf("%s SMs=%d\n", pr.name, pr.multiProcessorCount);
  const int smem = 200 * 1024;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  for (int cs : {1, 2, 4, 8, 16}) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs * 64, 1, 1); cfg.blockDim = dim3(320, 1, 1); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = -1; cudaError_t e = cudaOccupancyMaxActiveClusters(&n, k, &cfg);
    printf("cluster size %2d: max active clusters %d (%d SMs busy) %s\n", cs, n, n * cs, e == cudaSuccess ? "" : cudaGetErrorString(e));
  }
  return 0;
}
