/* lane_occupancy.cu -- resources and residency of the lane kernel's record-mode instantiations: registers, static
 * shared memory and local memory (cudaFuncGetAttributes), and the blocks per SM cudaOccupancyMaxActiveBlocksPerMultiprocessor
 * gives at the launch geometry of hs_engine.cu (64 threads, no dynamic shared memory).  bench.py's headline runs
 * hs_lane_kernel<10> (SIMPLE | REC) over 65 536 replicas, i.e. 1 024 blocks.
 *
 *   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I include -I happy-simulator_b200/csrc \
 *        -o lane_occupancy tools/lane_occupancy.cu                  (tools/lane_occupancy.py builds and runs it) */
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#include "hs_b200.h"
#include "hs_lane_engine.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <int F>
static void report(const char *what, int sms)
{
    cudaFuncAttributes a;
    CK(cudaFuncGetAttributes(&a, hs_lane_kernel<F>));
    int blocks = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, hs_lane_kernel<F>, HS_LANE_THREADS, 0));
    const int grid = 65536 / HS_LANE_THREADS, wave = blocks * sms;
    printf("hs_lane_kernel<%2d> %-14s regs %3d  smem %6zu B  local %4zu B  blocks/SM %d  "
           "(1024 blocks on %d SMs: %d resident, %d in a second wave)\n", F, what, a.numRegs, a.sharedSizeBytes,
           a.localSizeBytes, blocks, sms, grid < wave ? grid : wave, grid > wave ? grid - wave : 0);
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("# device: %s, %d SMs, %zu B shared memory per SM, %zu B reserved per block\n", prop.name,
           prop.multiProcessorCount, prop.sharedMemPerMultiprocessor, prop.reservedSharedMemPerBlock);
    report<HS_LF_REC>("REC", prop.multiProcessorCount);
    report<HS_LF_REC | HS_LF_SIMPLE>("SIMPLE|REC", prop.multiProcessorCount);
    report<HS_LF_HASH | HS_LF_REC | HS_LF_SIMPLE>("HASH|SIMPLE|REC", prop.multiProcessorCount);
    report<HS_LF_SIMPLE>("SIMPLE", prop.multiProcessorCount);
    return 0;
}
