// reduce.cuh - block reduction shared by the loss (train_step.cuh) and evaluation (eval_metrics.cuh) kernels.
#pragma once
#include <cuda_runtime.h>

namespace s3g {

// sum of v over a 256-thread block; `red` is 8 floats of shared memory.  The result is valid in thread 0.
__device__ __forceinline__ float block_sum_256(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = 0.f;
    if (warp == 0) {
        s = lane < (256 / 32) ? red[lane] : 0.f;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    return s;
}

}  // namespace s3g
