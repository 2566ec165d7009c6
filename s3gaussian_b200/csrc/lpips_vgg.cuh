// lpips_vgg.cuh - LPIPS v0.1 with the VGG16 backbone (lpipsPyTorch/modules/networks.py:88-96) on the device, forward
// only: the table of torchvision vgg16().features' thirteen convolutions for lpips.cuh's weight preparation and
// convolution tile, the convolution kernel and the 2x2 max-pool.  Taps and reduction are lpips.cuh's.
//
// Every convolution is 3x3 / stride 1 / pad 1, so it runs on lp_conv_tile: conv 1_1 (Cin = 3, K = 27 padded to 32)
// through the image-reading, z-scoring gather, the other twelve through the channels-last gather.
//
// Tile width.  The VGG walk is 305 856 MACs per input pixel and nothing but convolutions, so the tile's BN matters
// here as it did not for AlexNet.  Both wgmma operands come from shared memory, and one m64nNk8 tf32 instruction
// reads 2 KB of A and N * 32 bytes of B for 64 * N * 8 MACs: at N = 64 that is 128 bytes per clock of operand reads
// for a tensor core that retires 1024 MACs per clock, which is all a Hopper SM's shared memory delivers, before the
// 48 KB per K chunk that the gather and the weight copy write.  At N = 128 the same reads are 96 bytes per clock and
// each gathered A row is used for twice the channels, so the convolutions with Cout >= 128 (eleven of the thirteen,
// 87% of the MACs) use 128 x 128 tiles: 64 accumulators per thread and M half, 128 KB of shared memory for the two
// stages, one CTA per SM, the gather of chunk c + 1 hidden behind the 48 wgmmas of chunk c of the same CTA.  Conv 1_1
// and 1_2 (Cout = 64) keep the 128 x 64 tile, two CTAs per SM.  A wider tile still (N = 256) would need the M = 128
// rows split over two warpgroups to fit the accumulators; not done here.
// Measured on an H100 80GB HBM3 at a 700 W power limit, one 1920x1280 pair (tools/bench_lpips.py --net vgg): 44.3 ms
// per call, against 59.1 ms with 128 x 64 tiles everywhere; 3.0 TFLOP of convolutions counted once, so 68 TFLOP/s, of
// which the tensor cores execute three times (3xTF32).  The same run: the reference's module on cuDNN, 92.2 ms with
// TF32 off (the accuracy class of this path) and 32.0 ms with TF32 on (relative error 3.5e-4 against float64, this
// path 8e-7).
//
// Workspace: the x and y images walk each layer together, activations ping-pong between two buffers, each as large
// as conv 1_1's output (2N * H * W * 64 floats); a tap reads the last convolution of its group before the max-pool
// overwrites the other buffer.  One 1920x1280 pair: 2 x 1.258 GB + the taps' partial sums = 2.52 GB.
#pragma once
#include "lpips.cuh"

namespace s3g {

// torchvision vgg16().features convolutions 0,2 | 5,7 | 10,12,14 | 17,19,21 | 24,26,28
struct LpVgg {
    static constexpr int CONVS = 13;
    __host__ __device__ static constexpr int cout(int l) { return l < 2 ? 64 : l < 4 ? 128 : l < 7 ? 256 : 512; }
    __host__ __device__ static constexpr int cin(int l) { return l == 0 ? 3 : cout(l - 1); }
    __host__ __device__ static constexpr int ks(int) { return 3; }
    __host__ __device__ static constexpr int stride(int) { return 1; }
    __host__ __device__ static constexpr int pad(int) { return 1; }
    __host__ __device__ static constexpr int bn(int l) { return cout(l) >= 128 ? 128 : 64; }
    // group g = 0..4 ends with convolution last(g): the tap reads its ReLU output, then (g < 4) the max-pool does
    __host__ __device__ static constexpr int last(int g) { return g == 0 ? 1 : g == 1 ? 3 : 3 * g; }
};

template <int L>
__global__ void __launch_bounds__(LP_THREADS, LpVgg::bn(L) == 64 ? 2 : 1)
lpips_vgg_conv_kernel(const __grid_constant__ LpConvArgs a) {
    lp_conv_tile<LpVgg, L, false>(a);
}

// ---- max-pool 2/2, no padding, floor mode, channels-last [NI][H][W][C] -> [NI][H/2][W/2][C] -------------------------
__global__ void __launch_bounds__(256) lpips_maxpool2_kernel(int total4, int C4, int H, int W, int Ho, int Wo,
                                                             const float4* __restrict__ in, float4* __restrict__ out) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total4; e += gridDim.x * blockDim.x) {
        const int c = e % C4;
        int r = e / C4;
        const int ox = r % Wo;
        r /= Wo;
        const int oy = r % Ho, n = r / Ho;
        const float4* p = in + (((size_t)n * H + 2 * oy) * W + 2 * ox) * C4 + c;
        const float4 q0 = __ldg(p), q1 = __ldg(p + C4), q2 = __ldg(p + (size_t)W * C4), q3 = __ldg(p + (size_t)(W + 1) * C4);
        out[e] = make_float4(fmaxf(fmaxf(q0.x, q1.x), fmaxf(q2.x, q3.x)), fmaxf(fmaxf(q0.y, q1.y), fmaxf(q2.y, q3.y)),
                             fmaxf(fmaxf(q0.z, q1.z), fmaxf(q2.z, q3.z)), fmaxf(fmaxf(q0.w, q1.w), fmaxf(q2.w, q3.w)));
    }
}

}  // namespace s3g
