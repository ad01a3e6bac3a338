// conv_tf32.cuh -- the fp32 helper kernels of the data_type::kFLOAT engine (include/hyperpose/operator/dnn/tensorrt.hpp:14-22,
// 48,61).  Its convolutions are conv_wgmma_kernel<float, ...> (conv_wgmma.cuh): fp32 activations in HBM, wgmma kind tf32, fp32
// accumulation.
//
// TensorRT runs an "FP32" network on tensor-core GPUs exactly like this (TF32 is its default FP32 convolution math since
// Ampere): tensors stay fp32 everywhere, the multiplier reads the 8-bit exponent and the top 10 mantissa bits of each operand.
// The tensor core TRUNCATES the low 13 mantissa bits of what it reads; left alone that is a systematic toward-zero bias that
// compounds over ~40 layers.  So every producer of a conv operand rounds to the TF32 grid with round-to-nearest
// (cvt.rna.tf32.f32) before it stores -- the weights when the plan is built, the activations in the epilogue / helper kernel
// that writes them -- and the truncation on read is then exact.  Bias, PReLU, residual adds, pools and the depthwise convs
// compute in full fp32; the network outputs handed to the parser are NOT rounded.
#pragma once
#include "conv_wgmma.cuh"

namespace hpb {

// ---- fp32 helper kernels of the tf32 engine (HBM-bound, off the critical path of the headline f16 configuration) -------------

// first-layer patch gather (OP_IM2COL3): u8 frames or pre-scaled f32 NCHW -> [N,OH,OW,C_ld] fp32, k = (r*R+s)*3 + c, zero-padded
template <bool U8>
__global__ void __launch_bounds__(256) im2col_f32_kernel(const void* __restrict__ in, float* __restrict__ out, int N, int H, int W, double factor, int flip,
                                                         float m0, float m1, float m2, int R, int stride, int OH, int OW, int pad_h, int pad_w, int C_ld)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int groups = C_ld / 4;
    const size_t total = (size_t)N * OH * OW * groups;
    if (idx >= total) return;
    const int g4 = (int)(idx % groups);
    size_t t = idx / groups;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    const float mean[3] = { m0, m1, m2 };
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = g4 * 4 + j;
        float x = 0.f;
        if (k < R * R * 3) {
            const int c = k % 3, rs = k / 3, s = rs % R, r = rs / R;
            const int hh = oh * stride - pad_h + r, ww = ow * stride - pad_w + s;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                if (U8) x = (float)((double)((const uint8_t*)in)[(((size_t)n * H + hh) * W + ww) * 3 + (flip ? 2 - c : c)] * factor) - mean[c];
                else x = ((const float*)in)[(((size_t)n * 3 + c) * H + hh) * W + ww] - mean[c];
            }
        }
        v[j] = ptx::round_tf32(x);   // conv operand: rounded to the TF32 grid by its producer
    }
    *(float4*)(out + idx * 4) = make_float4(v[0], v[1], v[2], v[3]);
}

// KxK stride-2 max pool (K = 2 or 3), TF "SAME": window clipped at the border; 4 channels per thread
__global__ void __launch_bounds__(256) maxpool_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C_in_ld, int C, int C_out_ld,
                                                          int OH, int OW, int K, int pad_h, int pad_w)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 4;
    const size_t total = (size_t)N * OH * OW * cv;
    if (idx >= total) return;
    const int c4 = (int)(idx % cv);
    size_t t = idx / cv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < K; ++r) {
        const int h = oh * 2 - pad_h + r;
        if (h < 0 || h >= H) continue;
        for (int s = 0; s < K; ++s) {
            const int w = ow * 2 - pad_w + s;
            if (w < 0 || w >= W) continue;
            const float4 v = *(const float4*)(in + (((size_t)n * H + h) * W + w) * C_in_ld + c4 * 4);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    *(float4*)(out + (((size_t)n * OH + oh) * OW + ow) * C_out_ld + c4 * 4) = m;
}

// depthwise KxK conv (K = 1 or 3, stride 1 / 2, taps `dil` pixels apart, TF "SAME") + bias + PReLU, fp32 in / out, 4 channels per
// thread; accumulation order tap-row major, tap-column ascending (as dwconv_kernel)
__global__ void __launch_bounds__(256) dwconv_f32_kernel(const float* __restrict__ in, int in_ld, float* __restrict__ out, int out_ld, const float* __restrict__ w /*[K*K][C]*/,
                                                         const float* __restrict__ bias, const float* __restrict__ alpha, int N, int H, int W, int C, int OH, int OW,
                                                         int K, int stride, int dil, int pad_h, int pad_w)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 4;
    const size_t total = (size_t)N * OH * OW * cv;
    if (idx >= total) return;
    const int c0 = (int)(idx % cv) * 4;
    size_t t = idx / cv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < K; ++r) {
        const int h = oh * stride - pad_h + r * dil;
        if (h < 0 || h >= H) continue;
        for (int s = 0; s < K; ++s) {
            const int x = ow * stride - pad_w + s * dil;
            if (x < 0 || x >= W) continue;
            const float4 v = *(const float4*)(in + (((size_t)n * H + h) * W + x) * in_ld + c0);
            const float4 k = __ldg((const float4*)(w + (size_t)(r * K + s) * C + c0));
            acc.x = fmaf(v.x, k.x, acc.x); acc.y = fmaf(v.y, k.y, acc.y); acc.z = fmaf(v.z, k.z, acc.z); acc.w = fmaf(v.w, k.w, acc.w);
        }
    }
    const float4 b = __ldg((const float4*)(bias + c0)), a = __ldg((const float4*)(alpha + c0));
    float4 y = make_float4(acc.x + b.x, acc.y + b.y, acc.z + b.z, acc.w + b.w);
    y.x = y.x > 0.f ? y.x : y.x * a.x; y.y = y.y > 0.f ? y.y : y.y * a.y; y.z = y.z > 0.f ? y.z : y.z * a.z; y.w = y.w > 0.f ? y.w : y.w * a.w;
    y.x = ptx::round_tf32(y.x); y.y = ptx::round_tf32(y.y); y.z = ptx::round_tf32(y.z); y.w = ptx::round_tf32(y.w);
    *(float4*)(out + (((size_t)n * OH + oh) * OW + ow) * out_ld + c0) = y;
}

} // namespace hpb
