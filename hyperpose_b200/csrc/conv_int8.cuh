// conv_int8.cuh -- the helper kernels of the data_type::kINT8 engine (include/hyperpose/operator/dnn/tensorrt.hpp:14-22).  Its
// convolutions are conv_wgmma_kernel<int8_t, ...> (conv_wgmma.cuh): int8 activations in HBM, wgmma kind s8, s32 accumulation.
//
// Symmetric quantization as TensorRT's: activation buffer b holds int8 q in [-127, 127] standing for q * s_b (one fp32 scale per
// buffer, from a calibration table in the model pack); weights carry one scale per output channel.  Everything around the integer
// GEMM is fp32 with every product and sum rounded on its own (__fmul_rn / __fadd_rn: no FMA contraction), so that a CPU model of the
// same operations reproduces every byte.  Max-pool works on the int8 values themselves (input and output share a scale).
#pragma once
#include "conv_wgmma.cuh"

namespace hpb {

// first-layer patch gather (OP_IM2COL3): u8 frames or pre-scaled f32 NCHW -> [N,OH,OW,C_ld] int8, k = (r*R+s)*3 + c, zero-padded;
// x is what im2col_f32_kernel computes before its TF32 rounding, quantized with the im2col buffer's scale
template <bool U8>
__global__ void __launch_bounds__(256) im2col_i8_kernel(const void* __restrict__ in, int8_t* __restrict__ out, int N, int H, int W, double factor, int flip,
                                                        float m0, float m1, float m2, int R, int stride, int OH, int OW, int pad_h, int pad_w, int C_ld,
                                                        float inv_s)
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
    int8_t v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = g4 * 4 + j;
        float x = 0.f;
        if (k < R * R * 3) {
            const int c = k % 3, rs = k / 3, s = rs % R, r = rs / R;
            const int hh = oh * stride - pad_h + r, ww = ow * stride - pad_w + s;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                if (U8) x = __fsub_rn((float)((double)((const uint8_t*)in)[(((size_t)n * H + hh) * W + ww) * 3 + (flip ? 2 - c : c)] * factor), mean[c]);
                else x = __fsub_rn(((const float*)in)[(((size_t)n * 3 + c) * H + hh) * W + ww], mean[c]);
            }
        }
        v[j] = quantize_i8(x, inv_s);
    }
    *(char4*)(out + idx * 4) = make_char4(v[0], v[1], v[2], v[3]);
}

// KxK stride-2 max pool (K = 2 or 3), TF "SAME": window clipped at the border; 4 channels per thread, on the int8 values
__global__ void __launch_bounds__(256) maxpool_i8_kernel(const int8_t* __restrict__ in, int8_t* __restrict__ out, int N, int H, int W, int C_in_ld, int C, int C_out_ld,
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
    unsigned m = 0x80808080u;   // four times -128: below every stored value
    for (int r = 0; r < K; ++r) {
        const int h = oh * 2 - pad_h + r;
        if (h < 0 || h >= H) continue;
        for (int s = 0; s < K; ++s) {
            const int w = ow * 2 - pad_w + s;
            if (w < 0 || w >= W) continue;
            m = __vmaxs4(m, *(const unsigned*)(in + (((size_t)n * H + h) * W + w) * C_in_ld + c4 * 4));
        }
    }
    *(unsigned*)(out + (((size_t)n * OH + oh) * OW + ow) * C_out_ld + c4 * 4) = m;
}

// depthwise KxK conv (K = 1 or 3, stride 1 / 2, taps `dil` pixels apart, TF "SAME") + bias + PReLU, int8 in / out, fp32 weights, 4
// channels per thread.  Per tap x = q * s_in, acc = acc + x * w from acc = 0, taps row major then by ascending column, each operation
// rounded on its own.
__global__ void __launch_bounds__(256) dwconv_i8_kernel(const int8_t* __restrict__ in, int in_ld, int8_t* __restrict__ out, int out_ld, const float* __restrict__ w /*[K*K][C]*/,
                                                        const float* __restrict__ bias, const float* __restrict__ alpha, int N, int H, int W, int C, int OH, int OW,
                                                        int K, int stride, int dil, int pad_h, int pad_w, float s_in, float inv_s_out)
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
    float acc[4] = { 0.f, 0.f, 0.f, 0.f };
    for (int r = 0; r < K; ++r) {
        const int h = oh * stride - pad_h + r * dil;
        if (h < 0 || h >= H) continue;
        for (int s = 0; s < K; ++s) {
            const int x = ow * stride - pad_w + s * dil;
            if (x < 0 || x >= W) continue;
            const char4 q = *(const char4*)(in + (((size_t)n * H + h) * W + x) * in_ld + c0);
            const float4 k = __ldg((const float4*)(w + (size_t)(r * K + s) * C + c0));
            acc[0] = __fadd_rn(acc[0], __fmul_rn(__fmul_rn((float)q.x, s_in), k.x));
            acc[1] = __fadd_rn(acc[1], __fmul_rn(__fmul_rn((float)q.y, s_in), k.y));
            acc[2] = __fadd_rn(acc[2], __fmul_rn(__fmul_rn((float)q.z, s_in), k.z));
            acc[3] = __fadd_rn(acc[3], __fmul_rn(__fmul_rn((float)q.w, s_in), k.w));
        }
    }
    int8_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float y = __fadd_rn(acc[j], __ldg(bias + c0 + j));
        y = y > 0.f ? y : __fmul_rn(y, __ldg(alpha + c0 + j));
        o[j] = quantize_i8(y, inv_s_out);
    }
    *(char4*)(out + (((size_t)n * OH + oh) * OW + ow) * out_ld + c0) = make_char4(o[0], o[1], o[2], o[3]);
}

// calibration: absmax[0] = max(absmax[0], max |x|) over n fp32 values (non-negative floats order like their bit patterns)
__global__ void __launch_bounds__(256) absmax_f32_kernel(const float* __restrict__ x, size_t n, unsigned* __restrict__ absmax)
{
    float m = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(absmax, __float_as_uint(m));
}

} // namespace hpb
