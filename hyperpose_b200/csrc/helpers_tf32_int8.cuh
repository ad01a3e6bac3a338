// helpers_tf32_int8.cuh -- the helper kernels (patch gather, max-pool, depthwise conv) of the data_type::kFLOAT and
// data_type::kINT8 engines (include/hyperpose/operator/dnn/tensorrt.hpp:14-22,48,61), one template per op over the engine's
// activation type T: float (TF32 engine) or int8_t (INT8 engine), 4 channels per thread.  Their convolutions are
// conv_wgmma_kernel<float, ...> (fp32 activations in HBM, wgmma kind tf32, fp32 accumulation) and conv_wgmma_kernel<int8_t, ...>
// (int8 activations in HBM, wgmma kind s8, s32 accumulation), conv_wgmma.cuh.
//
// TF32: TensorRT runs an "FP32" network on tensor-core GPUs exactly like this (TF32 is its default FP32 convolution math since
// Ampere): tensors stay fp32 everywhere, the multiplier reads the 8-bit exponent and the top 10 mantissa bits of each operand.
// The tensor core TRUNCATES the low 13 mantissa bits of what it reads; left alone that is a systematic toward-zero bias that
// compounds over ~40 layers.  So every producer of a conv operand rounds to the TF32 grid with round-to-nearest
// (cvt.rna.tf32.f32) before it stores -- the weights when the plan is built, the activations in the epilogue / helper kernel
// that writes them -- and the truncation on read is then exact.  Bias, PReLU, residual adds, pools and the depthwise convs
// compute in full fp32; the network outputs handed to the parser are NOT rounded.
//
// INT8: symmetric quantization as TensorRT's: activation buffer b holds int8 q in [-127, 127] standing for q * s_b (one fp32 scale
// per buffer, from a calibration table in the model pack); weights carry one scale per output channel.  Everything around the
// integer GEMM is fp32 with every product and sum rounded on its own (__fmul_rn / __fadd_rn: no FMA contraction), so that a CPU
// model of the same operations reproduces every byte.  Max-pool works on the int8 values themselves (input and output share a
// scale).
//
// Each precision keeps its own arithmetic where the two differ (if constexpr on T).  engine.cu compiles with nvcc's default
// -fmad=true, so the TF32 expressions stay as written: a product rewritten to feed a sum could be contracted into an FMA.
#pragma once
#include "conv_wgmma.cuh"

namespace hpb {

// four consecutive channels in one 16-byte (fp32) / 4-byte (int8) store
template <typename T>
__device__ __forceinline__ void store4(T* p, const T (&v)[4])
{
    if constexpr (std::is_same<T, int8_t>::value) *(char4*)p = make_char4(v[0], v[1], v[2], v[3]);
    else *(float4*)p = make_float4(v[0], v[1], v[2], v[3]);
}

// first-layer patch gather (OP_IM2COL3): u8 frames or pre-scaled f32 NCHW -> [N,OH,OW,C_ld] T, k = (r*R+s)*3 + c, zero-padded.
// x = (float)(u8 * factor in double) - mean, or f32 - mean; TF32 rounds x to the TF32 grid, INT8 computes the same x with __fsub_rn
// and quantizes it with the im2col buffer's scale (inv_s; unused by TF32)
template <typename T, bool U8>
__global__ void __launch_bounds__(256) im2col_c4_kernel(const void* __restrict__ in, T* __restrict__ out, int N, int H, int W, double factor, int flip,
                                                        float m0, float m1, float m2, int R, int stride, int OH, int OW, int pad_h, int pad_w, int C_ld,
                                                        float inv_s)
{
    constexpr bool kI8 = std::is_same<T, int8_t>::value;
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
    T v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = g4 * 4 + j;
        float x = 0.f;
        if (k < R * R * 3) {
            const int c = k % 3, rs = k / 3, s = rs % R, r = rs / R;
            const int hh = oh * stride - pad_h + r, ww = ow * stride - pad_w + s;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                const float u = U8 ? (float)((double)((const uint8_t*)in)[(((size_t)n * H + hh) * W + ww) * 3 + (flip ? 2 - c : c)] * factor)
                                   : ((const float*)in)[(((size_t)n * 3 + c) * H + hh) * W + ww];
                x = kI8 ? __fsub_rn(u, mean[c]) : u - mean[c];
            }
        }
        if constexpr (kI8) v[j] = quantize_i8(x, inv_s);
        else v[j] = ptx::round_tf32(x);   // conv operand: rounded to the TF32 grid by its producer
    }
    store4(out + idx * 4, v);
}

// KxK stride-2 max pool (K = 2 or 3), TF "SAME": window clipped at the border; 4 channels per thread: fmaxf on a float4 (TF32),
// __vmaxs4 on the four packed int8 values (INT8)
template <typename T>
__global__ void __launch_bounds__(256) maxpool_c4_kernel(const T* __restrict__ in, T* __restrict__ out, int N, int H, int W, int C_in_ld, int C, int C_out_ld,
                                                         int OH, int OW, int K, int pad_h, int pad_w)
{
    constexpr bool kI8 = std::is_same<T, int8_t>::value;
    using V = typename std::conditional<kI8, unsigned, float4>::type;   // 4 channels
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 4;
    const size_t total = (size_t)N * OH * OW * cv;
    if (idx >= total) return;
    const int c4 = (int)(idx % cv);
    size_t t = idx / cv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    V m;
    if constexpr (kI8) m = 0x80808080u;   // four times -128: below every stored value
    else m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < K; ++r) {
        const int h = oh * 2 - pad_h + r;
        if (h < 0 || h >= H) continue;
        for (int s = 0; s < K; ++s) {
            const int w = ow * 2 - pad_w + s;
            if (w < 0 || w >= W) continue;
            const V v = *(const V*)(in + (((size_t)n * H + h) * W + w) * C_in_ld + c4 * 4);
            if constexpr (kI8) m = __vmaxs4(m, v);
            else { m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w); }
        }
    }
    *(V*)(out + (((size_t)n * OH + oh) * OW + ow) * C_out_ld + c4 * 4) = m;
}

// depthwise KxK conv (K = 1 or 3, stride 1 / 2, taps `dil` pixels apart, TF "SAME") + bias + PReLU, T in / out, fp32 weights, 4
// channels per thread; from acc = 0, taps row major then by ascending column (as dwconv_kernel).
//   TF32: acc = fma(x, w, acc); y = acc + b; y > 0 ? y : y * a; rounded to the TF32 grid.
//   INT8: acc = acc + (q * s_in) * w, then + b and the PReLU slope, each operation rounded on its own; quantized with inv_s_out.
// (s_in and inv_s_out are unused by TF32.)
template <typename T>
__global__ void __launch_bounds__(256) dwconv_c4_kernel(const T* __restrict__ in, int in_ld, T* __restrict__ out, int out_ld, const float* __restrict__ w /*[K*K][C]*/,
                                                        const float* __restrict__ bias, const float* __restrict__ alpha, int N, int H, int W, int C, int OH, int OW,
                                                        int K, int stride, int dil, int pad_h, int pad_w, float s_in, float inv_s_out)
{
    constexpr bool kI8 = std::is_same<T, int8_t>::value;
    using V = typename std::conditional<kI8, char4, float4>::type;   // 4 channels
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
            const V v = *(const V*)(in + (((size_t)n * H + h) * W + x) * in_ld + c0);
            const float4 k = __ldg((const float4*)(w + (size_t)(r * K + s) * C + c0));
            if constexpr (kI8) {
                acc[0] = __fadd_rn(acc[0], __fmul_rn(__fmul_rn((float)v.x, s_in), k.x));
                acc[1] = __fadd_rn(acc[1], __fmul_rn(__fmul_rn((float)v.y, s_in), k.y));
                acc[2] = __fadd_rn(acc[2], __fmul_rn(__fmul_rn((float)v.z, s_in), k.z));
                acc[3] = __fadd_rn(acc[3], __fmul_rn(__fmul_rn((float)v.w, s_in), k.w));
            } else {
                acc[0] = fmaf(v.x, k.x, acc[0]); acc[1] = fmaf(v.y, k.y, acc[1]); acc[2] = fmaf(v.z, k.z, acc[2]); acc[3] = fmaf(v.w, k.w, acc[3]);
            }
        }
    }
    T o[4];
    if constexpr (kI8) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float y = __fadd_rn(acc[j], __ldg(bias + c0 + j));
            y = y > 0.f ? y : __fmul_rn(y, __ldg(alpha + c0 + j));
            o[j] = quantize_i8(y, inv_s_out);
        }
    } else {
        const float4 b4 = __ldg((const float4*)(bias + c0)), a4 = __ldg((const float4*)(alpha + c0));
        const float b[4] = { b4.x, b4.y, b4.z, b4.w }, a[4] = { a4.x, a4.y, a4.z, a4.w };
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float y = acc[j] + b[j];
            o[j] = ptx::round_tf32(y > 0.f ? y : y * a[j]);
        }
    }
    store4(out + (((size_t)n * OH + oh) * OW + ow) * out_ld + c0, o);
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
