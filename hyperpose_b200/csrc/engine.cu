// engine.cu -- the DNN engine: replaces hyperpose::dnn::tensorrt (include/hyperpose/operator/dnn/tensorrt.hpp:33-141,
// src/tensorrt.cpp:121-471).  No TensorRT: the network is a flat list of ops (pack_format.h) executed as
// hand-written sm_90a kernels on one stream:
//   OP_IM2COL3  : frame pre-processing fused with the first layer's patch gather
//                 (nhwc_images_append_nchw_batch, src/data.cpp:21-51: u8 HWC BGR -> x*factor, R/B swap;
//                  vgg mean subtraction, hyperpose/Model/backbones.py:455,497-498)
//   OP_CONV     : conv_wgmma_kernel (conv_wgmma.cuh)
//   OP_MAXPOOL2 : 2x2/2 max-pool on fp16 NHWC
// Activations stay on the device in fp16 NHWC; only the final conf/paf maps are produced as fp32 NCHW
// (the layout hyperpose::parser::paf consumes, src/tensorrt.cpp:398-431) and they, too, stay on the device
// for the parser hand-off.  Precision: fp16 operands, fp32 accumulation (same mantissa as TF32).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "../../include/hyperpose_b200.h"
#include "common.h"
#include "conv_wgmma.cuh"
#include "conv_tf32.cuh"
#include "conv_int8.cuh"
#include "handoff.h"
#include "pair_math.cuh"
#include "pack_format.h"

namespace {
using namespace hpb;

// ---------------------------------------------------------------------------------------------
// helper kernels
// ---------------------------------------------------------------------------------------------

// grid = (pixels / 256, chunks): the 64-entry chunk index is uniform per block and resolved at compile time below
template <bool U8, int R>
__global__ void __launch_bounds__(256) im2col3_kernel(const void* __restrict__ in, __half* __restrict__ out,
                                                      int N, int H, int W, double factor, int flip, float m0, float m1, float m2,
                                                      int stride, int OH, int OW, int pad_h, int pad_w, int chunks)
{
    // Each thread builds one 128-byte row.  With one chunk per pixel the block's 256 rows are contiguous in HBM:
    // they are staged in shared memory (16-byte pieces XOR-swizzled by the row) and written out fully coalesced.
    __shared__ uint4 stage[256 * 8];
    const size_t total = (size_t)N * OH * OW;
    const size_t idx0 = (size_t)blockIdx.x * blockDim.x, idx = idx0 + threadIdx.x;
    const int chunk = blockIdx.y;
    constexpr int nchunks = (R * R * 3 + 63) / 64;
    const bool staged = (nchunks == 1);
    if (idx < total) {
        const int w0 = (int)(idx % OW) * stride - pad_w;
        const int h0 = (int)((idx / OW) % OH) * stride - pad_h;
        const int n = (int)(idx / ((size_t)OW * OH));
        const float mean[3] = { m0, m1, m2 };
        uint4* o = staged ? stage + threadIdx.x * 8 : (uint4*)(out + (idx * chunks + chunk) * 64);
        const int swz = staged ? (threadIdx.x & 7) : 0;
        if (nchunks == 1 || chunk == 0) im2col_chunk<U8, R, 0>(in, o, swz, n, h0, w0, H, W, factor, flip, mean);
        else if (chunk == 1) im2col_chunk<U8, R, (nchunks > 1 ? 1 : 0)>(in, o, swz, n, h0, w0, H, W, factor, flip, mean);
        else im2col_chunk<U8, R, (nchunks > 2 ? 2 : 0)>(in, o, swz, n, h0, w0, H, W, factor, flip, mean);
    }
    if (staged) {
        __syncthreads();
        const size_t rows = total - idx0 < 256 ? total - idx0 : 256;
        uint4* dst = (uint4*)(out + idx0 * 64);
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int q = it * 256 + threadIdx.x, row = q >> 3, c = q & 7;
            if ((size_t)row < rows) dst[q] = stage[row * 8 + (c ^ (row & 7))];
        }
    }
}

// cv::resize(INTER_LINEAR) on CV_8UC3 frames (src/tensorrt.cpp:451), OpenCV's 11-bit fixed-point bilinear:
//   rows: S = src[sx]*a0 + src[sx+1]*a1 (a = round(coef*2048)); out = (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2
// x fractions are clamped at the borders, y keeps the fraction and clips the two row indices (resize.cpp).
// An exact 2x reduction is INTER_AREA in OpenCV: (a+b+c+d+2)>>2.  Pixels outside the resized region (letterbox,
// non_scaling_resize src/data.cpp:53-69) are set to 0.  One thread per destination pixel.
__global__ void __launch_bounds__(256) resize_u8c3_kernel(const uint8_t* __restrict__ src, int sh, int sw, uint8_t* __restrict__ dst, int dh, int dw,
                                                          int rh, int rw, const int* __restrict__ xi, const short* __restrict__ xa,
                                                          const int* __restrict__ yi, const short* __restrict__ ya, int area2x)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= dh * dw) return;
    const int y = idx / dw, x = idx - y * dw;
    uint8_t* o = dst + (size_t)idx * 3;
    if (y >= rh || x >= rw) { o[0] = 0; o[1] = 0; o[2] = 0; return; }
    if (area2x) {
        const uint8_t* p = src + ((size_t)(2 * y) * sw + 2 * x) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = (uint8_t)((p[c] + p[3 + c] + p[(size_t)sw * 3 + c] + p[(size_t)sw * 3 + 3 + c] + 2) >> 2);
        return;
    }
    const int x0 = xi[x], x1 = min(x0 + 1, sw - 1);
    const int y0 = min(max(yi[y], 0), sh - 1), y1 = min(max(yi[y] + 1, 0), sh - 1);
    const int a0 = xa[2 * x], a1 = xa[2 * x + 1], b0 = ya[2 * y], b1 = ya[2 * y + 1];
    const uint8_t* r0 = src + (size_t)y0 * sw * 3;
    const uint8_t* r1 = src + (size_t)y1 * sw * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int S0 = r0[x0 * 3 + c] * a0 + r0[x1 * 3 + c] * a1;
        const int S1 = r1[x0 * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
        const int v = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;
        o[c] = (uint8_t)min(max(v, 0), 255);
    }
}

// depthwise KxK conv (K in {1,3}) + bias + PReLU on fp16 NHWC, 8 channels per thread (one 16-byte load per tap),
// fp32 accumulation.  HBM-bound: reads each input element ~once (taps hit L1/L2), writes the output once.
// Reference layers: DepthwiseConv2d + BatchNorm2d(act) of separable_block (hyperpose/Model/backbones.py:240-248), BN folded.
// Each thread produces DW_STRIP consecutive output pixels of one row for 8 channels with a sliding window over the input
// columns: every input column of the window is loaded once (3 x (strip*stride + K - stride) 16-byte loads per strip instead of 9 per
// output) and the K*K*8 weights live in registers.
constexpr int DW_STRIP = 4;
template <int K, int stride>
__global__ void __launch_bounds__(256, 3) dwconv_kernel(const __half* __restrict__ in, int in_ld, __half* __restrict__ out, int out_ld,
                                                     const float* __restrict__ w /*[K*K][C]*/, const float* __restrict__ bias,
                                                     const float* __restrict__ alpha, int N, int H, int W, int C,
                                                     int OH, int OW, int pad_h, int pad_w)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 8;
    const int strips = (OW + DW_STRIP - 1) / DW_STRIP;
    const size_t total = (size_t)N * OH * strips * cv;
    if (idx >= total) return;
    const int c0 = (int)(idx % cv) * 8;
    size_t t = idx / cv;
    const int ow0 = (int)(t % strips) * DW_STRIP; t /= strips;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    float wt[K * K][8];
#pragma unroll
    for (int k = 0; k < K * K; ++k) {
        const float4 w0 = __ldg((const float4*)(w + (size_t)k * C + c0)), w1 = __ldg((const float4*)(w + (size_t)k * C + c0 + 4));
        wt[k][0] = w0.x; wt[k][1] = w0.y; wt[k][2] = w0.z; wt[k][3] = w0.w; wt[k][4] = w1.x; wt[k][5] = w1.y; wt[k][6] = w1.z; wt[k][7] = w1.w;
    }
    float acc[DW_STRIP][8];
#pragma unroll
    for (int o = 0; o < DW_STRIP; ++o)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[o][j] = 0.f;
    const int x_first = ow0 * stride - pad_w;
    constexpr int ncols = (DW_STRIP - 1) * stride + K; // input columns touched by the strip
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int h = oh * stride - pad_h + r;
        if (h < 0 || h >= H) continue;
        const __half* rowp = in + (((size_t)n * H + h) * W + x_first) * in_ld + c0;
#pragma unroll
        for (int ci = 0; ci < ncols; ++ci) {
            if ((unsigned)(x_first + ci) >= (unsigned)W) continue;
            const uint4 v = *(const uint4*)(rowp + (size_t)ci * in_ld);
            const __half2* h2 = (const __half2*)&v;
            const float2 a = __half22float2(h2[0]), b = __half22float2(h2[1]), c = __half22float2(h2[2]), d = __half22float2(h2[3]);
            const float xv[8] = { a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y };
#pragma unroll
            for (int o = 0; o < DW_STRIP; ++o) {
                const int s = ci - o * stride; // tap column of output o that reads input column ci
                if (s < 0 || s >= K) continue;
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[o][j] = fmaf(xv[j], wt[r * K + s][j], acc[o][j]);
            }
        }
    }
    float bs[8], al[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { bs[j] = __ldg(bias + c0 + j); al[j] = __ldg(alpha + c0 + j); }
#pragma unroll
    for (int o = 0; o < DW_STRIP; ++o) {
        const int ow = ow0 + o;
        if (ow >= OW) break;
        uint4 ov;
        __half2* oh2 = (__half2*)&ov;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float y0 = acc[o][2 * j] + bs[2 * j], y1 = acc[o][2 * j + 1] + bs[2 * j + 1];
            y0 = y0 > 0.f ? y0 : y0 * al[2 * j];
            y1 = y1 > 0.f ? y1 : y1 * al[2 * j + 1];
            oh2[j] = __floats2half2_rn(y0, y1);
        }
        *(uint4*)(out + (((size_t)n * OH + oh) * OW + ow) * out_ld + c0) = ov;
    }
}

// Depthwise 3x3, stride 1 (every separable block of MobilenetThin-OpenPose except two): column-marching variant.
// A thread owns one image column x, 4 channels and a run of output rows: it walks DOWN the column, loads the three
// neighbouring input pixels of each input row once (3 x 8-byte loads, lanes along channels => 256-byte coalesced
// segments; the x-1 / x+1 neighbours are L1 hits of the adjacent columns' threads) and scatters the row into the three
// output rows it feeds, so per output there are 3 loads + 36 FMAs and the 36 weights stay in registers for the whole run.
// Accumulation order per output is tap-row major, tap-column ascending -- the same as dwconv_kernel (bit-identical).
__global__ void __launch_bounds__(256, 3) dwconv3_col_kernel(const __half* __restrict__ in, int in_ld, __half* __restrict__ out, int out_ld,
                                                          const float* __restrict__ w /*[9][C]*/, const float* __restrict__ bias,
                                                          const float* __restrict__ alpha, int N, int H, int W, int C, int rows_per_chunk, int chunks)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 4;
    const size_t total = (size_t)N * chunks * W * cv;
    if (idx >= total) return;
    const int c0 = (int)(idx % cv) * 4;
    size_t t = idx / cv;
    const int x = (int)(t % W); t /= W;
    const int chunk = (int)(t % chunks);
    const int n = (int)(t / chunks);
    const int oh0 = chunk * rows_per_chunk, oh1 = min(oh0 + rows_per_chunk, H);
    if (oh0 >= oh1) return;
    float4 wt[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wt[k] = __ldg((const float4*)(w + (size_t)k * C + c0));
    const float4 bs = __ldg((const float4*)(bias + c0)), al = __ldg((const float4*)(alpha + c0));
    const bool has_l = x > 0, has_r = x + 1 < W;
    const __half* colp = in + ((size_t)n * H * W + x) * in_ld + c0;
    __half* outp = out + ((size_t)n * H * W + x) * out_ld + c0;
    float4 a0 = { 0.f, 0.f, 0.f, 0.f }, a1 = a0, a2 = a0;   // output rows ih-1, ih, ih+1 while input row ih is being read
#define HP_FMA4(acc, wv, xv) { acc.x = fmaf(xv.x, wv.x, acc.x); acc.y = fmaf(xv.y, wv.y, acc.y); acc.z = fmaf(xv.z, wv.z, acc.z); acc.w = fmaf(xv.w, wv.w, acc.w); }
    // one input row: it is tap row 2 of output ih-1 (A, complete afterwards -> stored), tap row 1 of output ih (B), tap row 0 of
    // output ih+1 (Cc, starts from zero).  Absent neighbours are zeros: fma(0, w, acc) leaves acc unchanged.
#define HP_DW_STEP(A, B, Cc, IH)                                                                                                   \
    {                                                                                                                               \
        uint2 ul = { 0u, 0u }, ur = { 0u, 0u };                                                                                      \
        const uint2 uc = *(const uint2*)rp;                                                                                          \
        if (has_l) ul = *(const uint2*)(rp - in_ld);                                                                                 \
        if (has_r) ur = *(const uint2*)(rp + in_ld);                                                                                 \
        rp += row_in;                                                                                                                \
        const float2 l0 = __half22float2(*(const __half2*)&ul.x), l1 = __half22float2(*(const __half2*)&ul.y);                       \
        const float2 m0 = __half22float2(*(const __half2*)&uc.x), m1 = __half22float2(*(const __half2*)&uc.y);                       \
        const float2 r0 = __half22float2(*(const __half2*)&ur.x), r1 = __half22float2(*(const __half2*)&ur.y);                       \
        const float4 vl = { l0.x, l0.y, l1.x, l1.y }, vm = { m0.x, m0.y, m1.x, m1.y }, vr = { r0.x, r0.y, r1.x, r1.y };              \
        HP_FMA4(A, wt[6], vl); HP_FMA4(A, wt[7], vm); HP_FMA4(A, wt[8], vr);                                                         \
        HP_FMA4(B, wt[3], vl); HP_FMA4(B, wt[4], vm); HP_FMA4(B, wt[5], vr);                                                         \
        Cc = make_float4(0.f, 0.f, 0.f, 0.f);                                                                                        \
        HP_FMA4(Cc, wt[0], vl); HP_FMA4(Cc, wt[1], vm); HP_FMA4(Cc, wt[2], vr);                                                      \
        if ((IH) - 1 >= oh0) HP_DW_EMIT(A);                                                                                          \
    }
#define HP_DW_EMIT(A)                                                                                                              \
    {                                                                                                                               \
        float y0 = A.x + bs.x, y1 = A.y + bs.y, y2 = A.z + bs.z, y3 = A.w + bs.w;                                                    \
        y0 = y0 > 0.f ? y0 : y0 * al.x; y1 = y1 > 0.f ? y1 : y1 * al.y; y2 = y2 > 0.f ? y2 : y2 * al.z; y3 = y3 > 0.f ? y3 : y3 * al.w; \
        uint2 ov;                                                                                                                    \
        *(__half2*)&ov.x = __floats2half2_rn(y0, y1);                                                                                \
        *(__half2*)&ov.y = __floats2half2_rn(y2, y3);                                                                                \
        *(uint2*)op = ov;                                                                                                            \
        op += row_out;                                                                                                               \
    }
    const size_t row_in = (size_t)W * in_ld, row_out = (size_t)W * out_ld;
    const int ih_first = max(oh0 - 1, 0), ih_last = min(oh1, H - 1);   // valid input rows feeding this run
    const __half* rp = colp + (size_t)ih_first * row_in;
    __half* op = outp + (size_t)oh0 * row_out;
    int ih = ih_first;
    for (; ih + 2 <= ih_last; ih += 3) {   // three rows per trip: the accumulators rotate by renaming, not by moves
        HP_DW_STEP(a0, a1, a2, ih);
        HP_DW_STEP(a1, a2, a0, ih + 1);
        HP_DW_STEP(a2, a0, a1, ih + 2);
    }
    for (; ih <= ih_last; ++ih) {
        HP_DW_STEP(a0, a1, a2, ih);
        a0 = a1; a1 = a2;
    }
    if (oh1 - 1 >= ih_last) HP_DW_EMIT(a0);   // bottom image row: its last input row is padding (after the loop a0 holds output row ih_last)
#undef HP_DW_STEP
#undef HP_DW_EMIT
#undef HP_FMA4
}

// Depthwise 3x3 / stride 1 with the input staged by TMA (channel counts that are multiples of 64; NB = 1: one filter set, NB = 2: the two
// filter sets of a MobilenetThin stage's conf / paf branch on the same input).  The per-lane loads of dwconv3_col_kernel keep too few
// bytes in flight (the warps mostly wait on L1TEX loads at a small fraction of the DRAM bandwidth), so here a persistent CTA pulls
// whole tiles -- {64 channels, wbo + 2 columns, hb + 2 rows} of one frame, the 1-pixel halo included, out-of-image elements zero-filled
// by the TMA unit = the SAME padding -- through a ring of `stages` shared-memory buffers, one bulk tensor copy per tile, issued
// `stages - 1` tiles ahead.  Compute is the column march of dwconv3_col_kernel from shared memory: a lane owns a channel pair (the 32
// lanes of a warp read one pixel's 128 bytes: conflict-free), a warp a column of the tile; the accumulation order per output is the
// same (tap-row major, tap-column ascending, absent taps as zeros), as fmas on channel pairs (pair_math.cuh): bit-identical.
struct DwTmaParams {
    __half* out0; __half* out1; int out_ld;
    const float* w0; const float* w1;   // [9][C] | bias[C] | alpha[C]
    int H, W, C, ctiles, tiles_x, tiles_y, wbo, hb, n_items, stages;
};
constexpr int DWT_THREADS = 384;   // 12 warps
constexpr int DWT_STAGE_MAX = 73728;   // bytes of one tile buffer at most (3 of them + barriers fit 227 KB)

template <int NB>
__global__ void __launch_bounds__(DWT_THREADS, 1) dwconv3_tma_kernel(const __grid_constant__ CUtensorMap tmap_in, const DwTmaParams p)
{
    extern __shared__ uint8_t dwt_smem_raw[];
    const uint32_t base = (ptx::smem_u32(dwt_smem_raw) + 127u) & ~127u;
    const int bw = p.wbo + 2;
    const uint32_t stage_bytes = (uint32_t)(p.hb + 2) * (uint32_t)bw * 128u;
    const uint32_t bars = base + (uint32_t)p.stages * stage_bytes;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ptx::pdl_launch_dependents();
    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmap_in);
        for (int s = 0; s < p.stages; ++s) ptx::mbar_init(bars + 8u * s, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // work item -> tile: item = ((n * tiles_y + ty) * tiles_x + tx) * ctiles + ct, the channel tile fastest so that concurrent CTAs
    // read whole pixels
    auto tile_of = [&](int item, int& ct, int& tx, int& ty, int& n) {
        ct = item % p.ctiles; item /= p.ctiles;
        tx = item % p.tiles_x; item /= p.tiles_x;
        ty = item % p.tiles_y;
        n = item / p.tiles_y;
    };
    // k-th tile of this CTA -> its buffer (thread 0 only)
    auto issue = [&](int k) {
        const int item = (int)blockIdx.x + k * (int)gridDim.x;
        if (item >= p.n_items) return;
        int ct, tx, ty, n;
        tile_of(item, ct, tx, ty, n);
        const int s = k % p.stages;
        ptx::mbar_expect_tx(bars + 8u * s, stage_bytes);
        ptx::tma_load_4d(base + (uint32_t)s * stage_bytes, &tmap_in, bars + 8u * s, ct * 64, tx * p.wbo - 1, ty * p.hb - 1, n);
    };
    ptx::pdl_wait();   // the prologue above may run under the previous kernel's tail; its results are visible from here on
    if (threadIdx.x == 0)
        for (int k = 0; k < p.stages - 1; ++k) issue(k);
    const size_t row_out = (size_t)p.W * p.out_ld;
    float2 wa[9], wb[9], bsa, ala, bsb, alb;
    int ct_loaded = -1;
    for (int k = 0;; ++k) {
        const int item = (int)blockIdx.x + k * (int)gridDim.x;
        if (item >= p.n_items) break;
        __syncthreads();   // every warp is done with tile k-1: its buffer takes tile k + stages - 1
        if (threadIdx.x == 0) issue(k + p.stages - 1);
        int ct, tx, ty, n;
        tile_of(item, ct, tx, ty, n);
        const int c0 = ct * 64 + lane * 2;
        if (ct != ct_loaded) {
            ct_loaded = ct;
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                wa[q] = __ldg((const float2*)(p.w0 + (size_t)q * p.C + c0));
                if (NB == 2) wb[q] = __ldg((const float2*)(p.w1 + (size_t)q * p.C + c0));
            }
            bsa = __ldg((const float2*)(p.w0 + (size_t)9 * p.C + c0)); ala = __ldg((const float2*)(p.w0 + (size_t)10 * p.C + c0));
            if (NB == 2) { bsb = __ldg((const float2*)(p.w1 + (size_t)9 * p.C + c0)); alb = __ldg((const float2*)(p.w1 + (size_t)10 * p.C + c0)); }
        }
        const int x_lo = tx * p.wbo, y_lo = ty * p.hb;
        const int ncols = min(p.wbo, p.W - x_lo), nrows = min(p.hb, p.H - y_lo);
        const int s = k % p.stages;
        ptx::mbar_wait(bars + 8u * s, (uint32_t)(k / p.stages) & 1u);
        const uint32_t* tile = (const uint32_t*)(dwt_smem_raw + (base - ptx::smem_u32(dwt_smem_raw)) + (size_t)s * stage_bytes) + lane;
        const int row_words = bw * 32;
        for (int col = warp; col < ncols; col += (int)(blockDim.x >> 5)) {
            const uint32_t* sp = tile + col * 32;   // box row 0 (image row y_lo - 1), box columns col, col+1, col+2 = image x-1, x, x+1
            const size_t o = (((size_t)n * p.H + y_lo) * p.W + x_lo + col) * p.out_ld + c0;
            __half* opa = p.out0 + o;
            __half* opb = NB == 2 ? p.out1 + o : nullptr;
            float2 a0 = { 0.f, 0.f }, a1 = a0, a2 = a0, b0 = a0, b1 = a0, b2 = a0;
#define HP_DWT_EMIT(A, B)                                                                                                          \
            {                                                                                                                       \
                const float2 y = fadd2_rn(A, bsa), ys = fmul2_rn(y, ala);                                                        \
                *(__half2*)opa = __floats2half2_rn(y.x > 0.f ? y.x : ys.x, y.y > 0.f ? y.y : ys.y); opa += row_out;                  \
                if (NB == 2) {                                                                                                      \
                    const float2 z = fadd2_rn(B, bsb), zs = fmul2_rn(z, alb);                                                    \
                    *(__half2*)opb = __floats2half2_rn(z.x > 0.f ? z.x : zs.x, z.y > 0.f ? z.y : zs.y); opb += row_out;              \
                }                                                                                                                   \
            }
            // box row I: tap row 2 of output row I-2 (A0/B0, complete -> stored), tap row 1 of I-1 (A1/B1), tap row 0 of I (A2/B2, from zero)
#define HP_DWT_STEP(A0, A1, A2, B0, B1, B2, I)                                                                                     \
            {                                                                                                                       \
                const uint32_t ul = sp[0], uc = sp[32], ur = sp[64];                                                                 \
                sp += row_words;                                                                                                     \
                const float2 vl = __half22float2(*(const __half2*)&ul), vm = __half22float2(*(const __half2*)&uc), vr = __half22float2(*(const __half2*)&ur); \
                A0 = ffma2_rn(vl, wa[6], A0); A0 = ffma2_rn(vm, wa[7], A0); A0 = ffma2_rn(vr, wa[8], A0);                      \
                A1 = ffma2_rn(vl, wa[3], A1); A1 = ffma2_rn(vm, wa[4], A1); A1 = ffma2_rn(vr, wa[5], A1);                      \
                A2 = ffma2_rn(vl, wa[0], make_float2(0.f, 0.f)); A2 = ffma2_rn(vm, wa[1], A2); A2 = ffma2_rn(vr, wa[2], A2);   \
                if (NB == 2) {                                                                                                      \
                    B0 = ffma2_rn(vl, wb[6], B0); B0 = ffma2_rn(vm, wb[7], B0); B0 = ffma2_rn(vr, wb[8], B0);                  \
                    B1 = ffma2_rn(vl, wb[3], B1); B1 = ffma2_rn(vm, wb[4], B1); B1 = ffma2_rn(vr, wb[5], B1);                  \
                    B2 = ffma2_rn(vl, wb[0], make_float2(0.f, 0.f)); B2 = ffma2_rn(vm, wb[1], B2); B2 = ffma2_rn(vr, wb[2], B2); \
                }                                                                                                                   \
                if ((I) >= 2) HP_DWT_EMIT(A0, B0);                                                                                   \
            }
            const int R = nrows + 2;
            int i = 0;
            for (; i + 2 < R; i += 3) {   // three rows per trip: the accumulators rotate by renaming
                HP_DWT_STEP(a0, a1, a2, b0, b1, b2, i);
                HP_DWT_STEP(a1, a2, a0, b1, b2, b0, i + 1);
                HP_DWT_STEP(a2, a0, a1, b2, b0, b1, i + 2);
            }
            for (; i < R; ++i) {
                HP_DWT_STEP(a0, a1, a2, b0, b1, b2, i);
                a0 = a1; a1 = a2; b0 = b1; b1 = b2;
            }
#undef HP_DWT_STEP
#undef HP_DWT_EMIT
        }
    }
}

// OpenPifPaf heads (hyperpose/Model/pifpaf/model.py:215-281): raw 1x1-conv outputs [N,hc,wc,C] fp16 ->
//   pixel_shuffle(scale 2) (pifpaf/utils.py:371-379: in-channel ((nc*2+dy)*2+dx) -> out[nc, 2h+dy, 2w+dx]), crop to 2*hc-1,
//   reshape [fields, comps, ho, wo]; sigmoid on the confidences, softplus on the scales (inference branch, model.py:238-241,270-274);
//   regressed vectors are offsets from the cell, the C++ decoder wants absolute cell coordinates (postprocessor.cpp:326-328):
//   the index grid is added here (what the exported OpenPifPaf graph does).
template <typename T>
__global__ void __launch_bounds__(256) pifpaf_head_kernel(const T* __restrict__ raw, int raw_ld, float* __restrict__ out, int N, int hc, int wc,
                                                          int fields, int comps, int ho, int wo, int is_paf)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)N * fields * comps * ho * wo;
    if (idx >= total) return;
    const int x = (int)(idx % wo);
    size_t t = idx / wo;
    const int y = (int)(t % ho); t /= ho;
    const int comp = (int)(t % comps); t /= comps;
    const int k = (int)(t % fields);
    const int n = (int)(t / fields);
    const int nc = k * comps + comp;
    const int ch = (nc * 2 + (y & 1)) * 2 + (x & 1);
    float v = (float)raw[(((size_t)n * hc + (y >> 1)) * wc + (x >> 1)) * raw_ld + ch];
    const bool is_conf = comp == 0;
    const bool is_scale = is_paf ? (comp == 7 || comp == 8) : (comp == 4);
    const bool is_x = is_paf ? (comp == 1 || comp == 3) : (comp == 1);
    const bool is_y = is_paf ? (comp == 2 || comp == 4) : (comp == 2);
    if (is_conf) v = 1.f / (1.f + expf(-v));
    else if (is_scale) v = v > 20.f ? v : log1pf(expf(v));
    else if (is_x) v += (float)x;
    else if (is_y) v += (float)y;
    out[idx] = v;
}

// Pose Proposal Network head (hyperpose/Model/pose_proposal/model.py:84-93 + restore_coor :111-119, inference branch): the raw
// 1x1-conv output [N,gh,gw,raw_ld] -> sigmoid -> conf slot [N,6,K,gh,gw] (conf_point, conf_iou, x, y, w, h; the cell's offset and the
// size scaled to the network input) and edge slot [N,L*nh*nw,gh,gw] (the tf.reshape of :93 moves no data).  One thread per output
// element, in output order; every operation rounded on its own.
template <typename T>
__global__ void __launch_bounds__(256) ppn_head_kernel(const T* __restrict__ raw, int raw_ld, float* __restrict__ conf, float* __restrict__ edge,
                                                       int N, int gh, int gw, int K, int n_edge, float cw, float ch, float in_w, float in_h)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int G = gh * gw, nb = 6 * K, C = nb + n_edge;
    if (idx >= (size_t)N * C * G) return;
    const int pix = (int)(idx % G);
    const size_t t = idx / G;
    const int c = (int)(t % C), n = (int)(t / C);
    const int x = pix % gw, y = pix / gw;
    const float v = (float)raw[((size_t)n * G + pix) * raw_ld + c];
    const float s = 1.f / (1.f + expf(-v));
    if (c >= nb) { edge[((size_t)n * n_edge + (c - nb)) * G + pix] = s; return; }
    float o = s;
    switch (c / K) {
    case 2: o = __fmul_rn(__fadd_rn(s, (float)x), cw); break;
    case 3: o = __fmul_rn(__fadd_rn(s, (float)y), ch); break;
    case 4: o = __fmul_rn(s, in_w); break;
    case 5: o = __fmul_rn(s, in_h); break;
    default: break;   // conf_point, conf_iou
    }
    conf[((size_t)n * nb + c) * G + pix] = o;
}

// KxK (K = 2 or 3) stride-2 max pool, NHWC fp16, 8 channels per thread; TF "SAME" semantics (window clipped at the border).
template <int K>
__global__ void __launch_bounds__(256) maxpool2_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                                       int N, int H, int W, int C_in_ld, int C, int C_out_ld, int OH, int OW, int pad_h, int pad_w)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int cv = C / 8;
    const size_t total = (size_t)N * OH * OW * cv;
    if (idx >= total) return;
    const int c8 = (int)(idx % cv);
    size_t t = idx / cv;
    const int ow = (int)(t % OW); t /= OW;
    const int oh = (int)(t % OH);
    const int n = (int)(t / OH);
    if (K == 2) { // window rows/cols clamped to the last one: max(a, a) == a reproduces the clipped SAME window
        const int h0 = oh * 2, w0 = ow * 2;
        const int h1 = min(h0 + 1, H - 1), w1 = min(w0 + 1, W - 1);
        auto ld = [&](int h, int w) { return *(const uint4*)(in + (((size_t)n * H + h) * W + w) * C_in_ld + c8 * 8); };
        const uint4 a = ld(h0, w0), b = ld(h0, w1), c = ld(h1, w0), d = ld(h1, w1);
        const __half2* ra = (const __half2*)&a; const __half2* rb = (const __half2*)&b; const __half2* rc = (const __half2*)&c; const __half2* rd = (const __half2*)&d;
        uint4 r;
        __half2* rr = (__half2*)&r;
#pragma unroll
        for (int i = 0; i < 4; ++i) rr[i] = __hmax2(__hmax2(ra[i], rb[i]), __hmax2(rc[i], rd[i]));
        *(uint4*)(out + (((size_t)n * OH + oh) * OW + ow) * C_out_ld + c8 * 8) = r;
        return;
    }
    __half2 m[4];
    bool first = true;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int h = oh * 2 - pad_h + r;
        if (h < 0 || h >= H) continue;
#pragma unroll
        for (int s = 0; s < K; ++s) {
            const int w = ow * 2 - pad_w + s;
            if (w < 0 || w >= W) continue;
            const uint4 v = *(const uint4*)(in + (((size_t)n * H + h) * W + w) * C_in_ld + c8 * 8);
            const __half2* hv = (const __half2*)&v;
#pragma unroll
            for (int i = 0; i < 4; ++i) m[i] = first ? hv[i] : __hmax2(m[i], hv[i]);
            first = false;
        }
    }
    uint4 r4;
    __half2* rr = (__half2*)&r4;
#pragma unroll
    for (int i = 0; i < 4; ++i) rr[i] = m[i];
    *(uint4*)(out + (((size_t)n * OH + oh) * OW + ow) * C_out_ld + c8 * 8) = r4;
}

// ---------------------------------------------------------------------------------------------
// tensor maps (driver entry points fetched at run time: no link-time dependency on libcuda)
// ---------------------------------------------------------------------------------------------
void* driver_entry_point(const char* name)
{
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
    return p;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*, const int*,
                                     cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);
// TMA element type and size of an engine's activations / weights (the copy ignores signedness: int8 travels as UINT8)
CUtensorMapDataType tmap_type(int dtype)
{
    return dtype == HP_DTYPE_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : dtype == HP_DTYPE_INT8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}
int elem_bytes(int dtype) { return dtype == HP_DTYPE_TF32 ? 4 : dtype == HP_DTYPE_INT8 ? 1 : 2; }

// activations [N,H,W,C] fp16 (fp32, int8) in im2col mode: 128 consecutive output pixels x 128 bytes of channels per load; the bounding
// box [-pad, dim - pad) holds one base position per output pixel, filter taps are the im2col offsets of the copy instruction.
// Channels past C read as zeros.
int make_tmap_act_im2col(CUtensorMap* m, const void* base, int N, int H, int W, int C, int R, int S, int dtype)
{
    const int es = elem_bytes(dtype);
    const auto enc = (PFN_encodeIm2col)driver_entry_point("cuTensorMapEncodeIm2col");
    if (!enc) { set_error("cuTensorMapEncodeIm2col entry point not available"); return HP_ERR_CUDA; }
    cuuint64_t dims[4] = { (cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N };
    cuuint64_t strides[3] = { (cuuint64_t)C * es, (cuuint64_t)W * C * es, (cuuint64_t)H * W * C * es };
    const int pad_w = S / 2, pad_h = R / 2;
    int lower[2] = { -pad_w, -pad_h };
    int upper[2] = { pad_w - (S - 1), pad_h - (R - 1) };
    cuuint32_t estr[4] = { 1, 1, 1, 1 };
    CUresult r = enc(m, tmap_type(dtype), 4, (void*)base, dims, strides, lower, upper, 128 / es, (cuuint32_t)CONV_BLOCK_M, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeIm2col failed: %d (N=%d H=%d W=%d C=%d R=%d S=%d)", (int)r, N, H, W, C, R, S); return HP_ERR_CUDA; }
    return HP_OK;
}
// weights [rows, K] fp16 (fp32, int8) K-major: dims (K, rows), box (128 bytes, BN)
int make_tmap_wgt(CUtensorMap* m, const void* base, int rows, int K, int BN, int dtype)
{
    const int es = elem_bytes(dtype);
    const auto enc = (PFN_encodeTiled)driver_entry_point("cuTensorMapEncodeTiled");
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return HP_ERR_CUDA; }
    cuuint64_t dims[2] = { (cuuint64_t)K, (cuuint64_t)rows };
    cuuint64_t strides[1] = { (cuuint64_t)K * es };
    cuuint32_t box[2] = { (cuuint32_t)(128 / es), (cuuint32_t)BN };
    cuuint32_t estr[2] = { 1, 1 };
    CUresult r = enc(m, tmap_type(dtype), 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weights) failed: %d (rows=%d K=%d BN=%d)", (int)r, rows, K, BN); return HP_ERR_CUDA; }
    return HP_OK;
}

// a C-channel view (channel stride ld) of activations [N,H,W,ld] fp16 as a 4-D tiled tensor (C, W, H, N), box {64 ch, box_w, box_h, 1},
// out-of-tensor elements zero-filled on load.  The halo-box loads of conv_halo_kernel take the 128B swizzle, the halo'd tiles of
// dwconv3_tma_kernel none (a pixel's 64 channels = 128 contiguous bytes of shared memory).
int make_tmap_act_box(CUtensorMap* m, const __half* base, int N, int H, int W, int C, int ld, int box_w, int box_h, CUtensorMapSwizzle swizzle)
{
    const auto enc = (PFN_encodeTiled)driver_entry_point("cuTensorMapEncodeTiled");
    if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return HP_ERR_CUDA; }
    cuuint64_t dims[4] = { (cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N };
    cuuint64_t strides[3] = { (cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2 };
    cuuint32_t box[4] = { 64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1 };
    cuuint32_t estr[4] = { 1, 1, 1, 1 };
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(box) failed: %d (N=%d H=%d W=%d C=%d ld=%d box %dx%d)", (int)r, N, H, W, C, ld, box_w, box_h); return HP_ERR_CUDA; }
    return HP_OK;
}

int round_up(int a, int b) { return (a + b - 1) / b * b; }

int pick_bn(int cout_g)
{
    if (cout_g <= 16) return 16;
    if (cout_g <= 32) return 32;
    if (cout_g <= 48) return 48;
    if (cout_g <= 64) return 64;
    if (cout_g <= 96) return 96;
    if (cout_g <= 128) return 128;
    // wider layers: n-tiles of at most 128 channels (a 64 x 128 fp32 accumulator is 64 registers per thread); the width that pads
    // least, the wider one on a tie
    int best = 128;
    for (int bn : { 96, 64 })
        if (round_up(cout_g, bn) < round_up(cout_g, best)) best = bn;
    return best;
}

struct ConvPlan {
    ConvParams prm;
    CUtensorMap tmap_a, tmap_b;
    CUtensorMap tmap_x;          // halo plan: the input as a 4-D tensor with a (16+R-1) x (8+S-1)-pixel box
    void* d_w = nullptr;         // K-major weights: fp16, or fp32 rounded to TF32 (the engine's dtype)
    bool monotone_act = false;   // every PReLU slope of the layer is >= 0
    HaloParams hp;               // halo plan: conv_halo_kernel's parameters
    float* d_bias = nullptr;
    float* d_alpha = nullptr;
    float* d_mul = nullptr;      // INT8 engine: s_in * s_w[o] per (padded) output channel
    size_t smem = 0;
    double flops_per_frame = 0;
};

// What run_graph launches for an op: decided once when the engine is created, by build_conv_plan and the fusion passes
enum class Launch : uint8_t {
    None,           // taken by the launch of a neighbouring op (a conv epilogue, or the first op of a TMA depthwise pair)
    Im2col,         // im2col3_kernel
    StemOrIm2col,   // u8 frames: nothing, the consumer conv (ConvStem) gathers its patches from the frames; f32 entry: im2col3_kernel
    Conv,           // conv_wgmma_kernel
    ConvStem,       // u8 frames: conv_wgmma_kernel with the fused R x R stem (R = po.R); f32 entry: as Conv
    Halo,           // conv_halo_kernel: one TMA box per 16 x 8-pixel tile and channel chunk serves every filter tap
    HaloPool,       // conv_halo_kernel with the 2x2 max-pool that follows in its epilogue (hp.out is the POOLED buffer)
    HaloWide,       // conv_halo_kernel with 256-pixel work items: two 16 x 8 tiles share every weight tile
    HaloPP,         // conv_halo_kernel with ping-pong items: one 16 x 8 tile per consumer warpgroup, the two take turns on the tensor pipe
    HaloPoolPP,     // HaloPool on ping-pong items
    DwTma,          // dwconv3_tma_kernel<1>
    DwTmaPair,      // dwconv3_tma_kernel<2>: this op and the next one (same input, other filters)
    DwCol,          // dwconv3_col_kernel
    DwStrip,        // dwconv_kernel<K, stride>
    MaxPool,        // maxpool2_kernel
    Heads,          // two pifpaf_head_kernel launches
    PpnHead,        // ppn_head_kernel
    // TF32 engine: fp32 activations (conv_tf32.cuh); its convs are Conv
    Im2colF32, DwF32, MaxPoolF32, HeadsF32, PpnHeadF32,
    // INT8 engine: int8 activations (conv_int8.cuh); its convs are Conv
    Im2colI8, DwI8, MaxPoolI8,
};

// kernels an op launches per run: what launch_count counts, and what a graph replay of the step stands for
int kernels_launched(Launch k, bool u8_input)
{
    switch (k) {
    case Launch::None: return 0;
    case Launch::StemOrIm2col: return u8_input ? 0 : 1;
    case Launch::Heads: case Launch::HeadsF32: return 2;
    default: return 1;
    }
}

// does op q read buffer b (its input, a residual, or the second head input)?  The im2col op reads the frames.
bool reads_buffer(const PackOp& q, uint32_t b)
{
    if (q.type == OP_IM2COL3) return false;
    return q.in_buf == b || (((q.type == OP_CONV && q.res_mode) || q.type == OP_PIFPAF_HEAD) && q.res_buf == b);
}

struct EngOp {
    Launch launch = Launch::None;
    PackOp po;
    ConvPlan plan;              // OP_CONV only
    float* d_dw = nullptr;      // OP_DWCONV: [K*K][C] weights | bias[C] | alpha[C]
    // DwTma / DwTmaPair: the input's halo'd tiles
    CUtensorMap tmap_dw;
    int dwt_wbo = 0, dwt_hb = 0, dwt_tiles_x = 0, dwt_tiles_y = 0, dwt_stages = 0;
    size_t dwt_smem = 0;
};

// Environment switches, read once by hp_engine_create_ex.  Each selects the plainer form of a fused or TMA kernel path, the
// reference the tests compare the default against.
struct EngOptions {
    enum { HALO_AUTO, HALO_NONE, HALO_ALL } halo = HALO_AUTO;   // HPB_HALO=all | anything else; unset: build_conv_plan's rule
    bool halo_wide = true;       // HPB_HALO_NARROW: every halo layer takes the 128-pixel work item (neither wide nor ping-pong)
    bool stem3 = true;           // fused 3x3 stem; HPB_NO_STEM3 keeps the im2col buffer
    bool pool_fuse = true;       // HPB_NO_POOL_FUSE
    bool dw1_fuse = true;        // HPB_NO_DW1_FUSE
    bool dw_pair = true;         // HPB_NO_DW_DUAL
    bool dw_tma = true;          // HPB_NO_DW_TMA
    int pifpaf_reserve_sms = 0;  // HPB_PIFPAF_RESERVE_SMS (default min(max_batch, 16)), bounded by half the SMs
};

// TF "SAME": out = ceil(in / stride), pad_before = max((out - 1) * stride + k - in, 0) / 2
inline int same_pad_before(int in, int k, int stride)
{
    const int out = (in + stride - 1) / stride;
    const int total = std::max((out - 1) * stride + k - in, 0);
    return total / 2;
}

struct EngBuffer {
    bool fused_away = false;   // never written: its only consumer (a 2x2 max-pool / 1x1 depthwise op) runs inside the producing conv's epilogue
    int channels = 0, down = 0, H = 0, W = 0;
    __half* d = nullptr;
};

} // namespace

struct hp_engine {
    int device = 0;
    int dtype = 0;   // HP_DTYPE_F16 | HP_DTYPE_TF32 | HP_DTYPE_INT8
    std::vector<float> act_scale;   // INT8 engine: the pack's scale of every activation buffer
    int in_h = 0, in_w = 0, max_batch = 0;
    double factor = 1.0 / 255;
    int flip_rgb = 1;
    int num_sms = 132;
    EngOptions opt;
    PackHeader hdr;
    std::vector<EngBuffer> bufs;
    std::vector<EngOp> ops;
    int step_kernels = 0;          // kernels of one run of the whole graph on u8 frames
    float* d_conf = nullptr;
    float* d_paf = nullptr;
    int out_h = 0, out_w = 0;
    uint8_t* d_frames = nullptr;   // [max_batch, in_h, in_w, 3]
    float* d_input_f32 = nullptr;  // [max_batch, 3, in_h, in_w] (lazily)
    uint8_t* pin_frames = nullptr;
    cudaStream_t stream = nullptr;
    long long launches = 0;
    double flops_per_frame = 0;
    int last_N = 0;
    // frame staging with on-device resize (arbitrary-size frames)
    uint8_t* d_src = nullptr; size_t d_src_bytes = 0;
    uint8_t* pin_src = nullptr; size_t pin_src_bytes = 0;
    int* d_rz_xi = nullptr; short* d_rz_xa = nullptr; int* d_rz_yi = nullptr; short* d_rz_ya = nullptr;
    int rz_sh = -1, rz_sw = -1, rz_rh = 0, rz_rw = 0, rz_keep = -1, rz_area = 0;
    // benchmark hook: synthetic conf/paf copied over the outputs after the last conv (SURVEY 8d)
    const float* override_conf = nullptr;
    const float* override_paf = nullptr;
    // per-op CUDA-event profiling (bench.py roofline leg)
    bool profiling = false;
    static constexpr int EV_DEPTH = 4; // runs in flight: the host never waits for the GPU to read a run's events back
    std::vector<cudaEvent_t> ev;       // EV_DEPTH sets of n_ops + 1 events
    std::vector<double> op_ms_sum;     // accumulated per op
    long long profiled_runs = 0;
    long long ev_head = 0, ev_tail = 0; // event sets recorded / folded in
    // host read-back of the outputs (tensorrt::inference's per-image D2H) + the published device snapshots (handoff.h)
    float* pin_out = nullptr; size_t pin_out_floats = 0;
    std::shared_ptr<hpb::handoff::Batch> ho_ring[hpb::handoff::HANDOFF_RING];
    int ho_pos = 0;
    // network input of the NEXT run_graph: d_frames, or a slot buffer of the pipelined pose call
    const uint8_t* cur_frames = nullptr;
    bool stage_synced = false;     // hp_engine_stage_frame_u8: the previous batch's staging copies have been waited for
    // pipelined end-to-end call (hp_pose_submit_u8_host / hp_pose_collect): two batches in flight
    struct PoseSlot {
        uint8_t* d_frames = nullptr;       // this slot's device input
        uint8_t* pin_frames = nullptr;     // staging for pageable callers
        hp_human* pin_humans = nullptr; size_t pin_humans_n = 0;
        int* pin_counts = nullptr; size_t pin_counts_n = 0;   // [N counts | N flags]
        cudaEvent_t h2d_done = nullptr, done = nullptr;
        bool busy = false;
        int N = 0, hcap = 0;
        hp_paf* parser = nullptr;
        hp_pifpaf* decoder = nullptr;      // OpenPifPaf packs: the slot's batch is decoded on the decoder's stream
        cudaEvent_t conv_done = nullptr;   // (pifpaf) the engine's kernels of this slot have finished: the decoder may start
        cudaGraphExec_t graph = nullptr;   // captured launch sequence (convs + parse + result D2H) of this slot
        float key_f[2] = { 0, 0 }; int key_i[6] = { 0, 0, 0, 0, 0, 0 }; int key_N = 0; const void* key_parser = nullptr;
        const void* key_ovr[2] = { nullptr, nullptr };
    } slots[2];
    int next_slot = 0;
    bool use_pdl = false;                  // programmatic dependent launch for the conv / depthwise kernels (launch-bound networks)
    int reserve_sms = 0;                   // SMs the persistent conv kernels leave to a decoder running underneath them (pipelined pifpaf call)
    cudaEvent_t heads_wait = nullptr;      // run_graph: the head op waits for this event (the previous batch's fields have been consumed)
    cudaStream_t copy_stream = nullptr;
    bool graphs_ok = true;
    long long graph_launches = 0, graph_captures = 0;
};

namespace {

// round-to-nearest (ties away from zero in magnitude) onto the TF32 grid: 8-bit exponent, 10-bit mantissa
inline float tf32_round(float x)
{
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & 0xffffe000u;
    memcpy(&x, &u, 4);
    return x;
}

bool is_halo(Launch k)
{
    return k == Launch::Halo || k == Launch::HaloPool || k == Launch::HaloWide || k == Launch::HaloPP || k == Launch::HaloPoolPP;
}
HaloItem halo_item_of(Launch k)
{
    return k == Launch::HaloWide ? HaloItem::Wide : k == Launch::HaloPP || k == Launch::HaloPoolPP ? HaloItem::PingPong : HaloItem::Narrow;
}

// The halo plan's work item: one 16 x 8 tile (128 pixels) on both consumer warpgroups, two tiles sharing every weight tile
// (conv_halo_kernel<128, false, true>), or one tile per warpgroup with the two taking turns (conv_halo_kernel<BN, kPool, false, true>)
void set_halo_item(EngOp& op, HaloItem item, bool pool)
{
    HaloParams& h = op.plan.hp;
    h.num_stages = conv_halo_pick_stages(h.R, h.S, op.plan.prm.BN, item);
    op.plan.smem = conv_halo_smem_bytes(h.R, h.S, op.plan.prm.BN, h.num_stages, item);
    op.launch = item == HaloItem::Wide ? Launch::HaloWide : item == HaloItem::PingPong ? (pool ? Launch::HaloPoolPP : Launch::HaloPP)
                                                                                   : (pool ? Launch::HaloPool : Launch::Halo);
}

// Which halo layers take the wide item, from per-layer times of both items at the cfg3 / cfg4 / cfg5 benchmark batch sizes
// (tools/layer_times.py with and without HPB_HALO_NARROW, DESIGN.md §4): OpenPose's 7x7 refinement convs, 49 weight tiles per box,
// run 13-15 % faster.  The 3x3 layers gain at most 5 % (cin 512 at 46x82 and 46x54) and lose up to 46 % where a launch is a few
// rounds of short items (cfg4 / cfg5's 128- and 256-channel layers), so they keep the 128-pixel item.  Launches of fewer wide items
// than SMs were not measured; they leave SMs idle that the 128-pixel launch would use, and keep it.
bool halo_wide_faster(int R, long wide_items, int sms)
{
    return R == 7 && wide_items >= sms;
}

// The ping-pong item exists for 3x3 layers at BN = 64 and 128 (the VGG trunk's widths).  Which of them take it, from per-layer times
// of both items at the cfg3 / cfg4 / cfg5 benchmark batch sizes (tools/layer_times.py, DESIGN.md §4): layers of four or more
// 64-channel chunks (36+ k-steps per item: 12-17 % faster) and layers with the 2x2 max-pool in their epilogue (a quarter of the stores:
// 14-24 % faster, down to one chunk).  Shorter items with the full epilogue lose up to 14 %: one warpgroup's epilogue of a whole
// 16 x 8 x BN tile outlasts the other's 9 or 18 k-steps.  Launches of fewer than two items per CTA leave one warpgroup idle; they
// were not measured and keep the 128-pixel item.
bool halo_pp_exists(int R, int BN) { return R == 3 && (BN == 64 || BN == 128); }
bool halo_pp_faster(int chunks, bool pooled, long items, int sms) { return (chunks >= 4 || pooled) && items >= 2L * sms; }

// The halo layer's work item (halo_wide_faster, halo_pp_faster), its pool fused or not.  HPB_HALO=all takes the wide item wherever
// it exists and the ping-pong item where the wide one does not; HPB_HALO_NARROW=1 the 128-pixel item.
HaloItem pick_halo_item(const hp_engine* e, const EngOp& op, bool pooled)
{
    const HaloParams& h = op.plan.hp;
    const int BN = op.plan.prm.BN, sms = e->num_sms - e->reserve_sms;
    const long tiles = (long)h.Nb * h.tiles_x * h.tiles_y, n_tiles = (long)h.groups * (h.cout_g_pad / BN);
    const bool all = e->opt.halo == EngOptions::HALO_ALL;
    if (!e->opt.halo_wide) return HaloItem::Narrow;
    // the wide item: BN = 128 without the pool, and at least 3 weight stages next to its four boxes
    if (!pooled && BN == 128 && conv_halo_pick_stages(h.R, h.S, BN, HaloItem::Wide) >= 3 && (all || halo_wide_faster(h.R, (tiles + 1) / 2 * n_tiles, sms)))
        return HaloItem::Wide;
    if (halo_pp_exists(h.R, BN) && (all || halo_pp_faster(h.cin_g / CONV_BLOCK_K, pooled, tiles * n_tiles, sms))) return HaloItem::PingPong;
    return HaloItem::Narrow;
}

// The conv's GEMM operands, epilogue and tensor maps.  data_type::kHALF: fp16 activations and weights, 64-channel chunks;
// data_type::kFLOAT (HP_DTYPE_TF32): fp32 activations on the TF32 grid, 32-channel chunks (conv_wgmma_kernel<float, ...>);
// data_type::kINT8 (HP_DTYPE_INT8): int8 activations and per-output-channel int8 weights, 128-channel chunks
// (conv_wgmma_kernel<int8_t, ...>).  An INT8 k-step may run past the input buffer's last channel: the TMA reads those as zeros.
int build_conv_plan(hp_engine* e, EngOp& op, const float* blob)
{
    const PackOp& po = op.po;
    ConvPlan& pl = op.plan;
    const bool tf32 = e->dtype == HP_DTYPE_TF32, i8 = e->dtype == HP_DTYPE_INT8;
    const int chunk = tf32 ? 32 : i8 ? 128 : 64;
    const size_t es = (size_t)elem_bytes(e->dtype);
    const EngBuffer& ib = e->bufs[po.in_buf];
    const int G = (int)po.groups, R = (int)po.R, S = (int)po.S, cin_g = (int)po.cin_g, cout_g = (int)po.cout_g;
    const bool im2col = po.im2col_input != 0;
    if (im2col && (G != 1 || R * S * cin_g > ib.channels)) { set_error("engine: bad im2col conv"); return HP_ERR_ARG; }
    if (!im2col && G > 1 && cin_g % (i8 ? 16 : chunk) != 0) { set_error("engine: grouped conv needs cin_g %% %d == 0 (got %d)", i8 ? 16 : chunk, cin_g); return HP_ERR_UNSUPPORTED; }
    // effective GEMM view
    const int eR = im2col ? 1 : R, eS = im2col ? 1 : S;
    const int ecin = im2col ? round_up(R * S * cin_g, chunk) : round_up(cin_g, chunk);
    const int reads = i8 ? (im2col ? R * S * cin_g : G * cin_g) : G * ecin;   // channels that must lie inside the buffer
    if ((int)po.in_ch_off + reads > ib.channels) {
        set_error("engine: conv reads channels [%d,%d) of a %d-channel buffer", po.in_ch_off, po.in_ch_off + reads, ib.channels);
        return HP_ERR_ARG;
    }
    if (i8 && (long long)R * S * cin_g * 127 * 127 > 0x7fffffffLL) {   // the s32 accumulator must stay exact
        set_error("engine: INT8 conv op %d sums %d products per output (%dx%dx%d); the s32 accumulator is exact up to %d", (int)(&op - e->ops.data()), R * S * cin_g,
                  R, S, cin_g, 0x7fffffff / (127 * 127));
        return HP_ERR_UNSUPPORTED;
    }
    if (i8 && ib.channels % 16) {   // a TMA row stride is a multiple of 16 bytes
        set_error("engine: INT8 conv op %d reads buffer %u of %d channels (needs a multiple of 16)", (int)(&op - e->ops.data()), po.in_buf, ib.channels);
        return HP_ERR_ARG;
    }
    const int BN = pick_bn(cout_g);
    const int cout_pad = round_up(cout_g, BN);
    const int K = eR * eS * ecin;
    // repack fp32 [G][cout][cin][R][S] -> [G][cout_pad][R][S][cin_pad]
    std::vector<float> w((size_t)G * cout_pad * K, 0.f), bias((size_t)G * cout_pad, 0.f), alpha((size_t)G * cout_pad, 0.f);
    const float* W = blob + po.w_off;
    for (int g = 0; g < G; ++g)
        for (int o = 0; o < cout_g; ++o) {
            bias[(size_t)g * cout_pad + o] = blob[po.b_off + (size_t)g * cout_g + o];
            alpha[(size_t)g * cout_pad + o] = blob[po.a_off + (size_t)g * cout_g + o];
            for (int c = 0; c < cin_g; ++c)
                for (int r = 0; r < R; ++r)
                    for (int s = 0; s < S; ++s) {
                        const float v = W[((((size_t)g * cout_g + o) * cin_g + c) * R + r) * S + s];
                        const size_t k = im2col ? (size_t)((r * S + s) * cin_g + c) : ((size_t)(r * S + s) * ecin + c);
                        w[((size_t)g * cout_pad + o) * K + k] = tf32 ? tf32_round(v) : v;
                    }
        }
    std::vector<__half> wh;
    if (!tf32 && !i8) {
        wh.resize(w.size());
        for (size_t i = 0; i < w.size(); ++i) wh[i] = __float2half_rn(w[i]);
    }
    // INT8: s_w[o] = max |W[o]| / 127 (1 for an all-zero row), q = clamp(nearbyint(W / s_w), -127, 127), mul[o] = s_in * s_w[o]
    std::vector<int8_t> wq;
    std::vector<float> mul;
    if (i8) {
        wq.assign(w.size(), 0);
        mul.assign(bias.size(), 0.f);
        const float s_in = e->act_scale[po.in_buf];
        for (size_t row = 0; row < (size_t)G * cout_pad; ++row) {
            if ((int)(row % cout_pad) >= cout_g) continue;
            const float* wr = w.data() + row * K;
            float amax = 0.f;
            for (int k = 0; k < K; ++k) amax = std::max(amax, fabsf(wr[k]));
            const float sw = amax > 0.f ? amax / 127.0f : 1.0f;
            for (int k = 0; k < K; ++k) wq[row * K + k] = (int8_t)std::min(127.0f, std::max(-127.0f, nearbyintf(wr[k] / sw)));
            mul[row] = s_in * sw;
        }
        HP_CUDA_TRY(cudaMalloc(&pl.d_mul, mul.size() * sizeof(float)));
        HP_CUDA_TRY(cudaMemcpy(pl.d_mul, mul.data(), mul.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    HP_CUDA_TRY(cudaMalloc(&pl.d_w, w.size() * es));
    HP_CUDA_TRY(cudaMalloc(&pl.d_bias, bias.size() * sizeof(float)));
    HP_CUDA_TRY(cudaMalloc(&pl.d_alpha, alpha.size() * sizeof(float)));
    HP_CUDA_TRY(cudaMemcpy(pl.d_w, tf32 ? (const void*)w.data() : i8 ? (const void*)wq.data() : (const void*)wh.data(), w.size() * es, cudaMemcpyHostToDevice));
    HP_CUDA_TRY(cudaMemcpy(pl.d_bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
    HP_CUDA_TRY(cudaMemcpy(pl.d_alpha, alpha.data(), alpha.size() * sizeof(float), cudaMemcpyHostToDevice));

    ConvParams& p = pl.prm;
    memset(&p, 0, sizeof(p));
    p.Nb = e->max_batch; p.H = ib.H; p.W = ib.W;
    p.R = eR; p.S = eS; p.groups = G; p.cin_g = ecin;
    p.cout_g = cout_g; p.cout_g_pad = cout_pad; p.BN = BN;
    p.m_tiles = (int)(((size_t)e->max_batch * p.H * p.W + CONV_BLOCK_M - 1) / CONV_BLOCK_M);
    p.in_ch_off = (int)po.in_ch_off;
    p.num_stages = conv_pick_stages(BN);
    p.bias = pl.d_bias; p.alpha = pl.d_alpha;
    p.out_mode = (int)po.out_mode;
    if (po.out_mode == OUT_F32_NCHW_SPLIT) {
        p.out = e->d_conf; p.out2 = e->d_paf; p.split = (int)po.split;
        if ((int)po.split != (int)e->hdr.conf_channels || cout_g - (int)po.split != (int)e->hdr.paf_channels || G != 1) {
            set_error("engine: output conv must produce conf(%u)+paf(%u) channels", e->hdr.conf_channels, e->hdr.paf_channels);
            return HP_ERR_ARG;
        }
        // the conf / paf outputs hold out_h x out_w planes: the conv writes one per input pixel
        if (e->hdr.head_type != 0 || ib.H != e->out_h || ib.W != e->out_w) {
            set_error("engine: output conv op %d reads a %dx%d buffer but the outputs are %dx%d conf/paf planes (head_type %u)",
                      (int)(&op - e->ops.data()), ib.H, ib.W, e->out_h, e->out_w, e->hdr.head_type);
            return HP_ERR_ARG;
        }
    } else {
        const EngBuffer& ob = e->bufs[po.out_buf];
        if (ob.H != ib.H || ob.W != ib.W || (int)po.out_ch_off + G * cout_g > ob.channels) { set_error("engine: conv output buffer mismatch"); return HP_ERR_ARG; }
        p.out = ob.d; p.out_ld = ob.channels; p.out_ch_off = (int)po.out_ch_off;
        if (i8) p.out_inv_scale = 1.0f / e->act_scale[po.out_buf];
    }
    if (i8) { p.mul = pl.d_mul; p.in_g_stride = cin_g; }
    if (po.res_mode) {
        if (po.out_mode != OUT_F16_NHWC || po.res_buf >= e->bufs.size()) { set_error("engine: bad residual"); return HP_ERR_ARG; }
        const EngBuffer& rb = e->bufs[po.res_buf];
        if (rb.H != ib.H || rb.W != ib.W || (int)po.res_ch_off + G * cout_g > rb.channels || po.res_ch_off % 8 || cout_g % 16) { set_error("engine: residual buffer mismatch"); return HP_ERR_ARG; }
        p.res = rb.d; p.res_ld = rb.channels; p.res_ch_off = (int)po.res_ch_off; p.res_mode = (int)po.res_mode;
        if (i8) p.res_scale = e->act_scale[po.res_buf];
    }
    int rc = make_tmap_act_im2col(&pl.tmap_a, ib.d, e->max_batch, ib.H, ib.W, ib.channels, eR, eS, e->dtype);
    if (rc) return rc;
    rc = make_tmap_wgt(&pl.tmap_b, pl.d_w, G * cout_pad, K, BN, e->dtype);
    if (rc) return rc;
    pl.smem = conv_smem_bytes(BN, p.num_stages);
    pl.flops_per_frame = 2.0 * ib.H * ib.W * (double)G * cout_g * cin_g * R * S;
    op.launch = Launch::Conv;
    if (e->dtype != HP_DTYPE_F16) return HP_OK;   // the TF32 and INT8 engines have no halo kernel
    pl.monotone_act = true;
    for (float a : alpha) if (!(a >= 0.f)) { pl.monotone_act = false; break; }
    // Halo-box kernel: the A operand comes from L2 once per chunk instead of once per tap, in exchange for the pixels its 16 x 8 tile
    // grid computes outside the image (waste).  Per-layer times of the cfg3 / cfg4 / cfg5 graphs at their benchmark batch sizes on
    // both kernels (tools/layer_times.py, DESIGN.md §4) give the rule:
    //  * 3x3 layers whose grid wastes at most 6 % of the image: always (VGG conv1_2 -- conv2_2, 1.4-1.6x faster);
    //  * layers of two or more 64-channel chunks whose grid wastes at most 25 %, when the im2col grid needs more than one round of
    //    CTAs: the 3x3 layers of 128-512 channels at 46x54 to 193x193 (5-32 % faster) and OpenPose's 7x7 refinement convs (within 3 % either way).
    // It loses on one-chunk layers (ResNet-50's 64-channel 3x3 at 92x108 and 193x193: 7-17 % slower) and where the grid wastes half the
    // image (49x49 and 25x25: 6-10 % slower).  Launches of at most one round were not measured; they keep the first rule only.
    const int ty = (ib.H + HALO_TH - 1) / HALO_TH, tx = (ib.W + HALO_TW - 1) / HALO_TW;
    const double waste = (double)ty * HALO_TH * tx * HALO_TW / ((double)ib.H * ib.W) - 1.0;
    const bool shape_ok = !im2col && eR == eS && (eR == 3 || eR == 5 || eR == 7) && !po.res_mode && po.out_mode == OUT_F16_NHWC;
    const bool rounds = (long)p.m_tiles * G * (cout_pad / BN) > e->num_sms - e->reserve_sms;
    const bool faster = (eR == 3 && waste <= 0.06) || (rounds && ecin >= 2 * CONV_BLOCK_K && waste <= 0.25);
    const bool want = e->opt.halo == EngOptions::HALO_AUTO ? faster : e->opt.halo == EngOptions::HALO_ALL;
    if (shape_ok && want) {
        const EngBuffer& ob = e->bufs[po.out_buf];
        HaloParams& h = pl.hp;
        memset(&h, 0, sizeof(h));
        h.Nb = e->max_batch; h.H = ib.H; h.W = ib.W; h.R = eR; h.S = eS; h.groups = G; h.cin_g = ecin;
        h.cout_g = cout_g; h.cout_g_pad = cout_pad; h.in_ch_off = (int)po.in_ch_off;
        h.tiles_x = tx; h.tiles_y = ty;
        h.box_bytes = halo_box_bytes(eR, eS);
        h.bias = pl.d_bias; h.alpha = pl.d_alpha;
        h.out = ob.d; h.out_ld = ob.channels; h.out_ch_off = (int)po.out_ch_off;
        rc = make_tmap_act_box(&pl.tmap_x, ib.d, e->max_batch, ib.H, ib.W, ib.channels, ib.channels, HALO_TW + eS - 1, HALO_TH + eR - 1, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
        set_halo_item(op, pick_halo_item(e, op, false), false);
    }
    return HP_OK;
}

// Launch with programmatic dependent launch allowed: the kernel may begin (prologue: barrier init, tensor-map prefetch) on every SM
// the previous kernel of the stream has already left, and orders itself behind that kernel's completion with griddepcontrol.wait
// before it touches memory.  The persistent conv kernels trigger their dependents at their own start.  It pays where a step is a
// chain of short kernels and costs where they are long, so the engine turns it on by itself when the mean work per launch is small
// (hp_engine::use_pdl, decided at creation).
thread_local bool tl_use_pdl = false;   // set by the op loop from hp_engine::use_pdl for the launches it issues on this thread
static inline cudaLaunchConfig_t pdl_config(int grid, int block, size_t smem, cudaStream_t st, cudaLaunchAttribute* at)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = tl_use_pdl ? 1 : 0;
    return cfg;
}
template <typename... KArgs, typename... Args>
static inline void launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args&&... args)
{
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = pdl_config(grid, block, smem, st, at);
    cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// conv_wgmma_kernel instantiations: activation type (fp16 / TF32 engine) x tile width x residual epilogue x fused u8 stem
template <typename T, bool kRes, int kStemR = 0>
const void* conv_kernel_bn(int BN)
{
    switch (BN) {
    case 16: return (const void*)conv_wgmma_kernel<T, 16, kRes, kStemR>;
    case 32: return (const void*)conv_wgmma_kernel<T, 32, kRes, kStemR>;
    case 48: return (const void*)conv_wgmma_kernel<T, 48, kRes, kStemR>;
    case 64: return (const void*)conv_wgmma_kernel<T, 64, kRes, kStemR>;
    case 96: return (const void*)conv_wgmma_kernel<T, 96, kRes, kStemR>;
    case 128: return (const void*)conv_wgmma_kernel<T, 128, kRes, kStemR>;
    }
    return nullptr;
}
template <bool kPool>
const void* halo_kernel_bn(int BN)
{
    switch (BN) {
    case 16: return (const void*)conv_halo_kernel<16, kPool>;
    case 32: return (const void*)conv_halo_kernel<32, kPool>;
    case 48: return (const void*)conv_halo_kernel<48, kPool>;
    case 64: return (const void*)conv_halo_kernel<64, kPool>;
    case 96: return (const void*)conv_halo_kernel<96, kPool>;
    case 128: return (const void*)conv_halo_kernel<128, kPool>;
    }
    return nullptr;
}
// Launch::Halo / HaloPool / HaloWide / HaloPP / HaloPoolPP (the wide item exists for BN = 128 only, the ping-pong item for BN = 64
// and 128, see build_conv_plan)
const void* halo_kernel(Launch k, int BN)
{
    if (k == Launch::HaloWide) return BN == 128 ? (const void*)conv_halo_kernel<128, false, true> : nullptr;
    if (k == Launch::HaloPP || k == Launch::HaloPoolPP) {
        const bool pool = k == Launch::HaloPoolPP;
        if (BN == 64) return pool ? (const void*)conv_halo_kernel<64, true, false, true> : (const void*)conv_halo_kernel<64, false, false, true>;
        if (BN == 128) return pool ? (const void*)conv_halo_kernel<128, true, false, true> : (const void*)conv_halo_kernel<128, false, false, true>;
        return nullptr;
    }
    return k == Launch::HaloPool ? halo_kernel_bn<true>(BN) : halo_kernel_bn<false>(BN);
}
const void* conv_kernel(int dtype, bool res, int BN, int stem_R = 0)
{
    if (stem_R == 3) return conv_kernel_bn<__half, false, 3>(BN);
    if (stem_R == 7) return conv_kernel_bn<__half, false, 7>(BN);
    if (dtype == HP_DTYPE_TF32) return res ? conv_kernel_bn<float, true>(BN) : conv_kernel_bn<float, false>(BN);
    if (dtype == HP_DTYPE_INT8) return res ? conv_kernel_bn<int8_t, true>(BN) : conv_kernel_bn<int8_t, false>(BN);
    return res ? conv_kernel_bn<__half, true>(BN) : conv_kernel_bn<__half, false>(BN);
}

// depthwise 3x3 / stride 1 through dwconv3_tma_kernel; `pair` = the second depthwise op of a conf / paf branch pair (same input) or nullptr
void launch_dw_tma(hp_engine* e, const EngOp& op, const EngOp* pair, int N, cudaStream_t st)
{
    const PackOp& po = op.po;
    const EngBuffer& ib = e->bufs[po.in_buf];
    const EngBuffer& ob = e->bufs[po.out_buf];
    DwTmaParams p;
    p.out0 = ob.d + po.out_ch_off;
    p.out1 = pair ? e->bufs[pair->po.out_buf].d + pair->po.out_ch_off : nullptr;
    p.out_ld = ob.channels;
    p.w0 = op.d_dw; p.w1 = pair ? pair->d_dw : nullptr;
    p.H = ib.H; p.W = ib.W; p.C = (int)po.cout_g; p.ctiles = p.C / 64;
    p.tiles_x = op.dwt_tiles_x; p.tiles_y = op.dwt_tiles_y; p.wbo = op.dwt_wbo; p.hb = op.dwt_hb; p.stages = op.dwt_stages;
    p.n_items = N * p.tiles_y * p.tiles_x * p.ctiles;
    const int grid = std::min(p.n_items, std::max(1, e->num_sms - e->reserve_sms));
    if (pair) launch_pdl(dwconv3_tma_kernel<2>, grid, DWT_THREADS, op.dwt_smem, st, op.tmap_dw, p);
    else      launch_pdl(dwconv3_tma_kernel<1>, grid, DWT_THREADS, op.dwt_smem, st, op.tmap_dw, p);
}

// conv_wgmma_kernel, or conv_halo_kernel for the Halo* launches
int launch_conv(hp_engine* e, EngOp& op, int N, cudaStream_t st, bool u8_input)
{
    ConvPlan& pl = op.plan;
    ConvParams p = pl.prm;
    p.Nb = N;
    const int stem_R = op.launch == Launch::ConvStem && u8_input ? (int)op.po.R : 0;
    p.frames = e->cur_frames ? e->cur_frames : e->d_frames;
    if (is_halo(op.launch)) {
        HaloParams h = pl.hp;
        h.Nb = N;
        const int tiles = op.launch == Launch::HaloWide ? 2 : 1;
        const long items = ((long)N * h.tiles_x * h.tiles_y + tiles - 1) / tiles * h.groups * (h.cout_g_pad / p.BN);
        cudaLaunchAttribute at[1];
        const cudaLaunchConfig_t cfg = pdl_config((int)std::min<long>(e->num_sms - e->reserve_sms, items), CONV_THREADS, pl.smem, st, at);
        void* args[] = { (void*)&pl.tmap_x, (void*)&pl.tmap_b, (void*)&h };
        HP_CUDA_TRY(cudaLaunchKernelExC(&cfg, halo_kernel(op.launch, p.BN), args));
        return HP_OK;
    }
    p.m_tiles = (int)(((size_t)N * p.H * p.W + CONV_BLOCK_M - 1) / CONV_BLOCK_M);
    const int n_tiles = p.m_tiles * p.groups * (p.cout_g_pad / p.BN);
    const int grid = std::min(e->num_sms - e->reserve_sms, n_tiles);
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = pdl_config(grid, CONV_THREADS, pl.smem, st, at);
    void* args[] = { (void*)&pl.tmap_a, (void*)&pl.tmap_b, (void*)&p };
    HP_CUDA_TRY(cudaLaunchKernelExC(&cfg, conv_kernel(e->dtype, p.res_mode != 0, p.BN, stem_R), args));
    return HP_OK;
}

// folds the oldest recorded event set into the per-op sums; non-blocking mode gives up if that run is still executing
bool collect_one(hp_engine* e, bool blocking)
{
    if (e->ev_tail >= e->ev_head) return false;
    const size_t n = e->ops.size();
    cudaEvent_t* set = e->ev.data() + (size_t)(e->ev_tail % hp_engine::EV_DEPTH) * (n + 1);
    if (!blocking && cudaEventQuery(set[n]) != cudaSuccess) { cudaGetLastError(); return false; }
    cudaEventSynchronize(set[n]);
    for (size_t i = 0; i < n; ++i) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, set[i], set[i + 1]) == cudaSuccess) e->op_ms_sum[i] += ms;
    }
    e->profiled_runs++;
    e->ev_tail++;
    return true;
}

void collect_profile(hp_engine* e)
{
    while (collect_one(e, true)) {}
}

// the OpenPifPaf head op: pif fields [N,17,5,h,w] from in_buf, paf fields [N,19,9,h,w] from res_buf
template <typename T>
void launch_heads(hp_engine* e, const PackOp& po, int N, cudaStream_t st)
{
    if (e->heads_wait) cudaStreamWaitEvent(st, e->heads_wait, 0);   // the previous batch's decoder has read the field tensors
    const EngBuffer& a = e->bufs[po.in_buf];
    const EngBuffer& b = e->bufs[po.res_buf];
    const size_t t1 = (size_t)N * 17 * 5 * e->out_h * e->out_w, t2 = (size_t)N * 19 * 9 * e->out_h * e->out_w;
    pifpaf_head_kernel<T><<<(int)((t1 + 255) / 256), 256, 0, st>>>((const T*)a.d, a.channels, e->d_conf, N, a.H, a.W, 17, 5, e->out_h, e->out_w, 0);
    pifpaf_head_kernel<T><<<(int)((t2 + 255) / 256), 256, 0, st>>>((const T*)b.d, b.channels, e->d_paf, N, b.H, b.W, 19, 9, e->out_h, e->out_w, 1);
}

// the PPN head op: boxes [N,6,K,gh,gw] into the conf slot, edges [N,L,nh,nw,gh,gw] into the paf slot, from in_buf.  restore_coor's grid
// size is the engine's input size over the output grid, rounded once to fp32.
template <typename T>
void launch_ppn_head(hp_engine* e, const PackOp& po, int N, cudaStream_t st)
{
    const EngBuffer& a = e->bufs[po.in_buf];
    const int K = (int)po.cout_g, n_edge = (int)(po.groups * po.R * po.S);
    const size_t total = (size_t)N * (6 * K + n_edge) * e->out_h * e->out_w;
    ppn_head_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const T*)a.d, a.channels, e->d_conf, e->d_paf, N, e->out_h, e->out_w, K, n_edge,
                                                                        (float)((double)e->in_w / e->out_w), (float)((double)e->in_h / e->out_h),
                                                                        (float)e->in_w, (float)e->in_h);
}

int run_graph(hp_engine* e, int N, bool u8_input, cudaStream_t st, int first = 0, int last = -1)
{
    if (last < 0) last = (int)e->ops.size() - 1;
    const bool prof = e->profiling && first == 0 && last == (int)e->ops.size() - 1;
    cudaEvent_t* evset = nullptr;
    if (prof) {
        while (collect_one(e, false)) {}                                            // finished runs, without waiting
        if (e->ev_head - e->ev_tail >= hp_engine::EV_DEPTH) collect_one(e, true);   // ring full: wait for the oldest
        evset = e->ev.data() + (size_t)(e->ev_head % hp_engine::EV_DEPTH) * (e->ops.size() + 1);
        cudaEventRecord(evset[0], st);
    }
    tl_use_pdl = e->use_pdl;
    const uint8_t* frames = e->cur_frames ? e->cur_frames : e->d_frames;
    for (int oi = first; oi <= last; ++oi) {
        EngOp& op = e->ops[oi];
        const PackOp& po = op.po;
        const int K = (int)po.R, stride = po.stride ? (int)po.stride : 1;
        switch (op.launch) {
        case Launch::None:
            break;
        case Launch::StemOrIm2col:
            if (u8_input) break;   // the consumer conv gathers its patches from the frames itself
            [[fallthrough]];
        case Launch::Im2col: {
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int R = K ? K : 3, chunks = ob.channels / 64;
            const dim3 blocks((unsigned)(((size_t)N * ob.H * ob.W + 255) / 256), (unsigned)chunks);
            const int ph = same_pad_before(e->in_h, R, stride), pw = same_pad_before(e->in_w, R, stride);
#define HP_IM2COL(U8, RR, SRC, FAC, FLIP) im2col3_kernel<U8, RR><<<blocks, 256, 0, st>>>(SRC, ob.d, N, e->in_h, e->in_w, FAC, FLIP, \
                e->hdr.mean[0], e->hdr.mean[1], e->hdr.mean[2], stride, ob.H, ob.W, ph, pw, chunks)
            if (u8_input) { if (R == 3) HP_IM2COL(true, 3, frames, e->factor, e->flip_rgb); else HP_IM2COL(true, 7, frames, e->factor, e->flip_rgb); }
            else          { if (R == 3) HP_IM2COL(false, 3, e->d_input_f32, 1.0, 0); else HP_IM2COL(false, 7, e->d_input_f32, 1.0, 0); }
#undef HP_IM2COL
            break;
        }
        case Launch::Conv: case Launch::ConvStem: case Launch::Halo: case Launch::HaloPool: case Launch::HaloWide: case Launch::HaloPP: case Launch::HaloPoolPP:
            launch_conv(e, op, N, st, u8_input);
            break;
        case Launch::DwTma:
            launch_dw_tma(e, op, nullptr, N, st);
            break;
        case Launch::DwTmaPair:
            launch_dw_tma(e, op, &e->ops[oi + 1], N, st);
            break;
        case Launch::DwCol: {
            // column-marching kernel: enough row chunks to give every SM a few blocks
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g;
            const size_t base = ((size_t)N * ib.W * (C / 4) + 255) / 256;
            int chunks = (int)((4 * (size_t)e->num_sms + base - 1) / base);
            chunks = std::max(1, std::min(chunks, std::max(1, ib.H / 4)));
            const int rows = (ib.H + chunks - 1) / chunks;
            chunks = (ib.H + rows - 1) / rows;
            const size_t tot = (size_t)N * chunks * ib.W * (C / 4);
            dwconv3_col_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(ib.d + po.in_ch_off, ib.channels, ob.d + po.out_ch_off, ob.channels, op.d_dw,
                op.d_dw + (size_t)9 * C, op.d_dw + (size_t)9 * C + C, N, ib.H, ib.W, C, rows, chunks);
            break;
        }
        case Launch::DwStrip: {   // 3x3 / stride 2 and 1x1
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g;
            const size_t total = (size_t)N * ob.H * ((ob.W + DW_STRIP - 1) / DW_STRIP) * (C / 8);
            const int blocks = (int)((total + 255) / 256);
            const float* dw = op.d_dw;
#define HP_DW(KK, SS) dwconv_kernel<KK, SS><<<blocks, 256, 0, st>>>(ib.d + po.in_ch_off, ib.channels, ob.d + po.out_ch_off, ob.channels, dw, \
                dw + (size_t)KK * KK * C, dw + (size_t)KK * KK * C + C, N, ib.H, ib.W, C, ob.H, ob.W, same_pad_before(ib.H, KK, SS), same_pad_before(ib.W, KK, SS))
            if (K == 3) HP_DW(3, 2);
            else if (stride == 2) HP_DW(1, 2);
            else HP_DW(1, 1);
#undef HP_DW
            break;
        }
        case Launch::MaxPool: {
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g;
            const int blocks = (int)(((size_t)N * ob.H * ob.W * (C / 8) + 255) / 256);
            if (K == 3)
                maxpool2_kernel<3><<<blocks, 256, 0, st>>>(ib.d + po.in_ch_off, ob.d + po.out_ch_off, N, ib.H, ib.W, ib.channels, C, ob.channels, ob.H, ob.W,
                                                           same_pad_before(ib.H, 3, 2), same_pad_before(ib.W, 3, 2));
            else
                maxpool2_kernel<2><<<blocks, 256, 0, st>>>(ib.d + po.in_ch_off, ob.d + po.out_ch_off, N, ib.H, ib.W, ib.channels, C, ob.channels, ob.H, ob.W,
                                                           same_pad_before(ib.H, 2, 2), same_pad_before(ib.W, 2, 2));
            break;
        }
        case Launch::Heads:
            launch_heads<__half>(e, po, N, st);
            break;
        case Launch::Im2colF32: {
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int R = K ? K : 3;
            const int ph = same_pad_before(e->in_h, R, stride), pw = same_pad_before(e->in_w, R, stride);
            const unsigned blocks = (unsigned)(((size_t)N * ob.H * ob.W * (ob.channels / 4) + 255) / 256);
            if (u8_input) im2col_f32_kernel<true><<<blocks, 256, 0, st>>>(frames, (float*)ob.d, N, e->in_h, e->in_w, e->factor, e->flip_rgb, e->hdr.mean[0], e->hdr.mean[1], e->hdr.mean[2],
                                                                         R, stride, ob.H, ob.W, ph, pw, ob.channels);
            else im2col_f32_kernel<false><<<blocks, 256, 0, st>>>(e->d_input_f32, (float*)ob.d, N, e->in_h, e->in_w, 1.0, 0, e->hdr.mean[0], e->hdr.mean[1], e->hdr.mean[2],
                                                                  R, stride, ob.H, ob.W, ph, pw, ob.channels);
            break;
        }
        case Launch::DwF32: {
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g;
            const size_t total = (size_t)N * ob.H * ob.W * (C / 4);
            const float* dw = op.d_dw;
            dwconv_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float*)ib.d + po.in_ch_off, ib.channels, (float*)ob.d + po.out_ch_off, ob.channels, dw,
                dw + (size_t)K * K * C, dw + (size_t)K * K * C + C, N, ib.H, ib.W, C, ob.H, ob.W, K, stride, same_pad_before(ib.H, K, stride), same_pad_before(ib.W, K, stride));
            break;
        }
        case Launch::MaxPoolF32: {
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g, KP = K ? K : 2;
            const size_t total = (size_t)N * ob.H * ob.W * (C / 4);
            maxpool_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float*)ib.d + po.in_ch_off, (float*)ob.d + po.out_ch_off, N, ib.H, ib.W, ib.channels, C, ob.channels,
                                                                               ob.H, ob.W, KP, same_pad_before(ib.H, KP, 2), same_pad_before(ib.W, KP, 2));
            break;
        }
        case Launch::HeadsF32:
            launch_heads<float>(e, po, N, st);
            break;
        case Launch::PpnHead:
            launch_ppn_head<__half>(e, po, N, st);
            break;
        case Launch::PpnHeadF32:
            launch_ppn_head<float>(e, po, N, st);
            break;
        case Launch::Im2colI8: {
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int R = K ? K : 3;
            const int ph = same_pad_before(e->in_h, R, stride), pw = same_pad_before(e->in_w, R, stride);
            const unsigned blocks = (unsigned)(((size_t)N * ob.H * ob.W * (ob.channels / 4) + 255) / 256);
            const float inv_s = 1.0f / e->act_scale[po.out_buf];
            if (u8_input) im2col_i8_kernel<true><<<blocks, 256, 0, st>>>(frames, (int8_t*)ob.d, N, e->in_h, e->in_w, e->factor, e->flip_rgb, e->hdr.mean[0], e->hdr.mean[1],
                                                                        e->hdr.mean[2], R, stride, ob.H, ob.W, ph, pw, ob.channels, inv_s);
            else im2col_i8_kernel<false><<<blocks, 256, 0, st>>>(e->d_input_f32, (int8_t*)ob.d, N, e->in_h, e->in_w, 1.0, 0, e->hdr.mean[0], e->hdr.mean[1], e->hdr.mean[2],
                                                                 R, stride, ob.H, ob.W, ph, pw, ob.channels, inv_s);
            break;
        }
        case Launch::DwI8: {
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g;
            const size_t total = (size_t)N * ob.H * ob.W * (C / 4);
            const float* dw = op.d_dw;
            dwconv_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const int8_t*)ib.d + po.in_ch_off, ib.channels, (int8_t*)ob.d + po.out_ch_off, ob.channels, dw,
                dw + (size_t)K * K * C, dw + (size_t)K * K * C + C, N, ib.H, ib.W, C, ob.H, ob.W, K, stride, same_pad_before(ib.H, K, stride), same_pad_before(ib.W, K, stride),
                e->act_scale[po.in_buf], 1.0f / e->act_scale[po.out_buf]);
            break;
        }
        case Launch::MaxPoolI8: {
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            const int C = (int)po.cout_g, KP = K ? K : 2;
            const size_t total = (size_t)N * ob.H * ob.W * (C / 4);
            maxpool_i8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const int8_t*)ib.d + po.in_ch_off, (int8_t*)ob.d + po.out_ch_off, N, ib.H, ib.W, ib.channels, C, ob.channels,
                                                                              ob.H, ob.W, KP, same_pad_before(ib.H, KP, 2), same_pad_before(ib.W, KP, 2));
            break;
        }
        }
        e->launches += kernels_launched(op.launch, u8_input);
        if (prof) cudaEventRecord(evset[oi + 1], st);
    }
    if (prof) e->ev_head++;
    if (e->override_conf && e->override_paf && last == (int)e->ops.size() - 1) {
        const size_t plane = (size_t)e->out_h * e->out_w;
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_conf, e->override_conf, N * e->hdr.conf_channels * plane * sizeof(float), cudaMemcpyDeviceToDevice, st));
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_paf, e->override_paf, N * e->hdr.paf_channels * plane * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    HP_CUDA_TRY(cudaGetLastError());
    e->last_N = N;
    return HP_OK;
}

void free_engine(hp_engine* e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    hpb::handoff::retire_ring(e->ho_ring);
    if (e->pin_out) cudaFreeHost(e->pin_out);
    for (auto& b : e->bufs) if (b.d) cudaFree(b.d);
    for (auto& o : e->ops) {
        if (o.plan.d_w) cudaFree(o.plan.d_w);
        if (o.plan.d_bias) cudaFree(o.plan.d_bias);
        if (o.plan.d_alpha) cudaFree(o.plan.d_alpha);
        if (o.plan.d_mul) cudaFree(o.plan.d_mul);
        if (o.d_dw) cudaFree(o.d_dw);
    }
    if (e->d_conf) cudaFree(e->d_conf);
    if (e->d_paf) cudaFree(e->d_paf);
    if (e->d_frames) cudaFree(e->d_frames);
    if (e->d_input_f32) cudaFree(e->d_input_f32);
    if (e->pin_frames) cudaFreeHost(e->pin_frames);
    if (e->d_src) cudaFree(e->d_src);
    if (e->pin_src) cudaFreeHost(e->pin_src);
    if (e->d_rz_xi) cudaFree(e->d_rz_xi);
    if (e->d_rz_xa) cudaFree(e->d_rz_xa);
    if (e->d_rz_yi) cudaFree(e->d_rz_yi);
    if (e->d_rz_ya) cudaFree(e->d_rz_ya);
    for (auto& ev : e->ev) cudaEventDestroy(ev);
    for (int i = 0; i < 2; ++i) {
        auto& sl = e->slots[i];
        if (sl.graph) cudaGraphExecDestroy(sl.graph);
        if (sl.d_frames) cudaFree(sl.d_frames);
        if (sl.pin_frames) cudaFreeHost(sl.pin_frames);
        if (sl.pin_humans) cudaFreeHost(sl.pin_humans);
        if (sl.pin_counts) cudaFreeHost(sl.pin_counts);
        if (sl.h2d_done) cudaEventDestroy(sl.h2d_done);
        if (sl.done) cudaEventDestroy(sl.done);
        if (sl.conv_done) cudaEventDestroy(sl.conv_done);
    }
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

} // namespace

extern "C" {

int hp_engine_create(hp_engine** out, const void* pack, size_t pack_bytes, int in_w, int in_h, int max_batch,
                     double factor, int flip_rgb, int device)
{
    return hp_engine_create_ex(out, pack, pack_bytes, in_w, in_h, max_batch, factor, flip_rgb, device, HP_DTYPE_F16);
}

int hp_engine_dtype(const hp_engine* e) { return e ? e->dtype : HP_ERR_ARG; }

int hp_engine_create_ex(hp_engine** out, const void* pack, size_t pack_bytes, int in_w, int in_h, int max_batch,
                        double factor, int flip_rgb, int device, int dtype)
{
    if (dtype != HP_DTYPE_F16 && dtype != HP_DTYPE_TF32 && dtype != HP_DTYPE_INT8) { set_error("hp_engine_create_ex: unknown dtype %d", dtype); return HP_ERR_ARG; }

    if (!out || !pack) { set_error("hp_engine_create: null argument"); return HP_ERR_ARG; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error("hp_engine_create: no CUDA device (this library has no CPU fallback)");
        return HP_ERR_CUDA;
    }
    if (device < 0 || device >= ndev || in_w <= 0 || in_h <= 0 || max_batch <= 0) { set_error("hp_engine_create: bad device/size/batch"); return HP_ERR_ARG; }
    if (pack_bytes < sizeof(PackHeader)) { set_error("hp_engine_create: pack too small"); return HP_ERR_ARG; }
    PackHeader hdr;
    memcpy(&hdr, pack, sizeof(hdr));
    if (memcmp(hdr.magic, PACK_MAGIC, 8) != 0 || hdr.version != PACK_VERSION) { set_error("hp_engine_create: not an HPB2PACK v%u model pack", PACK_VERSION); return HP_ERR_ARG; }
    // the file is untrusted: bound the counts before any size arithmetic (no overflow), then check every blob range an op names
    if (hdr.n_buffers == 0 || hdr.n_buffers > 65536 || hdr.n_ops == 0 || hdr.n_ops > 65536 || hdr.blob_floats > ((uint64_t)1 << 34)) {
        set_error("hp_engine_create: implausible pack header (%u buffers, %u ops, %llu blob floats)", hdr.n_buffers, hdr.n_ops, (unsigned long long)hdr.blob_floats);
        return HP_ERR_ARG;
    }
    const uint32_t n_scales = hdr.reserved[0];   // INT8 calibration table: 0 or n_buffers scales after the blob
    if (n_scales != 0 && n_scales != hdr.n_buffers) { set_error("hp_engine_create: the pack's scale table has %u entries for %u buffers", n_scales, hdr.n_buffers); return HP_ERR_ARG; }
    const size_t need = sizeof(PackHeader) + (size_t)hdr.n_buffers * sizeof(PackBuffer) + (size_t)hdr.n_ops * sizeof(PackOp) + (size_t)hdr.blob_floats * sizeof(float) +
                        (size_t)n_scales * sizeof(float);
    if (pack_bytes < need) { set_error("hp_engine_create: truncated pack (%zu < %zu bytes)", pack_bytes, need); return HP_ERR_ARG; }
    std::vector<float> act_scale;
    if (dtype == HP_DTYPE_INT8) {
        if (hdr.head_type != 0) { set_error("hp_engine_create: the INT8 engine has no OpenPifPaf or PPN heads (pack head_type %u)", hdr.head_type); return HP_ERR_ARG; }
        if (n_scales == 0) { set_error("hp_engine_create: the pack has no INT8 scale table (export it with an INT8 calibration)"); return HP_ERR_ARG; }
        act_scale.resize(n_scales);
        memcpy(act_scale.data(), (const uint8_t*)pack + need - (size_t)n_scales * sizeof(float), (size_t)n_scales * sizeof(float));
        for (uint32_t b = 0; b < n_scales; ++b)
            if (!(std::isfinite(act_scale[b]) && act_scale[b] > 0.f)) { set_error("hp_engine_create: INT8 scale of buffer %u is %g (needs a finite value > 0)", b, (double)act_scale[b]); return HP_ERR_ARG; }
        const PackOp* vops = (const PackOp*)((const uint8_t*)pack + sizeof(PackHeader) + (size_t)hdr.n_buffers * sizeof(PackBuffer));
        for (uint32_t i = 0; i < hdr.n_ops; ++i) {
            PackOp po;
            memcpy(&po, vops + i, sizeof(po));
            if (po.type == OP_MAXPOOL2 && po.in_buf < n_scales && po.out_buf < n_scales && act_scale[po.in_buf] != act_scale[po.out_buf]) {
                set_error("hp_engine_create: INT8 max-pool op %u reads buffer %u (scale %g) but writes buffer %u (scale %g); they must be equal", i, po.in_buf,
                          (double)act_scale[po.in_buf], po.out_buf, (double)act_scale[po.out_buf]);
                return HP_ERR_ARG;
            }
        }
    }
    {
        const PackOp* vops = (const PackOp*)((const uint8_t*)pack + sizeof(PackHeader) + (size_t)hdr.n_buffers * sizeof(PackBuffer));
        auto in_blob = [&](uint64_t off, uint64_t count) { return off <= hdr.blob_floats && count <= hdr.blob_floats - off; };
        for (uint32_t i = 0; i < hdr.n_ops; ++i) {
            PackOp po;
            memcpy(&po, vops + i, sizeof(po));
            if (po.type != OP_CONV && po.type != OP_DWCONV) continue;
            const uint64_t lim = 1u << 16;   // per-dimension bound: keeps the products below 2^64
            const bool dw = po.type == OP_DWCONV;
            const uint64_t G = dw ? 1 : po.groups, co = po.cout_g, ci = dw ? 1 : po.cin_g, R = po.R, S = po.S;
            if (G == 0 || co == 0 || ci == 0 || R == 0 || S == 0 || G > lim || co > lim || ci > lim || R > 15 || S > 15 ||
                !in_blob(po.w_off, G * co * ci * R * S) || !in_blob(po.b_off, G * co) || !in_blob(po.a_off, G * co)) {
                set_error("hp_engine_create: op %u names weights outside the pack (groups %u, cout %u, cin %u, %ux%u)", i, po.groups, po.cout_g, po.cin_g, po.R, po.S);
                return HP_ERR_ARG;
            }
        }
    }
    HP_CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    HP_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) { set_error("hp_engine_create: device is sm_%d%d; this engine is wgmma/TMA code for sm_90a only", prop.major, prop.minor); return HP_ERR_UNSUPPORTED; }

    hp_engine* e = new hp_engine();
    e->device = device; e->dtype = dtype; e->in_h = in_h; e->in_w = in_w; e->max_batch = max_batch;
    e->factor = factor; e->flip_rgb = flip_rgb; e->hdr = hdr; e->num_sms = prop.multiProcessorCount;
    e->act_scale = std::move(act_scale);
    EngOptions& opt = e->opt;
    if (const char* v = getenv("HPB_HALO")) opt.halo = strcmp(v, "all") == 0 ? EngOptions::HALO_ALL : EngOptions::HALO_NONE;
    opt.halo_wide = !getenv("HPB_HALO_NARROW");
    opt.stem3 = !getenv("HPB_NO_STEM3");
    opt.pool_fuse = !getenv("HPB_NO_POOL_FUSE");
    opt.dw1_fuse = !getenv("HPB_NO_DW1_FUSE");
    opt.dw_pair = !getenv("HPB_NO_DW_DUAL");
    opt.dw_tma = !getenv("HPB_NO_DW_TMA");
    const char* rs = getenv("HPB_PIFPAF_RESERVE_SMS");
    opt.pifpaf_reserve_sms = std::max(0, std::min(rs ? atoi(rs) : std::min(max_batch, 16), e->num_sms / 2));
    const uint8_t* ptr = (const uint8_t*)pack + sizeof(PackHeader);
    const PackBuffer* pb = (const PackBuffer*)ptr;
    const PackOp* pops = (const PackOp*)(ptr + hdr.n_buffers * sizeof(PackBuffer));
    std::vector<float> blob(hdr.blob_floats);
    memcpy(blob.data(), (const uint8_t*)pops + hdr.n_ops * sizeof(PackOp), hdr.blob_floats * sizeof(float));

    int rc = HP_OK;
    auto fail = [&](int code) { free_engine(e); return code; };
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate failed"); return fail(HP_ERR_CUDA); }
    e->bufs.resize(hdr.n_buffers);
    for (uint32_t i = 0; i < hdr.n_buffers; ++i) {
        EngBuffer& b = e->bufs[i];
        b.channels = (int)pb[i].channels; b.down = (int)pb[i].down_shift;
        b.H = in_h; b.W = in_w;
        for (int d = 0; d < b.down; ++d) { b.H = (b.H + 1) / 2; b.W = (b.W + 1) / 2; }
        if (b.channels % 8) { set_error("engine: buffer %u has %d channels (need a multiple of 8)", i, b.channels); return fail(HP_ERR_ARG); }
        const size_t bytes = (size_t)max_batch * b.H * b.W * b.channels * (size_t)elem_bytes(dtype);
        if (cudaMalloc(&b.d, bytes) != cudaSuccess) { set_error("engine: cudaMalloc(%zu) failed", bytes); return fail(HP_ERR_CUDA); }
        cudaMemset(b.d, 0, bytes); // padding channels must read as zero
    }
    e->out_h = in_h; e->out_w = in_w;
    for (uint32_t d = 0; d < hdr.out_down_shift; ++d) { e->out_h = (e->out_h + 1) / 2; e->out_w = (e->out_w + 1) / 2; }
    if (hdr.head_type == 1) { e->out_h = 2 * e->out_h - 1; e->out_w = 2 * e->out_w - 1; } // pixel-shuffled and cropped
    if (cudaMalloc(&e->d_conf, (size_t)max_batch * hdr.conf_channels * e->out_h * e->out_w * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&e->d_paf, (size_t)max_batch * hdr.paf_channels * e->out_h * e->out_w * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&e->d_frames, (size_t)max_batch * in_h * in_w * 3 + 16) != cudaSuccess || // + slack: the 3x3 stem reads whole 32-bit words
        cudaMallocHost(&e->pin_frames, (size_t)max_batch * in_h * in_w * 3) != cudaSuccess) {
        set_error("engine: output/frame allocation failed");
        return fail(HP_ERR_CUDA);
    }
    e->ops.resize(hdr.n_ops);
    size_t max_smem = 0;
    const bool tf32 = dtype == HP_DTYPE_TF32, i8 = dtype == HP_DTYPE_INT8;
    for (uint32_t i = 0; i < hdr.n_ops; ++i) {
        EngOp& op = e->ops[i];
        op.po = pops[i];
        const PackOp& po = op.po;
        if ((po.type != OP_IM2COL3 && po.in_buf >= hdr.n_buffers) ||
            (po.out_mode != OUT_F32_NCHW_SPLIT && po.type != OP_PIFPAF_HEAD && po.type != OP_PPN_HEAD && po.out_buf >= hdr.n_buffers)) {
            set_error("engine: op %u references a missing buffer", i);
            return fail(HP_ERR_ARG);
        }
        if (po.type == OP_CONV) {
            rc = build_conv_plan(e, op, blob.data());
            if (rc) return fail(rc);
            max_smem = std::max(max_smem, op.plan.smem);
            e->flops_per_frame += op.plan.flops_per_frame;
        } else if (po.type == OP_IM2COL3) {
            const int stride = po.stride ? (int)po.stride : 1;
            const int R = po.R ? (int)po.R : 3;
            if (e->bufs[po.out_buf].channels != round_up(R * R * 3, 64) || e->bufs[po.out_buf].down != (stride == 2 ? 1 : 0) || stride > 2 || (R != 3 && R != 7)) {
                set_error("engine: im2col buffer must hold roundup(R*R*3,64) channels at the stem resolution");
                return fail(HP_ERR_ARG);
            }
            op.launch = tf32 ? Launch::Im2colF32 : i8 ? Launch::Im2colI8 : Launch::Im2col;
        } else if (po.type == OP_DWCONV) {
            const int C = (int)po.cout_g, K = (int)po.R, stride = po.stride ? (int)po.stride : 1;
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            if (C % 8 || (K != 1 && K != 3) || po.S != po.R || stride < 1 || stride > 2 || ob.down != ib.down + (stride == 2 ? 1 : 0) ||
                (int)po.in_ch_off + C > ib.channels || (int)po.out_ch_off + C > ob.channels || po.in_ch_off % 8 || po.out_ch_off % 8) {
                set_error("engine: bad depthwise op %u", i);
                return fail(HP_ERR_ARG);
            }
            // blob W[C][K][K] -> device [K*K][C] (tap-major so that 8 consecutive channels are one 32-byte load)
            std::vector<float> w((size_t)K * K * C + 2 * (size_t)C);
            for (int c = 0; c < C; ++c) {
                for (int t = 0; t < K * K; ++t) w[(size_t)t * C + c] = blob[po.w_off + (size_t)c * K * K + t];
                w[(size_t)K * K * C + c] = blob[po.b_off + c];
                w[(size_t)K * K * C + C + c] = blob[po.a_off + c];
            }
            if (cudaMalloc(&op.d_dw, w.size() * sizeof(float)) != cudaSuccess ||
                cudaMemcpy(op.d_dw, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
                set_error("engine: depthwise weight upload failed");
                return fail(HP_ERR_CUDA);
            }
            e->flops_per_frame += 2.0 * ob.H * ob.W * C * K * K;
            op.launch = tf32 ? Launch::DwF32 : i8 ? Launch::DwI8 : K == 3 && stride == 1 ? Launch::DwCol : Launch::DwStrip;
        } else if (po.type == OP_MAXPOOL2) {
            // 8 channels per 16-byte load (fp16) / two float4 loads (fp32): both offsets aligned, both channel ranges inside their buffers
            const EngBuffer& ib = e->bufs[po.in_buf];
            const EngBuffer& ob = e->bufs[po.out_buf];
            if (po.cout_g % 8 || ob.down != ib.down + 1 || (po.R != 0 && po.R != 2 && po.R != 3) || po.in_ch_off % 8 || po.out_ch_off % 8 ||
                (uint64_t)po.in_ch_off + po.cout_g > (uint64_t)ib.channels || (uint64_t)po.out_ch_off + po.cout_g > (uint64_t)ob.channels) {
                set_error("engine: bad maxpool op %u", i);
                return fail(HP_ERR_ARG);
            }
            op.launch = tf32 ? Launch::MaxPoolF32 : i8 ? Launch::MaxPoolI8 : Launch::MaxPool;
        } else if (po.type == OP_PIFPAF_HEAD) {
            // the head kernels read input row y >> 1 for every output row y < out_h: both inputs must be at the output resolution
            if (hdr.head_type != 1 || po.res_buf >= hdr.n_buffers || hdr.conf_channels != 85 || hdr.paf_channels != 171 ||
                e->bufs[po.in_buf].channels < 340 || e->bufs[po.res_buf].channels < 684 ||
                e->bufs[po.in_buf].down != (int)hdr.out_down_shift || e->bufs[po.res_buf].down != (int)hdr.out_down_shift) {
                set_error("engine: bad pifpaf head op %u", i);
                return fail(HP_ERR_ARG);
            }
            op.launch = tf32 ? Launch::HeadsF32 : Launch::Heads;
        } else if (po.type == OP_PPN_HEAD) {
            // one thread per output element reads raw channel c < 6K + L*nh*nw of the pixel it writes: the input must hold them all at
            // the output resolution; the parser indexes key points 0..17 (COCO limb table)
            const uint64_t K = po.cout_g, n_edge = (uint64_t)po.groups * po.R * po.S;
            const EngBuffer& ib = e->bufs[po.in_buf];
            if (hdr.head_type != 2) { set_error("engine: PPN head op %u in a pack with head_type %u (needs 2)", i, hdr.head_type); return fail(HP_ERR_ARG); }
            if (ib.down != (int)hdr.out_down_shift) {
                set_error("engine: PPN head op %u reads buffer %u at down-shift %d but the outputs are at %u", i, po.in_buf, ib.down, hdr.out_down_shift);
                return fail(HP_ERR_ARG);
            }
            if (K < 18 || K > 4096 || n_edge == 0 || n_edge > (1u << 20)) {
                set_error("engine: PPN head op %u has K=%llu key points and %llu edge channels (needs K >= 18 for the COCO limb table)", i,
                          (unsigned long long)K, (unsigned long long)n_edge);
                return fail(HP_ERR_ARG);
            }
            if ((uint64_t)ib.channels < 6 * K + n_edge) {
                set_error("engine: PPN head op %u reads %llu channels of a %d-channel buffer", i, (unsigned long long)(6 * K + n_edge), ib.channels);
                return fail(HP_ERR_ARG);
            }
            if (hdr.conf_channels != 6 * K || hdr.paf_channels != n_edge) {
                set_error("engine: PPN head op %u writes %llu box and %llu edge channels but the pack header says conf %u / paf %u", i,
                          (unsigned long long)(6 * K), (unsigned long long)n_edge, hdr.conf_channels, hdr.paf_channels);
                return fail(HP_ERR_ARG);
            }
            op.launch = tf32 ? Launch::PpnHeadF32 : Launch::PpnHead;
        } else {
            set_error("engine: unknown op type %u", po.type);
            return fail(HP_ERR_UNSUPPORTED);
        }
    }
    // The fusion passes below (fp16 engines; the TF32 and INT8 engines launch every op on its own) settle how each op launches.
    // Fused stem: the first conv gathers its patches from the u8 frames itself, the im2col buffer is never written.
    for (EngOp& c : e->ops) {
        const PackOp& po = c.po;
        const int R = (int)po.R;
        if (dtype != HP_DTYPE_F16 || c.launch != Launch::Conv || !po.im2col_input || po.res_mode || po.out_mode != OUT_F16_NHWC || po.S != po.R || !(R == 7 || (R == 3 && opt.stem3))) continue;
        for (EngOp& m : e->ops) {   // the patch-gather op feeding this conv: its stride / tap size define the stem geometry
            if (m.po.type != OP_IM2COL3 || m.po.out_buf != po.in_buf) continue;
            if ((int)(m.po.R ? m.po.R : 3) != R || po.cin_g != 3) break;
            ConvParams& p = c.plan.prm;
            const int stride = m.po.stride ? (int)m.po.stride : 1;
            p.in_h = in_h; p.in_w = in_w; p.stem_stride = stride;
            p.stem_pad_h = same_pad_before(in_h, R, stride); p.stem_pad_w = same_pad_before(in_w, R, stride);
            p.factor = factor; p.flip = flip_rgb;
            p.mean[0] = hdr.mean[0]; p.mean[1] = hdr.mean[1]; p.mean[2] = hdr.mean[2];
            c.launch = Launch::ConvStem;
            m.launch = Launch::StemOrIm2col;
            break;
        }
    }
    // conv (halo kernel) -> 2x2 max-pool: the pool moves into the conv's epilogue when nobody else reads the un-pooled tensor
    for (size_t i = 0; opt.pool_fuse && i + 1 < e->ops.size(); ++i) {
        EngOp& c = e->ops[i]; EngOp& m = e->ops[i + 1];
        if ((c.launch != Launch::Halo && c.launch != Launch::HaloWide && c.launch != Launch::HaloPP) || !c.plan.monotone_act || m.po.type != OP_MAXPOOL2 || (m.po.R != 0 && m.po.R != 2)) continue;
        const EngBuffer& cb = e->bufs[c.po.out_buf];
        const EngBuffer& pb = e->bufs[m.po.out_buf];
        const int C = (int)c.po.groups * (int)c.po.cout_g;
        if (m.po.in_buf != c.po.out_buf || m.po.in_ch_off != c.po.out_ch_off || (int)m.po.cout_g != C || c.plan.hp.cout_g_pad != c.plan.hp.cout_g ||
            (cb.H & 1) || (cb.W & 1) || pb.H != cb.H / 2 || pb.W != cb.W / 2 || (int)m.po.out_ch_off + C > pb.channels) continue;
        bool other_reader = false;
        for (size_t k = 0; k < e->ops.size(); ++k)
            if (k != i + 1 && reads_buffer(e->ops[k].po, c.po.out_buf)) other_reader = true;
        if (other_reader) continue;
        c.plan.hp.out = pb.d; c.plan.hp.out_ld = pb.channels; c.plan.hp.out_ch_off = (int)m.po.out_ch_off;
        // the item is picked again for the pooled epilogue: it has no wide form, and pooled layers take the ping-pong item at any depth
        set_halo_item(c, pick_halo_item(e, c, true), true);
        max_smem = std::max(max_smem, c.plan.smem);
        m.launch = Launch::None;
        e->bufs[c.po.out_buf].fused_away = true;
    }
    // conv -> 1x1 "depthwise" (per-channel affine + PReLU; the filter_size (1,1) separable blocks, mbv2_th_openpose.py:121,127,144,151):
    // applied in the epilogue of conv_wgmma_kernel when the tensor in between has no other reader before it is overwritten
    for (size_t i = 0; opt.dw1_fuse && i + 1 < e->ops.size(); ++i) {
        EngOp& c = e->ops[i]; EngOp& d = e->ops[i + 1];
        if ((c.launch != Launch::Conv && c.launch != Launch::ConvStem) || d.launch != Launch::DwStrip || d.po.R != 1 || (d.po.stride ? d.po.stride : 1) != 1) continue;
        const ConvParams& cp = c.plan.prm;
        const int Ctot = (int)c.po.groups * (int)c.po.cout_g;
        if (c.po.out_mode != OUT_F16_NHWC || cp.cout_g_pad != cp.cout_g || cp.cout_g % 16 ||
            d.po.in_buf != c.po.out_buf || d.po.in_ch_off != c.po.out_ch_off || (int)d.po.cout_g != Ctot || d.po.out_buf == c.po.out_buf) continue;
        if (d.po.out_buf == c.po.in_buf) {
            // the fused conv would write the tensor it reads.  That is safe only when every tile reads exactly the (pixels, channels) it
            // writes and has consumed them before its epilogue: a 1x1 conv whose group g maps channels [off + g*c, off + (g+1)*c) onto
            // themselves with ONE n-tile per group (MobilenetThin's grouped 128 -> 128 pointwise convs on the ping-pong buffers)
            if (cp.R != 1 || cp.S != 1 || cp.cin_g != cp.cout_g || cp.BN != cp.cout_g || (int)d.po.out_ch_off != cp.in_ch_off) continue;
        }
        if (c.po.res_mode && d.po.out_buf == c.po.res_buf) continue;
        // the tensor between the two must be dead afterwards: no reader before the next writer of the same channels
        bool safe = true, rewritten = false;
        for (size_t k = i + 2; k < e->ops.size() && safe && !rewritten; ++k) {
            const PackOp& q = e->ops[k].po;
            if (reads_buffer(q, c.po.out_buf)) safe = false;
            else if (q.type != OP_IM2COL3 && q.type != OP_PIFPAF_HEAD && q.type != OP_PPN_HEAD && q.out_mode != OUT_F32_NCHW_SPLIT && q.out_buf == c.po.out_buf) {
                const int qc = q.type == OP_CONV ? (int)q.groups * (int)q.cout_g : (int)q.cout_g;
                if (q.out_ch_off <= c.po.out_ch_off && (int)q.out_ch_off + qc >= (int)c.po.out_ch_off + Ctot) rewritten = true; else safe = false;
            }
        }
        if (!safe) continue;
        const EngBuffer& ob = e->bufs[d.po.out_buf];
        if ((int)d.po.out_ch_off + Ctot > ob.channels) continue;
        c.plan.prm.out = ob.d; c.plan.prm.out_ld = ob.channels; c.plan.prm.out_ch_off = (int)d.po.out_ch_off;
        c.plan.prm.post_w = d.d_dw; c.plan.prm.post_b = d.d_dw + Ctot; c.plan.prm.post_a = d.d_dw + 2 * (size_t)Ctot;
        d.launch = Launch::None;
        if (!rewritten) e->bufs[c.po.out_buf].fused_away = true;   // its final content would have been this conv's output
    }
    // depthwise 3x3 / stride 1 on a multiple of 64 channels: input tiles through TMA (dwconv3_tma_kernel)
    size_t dwt_max = 0;
    for (EngOp& a : e->ops) {
        const PackOp& po = a.po;
        if (!opt.dw_tma || a.launch != Launch::DwCol || po.cout_g % 64 || po.in_buf == po.out_buf) continue;
        const EngBuffer& ib = e->bufs[po.in_buf];
        const int C = (int)po.cout_g;
        const int nx = (ib.W + 61) / 62, wbo = (ib.W + nx - 1) / nx, bw = wbo + 2;
        // tile height: the tallest of 8 / 6 / 4 / 3 / 2 rows that fits a buffer and still gives every SM two tiles at the full batch
        int hb = 2;
        for (int cand : { 8, 6, 4, 3, 2 }) {
            if (cand > std::max(2, ib.H) || (size_t)(cand + 2) * bw * 128 > (size_t)DWT_STAGE_MAX) continue;
            const size_t items = (size_t)e->max_batch * ((ib.H + cand - 1) / cand) * nx * (C / 64);
            hb = cand;
            if (items >= 2 * (size_t)e->num_sms) break;
        }
        const size_t stage = (size_t)(hb + 2) * bw * 128;
        if (stage > (size_t)DWT_STAGE_MAX) continue;
        a.dwt_stages = (int)std::min<size_t>(4, (200 * 1024) / stage);
        if (a.dwt_stages < 2) continue;
        a.dwt_wbo = wbo; a.dwt_hb = hb; a.dwt_tiles_x = nx; a.dwt_tiles_y = (ib.H + hb - 1) / hb;
        a.dwt_smem = a.dwt_stages * stage + 128 + 64;
        if (make_tmap_act_box(&a.tmap_dw, ib.d + po.in_ch_off, e->max_batch, ib.H, ib.W, C, ib.channels, bw, hb + 2, CU_TENSOR_MAP_SWIZZLE_NONE) != HP_OK) return fail(HP_ERR_CUDA);
        a.launch = Launch::DwTma;
        dwt_max = std::max(dwt_max, a.dwt_smem);
    }
    if (dwt_max > 0 && (cudaFuncSetAttribute(dwconv3_tma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dwt_max) != cudaSuccess ||
                        cudaFuncSetAttribute(dwconv3_tma_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dwt_max) != cudaSuccess)) {
        set_error("engine: cannot opt in to %zu bytes of dynamic shared memory (depthwise)", dwt_max);
        return fail(HP_ERR_CUDA);
    }
    // two TMA depthwise convs of the same input (the conf / paf branch of a MobilenetThin stage): one launch with both filter sets
    for (size_t i = 0; opt.dw_pair && i + 1 < e->ops.size(); ++i) {
        EngOp& a = e->ops[i]; EngOp& b = e->ops[i + 1];
        if (a.launch != Launch::DwTma || b.launch != Launch::DwTma || a.po.in_buf != b.po.in_buf || a.po.in_ch_off != b.po.in_ch_off ||
            a.po.cout_g != b.po.cout_g || a.po.out_buf != b.po.out_buf) continue;
        a.launch = Launch::DwTmaPair;
        b.launch = Launch::None;
    }
    // programmatic dependent launch pays where the step is a chain of short kernels (MobilenetThin: 73 launches of ~2 GFLOP at batch 8)
    // and costs where they are long (VGG19: 140 GFLOP per launch); see launch_pdl
    int launches = 0;
    for (const EngOp& o : e->ops) {
        if ((o.po.type == OP_CONV || o.po.type == OP_DWCONV || o.po.type == OP_MAXPOOL2) && o.launch != Launch::None) ++launches;
        e->step_kernels += kernels_launched(o.launch, true);
    }
    const double per_launch = launches ? e->flops_per_frame * e->max_batch / launches : 0.0;
    e->use_pdl = dtype == HP_DTYPE_F16 && launches > 0 && per_launch < 10e9;
    for (const EngOp& o : e->ops) {
        if (o.po.type != OP_CONV) continue;
        if (is_halo(o.launch) &&
            cudaFuncSetAttribute(halo_kernel(o.launch, o.plan.prm.BN), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem) != cudaSuccess) {
            set_error("engine: cannot opt in to %zu bytes of dynamic shared memory (halo)", max_smem);
            return fail(HP_ERR_CUDA);
        }
        const int stem_R = o.launch == Launch::ConvStem ? (int)o.po.R : 0;
        for (int v = 0; v < 3; ++v)   // plain, residual, and (for a stem) the fused u8 form
            if ((v < 2 || stem_R) &&
                cudaFuncSetAttribute(conv_kernel(dtype, v == 1, o.plan.prm.BN, v == 2 ? stem_R : 0), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem) != cudaSuccess) {
                set_error("engine: cannot opt in to %zu bytes of dynamic shared memory", max_smem);
                return fail(HP_ERR_CUDA);
            }
    }
    if (cudaDeviceSynchronize() != cudaSuccess) { set_error("hp_engine_create: device error during set-up: %s", cudaGetErrorString(cudaGetLastError())); return fail(HP_ERR_CUDA); }
    *out = e;
    return HP_OK;
}

void hp_engine_destroy(hp_engine* e) { free_engine(e); }

int hp_engine_info(const hp_engine* e, int* in_w, int* in_h, int* max_batch, int* c_conf, int* c_paf, int* out_h, int* out_w, double* flops_per_frame)
{
    if (!e) return HP_ERR_ARG;
    if (in_w) *in_w = e->in_w;
    if (in_h) *in_h = e->in_h;
    if (max_batch) *max_batch = e->max_batch;
    if (c_conf) *c_conf = (int)e->hdr.conf_channels;
    if (c_paf) *c_paf = (int)e->hdr.paf_channels;
    if (out_h) *out_h = e->out_h;
    if (out_w) *out_w = e->out_w;
    if (flops_per_frame) *flops_per_frame = e->flops_per_frame;
    return HP_OK;
}

// 0: conf[c_conf,h,w] / paf[c_paf,h,w] for hyperpose::parser::paf; 1: OpenPifPaf fields pif[17,5,h,w] / paf[19,9,h,w]
// 2: Pose Proposal Network boxes [6,K,h,w] / edges [L,nh,nw,h,w] for hyperpose::parser::pose_proposal
int hp_engine_head_type(const hp_engine* e) { return e ? (int)e->hdr.head_type : HP_ERR_ARG; }

// frames: HOST u8 [N, in_h, in_w, 3] (already network-sized, BGR like cv::Mat).  Asynchronous on the engine stream.
int hp_engine_infer_u8_host(hp_engine* e, const uint8_t* frames, int N)
{
    if (!e || !frames) { set_error("hp_engine_infer_u8_host: null argument"); return HP_ERR_ARG; }
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const size_t bytes = (size_t)N * e->in_h * e->in_w * 3;
    cudaPointerAttributes attr;
    const bool pinned = (cudaPointerGetAttributes(&attr, frames) == cudaSuccess && attr.type == cudaMemoryTypeHost);
    if (!pinned) cudaGetLastError();
    if (pinned) { // page-locked caller memory: DMA straight from it
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_frames, frames, bytes, cudaMemcpyHostToDevice, e->stream));
    } else {
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream)); // pin_frames may still feed the previous batch
        memcpy(e->pin_frames, frames, bytes);
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_frames, e->pin_frames, bytes, cudaMemcpyHostToDevice, e->stream));
    }
    return run_graph(e, N, true, e->stream);
}

// frames: DEVICE u8 [N, in_h, in_w, 3]; stream: cudaStream_t or NULL for the engine's own stream.
int hp_engine_infer_u8_device(hp_engine* e, const uint8_t* d_frames, int N, void* stream)
{
    if (!e || !d_frames) { set_error("hp_engine_infer_u8_device: null argument"); return HP_ERR_ARG; }
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : e->stream;
    HP_CUDA_TRY(cudaMemcpyAsync(e->d_frames, d_frames, (size_t)N * e->in_h * e->in_w * 3, cudaMemcpyDeviceToDevice, st));
    return run_graph(e, N, true, st);
}

// tensorrt::inference(const std::vector<float>&, size_t) (src/tensorrt.cpp:364): HOST f32 NCHW, already scaled.
int hp_engine_infer_f32_host(hp_engine* e, const float* nchw, int N)
{
    if (!e || !nchw) { set_error("hp_engine_infer_f32_host: null argument"); return HP_ERR_ARG; }
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const size_t n = (size_t)e->max_batch * 3 * e->in_h * e->in_w;
    if (!e->d_input_f32) HP_CUDA_TRY(cudaMalloc(&e->d_input_f32, n * sizeof(float)));
    HP_CUDA_TRY(cudaMemcpyAsync(e->d_input_f32, nchw, (size_t)N * 3 * e->in_h * e->in_w * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    return run_graph(e, N, false, e->stream);
}

// Stages ONE host frame of arbitrary size into batch slot `slot`: H2D of the original pixels, then the reference's
// resize step on the GPU -- cv::resize(INTER_LINEAR) or, with keep_ratio, non_scaling_resize (src/tensorrt.cpp:446-451).
int hp_engine_stage_frame_u8(hp_engine* e, int slot, const uint8_t* frame, int src_h, int src_w, int keep_ratio)
{
    if (!e || !frame || slot < 0 || slot >= e->max_batch || src_h <= 0 || src_w <= 0) { set_error("hp_engine_stage_frame_u8: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const size_t bytes = (size_t)src_h * src_w * 3;
    uint8_t* dst = e->d_frames + (size_t)slot * e->in_h * e->in_w * 3;
    // Staging memory is one region per batch slot, so the frames of a batch never wait for each other: the stream is
    // synchronised ONCE per batch (first stage call after a run), not once per frame.
    if (!e->stage_synced) { HP_CUDA_TRY(cudaStreamSynchronize(e->stream)); e->stage_synced = true; }
    const size_t slot_bytes = (bytes + 255) & ~(size_t)255;
    if (e->pin_src_bytes < slot_bytes * e->max_batch) {
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
        if (e->pin_src) cudaFreeHost(e->pin_src);
        e->pin_src = nullptr; e->pin_src_bytes = 0;
        HP_CUDA_TRY(cudaMallocHost(&e->pin_src, slot_bytes * e->max_batch));
        e->pin_src_bytes = slot_bytes * e->max_batch;
    }
    uint8_t* pin = e->pin_src + (e->pin_src_bytes / e->max_batch / 256 * 256) * slot;
    if (src_h == e->in_h && src_w == e->in_w) { // already network-sized: both resize variants are the identity
        memcpy(pin, frame, bytes);
        HP_CUDA_TRY(cudaMemcpyAsync(dst, pin, bytes, cudaMemcpyHostToDevice, e->stream));
        return HP_OK;
    }
    if (src_h != e->rz_sh || src_w != e->rz_sw || keep_ratio != e->rz_keep) {
        int rh = e->in_h, rw = e->in_w;
        if (keep_ratio) { // non_scaling_resize (src/data.cpp:53-69)
            const double h1 = e->in_w * (src_h / (double)src_w);
            const double w2 = e->in_h * (src_w / (double)src_h);
            if (h1 <= e->in_h) { rw = e->in_w; rh = (int)h1; } else { rw = (int)w2; rh = e->in_h; }
            if (rh <= 0 || rw <= 0) { set_error("hp_engine_stage_frame_u8: degenerate letterbox"); return HP_ERR_ARG; }
        }
        auto table = [](int src, int dst, bool clamp, std::vector<int>& idx, std::vector<short>& coef) {
            idx.resize(dst); coef.resize(2 * (size_t)dst);
            const double inv = (double)dst / (double)src, scale = 1.0 / inv;
            for (int d = 0; d < dst; ++d) {
                float f = (float)((d + 0.5) * scale - 0.5);
                int s = (int)floorf(f);
                f -= (float)s;
                if (clamp) {
                    if (s < 0) { f = 0.f; s = 0; }
                    if (s >= src - 1) { f = 0.f; s = src - 1; }
                }
                idx[d] = s;
                coef[2 * d] = (short)lrintf((1.f - f) * 2048.f);   // saturate_cast<short>(float): round half to even
                coef[2 * d + 1] = (short)lrintf(f * 2048.f);
            }
        };
        std::vector<int> xi, yi; std::vector<short> xa, ya;
        table(src_w, rw, true, xi, xa);
        table(src_h, rh, false, yi, ya);
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));   // earlier frames of this batch may still read the old tables
        if (!e->d_rz_xi) {
            HP_CUDA_TRY(cudaMalloc(&e->d_rz_xi, e->in_w * sizeof(int)));
            HP_CUDA_TRY(cudaMalloc(&e->d_rz_xa, e->in_w * 2 * sizeof(short)));
            HP_CUDA_TRY(cudaMalloc(&e->d_rz_yi, e->in_h * sizeof(int)));
            HP_CUDA_TRY(cudaMalloc(&e->d_rz_ya, e->in_h * 2 * sizeof(short)));
        }
        // on the engine's (non-blocking) stream, so that the resize kernels are ordered behind the upload; the vectors are locals
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_rz_xi, xi.data(), rw * sizeof(int), cudaMemcpyHostToDevice, e->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_rz_xa, xa.data(), rw * 2 * sizeof(short), cudaMemcpyHostToDevice, e->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_rz_yi, yi.data(), rh * sizeof(int), cudaMemcpyHostToDevice, e->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(e->d_rz_ya, ya.data(), rh * 2 * sizeof(short), cudaMemcpyHostToDevice, e->stream));
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
        e->rz_sh = src_h; e->rz_sw = src_w; e->rz_keep = keep_ratio; e->rz_rh = rh; e->rz_rw = rw;
        e->rz_area = (src_h == 2 * rh && src_w == 2 * rw) ? 1 : 0;
    }
    if (e->d_src_bytes < slot_bytes * e->max_batch) {
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
        if (e->d_src) cudaFree(e->d_src);
        e->d_src = nullptr; e->d_src_bytes = 0;
        HP_CUDA_TRY(cudaMalloc(&e->d_src, slot_bytes * e->max_batch));
        e->d_src_bytes = slot_bytes * e->max_batch;
    }
    uint8_t* dsrc = e->d_src + (e->d_src_bytes / e->max_batch / 256 * 256) * slot;
    memcpy(pin, frame, bytes);
    HP_CUDA_TRY(cudaMemcpyAsync(dsrc, pin, bytes, cudaMemcpyHostToDevice, e->stream));
    const int total = e->in_h * e->in_w;
    resize_u8c3_kernel<<<(total + 255) / 256, 256, 0, e->stream>>>(dsrc, src_h, src_w, dst, e->in_h, e->in_w, e->rz_rh, e->rz_rw,
                                                                 e->d_rz_xi, e->d_rz_xa, e->d_rz_yi, e->d_rz_ya, e->rz_area);
    e->launches++;
    HP_CUDA_TRY(cudaGetLastError());
    return HP_OK;
}

// runs the network on the N frames staged by hp_engine_stage_frame_u8
int hp_engine_infer_staged(hp_engine* e, int N)
{
    if (!e) return HP_ERR_ARG;
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    e->stage_synced = false;   // the next batch's first stage call waits for this one's staging copies
    return run_graph(e, N, true, e->stream);
}

// test hook: the staged (resized) u8 frames back on the host
int hp_engine_debug_read_frames(hp_engine* e, uint8_t* out, int N)
{
    if (!e || !out || N <= 0 || N > e->max_batch) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(e->device));
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    HP_CUDA_TRY(cudaMemcpy(out, e->d_frames, (size_t)N * e->in_h * e->in_w * 3, cudaMemcpyDeviceToHost));
    return HP_OK;
}

int hp_engine_outputs(hp_engine* e, const float** d_conf, const float** d_paf, void** stream)
{
    if (!e) return HP_ERR_ARG;
    if (d_conf) *d_conf = e->d_conf;
    if (d_paf) *d_paf = e->d_paf;
    if (stream) *stream = (void*)e->stream;
    return HP_OK;
}

// D2H of the last batch's outputs: conf[N,c_conf,h,w], paf[N,c_paf,h,w] (what tensorrt::inference returns per image)
int hp_engine_read_outputs_host(hp_engine* e, float* conf, float* paf, int N)
{
    if (!e || N <= 0 || N > e->max_batch) { set_error("hp_engine_read_outputs_host: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const size_t plane = (size_t)e->out_h * e->out_w;
    if (conf) HP_CUDA_TRY(cudaMemcpyAsync(conf, e->d_conf, N * e->hdr.conf_channels * plane * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    if (paf) HP_CUDA_TRY(cudaMemcpyAsync(paf, e->d_paf, N * e->hdr.paf_channels * plane * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return HP_OK;
}

// tensorrt::inference's read-back loop (src/tensorrt.cpp:398-431): frame i of the last batch lands in the caller's
// conf_frames[i] / paf_frames[i] (the storage of the per-image feature_map_t objects).  With publish != 0 a device
// snapshot of the batch is kept and the host addresses are registered, so that hp_paf_process_host /
// hp_pifpaf_process_host called later with exactly these buffers parse from the device copy, the whole batch at once
// (handoff.h).  Results are identical with or without the publication.
int hp_engine_read_outputs_frames(hp_engine* e, float* const* conf_frames, float* const* paf_frames, int N, int publish)
{
    if (!e || !conf_frames || !paf_frames || N <= 0 || N > e->max_batch) { set_error("hp_engine_read_outputs_frames: bad argument"); return HP_ERR_ARG; }
    for (int i = 0; i < N; ++i)
        if (!conf_frames[i] || !paf_frames[i]) { set_error("hp_engine_read_outputs_frames: null frame buffer %d", i); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const size_t plane = (size_t)e->out_h * e->out_w;
    const size_t ea = e->hdr.conf_channels * plane, eb = e->hdr.paf_channels * plane;
    if (publish && hpb::handoff::enabled())   // D2H into the publication's own pinned copy, then into the caller's buffers
        return hpb::handoff::publish(e->ho_ring, &e->ho_pos, e->device, e->stream, e->d_conf, e->d_paf, N, ea, eb, conf_frames, paf_frames);
    const size_t need = (size_t)e->max_batch * (ea + eb);
    if (e->pin_out_floats < need) {
        if (e->pin_out) cudaFreeHost(e->pin_out);
        e->pin_out = nullptr; e->pin_out_floats = 0;
        HP_CUDA_TRY(cudaMallocHost(&e->pin_out, need * sizeof(float)));
        e->pin_out_floats = need;
    }
    float* ha = e->pin_out;
    float* hb = e->pin_out + (size_t)N * ea;
    HP_CUDA_TRY(cudaMemcpyAsync(ha, e->d_conf, (size_t)N * ea * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    HP_CUDA_TRY(cudaMemcpyAsync(hb, e->d_paf, (size_t)N * eb * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < N; ++i) {
        memcpy(conf_frames[i], ha + (size_t)i * ea, ea * sizeof(float));
        memcpy(paf_frames[i], hb + (size_t)i * eb, eb * sizeof(float));
    }
    return HP_OK;
}

// D2D snapshot of the last batch's outputs into caller-owned device tensors, asynchronously on `stream`
// (lets a pipelined caller parse batch i on another stream while batch i+1 overwrites the engine's outputs)
int hp_engine_copy_outputs_device(hp_engine* e, float* d_conf, float* d_paf, int N, void* stream)
{
    if (!e || !d_conf || !d_paf || N <= 0 || N > e->max_batch) { set_error("hp_engine_copy_outputs_device: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : e->stream;
    const size_t plane = (size_t)e->out_h * e->out_w;
    HP_CUDA_TRY(cudaMemcpyAsync(d_conf, e->d_conf, N * e->hdr.conf_channels * plane * sizeof(float), cudaMemcpyDeviceToDevice, st));
    HP_CUDA_TRY(cudaMemcpyAsync(d_paf, e->d_paf, N * e->hdr.paf_channels * plane * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return HP_OK;
}

int hp_engine_sync(hp_engine* e)
{
    if (!e) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(e->device));
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return HP_OK;
}

// test hook: copies activation buffer `buf` (fp16 NHWC, N frames) to the host
int hp_engine_debug_read_buffer(hp_engine* e, int buf, void* out_f16, int N, int* H, int* W, int* C)
{
    if (!e || buf < 0 || buf >= (int)e->bufs.size()) { set_error("hp_engine_debug_read_buffer: bad buffer"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const EngBuffer& b = e->bufs[buf];
    if (H) *H = b.H;
    if (W) *W = b.W;
    if (C) *C = b.channels;
    if (b.fused_away && out_f16) { set_error("hp_engine_debug_read_buffer: buffer %d is not materialised (the max-pool / 1x1 depthwise op that reads it runs in the producing conv's epilogue; HPB_NO_POOL_FUSE=1 / HPB_NO_DW1_FUSE=1 keep it)", buf); return HP_ERR_UNSUPPORTED; }
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    const size_t es = (size_t)elem_bytes(e->dtype);   // element type follows the engine's dtype
    if (out_f16) HP_CUDA_TRY(cudaMemcpy(out_f16, b.d, (size_t)N * b.H * b.W * b.channels * es, cudaMemcpyDeviceToHost));
    return HP_OK;
}

int hp_engine_debug_write_buffer(hp_engine* e, int buf, const void* in_f16, int N)
{
    if (!e || buf < 0 || buf >= (int)e->bufs.size() || !in_f16 || N <= 0 || N > e->max_batch) { set_error("hp_engine_debug_write_buffer: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const EngBuffer& b = e->bufs[buf];
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    const size_t es = (size_t)elem_bytes(e->dtype);
    HP_CUDA_TRY(cudaMemcpy(b.d, in_f16, (size_t)N * b.H * b.W * b.channels * es, cudaMemcpyHostToDevice));
    return HP_OK;
}

int hp_engine_debug_run_ops(hp_engine* e, int first_op, int last_op, int N)
{
    if (!e || first_op < 0 || last_op >= (int)e->ops.size() || first_op > last_op || N <= 0 || N > e->max_batch) { set_error("hp_engine_debug_run_ops: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    int rc = run_graph(e, N, true, e->stream, first_op, last_op);
    if (rc) return rc;
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return HP_OK;
}

// INT8 calibration (TensorRT's IInt8MinMaxCalibrator): runs the graph op by op on a TF32 engine and folds max |x| of every op's
// output buffer into absmax[out_buf] -- a running maximum over calls and over the max_batch-frame chunks of the N frames
int hp_engine_calibrate_u8(hp_engine* e, const uint8_t* frames, int N, float* absmax, int n_buffers)
{
    if (!e || !frames || !absmax || N <= 0) { set_error("hp_engine_calibrate_u8: bad argument"); return HP_ERR_ARG; }
    if (e->dtype != HP_DTYPE_TF32) { set_error("hp_engine_calibrate_u8: calibration runs on a TF32 engine (this one has dtype %d)", e->dtype); return HP_ERR_ARG; }
    if (n_buffers != (int)e->bufs.size()) { set_error("hp_engine_calibrate_u8: %d absmax entries for %zu buffers", n_buffers, e->bufs.size()); return HP_ERR_ARG; }
    for (int b = 0; b < n_buffers; ++b)
        if (!(absmax[b] >= 0.f)) { set_error("hp_engine_calibrate_u8: absmax[%d] = %g (the running maximum starts at values >= 0)", b, (double)absmax[b]); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    unsigned* d_amax = nullptr;
    HP_CUDA_TRY(cudaMalloc(&d_amax, (size_t)n_buffers * sizeof(unsigned)));
    auto done = [&](int rc) { cudaFree(d_amax); return rc; };
    if (cudaMemcpy(d_amax, absmax, (size_t)n_buffers * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) { set_error("hp_engine_calibrate_u8: upload failed"); return done(HP_ERR_CUDA); }
    const size_t frame_bytes = (size_t)e->in_h * e->in_w * 3;
    for (int f0 = 0; f0 < N; f0 += e->max_batch) {
        const int n = std::min(e->max_batch, N - f0);
        memcpy(e->pin_frames, frames + (size_t)f0 * frame_bytes, (size_t)n * frame_bytes);
        if (cudaMemcpyAsync(e->d_frames, e->pin_frames, (size_t)n * frame_bytes, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) { set_error("hp_engine_calibrate_u8: H2D failed"); return done(HP_ERR_CUDA); }
        for (int oi = 0; oi < (int)e->ops.size(); ++oi) {
            const int rc = run_graph(e, n, true, e->stream, oi, oi);
            if (rc) return done(rc);
            const PackOp& po = e->ops[oi].po;
            if (po.type == OP_PIFPAF_HEAD || po.type == OP_PPN_HEAD || (po.type == OP_CONV && po.out_mode == OUT_F32_NCHW_SPLIT)) continue;
            const EngBuffer& b = e->bufs[po.out_buf];
            const size_t cnt = (size_t)n * b.H * b.W * b.channels;
            absmax_f32_kernel<<<(unsigned)std::min<size_t>(1024, (cnt + 255) / 256), 256, 0, e->stream>>>((const float*)b.d, cnt, d_amax + po.out_buf);
        }
        if (cudaStreamSynchronize(e->stream) != cudaSuccess) { set_error("hp_engine_calibrate_u8: %s", cudaGetErrorString(cudaGetLastError())); return done(HP_ERR_CUDA); }
    }
    if (cudaMemcpy(absmax, d_amax, (size_t)n_buffers * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) { set_error("hp_engine_calibrate_u8: read-back failed"); return done(HP_ERR_CUDA); }
    return done(HP_OK);
}

// 1 when `pack` is a model pack that carries an INT8 scale table (what data_type::kINT8 needs), else 0; host only
int hp_pack_int8_calibrated(const void* pack, size_t pack_bytes)
{
    if (!pack || pack_bytes < sizeof(PackHeader)) return 0;
    PackHeader hdr;
    memcpy(&hdr, pack, sizeof(hdr));
    if (memcmp(hdr.magic, PACK_MAGIC, 8) != 0 || hdr.version != PACK_VERSION || hdr.n_buffers == 0 || hdr.reserved[0] != hdr.n_buffers ||
        hdr.n_buffers > 65536 || hdr.n_ops > 65536 || hdr.blob_floats > ((uint64_t)1 << 34))
        return 0;
    const size_t need = sizeof(PackHeader) + (size_t)hdr.n_buffers * sizeof(PackBuffer) + (size_t)hdr.n_ops * sizeof(PackOp) +
                        ((size_t)hdr.blob_floats + hdr.n_buffers) * sizeof(float);
    return pack_bytes >= need ? 1 : 0;
}

// test hook: the kernel op `op` launches on the next run over u8 frames, as decided when the engine was created (EngOp::launch and
// the conv plan's tile width): conv<f16|tf32|i8,BN[,res][,stem3|stem7]>, halo<BN[,pool|,wide|,pp|,pool,pp]>, dw_strip<K,S>, dw_col, dw_tma<1|2>, dw_f32,
// dw_i8, maxpool<K>, maxpool_f32, maxpool_i8, im2col, im2col_i8, heads, ppn_head, or none when a neighbouring op's launch covers it
int hp_engine_debug_op_kernel(const hp_engine* e, int op, char* name, int cap)
{
    if (!e || op < 0 || op >= (int)e->ops.size() || !name || cap <= 0) { set_error("hp_engine_debug_op_kernel: bad argument"); return HP_ERR_ARG; }
    const EngOp& o = e->ops[op];
    const PackOp& po = o.po;
    const int BN = o.plan.prm.BN;
    const char* dt = e->dtype == HP_DTYPE_TF32 ? "tf32," : e->dtype == HP_DTYPE_INT8 ? "i8," : "f16,";
    std::string s;
    switch (o.launch) {
    case Launch::None: case Launch::StemOrIm2col: s = "none"; break;
    case Launch::Im2col: case Launch::Im2colF32: s = "im2col"; break;
    case Launch::Conv:
        s = std::string("conv<") + dt + std::to_string(BN) + (o.plan.prm.res_mode ? ",res>" : ">");
        break;
    case Launch::ConvStem: s = "conv<f16," + std::to_string(BN) + ",stem" + std::to_string(po.R) + ">"; break;
    case Launch::Halo: s = "halo<" + std::to_string(BN) + ">"; break;
    case Launch::HaloPool: s = "halo<" + std::to_string(BN) + ",pool>"; break;
    case Launch::HaloWide: s = "halo<" + std::to_string(BN) + ",wide>"; break;
    case Launch::HaloPP: s = "halo<" + std::to_string(BN) + ",pp>"; break;
    case Launch::HaloPoolPP: s = "halo<" + std::to_string(BN) + ",pool,pp>"; break;
    case Launch::DwTma: s = "dw_tma<1>"; break;
    case Launch::DwTmaPair: s = "dw_tma<2>"; break;
    case Launch::DwCol: s = "dw_col"; break;
    case Launch::DwStrip: s = "dw_strip<" + std::to_string(po.R) + "," + std::to_string(po.stride ? po.stride : 1) + ">"; break;
    case Launch::MaxPool: s = "maxpool<" + std::to_string(po.R ? po.R : 2) + ">"; break;
    case Launch::Heads: case Launch::HeadsF32: s = "heads"; break;
    case Launch::PpnHead: case Launch::PpnHeadF32: s = "ppn_head"; break;
    case Launch::DwF32: s = "dw_f32"; break;
    case Launch::MaxPoolF32: s = "maxpool_f32"; break;
    case Launch::Im2colI8: s = "im2col_i8"; break;
    case Launch::DwI8: s = "dw_i8"; break;
    case Launch::MaxPoolI8: s = "maxpool_i8"; break;
    }
    if ((int)s.size() >= cap) { set_error("hp_engine_debug_op_kernel: %zu-character name, capacity %d", s.size(), cap); return HP_ERR_CAPACITY; }
    memcpy(name, s.c_str(), s.size() + 1);
    return HP_OK;
}

long long hp_engine_launch_count(const hp_engine* e) { return e ? e->launches : 0; }

int hp_engine_set_output_override(hp_engine* e, const float* d_conf, const float* d_paf)
{
    if (!e) return HP_ERR_ARG;
    e->override_conf = d_conf;
    e->override_paf = d_paf;
    return HP_OK;
}

int hp_engine_set_profiling(hp_engine* e, int enable)
{
    if (!e) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(e->device));
    if (enable && e->ev.empty()) {
        e->ev.resize((e->ops.size() + 1) * hp_engine::EV_DEPTH);
        for (auto& ev : e->ev) HP_CUDA_TRY(cudaEventCreate(&ev));
    }
    if (enable) {
        e->op_ms_sum.assign(e->ops.size(), 0.0);
        e->profiled_runs = 0;
        e->ev_head = e->ev_tail = 0;
    } else {
        collect_profile(e);
    }
    e->profiling = enable != 0;
    return HP_OK;
}

int hp_engine_get_profile(hp_engine* e, double* ms_per_op, int* op_type, double* flops_per_op, int cap, int* n_ops, long long* runs)
{
    if (!e) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(e->device));
    collect_profile(e);
    const int n = (int)e->ops.size();
    if (n_ops) *n_ops = n;
    if (runs) *runs = e->profiled_runs;
    if (cap < n) { set_error("hp_engine_get_profile: cap %d < %d ops", cap, n); return HP_ERR_CAPACITY; }
    for (int i = 0; i < n; ++i) {
        if (ms_per_op) ms_per_op[i] = (e->profiled_runs && i < (int)e->op_ms_sum.size()) ? e->op_ms_sum[i] / e->profiled_runs : 0.0;
        if (op_type) op_type[i] = (int)e->ops[i].po.type;
        if (flops_per_op) flops_per_op[i] = e->ops[i].po.type == OP_CONV ? e->ops[i].plan.flops_per_frame : 0.0;
    }
    return HP_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// End-to-end pose call: HOST u8 frames -> humans on the host, tensors never leave the device in between
// (operator API sequence engine.inference(batch) + parser.process(packet) per image,
//  examples/operator_api_batched_images_paf.example.cpp:64-74), two batches in flight:
//
//   hp_pose_submit_u8_host(i+1)  H2D of batch i+1 on the copy stream  | overlaps the convs of batch i
//   hp_pose_collect(i)           waits for batch i's records (their D2H was enqueued right behind its parse)
//
// The per-batch launch sequence (every conv + the two parser kernels + the result D2H, ~60 nodes at cfg3) is captured
// once per slot into a CUDA graph and replayed with one cudaGraphLaunch; it is re-captured when anything baked into it
// changes (batch size, parser thresholds / capacities, benchmark override).
// ---------------------------------------------------------------------------------------------------------------------
int hp_paf_prepare(hp_paf* p, int N, int c_conf, int c_paf, int H, int W);
int hp_paf_state(const hp_paf* p, float* thresholds2, int* ints6);
int hp_paf_copy_results_host_async(hp_paf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream);
int hp_paf_grow_capacity(hp_paf* p, int flags);
int hp_pifpaf_process_device(hp_pifpaf* p, const float* d_pif, const float* d_paf, int N, int h, int w, void* stream);
int hp_pifpaf_pipeline_info(hp_pifpaf* p, void** stream, void** inputs_free_event, int* hcap);
int hp_pifpaf_copy_results_host_async(hp_pifpaf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream);
int hp_pifpaf_grow_capacity(hp_pifpaf* p, int flags);

#ifdef HPB_HALO_PHASES
// instrumented build only (-DHPB_HALO_PHASES, tools/halo_phases.py): the cycle counts conv_halo_kernel has summed since the last
// reset, in HALO_PH_* order (total, operand A late, operand B late, wgmma wait, epilogue, turn wait); reset != 0 zeroes them after
int hp_debug_halo_phases(unsigned long long* out, int n, int reset)
{
    if (!out || n != HALO_PH_COUNT) { set_error("hp_debug_halo_phases: expected %d counters", (int)HALO_PH_COUNT); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaDeviceSynchronize());
    HP_CUDA_TRY(cudaMemcpyFromSymbol(out, g_halo_phases, sizeof(unsigned long long) * HALO_PH_COUNT));
    if (reset) {
        const unsigned long long zero[HALO_PH_COUNT] = {};
        HP_CUDA_TRY(cudaMemcpyToSymbol(g_halo_phases, zero, sizeof(zero)));
    }
    return HP_OK;
}
#endif

} // extern "C" (helpers below are C++)

namespace {

int pose_enqueue_compute(hp_engine* e, hp_engine::PoseSlot& sl, cudaStream_t st)
{
    e->cur_frames = sl.d_frames;
    int rc = run_graph(e, sl.N, true, st);
    e->cur_frames = nullptr;
    if (rc) return rc;
    rc = hp_paf_process_device(sl.parser, e->d_conf, e->d_paf, sl.N, (int)e->hdr.conf_channels, (int)e->hdr.paf_channels, e->out_h, e->out_w, (void*)st);
    if (rc) return rc;
    return hp_paf_copy_results_host_async(sl.parser, sl.pin_humans, sl.pin_counts, sl.N, (void*)st);
}

// what both pipelined calls need in a slot: its own frame buffer (the plain entry points keep hp_engine::d_frames), the upload and
// completion events, and pinned record buffers for hcap humans per frame.  A captured graph holds their addresses: it goes when they move.
int slot_alloc(hp_engine* e, hp_engine::PoseSlot& sl, int hcap)
{
    if (!e->copy_stream) HP_CUDA_TRY(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    if (!sl.d_frames) HP_CUDA_TRY(cudaMalloc(&sl.d_frames, (size_t)e->max_batch * e->in_h * e->in_w * 3 + 16));
    if (!sl.h2d_done) HP_CUDA_TRY(cudaEventCreateWithFlags(&sl.h2d_done, cudaEventDisableTiming));
    if (!sl.done) HP_CUDA_TRY(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
    const size_t need_h = (size_t)e->max_batch * hcap, need_c = (size_t)2 * e->max_batch;
    if ((sl.pin_humans_n < need_h || sl.pin_counts_n < need_c) && sl.graph) { cudaGraphExecDestroy(sl.graph); sl.graph = nullptr; }
    if (sl.pin_humans_n < need_h) {
        if (sl.pin_humans) cudaFreeHost(sl.pin_humans);
        sl.pin_humans = nullptr; sl.pin_humans_n = 0;
        HP_CUDA_TRY(cudaMallocHost(&sl.pin_humans, need_h * sizeof(hp_human)));
        sl.pin_humans_n = need_h;
    }
    if (sl.pin_counts_n < need_c) {
        if (sl.pin_counts) cudaFreeHost(sl.pin_counts);
        sl.pin_counts = nullptr; sl.pin_counts_n = 0;
        HP_CUDA_TRY(cudaMallocHost(&sl.pin_counts, need_c * sizeof(int)));
        sl.pin_counts_n = need_c;
    }
    sl.hcap = hcap;
    return HP_OK;
}

// the N frames of a submitted batch into the slot's device buffer, ordered before the engine stream's next work: frames already in
// HBM by a D2D copy on the engine stream, host frames by an H2D on the copy stream (pageable ones through the slot's pinned staging,
// free since the slot was collected)
int slot_upload(hp_engine* e, hp_engine::PoseSlot& sl, const uint8_t* frames, int N, bool device_src)
{
    const size_t bytes = (size_t)N * e->in_h * e->in_w * 3;
    if (device_src) {
        HP_CUDA_TRY(cudaMemcpyAsync(sl.d_frames, frames, bytes, cudaMemcpyDeviceToDevice, e->stream));
        return HP_OK;
    }
    cudaPointerAttributes attr;
    const bool pinned = (cudaPointerGetAttributes(&attr, frames) == cudaSuccess && attr.type == cudaMemoryTypeHost);
    if (!pinned) cudaGetLastError();
    const uint8_t* src = frames;
    if (!pinned) {
        if (!sl.pin_frames) HP_CUDA_TRY(cudaMallocHost(&sl.pin_frames, (size_t)e->max_batch * e->in_h * e->in_w * 3));
        memcpy(sl.pin_frames, frames, bytes);
        src = sl.pin_frames;
    }
    HP_CUDA_TRY(cudaMemcpyAsync(sl.d_frames, src, bytes, cudaMemcpyHostToDevice, e->copy_stream));
    HP_CUDA_TRY(cudaEventRecord(sl.h2d_done, e->copy_stream));
    HP_CUDA_TRY(cudaStreamWaitEvent(e->stream, sl.h2d_done, 0));
    return HP_OK;
}

int pose_slot_prepare(hp_engine* e, hp_engine::PoseSlot& sl, hp_paf* parser, int N)
{
    int rc = hp_paf_prepare(parser, N, (int)e->hdr.conf_channels, (int)e->hdr.paf_channels, e->out_h, e->out_w);
    if (rc) return rc;
    float kf[2]; int ki[6];
    hp_paf_state(parser, kf, ki);
    rc = slot_alloc(e, sl, ki[4]);
    if (rc) return rc;
    // anything the captured sequence bakes in
    const bool same = sl.graph && sl.key_N == N && sl.key_parser == (const void*)parser && memcmp(sl.key_f, kf, sizeof(kf)) == 0 && memcmp(sl.key_i, ki, sizeof(ki)) == 0 &&
                      sl.key_ovr[0] == (const void*)e->override_conf && sl.key_ovr[1] == (const void*)e->override_paf;
    if (!same && sl.graph) { cudaGraphExecDestroy(sl.graph); sl.graph = nullptr; }
    sl.key_N = N; sl.key_parser = parser; memcpy(sl.key_f, kf, sizeof(kf)); memcpy(sl.key_i, ki, sizeof(ki));
    sl.key_ovr[0] = e->override_conf; sl.key_ovr[1] = e->override_paf;
    sl.N = N; sl.parser = parser; sl.decoder = nullptr;
    return HP_OK;
}

// enqueue this slot's compute on the engine stream: graph replay when possible, direct launches otherwise
int pose_launch(hp_engine* e, hp_engine::PoseSlot& sl)
{
    if (e->graphs_ok && !e->profiling) {
        if (!sl.graph) {
            cudaGraph_t g = nullptr;
            if (cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
                const long long l0 = e->launches;
                const int rc = pose_enqueue_compute(e, sl, e->stream);
                const cudaError_t ce = cudaStreamEndCapture(e->stream, &g);
                e->launches = l0 - 2;   // capturing launches nothing (the parser counted its two kernels: taken back here)
                if (rc == HP_OK && ce == cudaSuccess && g && cudaGraphInstantiate(&sl.graph, g, 0) == cudaSuccess) e->graph_captures++;
                else { sl.graph = nullptr; e->graphs_ok = false; cudaGetLastError(); }
                if (g) cudaGraphDestroy(g);
            } else { e->graphs_ok = false; cudaGetLastError(); }
        }
        if (sl.graph) {
            HP_CUDA_TRY(cudaGraphLaunch(sl.graph, e->stream));
            e->graph_launches++;
            e->launches += e->step_kernels + 2;   // the replay runs what the direct path counts: the engine's step + the parser's two kernels
            return HP_OK;
        }
    }
    return pose_enqueue_compute(e, sl, e->stream);
}

} // namespace

extern "C" {

// ---- OpenPifPaf packs: engine on its stream, decoder on the decoder's stream, two batches in flight ----
static int pifpaf_slot_prepare(hp_engine* e, hp_engine::PoseSlot& sl, hp_pifpaf* dec, int N)
{
    if (sl.graph) { cudaGraphExecDestroy(sl.graph); sl.graph = nullptr; }   // (a PAF-parser graph of an earlier use of this slot)
    int hcap = 0;
    hp_pifpaf_pipeline_info(dec, nullptr, nullptr, &hcap);
    const int rc = slot_alloc(e, sl, hcap);
    if (rc) return rc;
    if (!sl.conv_done) HP_CUDA_TRY(cudaEventCreateWithFlags(&sl.conv_done, cudaEventDisableTiming));
    sl.N = N; sl.parser = nullptr; sl.decoder = dec;
    return HP_OK;
}

// engine kernels of the slot on the engine stream, then the decoder + the record D2H on the decoder's stream
static int pifpaf_enqueue(hp_engine* e, hp_engine::PoseSlot& sl)
{
    void* dst = nullptr; void* free_ev = nullptr;
    hp_pifpaf_pipeline_info(sl.decoder, &dst, &free_ev, nullptr);
    cudaStream_t dec_stream = (cudaStream_t)dst;
    e->cur_frames = sl.d_frames;
    e->heads_wait = (cudaEvent_t)free_ev;    // NULL before the decoder's first batch
    int rc = run_graph(e, sl.N, true, e->stream);
    e->cur_frames = nullptr;
    e->heads_wait = nullptr;
    if (rc) return rc;
    HP_CUDA_TRY(cudaEventRecord(sl.conv_done, e->stream));
    HP_CUDA_TRY(cudaStreamWaitEvent(dec_stream, sl.conv_done, 0));
    rc = hp_pifpaf_process_device(sl.decoder, e->d_conf, e->d_paf, sl.N, e->out_h, e->out_w, (void*)dec_stream);
    if (rc) return rc;
    rc = hp_pifpaf_copy_results_host_async(sl.decoder, sl.pin_humans, sl.pin_counts, sl.N, (void*)dec_stream);
    if (rc) return rc;
    HP_CUDA_TRY(cudaEventRecord(sl.done, dec_stream));
    return HP_OK;
}

static int pose_submit_pifpaf(hp_engine* e, hp_pifpaf* dec, const uint8_t* frames, int N, int* ticket, bool device_src)
{
    if (!e || !dec || !frames || !ticket) { set_error("hp_pose_submit_pifpaf: null argument"); return HP_ERR_ARG; }
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    if (e->hdr.head_type != 1) { set_error("hp_pose_submit_pifpaf: the model pack has no OpenPifPaf heads (head_type %u)", e->hdr.head_type); return HP_ERR_UNSUPPORTED; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const int idx = e->next_slot;
    hp_engine::PoseSlot& sl = e->slots[idx];
    if (sl.busy) { set_error("hp_pose_submit_pifpaf: two batches are already in flight -- collect ticket %d first", idx); return HP_ERR_ARG; }
    int rc = pifpaf_slot_prepare(e, sl, dec, N);
    if (rc) return rc;
    e->reserve_sms = e->opt.pifpaf_reserve_sms;   // the decoder's growth kernel (one warp per frame) runs underneath the next batch's convolutions
    rc = slot_upload(e, sl, frames, N, device_src);
    if (rc) return rc;
    rc = pifpaf_enqueue(e, sl);
    if (rc) return rc;
    sl.busy = true;
    e->next_slot = idx ^ 1;
    *ticket = idx;
    return HP_OK;
}

static int pose_submit(hp_engine* e, hp_paf* parser, const uint8_t* frames, int N, int* ticket, bool device_src)
{
    if (!e || !parser || !frames || !ticket) { set_error("hp_pose_submit: null argument"); return HP_ERR_ARG; }
    if (N <= 0 || N > e->max_batch) { set_error("Input batch size overflow: Yours@%d Max@%d", N, e->max_batch); return HP_ERR_BATCH; }
    if (e->hdr.head_type == 1) { set_error("hp_pose_submit: the model pack has OpenPifPaf heads (use hp_engine_infer_u8_host + hp_pifpaf_process_device)"); return HP_ERR_UNSUPPORTED; }
    if (e->hdr.head_type != 0) {
        set_error("hp_pose_submit: the model pack has Pose Proposal Network heads (use hp_engine_infer_u8_device + hp_ppn_process_device_strided on the engine's outputs)");
        return HP_ERR_UNSUPPORTED;
    }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    const int idx = e->next_slot;
    hp_engine::PoseSlot& sl = e->slots[idx];
    if (sl.busy) { set_error("hp_pose_submit: two batches are already in flight -- collect ticket %d first", idx); return HP_ERR_ARG; }
    int rc = pose_slot_prepare(e, sl, parser, N);
    if (rc) return rc;
    rc = slot_upload(e, sl, frames, N, device_src);   // (the captured graph reads the slot's buffer)
    if (rc) return rc;
    rc = pose_launch(e, sl);
    if (rc) return rc;
    HP_CUDA_TRY(cudaEventRecord(sl.done, e->stream));
    sl.busy = true;
    e->next_slot = idx ^ 1;
    *ticket = idx;
    return HP_OK;
}

int hp_pose_submit_u8_host(hp_engine* e, hp_paf* parser, const uint8_t* frames, int N, int* ticket)
{
    return pose_submit(e, parser, frames, N, ticket, false);
}

// the same with the frames already resident in device memory (what a decoder / capture pipeline on the GPU hands over)
int hp_pose_submit_u8_device(hp_engine* e, hp_paf* parser, const uint8_t* d_frames, int N, int* ticket)
{
    return pose_submit(e, parser, d_frames, N, ticket, true);
}

int hp_pose_submit_pifpaf_u8_host(hp_engine* e, hp_pifpaf* decoder, const uint8_t* frames, int N, int* ticket)
{
    return pose_submit_pifpaf(e, decoder, frames, N, ticket, false);
}

int hp_pose_submit_pifpaf_u8_device(hp_engine* e, hp_pifpaf* decoder, const uint8_t* d_frames, int N, int* ticket)
{
    return pose_submit_pifpaf(e, decoder, d_frames, N, ticket, true);
}

int hp_pose_collect(hp_engine* e, int ticket, hp_human* out, int cap, int* n_out)
{
    if (!e || ticket < 0 || ticket > 1 || !out || !n_out || cap < 0) { set_error("hp_pose_collect: bad argument"); return HP_ERR_ARG; }
    hp_engine::PoseSlot& sl = e->slots[ticket];
    if (!sl.busy) { set_error("hp_pose_collect: ticket %d is not in flight", ticket); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(e->device));
    HP_CUDA_TRY(cudaEventSynchronize(sl.done));
    sl.busy = false;
    const int N = sl.N;
    for (int attempt = 0; sl.decoder && attempt < 5; ++attempt) {
        int flags = 0;
        for (int f = 0; f < N; ++f) flags |= sl.pin_counts[N + f];
        if (!flags) break;
        // the reference decoder is unbounded: grow what overflowed and run this slot again, alone (the other batch in flight is
        // waited for first: its fields live in the same engine outputs)
        if (hp_pifpaf_grow_capacity(sl.decoder, flags) != HP_OK) { set_error("hp_pose_collect: decoder capacity limit reached (flags=%d)", flags); return HP_ERR_CAPACITY; }
        void* dst = nullptr;
        hp_pifpaf_pipeline_info(sl.decoder, &dst, nullptr, nullptr);
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
        HP_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)dst));
        int rc = pifpaf_slot_prepare(e, sl, sl.decoder, N);
        if (rc) return rc;
        rc = pifpaf_enqueue(e, sl);
        if (rc) return rc;
        HP_CUDA_TRY(cudaEventSynchronize(sl.done));
    }
    for (int attempt = 0; !sl.decoder && attempt < 8; ++attempt) {
        int flags = 0;
        for (int f = 0; f < N; ++f) flags |= sl.pin_counts[N + f];
        if (!flags) break;
        // the reference is unbounded: grow the parser capacity that overflowed and run this slot's frames again (they are still
        // in its device buffer), synchronously and outside the graph
        if (hp_paf_grow_capacity(sl.parser, flags) != HP_OK) { set_error("hp_pose_collect: parser capacity limit reached (flags=%d)", flags); return HP_ERR_CAPACITY; }
        int rc = pose_slot_prepare(e, sl, sl.parser, N);
        if (rc) return rc;
        rc = pose_enqueue_compute(e, sl, e->stream);
        if (rc) return rc;
        HP_CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    for (int f = 0; f < N; ++f) if (sl.pin_counts[N + f]) { set_error("hp_pose_collect: parser capacity exceeded"); return HP_ERR_CAPACITY; }
    for (int f = 0; f < N; ++f) {
        const int n = sl.pin_counts[f];
        if (n > cap) { set_error("hp_pose_collect: frame %d has %d humans but the caller's capacity is %d", f, n, cap); return HP_ERR_CAPACITY; }
        n_out[f] = n;
        memcpy(out + (size_t)f * cap, sl.pin_humans + (size_t)f * sl.hcap, sizeof(hp_human) * n);
    }
    return HP_OK;
}

// the synchronous form: one batch in, its humans out
int hp_pose_run_u8_host(hp_engine* e, hp_paf* parser, const uint8_t* frames, int N, hp_human* out, int cap, int* n_out)
{
    if (e) for (int t = 0; t < 2; ++t) if (e->slots[t].busy) { set_error("hp_pose_run_u8_host: a submitted batch (ticket %d) has not been collected", t); return HP_ERR_ARG; }
    int ticket = -1;
    int rc = hp_pose_submit_u8_host(e, parser, frames, N, &ticket);
    if (rc) return rc;
    return hp_pose_collect(e, ticket, out, cap, n_out);
}

int hp_pose_stats(const hp_engine* e, long long* graph_captures, long long* graph_launches)
{
    if (!e) return HP_ERR_ARG;
    if (graph_captures) *graph_captures = e->graph_captures;
    if (graph_launches) *graph_launches = e->graph_launches;
    return HP_OK;
}

} // extern "C"
