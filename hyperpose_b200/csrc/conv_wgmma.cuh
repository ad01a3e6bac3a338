// conv_wgmma.cuh -- implicit-GEMM convolution on the sm_90a (Hopper) tensor cores.
//
// Replaces the TensorRT-executed CNN of the reference (IExecutionContext::executeV2,
// src/tensorrt.cpp:387-396; layer shapes from hyperpose/Model/backbones.py:447-509 and
// hyperpose/Model/openpose/model/openpose.py:36-199).
//
//   D[128 pixels, BN out-channels] += A[128 pixels, 128 bytes of in-channels] * B[BN, 128 bytes]^T
//   summed over (filter tap r,s) x (channel chunk): one "k-step" per (r, s, chunk).
//
// * activations are NHWC (fp16, or fp32 rounded to the TF32 grid for the kFLOAT engine); the A tile of a k-step is ONE
//   im2col-mode TMA load (cp.async.bulk.tensor.4d...im2col): 128 consecutive output pixels (in n,h,w order, wrapping over rows
//   and images inside the TMA unit) x 128 bytes of channels at filter offset (s, r); out-of-image elements are zero-filled by
//   the TMA unit = "SAME" padding, no im2col buffer in HBM and no tile padding waste;
// * weights are [G][Cout_pad][R][S][Cin_g] (K-major); the B tile is a 2-D TMA box {128 bytes, BN};
// * both land in shared memory in the 128-byte-swizzled K-major layout wgmma reads through its matrix descriptors;
// * persistent CTAs (one per SM), warp-specialised: one thread of warpgroup 0 issues the TMA loads into a ring of
//   mbarrier-guarded stages; warpgroups 1 and 2 each own 64 of the 128 pixel rows, run wgmma.mma_async m64nBN with the fp32
//   accumulators in registers, and apply the epilogue (bias (+ residual) + PReLU -> fp16 / TF32 NHWC, or fp32 NCHW planes for
//   the parser) while the producer already streams the next tile: fp16 NHWC outputs at BN = 64 / 128 go through a shared-memory
//   staging slot and TMA stores (conv_epilogue_tma), everything else straight from the registers.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace hpb {

constexpr int CONV_BLOCK_M = 128;   // pixels per tile
constexpr int CONV_BLOCK_K = 64;    // fp16 channels per k-step == one 128-byte swizzle row
constexpr int TF32_BLOCK_K = 32;    // fp32 channels per k-step == one 128-byte swizzle row
constexpr int CONV_MAX_STAGES = 8;
constexpr int CONV_THREADS = 384;   // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma + epilogue of pixel rows 0-63 / 64-127
constexpr int CONV_A_BYTES = CONV_BLOCK_M * 128; // 16 KiB
constexpr size_t CONV_SMEM_LIMIT = 227 * 1024;

enum ConvOutMode : int {
    OUT_F16_NHWC = 0,       // NHWC activations (fp16; fp32 in the TF32 engine), out[pixel * ld + ch_off + g * cout_g + n]
    OUT_F32_NCHW_SPLIT = 1, // fp32 planar; channels [0,split) -> out, [split,cout_g) -> out2 (conf / paf for the parser)
};

struct ConvParams {
    int Nb, H, W;              // batch, spatial size (stride 1, "SAME" padding: output size == input size)
    int R, S;                  // filter taps
    int groups, cin_g;         // cin_g: multiple of one k-step (64 fp16 / 32 fp32 channels)
    int cout_g, cout_g_pad;    // real / padded (multiple of BN) output channels per group
    int BN;                    // tile N == wgmma N (16, 32, 48, 64, 96 or 128)
    int m_tiles;               // ceil(Nb * H * W / 128): a tile is 128 CONSECUTIVE output pixels in (n, h, w) order
    int in_ch_off;             // first input channel inside the input buffer
    int num_stages;
    const float* bias;         // [groups * cout_g_pad]
    const float* alpha;        // [groups * cout_g_pad]   y = v > 0 ? v : alpha * v   (0 => ReLU, 1 => linear)
    int out_mode;
    void* out; void* out2;
    int out_ld, out_ch_off;    // NHWC: channels per pixel of the output buffer / first channel written
    int split;                 // NCHW_SPLIT: channels [0,split) go to out, the rest to out2
    const void* res;           // residual input [pixels, res_ld] (+ res_ch_off), same element type as the activations, or nullptr
    int res_ld, res_ch_off;
    int res_mode;              // 1: y = act(v + res)   2: y = act(v) + res
    // a 1x1 "depthwise" op that follows the conv (per-channel scale + bias + PReLU: the filter_size (1,1) separable blocks of
    // MobilenetThin-OpenPose) applied in the epilogue, with the fp16 rounding of the tensor in between kept: bit-identical with the two launches
    const float* post_w; const float* post_b; const float* post_a;   // [groups * cout_g] each, or nullptr
    // fused u8 stem (conv_wgmma_kernel<__half, BN, false, R>): the first conv gathers its RxRx3 patches from the u8 frames itself
    const uint8_t* frames;     // [Nb, in_h, in_w, 3]
    int in_h, in_w, stem_stride, stem_pad_h, stem_pad_w, flip;
    double factor;
    float mean[3];
    // INT8 engine (conv_wgmma_kernel<int8_t, ...>): v = (float)acc * mul[c] + bias[c], mul = s_in * s_w[c]; a residual reads
    // q_r * res_scale; NHWC stores clamp(rint(y * out_inv_scale), -127, 127)
    const float* mul;          // [groups * cout_g_pad]
    float out_inv_scale, res_scale;
    int in_g_stride;           // input channels between groups (the real cin_g: a group's padded last k-step reads on into the next
                               // group's channels, or past the buffer's end as zeros, against zero weights)
    int tma_store;             // 1: fp16 NHWC outputs go through shared memory and TMA stores (conv_epilogue_tma, BN = 64 or 128)
};

// accumulator element of conv_wgmma_kernel<T, ...>: fp32 for the fp16 / TF32 engines, s32 for the INT8 engine
template <typename T> struct ConvAcc { using type = float; };
template <> struct ConvAcc<int8_t> { using type = int; };

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// im2col-mode load: {c, w, h, n} = channel + base pixel (output pixel minus padding); {offw, offh} = filter tap
__device__ __forceinline__ void tma_load_im2col_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c, int w, int h, int n, int offw, int offh)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(dst), "l"(m), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"((unsigned short)offw), "h"((unsigned short)offh)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(m), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
// four 8 x 8 fp16 matrices, one per register: the thread holds row lane / 4, columns 2 (lane % 4) + {0, 1} of each (the accumulator
// fragment's layout); lane 8 i + r gives the address of row r of matrix i
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3)
{
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}
__device__ __forceinline__ void named_barrier_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the thread's bulk groups but the newest N have finished reading shared memory / have completed (their writes are performed)
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint32_t half2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
// programmatic dependent launch (no-ops when the kernel was launched without the attribute)
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// round-to-nearest onto the TF32 grid (the value stays an fp32 bit pattern with 13 zero low mantissa bits)
__device__ __forceinline__ float round_tf32(float x)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// wgmma shared-memory matrix descriptor (sm_90), K-major, 128-byte swizzle:
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major, 1 by convention)
//   [32,46) stride byte offset >> 4 (= 1024 B between 8-row groups) | [49,52) base offset = 0 (1024-byte aligned tiles)
//   [62,64) layout type = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffffu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator register across the wgmma issue / wait statements
template <int R> __device__ __forceinline__ void fence_acc(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R> __device__ __forceinline__ void fence_acc(int (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x K] * B[N x K]^T, both operands K-major in 128B-swizzled shared memory; K = 32 bytes of the element type
// (16 fp16 / 8 tf32); scale_d = 0 overwrites D.  One specialisation per (element type, N) because the register list is part of the
// instruction.
template <typename T, int N> __device__ __forceinline__ void wgmma(typename ConvAcc<T>::type (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma<__half, 16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<__half, 32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<__half, 48>(float (&d)[24], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "%24, %25, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<__half, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<__half, 96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<__half, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 48>(float (&d)[24], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "%24, %25, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<float, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wgmma<int8_t, 16>(int (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<int8_t, 32>(int (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<int8_t, 48>(int (&d)[24], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "%24, %25, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<int8_t, 64>(int (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<int8_t, 96>(int (&d)[48], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
        "%48, %49, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma<int8_t, 128>(int (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
} // namespace ptx

struct ConvTile {
    int p0, g, n0; // first output pixel (flattened n,h,w), group, first output channel of the tile
};

// work item -> tile: n-tiles (over all groups) fastest, then 128-pixel blocks
__device__ __forceinline__ ConvTile decode_tile(const ConvParams& p, int tile, int n_tiles_g)
{
    ConvTile t;
    const int n_tiles_total = p.groups * n_tiles_g;
    const int nt = tile % n_tiles_total;
    const int mt = tile / n_tiles_total;
    t.g = nt / n_tiles_g;
    t.n0 = (nt - t.g * n_tiles_g) * p.BN;
    t.p0 = mt * CONV_BLOCK_M;
    return t;
}

struct PixelPos {
    int n, h, w;
};
__device__ __forceinline__ PixelPos unflatten(const ConvParams& p, int px)
{
    PixelPos q;
    const int hw = p.H * p.W;
    q.n = px / hw;
    const int rem = px - q.n * hw;
    q.h = rem / p.W;
    q.w = rem - q.h * p.W;
    return q;
}

// position in a ring of mbarrier-guarded buffers: the slot, and the parity of the phase its barriers are in.  (The member order
// steers ptxas's register assignment: phase first compiles conv_wgmma_kernel's producer and consumer loops to the same SASS as two
// separate counters.)
struct RingPos {
    uint32_t phase = 0;
    int slot = 0;
    __device__ __forceinline__ void step(int depth)
    {
        if (++slot == depth) { slot = 0; phase ^= 1; }
    }
    __device__ __forceinline__ void advance(int n, int depth)
    {
        slot += n;
        phase ^= (uint32_t)(slot / depth) & 1u;
        slot %= depth;
    }
};

// One thread per (output pixel, 64-channel chunk): gathers the RxRx3 neighbourhood (k = (r*R+s)*3 + c, c = model channel)
// into roundup(R*R*3, 64) fp16 channels.  SAME padding pads the *normalised* input with zeros.
//   u8 path : v = (float)((double)u8 * factor) (data.cpp:48); model channel c reads byte (flip ? 2-c : c)
//   f32 path: input is already scaled NCHW (tensorrt::inference(const std::vector<float>&, size_t))
// stride 2 (MobileNet / ResNet stems): TF "SAME" padding, pad_before = max((OH-1)*2 + R - H, 0) / 2.
template <bool U8, int R, int CHUNK>
__device__ __forceinline__ void im2col_chunk(const void* __restrict__ in, uint4* __restrict__ o, int oswz, int n, int h0, int w0, int H, int W,
                                             double factor, int flip, const float (&mean)[3])
{
    // 64 consecutive K entries of one output pixel: k = (r * R + s) * 3 + c, every index a compile-time constant
    constexpr int kmax = R * R * 3;
    __align__(16) __half vals[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) {
        const int k = CHUNK * 64 + j;
        float v = 0.f;
        if (k < kmax) {
            const int c = k % 3, rs = k / 3, s = rs % R, r = rs / R;
            const int hh = h0 + r, ww = w0 + s;
            if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
                if (U8) {
                    const uint8_t* px = (const uint8_t*)in + (((size_t)n * H + hh) * W + ww) * 3;
                    v = (float)((double)px[flip ? 2 - c : c] * factor) - mean[c];
                } else {
                    v = ((const float*)in)[(((size_t)n * 3 + c) * H + hh) * W + ww] - mean[c];
                }
            }
        }
        vals[j] = __float2half_rn(v);
    }
    const uint4* v4 = (const uint4*)vals;
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i ^ oswz] = v4[i];
}

// T = __half: fp16 activations, kind f16; T = float: fp32 activations on the TF32 grid, kind tf32 (the data_type::kFLOAT engine:
// every producer of a conv operand rounds to TF32 with round-to-nearest, so the tensor core's truncation on read is exact).
// T = int8_t: the INT8 engine -- symmetric int8 activations and per-output-channel int8 weights, kind s8 (k32) with exact s32
// accumulation; the epilogue (conv_epilogue_i8) rescales, adds bias / residual, applies PReLU and requantizes in fp32 with
// separately rounded operations, so that a CPU model reproduces every output byte.
// kRes: residual epilogue compiled in (ResNet / LW-OpenPose blocks).
// kStemR = 3 | 7: fused u8 stem -- the conv's input is the RxRx3 patch of each output pixel gathered from the u8 frames by the 128
// threads of warpgroup 0 straight into the swizzled A tile (im2col_chunk, the same values im2col3_kernel writes), so the im2col
// buffer is never written; the B tile still comes by TMA.
// y -> int8 of the output buffer: clamp(rint(y * inv_s), -127, 127), the product rounded on its own
__device__ __forceinline__ int8_t quantize_i8(float y, float inv_s)
{
    return (int8_t)min(max(__float2int_rn(__fmul_rn(y, inv_s)), -127), 127);
}

// The fp16 epilogue of one consumer warpgroup's m64 block (tile pixels p0 + 64 half .. + 63, all inside the batch) written through
// shared memory: the arithmetic of conv_wgmma_kernel's register epilogue, operation for operation, then the fp16 block goes into the
// warpgroup's staging slot (BN / 64 slices of {64 channels x 64 pixels}, each in the 128B-swizzled layout of one TMA box: pixel row q,
// 16-byte chunk j at q * 128 + ((j ^ q % 8) * 16)) and the leader thread stores each slice with one box of tmap_o, a 2-D map over
// [pixels of max_batch frames, the output's channels up to the layer's last].  The map clips the padding channels of a partial
// n-tile; the caller keeps pixels past the batch (a partial last tile, or N < max_batch) on the register epilogue.
template <int BN, bool kRes>
__device__ __forceinline__ void conv_epilogue_tma(const float (&acc)[BN / 2], const ConvParams& p, const ConvTile& t, const CUtensorMap* tmap_o,
                                                  uint32_t slot, int half, int warp, int lane)
{
    static_assert(BN == 64 || BN == 128, "one TMA box per 64-channel slice, at most two");
    constexpr int kSliceBytes = 64 * 128;
    const bool leader = (threadIdx.x & 127) == 0;
    const int bar_id = 1 + half;   // named barrier 1 / 2: consumer warpgroup 1 / 2
    const int col0 = 2 * (lane & 3);
    const float* bias = p.bias + t.g * p.cout_g_pad + t.n0;
    const float* alpha = p.alpha + t.g * p.cout_g_pad + t.n0;
    const int n_valid = min(BN, p.cout_g - t.n0);   // a multiple of 8: both channels of a pair are real, or neither
    const int och = p.out_ch_off + t.g * p.cout_g + t.n0;
    const int px0 = t.p0 + half * 64;
    if (leader) ptx::bulk_wait_read<0>();
    ptx::named_barrier_sync(bar_id, 128);   // the previous tile's store has read the slot
    // stmatrix: register i of a thread holds rows lane / 4 (+ 8 h) and channels 8 (4 jb + i) + col0 + {0, 1}; lane 8 i + r addresses
    // pixel row r of matrix i, so (row % 8) == r
    const int r = lane & 7, i = lane >> 3;
#pragma unroll
    for (int jb = 0; jb < BN / 32; ++jb) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const size_t pix = (size_t)(px0 + (warp & 3) * 16 + 8 * h + (lane >> 2));
            uint32_t v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int j = 4 * jb + k, c = 8 * j + col0;
                const bool real = c < n_valid;
                float a0 = acc[4 * j + 2 * h] + __ldg(bias + c), a1 = acc[4 * j + 2 * h + 1] + __ldg(bias + c + 1);
                float r0 = 0.f, r1 = 0.f;
                if (kRes && p.res_mode && real) {
                    const size_t ri = pix * p.res_ld + p.res_ch_off + t.g * p.cout_g + t.n0 + c;
                    const float2 rf = __half22float2(*((const __half2*)p.res + ri / 2)); r0 = rf.x; r1 = rf.y;
                }
                if (kRes && p.res_mode == 1) { a0 += r0; a1 += r1; }
                a0 = a0 > 0.f ? a0 : a0 * __ldg(alpha + c);
                a1 = a1 > 0.f ? a1 : a1 * __ldg(alpha + c + 1);
                if (kRes && p.res_mode == 2) { a0 += r0; a1 += r1; }
                __half2 h2 = __floats2half2_rn(a0, a1);
                if (p.post_w && real) {   // the fused 1x1 depthwise stage, as in the register epilogue
                    const int pc = t.g * p.cout_g + t.n0 + c;
                    const float2 x = __half22float2(h2);
                    float y0 = fmaf(x.x, __ldg(p.post_w + pc), 0.f) + __ldg(p.post_b + pc);
                    float y1 = fmaf(x.y, __ldg(p.post_w + pc + 1), 0.f) + __ldg(p.post_b + pc + 1);
                    y0 = y0 > 0.f ? y0 : y0 * __ldg(p.post_a + pc);
                    y1 = y1 > 0.f ? y1 : y1 * __ldg(p.post_a + pc + 1);
                    h2 = __floats2half2_rn(y0, y1);
                }
                v[k] = ptx::half2_bits(h2);
            }
            const int j = 4 * jb + i, row = (warp & 3) * 16 + 8 * h + r;
            ptx::stmatrix_x4(slot + (uint32_t)((j >> 3) * kSliceBytes + row * 128 + (((j & 7) ^ r) << 4)), v[0], v[1], v[2], v[3]);
        }
    }
    ptx::fence_proxy_async();   // the generic-proxy writes -> visible to the TMA store
    ptx::named_barrier_sync(bar_id, 128);
    if (leader) {
        ptx::tma_store_2d(tmap_o, slot, och, px0);
        if (BN == 128 && t.n0 + 64 < p.cout_g)   // (not a slice of padding channels only)
            ptx::tma_store_2d(tmap_o, slot + (uint32_t)kSliceBytes, och + 64, px0);
        ptx::bulk_commit();
    }
}

template <typename T, int BN, bool kRes, int kStemR = 0>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_o,
                  const ConvParams p)
{
    constexpr bool kF16 = std::is_same<T, __half>::value;
    constexpr bool kI8 = std::is_same<T, int8_t>::value;
    constexpr int BK = 128 / (int)sizeof(T);                 // channels per k-step
    constexpr int STAGE_BYTES = CONV_A_BYTES + BN * 128;      // a multiple of 1024: every tile stays aligned to the swizzle atom
    // the TMA-store epilogue (p.tma_store) exists for fp16 at BN = 64 and 128; other kernels always store from registers
    constexpr bool kTmaForm = kF16 && (BN == 64 || BN == 128);
    extern __shared__ uint8_t smem_raw[];
    ptx::pdl_launch_dependents();   // the next kernel may start its prologue on every SM this grid has left
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* s_stage = smem + (size_t)p.num_stages * STAGE_BYTES;                  // tma_store: [2][BN x 128 B], one slot per consumer warpgroup
    uint64_t* full_bar = (uint64_t*)(s_stage + (p.tma_store ? 2 * BN * 128 : 0)); // [stages]  TMA -> wgmma
    uint64_t* empty_bar = full_bar + CONV_MAX_STAGES;                             // [stages]  wgmma -> TMA

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles_g = p.cout_g_pad / BN;
    const int total_tiles = p.m_tiles * p.groups * n_tiles_g;
    const int chunks = p.cin_g / BK;
    const int ksteps = p.R * p.S * chunks;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmap_a);
        ptx::prefetch_tmap(&tmap_b);
        if (kTmaForm && p.tma_store) ptx::prefetch_tmap(&tmap_o);
        for (int i = 0; i < p.num_stages; ++i) {
            ptx::mbar_init(ptx::smem_u32(full_bar + i), kStemR ? 129 : 1);   // stem: 128 gathering threads + the weight load
            ptx::mbar_init(ptx::smem_u32(empty_bar + i), 8);   // one arrive per consumer warp
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    ptx::pdl_wait();   // everything above overlapped the previous kernel's tail; its results are visible from here on

    if constexpr (kStemR > 0) {
        if (wg == 0) {
            // ===================== u8 patch gather (one pixel row of the A tile per thread) + weight TMA =====================
            const int row = threadIdx.x;
            const int total_px = p.Nb * p.H * p.W;
            // two counters rather than a RingPos: with the struct, ptxas gives conv_wgmma_kernel<__half, 96, false, 3> two more registers
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const ConvTile t = decode_tile(p, tile, n_tiles_g);
                const int px = t.p0 + row;
                const PixelPos q = unflatten(p, px < total_px ? px : 0);
                const int h0 = q.h * p.stem_stride - p.stem_pad_h, w0 = q.w * p.stem_stride - p.stem_pad_w;
                for (int c = 0; c < chunks; ++c) {
                    ptx::mbar_wait(ptx::smem_u32(empty_bar + stage), phase ^ 1);
                    const uint32_t fb = ptx::smem_u32(full_bar + stage);
                    uint8_t* sa = smem + (size_t)stage * STAGE_BYTES;
                    if (row == 0) {
                        ptx::mbar_expect_tx(fb, (uint32_t)(BN * 128));
                        ptx::tma_load_2d(ptx::smem_u32(sa + CONV_A_BYTES), &tmap_b, fb, c * BK, t.g * p.cout_g_pad + t.n0);
                    }
                    uint4* o = (uint4*)(sa + row * 128);
                    if (px >= total_px) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) o[i] = make_uint4(0u, 0u, 0u, 0u);
                    } else if (c == 0) {
                        im2col_chunk<true, kStemR, 0>(p.frames, o, row & 7, q.n, h0, w0, p.in_h, p.in_w, p.factor, p.flip, p.mean);
                    } else if (c == 1) {
                        im2col_chunk<true, kStemR, 1>(p.frames, o, row & 7, q.n, h0, w0, p.in_h, p.in_w, p.factor, p.flip, p.mean);
                    } else {
                        im2col_chunk<true, kStemR, 2>(p.frames, o, row & 7, q.n, h0, w0, p.in_h, p.in_w, p.factor, p.flip, p.mean);
                    }
                    ptx::fence_proxy_async();   // generic-proxy shared-memory writes -> visible to wgmma
                    ptx::mbar_arrive(fb);
                    if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
                }
            }
            return;
        }
    }
    if (wg == 0) {
        // ===================== TMA producer =====================
        if (warp == 0 && ptx::elect_one()) {
            RingPos ring;
            const int pad_h = p.R / 2, pad_w = p.S / 2;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const ConvTile t = decode_tile(p, tile, n_tiles_g);
                const PixelPos q0 = unflatten(p, t.p0);
                const int a_ch0 = p.in_ch_off + t.g * (kI8 ? p.in_g_stride : p.cin_g);
                const int b_row = t.g * p.cout_g_pad + t.n0;
                int kcol = 0;
                for (int r = 0; r < p.R; ++r)
                    for (int s = 0; s < p.S; ++s)
                        for (int c = 0; c < chunks; ++c, kcol += BK) {
                            ptx::mbar_wait(ptx::smem_u32(empty_bar + ring.slot), ring.phase ^ 1);
                            const uint32_t fb = ptx::smem_u32(full_bar + ring.slot);
                            uint8_t* sa = smem + (size_t)ring.slot * STAGE_BYTES;
                            ptx::mbar_expect_tx(fb, (uint32_t)STAGE_BYTES);
                            ptx::tma_load_im2col_4d(ptx::smem_u32(sa), &tmap_a, fb, a_ch0 + c * BK, q0.w - pad_w, q0.h - pad_h, q0.n, s, r);
                            ptx::tma_load_2d(ptx::smem_u32(sa + CONV_A_BYTES), &tmap_b, fb, kcol, b_row);
                            ring.step(p.num_stages);
                        }
            }
        }
        return;
    }

    // ===================== wgmma + epilogue (warpgroups 1, 2) =====================
    const int half = wg - 1;                                   // pixel rows [64 half, 64 half + 64) of every tile
    const int row0 = half * 64 + (warp & 3) * 16 + (lane >> 2); // accumulator rows row0 and row0 + 8 of this thread
    const int col0 = 2 * (lane & 3);                           // columns col0 + 8 j + {0, 1}
    const int total_px = p.Nb * p.H * p.W;
    const uint32_t smem0 = ptx::smem_u32(smem);
    const bool tma = kTmaForm && p.tma_store;
    typename ConvAcc<T>::type acc[BN / 2];
    RingPos ring;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const ConvTile t = decode_tile(p, tile, n_tiles_g);
        int prev = 0;
        for (int ks = 0; ks < ksteps; ++ks) {
            const uint32_t sa = smem0 + (uint32_t)(ring.slot * STAGE_BYTES);
            const uint64_t da = ptx::make_sw128_kmajor_desc(sa + (uint32_t)(half * 64 * 128)), db = ptx::make_sw128_kmajor_desc(sa + CONV_A_BYTES);
            ptx::mbar_wait(ptx::smem_u32(full_bar + ring.slot), ring.phase);
            ptx::fence_acc(acc);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)   // K advances by 32 bytes inside the 128-byte swizzled row: +2 in the (>>4) address field
                ptx::wgmma<T, BN>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (ks | k) != 0 ? 1u : 0u);
            ptx::wgmma_commit();
            ptx::fence_acc(acc);
            if (ks > 0) {   // the previous k-step's wgmma have retired: its stage goes back to the producer
                ptx::wgmma_wait<1>();
                if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(empty_bar + prev));
            }
            prev = ring.slot;
            ring.step(p.num_stages);
        }
        ptx::wgmma_wait<0>();
        ptx::fence_acc(acc);
        if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(empty_bar + prev));

        if constexpr (kTmaForm) {
            if (tma && t.p0 + half * 64 + 64 <= total_px) {   // (the tensor map spans max_batch frames: a block past the batch stays below)
                conv_epilogue_tma<BN, kRes>(acc, p, t, &tmap_o, ptx::smem_u32(s_stage + (size_t)half * BN * 128), half, warp, lane);
                continue;
            }
        }
        // epilogue: this thread holds rows row0 / row0 + 8, columns col0 + 8 j + {0, 1}: acc[4 j + 2 h + {0, 1}]
        const float* bias = p.bias + t.g * p.cout_g_pad + t.n0;
        const float* alpha = p.alpha + t.g * p.cout_g_pad + t.n0;
        const int n_valid = min(BN, p.cout_g - t.n0);   // real (unpadded) channels of this tile
        const int och = p.out_ch_off + t.g * p.cout_g + t.n0;
        const bool pair_ok = ((och | p.out_ld) & 1) == 0;   // two neighbouring channels form one aligned 4- / 8-byte store
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int px = t.p0 + row0 + 8 * h;
            if (px >= total_px) continue;
            const size_t pix = (size_t)px;
            const PixelPos q = unflatten(p, px);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int c = 8 * j + col0;
                if (c >= n_valid) break;
                if constexpr (kI8) {   // no FMA contraction anywhere: every product and sum is rounded on its own
                    const float* mul = p.mul + t.g * p.cout_g_pad + t.n0;
                    const bool two = c + 1 < n_valid;
                    float y[2], r[2] = { 0.f, 0.f };
                    if (kRes && p.res_mode) {
                        const size_t ri = pix * p.res_ld + p.res_ch_off + t.g * p.cout_g + t.n0 + c;
                        const char2 rq = *(const char2*)((const int8_t*)p.res + ri);
                        r[0] = __fmul_rn((float)rq.x, p.res_scale); r[1] = __fmul_rn((float)rq.y, p.res_scale);
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float v = __fadd_rn(__fmul_rn((float)acc[4 * j + 2 * h + e], __ldg(mul + c + e)), __ldg(bias + c + e));
                        if (kRes && p.res_mode == 1) v = __fadd_rn(v, r[e]);
                        v = v > 0.f ? v : __fmul_rn(v, __ldg(alpha + c + e));
                        if (kRes && p.res_mode == 2) v = __fadd_rn(v, r[e]);
                        y[e] = v;
                    }
                    if (p.out_mode == OUT_F16_NHWC) {
                        int8_t* o = (int8_t*)p.out + pix * p.out_ld + och + c;
                        const int8_t q0 = quantize_i8(y[0], p.out_inv_scale), q1 = quantize_i8(y[1], p.out_inv_scale);
                        if (two && pair_ok) *(char2*)o = make_char2(q0, q1);
                        else { o[0] = q0; if (two) o[1] = q1; }
                    } else {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            if (e == 1 && !two) break;
                            const int ch = t.n0 + c + e;
                            if (ch < p.split) {
                                ((float*)p.out)[(((size_t)q.n * p.split + ch) * p.H + q.h) * p.W + q.w] = y[e];
                            } else {
                                const int c2 = ch - p.split, n2 = p.cout_g - p.split;
                                ((float*)p.out2)[(((size_t)q.n * n2 + c2) * p.H + q.h) * p.W + q.w] = y[e];
                            }
                        }
                    }
                    continue;
                }
                float a0 = acc[4 * j + 2 * h] + __ldg(bias + c), a1 = acc[4 * j + 2 * h + 1] + __ldg(bias + c + 1);
                float r0 = 0.f, r1 = 0.f;
                if (kRes && p.res_mode) {   // (residual layers: cout_g % 16 == 0, so both channels exist and the pair is aligned)
                    const size_t ri = pix * p.res_ld + p.res_ch_off + t.g * p.cout_g + t.n0 + c;
                    if constexpr (kF16) { const float2 rf = __half22float2(*((const __half2*)p.res + ri / 2)); r0 = rf.x; r1 = rf.y; }
                    else { const float2 rf = *(const float2*)((const float*)p.res + ri); r0 = rf.x; r1 = rf.y; }
                }
                if (kRes && p.res_mode == 1) { a0 += r0; a1 += r1; }
                a0 = a0 > 0.f ? a0 : a0 * __ldg(alpha + c);
                a1 = a1 > 0.f ? a1 : a1 * __ldg(alpha + c + 1);
                if (kRes && p.res_mode == 2) { a0 += r0; a1 += r1; }
                const bool two = c + 1 < n_valid;
                if (p.out_mode == OUT_F16_NHWC) {
                    if constexpr (kF16) {
                        __half2 h2 = __floats2half2_rn(a0, a1);
                        if (p.post_w) {   // the fused 1x1 depthwise stage with dwconv_kernel<1, 1>'s arithmetic: fp16(act(x * w + b))
                            const int pc = t.g * p.cout_g + t.n0 + c;
                            const float2 x = __half22float2(h2);
                            float y0 = fmaf(x.x, __ldg(p.post_w + pc), 0.f) + __ldg(p.post_b + pc);
                            float y1 = two ? fmaf(x.y, __ldg(p.post_w + pc + 1), 0.f) + __ldg(p.post_b + pc + 1) : 0.f;
                            y0 = y0 > 0.f ? y0 : y0 * __ldg(p.post_a + pc);
                            if (two) y1 = y1 > 0.f ? y1 : y1 * __ldg(p.post_a + pc + 1);
                            h2 = __floats2half2_rn(y0, y1);
                        }
                        __half* o = (__half*)p.out + pix * p.out_ld + och + c;
                        if (two && pair_ok) *(__half2*)o = h2;
                        else { o[0] = __low2half(h2); if (two) o[1] = __high2half(h2); }
                    } else {
                        float* o = (float*)p.out + pix * p.out_ld + och + c;
                        const float y0 = ptx::round_tf32(a0), y1 = ptx::round_tf32(a1);
                        if (two && pair_ok) *(float2*)o = make_float2(y0, y1);
                        else { o[0] = y0; if (two) o[1] = y1; }
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (e == 1 && !two) break;
                        const int ch = t.n0 + c + e;
                        const float y = e ? a1 : a0;
                        if (ch < p.split) {
                            ((float*)p.out)[(((size_t)q.n * p.split + ch) * p.H + q.h) * p.W + q.w] = y;
                        } else {
                            const int c2 = ch - p.split, n2 = p.cout_g - p.split;
                            ((float*)p.out2)[(((size_t)q.n * n2 + c2) * p.H + q.h) * p.W + q.w] = y;
                        }
                    }
                }
            }
        }
    }
    if (tma && (threadIdx.x & 127) == 0) ptx::bulk_wait<0>();   // every store has completed before the CTA exits (the next kernel reads them)
}

constexpr size_t CONV_SMEM_FIXED = 1024 /*base alignment*/ + 2 * CONV_MAX_STAGES * 8;
// conv_wgmma_kernel's dynamic shared memory: alignment, the A/B ring, with tma_store the two consumer warpgroups' staging slots
// (BN x 128 B each), and the barriers
inline size_t conv_smem_bytes(int BN, int stages, bool tma_store)
{
    return CONV_SMEM_FIXED + (size_t)stages * (CONV_A_BYTES + BN * 128) + (tma_store ? 2 * (size_t)BN * 128 : 0);
}
// as many stages as fit, up to CONV_MAX_STAGES
inline int conv_pick_stages(int BN, bool tma_store)
{
    int s = CONV_MAX_STAGES;
    while (s > 2 && conv_smem_bytes(BN, s, tma_store) > CONV_SMEM_LIMIT) --s;
    return s;
}

// ---------------------------------------------------------------------------------------------
// Halo-box variant for RxS convolutions on large images (the early VGG layers).
// conv_wgmma_kernel fetches the A operand once PER FILTER TAP: a 3x3 layer pulls every input pixel nine times from L2 into shared
// memory.  Here a work item is a SPATIAL tile of 16 rows x 8 columns of output pixels (= the 128 accumulator rows; warpgroup 1 takes
// tile rows 0-7, warpgroup 2 rows 8-15).  Per 64-channel chunk ONE tiled-mode TMA load brings the (16+R-1) x (8+S-1) pixel halo box
// (out-of-image pixels zero-filled = "SAME" padding) into a 128B-swizzled buffer, and every filter tap (r, s) multiplies straight out
// of it: the A descriptor starts at the box address + ((row0 + r) * box_width + s) * 128 B, with a stride byte offset of one box row
// (box_width * 128 B) between the 8-pixel row groups; such a start is not 1024-byte aligned, which the address-based 128B swizzle
// reads back exactly as the TMA wrote it.  A traffic drops from R*S x 16 KiB to one 22.5 KiB box per chunk
// (3x3: 6.4x less); the weights stream through their own ring, one BN x 64 tile per (tap, chunk).
// kPool: the 2x2 / stride-2 max-pool that follows the layer is taken in the epilogue, so the un-pooled activation is never written.
// Accumulator rows m and m + 8 of a thread are pixels (y, x) and (y + 1, x) with y even, and lane ^ 4 holds (y, x ^ 1): the window
// maximum is taken on the raw fp32 accumulators BEFORE bias / activation / rounding -- all three are monotone (slopes >= 0 are
// required), so fp16(act(max(v) + b)) == max(fp16(act(v + b))) bit for bit.
// ---------------------------------------------------------------------------------------------
constexpr int HALO_TH = 16, HALO_TW = 8;

// The wide item (HaloItem::Wide): a work item is TWO consecutive 16 x 8 tiles of the same grid (tiles 2i and 2i + 1 in (image, ty, tx) order, each with its
// own halo box, so a pair may straddle two rows or two frames) x one n-tile.  Warpgroup 1 computes all 128 pixels of the first tile,
// warpgroup 2 those of the second (two m64 accumulator blocks each: tile rows 0-7 and 8-15), and both read the same weight stage: one
// 16 KiB weight tile, one full-barrier wait and one release serve 256 x 128 x 64 MACs instead of 128 x 128 x 64.  Every accumulator
// row sees the same wgmma sequence (chunk, tap, k16) as in the 128-pixel item, so the outputs are identical.  128 fp32 accumulators
// per consumer thread need more than the 168 registers of an even 384-thread split: setmaxnreg moves registers from the producer
// warpgroup (40) to the consumers (232).  With an odd tile count the last item's second tile lies past the batch: its box is loaded
// (out-of-tensor rows are zero-filled, or a frame beyond N of the max-batch buffer) and computed, and its epilogue is skipped.
constexpr int HALO_WIDE_PRODUCER_REGS = 40, HALO_WIDE_CONSUMER_REGS = 232;

// The ping-pong item (HaloItem::PingPong, 3x3 layers): a work item is one 16 x 8 tile x one n-tile, as in the 128-pixel item, but ONE warpgroup computes
// all of it (two m64 blocks, tile rows 0-7 and 8-15, the same accumulators and register split as the wide item).  A CTA's items
// alternate between warpgroups 1 and 2, and both consume the producer's box and weight rings in the CTA's item order.  Two turn
// barriers pass the tensor pipe back and forth: a warpgroup starts an item's MMAs once the other has ISSUED (not finished) its
// previous item's, so the pipe does not drain at the hand-off, and each warpgroup's final wait and epilogue run under the other's
// main loop.  Within an item nothing drains at a chunk boundary: box c is released after the first wait<1> of chunk c + 1, which
// has seen every MMA of chunk c complete; the box ring's four slots keep the producer a chunk ahead.  Every accumulator row sees
// the same (chunk, tap, k16) wgmma sequence as in the 128-pixel item, so the outputs are identical.

#ifdef HPB_HALO_PHASES
// instrumented build (tools/halo_phases.py): clock64 cycles of every consumer warpgroup, summed over the CTAs of all halo launches.
// HALO_PH_EPILOGUE: accumulators -> output (registers -> global, or -> the staging buffer and the TMA store's issue);
// HALO_PH_STAGE_WAIT: waiting for the staging buffer's previous TMA store to have read it
enum { HALO_PH_TOTAL, HALO_PH_A_WAIT, HALO_PH_B_WAIT, HALO_PH_MMA_WAIT, HALO_PH_EPILOGUE, HALO_PH_TURN_WAIT, HALO_PH_STAGE_WAIT, HALO_PH_COUNT };
__device__ unsigned long long g_halo_phases[HALO_PH_COUNT];
#define HALO_PH_MARK(t) const long long t = clock64()
#define HALO_TIMED(i, ...) do { const long long t0_ = clock64(); __VA_ARGS__; ph[i] += clock64() - t0_; } while (0)
#define HALO_PH_ADD(i, t) (ph[i] += clock64() - (t))
#define HALO_PH_PARAM , long long (&ph)[HALO_PH_COUNT]
#define HALO_PH_ARG , ph
#else
#define HALO_PH_MARK(t) do {} while (0)
#define HALO_TIMED(i, ...) do { __VA_ARGS__; } while (0)
#define HALO_PH_ADD(i, t) do {} while (0)
#define HALO_PH_PARAM
#define HALO_PH_ARG
#endif

struct HaloParams {
    int Nb, H, W;
    int R, S, groups, cin_g;
    int cout_g, cout_g_pad;
    int in_ch_off;
    int tiles_x, tiles_y;
    int box_bytes;              // one tile's box: (16+R-1) * (8+S-1) * 128 rounded up to a multiple of 1024
    int num_stages;             // weight ring depth
    const float* bias; const float* alpha;
    __half* out; int out_ld, out_ch_off;   // NHWC output (kPool: the pooled tensor, [Nb, H/2, W/2, out_ld])
    int tma_store;              // 1: the epilogue stages the fp16 tile in shared memory and TMA-stores it (halo_epilogue_tma)
    int stage_bytes;            // tma_store: each consumer warpgroup's staging region (halo_stage_bytes; 0 on the wide item)
};

// the work item of conv_halo_kernel: one 16 x 8 tile on both consumer warpgroups (the 128-pixel item), two tiles (Wide), or one tile
// on one warpgroup (PingPong)
enum class HaloItem { Narrow, Wide, PingPong };
// What an item is made of.  The kernel's loops and shared-memory layout and the host's sizing of that memory all read it from here.
struct HaloShape {
    int tiles;         // 16 x 8 tiles per item = halo boxes per box slot
    int blocks;        // m64 accumulator blocks per consumer warpgroup
    int box_slots;     // box ring depth
    int slot_warps;    // consumer warps that read (and release) one box slot / weight stage
    int stage_slots;   // staging slots of one consumer warpgroup for the TMA-store epilogue, BN x 128 B each (one m64 block)
    bool move_regs;    // setmaxnreg moves registers from the producer warpgroup to the consumers (HALO_WIDE_*_REGS)
};
// The wide item stages its two blocks in its own box of the item's last chunk, so it has no staging slots; the ping-pong item at
// BN = 128 stores its two blocks through one 16 KiB slot in turn (a full 32 KiB per warpgroup would cost two more of its weight stages).
__host__ __device__ constexpr HaloShape halo_shape(HaloItem it, int BN)
{
    return it == HaloItem::Wide       ? HaloShape{ 2, 2, 2, 8, 0, true }
           : it == HaloItem::PingPong ? HaloShape{ 1, 2, 4, 4, BN == 64 ? 2 : 1, true }
                                      : HaloShape{ 1, 1, 2, 8, 1, false };
}
inline int halo_stage_bytes(int BN, HaloItem it) { return halo_shape(it, BN).stage_slots * BN * 128; }

namespace ptx {
// K-major 128B-swizzled operand whose 8-row groups are `sbo` bytes apart and whose start need not be 1024-byte aligned.  The swizzle
// is a function of the absolute shared-memory address (as for the TMA that wrote the box), so the base-offset field stays 0: setting
// it to the start's phase ((address >> 7) & 7) reads the wrong 16-byte chunks (measured on H100).
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc_at(uint32_t smem_addr, uint32_t sbo)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffffu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)((sbo >> 4) & 0x3fffu) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3)
{
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(m), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
} // namespace ptx

// Stores m64 blocks 0 .. kBlocks - 1 of one warpgroup's accumulators: block m holds tile rows row_base + 8 m .. row_base + 8 m + 7 of
// the tile at (n, y0, x0).  kPool: the 2x2 max-pool of each block (its rows pair up as (y, y + 1) with y even, see above).
template <int BN, bool kPool, int kBlocks>
__device__ __forceinline__ void halo_epilogue(const float (&acc)[kBlocks][BN / 2], const HaloParams& p, int n, int y0, int x0, int g, int n0,
                                              int row_base, int warp, int lane)
{
    const int col0 = 2 * (lane & 3);
    const int tx = lane >> 2;                    // tile column of this thread's pixels
    const float* bias = p.bias + g * p.cout_g_pad + n0;
    const float* alpha = p.alpha + g * p.cout_g_pad + n0;
    const int och = p.out_ch_off + g * p.cout_g + n0;
    const bool pair_ok = ((och | p.out_ld) & 1) == 0;
    if constexpr (kPool) {
#pragma unroll
        for (int m = 0; m < kBlocks; ++m) {
            const int ty0 = row_base + m * 8 + (warp & 3) * 2;   // tile row of accumulator row 0 of this thread (row 8: ty0 + 1)
            const float (&acc0)[BN / 2] = acc[m];
            // rows ty0 / ty0 + 1 of this thread, then the column partner lane ^ 4; lanes with an even tile column store the pooled pixel
            const int py = (y0 + ty0) >> 1, px = (x0 + tx) >> 1;
            const bool store = (tx & 1) == 0 && py < (p.H >> 1) && px < (p.W >> 1);
            __half* o = p.out + (((size_t)n * (p.H >> 1) + py) * (p.W >> 1) + px) * p.out_ld + och;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                float v0 = fmaxf(acc0[4 * j], acc0[4 * j + 2]), v1 = fmaxf(acc0[4 * j + 1], acc0[4 * j + 3]);
                v0 = fmaxf(v0, __shfl_xor_sync(0xffffffffu, v0, 4));
                v1 = fmaxf(v1, __shfl_xor_sync(0xffffffffu, v1, 4));
                const int c = 8 * j + col0;
                if (!store) continue;
                float a0 = v0 + __ldg(bias + c), a1 = v1 + __ldg(bias + c + 1);
                a0 = a0 > 0.f ? a0 : a0 * __ldg(alpha + c);
                a1 = a1 > 0.f ? a1 : a1 * __ldg(alpha + c + 1);
                const __half2 h2 = __floats2half2_rn(a0, a1);
                if (pair_ok) *(__half2*)(o + c) = h2;
                else { o[c] = __low2half(h2); o[c + 1] = __high2half(h2); }
            }
        }
    } else {
        const int n_valid = min(BN, p.cout_g - n0);
#pragma unroll
        for (int m = 0; m < kBlocks; ++m) {
            const int ty0 = row_base + m * 8 + (warp & 3) * 2;   // tile row of accumulator row 0 of this thread (row 8: ty0 + 1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int oy = y0 + ty0 + h, ox = x0 + tx;
                if (oy >= p.H || ox >= p.W) continue;
                __half* o = p.out + (((size_t)n * p.H + oy) * p.W + ox) * p.out_ld + och;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = 8 * j + col0;
                    if (c >= n_valid) break;
                    float a0 = acc[m][4 * j + 2 * h] + __ldg(bias + c), a1 = acc[m][4 * j + 2 * h + 1] + __ldg(bias + c + 1);
                    a0 = a0 > 0.f ? a0 : a0 * __ldg(alpha + c);
                    a1 = a1 > 0.f ? a1 : a1 * __ldg(alpha + c + 1);
                    const __half2 h2 = __floats2half2_rn(a0, a1);
                    const bool two = c + 1 < n_valid;
                    if (two && pair_ok) *(__half2*)(o + c) = h2;
                    else { o[c] = __low2half(h2); if (two) o[c + 1] = __high2half(h2); }
                }
            }
        }
    }
}

// halo_epilogue with the same fp32 arithmetic, written through shared memory: block m's fp16 outputs go into staging slot m % kSlots
// (BN / 64 slices of {64 channels x 8 x 8 pixels}, pooled {64 x 4 x 4}, each in the 128B-swizzled layout of one TMA box: pixel row q,
// 16-byte chunk j at q * 128 + ((j ^ q % 8) * 16)), and the warpgroup's leader thread stores each slice with one TMA box of tmap_o and
// commits one bulk group per block.  The tensor map clips what lies past the image's right / bottom edge (or the floor-pooled map)
// and past the layer's last channel.  kWait: before a slot is written again, the leader waits until the group that read it last is
// done reading (the wide item stages into its own box instead, which its caller hands back to the producer once that store has read it).
template <int BN, bool kPool, int kBlocks, int kSlots, bool kWait>
__device__ __forceinline__ void halo_epilogue_tma(const float (&acc)[kBlocks][BN / 2], const HaloParams& p, const CUtensorMap* tmap_o, uint32_t stage,
                                                  int n, int y0, int x0, int g, int n0, int row_base, int warp, int lane, bool leader HALO_PH_PARAM)
{
    static_assert(BN == 64 || BN == 128, "one TMA box per 64-channel slice, at most two");
    constexpr int kSliceBytes = (kPool ? 16 : 64) * 128;
    constexpr int kSlotBytes = BN / 64 * kSliceBytes;
    const int col0 = 2 * (lane & 3);
    const float* bias = p.bias + g * p.cout_g_pad + n0;
    const float* alpha = p.alpha + g * p.cout_g_pad + n0;
    const int och = p.out_ch_off + g * p.cout_g + n0;
    const int bar_id = warp >> 2;   // named barrier 1 / 2: consumer warpgroup 1 / 2
#pragma unroll
    for (int m = 0; m < kBlocks; ++m) {
        const uint32_t slot = stage + (uint32_t)((m % kSlots) * kSlotBytes);
        HALO_PH_MARK(t_wait);
        if (kWait && leader) ptx::bulk_wait_read<kSlots - 1>();
        ptx::named_barrier_sync(bar_id, 128);   // the slot is free, and the whole warpgroup is past its last wgmma
#ifdef HPB_HALO_PHASES
        { const long long d = clock64() - t_wait; ph[HALO_PH_STAGE_WAIT] += d; ph[HALO_PH_EPILOGUE] -= d; }
#endif
        const int ty0 = row_base + m * 8;   // tile row of the block's first pixel row
        if constexpr (kPool) {
            // the pooled pixel of this thread's rows (ty0 + 2 (warp % 4), + 1) and columns (tx, tx ^ 1): slot row (warp % 4) * 4 + tx / 2
            const int q = (warp & 3) * 4 + (lane >> 3);
            const bool store = ((lane >> 2) & 1) == 0;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                float v0 = fmaxf(acc[m][4 * j], acc[m][4 * j + 2]), v1 = fmaxf(acc[m][4 * j + 1], acc[m][4 * j + 3]);
                v0 = fmaxf(v0, __shfl_xor_sync(0xffffffffu, v0, 4));
                v1 = fmaxf(v1, __shfl_xor_sync(0xffffffffu, v1, 4));
                if (!store) continue;
                const int c = 8 * j + col0;
                const float2 b = __ldg((const float2*)(bias + c)), a = __ldg((const float2*)(alpha + c));
                float a0 = v0 + b.x, a1 = v1 + b.y;
                a0 = a0 > 0.f ? a0 : a0 * a.x;
                a1 = a1 > 0.f ? a1 : a1 * a.y;
                ptx::st_shared_u32(slot + (uint32_t)((j >> 3) * kSliceBytes + q * 128 + (((j & 7) ^ (q & 7)) << 4) + (lane & 3) * 4),
                                   ptx::half2_bits(__floats2half2_rn(a0, a1)));
            }
        } else {
            // stmatrix: register i of a thread holds rows lane / 4 (+ 8 h) and channels 8 (4 jb + i) + col0 + {0, 1}; lane 8 i + r
            // addresses pixel row r of matrix i, so (row % 8) == r
            const int r = lane & 7, i = lane >> 3;
#pragma unroll
            for (int jb = 0; jb < BN / 32; ++jb) {
                float2 b[4], a[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int c = 8 * (4 * jb + k) + col0;
                    b[k] = __ldg((const float2*)(bias + c));
                    a[k] = __ldg((const float2*)(alpha + c));
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    uint32_t v[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float a0 = acc[m][4 * (4 * jb + k) + 2 * h] + b[k].x, a1 = acc[m][4 * (4 * jb + k) + 2 * h + 1] + b[k].y;
                        a0 = a0 > 0.f ? a0 : a0 * a[k].x;
                        a1 = a1 > 0.f ? a1 : a1 * a[k].y;
                        v[k] = ptx::half2_bits(__floats2half2_rn(a0, a1));
                    }
                    const int j = 4 * jb + i, row = (warp & 3) * 16 + 8 * h + r;
                    ptx::stmatrix_x4(slot + (uint32_t)((j >> 3) * kSliceBytes + row * 128 + (((j & 7) ^ r) << 4)), v[0], v[1], v[2], v[3]);
                }
            }
        }
        ptx::fence_proxy_async();   // the generic-proxy writes -> visible to the TMA store
        ptx::named_barrier_sync(bar_id, 128);
        if (leader) {
            const int x = kPool ? x0 >> 1 : x0, y = kPool ? (y0 + ty0) >> 1 : y0 + ty0;
            ptx::tma_store_4d(tmap_o, slot, och, x, y, n);
            if (BN == 128 && n0 + 64 < p.cout_g)   // (not a slice of padding channels only)
                ptx::tma_store_4d(tmap_o, slot + (uint32_t)kSliceBytes, och + 64, x, y, n);
            ptx::bulk_commit();
        }
    }
}

// One k-step (chunk, tap (r, s)) of a consumer warpgroup: m64 block m, the tile rows 8 m .. 8 m + 7 below the box row at `abase`,
// times the weight tile in slot b.slot of the ring, once that slot's full barrier has completed phase b.phase.  The first k-step of
// an item (c | tap == 0) overwrites the accumulators.
template <int BN, int kBlocks>
__device__ __forceinline__ void halo_kstep(float (&acc)[kBlocks][BN / 2], uint32_t abase, int r, int s, int BW, uint32_t sbo, const uint8_t* s_b,
                                           uint64_t* b_full, RingPos b, int c_or_tap HALO_PH_PARAM)
{
    uint64_t da[kBlocks];
#pragma unroll
    for (int m = 0; m < kBlocks; ++m) da[m] = ptx::make_sw128_kmajor_desc_at(abase + (uint32_t)(((m * 8 + r) * BW + s) * 128), sbo);
    const uint64_t db = ptx::make_sw128_kmajor_desc(ptx::smem_u32(s_b + (size_t)b.slot * BN * 128));
    HALO_TIMED(HALO_PH_B_WAIT, ptx::mbar_wait(ptx::smem_u32(b_full + b.slot), b.phase));
#pragma unroll
    for (int m = 0; m < kBlocks; ++m) ptx::fence_acc(acc[m]);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int m = 0; m < kBlocks; ++m)
            ptx::wgmma<__half, BN>(acc[m], da[m] + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (c_or_tap | k) != 0 ? 1u : 0u);
    ptx::wgmma_commit();
#pragma unroll
    for (int m = 0; m < kBlocks; ++m) ptx::fence_acc(acc[m]);
}

// The epilogue of one warpgroup's share of an item: with `tma` (p.tma_store, at a width with a TMA form) halo_epilogue_tma through
// the staging slots at `stage`, else halo_epilogue from registers.  The wide item's `stage` is its own box of the item's last chunk:
// a 7x7 box (39 KiB) holds both m64 blocks at once, a smaller one (3x3: 23 KiB) one block at a time.
template <int BN, bool kPool, HaloItem kItem>
__device__ __forceinline__ void halo_store(const float (&acc)[halo_shape(kItem, BN).blocks][BN / 2], const HaloParams& p, const CUtensorMap* tmap_o,
                                           bool tma, uint32_t stage, int n, int y0, int x0, int g, int n0, int row_base, int warp, int lane,
                                           bool leader HALO_PH_PARAM)
{
    constexpr HaloShape kShape = halo_shape(kItem, BN);
    if constexpr (BN % 64 == 0) {
        if (tma) {
            if constexpr (kItem != HaloItem::Wide)
                halo_epilogue_tma<BN, kPool, kShape.blocks, kShape.stage_slots, true>(acc, p, tmap_o, stage, n, y0, x0, g, n0, row_base, warp, lane,
                                                                                     leader HALO_PH_ARG);
            else if (p.box_bytes >= kShape.blocks * BN * 128)
                halo_epilogue_tma<BN, kPool, kShape.blocks, kShape.blocks, false>(acc, p, tmap_o, stage, n, y0, x0, g, n0, row_base, warp, lane,
                                                                                 leader HALO_PH_ARG);
            else
                halo_epilogue_tma<BN, kPool, kShape.blocks, 1, true>(acc, p, tmap_o, stage, n, y0, x0, g, n0, row_base, warp, lane, leader HALO_PH_ARG);
            return;
        }
    }
    halo_epilogue<BN, kPool, kShape.blocks>(acc, p, n, y0, x0, g, n0, row_base, warp, lane);
}

template <int BN, bool kPool, HaloItem kItem>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_b, const __grid_constant__ CUtensorMap tmap_o,
                 const HaloParams p)
{
    static_assert(!(kItem == HaloItem::Wide && kPool), "the pooled epilogue pairs pixel rows of one m64 block; it has no wide form");
    static_assert(kItem != HaloItem::PingPong || BN == 64 || BN == 128, "the ping-pong item is built for the VGG trunk's widths, BN = 64 and 128");
    constexpr HaloShape kShape = halo_shape(kItem, BN);
    constexpr int B_BYTES = BN * 128;
    // the TMA-store epilogue (p.tma_store) exists for BN = 64 and 128; other widths always take halo_epilogue
    constexpr bool kTmaForm = BN % 64 == 0;
    extern __shared__ uint8_t smem_raw[];
    ptx::pdl_launch_dependents();
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* s_box = smem;                                                           // [box_slots][tiles][box_bytes]
    uint8_t* s_b = s_box + (size_t)kShape.box_slots * kShape.tiles * p.box_bytes;    // [num_stages][BN x 128 B]
    uint8_t* s_stage = s_b + (size_t)p.num_stages * B_BYTES;                         // [2][stage_bytes]: TMA-store staging per consumer warpgroup
    uint64_t* a_full = (uint64_t*)(s_stage + 2 * (size_t)p.stage_bytes);             // [box_slots]
    uint64_t* a_empty = a_full + kShape.box_slots;
    uint64_t* b_full = a_empty + kShape.box_slots;                                   // [CONV_MAX_STAGES]
    uint64_t* b_empty = b_full + CONV_MAX_STAGES;
    uint64_t* turn = b_empty + CONV_MAX_STAGES;                                      // ping-pong item: [2], warpgroup 1 + i may start its next item

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles_g = p.cout_g_pad / BN;
    const int nt_total = p.groups * n_tiles_g;
    const int sp_per_img = p.tiles_x * p.tiles_y;
    const int total_items = (p.Nb * sp_per_img + kShape.tiles - 1) / kShape.tiles * nt_total;
    const int chunks = p.cin_g / CONV_BLOCK_K;
    const int taps = p.R * p.S;
    const int BW = HALO_TW + p.S - 1, BH = HALO_TH + p.R - 1;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmap_x);
        ptx::prefetch_tmap(&tmap_b);
        if (kTmaForm && p.tma_store) ptx::prefetch_tmap(&tmap_o);
        for (int i = 0; i < kShape.box_slots; ++i) {
            ptx::mbar_init(ptx::smem_u32(a_full + i), 1);
            ptx::mbar_init(ptx::smem_u32(a_empty + i), kShape.slot_warps);   // one arrive per consumer warp that reads it
        }
        for (int i = 0; i < p.num_stages; ++i) {
            ptx::mbar_init(ptx::smem_u32(b_full + i), 1);
            ptx::mbar_init(ptx::smem_u32(b_empty + i), kShape.slot_warps);
        }
        if constexpr (kItem == HaloItem::PingPong) {
            ptx::mbar_init(ptx::smem_u32(turn), 4);       // one arrive per warp of the warpgroup that hands over
            ptx::mbar_init(ptx::smem_u32(turn + 1), 4);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    ptx::pdl_wait();

    // item -> (first spatial tile, group, n-tile); n-tiles vary fastest so that neighbouring CTAs share a halo box in L2
    auto decode = [&](int item, int& sp, int& g, int& n0) {
        const int nt = item % nt_total;
        sp = item / nt_total * kShape.tiles;
        g = nt / n_tiles_g;
        n0 = (nt - g * n_tiles_g) * BN;
    };
    // spatial tile -> (image, first output row, first output column)
    auto tile_pos = [&](int sp, int& n, int& y0, int& x0) {
        n = sp / sp_per_img;
        const int t = sp - n * sp_per_img;
        const int ty = t / p.tiles_x;
        y0 = ty * HALO_TH;
        x0 = (t - ty * p.tiles_x) * HALO_TW;
    };

#ifdef HPB_HALO_PHASES
    long long ph[HALO_PH_COUNT] = {};
    HALO_PH_MARK(t_start);
#endif
    RingPos a, b;   // box ring (a_full / a_empty), weight ring (b_full / b_empty)
    if (wg == 0) {
        if constexpr (kShape.move_regs) ptx::setmaxnreg_dec<HALO_WIDE_PRODUCER_REGS>();
        // ===================== TMA producer: kShape.tiles halo boxes per (item, chunk), one weight tile per (item, chunk, tap) =====================
        if (warp == 0 && ptx::elect_one()) {
            const int pad_h = p.R / 2, pad_w = p.S / 2;
            for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
                int sp, g, n0;
                decode(item, sp, g, n0);
                for (int c = 0; c < chunks; ++c) {
                    ptx::mbar_wait(ptx::smem_u32(a_empty + a.slot), a.phase ^ 1);
                    const uint32_t fa = ptx::smem_u32(a_full + a.slot);
                    ptx::mbar_expect_tx(fa, (uint32_t)(kShape.tiles * BH * BW * 128));
#pragma unroll
                    for (int t = 0; t < kShape.tiles; ++t) {
                        int n, y0, x0;
                        tile_pos(sp + t, n, y0, x0);
                        ptx::tma_load_4d(ptx::smem_u32(s_box + (size_t)(a.slot * kShape.tiles + t) * p.box_bytes), &tmap_x, fa,
                                         p.in_ch_off + g * p.cin_g + c * CONV_BLOCK_K, x0 - pad_w, y0 - pad_h, n);
                    }
                    a.step(kShape.box_slots);
                    for (int tap = 0; tap < taps; ++tap) {
                        ptx::mbar_wait(ptx::smem_u32(b_empty + b.slot), b.phase ^ 1);
                        const uint32_t fb = ptx::smem_u32(b_full + b.slot);
                        ptx::mbar_expect_tx(fb, (uint32_t)B_BYTES);
                        ptx::tma_load_2d(ptx::smem_u32(s_b + (size_t)b.slot * B_BYTES), &tmap_b, fb, tap * p.cin_g + c * CONV_BLOCK_K, g * p.cout_g_pad + n0);
                        b.step(p.num_stages);
                    }
                }
            }
        }
        return;
    }

    // ===================== wgmma + epilogue =====================
    // 128-pixel item: warpgroups 1, 2 take tile rows 8 half .. 8 half + 7 of the item's tile (one m64 block each).
    // wide item: warpgroup 1 + half takes tile `half` of the pair, m64 block m = its tile rows 8 m .. 8 m + 7.
    // ping-pong item: warpgroup 1 + half takes the CTA's items half, half + 2, ..., m64 block m = tile rows 8 m .. 8 m + 7.
    if constexpr (kShape.move_regs) ptx::setmaxnreg_inc<HALO_WIDE_CONSUMER_REGS>();
    const int half = wg - 1;
    const uint32_t sbo = (uint32_t)BW * 128u;
    const bool tma = kTmaForm && p.tma_store;
    const bool leader = (threadIdx.x & 127) == 0;   // issues (and waits for) the warpgroup's TMA stores
    const uint32_t stage = ptx::smem_u32(s_stage + (size_t)half * p.stage_bytes);
    float acc[kShape.blocks][BN / 2];
    if constexpr (kItem == HaloItem::PingPong) {
        const int item_stages = chunks * taps;
        if (half) {   // warpgroup 2 starts behind the CTA's first item
            a.advance(chunks, kShape.box_slots);
            b.advance(item_stages, p.num_stages);
        }
        for (int j = half, item = blockIdx.x + half * gridDim.x; item < total_items; j += 2, item += 2 * gridDim.x) {
            int sp, g, n0;
            decode(item, sp, g, n0);
            // the tensor pipe is ours once the other warpgroup has issued every MMA of item j - 1
            if (j > 0) HALO_TIMED(HALO_PH_TURN_WAIT, ptx::mbar_wait(ptx::smem_u32(turn + half), (uint32_t)((j - 1) >> 1) & 1u));
            int prev_st = 0, prev_bs = 0;
            for (int c = 0; c < chunks; ++c) {
                HALO_TIMED(HALO_PH_A_WAIT, ptx::mbar_wait(ptx::smem_u32(a_full + a.slot), a.phase));
                const uint32_t abase = ptx::smem_u32(s_box + (size_t)a.slot * p.box_bytes);
                for (int tap = 0; tap < taps; ++tap) {
                    const int r = tap / p.S, s = tap - r * p.S;
                    halo_kstep<BN, kShape.blocks>(acc, abase, r, s, BW, sbo, s_b, b_full, b, c | tap HALO_PH_ARG);
                    if ((c | tap) != 0) {
                        // the previous k-step's MMAs are done: its weight stage, and at a chunk's first tap the previous box, are free
                        HALO_TIMED(HALO_PH_MMA_WAIT, ptx::wgmma_wait<1>());
                        if (lane == 0) {
                            ptx::mbar_arrive(ptx::smem_u32(b_empty + prev_st));
                            if (tap == 0) ptx::mbar_arrive(ptx::smem_u32(a_empty + prev_bs));
                        }
                    }
                    prev_st = b.slot;
                    b.step(p.num_stages);
                }
                prev_bs = a.slot;
                a.step(kShape.box_slots);
            }
            if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(turn + (half ^ 1)));   // every MMA of item j is issued: hand over the pipe
            HALO_TIMED(HALO_PH_MMA_WAIT, ptx::wgmma_wait<0>());
#pragma unroll
            for (int m = 0; m < kShape.blocks; ++m) ptx::fence_acc(acc[m]);
            if (lane == 0) {
                ptx::mbar_arrive(ptx::smem_u32(b_empty + prev_st));
                ptx::mbar_arrive(ptx::smem_u32(a_empty + prev_bs));
            }
            a.advance(chunks, kShape.box_slots);   // item j + 1 is the other warpgroup's
            b.advance(item_stages, p.num_stages);
            HALO_PH_MARK(t_epi);
            int n, y0, x0;
            tile_pos(sp, n, y0, x0);
            halo_store<BN, kPool, kItem>(acc, p, &tmap_o, tma, stage, n, y0, x0, g, n0, 0, warp, lane, leader HALO_PH_ARG);
            HALO_PH_ADD(HALO_PH_EPILOGUE, t_epi);
        }
    } else {
        const int box = kItem == HaloItem::Wide ? half : 0;            // this warpgroup's box inside a box slot
        const int row_base = kItem == HaloItem::Wide ? 0 : half * 8;   // tile row of block 0's first accumulator row
        // wide item, TMA store: the box slot the leader has not released yet -- the previous item's last chunk, which holds its staged
        // tile until the store has read it (the producer's next load into it is a chunk away)
        int held = -1;
        for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
            int sp, g, n0;
            decode(item, sp, g, n0);
            for (int c = 0; c < chunks; ++c) {
                HALO_TIMED(HALO_PH_A_WAIT, ptx::mbar_wait(ptx::smem_u32(a_full + a.slot), a.phase));
                const uint32_t abase = ptx::smem_u32(s_box + (size_t)(a.slot * kShape.tiles + box) * p.box_bytes) + (uint32_t)(row_base * BW * 128);
                int prev = 0;
                for (int tap = 0; tap < taps; ++tap) {
                    const int r = tap / p.S, s = tap - r * p.S;
                    halo_kstep<BN, kShape.blocks>(acc, abase, r, s, BW, sbo, s_b, b_full, b, c | tap HALO_PH_ARG);
                    if (tap > 0) {
                        HALO_TIMED(HALO_PH_MMA_WAIT, ptx::wgmma_wait<1>());
                        if (lane == 0) ptx::mbar_arrive(ptx::smem_u32(b_empty + prev));
                    }
                    if (kItem == HaloItem::Wide && held >= 0 && tap == taps / 2) {
                        HALO_TIMED(HALO_PH_STAGE_WAIT, ptx::bulk_wait_read<0>());
                        ptx::mbar_arrive(ptx::smem_u32(a_empty + held));
                        held = -1;
                    }
                    prev = b.slot;
                    b.step(p.num_stages);
                }
                HALO_TIMED(HALO_PH_MMA_WAIT, ptx::wgmma_wait<0>());   // every tap of this chunk has read the box
#pragma unroll
                for (int m = 0; m < kShape.blocks; ++m) ptx::fence_acc(acc[m]);
                if (lane == 0) {
                    ptx::mbar_arrive(ptx::smem_u32(b_empty + prev));
                    if (kItem == HaloItem::Wide && tma && leader && c == chunks - 1) held = a.slot;   // this box stages the tile's outputs
                    else ptx::mbar_arrive(ptx::smem_u32(a_empty + a.slot));
                }
                a.step(kShape.box_slots);
            }

            HALO_PH_MARK(t_epi);
            int n, y0, x0;
            tile_pos(sp + box, n, y0, x0);
            if (kItem == HaloItem::Wide && n >= p.Nb) {   // the second tile of an odd tile count's last item
                if (held >= 0) { ptx::mbar_arrive(ptx::smem_u32(a_empty + held)); held = -1; }
                continue;
            }
            // the wide item stages its outputs in this warpgroup's box of the chunk just read, one ring position back
            const int last = (a.slot + kShape.box_slots - 1) % kShape.box_slots;
            const uint32_t dst = kItem == HaloItem::Wide ? ptx::smem_u32(s_box + (size_t)(last * kShape.tiles + box) * p.box_bytes) : stage;
            halo_store<BN, kPool, kItem>(acc, p, &tmap_o, tma, dst, n, y0, x0, g, n0, row_base, warp, lane, leader HALO_PH_ARG);
            HALO_PH_ADD(HALO_PH_EPILOGUE, t_epi);
        }
    }
    if (tma && leader) ptx::bulk_wait<0>();   // every store has completed before the CTA exits (the next kernel reads them)
#ifdef HPB_HALO_PHASES
    HALO_PH_ADD(HALO_PH_TOTAL, t_start);
    if ((threadIdx.x & 127) == 0)
        for (int i = 0; i < HALO_PH_COUNT; ++i) atomicAdd(g_halo_phases + i, (unsigned long long)ph[i]);
#endif
}

inline int halo_box_bytes(int R, int S) { return ((HALO_TH + R - 1) * (HALO_TW + S - 1) * 128 + 1023) & ~1023; }
// conv_halo_kernel's dynamic shared memory: alignment, box ring, weight ring, staging regions (with tma_store: halo_stage_bytes per
// consumer warpgroup) and barriers
inline size_t conv_halo_smem_bytes(int R, int S, int BN, int stages, HaloItem it, bool tma_store)
{
    const HaloShape sh = halo_shape(it, BN);
    return 1024 + (size_t)sh.box_slots * sh.tiles * halo_box_bytes(R, S) + (size_t)stages * BN * 128 +
           (tma_store ? 2 * (size_t)halo_stage_bytes(BN, it) : 0) + (2 * sh.box_slots + 2 * CONV_MAX_STAGES + 2) * 8;
}
// as many weight stages as fit, up to CONV_MAX_STAGES (at least 2: a caller that needs more checks the result)
inline int conv_halo_pick_stages(int R, int S, int BN, HaloItem it, bool tma_store)
{
    int s = CONV_MAX_STAGES;
    while (s > 2 && conv_halo_smem_bytes(R, S, BN, s, it, tma_store) > CONV_SMEM_LIMIT) --s;
    return s;
}

} // namespace hpb
