// paf_parser.cu -- H100 (sm_90a) PAF post-processing: conf/PAF tensors -> human_t records.
//
// Replaces the reference's CPU parser hyperpose::parser::paf
//   src/paf.cpp:57-375, src/post_process.hpp:26-205, src/coco.hpp:6-52
// with two batched CUDA kernels (grid covers every frame of the batch):
//
//   K1 paf_peaks_kernel    resize_area (post_process.hpp:26-52) + smooth (:54-69) + 3x3 max-pool NMS
//                          (:71-102) + peak scan (:175-192), fused per smem tile.  The 4x up-sampled maps
//                          are never written to HBM.  Tiles whose source values cannot reach conf_thresh
//                          are skipped (provably peak-free, see tile_can_skip()).
//   K2 paf_limbs_kernel    one CTA per (limb, frame): restores the reference's channel-major / row-major peak order and ids,
//                          get_connection_candidates + get_connections (paf.cpp:93-144, 234-272: 10 lanes per peak pair sample
//                          the PAF line integral -- up-sampling recomputed on the fly from the 1/8-resolution field staged in
//                          shared memory -- ballot/shuffle reductions, score-ordered greedy matching), and, in the last CTA of a
//                          frame to finish, get_humans (paf.cpp:146-232) + conversion (:359-372).
//
// Arithmetic contract (bit-exactness with oracle/paf_oracle.c): every fp32 operation on the result path
// is spelled with an explicit round-to-nearest intrinsic (__fmul_rn/__fadd_rn/__fmaf_rn/__fdiv_rn) in
// the order the oracle documents; the double-precision steps of the reference (paf.cpp:74,104,129) are
// done in double.  The file is additionally compiled with -fmad=false.
//
// No CPU fallback exists: every entry point fails with HP_ERR_CUDA when CUDA is unavailable.

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/hyperpose_b200.h"
#include "common.h"
#include "handoff.h"
#include "pair_math.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// topology (src/coco.hpp:10-52)
// ---------------------------------------------------------------------------------------------
__constant__ int c_pairs_net[HP_N_PAIRS][2] = {
    {12, 13}, {20, 21}, {14, 15}, {16, 17}, {22, 23}, {24, 25}, {0, 1}, {2, 3}, {4, 5}, {6, 7},
    {8, 9}, {10, 11}, {28, 29}, {30, 31}, {34, 35}, {32, 33}, {36, 37}, {18, 19}, {26, 27}};
__constant__ int c_pairs[HP_N_PAIRS][2] = {
    {1, 2}, {1, 5}, {2, 3}, {3, 4}, {5, 6}, {6, 7}, {1, 8}, {8, 9}, {9, 10}, {1, 11},
    {11, 12}, {12, 13}, {1, 0}, {0, 14}, {14, 16}, {0, 15}, {15, 17}, {2, 16}, {5, 17}};

// cv::getGaussianKernel(17, 3.0, CV_32F) (post_process.hpp:58,66-67; ksize 17 from paf.cpp:330-331):
// exp(-(i-8)^2/18) normalised in double, rounded to fp32.
__constant__ float c_g17[17] = {
    0x1.f41be6p-9f, 0x1.1faf48p-7f, 0x1.282c02p-6f, 0x1.10d854p-5f, 0x1.c1d86ep-5f,
    0x1.4bd66ep-4f, 0x1.b616fp-4f, 0x1.02c558p-3f, 0x1.118dcap-3f, 0x1.02c558p-3f,
    0x1.b616fp-4f, 0x1.4bd66ep-4f, 0x1.c1d86ep-5f, 0x1.10d854p-5f, 0x1.282c02p-6f,
    0x1.1faf48p-7f, 0x1.f41be6p-9f};

constexpr int THRESH_VECTOR_CNT1 = 8; // paf.cpp:57
constexpr int THRESH_PART_CNT = 4;    // paf.cpp:58
constexpr int STEP_PAF = 10;          // paf.cpp:60

enum : int { FLAG_PEAK_OVERFLOW = 1, FLAG_CAND_OVERFLOW = 2, FLAG_HUMAN_OVERFLOW = 4 };

// cv::borderInterpolate(BORDER_REFLECT_101)
__host__ __device__ inline int refl101(int p, int len)
{
    if ((unsigned)p < (unsigned)len) return p;
    if (len == 1) return 0;
    do {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    } while ((unsigned)p >= (unsigned)len);
    return p;
}

// ---------------------------------------------------------------------------------------------
// K1: fused up-sample + Gaussian + NMS + peak emission
// ---------------------------------------------------------------------------------------------
// The kernel is ISSUE-bound (~9.3k warp instructions per tile, 9504 tiles per 16-frame batch), so this
// version is organised around instruction count: the horizontal lerp of the up-sampling is computed once per SOURCE row (the
// default resolution stretches rows 7x: ~9 source rows feed 48 tile rows), both filter passes produce 16 outputs per thread
// from one 32-value register window (1 shared load per 8.5 FMAs), every pass is exactly one round of the 192-thread CTA, and
// the source bounds of a tile come from host tables instead of shared-memory atomics.
// Both filter passes work on float2 pairs (pair_math.cuh: each lane rounded exactly like the scalar instruction): the row pass pairs two ROWS (the up-sampled tile is
// stored as float2 {row 2r, row 2r+1}), the column pass pairs two COLUMNS (the row-pass output is row-major with an even stride).
constexpr int K1_THREADS = 192;
constexpr int TH = 30, TW = 62;          // interior tile of the up-map handled by one CTA
constexpr int HALO = 9;                  // 8 (17-tap blur) + 1 (3x3 NMS)
constexpr int UT_H = TH + 2 * HALO;      // 48 rows of up-sampled values (virtual = reflected coordinates)
constexpr int UT_W = TW + 2 * HALO;      // 80 cols
constexpr int UT_LD = UT_W + 1;          // 81: odd stride -> row-parallel accesses are conflict-free
constexpr int RT_W = TW + 2;             // 64 row-pass output columns (interior + 1 each side)
constexpr int RT_LD = RT_W + 2;          // 66: even, so that a column pair is one aligned 8-byte shared-memory access
constexpr int CT_H = TH + 2;             // 32 column-pass output rows
constexpr int SRC_MAX_H = UT_H + 1, SRC_MAX_W = UT_W + 1; // scale >= 1 => at most one source px per up px (+1)
constexpr int RUN = 8;                   // outputs per thread per pass and lane of the pair (sliding window of RUN+16 inputs)
constexpr int HL_ROWS = 16;              // source rows per tile for which the horizontal lerp is cached (more: direct path)
constexpr int SRC_COLS = 64;             // source columns per tile the (row mod 3, column) staging loop covers (more: generic loop)
static_assert(K1_THREADS % SRC_COLS == 0 && (SRC_COLS & (SRC_COLS - 1)) == 0, "source staging: thread = (row mod 3, column)");
static_assert(UT_H % 4 == 0 && 2 * UT_W <= K1_THREADS, "up-sampling: one (tile column, half of the row pairs) per thread");
static_assert(UT_H % 2 == 0 && (UT_H / 2) * (RT_W / RUN) == K1_THREADS, "row pass: one (row pair, run) per thread");
static_assert(RT_W % 2 == 0 && (RT_W / 2) * (CT_H / RUN) <= K1_THREADS && CT_H % RUN == 0, "column pass: one (column pair, run) per thread");

// up-sampled tile, rows paired: element (vy, vx) of the 48 x 80 tile
__device__ __forceinline__ float& tile_u(float2* sU2, int vy, int vx) { return reinterpret_cast<float*>(sU2 + (vy >> 1) * UT_LD + vx)[vy & 1]; }

struct PeakParams {
    const float* conf; // [N, c_conf, H, W]
    int c_conf, H, W, UH, UW;
    const int* xi; const float* xf; // [UW] area-upscale table
    const int* yi; const float* yf; // [UH]
    const int* tile_bounds;         // [tiles_y][2] source row lo/hi, then [tiles_x][2] source col lo/hi (host: tile_source_bounds)
    float thresh;
    float skip_below; // tiles whose source max is <= this cannot contain a peak; -inf disables skipping
    int tiles_x, tiles_y;
    int pcap;            // capacity per (frame, part)
    int* peak_cnt;       // [N,18]
    int* raw_key;        // [N,18,pcap]  y*UW + x
    float* raw_score;    // [N,18,pcap]
    int* flags;          // [N]
    int n8, n4;          // column classes of the separable filter (see oracle/paf_oracle.c)
    const float* up;     // kFromUp: resized maps [N, c_conf, UH, UW] written by resize_area_generic_kernel
};

// kFromUp = false: the default, fused path (resolution >= feature map on both axes: 2-tap area-mode up-sampling recomputed per tile).
// kFromUp = true : resolutions that SHRINK an axis (true INTER_AREA averaging, or the mixed regime): the resized maps were
//                  materialised by resize_area_generic_kernel and the tile is loaded from them (reflected coordinates).
template <bool kFromUp>
__global__ void __launch_bounds__(K1_THREADS) paf_peaks_kernel(const PeakParams p)
{
    // sSrc (dead after the up-sample) and sTmp (row-pass output) share storage.
    __shared__ float2 sU2[(UT_H / 2) * UT_LD];   // {row 2r, row 2r+1} per column
    __shared__ __align__(8) float sA[(SRC_MAX_H * SRC_MAX_W > UT_H * RT_LD) ? SRC_MAX_H * SRC_MAX_W : UT_H * RT_LD];
    __shared__ __align__(8) float sS[CT_H * RT_LD];
    __shared__ float sHl[HL_ROWS * UT_LD];   // horizontal lerp of the tile's source rows
    __shared__ int sXi[UT_W], sYi[UT_H];
    __shared__ float sXf[UT_W], sYf[UT_H];
    __shared__ int2 sYo[UT_H];
    __shared__ float sMax[K1_THREADS / 32];
    __shared__ int sSkip;

    const int tid = threadIdx.x;
    const int tx = blockIdx.x, ty = blockIdx.y / HP_N_PARTS;        // grid (tiles_x, tiles_y * 18, N): no run-time division
    const int part = blockIdx.y - ty * HP_N_PARTS, frame = blockIdx.z;
    const int x0 = tx * TW, y0 = ty * TH;
    const int H = p.H, W = p.W, UH = p.UH, UW = p.UW;
    const float* src = p.conf + ((size_t)frame * p.c_conf + part) * H * W;

    if (kFromUp) {
        const float* up = p.up + ((size_t)frame * p.c_conf + part) * UH * UW;
        float lmax = -INFINITY;
        for (int i = tid; i < UT_H * UT_W; i += K1_THREADS) {
            const int vy = i / UT_W, vx = i - vy * UT_W;
            const float v = __ldg(up + (size_t)refl101(y0 - HALO + vy, UH) * UW + refl101(x0 - HALO + vx, UW));
            tile_u(sU2, vy, vx) = v;
            lmax = fmaxf(lmax, v);
            if (v != v) lmax = INFINITY;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        if ((tid & 31) == 0) sMax[tid >> 5] = lmax;
        __syncthreads();
        if (tid == 0) {
            float m = sMax[0];
            for (int i = 1; i < K1_THREADS / 32; ++i) m = fmaxf(m, sMax[i]);
            sSkip = (m <= p.skip_below) ? 1 : 0;   // smoothed <= max of the window (1 + 3e-6): same bound as below
        }
        __syncthreads();
        if (sSkip) return;
    } else {
    // source rows / columns this tile's (reflected) rows and columns touch: precomputed on the host
    const int sr0 = __ldg(p.tile_bounds + 2 * ty), sr1 = __ldg(p.tile_bounds + 2 * ty + 1);
    const int sc0 = __ldg(p.tile_bounds + 2 * p.tiles_y + 2 * tx), sc1 = __ldg(p.tile_bounds + 2 * p.tiles_y + 2 * tx + 1);
    const int sh = sr1 - sr0 + 1, sw = sc1 - sc0 + 1; // <= SRC_MAX_H x SRC_MAX_W because UH >= H, UW >= W
    float* sSrc = sA;
    float lmax = -INFINITY;
    if (sw <= SRC_COLS) {   // thread = (row mod 3, column): no run-time division (the default resolutions: sw ~ 37)
        const int c = tid & (SRC_COLS - 1);
        if (c < sw)
            for (int r = tid / SRC_COLS; r < sh; r += K1_THREADS / SRC_COLS) {
                const float v = __ldg(src + (size_t)(sr0 + r) * W + sc0 + c);
                sSrc[r * sw + c] = v;
                lmax = fmaxf(lmax, v); // fmaxf ignores NaN: a NaN never enables the skip on its own
                if (v != v) lmax = INFINITY;
            }
    } else {
        for (int i = tid; i < sh * sw; i += K1_THREADS) {
            const int r = i / sw, c = i - r * sw;
            const float v = __ldg(src + (size_t)(sr0 + r) * W + sc0 + c);
            sSrc[i] = v;
            lmax = fmaxf(lmax, v);
            if (v != v) lmax = INFINITY;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    if ((tid & 31) == 0) sMax[tid >> 5] = lmax;
    // the coefficient tables of the (reflected) rows / columns this tile needs
    for (int i = tid; i < UT_W + UT_H; i += K1_THREADS) {
        if (i < UT_W) {
            const int rx = refl101(x0 - HALO + i, UW);
            sXi[i] = __ldg(p.xi + rx);
            sXf[i] = __ldg(p.xf + rx);
        } else {
            const int j = i - UT_W;
            const int ry = refl101(y0 - HALO + j, UH);
            const int sy0 = __ldg(p.yi + ry);
            sYi[j] = sy0;
            sYf[j] = __ldg(p.yf + ry);
            sYo[j] = make_int2((sy0 - sr0) * UT_LD, (min(sy0 + 1, H - 1) - sr0) * UT_LD);   // offsets into the cached horizontal lerp
        }
    }
    __syncthreads();
    if (tid == 0) {
        float m = sMax[0];
        for (int i = 1; i < K1_THREADS / 32; ++i) m = fmaxf(m, sMax[i]);
        // tile_can_skip: every smoothed value is a (rounded) convex combination of source values:
        //   |lerp| <= m(1+2^-22), two 17-tap passes with sum(k) <= 1+1.3e-8 and <= 34 roundings
        //   => smoothed <= m(1+3e-6) for m >= 0;  skip_below = thresh*(1-1e-5) keeps a 3x margin.
        sSkip = (m <= p.skip_below) ? 1 : 0;
    }
    __syncthreads();
    if (sSkip) return;

    // ---- up-sample into virtual (reflected) coordinates: sU[vy][vx] = up(refl(y0-9+vy), refl(x0-9+vx))
    //      HResizeLinear then VResizeLinear, products rounded separately (oracle orc_resize_area_up).
    //      The horizontal pass depends on the SOURCE row only: computed once per source row when few rows feed the tile.
    if (sh <= HL_ROWS) {
        for (int i = tid; i < sh * UT_W; i += K1_THREADS) {
            const int r = i / UT_W, vx = i - r * UT_W;
            const int sx0 = sXi[vx], sx1 = min(sx0 + 1, W - 1);
            const float a1 = sXf[vx], a0 = __fsub_rn(1.f, a1);
            const float* row = sSrc + r * sw - sc0;
            sHl[r * UT_LD + vx] = __fadd_rn(__fmul_rn(row[sx0], a0), __fmul_rn(row[sx1], a1));
        }
        __syncthreads();
        // vertical pass: a thread owns one tile column and walks down half of the row pairs; one packed 8-byte store per pair
        if (tid < 2 * UT_W) {
            const int vx = tid % UT_W, rp0 = (tid / UT_W) * (UT_H / 4);
            const float* col = sHl + vx;
#pragma unroll 4
            for (int rp = rp0; rp < rp0 + UT_H / 4; ++rp) {
                float2 o;
                {
                    const int2 so = sYo[2 * rp];
                    const float b1 = sYf[2 * rp], b0 = __fsub_rn(1.f, b1);
                    o.x = __fadd_rn(__fmul_rn(col[so.x], b0), __fmul_rn(col[so.y], b1));
                }
                {
                    const int2 so = sYo[2 * rp + 1];
                    const float b1 = sYf[2 * rp + 1], b0 = __fsub_rn(1.f, b1);
                    o.y = __fadd_rn(__fmul_rn(col[so.x], b0), __fmul_rn(col[so.y], b1));
                }
                sU2[rp * UT_LD + vx] = o;
            }
        }
    } else {
        for (int i = tid; i < UT_H * UT_W; i += K1_THREADS) {
            const int vy = i / UT_W, vx = i - vy * UT_W;
            const int sx0 = sXi[vx], sx1 = min(sx0 + 1, W - 1);
            const int sy0 = sYi[vy], sy1 = min(sy0 + 1, H - 1);
            const float a1 = sXf[vx], a0 = __fsub_rn(1.f, a1);
            const float b1 = sYf[vy], b0 = __fsub_rn(1.f, b1);
            const float* r0 = sSrc + (sy0 - sr0) * sw - sc0;
            const float* r1 = sSrc + (sy1 - sr0) * sw - sc0;
            const float h0 = __fadd_rn(__fmul_rn(r0[sx0], a0), __fmul_rn(r0[sx1], a1));
            const float h1 = __fadd_rn(__fmul_rn(r1[sx0], a0), __fmul_rn(r1[sx1], a1));
            tile_u(sU2, vy, vx) = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
        }
    }
    __syncthreads(); // sSrc is dead from here; sA becomes sTmp
    }

    // ---- row pass: sTmp[vy][c], c = 0..63 <-> real column j = x0 - 1 + c; taps left->right.
    //      work item = (row PAIR, run of 8 columns), one per thread: every packed instruction serves rows 2rp and 2rp+1.
    float* sTmp = sA;
    {
        const int rp = tid % (UT_H / 2), run = tid / (UT_H / 2);
        const int c0 = run * RUN;
        const float2* in = sU2 + rp * UT_LD + c0; // window input k for output c is in[c - c0 + k] (vx = c + k)
        float2 w[RUN + 16];
#pragma unroll
        for (int k = 0; k < RUN + 16; ++k) w[k] = in[k];
        const int jlast = x0 - 1 + c0 + RUN - 1;
        float2 acc[RUN];
        if (jlast < p.n4) {
            const float2 g0 = make_float2(c_g17[0], c_g17[0]);
#pragma unroll
            for (int o = 0; o < RUN; ++o) acc[o] = fmul2_rn(g0, w[o]);
#pragma unroll
            for (int t = 1; t < 17; ++t) {
                const float2 g = make_float2(c_g17[t], c_g17[t]);
#pragma unroll
                for (int o = 0; o < RUN; ++o) acc[o] = ffma2_rn(g, w[o + t], acc[o]);
            }
        } else {
#pragma unroll
            for (int o = 0; o < RUN; ++o) {
                const bool fma = (x0 - 1 + c0 + o) < p.n4;
                float2 s2 = fmul2_rn(make_float2(c_g17[0], c_g17[0]), w[o]);
#pragma unroll
                for (int t = 1; t < 17; ++t) {
                    const float2 g = make_float2(c_g17[t], c_g17[t]);
                    s2 = fma ? ffma2_rn(g, w[o + t], s2) : fadd2_rn(s2, fmul2_rn(g, w[o + t]));
                }
                acc[o] = s2;
            }
        }
#pragma unroll
        for (int o = 0; o < RUN; ++o) {
            sTmp[(2 * rp) * RT_LD + c0 + o] = acc[o].x;
            sTmp[(2 * rp + 1) * RT_LD + c0 + o] = acc[o].y;
        }
    }
    __syncthreads();

    // ---- column pass (symmetric): sS[r][c], r = 0..31 <-> real row i = y0 - 1 + r (virtual row r + 8).
    //      work item = (column PAIR c, c+1; run of 8 rows); the two columns can fall into different column classes of the
    //      reference's SIMD filter (FMA below n8, mul + add from n8 on): then both chains are computed and each lane keeps its own.
    if (tid < (RT_W / 2) * (CT_H / RUN)) {
        const int c = (tid % (RT_W / 2)) * 2, r0 = (tid / (RT_W / 2)) * RUN;
        const int j0 = x0 - 1 + c, j1 = j0 + 1;
        const bool fma0 = j0 < p.n8, fma1 = j1 < p.n8;
        float2 w[RUN + 16];
#pragma unroll
        for (int k = 0; k < RUN + 16; ++k) w[k] = *reinterpret_cast<const float2*>(sTmp + (r0 + k) * RT_LD + c);
        const float2 g8 = make_float2(c_g17[8], c_g17[8]);
        float2 res[RUN];
        // the whole tile lies in one column class almost always (CTA-uniform tests): one chain, taps outermost so that a
        // coefficient pair serves all RUN outputs
        const int jlo = x0 - 1, jhi = x0 - 1 + RT_W - 1;
        if (jhi < p.n8) {
#pragma unroll
            for (int o = 0; o < RUN; ++o) res[o] = fmul2_rn(g8, w[o + 8]);
#pragma unroll
            for (int t = 1; t <= 8; ++t) {
                const float2 g = make_float2(c_g17[8 + t], c_g17[8 + t]);
#pragma unroll
                for (int o = 0; o < RUN; ++o) res[o] = ffma2_rn(g, fadd2_rn(w[o + 8 + t], w[o + 8 - t]), res[o]);
            }
        } else if (jlo >= p.n8) {
#pragma unroll
            for (int o = 0; o < RUN; ++o) res[o] = fmul2_rn(g8, w[o + 8]);
#pragma unroll
            for (int t = 1; t <= 8; ++t) {
                const float2 g = make_float2(c_g17[8 + t], c_g17[8 + t]);
#pragma unroll
                for (int o = 0; o < RUN; ++o) res[o] = fadd2_rn(res[o], fmul2_rn(g, fadd2_rn(w[o + 8 + t], w[o + 8 - t])));
            }
        } else {   // the class boundary runs through this tile: both chains, each lane keeps its own
#pragma unroll
            for (int o = 0; o < RUN; ++o) {
                float2 sf = fmul2_rn(g8, w[o + 8]), sn = sf;
#pragma unroll
                for (int t = 1; t <= 8; ++t) {
                    const float2 a = fadd2_rn(w[o + 8 + t], w[o + 8 - t]);
                    const float2 g = make_float2(c_g17[8 + t], c_g17[8 + t]);
                    sf = ffma2_rn(g, a, sf);
                    sn = fadd2_rn(sn, fmul2_rn(g, a));
                }
                res[o] = make_float2(fma0 ? sf.x : sn.x, fma1 ? sf.y : sn.y);
            }
        }
        const bool col0 = j0 >= 0 && j0 < UW, col1 = j1 >= 0 && j1 < UW;
#pragma unroll
        for (int o = 0; o < RUN; ++o) {
            const int i = y0 - 1 + r0 + o;
            const bool row_ok = i >= 0 && i < UH;
            float2 v;   // out-of-image neighbours never win the max
            v.x = (row_ok && col0) ? res[o].x : -INFINITY;
            v.y = (row_ok && col1) ? res[o].y : -INFINITY;
            *reinterpret_cast<float2*>(sS + (r0 + o) * RT_LD + c) = v;
        }
    }
    __syncthreads();

    // ---- threshold + 3x3 NMS (same_max_pool_3x3_2d skips out-of-range neighbours) + emission
    static_assert(TW <= 64 && K1_THREADS % 64 == 0, "NMS: thread = (row mod 3, column)");
    const int c = tid & 63;
    for (int r = tid >> 6; r < TH; r += K1_THREADS / 64) {
        const int i = y0 + r, j = x0 + c;
        if (c >= TW || i >= UH || j >= UW) continue;
        const float* q = sS + (r + 1) * RT_LD + (c + 1);
        const float v = q[0];
        if (!(v > p.thresh)) continue;
        float m = v;
        m = fmaxf(m, q[-RT_LD - 1]); m = fmaxf(m, q[-RT_LD]); m = fmaxf(m, q[-RT_LD + 1]);
        m = fmaxf(m, q[-1]);                                   m = fmaxf(m, q[1]);
        m = fmaxf(m, q[RT_LD - 1]);  m = fmaxf(m, q[RT_LD]);   m = fmaxf(m, q[RT_LD + 1]);
        if (v == m) {
            int* cnt = p.peak_cnt + frame * HP_N_PARTS + part;
            const int slot = atomicAdd(cnt, 1);
            if (slot < p.pcap) {
                const size_t o = ((size_t)frame * HP_N_PARTS + part) * p.pcap + slot;
                p.raw_key[o] = i * UW + j;
                p.raw_score[o] = tile_u(sU2, r + HALO, c + HALO); // score = UNsmoothed up-map value
            } else {
                atomicOr(p.flags + frame, FLAG_PEAK_OVERFLOW);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K0 (only for resolutions that shrink an axis): cv::resize(INTER_AREA) of every channel into HBM, one thread per destination
// value, the reference's arithmetic in the reference's order (oracle/paf_oracle.c orc_resize_area, pinned to cv2):
//   mode 0  2-tap area-mode lerp on both axes (mixed regime: one axis grows);
//   mode 1  integer factors: block sum in row-major order, four at a time (sum += ((s0+s1)+s2)+s3), times (float)(1/area);
//           the 2 x 2 case is ((a+b)+(c+d)) * 0.25 for dx < (dw & ~3) (OpenCV's SIMD kernel) and the scalar order on the tail;
//   mode 2  fractional: DecimateAlpha tables -- buf = sum_k S[sx_k] * alpha_k per source row, dst = beta_0 buf_0 + beta_1 buf_1 + ...
// ---------------------------------------------------------------------------------------------
struct ResizeParams {
    const float* src; float* dst;   // [N*C, H, W] -> [N*C, UH, UW]
    int planes, H, W, UH, UW;
    int mode, isx, isy;
    const int* xi; const float* xf; const int* yi; const float* yf;           // mode 0
    const int* xofs; const int* xsi; const float* xal;                          // mode 2: entries [xofs[dx], xofs[dx+1])
    const int* yofs; const int* ysi; const float* yal;
};

__global__ void __launch_bounds__(256) resize_area_generic_kernel(const ResizeParams p)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)p.planes * p.UH * p.UW;
    if (idx >= total) return;
    const int dx = (int)(idx % p.UW);
    const int dy = (int)((idx / p.UW) % p.UH);
    const int pl = (int)(idx / ((size_t)p.UW * p.UH));
    const float* S = p.src + (size_t)pl * p.H * p.W;
    const int W = p.W;
    float out;
    if (p.mode == 0) {
        const int x0 = __ldg(p.xi + dx), x1 = min(x0 + 1, W - 1);
        const int y0 = __ldg(p.yi + dy), y1 = min(y0 + 1, p.H - 1);
        const float a1 = __ldg(p.xf + dx), a0 = __fsub_rn(1.f, a1);
        const float b1 = __ldg(p.yf + dy), b0 = __fsub_rn(1.f, b1);
        const float h0 = __fadd_rn(__fmul_rn(S[y0 * W + x0], a0), __fmul_rn(S[y0 * W + x1], a1));
        const float h1 = __fadd_rn(__fmul_rn(S[y1 * W + x0], a0), __fmul_rn(S[y1 * W + x1], a1));
        out = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
    } else if (p.mode == 1) {
        const int isx = p.isx, isy = p.isy, area = isx * isy;
        const float* B = S + (size_t)dy * isy * W + (size_t)dx * isx;
        if (isx == 2 && isy == 2 && dx < (p.UW & ~3)) {
            out = __fmul_rn(__fadd_rn(__fadd_rn(B[0], B[1]), __fadd_rn(B[W], B[W + 1])), 0.25f);
        } else {
            float sum = 0.f;
            int k = 0;
            for (; k <= area - 4; k += 4) {
                float g = __fadd_rn(B[(k / isx) * W + k % isx], B[((k + 1) / isx) * W + (k + 1) % isx]);
                g = __fadd_rn(g, B[((k + 2) / isx) * W + (k + 2) % isx]);
                g = __fadd_rn(g, B[((k + 3) / isx) * W + (k + 3) % isx]);
                sum = __fadd_rn(sum, g);
            }
            for (; k < area; ++k) sum = __fadd_rn(sum, B[(k / isx) * W + k % isx]);
            out = __fmul_rn(sum, __fdiv_rn(1.f, (float)area));
        }
    } else {
        const int xb = __ldg(p.xofs + dx), xe = __ldg(p.xofs + dx + 1);
        const int yb = __ldg(p.yofs + dy), ye = __ldg(p.yofs + dy + 1);
        float sum = 0.f;
        for (int j = yb; j < ye; ++j) {
            const float* R = S + (size_t)__ldg(p.ysi + j) * W;
            float buf = 0.f;
            for (int k = xb; k < xe; ++k) buf = __fadd_rn(buf, __fmul_rn(R[__ldg(p.xsi + k)], __ldg(p.xal + k)));
            const float t = __fmul_rn(__ldg(p.yal + j), buf);
            sum = (j == yb) ? t : __fadd_rn(sum, t);
        }
        out = sum;
    }
    p.dst[idx] = out;
}

// ---------------------------------------------------------------------------------------------
// K2: everything after the peak scan, one CTA per (limb, frame):
//   (a) peak ordering   -- the CTA restores the reference's channel-major / row-major peak order (ids = index) for the two
//                          parts of its limb: rank-sort by scan position.  A part belongs to several limbs; every CTA that
//                          needs it writes the SAME ordered records to the same place (idempotent), so no CTA waits for another.
//   (b) limb scoring    -- get_connection_candidates (paf.cpp:93-144): 10 lanes per peak pair, ballot / shuffle reductions
//   (c) matching        -- std::sort by score + greedy one-to-one (paf.cpp:234-272), candidates kept in shared memory
//   (d) assembly        -- get_humans + filter + conversion (paf.cpp:146-232, 359-372) by the LAST CTA of the frame to finish
//                          (threadfence + per-frame arrival counter): one lane per connected component of the (peaks,
//                          connections) graph, or, for the frames that path hands back, the strictly ordered merge on one warp
//                          out of shared memory (assemble_sequential).
// ---------------------------------------------------------------------------------------------
constexpr int K3_THREADS = 256;
constexpr int MAX_PCAP = 4096;   // bitmap size for the greedy pass
constexpr int SM_CAND = 512;     // candidates per limb kept in shared memory (more: global scratch)
constexpr int SM_KEYS = 512;     // raw peak keys per part staged for the rank sort
constexpr int SM_CONN = 1024;    // connections per frame staged for the assembly
constexpr int SM_PSC = 2048;     // peak scores per frame staged for the assembly
constexpr int SM_TAB = 1024;     // up-sampling table entries (UW + UH) staged for the line integrals
constexpr int ASM_WARPS = 2;     // component-parallel assembly: one LANE per connected component, 32 * ASM_WARPS components per frame
constexpr int ASM_CMAX = 32 * ASM_WARPS;
constexpr int ASM_SLOTS = 8;     // partial humans ever created inside one component (more: sequential fallback)
constexpr int ASM_IFIELDS = 3;   // per slot: score, n_parts, creation index as 32-bit words; the 18 part ids as 16-bit values (ids < SM_PSC)

// whether paf_limbs_kernel stages the up-sampling tables in shared memory (else it reads them from global memory); `from_up`: the
// resolution shrinks an axis and the line integrals read the materialised up-maps instead
__host__ __device__ constexpr bool limb_tables_staged(bool from_up, int UW, int UH) { return !from_up && UW + UH <= SM_TAB; }

struct LimbParams {
    const float* paf; // [N, c_paf, H, W]
    int c_paf, H, W, UH, UW;
    const int* xi; const float* xf; const int* yi; const float* yf;
    float paf_thresh;
    int feat_height; // m_feature_size.height == W of the feature map of the handle's first call (paf.cpp:321-332,354)
    int pcap, ccap, hcap, max_refs;
    const int* peak_cnt;             // [N,18]
    const int* raw_key;              // [N,18,pcap]  y*UW + x
    const float* raw_score;          // [N,18,pcap]
    int* part_base;                  // [N,19]
    int* px; int* py; float* pscore; // [N, 18*pcap] ordered peaks
    unsigned long long* cand;        // [N,19,ccap]
    unsigned long long* cand_sorted; // [N,19,ccap]
    hp_connection* conn;             // [N,19,pcap]
    int* conn_cnt;                   // [N,19]
    int* frame_done;                 // [N] arrival counter of the frame's limb CTAs
    hp_human* humans;                // [N,hcap]
    int* human_cnt;                  // [N]
    int* flags;
    int stage_bytes; // dynamic smem available for staging the two PAF channels (0 = never stage)
    int fast_asm;    // 1: the dynamic shared memory holds the component-parallel assembly state
    const float* up_paf; // resolutions that shrink an axis: resized PAF maps [N, c_paf, UH, UW] (resize_area_generic_kernel); else null
    unsigned long long* dbg_t; // optional phase timestamps (%globaltimer, ns): [N][19][4] per CTA (start, ordered, candidates, matched) + [N][2] assembly (start, end); null = off
};

__device__ __forceinline__ unsigned long long gtimer()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// up-sampled PAF value at up-map pixel (lx, ly), recomputed from the low-resolution field
// exactly as orc_resize_area_up does (horizontal lerp on two source rows, then vertical).
template <bool kTabSmem> // kTabSmem: the tables were staged in shared memory (plain loads); else global memory through the read-only path
__device__ __forceinline__ float up_sample(const float* P, int W, int H, int lx, int ly,
                                           const int* xi, const float* xf, const int* yi, const float* yf)
{
    const int sx0 = kTabSmem ? xi[lx] : __ldg(xi + lx), sx1 = min(sx0 + 1, W - 1);
    const int sy0 = kTabSmem ? yi[ly] : __ldg(yi + ly), sy1 = min(sy0 + 1, H - 1);
    const float a1 = kTabSmem ? xf[lx] : __ldg(xf + lx), a0 = __fsub_rn(1.f, a1);
    const float b1 = kTabSmem ? yf[ly] : __ldg(yf + ly), b0 = __fsub_rn(1.f, b1);
    const float h0 = __fadd_rn(__fmul_rn(P[sy0 * W + sx0], a0), __fmul_rn(P[sy0 * W + sx1], a1));
    const float h1 = __fadd_rn(__fmul_rn(P[sy1 * W + sx0], a0), __fmul_rn(P[sy1 * W + sx1], a1));
    return __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
}

// candidate key: score bits (positive floats order like unsigned ints) | inverted (idx1, idx2)
// => max key == best score, ties broken by idx1 asc then idx2 asc (frozen tie-break, SURVEY 8c).
__device__ __forceinline__ unsigned long long make_key(float score, int ia, int ib)
{
    return ((unsigned long long)__float_as_uint(score) << 32) | (unsigned)(0xffffffffu - (((unsigned)ia << 16) | (unsigned)ib));
}

__device__ __forceinline__ hp_connection ld_conn_cg(const hp_connection* c)
{
    hp_connection r;
    r.cid1 = __ldcg(&c->cid1); r.cid2 = __ldcg(&c->cid2); r.score = __ldcg(&c->score);
    return r;
}

// the filter of get_humans (paf.cpp:226-230)
__device__ __forceinline__ bool keep_human(const int n_parts, const float score)
{
    return !(n_parts < THRESH_PART_CNT || __fdiv_rn(score, (float)n_parts) < 0.4f);
}

// part id -> hp_body_part (paf.cpp:359-372).  Ids fabricated by the `+=` merge quirk would be an out-of-bounds read (UB) in the
// reference; like the oracle, such parts are reported absent.  sPsc: the frame's peak scores staged in shared memory, or null.
__device__ __forceinline__ hp_body_part body_part(const LimbParams& p, const int frame, const int n_peaks, const float* sPsc, const int id)
{
    hp_body_part bp;
    bp.has_value = 0; bp.x = 0.f; bp.y = 0.f; bp.score = 0.f;
    if (id >= 0 && id < n_peaks) {
        const size_t k = (size_t)frame * HP_N_PARTS * p.pcap + id;   // other CTAs wrote the peaks: read past L1
        bp.has_value = 1;
        bp.score = sPsc ? sPsc[id] : __ldcg(p.pscore + k);
        bp.x = __fdiv_rn((float)__ldcg(p.px + k), (float)p.UW);
        bp.y = __fdiv_rn((float)__ldcg(p.py + k), (float)p.UH);
    }
    return bp;
}

// The strictly sequential get_humans (one warp), the partial humans in shared memory: stored part-major so that the 32-wide "touch"
// test is bank-conflict free, the per-part loops of a merge on 18 lanes.  Runs for the frames the component-parallel path of
// paf_limbs_kernel hands back (fabricated ids, > 64 components, > 8 partial humans in a component, > 1024 connections, > 2048 peaks)
// and for every frame when that path is off.  The connections are read from shared memory when they were staged, else from global
// memory; the peak scores likewise (sPsc null: not staged).
__device__ __forceinline__ void assemble_sequential(const LimbParams& p, const int frame, const int lane, const bool conn_staged,
                                                    const int n_peaks, const int* sCnt, const hp_connection* sConn, const float* sPsc,
                                                    int* rParts, float* rScore, int* rNparts, unsigned long long* dbg_a)
{
    const int MAXR = p.max_refs;
    const hp_connection* gconn = p.conn + (size_t)frame * HP_N_PAIRS * p.pcap;
    // (unstaged: > 2048 peaks in one frame; plain loads are fine for values no earlier read of this SM cached)
    const float* psc = sPsc ? sPsc : p.pscore + (size_t)frame * HP_N_PARTS * p.pcap;

    int nh = 0;
    for (int pair_id = 0; pair_id < HP_N_PAIRS; ++pair_id) {
        const int part1 = c_pairs[pair_id][0], part2 = c_pairs[pair_id][1];
        const int ncn = sCnt[pair_id + 1] - sCnt[pair_id];
        const hp_connection* conns = conn_staged ? sConn + sCnt[pair_id] : gconn + (size_t)pair_id * p.pcap;
        for (int ci = 0; ci < ncn; ++ci) {
            const hp_connection cn = conn_staged ? conns[ci] : ld_conn_cg(conns + ci);
            // touches (paf.cpp:33-36) evaluated for 32 humans at a time; first two hits in vector order
            int t0 = -1, t1 = -1, nt = 0;
            for (int hb = 0; hb < nh && nt < 2; hb += 32) {
                const int h = hb + lane;
                const bool touch = (h < nh) && (rParts[part1 * MAXR + h] == cn.cid1 || rParts[part2 * MAXR + h] == cn.cid2);
                unsigned bal = __ballot_sync(0xffffffffu, touch);
                while (bal && nt < 2) {
                    const int l = __ffs(bal) - 1;
                    if (nt == 0) t0 = hb + l; else t1 = hb + l;
                    ++nt;
                    bal &= bal - 1;
                }
            }
            // every branch below is warp-uniform (nt, t0, t1, nh are the same on all lanes)
            if (nt == 1) { // paf.cpp:172-178
                if (lane == 0 && rParts[part2 * MAXR + t0] != cn.cid2) {
                    rParts[part2 * MAXR + t0] = cn.cid2;
                    rNparts[t0] += 1;
                    rScore[t0] = __fadd_rn(rScore[t0], __fadd_rn(psc[cn.cid2], cn.score));
                }
            } else if (nt >= 2) { // paf.cpp:179-210
                int va = 0, vb = 0;
                if (lane < HP_N_PARTS) { va = rParts[lane * MAXR + t0]; vb = rParts[lane * MAXR + t1]; }
                const bool shared_part = __ballot_sync(0xffffffffu, lane < HP_N_PARTS && va > 0 && vb > 0) != 0u; // `id > 0` quirk (paf.cpp:185)
                if (!shared_part) {
                    if (lane < HP_N_PARTS) rParts[lane * MAXR + t0] = va + vb + 1; // paf.cpp:193
                    if (lane == 0) {
                        rNparts[t0] += rNparts[t1];
                        rScore[t0] = __fadd_rn(__fadd_rn(rScore[t0], rScore[t1]), cn.score);
                    }
                    __syncwarp();
                    // vector::erase (paf.cpp:201-205): lanes 0..17 shift one part column each, 18 the scores, 19 the counts
                    for (int h = t1; h + 1 < nh; ++h) {
                        if (lane < HP_N_PARTS) rParts[lane * MAXR + h] = rParts[lane * MAXR + h + 1];
                        else if (lane == HP_N_PARTS) rScore[h] = rScore[h + 1];
                        else if (lane == HP_N_PARTS + 1) rNparts[h] = rNparts[h + 1];
                    }
                    nh -= 1;
                } else if (lane == 0) {
                    rParts[part2 * MAXR + t0] = cn.cid2;
                    rNparts[t0] += 1;
                    rScore[t0] = __fadd_rn(rScore[t0], __fadd_rn(psc[cn.cid2], cn.score));
                }
            } else if (pair_id <= 16) { // !is_virtual_pair (coco.hpp:6, paf.cpp:211-220)
                if (nh < MAXR) {
                    if (lane < HP_N_PARTS) rParts[lane * MAXR + nh] = (lane == part1) ? cn.cid1 : (lane == part2) ? cn.cid2 : -1;
                    if (lane == 0) {
                        rNparts[nh] = 2;
                        rScore[nh] = __fadd_rn(__fadd_rn(psc[cn.cid1], psc[cn.cid2]), cn.score);
                    }
                    nh += 1;
                } else if (lane == 0) {
                    atomicOr(p.flags + frame, FLAG_HUMAN_OVERFLOW);
                }
            }
            __syncwarp();
        }
    }

    // filter (stable like remove_if) + conversion to human_t
    int no = 0;
    for (int hb = 0; hb < nh; hb += 32) {
        const int h = hb + lane;
        const bool keep = h < nh && keep_human(rNparts[h], rScore[h]);
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const int idx = no + __popc(bal & ((1u << lane) - 1u));
        if (keep) {
            if (idx < p.hcap) {
                hp_human* o = p.humans + (size_t)frame * p.hcap + idx;
                o->score = rScore[h];
                for (int i = 0; i < HP_N_PARTS; ++i) o->parts[i] = body_part(p, frame, n_peaks, sPsc, rParts[i * MAXR + h]);
            } else {
                atomicOr(p.flags + frame, FLAG_HUMAN_OVERFLOW);
            }
        }
        no += __popc(bal);
    }
    if (lane == 0) p.human_cnt[frame] = min(no, p.hcap);
    if (dbg_a && lane == 0) dbg_a[1] = (gtimer() & ~3ull) | 1ull;   // low bits 1: the shared-memory path ran
}

__global__ void __launch_bounds__(K3_THREADS, 3) paf_limbs_kernel(const LimbParams p)
{
    extern __shared__ __align__(16) unsigned char sDyn[];   // phase (b): the two PAF channels; phase (d): the assembly state
    __shared__ int sNcand, sLast, sFast, sNComp, sNKeep;
    __shared__ __align__(8) unsigned long long sBulkBar;
    __shared__ int sBase[HP_N_PARTS + 1];
    __shared__ unsigned sUsedA[MAX_PCAP / 32], sUsedB[MAX_PCAP / 32];
    __shared__ unsigned long long sCand[SM_CAND], sSorted[SM_CAND];
    __shared__ int sKeys[SM_KEYS];
    // behind the staged PAF planes (phase b only; the assembly of phase d reuses the whole dynamic region):
    int* sTabI = reinterpret_cast<int*>(sDyn + p.stage_bytes);     // [SM_TAB] xi[UW] then yi[UH]
    float* sTabF = reinterpret_cast<float*>(sTabI + SM_TAB);       // [SM_TAB] xf[UW] then yf[UH]
    int (*sPk)[SM_KEYS] = reinterpret_cast<int (*)[SM_KEYS]>(sTabF + SM_TAB);   // [2][SM_KEYS] ordered peaks of the limb's two parts, x | y << 16

    const int limb = blockIdx.x, frame = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pa = c_pairs[limb][0], pb = c_pairs[limb][1];
    const int* cnt = p.peak_cnt + frame * HP_N_PARTS;
    unsigned long long* dbg = p.dbg_t ? p.dbg_t + ((size_t)frame * HP_N_PAIRS + limb) * 4 : nullptr;
    if (dbg && tid == 0) dbg[0] = gtimer();
    if (tid == 0) {
        int bsum = 0;
        for (int q = 0; q < HP_N_PARTS; ++q) { sBase[q] = bsum; bsum += min(cnt[q], p.pcap); }
        sBase[HP_N_PARTS] = bsum;
        sNcand = 0;
    }
    // the up-sampling tables of the line integrals: one coalesced pass instead of four dependent global loads per sample
    const bool tab_staged = limb_tables_staged(p.up_paf != nullptr, p.UW, p.UH);
    if (tab_staged) {
        for (int i = tid; i < p.UW + p.UH; i += K3_THREADS) {
            const bool isx = i < p.UW;
            sTabI[i] = isx ? __ldg(p.xi + i) : __ldg(p.yi + (i - p.UW));
            sTabF[i] = isx ? __ldg(p.xf + i) : __ldg(p.yf + (i - p.UW));
        }
    }
    __syncthreads();
    if (limb == 0 && tid <= HP_N_PARTS) p.part_base[frame * (HP_N_PARTS + 1) + tid] = sBase[tid];
    const size_t peak_off = (size_t)frame * HP_N_PARTS * p.pcap;
    int* px = p.px + peak_off;
    int* py = p.py + peak_off;
    float* pscore = p.pscore + peak_off;

    // ---- (a) order the peaks of this limb's two parts (post_process.hpp:175-192: ids follow the scan order)
    const bool pk_staged = p.UW < 65536 && p.UH < 32768 && sBase[pa + 1] - sBase[pa] <= SM_KEYS && sBase[pb + 1] - sBase[pb] <= SM_KEYS;
    for (int which = 0; which < 2; ++which) {
        const int part = which ? pb : pa;
        const int n = sBase[part + 1] - sBase[part];
        const size_t raw = ((size_t)frame * HP_N_PARTS + part) * p.pcap;
        const int* keys = p.raw_key + raw;
        const bool staged = n <= SM_KEYS;
        __syncthreads();   // sKeys of the previous part is dead
        if (staged) {
            for (int i = tid; i < n; i += K3_THREADS) sKeys[i] = keys[i];
            __syncthreads();
        }
        const int out = sBase[part];
        for (int i = tid; i < n; i += K3_THREADS) {
            const int k = staged ? sKeys[i] : keys[i];
            int rank = 0;
            if (staged) { for (int q = 0; q < n; ++q) rank += (sKeys[q] < k); }   // keys are unique pixel positions
            else        { for (int q = 0; q < n; ++q) rank += (keys[q] < k); }
            const int x = k % p.UW, y = k / p.UW;
            px[out + rank] = x;
            py[out + rank] = y;
            pscore[out + rank] = p.raw_score[raw + i];
            if (pk_staged) sPk[which][rank] = x | (y << 16);
        }
    }
    __syncthreads();   // this CTA's own global writes are visible to all of its threads from here on
    if (dbg && tid == 0) dbg[1] = gtimer();

    const int base_a = sBase[pa], na = sBase[pa + 1] - base_a;
    const int base_b = sBase[pb], nb = sBase[pb + 1] - base_b;
    int* conn_cnt = p.conn_cnt + frame * HP_N_PAIRS + limb;
    const int H = p.H, W = p.W;
    if (na == 0 || nb == 0) {
        if (tid == 0) *conn_cnt = 0;
    } else {
        const float* P1 = p.paf + ((size_t)frame * p.c_paf + c_pairs_net[limb][0]) * H * W;
        const float* P2 = p.paf + ((size_t)frame * p.c_paf + c_pairs_net[limb][1]) * H * W;
        const int npairs = na * nb;
        const float* U1 = nullptr; const float* U2 = nullptr;   // materialised up-maps of the two channels (shrinking resolutions)
        if (p.up_paf) {
            U1 = p.up_paf + ((size_t)frame * p.c_paf + c_pairs_net[limb][0]) * p.UH * p.UW;
            U2 = p.up_paf + ((size_t)frame * p.c_paf + c_pairs_net[limb][1]) * p.UH * p.UW;
        }
        // stage both channels when enough pairs will reuse them (one coalesced pass instead of scattered gathers)
        if (!p.up_paf && npairs >= 6 && (int)(2 * H * W * sizeof(float)) <= p.stage_bytes) {
            float* sPaf = reinterpret_cast<float*>(sDyn);
            const unsigned plane_bytes = (unsigned)(H * W * sizeof(float));
            if ((plane_bytes & 15u) == 0u && ((size_t)P1 & 15) == 0 && ((size_t)P2 & 15) == 0) {
                // two bulk async copies (TMA, 1-D) issued by one thread instead of ~60 dependent load / store rounds per thread
                const unsigned bar = (unsigned)__cvta_generic_to_shared(&sBulkBar);
                if (tid == 0) {
                    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
                    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(2u * plane_bytes) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"((unsigned)__cvta_generic_to_shared(sPaf)), "l"(P1), "r"(plane_bytes), "r"(bar) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"((unsigned)__cvta_generic_to_shared(sPaf + H * W)), "l"(P2), "r"(plane_bytes), "r"(bar) : "memory");
                }
                __syncthreads();   // the barrier is initialised before anybody polls it
                unsigned done;
                do {
                    asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], 0;\n\tselp.u32 %0, 1, 0, q;\n\t}" : "=r"(done) : "r"(bar) : "memory");
                } while (!done);
            } else {
                for (int i = tid; i < H * W; i += K3_THREADS) {
                    sPaf[i] = __ldg(P1 + i);
                    sPaf[H * W + i] = __ldg(P2 + i);
                }
            }
            P1 = sPaf;
            P2 = sPaf + H * W;
        }
        __syncthreads();

        unsigned long long* cand = p.cand + ((size_t)frame * HP_N_PAIRS + limb) * p.ccap;
        unsigned long long* sorted = p.cand_sorted + ((size_t)frame * HP_N_PAIRS + limb) * p.ccap;

        // ---- (b) get_connection_candidates: 3 peak pairs per warp pass, 10 lanes (= 10 samples) per pair
        const int grp = lane / STEP_PAF, smp = lane - grp * STEP_PAF;
        const unsigned gmask = (grp < 3) ? (0x3ffu << (grp * STEP_PAF)) : 0u;
        constexpr int NW = K3_THREADS / 32;
        for (int pb0 = warp * 3; pb0 < npairs; pb0 += NW * 3) { // warp-uniform trip count
            const int pidx = pb0 + grp;
            const bool active = (grp < 3) && (pidx < npairs);
            int ia = 0, ib = 0;
            float score = 0.f, norm = 1.f;
            bool valid = false;
            if (active) {
                ia = pidx / nb;
                ib = pidx - ia * nb;
                int ax, ay, bx, by;
                if (pk_staged) {
                    const int ka = sPk[0][ia], kb = sPk[1][ib];
                    ax = ka & 0xffff; ay = ka >> 16; bx = kb & 0xffff; by = kb >> 16;
                } else {
                    ax = px[base_a + ia]; ay = py[base_a + ia]; bx = px[base_b + ib]; by = py[base_b + ib];
                }
                const int dx = bx - ax, dy = by - ay;
                norm = (float)sqrt((double)(dx * dx + dy * dy)); // paf.cpp:104
                valid = !((double)norm < 1e-12);                   // paf.cpp:105
                if (valid) {
                    const float vx = __fdiv_rn((float)dx, norm), vy = __fdiv_rn((float)dy, norm);
                    const float stepx = __fdiv_rn((float)dx, (float)STEP_PAF); // paf.cpp:77-78
                    const float stepy = __fdiv_rn((float)dy, (float)STEP_PAF);
                    const float fx = __fadd_rn((float)ax, __fmul_rn((float)smp, stepx));
                    const float fy = __fadd_rn((float)ay, __fmul_rn((float)smp, stepy));
                    const int lx = (int)((double)fx + 0.5); // roundpaf (paf.cpp:74): float + double literal
                    const int ly = (int)((double)fy + 0.5);
                    float vpx, vpy;
                    if (U1) {
                        vpx = __ldg(U1 + (size_t)ly * p.UW + lx);
                        vpy = __ldg(U2 + (size_t)ly * p.UW + lx);
                    } else if (tab_staged) {
                        vpx = up_sample<true>(P1, W, H, lx, ly, sTabI, sTabF, sTabI + p.UW, sTabF + p.UW);
                        vpy = up_sample<true>(P2, W, H, lx, ly, sTabI, sTabF, sTabI + p.UW, sTabF + p.UW);
                    } else {
                        vpx = up_sample<false>(P1, W, H, lx, ly, p.xi, p.xf, p.yi, p.yf);
                        vpy = up_sample<false>(P2, W, H, lx, ly, p.xi, p.xf, p.yi, p.yf);
                    }
                    score = __fadd_rn(__fmul_rn(vx, vpx), __fmul_rn(vy, vpy)); // paf.cpp:122
                }
            }
            const unsigned ball = __ballot_sync(0xffffffffu, valid && score > p.paf_thresh);
            const int criterion1 = __popc(ball & gmask);
            float sum = 0.f; // sequential i = 0..9 accumulation order of paf.cpp:121-127
#pragma unroll
            for (int i = 0; i < STEP_PAF; ++i) {
                const int srcl = min(grp * STEP_PAF + i, 31);
                sum = __fadd_rn(sum, __shfl_sync(0xffffffffu, score, srcl));
            }
            if (valid && smp == 0) {
                double pen = 0.5 * (double)p.feat_height / (double)norm - 1.0; // paf.cpp:129
                if (pen > 0.0) pen = 0.0;
                const float criterion2 = (float)((double)__fdiv_rn(sum, (float)STEP_PAF) + pen);
                if (criterion1 > THRESH_VECTOR_CNT1 && criterion2 > 0.f) {
                    const int slot = atomicAdd(&sNcand, 1);
                    const unsigned long long key = make_key(criterion2, ia, ib);
                    if (slot < SM_CAND) sCand[slot] = key;
                    else if (slot < p.ccap) cand[slot] = key;
                }
            }
        }
        __syncthreads();
        if (dbg && tid == 0) dbg[2] = gtimer();
        int ncand = sNcand;
        if (ncand > p.ccap) {
            if (tid == 0) atomicOr(p.flags + frame, FLAG_CAND_OVERFLOW);
            ncand = p.ccap;
        }
        // the common case keeps the whole list in shared memory; a longer one moves to the global scratch arrays
        const bool in_smem = ncand <= SM_CAND;
        if (!in_smem) {
            for (int i = tid; i < SM_CAND; i += K3_THREADS) cand[i] = sCand[i];
            __threadfence_block();
            __syncthreads();
        }
        const unsigned long long* cin = in_smem ? sCand : cand;
        unsigned long long* cout = in_smem ? sSorted : sorted;

        // ---- (c) std::sort by score desc (paf.cpp:249-250): rank sort on unique keys
        for (int i = tid; i < ncand; i += K3_THREADS) {
            const unsigned long long k = cin[i];
            int rank = 0;
            for (int q = 0; q < ncand; ++q) rank += (cin[q] > k);
            cout[rank] = k;
        }
        for (int i = tid; i < MAX_PCAP / 32; i += K3_THREADS) { sUsedA[i] = 0u; sUsedB[i] = 0u; }
        __threadfence_block();
        __syncthreads();

        // greedy one-to-one selection in score order (paf.cpp:252-270)
        if (tid == 0) {
            hp_connection* conn = p.conn + ((size_t)frame * HP_N_PAIRS + limb) * p.pcap;
            const int max_conn = min(na, nb);
            int nconn = 0;
            for (int i = 0; i < ncand && nconn < max_conn; ++i) {
                const unsigned long long k = cout[i];
                const unsigned inv = 0xffffffffu - (unsigned)(k & 0xffffffffu);
                const int ia = (int)(inv >> 16), ib = (int)(inv & 0xffffu);
                if ((sUsedA[ia >> 5] >> (ia & 31)) & 1u) continue;
                if ((sUsedB[ib >> 5] >> (ib & 31)) & 1u) continue;
                sUsedA[ia >> 5] |= 1u << (ia & 31);
                sUsedB[ib >> 5] |= 1u << (ib & 31);
                hp_connection c;
                c.cid1 = base_a + ia; // peak ids == index in the ordered all_peaks list
                c.cid2 = base_b + ib;
                c.score = __uint_as_float((unsigned)(k >> 32));
                conn[nconn++] = c;
            }
            *conn_cnt = nconn;
        }
    }

    // ---- (d) the last CTA of the frame to arrive assembles the humans
    if (dbg && tid == 0) dbg[3] = gtimer();
    __threadfence();   // ordered peaks, connections and counts of this CTA: visible device-wide before the arrival is counted
    __syncthreads();
    if (tid == 0) sLast = (atomicAdd(p.frame_done + frame, 1) == HP_N_PAIRS - 1) ? 1 : 0;
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    unsigned long long* dbg_a = p.dbg_t ? p.dbg_t + (size_t)gridDim.y * HP_N_PAIRS * 4 + (size_t)frame * 6 : nullptr;
    if (dbg_a && tid == 0) dbg_a[0] = gtimer();

    const int n_peaks = sBase[HP_N_PARTS];
    const int MAXR = p.max_refs;
    // dynamic shared memory of the assembly: [connections | their peak scores | UNION { component-parallel state ;
    // all peak scores + partial humans of the sequential path }]
    hp_connection* sConn = reinterpret_cast<hp_connection*>(sDyn);             // [SM_CONN]
    float2* sConnPs = reinterpret_cast<float2*>(sConn + SM_CONN);              // [SM_CONN] peak scores of (cid1, cid2)
    int* uni = reinterpret_cast<int*>(sConnPs + SM_CONN);
    float* sPsc = reinterpret_cast<float*>(uni);                               // [SM_PSC]
    int* rParts = uni + SM_PSC;                                       // [18][MAXR] part-major: lane h reads parts[q][h] conflict-free
    float* rScore = reinterpret_cast<float*>(rParts + HP_N_PARTS * MAXR);
    int* rNparts = reinterpret_cast<int*>(rScore + MAXR);
    int* sLabel = uni;                                                         // [SM_PSC] component labels of the peaks
    int* sCompCnt = sLabel + SM_PSC;                                           // [ASM_CMAX] fill pointers
    int* sCompOff = sCompCnt + ASM_CMAX;                                       // [ASM_CMAX + 1]
    int* sKeep = sCompOff + ASM_CMAX + 1;                                      // [ASM_CMAX * ASM_SLOTS] keys of the surviving humans
    int* sSlotI = sKeep + ASM_CMAX * ASM_SLOTS;                                // [ASM_WARPS][ASM_SLOTS][ASM_IFIELDS][32]
    short* sSlotP = reinterpret_cast<short*>(sSlotI + ASM_WARPS * ASM_SLOTS * ASM_IFIELDS * 32);   // [ASM_WARPS][ASM_SLOTS][18][32] part ids, -1 = absent
    unsigned short* sList = reinterpret_cast<unsigned short*>(sSlotP + ASM_WARPS * ASM_SLOTS * HP_N_PARTS * 32);   // [SM_CONN] connections grouped by component
    unsigned short* sConnPair = sList + SM_CONN;                               // [SM_CONN] part1 | part2 << 5 | pair << 10
    unsigned char* sConnComp = reinterpret_cast<unsigned char*>(sConnPair + SM_CONN);   // [SM_CONN] component of the connection
    int* sCnt = reinterpret_cast<int*>(sUsedA);                                // [20] connection offsets (bitmaps are dead)
    if (tid < 32) {   // connection counts of the 19 limbs (other CTAs wrote them: read past L1), exclusive prefix by shuffles
        const int c = tid < HP_N_PAIRS ? __ldcg(p.conn_cnt + frame * HP_N_PAIRS + tid) : 0;
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (tid >= o) incl += v;
        }
        if (tid <= HP_N_PAIRS) sCnt[tid] = incl - c;   // sCnt[19] = total (lane 19 holds c = 0)
    }
    __syncthreads();
    const int n_conn = sCnt[HP_N_PAIRS];
    const bool conn_staged = n_conn <= SM_CONN, psc_staged = n_peaks <= SM_PSC;
    const hp_connection* gconn = p.conn + (size_t)frame * HP_N_PAIRS * p.pcap;
    const bool fast_try = p.fast_asm && conn_staged && psc_staged;
    if (conn_staged)   // one connection per thread and round: the loads of all limbs are in flight together (two dependent L2 latencies in total)
        for (int i = tid; i < n_conn; i += K3_THREADS) {
            int q = 0;
            while (sCnt[q + 1] <= i) ++q;
            const hp_connection c = ld_conn_cg(gconn + (size_t)q * p.pcap + (i - sCnt[q]));
            sConn[i] = c;
            sConnPs[i] = make_float2(__ldcg(pscore + c.cid1), __ldcg(pscore + c.cid2));
            if (fast_try) sConnPair[i] = (unsigned short)(c_pairs[q][0] | (c_pairs[q][1] << 5) | (q << 10));
        }

    // ---- component-parallel get_humans.  The reference walks the connections strictly in order, but a connection can only
    // "touch" (paf.cpp:33-36) a partial human that already holds one of its two peaks, so partial humans of different CONNECTED
    // COMPONENTS of the (peaks, connections) graph never interact: each component is replayed sequentially by ONE LANE, all
    // components at once, and the survivors are put back into the reference's vector order afterwards -- a human's position in
    // the vector follows its creation (erase keeps the relative order, a merge keeps the earlier human, paf.cpp:191-205), so the
    // order is the ascending index of the creating connection.  The one cross-component effect of the reference is the id
    // FABRICATED by `parts[i] += other.parts[i] + 1` when both humans hold a part and one of the ids is 0 (the `id > 0` quirk,
    // paf.cpp:185): such a frame -- like one with more components / partial humans than fit -- is redone by the sequential path below.
    if (fast_try) {
        if (tid == 0) { sFast = 1; sNComp = 0; sNKeep = 0; }
        for (int i = tid; i < n_peaks; i += K3_THREADS) sLabel[i] = i | 0x40000000;   // not an end point of any connection
        for (int i = tid; i < ASM_CMAX; i += K3_THREADS) sCompCnt[i] = 0;
        for (int i = tid; i < ASM_WARPS * ASM_SLOTS * (ASM_IFIELDS + HP_N_PARTS / 2) * 32; i += K3_THREADS) sSlotI[i] = -1;   // every part of every slot absent, n_parts < 0 (the 16-bit part array follows the words)
        __syncthreads();
        if (dbg_a && tid == 0) dbg_a[2] = gtimer();
        for (int i = tid; i < n_conn; i += K3_THREADS) { const hp_connection c = sConn[i]; sLabel[c.cid1] = c.cid1; sLabel[c.cid2] = c.cid2; }
        __syncthreads();
        while (true) {   // min-label propagation with one pointer jump per visit; labels are always end points of the same component
            int changed = 0;
            for (int i = tid; i < n_conn; i += K3_THREADS) {
                const hp_connection c = sConn[i];
                int a = sLabel[c.cid1], b = sLabel[c.cid2];
                a = min(a, sLabel[a]); b = min(b, sLabel[b]);
                const int m = min(a, b);
                if (sLabel[c.cid1] > m) { atomicMin(&sLabel[c.cid1], m); changed = 1; }
                if (sLabel[c.cid2] > m) { atomicMin(&sLabel[c.cid2], m); changed = 1; }
            }
            if (!__syncthreads_or(changed)) break;
        }
        // fixed point: one label L per component with sLabel[L] == L; number the components (any order: the output order is restored below)
        for (int i = tid; i < n_peaks; i += K3_THREADS)
            if (sLabel[i] == i) sLabel[i] = -(atomicAdd(&sNComp, 1) + 1);
        __syncthreads();
        const int n_comp = sNComp;
        if (dbg_a && tid == 0) dbg_a[3] = gtimer();
        if (n_comp <= ASM_CMAX) {
            for (int i = tid; i < n_conn; i += K3_THREADS) {
                int l = sLabel[sConn[i].cid1];
                if (l >= 0) l = sLabel[l];
                const int cc = -l - 1;
                sConnComp[i] = (unsigned char)cc;
                atomicAdd(&sCompCnt[cc], 1);
            }
            __syncthreads();
            if (warp == 0) {
                // exclusive scan of the component sizes (ASM_CMAX = 32 * ASM_WARPS values, ASM_WARPS per lane)
                int v[ASM_WARPS], tot = 0;
#pragma unroll
                for (int k = 0; k < ASM_WARPS; ++k) { v[k] = sCompCnt[lane * ASM_WARPS + k]; tot += v[k]; }
                int incl = tot;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int u = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += u;
                }
                int run = incl - tot;
#pragma unroll
                for (int k = 0; k < ASM_WARPS; ++k) { sCompOff[lane * ASM_WARPS + k] = run; sCompCnt[lane * ASM_WARPS + k] = run; run += v[k]; }
                if (lane == 31) sCompOff[ASM_CMAX] = run;
                __syncwarp();
                // stable grouping: the connections of a component keep their global order
                for (int base = 0; base < n_conn; base += 32) {
                    const int i = base + lane;
                    const unsigned cc = i < n_conn ? (unsigned)sConnComp[i] : 0xffffu;
                    const unsigned peers = __match_any_sync(0xffffffffu, cc);
                    const int rank = __popc(peers & ((1u << lane) - 1u));
                    const int pos = cc != 0xffffu ? sCompCnt[cc] + rank : 0;
                    __syncwarp();
                    if (cc != 0xffffu && rank == 0) sCompCnt[cc] += __popc(peers);
                    __syncwarp();
                    if (cc != 0xffffu) sList[pos] = (unsigned short)i;
                }
            }
            __syncthreads();
            if (dbg_a && tid == 0) dbg_a[4] = gtimer();
            if (warp < ASM_WARPS) {
                const int ci = warp * 32 + lane;
                int* S = sSlotI + warp * ASM_SLOTS * ASM_IFIELDS * 32 + lane;   // lane-private columns: the bank follows the lane, never a conflict
                short* Q = sSlotP + warp * ASM_SLOTS * HP_N_PARTS * 32 + lane;
#define HP_SI(slot, f) S[((slot) * ASM_IFIELDS + (f)) * 32]
#define HP_SP(slot, f) Q[((slot) * HP_N_PARTS + (f)) * 32]
                constexpr int F_SCORE = 0, F_NP = 1, F_MADE = 2;
                bool ok = true;
                int ns = 0;   // partial humans ever created in this component (slots are never reused: a merged-away human is marked dead)
                if (ci < n_comp) {
                    const int beg = sCompOff[ci], end = sCompOff[ci + 1];
                    int gi_next = sList[beg];   // (a component has at least one connection)
                    for (int k = beg; k < end; ++k) {
                        const int gi = gi_next;
                        if (k + 1 < end) gi_next = sList[k + 1];
                        const hp_connection cn = sConn[gi];
                        const float2 ps = sConnPs[gi];
                        const int code = sConnPair[gi];
                        const int P1 = code & 31, P2 = (code >> 5) & 31, pair_id = code >> 10;
                        // one batch of independent loads for every slot created so far (one shared-memory latency, not one per slot)
                        int vn[ASM_SLOTS], v1[ASM_SLOTS], v2[ASM_SLOTS];
#pragma unroll
                        for (int sl = 0; sl < ASM_SLOTS; ++sl) {
                            vn[sl] = -1; v1[sl] = -2; v2[sl] = -2;
                            if (sl < ns) { vn[sl] = HP_SI(sl, F_NP); v1[sl] = HP_SP(sl, P1); v2[sl] = HP_SP(sl, P2); }
                        }
                        int t0 = -1, t1 = -1, np0 = 0, p2_0 = -2;   // first two touching humans in vector order (paf.cpp:33-36,160-170)
#pragma unroll
                        for (int sl = ASM_SLOTS - 1; sl >= 0; --sl)
                            if (vn[sl] >= 0 && (v1[sl] == cn.cid1 || v2[sl] == cn.cid2)) { t1 = t0; t0 = sl; np0 = vn[sl]; p2_0 = v2[sl]; }
                        if (t0 < 0) {
                            if (pair_id <= 16) {   // !is_virtual_pair (coco.hpp:6, paf.cpp:211-220)
                                if (ns >= ASM_SLOTS) { ok = false; break; }
                                HP_SP(ns, P1) = (short)cn.cid1; HP_SP(ns, P2) = (short)cn.cid2;   // (the other parts were preset to -1)
                                HP_SI(ns, F_NP) = 2;
                                HP_SI(ns, F_SCORE) = __float_as_int(__fadd_rn(__fadd_rn(ps.x, ps.y), cn.score));
                                HP_SI(ns, F_MADE) = gi;
                                ++ns;
                            }
                        } else if (t1 < 0) {   // paf.cpp:172-178
                            if (p2_0 != cn.cid2) {
                                HP_SP(t0, P2) = (short)cn.cid2;
                                HP_SI(t0, F_NP) = np0 + 1;
                                HP_SI(t0, F_SCORE) = __float_as_int(__fadd_rn(__int_as_float(HP_SI(t0, F_SCORE)), __fadd_rn(ps.y, cn.score)));
                            }
                        } else {               // paf.cpp:179-210
                            bool shared_part = false, fabricates = false;
                            int a[HP_N_PARTS], b[HP_N_PARTS];
#pragma unroll
                            for (int f = 0; f < HP_N_PARTS; ++f) { a[f] = HP_SP(t0, f); b[f] = HP_SP(t1, f); }
#pragma unroll
                            for (int f = 0; f < HP_N_PARTS; ++f) {
                                shared_part |= (a[f] > 0 && b[f] > 0);   // `id > 0` quirk (paf.cpp:185)
                                fabricates |= (a[f] >= 0 && b[f] >= 0);
                            }
                            if (!shared_part) {
                                if (fabricates) { ok = false; break; }   // the merge would invent a peak id: sequential path
#pragma unroll
                                for (int f = 0; f < HP_N_PARTS; ++f) HP_SP(t0, f) = (short)(a[f] + b[f] + 1);   // paf.cpp:193
                                HP_SI(t0, F_NP) = np0 + HP_SI(t1, F_NP);
                                HP_SI(t0, F_SCORE) = __float_as_int(__fadd_rn(__fadd_rn(__int_as_float(HP_SI(t0, F_SCORE)), __int_as_float(HP_SI(t1, F_SCORE))), cn.score));
                                HP_SI(t1, F_NP) = -1;   // vector::erase (paf.cpp:201-205)
                            } else {
                                HP_SP(t0, P2) = (short)cn.cid2;
                                HP_SI(t0, F_NP) = np0 + 1;
                                HP_SI(t0, F_SCORE) = __float_as_int(__fadd_rn(__int_as_float(HP_SI(t0, F_SCORE)), __fadd_rn(ps.y, cn.score)));
                            }
                        }
                    }
                    if (ok) {   // filter (paf.cpp:226-230)
                        for (int sl = 0; sl < ns; ++sl) {
                            const int np = HP_SI(sl, F_NP);
                            if (np < 0 || np < THRESH_PART_CNT || __fdiv_rn(__int_as_float(HP_SI(sl, F_SCORE)), (float)np) < 0.4f) continue;
                            sKeep[atomicAdd(&sNKeep, 1)] = (HP_SI(sl, F_MADE) << 9) | (ci << 3) | sl;
                        }
                    }
                }
                if (!ok) sFast = 0;
#undef HP_SI
#undef HP_SP
            }
            __syncthreads();
            if (dbg_a && tid == 0) dbg_a[5] = gtimer();
            if (sFast) {
                // conversion (paf.cpp:359-372) in vector order: one warp per surviving human, one lane per part
                const int nk = sNKeep;
                for (int h = warp; h < nk; h += K3_THREADS / 32) {
                    const int key = sKeep[h];
                    int rank = 0;
                    for (int q = lane; q < nk; q += 32) rank += (sKeep[q] < key);
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
                    if (rank >= p.hcap) { if (lane == 0) atomicOr(p.flags + frame, FLAG_HUMAN_OVERFLOW); continue; }
                    const int ci = (key >> 3) & (ASM_CMAX - 1), sl = key & 7;
                    const int* Sx = sSlotI + ((ci >> 5) * ASM_SLOTS + sl) * ASM_IFIELDS * 32 + (ci & 31);
                    const short* Qx = sSlotP + ((ci >> 5) * ASM_SLOTS + sl) * HP_N_PARTS * 32 + (ci & 31);
                    hp_human* o = p.humans + (size_t)frame * p.hcap + rank;
                    if (lane < HP_N_PARTS) {
                        o->parts[lane] = body_part(p, frame, n_peaks, nullptr, Qx[lane * 32]);
                    } else if (lane == HP_N_PARTS) {
                        o->score = __int_as_float(Sx[0]);
                    }
                }
                if (tid == 0) p.human_cnt[frame] = min(nk, p.hcap);
                if (dbg_a && tid == 0) dbg_a[1] = (gtimer() & ~3ull) | 2ull;   // low bits 2: the component-parallel path ran
                return;
            }
        }
    }
    // every thread has passed a barrier after its last access to the component-parallel state: its space takes the peak scores
    if (psc_staged)
        for (int i = tid; i < n_peaks; i += K3_THREADS) sPsc[i] = __ldcg(pscore + i);   // other CTAs wrote these: read past L1
    __syncthreads();
    if (warp != 0) return;
    assemble_sequential(p, frame, lane, conn_staged, n_peaks, sCnt, sConn, psc_staged ? sPsc : nullptr, rParts, rScore, rNparts, dbg_a);
}

// bytes of dynamic shared memory the assembly phase of paf_limbs_kernel needs for `max_refs` partial humans
constexpr size_t ASM_COMMON_BYTES = (size_t)SM_CONN * sizeof(hp_connection) + (size_t)SM_CONN * sizeof(float2);
// the component-parallel state; it shares the union region with the peak scores + partial humans of the sequential path
constexpr size_t ASM_FAST_BYTES = ((size_t)SM_PSC + ASM_CMAX + ASM_CMAX + 1 + ASM_CMAX * ASM_SLOTS + ASM_WARPS * ASM_SLOTS * (ASM_IFIELDS + HP_N_PARTS / 2) * 32) * 4
                                  + (size_t)SM_CONN * 2 * 2 + SM_CONN + 16;
constexpr size_t assemble_smem_bytes(int max_refs, bool fast)
{
    return ASM_COMMON_BYTES + std::max((size_t)SM_PSC * 4 + (size_t)max_refs * (HP_N_PARTS + 2) * 4, fast ? ASM_FAST_BYTES : (size_t)0);
}
// phase (b) keeps the up-sampling tables and the packed peaks of the limb behind the staged PAF planes
constexpr size_t LIMB_PHASE_B_EXTRA = (size_t)SM_TAB * 8 + (size_t)2 * SM_KEYS * 4;

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
// OpenCV resize.cpp, INTER_AREA with dst >= src ("area_mode" 2-tap interpolation):
//   inv = dst/src (double), scale = 1/inv, sx = floor(dx*scale),
//   fx = (float)((dx+1) - (sx+1)*inv); fx = fx <= 0 ? 0 : fx - floor(fx); clamp at the last source px.
void area_up_table(int src, int dst, std::vector<int>& idx, std::vector<float>& frac)
{
    idx.resize(dst);
    frac.resize(dst);
    const double inv = (double)dst / (double)src;
    const double scale = 1.0 / inv;
    for (int d = 0; d < dst; ++d) {
        int s = (int)floor(d * scale);
        float f = (float)((double)(d + 1) - (double)(s + 1) * inv);
        f = f <= 0.f ? 0.f : f - floorf(f);
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
        idx[d] = s;
        frac[d] = f;
    }
}

// OpenCV computeResizeAreaTab (resize.cpp), grouped by destination index: entries [ofs[d], ofs[d+1]) = (source index, weight)
void decimate_table(int ssize, int dsize, double scale, std::vector<int>& ofs, std::vector<int>& si, std::vector<float>& al)
{
    ofs.assign(1, 0); si.clear(); al.clear();
    for (int dx = 0; dx < dsize; ++dx) {
        const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        const double cell = std::min(scale, ssize - fsx1);
        int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
        sx2 = std::min(sx2, ssize - 1);
        sx1 = std::min(sx1, sx2);
        if (sx1 - fsx1 > 1e-3) { si.push_back(sx1 - 1); al.push_back((float)((sx1 - fsx1) / cell)); }
        for (int sx = sx1; sx < sx2; ++sx) { si.push_back(sx); al.push_back((float)(1.0 / cell)); }
        if (fsx2 - sx2 > 1e-3) { si.push_back(sx2); al.push_back((float)(std::min(std::min(fsx2 - sx2, 1.0), cell) / cell)); }
        ofs.push_back((int)si.size());
    }
}

// Source rows (or columns) the tile starting at up-map position t0 reads: the tile's window [t0 - 9, t0 + extent + 9) in
// reflected coordinates (BORDER_REFLECT_101), each position touching source index idx[.] and idx[.] + 1 (clamped).
void tile_source_bounds(const std::vector<int>& idx, int src_len, int up_len, int tile, int window, std::vector<int>& out)
{
    const int tiles = (up_len + tile - 1) / tile;
    for (int t = 0; t < tiles; ++t) {
        int lo = 0x7fffffff, hi = -1;
        for (int k = 0; k < window; ++k) {
            const int s = idx[refl101(t * tile - HALO + k, up_len)];
            lo = std::min(lo, s);
            hi = std::max(hi, std::min(s + 1, src_len - 1));
        }
        out.push_back(lo);
        out.push_back(hi);
    }
}

template <typename T> struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaError_t ensure(size_t count)
    {
        if (count <= n) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
        cudaError_t e = cudaMalloc(&p, count * sizeof(T));
        if (e == cudaSuccess) {
            n = count;
            // unused record slots travel to the host with the used ones: zero them.  On a private non-blocking stream + a stream
            // (not device) synchronise: another host thread of the process may be capturing a CUDA graph on this device (pool
            // workers), during which neither the legacy stream nor cudaDeviceSynchronize may be touched.
            static thread_local cudaStream_t zs = nullptr;
            static thread_local int zs_dev = -1;
            int dev = 0;
            cudaGetDevice(&dev);
            if (!zs || zs_dev != dev) { if (cudaStreamCreateWithFlags(&zs, cudaStreamNonBlocking) != cudaSuccess) return cudaGetLastError(); zs_dev = dev; }
            e = cudaMemsetAsync(p, 0, count * sizeof(T), zs);
            if (e == cudaSuccess) e = cudaStreamSynchronize(zs);
        }
        return e;
    }
    void release()
    {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
};

template <typename T> struct PinnedBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaError_t ensure(size_t count)
    {
        if (count <= n) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        n = 0;
        cudaError_t e = cudaMallocHost(&p, count * sizeof(T));
        if (e == cudaSuccess) n = count;
        return e;
    }
    void release()
    {
        if (p) cudaFreeHost(p);
        p = nullptr;
        n = 0;
    }
};

} // namespace

struct hp_paf {
    int device = 0;
    float conf_thresh = 0.05f, paf_thresh = 0.05f;
    int res_w = -1, res_h = -1; // user resolution (-1 = reference default, fixed at the first call like paf.cpp:314-315)
    int feat_height = -1;       // length-penalty height: W of the first call's maps (m_feature_size, paf.cpp:321-332,354)
    int pcap = 128, ccap = 2048, hcap = 64, max_refs = 256;
    cudaStream_t stream = nullptr;
    long long launches = 0;

    // geometry of the current buffers
    int N = 0, c_conf = 0, c_paf = 0, H = 0, W = 0, UH = 0, UW = 0;
    int cap_pcap = 0, cap_ccap = 0, cap_hcap = 0, cap_N = 0;

    DevBuf<int> xi, yi, tile_bounds;
    DevBuf<float> xf, yf;
    // resolutions that shrink an axis (cv::resize INTER_AREA beyond pure up-scaling): materialised maps + the resize description
    bool generic = false;
    int rz_mode = 0, rz_isx = 1, rz_isy = 1;
    DevBuf<int> rz_xofs, rz_xsi, rz_yofs, rz_ysi;
    DevBuf<float> rz_xal, rz_yal, up_conf, up_paf;
    DevBuf<unsigned long long> dbg_t;   // HPB_PAF_TIMING=1: phase timestamps of the last batch (hp_paf_debug_timing)
    DevBuf<int> counters; // [N*18 peak_cnt | N*19 conn_cnt | N human_cnt | N flags | N frame_done]
    DevBuf<int> raw_key, part_base, px, py;
    DevBuf<float> raw_score, pscore;
    DevBuf<unsigned long long> cand, cand_sorted;
    DevBuf<hp_connection> conn;
    DevBuf<hp_human> humans;
    DevBuf<float> in_conf, in_paf; // device staging for host inputs
    PinnedBuf<float> pin_in;
    PinnedBuf<hp_human> pin_humans;
    PinnedBuf<int> pin_counts; // [N human_cnt | N flags]
    int last_N = 0;
    cudaStream_t last_stream = nullptr;
    int limb_dyn_bytes = 0;       // dynamic shared memory paf_limbs_kernel may use (opted in at create)
    int assemble_max_refs = 256;  // partial humans that fit next to the staged connections / scores
    // tile rows of paf_peaks_kernel with more than HL_ROWS source rows / tile columns with more than SRC_COLS source columns
    int wide_tile_rows = 0, wide_tile_cols = 0;
    int plan[HP_PAF_PLAN_FIELDS] = {};   // the code paths of the last launch_pipeline (hp_paf_debug_plan)

    int* peak_cnt() { return counters.p; }
    int* conn_cnt() { return counters.p + (size_t)cap_N * HP_N_PARTS; }
    int* human_cnt() { return counters.p + (size_t)cap_N * (HP_N_PARTS + HP_N_PAIRS); }
    int* flags() { return counters.p + (size_t)cap_N * (HP_N_PARTS + HP_N_PAIRS + 1); }
    int* frame_done() { return counters.p + (size_t)cap_N * (HP_N_PARTS + HP_N_PAIRS + 2); }
    static constexpr int COUNTERS_PER_FRAME = HP_N_PARTS + HP_N_PAIRS + 3;
};

namespace {

int ensure_geometry(hp_paf* p, int N, int c_conf, int c_paf, int H, int W)
{
    if (N <= 0 || H <= 0 || W <= 0 || c_conf < HP_N_PARTS || c_paf < 2 * HP_N_PAIRS) {
        hpb::set_error("hp_paf: bad tensor shape N=%d conf=[%d,%d,%d] paf=[%d,%d,%d] (need >=18 / >=38 channels)",
                       N, c_conf, H, W, c_paf, H, W);
        return HP_ERR_ARG;
    }
    // paf.cpp:311-315: dims() of the [C,H,W] view are bound to (C, fw, fh): fw = H, fh = W, and the
    // default resolution is cv::Size(width = fw*4, height = fh*4).  Fixed at the first call.
    if (p->res_w == -1 || p->res_h == -1) {
        p->res_w = H * 4;
        p->res_h = W * 4;
    }
    if (p->feat_height == -1) p->feat_height = W;
    const int UW = p->res_w, UH = p->res_h;
    if (p->pcap > MAX_PCAP) p->pcap = MAX_PCAP;
    const bool geo_changed = (H != p->H || W != p->W || UH != p->UH || UW != p->UW);
    if (geo_changed) {
        // cv::resize's dispatch (resize.cpp): true area averaging when BOTH axes shrink or keep, else 2-tap area-mode interpolation
        p->generic = (UW < W || UH < H);
        const double scale_x = 1.0 / ((double)UW / (double)W), scale_y = 1.0 / ((double)UH / (double)H);
        p->rz_mode = 0;
        if (p->generic && scale_x >= 1.0 && scale_y >= 1.0) {
            const int isx = (int)lrint(scale_x), isy = (int)lrint(scale_y);
            if (fabs(scale_x - isx) < 2.220446049250313e-16 && fabs(scale_y - isy) < 2.220446049250313e-16) {
                p->rz_mode = 1; p->rz_isx = isx; p->rz_isy = isy;
            } else {
                p->rz_mode = 2;
                std::vector<int> ofs, si; std::vector<float> al;
                decimate_table(W, UW, scale_x, ofs, si, al);
                HP_CUDA_TRY(p->rz_xofs.ensure(ofs.size())); HP_CUDA_TRY(p->rz_xsi.ensure(si.size())); HP_CUDA_TRY(p->rz_xal.ensure(al.size()));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_xofs.p, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_xsi.p, si.data(), si.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_xal.p, al.data(), al.size() * sizeof(float), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaStreamSynchronize(p->stream));
                decimate_table(H, UH, scale_y, ofs, si, al);
                HP_CUDA_TRY(p->rz_yofs.ensure(ofs.size())); HP_CUDA_TRY(p->rz_ysi.ensure(si.size())); HP_CUDA_TRY(p->rz_yal.ensure(al.size()));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_yofs.p, ofs.data(), ofs.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_ysi.p, si.data(), si.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaMemcpyAsync(p->rz_yal.p, al.data(), al.size() * sizeof(float), cudaMemcpyHostToDevice, p->stream));
                HP_CUDA_TRY(cudaStreamSynchronize(p->stream));
            }
        }
        std::vector<int> idx_x, idx_y;
        std::vector<float> fr;
        area_up_table(W, UW, idx_x, fr);
        HP_CUDA_TRY(p->xi.ensure(UW));
        HP_CUDA_TRY(p->xf.ensure(UW));
        HP_CUDA_TRY(cudaMemcpyAsync(p->xi.p, idx_x.data(), UW * sizeof(int), cudaMemcpyHostToDevice, p->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(p->xf.p, fr.data(), UW * sizeof(float), cudaMemcpyHostToDevice, p->stream));
        HP_CUDA_TRY(cudaStreamSynchronize(p->stream)); // the vectors are locals
        area_up_table(H, UH, idx_y, fr);
        HP_CUDA_TRY(p->yi.ensure(UH));
        HP_CUDA_TRY(p->yf.ensure(UH));
        HP_CUDA_TRY(cudaMemcpyAsync(p->yi.p, idx_y.data(), UH * sizeof(int), cudaMemcpyHostToDevice, p->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(p->yf.p, fr.data(), UH * sizeof(float), cudaMemcpyHostToDevice, p->stream));
        // per tile row / tile column: the source rows / columns its halo window reads (K1 stages exactly that rectangle)
        std::vector<int> tb;
        p->wide_tile_rows = p->wide_tile_cols = 0;
        if (!p->generic) {
            tile_source_bounds(idx_y, H, UH, TH, UT_H, tb);
            const size_t rows_end = tb.size();
            tile_source_bounds(idx_x, W, UW, TW, UT_W, tb);
            for (size_t i = 0; i < tb.size(); i += 2) {
                const int n = tb[i + 1] - tb[i] + 1;
                if (i < rows_end) p->wide_tile_rows += n > HL_ROWS;
                else p->wide_tile_cols += n > SRC_COLS;
            }
        } else {
            tb.assign(4, 0);
        }
        HP_CUDA_TRY(p->tile_bounds.ensure(tb.size()));
        HP_CUDA_TRY(cudaMemcpyAsync(p->tile_bounds.p, tb.data(), tb.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
        HP_CUDA_TRY(cudaStreamSynchronize(p->stream));
    }
    p->H = H; p->W = W; p->UH = UH; p->UW = UW; p->c_conf = c_conf; p->c_paf = c_paf;
    if (N > p->cap_N || p->pcap != p->cap_pcap || p->ccap != p->cap_ccap || p->hcap != p->cap_hcap) {
        const int cN = std::max(N, p->cap_N);
        p->cap_N = cN;
        p->cap_pcap = p->pcap; p->cap_ccap = p->ccap; p->cap_hcap = p->hcap;
        HP_CUDA_TRY(p->counters.ensure((size_t)cN * hp_paf::COUNTERS_PER_FRAME));
        HP_CUDA_TRY(p->raw_key.ensure((size_t)cN * HP_N_PARTS * p->pcap));
        HP_CUDA_TRY(p->raw_score.ensure((size_t)cN * HP_N_PARTS * p->pcap));
        HP_CUDA_TRY(p->part_base.ensure((size_t)cN * (HP_N_PARTS + 1)));
        HP_CUDA_TRY(p->px.ensure((size_t)cN * HP_N_PARTS * p->pcap));
        HP_CUDA_TRY(p->py.ensure((size_t)cN * HP_N_PARTS * p->pcap));
        HP_CUDA_TRY(p->pscore.ensure((size_t)cN * HP_N_PARTS * p->pcap));
        HP_CUDA_TRY(p->cand.ensure((size_t)cN * HP_N_PAIRS * p->ccap));
        HP_CUDA_TRY(p->cand_sorted.ensure((size_t)cN * HP_N_PAIRS * p->ccap));
        HP_CUDA_TRY(p->conn.ensure((size_t)cN * HP_N_PAIRS * p->pcap));
        HP_CUDA_TRY(p->humans.ensure((size_t)cN * p->hcap));
        HP_CUDA_TRY(p->pin_humans.ensure((size_t)cN * p->hcap));
        HP_CUDA_TRY(p->pin_counts.ensure((size_t)cN * 2));
    }
    if (p->generic) {
        HP_CUDA_TRY(p->up_conf.ensure((size_t)std::max(N, p->cap_N) * c_conf * UH * UW));
        HP_CUDA_TRY(p->up_paf.ensure((size_t)std::max(N, p->cap_N) * c_paf * UH * UW));
    }
    p->N = N;
    return HP_OK;
}

int launch_pipeline(hp_paf* p, const float* d_conf, const float* d_paf, int N, cudaStream_t st)
{
    const int UH = p->UH, UW = p->UW;
    HP_CUDA_TRY(cudaMemsetAsync(p->counters.p, 0, (size_t)p->cap_N * hp_paf::COUNTERS_PER_FRAME * sizeof(int), st));

    PeakParams k1;
    k1.conf = d_conf; k1.c_conf = p->c_conf; k1.H = p->H; k1.W = p->W; k1.UH = UH; k1.UW = UW;
    k1.xi = p->xi.p; k1.xf = p->xf.p; k1.yi = p->yi.p; k1.yf = p->yf.p;
    k1.thresh = p->conf_thresh;
    k1.skip_below = (p->conf_thresh > 0.f) ? p->conf_thresh * (1.f - 1e-5f) : -INFINITY;
    k1.tiles_x = (UW + TW - 1) / TW;
    k1.tiles_y = (UH + TH - 1) / TH;
    k1.tile_bounds = p->tile_bounds.p;
    k1.pcap = p->pcap;
    k1.peak_cnt = p->peak_cnt(); k1.raw_key = p->raw_key.p; k1.raw_score = p->raw_score.p; k1.flags = p->flags();
    k1.n8 = UW & ~7;
    k1.n4 = (UW - k1.n8 >= 4) ? k1.n8 + 4 : k1.n8;
    dim3 g1(k1.tiles_x, k1.tiles_y * HP_N_PARTS, N);
    k1.up = nullptr;
    if (p->generic) {   // resolutions that shrink an axis: materialise cv::resize(INTER_AREA) of every channel, then run from the maps
        ResizeParams rz;
        rz.H = p->H; rz.W = p->W; rz.UH = UH; rz.UW = UW; rz.mode = p->rz_mode; rz.isx = p->rz_isx; rz.isy = p->rz_isy;
        rz.xi = p->xi.p; rz.xf = p->xf.p; rz.yi = p->yi.p; rz.yf = p->yf.p;
        rz.xofs = p->rz_xofs.p; rz.xsi = p->rz_xsi.p; rz.xal = p->rz_xal.p; rz.yofs = p->rz_yofs.p; rz.ysi = p->rz_ysi.p; rz.yal = p->rz_yal.p;
        rz.src = d_conf; rz.dst = p->up_conf.p; rz.planes = N * p->c_conf;
        resize_area_generic_kernel<<<(unsigned)(((size_t)rz.planes * UH * UW + 255) / 256), 256, 0, st>>>(rz);
        rz.src = d_paf; rz.dst = p->up_paf.p; rz.planes = N * p->c_paf;
        resize_area_generic_kernel<<<(unsigned)(((size_t)rz.planes * UH * UW + 255) / 256), 256, 0, st>>>(rz);
        p->launches += 2;
        k1.up = p->up_conf.p;
        paf_peaks_kernel<true><<<g1, K1_THREADS, 0, st>>>(k1);
    } else {
        paf_peaks_kernel<false><<<g1, K1_THREADS, 0, st>>>(k1);
    }

    LimbParams k3;
    k3.paf = d_paf; k3.c_paf = p->c_paf; k3.H = p->H; k3.W = p->W; k3.UH = UH; k3.UW = UW;
    k3.xi = p->xi.p; k3.xf = p->xf.p; k3.yi = p->yi.p; k3.yf = p->yf.p;
    k3.paf_thresh = p->paf_thresh;
    k3.feat_height = p->feat_height; // m_feature_size = cv::Size(fw, fh) with fh = W, set at the first call (paf.cpp:321-332); .height -> get_connections (:354)
    k3.pcap = p->pcap; k3.ccap = p->ccap; k3.hcap = p->hcap; k3.max_refs = p->max_refs;
    k3.peak_cnt = p->peak_cnt(); k3.raw_key = p->raw_key.p; k3.raw_score = p->raw_score.p;
    k3.part_base = p->part_base.p; k3.px = p->px.p; k3.py = p->py.p; k3.pscore = p->pscore.p;
    k3.cand = p->cand.p; k3.cand_sorted = p->cand_sorted.p; k3.conn = p->conn.p; k3.conn_cnt = p->conn_cnt();
    k3.frame_done = p->frame_done(); k3.humans = p->humans.p; k3.human_cnt = p->human_cnt();
    k3.flags = p->flags();
    k3.up_paf = p->generic ? p->up_paf.p : nullptr;
    k3.dbg_t = nullptr;
    if (getenv("HPB_PAF_TIMING")) {
        HP_CUDA_TRY(p->dbg_t.ensure((size_t)p->cap_N * (HP_N_PAIRS * 4 + 6)));
        k3.dbg_t = p->dbg_t.p;
    }
    const int want = 2 * p->H * p->W * (int)sizeof(float);
    k3.stage_bytes = (want + (int)LIMB_PHASE_B_EXTRA <= p->limb_dyn_bytes) ? want : 0;
    k3.fast_asm = (ASM_COMMON_BYTES + ASM_FAST_BYTES <= (size_t)p->limb_dyn_bytes && !getenv("HPB_PAF_SEQ_ASSEMBLY")) ? 1 : 0;
    const size_t dyn = std::max((size_t)k3.stage_bytes + LIMB_PHASE_B_EXTRA, assemble_smem_bytes(p->max_refs, k3.fast_asm != 0));
    paf_limbs_kernel<<<dim3(HP_N_PAIRS, N), K3_THREADS, dyn, st>>>(k3);
    HP_CUDA_TRY(cudaGetLastError());
    const int plan[HP_PAF_PLAN_FIELDS] = {p->generic ? 1 : 0, p->generic ? p->rz_mode : -1, limb_tables_staged(p->generic, UW, UH) ? 1 : 0,
                                          k3.stage_bytes, p->limb_dyn_bytes, k3.fast_asm,
                                          p->generic ? 0 : p->wide_tile_rows, p->generic ? 0 : p->wide_tile_cols};
    memcpy(p->plan, plan, sizeof(plan));
    p->launches += 2;
    p->last_N = N;
    p->last_stream = st;
    return HP_OK;
}

int fetch_results(hp_paf* p, hp_human* out, int cap, int* n_out, int N)
{
    if (N != p->last_N || !out || !n_out || cap < 0) {
        hpb::set_error("hp_paf_fetch: N=%d does not match the last processed batch (%d) or null output", N, p->last_N);
        return HP_ERR_ARG;
    }
    cudaStream_t st = p->last_stream;
    HP_CUDA_TRY(cudaMemcpyAsync(p->pin_counts.p, p->human_cnt(), sizeof(int) * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(p->pin_counts.p + N, p->flags(), sizeof(int) * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(p->pin_humans.p, p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaStreamSynchronize(st));
    int flags = 0;
    for (int f = 0; f < N; ++f) flags |= p->pin_counts.p[N + f];
    if (flags) {
        hpb::set_error("hp_paf: internal capacity exceeded (flags=%d: 1 peaks/part>%d, 2 candidates/limb>%d, 4 humans>%d)",
                       flags, p->pcap, p->ccap, p->hcap);
        return HP_ERR_CAPACITY;
    }
    for (int f = 0; f < N; ++f) {
        const int n = p->pin_counts.p[f];
        if (n > cap) {
            hpb::set_error("hp_paf: frame %d has %d humans but the caller's capacity is %d", f, n, cap);
            return HP_ERR_CAPACITY;
        }
        n_out[f] = n;
        memcpy(out + (size_t)f * cap, p->pin_humans.p + (size_t)f * p->hcap, sizeof(hp_human) * n);
    }
    return HP_OK;
}

// The reference is unbounded (std::vector everywhere): after a run that raised overflow flags, enlarge exactly the capacities
// that overflowed.  HP_ERR_CAPACITY when a hard limit is reached (4096 peaks per part: the greedy pass' bitmaps).
int grow_after_overflow(hp_paf* p, int flags)
{
    if ((flags & FLAG_PEAK_OVERFLOW) && p->pcap >= MAX_PCAP) return HP_ERR_CAPACITY;
    if (flags & FLAG_PEAK_OVERFLOW) p->pcap = std::min(p->pcap * 4, MAX_PCAP);
    if (flags & FLAG_CAND_OVERFLOW) p->ccap *= 4;
    if (flags & FLAG_HUMAN_OVERFLOW) {
        if (p->hcap >= 4096 && p->max_refs >= p->assemble_max_refs) return HP_ERR_CAPACITY; // > ~2500 partial humans in one frame
        hp_paf_set_capacity(p, 0, 0, std::min(p->hcap * 4, 4096));
    }
    return HP_OK;
}

// Published-batch path of hp_paf_process_host (handoff.h): `conf` / `paf` are host buffers the engine filled AND published.
// The first call on a batch parses all of its frames from the device snapshot with this handle's parameters; the
// other frames (any handle with the same parameters, any thread) are served from the cached records.
constexpr int HANDOFF_MISS = 1;
int process_from_handoff(hp_paf* p, const float* conf, const float* paf, int c_conf, int c_paf, int H, int W, hp_human* out, int cap, int* n_out)
{
    namespace ho = hpb::handoff;
    if (H <= 0 || W <= 0 || c_conf <= 0 || c_paf <= 0) return HANDOFF_MISS;
    const size_t ea = (size_t)c_conf * H * W, eb = (size_t)c_paf * H * W;
    ho::Hit hit = ho::lookup(conf, paf, ea, eb);
    if (!hit.batch) return HANDOFF_MISS;
    ho::Batch& b = *hit.batch;
    std::lock_guard<std::mutex> lk(b.mu);
    const int f = hit.frame;
    if (!b.valid || b.fail_count >= 2 || b.device != p->device || f >= b.N || b.host_a[f] != conf || b.host_b[f] != paf ||
        b.elems_a != ea || b.elems_b != eb || !ho::contents_match(b, f)) {
        ho::count_miss();
        return HANDOFF_MISS;
    }
    if (ensure_geometry(p, b.N, c_conf, c_paf, H, W) != HP_OK) return HANDOFF_MISS; // the host path reports the error
    const bool cached = b.cache_kind == 1 && b.key_f[0] == p->conf_thresh && b.key_f[1] == p->paf_thresh && b.key_i[0] == p->res_w && b.key_i[1] == p->res_h &&
                        b.key_i[2] == p->feat_height;
    if (!cached) {
        b.cache_kind = 0;
        HP_CUDA_TRY(cudaStreamWaitEvent(p->stream, b.ready, 0));
        int rc = launch_pipeline(p, b.d_a, b.d_b, b.N, p->stream);
        if (rc) return rc;
        b.humans.resize((size_t)b.N * p->hcap);
        b.counts.resize(b.N);
        rc = fetch_results(p, b.humans.data(), p->hcap, b.counts.data(), b.N);
        if (rc == HP_ERR_CAPACITY) { // the host path grows this handle's capacities; a later frame may try again
            b.fail_count++;
            ho::count_miss();
            return HANDOFF_MISS;
        }
        if (rc) return rc;
        b.cache_kind = 1;
        b.key_f[0] = p->conf_thresh; b.key_f[1] = p->paf_thresh; b.key_i[0] = p->res_w; b.key_i[1] = p->res_h; b.key_i[2] = p->feat_height;
        b.hcap = p->hcap;
        ho::count_batch_parse();
    }
    const int n = b.counts[f];
    if (n > cap) {
        hpb::set_error("hp_paf: frame has %d humans but the caller's capacity is %d", n, cap);
        return HP_ERR_CAPACITY;
    }
    memcpy(out, b.humans.data() + (size_t)f * b.hcap, sizeof(hp_human) * n);
    *n_out = n;
    ho::count_hit();
    return HP_OK;
}

} // namespace

extern "C" {

int hp_paf_create(hp_paf** out, float conf_thresh, float paf_thresh, int res_w, int res_h, int device)
{
    if (!out) { hpb::set_error("hp_paf_create: null out"); return HP_ERR_ARG; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        hpb::set_error("hp_paf_create: no CUDA device (this library has no CPU fallback)");
        return HP_ERR_CUDA;
    }
    if (device < 0 || device >= ndev) { hpb::set_error("hp_paf_create: device %d out of range (%d devices)", device, ndev); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(device));
    hp_paf* p = new hp_paf();
    p->device = device;
    p->conf_thresh = conf_thresh;
    p->paf_thresh = paf_thresh;
    p->res_w = res_w;
    p->res_h = res_h;
    cudaError_t e = cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete p; hpb::set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); return HP_ERR_CUDA; }
    // opt in to the large dynamic shared-memory carve-out of paf_limbs_kernel: the two PAF channels of a limb in phase (b),
    // the partial humans + connections + peak scores of a frame in phase (d)
    int max_optin = 0;
    cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    cudaFuncAttributes fa;
    size_t static_smem = 16 * 1024;
    if (cudaFuncGetAttributes(&fa, paf_limbs_kernel) == cudaSuccess) static_smem = fa.sharedSizeBytes;
    else cudaGetLastError();
    int dyn = max_optin - (int)static_smem - 1024;
    if (dyn > 200 * 1024) dyn = 200 * 1024;
    if (dyn > 48 * 1024 - (int)static_smem && cudaFuncSetAttribute(paf_limbs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn) == cudaSuccess)
        p->limb_dyn_bytes = dyn;
    else {
        cudaGetLastError();
        p->limb_dyn_bytes = 48 * 1024 - (int)static_smem;
    }
    p->assemble_max_refs = (int)((p->limb_dyn_bytes - (ASM_COMMON_BYTES + SM_PSC * 4)) / ((HP_N_PARTS + 2) * 4));
    if (p->max_refs > p->assemble_max_refs) p->max_refs = p->assemble_max_refs;
    *out = p;
    return HP_OK;
}

void hp_paf_destroy(hp_paf* p)
{
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) { cudaStreamSynchronize(p->stream); cudaStreamDestroy(p->stream); }
    p->xi.release(); p->yi.release(); p->xf.release(); p->yf.release(); p->tile_bounds.release(); p->counters.release();
    p->dbg_t.release(); p->rz_xofs.release(); p->rz_xsi.release(); p->rz_yofs.release(); p->rz_ysi.release(); p->rz_xal.release(); p->rz_yal.release(); p->up_conf.release(); p->up_paf.release();
    p->raw_key.release(); p->part_base.release(); p->px.release(); p->py.release();
    p->raw_score.release(); p->pscore.release(); p->cand.release(); p->cand_sorted.release();
    p->conn.release(); p->humans.release(); p->in_conf.release(); p->in_paf.release();
    p->pin_in.release(); p->pin_humans.release(); p->pin_counts.release();
    delete p;
}

int hp_paf_set_conf_thresh(hp_paf* p, float t) { if (!p) return HP_ERR_ARG; p->conf_thresh = t; return HP_OK; }
int hp_paf_set_paf_thresh(hp_paf* p, float t) { if (!p) return HP_ERR_ARG; p->paf_thresh = t; return HP_OK; }

int hp_paf_set_capacity(hp_paf* p, int max_peaks_per_part, int max_candidates_per_limb, int max_humans)
{
    if (!p) return HP_ERR_ARG;
    if (max_peaks_per_part > 0) p->pcap = std::min(max_peaks_per_part, MAX_PCAP);
    if (max_candidates_per_limb > 0) p->ccap = max_candidates_per_limb;
    if (max_humans > 0) {
        p->hcap = max_humans;
        // partial humans (paf.cpp:152 `human_refs`) live in shared memory: 80 B each, up to the opted-in carve-out
        p->max_refs = std::min(std::max(256, 4 * max_humans), p->assemble_max_refs);
    }
    return HP_OK;
}

int hp_paf_process_device(hp_paf* p, const float* d_conf, const float* d_paf, int N, int c_conf, int c_paf, int H, int W, void* stream)
{
    if (!p || !d_conf || !d_paf) { hpb::set_error("hp_paf_process_device: null argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    int rc = ensure_geometry(p, N, c_conf, c_paf, H, W);
    if (rc) return rc;
    return launch_pipeline(p, d_conf, d_paf, N, stream ? (cudaStream_t)stream : p->stream);
}

int hp_paf_fetch(hp_paf* p, hp_human* out, int cap, int* n_out, int N)
{
    if (!p) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    return fetch_results(p, out, cap, n_out, N);
}

int hp_paf_process_host_batched(hp_paf* p, const float* conf, const float* paf, int N, int c_conf, int c_paf, int H, int W,
                                hp_human* out, int cap, int* n_out)
{
    if (!p || !conf || !paf || !out || !n_out) { hpb::set_error("hp_paf_process_host: null argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    for (int attempt = 0; attempt < 8; ++attempt) {
        int rc = ensure_geometry(p, N, c_conf, c_paf, H, W);
        if (rc) return rc;
        const size_t n_conf = (size_t)N * c_conf * H * W, n_paf = (size_t)N * c_paf * H * W;
        HP_CUDA_TRY(p->in_conf.ensure(n_conf));
        HP_CUDA_TRY(p->in_paf.ensure(n_paf));
        HP_CUDA_TRY(p->pin_in.ensure(n_conf + n_paf));
        memcpy(p->pin_in.p, conf, n_conf * sizeof(float));
        memcpy(p->pin_in.p + n_conf, paf, n_paf * sizeof(float));
        HP_CUDA_TRY(cudaMemcpyAsync(p->in_conf.p, p->pin_in.p, n_conf * sizeof(float), cudaMemcpyHostToDevice, p->stream));
        HP_CUDA_TRY(cudaMemcpyAsync(p->in_paf.p, p->pin_in.p + n_conf, n_paf * sizeof(float), cudaMemcpyHostToDevice, p->stream));
        rc = launch_pipeline(p, p->in_conf.p, p->in_paf.p, N, p->stream);
        if (rc) return rc;
        rc = fetch_results(p, out, cap, n_out, N);
        if (rc != HP_ERR_CAPACITY) return rc;
        // the reference is unbounded: grow whichever internal capacity overflowed and retry
        int flags = 0;
        for (int f = 0; f < N; ++f) flags |= p->pin_counts.p[N + f];
        if (!flags) return rc; // the caller's own `cap` was too small
        if (grow_after_overflow(p, flags) != HP_OK) return rc;
    }
    return HP_ERR_CAPACITY;
}

int hp_paf_process_host(hp_paf* p, const float* conf, const float* paf, int c_conf, int c_paf, int H, int W,
                        hp_human* out, int cap, int* n_out)
{
    if (p && conf && paf && out && n_out && cudaSetDevice(p->device) == cudaSuccess) {
        const int rc = process_from_handoff(p, conf, paf, c_conf, c_paf, H, W, out, cap, n_out);
        if (rc != HANDOFF_MISS) return rc;
    }
    return hp_paf_process_host_batched(p, conf, paf, 1, c_conf, c_paf, H, W, out, cap, n_out);
}

// ---- building blocks of the pipelined end-to-end call (engine.cu: hp_pose_submit_u8_host / hp_pose_collect) ----------------
// Allocates everything a batch of this geometry needs (nothing is allocated inside a CUDA-graph capture afterwards).
int hp_paf_prepare(hp_paf* p, int N, int c_conf, int c_paf, int H, int W)
{
    if (!p) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    return ensure_geometry(p, N, c_conf, c_paf, H, W);
}
// Everything a captured launch sequence bakes in: thresholds, resolution, capacities (a change invalidates the graph).
int hp_paf_state(const hp_paf* p, float* thresholds2, int* ints6)
{
    if (!p) return HP_ERR_ARG;
    if (thresholds2) { thresholds2[0] = p->conf_thresh; thresholds2[1] = p->paf_thresh; }
    if (ints6) { ints6[0] = p->res_w; ints6[1] = p->res_h; ints6[2] = p->pcap; ints6[3] = p->ccap; ints6[4] = p->hcap; ints6[5] = p->cap_N; }
    return HP_OK;
}
// Enqueues the D2H of the last batch's records on `stream`: humans[N * hcap] and counts_flags[2N] (counts, then overflow flags)
// into caller-owned PINNED host memory; no synchronisation.
int hp_paf_copy_results_host_async(hp_paf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream)
{
    if (!p || !pin_humans || !pin_counts_flags || N != p->last_N) { hpb::set_error("hp_paf_copy_results_host_async: bad argument"); return HP_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : p->last_stream;
    HP_CUDA_TRY(cudaMemcpyAsync(pin_counts_flags, p->human_cnt(), sizeof(int) * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(pin_counts_flags + N, p->flags(), sizeof(int) * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(pin_humans, p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost, st));
    return HP_OK;
}
// After a batch whose flags (OR over its frames) report an overflow: grow those capacities (see grow_after_overflow).
int hp_paf_grow_capacity(hp_paf* p, int flags)
{
    if (!p) return HP_ERR_ARG;
    return grow_after_overflow(p, flags);
}

int hp_paf_debug_peaks(hp_paf* p, int frame, hp_peak* out, int cap, int* n_out)
{
    if (!p || frame < 0 || frame >= p->last_N || !out || !n_out) { hpb::set_error("hp_paf_debug_peaks: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaStreamSynchronize(p->last_stream));
    int base[HP_N_PARTS + 1];
    HP_CUDA_TRY(cudaMemcpy(base, p->part_base.p + (size_t)frame * (HP_N_PARTS + 1), sizeof(base), cudaMemcpyDeviceToHost));
    const int n = base[HP_N_PARTS];
    *n_out = n;
    if (n > cap) { hpb::set_error("hp_paf_debug_peaks: %d peaks > cap %d", n, cap); return HP_ERR_CAPACITY; }
    std::vector<int> x(n), y(n);
    std::vector<float> s(n);
    const size_t off = (size_t)frame * HP_N_PARTS * p->pcap;
    if (n) {
        HP_CUDA_TRY(cudaMemcpy(x.data(), p->px.p + off, n * sizeof(int), cudaMemcpyDeviceToHost));
        HP_CUDA_TRY(cudaMemcpy(y.data(), p->py.p + off, n * sizeof(int), cudaMemcpyDeviceToHost));
        HP_CUDA_TRY(cudaMemcpy(s.data(), p->pscore.p + off, n * sizeof(float), cudaMemcpyDeviceToHost));
    }
    int part = 0;
    for (int i = 0; i < n; ++i) {
        while (part < HP_N_PARTS - 1 && i >= base[part + 1]) ++part;
        out[i].part_id = part; out[i].x = x[i]; out[i].y = y[i]; out[i].score = s[i]; out[i].id = i;
    }
    return HP_OK;
}

int hp_paf_debug_connections(hp_paf* p, int frame, int pair_id, hp_connection* out, int cap, int* n_out)
{
    if (!p || frame < 0 || frame >= p->last_N || pair_id < 0 || pair_id >= HP_N_PAIRS || !out || !n_out) {
        hpb::set_error("hp_paf_debug_connections: bad argument");
        return HP_ERR_ARG;
    }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaStreamSynchronize(p->last_stream));
    int n = 0;
    HP_CUDA_TRY(cudaMemcpy(&n, p->conn_cnt() + frame * HP_N_PAIRS + pair_id, sizeof(int), cudaMemcpyDeviceToHost));
    *n_out = n;
    if (n > cap) { hpb::set_error("hp_paf_debug_connections: %d > cap %d", n, cap); return HP_ERR_CAPACITY; }
    if (n) HP_CUDA_TRY(cudaMemcpy(out, p->conn.p + ((size_t)frame * HP_N_PAIRS + pair_id) * p->pcap, n * sizeof(hp_connection), cudaMemcpyDeviceToHost));
    return HP_OK;
}

long long hp_paf_launch_count(const hp_paf* p) { return p ? p->launches : 0; }

// diagnostics (HPB_PAF_TIMING=1): %globaltimer stamps of the last batch's paf_limbs_kernel, N * (19 * 4 + 6) values
int hp_paf_debug_timing(hp_paf* p, unsigned long long* out, int N)
{
    if (!p || !out || N != p->last_N || !p->dbg_t.p) { hpb::set_error("hp_paf_debug_timing: no timing data (set HPB_PAF_TIMING=1)"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaStreamSynchronize(p->last_stream));
    HP_CUDA_TRY(cudaMemcpy(out, p->dbg_t.p, (size_t)N * (HP_N_PAIRS * 4 + 6) * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return HP_OK;
}

int hp_paf_debug_plan(hp_paf* p, int* out, int n)
{
    if (!p || !out || n < HP_PAF_PLAN_FIELDS || p->last_N == 0) {
        hpb::set_error("hp_paf_debug_plan: bad argument or nothing launched yet (need %d values)", HP_PAF_PLAN_FIELDS);
        return HP_ERR_ARG;
    }
    memcpy(out, p->plan, sizeof(p->plan));
    return HP_OK;
}

int hp_paf_copy_results_device(hp_paf* p, hp_human* d_humans, int* d_counts, int N, int cap, void* stream)
{
    if (!p || !d_humans || !d_counts || N != p->last_N || cap < p->hcap) {
        hpb::set_error("hp_paf_copy_results_device: bad argument (N=%d last=%d cap=%d hcap=%d)", N, p ? p->last_N : -1, cap, p ? p->hcap : -1);
        return HP_ERR_ARG;
    }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : p->last_stream;
    HP_CUDA_TRY(cudaMemcpy2DAsync(d_humans, (size_t)cap * sizeof(hp_human), p->humans.p, (size_t)p->hcap * sizeof(hp_human),
                                  (size_t)p->hcap * sizeof(hp_human), N, cudaMemcpyDeviceToDevice, st));
    HP_CUDA_TRY(cudaMemcpyAsync(d_counts, p->human_cnt(), sizeof(int) * N, cudaMemcpyDeviceToDevice, st));
    return HP_OK;
}

} // extern "C"
