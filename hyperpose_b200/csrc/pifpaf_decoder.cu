// pifpaf_decoder.cu -- H100 (sm_90a) OpenPifPaf decode: PIF / PAF fields -> human_t records.
//
// Replaces the reference's CPU decoder hyperpose::parser::pifpaf::process
//   src/pifpaf.cpp:7-95  +  src/pifpaf_decoder/openpifpaf_postprocessor.cpp:142-926 (SURVEY 8a A12)
// with four batched kernels (grid covers every frame of the batch):
//
//   P1 pif_hr_kernel      targetIntensities (:284-380): the high-resolution "core" confidence map of every keypoint
//                         field.  The reference zero-fills 4 x 17 x H_hr x W_hr floats and scatters Gaussians
//                         sequentially on one core; only `targetsCoreOnly` is ever consumed downstream (:669-671,
//                         the other three maps are dead), so only that one is built.  One CTA per (field, frame):
//                         cells are applied in the reference's order, but all pixels of a cell's footprint in
//                         parallel -- each pixel is always owned by the same thread, so every pixel sees exactly
//                         the reference's add / clamp sequence (bit-identical accumulation).
//   P2 pif_seeds_kernel   seed extraction (:679-706) + descending sort (:772).
//   P3 caf_filter_kernel  CAF scoring / filtering into forward and backward lists (:712-762), order preserving.
//   P4 pifpaf_grow_kernel greedy decoding (:776-799, grow :457-572, growConnectionBlend :382-437), soft NMS
//                         (:574-635), thresholds / sort (:837-851), and the 17 -> 18 keypoint remap of
//                         src/pifpaf.cpp:52-92.  One warp per frame: the CAF scans run on all 32 lanes with the
//                         reference's exact top-2 tie semantics, the small sequential state machine on lane 0.
//
// Arithmetic follows the reference expression by expression (float vs double promotion included); compiled with
// -fmad=false.  Undefined behaviour of the reference given a defined result here: negative coordinates cast to
// size_t when indexing the high-resolution map (:693, :741) are clamped to 0.
// No CPU fallback exists.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "../../include/hyperpose_b200.h"
#include "common.h"
#include "handoff.h"

namespace {

constexpr int NKP = 17, NBONE = 19;
constexpr float PP_STRIDE = 8.0f;
constexpr float SEED_THRESHOLD = 0.3f;     // :141
constexpr float INSTANCE_THRESHOLD = 0.2f; // :143

// bones, 1-based (:64-84)
__constant__ int c_bones[NBONE][2] = { { 16, 14 }, { 14, 12 }, { 17, 15 }, { 15, 13 }, { 12, 13 }, { 6, 12 }, { 7, 13 }, { 6, 7 }, { 6, 8 }, { 7, 9 },
    { 8, 10 }, { 9, 11 }, { 2, 3 }, { 1, 2 }, { 1, 3 }, { 2, 4 }, { 3, 5 }, { 4, 6 }, { 5, 7 } };
// BY_SOURCE_MAP (:91-137): for every start joint the (end joint, caf field, forward?) triples, iterated in DESCENDING end
// joint order (std::map<int, to_point, std::greater<>>)
struct Edge { int8_t end, field, fwd; };
__constant__ Edge c_edges[NKP][4] = {
    /*0*/ { { 2, 14, 1 }, { 1, 13, 1 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*1*/ { { 3, 15, 1 }, { 2, 12, 1 }, { 0, 13, 0 }, { -1, 0, 0 } },
    /*2*/ { { 4, 16, 1 }, { 1, 12, 0 }, { 0, 14, 0 }, { -1, 0, 0 } },
    /*3*/ { { 5, 17, 1 }, { 1, 15, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*4*/ { { 6, 18, 1 }, { 2, 16, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*5*/ { { 11, 5, 1 }, { 7, 8, 1 }, { 6, 7, 1 }, { 3, 17, 0 } },
    /*6*/ { { 12, 6, 1 }, { 8, 9, 1 }, { 5, 7, 0 }, { 4, 18, 0 } },
    /*7*/ { { 9, 10, 1 }, { 5, 8, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*8*/ { { 10, 11, 1 }, { 6, 9, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*9*/ { { 7, 10, 0 }, { -1, 0, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*10*/ { { 8, 11, 0 }, { -1, 0, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*11*/ { { 13, 1, 0 }, { 12, 4, 1 }, { 5, 5, 0 }, { -1, 0, 0 } },
    /*12*/ { { 14, 3, 0 }, { 11, 4, 0 }, { 6, 6, 0 }, { -1, 0, 0 } },
    /*13*/ { { 15, 0, 0 }, { 11, 1, 1 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*14*/ { { 16, 2, 0 }, { 12, 3, 1 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*15*/ { { 13, 0, 1 }, { -1, 0, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
    /*16*/ { { 14, 2, 1 }, { -1, 0, 0 }, { -1, 0, 0 }, { -1, 0, 0 } },
};

enum : int { PP_FLAG_SEEDS = 1, PP_FLAG_ANNS = 2, PP_FLAG_NMS_DIM = 4, PP_FLAG_HUMANS = 8 };

struct Geo {
    int H, W, HR, WR; // field size, high-resolution size = (H-1)*8+1 (:641-642)
};

// ---------------------------------------------------------------------------------------------
// P1: high-resolution core map
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float clipf(float v, float lo, float hi) { return fmaxf(lo, fminf(hi, v)); }

__device__ __forceinline__ float approx_exp(float x) // :224-232
{
    if (x > 2 || x < -2) return 0.f;
    x = __fadd_rn(1.f, __fdiv_rn(x, 8.f));
    x = __fmul_rn(x, x);
    x = __fmul_rn(x, x);
    x = __fmul_rn(x, x);
    return x;
}

// Qualifying cells are compacted into shared memory in chunks of at most HR_CHUNK, and each chunk is applied before the
// next is compacted: the cells still reach the map in ascending order, and the field size is not limited by shared memory.
constexpr int HR_CHUNK = 2048;

__global__ void __launch_bounds__(256) pif_hr_kernel(const float* __restrict__ pif, float* __restrict__ hr, Geo g, float v_th)
{
    __shared__ int sCells[HR_CHUNK]; // qualifying cells of this chunk, ascending (the reference's scan order)
    __shared__ int sCount, sWarpCnt[8];
    const int field = blockIdx.x, frame = blockIdx.y;
    const int hw = g.H * g.W;
    const float* p = pif + ((size_t)frame * NKP + field) * 5 * hw;
    float* map = hr + ((size_t)frame * NKP + field) * g.HR * g.WR;
    const int tid = threadIdx.x;
    for (int i = tid; i < g.HR * g.WR; i += 256) map[i] = 0.f; // vfill (:296)
    const int ty = tid >> 4, tx = tid & 15; // this thread owns the pixels with (yy % 16, xx % 16) == (ty, tx)
    for (int base = 0; base < hw;) {
        if (tid == 0) sCount = 0;
        __syncthreads(); // also orders the zero fill before the first chunk is applied (pixels are filled by other threads)
        // ordered compaction of the cells with conf > v_th (:322-330); one step adds at most 256 cells
        for (; base < hw && sCount <= HR_CHUNK - 256; base += 256) {
            const int j = base + tid;
            const bool q = j < hw && p[j] > v_th;
            const unsigned b = __ballot_sync(0xffffffffu, q);
            if ((tid & 31) == 0) sWarpCnt[tid >> 5] = __popc(b);
            __syncthreads();
            int off = sCount;
            for (int w = 0; w < (tid >> 5); ++w) off += sWarpCnt[w];
            if (q) sCells[off + __popc(b & ((1u << (tid & 31)) - 1u))] = j;
            __syncthreads();
            if (tid == 0) {
                int t = 0;
                for (int w = 0; w < 8; ++w) t += sWarpCnt[w];
                sCount += t;
            }
            __syncthreads();
        }
        const int n = sCount;
        for (int c = 0; c < n; ++c) {
            const int j = sCells[c];
            const float conf = p[j];
            const float cx = __fmul_rn(p[hw + j], PP_STRIDE);
            const float cy = __fmul_rn(p[2 * hw + j], PP_STRIDE);
            const float cs = (float)fmax(1.0, 0.5 * (double)p[4 * hw + j] * (double)PP_STRIDE); // :329 (double promotion)
            const float cv = __fmul_rn(conf, 0.0625f);                                          // v / PIF_NN (:349)
            const float tc = __fmul_rn(cs, 1.0f);                                               // truncate = 1 (:352)
            // scalarSquareAddGaussWitMax bounds (:210-213): clip in float, then truncate to integer
            const long long minx = (long long)clipf(__fsub_rn(cx, tc), 0.f, (float)(g.WR - 1));
            const long long maxx = (long long)clipf(__fadd_rn(__fadd_rn(cx, tc), 1.f), (float)(minx + 1), (float)g.WR);
            const long long miny = (long long)clipf(__fsub_rn(cy, tc), 0.f, (float)(g.HR - 1));
            const long long maxy = (long long)clipf(__fadd_rn(__fadd_rn(cy, tc), 1.f), (float)(miny + 1), (float)g.HR);
            const float tc2 = __fmul_rn(tc, tc);
            const float cs2 = __fmul_rn(cs, cs);
            long long x0 = minx + ((tx - (int)(minx & 15)) & 15);
            long long y0 = miny + ((ty - (int)(miny & 15)) & 15);
            for (long long xx = x0; xx < maxx; xx += 16) {
                const float dx = __fsub_rn((float)xx, cx), dx2 = __fmul_rn(dx, dx);
                for (long long yy = y0; yy < maxy; yy += 16) {
                    const float dy = __fsub_rn((float)yy, cy), dy2 = __fmul_rn(dy, dy);
                    const float d2 = __fadd_rn(dx2, dy2);
                    if (d2 > tc2) continue;
                    float vv;
                    if (dx2 < 0.25f && dy2 < 0.25f) vv = cv;
                    else vv = __fmul_rn(cv, approx_exp((float)(-0.5 * (double)d2 / (double)cs2))); // :233
                    float* px = map + yy * g.WR + xx;
                    *px = fminf(1.0f, __fadd_rn(*px, vv)); // += then clamp (:234-235)
                }
            }
        }
        __syncthreads(); // every thread has read sCount and sCells before the next chunk is compacted
    }
}

// ---------------------------------------------------------------------------------------------
// P2: seeds
// ---------------------------------------------------------------------------------------------
struct Seed { float v; int f; float x, y, s; };

__device__ __forceinline__ bool seed_greater(const Seed& a, const Seed& b) // std::greater on (v, f, x, y, s) tuples (:772)
{
    if (a.v != b.v) return a.v > b.v;
    if (a.f != b.f) return a.f > b.f;
    if (a.x != b.x) return a.x > b.x;
    if (a.y != b.y) return a.y > b.y;
    return a.s > b.s;
}

// (size_t)(y + 0.5) * W_hr + (size_t)(x + 0.5) (:693, :741); `fy`, `fx` already include the + 0.5 (double).
// Negative or out-of-map values are undefined behaviour in the reference (its range test compares cell units with
// high-resolution bounds); they are clamped into the map here.
__device__ __forceinline__ size_t hr_index(double fy, double fx, int HR, int WR)
{
    size_t iy = fy < 0 ? 0 : (size_t)fy, ix = fx < 0 ? 0 : (size_t)fx;
    if (iy > (size_t)(HR - 1)) iy = HR - 1;
    if (ix > (size_t)(WR - 1)) ix = WR - 1;
    return iy * WR + ix;
}

__global__ void __launch_bounds__(256) pif_seeds_kernel(const float* __restrict__ pif, const float* __restrict__ hr, Geo g,
                                                        Seed* __restrict__ raw, int* __restrict__ count, int cap, int* __restrict__ flags)
{
    __shared__ int sN;
    const int frame = blockIdx.x, tid = threadIdx.x;
    const int hw = g.H * g.W;
    if (tid == 0) sN = 0;
    __syncthreads();
    Seed* out = raw + (size_t)frame * cap;
    const float maxx = (float)(g.WR - 0.51), maxy = (float)(g.HR - 0.51); // :683 (double literal, stored as float)
    for (int i = tid; i < NKP * hw; i += 256) {
        const int f = i / hw, j = i - f * hw;
        const float* p = pif + ((size_t)frame * NKP + f) * 5 * hw;
        const float c = p[j];
        if (!(c > SEED_THRESHOLD)) continue;
        const float x = p[hw + j], y = p[2 * hw + j], s = p[4 * hw + j];
        if ((double)x < -0.49 || (double)y < -0.49 || x > maxx || y > maxy) continue; // :691
        const double fy = (double)__fmul_rn(y, PP_STRIDE) + 0.5, fx = (double)__fmul_rn(x, PP_STRIDE) + 0.5; // :693
        float v = hr[((size_t)frame * NKP + f) * g.HR * g.WR + hr_index(fy, fx, g.HR, g.WR)];
        v = (float)(0.9 * (double)v + 0.1 * (double)c); // :696
        if (v > SEED_THRESHOLD) {
            const int slot = atomicAdd(&sN, 1);
            if (slot < cap) {
                Seed sd; sd.v = v; sd.f = f; sd.x = __fmul_rn(x, PP_STRIDE); sd.y = __fmul_rn(y, PP_STRIDE); sd.s = __fmul_rn(s, PP_STRIDE);
                out[slot] = sd;
            }
        }
    }
    __syncthreads();
    if (tid == 0) {
        int n = sN;
        if (n > cap) { atomicOr(flags + frame, PP_FLAG_SEEDS); n = cap; }
        count[frame] = n;
    }
}

// descending rank sort of the seeds (std::sort(seeds, std::greater{}), :772): one thread per seed, grid (cap/256, N)
__global__ void __launch_bounds__(256) pif_seed_sort_kernel(const Seed* __restrict__ raw, Seed* __restrict__ sorted, const int* __restrict__ count, int cap)
{
    const int frame = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    const int n = count[frame];
    if (i >= n) return;
    const Seed* in = raw + (size_t)frame * cap;
    const Seed a = in[i];
    int rank = 0;
    for (int q = 0; q < n; ++q) {
        const Seed b = in[q];
        rank += (seed_greater(b, a) || (!seed_greater(a, b) && q < i)) ? 1 : 0;
    }
    sorted[(size_t)frame * cap + rank] = a;
}

// ---------------------------------------------------------------------------------------------
// P3: CAF filter -> forward / backward lists [frame][field][dir][9][hw]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) caf_filter_kernel(const float* __restrict__ paf, const float* __restrict__ hr, Geo g,
                                                         float* __restrict__ lists, int* __restrict__ counts)
{
    __shared__ int sCnt[2], sWarp[2][8];
    const int field = blockIdx.x, frame = blockIdx.y, tid = threadIdx.x;
    const int hw = g.H * g.W;
    const float* p = paf + ((size_t)frame * NBONE + field) * 9 * hw;
    const float maxx = (float)(g.WR - 0.51), maxy = (float)(g.HR - 0.51);
    const int pif_back = c_bones[field][0] - 1, pif_fwd = c_bones[field][1] - 1; // :733-734
    const int BACKWARD_IDX[9] = { 0, 3, 4, 1, 2, 6, 5, 8, 7 };                    // :736
    if (tid < 2) sCnt[tid] = 0;
    __syncthreads();
    for (int base = 0; base < hw; base += 256) {
        const int j = base + tid;
        float ch[9];
        bool pass[2] = { false, false }; // [0] backward, [1] forward
        float newv[2] = { 0.f, 0.f };
        if (j < hw && p[j] > 0.2f) {     // PAF_SCORE_THRE (:718,723)
            ch[0] = p[j];
#pragma unroll
            for (int c = 1; c < 9; ++c) ch[c] = __fmul_rn(p[(size_t)c * hw + j], PP_STRIDE); // :728-730
#pragma unroll
            for (int d = 0; d < 2; ++d) {
                const float x = d == 0 ? ch[1] : ch[3], y = d == 0 ? ch[2] : ch[4]; // this_ch[idx_mapping[3]], [4]
                if (!((double)x < -0.49 || (double)y < -0.49 || x > maxx || y > maxy)) {
                    const double fy = (double)y + 0.5, fx = (double)x + 0.5;
                    const int pf = d == 0 ? pif_back : pif_fwd;
                    const float t = hr[((size_t)frame * NKP + pf) * g.HR * g.WR + hr_index(fy, fx, g.HR, g.WR)];
                    const float nv = __fmul_rn(ch[0], __fadd_rn(0.1f, __fmul_rn(__fsub_rn(1.f, 0.1f), t))); // :744
                    if (nv > 0.2f) { pass[d] = true; newv[d] = nv; }
                }
            }
        }
#pragma unroll
        for (int d = 0; d < 2; ++d) {
            const unsigned b = __ballot_sync(0xffffffffu, pass[d]);
            if ((tid & 31) == 0) sWarp[d][tid >> 5] = __popc(b);
            __syncthreads();
            int off = sCnt[d];
            for (int w = 0; w < (tid >> 5); ++w) off += sWarp[d][w];
            if (pass[d]) {
                const int slot = off + __popc(b & ((1u << (tid & 31)) - 1u));
                float* L = lists + ((((size_t)frame * NBONE + field) * 2 + d) * 9) * hw;
#pragma unroll
                for (int c = 0; c < 9; ++c) L[(size_t)c * hw + slot] = ch[d == 0 ? BACKWARD_IDX[c] : c];
                L[slot] = newv[d]; // cont[field_i][0].back() = new_v (:751)
            }
            __syncthreads();
            if (tid == 0) {
                int t = 0;
                for (int w = 0; w < 8; ++w) t += sWarp[d][w];
                sCnt[d] += t;
            }
            __syncthreads();
        }
    }
    if (tid < 2) counts[((size_t)frame * NBONE + field) * 2 + tid] = sCnt[tid];
}

// ---------------------------------------------------------------------------------------------
// P4: greedy decode, one warp per frame
// ---------------------------------------------------------------------------------------------
struct Ann {
    float kp[NKP * 3];
    float js[NKP];
};

__device__ __forceinline__ float ann_score(const Ann& a) // openpifpaf_postprocessor.hpp:72-84
{
    float maxv = 0.f, vv = 0.f;
    for (int k = 0; k < NKP; ++k) {
        const float v = a.kp[k * 3 + 2];
        if (v > maxv) maxv = v;
        vv = __fadd_rn(vv, __fmul_rn(v, v));
    }
    return __fadd_rn(__fmul_rn(0.1f, maxv), __fdiv_rn(__fmul_rn(0.9f, vv), (float)NKP));
}

struct Blend { float x, y, s, v; };

// growConnectionBlend (:382-437) on all 32 lanes.  Sequential semantics of the reference's top-2 scan:
//   i1 = LAST index with the maximum score; (s2, i2) = best of the others where, before i1, ties prefer the LAST index
//   and, after i1, a later element replaces only if STRICTLY greater (first index of the suffix maximum); the prefix
//   wins ties against the suffix.
__device__ Blend grow_connection_blend(float x, float y, float s, const float* L, int n, int hw, int lane)
{
    const float sigma = (float)(2.0 * (double)s);
    const float sigma2 = (float)(0.25 * (double)s * (double)s);
    const float xlo = __fsub_rn(x, sigma), xhi = __fadd_rn(x, sigma), ylo = __fsub_rn(y, sigma), yhi = __fadd_rn(y, sigma);
    auto score_of = [&](int i, bool& ok) -> float {
        const float px = L[(size_t)1 * hw + i], py = L[(size_t)2 * hw + i];
        ok = !((px < xlo) || (px > xhi) || (py < ylo) || (py > yhi));
        if (!ok) return 0.f;
        const float ax = __fsub_rn(px, x), ay = __fsub_rn(py, y);
        const float d2 = __fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay));
        return (float)(exp(-0.5 * (double)d2 / (double)sigma2) * (double)L[i]); // :399 (double exp, then float)
    };
    // pass 1: maximum score and its LAST index (score >= score_1 replaces).  The scores of the first 8 entries of each
    // lane (lists up to 256 long) are kept in registers for pass 2 (the double-precision exp dominates this function).
    float cache[8]; unsigned cache_ok = 0;
    float m1 = -1.f; int i1 = -1;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int i = lane + 32 * c;
        cache[c] = 0.f;
        if (i < n) {
            bool ok; const float sc = score_of(i, ok);
            cache[c] = sc; cache_ok |= (ok ? 1u : 0u) << c;
            if (ok && (sc > m1 || (sc == m1 && i > i1))) { m1 = sc; i1 = i; }
        }
    }
    for (int i = lane + 256; i < n; i += 32) {
        bool ok; const float sc = score_of(i, ok);
        if (ok && (sc > m1 || (sc == m1 && i > i1))) { m1 = sc; i1 = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m1, o); const int oi = __shfl_xor_sync(0xffffffffu, i1, o);
        if (om > m1 || (om == m1 && oi > i1)) { m1 = om; i1 = oi; }
    }
    Blend r; r.x = r.y = r.s = r.v = 0.f;
    if (i1 < 0 || m1 == 0.f) return r; // no candidate, or score_1 == 0 (:411-412)
    // NOTE: with an initial score_1 of 0, elements scoring exactly 0 before the first positive one only shuffle the
    // zero-valued slots; they can never be selected because score_1 == 0 returns early and score_2 < 0.01 drops them.
    // pass 2: best of the others
    float mp = -1.f; int ip = -1; // prefix (i < i1): larger score, then LARGER index
    float ms = -1.f; int is = -1; // suffix (i > i1): larger score, then SMALLER index
    auto consider = [&](int i, float sc) {
        if (i < i1) { if (sc > mp || (sc == mp && i > ip)) { mp = sc; ip = i; } }
        else        { if (sc > ms || (sc == ms && (is < 0 || i < is))) { ms = sc; is = i; } }
    };
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int i = lane + 32 * c;
        if (i < n && i != i1 && ((cache_ok >> c) & 1u)) consider(i, cache[c]);
    }
    for (int i = lane + 256; i < n; i += 32) {
        if (i == i1) continue;
        bool ok; const float sc = score_of(i, ok);
        if (ok) consider(i, sc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float op = __shfl_xor_sync(0xffffffffu, mp, o); const int oip = __shfl_xor_sync(0xffffffffu, ip, o);
        if (op > mp || (op == mp && oip > ip)) { mp = op; ip = oip; }
        const float os = __shfl_xor_sync(0xffffffffu, ms, o); const int ois = __shfl_xor_sync(0xffffffffu, is, o);
        if (os > ms || (os == ms && ois >= 0 && (is < 0 || ois < is))) { ms = os; is = ois; }
    }
    float m2 = 0.f; int i2 = 0; // score_2 starts at 0 (:391)
    if (ip >= 0 && (is < 0 || mp >= ms)) { if (mp > 0.f) { m2 = mp; i2 = ip; } }
    else if (is >= 0) { if (ms > 0.f) { m2 = ms; i2 = is; } }
    const float ex1 = L[(size_t)3 * hw + i1], ey1 = L[(size_t)4 * hw + i1], es1 = L[(size_t)8 * hw + i1];
    if ((double)m2 < 0.01 || (double)m2 < 0.5 * (double)m1) { // :418
        r.x = ex1; r.y = ey1; r.s = es1; r.v = (float)((double)m1 * 0.5);
        return r;
    }
    const float ex2 = L[(size_t)3 * hw + i2], ey2 = L[(size_t)4 * hw + i2], es2 = L[(size_t)8 * hw + i2];
    const float bx = __fsub_rn(ex1, ex2), by = __fsub_rn(ey1, ey2);
    const float blend_d2 = __fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by));
    if (blend_d2 > __fdiv_rn(__fmul_rn(es1, es1), 4.f)) { // :426
        r.x = ex1; r.y = ey1; r.s = es1; r.v = (float)((double)m1 * 0.5);
        return r;
    }
    const float den = __fadd_rn(m1, m2);
    r.x = __fdiv_rn(__fadd_rn(__fmul_rn(m1, ex1), __fmul_rn(m2, ex2)), den);
    r.y = __fdiv_rn(__fadd_rn(__fmul_rn(m1, ey1), __fmul_rn(m2, ey2)), den);
    r.s = __fdiv_rn(__fadd_rn(__fmul_rn(m1, es1), __fmul_rn(m2, es2)), den);
    r.v = (float)(0.5 * (double)den);
    return r;
}

struct Occ { // Occupancy (:20-60)
    uint8_t* m; int d0, d1, d2;
    __device__ bool get(size_t a, size_t b, size_t c) const { return m[((size_t)d1 * d2) * a + (size_t)d2 * b + c] != 0; }
    __device__ bool fuzz_get(int f, float y, float x) const
    {
        if (f >= d0) return true;
        const float xx = fminf((float)d2 - 1.f, fmaxf(0.f, __fdiv_rn(x, 2.f)));
        const float yy = fminf((float)d1 - 1.f, fmaxf(0.f, __fdiv_rn(y, 2.f)));
        return get((size_t)f, (size_t)yy, (size_t)xx);
    }
};

// scalarSquareAddSingle (:245-277), the rectangle filled by all lanes
__device__ void occ_add(Occ& o, int f, int fieldH, int fieldW, float x, float y, float width, float reduction, float min_scaled, int lane)
{
    if (reduction != 1.0f) {
        x = __fdiv_rn(x, reduction); y = __fdiv_rn(y, reduction);
        width = fmaxf(min_scaled, __fdiv_rn(width, reduction));
    }
    const int minx = min(fieldW - 1, max(0, (int)__fsub_rn(x, width)));
    const int miny = min(fieldH - 1, max(0, (int)__fsub_rn(y, width)));
    const int maxx = min(fieldW, max(minx + 1, min(fieldW, (int)__fadd_rn(x, width) + 1)));
    const int maxy = min(fieldH, max(miny + 1, min(fieldH, (int)__fadd_rn(y, width) + 1)));
    const int w = maxx - minx, n = w * (maxy - miny);
    for (int i = lane; i < n; i += 32) {
        const int yy = miny + i / w, xx = minx + i % w;
        o.m[((size_t)o.d1 * o.d2) * f + (size_t)o.d2 * yy + xx] = 1;
    }
}

struct GrowParams {
    Geo g;
    const Seed* seeds; const int* seed_cnt; int seed_cap;
    const float* lists; const int* list_cnt;
    uint8_t* occ_grow;   // [N][17][HR][WR]
    uint8_t* occ_nms;    // [N][17][nms_h][nms_w]
    int nms_h, nms_w;
    Ann* anns; int ann_cap; // [N][ann_cap]
    float keypoint_thresh;
    int net_h, net_w;
    hp_human* humans; int hcap; int* human_cnt; int* flags;
    int* dbg; // [N][4]: annotations grown, kept after thresholds, NMS map h, w
};

struct QItem { float score; int has; float x, y, s, v; int start, end; };

__global__ void __launch_bounds__(32) pifpaf_grow_kernel(const GrowParams p)
{
    __shared__ QItem q[96];     // frontier: every directed edge at most once as placeholder and once scored
    __shared__ int order[512];  // sort permutations
    __shared__ Ann sAnn;        // the annotation being grown (copied to global memory when finished)
    const int frame = blockIdx.x, lane = threadIdx.x;
    const Geo g = p.g;
    const int hw = g.H * g.W;
    const Seed* seeds = p.seeds + (size_t)frame * p.seed_cap;
    const int n_seeds = p.seed_cnt[frame];
    Occ og; og.m = p.occ_grow + (size_t)frame * NKP * g.HR * g.WR; og.d0 = NKP; og.d1 = g.HR; og.d2 = g.WR;
    Ann* anns = p.anns + (size_t)frame * p.ann_cap;
    int n_ann = 0;
    auto list_of = [&](int field, int fwd) { return p.lists + ((((size_t)frame * NBONE + field) * 2 + fwd) * 9) * hw; };
    auto count_of = [&](int field, int fwd) { return p.list_cnt[((size_t)frame * NBONE + field) * 2 + fwd]; };

    for (int si = 0; si < n_seeds; ++si) {
        const Seed sd = seeds[si];
        if (og.fuzz_get(sd.f, sd.y, sd.x)) continue; // :779 (warp-uniform)
        if (n_ann >= p.ann_cap) { if (lane == 0) atomicOr(p.flags + frame, PP_FLAG_ANNS); break; }
        Ann& ann = sAnn;
        if (lane == 0) {
            for (int i = 0; i < NKP * 3; ++i) ann.kp[i] = 0.f;
            for (int i = 0; i < NKP; ++i) ann.js[i] = 0.f;
            ann.kp[sd.f * 3] = sd.x; ann.kp[sd.f * 3 + 1] = sd.y; ann.kp[sd.f * 3 + 2] = sd.v;
            ann.js[sd.f] = sd.s;
        }
        __syncwarp();
        // ---- grow (:457-572) ----
        int nq = 0;                         // live frontier entries (warp-uniform copy)
        unsigned long long in_frontier[NKP]; // bit end_i of word start_i (lane-local copies stay identical)
        for (int i = 0; i < NKP; ++i) in_frontier[i] = 0ull;
        auto add_to_frontier = [&](int start_i) {
            for (int e = 0; e < 4; ++e) {
                const Edge ed = c_edges[start_i][e];
                if (ed.end < 0) break;
                if (ann.kp[3 * ed.end + 2] > 0.0f) continue;
                if ((in_frontier[start_i] >> ed.end) & 1ull) continue;
                if (nq < 96) {
                    if (lane == 0) {
                        QItem it; it.score = sqrtf(ann.kp[3 * start_i + 2]); it.has = 0; it.x = it.y = it.s = it.v = 0.f; it.start = start_i; it.end = ed.end;
                        q[nq] = it;
                    }
                    ++nq;
                }
                in_frontier[start_i] |= 1ull << ed.end;
            }
            __syncwarp();
        };
        for (int j = 0; j < NKP; ++j)
            if (ann.kp[3 * j + 2] != 0.0f) add_to_frontier(j);
        for (;;) {
            // frontier_get (:488-546): pop the entry with the largest score (priority = -score)
            bool got = false; QItem cur;
            while (nq > 0) {
                int best = 0;
                for (int i = 1; i < nq; ++i) if (q[i].score > q[best].score) best = i;
                cur = q[best];
                __syncwarp();
                if (lane == 0) q[best] = q[nq - 1];
                --nq;
                __syncwarp();
                if (cur.has) { got = true; break; }
                if (ann.kp[cur.end * 3 + 2] > 0.0f) continue;
                // connection value (:506-538)
                Edge ed; ed.end = -1; ed.field = 0; ed.fwd = 0;
                for (int e = 0; e < 4; ++e) if (c_edges[cur.start][e].end == cur.end) ed = c_edges[cur.start][e];
                const float x = ann.kp[cur.start * 3], y = ann.kp[cur.start * 3 + 1], v = ann.kp[cur.start * 3 + 2];
                const float xy_scale_s = fmaxf(0.f, ann.js[cur.start]);
                const Blend nb = grow_connection_blend(x, y, xy_scale_s, list_of(ed.field, ed.fwd ? 1 : 0), count_of(ed.field, ed.fwd ? 1 : 0), hw, lane);
                if (nb.v == 0.f) continue;
                const float kscore = sqrtf(__fmul_rn(nb.v, v));
                if (kscore < p.keypoint_thresh) continue;
                if (kscore < __fmul_rn(v, 0.5f)) continue;
                const float xy_scale_t = fmaxf(0.f, nb.s);
                const Blend rb = grow_connection_blend(nb.x, nb.y, xy_scale_t, list_of(ed.field, ed.fwd ? 0 : 1), count_of(ed.field, ed.fwd ? 0 : 1), hw, lane);
                if (rb.s == 0.f || __fadd_rn(fabsf(__fsub_rn(x, rb.x)), fabsf(__fsub_rn(y, rb.y))) > xy_scale_s) continue;
                if (nq < 96) {
                    if (lane == 0) {
                        QItem it; it.score = kscore; it.has = 1; it.x = nb.x; it.y = nb.y; it.s = nb.s; it.v = kscore; it.start = cur.start; it.end = cur.end;
                        q[nq] = it;
                    }
                    ++nq;
                }
                __syncwarp();
            }
            if (!got) break;
            const bool taken = ann.kp[cur.end * 3 + 2] > 0.0f;
            __syncwarp();   // every lane has read the slot before lane 0 may fill it
            if (taken) continue;
            if (lane == 0) {
                ann.kp[cur.end * 3] = cur.x; ann.kp[cur.end * 3 + 1] = cur.y; ann.kp[cur.end * 3 + 2] = cur.v;
                ann.js[cur.end] = cur.s;
            }
            __syncwarp();
            add_to_frontier(cur.end);
        }
        // ---- mark occupancy (:787-798) ----
        for (int i = 0; i < NKP; ++i) {
            if (ann.kp[i * 3 + 2] == 0.f) continue;
            occ_add(og, i, g.HR, g.WR, ann.kp[i * 3], ann.kp[i * 3 + 1], ann.js[i], 2.f, 2.f, lane);
        }
        __syncwarp();
        for (int i = lane; i < NKP * 3; i += 32) anns[n_ann].kp[i] = sAnn.kp[i];
        if (lane < NKP) anns[n_ann].js[lane] = sAnn.js[lane];
        __syncwarp();
        ++n_ann;
    }

    if (lane == 0) p.dbg[frame * 4 + 0] = n_ann;
    // ---- soft NMS (:574-635) ----
    int n_keep = 0;
    if (n_ann > 0) {
        float mx = 0.f, my = 0.f;
        for (int a = 0; a < n_ann; ++a)
            for (int k = 0; k < NKP; ++k) { mx = fmaxf(mx, anns[a].kp[k * 3]); my = fmaxf(my, anns[a].kp[k * 3 + 1]); }
        const int h = (int)__fadd_rn(my, 1.f), w = (int)__fadd_rn(mx, 1.f);
        if (lane == 0) { p.dbg[frame * 4 + 2] = h; p.dbg[frame * 4 + 3] = w; }
        if (h > p.nms_h || w > p.nms_w || n_ann > 512) {
            if (lane == 0) atomicOr(p.flags + frame, PP_FLAG_NMS_DIM);
            if (lane == 0) p.human_cnt[frame] = 0;
            return;
        }
        Occ on; on.m = p.occ_nms + (size_t)frame * NKP * p.nms_h * p.nms_w; on.d0 = NKP; on.d1 = h; on.d2 = w;
        // sorted by score, descending (std::sort :592; ties between distinct annotations are not expected)
        if (lane == 0) {
            for (int a = 0; a < n_ann; ++a) order[a] = a;
            for (int a = 1; a < n_ann; ++a) { // insertion sort (stable)
                const int key = order[a]; const float ks = ann_score(anns[key]);
                int b = a - 1;
                while (b >= 0 && ann_score(anns[order[b]]) < ks) { order[b + 1] = order[b]; --b; }
                order[b + 1] = key;
            }
        }
        __syncwarp();
        for (int oi = 0; oi < n_ann; ++oi) {
            Ann& ann = anns[order[oi]];
            for (int k = 0; k < NKP; ++k) {
                const float x = ann.kp[k * 3], y = ann.kp[k * 3 + 1], v = ann.kp[k * 3 + 2];
                if (v == 0.f) continue;
                const int i = min(max(0, (int)roundf(x)), w - 1), j = min(max(0, (int)roundf(y)), h - 1);
                if (on.fuzz_get(k, (float)j, (float)i)) {
                    __syncwarp();
                    if (lane == 0) ann.kp[k * 3 + 2] = 0.0f;
                    __syncwarp();
                } else {
                    occ_add(on, k, h, w, x, y, ann.js[k], 1.f, 0.f, lane);
                    __syncwarp();
                }
            }
        }
    }
    // ---- threshold (:837-847), sort (:849-851), convert (:876-925 + src/pifpaf.cpp:52-92) ----
    if (lane == 0) {
        for (int a = 0; a < n_ann; ++a) {
            bool any = false;
            for (int k = 0; k < NKP; ++k) if (anns[a].kp[k * 3 + 2] > 0.0f) any = true; // softNMS `filtered`
            if (!any) continue;
            for (int k = 0; k < NKP; ++k) if (anns[a].kp[k * 3 + 2] < p.keypoint_thresh) anns[a].kp[k * 3 + 2] = 0.0f;
            if (ann_score(anns[a]) >= INSTANCE_THRESHOLD) order[n_keep++] = a;
        }
        for (int a = 1; a < n_keep; ++a) {
            const int key = order[a]; const float ks = ann_score(anns[key]);
            int b = a - 1;
            while (b >= 0 && ann_score(anns[order[b]]) < ks) { order[b + 1] = order[b]; --b; }
            order[b + 1] = key;
        }
        const int from_index[16] = { 6, 8, 10, 5, 7, 9, 12, 14, 16, 11, 13, 15, 2, 1, 4, 3 }; // pifpaf.cpp:73-77
        int n_out = 0;
        for (int oi = 0; oi < n_keep; ++oi) {
            if (n_out >= p.hcap) { atomicOr(p.flags + frame, PP_FLAG_HUMANS); break; }
            const Ann& ann = anns[order[oi]];
            hp_human* o = p.humans + (size_t)frame * p.hcap + n_out++;
            o->score = ann_score(ann);
            for (int k = 0; k < HP_N_PARTS; ++k) { o->parts[k].has_value = 0; o->parts[k].x = o->parts[k].y = o->parts[k].score = 0.f; }
            auto p2p = [&](int src, int dst) {
                const float v = ann.kp[src * 3 + 2];
                if ((double)v > 0.) {
                    const int xi = (int)ann.kp[src * 3], yi = (int)ann.kp[src * 3 + 1]; // truncated to int pixels (:888-889)
                    o->parts[dst].score = 1.f;
                    o->parts[dst].x = __fdiv_rn((float)xi, (float)p.net_w);
                    o->parts[dst].y = __fdiv_rn((float)yi, (float)p.net_h);
                    o->parts[dst].has_value = 1;
                }
            };
            p2p(0, 0);
            for (int i = 0; i < 16; ++i) p2p(from_index[i], i + 2);
            if (o->parts[2].has_value && o->parts[5].has_value) { // neck = mean of the shoulders (pifpaf.cpp:83-90)
                o->parts[1].x = __fdiv_rn(__fadd_rn(o->parts[2].x, o->parts[5].x), 2.f);
                o->parts[1].y = __fdiv_rn(__fadd_rn(o->parts[2].y, o->parts[5].y), 2.f);
                o->parts[1].has_value = 1;
                o->parts[1].score = __fdiv_rn(__fadd_rn(o->parts[2].score, o->parts[5].score), 2.f);
            }
        }
        p.human_cnt[frame] = n_out;
        p.dbg[frame * 4 + 1] = n_keep;
    }
}

template <typename T> struct DBuf {
    T* p = nullptr; size_t n = 0;
    cudaError_t ensure(size_t c) { if (c <= n) return cudaSuccess; if (p) cudaFree(p); p = nullptr; n = 0; cudaError_t e = cudaMalloc(&p, c * sizeof(T)); if (e == cudaSuccess) { n = c; e = cudaMemset(p, 0, c * sizeof(T)); }
        // the memset runs on the legacy default stream, the parser's work on a NON-BLOCKING stream: without this the zero fill can
        // land after the first copy / kernel that uses the new buffer
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        return e; }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

} // namespace

struct hp_pifpaf {
    int device = 0, net_h = 0, net_w = 0;
    float thresh = 0.1f;
    cudaStream_t stream = nullptr;
    int seed_cap = 8192, ann_cap = 256, hcap = 128;
    int N = 0, H = 0, W = 0;
    DBuf<float> hr, lists, in_pif, in_paf;
    DBuf<Seed> seeds_raw, seeds;
    DBuf<int> counters; // [N seed_cnt | N*19*2 list_cnt | N human_cnt | N flags | N*4 dbg]
    DBuf<uint8_t> occ_grow, occ_nms;
    DBuf<Ann> anns;
    DBuf<hp_human> humans;
    std::vector<hp_human> host_h; std::vector<int> host_c;
    long long launches = 0;
    int last_N = 0;
    cudaEvent_t inputs_free = nullptr;   // recorded behind the last kernel that reads the field tensors (the greedy growth reads the decoder's own lists)
};

extern "C" {

// pifpaf::pifpaf(int h, int w, float thresh) (include/hyperpose/operator/parser/pifpaf.hpp:10-13): network input size + keypoint threshold
int hp_pifpaf_create(hp_pifpaf** out, int net_h, int net_w, float thresh, int device)
{
    if (!out) return HP_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); hpb::set_error("hp_pifpaf_create: no CUDA device (this library has no CPU fallback)"); return HP_ERR_CUDA; }
    if (device < 0 || device >= ndev || net_h <= 0 || net_w <= 0) { hpb::set_error("hp_pifpaf_create: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(device));
    hp_pifpaf* p = new hp_pifpaf();
    p->device = device; p->net_h = net_h; p->net_w = net_w; p->thresh = thresh;
    if (cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) != cudaSuccess) { delete p; hpb::set_error("cudaStreamCreate failed"); return HP_ERR_CUDA; }
    *out = p;
    return HP_OK;
}

void hp_pifpaf_destroy(hp_pifpaf* p)
{
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) { cudaStreamSynchronize(p->stream); cudaStreamDestroy(p->stream); }
    if (p->inputs_free) cudaEventDestroy(p->inputs_free);
    p->hr.release(); p->lists.release(); p->in_pif.release(); p->in_paf.release(); p->seeds_raw.release(); p->seeds.release();
    p->counters.release(); p->occ_grow.release(); p->occ_nms.release(); p->anns.release(); p->humans.release();
    delete p;
}

// pifpaf::process for N frames with DEVICE tensors pif[N,17,5,h,w], paf[N,19,9,h,w]; results fetched by hp_pifpaf_fetch
int hp_pifpaf_process_device(hp_pifpaf* p, const float* d_pif, const float* d_paf, int N, int h, int w, void* stream)
{
    if (!p || !d_pif || !d_paf || N <= 0 || h <= 1 || w <= 1) { hpb::set_error("hp_pifpaf_process_device: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : p->stream;
    Geo g; g.H = h; g.W = w; g.HR = (h - 1) * 8 + 1; g.WR = (w - 1) * 8 + 1;
    const size_t hr_px = (size_t)g.HR * g.WR, hw = (size_t)h * w;
    const int nms_h = g.HR + 256, nms_w = g.WR + 256;
    HP_CUDA_TRY(p->hr.ensure((size_t)N * NKP * hr_px));
    HP_CUDA_TRY(p->lists.ensure((size_t)N * NBONE * 2 * 9 * hw));
    HP_CUDA_TRY(p->seeds_raw.ensure((size_t)N * p->seed_cap));
    HP_CUDA_TRY(p->seeds.ensure((size_t)N * p->seed_cap));
    HP_CUDA_TRY(p->counters.ensure((size_t)N * (1 + NBONE * 2 + 2 + 4)));
    HP_CUDA_TRY(p->occ_grow.ensure((size_t)N * NKP * hr_px));
    HP_CUDA_TRY(p->occ_nms.ensure((size_t)N * NKP * nms_h * nms_w));
    HP_CUDA_TRY(p->anns.ensure((size_t)N * p->ann_cap));
    HP_CUDA_TRY(p->humans.ensure((size_t)N * p->hcap));
    int* seed_cnt = p->counters.p;
    int* list_cnt = seed_cnt + N;
    int* human_cnt = list_cnt + (size_t)N * NBONE * 2;
    int* flags = human_cnt + N;
    HP_CUDA_TRY(cudaMemsetAsync(p->counters.p, 0, (size_t)N * (1 + NBONE * 2 + 2 + 4) * sizeof(int), st));
    HP_CUDA_TRY(cudaMemsetAsync(p->occ_grow.p, 0, (size_t)N * NKP * hr_px, st));
    HP_CUDA_TRY(cudaMemsetAsync(p->occ_nms.p, 0, (size_t)N * NKP * nms_h * nms_w, st));
    pif_hr_kernel<<<dim3(NKP, N), 256, 0, st>>>(d_pif, p->hr.p, g, 0.1f);
    pif_seeds_kernel<<<N, 256, 0, st>>>(d_pif, p->hr.p, g, p->seeds_raw.p, seed_cnt, p->seed_cap, flags);
    pif_seed_sort_kernel<<<dim3((p->seed_cap + 255) / 256, N), 256, 0, st>>>(p->seeds_raw.p, p->seeds.p, seed_cnt, p->seed_cap);
    caf_filter_kernel<<<dim3(NBONE, N), 256, 0, st>>>(d_paf, p->hr.p, g, p->lists.p, list_cnt);
    if (!p->inputs_free) HP_CUDA_TRY(cudaEventCreateWithFlags(&p->inputs_free, cudaEventDisableTiming));
    HP_CUDA_TRY(cudaEventRecord(p->inputs_free, st));   // d_pif / d_paf may be overwritten from here on (pipelined callers wait for this, not for the growth)
    GrowParams gp;
    gp.g = g; gp.seeds = p->seeds.p; gp.seed_cnt = seed_cnt; gp.seed_cap = p->seed_cap; gp.lists = p->lists.p; gp.list_cnt = list_cnt;
    gp.occ_grow = p->occ_grow.p; gp.occ_nms = p->occ_nms.p; gp.nms_h = nms_h; gp.nms_w = nms_w; gp.anns = p->anns.p; gp.ann_cap = p->ann_cap;
    gp.keypoint_thresh = p->thresh; gp.net_h = p->net_h; gp.net_w = p->net_w; gp.humans = p->humans.p; gp.hcap = p->hcap; gp.human_cnt = human_cnt; gp.flags = flags; gp.dbg = flags + N;
    pifpaf_grow_kernel<<<N, 32, 0, st>>>(gp);
    HP_CUDA_TRY(cudaGetLastError());
    p->launches += 5;
    p->N = N; p->H = h; p->W = w; p->last_N = N;
    return HP_OK;
}

int hp_pifpaf_fetch(hp_pifpaf* p, hp_human* out, int cap, int* n_out, int N)
{
    if (!p || !out || !n_out || N != p->last_N) { hpb::set_error("hp_pifpaf_fetch: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaDeviceSynchronize());
    p->host_h.resize((size_t)N * p->hcap); p->host_c.resize((size_t)N * 2);
    int* human_cnt = p->counters.p + N + (size_t)N * NBONE * 2;
    HP_CUDA_TRY(cudaMemcpy(p->host_c.data(), human_cnt, sizeof(int) * 2 * N, cudaMemcpyDeviceToHost));
    HP_CUDA_TRY(cudaMemcpy(p->host_h.data(), p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost));
    int fl = 0;
    for (int f = 0; f < N; ++f) fl |= p->host_c[N + f];
    if (fl) { hpb::set_error("hp_pifpaf: internal capacity exceeded (flags=%d: 1 seeds>%d, 2 annotations>%d, 4 NMS map, 8 humans>%d)", fl, p->seed_cap, p->ann_cap, p->hcap); return HP_ERR_CAPACITY; }
    for (int f = 0; f < N; ++f) {
        const int n = p->host_c[f];
        if (n > cap) { hpb::set_error("hp_pifpaf: frame %d has %d humans but the caller's capacity is %d", f, n, cap); return HP_ERR_CAPACITY; }
        n_out[f] = n;
        memcpy(out + (size_t)f * cap, p->host_h.data() + (size_t)f * p->hcap, sizeof(hp_human) * n);
    }
    return HP_OK;
}

// Published-batch path (handoff.h): `pif` / `paf` are host buffers the engine filled and published -> decode the whole
// batch once from the device snapshot, serve the other frames from the cached records.  Returns 1 on a miss.
static int pifpaf_from_handoff(hp_pifpaf* p, const float* pif, const float* paf, int h, int w, hp_human* out, int cap, int* n_out)
{
    namespace ho = hpb::handoff;
    if (h <= 1 || w <= 1) return 1;
    const size_t ea = (size_t)NKP * 5 * h * w, eb = (size_t)NBONE * 9 * h * w;
    ho::Hit hit = ho::lookup(pif, paf, ea, eb);
    if (!hit.batch) return 1;
    ho::Batch& b = *hit.batch;
    std::lock_guard<std::mutex> lk(b.mu);
    const int f = hit.frame;
    if (!b.valid || b.fail_count >= 2 || b.device != p->device || f >= b.N || b.host_a[f] != pif || b.host_b[f] != paf ||
        b.elems_a != ea || b.elems_b != eb || !ho::contents_match(b, f)) {
        ho::count_miss();
        return 1;
    }
    const bool cached = b.cache_kind == 2 && b.key_f[0] == p->thresh && b.key_i[0] == p->net_h && b.key_i[1] == p->net_w;
    if (!cached) {
        b.cache_kind = 0;
        HP_CUDA_TRY(cudaStreamWaitEvent(p->stream, b.ready, 0));
        int rc = hp_pifpaf_process_device(p, b.d_a, b.d_b, b.N, h, w, p->stream);
        if (rc) return rc;
        b.humans.resize((size_t)b.N * p->hcap);
        b.counts.resize(b.N);
        rc = hp_pifpaf_fetch(p, b.humans.data(), p->hcap, b.counts.data(), b.N);
        if (rc == HP_ERR_CAPACITY) { b.fail_count++; ho::count_miss(); return 1; }
        if (rc) return rc;
        b.cache_kind = 2;
        b.key_f[0] = p->thresh; b.key_f[1] = 0.f; b.key_i[0] = p->net_h; b.key_i[1] = p->net_w;
        b.hcap = p->hcap;
        ho::count_batch_parse();
    }
    const int n = b.counts[f];
    if (n > cap) { hpb::set_error("hp_pifpaf: frame has %d humans but the caller's capacity is %d", n, cap); return HP_ERR_CAPACITY; }
    memcpy(out, b.humans.data() + (size_t)f * b.hcap, sizeof(hp_human) * n);
    *n_out = n;
    ho::count_hit();
    return HP_OK;
}

// pifpaf::process(pif, paf) (pifpaf.hpp:14; src/pifpaf.cpp:7-95) with HOST tensors, N frames
int hp_pifpaf_process_host(hp_pifpaf* p, const float* pif, const float* paf, int N, int h, int w, hp_human* out, int cap, int* n_out)
{
    if (!p || !pif || !paf || !out || !n_out || N <= 0) { hpb::set_error("hp_pifpaf_process_host: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    if (N == 1) {
        const int rc = pifpaf_from_handoff(p, pif, paf, h, w, out, cap, n_out);
        if (rc != 1) return rc;
    }
    const size_t n_pif = (size_t)N * NKP * 5 * h * w, n_paf = (size_t)N * NBONE * 9 * h * w;
    HP_CUDA_TRY(p->in_pif.ensure(n_pif));
    HP_CUDA_TRY(p->in_paf.ensure(n_paf));
    HP_CUDA_TRY(cudaMemcpyAsync(p->in_pif.p, pif, n_pif * sizeof(float), cudaMemcpyHostToDevice, p->stream));
    HP_CUDA_TRY(cudaMemcpyAsync(p->in_paf.p, paf, n_paf * sizeof(float), cudaMemcpyHostToDevice, p->stream));
    for (int attempt = 0; attempt < 5; ++attempt) {
        int rc = hp_pifpaf_process_device(p, p->in_pif.p, p->in_paf.p, N, h, w, p->stream);
        if (rc) return rc;
        rc = hp_pifpaf_fetch(p, out, cap, n_out, N);
        if (rc != HP_ERR_CAPACITY) return rc;
        // the reference decoder is unbounded (std::vector): grow the internal capacity that overflowed and decode again
        int fl = 0;
        for (int f = 0; f < N; ++f) fl |= p->host_c[N + f];
        if (!(fl & (1 | 2 | 8))) return rc;   // the caller's own `cap`, or the fixed NMS map
        if (fl & 1) p->seed_cap *= 4;
        if (fl & 2) p->ann_cap *= 4;
        if (fl & 8) p->hcap *= 4;
        if (p->seed_cap > (1 << 20) || p->ann_cap > (1 << 18) || p->hcap > (1 << 16)) return rc;
    }
    return HP_ERR_CAPACITY;
}

long long hp_pifpaf_launch_count(const hp_pifpaf* p) { return p ? p->launches : 0; }

// ---- building blocks of the pipelined end-to-end call (engine.cu: hp_pose_submit_pifpaf_u8_host / hp_pose_collect) ----
// the decoder's own stream, the event recorded once the field tensors of the last hp_pifpaf_process_device call have been consumed
// (NULL before the first call), and the per-frame human capacity of the result buffer
int hp_pifpaf_pipeline_info(hp_pifpaf* p, void** stream, void** inputs_free_event, int* hcap)
{
    if (!p) return HP_ERR_ARG;
    if (stream) *stream = (void*)p->stream;
    if (inputs_free_event) *inputs_free_event = (void*)p->inputs_free;
    if (hcap) *hcap = p->hcap;
    return HP_OK;
}
// Enqueues the D2H of the last batch's records on `stream`: humans[N * hcap] and counts_flags[2N] (counts, then overflow flags)
// into caller-owned PINNED host memory; no synchronisation.
int hp_pifpaf_copy_results_host_async(hp_pifpaf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream)
{
    if (!p || !pin_humans || !pin_counts_flags || N != p->last_N) { hpb::set_error("hp_pifpaf_copy_results_host_async: bad argument"); return HP_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : p->stream;
    const int* human_cnt = p->counters.p + N + (size_t)N * NBONE * 2;   // [N counts | N flags] are adjacent
    HP_CUDA_TRY(cudaMemcpyAsync(pin_counts_flags, human_cnt, sizeof(int) * 2 * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(pin_humans, p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost, st));
    return HP_OK;
}
// After a batch whose flags (OR over its frames) report an overflow: grow those capacities like hp_pifpaf_process_host does.
int hp_pifpaf_grow_capacity(hp_pifpaf* p, int flags)
{
    if (!p) return HP_ERR_ARG;
    if (!(flags & (1 | 2 | 8))) return HP_ERR_CAPACITY;   // the fixed NMS map
    if (flags & 1) p->seed_cap *= 4;
    if (flags & 2) p->ann_cap *= 4;
    if (flags & 8) p->hcap *= 4;
    if (p->seed_cap > (1 << 20) || p->ann_cap > (1 << 18) || p->hcap > (1 << 16)) return HP_ERR_CAPACITY;
    return HP_OK;
}

// test hook: the high-resolution core map of (frame, field) of the last call, HR x WR floats
int hp_pifpaf_debug_hr(hp_pifpaf* p, int frame, int field, float* out)
{
    if (!p || !out || frame < 0 || frame >= p->last_N || field < 0 || field >= NKP) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaDeviceSynchronize());
    const size_t hr_px = (size_t)((p->H - 1) * 8 + 1) * ((p->W - 1) * 8 + 1);
    HP_CUDA_TRY(cudaMemcpy(out, p->hr.p + ((size_t)frame * NKP + field) * hr_px, hr_px * sizeof(float), cudaMemcpyDeviceToHost));
    return HP_OK;
}

// test hook: per-frame counters of the last call: out[0] seeds, out[1] annotations grown, out[2] kept after thresholds,
// out[3] flags, out[4..5] NMS map h, w, out[6] sum of CAF list lengths
int hp_pifpaf_debug_counts(hp_pifpaf* p, int frame, int* out)
{
    if (!p || !out || frame < 0 || frame >= p->last_N) return HP_ERR_ARG;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaDeviceSynchronize());
    const int N = p->last_N;
    std::vector<int> c((size_t)N * (1 + NBONE * 2 + 2 + 4));
    HP_CUDA_TRY(cudaMemcpy(c.data(), p->counters.p, c.size() * sizeof(int), cudaMemcpyDeviceToHost));
    const int* list_cnt = c.data() + N; const int* human_cnt = list_cnt + (size_t)N * NBONE * 2; const int* flags = human_cnt + N; const int* dbg = flags + N;
    out[0] = c[frame]; out[1] = dbg[frame * 4]; out[2] = dbg[frame * 4 + 1]; out[3] = flags[frame]; out[4] = dbg[frame * 4 + 2]; out[5] = dbg[frame * 4 + 3];
    int t = 0;
    for (int i = 0; i < NBONE * 2; ++i) t += list_cnt[(size_t)frame * NBONE * 2 + i];
    out[6] = t;
    return HP_OK;
}

} // extern "C"
