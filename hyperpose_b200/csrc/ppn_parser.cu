// ppn_parser.cu -- Pose Proposal Network parser on the GPU: hyperpose::parser::pose_proposal::process
// (src/pose_proposal.cpp:68-337) for a batch of frames, one CTA per frame, everything in shared memory.
//
// The reference algorithm is four short, order-dependent stages over tiny tensors ([18,12,12] boxes, [17,9,9,12,12]
// edges, 0.86 MB/frame); the work per frame is far too small to spread over the device, so the batch is the parallel
// axis (frame f = blockIdx.x) and inside a CTA only the data-parallel parts are spread over the threads:
//   A. threshold + box decode + sort            (:136-152,:104-106)  warp per key-point type, rank sort
//   B. box NMS with the reference's skipping scan (:117-123)          same warp; IoUs in parallel, scan by lane 0
//   C. per limb: candidate edges (:186-211) by all threads -> bitonic sort of 64-bit keys (:223-225) -> the
//      root/attach pass (:231-268), which is inherently sequential (thread 0)
//   D. duplicate merge through the 64 x 64 spatial hash (:275-326), sequential, linked cell lists in smem
// Results are bit-identical to the reference: all arithmetic that reaches the output is integer box arithmetic plus
// one IEEE fp32 division per coordinate (__fdiv_rn), and the two unstable std::sort calls are frozen to
// (conf, grid index) / (conf, from_index * n_neighbors + neighbor) -- see oracle/ppn_oracle.py.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <mutex>
#include <type_traits>
#include <vector>

#include "../../include/hyperpose_b200.h"
#include "common.h"

namespace {

constexpr int NPARTS = 18;
constexpr int NPAIRS = 17;
constexpr int THREADS = 256;
constexpr int NWARPS = THREADS / 32;
constexpr int HASH = 64;          // :275
// Capacities of the sequential stages (the reference is unbounded).  The fast variant keeps humans and hash-cell
// registrations in shared memory; when a frame overflows them (very low thresholds: every candidate whose two boxes are
// both rooted opens a new human, :240-243) the host re-runs the batch with the spill variant, which keeps them in a
// per-frame global scratch area.
constexpr int CAP_H = 512, CAP_ENT = 8192;                 // shared-memory variant
constexpr int SPILL_CAP_H = 16384, SPILL_CAP_ENT = 262144; // global-scratch variant (positions must fit the reference's uint16_t ids)

// src/pose_proposal.cpp:24-42
__constant__ int8_t c_pair[NPAIRS][2] = { { 1, 8 }, { 8, 9 }, { 9, 10 }, { 1, 11 }, { 11, 12 }, { 12, 13 }, { 1, 2 }, { 2, 3 }, { 3, 4 },
    { 1, 5 }, { 5, 6 }, { 6, 7 }, { 1, 0 }, { 0, 14 }, { 0, 15 }, { 14, 16 }, { 15, 17 } };

struct __align__(16) Box {
    short x, y, w, h;   // cv::Rect clamped to [0, net] (:143-146)
    float conf;
    short grid;         // cell index gy * gw + gx
    short root;         // meta_info::human_index (:91-99)
};

struct PpnParams {
    const float *conf, *x, *y, *w, *h, *edge;
    int K, gh, gw, E, nh, nw, net_w, net_h;
    size_t box_stride, edge_stride;   // floats from one frame's box / edge maps to the next (the engine's conf slot holds 6 maps per frame)
    float pt, lt, nt;
    int cap_c;              // candidate keys (power of two)
    hp_human* humans; int hcap;
    int* human_cnt; int* flags;
    unsigned char* spill;   // kSpill: per-frame scratch of spill_bytes()
};

__host__ __device__ constexpr size_t spill_bytes()
{
    return (size_t)SPILL_CAP_H * (NPARTS + 2) * sizeof(short) + (size_t)SPILL_CAP_ENT * (sizeof(unsigned short) + sizeof(int));
}

// flags
enum { F_CAND = 1, F_HUMANS = 2, F_ENTRIES = 4, F_OUT = 8 };

__device__ __forceinline__ float iou_of(const Box& a, const Box& b)
{
    // (l & r).area() / (l.area() + r.area() - int_area), int areas, fp32 division (:108-113); 0/0 = NaN compares false
    const int x1 = max((int)a.x, (int)b.x), y1 = max((int)a.y, (int)b.y);
    int iw = min(a.x + a.w, b.x + b.w) - x1, ih = min(a.y + a.h, b.y + b.h) - y1;
    if (iw <= 0 || ih <= 0) { iw = 0; ih = 0; }
    const float ia = (float)(iw * ih);
    const float un = __fsub_rn((float)(a.w * a.h + b.w * b.h), ia);
    return __fdiv_rn(ia, un);
}

__device__ __forceinline__ unsigned orderable(float v)
{
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ int hash_cell(int c, int net)
{
    // size_t(part.x * grid_size), 64 -> 63 (:278-286).  A centre beyond the network size would index past the
    // reference's 64 x 64 std::array (undefined behaviour there); it is clamped to the last cell here.
    const float v = __fmul_rn(__fdiv_rn((float)c, (float)net), (float)HASH);
    int i = (int)v;
    return i >= HASH ? HASH - 1 : i;
}

template <bool kSpill>
__global__ void __launch_bounds__(THREADS, 1) ppn_parse_kernel(PpnParams P)
{
    using EIdx = typename std::conditional<kSpill, int, short>::type;   // hash-cell list links
    constexpr int cap_h = kSpill ? SPILL_CAP_H : CAP_H, cap_ent = kSpill ? SPILL_CAP_ENT : CAP_ENT;
    extern __shared__ __align__(16) unsigned char smem[];
    const int f = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = P.gh * P.gw, nn = P.nh * P.nw;
    // ---- shared memory carve-up ----
    Box* boxes = reinterpret_cast<Box*>(smem);                                    // [18][G]
    float* wscr = reinterpret_cast<float*>(boxes + NPARTS * G);                   // [NWARPS][G] conf copy / suppress flags
    short* to_at = reinterpret_cast<short*>(wscr + NWARPS * G);                   // [G] (padded to even)
    short* s_h = to_at + ((G + 7) & ~7);                                          // fast variant: humans live here
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(s_h + CAP_H * (NPARTS + 2)); // [cap_c]; phase D re-uses this region:
    EIdx* cell_head = reinterpret_cast<EIdx*>(keys);                              // [64*64]
    EIdx* cell_tail = cell_head + HASH * HASH;                                    // [64*64]
    unsigned char* gs = kSpill ? P.spill + (size_t)blockIdx.x * spill_bytes() : nullptr;
    short* hparts = kSpill ? reinterpret_cast<short*>(gs) : s_h;                  // [cap_h][18] index into boxes[type], -1 = absent
    short* hcount = hparts + cap_h * NPARTS;                                      // [cap_h] human_t::score (a count)
    unsigned short* order = reinterpret_cast<unsigned short*>(hcount + cap_h);    // [cap_h] position -> slot
    EIdx* ent_next = kSpill ? reinterpret_cast<EIdx*>(order + cap_h) : reinterpret_cast<EIdx*>(cell_tail + HASH * HASH); // [cap_ent]
    unsigned short* ent_id = reinterpret_cast<unsigned short*>(ent_next + cap_ent); // [cap_ent] POSITIONS, uint16_t like the reference's table
    __shared__ int s_nthr[NPARTS], s_nret[NPARTS];
    __shared__ int s_cnt, s_nh, s_flags, s_nkeep;

    const float* conf = P.conf + (size_t)f * P.box_stride;
    const float* bx = P.x + (size_t)f * P.box_stride;
    const float* by = P.y + (size_t)f * P.box_stride;
    const float* bw = P.w + (size_t)f * P.box_stride;
    const float* bh = P.h + (size_t)f * P.box_stride;
    const float* edge = P.edge + (size_t)f * P.edge_stride;
    if (tid == 0) { s_nh = 0; s_flags = 0; }

    // ---- A + B: threshold, decode, sort ascending by (conf, grid), NMS -- one warp per key-point type ----
    float* sc = wscr + warp * G;
    for (int k = warp; k < NPARTS; k += NWARPS) {
        int n = 0;
        for (int j0 = 0; j0 < G; j0 += 32) {
            const int j = j0 + lane;
            const float c = j < G ? conf[k * G + j] : 0.f;
            const bool on = j < G && P.pt < c;
            if (j < G) sc[j] = on ? c : __int_as_float(0x7fc00000);   // NaN = below threshold
            n += __popc(__ballot_sync(0xffffffffu, on));
        }
        __syncwarp();
        Box* B = boxes + k * G;
        for (int j = lane; j < G; j += 32) {
            const float c = sc[j];
            if (c != c) continue;
            int rank = 0;
            for (int q = 0; q < G; ++q) {
                const float c2 = sc[q];
                rank += (c2 < c || (c2 == c && q < j)) ? 1 : 0;
            }
            const int q = k * G + j;
            Box b;
            b.x = (short)max(min(P.net_w, __float2int_rz(__fsub_rn(bx[q], __fmul_rn(bw[q], 0.5f)))), 0);
            b.y = (short)max(min(P.net_h, __float2int_rz(__fsub_rn(by[q], __fmul_rn(bh[q], 0.5f)))), 0);
            b.w = (short)max(min(P.net_w, __float2int_rz(bw[q])), 0);
            b.h = (short)max(min(P.net_h, __float2int_rz(bh[q])), 0);
            b.conf = c; b.grid = (short)j; b.root = -1;
            B[rank] = b;
        }
        __syncwarp();
        // NMS: the pick is the back of the ascending list; ret[r] is stored at index n-1-r (the vacated tail)
        int* sup = reinterpret_cast<int*>(sc);
        int nB = n, r = 0;
        while (nB > 0) {
            const Box pick = B[nB - 1];
            --nB;
            __syncwarp();
            if (lane == 0) B[n - 1 - r] = pick;
            ++r;
            for (int i = lane; i < nB; i += 32) sup[i] = iou_of(pick, B[i]) >= P.nt ? 1 : 0;
            __syncwarp();
            if (lane == 0) {
                // `boxes.erase(begin + i)` without stepping i back (:121-123): the element sliding into slot i escapes
                int p = 0, q = 0;
                while (p < nB) {
                    if (sup[p]) {
                        ++p;
                        if (p < nB) { B[q++] = B[p]; ++p; }
                    } else {
                        if (q != p) B[q] = B[p];
                        ++q; ++p;
                    }
                }
                sup[0] = q;   // (read back below, after the barrier)
            }
            __syncwarp();
            nB = sup[0];
            __syncwarp();
        }
        if (lane == 0) { s_nthr[k] = n; s_nret[k] = r; }
    }
    __syncthreads();

    // ---- C: limbs in COCOPAIR_STD order ----
    const int n_range = min(P.E, NPAIRS);
    for (int i = 0; i < n_range; ++i) {
        const int ta = c_pair[i][0], tb = c_pair[i][1];
        const int nfrom = s_nret[ta], nto = s_nret[tb];
        Box* A = boxes + ta * G + (s_nthr[ta] - 1);   // ret[fi] = A[-fi]
        Box* T = boxes + tb * G + (s_nthr[tb] - 1);
        if (tid == 0) s_cnt = 0;
        for (int g = tid; g < G; g += THREADS) to_at[g] = -1;
        __syncthreads();
        for (int t = tid; t < nto; t += THREADS) to_at[T[-t].grid] = (short)t;
        __syncthreads();
        const float* ed = edge + (size_t)i * nn * G;
        for (int it = tid; it < nfrom * nn; it += THREADS) {
            const int fi = it / nn, j = it - fi * nn;
            const int fg = A[-fi].grid;
            const int fy = fg / P.gw, fx = fg - fy * P.gw;
            const int ny = j / P.nw, nx = j - ny * P.nw;
            const int ty = fy + ny - P.nh / 2, tx = fx + nx - P.nw / 2;
            if (tx < 0 || tx >= P.gw || ty < 0 || ty >= P.gh) continue;
            const float c = ed[(size_t)j * G + fg];
            if (!(c > P.lt)) continue;
            if (to_at[ty * P.gw + tx] < 0) continue;
            const int slot = atomicAdd(&s_cnt, 1);
            if (slot < P.cap_c) keys[slot] = ((unsigned long long)orderable(c) << 32) | (unsigned)it;
        }
        __syncthreads();
        int cnt = s_cnt;
        if (cnt > P.cap_c) { if (tid == 0) s_flags |= F_CAND; cnt = P.cap_c; }
        int m = 1;
        while (m < cnt) m <<= 1;
        for (int t = cnt + tid; t < m; t += THREADS) keys[t] = 0ull;
        __syncthreads();
        // bitonic sort, descending: (conf, generation order) -- the back of the reference's ascending list first
        for (int size = 2; size <= m; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = tid; t < (m >> 1); t += THREADS) {
                    const int lo = (t / stride) * (stride << 1) + (t % stride), hi = lo + stride;
                    const bool desc = ((lo & size) == 0);
                    const unsigned long long a = keys[lo], b = keys[hi];
                    if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
                }
                __syncthreads();
            }
        }
        if (tid == 0) {
            int nh_ = s_nh;
            for (int c = 0; c < cnt; ++c) {
                const int it = (int)(unsigned)(keys[c] & 0xffffffffu);
                const int fi = it / nn, j = it - fi * nn;
                Box& fb = A[-fi];
                const int fg = fb.grid;
                const int fy = fg / P.gw, fx = fg - fy * P.gw;
                const int ny = j / P.nw, nx = j - ny * P.nw;
                const int ti = to_at[(fy + ny - P.nh / 2) * P.gw + (fx + nx - P.nw / 2)];
                Box& tb_ = T[-ti];
                // from_check / to_check are tested but never set by the reference (:228-235): every candidate is visited
                int root;
                if ((fb.root != -1) == (tb_.root != -1)) {       // both rooted or both free: a NEW human (:240-243)
                    if (nh_ >= cap_h) { s_flags |= F_HUMANS; break; }
                    root = nh_++;
                    for (int u = 0; u < NPARTS; ++u) hparts[root * NPARTS + u] = -1;
                    hcount[root] = 0;
                } else
                    root = fb.root != -1 ? fb.root : tb_.root;
                if (hparts[root * NPARTS + ta] < 0) {
                    hparts[root * NPARTS + ta] = (short)(s_nthr[ta] - 1 - fi);
                    fb.root = (short)root;
                    ++hcount[root];
                }
                if (hparts[root * NPARTS + tb] < 0) {
                    hparts[root * NPARTS + tb] = (short)(s_nthr[tb] - 1 - ti);
                    tb_.root = (short)root;
                    ++hcount[root];
                }
            }
            s_nh = nh_;
        }
        __syncthreads();
    }

    // ---- D: merge humans sharing a part position, through the 64 x 64 hash of part centres (:275-326) ----
    for (int t = tid; t < HASH * HASH; t += THREADS) { cell_head[t] = -1; cell_tail[t] = -1; }
    for (int t = tid; t < s_nh; t += THREADS) order[t] = (unsigned short)t;
    __syncthreads();
    if (tid == 0) {
        int nh_ = s_nh, n_ent = 0;
        bool overflow = false;
        // centre of a part in pixels; an absent part is a default body_part_t at (0, 0) (human.hpp:14-19)
        auto centre = [&](int slot, int u, int& cx, int& cy) {
            const int bi = hparts[slot * NPARTS + u];
            if (bi < 0) { cx = 0; cy = 0; return; }
            const Box& b = boxes[u * G + bi];
            cx = b.x + b.w / 2; cy = b.y + b.h / 2;
        };
        auto push = [&](int cell, int id) {
            if (n_ent >= cap_ent) { overflow = true; return; }
            ent_id[n_ent] = (unsigned short)id; ent_next[n_ent] = -1;
            if (cell_tail[cell] < 0) cell_head[cell] = (EIdx)n_ent; else ent_next[cell_tail[cell]] = (EIdx)n_ent;
            cell_tail[cell] = (EIdx)n_ent;
            ++n_ent;
        };
        for (int i = 0; i < nh_ && !overflow; ++i) {
            const int cur = order[i];
            if ((double)hcount[cur] > (double)P.K - 0.1) continue;
            for (int j = 0; j < NPARTS; ++j) {
                if (hparts[cur * NPARTS + j] < 0) continue;
                int cx, cy;
                centre(cur, j, cx, cy);
                const int cell = hash_cell(cx, P.net_w) * HASH + hash_cell(cy, P.net_h);
                bool removed = false;
                for (int e = cell_head[cell]; e >= 0; e = ent_next[e]) {
                    const int pid = ent_id[e];            // a POSITION, possibly stale after erasures -- as in the reference
                    if (pid == i || pid >= nh_) continue;
                    const int mc = order[pid];
                    int mx, my;
                    centre(mc, j, mx, my);
                    if (my != cy || mx != cx) continue;
                    removed = true;
                    for (int u = 0; u < NPARTS; ++u) {
                        if (hparts[cur * NPARTS + u] >= 0 && hparts[mc * NPARTS + u] < 0) {
                            hparts[mc * NPARTS + u] = hparts[cur * NPARTS + u];
                            ++hcount[mc];
                            int ux, uy;
                            centre(cur, u, ux, uy);
                            push(hash_cell(ux, P.net_w) * HASH + hash_cell(uy, P.net_h), i);
                        }
                    }
                    for (int t = i; t + 1 < nh_; ++t) order[t] = order[t + 1];
                    --nh_;
                    --i;
                    break;
                }
                if (removed) break;
                push(cell, i);
            }
        }
        if (overflow) s_flags |= F_ENTRIES;
        // final filter: score <= MIN_REQUIRED_POINTS_FOR_A_MAN removed (:330-333); survivors keep their order
        int nk = 0;
        for (int i = 0; i < nh_; ++i)
            if (hcount[order[i]] > 3) order[nk++] = order[i];
        s_nkeep = nk;
    }
    __syncthreads();
    const int nk = s_nkeep;
    if (nk > P.hcap && tid == 0) s_flags |= F_OUT;
    const int nw_ = min(nk, P.hcap);
    hp_human* out = P.humans + (size_t)f * P.hcap;
    for (int t = tid; t < nw_ * (NPARTS + 1); t += THREADS) {
        const int hi = t / (NPARTS + 1), u = t - hi * (NPARTS + 1);
        const int slot = order[hi];
        if (u == NPARTS) { out[hi].score = (float)hcount[slot]; continue; }
        const int bi = hparts[slot * NPARTS + u];
        hp_body_part bp;
        if (bi < 0) { bp.has_value = 0; bp.x = 0.f; bp.y = 0.f; bp.score = 0.f; }
        else {
            const Box& b = boxes[u * G + bi];
            bp.has_value = 1;
            bp.x = __fdiv_rn((float)(b.x + b.w / 2), (float)P.net_w);   // :246-249
            bp.y = __fdiv_rn((float)(b.y + b.h / 2), (float)P.net_h);
            bp.score = b.conf;
        }
        out[hi].parts[u] = bp;
    }
    __syncthreads();
    if (tid == 0) { P.human_cnt[f] = nk; P.flags[f] = s_flags; }
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

size_t fixed_smem(int G)
{
    return (size_t)NPARTS * G * sizeof(Box) + (size_t)NWARPS * G * sizeof(float) + (size_t)((G + 7) & ~7) * sizeof(short)
        + (size_t)CAP_H * (NPARTS + 2) * sizeof(short);   // (the spill variant leaves the human area unused)
}

} // namespace

struct hp_ppn {
    int device = 0, net_w = 0, net_h = 0;
    float pt = 0.10f, lt = 0.05f, nt = 0.3f;
    cudaStream_t stream = nullptr;
    int hcap = 128;
    int smem_optin = 0;
    DBuf<float> in;          // host-entry staging: conf | x | y | w | h | edge
    DBuf<hp_human> humans;
    DBuf<int> counters;      // [N human_cnt | N flags]
    DBuf<unsigned char> spill;
    bool use_spill = false;  // sticky once a frame overflowed the shared-memory capacities
    std::vector<hp_human> host_h; std::vector<int> host_c;
    long long launches = 0;
    int last_N = 0;
    int prep_N = 0;          // frames humans / counters / spill are allocated for (they only grow)
};

namespace {

// the launch shape of a grid: candidate-key capacity (a power of two) and dynamic shared memory, or a refusal
int launch_config(const hp_ppn* p, int gh, int gw, int nh, int nw, int* cap_c, size_t* smem)
{
    const int G = gh * gw;
    if (G > 16384) { hpb::set_error("hp_ppn: %dx%d grid not supported", gh, gw); return HP_ERR_UNSUPPORTED; }
    // candidate capacity: worst case one per (from box, neighbour) = G * nh * nw, rounded up to a power of two,
    // bounded by the shared memory left (the phase-D tables alias the same region)
    const size_t fixed = fixed_smem(G);
    const size_t tables = p->use_spill ? (size_t)2 * HASH * HASH * sizeof(int) : (size_t)(2 * HASH * HASH + 2 * CAP_ENT) * sizeof(short);
    size_t want = 1;
    while (want < (size_t)G * nh * nw) want <<= 1;
    const size_t budget = (size_t)p->smem_optin - 1024;
    if (fixed + tables > budget) { hpb::set_error("hp_ppn: %dx%d grid needs %zu B of shared memory (> %zu)", gh, gw, fixed + tables, budget); return HP_ERR_UNSUPPORTED; }
    while (want > 1 && fixed + want * 8 > budget) want >>= 1;
    size_t dyn = want * 8;
    if (dyn < tables) dyn = tables;
    *cap_c = (int)want;
    *smem = fixed + dyn;
    return HP_OK;
}

// the device buffers a launch of N frames writes, for at least every N prepared so far at the current capacities
int ensure_buffers(hp_ppn* p, int N)
{
    if (N > p->prep_N) p->prep_N = N;
    if (p->use_spill) HP_CUDA_TRY(p->spill.ensure((size_t)p->prep_N * spill_bytes()));
    HP_CUDA_TRY(p->humans.ensure((size_t)p->prep_N * p->hcap));
    HP_CUDA_TRY(p->counters.ensure((size_t)p->prep_N * 2));
    return HP_OK;
}

// after a batch whose flags (OR over its frames) report an overflow, in the order hp_ppn_fetch has always grown: the record buffer to
// the largest frame's count first, else the sticky global-scratch variant; anything else cannot grow
int grow_after_overflow(hp_ppn* p, int flags, int max_count)
{
    if (flags & F_OUT) {
        if (max_count > p->hcap) p->hcap = max_count;
        return HP_OK;
    }
    if ((flags & (F_HUMANS | F_ENTRIES)) && !p->use_spill) {
        p->use_spill = true;
        return HP_OK;
    }
    if (flags) { hpb::set_error("hp_ppn: internal capacity exceeded (flags=%d: 1 limb candidates, 2 humans>%d, 4 hash registrations>%d)", flags, SPILL_CAP_H, SPILL_CAP_ENT); return HP_ERR_CAPACITY; }
    return HP_OK;
}

} // namespace

extern "C" {

int hp_ppn_create(hp_ppn** out, int net_w, int net_h, float point_thresh, float limb_thresh, float nms_thresh, int device)
{
    if (!out) return HP_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); hpb::set_error("hp_ppn_create: no CUDA device (this library has no CPU fallback)"); return HP_ERR_CUDA; }
    if (device < 0 || device >= ndev || net_w <= 0 || net_h <= 0 || net_w > 16383 || net_h > 16383) { hpb::set_error("hp_ppn_create: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(device));
    hp_ppn* p = new hp_ppn();
    p->device = device; p->net_w = net_w; p->net_h = net_h; p->pt = point_thresh; p->lt = limb_thresh; p->nt = nms_thresh;
    if (cudaDeviceGetAttribute(&p->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) { delete p; hpb::set_error("cudaDeviceGetAttribute failed"); return HP_ERR_CUDA; }
    {
        // The dynamic shared-memory cap of the parse kernels is process-wide state.  It is raised once per device, to everything a
        // launch may ask for, before any parser of that device launches: parsers used from several threads at once (the reference's
        // stream scheduler parses on a thread pool, one parser per thread) never set it while another thread launches.
        static std::mutex mu;
        static std::vector<char> raised;
        std::lock_guard<std::mutex> lk(mu);
        if (raised.size() <= (size_t)device) raised.resize(device + 1, 0);
        if (!raised[device]) {
            const int cap = p->smem_optin - 1024;
            if (cudaFuncSetAttribute(ppn_parse_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap) != cudaSuccess ||
                cudaFuncSetAttribute(ppn_parse_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap) != cudaSuccess) {
                delete p; hpb::set_error("hp_ppn_create: cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError())); return HP_ERR_CUDA;
            }
            raised[device] = 1;
        }
    }
    if (cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) != cudaSuccess) { delete p; hpb::set_error("cudaStreamCreate failed"); return HP_ERR_CUDA; }
    *out = p;
    return HP_OK;
}

void hp_ppn_destroy(hp_ppn* p)
{
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) { cudaStreamSynchronize(p->stream); cudaStreamDestroy(p->stream); }
    p->in.release(); p->humans.release(); p->counters.release(); p->spill.release();
    delete p;
}

int hp_ppn_set_point_thresh(hp_ppn* p, float t) { if (!p) return HP_ERR_ARG; p->pt = t; return HP_OK; }
int hp_ppn_set_limb_thresh(hp_ppn* p, float t) { if (!p) return HP_ERR_ARG; p->lt = t; return HP_OK; }
int hp_ppn_set_nms_thresh(hp_ppn* p, float t) { if (!p) return HP_ERR_ARG; p->nt = t; return HP_OK; }

int hp_ppn_process_device(hp_ppn* p, const float* d_conf, const float* d_x, const float* d_y, const float* d_w, const float* d_h,
                          const float* d_edge, int N, int K, int gh, int gw, int E, int nh, int nw, void* stream)
{
    const size_t G = (size_t)(gh > 0 ? gh : 0) * (gw > 0 ? gw : 0);
    return hp_ppn_process_device_strided(p, d_conf, d_x, d_y, d_w, d_h, d_edge, N, K, gh, gw, E, nh, nw, (size_t)(K > 0 ? K : 0) * G,
                                         (size_t)(E > 0 ? E : 0) * (nh > 0 ? nh : 0) * (nw > 0 ? nw : 0) * G, stream);
}

int hp_ppn_process_device_strided(hp_ppn* p, const float* d_conf, const float* d_x, const float* d_y, const float* d_w, const float* d_h,
                                  const float* d_edge, int N, int K, int gh, int gw, int E, int nh, int nw, size_t box_frame_stride,
                                  size_t edge_frame_stride, void* stream)
{
    if (!p || !d_conf || !d_x || !d_y || !d_w || !d_h || !d_edge || N <= 0 || gh <= 0 || gw <= 0 || E < 0 || nh <= 0 || nw <= 0) {
        hpb::set_error("hp_ppn_process_device: bad argument"); return HP_ERR_ARG;
    }
    // COCOPAIR_STD indexes key-point lists 0..17: with fewer the reference's key_points.at() throws (:187-188)
    if (K < NPARTS) { hpb::set_error("hp_ppn: K=%d key-point maps, the COCO limb table needs 18", K); return HP_ERR_ARG; }
    // a frame's maps must not overlap the next frame's: K maps of gh*gw, E*nh*nw edge planes
    if (box_frame_stride < (size_t)K * gh * gw || edge_frame_stride < (size_t)E * nh * nw * gh * gw) {
        hpb::set_error("hp_ppn_process_device: frame strides %zu / %zu floats are shorter than one frame's %d box / %d edge maps of %dx%d",
                       box_frame_stride, edge_frame_stride, K, E * nh * nw, gh, gw);
        return HP_ERR_ARG;
    }
    int cap_c = 0;
    size_t smem = 0;
    int rc = launch_config(p, gh, gw, nh, nw, &cap_c, &smem);
    if (rc) return rc;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : p->stream;
    rc = ensure_buffers(p, N);   // (after hp_ppn_prepare for this N: allocates nothing, synchronises nothing)
    if (rc) return rc;
    PpnParams P;
    P.conf = d_conf; P.x = d_x; P.y = d_y; P.w = d_w; P.h = d_h; P.edge = d_edge;
    P.K = K; P.gh = gh; P.gw = gw; P.E = E; P.nh = nh; P.nw = nw; P.net_w = p->net_w; P.net_h = p->net_h;
    P.box_stride = box_frame_stride; P.edge_stride = edge_frame_stride;
    P.pt = p->pt; P.lt = p->lt; P.nt = p->nt; P.cap_c = cap_c;
    P.humans = p->humans.p; P.hcap = p->hcap; P.human_cnt = p->counters.p; P.flags = p->counters.p + N;
    P.spill = p->spill.p;
    if (p->use_spill) ppn_parse_kernel<true><<<N, THREADS, smem, st>>>(P);
    else ppn_parse_kernel<false><<<N, THREADS, smem, st>>>(P);
    HP_CUDA_TRY(cudaGetLastError());
    p->launches += 1;
    p->last_N = N;
    return HP_OK;
}

int hp_ppn_fetch(hp_ppn* p, hp_human* out, int cap, int* n_out, int N)
{
    if (!p || !out || !n_out || N != p->last_N) { hpb::set_error("hp_ppn_fetch: bad argument"); return HP_ERR_ARG; }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    HP_CUDA_TRY(cudaDeviceSynchronize());
    p->host_h.resize((size_t)N * p->hcap); p->host_c.resize((size_t)N * 2);
    HP_CUDA_TRY(cudaMemcpy(p->host_c.data(), p->counters.p, sizeof(int) * 2 * N, cudaMemcpyDeviceToHost));
    HP_CUDA_TRY(cudaMemcpy(p->host_h.data(), p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost));
    int fl = 0, mx = 0;
    for (int f = 0; f < N; ++f) { fl |= p->host_c[N + f]; mx = p->host_c[f] > mx ? p->host_c[f] : mx; }
    if (fl) {
        // grow what overflowed for the next call and tell the caller to retry
        const int hcap_before = p->hcap;
        const int rc = grow_after_overflow(p, fl, mx);
        if (rc) return rc;
        if (p->hcap != hcap_before) hpb::set_error("hp_ppn: %d humans in one frame; record buffer grown, call again", mx);
        else hpb::set_error("hp_ppn: a frame overflowed the shared-memory human/hash capacities (%d / %d); switched to the global-scratch variant, call again", CAP_H, CAP_ENT);
        return HP_ERR_CAPACITY;
    }
    for (int f = 0; f < N; ++f) {
        const int n = p->host_c[f];
        if (n > cap) { hpb::set_error("hp_ppn: frame %d has %d humans but the caller's capacity is %d", f, n, cap); return HP_ERR_CAPACITY; }
        n_out[f] = n;
        memcpy(out + (size_t)f * cap, p->host_h.data() + (size_t)f * p->hcap, sizeof(hp_human) * n);
    }
    return HP_OK;
}

int hp_ppn_process_host(hp_ppn* p, const float* conf_point, const float* x, const float* y, const float* w, const float* h,
                        const float* edge, int N, int K, int gh, int gw, int E, int nh, int nw, hp_human* out, int cap, int* n_out)
{
    if (!p || !conf_point || !x || !y || !w || !h || !edge || !out || !n_out || N <= 0 || K <= 0 || gh <= 0 || gw <= 0 || E < 0 || nh <= 0 || nw <= 0) {
        hpb::set_error("hp_ppn_process_host: bad argument"); return HP_ERR_ARG;
    }
    HP_CUDA_TRY(cudaSetDevice(p->device));
    const size_t nb = (size_t)N * K * gh * gw, ne = (size_t)N * E * nh * nw * gh * gw;
    HP_CUDA_TRY(p->in.ensure(5 * nb + ne + 1));
    const float* src[5] = { conf_point, x, y, w, h };
    for (int i = 0; i < 5; ++i) HP_CUDA_TRY(cudaMemcpyAsync(p->in.p + i * nb, src[i], nb * sizeof(float), cudaMemcpyHostToDevice, p->stream));
    if (ne) HP_CUDA_TRY(cudaMemcpyAsync(p->in.p + 5 * nb, edge, ne * sizeof(float), cudaMemcpyHostToDevice, p->stream));
    for (int attempt = 0; attempt < 3; ++attempt) {
        int rc = hp_ppn_process_device(p, p->in.p, p->in.p + nb, p->in.p + 2 * nb, p->in.p + 3 * nb, p->in.p + 4 * nb, p->in.p + 5 * nb,
                                       N, K, gh, gw, E, nh, nw, p->stream);
        if (rc) return rc;
        const int before = p->hcap;
        const bool spill_before = p->use_spill;
        rc = hp_ppn_fetch(p, out, cap, n_out, N);
        if (rc == HP_ERR_CAPACITY && (p->hcap != before || p->use_spill != spill_before)) continue;   // a capacity was raised: run again
        return rc;
    }
    return HP_ERR_CAPACITY;
}

long long hp_ppn_launch_count(const hp_ppn* p) { return p ? p->launches : 0; }

// ---- building blocks of the pipelined end-to-end call (engine.cu: hp_pose_submit_ppn_* / hp_pose_collect) -------------------
// Checks the geometry and allocates everything a launch of N frames needs: hp_ppn_process_device_strided for this geometry then
// allocates nothing and synchronises nothing, so it can be captured into a CUDA graph.
int hp_ppn_prepare(hp_ppn* p, int N, int K, int gh, int gw, int E, int nh, int nw)
{
    if (!p || N <= 0 || gh <= 0 || gw <= 0 || E < 0 || nh <= 0 || nw <= 0) { hpb::set_error("hp_ppn_prepare: bad argument"); return HP_ERR_ARG; }
    if (K < NPARTS) { hpb::set_error("hp_ppn: K=%d key-point maps, the COCO limb table needs 18", K); return HP_ERR_ARG; }
    int cap_c = 0;
    size_t smem = 0;
    const int rc = launch_config(p, gh, gw, nh, nw, &cap_c, &smem);
    if (rc) return rc;
    HP_CUDA_TRY(cudaSetDevice(p->device));
    return ensure_buffers(p, N);
}
// Everything a captured launch bakes in (a change invalidates the graph): point / limb / NMS thresholds, then net_w, net_h, hcap,
// use_spill, the prepared N (the buffers' frame capacity), and the device.
int hp_ppn_state(const hp_ppn* p, float* thresholds3, int* ints6)
{
    if (!p) return HP_ERR_ARG;
    if (thresholds3) { thresholds3[0] = p->pt; thresholds3[1] = p->lt; thresholds3[2] = p->nt; }
    if (ints6) { ints6[0] = p->net_w; ints6[1] = p->net_h; ints6[2] = p->hcap; ints6[3] = p->use_spill ? 1 : 0; ints6[4] = p->prep_N; ints6[5] = p->device; }
    return HP_OK;
}
// Enqueues the D2H of the last launch's results on `stream` (NULL = the parser's own) into caller-owned PINNED host memory:
// counts_flags[2N] (N counts, then N overflow flags, the layout of hp_paf_copy_results_host_async) and humans[N * hcap]; no
// synchronisation.
int hp_ppn_copy_results_host_async(hp_ppn* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream)
{
    if (!p || !pin_humans || !pin_counts_flags || N <= 0 || N != p->last_N) { hpb::set_error("hp_ppn_copy_results_host_async: bad argument"); return HP_ERR_ARG; }
    cudaStream_t st = stream ? (cudaStream_t)stream : p->stream;
    HP_CUDA_TRY(cudaMemcpyAsync(pin_counts_flags, p->counters.p, sizeof(int) * 2 * N, cudaMemcpyDeviceToHost, st));
    HP_CUDA_TRY(cudaMemcpyAsync(pin_humans, p->humans.p, sizeof(hp_human) * (size_t)N * p->hcap, cudaMemcpyDeviceToHost, st));
    return HP_OK;
}
// After a launch whose flags (OR over its frames) report an overflow, max_count being its largest per-frame count: F_OUT raises hcap
// to max_count; F_HUMANS / F_ENTRIES switch to the global-scratch variant (sticky); F_CAND, or the global-scratch variant overflowing,
// is HP_ERR_CAPACITY.  Call hp_ppn_prepare before the next launch.
int hp_ppn_grow_capacity(hp_ppn* p, int flags, int max_count)
{
    if (!p) return HP_ERR_ARG;
    return grow_after_overflow(p, flags, max_count);
}

} // extern "C"
