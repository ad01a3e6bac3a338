/*
 * oracle/paf_oracle.c -- CPU restatement of the reference PAF parser (plain C99).
 *
 * TEST INFRASTRUCTURE ONLY (see paf_oracle.h).  Build: see oracle/Makefile
 * (gcc -O2 -ffp-contract=off: every fp32 rounding below is explicit; fmaf() is
 * the correctly-rounded fused op, identical to CUDA's __fmaf_rn).
 *
 * Determinism decisions frozen here (the reference leaves them unspecified, SURVEY 8c):
 *   - Gaussian row pass: taps left->right, acc = k0*x0; acc = fma(k_i, x_i, acc);
 *     column pass: symmetric, acc = k8*x0; acc = fma(k_{8+j}, (x_{+j} + x_{-j}), acc).
 *     This is the order OpenCV's AVX2 RowVec_32f / SymmColumnVec_32f use; together with the
 *     tail-column classes documented at orc_gaussian17 it reproduces cv2 4.13.0 bit-for-bit
 *     for every width (tests/test_oracle_cv_pin.py).
 *   - candidate sort: score desc, then idx1 asc, then idx2 asc (std::sort is unstable, paf.cpp:249).
 *   - -Ofast of the reference build (CMakeLists.txt:9) is NOT replicated: IEEE fp32/fp64.
 */
#include "paf_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* src/coco.hpp:10-52 */
static const int COCOPAIRS_NET[ORC_N_PAIRS][2] = {
    {12, 13}, {20, 21}, {14, 15}, {16, 17}, {22, 23}, {24, 25}, {0, 1}, {2, 3}, {4, 5}, {6, 7},
    {8, 9}, {10, 11}, {28, 29}, {30, 31}, {34, 35}, {32, 33}, {36, 37}, {18, 19}, {26, 27}};
static const int COCOPAIRS[ORC_N_PAIRS][2] = {
    {1, 2}, {1, 5}, {2, 3}, {3, 4}, {5, 6}, {6, 7}, {1, 8}, {8, 9}, {9, 10}, {1, 11},
    {11, 12}, {12, 13}, {1, 0}, {0, 14}, {14, 16}, {0, 15}, {15, 17}, {2, 16}, {5, 17}};
static int is_virtual_pair(int pair_id) { return pair_id > 16; } /* coco.hpp:6 */

/* paf.cpp:57-60 */
#define THRESH_VECTOR_CNT1 8
#define THRESH_PART_CNT 4
static const float THRESH_HUMAN_SCORE = 0.4f;
#define STEP_PAF 10

/* cv::getGaussianKernel(17, 3.0, CV_32F) = exp(-(i-8)^2/18), normalised in double and
 * rounded to fp32.  Literal bit patterns (so no libm enters the parity path); checked
 * against cv2.getGaussianKernel in tests/test_oracle_cv_pin.py. */
static const float g_k[17] = {
    0x1.f41be6p-9f, 0x1.1faf48p-7f, 0x1.282c02p-6f, 0x1.10d854p-5f, 0x1.c1d86ep-5f,
    0x1.4bd66ep-4f, 0x1.b616fp-4f, 0x1.02c558p-3f, 0x1.118dcap-3f, 0x1.02c558p-3f,
    0x1.b616fp-4f, 0x1.4bd66ep-4f, 0x1.c1d86ep-5f, 0x1.10d854p-5f, 0x1.282c02p-6f,
    0x1.1faf48p-7f, 0x1.f41be6p-9f};
const float* orc_gauss17_kernel(void) { return g_k; }

/* OpenCV resize.cpp, INTER_AREA with dst>=src: "area_mode" 2-tap interpolation.
 *   inv_scale = dst/src (double); scale = 1/inv_scale;
 *   sx = floor(dx*scale); fx = (float)((dx+1) - (sx+1)*inv_scale); fx = fx<=0 ? 0 : fx-floor(fx)
 *   clamp at the last source column. */
void orc_area_up_tab(int src, int dst, int32_t* idx, float* frac)
{
    double inv = (double)dst / (double)src;
    double scale = 1.0 / inv;
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

/* cv::resize(..., INTER_AREA) on one CV_32FC1 plane, every size combination (OpenCV resize.cpp, cv::resize dispatch):
 *   scale = src/dst per axis (computed as 1 / (dst/src) in double, like OpenCV);
 *   * BOTH axes shrink or keep (scale_x >= 1 && scale_y >= 1): true area averaging --
 *       integer factors ("is_area_fast"): resizeAreaFast_: sum of the iscale_y x iscale_x block (row-major, the scalar loop
 *         unrolled by four: sum += ((s0 + s1) + s2) + s3), times (float)(1 / area); the 2 x 2 case runs the SIMD kernel
 *         ((a + b) + (c + d)) * 0.25f on dx < (dw & ~3) and the scalar loop on the tail;
 *       otherwise resizeArea_ with computeResizeAreaTab (DecimateAlpha): buf[dx] = sum_k S[sx_k] * alpha_k per source row,
 *         dst = beta_0 * buf_0 + beta_1 * buf_1 + ... in table order, all float, products and sums rounded separately;
 *   * any axis grows (scale < 1): the 2-tap "area_mode" interpolation on BOTH axes with orc_area_up_tab's index / fraction
 *     formula (for the shrinking axis the same formula simply skips source pixels).
 * Pinned bit-exactly against Python cv2 4.13 for all four regimes (tests/golden/cv_pin_area.npz). */
typedef struct { int di, si; float alpha; } orc_dec;

static int decimate_tab(int ssize, int dsize, double scale, orc_dec* tab)
{
    int k = 0;
    for (int dx = 0; dx < dsize; ++dx) {
        double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        double cell = scale < ssize - fsx1 ? scale : ssize - fsx1;
        int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
        if (sx2 > ssize - 1) sx2 = ssize - 1;
        if (sx1 > sx2) sx1 = sx2;
        if (sx1 - fsx1 > 1e-3) { tab[k].di = dx; tab[k].si = sx1 - 1; tab[k++].alpha = (float)((sx1 - fsx1) / cell); }
        for (int sx = sx1; sx < sx2; ++sx) { tab[k].di = dx; tab[k].si = sx; tab[k++].alpha = (float)(1.0 / cell); }
        if (fsx2 - sx2 > 1e-3) {
            double a = fsx2 - sx2;
            if (a > 1.0) a = 1.0;
            if (a > cell) a = cell;
            tab[k].di = dx; tab[k].si = sx2; tab[k++].alpha = (float)(a / cell);
        }
    }
    return k;
}

static int resize_lerp2(const float* src, int sh, int sw, float* dst, int dh, int dw)
{
    int32_t* xi = (int32_t*)malloc(sizeof(int32_t) * dw);
    int32_t* yi = (int32_t*)malloc(sizeof(int32_t) * dh);
    float* xf = (float*)malloc(sizeof(float) * dw);
    float* yf = (float*)malloc(sizeof(float) * dh);
    float* row0 = (float*)malloc(sizeof(float) * dw);
    float* row1 = (float*)malloc(sizeof(float) * dw);
    orc_area_up_tab(sw, dw, xi, xf);
    orc_area_up_tab(sh, dh, yi, yf);
    for (int y = 0; y < dh; ++y) {
        int y0 = yi[y], y1 = y0 + 1 < sh ? y0 + 1 : sh - 1;
        float b1 = yf[y], b0 = 1.f - b1;
        /* HResizeLinear: D = S[sx]*(1-fx) + S[sx+1]*fx, products rounded separately */
        for (int x = 0; x < dw; ++x) {
            int x0 = xi[x], x1 = x0 + 1 < sw ? x0 + 1 : sw - 1;
            float a1 = xf[x], a0 = 1.f - a1;
            float p, q;
            p = src[y0 * sw + x0] * a0; q = src[y0 * sw + x1] * a1; row0[x] = p + q;
            p = src[y1 * sw + x0] * a0; q = src[y1 * sw + x1] * a1; row1[x] = p + q;
        }
        /* VResizeLinear: dst = S0*b0 + S1*b1 */
        for (int x = 0; x < dw; ++x) {
            float p = row0[x] * b0, q = row1[x] * b1;
            dst[y * dw + x] = p + q;
        }
    }
    free(xi); free(yi); free(xf); free(yf); free(row0); free(row1);
    return 0;
}

int orc_resize_area(const float* src, int sh, int sw, float* dst, int dh, int dw)
{
    if (sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0) return -3;
    const double scale_x = 1.0 / ((double)dw / (double)sw), scale_y = 1.0 / ((double)dh / (double)sh);
    if (!(scale_x >= 1.0 && scale_y >= 1.0)) return resize_lerp2(src, sh, sw, dst, dh, dw);
    const int isx = (int)lrint(scale_x), isy = (int)lrint(scale_y);
    if (fabs(scale_x - isx) < 2.220446049250313e-16 && fabs(scale_y - isy) < 2.220446049250313e-16) {
        const int area = isx * isy;
        const float scale = 1.f / (float)area;
        for (int dy = 0; dy < dh; ++dy)
            for (int dx = 0; dx < dw; ++dx) {
                const float* S = src + (size_t)dy * isy * sw + (size_t)dx * isx;
                if (isx == 2 && isy == 2 && dx < (dw & ~3)) { /* ResizeAreaFastVec_SIMD_32f */
                    const float top = S[0] + S[1], bot = S[sw] + S[sw + 1];
                    dst[dy * dw + dx] = (top + bot) * 0.25f;
                    continue;
                }
                float sum = 0.f;
                int k = 0;
                for (; k <= area - 4; k += 4) { /* CV_ENABLE_UNROLLED */
                    float g = S[(k / isx) * sw + k % isx] + S[((k + 1) / isx) * sw + (k + 1) % isx];
                    g = g + S[((k + 2) / isx) * sw + (k + 2) % isx];
                    g = g + S[((k + 3) / isx) * sw + (k + 3) % isx];
                    sum = sum + g;
                }
                for (; k < area; ++k) sum = sum + S[(k / isx) * sw + k % isx];
                dst[dy * dw + dx] = sum * scale;
            }
        return 0;
    }
    orc_dec* xtab = (orc_dec*)malloc(sizeof(orc_dec) * ((size_t)sw * 2 + 2 * dw + 4));
    orc_dec* ytab = (orc_dec*)malloc(sizeof(orc_dec) * ((size_t)sh * 2 + 2 * dh + 4));
    const int nx = decimate_tab(sw, dw, scale_x, xtab), ny = decimate_tab(sh, dh, scale_y, ytab);
    float* buf = (float*)malloc(sizeof(float) * dw);
    float* sum = (float*)malloc(sizeof(float) * dw);
    int prev_dy = -1;
    for (int j = 0; j < ny; ++j) {
        const float beta = ytab[j].alpha;
        const int dy = ytab[j].di;
        const float* S = src + (size_t)ytab[j].si * sw;
        for (int dx = 0; dx < dw; ++dx) buf[dx] = 0.f;
        for (int k = 0; k < nx; ++k) {
            const float t = S[xtab[k].si] * xtab[k].alpha;
            buf[xtab[k].di] = buf[xtab[k].di] + t;
        }
        if (dy != prev_dy) {
            if (prev_dy >= 0) for (int dx = 0; dx < dw; ++dx) dst[prev_dy * dw + dx] = sum[dx];
            for (int dx = 0; dx < dw; ++dx) sum[dx] = beta * buf[dx];
            prev_dy = dy;
        } else {
            for (int dx = 0; dx < dw; ++dx) { const float t = beta * buf[dx]; sum[dx] = sum[dx] + t; }
        }
    }
    if (prev_dy >= 0) for (int dx = 0; dx < dw; ++dx) dst[prev_dy * dw + dx] = sum[dx];
    free(xtab); free(ytab); free(buf); free(sum);
    return 0;
}

/* the up-scaling regime only (kept for the callers that state it): dst >= src on both axes */
int orc_resize_area_up(const float* src, int sh, int sw, float* dst, int dh, int dw)
{
    if (dh < sh || dw < sw || sh <= 0 || sw <= 0) return -3;
    return resize_lerp2(src, sh, sw, dst, dh, dw);
}

/* cv::borderInterpolate(BORDER_REFLECT_101) */
static int refl101(int p, int len)
{
    if ((unsigned)p < (unsigned)len) return p;
    if (len == 1) return 0;
    do {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    } while ((unsigned)p >= (unsigned)len);
    return p;
}

/* Column classes of OpenCV's AVX2 separable filter (RowVec_32f / SymmColumnVec_32f with
 * 8-lane vectors, then one 4-lane step, then scalar code compiled without contraction):
 *   x <  n8           : row pass FMA,      column pass FMA
 *   n8 <= x < n4      : row pass FMA,      column pass mul+add
 *   x >= n4           : row pass mul+add,  column pass mul+add
 * with n8 = w & ~7, n4 = n8 + 4 if w - n8 >= 4.  Measured against cv2 4.13.0; for the
 * default resolution (width 4*Hf, Hf even) every column is in the first class. */
void orc_gaussian17(const float* src, float* dst, int h, int w)
{
    const float* k = g_k;
    const int n8 = w & ~7;
    const int n4 = (w - n8 >= 4) ? n8 + 4 : n8;
    float* tmp = (float*)malloc(sizeof(float) * (size_t)h * w);
    for (int i = 0; i < h; ++i)
        for (int j = 0; j < w; ++j) {
            float s = k[0] * src[i * w + refl101(j - 8, w)];
            if (j < n4)
                for (int t = 1; t < 17; ++t) s = fmaf(k[t], src[i * w + refl101(j + t - 8, w)], s);
            else
                for (int t = 1; t < 17; ++t) { float p = k[t] * src[i * w + refl101(j + t - 8, w)]; s = s + p; }
            tmp[i * w + j] = s;
        }
    for (int i = 0; i < h; ++i)
        for (int j = 0; j < w; ++j) {
            float s = k[8] * tmp[i * w + j];
            for (int t = 1; t <= 8; ++t) {
                float a = tmp[refl101(i + t, h) * w + j] + tmp[refl101(i - t, h) * w + j];
                if (j < n8) s = fmaf(k[8 + t], a, s);
                else { float p = k[8 + t] * a; s = s + p; }
            }
            dst[i * w + j] = s;
        }
    free(tmp);
}

/* post_process.hpp:71-92: 3x3 stride-1 max with out-of-range neighbours skipped */
static void same_max_pool_3x3_2d(int height, int width, const float* in, float* out)
{
    for (int i = 0; i < height; ++i)
        for (int j = 0; j < width; ++j) {
            float m = in[i * width + j];
            for (int dx = 0; dx < 3; ++dx)
                for (int dy = 0; dy < 3; ++dy) {
                    int nx = i + dx - 1, ny = j + dy - 1;
                    if (0 <= nx && nx < height && 0 <= ny && ny < width) {
                        float v = in[nx * width + ny];
                        m = m > v ? m : v;
                    }
                }
            out[i * width + j] = m;
        }
}

typedef struct { int idx1, idx2; float score, etc; } cand_t; /* paf.cpp:41-46 */
static int cand_cmp(const void* pa, const void* pb)
{
    const cand_t* a = (const cand_t*)pa; const cand_t* b = (const cand_t*)pb;
    if (a->score > b->score) return -1;
    if (a->score < b->score) return 1;
    if (a->idx1 != b->idx1) return a->idx1 < b->idx1 ? -1 : 1;
    if (a->idx2 != b->idx2) return a->idx2 < b->idx2 ? -1 : 1;
    return 0;
}

typedef struct { int id; int parts[ORC_N_PARTS]; float score; int n_parts; } href_t; /* paf.cpp:19-37 */

int orc_paf_process(const float* conf, const float* paf, int c_conf, int c_paf, int H, int W,
                    int res_w, int res_h, int feat_height, float conf_thresh, float paf_thresh,
                    orc_human* humans, int human_cap, int* n_humans,
                    orc_peak* peaks_out, int peak_cap, int* n_peaks_out,
                    orc_conn* conns_out, int conn_cap, int* n_conns_out)
{
    if (!conf || !paf || H <= 0 || W <= 0 || c_conf < ORC_N_PARTS || c_paf < 2 * ORC_N_PAIRS) return -1;
    /* paf.cpp:311-315: dims() of a [C,H,W] view are bound to (C, fw, fh) => fw = H, fh = W;
     * default resolution = cv::Size(width = fw*4, height = fh*4). */
    const int fw = H, fh = W;
    if (res_w == -1 || res_h == -1) { res_w = fw * 4; res_h = fh * 4; }
    const int UW = res_w, UH = res_h; /* up-maps are [C, UH, UW] (paf.cpp:326-327) */
    /* m_feature_size = cv::Size(fw, fh) of the handle's first call; .height passed on (paf.cpp:321-332,354) */
    if (feat_height == -1) feat_height = fh;

    const size_t plane = (size_t)UH * UW;
    float* up_conf = (float*)malloc(sizeof(float) * plane * c_conf);
    float* up_paf = (float*)malloc(sizeof(float) * plane * c_paf);
    float* smoothed = (float*)malloc(sizeof(float) * plane * c_conf);
    float* pooled = (float*)malloc(sizeof(float) * plane * c_conf);
    int rc = 0;
    /* resize_area (post_process.hpp:26-52). NOTE: when dims are equal the reference
     * returns without copying (post_process.hpp:31-32), leaving uninitialised buffers;
     * here equal dims degenerate to an exact copy (fx = 0), the evident intent. */
    for (int k = 0; k < c_conf; ++k) orc_resize_area(conf + (size_t)k * H * W, H, W, up_conf + k * plane, UH, UW);
    for (int k = 0; k < c_paf; ++k) orc_resize_area(paf + (size_t)k * H * W, H, W, up_paf + k * plane, UH, UW);

    /* find_peak_coords (post_process.hpp:147-195): smooth all channels, pool, scan. */
    for (int k = 0; k < c_conf; ++k) {
        orc_gaussian17(up_conf + k * plane, smoothed + k * plane, UH, UW);
        same_max_pool_3x3_2d(UH, UW, smoothed + k * plane, pooled + k * plane);
    }
    int n_peaks = 0, peaks_alloc = 1024;
    orc_peak* all_peaks = (orc_peak*)malloc(sizeof(orc_peak) * peaks_alloc);
    {
        size_t off = 0;
        for (int k = 0; k < c_conf; ++k)
            for (int i = 0; i < UH; ++i)
                for (int j = 0; j < UW; ++j, ++off)
                    if (k < ORC_N_PARTS && smoothed[off] > conf_thresh && smoothed[off] == pooled[off]) {
                        if (n_peaks == peaks_alloc) {
                            peaks_alloc *= 2;
                            all_peaks = (orc_peak*)realloc(all_peaks, sizeof(orc_peak) * peaks_alloc);
                        }
                        orc_peak p = {k, j, i, up_conf[off], n_peaks};
                        all_peaks[n_peaks++] = p;
                    }
    }
    /* group_by (post_process.hpp:197-205): ids are contiguous per part because of scan order */
    int part_begin[ORC_N_PARTS + 1];
    {
        int c = 0;
        for (int k = 0; k < ORC_N_PARTS; ++k) {
            part_begin[k] = c;
            while (c < n_peaks && all_peaks[c].part_id == k) ++c;
        }
        part_begin[ORC_N_PARTS] = c;
    }
    if (n_peaks_out) *n_peaks_out = n_peaks;
    if (peaks_out) {
        if (n_peaks > peak_cap) { rc = -2; goto done; }
        memcpy(peaks_out, all_peaks, sizeof(orc_peak) * n_peaks);
    }

    /* get_connections for every pair (paf.cpp:351-354, 234-272) */
    orc_conn* all_conns[ORC_N_PAIRS];
    int n_conns[ORC_N_PAIRS];
    for (int p = 0; p < ORC_N_PAIRS; ++p) { all_conns[p] = NULL; n_conns[p] = 0; }
    for (int pair_id = 0; pair_id < ORC_N_PAIRS; ++pair_id) {
        const int pa = COCOPAIRS[pair_id][0], pb = COCOPAIRS[pair_id][1];
        const int ch1 = COCOPAIRS_NET[pair_id][0], ch2 = COCOPAIRS_NET[pair_id][1];
        const int na = part_begin[pa + 1] - part_begin[pa], nb = part_begin[pb + 1] - part_begin[pb];
        cand_t* cands = (cand_t*)malloc(sizeof(cand_t) * ((size_t)na * nb + 1));
        int nc = 0;
        /* get_connection_candidates (paf.cpp:93-144) */
        for (int ia = 0; ia < na; ++ia)
            for (int ib = 0; ib < nb; ++ib) {
                const orc_peak* A = &all_peaks[part_begin[pa] + ia];
                const orc_peak* B = &all_peaks[part_begin[pb] + ib];
                const int dx = B->x - A->x, dy = B->y - A->y;
                const float norm = (float)sqrt((double)(dx * dx + dy * dy)); /* paf.cpp:104 */
                if (norm < 1e-12) continue;
                const float vx = (float)dx / norm, vy = (float)dy / norm;
                /* get_paf_vectors (paf.cpp:67-91) */
                const float STEP_X = (float)dx / (float)STEP_PAF;
                const float STEP_Y = (float)dy / (float)STEP_PAF;
                float scores = 0.0f;
                int criterion1 = 0;
                for (int i = 0; i < STEP_PAF; ++i) {
                    float fx = (float)i * STEP_X; fx = (float)A->x + fx;
                    float fy = (float)i * STEP_Y; fy = (float)A->y + fy;
                    const int lx = (int)((double)fx + 0.5); /* roundpaf: v + 0.5 is double (paf.cpp:74) */
                    const int ly = (int)((double)fy + 0.5);
                    const float px = up_paf[ch1 * plane + (size_t)ly * UW + lx];
                    const float py = up_paf[ch2 * plane + (size_t)ly * UW + lx];
                    const float m1 = vx * px, m2 = vy * py;
                    const float score = m1 + m2;
                    scores += score;
                    if (score > paf_thresh) criterion1 += 1;
                }
                /* paf.cpp:129: float + double -> double, stored to float */
                double pen = 0.5 * (double)feat_height / (double)norm - 1.0;
                if (pen > 0.0) pen = 0.0;
                const float criterion2 = (float)((double)(scores / (float)STEP_PAF) + pen);
                if (criterion1 > THRESH_VECTOR_CNT1 && criterion2 > 0) {
                    float e = criterion2 + A->score; e = e + B->score;
                    cand_t c = {A->id, B->id, criterion2, e};
                    cands[nc++] = c;
                }
            }
        qsort(cands, nc, sizeof(cand_t), cand_cmp); /* paf.cpp:249-250 + frozen tie-break */
        orc_conn* conns = (orc_conn*)malloc(sizeof(orc_conn) * (nc + 1));
        int ncn = 0;
        for (int c = 0; c < nc; ++c) { /* paf.cpp:252-270 */
            int assigned = 0;
            for (int q = 0; q < ncn; ++q)
                if (conns[q].cid1 == cands[c].idx1 || conns[q].cid2 == cands[c].idx2) { assigned = 1; break; }
            if (!assigned) { orc_conn cn = {cands[c].idx1, cands[c].idx2, cands[c].score}; conns[ncn++] = cn; }
        }
        free(cands);
        all_conns[pair_id] = conns;
        n_conns[pair_id] = ncn;
        if (n_conns_out) n_conns_out[pair_id] = ncn;
        if (conns_out) {
            if (ncn > conn_cap) { rc = -2; }
            else memcpy(conns_out + (size_t)pair_id * conn_cap, conns, sizeof(orc_conn) * ncn);
        }
    }
    if (rc) goto done_conns;

    /* get_humans (paf.cpp:146-232) */
    {
        int hcap = 64, nh = 0;
        href_t* hr = (href_t*)malloc(sizeof(href_t) * hcap);
        for (int pair_id = 0; pair_id < ORC_N_PAIRS; ++pair_id) {
            const int part_id1 = COCOPAIRS[pair_id][0], part_id2 = COCOPAIRS[pair_id][1];
            for (int ci = 0; ci < n_conns[pair_id]; ++ci) {
                const orc_conn conn = all_conns[pair_id][ci];
                int t0 = -1, t1 = -1, nt = 0;
                for (int h = 0; h < nh; ++h)
                    if (hr[h].parts[part_id1] == conn.cid1 || hr[h].parts[part_id2] == conn.cid2) {
                        if (nt == 0) t0 = hr[h].id; else if (nt == 1) t1 = hr[h].id;
                        ++nt;
                    }
                if (nt == 1) {
                    href_t* h1 = &hr[t0];
                    if (h1->parts[part_id2] != conn.cid2) {
                        h1->parts[part_id2] = conn.cid2;
                        ++h1->n_parts;
                        float s = all_peaks[conn.cid2].score + conn.score;
                        h1->score += s;
                    }
                } else if (nt >= 2) {
                    href_t* h1 = &hr[t0]; href_t* h2 = &hr[t1];
                    int membership = 0;
                    for (int i = 0; i < ORC_N_PARTS; ++i)
                        if (h1->parts[i] > 0 && h2->parts[i] > 0) membership = 2; /* `id > 0` quirk, paf.cpp:185 */
                    if (membership == 0) {
                        for (int i = 0; i < ORC_N_PARTS; ++i) h1->parts[i] += h2->parts[i] + 1; /* paf.cpp:193 */
                        h1->n_parts += h2->n_parts;
                        h1->score += h2->score;
                        h1->score += conn.score;
                        const int delete_id = t1;
                        memmove(&hr[delete_id], &hr[delete_id + 1], sizeof(href_t) * (nh - delete_id - 1));
                        --nh;
                        for (int h = 0; h < nh; ++h) if (hr[h].id > delete_id) --hr[h].id;
                    } else {
                        h1->parts[part_id2] = conn.cid2;
                        h1->n_parts += 1;
                        float s = all_peaks[conn.cid2].score + conn.score;
                        h1->score += s;
                    }
                } else if (nt == 0 && !is_virtual_pair(pair_id)) {
                    if (nh == hcap) { hcap *= 2; hr = (href_t*)realloc(hr, sizeof(href_t) * hcap); }
                    href_t h;
                    h.id = nh; h.score = 0; h.n_parts = 2;
                    for (int i = 0; i < ORC_N_PARTS; ++i) h.parts[i] = -1;
                    h.parts[part_id1] = conn.cid1;
                    h.parts[part_id2] = conn.cid2;
                    float s = all_peaks[conn.cid1].score + all_peaks[conn.cid2].score;
                    h.score = s + conn.score;
                    hr[nh++] = h;
                }
            }
        }
        /* filter (paf.cpp:226-230) + conversion (paf.cpp:359-372) */
        int no = 0;
        for (int h = 0; h < nh; ++h) {
            if (hr[h].n_parts < THRESH_PART_CNT || hr[h].score / (float)hr[h].n_parts < THRESH_HUMAN_SCORE) continue;
            if (humans) {
                if (no >= human_cap) { rc = -2; break; }
                orc_human* o = &humans[no];
                memset(o, 0, sizeof(*o));
                o->score = hr[h].score;
                for (int i = 0; i < ORC_N_PARTS; ++i) {
                    const int id = hr[h].parts[i];
                    if (id != -1) {
                        /* the `+=` merge quirk can fabricate ids; the reference would read out of
                         * bounds (UB) -- the oracle (and the GPU path) report such parts as absent. */
                        if (id < 0 || id >= n_peaks) continue;
                        o->parts[i].has_value = 1;
                        o->parts[i].score = all_peaks[id].score;
                        o->parts[i].x = (float)all_peaks[id].x / (float)UW;
                        o->parts[i].y = (float)all_peaks[id].y / (float)UH;
                    }
                }
            }
            ++no;
        }
        if (n_humans) *n_humans = no;
        free(hr);
    }
done_conns:
    for (int p = 0; p < ORC_N_PAIRS; ++p) free(all_conns[p]);
done:
    free(all_peaks);
    free(up_conf); free(up_paf); free(smoothed); free(pooled);
    return rc;
}


/* ------------------------------------------------------------------------------------------------
 * Frame resize of tensorrt::inference(std::vector<cv::Mat>) (src/tensorrt.cpp:446-451):
 * cv::resize(mat, mat, size) = INTER_LINEAR on CV_8UC3, and non_scaling_resize (src/data.cpp:53-69).
 * Restates OpenCV's 8-bit fixed-point bilinear path (resize.cpp: INTER_RESIZE_COEF_BITS = 11,
 * HResizeLinear / VResizeLinear<uchar,int,short>), including the exact-2x shortcut to INTER_AREA.
 * Pinned bit-exactly against cv2 4.13.0 (tests/golden/cv_pin.npz, tests/test_oracle_cv_pin.py).
 * ---------------------------------------------------------------------------------------------- */
static int cv_round_half_even(float v) { return (int)lrintf(v); } /* saturate_cast<short>(float) = cvRound */

void orc_linear_tab(int src, int dst, int clamp_frac, int32_t* idx, int16_t* coef /* [dst][2] */)
{
    const double inv = (double)dst / (double)src;
    const double scale = 1.0 / inv;
    for (int d = 0; d < dst; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        f -= (float)s;
        if (clamp_frac) { /* x direction: resize.cpp clamps the fraction at the borders ... */
            if (s < 0) { f = 0.f; s = 0; }
            if (s >= src - 1) { f = 0.f; s = src - 1; }
        } /* ... the y direction keeps the fraction and clips the two row indices instead */
        idx[d] = s;
        coef[2 * d] = (int16_t)cv_round_half_even((1.f - f) * 2048.f);
        coef[2 * d + 1] = (int16_t)cv_round_half_even(f * 2048.f);
    }
}

int orc_resize_linear_u8c3(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw)
{
    if (sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0) return -1;
    if (sh == dh && sw == dw) { memcpy(dst, src, (size_t)sh * sw * 3); return 0; }
    if (sh == 2 * dh && sw == 2 * dw) { /* INTER_LINEAR with integer scale 2 is switched to INTER_AREA: (a+b+c+d+2)>>2 */
        for (int y = 0; y < dh; ++y)
            for (int x = 0; x < dw; ++x)
                for (int c = 0; c < 3; ++c) {
                    const uint8_t* p = src + ((size_t)(2 * y) * sw + 2 * x) * 3 + c;
                    dst[((size_t)y * dw + x) * 3 + c] = (uint8_t)((p[0] + p[3] + p[(size_t)sw * 3] + p[(size_t)sw * 3 + 3] + 2) >> 2);
                }
        return 0;
    }
    int32_t* xi = (int32_t*)malloc(sizeof(int32_t) * dw); int16_t* xa = (int16_t*)malloc(sizeof(int16_t) * 2 * dw);
    int32_t* yi = (int32_t*)malloc(sizeof(int32_t) * dh); int16_t* ya = (int16_t*)malloc(sizeof(int16_t) * 2 * dh);
    orc_linear_tab(sw, dw, 1, xi, xa);
    orc_linear_tab(sh, dh, 0, yi, ya);
    for (int y = 0; y < dh; ++y) {
        int y0 = yi[y], y1 = yi[y] + 1;
        y0 = y0 < 0 ? 0 : (y0 > sh - 1 ? sh - 1 : y0);
        y1 = y1 < 0 ? 0 : (y1 > sh - 1 ? sh - 1 : y1);
        const int b0 = ya[2 * y], b1 = ya[2 * y + 1];
        for (int x = 0; x < dw; ++x) {
            const int x0 = xi[x], x1 = x0 + 1 < sw ? x0 + 1 : sw - 1;
            const int a0 = xa[2 * x], a1 = xa[2 * x + 1];
            for (int c = 0; c < 3; ++c) {
                const int S0 = src[((size_t)y0 * sw + x0) * 3 + c] * a0 + src[((size_t)y0 * sw + x1) * 3 + c] * a1;
                const int S1 = src[((size_t)y1 * sw + x0) * 3 + c] * a0 + src[((size_t)y1 * sw + x1) * 3 + c] * a1;
                int v = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;
                dst[((size_t)y * dw + x) * 3 + c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
            }
        }
    }
    free(xi); free(xa); free(yi); free(ya);
    return 0;
}

/* non_scaling_resize (src/data.cpp:53-69): fit inside dst keeping the aspect ratio, pad right/bottom with 0 */
int orc_letterbox_u8c3(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw)
{
    const double h1 = dw * (sh / (double)sw);
    const double w2 = dh * (sw / (double)sh);
    int rh, rw;
    if (h1 <= dh) { rw = dw; rh = (int)h1; } else { rw = (int)w2; rh = dh; }
    if (rh <= 0 || rw <= 0) return -1;
    uint8_t* tmp = (uint8_t*)malloc((size_t)rh * rw * 3);
    int rc = orc_resize_linear_u8c3(src, sh, sw, tmp, rh, rw);
    memset(dst, 0, (size_t)dh * dw * 3);
    for (int y = 0; y < rh; ++y) memcpy(dst + (size_t)y * dw * 3, tmp + (size_t)y * rw * 3, (size_t)rw * 3);
    free(tmp);
    return rc;
}
