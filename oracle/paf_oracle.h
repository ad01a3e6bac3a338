/*
 * oracle/paf_oracle.h -- CPU restatement of the reference PAF parser.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under hyperpose_b200/ may include, link
 * or call this.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it (as the checker / CPU baseline).
 *
 * Follows (file:line under /root/reference):
 *   src/paf.cpp:57-375, src/post_process.hpp:26-205, src/coco.hpp:6-52,
 *   include/hyperpose/utility/human.hpp:10-31.
 * Third-party arithmetic restated (absent from /root/reference):
 *   OpenCV 4.4.0 (Dockerfile:32) cv::resize(INTER_AREA, upscale) and
 *   cv::GaussianBlur(17x17, sigma 3, BORDER_REFLECT_101); pinned bit-exactly
 *   against Python cv2 4.13.0 (tests/test_oracle_cv_pin.py, tests/golden/).
 * Parity pin: the reference holds no golden vectors for this path (SURVEY 4);
 *   the restatement is pinned (a) bit-exactly against cv2 for the two OpenCV
 *   primitives and (b) against oracle/_ref (the reference's own src/paf.cpp
 *   compiled verbatim over oracle/shim) for everything after them.
 */
#ifndef PAF_ORACLE_H
#define PAF_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ORC_N_PARTS 18
#define ORC_N_PAIRS 19

typedef struct { int32_t has_value; float x, y, score; } orc_body_part; /* human.hpp:14-19 */
typedef struct { orc_body_part parts[ORC_N_PARTS]; float score; } orc_human; /* human.hpp:23-27 */
typedef struct { int32_t part_id, x, y; float score; int32_t id; } orc_peak; /* post_process.hpp:126-131 */
typedef struct { int32_t cid1, cid2; float score; } orc_conn;             /* paf.cpp:7-13 */

/* cv::resize(INTER_AREA) for dst >= src in both axes (post_process.hpp:50). */
int orc_resize_area_up(const float* src, int sh, int sw, float* dst, int dh, int dw);
/* cv::resize(INTER_AREA), any source / destination size: true area averaging when both axes shrink, else the 2-tap area-mode lerp. */
int orc_resize_area(const float* src, int sh, int sw, float* dst, int dh, int dw);
/* coefficient table of the same (exposed for the GPU tests). */
void orc_area_up_tab(int src, int dst, int32_t* idx, float* frac);
/* cv::GaussianBlur(17x17, sigma=3, REFLECT_101) (post_process.hpp:66-67). */
void orc_gaussian17(const float* src, float* dst, int h, int w);
const float* orc_gauss17_kernel(void);

/*
 * paf::process (paf.cpp:300-375) on one frame.
 * conf [c_conf,H,W], paf [c_paf,H,W] row-major float32.
 * res_w/res_h: paf ctor resolution_size; pass -1,-1 for the default
 *   (width = 4*H, height = 4*W -- the reference's transposed default, paf.cpp:311-315).
 * feat_height: the length penalty's feature height (paf.cpp:129,354), which a paf handle takes from the W of its FIRST
 *   call (m_feature_size, paf.cpp:321-332); -1 = this frame's W (a handle's first call).
 * Optional debug outputs may be NULL.
 * returns 0, or <0 on error (-1 bad args, -2 capacity overflow, -3 unsupported resolution).
 */
int orc_paf_process(const float* conf, const float* paf, int c_conf, int c_paf, int H, int W,
                    int res_w, int res_h, int feat_height, float conf_thresh, float paf_thresh,
                    orc_human* humans, int human_cap, int* n_humans,
                    orc_peak* peaks, int peak_cap, int* n_peaks,
                    orc_conn* conns /* [19][conn_cap] */, int conn_cap, int* n_conns /* [19] */);

/* cv::resize(INTER_LINEAR) on CV_8UC3 (src/tensorrt.cpp:451) and non_scaling_resize (src/data.cpp:53-69) */
int orc_resize_linear_u8c3(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw);
int orc_letterbox_u8c3(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw);
void orc_linear_tab(int src, int dst, int clamp_frac, int32_t* idx, int16_t* coef);

#ifdef __cplusplus
}
#endif
#endif
