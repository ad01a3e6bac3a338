/*
 * hyperpose_b200.h -- C ABI of the H100-native HyperPose inference path.
 *
 * This is the drop-in boundary: the reference has no FFI, its seam is link-time
 * substitution of src/tensorrt.cpp + src/paf.cpp (CMakeLists.txt:28-34,
 * cmake/hyperpose.fake.cmake:6-19).  The C++ classes of include/hyperpose/operator/...
 * are re-implemented as thin wrappers over the functions below
 * (hyperpose_b200/csrc/hyperpose_api/); INTEGRATION.md shows the wiring.
 *
 * Conventions: plain pointers and sizes, no C++/torch types.  Every function returns
 * HP_OK (0) or a negative hp_status; hp_last_error() gives a thread-local message.
 * The C++ wrappers translate statuses to the reference's conventions
 * (error() -> std::exit(-1), src/logging.hpp:31-37; std::logic_error, src/tensorrt.cpp:439-443).
 * There is NO CPU fallback: without a CUDA device every entry point fails with HP_ERR_CUDA.
 */
#ifndef HYPERPOSE_B200_H
#define HYPERPOSE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HP_N_PARTS 18 /* include/hyperpose/utility/human.hpp:10 */
#define HP_N_PAIRS 19 /* include/hyperpose/utility/human.hpp:11 */

typedef enum hp_status {
    HP_OK = 0,
    HP_ERR_ARG = -1,      /* bad argument (rank/shape/null) -- reference: error() exit, paf.cpp:305-306 */
    HP_ERR_CAPACITY = -2, /* an internal or caller-provided capacity was exceeded */
    HP_ERR_UNSUPPORTED = -3,
    HP_ERR_CUDA = -4,     /* CUDA runtime failure / no device */
    HP_ERR_BATCH = -5     /* batch > max_batch -- reference: std::logic_error, tensorrt.cpp:439-443 */
} hp_status;

/* mirrors hyperpose::body_part_t / human_t (include/hyperpose/utility/human.hpp:14-31) */
typedef struct hp_body_part {
    int32_t has_value;
    float x, y, score;
} hp_body_part;
typedef struct hp_human {
    hp_body_part parts[HP_N_PARTS];
    float score;
} hp_human; /* 292 bytes */

/* debug/parity records (src/post_process.hpp:126-131, src/paf.cpp:7-13) */
typedef struct hp_peak {
    int32_t part_id, x, y;
    float score;
    int32_t id;
} hp_peak;
typedef struct hp_connection {
    int32_t cid1, cid2;
    float score;
} hp_connection;

const char* hp_last_error(void);
int hp_device_count(void);
const char* hp_version(void);

/* ------------------------------------------------------------------------------------------
 * PAF parser -- replaces hyperpose::parser::paf (include/hyperpose/operator/parser/paf.hpp:17-93,
 * src/paf.cpp:284-387, src/post_process.hpp:26-205).
 * ---------------------------------------------------------------------------------------- */
typedef struct hp_paf hp_paf;

/* paf::paf(conf_thresh, paf_thresh, resolution_size) (paf.hpp:27). res_w/res_h = -1 selects the
 * reference default (width 4*H, height 4*W of the first [C,H,W] input, paf.cpp:311-315).
 * device: CUDA ordinal. */
int hp_paf_create(hp_paf** out, float conf_thresh, float paf_thresh, int res_w, int res_h, int device);
void hp_paf_destroy(hp_paf* p);
/* paf::set_conf_thresh / set_paf_thresh (paf.hpp:66-70) */
int hp_paf_set_conf_thresh(hp_paf* p, float thresh);
int hp_paf_set_paf_thresh(hp_paf* p, float thresh);
/* internal capacities (the reference is unbounded; exceeding one returns HP_ERR_CAPACITY, the
 * *_host entry points grow and retry automatically). 0 keeps the current value. */
int hp_paf_set_capacity(hp_paf* p, int max_peaks_per_part, int max_candidates_per_limb, int max_humans);

/* paf::process(conf, paf) (paf.hpp:48, paf.cpp:300-375): one frame, HOST tensors
 * conf[c_conf,H,W], paf[c_paf,H,W] float32 row-major.  Writes <= cap humans, *n_out = count. */
int hp_paf_process_host(hp_paf* p, const float* conf, const float* paf, int c_conf, int c_paf, int H, int W,
                        hp_human* out, int cap, int* n_out);
/* N frames in one call (what the stream's parse stage would hand over, stream.hpp:347-385):
 * conf[N,c_conf,H,W], paf[N,c_paf,H,W]; out[N*cap], n_out[N]. */
int hp_paf_process_host_batched(hp_paf* p, const float* conf, const float* paf, int N, int c_conf, int c_paf, int H, int W,
                                hp_human* out, int cap, int* n_out);
/* Device-resident inputs (engine -> parser hand-off without the reference's D2H/H2D,
 * tensorrt.cpp:398-431).  Enqueues on `stream` (a cudaStream_t; NULL = the parser's own stream);
 * results stay on the device until hp_paf_fetch. */
int hp_paf_process_device(hp_paf* p, const float* d_conf, const float* d_paf, int N, int c_conf, int c_paf, int H, int W,
                          void* stream);
/* Copies the humans of the last hp_paf_process_device call to the host (synchronises its stream). */
int hp_paf_fetch(hp_paf* p, hp_human* out, int cap, int* n_out, int N);

/* parity/debug: peak list (scan-ordered, ids as in post_process.hpp:175-192) and per-limb
 * connections (paf.cpp:252-270) of frame `frame` of the last call. */
int hp_paf_debug_peaks(hp_paf* p, int frame, hp_peak* out, int cap, int* n_out);
int hp_paf_debug_connections(hp_paf* p, int frame, int pair_id, hp_connection* out, int cap, int* n_out);
/* kernels launched by this handle since creation (bench.py's gpu_launches) */
long long hp_paf_launch_count(const hp_paf* p);
/* diagnostics: with HPB_PAF_TIMING=1 in the environment the limb kernel stamps its phases (%globaltimer, ns); N * (19 * 4 + 6) values */
int hp_paf_debug_timing(hp_paf* p, unsigned long long* out, int N);
/* diagnostics: the code paths the last launch took, n >= HP_PAF_PLAN_FIELDS ints: generic (1: the resolution shrinks an axis and the
 * up-maps are materialised), rz_mode (resize regime of that path, -1 otherwise), tab_staged (limb kernel: up-sampling tables in shared
 * memory), stage_bytes (limb kernel: shared memory for the two PAF planes of a limb, 0 = read from global memory), limb_dyn_bytes
 * (dynamic shared memory the limb kernel may use), fast_asm (component-parallel assembly enabled), then the peak kernel's tile rows
 * with more than 16 source rows (direct up-sampling) and tile columns with more than 64 source columns (generic staging loop). */
#define HP_PAF_PLAN_FIELDS 8
int hp_paf_debug_plan(hp_paf* p, int* out, int n);
/* multi-GPU gather leg: copies the last batch's records (padded to `cap` >= the parser's human capacity per
 * frame) and counts into caller-owned DEVICE buffers, asynchronously on `stream` (NULL = the batch's stream),
 * so they can be handed to NCCL without a host round trip. */
int hp_paf_copy_results_device(hp_paf* p, hp_human* d_humans, int* d_counts, int N, int cap, void* stream);

/* ------------------------------------------------------------------------------------------
 * OpenPifPaf decoder -- replaces hyperpose::parser::pifpaf (include/hyperpose/operator/parser/pifpaf.hpp:8-26,
 * src/pifpaf.cpp:7-95, src/pifpaf_decoder/openpifpaf_postprocessor.cpp).
 * Tensors: pif[N,17,5,h,w] = {conf,x,y,b,scale}, paf[N,19,9,h,w] = {conf,x1,y1,x2,y2,b1,b2,s1,s2}, feature-cell units.
 * ---------------------------------------------------------------------------------------- */
typedef struct hp_pifpaf hp_pifpaf;
/* pifpaf::pifpaf(int h, int w, float thresh = 0.1) (pifpaf.hpp:10-13) */
int hp_pifpaf_create(hp_pifpaf** out, int net_h, int net_w, float thresh, int device);
void hp_pifpaf_destroy(hp_pifpaf* p);
/* pifpaf::process (pifpaf.hpp:14; defined with the (paf, pif) argument order at src/pifpaf.cpp:7): HOST tensors, N frames */
int hp_pifpaf_process_host(hp_pifpaf* p, const float* pif, const float* paf, int N, int h, int w, hp_human* out, int cap, int* n_out);
int hp_pifpaf_process_device(hp_pifpaf* p, const float* d_pif, const float* d_paf, int N, int h, int w, void* stream);
int hp_pifpaf_fetch(hp_pifpaf* p, hp_human* out, int cap, int* n_out, int N);
long long hp_pifpaf_launch_count(const hp_pifpaf* p);
int hp_pifpaf_debug_counts(hp_pifpaf* p, int frame, int* out7);
int hp_pifpaf_debug_hr(hp_pifpaf* p, int frame, int field, float* out);

/* ------------------------------------------------------------------------------------------
 * Pose Proposal Network parser -- replaces hyperpose::parser::pose_proposal
 * (include/hyperpose/operator/parser/proposal_network.hpp:18-80, src/pose_proposal.cpp:44-337).
 * Tensors per frame: conf_point / x / y / w / h f32[K,gh,gw] (boxes in network-input pixels) and
 * edge f32[E,nh,nw,gh,gw] (src/pose_proposal.cpp:14-20).  conf_iou is ignored by the reference except for its
 * leading dimension (:74,:84), which is the K passed here (K >= 18: COCOPAIR_STD indexes key points 0..17).
 * ---------------------------------------------------------------------------------------- */
typedef struct hp_ppn hp_ppn;
/* pose_proposal::pose_proposal(net_resolution, point_thresh = 0.10, limb_thresh = 0.05, nms_thresh = 0.3)
 * (proposal_network.hpp:26) */
int hp_ppn_create(hp_ppn** out, int net_w, int net_h, float point_thresh, float limb_thresh, float nms_thresh, int device);
void hp_ppn_destroy(hp_ppn* p);
/* set_point_thresh / set_limb_thresh / set_nms_thresh (proposal_network.hpp:67-75) */
int hp_ppn_set_point_thresh(hp_ppn* p, float thresh);
int hp_ppn_set_limb_thresh(hp_ppn* p, float thresh);
int hp_ppn_set_nms_thresh(hp_ppn* p, float thresh);
/* pose_proposal::process (proposal_network.hpp:44-47; src/pose_proposal.cpp:68-337) for N frames, HOST tensors
 * [N,K,gh,gw] x5 and [N,E,nh,nw,gh,gw]; out[N*cap], n_out[N]. */
int hp_ppn_process_host(hp_ppn* p, const float* conf_point, const float* x, const float* y, const float* w, const float* h,
                        const float* edge, int N, int K, int gh, int gw, int E, int nh, int nw, hp_human* out, int cap, int* n_out);
/* same with DEVICE tensors, asynchronous on `stream` (NULL = the parser's own); results by hp_ppn_fetch */
int hp_ppn_process_device(hp_ppn* p, const float* d_conf_point, const float* d_x, const float* d_y, const float* d_w, const float* d_h,
                          const float* d_edge, int N, int K, int gh, int gw, int E, int nh, int nw, void* stream);
/* the same with the distance from one frame's maps to the next given in floats: box_frame_stride for conf_point / x / y / w / h
 * (hp_ppn_process_device: K*gh*gw), edge_frame_stride for edge (E*nh*nw*gh*gw).  A PPN engine's outputs (head_type 2) are parsed
 * in place with d_conf_point = conf slot + 0, d_x = + 2*K*gh*gw, d_y = + 3*K*gh*gw, d_w = + 4*K*gh*gw, d_h = + 5*K*gh*gw,
 * box_frame_stride = 6*K*gh*gw, d_edge = the paf slot, edge_frame_stride = E*nh*nw*gh*gw. */
int hp_ppn_process_device_strided(hp_ppn* p, const float* d_conf_point, const float* d_x, const float* d_y, const float* d_w, const float* d_h,
                                  const float* d_edge, int N, int K, int gh, int gw, int E, int nh, int nw, size_t box_frame_stride,
                                  size_t edge_frame_stride, void* stream);
int hp_ppn_fetch(hp_ppn* p, hp_human* out, int cap, int* n_out, int N);
long long hp_ppn_launch_count(const hp_ppn* p);

/* ------------------------------------------------------------------------------------------
 * DNN engine -- replaces hyperpose::dnn::tensorrt (include/hyperpose/operator/dnn/tensorrt.hpp:33-141,
 * src/tensorrt.cpp:121-471).  The model file is a flat "HPB2PACK" pack (hyperpose_b200/csrc/pack_format.h,
 * written by hyperpose_b200/models.py) instead of .onnx/.uff/.trt (utility/model.hpp:13-32).
 * ---------------------------------------------------------------------------------------- */
typedef struct hp_engine hp_engine;

/* tensorrt::tensorrt(model, input_size(w,h), max_batch_size, keep_ratio, dtype, factor, flip_rgb)
 * (tensorrt.hpp:44-74).  pack/pack_bytes: model pack image in host memory. */
int hp_engine_create(hp_engine** out, const void* pack, size_t pack_bytes, int in_w, int in_h, int max_batch,
                     double factor, int flip_rgb, int device);
/* The same with the arithmetic the reference's `data_type` ctor argument selects (tensorrt.hpp:14-22,48,61):
 *   HP_DTYPE_F16  (= data_type::kHALF):  fp16 operands and activations, fp32 accumulation -- what hp_engine_create builds;
 *   HP_DTYPE_TF32 (= data_type::kFLOAT, the reference default): fp32 activations in HBM, wgmma kind tf32 (fp32 operands
 *                 read with a 10-bit mantissa by the tensor core, fp32 accumulation) -- TensorRT's own FP32 mode on tensor-core GPUs;
 *   HP_DTYPE_INT8 (= data_type::kINT8): symmetric int8 activations (one fp32 scale per buffer, from the pack's calibration table)
 *                 and per-output-channel int8 weights, wgmma kind s8 with s32 accumulation.  Needs a pack with a scale table
 *                 (hp_pack_int8_calibrated); no OpenPifPaf heads.  HP_ERR_ARG names the op or buffer a pack is refused for. */
#define HP_DTYPE_F16 0
#define HP_DTYPE_TF32 1
#define HP_DTYPE_INT8 2
int hp_engine_create_ex(hp_engine** out, const void* pack, size_t pack_bytes, int in_w, int in_h, int max_batch,
                        double factor, int flip_rgb, int device, int dtype);
int hp_engine_dtype(const hp_engine* e);
/* 1 when the model pack carries an INT8 scale table (one scale per activation buffer), else 0.  Host only. */
int hp_pack_int8_calibrated(const void* pack, size_t pack_bytes);
/* INT8 calibration as TensorRT's IInt8MinMaxCalibrator: on an HP_DTYPE_TF32 engine (HP_ERR_ARG on any other), runs the graph op by
 * op on HOST u8 frames [N,in_h,in_w,3] (N may exceed max_batch) and folds max |x| of every op's output buffer into
 * absmax[n_buffers] -- a running maximum, so start from zeros and call again for more frames.  Scale = absmax / 127. */
int hp_engine_calibrate_u8(hp_engine* e, const uint8_t* frames, int N, float* absmax, int n_buffers);
void hp_engine_destroy(hp_engine* e);
/* max_batch_size() / input_size() (tensorrt.hpp:81-85) + output geometry; any pointer may be NULL */
int hp_engine_info(const hp_engine* e, int* in_w, int* in_h, int* max_batch, int* c_conf, int* c_paf, int* out_h, int* out_w,
                   double* flops_per_frame);
/* tensorrt::inference(std::vector<cv::Mat>) (tensorrt.cpp:436-461) after the resize step: HOST u8
 * [N,in_h,in_w,3] BGR frames.  N > max_batch -> HP_ERR_BATCH (std::logic_error in the reference).
 * Asynchronous: outputs stay on the device (hp_engine_outputs / hp_engine_read_outputs_host). */
int hp_engine_infer_u8_host(hp_engine* e, const uint8_t* frames, int N);
int hp_engine_infer_u8_device(hp_engine* e, const uint8_t* d_frames, int N, void* stream);
/* The resize step of tensorrt::inference (tensorrt.cpp:446-451) on the GPU: stages ONE host frame of any size into
 * batch slot `slot` -- cv::resize(INTER_LINEAR) or, with keep_ratio, non_scaling_resize (src/data.cpp:53-69),
 * bit-exact with OpenCV's 8-bit fixed-point bilinear.  hp_engine_infer_staged then runs the network on N slots. */
int hp_engine_stage_frame_u8(hp_engine* e, int slot, const uint8_t* frame, int src_h, int src_w, int keep_ratio);
int hp_engine_infer_staged(hp_engine* e, int N);
int hp_engine_debug_read_frames(hp_engine* e, uint8_t* out, int N);
/* tensorrt::inference(const std::vector<float>&, size_t) (tensorrt.cpp:364-434): HOST f32 NCHW, pre-scaled */
int hp_engine_infer_f32_host(hp_engine* e, const float* nchw, int N);
/* device pointers of the fp32 NCHW outputs conf[N,c_conf,h,w] / paf[N,c_paf,h,w] and the engine stream */
int hp_engine_outputs(hp_engine* e, const float** d_conf, const float** d_paf, void** stream);
/* the reference's per-image D2H of every output (tensorrt.cpp:398-431), as two contiguous host tensors */
int hp_engine_read_outputs_host(hp_engine* e, float* conf, float* paf, int N);
/* The same read-back into N SEPARATE per-image buffers -- the storage of the feature_map_t objects
 * tensorrt::inference returns (tensorrt.cpp:398-431): conf_frames[i] receives [c_conf,h,w], paf_frames[i] [c_paf,h,w]
 * (OpenPifPaf packs: pif [17,5,h,w] / paf [19,9,h,w]).  publish != 0 additionally keeps a device snapshot of the
 * batch and registers the host addresses: hp_paf_process_host / hp_pifpaf_process_host called later with exactly
 * these buffers (what parser.process(packet[0], packet[1]) does per image, operator_api_batched_images_paf.example.cpp:
 * 70-74, and what the stream's parse tasks do, stream.hpp:347-373) parse the whole batch ONCE from the device copy and
 * serve the remaining images from the cached records -- no second trip of the tensors over PCIe, one launch sequence
 * per batch.  The look-up compares EVERY byte of the two host tensors with the pinned copy the publication keeps: a
 * buffer edited in place, or freed and re-allocated at the same address, is never served stale results.  Any mismatch
 * (other address, other shape, any changed byte, publication older than 4 batches) takes the ordinary host path; the
 * results are identical.  Publishing is opt-in (publish = 0 is a plain read-back). */
int hp_engine_read_outputs_frames(hp_engine* e, float* const* conf_frames, float* const* paf_frames, int N, int publish);
/* 0: conf/paf maps for hyperpose::parser::paf; 1: OpenPifPaf fields (pif, paf) for hyperpose::parser::pifpaf;
 * 2: Pose Proposal Network outputs for hyperpose::parser::pose_proposal -- conf slot [6,K,gh,gw] (conf_point, conf_iou, x, y, w, h;
 * boxes in network-input pixels), paf slot [L,nh,nw,gh,gw] (edges), c_conf = 6K, c_paf = L*nh*nw.  The PAF-parser hp_pose_* calls
 * refuse it: use hp_pose_submit_ppn_* (below), or parse with hp_ppn_process_device_strided on the engine's device outputs. */
int hp_engine_head_type(const hp_engine* e);
/* the publication mechanism above: global switch (default on; env HPB_NO_HANDOFF disables) and counters
 * (batches published, process() calls served from a device snapshot, batched parses run, look-ups that fell back) */
int hp_handoff_enable(int on);
int hp_handoff_stats(long long* published, long long* hits, long long* batch_parses, long long* misses);
/* asynchronous D2D snapshot of the outputs into caller-owned device tensors (software-pipelined callers) */
int hp_engine_copy_outputs_device(hp_engine* e, float* d_conf, float* d_paf, int N, void* stream);
int hp_engine_sync(hp_engine* e);
long long hp_engine_launch_count(const hp_engine* e);
/* test hooks: read / write an activation buffer (NHWC; fp16 elements on an HP_DTYPE_F16 engine, fp32 on HP_DTYPE_TF32, int8 on HP_DTYPE_INT8),
 * run a sub-range [first,last] of the op list */
int hp_engine_debug_read_buffer(hp_engine* e, int buf, void* out_f16, int N, int* H, int* W, int* C);
int hp_engine_debug_write_buffer(hp_engine* e, int buf, const void* in_f16, int N);
int hp_engine_debug_run_ops(hp_engine* e, int first_op, int last_op, int N);
/* test hooks: read a buffer's memory as it stands, including a buffer hp_engine_debug_read_buffer refuses because its final
 * content is never stored (earlier ops may still use it); write N frames of the fp32 conf / paf outputs */
int hp_engine_debug_read_buffer_raw(hp_engine* e, int buf, void* out, int N);
int hp_engine_debug_write_outputs(hp_engine* e, const float* conf, const float* paf, int N);
/* test hook: the kernel op `op` launches on the next run over u8 frames, fixed at creation, as a NUL-terminated name in
 * name[cap]: "conv<f16|tf32|i8,BN[,res][,stem3|stem7]>", "halo<BN[,pool|,wide|,pp|,pool,pp]>", "dw_strip<K,S>", "dw_col", "dw_tma<1|2>",
 * "dw_f32", "dw_i8", "maxpool<K>", "maxpool_f32", "maxpool_i8", "im2col" (fp16 and TF32), "im2col_i8", "heads", "ppn_head", or "none" for
 * an op that a neighbouring op's launch covers.  A dilated depthwise op adds its dilation: "dw_tma<1,d2>", "dw_col<d2>", "dw_f32<d2>",
 * "dw_i8<d2>". */
int hp_engine_debug_op_kernel(const hp_engine* e, int op, char* name, int cap);
/* test hook: *tma_store = 1 when op `op` runs the halo conv kernel with its TMA-store epilogue, 0 otherwise (HPB_HALO_REG_EPILOGUE=1
 * or a plan the TMA store cannot express: per-thread stores from registers) */
int hp_engine_debug_op_epilogue(const hp_engine* e, int op, int* tma_store);
/* test hook: the same for the im2col conv kernel ("conv<f16,...>"): *tma_store = 1 when op `op` stages its fp16 outputs in shared
 * memory and TMA-stores them, 0 otherwise (HPB_CONV_REG_EPILOGUE=1, the TF32 / INT8 engines, the fp32 conf / PAF output, or a plan
 * the TMA store cannot express: per-thread stores from registers) */
int hp_engine_debug_op_conv_epilogue(const hp_engine* e, int op, int* tma_store);
/* test hook: *pdl = 1 when the engine launches its conv and depthwise kernels with programmatic dependent launch, each kernel's
 * prologue running under its predecessor's tail, 0 otherwise.  Decided at creation from the work per launch at max_batch. */
int hp_engine_debug_uses_pdl(const hp_engine* e, int* pdl);

/* benchmark hook (SURVEY 8d): after the last conv of every run, copy these DEVICE tensors over the engine's
 * conf/paf outputs, so that random-init weights still give the parser a realistic load.  NULL disables it. */
int hp_engine_set_output_override(hp_engine* e, const float* d_conf, const float* d_paf);
/* per-op CUDA-event timing on the engine's launching stream (bench.py roofline leg) */
int hp_engine_set_profiling(hp_engine* e, int enable);
int hp_engine_get_profile(hp_engine* e, double* ms_per_op, int* op_type, double* flops_per_op, int cap, int* n_ops, long long* runs);

/* engine.inference(batch) + parser.process(packet) for every image of the batch
 * (examples/operator_api_batched_images_paf.example.cpp:64-74) as ONE call: host u8 frames in,
 * human_t records out, conf/paf never leave the device.  Synchronous form of the two calls below; a parser capacity that
 * overflows is grown and the batch re-run (the reference is unbounded), so HP_ERR_CAPACITY means the CALLER's `cap`. */
int hp_pose_run_u8_host(hp_engine* e, hp_paf* parser, const uint8_t* frames, int N, hp_human* out, int cap, int* n_out);
/* The same, two batches in flight: submit enqueues the H2D copy of the frames (own copy stream: it overlaps the convs of
 * the previously submitted batch), the whole launch sequence (replayed from a CUDA graph captured on first use) and the
 * D2H of the records, and returns a ticket (0 or 1) at once; collect waits for that batch and hands out its humans.
 * At most two tickets are outstanding; a third submit without a collect is HP_ERR_ARG.  `frames` may be pageable (it is
 * copied into pinned staging before submit returns) or page-locked (DMA straight from it: keep it alive until collect). */
int hp_pose_submit_u8_host(hp_engine* e, hp_paf* parser, const uint8_t* frames, int N, int* ticket);
int hp_pose_submit_u8_device(hp_engine* e, hp_paf* parser, const uint8_t* d_frames, int N, int* ticket);   /* frames already in HBM */
int hp_pose_collect(hp_engine* e, int ticket, hp_human* out, int cap, int* n_out);
int hp_pose_stats(const hp_engine* e, long long* graph_captures, long long* graph_launches);
/* The pipelined call for OpenPifPaf packs: engine.inference(batch) + pifpaf.process(packet[0], packet[1]) per image
 * (examples/operator_api_batched_images_pifpaf.example.cpp:48-64), two batches in flight.  The decoder's greedy growth is a
 * latency chain on one warp per frame (milliseconds per batch of 16 while 16 of 132 SMs do anything at all), so it runs on the DECODER's
 * stream underneath the convolutions of the next batch: the engine's persistent kernels leave `reserve` SMs to it (default
 * min(max_batch, 16); env HPB_PIFPAF_RESERVE_SMS), and the next batch's head kernels wait only until the field tensors have
 * been consumed (decoder kernels P1-P3), not for the growth.  Tickets / hp_pose_collect as above. */
int hp_pose_submit_pifpaf_u8_host(hp_engine* e, hp_pifpaf* decoder, const uint8_t* frames, int N, int* ticket);
int hp_pose_submit_pifpaf_u8_device(hp_engine* e, hp_pifpaf* decoder, const uint8_t* d_frames, int N, int* ticket);
/* The pipelined calls for frames of ANY size (cameras, video files: 640x360, 1280x720, 1920x1080 ...): each frame goes through the
 * reference's resize step -- cv::resize(INTER_LINEAR) or, with keep_ratio, non_scaling_resize (src/tensorrt.cpp:446-451,
 * src/data.cpp:53-69) -- bit-exact with OpenCV, in ONE batched kernel on the engine stream ahead of the network; the frames of a batch
 * may all differ in size.  Results by hp_pose_collect, as above.  N > max_batch is HP_ERR_BATCH, a null frame or a size <= 0
 * HP_ERR_ARG; packs the network-size calls refuse are refused alike.
 * _host: the source pixels are copied on the copy stream (overlapping the previous batch's convolutions): page-locked frames by DMA
 * straight from them (keep them alive until collect), pageable ones through pinned staging before submit returns.  Page-locked
 * frames save a host memcpy of every frame.
 * _device: the frames are read in place from device memory by the resize kernel: they must stay valid and unchanged until the
 * ticket is collected. */
typedef struct hp_frame_u8 { const uint8_t* data; int32_t height, width; } hp_frame_u8;   /* HWC BGR, rows packed */
int hp_pose_submit_frames_u8_host(hp_engine* e, hp_paf* parser, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_frames_u8_device(hp_engine* e, hp_paf* parser, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_u8_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_u8_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
/* The pipelined calls for Pose Proposal Network packs (head_type 2): engine.inference(batch) + pose_proposal.process(packet) per image
 * (examples/operator_api_batched_images_pose_proposal.example.cpp), two batches in flight, frames at the network size or (_frames_)
 * of any size as above.  The parse of a batch runs on the engine stream right behind its network, reading the engine's outputs in
 * place (the pointers and strides of hp_ppn_process_device_strided, with K, E, nh, nw from the pack's PPN head op), and the network,
 * the parse and the record D2H are replayed from one CUDA graph per ticket.  The records are byte-identical to hp_engine_infer_u8_device
 * + hp_ppn_process_device_strided + hp_ppn_fetch (retried on HP_ERR_CAPACITY).  A pack without PPN heads is HP_ERR_UNSUPPORTED, a
 * parser on another device than the engine HP_ERR_ARG.  Tickets / hp_pose_collect as above: a parser capacity that overflows is grown
 * in collect and the ticket's frames run again, so HP_ERR_CAPACITY there means the CALLER's `cap`. */
int hp_pose_submit_ppn_u8_host(hp_engine* e, hp_ppn* parser, const uint8_t* frames, int N, int* ticket);
int hp_pose_submit_ppn_u8_device(hp_engine* e, hp_ppn* parser, const uint8_t* d_frames, int N, int* ticket);
int hp_pose_submit_ppn_frames_u8_host(hp_engine* e, hp_ppn* parser, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_u8_device(hp_engine* e, hp_ppn* parser, const hp_frame_u8* frames, int N, int keep_ratio, int* ticket);
/* The same calls for YUV 4:2:0 video frames (NVDEC's NV12, libavcodec's I420, camera NV12 / NV21, YV12), for all three head types.
 * Each source pixel is converted to BGR as cv::cvtColor(COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12) does -- BT.601 limited range,
 * OpenCV's 20-bit fixed point, each chroma sample covering its 2x2 luma block -- inside the batched resize's fetch, before any
 * interpolation: the network-size frame is byte-identical to cv::resize(cv::cvtColor(src, code), ...) (or non_scaling_resize of it),
 * the regime chosen from the luma size as for BGR frames.  No extra pass and no extra buffer.  The frames of a batch may mix layouts
 * and sizes.  N > max_batch is HP_ERR_BATCH.  HP_ERR_ARG, before anything is enqueued: a null plane, a height or width <= 0 or odd,
 * pitch_y < width, pitch_uv < (width / 2) * uv_step, uv_step not 1 or 2, semi-planar u and v not one byte apart.
 * _host: each plane is copied row-compacted (1.5 bytes per pixel; a semi-planar UV plane once), by DMA from page-locked planes,
 * through pinned staging from pageable ones.  _device: the planes are read in place with the given pitches (an NVDEC surface as it
 * stands) and must stay valid and unchanged until the ticket is collected. */
typedef struct hp_frame_yuv420 {
    const uint8_t *y, *u, *v;
    int32_t height, width;       /* luma size, both even */
    int32_t pitch_y, pitch_uv;   /* bytes from one row to the next */
    int32_t uv_step;             /* 2: semi-planar (NV12 v = u + 1, NV21 u = v + 1); 1: planar (I420, YV12) */
} hp_frame_yuv420;
int hp_pose_submit_frames_yuv420_host(hp_engine* e, hp_paf* parser, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_frames_yuv420_device(hp_engine* e, hp_paf* parser, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_host(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_device(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420* frames, int N, int keep_ratio, int* ticket);
/* The same calls for interleaved frames with a row pitch: webcams' YUYV (the V4L2 / UVC default), capture cards' UYVY, YVYU, 4-byte
 * surfaces (GStreamer BGRx / RGBx, DeepStream's RGBA NvBufSurface, desktop capture's BGRA), RGB (PIL, torchvision, PyAV), gray (IR
 * and industrial cameras) and BGR, for all three head types.  Each source pixel is converted to BGR as cv::cvtColor does --
 * COLOR_RGB2BGR, _BGRA2BGR, _RGBA2BGR (alpha / x ignored), _GRAY2BGR (replicated), _YUV2BGR_YUYV / _UYVY / _YVYU (one U, V pair per
 * 2x1 pixel pair, BT.601 limited range in OpenCV's 20-bit fixed point, as the 4:2:0 calls) -- inside the batched resize's fetch,
 * before any interpolation: the network-size frame is byte-identical to cv::resize(cv::cvtColor(src, code), ...) (or
 * non_scaling_resize of it), the regime chosen from the pixel size as for hp_frame_u8.  HP_PIX_BGR with pitch = 3 * width is the
 * hp_frame_u8 call.  The frames of a batch may mix formats and sizes.  N > max_batch is HP_ERR_BATCH.  HP_ERR_ARG, before anything
 * is enqueued: a null data, a height or width <= 0, an unknown format, a 4:2:2 frame of odd width, pitch < width * bytes per pixel.
 * _host: each frame is copied row-compacted (width * bytes per pixel per row: 2 for 4:2:2, 1 for gray), by a pitched DMA from
 * page-locked frames (keep them alive until collect), through pinned staging from pageable ones before submit returns.  _device: the
 * frames are read in place with their pitch (a cudaMallocPitch / NvBufSurface / cropped surface as it stands) and must stay valid and
 * unchanged until the ticket is collected; the bytes between a row's end and the pitch are never read. */
typedef enum hp_pixel_format {
    HP_PIX_BGR = 0, HP_PIX_RGB, HP_PIX_BGRA, HP_PIX_RGBA, HP_PIX_GRAY,   /* 3, 3, 4, 4, 1 bytes per pixel */
    HP_PIX_YUYV, HP_PIX_UYVY, HP_PIX_YVYU                               /* 4:2:2, 2 bytes per pixel: Y0 U Y1 V, U Y0 V Y1, Y0 V Y1 U */
} hp_pixel_format;
typedef struct hp_frame_interleaved {
    const uint8_t* data;
    int32_t height, width;
    int32_t pitch;    /* bytes from one row to the next */
    int32_t format;   /* hp_pixel_format */
} hp_frame_interleaved;
int hp_pose_submit_frames_interleaved_host(hp_engine* e, hp_paf* parser, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_frames_interleaved_device(hp_engine* e, hp_paf* parser, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved_host(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved_device(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved* frames, int N, int keep_ratio, int* ticket);
/* The YUV 4:2:0 and interleaved calls for rotated frames: phone video stored landscape with a rotation in its display matrix, cameras
 * mounted sideways or upside down.  rotation[f] is frame f's clockwise rotation in degrees: 0, 90 (cv::ROTATE_90_CLOCKWISE), 180
 * (cv::ROTATE_180) or 270 (cv::ROTATE_90_COUNTERCLOCKWISE); rotation NULL is every frame upright, the calls above.  The network-size
 * frame is byte-identical to cv::resize(cv::rotate(cv::cvtColor(src, code), rotate_code), ...) (or non_scaling_resize of it): the
 * conversion happens in the stored grid (a 4:2:0 pixel takes the chroma of its 2x2 block, a 4:2:2 pixel the U, V pair of its pixel
 * pair, as stored), the rotation is a permutation of the fetch inside the same batched resize (no extra pass, no extra buffer), and
 * the regime and the letterbox come from the rotated size (height and width swapped for 90 and 270).  The records describe the
 * rotated frame: they are what the calls above return for the frame rotated beforehand.  A rotation other than 0, 90, 180 or 270 is
 * HP_ERR_ARG before anything is enqueued, as is everything the calls above refuse.  _host frames are copied in their stored
 * orientation, as above; _device frames are read in place with their pitch (a rotated NVDEC surface as it stands).  For hp_frame_u8,
 * use HP_PIX_BGR with pitch = 3 * width. */
int hp_pose_submit_frames_yuv420_rotated_host(hp_engine* e, hp_paf* parser, const hp_frame_yuv420* frames, const int32_t* rotation, int N,
                                              int keep_ratio, int* ticket);
int hp_pose_submit_frames_yuv420_rotated_device(hp_engine* e, hp_paf* parser, const hp_frame_yuv420* frames, const int32_t* rotation, int N,
                                                int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_rotated_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420* frames, const int32_t* rotation,
                                                     int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_rotated_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420* frames, const int32_t* rotation,
                                                       int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_rotated_host(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420* frames, const int32_t* rotation, int N,
                                                  int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_rotated_device(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420* frames, const int32_t* rotation, int N,
                                                    int keep_ratio, int* ticket);
int hp_pose_submit_frames_interleaved_rotated_host(hp_engine* e, hp_paf* parser, const hp_frame_interleaved* frames, const int32_t* rotation,
                                                   int N, int keep_ratio, int* ticket);
int hp_pose_submit_frames_interleaved_rotated_device(hp_engine* e, hp_paf* parser, const hp_frame_interleaved* frames, const int32_t* rotation,
                                                     int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved_rotated_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved* frames,
                                                          const int32_t* rotation, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved_rotated_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved* frames,
                                                            const int32_t* rotation, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved_rotated_host(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved* frames,
                                                       const int32_t* rotation, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved_rotated_device(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved* frames,
                                                         const int32_t* rotation, int N, int keep_ratio, int* ticket);
/* The YUV 4:2:0 and interleaved calls for frames whose samples are 16-bit words: 10 / 12-bit video (NVDEC's P010 / P016, FFmpeg's
 * p010le / p016le, yuv420p10le / p12le / p16le), 16-bit images (Mono12 / Mono16 cameras, 16-bit PNG / TIFF gray, RGB, RGBA).  Each
 * sample v, holding `bits` significant bits LSB-aligned (9 <= bits <= 16), is first reduced to the byte that OpenCV's
 * src.convertTo(dst, CV_8U, 1.0 / (1 << (bits - 8))) gives: saturate(rint_half_even(v * 2^-(bits - 8))).  P010 / P016 are
 * MSB-aligned: pass bits = 16; yuv420p10le is bits = 10 (1023 saturates to 255).  The 8-bit calls above then run on the reduced
 * bytes, unchanged, inside the same batched resize's fetch: the network-size frame is byte-identical to
 * cv::resize(cv::rotate(cv::cvtColor(convertTo(src16, CV_8U, 2^-(bits-8)), code), rotate_code), ...) (or non_scaling_resize of it).
 * rotation as for the _rotated_ calls (NULL: every frame upright).  No extra pass and no extra buffer.  The frames of a batch may mix
 * layouts, formats, sizes, bits and rotations.  Every pointer, pitch and uv_step is as in the 8-bit records, but counted over 16-bit
 * samples where the 8-bit ones count bytes: pitches stay in bytes, uv_step is in samples.  HP_ERR_ARG, before anything is enqueued:
 * everything the 8-bit calls refuse, bits outside 9..16, a pointer or pitch that is not 2-byte aligned, semi-planar u and v not one
 * sample apart, and in the interleaved call a 4:2:2 format (only HP_PIX_BGR, _RGB, _BGRA, _RGBA, _GRAY: BGR48, RGB48, BGRA64,
 * RGBA64, GRAY16).  _host: copied row-compacted at 2 bytes per sample, by a pitched DMA from page-locked frames, through pinned
 * staging from pageable ones.  _device: read in place with their pitch; the bytes between a row's end and the pitch are never read. */
typedef struct hp_frame_yuv420_16 {
    const uint16_t *y, *u, *v;
    int32_t height, width;       /* luma size, both even */
    int32_t pitch_y, pitch_uv;   /* bytes from one row to the next, even */
    int32_t uv_step;             /* samples: 2 semi-planar (P010 / P016 v = u + 1, V-first u = v + 1); 1 planar (I420, YV12 order) */
    int32_t bits;                /* significant bits per sample, LSB-aligned: 9..16 (16 for P010 / P016) */
} hp_frame_yuv420_16;
typedef struct hp_frame_interleaved16 {
    const uint16_t* data;
    int32_t height, width;
    int32_t pitch;    /* bytes from one row to the next, even */
    int32_t format;   /* HP_PIX_BGR, _RGB, _BGRA, _RGBA or _GRAY: 3, 3, 4, 4, 1 samples per pixel */
    int32_t bits;     /* as in hp_frame_yuv420_16 */
} hp_frame_interleaved16;
int hp_pose_submit_frames_yuv420_16_host(hp_engine* e, hp_paf* parser, const hp_frame_yuv420_16* frames, const int32_t* rotation, int N,
                                         int keep_ratio, int* ticket);
int hp_pose_submit_frames_yuv420_16_device(hp_engine* e, hp_paf* parser, const hp_frame_yuv420_16* frames, const int32_t* rotation, int N,
                                           int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_16_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420_16* frames, const int32_t* rotation,
                                                int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_yuv420_16_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_yuv420_16* frames, const int32_t* rotation,
                                                  int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_16_host(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420_16* frames, const int32_t* rotation, int N,
                                             int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_yuv420_16_device(hp_engine* e, hp_ppn* parser, const hp_frame_yuv420_16* frames, const int32_t* rotation, int N,
                                               int keep_ratio, int* ticket);
int hp_pose_submit_frames_interleaved16_host(hp_engine* e, hp_paf* parser, const hp_frame_interleaved16* frames, const int32_t* rotation,
                                             int N, int keep_ratio, int* ticket);
int hp_pose_submit_frames_interleaved16_device(hp_engine* e, hp_paf* parser, const hp_frame_interleaved16* frames, const int32_t* rotation,
                                               int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved16_host(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved16* frames,
                                                    const int32_t* rotation, int N, int keep_ratio, int* ticket);
int hp_pose_submit_pifpaf_frames_interleaved16_device(hp_engine* e, hp_pifpaf* decoder, const hp_frame_interleaved16* frames,
                                                      const int32_t* rotation, int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved16_host(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved16* frames, const int32_t* rotation,
                                                 int N, int keep_ratio, int* ticket);
int hp_pose_submit_ppn_frames_interleaved16_device(hp_engine* e, hp_ppn* parser, const hp_frame_interleaved16* frames,
                                                   const int32_t* rotation, int N, int keep_ratio, int* ticket);
/* test hook: the first N resized network-size frames [N,in_h,in_w,3] of an in-flight or collected ticket */
int hp_pose_debug_read_slot_frames(hp_engine* e, int ticket, uint8_t* out, int N);
int hp_pifpaf_pipeline_info(hp_pifpaf* p, void** stream, void** inputs_free_event, int* hcap);
int hp_pifpaf_copy_results_host_async(hp_pifpaf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream);
int hp_pifpaf_grow_capacity(hp_pifpaf* p, int flags);
/* building blocks of the above (also usable on their own): pre-allocate for a geometry / read the state a captured launch
 * sequence bakes in / enqueue the record D2H into PINNED caller memory / grow after an overflow */
int hp_paf_prepare(hp_paf* p, int N, int c_conf, int c_paf, int H, int W);
int hp_paf_state(const hp_paf* p, float* thresholds2, int* ints6);
int hp_paf_copy_results_host_async(hp_paf* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream);
int hp_paf_grow_capacity(hp_paf* p, int flags);
/* the same for the Pose Proposal Network parser: prepare checks the geometry and allocates for N frames; state gives the point / limb /
 * NMS thresholds and {net_w, net_h, hcap, use_spill, prepared N, device}; the D2H writes counts_flags[2N] ([N counts | N flags]) and
 * humans[N * hcap]; grow takes the flags OR-ed over the batch and its largest per-frame count (HP_ERR_CAPACITY: nothing left to grow) */
int hp_ppn_prepare(hp_ppn* p, int N, int K, int gh, int gw, int E, int nh, int nw);
int hp_ppn_state(const hp_ppn* p, float* thresholds3, int* ints6);
int hp_ppn_copy_results_host_async(hp_ppn* p, hp_human* pin_humans, int* pin_counts_flags, int N, void* stream);
int hp_ppn_grow_capacity(hp_ppn* p, int flags, int max_count);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU (SURVEY 8e): frames are independent, so they shard across the GPUs of one box with no data-path collective.
 * One PROCESS, one host thread + engine + parser + stream pair per GPU (weights replicated).  N_total frames are cut into
 * blocks of max_batch; block k (frames [k*B, (k+1)*B)) runs on GPU k % n -- GPU g gets frames [g*B, (g+1)*B) of every
 * super-batch of n*B frames -- each GPU pipelines its blocks two deep, and the humans come back in frame order.
 * The reference has no multi-GPU path at all (one TensorRT context, src/tensorrt.cpp:387-396).
 * ---------------------------------------------------------------------------------------- */
typedef struct hp_pool hp_pool;
/* devices: n CUDA ordinals (NULL = 0..n-1); the remaining arguments as hp_engine_create / hp_paf_create */
int hp_pool_create(hp_pool** out, const int* devices, int n_devices, const void* pack, size_t pack_bytes, int in_w, int in_h,
                   int max_batch, double factor, int flip_rgb, float conf_thresh, float paf_thresh);
void hp_pool_destroy(hp_pool* p);
int hp_pool_size(const hp_pool* p);
int hp_pool_set_capacity(hp_pool* p, int max_peaks_per_part, int max_candidates_per_limb, int max_humans);
/* frames: HOST u8 [n_total, in_h, in_w, 3]; out[n_total * cap], n_out[n_total] */
int hp_pool_run_u8_host(hp_pool* p, const uint8_t* frames, int n_total, hp_human* out, int cap, int* n_out);
int hp_pool_set_output_override(hp_pool* p, const float* const* d_conf, const float* const* d_paf);
long long hp_pool_launch_count(const hp_pool* p);
/* Device of the C++ drop-in classes (hyperpose::dnn::tensorrt has no device argument): env HPB_DEVICE = <ordinal> | "rr"
 * (engine instances take the GPUs round-robin); unset = 0.  A parser created by the drop-in follows the engine whose
 * published batch it is first handed (hp_handoff_device_of), else this default. */
int hp_default_device(void);
/* device of the published batch that owns this host buffer (engine -> parser hand-off), or -1 */
int hp_handoff_device_of(const float* host_conf);

#ifdef __cplusplus
}
#endif
#endif /* HYPERPOSE_B200_H */
