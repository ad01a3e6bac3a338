// pack_format.h -- the flat model pack consumed by hp_engine_create (replaces the reference's
// .onnx/.uff/.trt model files, include/hyperpose/utility/model.hpp:13-32; SURVEY 8f rank 1).
// Little-endian; written by hyperpose_b200/models.py.
//   PackHeader | PackBuffer[n_buffers] | PackOp[n_ops] | float blob[] | float act_scale[n_act_scales]
// The graph is a straight list of ops over numbered activation buffers (fp16 NHWC on the device).
#pragma once
#include <stdint.h>

namespace hpb {

constexpr char PACK_MAGIC[8] = { 'H', 'P', 'B', '2', 'P', 'A', 'C', 'K' };
constexpr uint32_t PACK_VERSION = 2;

enum PackOpType : uint32_t {
    OP_IM2COL3 = 1, // network input (u8 HWC frames or f32 NCHW) -> [N,OH,OW,roundup(R*R*3,64)] fp16: RxRx3 patches (k = (r*R+s)*3+c) + zeros,
                    // minus mean; R in {3,7}, stride 1/2, TF "SAME" padding
    OP_CONV = 2,    // stride-1 SAME convolution (odd R and S) + bias + PReLU (alpha 0 = ReLU, alpha 1 = linear)
    OP_MAXPOOL2 = 3, // RxR (R = 2 or 3) stride-2 max-pool, TF "SAME" semantics (out = ceil(in/2), window clipped at the border)
    OP_PIFPAF_HEAD = 5, // OpenPifPaf heads: pixel-shuffle(2) + crop + sigmoid/softplus + index grid of the two raw 1x1-conv outputs
                        // (in_buf = pif raw [.,.,340+], res_buf = paf raw [.,.,684+]) -> engine outputs pif[N,17,5,ho,wo], paf[N,19,9,ho,wo]
    OP_DWCONV = 4,   // depthwise KxK (K = 1 or 3) conv, stride 1/2, dilation 1 (or 2 for 3x3 / stride 1), TF "SAME" padding,
                     // + bias + PReLU; HBM-bound CUDA-core kernel
    OP_PPN_HEAD = 6  // Pose Proposal Network head: sigmoid + restore_coor of one raw 1x1-conv output (in_buf [.,.,6K + L*nh*nw+]) ->
                     // engine outputs conf[N,6,K,gh,gw] (conf_point, conf_iou, x, y, w, h) and paf[N,L,nh,nw,gh,gw];
                     // cout_g = K, groups = L, R x S = nh x nw
};

struct PackHeader {
    char magic[8];
    uint32_t version;
    uint32_t n_buffers, n_ops;
    uint32_t conf_channels, paf_channels; // channels of the two fp32 NCHW outputs handed to the parser
    uint32_t out_down_shift;              // outputs are at (H >> shift, W >> shift)
    float mean[3];                        // subtracted after scaling, per model-input channel (backbones.py:455)
    uint32_t head_type;                   // 0: conf/paf at (H >> shift); 1: OpenPifPaf fields at 2*(H >> shift) - 1 (pixel-shuffled, cropped);
                                          // 2: Pose Proposal Network boxes / edges at (H >> shift) (OP_PPN_HEAD)
    uint32_t reserved[4];                 // keeps blob_floats 8-byte aligned at offset 64.  reserved[0] = n_act_scales: 0, or n_buffers
                                          // when the INT8 calibration table (one fp32 scale per activation buffer) follows the blob
    uint64_t blob_floats;
};

struct PackBuffer {
    uint32_t channels;   // multiple of 8
    uint32_t down_shift; // spatial size = (in_h >> down_shift, in_w >> down_shift), ceil
};

struct PackOp {
    uint32_t type;
    uint32_t in_buf, out_buf;       // OP_IM2COL3 ignores in_buf
    uint32_t in_ch_off, out_ch_off;
    uint32_t R, S, groups, cin_g, cout_g;
    uint32_t out_mode;              // ConvOutMode; OUT_F32_NCHW_SPLIT writes the engine's conf/paf outputs
    uint32_t split;
    uint32_t im2col_input;          // 1: this conv consumes an OP_IM2COL3 buffer (R*S*cin_g <= 64 packed as one 64-ch k-step)
    uint32_t stride;                // OP_IM2COL3 / OP_DWCONV: 1 or 2 (0 = 1)
    uint32_t res_buf, res_ch_off;   // OP_CONV residual input (fp16 NHWC buffer of the output's geometry)
    uint32_t res_mode;              // 0 none | 1 y = act(conv + bias + res) (ResNet) | 2 y = act(conv + bias) + res (LW-OpenPose blocks)
    uint32_t dilation;              // OP_DWCONV: 1 or 2 (0 = 1), 2 only for 3x3 at stride 1 (SAME pads (3-1)*2/2 = 2 per side);
                                    // 0 for every other op
    uint64_t w_off, b_off, a_off;   // float offsets into the blob: W[G][cout_g][cin_g][R][S], bias[G*cout_g], alpha[G*cout_g]
                                    // OP_DWCONV: W[C][R][S], bias[C], alpha[C] with C = cout_g
};

static_assert(sizeof(PackHeader) == 72 && sizeof(PackBuffer) == 8 && sizeof(PackOp) == 96, "pack layout");

} // namespace hpb
