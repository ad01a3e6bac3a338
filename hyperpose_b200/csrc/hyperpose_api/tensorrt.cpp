// hyperpose_api/tensorrt.cpp -- hyperpose::dnn::tensorrt implemented on the hyperpose_b200 C ABI (no TensorRT).
//
// Drop-in replacement for the reference's src/tensorrt.cpp (same seam as src/fake/fake_tensorrt.cpp),
// compiled against the UNCHANGED include/hyperpose/operator/dnn/tensorrt.hpp.  All three constructors
// accept the path of an HPB2PACK model pack (hyperpose_b200/models.py) in place of the .uff/.onnx/.trt file;
// a file that is not a pack is a fatal error, like an unparsable model in the reference (tensorrt.cpp:141-158).
// inference() returns, per image, the outputs ordered by name (conf < paf, tensorrt.cpp:405; paf < pif for OpenPifPaf
// packs; the seven Pose Proposal Network maps for PPN packs) as host feature_map_t objects with shape [C,H,W] ([19,9,h,w] /
// [17,5,h,w]; [K,gh,gw] x6 and [17,9,9,gh,gw]), exactly as the reference does;
// the same buffers are published for the device-resident hand-off to the parsers (csrc/handoff.h).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
#include <stdexcept>

#include <hyperpose/operator/dnn/tensorrt.hpp>

#include "hyperpose_b200.h"

namespace hyperpose {
namespace dnn {

    namespace {
        [[noreturn]] void die(const std::string& what)
        {
            std::cerr << "[HyperPose::ERROR  ] " << what << ": " << hp_last_error() << '\n';
            std::exit(1);
        }
        // data_type of the reference ctor (tensorrt.hpp:14-22,48,61): kFLOAT (the default every example uses) selects the wgmma
        // kind tf32 engine (fp32 tensors, TF32 multiplies -- TensorRT's own FP32 convolution math on tensor-core GPUs), kHALF the
        // f16 engine, kINT8 the int8 engine when the pack carries a calibration table (hyperpose_b200.export --int8-calibration) and
        // the tf32 engine otherwise.  A serialized engine carries no precision argument in the reference API (its plan was built with
        // one): the pack runs as kHALF unless HPB_DTYPE=tf32 | int8 says otherwise.
        constexpr int INT8_IF_CALIBRATED = -1;
        int dtype_of(const data_type& t)
        {
            return t.val == data_type::kHALF ? HP_DTYPE_F16 : t.val == data_type::kINT8 ? INT8_IF_CALIBRATED : HP_DTYPE_TF32;
        }
        int serialized_dtype()
        {
            const char* v = std::getenv("HPB_DTYPE");
            if (v && std::string(v) == "tf32") return HP_DTYPE_TF32;
            if (v && std::string(v) == "int8") return HP_DTYPE_INT8;
            return HP_DTYPE_F16;
        }
        hp_engine* load_engine(const std::string& path, cv::Size input_size, int max_batch, double factor, bool flip_rgb, int dtype)
        {
            std::ifstream f(path, std::ios::binary | std::ios::ate);
            if (!f) die("cannot open model pack " + path);
            const std::streamsize n = f.tellg();
            f.seekg(0);
            std::vector<char> blob((size_t)n);
            if (!f.read(blob.data(), n)) die("cannot read model pack " + path);
            if (dtype == INT8_IF_CALIBRATED) dtype = hp_pack_int8_calibrated(blob.data(), blob.size()) ? HP_DTYPE_INT8 : HP_DTYPE_TF32;
            hp_engine* e = nullptr;
            // the reference API has no device argument: HPB_DEVICE=<ordinal> | rr (round-robin per engine instance), default 0
            if (hp_engine_create_ex(&e, blob.data(), blob.size(), input_size.width, input_size.height, max_batch, factor, flip_rgb ? 1 : 0, hp_default_device(), dtype) != HP_OK)
                die("hp_engine_create(" + path + ")");
            return e;
        }
    }

    struct tensorrt::cuda_dep {
        hp_engine* engine = nullptr;
        std::string pack_path; // what save() re-emits
        int c_conf = 0, c_paf = 0, out_h = 0, out_w = 0;
        ~cuda_dep() { hp_engine_destroy(engine); }
    };

    tensorrt::tensorrt(const uff& m, cv::Size input_size, int max_batch_size, bool keep_ratio, data_type dtype, double factor, bool flip_rgb)
        : m_inp_size(input_size), m_max_batch_size(max_batch_size), m_keep_ratio(keep_ratio), m_factor(factor), m_flip_rgb(flip_rgb)
        , m_cuda_dep(std::make_unique<cuda_dep>())
    {
        m_cuda_dep->engine = load_engine(m.model_path, input_size, max_batch_size, factor, flip_rgb, dtype_of(dtype));
        m_cuda_dep->pack_path = m.model_path;
        _create_binding_buffers();
    }
    tensorrt::tensorrt(const onnx& m, cv::Size input_size, int max_batch_size, bool keep_ratio, data_type dtype, double factor, bool flip_rgb)
        : m_inp_size(input_size), m_max_batch_size(max_batch_size), m_keep_ratio(keep_ratio), m_factor(factor), m_flip_rgb(flip_rgb)
        , m_cuda_dep(std::make_unique<cuda_dep>())
    {
        m_cuda_dep->engine = load_engine(m.model_path, input_size, max_batch_size, factor, flip_rgb, dtype_of(dtype));
        m_cuda_dep->pack_path = m.model_path;
        _create_binding_buffers();
    }
    tensorrt::tensorrt(const tensorrt_serialized& m, cv::Size input_size, int max_batch_size, bool keep_ratio, double factor, bool flip_rgb)
        : m_inp_size(input_size), m_max_batch_size(max_batch_size), m_keep_ratio(keep_ratio), m_factor(factor), m_flip_rgb(flip_rgb)
        , m_cuda_dep(std::make_unique<cuda_dep>())
    {
        m_cuda_dep->engine = load_engine(m.model_path, input_size, max_batch_size, factor, flip_rgb, serialized_dtype());
        m_cuda_dep->pack_path = m.model_path;
        _create_binding_buffers();
    }

    void tensorrt::_create_binding_buffers()
    {
        hp_engine_info(m_cuda_dep->engine, nullptr, nullptr, nullptr, &m_cuda_dep->c_conf, &m_cuda_dep->c_paf, &m_cuda_dep->out_h, &m_cuda_dep->out_w, nullptr);
    }

    void tensorrt::_batching(std::vector<cv::Mat>&, std::vector<float>&) {} // batching happens on the GPU (im2col3_kernel)

    namespace {
        // tensorrt::inference's read-back (tensorrt.cpp:398-431): one host feature_map_t per image and output, ordered by
        // tensor name (:405).  PAF networks: "conf" [C,h,w] < "paf" [2L,h,w]; OpenPifPaf networks: "paf" [19,9,h,w] < "pif"
        // [17,5,h,w] -- the order pifpaf::process(packet[0], packet[1]) relies on (src/pifpaf.cpp:6-7).
        // The buffers are filled by ONE call that also publishes them for the device-resident hand-off (handoff.h): the
        // parser.process() calls that follow find the batch on the device and parse it once.
        // Pose Proposal Network packs (head_type 2): seven maps per image, conf_point, conf_iou, x, y, w, h [K,gh,gw] and edge
        // [L,nh,nw,gh,gw] -- the order pose_proposal::process(const std::vector<feature_map_t>&) reads them in
        // (proposal_network.hpp:51-62), under names that sort in that order.  A plain read-back: no parser looks PPN tensors up.
        std::vector<internal_t> collect_ppn(hp_engine* e, size_t batch, int cc, int cp, int oh, int ow)
        {
            static const char* const names[6] = { "0_conf_point", "1_conf_iou", "2_x", "3_y", "4_w", "5_h" };
            const size_t plane = (size_t)oh * ow, K = (size_t)cc / 6, n_edge = 17 * 9 * 9;
            if (cc % 6 || (size_t)cp != n_edge) die("PPN pack with " + std::to_string(cc) + " box / " + std::to_string(cp) + " edge channels (needs 6K / 17*9*9)");
            std::vector<std::unique_ptr<float[]>> boxes(batch);
            std::vector<std::unique_ptr<char[]>> edges(batch);
            std::vector<float*> pa(batch), pb(batch);
            for (size_t j = 0; j < batch; ++j) {
                boxes[j].reset(new float[cc * plane]);
                edges[j].reset(new char[cp * plane * sizeof(float)]);
                pa[j] = boxes[j].get();
                pb[j] = reinterpret_cast<float*>(edges[j].get());
            }
            if (hp_engine_read_outputs_frames(e, pa.data(), pb.data(), (int)batch, 0) != HP_OK) die("hp_engine_read_outputs_frames");
            std::vector<internal_t> ret(batch);
            for (size_t j = 0; j < batch; ++j) {
                for (int t = 0; t < 6; ++t) {
                    std::unique_ptr<char[]> m(new char[K * plane * sizeof(float)]);
                    std::memcpy(m.get(), pa[j] + t * K * plane, K * plane * sizeof(float));
                    ret[j].emplace_back(names[t], std::move(m), std::vector<int>{ (int)K, oh, ow });
                }
                ret[j].emplace_back("6_edge", std::move(edges[j]), std::vector<int>{ 17, 9, 9, oh, ow });
            }
            return ret;
        }

        std::vector<internal_t> collect(hp_engine* e, size_t batch, int cc, int cp, int oh, int ow)
        {
            const size_t plane = (size_t)oh * ow;
            const int head = hp_engine_head_type(e);
            if (head == 2) return collect_ppn(e, batch, cc, cp, oh, ow);
            const bool pifpaf = head == 1;
            std::vector<std::unique_ptr<char[]>> a(batch), b(batch);
            std::vector<float*> pa(batch), pb(batch);
            for (size_t j = 0; j < batch; ++j) {
                a[j].reset(new char[cc * plane * sizeof(float)]);
                b[j].reset(new char[cp * plane * sizeof(float)]);
                pa[j] = reinterpret_cast<float*>(a[j].get());
                pb[j] = reinterpret_cast<float*>(b[j].get());
            }
            if (hp_engine_read_outputs_frames(e, pa.data(), pb.data(), (int)batch, 1) != HP_OK) die("hp_engine_read_outputs_frames");
            std::vector<internal_t> ret(batch);
            for (size_t j = 0; j < batch; ++j) {
                if (pifpaf) { // engine tensor a = pif fields, b = paf fields
                    ret[j].emplace_back("paf", std::move(b[j]), std::vector<int>{ 19, 9, oh, ow });
                    ret[j].emplace_back("pif", std::move(a[j]), std::vector<int>{ 17, 5, oh, ow });
                } else {
                    ret[j].emplace_back("conf", std::move(a[j]), std::vector<int>{ cc, oh, ow });
                    ret[j].emplace_back("paf", std::move(b[j]), std::vector<int>{ cp, oh, ow });
                }
            }
            return ret;
        }
    }

    std::vector<internal_t> tensorrt::inference(const std::vector<float>& buffer, size_t batch_size)
    {
        const int rc = hp_engine_infer_f32_host(m_cuda_dep->engine, buffer.data(), (int)batch_size);
        if (rc == HP_ERR_BATCH) throw std::logic_error(hp_last_error());
        if (rc != HP_OK) die("hp_engine_infer_f32_host");
        return collect(m_cuda_dep->engine, batch_size, m_cuda_dep->c_conf, m_cuda_dep->c_paf, m_cuda_dep->out_h, m_cuda_dep->out_w);
    }

    std::vector<internal_t> tensorrt::inference(std::vector<cv::Mat> batch)
    {
        if (batch.size() > (size_t)m_max_batch_size)
            throw std::logic_error("Input batch size overflow: Yours@" + std::to_string(batch.size()) + " Max@" + std::to_string(m_max_batch_size));
        // Step 1 of the reference (cv::resize / non_scaling_resize on the CPU, tensorrt.cpp:446-451) runs on the GPU,
        // bit-exact with OpenCV's 8-bit bilinear; step 2 (_batching, NHWC->NCHW) is fused into the first conv's gather.
        for (size_t i = 0; i < batch.size(); ++i) {
            const cv::Mat& m = batch[i];
            if (m.type() != CV_8UC3 || !m.isContinuous() || m.empty()) {
                std::cerr << "[HyperPose::ERROR  ] engine: frames must be continuous CV_8UC3\n";
                std::exit(-1);
            }
            if (hp_engine_stage_frame_u8(m_cuda_dep->engine, (int)i, m.data, m.rows, m.cols, m_keep_ratio ? 1 : 0) != HP_OK) die("hp_engine_stage_frame_u8");
        }
        if (hp_engine_infer_staged(m_cuda_dep->engine, (int)batch.size()) != HP_OK) die("hp_engine_infer_staged");
        return collect(m_cuda_dep->engine, batch.size(), m_cuda_dep->c_conf, m_cuda_dep->c_paf, m_cuda_dep->out_h, m_cuda_dep->out_w);
    }

    // tensorrt.cpp:463-471 serialises the built TensorRT plan.  Here the model pack IS the serialised engine (there
    // is no build step whose result would be worth caching), so save() re-emits the pack: the saved file is accepted
    // by tensorrt(tensorrt_serialized{path}, ...) exactly like the plan file in the reference
    // (examples/gen_serialized_engine.example.cpp:28-46).
    void tensorrt::save(const std::string path)
    {
        std::ifstream src(m_cuda_dep->pack_path, std::ios::binary);
        std::ofstream dst(path, std::ios::binary | std::ios::trunc);
        if (!src || !dst) die("save: cannot copy model pack " + m_cuda_dep->pack_path + " -> " + path);
        dst << src.rdbuf();
        if (!dst) die("save: write failed for " + path);
    }

    tensorrt::~tensorrt() = default;

} // namespace dnn

// member-wise constructor + printer of feature_map_t (include/hyperpose/utility/data.hpp:22,28): in a full
// integration these come from the reference's own src/data.cpp; they are repeated here only so that this
// translation unit links stand-alone (tests, the drop-in example) without OpenCV.
#ifdef HP_B200_STANDALONE
feature_map_t::feature_map_t(std::string name, std::unique_ptr<char[]>&& tensor, std::vector<int> shape)
    : m_name(std::move(name)), m_data(std::move(tensor)), m_shape(std::move(shape))
{
}
std::ostream& operator<<(std::ostream& out, const feature_map_t& map)
{
    out << map.m_name << ":[";
    for (auto& s : map.m_shape) out << s << ", ";
    return out << ']';
}
#endif
} // namespace hyperpose
