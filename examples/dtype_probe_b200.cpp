// examples/dtype_probe_b200.cpp -- the `data_type` a drop-in `hyperpose::dnn::tensorrt` is built with, seen from its outputs: one
// f32 frame through tensorrt::inference(const std::vector<float>&, 1) (tensorrt.hpp:119), conf then PAF written as raw float32.
// The same frame through an engine of each dtype tells which arithmetic the drop-in selected.  Only the reference's public headers.
//   usage: dtype_probe_b200 <model.pack> <width> <height> <kfloat|khalf|kint8|serialized> <out.bin>
//   serialized: tensorrt(tensorrt_serialized{pack}) -- no dtype argument; HPB_DTYPE selects it
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <memory>

#include <hyperpose/operator/dnn/tensorrt.hpp>

int main(int argc, char** argv)
{
    if (argc != 6) { std::cerr << "usage: " << argv[0] << " model.pack width height kfloat|khalf|kint8|serialized out.bin\n"; return 2; }
    namespace hp = hyperpose;
    const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
    const std::string mode = argv[4];
    std::unique_ptr<hp::dnn::tensorrt> engine;
    if (mode == "serialized") {
        engine = std::make_unique<hp::dnn::tensorrt>(hp::dnn::tensorrt_serialized{ argv[1] }, cv::Size(w, h), 1);
    } else {
        const int dt = mode == "kint8" ? hp::data_type::kINT8 : mode == "khalf" ? hp::data_type::kHALF : hp::data_type::kFLOAT;
        engine = std::make_unique<hp::dnn::tensorrt>(hp::dnn::onnx{ argv[1] }, cv::Size(w, h), 1, false, hp::data_type(dt));
    }
    std::vector<float> x((size_t)3 * h * w);
    for (size_t i = 0; i < x.size(); ++i) x[i] = (float)((i * 2654435761u) % 1024) / 1024.0f;   // pre-scaled NCHW, [0, 1)
    auto packets = engine->inference(x, 1);
    FILE* f = std::fopen(argv[5], "wb");
    if (!f) { std::cerr << "cannot write " << argv[5] << '\n'; return 1; }
    for (auto&& m : packets[0]) {
        size_t n = 1;
        for (int d : m.shape()) n *= (size_t)d;
        std::fwrite(m.view<float>(), sizeof(float), n, f);
        std::cout << m << '\n';
    }
    std::fclose(f);
    return 0;
}
