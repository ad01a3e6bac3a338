// examples/operator_api_b200.cpp -- the reference's operator-API call sequence
// (examples/operator_api_batched_images_paf.example.cpp:58-74 and ..._pifpaf.example.cpp:48-64: engine.inference(batch),
// then parser.process(packet[0], packet[1]) per image) against the drop-in, using only the reference's
// public headers.  Frames are synthetic (no OpenCV image I/O here); the model is an HPB2PACK file.
//   usage: operator_api_b200 <model.pack> <width> <height> <batch> [save-as.pack|-] [iterations] [paf|pifpaf]
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <random>

#include <hyperpose/operator/dnn/tensorrt.hpp>
#include <hyperpose/operator/parser/paf.hpp>
#include <hyperpose/operator/parser/pifpaf.hpp>

int main(int argc, char** argv)
{
    if (argc < 5) { std::cerr << "usage: " << argv[0] << " model.pack width height batch [save-as.pack|-] [iterations] [paf|pifpaf]\n"; return 2; }
    const int w = std::atoi(argv[2]), h = std::atoi(argv[3]), n = std::atoi(argv[4]);
    const int iters = argc > 6 ? std::atoi(argv[6]) : 1;
    const bool use_pifpaf = argc > 7 && std::strcmp(argv[7], "pifpaf") == 0;
    namespace hp = hyperpose;
    hp::dnn::tensorrt engine(hp::dnn::tensorrt_serialized{ argv[1] }, { w, h }, n);
    if (argc > 5 && std::strcmp(argv[5], "-") != 0) engine.save(argv[5]); // examples/gen_serialized_engine.example.cpp:44
    hp::parser::paf paf_parser{};
    hp::parser::pifpaf pifpaf_parser(engine.input_size().height, engine.input_size().width);
    std::mt19937 rng(1);
    std::vector<cv::Mat> batch;
    for (int i = 0; i < n; ++i) {
        cv::Mat m(cv::Size(w, h), CV_8UC3);
        for (size_t k = 0; k < m.total() * 3; ++k) m.data[k] = (unsigned char)(rng() & 0xff);
        batch.push_back(m);
    }
    for (int it = 0; it < iters; ++it) {
        auto beg = std::chrono::high_resolution_clock::now();
        auto packets = engine.inference(batch);
        size_t humans = 0;
        for (auto&& packet : packets) {
            if (it == 0) std::cout << packet[0] << ' ' << packet[1] << '\n';
            humans += use_pifpaf ? pifpaf_parser.process(packet[0], packet[1]).size() : paf_parser.process(packet[0], packet[1]).size();
        }
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - beg).count();
        std::cout << batch.size() << " images got processed. FPS = " << 1000. * batch.size() / ms << " humans = " << humans << '\n';
    }
    return 0;
}
