// examples/stream_api_b200.cpp -- the reference's STREAM API (examples/stream_api_video_paf.example.cpp:80-95:
// hp::make_stream(engine, parser); stream.async() << input; stream.sync() >> writer) on the drop-in.
// The scheduler is the reference's own: include/hyperpose/stream/stream.hpp is instantiated as it is and src/stream.cpp,
// src/thread_pool.cpp, src/logging.cpp are compiled from the reference tree unchanged (hyperpose_b200/build.py::
// build_stream_example); only the engine and the parser underneath are the drop-in classes.  Input = in-memory frames
// (std::vector<cv::Mat>, one of the stream's input types), output = a frame sink; the poses the stream hands to its drawing
// stage are counted and compared with the operator-API sequence on the same frames.
//   usage: stream_api_b200 <model.pack> <width> <height> <max_batch> <frames>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <iostream>
#include <random>

#include <hyperpose/operator/dnn/tensorrt.hpp>
#include <hyperpose/operator/parser/paf.hpp>
#include <hyperpose/stream/stream.hpp>

#ifdef HP_STREAM_MOCK
// CPU self-check of this program's plumbing (tests/test_cpp_dropin.py): the reference's scheduler, this file's input / output
// handling and the shim, with a stand-in engine and parser that need no GPU.  Every frame "contains" (first byte % 3) people.
namespace mock {
struct engine {
    cv::Size size; int mb;
    cv::Size input_size() const { return size; }
    int max_batch_size() const { return mb; }
    std::vector<hyperpose::internal_t> inference(std::vector<cv::Mat> batch)
    {
        std::vector<hyperpose::internal_t> out(batch.size());
        for (size_t i = 0; i < batch.size(); ++i) {
            std::unique_ptr<char[]> a(new char[sizeof(float)]), b(new char[sizeof(float)]);
            *reinterpret_cast<float*>(a.get()) = (float)(batch[i].data[0] % 3);
            *reinterpret_cast<float*>(b.get()) = 0.f;
            out[i].emplace_back("conf", std::move(a), std::vector<int>{ 1, 1, 1 });
            out[i].emplace_back("paf", std::move(b), std::vector<int>{ 1, 1, 1 });
        }
        return out;
    }
};
struct parser {
    std::vector<hyperpose::human_t> process(const hyperpose::feature_map_t& conf, const hyperpose::feature_map_t&)
    {
        return std::vector<hyperpose::human_t>((size_t)conf.view<float>()[0]);
    }
    template <typename C> std::vector<hyperpose::human_t> process(C&& maps) { return process(maps[0], maps[1]); }
};
}
namespace hyperpose {
feature_map_t::feature_map_t(std::string name, std::unique_ptr<char[]>&& tensor, std::vector<int> shape)
    : m_name(std::move(name)), m_data(std::move(tensor)), m_shape(std::move(shape)) {}
}
#endif

namespace {
std::atomic<size_t> g_drawn{ 0 };
}

namespace hyperpose {
// the two drawing / letterbox helpers the stream's output stage calls live in the reference's src/human.cpp and src/data.cpp,
// which need real OpenCV drawing; here they record instead of drawing
void draw_human(cv::Mat&, const human_t&) { ++g_drawn; }
cv::Mat non_scaling_resize(const cv::Mat& input, const cv::Size& size, const cv::Scalar)
{
    cv::Mat out;
    cv::resize(input, out, size);
    return out;
}
}

int main(int argc, char** argv)
{
    if (argc < 6) { std::cerr << "usage: " << argv[0] << " model.pack width height max_batch frames\n"; return 2; }
    const int w = std::atoi(argv[2]), h = std::atoi(argv[3]), mb = std::atoi(argv[4]), n = std::atoi(argv[5]);
    namespace hp = hyperpose;
#ifdef HP_STREAM_MOCK
    mock::engine engine{ cv::Size(w, h), mb };
    mock::parser parser;
#else
    hp::dnn::tensorrt engine(hp::dnn::tensorrt_serialized{ argv[1] }, { w, h }, mb);
    hp::parser::paf parser{};
#endif

    std::mt19937 rng(7);
    std::vector<cv::Mat> frames;
    for (int i = 0; i < n; ++i) {
        cv::Mat m(cv::Size(w, h), CV_8UC3);
        for (size_t k = 0; k < m.total() * 3; ++k) m.data[k] = (unsigned char)(rng() & 0xff);
        frames.push_back(m);
    }

    // operator API on the same frames: the count the stream has to reproduce
    size_t want = 0;
    for (int i = 0; i < n; i += mb) {
        std::vector<cv::Mat> batch(frames.begin() + i, frames.begin() + std::min(n, i + mb));
        for (auto&& packet : engine.inference(batch)) want += parser.process(packet[0], packet[1]).size();
    }

    cv::VideoWriter writer("unused.avi", 0, 25.0, cv::Size(w, h));
    const auto beg = std::chrono::high_resolution_clock::now();
    {
        auto stream = hp::make_stream(engine, parser, false);
        // one frame at a time (basic_stream_manager::read_from(cv::Mat), src/stream.cpp:60-66).  The std::vector<cv::Mat> overload
        // (src/stream.cpp:18-30) is not usable: its loop condition `distance(it, end) <= step_size` copies step_size elements
        // from a vector that holds fewer -- it reads past the end for any input shorter than half the queue (seen as a
        // segmentation fault here); the reference's own examples only ever feed a cv::VideoCapture.
        for (auto& f : frames) stream.async() << f;
        stream.sync() >> writer;
    }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::high_resolution_clock::now() - beg).count();
    std::cout << writer.frames_written << " frames through the stream in " << ms << " ms, humans drawn = " << g_drawn.load()
              << ", operator API humans = " << want << '\n';
    const bool ok = writer.frames_written == (size_t)n && g_drawn.load() == want;
    std::cout << (ok ? "stream == operator API" : "MISMATCH") << '\n';
    return ok ? 0 : 1;
}
