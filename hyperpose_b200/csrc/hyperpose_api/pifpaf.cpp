// hyperpose_api/pifpaf.cpp -- hyperpose::parser::pifpaf::process implemented on the hyperpose_b200 C ABI.
// Drop-in replacement for the reference's src/pifpaf.cpp (+ src/pifpaf_decoder/*), compiled against the UNCHANGED
// include/hyperpose/operator/parser/pifpaf.hpp.  The argument-order quirk is kept: the definition takes (paf, pif)
// (src/pifpaf.cpp:6-7, "TODO: Name ORDER!") because the engine returns its outputs sorted by name.
#include <cstdlib>
#include <iostream>

#include <hyperpose/operator/parser/pifpaf.hpp>

#include "hyperpose_b200.h"

namespace hyperpose::parser {

std::vector<human_t> pifpaf::process(const feature_map_t& paf, const feature_map_t& pif)
{
    if (pif.shape().size() != 4 || paf.shape().size() != 4) {
        std::cerr << "[HyperPose::ERROR  ] pifpaf::process expects [19,9,h,w] and [17,5,h,w] tensors\n";
        std::exit(-1);
    }
    const int h = pif.shape()[2], w = pif.shape()[3];
    // the reference constructs a fresh decoder per call (src/pifpaf.cpp:21); the device buffers are kept per thread here
    thread_local hp_pifpaf* handle = nullptr;
    thread_local int cur_h = 0, cur_w = 0;
    thread_local float cur_t = -1.f;
    if (!handle || cur_h != m_net_h || cur_w != m_net_w || cur_t != m_keypoint_thresh) {
        if (handle) hp_pifpaf_destroy(handle);
        int dev = hp_handoff_device_of(pif.view<float>());
        if (dev < 0) dev = hp_default_device();
        if (hp_pifpaf_create(&handle, m_net_h, m_net_w, m_keypoint_thresh, dev) != HP_OK) {
            std::cerr << "[HyperPose::ERROR  ] hp_pifpaf_create: " << hp_last_error() << '\n';
            std::exit(-1);
        }
        cur_h = m_net_h; cur_w = m_net_w; cur_t = m_keypoint_thresh;
    }
    // the reference returns however many poses the decoder finds: grow the output array on HP_ERR_CAPACITY
    std::vector<hp_human> buf(256);
    int n = 0;
    for (;;) {
        const int rc = hp_pifpaf_process_host(handle, pif.view<float>(), paf.view<float>(), 1, h, w, buf.data(), (int)buf.size(), &n);
        if (rc == HP_OK) break;
        if (rc == HP_ERR_CAPACITY && buf.size() < (1u << 16)) { buf.resize(buf.size() * 4); continue; }
        std::cerr << "[HyperPose::ERROR  ] hp_pifpaf_process_host: " << hp_last_error() << '\n';
        std::exit(-1);
    }
    std::vector<human_t> ret(n);
    for (int i = 0; i < n; ++i) {
        ret[i].score = buf[i].score;
        for (int k = 0; k < COCO_N_PARTS; ++k) {
            ret[i].parts[k].has_value = buf[i].parts[k].has_value != 0;
            ret[i].parts[k].x = buf[i].parts[k].x;
            ret[i].parts[k].y = buf[i].parts[k].y;
            ret[i].parts[k].score = buf[i].parts[k].score;
        }
    }
    return ret;
}

} // namespace hyperpose::parser
