// hyperpose_api/pose_proposal.cpp -- hyperpose::parser::pose_proposal implemented on the hyperpose_b200 C ABI.
// Drop-in replacement for the reference's src/pose_proposal.cpp, compiled against the UNCHANGED
// include/hyperpose/operator/parser/proposal_network.hpp.  The class holds only its parameters (no pimpl slot), so the
// device handle lives per thread, like the reference's stateless process() allows (one parser copy per pool thread,
// stream.hpp:139).
#include <cassert>
#include <cstdlib>
#include <iostream>

#include <hyperpose/operator/parser/proposal_network.hpp>

#include "hyperpose_b200.h"

namespace hyperpose {
namespace parser {

    pose_proposal::pose_proposal(cv::Size net_resolution, float point_thresh, float limb_thresh, float mns_thresh)
        : m_net_resolution(std::move(net_resolution))
        , m_point_thresh(point_thresh)
        , m_limb_thresh(limb_thresh)
        , m_nms_thresh(mns_thresh)
    {
    }

    void pose_proposal::set_point_thresh(float thresh) { m_point_thresh = thresh; }
    void pose_proposal::set_limb_thresh(float thresh) { m_limb_thresh = thresh; }
    void pose_proposal::set_nms_thresh(float thresh) { m_nms_thresh = thresh; }

    std::vector<human_t> pose_proposal::process(
        const feature_map_t& conf_point, const feature_map_t& conf_iou,
        const feature_map_t& x, const feature_map_t& y, const feature_map_t& w, const feature_map_t& h,
        const feature_map_t& edge)
    {
        // same preconditions as the reference's asserts (src/pose_proposal.cpp:76-80), but always checked
        if (conf_point.shape().size() != 3 || edge.shape().size() < 3 || conf_iou.shape().empty()
            || x.shape() != conf_point.shape() || y.shape() != conf_point.shape() || w.shape() != conf_point.shape() || h.shape() != conf_point.shape()
            || conf_iou.shape().front() > conf_point.shape().front()) {
            std::cerr << "[HyperPose::ERROR  ] pose_proposal::process expects [K,gh,gw] x6 and [E,nh,nw,gh,gw] tensors\n";
            std::exit(-1);
        }
        thread_local hp_ppn* handle = nullptr;
        thread_local int cur_w = 0, cur_h = 0;
        if (!handle || cur_w != m_net_resolution.width || cur_h != m_net_resolution.height) {
            if (handle) hp_ppn_destroy(handle);
            if (hp_ppn_create(&handle, m_net_resolution.width, m_net_resolution.height, m_point_thresh, m_limb_thresh, m_nms_thresh, hp_default_device()) != HP_OK) {
                std::cerr << "[HyperPose::ERROR  ] hp_ppn_create: " << hp_last_error() << '\n';
                std::exit(-1);
            }
            cur_w = m_net_resolution.width; cur_h = m_net_resolution.height;
        }
        hp_ppn_set_point_thresh(handle, m_point_thresh);
        hp_ppn_set_limb_thresh(handle, m_limb_thresh);
        hp_ppn_set_nms_thresh(handle, m_nms_thresh);
        // n_key_points is conf_iou's leading dimension (:84); the five box tensors are indexed with the conf_point strides
        const int K = conf_iou.shape().front(), gh = conf_point.shape()[1], gw = conf_point.shape()[2];
        std::vector<hp_human> buf(512);
        int n = 0;
        if (hp_ppn_process_host(handle, conf_point.view<float>(), x.view<float>(), y.view<float>(), w.view<float>(), h.view<float>(),
                edge.view<float>(), 1, K, gh, gw, edge.shape()[0], edge.shape()[1], edge.shape()[2], buf.data(), (int)buf.size(), &n)
            != HP_OK) {
            std::cerr << "[HyperPose::ERROR  ] hp_ppn_process_host: " << hp_last_error() << '\n';
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

}
} // namespace hyperpose
