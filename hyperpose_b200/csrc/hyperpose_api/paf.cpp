// hyperpose_api/paf.cpp -- hyperpose::parser::paf implemented on the hyperpose_b200 C ABI.
//
// Drop-in replacement for the reference's src/paf.cpp (the same seam src/fake/fake_paf.cpp uses,
// cmake/hyperpose.fake.cmake:6-19): compiled against the reference's UNCHANGED
// include/hyperpose/operator/parser/paf.hpp, it defines exactly the symbols that header declares
// (ctor, copy-ctor, dtor, process, set_paf_thresh, set_conf_thresh, the two pimpl structs).
// Error conventions follow the reference: bad tensor rank / CUDA failure -> message on the error logger
// and std::exit(-1) (src/logging.hpp:31-37, src/paf.cpp:305-306).
#include <cstdio>
#include <cstdlib>
#include <iostream>

#include <hyperpose/operator/parser/paf.hpp>
#include <hyperpose/utility/logging.hpp>

#include "hyperpose_b200.h"

namespace hyperpose {
namespace parser {

    namespace {
        [[noreturn]] void die(const char* what)
        {
            std::cerr << "[HyperPose::ERROR  ] " << what << ": " << hp_last_error() << '\n';
            std::exit(-1);
        }
    }

    struct paf::ttl_impl {
        hp_paf* handle = nullptr;
        ~ttl_impl() { hp_paf_destroy(handle); }
    };
    struct paf::peak_finder_impl {
    };

    paf::paf(float conf_thresh, float paf_thresh, cv::Size resolution_size)
        : m_conf_thresh(conf_thresh)
        , m_paf_thresh(paf_thresh)
        , m_resolution_size(resolution_size)
        , m_ttl(UNINITIALIZED_PTR)
    {
    }

    // like the reference (paf.cpp:292-298) a copy shares nothing but the parameters; buffers are lazily created
    paf::paf(const paf& p)
        : m_conf_thresh(p.m_conf_thresh)
        , m_paf_thresh(p.m_paf_thresh)
        , m_resolution_size(p.m_resolution_size)
        , m_ttl(UNINITIALIZED_PTR)
    {
    }

    std::vector<human_t> paf::process(const feature_map_t& conf_map, const feature_map_t& paf_map)
    {
        if (conf_map.shape().size() != 3 || paf_map.shape().size() != 3) {
            std::cerr << "[HyperPose::ERROR  ] Input of PAF::PROCESS didn't meet requirements: [conf, paf], tensor.dims() == 3\n";
            std::exit(-1);
        }
        if (!m_ttl) {
            m_ttl = std::make_unique<ttl_impl>();
            // device: the GPU of the engine whose published batch these tensors belong to (engine -> parser hand-off), else the default
            int dev = hp_handoff_device_of(conf_map.view<float>());
            if (dev < 0) dev = hp_default_device();
            if (hp_paf_create(&m_ttl->handle, m_conf_thresh, m_paf_thresh, m_resolution_size.width, m_resolution_size.height, dev) != HP_OK)
                die("hp_paf_create");
            m_n_joints = conf_map.shape()[0];
            m_n_connections = paf_map.shape()[0] / 2;
            m_feature_size = cv::Size(conf_map.shape()[1], conf_map.shape()[2]); // (fw, fh) as in paf.cpp:329
            if (m_resolution_size.width == UNINITIALIZED_VAL || m_resolution_size.height == UNINITIALIZED_VAL)
                m_resolution_size = cv::Size(conf_map.shape()[1] * 4, conf_map.shape()[2] * 4); // paf.cpp:314-315
        }
        hp_paf_set_conf_thresh(m_ttl->handle, m_conf_thresh);
        hp_paf_set_paf_thresh(m_ttl->handle, m_paf_thresh);

        int cap = 64, n = 0;
        std::vector<hp_human> buf;
        for (;;) {
            buf.resize(cap);
            const int rc = hp_paf_process_host(m_ttl->handle, conf_map.view<float>(), paf_map.view<float>(), conf_map.shape()[0],
                paf_map.shape()[0], conf_map.shape()[1], conf_map.shape()[2], buf.data(), cap, &n);
            if (rc == HP_OK) break;
            if (rc == HP_ERR_CAPACITY && cap < (1 << 16)) { cap *= 4; continue; }
            die("hp_paf_process_host");
        }
        std::vector<human_t> humans(n);
        for (int i = 0; i < n; ++i) {
            humans[i].score = buf[i].score;
            for (int k = 0; k < COCO_N_PARTS; ++k) {
                humans[i].parts[k].has_value = buf[i].parts[k].has_value != 0;
                humans[i].parts[k].x = buf[i].parts[k].x;
                humans[i].parts[k].y = buf[i].parts[k].y;
                humans[i].parts[k].score = buf[i].parts[k].score;
            }
        }
        return humans;
    }

    void paf::set_paf_thresh(float thresh) { m_paf_thresh = thresh; }
    void paf::set_conf_thresh(float thresh) { m_conf_thresh = thresh; }

    paf::~paf() = default;

} // namespace parser
} // namespace hyperpose
