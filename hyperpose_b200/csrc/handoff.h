// handoff.h -- device-resident engine -> parser hand-off BEHIND the reference's host-only `feature_map_t`
// (SURVEY 8f rank 2; include/hyperpose/stream/stream.hpp:326-385, src/tensorrt.cpp:398-431).
//
// The reference API moves every network output through host memory: tensorrt::inference() returns one host
// `feature_map_t` per image and output, and the caller (operator API loop, or the stream's thread-pool tasks) hands
// them to parser.process() one image at a time.  The drop-in keeps that interface (the headers are unchanged), but the
// bytes do not have to travel twice: when the engine fills the host buffers it also keeps a device-side snapshot of the
// batch and PUBLISHES the host addresses.  A parser that is handed a published address -- same pointers, same shape,
// and EVERY BYTE of both tensors still equal to what was published -- parses the whole batch once from the snapshot
// (one batched launch sequence instead of N H2D copies + N launch sequences) and serves the other N-1 process() calls
// from the cached records.  The content check is a full memcmp of the caller's buffers against the pinned host copy
// the publication keeps (the very bytes the D2H delivered; ~0.05 ms per 860 KB frame, against ~0.5 ms for the H2D +
// launch sequence it saves): a buffer that was edited in place, or freed and re-allocated at the same address with
// other contents, can never be served the previous batch's humans -- not even when the edit touches a single float.
// `feature_map_t` exposes its data only through `const T* view() const` (include/hyperpose/utility/data.hpp:40-45);
// the check does not rely on that.  A miss of any kind falls back to the ordinary host path; results are identical
// either way (same kernels).
#pragma once
#include <cuda_runtime.h>

#include <array>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/hyperpose_b200.h"

namespace hpb {
namespace handoff {

constexpr int HANDOFF_RING = 4;     // published batches kept per engine

// One published batch: device snapshot of the two output tensors + the host addresses they were copied to.
struct Batch {
    std::mutex mu;                   // serialises the lazy batched parse, content checks and retirement
    bool valid = false;
    int fail_count = 0;              // batched parses that overflowed a parser capacity; >= 2: stop trying on this batch
    int device = 0;
    int N = 0;
    size_t elems_a = 0, elems_b = 0; // floats per frame of tensor a (conf | pif) and b (paf)
    float* d_a = nullptr; float* d_b = nullptr;
    size_t cap_a = 0, cap_b = 0;     // floats allocated
    cudaEvent_t ready = nullptr;     // snapshot copies complete
    std::vector<const float*> host_a, host_b;
    float* pin = nullptr;            // pinned host copy of the published bytes: [N * elems_a | N * elems_b]
    size_t pin_floats = 0;
    // cache of the batched parse: key = parser kind + its parameters
    int cache_kind = 0;              // 0 empty | 1 PAF | 2 PifPaf
    float key_f[2] = { 0, 0 };
    int key_i[3] = { 0, 0, 0 };
    int hcap = 0;
    std::vector<hp_human> humans;    // [N][hcap]
    std::vector<int> counts;         // [N]
};

struct Hit {
    std::shared_ptr<Batch> batch;
    int frame = -1;
};

bool enabled();
void set_enabled(bool on);

// engine side -------------------------------------------------------------------------------------------------------
// Takes the engine's next ring slot (retiring whatever it held), snapshots d_a / d_b (N frames) on `st`, copies them to
// the slot's pinned host buffer (one D2H per tensor, synchronises `st`), fills the caller's per-frame buffers from it
// and registers their addresses.
int publish(std::shared_ptr<Batch>* ring, int* ring_pos, int device, cudaStream_t st, const float* d_a, const float* d_b, int N,
            size_t elems_a, size_t elems_b, float* const* host_a, float* const* host_b);
// engine teardown: unregister and free every slot of the ring
void retire_ring(std::shared_ptr<Batch>* ring);

// parser side -------------------------------------------------------------------------------------------------------
// Registry lookup by host address of tensor a (then b and the per-frame sizes must match).  No content check yet.
Hit lookup(const float* host_a, const float* host_b, size_t elems_a, size_t elems_b);
// Content check of frame `frame` (caller holds batch->mu): every byte of both host tensors still equals what was published.
bool contents_match(const Batch& b, int frame);

std::mutex& registry_mutex();
int device_of_locked(const float* host_a);   // caller holds registry_mutex()

void count_hit();
void count_batch_parse();
void count_miss();
void stats(long long* published, long long* hits, long long* batch_parses, long long* misses);

} // namespace handoff
} // namespace hpb
