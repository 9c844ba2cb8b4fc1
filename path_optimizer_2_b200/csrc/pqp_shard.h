// pqp_shard.h — how the multi-device ABIs (pqp_multi.h, pqp_plan_multi.h) split a batch over their devices, and the
// one-host-thread-per-device fan-out of their host calls. No device code here.
#pragma once
#include <algorithm>
#include <thread>
#include <vector>

namespace pqp {

// contiguous shards of `per` = ceil(batch / devices) paths: device i takes [i * per, min(batch, (i + 1) * per)),
// empty when batch < devices
inline int shard_per(int batch, int devices) { return (batch + devices - 1) / devices; }

struct Shard {
    int first, count;
};

inline Shard shard_of(int batch, int per, int i) {
    const int lo = std::min(batch, i * per), hi = std::min(batch, lo + per);
    return {lo, hi - lo};
}

// work(i) for every device index i < devices: index 0 on the calling thread, every other on a host thread of its
// own; returns when all have. The callers are C entry points that never throw: a device whose thread cannot be
// started (std::system_error, or no memory for it) runs its work on the calling thread instead, so every index still
// runs exactly once.
template <typename F>
void fan_out(int devices, F &&work) {
    std::vector<std::thread> workers;
    for (int d = 1; d < devices; ++d) {
        try {
            workers.emplace_back(work, d);
        } catch (...) {
            work(d);
        }
    }
    work(0);
    for (auto &t : workers) t.join();
}

}  // namespace pqp
