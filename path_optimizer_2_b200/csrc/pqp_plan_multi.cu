// pqp_plan_multi.cu — include/pqp_plan_multi.h: the whole plan over the GPUs of one box, one pqp_plan_handle per
// device, contiguous shards, no collective. Built on the public single-device plan ABI (pqp_plan.h) only.
//
// Refusals: every device's handle has the same params, capacities and slot count, so an argument one handle refuses
// every handle refuses, before it enqueues anything. The device forms call the home handle first, so a refused call
// enqueues nothing on any device.
#include <cuda_runtime.h>

#include <new>
#include <string>
#include <vector>

#include "../../include/pqp_plan_multi.h"
#include "pqp_host_handle.h"
#include "pqp_plan_trace.h"
#include "pqp_shard.h"

namespace {

thread_local std::string g_plan_multi_create_error;

// the device-form staging of one device other than the home one, for per_max paths
struct Staging {
    double *x = nullptr, *y = nullptr, *start = nullptr, *target = nullptr, *path = nullptr, *cost = nullptr;
    int32_t *cnt = nullptr, *map_index = nullptr, *status = nullptr, *n = nullptr, *iters = nullptr;
    uint8_t *occ = nullptr;  // n_maps * cap_cells: the images of a device-form occupancy update
    double *boxes = nullptr;  // PQP_MAX_BOXES * PQP_BOX_FIELDS: the boxes of a device-form box update
    int32_t *box_k = nullptr;  // n_maps: their counts
};

}  // namespace

struct pqp_plan_multi_t {
    int n_dev = 0, batch_max = 0, per_max = 0, R = 0, P = 0, L = 0, N = 0;
    size_t cap_cells = 0;  // cells of the largest map given at create: those of a slot
    std::vector<int> dev;
    std::vector<pqp_plan_handle *> h;
    std::vector<cudaStream_t> stream;  // per device index: the device forms' stream (index 0: the caller's)
    std::vector<cudaEvent_t> done;     // per device index: its shard's work of a device-form call is complete
    cudaEvent_t fork = nullptr;        // on the home device: the point of the caller's stream the others wait for
    std::vector<Staging> st;
    int last_batch = 0, last_per = 0;
    std::string err;
    std::vector<pqp::Resources> res;  // one per device; last member: releasing clears the members above
};

namespace {

using pqp::fail;

template <typename T>
T *at(T *p, size_t offset) {
    return p ? p + offset : nullptr;
}

// a device handle's refusal or error as the multi-device handle's
int device_fail(pqp_plan_multi_t *m, int d, int rc) {
    return fail(m->err, rc, "device " + std::to_string(m->dev[d]) + ": " + pqp_plan_last_error(m->h[d]));
}

// the fields of one plan call that differ between the points and the samples form
struct Call {
    const pqp_plan_in *in;          // samples form, or NULL
    const pqp_plan_points_in *pts;  // points form, or NULL
    int batch() const { return pts ? pts->batch : in->batch; }
    int stride() const { return pts ? pts->m_max : in->r_max; }
    const double *x() const { return pts ? pts->ref_x : in->raw_x; }
    const double *y() const { return pts ? pts->ref_y : in->raw_y; }
    const int32_t *cnt() const { return pts ? pts->m : in->r; }
    const double *start() const { return pts ? pts->start : in->start; }
    const double *target() const { return pts ? pts->target : in->target; }
    // handle d plans `count` paths from these buffers into `out`
    int run(pqp_plan_handle *h, int count, const double *x, const double *y, const int32_t *cnt, const double *start,
            const double *target, const int32_t *map_index, const pqp_plan_out *out, cudaStream_t *stream) const {
        if (pts) {
            const pqp_plan_points_in v = {count, pts->m_max, x, y, cnt, start, target};
            if (stream) return map_index ? pqp_plan_points_mapped_device(h, &v, map_index, out, *stream)
                                         : pqp_plan_points_device(h, &v, out, *stream);
            return map_index ? pqp_plan_points_mapped(h, &v, map_index, out) : pqp_plan_points(h, &v, out);
        }
        const pqp_plan_in v = {count, in->r_max, x, y, cnt, start, target};
        if (stream) return map_index ? pqp_plan_mapped_device(h, &v, map_index, out, *stream)
                                     : pqp_plan_device(h, &v, out, *stream);
        return map_index ? pqp_plan_mapped(h, &v, map_index, out) : pqp_plan(h, &v, out);
    }
};

int validate(pqp_plan_multi_t *m, const Call &c, const pqp_plan_out *out) {
    if (!m) return PQP_E_INVALID;
    if (!(c.in || c.pts) || !out) return fail(m->err, PQP_E_INVALID, "null batch");
    if (c.batch() < 1 || c.batch() > m->batch_max) return fail(m->err, PQP_E_INVALID, "batch out of range");
    return PQP_OK;
}

// the outputs of `out` from path `first` on; `trace`: where the shard's trace view is kept
pqp_plan_out out_from(const pqp_plan_multi_t *m, const pqp_plan_out *out, size_t first, pqp_plan_trace *trace) {
    pqp_plan_out v = {at(out->status, first), at(out->n, first), at(out->path, first * PQP_PLAN_PATH_ROWS * m->N),
                      at(out->cost, first), at(out->iters, 2 * first), nullptr};
    if (out->trace) {
        *trace = pqpl::trace_from(*out->trace, first, m->P, m->L, m->N, m->R);
        v.trace = trace;
    }
    return v;
}

int plan_host(pqp_plan_multi_t *m, const Call &c, const int32_t *map_index, const pqp_plan_out *out) {
    int rc = validate(m, c, out);
    if (rc != PQP_OK) return rc;
    const int G = m->n_dev, B = c.batch(), per = pqp::shard_per(B, G);
    const size_t S = c.stride();
    std::vector<int> rcs(G, PQP_OK);
    std::vector<pqp_plan_trace> traces(G);
    pqp::fan_out(G, [&](int d) {
        const pqp::Shard sh = pqp::shard_of(B, per, d);
        if (sh.count == 0) return;
        const size_t lo = sh.first;
        const pqp_plan_out o = out_from(m, out, lo, &traces[d]);
        rcs[d] = c.run(m->h[d], sh.count, at(c.x(), lo * S), at(c.y(), lo * S), at(c.cnt(), lo), at(c.start(), 4 * lo),
                       at(c.target(), 3 * lo), at(map_index, lo), &o, nullptr);
    });
    for (int d = 0; d < G; ++d)
        if (rcs[d] != PQP_OK) return device_fail(m, d, rcs[d]);
    m->last_batch = B;
    m->last_per = per;
    return PQP_OK;
}

// lets `from` reach `to`'s memory directly, so that copies between the two go device to device rather than through
// the host; a pair the process already enabled stays as it is
cudaError_t enable_peer(int from, int to) {
    pqp::DeviceGuard g(from);
    const cudaError_t e = cudaDeviceEnablePeerAccess(to, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) {
        cudaGetLastError();  // clears it
        return cudaSuccess;
    }
    return e;
}

template <typename T>
cudaError_t peer_copy(T *dst, int dst_dev, const T *src, int src_dev, size_t count, cudaStream_t s) {
    return cudaMemcpyPeerAsync(dst, dst_dev, src, src_dev, count * sizeof(T), s);
}

// A device-form call on every device: `run(d, s)` enqueues device index d's part on stream s (a handle's refusal
// through device_fail). The home part runs first, on the caller's stream, so its refusal enqueues nothing anywhere;
// every other device with active(d) runs on its own stream between the fork and the caller's stream's join.
template <typename Run, typename Active>
int fork_join(pqp_plan_multi_t *m, cudaStream_t stream, Run &&run, Active &&active) {
    const int home = m->dev[0];
    {
        pqp::DeviceGuard g(home);
        PQP_CUDA(m->err, cudaEventRecord(m->fork, stream));
    }
    int rc = run(0, stream);
    if (rc != PQP_OK) return rc;
    for (int d = 1; d < m->n_dev; ++d) {
        if (!active(d)) continue;
        pqp::DeviceGuard g(m->dev[d]);
        PQP_CUDA(m->err, cudaStreamWaitEvent(m->stream[d], m->fork, 0));
        rc = run(d, m->stream[d]);
        if (rc != PQP_OK) return rc;
        PQP_CUDA(m->err, cudaEventRecord(m->done[d], m->stream[d]));
    }
    pqp::DeviceGuard g(home);
    for (int d = 1; d < m->n_dev; ++d)
        if (active(d)) PQP_CUDA(m->err, cudaStreamWaitEvent(stream, m->done[d], 0));
    return PQP_OK;
}

int plan_device(pqp_plan_multi_t *m, const Call &c, const int32_t *map_index, const pqp_plan_out *out,
                cudaStream_t stream) {
    int rc = validate(m, c, out);
    if (rc != PQP_OK) return rc;
    if (out->trace)
        return fail(m->err, PQP_E_INVALID,
                    "the device forms take no trace (a traced shard would need staging for every trace field); use the "
                    "host form");
    const int G = m->n_dev, B = c.batch(), per = pqp::shard_per(B, G), home = m->dev[0];
    const size_t S = c.stride(), N = m->N;
    rc = fork_join(m, stream, [&](int d, cudaStream_t sd) -> int {
        const pqp::Shard sh = pqp::shard_of(B, per, d);
        if (d == 0) {  // the home shard [0, per) on the caller's buffers
            const int hrc = c.run(m->h[0], sh.count, c.x(), c.y(), c.cnt(), c.start(), c.target(), map_index, out, &sd);
            return hrc == PQP_OK ? PQP_OK : device_fail(m, 0, hrc);
        }
        const size_t lo = sh.first, n = sh.count;
        const int dv = m->dev[d];
        const Staging &s = m->st[d];
        PQP_CUDA(m->err, peer_copy(s.x, dv, c.x() + lo * S, home, n * S, sd));
        PQP_CUDA(m->err, peer_copy(s.y, dv, c.y() + lo * S, home, n * S, sd));
        PQP_CUDA(m->err, peer_copy(s.cnt, dv, c.cnt() + lo, home, n, sd));
        PQP_CUDA(m->err, peer_copy(s.start, dv, c.start() + 4 * lo, home, 4 * n, sd));
        PQP_CUDA(m->err, peer_copy(s.target, dv, c.target() + 3 * lo, home, 3 * n, sd));
        if (map_index) PQP_CUDA(m->err, peer_copy(s.map_index, dv, map_index + lo, home, n, sd));
        const pqp_plan_out o = {s.status, s.n, s.path, s.cost, s.iters, nullptr};
        const int drc = c.run(m->h[d], sh.count, s.x, s.y, s.cnt, s.start, s.target, map_index ? s.map_index : nullptr,
                              &o, &sd);
        if (drc != PQP_OK) return device_fail(m, d, drc);
        PQP_CUDA(m->err, peer_copy(out->status + lo, home, s.status, dv, n, sd));
        PQP_CUDA(m->err, peer_copy(out->n + lo, home, s.n, dv, n, sd));
        PQP_CUDA(m->err, peer_copy(out->path + lo * PQP_PLAN_PATH_ROWS * N, home, s.path, dv, n * PQP_PLAN_PATH_ROWS * N, sd));
        PQP_CUDA(m->err, peer_copy(out->cost + lo, home, s.cost, dv, n, sd));
        PQP_CUDA(m->err, peer_copy(out->iters + 2 * lo, home, s.iters, dv, 2 * n, sd));
        return PQP_OK;
    }, [&](int d) { return pqp::shard_of(B, per, d).count > 0; });
    if (rc != PQP_OK) return rc;
    m->last_batch = B;
    m->last_per = per;
    return PQP_OK;
}

// A device-form occupancy update of slots first .. first + count - 1: pqp_plan_set_occupancy_boxes_device when
// `boxed`, else pqp_plan_set_occupancy_slots_device.
struct Occupancy {
    int first;
    const pqp_occupancy_stack *stack;
    bool boxed;
    int shared_base;
    const pqp_obstacle_boxes *boxes;
};

// An update the home handle accepted, peer-copied on sd into device index d's staging: the image(s), and k and the
// boxes when there are any. `r` becomes the update that reads them there, through `stack` and `boxes`.
int stage(pqp_plan_multi_t *m, int d, cudaStream_t sd, Occupancy &r, pqp_occupancy_stack &stack,
          pqp_obstacle_boxes &boxes) {
    const int dv = m->dev[d], home = m->dev[0];
    const Staging &st = m->st[d];
    stack = *r.stack;
    boxes = r.boxed ? *r.boxes : pqp_obstacle_boxes{};
    const size_t bytes = (size_t)(r.shared_base ? 1 : stack.count) * stack.rows * stack.cols;
    const size_t n_box = (size_t)stack.count * boxes.k_max;
    PQP_CUDA(m->err, peer_copy(st.occ, dv, stack.cells, home, bytes, sd));
    if (n_box) {
        PQP_CUDA(m->err, peer_copy(st.box_k, dv, boxes.k, home, (size_t)stack.count, sd));
        PQP_CUDA(m->err, peer_copy(st.boxes, dv, boxes.boxes, home, n_box * PQP_BOX_FIELDS, sd));
        boxes.k = st.box_k;
        boxes.boxes = st.boxes;
    }
    stack.cells = st.occ;
    r.stack = &stack;
    if (r.boxed) r.boxes = &boxes;
    return PQP_OK;
}

// the occupancy update on every device: once the caller's stream has passed it, every device's slots are final, as the
// single-device call's are, whichever stream (a host form's included) reads them next
int occupancy_device(pqp_plan_multi_t *m, const Occupancy &r, cudaStream_t stream) {
    if (!m) return PQP_E_INVALID;
    return fork_join(m, stream, [&](int d, cudaStream_t sd) -> int {
        Occupancy u = r;
        pqp_occupancy_stack stack;
        pqp_obstacle_boxes boxes;
        if (d > 0) {
            const int rc = stage(m, d, sd, u, stack, boxes);
            if (rc != PQP_OK) return rc;
        }
        const int rc = u.boxed ? pqp_plan_set_occupancy_boxes_device(m->h[d], u.first, u.stack, u.shared_base, u.boxes, sd)
                               : pqp_plan_set_occupancy_slots_device(m->h[d], u.first, u.stack, sd);
        return rc == PQP_OK ? PQP_OK : device_fail(m, d, rc);
    }, [](int) { return true; });
}

// a host-form update of every device's handle, concurrently
template <typename F>
int update_all(pqp_plan_multi_t *m, F &&update) {
    std::vector<int> rcs(m->n_dev, PQP_OK);
    pqp::fan_out(m->n_dev, [&](int d) { rcs[d] = update(m->h[d]); });
    for (int d = 0; d < m->n_dev; ++d)
        if (rcs[d] != PQP_OK) return device_fail(m, d, rcs[d]);
    return PQP_OK;
}

}  // namespace

extern "C" {

const char *pqp_plan_multi_last_error(const pqp_plan_multi_t *m) {
    return m ? m->err.c_str() : g_plan_multi_create_error.c_str();
}

int pqp_plan_multi_create_maps(const pqp_bounds_map *maps, int32_t n_maps, const pqp_plan_params *params,
                               int32_t r_max, int32_t p_max, int32_t layers_max, int32_t n_max, int32_t batch_max,
                               int32_t n_devices, const int32_t *devices, pqp_plan_multi_t **out) {
    std::string &err = g_plan_multi_create_error;
    if (!out) return fail(err, PQP_E_INVALID, "pqp_plan_multi_create_maps: out is null");
    *out = nullptr;
    if (!params || n_devices < 1 || batch_max < 1)
        return fail(err, PQP_E_INVALID, "pqp_plan_multi_create_maps: params required, n_devices >= 1, batch_max >= 1");
    if (!maps || n_maps < 1) return fail(err, PQP_E_INVALID, "pqp_plan_multi_create_maps: a map is required");
    // pqp_plan_create_maps' capacity rule, checked here too so that it refuses before the device lookup
    if (r_max < 3 || p_max < 4 || layers_max < 4 || n_max < 2 || n_max > 511)
        return fail(err, PQP_E_INVALID,
                    "pqp_plan_multi_create_maps: r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511");
    int visible = 0;
    if (cudaGetDeviceCount(&visible) != cudaSuccess) visible = 0;
    for (int d = 0; d < n_devices; ++d) {
        const int dv = devices ? devices[d] : d;
        if (dv < 0 || dv >= visible)
            return fail(err, PQP_E_NO_DEVICE, "pqp_plan_multi_create_maps: device " + std::to_string(dv) + " requested, " +
                                                  std::to_string(visible) +
                                                  " CUDA devices visible (there is no CPU fallback)");
    }
    pqp_plan_multi_t *m = new (std::nothrow) pqp_plan_multi_t;
    if (!m) return fail(err, PQP_E_INVALID, "out of host memory");
    const size_t G = n_devices;
    m->n_dev = n_devices;
    m->batch_max = batch_max;
    m->per_max = pqp::shard_per(batch_max, n_devices);
    m->R = r_max;
    m->P = p_max;
    m->L = layers_max;
    m->N = n_max;
    for (int i = 0; i < n_maps; ++i) {
        const size_t cells = (size_t)(maps[i].rows > 0 ? maps[i].rows : 0) * (size_t)(maps[i].cols > 0 ? maps[i].cols : 0);
        m->cap_cells = cells > m->cap_cells ? cells : m->cap_cells;
    }
    m->dev.resize(G);
    m->h.assign(G, nullptr);
    m->stream.assign(G, nullptr);
    m->done.assign(G, nullptr);
    m->st.assign(G, Staging{});
    m->res = std::vector<pqp::Resources>(G);
    for (int d = 0; d < n_devices; ++d) m->dev[d] = m->res[d].device = devices ? devices[d] : d;
    const int home = m->dev[0];
    const int rc = [&]() -> int {
        for (int d = 0; d < n_devices; ++d) {
            const int hrc = pqp_plan_create_maps(maps, n_maps, params, r_max, p_max, layers_max, n_max, m->per_max,
                                                 m->dev[d], &m->h[d]);
            if (hrc != PQP_OK)
                return fail(err, hrc, "device " + std::to_string(m->dev[d]) + ": " + pqp_plan_last_error(nullptr));
            pqp::DeviceGuard g(m->dev[d]);
            pqp::Resources &r = m->res[d];
            if (d == 0) {
                PQP_CUDA(err, r.event(m->fork, cudaEventDisableTiming));
                continue;
            }
            PQP_CUDA(err, r.stream(m->stream[d]));
            PQP_CUDA(err, r.event(m->done[d], cudaEventDisableTiming));
            Staging &s = m->st[d];
            const size_t B = m->per_max, R = r_max, N = n_max;
            PQP_CUDA(err, r.alloc(s.x, B * R));
            PQP_CUDA(err, r.alloc(s.y, B * R));
            PQP_CUDA(err, r.alloc(s.cnt, B));
            PQP_CUDA(err, r.alloc(s.start, B * 4));
            PQP_CUDA(err, r.alloc(s.target, B * 3));
            PQP_CUDA(err, r.alloc(s.map_index, B));
            PQP_CUDA(err, r.alloc(s.status, B));
            PQP_CUDA(err, r.alloc(s.n, B));
            PQP_CUDA(err, r.alloc(s.path, B * PQP_PLAN_PATH_ROWS * N));
            PQP_CUDA(err, r.alloc(s.cost, B));
            PQP_CUDA(err, r.alloc(s.iters, B * 2));
            PQP_CUDA(err, r.alloc(s.occ, (size_t)n_maps * m->cap_cells));
            PQP_CUDA(err, r.alloc(s.boxes, (size_t)PQP_MAX_BOXES * PQP_BOX_FIELDS));
            PQP_CUDA(err, r.alloc(s.box_k, (size_t)n_maps));
            // direct copies over NVLink / PCIe between this device and the home one where the pair allows it
            int there = 0, back = 0;
            if (m->dev[d] != home && cudaDeviceCanAccessPeer(&there, m->dev[d], home) == cudaSuccess && there &&
                cudaDeviceCanAccessPeer(&back, home, m->dev[d]) == cudaSuccess && back) {
                PQP_CUDA(err, enable_peer(m->dev[d], home));
                PQP_CUDA(err, enable_peer(home, m->dev[d]));
            }
        }
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        const std::string msg = err;
        pqp_plan_multi_destroy(m);
        err = msg;
        return rc;
    }
    *out = m;
    return PQP_OK;
}

int pqp_plan_multi_destroy(pqp_plan_multi_t *m) {
    if (!m) return PQP_OK;
    for (int d = 0; d < m->n_dev; ++d) {
        pqp::DeviceGuard g(m->dev[d]);
        if (m->stream[d]) cudaStreamSynchronize(m->stream[d]);
        if (m->h[d]) pqp_plan_destroy(m->h[d]);
    }
    delete m;
    return PQP_OK;
}

int pqp_plan_multi_points(pqp_plan_multi_t *m, const pqp_plan_points_in *in, const int32_t *map_index,
                          const pqp_plan_out *out) {
    return plan_host(m, Call{nullptr, in}, map_index, out);
}

int pqp_plan_multi(pqp_plan_multi_t *m, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out) {
    return plan_host(m, Call{in, nullptr}, map_index, out);
}

int pqp_plan_multi_points_device(pqp_plan_multi_t *m, const pqp_plan_points_in *in, const int32_t *map_index,
                                 const pqp_plan_out *out, void *stream) {
    return plan_device(m, Call{nullptr, in}, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan_multi_device(pqp_plan_multi_t *m, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out,
                          void *stream) {
    return plan_device(m, Call{in, nullptr}, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan_multi_set_map_slot(pqp_plan_multi_t *m, int32_t slot, const pqp_bounds_map *map) {
    if (!m) return PQP_E_INVALID;
    return update_all(m, [&](pqp_plan_handle *h) { return pqp_plan_set_map_slot(h, slot, map); });
}

int pqp_plan_multi_set_occupancy_slots(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *stack) {
    if (!m) return PQP_E_INVALID;
    return update_all(m, [&](pqp_plan_handle *h) { return pqp_plan_set_occupancy_slots(h, first_slot, stack); });
}

int pqp_plan_multi_set_occupancy_slots_device(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *stack,
                                              void *stream) {
    return occupancy_device(m, {first_slot, stack, false, 0, nullptr}, static_cast<cudaStream_t>(stream));
}

int pqp_plan_multi_set_occupancy_boxes(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *base,
                                       int32_t shared_base, const pqp_obstacle_boxes *boxes) {
    if (!m) return PQP_E_INVALID;
    return update_all(m, [&](pqp_plan_handle *h) {
        return pqp_plan_set_occupancy_boxes(h, first_slot, base, shared_base, boxes);
    });
}

int pqp_plan_multi_set_occupancy_boxes_device(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *base,
                                              int32_t shared_base, const pqp_obstacle_boxes *boxes, void *stream) {
    return occupancy_device(m, {first_slot, base, true, shared_base, boxes}, static_cast<cudaStream_t>(stream));
}

int pqp_plan_multi_get_map_slot(pqp_plan_multi_t *m, int32_t device_index, int32_t slot, pqp_bounds_map *meta,
                                float *distance) {
    if (!m || device_index < 0 || device_index >= m->n_dev) return PQP_E_INVALID;
    const int rc = pqp_plan_get_map_slot(m->h[device_index], slot, meta, distance);
    return rc == PQP_OK ? PQP_OK : device_fail(m, device_index, rc);
}

int pqp_plan_multi_shard(pqp_plan_multi_t *m, int32_t device_index, int32_t *first, int32_t *count) {
    if (!m || device_index < 0 || device_index >= m->n_dev) return PQP_E_INVALID;
    const pqp::Shard sh = pqp::shard_of(m->last_batch, m->last_per, device_index);
    if (first) *first = sh.first;
    if (count) *count = sh.count;
    return PQP_OK;
}

int pqp_plan_multi_handle(pqp_plan_multi_t *m, int32_t device_index, pqp_plan_handle **h) {
    if (!m || !h || device_index < 0 || device_index >= m->n_dev) return PQP_E_INVALID;
    *h = m->h[device_index];
    return PQP_OK;
}

}  // extern "C"
