// pqp_dp.cu — include/pqp_dp.h: the lattice DP search on the GPU, one CTA of 256 threads per path.
// The per-path routine is pqp_dp_core.cuh (shared with the CPU test driver); this file supplies the CUDA
// execution context (4 lanes per node share a layer's 34 predecessors and min-reduce with shuffles under the
// reference's first-minimum rule), the handle and the C ABI. Built with --fmad=false: the decision chain
// (feasibility thresholds, strict cost comparisons) follows separately rounded FP64 operations like the host code.
#include <cuda_runtime.h>

#include <new>
#include <optional>
#include <string>

#include "../../include/pqp_dp.h"
#include "pqp_bounds_internal.h"
#include "pqp_dp_core.cuh"
#include "pqp_host_handle.h"

namespace {

thread_local std::string g_dp_create_error;
constexpr int kThreads = 256;

struct CudaCtx {
    static constexpr int kPredLanes = 4;
    __device__ int tid() const { return threadIdx.x; }
    __device__ int nthreads() const { return blockDim.x; }
    __device__ void sync() const { __syncthreads(); }
    // lanes 4 j .. 4 j + 3 hold partial minima over predecessors p = g, g + 4, ...: smaller total wins, equal
    // totals go to the smaller predecessor index (what a sequential strict-< scan in index order keeps)
    __device__ void reduce_pred(double &best, int &bp, double &bdir) const {
#pragma unroll
        for (int m = 1; m < kPredLanes; m <<= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, m);
            const int op = __shfl_xor_sync(0xffffffffu, bp, m);
            const double od = __shfl_xor_sync(0xffffffffu, bdir, m);
            if (op >= 0 && (bp < 0 || ob < best || (ob == best && op < bp))) {
                best = ob;
                bp = op;
                bdir = od;
            }
        }
    }
    __device__ bool any(bool v) const { return __syncthreads_or(v ? 1 : 0) != 0; }
};

struct DpArgs {
    int batch, k_max, layers_max, J;
    const double *spline, *length, *start;
    const int32_t *k;
    int32_t *status, *n_layers, *n_out, *chosen;
    double *layer_s, *lower, *upper, *vehicle_l, *target_s, *cost;
    int8_t *parent;
    uint8_t *feasible;
    double *nx, *ny, *dis, *ref;
    const pqb::MapView *table;  // per-path maps: path b reads table[map_index[b]]; map_index NULL: the shared map
    const int32_t *map_index;
    int n_maps;
};

// Three CTAs per SM, as before the per-path map: left free, ptxas gives the kernel 104 registers (two CTAs per SM)
// once the view may come from the slot table; capped at 80 it keeps its occupancy with a 4-byte spill.
__global__ void __launch_bounds__(kThreads, 3) dp_search_kernel(const pqb::MapView shared_map, const pqdp::Params prm,
                                                             const DpArgs a) {
    __shared__ double shd[6 * pqdp::kJMax + 8];
    __shared__ int shi[8];
    const int b = blockIdx.x;
    if (b >= a.batch) return;
    pqb::MapView map = shared_map;
    if (a.map_index) {
        const pqb::MapView *slot = pqb::slot_view(a.table, a.n_maps, a.map_index, b);
        if (slot) {
            map = *slot;
        } else {  // no map to search: nothing sampled, nothing kept
            if (threadIdx.x == 0) {
                a.status[b] = PQP_DP_MAP_INDEX;
                a.n_layers[b] = 0;
                a.n_out[b] = 0;
            }
            return;
        }
    }
    pqdp::PathIO io;
    const double *row = a.spline + (size_t)b * PQP_SPLINE_ROWS * a.k_max;
    io.sp.sx = row;
    io.sp.xa = row + a.k_max;
    io.sp.xb = row + 2 * (size_t)a.k_max;
    io.sp.xc = row + 3 * (size_t)a.k_max;
    io.sp.xy = row + 4 * (size_t)a.k_max;
    io.sp.ya = row + 5 * (size_t)a.k_max;
    io.sp.yb = row + 6 * (size_t)a.k_max;
    io.sp.yc = row + 7 * (size_t)a.k_max;
    io.sp.yy = row + 8 * (size_t)a.k_max;
    io.sp.k = a.k[b];
    io.length = a.length[b];
    io.sx = a.start[3 * b];
    io.sy = a.start[3 * b + 1];
    io.sh = a.start[3 * b + 2];
    io.layers_max = a.layers_max;
    const size_t lo = (size_t)b * a.layers_max, t = lo * a.J;
    io.ok = a.status + b;
    io.n_layers = a.n_layers + b;
    io.n_out = a.n_out + b;
    io.chosen = a.chosen + lo;
    io.layer_s = a.layer_s + lo;
    io.lower = a.lower + lo;
    io.upper = a.upper + lo;
    io.vehicle_l = a.vehicle_l + b;
    io.target_s = a.target_s + b;
    io.cost = a.cost + t;
    io.parent = a.parent + t;
    io.feasible = a.feasible + t;
    io.nx = a.nx + t;
    io.ny = a.ny + t;
    io.dis = a.dis + t;
    io.ref = a.ref + lo * 4;
    pqdp::dp_search_path(CudaCtx(), map, prm, io, shd, shi);
}

}  // namespace

struct pqp_dp_handle {
    pqp_bounds_handle *owner = nullptr;
    int device = 0, layers_max = 0, batch_max = 0, J = 0;
    pqdp::Params prm{};
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // scratch + default tables (per path: layers_max x J)
    double *d_nx = nullptr, *d_ny = nullptr, *d_dis = nullptr, *d_ref = nullptr, *d_cost = nullptr;
    int8_t *d_parent = nullptr;
    uint8_t *d_feasible = nullptr;
    // staging of the host-pointer call
    double *d_spline = nullptr, *d_length = nullptr, *d_start = nullptr, *d_layer_s = nullptr, *d_lower = nullptr, *d_upper = nullptr;
    double *d_vehicle_l = nullptr, *d_target_s = nullptr;
    int32_t *d_k = nullptr, *d_status = nullptr, *d_n_layers = nullptr, *d_n_out = nullptr, *d_chosen = nullptr;
    int32_t *d_map_index = nullptr;  // grown on demand
    float last_ms = 0.0f;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace {

using pqp::fail;

int search(pqp_dp_handle *h, const pqp_dp_in *in, bool mapped, const int32_t *map_index, const pqp_dp_out *out,
           std::optional<cudaStream_t> stream);

int validate(pqp_dp_handle *h, const pqp_dp_in *in, const pqp_dp_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out) return fail(h->err, PQP_E_INVALID, "null batch");
    if (!in->spline || !in->k || !in->length || !in->start) return fail(h->err, PQP_E_INVALID, "null input buffer");
    if (!out->status || !out->n_layers || !out->n_out || !out->layer_s || !out->lower || !out->upper || !out->chosen ||
        !out->vehicle_l || !out->target_s)
        return fail(h->err, PQP_E_INVALID, "null output buffer");
    if (in->batch < 1 || in->batch > h->batch_max) return fail(h->err, PQP_E_INVALID, "batch out of range");
    if (in->k_max < 3) return fail(h->err, PQP_E_INVALID, "k_max must be >= 3");
    return PQP_OK;
}

int launch(pqp_dp_handle *h, const pqp_dp_in *in, const int32_t *map_index, const pqp_dp_out *out, cudaStream_t s) {
    DpArgs a;
    a.table = pqb::handle_table(h->owner);
    a.map_index = map_index;
    a.n_maps = pqb::handle_map_count(h->owner);
    a.batch = in->batch;
    a.k_max = in->k_max;
    a.layers_max = h->layers_max;
    a.J = h->J;
    a.spline = in->spline;
    a.length = in->length;
    a.start = in->start;
    a.k = in->k;
    a.status = out->status;
    a.n_layers = out->n_layers;
    a.n_out = out->n_out;
    a.chosen = out->chosen;
    a.layer_s = out->layer_s;
    a.lower = out->lower;
    a.upper = out->upper;
    a.vehicle_l = out->vehicle_l;
    a.target_s = out->target_s;
    a.cost = out->cost ? out->cost : h->d_cost;
    a.parent = out->parent ? out->parent : h->d_parent;
    a.feasible = out->feasible ? out->feasible : h->d_feasible;
    a.nx = h->d_nx;
    a.ny = h->d_ny;
    a.dis = h->d_dis;
    a.ref = h->d_ref;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    dp_search_kernel<<<in->batch, kThreads, 0, s>>>(*pqb::handle_map(h->owner), h->prm, a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    return PQP_OK;
}

}  // namespace

extern "C" {

void pqp_dp_default_params(pqp_dp_params *p) {
    if (!p) return;
    p->lateral_range = 10.0;
    p->lateral_spacing = 0.6;
    p->longitudinal_spacing = 1.5;
    p->car_width = 2.0;
}

const char *pqp_dp_last_error(const pqp_dp_handle *h) { return h ? h->err.c_str() : g_dp_create_error.c_str(); }

int pqp_dp_create(pqp_bounds_handle *owner, const pqp_dp_params *params, int32_t layers_max, int32_t batch_max,
                  pqp_dp_handle **out) {
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (!owner) return fail(g_dp_create_error, PQP_E_INVALID, "pqp_dp_create: a pqp_bounds_handle (the map) is required");
    if (layers_max < 2 || batch_max < 1) return fail(g_dp_create_error, PQP_E_INVALID, "pqp_dp_create: layers_max >= 2, batch_max >= 1");
    pqp_dp_params dflt;
    pqp_dp_default_params(&dflt);
    const pqp_dp_params &p = params ? *params : dflt;
    if (!(p.lateral_spacing > 0) || !(p.lateral_range > 0) || !(p.longitudinal_spacing > 0))
        return fail(g_dp_create_error, PQP_E_INVALID, "pqp_dp_create: spacings and range must be positive");
    {
        double cl = -p.lateral_range;
        int n = 0;
        while (cl <= p.lateral_range) { ++n; cl += p.lateral_spacing; }
        if (n > pqdp::kJMax) return fail(g_dp_create_error, PQP_E_INVALID, "pqp_dp_create: more than 64 lateral samples per layer");
    }
    pqp_dp_handle *h = new (std::nothrow) pqp_dp_handle;
    if (!h) return fail(g_dp_create_error, PQP_E_INVALID, "out of host memory");
    h->owner = owner;
    h->device = h->res.device = pqb::handle_device(owner);
    h->layers_max = layers_max;
    h->batch_max = batch_max;
    h->prm.lateral_range = p.lateral_range;
    h->prm.lateral_spacing = p.lateral_spacing;
    h->prm.lon_spacing = p.longitudinal_spacing;
    h->prm.car_width = p.car_width;
    h->J = pqdp::lateral_count(h->prm);
    pqp::DeviceGuard guard_(h->device);
    const int rc = [&]() -> int {
        std::string &err = g_dp_create_error;
        pqp::Resources &r = h->res;
        const size_t B = batch_max, T = B * layers_max * h->J, Ls = B * layers_max;
        PQP_CUDA(err, r.stream(h->stream));
        PQP_CUDA(err, r.event(h->ev0));
        PQP_CUDA(err, r.event(h->ev1));
        PQP_CUDA(err, r.alloc(h->d_nx, T));
        PQP_CUDA(err, r.alloc(h->d_ny, T));
        PQP_CUDA(err, r.alloc(h->d_dis, T));
        PQP_CUDA(err, r.alloc(h->d_cost, T));
        PQP_CUDA(err, r.alloc(h->d_parent, T));
        PQP_CUDA(err, r.alloc(h->d_feasible, T));
        PQP_CUDA(err, r.alloc(h->d_ref, Ls * 4));
        PQP_CUDA(err, r.alloc(h->d_length, B));
        PQP_CUDA(err, r.alloc(h->d_start, B * 3));
        PQP_CUDA(err, r.alloc(h->d_k, B));
        PQP_CUDA(err, r.alloc(h->d_status, B));
        PQP_CUDA(err, r.alloc(h->d_n_layers, B));
        PQP_CUDA(err, r.alloc(h->d_n_out, B));
        PQP_CUDA(err, r.alloc(h->d_vehicle_l, B));
        PQP_CUDA(err, r.alloc(h->d_target_s, B));
        PQP_CUDA(err, r.alloc(h->d_layer_s, Ls));
        PQP_CUDA(err, r.alloc(h->d_lower, Ls));
        PQP_CUDA(err, r.alloc(h->d_upper, Ls));
        PQP_CUDA(err, r.alloc(h->d_chosen, Ls));
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_dp_destroy(h);
        return rc;
    }
    *out = h;
    return PQP_OK;
}

void pqp_dp_destroy(pqp_dp_handle *h) {
    if (!h) return;
    pqp::DeviceGuard guard_(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    delete h;
}

int32_t pqp_dp_lateral_count(const pqp_dp_handle *h) { return h ? h->J : 0; }

int pqp_dp_search_device(pqp_dp_handle *h, const pqp_dp_in *in, const pqp_dp_out *out, void *stream) {
    return search(h, in, false, nullptr, out, static_cast<cudaStream_t>(stream));
}

int pqp_dp_search_mapped_device(pqp_dp_handle *h, const pqp_dp_in *in, const int32_t *map_index, const pqp_dp_out *out,
                                void *stream) {
    return search(h, in, true, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_dp_search(pqp_dp_handle *h, const pqp_dp_in *in, const pqp_dp_out *out) {
    return search(h, in, false, nullptr, out, std::nullopt);
}

int pqp_dp_search_mapped(pqp_dp_handle *h, const pqp_dp_in *in, const int32_t *map_index, const pqp_dp_out *out) {
    return search(h, in, true, map_index, out, std::nullopt);
}

int pqp_dp_last_kernel_ms(pqp_dp_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    *ms = h->last_ms;
    return PQP_OK;
}

}  // extern "C"

namespace {

// every pqp_dp_search* entry point: `mapped` for the mapped forms (path b on slot map_index[b]), `stream` empty for
// the host forms, which stage the inputs into the handle's buffers, search on the handle's stream, copy the outputs
// back and wait
int search(pqp_dp_handle *h, const pqp_dp_in *in, bool mapped, const int32_t *map_index, const pqp_dp_out *out,
           std::optional<cudaStream_t> stream) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    if (mapped && !map_index) return fail(h->err, PQP_E_INVALID, "null map_index");
    pqp::DeviceGuard guard_(h->device);
    if (stream) return launch(h, in, map_index, out, *stream);
    const size_t B = in->batch, nsp = B * PQP_SPLINE_ROWS * in->k_max, Ls = B * h->layers_max, T = Ls * h->J;
    PQP_CUDA(h->err, h->res.grow(h->d_spline, nsp));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_spline, in->spline, nsp * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_k, in->k, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_length, in->length, B * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_start, in->start, B * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_chosen, 0, Ls * sizeof(int32_t), s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_layer_s, 0, Ls * sizeof(double), s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_lower, 0, Ls * sizeof(double), s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_upper, 0, Ls * sizeof(double), s));
    pqp_dp_in din = {in->batch, in->k_max, h->d_spline, h->d_k, h->d_length, h->d_start};
    pqp_dp_out dout = {h->d_status, h->d_n_layers, h->d_n_out, h->d_layer_s, h->d_lower, h->d_upper, h->d_chosen,
                       h->d_vehicle_l, h->d_target_s, nullptr, nullptr, nullptr};
    if (mapped) {
        PQP_CUDA(h->err, h->res.grow(h->d_map_index, B));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->d_map_index, map_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    }
    rc = launch(h, &din, mapped ? h->d_map_index : nullptr, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n_layers, h->d_n_layers, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n_out, h->d_n_out, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->vehicle_l, h->d_vehicle_l, B * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->target_s, h->d_target_s, B * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->layer_s, h->d_layer_s, Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->lower, h->d_lower, Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->upper, h->d_upper, Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->chosen, h->d_chosen, Ls * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->cost) PQP_CUDA(h->err, cudaMemcpyAsync(out->cost, h->d_cost, T * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (out->parent) PQP_CUDA(h->err, cudaMemcpyAsync(out->parent, h->d_parent, T * sizeof(int8_t), cudaMemcpyDeviceToHost, s));
    if (out->feasible) PQP_CUDA(h->err, cudaMemcpyAsync(out->feasible, h->d_feasible, T * sizeof(uint8_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    PQP_CUDA(h->err, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return PQP_OK;
}

}  // namespace
