// pqp_bounds.cu — clearance-bounds kernel and its C ABI (include/pqp_bounds.h).
//
// One thread per (path, reference state, anchor); a warp = one anchor type of 32 consecutive
// states, so its ray-marches walk neighbouring map cells in lock step. The
// float distance layer (2 MB for the demo map) is read through the read-only path and stays in
// the 126 MB L2; per state the kernel reads 32 B of state + its share of the spline and writes
// 48 B of bounds - it is gather-latency bound, not HBM bound (DESIGN.md §5).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>

#include "../../include/pqp_bounds.h"
#include "pqp_bounds_core.cuh"
#include "pqp_bounds_internal.h"
#include "pqp_host_handle.h"
#include "pqp_map_core.cuh"

namespace {

struct BoundsArgs {
    pqb::MapView map;
    pqb::Params prm;
    int batch, n_max, k_max;
    const double *states;
    const int32_t *n;
    const double *spline;
    const int32_t *k;
    double *bounds;
    int32_t *n_valid;
    double *knots;
};

__global__ void init_n_valid_kernel(const int32_t *__restrict__ n, int32_t *__restrict__ n_valid, int batch, int n_max) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) {
        int v = n[b];
        n_valid[b] = v < 0 ? 0 : (v > n_max ? n_max : v);
    }
}

// grid.x covers (path, state) pairs, grid.y the anchor: a warp handles one anchor type of 32
// consecutive states (0.15-0.3 m apart), so its lanes run the same Newton / march phases over
// neighbouring map cells.
__global__ void __launch_bounds__(128) clearance_bounds_kernel(const BoundsArgs a) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)a.batch * a.n_max;
    if (t >= total) return;
    const int anchor = (int)blockIdx.y;
    const int i = (int)(t % a.n_max);
    const int b = (int)(t / a.n_max);
    int nb = a.n[b];
    nb = nb > a.n_max ? a.n_max : nb;
    if (i >= nb) return;
    const double *st = a.states + (size_t)b * PQP_STATE_ROWS * a.n_max;
    const double s = st[i], x = st[a.n_max + i], y = st[2 * a.n_max + i], heading = st[3 * a.n_max + i];
    const double *sb = a.spline + (size_t)b * PQP_SPLINE_ROWS * a.k_max;
    pqb::SplineView sp;
    sp.sx = sb;
    sp.xa = sb + 1 * (size_t)a.k_max; sp.xb = sb + 2 * (size_t)a.k_max; sp.xc = sb + 3 * (size_t)a.k_max; sp.xy = sb + 4 * (size_t)a.k_max;
    sp.ya = sb + 5 * (size_t)a.k_max; sp.yb = sb + 6 * (size_t)a.k_max; sp.yc = sb + 7 * (size_t)a.k_max; sp.yy = sb + 8 * (size_t)a.k_max;
    sp.k = a.k[b] > a.k_max ? a.k_max : a.k[b];
    double lb, ub;
    pqb::anchor_bounds(a.map, a.prm, sp, s, x, y, heading, anchor, lb, ub);
    double *ob = a.bounds + (size_t)b * PQP_BOUND_ROWS * a.n_max;
    ob[(size_t)(2 * anchor) * a.n_max + i] = lb;
    ob[(size_t)(2 * anchor + 1) * a.n_max + i] = ub;
    if (anchor < 2) {
        if (a.knots) {
            double *kb = a.knots + (size_t)b * PQP_NFIELDS * a.n_max;
            const int f = anchor == 0 ? PQP_F_B0_LB : PQP_F_B1_LB;
            kb[(size_t)f * a.n_max + i] = lb;
            kb[(size_t)(f + 1) * a.n_max + i] = ub;
        }
        // isEqual(bound[0], bound[1]) -> "Path is blocked" (reference_path_impl.cpp:216-220)
        if (fabs(ub - lb) < a.prm.epsilon) atomicMin(a.n_valid + b, i);
    }
}

struct StatesArgs {
    int batch, n_max, k_max;
    const double *spline;
    const int32_t *k;
    const double *max_s;
    double ds_small, ds_large;
    int dynamic;
    double *states, *curvature, *knots;
    int32_t *n, *total;
};

// one thread per path: the walk is sequential in s (each step depends on the curvature at the last)
__global__ void __launch_bounds__(64) reference_states_kernel(const StatesArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch) return;
    const double *sb = a.spline + (size_t)b * PQP_SPLINE_ROWS * a.k_max;
    pqb::SplineView sp;
    sp.sx = sb;
    sp.xa = sb + 1 * (size_t)a.k_max; sp.xb = sb + 2 * (size_t)a.k_max; sp.xc = sb + 3 * (size_t)a.k_max; sp.xy = sb + 4 * (size_t)a.k_max;
    sp.ya = sb + 5 * (size_t)a.k_max; sp.yb = sb + 6 * (size_t)a.k_max; sp.yc = sb + 7 * (size_t)a.k_max; sp.yy = sb + 8 * (size_t)a.k_max;
    sp.k = a.k[b] > a.k_max ? a.k_max : a.k[b];
    double *st = a.states + (size_t)b * PQP_STATE_ROWS * a.n_max;
    double *cv = a.curvature + (size_t)b * a.n_max;
    const int total = pqb::build_states(sp, a.max_s[b], a.ds_small, a.ds_large, a.dynamic != 0, a.n_max, a.total != nullptr, st, cv);
    const int nb = total < a.n_max ? total : a.n_max;
    a.n[b] = nb;
    if (a.total) a.total[b] = total;
    if (a.knots) {
        double *kb = a.knots + (size_t)b * PQP_NFIELDS * a.n_max;
        for (int i = 0; i < nb; ++i) {
            kb[(size_t)PQP_F_S * a.n_max + i] = st[i];
            kb[(size_t)PQP_F_KREF * a.n_max + i] = cv[i];
            kb[(size_t)PQP_F_L * a.n_max + i] = 0.0;
            kb[(size_t)PQP_F_PSI * a.n_max + i] = 0.0;
            kb[(size_t)PQP_F_K * a.n_max + i] = cv[i];
        }
    }
}

}  // namespace

// The exact Euclidean distance transform of pqp_bounds_set_occupancy* (pqp_map_core.cuh), in place in the
// distance layer: the column pass writes int32 g over the layer, the row pass reads its row of g into shared
// memory and writes the row's floats back. Named namespace: the kernels keep stable names in profiles.
namespace pqm {

constexpr int kEdtColumnThreads = 128;
constexpr int kEdtRowThreads = 64;

// one thread per column: consecutive threads read consecutive bytes of a row
__global__ void __launch_bounds__(kEdtColumnThreads) edt_column_kernel(const uint8_t *__restrict__ img, int rows, int cols,
                                                                        int obstacle_max, int32_t *__restrict__ g) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < cols) pqm::column_pass(img, rows, cols, j, obstacle_max, g);
}

// one block per row: the block loads the row's g, thread 0 builds the lower envelope, the block fills d2 per
// envelope parabola and converts it to the layer's floats
__global__ void __launch_bounds__(kEdtRowThreads) edt_row_kernel(void *layer, int rows, int cols, float res) {
    extern __shared__ int4 edt_smem[];
    int32_t *g = reinterpret_cast<int32_t *>(edt_smem);
    int32_t *h = g + cols;
    int16_t *s = reinterpret_cast<int16_t *>(h + cols);
    int16_t *t = s + cols;
    __shared__ int n_env;
    const size_t row = (size_t)blockIdx.x * cols;
    const int32_t *gin = static_cast<const int32_t *>(layer) + row;
    for (int u = threadIdx.x; u < cols; u += blockDim.x) g[u] = gin[u];
    __syncthreads();
    if (threadIdx.x == 0) n_env = pqm::envelope(g, cols, s, t, h);
    __syncthreads();
    const int n = n_env;
    for (int k = threadIdx.x; k < n; k += blockDim.x) pqm::fill(s, t, h, n, cols, k, g);
    __syncthreads();
    const int32_t inf = pqm::inf_g(rows, cols);
    float *out = static_cast<float *>(layer) + row;
    for (int u = threadIdx.x; u < cols; u += blockDim.x) out[u] = pqm::layer_value(g[u], inf * inf, res);
}

}  // namespace pqm

struct pqp_bounds_handle {
    int device = 0;
    pqb::MapView map{};
    pqb::Params prm{};
    float *d_dist = nullptr;
    size_t cap_cells = 0;        // cells of the map the handle was created with: the most any later map may have
    uint8_t *d_occ = nullptr;    // [cap_cells] staging of pqp_bounds_set_occupancy's host image
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // staging for the host-pointer call (grown on demand)
    double *d_states = nullptr, *d_spline = nullptr, *d_bounds = nullptr, *d_knots = nullptr;
    int32_t *d_n = nullptr, *d_k = nullptr, *d_nvalid = nullptr;
    double *d_maxs = nullptr, *d_curv = nullptr;
    int32_t *d_total = nullptr;
    bool timed = false;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace pqb {
const MapView *handle_map(const pqp_bounds_handle *h) { return h ? &h->map : nullptr; }
int handle_device(const pqp_bounds_handle *h) { return h ? h->device : -1; }
}  // namespace pqb

namespace {

thread_local std::string g_bounds_create_error;

using pqp::fail;

int validate(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || in->batch <= 0 || in->n_max <= 0 || in->k_max < 3 || !in->states || !in->n || !in->spline ||
        !in->k || !out->bounds || !out->n_valid)
        return fail(h->err, PQP_E_INVALID, "pqp_bounds: null pointer or non-positive size (batch, n_max > 0, k_max >= 3)");
    return PQP_OK;
}

int launch(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out, cudaStream_t s) {
    BoundsArgs a;
    a.map = h->map;
    a.prm = h->prm;
    a.batch = in->batch;
    a.n_max = in->n_max;
    a.k_max = in->k_max;
    a.states = in->states;
    a.n = in->n;
    a.spline = in->spline;
    a.k = in->k;
    a.bounds = out->bounds;
    a.n_valid = out->n_valid;
    a.knots = out->knots;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    init_n_valid_kernel<<<(in->batch + 255) / 256, 256, 0, s>>>(in->n, out->n_valid, in->batch, in->n_max);
    const long long total = (long long)in->batch * in->n_max;
    const long long blocks = (total + 127) / 128;
    if (blocks > 0x7fffffffLL) return fail(h->err, PQP_E_INVALID, "pqp_bounds: batch * n_max too large for one launch");
    clearance_bounds_kernel<<<dim3((unsigned)blocks, 3), 128, 0, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->timed = true;
    return PQP_OK;
}

void set_meta(pqp_bounds_handle *h, int rows, int cols, double res, double cx, double cy) {
    h->map.dist = h->d_dist;
    h->map.rows = rows;
    h->map.cols = cols;
    h->map.res = res;
    h->map.inv_res = 1.0 / res;
    h->map.half_lx = 0.5 * rows * res;
    h->map.half_ly = 0.5 * cols * res;
    h->map.cx = cx;
    h->map.cy = cy;
}

// what pqp_bounds_set_map* and pqp_bounds_set_occupancy* accept; a refused map leaves the handle's map untouched
int validate_map(pqp_bounds_handle *h, const void *m, int rows, int cols, double res, double cx, double cy,
                 const void *data, const char *what) {
    if (!h) return PQP_E_INVALID;
    std::string why;
    if (!m || !data) why = "null map or layer";
    else if (rows < 2 || cols < 2) why = "rows, cols >= 2 required";
    else if ((size_t)rows * (size_t)cols > h->cap_cells) why = "rows * cols exceeds the cells the handle was created with";
    else if (!(res > 0.0) || !std::isfinite(res)) why = "resolution must be finite and > 0";
    else if (!std::isfinite(cx) || !std::isfinite(cy)) why = "centre must be finite";
    return why.empty() ? PQP_OK : fail(h->err, PQP_E_INVALID, std::string(what) + ": " + why);
}

int launch_edt(pqp_bounds_handle *h, const pqp_occupancy_map *occ, const uint8_t *cells, cudaStream_t s) {
    const int rows = occ->rows, cols = occ->cols;
    const size_t smem = (size_t)pqm::kRowSmemPerCol * cols;
    // the dynamic share plus the kernel's static n_env may pass the 48 KB default at any width: always opt in
    PQP_CUDA(h->err, cudaFuncSetAttribute(pqm::edt_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pqm::edt_column_kernel<<<(cols + pqm::kEdtColumnThreads - 1) / pqm::kEdtColumnThreads, pqm::kEdtColumnThreads, 0,
                             s>>>(cells, rows, cols, occ->obstacle_max, reinterpret_cast<int32_t *>(h->d_dist));
    PQP_CUDA(h->err, cudaGetLastError());
    pqm::edt_row_kernel<<<rows, pqm::kEdtRowThreads, smem, s>>>(h->d_dist, rows, cols, (float)occ->resolution);
    PQP_CUDA(h->err, cudaGetLastError());
    return PQP_OK;
}

int validate_occupancy(pqp_bounds_handle *h, const pqp_occupancy_map *occ, const char *what) {
    const int rc = occ ? validate_map(h, occ, occ->rows, occ->cols, occ->resolution, occ->center_x, occ->center_y,
                                      occ->cells, what)
                       : validate_map(h, nullptr, 0, 0, 0.0, 0.0, 0.0, nullptr, what);
    if (rc != PQP_OK) return rc;
    if (occ->rows > pqm::kMaxSide || occ->cols > pqm::kMaxSide)
        return fail(h->err, PQP_E_INVALID, std::string(what) + ": rows and cols must be <= 16384 for the distance transform");
    return PQP_OK;
}

}  // namespace

extern "C" {

void pqp_bounds_default_params(pqp_bounds_params *p) {
    if (!p) return;
    p->front_length = 3.9;
    p->rear_length = -1.0;
    p->car_width = 2.0;
    p->safety_margin = 0.3;
    p->epsilon = 1e-6;
}

int pqp_bounds_create(const pqp_bounds_map *map, const pqp_bounds_params *params, int32_t device,
                      pqp_bounds_handle **out) {
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (!map || !map->distance || map->rows < 2 || map->cols < 2 || !(map->resolution > 0.0))
        return fail(g_bounds_create_error, PQP_E_INVALID,
                    "pqp_bounds_create: map needs rows, cols >= 2, resolution > 0 and a distance layer");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return fail(g_bounds_create_error, PQP_E_NO_DEVICE, "pqp_bounds_create: no CUDA device (there is no CPU fallback)");
    pqp_bounds_handle *h = new (std::nothrow) pqp_bounds_handle();
    if (!h) return PQP_E_CUDA;
    h->device = h->res.device = device;
    pqp_bounds_params dflt;
    pqp_bounds_default_params(&dflt);
    const pqp_bounds_params &p = params ? *params : dflt;
    h->prm.front_length = p.front_length;
    h->prm.rear_length = p.rear_length;
    h->prm.car_width = p.car_width;
    h->prm.safety_margin = p.safety_margin;
    h->prm.epsilon = p.epsilon;
    const size_t cells = (size_t)map->rows * map->cols;
    pqp::DeviceGuard guard_(device);
    const int rc = [&]() -> int {
        PQP_CUDA(g_bounds_create_error, h->res.alloc(h->d_dist, cells));
        PQP_CUDA(g_bounds_create_error, cudaMemcpy(h->d_dist, map->distance, cells * sizeof(float), cudaMemcpyHostToDevice));
        PQP_CUDA(g_bounds_create_error, h->res.alloc(h->d_occ, cells));
        PQP_CUDA(g_bounds_create_error, h->res.stream(h->stream));
        PQP_CUDA(g_bounds_create_error, h->res.event(h->ev0));
        PQP_CUDA(g_bounds_create_error, h->res.event(h->ev1));
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_bounds_destroy(h);
        return rc;
    }
    h->cap_cells = cells;
    set_meta(h, map->rows, map->cols, map->resolution, map->center_x, map->center_y);
    *out = h;
    return PQP_OK;
}

void pqp_bounds_destroy(pqp_bounds_handle *h) {
    delete h;
}

int pqp_bounds_compute_device(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out, void *stream) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    return launch(h, in, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_compute(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const size_t B = in->batch, ns = B * PQP_STATE_ROWS * in->n_max, nsp = B * PQP_SPLINE_ROWS * in->k_max;
    const size_t nb = B * PQP_BOUND_ROWS * in->n_max, nk = out->knots ? B * PQP_NFIELDS * in->n_max : 0;
    PQP_CUDA(h->err, h->res.grow(h->d_states, ns));
    PQP_CUDA(h->err, h->res.grow(h->d_bounds, nb));
    PQP_CUDA(h->err, h->res.grow(h->d_spline, nsp));
    if (nk) PQP_CUDA(h->err, h->res.grow(h->d_knots, nk));
    PQP_CUDA(h->err, h->res.grow(h->d_n, B));
    PQP_CUDA(h->err, h->res.grow(h->d_k, B));
    PQP_CUDA(h->err, h->res.grow(h->d_nvalid, B));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_states, in->states, ns * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_spline, in->spline, nsp * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_n, in->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_k, in->k, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_knots, out->knots, nk * sizeof(double), cudaMemcpyHostToDevice, s));
    pqp_bounds_in din = *in;
    din.states = h->d_states;
    din.spline = h->d_spline;
    din.n = h->d_n;
    din.k = h->d_k;
    pqp_bounds_out dout;
    dout.bounds = h->d_bounds;
    dout.n_valid = h->d_nvalid;
    dout.knots = nk ? h->d_knots : nullptr;
    rc = launch(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->bounds, h->d_bounds, nb * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n_valid, h->d_nvalid, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(out->knots, h->d_knots, nk * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

static int validate_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || in->batch <= 0 || in->n_max <= 0 || in->k_max < 3 || !in->spline || !in->k || !in->max_s ||
        !out->states || !out->curvature || !out->n || !(in->delta_s_larger > 0.0) || !(in->delta_s_smaller > 0.0) ||
        in->delta_s_smaller > in->delta_s_larger)
        return fail(h->err, PQP_E_INVALID,
                    "pqp_bounds_build_states: null pointer, non-positive size, or 0 < delta_s_smaller <= delta_s_larger violated");
    return PQP_OK;
}

static int launch_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out, cudaStream_t s) {
    StatesArgs a;
    a.batch = in->batch;
    a.n_max = in->n_max;
    a.k_max = in->k_max;
    a.spline = in->spline;
    a.k = in->k;
    a.max_s = in->max_s;
    a.ds_small = in->delta_s_smaller;
    a.ds_large = in->delta_s_larger;
    a.dynamic = in->dynamic_segmentation;
    a.states = out->states;
    a.curvature = out->curvature;
    a.knots = out->knots;
    a.n = out->n;
    a.total = out->total;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    reference_states_kernel<<<(in->batch + 63) / 64, 64, 0, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->timed = true;
    return PQP_OK;
}

int pqp_bounds_build_states_device(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out, void *stream) {
    int rc = validate_states(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    return launch_states(h, in, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_build_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out) {
    int rc = validate_states(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const size_t B = in->batch, ns = B * PQP_STATE_ROWS * in->n_max, nsp = B * PQP_SPLINE_ROWS * in->k_max;
    const size_t nc = B * in->n_max, nk = out->knots ? B * PQP_NFIELDS * in->n_max : 0;
    PQP_CUDA(h->err, h->res.grow(h->d_states, ns));
    PQP_CUDA(h->err, h->res.grow(h->d_curv, nc));
    PQP_CUDA(h->err, h->res.grow(h->d_spline, nsp));
    if (nk) PQP_CUDA(h->err, h->res.grow(h->d_knots, nk));
    PQP_CUDA(h->err, h->res.grow(h->d_n, B));
    PQP_CUDA(h->err, h->res.grow(h->d_k, B));
    PQP_CUDA(h->err, h->res.grow(h->d_total, B));
    PQP_CUDA(h->err, h->res.grow(h->d_maxs, B));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_spline, in->spline, nsp * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_k, in->k, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_maxs, in->max_s, B * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_states, 0, ns * sizeof(double), s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_curv, 0, nc * sizeof(double), s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_knots, out->knots, nk * sizeof(double), cudaMemcpyHostToDevice, s));
    pqp_states_in din = *in;
    din.spline = h->d_spline;
    din.k = h->d_k;
    din.max_s = h->d_maxs;
    pqp_states_out dout;
    dout.states = h->d_states;
    dout.curvature = h->d_curv;
    dout.n = h->d_n;
    dout.total = h->d_total;
    dout.knots = nk ? h->d_knots : nullptr;
    rc = launch_states(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->states, h->d_states, ns * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->curvature, h->d_curv, nc * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n, h->d_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->total) PQP_CUDA(h->err, cudaMemcpyAsync(out->total, h->d_total, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(out->knots, h->d_knots, nk * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

int pqp_bounds_last_kernel_ms(pqp_bounds_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    if (!h->timed) {
        *ms = 0.0f;
        return PQP_OK;
    }
    PQP_CUDA(h->err, cudaEventSynchronize(h->ev1));
    PQP_CUDA(h->err, cudaEventElapsedTime(ms, h->ev0, h->ev1));
    return PQP_OK;
}

const char *pqp_bounds_last_error(pqp_bounds_handle *h) { return h ? h->err.c_str() : g_bounds_create_error.c_str(); }

int pqp_bounds_set_map_device(pqp_bounds_handle *h, const pqp_bounds_map *map, void *stream) {
    const int rc = map ? validate_map(h, map, map->rows, map->cols, map->resolution, map->center_x, map->center_y,
                                      map->distance, "pqp_bounds_set_map")
                       : validate_map(h, nullptr, 0, 0, 0.0, 0.0, 0.0, nullptr, "pqp_bounds_set_map");
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const size_t cells = (size_t)map->rows * map->cols;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_dist, map->distance, cells * sizeof(float), cudaMemcpyDefault,
                                static_cast<cudaStream_t>(stream)));
    set_meta(h, map->rows, map->cols, map->resolution, map->center_x, map->center_y);
    return PQP_OK;
}

int pqp_bounds_set_map(pqp_bounds_handle *h, const pqp_bounds_map *map) {
    const int rc = pqp_bounds_set_map_device(h, map, h ? h->stream : nullptr);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    PQP_CUDA(h->err, cudaStreamSynchronize(h->stream));
    return PQP_OK;
}

int pqp_bounds_set_occupancy_device(pqp_bounds_handle *h, const pqp_occupancy_map *occ, void *stream) {
    const int rc = validate_occupancy(h, occ, "pqp_bounds_set_occupancy_device");
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const int lrc = launch_edt(h, occ, occ->cells, static_cast<cudaStream_t>(stream));
    if (lrc != PQP_OK) return lrc;
    set_meta(h, occ->rows, occ->cols, occ->resolution, occ->center_x, occ->center_y);
    return PQP_OK;
}

int pqp_bounds_set_occupancy(pqp_bounds_handle *h, const pqp_occupancy_map *occ) {
    const int rc = validate_occupancy(h, occ, "pqp_bounds_set_occupancy");
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const size_t cells = (size_t)occ->rows * occ->cols;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_occ, occ->cells, cells, cudaMemcpyHostToDevice, h->stream));
    const int lrc = launch_edt(h, occ, h->d_occ, h->stream);
    if (lrc != PQP_OK) return lrc;
    set_meta(h, occ->rows, occ->cols, occ->resolution, occ->center_x, occ->center_y);
    PQP_CUDA(h->err, cudaStreamSynchronize(h->stream));
    return PQP_OK;
}

int pqp_bounds_get_map(pqp_bounds_handle *h, pqp_bounds_map *meta, float *distance) {
    if (!h) return PQP_E_INVALID;
    if (!meta) return fail(h->err, PQP_E_INVALID, "pqp_bounds_get_map: null metadata");
    pqp::DeviceGuard guard_(h->device);
    meta->rows = h->map.rows;
    meta->cols = h->map.cols;
    meta->resolution = h->map.res;
    meta->center_x = h->map.cx;
    meta->center_y = h->map.cy;
    meta->distance = nullptr;
    if (distance) {
        PQP_CUDA(h->err, cudaDeviceSynchronize());
        PQP_CUDA(h->err, cudaMemcpy(distance, h->d_dist, (size_t)h->map.rows * h->map.cols * sizeof(float),
                               cudaMemcpyDeviceToHost));
    }
    return PQP_OK;
}

}  // extern "C"
