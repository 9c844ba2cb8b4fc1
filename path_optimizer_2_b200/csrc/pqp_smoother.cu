// pqp_smoother.cu — include/pqp_smoother.h: the three smoother QPs of the reference's front end on the GPU.
// One warp (= one CTA) per QP runs pqp_smoother_core.cuh (OSQP on a stage-banded QP, FP64). The serial part of an
// iteration is the banded forward / backward substitution, so its band factor and right-hand side live in shared
// memory; everything else (problem data, iterates) is per-CTA scratch in global memory that stays in L1/L2. A grid
// of min(batch, resident CTAs) loops over the QPs.
#include <cuda_runtime.h>

#include <new>
#include <string>

#include "../../include/pqp_smoother.h"
#include "pqp_host_handle.h"
#include "pqp_smoother_core.cuh"
#include "pqp_smoother_internal.h"

namespace {

thread_local std::string g_smoother_create_error;

struct WarpLane {
    __device__ int lane() const { return threadIdx.x; }
    __device__ int lanes() const { return 32; }
    __device__ void sync() const { __syncwarp(); }
    __device__ double max(double v) const {
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, m));
        return v;
    }
    __device__ double sum(double v) const {
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
        return v;
    }
    __device__ int all(int v) const { return __all_sync(0xffffffffu, v); }
};

struct KArgs {
    int batch, p_max, mode;  // mode 0 tension, 1 post
    pqs::Settings st;
    pqs::TensionWeights tw;
    pqs::PostWeights pw;
    const int32_t *p;
    const double *a0, *a1, *a2, *a3, *a4;  // tension: x, y, angle, k, s; post: layer_s, lower, upper, vehicle_l
    double *o0, *o1, *o2, *x_full;         // tension: x, y, s; post: offsets
    int32_t *status, *iters;
    unsigned char *scratch;
    size_t scratch_stride;
};

__global__ void __launch_bounds__(32) smoother_kernel(const KArgs a) {
    extern __shared__ __align__(16) double band[];
    pqs::Work W;
    pqs::carve(W, a.scratch + (size_t)blockIdx.x * a.scratch_stride, a.p_max, band);
    const WarpLane c;
    for (int b = blockIdx.x; b < a.batch; b += gridDim.x) {
        const int p = a.p[b];
        const size_t o = (size_t)b * a.p_max;
        pqs::Result R;
        if (a.mode == 0) {
            if (p < 3 || p > a.p_max) {
                if (threadIdx.x == 0) { a.status[b] = pqs::kNumerical; a.iters[b] = 0; }
                continue;
            }
            R = pqs::tension_smooth(c, W, a.st, a.tw, p, a.a0 + o, a.a1 + o, a.a2 + o, a.a3 + o, a.a4 + o, a.o0 + o, a.o1 + o,
                                    a.o2 + o, a.x_full ? a.x_full + (size_t)b * 4 * a.p_max : nullptr);
        } else {
            if (p < 2 || p > a.p_max) {
                if (threadIdx.x == 0) { a.status[b] = pqs::kNumerical; a.iters[b] = 0; }
                continue;
            }
            R = pqs::post_smooth(c, W, a.st, a.pw, p, a.a0 + o, a.a1 + o, a.a2 + o, a.a3[b], a.o0 + o,
                                 a.x_full ? a.x_full + (size_t)b * 3 * a.p_max : nullptr);
        }
        if (threadIdx.x == 0) {
            a.status[b] = R.status;
            a.iters[b] = R.iters;
        }
        __syncwarp();
    }
}

struct CArgs {
    int batch, p_max;
    pqs::Settings st;
    pqs::CartesianWeights cw;
    const int32_t *p;
    const double *x, *y, *angle, *clearance;
    double *ox, *oy, *os, *x_full;
    int32_t *status, *iters;
    unsigned char *scratch;
    size_t scratch_stride;
};

// TensionSmoother::osqpSmooth: the same solver at half-bandwidth 9, so its own kernel (band in shared memory:
// (3 p_max + 9) * 11 doubles). The minimum of one block per SM lets ptxas keep the wider band loops in registers
// (191, no spills, CUDA 12.9) instead of capping at 168 with spills; shared memory bounds the residency anyway.
__global__ void __launch_bounds__(32, 1) cartesian_kernel(const CArgs a) {
    extern __shared__ __align__(16) double band[];
    pqs::Work W;
    pqs::cartesian_carve(W, a.scratch + (size_t)blockIdx.x * a.scratch_stride, a.p_max, band);
    const WarpLane c;
    for (int b = blockIdx.x; b < a.batch; b += gridDim.x) {
        const int p = a.p[b];
        const size_t o = (size_t)b * a.p_max;
        if (p < 3 || p > a.p_max) {
            if (threadIdx.x == 0) { a.status[b] = pqs::kNumerical; a.iters[b] = 0; }
            continue;
        }
        const pqs::Result R = pqs::cartesian_tension_smooth(c, W, a.st, a.cw, p, a.x + o, a.y + o, a.angle + o, a.clearance + o,
                                                            a.ox + o, a.oy + o, a.os + o,
                                                            a.x_full ? a.x_full + (size_t)b * 3 * a.p_max : nullptr);
        if (threadIdx.x == 0) {
            a.status[b] = R.status;
            a.iters[b] = R.iters;
        }
        __syncwarp();
    }
}

}  // namespace

struct pqp_smoother_handle {
    pqp_smoother_params prm{};
    int device = 0, p_max = 0, batch_max = 0, grid_max = 0;
    size_t scratch_stride = 0, smem = 0, scratch_total = 0;
    // Cartesian tension QP: its own working-set size, band and resident-CTA count; cart_err is set when p_max is
    // beyond its shared-memory limit (the other calls are unaffected)
    int cart_grid_max = 0;
    size_t cart_stride = 0, cart_smem = 0;
    std::string cart_err;
    unsigned char *d_scratch = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // staging of the host-pointer calls: 5 input lists, 3 output lists, x_full, p / status / iters, vehicle_l
    double *d_in[5] = {}, *d_out[3] = {}, *d_xfull = nullptr, *d_vl = nullptr;
    int32_t *d_p = nullptr, *d_status = nullptr, *d_iters = nullptr;
    float last_ms = 0.0f;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace {

using pqp::fail;

pqs::Settings settings_of(const pqp_smoother_params &p) {
    pqs::Settings s;
    s.rho = p.rho; s.sigma = p.sigma; s.alpha = p.alpha; s.eps_abs = p.eps_abs; s.eps_rel = p.eps_rel;
    s.eps_prim_inf = p.eps_prim_inf; s.eps_dual_inf = p.eps_dual_inf; s.adaptive_rho_tolerance = p.adaptive_rho_tolerance;
    s.max_iter = p.max_iter; s.check_termination = p.check_termination; s.scaling = p.scaling;
    s.adaptive_rho = p.adaptive_rho; s.adaptive_rho_interval = p.adaptive_rho_interval;
    return s;
}

// resident one-warp CTAs of `kernel` at `smem` bytes of band: 1 to 16 per SM, at most batch_max in all
template <typename Kernel>
cudaError_t resident_grid(Kernel *kernel, size_t smem, int sm_count, int batch_max, int *grid) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int per_sm = 1;
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 32, smem);
    per_sm = per_sm < 1 ? 1 : (per_sm > 16 ? 16 : per_sm);
    *grid = sm_count * per_sm < batch_max ? sm_count * per_sm : batch_max;
    return e;
}

int launch(pqp_smoother_handle *h, KArgs &a, cudaStream_t s) {
    a.p_max = h->p_max;
    a.st = settings_of(h->prm);
    a.tw = {h->prm.tension_deviation_weight, h->prm.tension_curvature_weight, h->prm.tension_curvature_rate_weight};
    a.pw = {h->prm.post_weight_x, h->prm.post_weight_dx, h->prm.post_weight_ddx};
    a.scratch = h->d_scratch;
    a.scratch_stride = h->scratch_stride;
    const int grid = a.batch < h->grid_max ? a.batch : h->grid_max;
    // the dynamic shared-memory limit is an attribute of the kernel, not of the handle: a handle created later with a
    // smaller p_max lowers it, so each launch sets this handle's own
    PQP_CUDA(h->err, cudaFuncSetAttribute(smoother_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem));
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    smoother_kernel<<<grid, 32, h->smem, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    return PQP_OK;
}

int launch_cartesian(pqp_smoother_handle *h, CArgs &a, cudaStream_t s) {
    a.p_max = h->p_max;
    a.st = settings_of(h->prm);
    a.cw = {h->prm.cartesian_curvature_weight, h->prm.cartesian_curvature_rate_weight, h->prm.cartesian_deviation_weight};
    a.scratch = h->d_scratch;
    a.scratch_stride = h->cart_stride;
    const int grid = a.batch < h->cart_grid_max ? a.batch : h->cart_grid_max;
    PQP_CUDA(h->err, cudaFuncSetAttribute(cartesian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->cart_smem));
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    cartesian_kernel<<<grid, 32, h->cart_smem, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    return PQP_OK;
}

// the argument checks of each call, shared by its host-pointer and device-pointer forms
int check_size(pqp_smoother_handle *h, int batch, int p_max) {
    if (batch < 1 || batch > h->batch_max || p_max != h->p_max) return fail(h->err, PQP_E_INVALID, "batch / p_max do not fit the handle");
    return PQP_OK;
}
int check(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->x || !in->y || !in->angle || !in->k || !in->s || !out->x || !out->y || !out->s ||
        !out->status || !out->iters)
        return fail(h->err, PQP_E_INVALID, "null buffer");
    return check_size(h, in->batch, in->p_max);
}
int check(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->layer_s || !in->lower || !in->upper || !in->vehicle_l || !out->offsets || !out->status || !out->iters)
        return fail(h->err, PQP_E_INVALID, "null buffer");
    return check_size(h, in->batch, in->p_max);
}
int check(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in, const pqp_tension_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!h->cart_err.empty()) return fail(h->err, PQP_E_INVALID, h->cart_err);
    if (!in || !out || !in->p || !in->x || !in->y || !in->angle || !in->clearance || !out->x || !out->y || !out->s ||
        !out->status || !out->iters)
        return fail(h->err, PQP_E_INVALID, "null buffer");
    return check_size(h, in->batch, in->p_max);
}

// A host-pointer call: its input lists (and post's vehicle_l) and p are staged into d_in / d_vl / d_p, its outputs
// cleared, the device form `run` is launched on the handle's stream with the staging buffers, and the outputs are
// copied back. `p_min` is the smallest p[b] the call accepts; `full_rows` the rows of one QP's x_full.
struct HostCall {
    int batch;
    const int32_t *p;
    int p_min;
    const double *const *in;
    int n_in;
    const double *vehicle_l;
    double *const *out;
    int n_out;
    int32_t *status, *iters;
    double *x_full;
    int full_rows;
};

template <typename Run>
int run_host(pqp_smoother_handle *h, const HostCall &c, Run run) {
    for (int b = 0; b < c.batch; ++b)
        if (c.p[b] < c.p_min || c.p[b] > h->p_max)
            return fail(h->err, PQP_E_INVALID, c.p_min == 2 ? "p[b] must be in [2, p_max]" : "p[b] must be in [3, p_max]");
    pqp::DeviceGuard guard_(h->device);
    cudaStream_t s = h->stream;
    const size_t B = c.batch, Ls = B * h->p_max, nf = Ls * c.full_rows;
    for (int i = 0; i < c.n_in; ++i) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_in[i], c.in[i], Ls * sizeof(double), cudaMemcpyHostToDevice, s));
    if (c.vehicle_l) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_vl, c.vehicle_l, B * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_p, c.p, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    for (int i = 0; i < c.n_out; ++i) PQP_CUDA(h->err, cudaMemsetAsync(h->d_out[i], 0, Ls * sizeof(double), s));
    if (c.x_full) PQP_CUDA(h->err, cudaMemsetAsync(h->d_xfull, 0, nf * sizeof(double), s));
    const int rc = run(s, c.x_full ? h->d_xfull : nullptr);
    if (rc != PQP_OK) return rc;
    for (int i = 0; i < c.n_out; ++i) PQP_CUDA(h->err, cudaMemcpyAsync(c.out[i], h->d_out[i], Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(c.status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(c.iters, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (c.x_full) PQP_CUDA(h->err, cudaMemcpyAsync(c.x_full, h->d_xfull, nf * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    PQP_CUDA(h->err, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return PQP_OK;
}

}  // namespace

const char *pqs::cartesian_unavailable(const pqp_smoother_handle *h) {
    return (h && !h->cart_err.empty()) ? h->cart_err.c_str() : nullptr;
}

extern "C" {

void pqp_smoother_default_params(pqp_smoother_params *p) {
    if (!p) return;
    p->tension_deviation_weight = 0.005;
    p->tension_curvature_weight = 1.0;
    p->tension_curvature_rate_weight = 10.0;
    p->post_weight_x = 1.0;
    p->post_weight_dx = 100.0;
    p->post_weight_ddx = 1000.0;
    p->rho = 0.1;
    p->sigma = 1e-6;
    p->alpha = 1.6;
    p->eps_abs = 1e-3;
    p->eps_rel = 1e-3;
    p->eps_prim_inf = 1e-4;
    p->eps_dual_inf = 1e-4;
    p->adaptive_rho_tolerance = 5.0;
    p->max_iter = 4000;
    p->check_termination = 25;
    p->scaling = 10;
    p->adaptive_rho = 1;
    p->adaptive_rho_interval = 25;
    p->reserved = 0;
    p->cartesian_curvature_weight = 1.0;
    p->cartesian_curvature_rate_weight = 50.0;
    p->cartesian_deviation_weight = 0.0;
}

const char *pqp_smoother_last_error(const pqp_smoother_handle *h) { return h ? h->err.c_str() : g_smoother_create_error.c_str(); }

int pqp_smoother_create(const pqp_smoother_params *params, int32_t p_max, int32_t batch_max, int32_t device,
                        pqp_smoother_handle **out) {
    std::string &err = g_smoother_create_error;
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (p_max < 4 || p_max > 2000 || batch_max < 1) return fail(err, PQP_E_INVALID, "pqp_smoother_create: 4 <= p_max <= 2000, batch_max >= 1");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return fail(err, PQP_E_NO_DEVICE, "pqp_smoother_create: no CUDA device (there is no CPU fallback)");
    pqp_smoother_params prm;
    if (params) prm = *params;
    else pqp_smoother_default_params(&prm);
    if (!(prm.rho > 0) || !(prm.sigma > 0) || !(prm.alpha > 0 && prm.alpha < 2) || prm.max_iter < 1)
        return fail(err, PQP_E_INVALID, "pqp_smoother_create: invalid OSQP settings");
    cudaDeviceProp prop;
    PQP_CUDA(err, cudaGetDeviceProperties(&prop, device));
    const size_t smem_limit = prop.sharedMemPerBlockOptin;
    if (pqs::band_doubles(p_max) * sizeof(double) > smem_limit)
        return fail(err, PQP_E_INVALID, "pqp_smoother_create: p_max too large for the shared-memory band");
    pqp_smoother_handle *h = new (std::nothrow) pqp_smoother_handle;
    if (!h) return fail(err, PQP_E_INVALID, "out of host memory");
    h->prm = prm;
    h->device = h->res.device = device;
    h->p_max = p_max;
    h->batch_max = batch_max;
    h->scratch_stride = pqs::scratch_bytes(p_max);
    h->smem = pqs::band_doubles(p_max) * sizeof(double);
    // the Cartesian QP's band is wider: beyond its limit only the Cartesian calls are refused
    h->cart_stride = pqs::cartesian_scratch_bytes(p_max);
    h->cart_smem = pqs::cartesian_band_doubles(p_max) * sizeof(double);
    if (h->cart_smem > smem_limit)
        h->cart_err = "pqp_cartesian_tension_smooth: p_max = " + std::to_string(p_max) +
                      " too large for the Cartesian QP's shared-memory band ((3 p_max + 9) * 11 doubles = " +
                      std::to_string(h->cart_smem) + " bytes, the device allows " + std::to_string(smem_limit) + " per block)";
    pqp::DeviceGuard guard_(device);
    const int rc = [&]() -> int {
        PQP_CUDA(err, resident_grid(smoother_kernel, h->smem, prop.multiProcessorCount, batch_max, &h->grid_max));
        if (h->cart_err.empty())
            PQP_CUDA(err, resident_grid(cartesian_kernel, h->cart_smem, prop.multiProcessorCount, batch_max, &h->cart_grid_max));
        // one scratch block serves both working-set shapes: the Cartesian grid is capped by how many of its (larger)
        // working sets fit, and the block holds at least one
        h->scratch_total = (size_t)h->grid_max * h->scratch_stride;
        if (h->cart_err.empty() && h->scratch_total < h->cart_stride) h->scratch_total = h->cart_stride;
        if (h->cart_err.empty() && (size_t)h->cart_grid_max > h->scratch_total / h->cart_stride)
            h->cart_grid_max = (int)(h->scratch_total / h->cart_stride);
        pqp::Resources &r = h->res;
        const size_t B = batch_max, Ls = B * p_max;
        PQP_CUDA(err, r.alloc(h->d_scratch, h->scratch_total));
        PQP_CUDA(err, r.stream(h->stream));
        PQP_CUDA(err, r.event(h->ev0));
        PQP_CUDA(err, r.event(h->ev1));
        for (int i = 0; i < 5; ++i) PQP_CUDA(err, r.alloc(h->d_in[i], Ls));
        for (int i = 0; i < 3; ++i) PQP_CUDA(err, r.alloc(h->d_out[i], Ls));
        PQP_CUDA(err, r.alloc(h->d_xfull, Ls * 4));
        PQP_CUDA(err, r.alloc(h->d_vl, B));
        PQP_CUDA(err, r.alloc(h->d_p, B));
        PQP_CUDA(err, r.alloc(h->d_status, B));
        PQP_CUDA(err, r.alloc(h->d_iters, B));
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_smoother_destroy(h);
        return rc;
    }
    *out = h;
    return PQP_OK;
}

void pqp_smoother_destroy(pqp_smoother_handle *h) {
    if (!h) return;
    pqp::DeviceGuard guard_(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    delete h;
}

int pqp_tension_smooth_device(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out, void *stream) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    KArgs a{};
    a.batch = in->batch;
    a.mode = 0;
    a.p = in->p;
    a.a0 = in->x; a.a1 = in->y; a.a2 = in->angle; a.a3 = in->k; a.a4 = in->s;
    a.o0 = out->x; a.o1 = out->y; a.o2 = out->s;
    a.x_full = out->x_full;
    a.status = out->status;
    a.iters = out->iters;
    return launch(h, a, static_cast<cudaStream_t>(stream));
}

int pqp_post_smooth_device(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out, void *stream) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    KArgs a{};
    a.batch = in->batch;
    a.mode = 1;
    a.p = in->p;
    a.a0 = in->layer_s; a.a1 = in->lower; a.a2 = in->upper; a.a3 = in->vehicle_l; a.a4 = nullptr;
    a.o0 = out->offsets; a.o1 = nullptr; a.o2 = nullptr;
    a.x_full = out->x_full;
    a.status = out->status;
    a.iters = out->iters;
    return launch(h, a, static_cast<cudaStream_t>(stream));
}

int pqp_cartesian_tension_smooth_device(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in,
                                        const pqp_tension_out *out, void *stream) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    CArgs a{};
    a.batch = in->batch;
    a.p = in->p;
    a.x = in->x; a.y = in->y; a.angle = in->angle; a.clearance = in->clearance;
    a.ox = out->x; a.oy = out->y; a.os = out->s;
    a.x_full = out->x_full;
    a.status = out->status;
    a.iters = out->iters;
    return launch_cartesian(h, a, static_cast<cudaStream_t>(stream));
}

int pqp_cartesian_tension_smooth(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in, const pqp_tension_out *out) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    const double *src[] = {in->x, in->y, in->angle, in->clearance};
    double *dst[] = {out->x, out->y, out->s};
    return run_host(h, {in->batch, in->p, 3, src, 4, nullptr, dst, 3, out->status, out->iters, out->x_full, 3},
                    [&](cudaStream_t s, double *x_full) {
                        const pqp_cartesian_tension_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_in[3]};
                        const pqp_tension_out dout = {h->d_out[0], h->d_out[1], h->d_out[2], h->d_status, h->d_iters, x_full};
                        return pqp_cartesian_tension_smooth_device(h, &din, &dout, s);
                    });
}

int pqp_tension_smooth(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    const double *src[] = {in->x, in->y, in->angle, in->k, in->s};
    double *dst[] = {out->x, out->y, out->s};
    return run_host(h, {in->batch, in->p, 3, src, 5, nullptr, dst, 3, out->status, out->iters, out->x_full, 4},
                    [&](cudaStream_t s, double *x_full) {
                        const pqp_tension_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_in[3], h->d_in[4]};
                        const pqp_tension_out dout = {h->d_out[0], h->d_out[1], h->d_out[2], h->d_status, h->d_iters, x_full};
                        return pqp_tension_smooth_device(h, &din, &dout, s);
                    });
}

int pqp_post_smooth(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out) {
    const int rc = check(h, in, out);
    if (rc != PQP_OK) return rc;
    const double *src[] = {in->layer_s, in->lower, in->upper};
    double *dst[] = {out->offsets};
    return run_host(h, {in->batch, in->p, 2, src, 3, in->vehicle_l, dst, 1, out->status, out->iters, out->x_full, 3},
                    [&](cudaStream_t s, double *x_full) {
                        const pqp_post_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_vl};
                        const pqp_post_out dout = {h->d_out[0], h->d_status, h->d_iters, x_full};
                        return pqp_post_smooth_device(h, &din, &dout, s);
                    });
}

int pqp_smoother_last_kernel_ms(pqp_smoother_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    *ms = h->last_ms;
    return PQP_OK;
}

}  // extern "C"
