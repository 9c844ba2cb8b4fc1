// pqp_smoother.cu — include/pqp_smoother.h: the three smoother QPs of the reference's front end on the GPU.
// One warp (= one CTA) per QP runs pqp_smoother_core.cuh (OSQP on a stage-banded QP, FP64). The serial part of an
// iteration is the banded forward / backward substitution, so its band factor and right-hand side live in shared
// memory; everything else (problem data, iterates) is per-CTA scratch in global memory that stays in L1/L2. A grid
// of min(batch, resident CTAs) loops over the QPs.
#include <cuda_runtime.h>

#include <new>
#include <string>

#include "../../include/pqp_smoother.h"
#include "pqp_device_guard.h"
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
};

namespace {

#define PQS_CUDA(h, call)                                                      \
    do {                                                                       \
        cudaError_t e_ = (call);                                               \
        if (e_ != cudaSuccess) {                                               \
            (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);     \
            return PQP_E_CUDA;                                                 \
        }                                                                      \
    } while (0)

int sfail(pqp_smoother_handle *h, int code, const char *msg) {
    if (h) h->err = msg;
    else g_smoother_create_error = msg;
    return code;
}

pqs::Settings settings_of(const pqp_smoother_params &p) {
    pqs::Settings s;
    s.rho = p.rho; s.sigma = p.sigma; s.alpha = p.alpha; s.eps_abs = p.eps_abs; s.eps_rel = p.eps_rel;
    s.eps_prim_inf = p.eps_prim_inf; s.eps_dual_inf = p.eps_dual_inf; s.adaptive_rho_tolerance = p.adaptive_rho_tolerance;
    s.max_iter = p.max_iter; s.check_termination = p.check_termination; s.scaling = p.scaling;
    s.adaptive_rho = p.adaptive_rho; s.adaptive_rho_interval = p.adaptive_rho_interval;
    return s;
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
    PQS_CUDA(h, cudaFuncSetAttribute(smoother_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem));
    PQS_CUDA(h, cudaEventRecord(h->ev0, s));
    smoother_kernel<<<grid, 32, h->smem, s>>>(a);
    PQS_CUDA(h, cudaGetLastError());
    PQS_CUDA(h, cudaEventRecord(h->ev1, s));
    return PQP_OK;
}

int launch_cartesian(pqp_smoother_handle *h, CArgs &a, cudaStream_t s) {
    a.p_max = h->p_max;
    a.st = settings_of(h->prm);
    a.cw = {h->prm.cartesian_curvature_weight, h->prm.cartesian_curvature_rate_weight, h->prm.cartesian_deviation_weight};
    a.scratch = h->d_scratch;
    a.scratch_stride = h->cart_stride;
    const int grid = a.batch < h->cart_grid_max ? a.batch : h->cart_grid_max;
    PQS_CUDA(h, cudaFuncSetAttribute(cartesian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->cart_smem));
    PQS_CUDA(h, cudaEventRecord(h->ev0, s));
    cartesian_kernel<<<grid, 32, h->cart_smem, s>>>(a);
    PQS_CUDA(h, cudaGetLastError());
    PQS_CUDA(h, cudaEventRecord(h->ev1, s));
    return PQP_OK;
}

int check_cartesian(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in, const pqp_tension_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!h->cart_err.empty()) return sfail(h, PQP_E_INVALID, h->cart_err.c_str());
    if (!in || !out || !in->p || !in->x || !in->y || !in->angle || !in->clearance || !out->x || !out->y || !out->s ||
        !out->status || !out->iters)
        return sfail(h, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max || in->p_max != h->p_max) return sfail(h, PQP_E_INVALID, "batch / p_max do not fit the handle");
    return PQP_OK;
}

template <typename T>
cudaError_t dalloc(T **p, size_t n) {
    return cudaMalloc(reinterpret_cast<void **>(p), (n ? n : 1) * sizeof(T));
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
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (p_max < 4 || p_max > 2000 || batch_max < 1) return sfail(nullptr, PQP_E_INVALID, "pqp_smoother_create: 4 <= p_max <= 2000, batch_max >= 1");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return sfail(nullptr, PQP_E_NO_DEVICE, "pqp_smoother_create: no CUDA device (there is no CPU fallback)");
    pqp_smoother_handle *h = new (std::nothrow) pqp_smoother_handle;
    if (!h) return sfail(nullptr, PQP_E_INVALID, "out of host memory");
    if (params) h->prm = *params;
    else pqp_smoother_default_params(&h->prm);
    if (!(h->prm.rho > 0) || !(h->prm.sigma > 0) || !(h->prm.alpha > 0 && h->prm.alpha < 2) || h->prm.max_iter < 1) {
        delete h;
        return sfail(nullptr, PQP_E_INVALID, "pqp_smoother_create: invalid OSQP settings");
    }
    h->device = device;
    h->p_max = p_max;
    h->batch_max = batch_max;
    h->scratch_stride = pqs::scratch_bytes(p_max);
    h->smem = pqs::band_doubles(p_max) * sizeof(double);
    pqp::DeviceGuard guard_(device);
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e == cudaSuccess && h->smem > (size_t)prop.sharedMemPerBlockOptin) {
        delete h;
        return sfail(nullptr, PQP_E_INVALID, "pqp_smoother_create: p_max too large for the shared-memory band");
    }
    if (e == cudaSuccess) e = cudaFuncSetAttribute(smoother_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem);
    int per_sm = 1;
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, smoother_kernel, 32, h->smem);
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 16) per_sm = 16;
    h->grid_max = prop.multiProcessorCount * per_sm;
    if (h->grid_max > batch_max) h->grid_max = batch_max;
    // the Cartesian QP's band is wider: beyond its limit only the Cartesian calls are refused
    h->cart_stride = pqs::cartesian_scratch_bytes(p_max);
    h->cart_smem = pqs::cartesian_band_doubles(p_max) * sizeof(double);
    if (e == cudaSuccess && h->cart_smem > (size_t)prop.sharedMemPerBlockOptin) {
        h->cart_err = "pqp_cartesian_tension_smooth: p_max = " + std::to_string(p_max) +
                      " too large for the Cartesian QP's shared-memory band ((3 p_max + 9) * 11 doubles = " +
                      std::to_string(h->cart_smem) + " bytes, the device allows " +
                      std::to_string((size_t)prop.sharedMemPerBlockOptin) + " per block)";
    } else if (e == cudaSuccess) {
        e = cudaFuncSetAttribute(cartesian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->cart_smem);
        int cart_per_sm = 1;
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cart_per_sm, cartesian_kernel, 32, h->cart_smem);
        if (cart_per_sm < 1) cart_per_sm = 1;
        if (cart_per_sm > 16) cart_per_sm = 16;
        h->cart_grid_max = prop.multiProcessorCount * cart_per_sm;
        if (h->cart_grid_max > batch_max) h->cart_grid_max = batch_max;
    }
    // one scratch block serves both working-set shapes: the Cartesian grid is capped by how many of its (larger)
    // working sets fit, and the block holds at least one
    h->scratch_total = (size_t)h->grid_max * h->scratch_stride;
    if (h->cart_err.empty() && h->scratch_total < h->cart_stride) h->scratch_total = h->cart_stride;
    if (h->cart_err.empty() && (size_t)h->cart_grid_max > h->scratch_total / h->cart_stride)
        h->cart_grid_max = (int)(h->scratch_total / h->cart_stride);
    const size_t B = batch_max, Ls = B * p_max;
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&h->d_scratch), h->scratch_total);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreate(&h->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&h->ev1);
    for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = dalloc(&h->d_in[i], Ls);
    for (int i = 0; i < 3 && e == cudaSuccess; ++i) e = dalloc(&h->d_out[i], Ls);
    if (e == cudaSuccess) e = dalloc(&h->d_xfull, Ls * 4);
    if (e == cudaSuccess) e = dalloc(&h->d_vl, B);
    if (e == cudaSuccess) e = dalloc(&h->d_p, B);
    if (e == cudaSuccess) e = dalloc(&h->d_status, B);
    if (e == cudaSuccess) e = dalloc(&h->d_iters, B);
    if (e != cudaSuccess) {
        g_smoother_create_error = std::string("pqp_smoother_create: ") + cudaGetErrorString(e);
        pqp_smoother_destroy(h);
        return PQP_E_CUDA;
    }
    *out = h;
    return PQP_OK;
}

void pqp_smoother_destroy(pqp_smoother_handle *h) {
    if (!h) return;
    pqp::DeviceGuard guard_(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    cudaFree(h->d_scratch);
    for (int i = 0; i < 5; ++i) cudaFree(h->d_in[i]);
    for (int i = 0; i < 3; ++i) cudaFree(h->d_out[i]);
    cudaFree(h->d_xfull); cudaFree(h->d_vl); cudaFree(h->d_p); cudaFree(h->d_status); cudaFree(h->d_iters);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int pqp_tension_smooth_device(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out, void *stream) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->x || !in->y || !in->angle || !in->k || !in->s || !out->x || !out->y || !out->s ||
        !out->status || !out->iters)
        return sfail(h, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max || in->p_max != h->p_max) return sfail(h, PQP_E_INVALID, "batch / p_max do not fit the handle");
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
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->layer_s || !in->lower || !in->upper || !in->vehicle_l || !out->offsets || !out->status || !out->iters)
        return sfail(h, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max || in->p_max != h->p_max) return sfail(h, PQP_E_INVALID, "batch / p_max do not fit the handle");
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
    const int rc = check_cartesian(h, in, out);
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
    int rc = check_cartesian(h, in, out);
    if (rc != PQP_OK) return rc;
    for (int b = 0; b < in->batch; ++b)
        if (in->p[b] < 3 || in->p[b] > in->p_max) return sfail(h, PQP_E_INVALID, "p[b] must be in [3, p_max]");
    pqp::DeviceGuard guard_(h->device);
    cudaStream_t s = h->stream;
    const size_t B = in->batch, Ls = B * h->p_max;
    const double *src[4] = {in->x, in->y, in->angle, in->clearance};
    for (int i = 0; i < 4; ++i) PQS_CUDA(h, cudaMemcpyAsync(h->d_in[i], src[i], Ls * sizeof(double), cudaMemcpyHostToDevice, s));
    PQS_CUDA(h, cudaMemcpyAsync(h->d_p, in->p, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    for (int i = 0; i < 3; ++i) PQS_CUDA(h, cudaMemsetAsync(h->d_out[i], 0, Ls * sizeof(double), s));
    if (out->x_full) PQS_CUDA(h, cudaMemsetAsync(h->d_xfull, 0, Ls * 3 * sizeof(double), s));
    pqp_cartesian_tension_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_in[3]};
    pqp_tension_out dout = {h->d_out[0], h->d_out[1], h->d_out[2], h->d_status, h->d_iters, out->x_full ? h->d_xfull : nullptr};
    rc = pqp_cartesian_tension_smooth_device(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    double *dst[3] = {out->x, out->y, out->s};
    for (int i = 0; i < 3; ++i) PQS_CUDA(h, cudaMemcpyAsync(dst[i], h->d_out[i], Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->iters, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->x_full) PQS_CUDA(h, cudaMemcpyAsync(out->x_full, h->d_xfull, Ls * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaStreamSynchronize(s));
    PQS_CUDA(h, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return PQP_OK;
}

int pqp_tension_smooth(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->x || !in->y || !in->angle || !in->k || !in->s || !out->x || !out->y || !out->s ||
        !out->status || !out->iters)
        return sfail(h, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max || in->p_max != h->p_max) return sfail(h, PQP_E_INVALID, "batch / p_max do not fit the handle");
    for (int b = 0; b < in->batch; ++b)
        if (in->p[b] < 3 || in->p[b] > in->p_max) return sfail(h, PQP_E_INVALID, "p[b] must be in [3, p_max]");
    pqp::DeviceGuard guard_(h->device);
    cudaStream_t s = h->stream;
    const size_t B = in->batch, Ls = B * h->p_max;
    const double *src[5] = {in->x, in->y, in->angle, in->k, in->s};
    for (int i = 0; i < 5; ++i) PQS_CUDA(h, cudaMemcpyAsync(h->d_in[i], src[i], Ls * sizeof(double), cudaMemcpyHostToDevice, s));
    PQS_CUDA(h, cudaMemcpyAsync(h->d_p, in->p, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    for (int i = 0; i < 3; ++i) PQS_CUDA(h, cudaMemsetAsync(h->d_out[i], 0, Ls * sizeof(double), s));
    if (out->x_full) PQS_CUDA(h, cudaMemsetAsync(h->d_xfull, 0, Ls * 4 * sizeof(double), s));
    pqp_tension_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_in[3], h->d_in[4]};
    pqp_tension_out dout = {h->d_out[0], h->d_out[1], h->d_out[2], h->d_status, h->d_iters, out->x_full ? h->d_xfull : nullptr};
    int rc = pqp_tension_smooth_device(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    double *dst[3] = {out->x, out->y, out->s};
    for (int i = 0; i < 3; ++i) PQS_CUDA(h, cudaMemcpyAsync(dst[i], h->d_out[i], Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->iters, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->x_full) PQS_CUDA(h, cudaMemcpyAsync(out->x_full, h->d_xfull, Ls * 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaStreamSynchronize(s));
    PQS_CUDA(h, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return PQP_OK;
}

int pqp_post_smooth(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->p || !in->layer_s || !in->lower || !in->upper || !in->vehicle_l || !out->offsets || !out->status || !out->iters)
        return sfail(h, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max || in->p_max != h->p_max) return sfail(h, PQP_E_INVALID, "batch / p_max do not fit the handle");
    for (int b = 0; b < in->batch; ++b)
        if (in->p[b] < 2 || in->p[b] > in->p_max) return sfail(h, PQP_E_INVALID, "p[b] must be in [2, p_max]");
    pqp::DeviceGuard guard_(h->device);
    cudaStream_t s = h->stream;
    const size_t B = in->batch, Ls = B * h->p_max;
    const double *src[3] = {in->layer_s, in->lower, in->upper};
    for (int i = 0; i < 3; ++i) PQS_CUDA(h, cudaMemcpyAsync(h->d_in[i], src[i], Ls * sizeof(double), cudaMemcpyHostToDevice, s));
    PQS_CUDA(h, cudaMemcpyAsync(h->d_vl, in->vehicle_l, B * sizeof(double), cudaMemcpyHostToDevice, s));
    PQS_CUDA(h, cudaMemcpyAsync(h->d_p, in->p, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQS_CUDA(h, cudaMemsetAsync(h->d_out[0], 0, Ls * sizeof(double), s));
    if (out->x_full) PQS_CUDA(h, cudaMemsetAsync(h->d_xfull, 0, Ls * 3 * sizeof(double), s));
    pqp_post_in din = {in->batch, in->p_max, h->d_p, h->d_in[0], h->d_in[1], h->d_in[2], h->d_vl};
    pqp_post_out dout = {h->d_out[0], h->d_status, h->d_iters, out->x_full ? h->d_xfull : nullptr};
    int rc = pqp_post_smooth_device(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    PQS_CUDA(h, cudaMemcpyAsync(out->offsets, h->d_out[0], Ls * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->status, h->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaMemcpyAsync(out->iters, h->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->x_full) PQS_CUDA(h, cudaMemcpyAsync(out->x_full, h->d_xfull, Ls * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQS_CUDA(h, cudaStreamSynchronize(s));
    PQS_CUDA(h, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return PQP_OK;
}

int pqp_smoother_last_kernel_ms(pqp_smoother_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    *ms = h->last_ms;
    return PQP_OK;
}

}  // extern "C"
