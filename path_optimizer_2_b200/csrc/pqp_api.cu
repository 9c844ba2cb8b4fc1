// pqp_api.cu — C ABI (include/pqp.h) of the batched path-QP solver for H100 (sm_90a).
//
// Host side: handle with device buffers + per-instance warm state, H2D/D2H staging for the
// host-pointer entry points, launches. Device side: the kernel entry (one warp = one CTA =
// one QP instance; the instance's knot block is staged into shared memory with one TMA
// bulk copy + mbarrier) around the QpWarp<C> solver of pqp_kernel.cuh, and the FP64
// Frenet->Cartesian epilogue kernel (base_solver.cpp:263-288).
//
// There is no CPU fallback in this library: every entry point needs a CUDA device.
#include <cuda_runtime.h>
#include <time.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/pqp_multi.h"
#include "pqp_batch_layout.h"
#include "pqp_host_common.h"
#include "pqp_host_handle.h"

namespace {

thread_local std::string g_create_error;

// ------------------------------------------------------------------ device: TMA staging
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D bulk copy global -> shared, completion counted on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// ------------------------------------------------------------------ device: kernel entry
// One CTA = one warp = one QP instance. Dynamic shared memory: NFIELD*C*32 floats of
// solver state (the factor region doubles as the FP64 input staging buffer) + 1 mbarrier.
template <int C, typename real, bool Incr>
__global__ void __launch_bounds__(32) pqp_admm_kernel(const __grid_constant__ pqp::KernelArgs ka) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    real *smem = reinterpret_cast<real *>(smem_raw);
    const int lane = threadIdx.x;
    const int qp = blockIdx.x;
    if (qp >= ka.batch) return;
    const double *src = ka.knots + (size_t)qp * PQP_NFIELDS * ka.n_max;
    if (ka.use_tma) {
        uint64_t *bar = reinterpret_cast<uint64_t *>(smem + pqp::NFIELD * C * 32);
        double *stage = reinterpret_cast<double *>(smem + pqp::FDI * C * 32);
        const uint32_t bytes = (uint32_t)(PQP_NFIELDS * ka.n_max * sizeof(double));
        if (lane == 0) {
            mbar_init(bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
        if (lane == 0) {
            mbar_expect_tx(bar, bytes);
            tma_load_1d(stage, src, bytes, bar);
        }
        mbar_wait(bar, 0);
        src = stage;
    }
    pqp::QpWarp<C, real, pqp::SmemStore<C, real>, Incr> w(ka, pqp::SmemStore<C, real>(smem, lane), lane, qp);
    w.run(src, ka.n_max, (size_t)(qp + ka.qp0));
}


// FP64 instantiation at C = 16 (256 <= n_max <= 511): its state (72 x 16 x 32 doubles = 288 KB per QP)
// exceeds shared memory, so the same storage policy is pointed at a per-CTA block of global memory
// (it lives in L1/L2; only the owning lane ever touches an element). This is the parity / escalation
// path, not the throughput path: a few resident CTAs loop over the instances.
template <int C, typename real, bool Incr>
__global__ void __launch_bounds__(32) pqp_admm_kernel_gmem(const __grid_constant__ pqp::KernelArgs ka, real *state) {
    const int lane = threadIdx.x;
    real *st = state + (size_t)blockIdx.x * pqp::NFIELD * C * 32;
    for (int qp = blockIdx.x; qp < ka.batch; qp += gridDim.x) {
        const double *src = ka.knots + (size_t)qp * PQP_NFIELDS * ka.n_max;
        pqp::QpWarp<C, real, pqp::SmemStore<C, real>, Incr> w(ka, pqp::SmemStore<C, real>(st, lane), lane, qp);
        w.run(src, ka.n_max, (size_t)(qp + ka.qp0));
        __syncwarp();
    }
}

// Persistent kernel (FP32): as many one-warp CTAs as fit on the SMs (shared memory bounds it: the
// whole per-QP state of SmemStore, 37 KB at C = 4, 74 KB at C = 8, 147 KB at C = 16); every warp
// solves one QP at a time and takes the next unsolved instance from a global work counter
// (iteration counts vary 3x between instances; a static assignment would idle). Each instance's
// knot block is staged into the warp's factor region by one TMA bulk copy, as in pqp_admm_kernel;
// the mbarrier is initialised once and its phase advances by one per instance. Scratch slots
// (Ruiz factors, delta_y) belong to the CTA, not to the instance.
template <int C, bool Incr>
__global__ void __launch_bounds__(32) pqp_admm_kernel_persistent(const __grid_constant__ pqp::KernelArgs ka) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *smem = reinterpret_cast<float *>(smem_raw);
    const int lane = threadIdx.x;
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + pqp::NFIELD * C * 32);
    double *stage = reinterpret_cast<double *>(smem + pqp::FDI * C * 32);
    const uint32_t bytes = (uint32_t)(PQP_NFIELDS * ka.n_max * sizeof(double));
    if (ka.use_tma && lane == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t phase = 0;
    for (;;) {
        int qp = 0;
        if (lane == 0) qp = atomicAdd(ka.work_counter, 1);
        qp = __shfl_sync(0xffffffffu, qp, 0);
        if (qp >= ka.batch) break;
        int chunk = 0;
        if (ka.ready) {
            // streamed launch: this instance's inputs may still be in flight
            while (chunk + 1 < ka.n_chunks && qp >= ka.chunk_lo[chunk + 1]) ++chunk;
            bool landed = true;
            if (lane == 0) {
                const volatile int *flag = ka.ready + chunk;
                const long long t0 = clock64();
                while (*flag == 0) {
                    __nanosleep(200);
                    if (clock64() - t0 > 20000000000LL) {  // ~10 s: give up, never hang
                        landed = false;
                        atomicExch(ka.work_counter, 1 << 30);  // and stop everybody else from taking work
                        break;
                    }
                }
                __threadfence();
            }
            landed = __shfl_sync(0xffffffffu, landed ? 1 : 0, 0) != 0;
            if (!landed) {
                if (lane == 0 && ka.status) ka.status[qp] = pqp::kUnsolved;
                continue;
            }
        }
        const double *src = ka.knots + (size_t)qp * PQP_NFIELDS * ka.n_max;
        if (ka.use_tma) {
            // the previous instance wrote the staging region through the generic proxy; order those writes
            // before the bulk copy (async proxy) overwrites it
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                mbar_expect_tx(bar, bytes);
                tma_load_1d(stage, src, bytes, bar);
            }
            mbar_wait(bar, phase);
            phase ^= 1u;
            src = stage;
        }
        pqp::QpWarp<C, float, pqp::SmemStore<C, float>, Incr> w(ka, pqp::SmemStore<C, float>(smem, lane), lane, qp);
        w.run(src, ka.n_max, (size_t)blockIdx.x);
        __syncwarp();
        if (ka.done) {
            if (lane == 0) {
                __threadfence();  // this instance's outputs before the count
                const int len = ka.chunk_lo[chunk + 1] - ka.chunk_lo[chunk];
                if (atomicAdd(ka.done + chunk, 1) + 1 == len) {
                    __threadfence_system();
                    *reinterpret_cast<volatile int *>(ka.host_done + chunk) = 1;
                }
            }
        }
    }
}

// BaseSolver::getOptimizedPath (base_solver.cpp:263-288) in FP64, one thread per knot.
__device__ __forceinline__ double constrain_angle(double a) {
    while (a > M_PI) a -= 2 * M_PI;
    while (a < -M_PI) a += 2 * M_PI;
    return a;
}
__global__ void frenet_to_cartesian_kernel(int batch, int n_max, const int *__restrict__ n,
                                           const double *__restrict__ ref, const double *__restrict__ sol,
                                           double *__restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= batch * n_max) return;
    const int b = idx / n_max, i = idx - b * n_max;
    if (i >= n[b]) return;
    const size_t r = (size_t)b * 3 * n_max, s = (size_t)b * 4 * n_max;
    const double angle = ref[r + 2 * n_max + i];
    const double l = sol[s + i], psi = sol[s + n_max + i];
    const double new_angle = constrain_angle(angle + M_PI_2);
    out[r + i] = ref[r + i] + l * cos(new_angle);
    out[r + n_max + i] = ref[r + n_max + i] + l * sin(new_angle);
    out[r + 2 * n_max + i] = constrain_angle(angle + psi);
}

// previous solution -> linearisation fields of the device knot buffer
__global__ void relinearise_kernel(int batch, int n_max, const double *__restrict__ sol,
                                   double *__restrict__ knots) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= batch * n_max) return;
    const int b = idx / n_max, i = idx - b * n_max;
    const size_t s = (size_t)b * 4 * n_max, k = (size_t)b * PQP_NFIELDS * n_max;
    knots[k + (size_t)PQP_F_L * n_max + i] = sol[s + i];
    knots[k + (size_t)PQP_F_PSI * n_max + i] = sol[s + n_max + i];
    knots[k + (size_t)PQP_F_K * n_max + i] = sol[s + 2 * (size_t)n_max + i];
}

// Receding-horizon tick (BASELINE configs[4]): the planning window advances by `tick` knots along
// an extended reference ext[b][9][ext_len]; the new linearisation point is the previous solution
// shifted by one knot (last knot repeated) and the new x0 is the previous solution at knot 1.
__global__ void advance_window_kernel(int batch, int n_max, int ext_len, int tick, const double *__restrict__ ext,
                                      const double *__restrict__ sol, double *__restrict__ knots,
                                      double *__restrict__ inst) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= batch * n_max) return;
    const int b = idx / n_max, i = idx - b * n_max;
    const double *e = ext + (size_t)b * PQP_NFIELDS * ext_len + tick + i;
    const double *sb = sol + (size_t)b * 4 * n_max;
    double *k = knots + (size_t)b * PQP_NFIELDS * n_max + i;
    const int src = i + 1 < n_max ? i + 1 : n_max - 1;
#pragma unroll
    for (int f = 0; f < PQP_NFIELDS; ++f) {
        double v = e[(size_t)f * ext_len];
        if (f == PQP_F_L) v = sb[src];
        if (f == PQP_F_PSI) v = sb[n_max + src];
        if (f == PQP_F_K) v = sb[2 * (size_t)n_max + src];
        k[(size_t)f * n_max] = v;
    }
    if (i == 0) {
        double *ib = inst + (size_t)b * PQP_NINST;
        const int one = n_max > 1 ? 1 : 0;
        ib[PQP_I_L0] = sb[one];
        ib[PQP_I_PSI0] = sb[n_max + one];
        ib[PQP_I_K0] = sb[2 * (size_t)n_max + one];
    }
}

// After an FP64 re-solve: the instance's warm slot (FP32) takes over the FP64 run's scaled iterates and rho, so
// that a later pqp_resolve warm-starts from the run whose result was returned, not from the abandoned FP32 one.
__global__ void adopt_warm_kernel(int count, size_t warm_len, const int *__restrict__ slots, const double *__restrict__ e_warm,
                                  const double *__restrict__ e_rho, float *__restrict__ d_warm, float *__restrict__ d_rho) {
    const int j = blockIdx.y;
    if (j >= count) return;
    const size_t b = (size_t)slots[j];
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < warm_len; i += (size_t)gridDim.x * blockDim.x)
        d_warm[b * warm_len + i] = (float)e_warm[(size_t)j * warm_len + i];
    if (blockIdx.x == 0 && threadIdx.x == 0) d_rho[b] = (float)e_rho[j];
}

// {cost, status, iters} -> one 16-byte record per instance (the payload of the multi-GPU all-gather)
__global__ void pack_results_kernel(int batch, const double *__restrict__ cost, const int *__restrict__ status,
                                    const int *__restrict__ iters, pqp_result_rec *__restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    pqp_result_rec r;
    r.cost = cost[b];
    r.status = status[b];
    r.iters = iters[b];
    out[b] = r;
}

using SolveKernel = void (*)(pqp::KernelArgs);

}  // namespace

// ------------------------------------------------------------------ handle
struct pqp_handle {
    pqp_params prm;
    int n_max = 0, batch_max = 0, device = 0, chunk = 0;
    int sm_count = 0, warps_per_sm = 0;
    size_t smem_bytes = 0;
    static const int kStreams = 8;
    cudaStream_t stream = nullptr;            // streams[0]
    cudaStream_t streams[kStreams] = {};      // one per pipeline chunk
    cudaEvent_t evs[kStreams] = {};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // device buffers owned by the handle
    double *d_knots = nullptr, *d_inst = nullptr, *d_sol = nullptr, *d_cost = nullptr, *d_info = nullptr;
    double *d_xf = nullptr, *d_yf = nullptr, *d_zf = nullptr, *d_ref = nullptr, *d_xy = nullptr;
    int *d_n = nullptr, *d_p = nullptr, *d_status = nullptr, *d_iters = nullptr;
    void *d_warm = nullptr, *d_scal = nullptr, *d_dy = nullptr, *d_rho = nullptr;
    double *d_state64 = nullptr;   // per-CTA state of the FP64 kernel at C = 16 (global memory)
    int *d_ready = nullptr, *d_done = nullptr;      // per-chunk flags of the streamed launch
    int *h_done = nullptr, *d_hdone = nullptr;     // mapped pinned host memory + its device alias
    static const int kCounters = 64;
    int *d_counters = nullptr;
    unsigned counter_next = 0;
    bool persistent = false;       // params.reserved bit 3: persistent launch with a work counter (FP32 kernel)
    bool incr = false;             // ADMM step in increment form (FP32 kernels)
    bool fp64 = false;             // params.reserved bit 1: iterate in FP64
    bool escalate = true;          // params.reserved bit 2 clears it
    bool cold_only = false;        // params.reserved bit 128: no warm state is kept (pqp_resolve* is refused)
    float stage_ms[PQP_NSTAGES] = {0, 0, 0, 0, 0};
    cudaEvent_t ev_st[4] = {};     // stage boundaries of the single-stream host call
    SolveKernel kernel = nullptr;  // the handle's solve kernel, chosen and prepared at create
    SolveKernel kernel64 = nullptr;  // the FP64 kernel of the escalation (nullptr at C = 16), prepared on first use
    size_t smem_bytes64 = 0;
    bool prepared64 = false;
    int *d_flags = nullptr;
    int *h_status = nullptr, *h_flags = nullptr;  // pinned host mirrors
    // FP64 escalation of suspected-infeasible instances (small side batch)
    int esc_cap = 0;
    double *e_knots = nullptr, *e_inst = nullptr, *e_sol = nullptr, *e_cost = nullptr, *e_info = nullptr;
    double *e_xf = nullptr, *e_yf = nullptr, *e_zf = nullptr;
    int *e_n = nullptr, *e_p = nullptr, *e_status = nullptr, *e_iters = nullptr, *e_slots = nullptr;
    void *e_warm = nullptr, *e_scal = nullptr, *e_dy = nullptr, *e_rho = nullptr;
    long long escalated = 0;
    double *d_sol2 = nullptr;
    int *d_n2 = nullptr;
    bool solved = false, host_inputs_resident = false, d_p_valid = false;
    int last_batch = 0;
    float last_ms = 0.0f;
    long long launches = 0;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace {

using pqp::DeviceGuard;
using pqp::fail;

// The solve kernel of C stages for (FP64, increment form, persistent launch). The increment form is only instantiated
// for FP32 (the FP64 kernel is exact in either form), and so is the persistent launch. FP64 at C = 16 has no
// shared-memory kernel (288 KB per QP): nullptr, run_device launches pqp_admm_kernel_gmem instead.
template <int C>
SolveKernel kernel_for(bool fp64, bool incr, bool persistent) {
    if (fp64) {
        if constexpr (C == 16) return nullptr;
        else return pqp_admm_kernel<C, double, false>;
    }
    if (persistent) return incr ? pqp_admm_kernel_persistent<C, true> : pqp_admm_kernel_persistent<C, false>;
    return incr ? pqp_admm_kernel<C, float, true> : pqp_admm_kernel<C, float, false>;
}
SolveKernel select_kernel(int chunk, bool fp64, bool incr, bool persistent) {
    switch (chunk) {
        case 1: return kernel_for<1>(fp64, incr, persistent);
        case 2: return kernel_for<2>(fp64, incr, persistent);
        case 4: return kernel_for<4>(fp64, incr, persistent);
        case 8: return kernel_for<8>(fp64, incr, persistent);
        default: return kernel_for<16>(fp64, incr, persistent);
    }
}

// opts `k` in to `smem` bytes of dynamic shared memory and counts its resident CTAs per SM
cudaError_t prepare(SolveKernel k, size_t smem, int *blocks_per_sm) {
    if (!k) {  // the global-memory kernel: nothing to prepare
        *blocks_per_sm = 2;
        return cudaSuccess;
    }
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, k, 32, smem);
}

int validate_batch(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out) return fail(h->err, PQP_E_INVALID, "null batch");
    if (!in->knots || !in->inst || !in->n || !out->sol) return fail(h->err, PQP_E_INVALID, "null buffer");
    if (in->batch < 1 || in->batch > h->batch_max) return fail(h->err, PQP_E_INVALID, "batch out of range");
    if (in->n_max != h->n_max) return fail(h->err, PQP_E_INVALID, "n_max differs from the handle's");
    return PQP_OK;
}

// device pointers in `in`/`out`; asynchronous
struct StreamedLaunch {
    const int *ready = nullptr;
    int *done = nullptr, *host_done = nullptr;
    int n_chunks = 0;
    int chunk_lo[9] = {};
};

int run_device(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out, int mode,
               cudaStream_t s, bool timed, int qp0 = 0, bool esc = false, int *flags = nullptr,
               const StreamedLaunch *sl = nullptr) {
    pqp::KernelArgs ka;
    ka.prm = pqp::make_dev_params(h->prm);
    ka.batch = in->batch;
    ka.n_max = in->n_max;
    ka.mode = mode | ((h->cold_only && !esc) ? 2 : 0);
    ka.qp0 = qp0;
    const size_t block_bytes = (size_t)PQP_NFIELDS * in->n_max * sizeof(double);
    ka.use_tma = ((block_bytes % 16) == 0 && (reinterpret_cast<uintptr_t>(in->knots) % 16) == 0) ? 1 : 0;
    ka.knots = in->knots;
    ka.inst = in->inst;
    ka.n = in->n;
    ka.p = in->p;
    ka.sol = out->sol;
    ka.cost = out->cost;
    ka.status = out->status;
    ka.iters = out->iters;
    ka.x_full = out->x_full;
    ka.y_full = out->y_full;
    ka.z_full = out->z_full;
    ka.info = out->info;
    ka.flags = flags;
    ka.work_counter = nullptr;
    ka.ready = sl ? sl->ready : nullptr;
    ka.done = sl ? sl->done : nullptr;
    ka.host_done = sl ? sl->host_done : nullptr;
    ka.n_chunks = sl ? sl->n_chunks : 0;
    for (int c = 0; c < 9; ++c) ka.chunk_lo[c] = sl ? sl->chunk_lo[c] : 0;
    ka.warm = esc ? h->e_warm : h->d_warm;
    ka.scal = esc ? h->e_scal : h->d_scal;
    ka.dy = esc ? h->e_dy : h->d_dy;
    ka.rho_state = esc ? h->e_rho : h->d_rho;
    if (timed) PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    const bool fp64 = esc || h->fp64;
    if (fp64 && !h->prepared64) {
        int bps = 0;
        PQP_CUDA(h->err, prepare(h->kernel64, h->smem_bytes64, &bps));
        h->prepared64 = true;
    }
    if (fp64 && h->chunk == 16) {
        const int ctas = std::min(ka.batch, 2 * h->sm_count);
        if (!h->d_state64) PQP_CUDA(h->err, h->res.alloc(h->d_state64, (size_t)2 * h->sm_count * pqp::smem_floats(16)));
        pqp_admm_kernel_gmem<16, double, false><<<ctas, 32, 0, s>>>(ka, h->d_state64);
    } else {
        int ctas = ka.batch;
        if (!fp64 && h->persistent) {
            // one work counter per concurrently running launch (pipeline chunk); counters rotate; min(batch, resident)
            // one-warp CTAs, resident = SMs x CTAs per SM at this shared-memory size
            int *ctr = h->d_counters + (h->counter_next++ % pqp_handle::kCounters);
            PQP_CUDA(h->err, cudaMemsetAsync(ctr, 0, sizeof(int), s));
            ka.work_counter = ctr;
            ctas = std::min(ka.batch, h->sm_count * h->warps_per_sm);
        }
        (fp64 ? h->kernel64 : h->kernel)<<<ctas, 32, fp64 ? h->smem_bytes64 : h->smem_bytes, s>>>(ka);
    }
    PQP_CUDA(h->err, cudaGetLastError());
    if (timed) PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->launches++;
    if (!esc) {
        h->solved = true;
        if (qp0 == 0) h->last_batch = in->batch;
    }
    return PQP_OK;
}

// The FP64 escalation's side batch of esc_cap instances, all or nothing: after a failed allocation it has no
// buffers, so the next escalation allocates again instead of running with a missing one.
cudaError_t alloc_escalation(pqp_handle *h) {
    const size_t E = h->esc_cap, c = h->chunk;
    const auto batch_of = [&](auto member) { return E * pqp::per_instance(member, h->n_max); };
    pqp::Resources &r = h->res;
    return r.group([&] {
        cudaError_t e = r.alloc(h->e_knots, batch_of(&pqp_batch_in::knots));
        if (e == cudaSuccess) e = r.alloc(h->e_inst, batch_of(&pqp_batch_in::inst));
        if (e == cudaSuccess) e = r.alloc(h->e_n, batch_of(&pqp_batch_in::n));
        if (e == cudaSuccess) e = r.alloc(h->e_p, batch_of(&pqp_batch_in::p));
        if (e == cudaSuccess) e = r.alloc(h->e_sol, batch_of(&pqp_batch_out::sol));
        if (e == cudaSuccess) e = r.alloc(h->e_cost, batch_of(&pqp_batch_out::cost));
        if (e == cudaSuccess) e = r.alloc(h->e_status, batch_of(&pqp_batch_out::status));
        if (e == cudaSuccess) e = r.alloc(h->e_iters, batch_of(&pqp_batch_out::iters));
        if (e == cudaSuccess) e = r.alloc(h->e_info, batch_of(&pqp_batch_out::info));
        if (e == cudaSuccess) e = r.alloc(h->e_xf, batch_of(&pqp_batch_out::x_full));
        if (e == cudaSuccess) e = r.alloc(h->e_yf, batch_of(&pqp_batch_out::y_full));
        if (e == cudaSuccess) e = r.alloc(h->e_zf, batch_of(&pqp_batch_out::z_full));
        if (e == cudaSuccess) e = r.alloc(h->e_warm, E * pqp::warm_floats(c) * sizeof(double));
        if (e == cudaSuccess) e = r.alloc(h->e_scal, E * pqp::scal_floats(c) * sizeof(double));
        if (e == cudaSuccess) e = r.alloc(h->e_dy, E * pqp::dy_floats(c) * sizeof(double));
        if (e == cudaSuccess) e = r.alloc(h->e_rho, E * sizeof(double));
        if (e == cudaSuccess) e = r.alloc(h->e_slots, E);
        return e;
    });
}

// Instances the FP32 kernel could neither solve nor certify (iteration cap reached while the
// first two conditions of OSQP's primal-infeasibility certificate held) are re-solved cold by
// the FP64 instantiation of the same kernel: FP32 iterates resolve |A'dy| < 1e-4 |dy| only to
// ~5e-4 (DESIGN.md), FP64 ones reproduce the reference's PRIMAL_INFEASIBLE status. Rare path,
// plain synchronous copies.
int escalate_fp64(pqp_handle *h, const pqp_batch_in &dev_in, const pqp_batch_out *out, int B) {
    std::vector<int> idx;
    for (int b = 0; b < B; ++b)
        // also an "inaccurate" certificate at the iteration cap: in FP32 the 10x-tolerance test can
        // pass on rounding noise alone, the FP64 run decides (normally: PRIMAL_INFEASIBLE proper)
        if ((h->h_status[b] == PQP_MAX_ITER_REACHED && (h->h_flags[b] & 1)) ||
            h->h_status[b] == PQP_PRIMAL_INFEASIBLE_INACCURATE)
            idx.push_back(b);
    if (idx.empty()) return PQP_OK;
    const int nmax = h->n_max;
    const size_t c = h->chunk;
    if (!h->e_knots) {
        h->esc_cap = h->batch_max < 256 ? h->batch_max : 256;
        PQP_CUDA(h->err, alloc_escalation(h));
    }
    cudaStream_t s = h->stream;
    // inputs come from the handle's device copy dev_in (valid for both host-batch and NULL-batch calls)
    const pqp_batch_in e_in = {h->esc_cap, nmax, h->e_knots, h->e_inst, h->e_n, h->d_p_valid ? h->e_p : nullptr};
    const pqp_batch_out e_out = {h->e_sol, h->e_cost, h->e_status, h->e_iters, h->e_xf, h->e_yf, h->e_zf, h->e_info};
    const pqp_batch_out e_full = {nullptr, nullptr, nullptr, nullptr, h->e_xf, h->e_yf, h->e_zf, nullptr};
    // the device-resident results are kept coherent too (resolve(NULL) linearises about d_sol)
    const pqp_batch_out resident = {h->d_sol, h->d_cost, h->d_status, h->d_iters, nullptr, nullptr, nullptr, nullptr};
    for (size_t start = 0; start < idx.size(); start += h->esc_cap) {
        const int E = (int)std::min(idx.size() - start, (size_t)h->esc_cap);
        for (int j = 0; j < E; ++j)
            PQP_CUDA(h->err, pqp::copy_batch(e_in, j, dev_in, idx[start + j], 1, nmax, cudaMemcpyDeviceToDevice, s));
        PQP_CUDA(h->err, pqp::zero_batch(e_full, 0, E, nmax, s));
        pqp_batch_in din = e_in;
        din.batch = E;
        int rc = run_device(h, &din, &e_out, 0, s, false, 0, true, nullptr);
        if (rc) return rc;
        for (int j = 0; j < E; ++j) {
            const int b = idx[start + j];
            PQP_CUDA(h->err, pqp::copy_batch(*out, b, e_out, j, 1, nmax, cudaMemcpyDeviceToHost, s));
            PQP_CUDA(h->err, pqp::copy_batch(resident, b, e_out, j, 1, nmax, cudaMemcpyDeviceToDevice, s));
        }
        // the warm slots of these instances adopt the FP64 run's scaled iterates and rho
        if (!h->cold_only) {
            PQP_CUDA(h->err, cudaMemcpyAsync(h->e_slots, idx.data() + start, (size_t)E * sizeof(int), cudaMemcpyHostToDevice, s));
            const size_t wf = pqp::warm_floats(c);
            adopt_warm_kernel<<<dim3((unsigned)((wf + 255) / 256), (unsigned)E), 256, 0, s>>>(
                E, wf, h->e_slots, static_cast<const double *>(h->e_warm), static_cast<const double *>(h->e_rho),
                static_cast<float *>(h->d_warm), static_cast<float *>(h->d_rho));
            PQP_CUDA(h->err, cudaGetLastError());
        }
        PQP_CUDA(h->err, cudaStreamSynchronize(s));
        h->escalated += E;
    }
    return PQP_OK;
}



// Host-buffer solve on the persistent kernel as ONE launch over the whole batch:
// the kernel starts immediately and each warp waits (ready[chunk]) until the H2D copy of the
// chunk its next instance belongs to has landed; finished chunks are announced through mapped
// host memory (host_done[chunk]) so their D2H copies overlap the rest of the solve. Compared
// with one launch per chunk this removes the per-launch tail of a persistent kernel.
int run_host_streamed(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out, const pqp_batch_in &dev_in,
                      const pqp_batch_out &dev_out, const pqp_batch_out &dev_full, int mode, int B) {
    const int nmax = h->n_max;
    // up to kStreams chunks of >= 256 instances: small batches (configs[1]: 1024) still overlap
    // their copies with the solve, large ones (8192) move 1024 instances per chunk
    const int min_chunk = 256;
    int nchunks = (B + min_chunk - 1) / min_chunk;
    if (nchunks > pqp_handle::kStreams) nchunks = pqp_handle::kStreams;
    const int per = (B + nchunks - 1) / nchunks;
    nchunks = (B + per - 1) / per;
    // chunk boundaries. Large batches use a ramp instead of equal chunks: nothing can start before the FIRST chunk
    // has landed and nothing is returned before the LAST chunk has finished, so those two are small (1/32 and 2/32 of
    // the batch) and the middle ones carry the volume.
    int lo_of[pqp_handle::kStreams + 1];
    if (nchunks == pqp_handle::kStreams && B >= 32 * min_chunk) {
        static const int w[pqp_handle::kStreams] = {1, 3, 6, 6, 6, 5, 3, 2};  // / 32
        int acc = 0;
        for (int c = 0; c < nchunks; ++c) {
            lo_of[c] = (int)((long long)B * acc / 32);
            acc += w[c];
        }
        lo_of[nchunks] = B;
    } else {
        for (int c = 0; c <= nchunks; ++c) lo_of[c] = (c * per < B) ? c * per : B;
    }
    cudaStream_t sk = h->streams[0], sc = h->streams[1], sd = h->streams[2];
    for (int c = 0; c < pqp_handle::kStreams; ++c) h->h_done[c] = 0;
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_ready, 0, pqp_handle::kStreams * sizeof(int), sk));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_done, 0, pqp_handle::kStreams * sizeof(int), sk));
    PQP_CUDA(h->err, pqp::zero_batch(dev_full, 0, B, nmax, sk));
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, sk));
    PQP_CUDA(h->err, cudaStreamWaitEvent(sc, h->ev0, 0));
    PQP_CUDA(h->err, cudaStreamWaitEvent(sd, h->ev0, 0));
    StreamedLaunch sl;
    sl.ready = h->d_ready;
    sl.done = h->d_done;
    sl.host_done = h->d_hdone;
    sl.n_chunks = nchunks;
    for (int c = 0; c <= pqp_handle::kStreams; ++c) sl.chunk_lo[c] = c <= nchunks ? lo_of[c] : B;
    // The chunk copies are queued BEFORE the launch: they are asynchronous (pinned buffers), so the
    // kernel still overlaps them, and a tool that makes launches blocking (ncu serialises kernels)
    // cannot leave the kernel waiting for copies the host has not issued yet.
    for (int c = 0; c < nchunks; ++c) {
        const int lo = lo_of[c];
        PQP_CUDA(h->err, pqp::copy_batch(dev_in, lo, *in, lo, lo_of[c + 1] - lo, nmax, cudaMemcpyHostToDevice, sc));
        PQP_CUDA(h->err, cudaMemsetAsync(h->d_ready + c, 1, sizeof(int), sc));  // "chunk c has landed"
    }
    int rc = run_device(h, &dev_in, &dev_out, mode, sk, false, 0, false, h->d_flags, &sl);
    if (rc) return rc;
    h->host_inputs_resident = true;
    for (int c = 0; c < nchunks; ++c) {
        const int lo = lo_of[c], hi = lo_of[c + 1];
        const size_t nb = (size_t)(hi - lo);
        // wait until the kernel announces the chunk (or has ended, e.g. after an error)
        // (short spin, then 20 us naps: a chunk takes ~ a millisecond, and a caller that drives several handles
        // from several threads must not burn a core per handle)
        volatile int *flag = h->h_done + c;
        for (unsigned spin = 0; *flag == 0; ++spin) {
            if (spin < 4096) continue;
            if ((spin & 0x3f) == 0 && cudaStreamQuery(sk) != cudaErrorNotReady) break;
            const struct timespec nap = {0, 20000};
            nanosleep(&nap, nullptr);
        }
        PQP_CUDA(h->err, cudaMemcpyAsync(h->h_status + lo, h->d_status + lo, nb * sizeof(int), cudaMemcpyDeviceToHost, sd));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->h_flags + lo, h->d_flags + lo, nb * sizeof(int), cudaMemcpyDeviceToHost, sd));
        PQP_CUDA(h->err, pqp::copy_batch(*out, lo, dev_out, lo, nb, nmax, cudaMemcpyDeviceToHost, sd));
    }
    h->last_batch = B;
    PQP_CUDA(h->err, cudaStreamSynchronize(sk));
    PQP_CUDA(h->err, cudaStreamSynchronize(sc));
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, sd));
    PQP_CUDA(h->err, cudaStreamSynchronize(sd));
    PQP_CUDA(h->err, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    for (int i = 0; i < PQP_NSTAGES; ++i) h->stage_ms[i] = -1.0f;  // copies and kernel overlap: only the total is defined
    h->stage_ms[PQP_STAGE_TOTAL] = h->last_ms;
    if (!h->fp64 && h->escalate && mode == 0) return escalate_fp64(h, dev_in, out, B);
    return PQP_OK;
}

// staging of the host-pointer pqp_frenet_to_cartesian, all or nothing (allocated on its first call)
cudaError_t alloc_frenet_staging(pqp_handle *h) {
    const size_t B = h->batch_max, nm = h->n_max;
    pqp::Resources &r = h->res;
    return r.group([&] {
        cudaError_t e = r.alloc(h->d_ref, B * 3 * nm);
        if (e == cudaSuccess) e = r.alloc(h->d_xy, B * 3 * nm);
        if (e == cudaSuccess) e = r.alloc(h->d_sol2, B * 4 * nm);
        if (e == cudaSuccess) e = r.alloc(h->d_n2, B);
        return e;
    });
}

int run_host(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out, int mode) {
    int rc;
    const int nmax = h->n_max;
    cudaStream_t s = h->stream;
    DeviceGuard guard_(h->device);
    int B;
    if (in) {
        rc = validate_batch(h, in, out);
        if (rc) return rc;
        B = in->batch;
        for (int b = 0; b < B; ++b) {
            if (in->n[b] < 2 || in->n[b] > nmax) return fail(h->err, PQP_E_INVALID, "n[b] must be in [2, n_max]");
            if (in->p && (in->p[b] < 0 || in->p[b] > in->n[b])) return fail(h->err, PQP_E_INVALID, "p[b] must be in [0, n[b]]");
        }
        if (mode == 1 && h->cold_only) return fail(h->err, PQP_E_STATE, "cold-only handle (option bit 128) keeps no warm state");
        if (mode == 1 && (!h->solved || B != h->last_batch)) return fail(h->err, PQP_E_STATE, "resolve needs a previous solve of the same batch");
        h->host_inputs_resident = true;
        h->d_p_valid = in->p != nullptr;
    } else {
        if (mode != 1) return fail(h->err, PQP_E_INVALID, "null batch");
        if (h->cold_only) return fail(h->err, PQP_E_STATE, "cold-only handle (option bit 128) keeps no warm state");
        if (!out || !out->sol) return fail(h->err, PQP_E_INVALID, "null output");
        if (!h->solved || !h->host_inputs_resident) return fail(h->err, PQP_E_STATE, "resolve(NULL) needs a previous host-API solve");
        B = h->last_batch;
        const int threads = 256, blocks = (B * nmax + threads - 1) / threads;
        relinearise_kernel<<<blocks, threads, 0, s>>>(B, nmax, h->d_sol, h->d_knots);
        PQP_CUDA(h->err, cudaGetLastError());
        h->launches++;
    }
    // optional full outputs are allocated on first use
    const auto batch_of = [&](auto member) { return (size_t)h->batch_max * pqp::per_instance(member, nmax); };
    if (out->x_full && !h->d_xf) PQP_CUDA(h->err, h->res.alloc(h->d_xf, batch_of(&pqp_batch_out::x_full)));
    if (out->y_full && !h->d_yf) PQP_CUDA(h->err, h->res.alloc(h->d_yf, batch_of(&pqp_batch_out::y_full)));
    if (out->z_full && !h->d_zf) PQP_CUDA(h->err, h->res.alloc(h->d_zf, batch_of(&pqp_batch_out::z_full)));
    // the handle's device buffers as one batch: inputs, outputs, and the requested full outputs alone (zeroed before a
    // solve: the kernel writes an instance's first nv / m entries only)
    const pqp_batch_in dev_in = {B, nmax, h->d_knots, h->d_inst, h->d_n, h->d_p_valid ? h->d_p : nullptr};
    const pqp_batch_out dev_full = {nullptr, nullptr, nullptr, nullptr, out->x_full ? h->d_xf : nullptr,
                                    out->y_full ? h->d_yf : nullptr, out->z_full ? h->d_zf : nullptr, nullptr};
    const pqp_batch_out dev_out = {h->d_sol,         h->d_cost,       h->d_status,     h->d_iters,
                                   dev_full.x_full, dev_full.y_full, dev_full.z_full, h->d_info};
    if (in && h->persistent && B >= 512) return run_host_streamed(h, in, out, dev_in, dev_out, dev_full, mode, B);
    // Chunked pipeline, one stream per chunk: chunk c+1's H2D copy and chunk c-1's D2H copy
    // overlap chunk c's kernel (fully asynchronous when the caller's buffers are pinned), and
    // because every chunk's kernel sits in its own stream the block scheduler back-fills SMs
    // from the next chunk as soon as its inputs have landed (no partial-wave bubble between
    // chunks). Scratch slots are addressed by the instance's index in the whole batch (qp0),
    // so chunking is invisible to the warm state.
    const int kMinChunk = 1024;
    int nchunks = (B + kMinChunk - 1) / kMinChunk;
    if (nchunks > pqp_handle::kStreams) nchunks = pqp_handle::kStreams;
    if (nchunks < 1) nchunks = 1;
    const int per = (B + nchunks - 1) / nchunks;
    cudaStream_t *streams = h->streams;
    // every chunk stream starts after whatever the handle's main stream has queued so far
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, streams[0]));
    for (int c = 1; c < nchunks; ++c) PQP_CUDA(h->err, cudaStreamWaitEvent(streams[c], h->ev0, 0));
    for (int c = 0; c < nchunks; ++c) {
        const int lo = c * per, hi = (lo + per < B) ? lo + per : B;
        if (lo >= hi) break;
        const size_t nb = (size_t)(hi - lo);
        cudaStream_t s = streams[c];
        if (in) PQP_CUDA(h->err, pqp::copy_batch(dev_in, lo, *in, lo, nb, nmax, cudaMemcpyHostToDevice, s));
        PQP_CUDA(h->err, pqp::zero_batch(dev_full, lo, nb, nmax, s));
        if (nchunks == 1) PQP_CUDA(h->err, cudaEventRecord(h->ev_st[0], s));
        pqp_batch_in din = pqp::batch_from(dev_in, lo, nmax);
        din.batch = (int32_t)nb;
        const pqp_batch_out dout = pqp::batch_from(dev_out, lo, nmax);
        rc = run_device(h, &din, &dout, mode, s, false, lo, false, h->d_flags + lo);
        if (rc) return rc;
        if (nchunks == 1) PQP_CUDA(h->err, cudaEventRecord(h->ev_st[1], s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->h_status + lo, dout.status, nb * sizeof(int), cudaMemcpyDeviceToHost, s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->h_flags + lo, h->d_flags + lo, nb * sizeof(int), cudaMemcpyDeviceToHost, s));
        PQP_CUDA(h->err, pqp::copy_batch(*out, lo, dev_out, lo, nb, nmax, cudaMemcpyDeviceToHost, s));
    }
    h->last_batch = B;
    // join: stream[0] waits for every chunk stream; ev1 marks the end of the whole pipeline
    for (int c = 1; c < nchunks; ++c) {
        PQP_CUDA(h->err, cudaEventRecord(h->evs[c], streams[c]));
        PQP_CUDA(h->err, cudaStreamWaitEvent(streams[0], h->evs[c], 0));
    }
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, streams[0]));
    PQP_CUDA(h->err, cudaStreamSynchronize(streams[0]));
    PQP_CUDA(h->err, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    // per-stage device times of a single-stream call (the reference's TimeRecorder stages of
    // BaseSolver::solve, base_solver.cpp:57-93; here cost / constraints / solver set-up / ADMM are one kernel)
    for (int i = 0; i < PQP_NSTAGES; ++i) h->stage_ms[i] = -1.0f;
    if (nchunks == 1) {
        PQP_CUDA(h->err, cudaEventElapsedTime(&h->stage_ms[PQP_STAGE_H2D], h->ev0, h->ev_st[0]));
        PQP_CUDA(h->err, cudaEventElapsedTime(&h->stage_ms[PQP_STAGE_KERNEL], h->ev_st[0], h->ev_st[1]));
        PQP_CUDA(h->err, cudaEventElapsedTime(&h->stage_ms[PQP_STAGE_D2H], h->ev_st[1], h->ev1));
    }
    h->stage_ms[PQP_STAGE_TOTAL] = h->last_ms;
    h->stage_ms[PQP_STAGE_ESCALATION] = 0.0f;
    // cold solves only: the FP64 re-solve starts cold, which is not what a warm re-solve under an iteration
    // cap (receding horizon) is; the increment-form kernel certifies infeasibility by itself there
    if (!h->fp64 && h->escalate && mode == 0) {
        PQP_CUDA(h->err, cudaEventRecord(h->ev_st[2], streams[0]));
        rc = escalate_fp64(h, dev_in, out, B);
        if (rc) return rc;
        PQP_CUDA(h->err, cudaEventRecord(h->ev_st[3], streams[0]));
        PQP_CUDA(h->err, cudaEventSynchronize(h->ev_st[3]));
        PQP_CUDA(h->err, cudaEventElapsedTime(&h->stage_ms[PQP_STAGE_ESCALATION], h->ev_st[2], h->ev_st[3]));
    }
    return PQP_OK;
}

}  // namespace

// ------------------------------------------------------------------ C ABI
extern "C" {

int pqp_version(void) { return PQP_VERSION; }

int pqp_default_params(pqp_params *params) {
    if (!params) return PQP_E_INVALID;
    pqp::default_params(params);
    return PQP_OK;
}

const char *pqp_last_error(const pqp_handle *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int pqp_create(const pqp_params *params, int32_t n_max, int32_t batch_max, int32_t device,
               pqp_handle **out) {
    if (!out) return fail(g_create_error, PQP_E_INVALID, "out is null");
    *out = nullptr;
    if (!params || !pqp::params_valid(*params)) return fail(g_create_error, PQP_E_INVALID, "invalid params");
    if (n_max < 2 || n_max > 32 * pqp::kMaxChunk - 1) return fail(g_create_error, PQP_E_INVALID, "n_max must be in [2, 511]");
    if (batch_max < 1) return fail(g_create_error, PQP_E_INVALID, "batch_max must be >= 1");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(g_create_error, PQP_E_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(g_create_error, PQP_E_NO_DEVICE, "device index out of range");
    cudaDeviceProp prop;
    PQP_CUDA(g_create_error, cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(g_create_error, PQP_E_NO_DEVICE, "this library is built for sm_90a (H100) only; found sm_" +
                                                  std::to_string(prop.major) + std::to_string(prop.minor));
    pqp_handle *h = new (std::nothrow) pqp_handle;
    if (!h) return fail(g_create_error, PQP_E_INVALID, "out of host memory");
    h->prm = *params;
    h->n_max = n_max;
    h->batch_max = batch_max;
    h->device = h->res.device = device;
    h->chunk = pqp::chunk_for(n_max);
    h->sm_count = prop.multiProcessorCount;
    h->smem_bytes = pqp::smem_floats(h->chunk) * sizeof(float) + 16;
    DeviceGuard guard_(device);
    const int rc = [&]() -> int {
        h->fp64 = (params->reserved & 2) != 0;
        h->escalate = (params->reserved & 4) == 0;
        h->cold_only = (params->reserved & 128) != 0;
        // launch of the FP32 kernel (measured on H100, 8192 instances, DESIGN.md §5): persistent (work counter, one
        // streamed launch per host call) for n_max >= 128, where three QPs fill an SM's shared memory (n = 240: 0.5-1 %
        // ahead); one CTA per instance below (n = 120: 2.7 % ahead, n = 60: equal). Both keep the state in shared
        // memory. Bits 8 / 16 force one or the other.
        const bool auto_persistent = h->chunk >= 8;
        h->persistent = !h->fp64 && ((params->reserved & 8) != 0 || (auto_persistent && (params->reserved & 16) == 0));
        // form of the ADMM step (FP32 kernels): the increment form (dx solve, row values A x carried and
        // advanced by alpha A dx) follows the FP64 oracle's rho schedule - the same iteration count in almost
        // every instance, fewer iterations on average - for a few per cent more work per iteration. Default:
        // increment form for n_max >= 64, textbook form below; bits 32 / 64 force one or the other.
        h->incr = !h->fp64 && ((params->reserved & 32) != 0 || ((params->reserved & 64) == 0 && h->chunk >= 4));
        h->smem_bytes64 = pqp::smem_floats(h->chunk) * sizeof(double) + 16;
        h->kernel = select_kernel(h->chunk, h->fp64, h->incr, h->persistent);
        h->kernel64 = select_kernel(h->chunk, true, false, false);
        h->prepared64 = h->fp64;
        int bps = 0;
        PQP_CUDA(g_create_error, prepare(h->kernel, h->fp64 ? h->smem_bytes64 : h->smem_bytes, &bps));
        if (bps < 1) return fail(g_create_error, PQP_E_CUDA, "the solve kernel does not fit on an SM");
        h->warps_per_sm = bps;
        pqp::Resources &r = h->res;
        for (int i = 0; i < pqp_handle::kStreams; ++i) {
            PQP_CUDA(g_create_error, r.stream(h->streams[i]));
            PQP_CUDA(g_create_error, r.event(h->evs[i], cudaEventDisableTiming));
        }
        h->stream = h->streams[0];
        PQP_CUDA(g_create_error, r.event(h->ev0));
        PQP_CUDA(g_create_error, r.event(h->ev1));
        const size_t B = batch_max, c = h->chunk;
        const auto batch_of = [&](auto member) { return B * pqp::per_instance(member, n_max); };
        PQP_CUDA(g_create_error, r.alloc(h->d_knots, batch_of(&pqp_batch_in::knots)));
        PQP_CUDA(g_create_error, r.alloc(h->d_inst, batch_of(&pqp_batch_in::inst)));
        PQP_CUDA(g_create_error, r.alloc(h->d_n, batch_of(&pqp_batch_in::n)));
        PQP_CUDA(g_create_error, r.alloc(h->d_p, batch_of(&pqp_batch_in::p)));
        PQP_CUDA(g_create_error, r.alloc(h->d_sol, batch_of(&pqp_batch_out::sol)));
        PQP_CUDA(g_create_error, r.alloc(h->d_cost, batch_of(&pqp_batch_out::cost)));
        PQP_CUDA(g_create_error, r.alloc(h->d_status, batch_of(&pqp_batch_out::status)));
        PQP_CUDA(g_create_error, r.alloc(h->d_iters, batch_of(&pqp_batch_out::iters)));
        PQP_CUDA(g_create_error, r.alloc(h->d_info, batch_of(&pqp_batch_out::info)));
        const size_t esz = h->fp64 ? sizeof(double) : sizeof(float);
        // Warm state (scaled x, z, y and rho: the OSQP workspace that persists between solve and
        // updateProblemFormulationAndSolve) is per instance; a cold-only handle keeps none. The Ruiz
        // factors and delta_y are scratch of one solve: per instance under the one-CTA-per-instance
        // launch, per resident warp under the persistent launch.
        if (!h->cold_only) {
            PQP_CUDA(g_create_error, r.alloc(h->d_warm, B * pqp::warm_floats(c) * esz));
            PQP_CUDA(g_create_error, cudaMemset(h->d_warm, 0, B * pqp::warm_floats(c) * esz));
            PQP_CUDA(g_create_error, r.alloc(h->d_rho, B * esz));
        }
        const size_t slots = h->persistent ? (size_t)h->sm_count * h->warps_per_sm : B;
        PQP_CUDA(g_create_error, r.alloc(h->d_scal, slots * pqp::scal_floats(c) * esz));
        PQP_CUDA(g_create_error, r.alloc(h->d_dy, slots * pqp::dy_floats(c) * esz));
        for (int i = 0; i < 4; ++i) PQP_CUDA(g_create_error, r.event(h->ev_st[i]));
        PQP_CUDA(g_create_error, r.alloc(h->d_counters, (size_t)pqp_handle::kCounters));
        PQP_CUDA(g_create_error, r.alloc(h->d_ready, (size_t)pqp_handle::kStreams));
        PQP_CUDA(g_create_error, r.alloc(h->d_done, (size_t)pqp_handle::kStreams));
        PQP_CUDA(g_create_error, r.alloc_host(h->h_done, (size_t)pqp_handle::kStreams, cudaHostAllocMapped));
        PQP_CUDA(g_create_error, cudaHostGetDevicePointer(reinterpret_cast<void **>(&h->d_hdone), h->h_done, 0));
        PQP_CUDA(g_create_error, r.alloc(h->d_flags, B));
        PQP_CUDA(g_create_error, cudaMemset(h->d_flags, 0, B * sizeof(int)));
        PQP_CUDA(g_create_error, r.alloc_host(h->h_status, B));
        PQP_CUDA(g_create_error, r.alloc_host(h->h_flags, B));
        PQP_CUDA(g_create_error, cudaMemset(h->d_sol, 0, batch_of(&pqp_batch_out::sol) * sizeof(double)));
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_destroy(h);
        return rc;
    }
    *out = h;
    return PQP_OK;
}

int pqp_destroy(pqp_handle *h) {
    if (!h) return PQP_OK;
    DeviceGuard guard_(h->device);
    for (int i = 0; i < pqp_handle::kStreams; ++i) if (h->streams[i]) cudaStreamSynchronize(h->streams[i]);
    delete h;
    return PQP_OK;
}

int pqp_solve(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in) return fail(h->err, PQP_E_INVALID, "null batch");
    return run_host(h, in, out, 0);
}

int pqp_resolve(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out) {
    if (!h) return PQP_E_INVALID;
    return run_host(h, in, out, 1);
}

int pqp_solve_device(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out, void *stream) {
    int rc = validate_batch(h, in, out);
    if (rc) return rc;
    DeviceGuard guard_(h->device);
    h->host_inputs_resident = false;
    return run_device(h, in, out, 0, static_cast<cudaStream_t>(stream), false);
}

int pqp_resolve_device(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out, void *stream) {
    int rc = validate_batch(h, in, out);
    if (rc) return rc;
    if (h->cold_only) return fail(h->err, PQP_E_STATE, "cold-only handle (option bit 128) keeps no warm state");
    if (!h->solved || in->batch != h->last_batch) return fail(h->err, PQP_E_STATE, "resolve needs a previous solve of the same batch");
    DeviceGuard guard_(h->device);
    return run_device(h, in, out, 1, static_cast<cudaStream_t>(stream), false);
}

int pqp_frenet_to_cartesian_device(pqp_handle *h, int32_t batch, const int32_t *n, const double *ref_xyh,
                                   const double *sol, double *out_xyh, void *stream) {
    if (!h) return PQP_E_INVALID;
    if (!n || !ref_xyh || !sol || !out_xyh || batch < 1) return fail(h->err, PQP_E_INVALID, "null buffer");
    DeviceGuard guard_(h->device);
    const int threads = 256, blocks = (batch * h->n_max + threads - 1) / threads;
    frenet_to_cartesian_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(batch, h->n_max, n, ref_xyh, sol, out_xyh);
    PQP_CUDA(h->err, cudaGetLastError());
    h->launches++;
    return PQP_OK;
}

int pqp_relinearise_device(pqp_handle *h, int32_t batch, const double *sol, double *knots, void *stream) {
    if (!h) return PQP_E_INVALID;
    if (!sol || !knots || batch < 1) return fail(h->err, PQP_E_INVALID, "null buffer");
    DeviceGuard guard_(h->device);
    const int threads = 256, blocks = (batch * h->n_max + threads - 1) / threads;
    relinearise_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(batch, h->n_max, sol, knots);
    PQP_CUDA(h->err, cudaGetLastError());
    h->launches++;
    return PQP_OK;
}

int pqp_advance_window_device(pqp_handle *h, int32_t batch, int32_t ext_len, int32_t tick, const double *ext_knots,
                              const double *sol, double *knots, double *inst, void *stream) {
    if (!h) return PQP_E_INVALID;
    if (!ext_knots || !sol || !knots || !inst || batch < 1) return fail(h->err, PQP_E_INVALID, "null buffer");
    if (tick < 0 || tick + h->n_max > ext_len) return fail(h->err, PQP_E_INVALID, "window [tick, tick + n_max) leaves the extended reference");
    DeviceGuard guard_(h->device);
    const int threads = 256, blocks = (batch * h->n_max + threads - 1) / threads;
    advance_window_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(batch, h->n_max, ext_len, tick, ext_knots, sol,
                                                                                   knots, inst);
    PQP_CUDA(h->err, cudaGetLastError());
    h->launches++;
    return PQP_OK;
}

int pqp_frenet_to_cartesian(pqp_handle *h, int32_t batch, const int32_t *n, const double *ref_xyh,
                            const double *sol, double *out_xyh) {
    if (!h) return PQP_E_INVALID;
    if (!n || !ref_xyh || !sol || !out_xyh || batch < 1 || batch > h->batch_max) return fail(h->err, PQP_E_INVALID, "bad arguments");
    DeviceGuard guard_(h->device);
    const size_t B = batch, nm = h->n_max;
    if (!h->d_ref) PQP_CUDA(h->err, alloc_frenet_staging(h));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_ref, ref_xyh, B * 3 * nm * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_sol2, sol, B * 4 * nm * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_n2, n, B * sizeof(int), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_xy, 0, B * 3 * nm * sizeof(double), s));
    int rc = pqp_frenet_to_cartesian_device(h, batch, h->d_n2, h->d_ref, h->d_sol2, h->d_xy, s);
    if (rc) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out_xyh, h->d_xy, B * 3 * nm * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

int pqp_last_kernel_ms(pqp_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    *ms = h->last_ms;
    return PQP_OK;
}

int pqp_pack_results_device(pqp_handle *h, int32_t batch, const double *cost, const int32_t *status,
                            const int32_t *iters, pqp_result_rec *packed, void *stream) {
    if (!h) return PQP_E_INVALID;
    if (!cost || !status || !iters || !packed || batch < 1) return fail(h->err, PQP_E_INVALID, "null buffer");
    DeviceGuard guard_(h->device);
    pack_results_kernel<<<(batch + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(batch, cost, status, iters, packed);
    PQP_CUDA(h->err, cudaGetLastError());
    h->launches++;
    return PQP_OK;
}

int pqp_resident_results(pqp_handle *h, const double **sol, const double **cost, const int32_t **status,
                         const int32_t **iters) {
    if (!h) return PQP_E_INVALID;
    if (!h->solved || !h->host_inputs_resident) return fail(h->err, PQP_E_STATE, "no host-pointer solve has run on this handle");
    if (sol) *sol = h->d_sol;
    if (cost) *cost = h->d_cost;
    if (status) *status = h->d_status;
    if (iters) *iters = h->d_iters;
    return PQP_OK;
}

int pqp_last_stage_ms(pqp_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    for (int i = 0; i < PQP_NSTAGES; ++i) ms[i] = h->stage_ms[i];
    return PQP_OK;
}

int pqp_launch_count(pqp_handle *h, int64_t *count) {
    if (!h || !count) return PQP_E_INVALID;
    *count = h->launches;
    return PQP_OK;
}

int pqp_kernel_info(pqp_handle *h, int32_t *sm_count, int32_t *warps_per_sm, int32_t *smem_per_warp) {
    if (!h) return PQP_E_INVALID;
    if (sm_count) *sm_count = h->sm_count;
    if (warps_per_sm) *warps_per_sm = h->warps_per_sm;
    if (smem_per_warp) *smem_per_warp = (int32_t)h->smem_bytes;
    return PQP_OK;
}

}  // extern "C"
