// pqp_multi.cu — include/pqp_multi.h: one process, the GPUs of one box, contiguous shards, one
// ncclAllGather of 16 B per instance. Built on the public single-device ABI (pqp.h) only.
//
// NCCL is bound at run time (dlopen): no link-time dependency, and a process that already carries a
// libnccl.so.2 (torch's) shares it.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "../../include/pqp_multi.h"
#include "pqp_batch_layout.h"
#include "pqp_host_handle.h"
#include "pqp_shard.h"

namespace {

thread_local std::string g_multi_create_error;

// the handful of NCCL entry points this file uses (signatures of nccl.h 2.x; ncclInt8 == 0)
typedef struct ncclComm *ncclComm_t;
struct Nccl {
    void *lib = nullptr;
    int (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool load(std::string *err) {
        if (lib) return true;
        for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
            lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (lib) break;
        }
        if (!lib) {
            *err = std::string("cannot load NCCL: ") + dlerror();
            return false;
        }
        CommInitAll = reinterpret_cast<decltype(CommInitAll)>(dlsym(lib, "ncclCommInitAll"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
        AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(lib, "ncclAllGather"));
        GroupStart = reinterpret_cast<decltype(GroupStart)>(dlsym(lib, "ncclGroupStart"));
        GroupEnd = reinterpret_cast<decltype(GroupEnd)>(dlsym(lib, "ncclGroupEnd"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
        if (!CommInitAll || !CommDestroy || !AllGather || !GroupStart || !GroupEnd || !GetErrorString) {
            *err = "libnccl.so.2 lacks an expected symbol";
            return false;
        }
        return true;
    }
};
Nccl &nccl() {
    static Nccl n;
    return n;
}

}  // namespace

struct pqp_multi {
    int n_dev = 0, n_max = 0, batch_max = 0, per_max = 0;
    std::vector<int> dev;
    std::vector<pqp_handle *> h;
    std::vector<cudaStream_t> stream;
    std::vector<cudaEvent_t> ev0, ev1;
    std::vector<pqp_result_rec *> d_send, d_table;  // per device: its packed shard / the gathered table
    std::vector<ncclComm_t> comm;
    int last_batch = 0, last_per = 0;
    float gather_ms = 0.0f;
    std::string err;
    std::vector<pqp::Resources> res;  // one per device; last member: releasing clears the members above
};

namespace {

using pqp::fail;

int run(pqp_multi *m, const pqp_batch_in *in, const pqp_batch_out *out, bool warm) {
    if (!m) return PQP_E_INVALID;
    if (!out || !out->sol) return fail(m->err, PQP_E_INVALID, "null output");
    int B;
    if (in) {
        if (!in->knots || !in->inst || !in->n) return fail(m->err, PQP_E_INVALID, "null buffer");
        if (in->batch < 1 || in->batch > m->batch_max) return fail(m->err, PQP_E_INVALID, "batch out of range");
        if (in->n_max != m->n_max) return fail(m->err, PQP_E_INVALID, "n_max differs from the handle's");
        B = in->batch;
    } else {
        if (!warm) return fail(m->err, PQP_E_INVALID, "null batch");
        B = m->last_batch;
        if (B < 1) return fail(m->err, PQP_E_STATE, "resolve(NULL) needs a previous solve");
    }
    if (warm && B != m->last_batch) return fail(m->err, PQP_E_STATE, "resolve needs a previous solve of the same batch");
    const int G = m->n_dev, nmax = m->n_max;
    const int per = pqp::shard_per(B, G);
    std::vector<int> rc(G, PQP_OK);
    // one host thread per device: each runs that device's own (pipelined, synchronous) host call
    pqp::fan_out(G, [&](int d) {
        const pqp::Shard sh = pqp::shard_of(B, per, d);
        const int lo = sh.first, hi = sh.first + sh.count;
        if (lo >= hi) return;
        pqp_batch_in din = in ? pqp::batch_from(*in, lo, nmax) : pqp_batch_in{};
        din.batch = hi - lo;
        const pqp_batch_out dout = pqp::batch_from(*out, lo, nmax);
        rc[d] = warm ? pqp_resolve(m->h[d], in ? &din : nullptr, &dout) : pqp_solve(m->h[d], &din, &dout);
    });
    for (int d = 0; d < G; ++d)
        if (rc[d] != PQP_OK) return fail(m->err, rc[d], std::string("device ") + std::to_string(m->dev[d]) + ": " + pqp_last_error(m->h[d]));
    m->last_batch = B;
    m->last_per = per;
    // pack on every device, then one all-gather of per * 16 bytes per device
    for (int d = 0; d < G; ++d) {
        pqp::DeviceGuard g(m->dev[d]);
        const pqp::Shard sh = pqp::shard_of(B, per, d);
        const int lo = sh.first, hi = sh.first + sh.count;
        cudaEventRecord(m->ev0[d], m->stream[d]);
        cudaMemsetAsync(m->d_send[d], 0, (size_t)per * sizeof(pqp_result_rec), m->stream[d]);
        if (hi > lo) {
            const double *cost;
            const int32_t *status, *iters;
            int r = pqp_resident_results(m->h[d], nullptr, &cost, &status, &iters);
            if (r == PQP_OK) r = pqp_pack_results_device(m->h[d], hi - lo, cost, status, iters, m->d_send[d], m->stream[d]);
            if (r != PQP_OK) return fail(m->err, r, pqp_last_error(m->h[d]));
        }
    }
    if (G == 1) {
        pqp::DeviceGuard g(m->dev[0]);
        cudaMemcpyAsync(m->d_table[0], m->d_send[0], (size_t)per * sizeof(pqp_result_rec), cudaMemcpyDeviceToDevice, m->stream[0]);
    } else {
        Nccl &N = nccl();
        int e = N.GroupStart();
        for (int d = 0; d < G && e == 0; ++d)
            e = N.AllGather(m->d_send[d], m->d_table[d], (size_t)per * sizeof(pqp_result_rec), /*ncclInt8*/ 0, m->comm[d], m->stream[d]);
        const int e2 = N.GroupEnd();
        if (e == 0) e = e2;
        if (e != 0) return fail(m->err, PQP_E_CUDA, std::string("ncclAllGather: ") + N.GetErrorString(e));
    }
    float worst = 0.0f;
    for (int d = 0; d < G; ++d) {
        pqp::DeviceGuard g(m->dev[d]);
        cudaEventRecord(m->ev1[d], m->stream[d]);
        PQP_CUDA(m->err, cudaStreamSynchronize(m->stream[d]));
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, m->ev0[d], m->ev1[d]);
        worst = std::max(worst, ms);
    }
    m->gather_ms = worst;
    return PQP_OK;
}

}  // namespace

extern "C" {

const char *pqp_multi_last_error(const pqp_multi *m) { return m ? m->err.c_str() : g_multi_create_error.c_str(); }

int pqp_multi_create(const pqp_params *params, int32_t n_max, int32_t batch_max, int32_t n_devices,
                     const int32_t *devices, pqp_multi **out) {
    std::string &err = g_multi_create_error;
    if (!out) return fail(err, PQP_E_INVALID, "out is null");
    *out = nullptr;
    if (!params || n_devices < 1 || batch_max < 1) return fail(err, PQP_E_INVALID, "invalid arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < n_devices)
        return fail(err, PQP_E_NO_DEVICE, "fewer CUDA devices than n_devices (there is no CPU fallback)");
    if (n_devices > 1 && !nccl().load(&g_multi_create_error)) return PQP_E_NO_DEVICE;
    pqp_multi *m = new (std::nothrow) pqp_multi;
    if (!m) return fail(err, PQP_E_INVALID, "out of host memory");
    m->n_dev = n_devices;
    m->n_max = n_max;
    m->batch_max = batch_max;
    m->per_max = (batch_max + n_devices - 1) / n_devices;
    const size_t G = n_devices;
    m->dev.resize(G);
    m->h.assign(G, nullptr);
    m->stream.assign(G, nullptr);
    m->ev0.assign(G, nullptr);
    m->ev1.assign(G, nullptr);
    m->d_send.assign(G, nullptr);
    m->d_table.assign(G, nullptr);
    m->comm.assign(G, nullptr);
    m->res = std::vector<pqp::Resources>(G);
    for (int d = 0; d < n_devices; ++d) m->dev[d] = m->res[d].device = devices ? devices[d] : d;
    const int rc = [&]() -> int {
        for (int d = 0; d < n_devices; ++d) {
            const int hrc = pqp_create(params, n_max, m->per_max, m->dev[d], &m->h[d]);
            if (hrc != PQP_OK) return fail(err, hrc, pqp_last_error(nullptr));
            pqp::DeviceGuard g(m->dev[d]);
            pqp::Resources &r = m->res[d];
            PQP_CUDA(err, r.stream(m->stream[d]));
            PQP_CUDA(err, r.event(m->ev0[d]));
            PQP_CUDA(err, r.event(m->ev1[d]));
            PQP_CUDA(err, r.alloc(m->d_send[d], (size_t)m->per_max));
            PQP_CUDA(err, r.alloc(m->d_table[d], G * m->per_max));
        }
        if (n_devices > 1) {
            const int e = nccl().CommInitAll(m->comm.data(), n_devices, m->dev.data());
            if (e != 0) {
                for (auto &c : m->comm) c = nullptr;
                return fail(err, PQP_E_CUDA, std::string("ncclCommInitAll: ") + nccl().GetErrorString(e));
            }
        }
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_multi_destroy(m);
        return rc;
    }
    *out = m;
    return PQP_OK;
}

int pqp_multi_destroy(pqp_multi *m) {
    if (!m) return PQP_OK;
    for (int d = 0; d < m->n_dev; ++d) {
        pqp::DeviceGuard g(m->dev[d]);
        if (m->stream[d]) cudaStreamSynchronize(m->stream[d]);
        if (m->comm[d]) nccl().CommDestroy(m->comm[d]);
        if (m->h[d]) pqp_destroy(m->h[d]);
    }
    delete m;
    return PQP_OK;
}

int pqp_multi_solve(pqp_multi *m, const pqp_batch_in *in, const pqp_batch_out *out) {
    if (!m) return PQP_E_INVALID;
    if (!in) return fail(m->err, PQP_E_INVALID, "null batch");
    return run(m, in, out, false);
}

int pqp_multi_resolve(pqp_multi *m, const pqp_batch_in *in, const pqp_batch_out *out) { return run(m, in, out, true); }

int pqp_multi_gathered(pqp_multi *m, int32_t i, const pqp_result_rec **table, int32_t *per) {
    if (!m || i < 0 || i >= m->n_dev) return PQP_E_INVALID;
    if (m->last_batch < 1) return fail(m->err, PQP_E_STATE, "nothing solved yet");
    if (table) *table = m->d_table[i];
    if (per) *per = m->last_per;
    return PQP_OK;
}

int pqp_multi_shard(pqp_multi *m, int32_t i, int32_t *first, int32_t *count) {
    if (!m || i < 0 || i >= m->n_dev) return PQP_E_INVALID;
    const pqp::Shard sh = pqp::shard_of(m->last_batch, m->last_per, i);
    if (first) *first = sh.first;
    if (count) *count = sh.count;
    return PQP_OK;
}

int pqp_multi_handle(pqp_multi *m, int32_t i, pqp_handle **h) {
    if (!m || !h || i < 0 || i >= m->n_dev) return PQP_E_INVALID;
    *h = m->h[i];
    return PQP_OK;
}

int pqp_multi_last_gather_ms(pqp_multi *m, float *ms) {
    if (!m || !ms) return PQP_E_INVALID;
    *ms = m->gather_ms;
    return PQP_OK;
}

}  // extern "C"
