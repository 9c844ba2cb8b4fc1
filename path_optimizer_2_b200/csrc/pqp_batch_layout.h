// pqp_batch_layout.h — the layout of a solver batch (include/pqp.h): every pointer member of pqp_batch_in and
// pqp_batch_out with the elements it holds per instance, for a handle of n_max knots. A NULL member is one the caller
// did not request; every routine here skips it. The solver's host calls stage, zero and slice their batches through
// it, the multi-device solver shards with it and the plan sizes its traced full outputs with it. The table and the
// slicing are host code that g++ compiles; the copies and the zeroing need the CUDA runtime.
#pragma once
#include <array>
#include <cstddef>
#include <cstdint>
#include <cstring>

#include "../../include/pqp.h"

namespace pqp {

struct BatchField {
    size_t offset;  // offsetof(struct, member)
    size_t count;   // elements of one instance
    size_t size;    // bytes of one element
    size_t bytes() const { return count * size; }
};

// The members of pqp_batch_in and of pqp_batch_out, each once. Every copy and zeroing of a batch runs in this order.
inline std::array<BatchField, 4> batch_fields(const pqp_batch_in *, size_t n_max) {
    const size_t d = sizeof(double), i4 = sizeof(int32_t);
    return {{{offsetof(pqp_batch_in, knots), PQP_NFIELDS * n_max, d},
             {offsetof(pqp_batch_in, inst), PQP_NINST, d},
             {offsetof(pqp_batch_in, n), 1, i4},
             {offsetof(pqp_batch_in, p), 1, i4}}};
}
inline std::array<BatchField, 8> batch_fields(const pqp_batch_out *, size_t n_max) {
    const size_t d = sizeof(double), i4 = sizeof(int32_t);
    return {{{offsetof(pqp_batch_out, sol), 4 * n_max, d},
             {offsetof(pqp_batch_out, cost), 1, d},
             {offsetof(pqp_batch_out, status), 1, i4},
             {offsetof(pqp_batch_out, iters), 1, i4},
             {offsetof(pqp_batch_out, info), PQP_NINFO, d},
             {offsetof(pqp_batch_out, x_full), 6 * n_max - 1, d},   // nv_max
             {offsetof(pqp_batch_out, y_full), 6 * n_max + 2, d},   // m_max
             {offsetof(pqp_batch_out, z_full), 6 * n_max + 2, d}}};
}

// elements of one instance in `member`, e.g. per_instance(&pqp_batch_out::x_full, n_max)
template <typename Batch, typename T>
size_t per_instance(T *Batch::*member, size_t n_max) {
    static const Batch b{};
    const size_t offset = (size_t)(reinterpret_cast<const char *>(&(b.*member)) - reinterpret_cast<const char *>(&b));
    for (const BatchField &f : batch_fields(&b, n_max))
        if (f.offset == offset) return f.count;
    return 0;
}

template <typename Batch>
char *field_of(const Batch &b, const BatchField &f) {
    void *p;
    std::memcpy(&p, reinterpret_cast<const char *>(&b) + f.offset, sizeof p);
    return static_cast<char *>(p);
}

// `b` from instance `first` on: every non-NULL member advanced by `first` instances; NULL members stay NULL. The
// batch and n_max of a pqp_batch_in are left as they are.
template <typename Batch>
Batch batch_from(const Batch &b, size_t first, size_t n_max) {
    Batch v = b;
    for (const BatchField &f : batch_fields(&b, n_max))
        if (char *p = field_of(b, f)) {
            p += first * f.bytes();
            std::memcpy(reinterpret_cast<char *>(&v) + f.offset, &p, sizeof p);
        }
    return v;
}

#ifdef __CUDACC__
// instances [src_first, src_first + count) of `src` to [dst_first, ...) of `dst`, one asynchronous copy per member
// that is non-NULL in both; a caller selects members by leaving the others NULL
template <typename Batch>
cudaError_t copy_batch(const Batch &dst, size_t dst_first, const Batch &src, size_t src_first, size_t count,
                       size_t n_max, cudaMemcpyKind kind, cudaStream_t s) {
    for (const BatchField &f : batch_fields(&dst, n_max)) {
        char *d = field_of(dst, f), *from = field_of(src, f);
        if (!d || !from) continue;
        const cudaError_t e = cudaMemcpyAsync(d + dst_first * f.bytes(), from + src_first * f.bytes(), count * f.bytes(),
                                              kind, s);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// zeroes instances [first, first + count) of every non-NULL member of `b`
template <typename Batch>
cudaError_t zero_batch(const Batch &b, size_t first, size_t count, size_t n_max, cudaStream_t s) {
    for (const BatchField &f : batch_fields(&b, n_max))
        if (char *p = field_of(b, f)) {
            const cudaError_t e = cudaMemsetAsync(p + first * f.bytes(), 0, count * f.bytes(), s);
            if (e != cudaSuccess) return e;
        }
    return cudaSuccess;
}
#endif

}  // namespace pqp
