// pqp_plan_trace.h — the layout of a pqp_plan_trace: every member with the bytes it holds per path, for a handle of
// capacities P = p_max, L = layers_max, N = n_max, R = r_max. The plan's copy_trace sizes its copies with it and the
// multi-device plan offsets a caller's trace to a shard's first path with it. Host code only.
#pragma once
#include <array>
#include <cstddef>
#include <cstdint>
#include <cstring>

#include "../../include/pqp_plan.h"
#include "pqp_batch_layout.h"

namespace pqpl {

struct TraceField {
    size_t offset;    // offsetof(pqp_plan_trace, member)
    size_t per_path;  // bytes of one path's entries
};

// every member of pqp_plan_trace is a pointer, and each is listed below once
constexpr int kTraceFields = (int)(sizeof(pqp_plan_trace) / sizeof(void *));

// in the member order of pqp_plan_trace
inline std::array<TraceField, kTraceFields> trace_fields(size_t P, size_t L, size_t N, size_t R) {
    const size_t d = sizeof(double), i4 = sizeof(int32_t);
    const size_t nv = pqp::per_instance(&pqp_batch_out::x_full, N), m = pqp::per_instance(&pqp_batch_out::y_full, N);
#define PQL_F(member, bytes) TraceField{offsetof(pqp_plan_trace, member), (bytes)}
    const TraceField f[] = {
        PQL_F(raw_spline, PQP_SPLINE_ROWS * R * d), PQL_F(seg_p, i4), PQL_F(seg_x, P * d), PQL_F(seg_y, P * d),
        PQL_F(seg_angle, P * d), PQL_F(seg_k, P * d), PQL_F(seg_s, P * d), PQL_F(tension_x, P * d),
        PQL_F(tension_y, P * d), PQL_F(tension_s, P * d), PQL_F(tension_status, i4), PQL_F(tension_iters, i4),
        PQL_F(tension_spline, PQP_SPLINE_ROWS * P * d), PQL_F(tension_length, d), PQL_F(dp_status, i4),
        PQL_F(dp_n_out, i4), PQL_F(dp_layer_s, L * d), PQL_F(dp_lower, L * d), PQL_F(dp_upper, L * d),
        PQL_F(dp_chosen, L * i4), PQL_F(dp_vehicle_l, d), PQL_F(post_offsets, L * d), PQL_F(post_status, i4),
        PQL_F(post_iters, i4), PQL_F(ref_spline, PQP_SPLINE_ROWS * L * d), PQL_F(max_s, d),
        PQL_F(states, PQP_STATE_ROWS * N * d), PQL_F(curvature, N * d), PQL_F(total, i4),
        PQL_F(bounds, PQP_BOUND_ROWS * N * d), PQL_F(n_valid, i4), PQL_F(knots, PQP_NFIELDS * N * d),
        PQL_F(inst, PQP_NINST * d), PQL_F(p, i4), PQL_F(sol1, 4 * N * d), PQL_F(status1, i4), PQL_F(iters1, i4),
        PQL_F(x_full1, nv * d), PQL_F(y_full1, m * d), PQL_F(z_full1, m * d), PQL_F(x_full2, nv * d),
        PQL_F(y_full2, m * d), PQL_F(z_full2, m * d), PQL_F(tension_clearance, P * d), PQL_F(raw_r, i4),
        PQL_F(bspline_degree, i4)
    };
#undef PQL_F
    static_assert(sizeof f / sizeof *f == kTraceFields, "a pqp_plan_trace member is missing from the table");
    std::array<TraceField, kTraceFields> a;
    for (int i = 0; i < kTraceFields; ++i) a[i] = f[i];
    return a;
}

// the member of `t` that `f` describes (as an untyped pointer)
inline void *trace_get(const pqp_plan_trace &t, const TraceField &f) {
    void *p;
    std::memcpy(&p, reinterpret_cast<const char *>(&t) + f.offset, sizeof p);
    return p;
}

inline void trace_set(pqp_plan_trace &t, const TraceField &f, void *p) {
    std::memcpy(reinterpret_cast<char *>(&t) + f.offset, &p, sizeof p);
}

// `t` from path `first` on: every non-NULL member advanced by `first` paths; NULL members stay NULL
inline pqp_plan_trace trace_from(const pqp_plan_trace &t, size_t first, size_t P, size_t L, size_t N, size_t R) {
    pqp_plan_trace v = t;
    for (const TraceField &f : trace_fields(P, L, N, R))
        if (char *p = static_cast<char *>(trace_get(t, f))) trace_set(v, f, p + first * f.per_path);
    return v;
}

}  // namespace pqpl
