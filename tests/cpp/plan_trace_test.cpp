// plan_trace_test.cpp — TEST ONLY, host code (g++). The trace table of pqp_plan_trace.h against the byte counts the
// plan's trace copy used per member before the table existed, written out member by member, and trace_from's
// offsets. Prints "ok <fields>" or the first mismatch and exits non-zero.
#include <cstdio>
#include <string>

#include "../../path_optimizer_2_b200/csrc/pqp_plan_trace.h"

namespace {

int fails = 0;

void expect(const char *what, size_t got, size_t want) {
    if (got != want && fails++ < 10) std::printf("mismatch %s: %zu bytes per path, expected %zu\n", what, got, want);
}

}  // namespace

int main() {
    const size_t P = 61, L = 47, N = 255, R = 73;
    const size_t d = sizeof(double), i4 = sizeof(int32_t), nv = 6 * N - 1, m = 6 * N + 2;
    const auto f = pqpl::trace_fields(P, L, N, R);
    size_t at = 0;
    // the expected count of one member, in member order (a missing or reordered member fails here)
#define CHECK(member, bytes)                                                                         \
    do {                                                                                             \
        if (at >= f.size() || f[at].offset != offsetof(pqp_plan_trace, member)) {                   \
            std::printf("mismatch %s: not field %zu of the table\n", #member, at);                 \
            return 1;                                                                                \
        }                                                                                            \
        expect(#member, f[at++].per_path, (bytes));                                                 \
    } while (0)
    CHECK(raw_spline, PQP_SPLINE_ROWS * R * d);
    CHECK(seg_p, i4);
    CHECK(seg_x, P * d);
    CHECK(seg_y, P * d);
    CHECK(seg_angle, P * d);
    CHECK(seg_k, P * d);
    CHECK(seg_s, P * d);
    CHECK(tension_x, P * d);
    CHECK(tension_y, P * d);
    CHECK(tension_s, P * d);
    CHECK(tension_status, i4);
    CHECK(tension_iters, i4);
    CHECK(tension_spline, PQP_SPLINE_ROWS * P * d);
    CHECK(tension_length, d);
    CHECK(dp_status, i4);
    CHECK(dp_n_out, i4);
    CHECK(dp_layer_s, L * d);
    CHECK(dp_lower, L * d);
    CHECK(dp_upper, L * d);
    CHECK(dp_chosen, L * i4);
    CHECK(dp_vehicle_l, d);
    CHECK(post_offsets, L * d);
    CHECK(post_status, i4);
    CHECK(post_iters, i4);
    CHECK(ref_spline, PQP_SPLINE_ROWS * L * d);
    CHECK(max_s, d);
    CHECK(states, PQP_STATE_ROWS * N * d);
    CHECK(curvature, N * d);
    CHECK(total, i4);
    CHECK(bounds, PQP_BOUND_ROWS * N * d);
    CHECK(n_valid, i4);
    CHECK(knots, PQP_NFIELDS * N * d);
    CHECK(inst, PQP_NINST * d);
    CHECK(p, i4);
    CHECK(sol1, 4 * N * d);
    CHECK(status1, i4);
    CHECK(iters1, i4);
    CHECK(x_full1, nv * d);
    CHECK(y_full1, m * d);
    CHECK(z_full1, m * d);
    CHECK(x_full2, nv * d);
    CHECK(y_full2, m * d);
    CHECK(z_full2, m * d);
    CHECK(tension_clearance, P * d);
    CHECK(raw_r, i4);
    CHECK(bspline_degree, i4);
#undef CHECK
    if (at != f.size()) {
        std::printf("mismatch: %zu members checked, the table has %zu\n", at, f.size());
        return 1;
    }
    // trace_from: a set member moves by first * its bytes per path, a NULL one stays NULL
    static double states[16 * PQP_STATE_ROWS * N];
    static int32_t p[16];
    pqp_plan_trace t{};
    t.states = states;
    t.p = p;
    const pqp_plan_trace v = pqpl::trace_from(t, 5, P, L, N, R);
    if (v.states != states + 5 * PQP_STATE_ROWS * N || v.p != p + 5 || v.sol1 != nullptr || v.raw_spline != nullptr) {
        std::printf("mismatch: trace_from offsets\n");
        return 1;
    }
    if (fails) return 1;
    std::printf("ok %zu\n", f.size());
    return 0;
}
