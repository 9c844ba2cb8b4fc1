// plan_driver.cpp — TEST ONLY. Compiles the plan glue's per-path source (path_optimizer_2_b200/csrc/pqp_plan_core.cuh)
// for the host, so its arithmetic can be checked against oracle/plan_oracle.py on a GPU-less box. The product has no
// CPU path; nothing in the package references this file.
#include <cmath>
#include <cstdint>

#include "../../path_optimizer_2_b200/csrc/pqp_plan_core.cuh"

extern "C" {

void plan_emu_fit(const double *sx, const double *y, int k, double *a, double *b, double *c) {
    pqpl::natural_spline_fit(sx, y, k, a, b, c);
}

int plan_emu_chord(const double *x, const double *y, int r, double *s) {
    pqpl::chord_length(x, y, r, s);
    return pqpl::increasing(s, r) ? 1 : 0;
}

int plan_emu_segment_count(double max_s, int cap) { return pqpl::segment_count(max_s, cap); }

// samples j = 0 .. p-1 of segmentRawReference: out[5][p] = x, y, angle, k, s
void plan_emu_segment(const double *rows, int stride, int k, int p, double *out) {
    const pqb::SplineView sp = pqpl::view(rows, stride, k);
    for (int j = 0; j < p; ++j) {
        const double s = pqpl::segment_s(j);
        pqpl::segment_sample(sp, s, out[j], out[p + j], out[2 * p + j], out[3 * p + j]);
        out[4 * p + j] = s;
    }
}

void plan_emu_post_points(const double *rows, int stride, int k, const double *layer_s, const double *offsets, int n,
                          double *s, double *x, double *y) {
    pqpl::post_points(pqpl::view(rows, stride, k), layer_s, offsets, n, s, x, y);
}

int plan_emu_process(const double *rows, int stride, int k, double length, const double *start, const double *target,
                     double epsilon, double *out) {
    return pqpl::process_reference(pqpl::view(rows, stride, k), length, start, target, epsilon, out[0], out[1], out[2]);
}

int plan_emu_precise(const double *s, int n, int rough, double precise_length) {
    return pqpl::precise_size(s, n, rough != 0, precise_length);
}

void plan_emu_end_heading(int constrain, int blocked, double target_heading, double last_heading, double *out) {
    pqpl::end_heading_rows(constrain != 0, blocked != 0, target_heading, last_heading, out[0], out[1]);
}

void plan_emu_placeholder(double *s, double *x, double *y) { pqpl::placeholder_points(s, x, y); }
}
