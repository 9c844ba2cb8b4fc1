// pqp_collision_core.cuh — per-state work of the footprint collision check (pqp_bounds_collision_check*,
// include/pqp_bounds.h). Plain FP64 scalar code with no CUDA intrinsics, so the same source is compiled by nvcc for
// the kernel (pqp_bounds.cu) and by g++ for the CPU test driver (tests/emu/collision_driver.cpp).
// Citations are relative to /root/reference/.
#pragma once
#include <math.h>

#include "pqp_bounds_core.cuh"

namespace pqc {

// The car's footprint in the rear-axle frame: circle 0 is CarGeometry's bounding circle, 1 .. 6 its circles_ in the
// order setCircles() writes them (rr, rl, fr, fl, fm, rm).
constexpr int kCircles = 7;
struct Footprint {
    double x[kCircles], y[kCircles], r[kCircles];
};

// CarGeometry(width, back_length, front_length) and setCircles() (src/tools/car_geometry.cpp:10-55), with the
// reference's expressions in double. Host only: the kernel receives the result as a parameter and never calls pow.
inline Footprint car_footprint(double width, double back_length, double front_length) {
    const double length = front_length + back_length;
    const double fl_x = front_length, fl_y = width / 2.0, fr_x = front_length, fr_y = -width / 2.0;
    const double rl_x = -back_length, rl_y = width / 2.0, rr_x = -back_length, rr_y = -width / 2.0;
    Footprint f;
    f.x[0] = (front_length - back_length) / 2.0;
    f.y[0] = 0;
    f.r[0] = sqrt(pow(length / 2, 2) + pow(width / 2, 2));
    const double small_circle_shift = width / 4.0;
    const double small_circle_radius = sqrt(2 * pow(small_circle_shift, 2));
    const double large_circle_radius = sqrt(pow(width, 2) + pow((length - width) / 2.0, 2)) / 2;
    const double cx[6] = {rr_x + small_circle_shift, rl_x + small_circle_shift, fr_x - small_circle_shift,
                          fl_x - small_circle_shift, f.x[0] + (length - width) / 4, f.x[0] - (length - width) / 4};
    const double cy[6] = {rr_y + small_circle_shift, rl_y - small_circle_shift, fr_y + small_circle_shift,
                          fl_y - small_circle_shift, 0, 0};
    for (int k = 0; k < 6; ++k) {
        f.x[k + 1] = cx[k];
        f.y[k + 1] = cy[k];
        f.r[k + 1] = k < 4 ? small_circle_radius : large_circle_radius;
    }
    return f;
}

// CollisionChecker::isSingleStateCollisionFreeImproved (src/tools/collision_checker.cpp:41-59) for the state
// (x, y, heading) at the rear axle, with the comparisons as the reference writes them: a NaN distance is not below
// a radius, and a state whose bounding circle clears the map is free without looking at the six circles.
// `clearance` is min over the six circles of d_i - r_i (NaN terms skipped), the margin of the exact test
// isSingleStateCollisionFree (:17-39); all seven lookups are made for every state.
PQB_HD bool state_free(const pqb::MapView &m, const Footprint &f, double x, double y, double heading,
                       double &clearance) {
    // local2Global (src/tools/tools.cpp:50-55)
    const double c = cos(heading), s = sin(heading);
    bool inside0 = false, below0 = false, exact = true;
    clearance = NAN;
    for (int k = 0; k < kCircles; ++k) {
        const double gx = f.x[k] * c - f.y[k] * s + x;
        const double gy = f.x[k] * s + f.y[k] * c + y;
        const bool inside = pqb::map_inside(m, gx, gy);
        const double d = pqb::map_distance(m, gx, gy);
        if (k == 0) {
            inside0 = inside;
            below0 = d < f.r[0];
        } else {
            if (!inside || d < f.r[k]) exact = false;
            clearance = fmin(clearance, d - f.r[k]);
        }
    }
    if (!inside0) return false;
    return below0 ? exact : true;
}

}  // namespace pqc
