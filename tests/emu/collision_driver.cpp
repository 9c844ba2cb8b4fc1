// collision_driver.cpp — TEST ONLY. Compiles the collision check's per-state source
// (path_optimizer_2_b200/csrc/pqp_collision_core.cuh) for the host and loops over the paths and states the CUDA
// grid would run, so the kernel arithmetic can be checked against the oracle on a GPU-less box. The product has no
// CPU path; nothing in the package references this file.
#include <cmath>
#include <cstdint>

#include "../../include/pqp_bounds.h"
#include "../../path_optimizer_2_b200/csrc/pqp_collision_core.cuh"

extern "C" int pqc_emu_check(const pqp_bounds_map *map, const pqp_bounds_params *p, const pqp_collision_in *in,
                             const pqp_collision_out *out) {
    pqb::MapView m;
    m.dist = map->distance;
    m.rows = map->rows;
    m.cols = map->cols;
    m.res = map->resolution;
    m.inv_res = 1.0 / map->resolution;
    m.half_lx = 0.5 * map->rows * map->resolution;
    m.half_ly = 0.5 * map->cols * map->resolution;
    m.cx = map->center_x;
    m.cy = map->center_y;
    const pqc::Footprint fp = pqc::car_footprint(p->car_width, fabs(p->rear_length), p->front_length);
    const int n_max = in->n_max;
    for (int b = 0; b < in->batch; ++b) {
        int nb = in->n[b];
        nb = nb < 0 ? 0 : (nb > n_max ? n_max : nb);
        const double *x = in->poses + (size_t)b * in->row_stride * n_max, *y = x + n_max, *h = y + n_max;
        int hit = nb;
        for (int i = 0; i < n_max; ++i) {
            bool free_ = false;
            double c = 0.0;
            if (i < nb) {
                free_ = pqc::state_free(m, fp, x[i], y[i], h[i], c);
                if (!free_ && i < hit) hit = i;
            }
            if (out->state_free) out->state_free[(size_t)b * n_max + i] = free_ ? 1 : 0;
            if (out->clearance) out->clearance[(size_t)b * n_max + i] = c;
        }
        out->first_hit[b] = hit;
    }
    return 0;
}

// the footprint circles as the kernel receives them: x[7], y[7], r[7] (bounding circle, rr, rl, fr, fl, fm, rm)
extern "C" void pqc_emu_footprint(const pqp_bounds_params *p, double *xyr) {
    const pqc::Footprint fp = pqc::car_footprint(p->car_width, fabs(p->rear_length), p->front_length);
    for (int k = 0; k < pqc::kCircles; ++k) {
        xyr[k] = fp.x[k];
        xyr[pqc::kCircles + k] = fp.y[k];
        xyr[2 * pqc::kCircles + k] = fp.r[k];
    }
}
