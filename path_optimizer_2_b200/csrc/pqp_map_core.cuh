// pqp_map_core.cuh — per-column and per-row work of the exact Euclidean distance transform that turns an
// occupancy image into the map's float distance layer (pqp_bounds_set_occupancy*, include/pqp_bounds.h).
// Plain C++ (the FP64 box test below names its CUDA rounding intrinsics under __CUDA_ARCH__ only), so the same source
// is compiled by nvcc for the kernels (pqp_bounds.cu) and by g++ for the CPU test drivers (tests/emu/map_driver.cpp,
// tests/emu/boxes_driver.cpp).
//
// Two separable passes (Meijster, Roerdink and Hesselink, "A general algorithm for computing distance
// transforms in linear time", 2000), both in int32:
//   column pass  g(i, j)  = |i - i'| to the nearest obstacle cell (i', j) of column j, or kInf(rows, cols) when
//                           column j has none;
//   row pass     d2(i, j) = min over j' of (j - j')^2 + g(i, j')^2, from the lower envelope of those parabolas.
// A column without obstacles keeps g = rows + cols, whose square exceeds every true squared distance
// ((rows - 1)^2 + (cols - 1)^2), so it never wins a row that has a finite g. A row has no finite g only when the
// whole image has no obstacle; then every d2 of it is kInf^2, which layer_value turns into the obstacle-free value.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PQM_HD __host__ __device__ __forceinline__
#else
#define PQM_HD inline
#endif

namespace pqm {

// rows, cols <= kMaxSide keeps every intermediate below 2^31: kInf^2 <= 2^30, (j - j')^2 < 2^28. The row pass
// holds 12 bytes per column in shared memory (192 KB at kMaxSide), and the envelope indices fit in int16.
constexpr int kMaxSide = 16384;
constexpr int kRowSmemPerCol = 4 + 2 + 2 + 4;  // g / d2 (int32), vertex s, start t (int16), g(s)^2 (int32)

PQM_HD int32_t inf_g(int rows, int cols) { return rows + cols; }

// Column pass, column j: forward sweep for the nearest obstacle above, backward sweep (over g itself: g = 0 marks
// an obstacle) for the nearest one below. `img` and `g` are row-major [rows][cols].
PQM_HD void column_pass(const uint8_t *__restrict__ img, int rows, int cols, int j, int obstacle_max,
                        int32_t *__restrict__ g) {
    const int32_t inf = inf_g(rows, cols);
    int32_t d = inf;
    for (int i = 0; i < rows; ++i) {
        const size_t k = (size_t)i * cols + j;
        d = (int32_t)img[k] <= obstacle_max ? 0 : (d < inf ? d + 1 : inf);
        g[k] = d;
    }
    d = inf;
    for (int i = rows - 1; i >= 0; --i) {
        const size_t k = (size_t)i * cols + j;
        const int32_t up = g[k];
        d = up == 0 ? 0 : (d < inf ? d + 1 : inf);
        if (d < up) g[k] = d;
    }
}

// Sep(i, u) of Meijster et al. for i < u: the last column x at which parabola i is not above parabola u,
// (x - i)^2 + gi2 <= (x - u)^2 + gu2  <=>  2 x (u - i) <= u^2 - i^2 + gu2 - gi2, i.e. floor of the quotient.
// envelope() calls it only where parabola i is not above u at a column t >= 0, so the quotient is >= t >= 0 and
// C's truncating division is the floor.
PQM_HD int32_t sep(int32_t i, int32_t u, int32_t gi2, int32_t gu2) {
    return (u * u - i * i + (gu2 - gi2)) / (2 * (u - i));
}

// Row pass, first half (one thread): the lower envelope of the parabolas (x - u)^2 + g[u]^2, u = 0 .. cols - 1.
// Parabola k of the envelope has its vertex at s[k], value h[k] = g[s[k]]^2 there, and is the lowest from column
// t[k] up to t[k + 1] - 1 (the last one up to cols - 1). Returns the number of parabolas.
PQM_HD int envelope(const int32_t *g, int cols, int16_t *s, int16_t *t, int32_t *h) {
    int q = 0;
    s[0] = 0;
    t[0] = 0;
    h[0] = g[0] * g[0];
    for (int u = 1; u < cols; ++u) {
        const int32_t gu2 = g[u] * g[u];
        // drop the parabolas that u undercuts at the first column where they are lowest
        while (q >= 0) {
            const int32_t tq = t[q], dq = tq - s[q], du = tq - u;
            if (dq * dq + h[q] <= du * du + gu2) break;
            --q;
        }
        if (q < 0) {
            q = 0;
            s[0] = (int16_t)u;
            t[0] = 0;
            h[0] = gu2;
        } else {
            const int32_t w = 1 + sep(s[q], u, h[q], gu2);
            if (w < cols) {
                ++q;
                s[q] = (int16_t)u;
                t[q] = (int16_t)w;
                h[q] = gu2;
            }
        }
    }
    return q + 1;
}

// Row pass, second half: parabola k of the envelope writes d2 over its columns. Independent per k.
PQM_HD void fill(const int16_t *s, const int16_t *t, const int32_t *h, int n, int cols, int k, int32_t *d2) {
    const int32_t sk = s[k], hk = h[k];
    const int end = k + 1 < n ? t[k + 1] : cols;
    for (int u = t[k]; u < end; ++u) d2[u] = (u - sk) * (u - sk) + hk;
}

// The layer value of one cell: sqrt in IEEE double, one rounding to float, a float multiply by the resolution
// (scipy.ndimage.distance_transform_edt(...).astype(float32) * float32(res)). An image without obstacles gives
// 2^64 per cell, as OpenCV's precise transform does.
PQM_HD float layer_value(int32_t d2, int32_t inf2, float res) {
    if (d2 >= inf2) return 18446744073709551616.0f * res;
    return (float)sqrt((double)d2) * res;
}

// ---- Obstacle boxes stamped into an occupancy image (pqp_bounds_set_occupancy_boxes*, include/pqp_bounds.h) ----
// Every product and sum rounds on its own: the intrinsics on the device (pqp_bounds.cu is compiled with contraction on),
// plain operators on the host (the drivers are compiled with -ffp-contract=off).
PQM_HD double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
PQM_HD double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
PQM_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// The map fields the cell centres come from (pqb::MapView's, as make_view sets them: half_lx = 0.5 * rows * res).
struct Cells {
    int rows, cols;
    double res, half_lx, half_ly, cx, cy;
};

// centre of row i / column j: cx + (half_lx - (i + 0.5) res), cy + (half_ly - (j + 0.5) res)
PQM_HD double cell_px(const Cells &m, int i) { return add_rn(m.cx, sub_rn(m.half_lx, mul_rn(i + 0.5, m.res))); }
PQM_HD double cell_py(const Cells &m, int j) { return add_rn(m.cy, sub_rn(m.half_ly, mul_rn(j + 0.5, m.res))); }

// The predicate: (px, py) lies inside or on the boundary of the box centred at (bx, by) whose length (2 half_l) runs
// along the heading with cosine c and sine s. A NaN anywhere, or a negative half size, fails a comparison: false.
PQM_HD bool in_box(double px, double py, double bx, double by, double c, double s, double half_l, double half_w) {
    const double dx = sub_rn(px, bx), dy = sub_rn(py, by);
    const double u = add_rn(mul_rn(dx, c), mul_rn(dy, s));
    const double v = sub_rn(mul_rn(dy, c), mul_rn(dx, s));
    return fabs(u) <= half_l && fabs(v) <= half_w;
}

constexpr int kBoxFields = 5;  // x, y, heading, length, width

// One box as the stamping reads it: the predicate's operands and the half extents (rx along x, ry along y) of a
// bounding box that holds every cell centre the predicate accepts, +inf where a field is infinite.
struct Box {
    double x, y, c, s, half_l, half_w, rx, ry;
};

// Rounding slack of the bounding boxes: the predicate's error is a few ulp of |px| + |bx| + |py| + |by|, far below
// 1e-9 of it.
PQM_HD double map_slack(const Cells &m) { return 1e-9 * (1.0 + fabs(m.cx) + fabs(m.cy) + m.half_lx + m.half_ly); }

// The Box of fields f[0 .. 4]; false for a box the predicate rejects at every point (a NaN field, a NaN cosine or sine
// from an infinite heading, a negative length or width), which stamps nothing.
PQM_HD bool make_box(const double *f, Box &b) {
    double s, c;
#ifdef __CUDA_ARCH__
    sincos(f[2], &s, &c);
#else
    s = sin(f[2]);
    c = cos(f[2]);
#endif
    b.x = f[0];
    b.y = f[1];
    b.c = c;
    b.s = s;
    b.half_l = mul_rn(0.5, f[3]);
    b.half_w = mul_rn(0.5, f[4]);
    if (!(b.half_l >= 0.0 && b.half_w >= 0.0) || b.x != b.x || b.y != b.y || c != c || s != s) return false;
    if (isfinite(b.x) && isfinite(b.y) && isfinite(b.half_l) && isfinite(b.half_w)) {
        const double rx = b.half_l * fabs(c) + b.half_w * fabs(s), ry = b.half_l * fabs(s) + b.half_w * fabs(c);
        const double slack = 1e-9 * (1.0 + fabs(b.x) + fabs(b.y) + rx + ry);
        b.rx = rx + slack;
        b.ry = ry + slack;
    } else {
        b.rx = b.ry = INFINITY;
    }
    return true;
}

// Whether the box can reach a column whose centre lies in [py_lo, py_hi] (already widened by map_slack).
PQM_HD bool box_reaches(const Box &b, double py_lo, double py_hi) { return !(b.y - b.ry > py_hi || b.y + b.ry < py_lo); }

// Column j of a stamped image: g = 0 on an obstacle of the base image, 1 elsewhere (the column sweeps read only that).
PQM_HD void column_init(const uint8_t *__restrict__ img, int rows, int cols, int j, int obstacle_max,
                        int32_t *__restrict__ g) {
    for (int i = 0; i < rows; ++i) {
        const size_t k = (size_t)i * cols + j;
        g[k] = (int32_t)img[k] <= obstacle_max ? 0 : 1;
    }
}

// Sets g = 0 on every cell of column j (centre py) that the predicate puts in box b. Only rows whose centre can lie
// within b.rx (+ ms, the map's slack) of b.x are tested, one row more at each end; every tested row is decided by the
// predicate itself.
PQM_HD void stamp_column(int32_t *__restrict__ g, const Cells &m, int j, double py, double ms, const Box &b) {
    if (!(fabs(py - b.y) <= b.ry + ms)) return;
    double lo = 0.0, hi = m.rows - 1;
    if (isfinite(b.rx)) {  // px(i) falls as i grows: px <= b.x + rx from row `lo` on, px >= b.x - rx up to row `hi`
        const double top = m.cx + m.half_lx;
        lo = (top - (b.x + b.rx + ms)) / m.res - 0.5;
        hi = (top - (b.x - b.rx - ms)) / m.res - 0.5;
        lo = lo < 0.0 ? 0.0 : lo;
        hi = hi > m.rows - 1 ? m.rows - 1 : hi;
        if (!(lo <= hi)) return;
    }
    int i0 = (int)floor(lo) - 1, i1 = (int)ceil(hi) + 1;
    i0 = i0 < 0 ? 0 : i0;
    i1 = i1 > m.rows - 1 ? m.rows - 1 : i1;
    for (int i = i0; i <= i1; ++i)
        if (in_box(cell_px(m, i), py, b.x, b.y, b.c, b.s, b.half_l, b.half_w)) g[(size_t)i * m.cols + j] = 0;
}

// The column pass over a column that column_init and stamp_column prepared: g = 0 marks an obstacle cell.
PQM_HD void column_sweeps(int rows, int cols, int j, int32_t *__restrict__ g) {
    const int32_t inf = inf_g(rows, cols);
    int32_t d = inf;
    for (int i = 0; i < rows; ++i) {
        const size_t k = (size_t)i * cols + j;
        d = g[k] == 0 ? 0 : (d < inf ? d + 1 : inf);
        g[k] = d;
    }
    d = inf;
    for (int i = rows - 1; i >= 0; --i) {
        const size_t k = (size_t)i * cols + j;
        const int32_t up = g[k];
        d = up == 0 ? 0 : (d < inf ? d + 1 : inf);
        if (d < up) g[k] = d;
    }
}

}  // namespace pqm
