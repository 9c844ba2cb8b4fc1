// pqp_map_core.cuh — per-column and per-row work of the exact Euclidean distance transform that turns an
// occupancy image into the map's float distance layer (pqp_bounds_set_occupancy*, include/pqp_bounds.h).
// Plain integer C++ with no CUDA intrinsics, so the same source is compiled by nvcc for the kernels
// (pqp_bounds.cu) and by g++ for the CPU test driver (tests/emu/map_driver.cpp).
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

}  // namespace pqm
