// pqp_smoother_core.cuh — the three QPs of the reference's front end (SURVEY.md §8 row f-3) through one
// OSQP-style ADMM routine for small stage-banded QPs, FP64, one warp per QP:
//   TensionSmoother2::osqpSmooth   /root/reference/src/reference_path_smoother/tension_smoother_2.cpp:20-158
//   TensionSmoother::osqpSmooth    src/reference_path_smoother/tension_smoother.cpp:49-177 (Cartesian tension)
//   ReferencePathSmoother::postSmooth (its QP)  src/reference_path_smoother/reference_path_smoother.cpp:526-636
// All hand OSQP (defaults, eps 1e-3: only verbosity and warm start are set, :33-34 / :62-63 / :533-534) a QP whose
// variables can be ordered stage by stage so that P + sigma I + A' diag(rho) A is banded (half-bandwidth 4 for
// TENSION2 and post, 9 for the Cartesian QP) and every row / column of A has at most 4 entries. The routine below is
// OSQP 0.6.x on such a QP - Ruiz equilibration with cost scaling, rho vector, relaxed ADMM step with the x-update
// done on the reduced banded system (banded LDL', refactored on rho updates), unscaled termination test, primal /
// dual infeasibility certificates, adaptive rho - i.e. the algorithm of oracle/osqp_generic.py, which is the oracle
// of this row. The half-bandwidths of the reduced matrix (HB) and of P (HBP) are template parameters of the band
// routines.
//
// One templated routine over a warp context: the CUDA kernel (pqp_smoother.cu) and the CPU test driver
// (tests/emu/smoother_driver.cpp, 1 "lane") compile this same source.
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PQS_HD __host__ __device__ __forceinline__
#else
#define PQS_HD inline
#endif

namespace pqs {

constexpr int kHB = 4;    // half-bandwidth of the reduced matrix (TENSION2, post: entries of a row lie within 4 columns)
constexpr int kHBP = 4;   // half-bandwidth of P (TENSION2, post)
constexpr int kHBC = 9;   // Cartesian tension QP: half-bandwidth of P and of the reduced matrix (x_i .. x_{i+3})
constexpr int kEll = 4;   // entries per row / column of A (all three QPs)

struct Settings {  // OSQP settings (defaults = OSQP 0.6.x defaults; the reference overrides none of them here)
    double rho, sigma, alpha, eps_abs, eps_rel, eps_prim_inf, eps_dual_inf, adaptive_rho_tolerance;
    int max_iter, check_termination, scaling, adaptive_rho, adaptive_rho_interval;
};

struct TensionWeights { double deviation, curvature, curvature_rate; };  // planning_flags.cpp:57-61: 0.005, 1, 10
struct PostWeights { double x, dx, ddx; };                               // reference_path_smoother.cpp:590-592: 1, 100, 1000
struct CartesianWeights { double curvature, curvature_rate, deviation; }; // planning_flags.cpp:51-55: 1, 50, 0

// status codes as in include/pqp.h
enum { kSolved = 0, kMaxIter = 1, kPrimInf = 2, kDualInf = 3, kSolvedInacc = 4, kPrimInfInacc = 5, kDualInfInacc = 6, kNumerical = 7 };

// Working set of one QP (pointers into the CTA's scratch; `Lb`, `w` may be shared memory)
struct Work {
    int N, M;            // variables, rows
    int Np;              // N padded for the band arrays (N + HB)
    double *Pb;          // [Np][HBP+1]  P(j, j+d), upper band, scaled in place
    double *q;           // [N]
    double *Av;          // [M][kEll] values, row-ELL
    int16_t *Ac;         // [M][kEll] columns (-1 = empty)
    int16_t *Cr;         // [N][kEll] col-ELL: row index (-1 = empty)
    int8_t *Ce;          // [N][kEll] col-ELL: position of the entry in its row
    int8_t *cnt;         // [N] entries per column (build_columns)
    double *l, *u;       // [M] (scaled after set-up)
    double *D, *E;       // [N], [M]
    double *rho_vec;     // [M]
    int8_t *ctype;       // [M]: -1 loose, 1 equality, 0 inequality
    double *x, *z, *y;   // iterates (scaled)
    double *xp;          // [N] previous x (delta_x for the dual certificate)
    double *dy;          // [M] delta_y
    double *Lb;          // [Np][HB+1] band of the reduced matrix -> its LDL' (d in [.][0], L(j+i, j) in [.][i])
    double *w;           // [Np] rhs / solution of the reduced solve
    double *t1, *t2;     // [max(N, M)] temporaries
    double c, rho;
};

// ------------------------------------------------------------------ warp contexts
struct SerialLane {  // CPU build: one lane
    PQS_HD int lane() const { return 0; }
    PQS_HD int lanes() const { return 1; }
    PQS_HD void sync() const {}
    PQS_HD double max(double v) const { return v; }
    PQS_HD double sum(double v) const { return v; }
    PQS_HD int all(int v) const { return v; }
};

PQS_HD double lim_scaling(double v) {
    v = v < 1e-4 ? 1.0 : v;
    return v > 1e4 ? 1e4 : v;
}
PQS_HD double dabs(double a) { return fabs(a); }
PQS_HD double dmax2(double a, double b) { return a > b ? a : b; }
PQS_HD double dmin2(double a, double b) { return a < b ? a : b; }

// ------------------------------------------------------------------ assembly
// TensionSmoother2 (tension_smoother_2.cpp:74-158), variables interleaved per point: x_i, y_i, theta_i, k_i at
// 4 i .. 4 i + 3 (k only for i < p - 1); rows per segment i: 3 i .. 3 i + 2 (x, y, theta update), then x_0, y_0.
// The reference's own index order (x block, y block, theta block, k block) is restored on output.
template <class Ctx>
PQS_HD void assemble_tension(const Ctx &c, Work &W, int p, const double *xl, const double *yl, const double *al, const double *kl,
                             const double *sl, const TensionWeights &tw) {
    const int N = 4 * p - 1, M = 3 * (p - 1) + 2;
    W.N = N;
    W.M = M;
    for (int j = c.lane(); j < W.Np * (kHBP + 1); j += c.lanes()) W.Pb[j] = 0.0;
    for (int r = c.lane(); r < M * kEll; r += c.lanes()) {
        W.Av[r] = 0.0;
        W.Ac[r] = -1;
    }
    c.sync();
    for (int i = c.lane(); i < p; i += c.lanes()) {
        double *Px = W.Pb + (size_t)(4 * i) * (kHBP + 1);
        Px[0] = tw.deviation * 2;                       // x_i  (:84-85)
        Px[kHBP + 1] = tw.deviation * 2;                // y_i
        Px[2 * (kHBP + 1)] = 0.0;                       // theta_i
        W.q[4 * i] = -2 * tw.deviation * xl[i];         // (:154-155)
        W.q[4 * i + 1] = -2 * tw.deviation * yl[i];
        W.q[4 * i + 2] = 0.0;
        if (i < p - 1) {
            // curvature weight + the [1 -1; -1 1] curvature-rate blocks on (k_i, k_{i+1}) for i < p - 2 (:86, :88-93)
            double dk = tw.curvature * 2;
            if (i <= p - 3) dk += 2 * tw.curvature_rate;   // block starting at i
            if (i >= 1) dk += 2 * tw.curvature_rate;       // block starting at i - 1
            double *Pk = W.Pb + (size_t)(4 * i + 3) * (kHBP + 1);
            Pk[0] = dk;
            Pk[4] = (i <= p - 3) ? -2 * tw.curvature_rate : 0.0;   // P(k_i, k_{i+1}), 4 columns apart
            W.q[4 * i + 3] = 0.0;
        }
    }
    for (int i = c.lane(); i < p - 1; i += c.lanes()) {
        const double ds = sl[i + 1] - sl[i];
        const double sa = sin(al[i]), ca = cos(al[i]);
        // x update:  x_{i+1} - x_i + ds sin(a_i) theta_i = ds cos(a_i)   (:113-121, :132-134)
        int r = 3 * i;
        W.Ac[r * kEll + 0] = (int16_t)(4 * i);         W.Av[r * kEll + 0] = -1;
        W.Ac[r * kEll + 1] = (int16_t)(4 * i + 2);     W.Av[r * kEll + 1] = ds * sa;
        W.Ac[r * kEll + 2] = (int16_t)(4 * (i + 1));   W.Av[r * kEll + 2] = 1;
        W.l[r] = W.u[r] = ds * ca;
        r = 3 * i + 1;  // y update
        W.Ac[r * kEll + 0] = (int16_t)(4 * i + 1);     W.Av[r * kEll + 0] = -1;
        W.Ac[r * kEll + 1] = (int16_t)(4 * i + 2);     W.Av[r * kEll + 1] = -ds * ca;
        W.Ac[r * kEll + 2] = (int16_t)(4 * (i + 1) + 1); W.Av[r * kEll + 2] = 1;
        W.l[r] = W.u[r] = ds * sa;
        r = 3 * i + 2;  // theta update: theta_{i+1} - theta_i - ds k_i = -ds k_list_i
        W.Ac[r * kEll + 0] = (int16_t)(4 * i + 2);     W.Av[r * kEll + 0] = -1;
        W.Ac[r * kEll + 1] = (int16_t)(4 * i + 3);     W.Av[r * kEll + 1] = -ds;
        W.Ac[r * kEll + 2] = (int16_t)(4 * (i + 1) + 2); W.Av[r * kEll + 2] = 1;
        W.l[r] = W.u[r] = -ds * kl[i];
    }
    if (c.lane() == 0) {
        int r = 3 * (p - 1);
        W.Ac[r * kEll] = 0;  W.Av[r * kEll] = 1;  W.l[r] = W.u[r] = xl[0];   // (:123, :140-141)
        ++r;
        W.Ac[r * kEll] = 1;  W.Av[r * kEll] = 1;  W.l[r] = W.u[r] = yl[0];
    }
    c.sync();
}

// postSmooth's QP (reference_path_smoother.cpp:584-636), variables interleaved per layer: x_i, dx_i, ddx_i at
// 3 i .. 3 i + 2; rows: x range i at 3 i, (x_{i+1} - x_i - ds dx_i = 0) at 3 i + 1, (dx_{i+1} - dx_i - ds ddx_i = 0) at 3 i + 2.
template <class Ctx>
PQS_HD void assemble_post(const Ctx &c, Work &W, int p, const double *layer_s, const double *lower, const double *upper,
                          double vehicle_l, const PostWeights &pw) {
    const int N = 3 * p, M = 3 * p - 2;
    W.N = N;
    W.M = M;
    for (int j = c.lane(); j < W.Np * (kHBP + 1); j += c.lanes()) W.Pb[j] = 0.0;
    for (int r = c.lane(); r < M * kEll; r += c.lanes()) {
        W.Av[r] = 0.0;
        W.Ac[r] = -1;
    }
    c.sync();
    for (int i = c.lane(); i < p; i += c.lanes()) {
        W.Pb[(size_t)(3 * i) * (kHBP + 1)] = pw.x;
        W.Pb[(size_t)(3 * i + 1) * (kHBP + 1)] = pw.dx;
        W.Pb[(size_t)(3 * i + 2) * (kHBP + 1)] = pw.ddx;
        W.q[3 * i] = W.q[3 * i + 1] = W.q[3 * i + 2] = 0.0;
    }
    // row numbering: the last layer has only its range row -> rows 3 i (range), 3 i + 1, 3 i + 2 for i < p - 1, and 3 (p - 1)
    for (int i = c.lane(); i < p; i += c.lanes()) {
        const int r = 3 * i;
        W.Ac[r * kEll] = (int16_t)(3 * i);
        W.Av[r * kEll] = 1;
        W.l[r] = (i == 0) ? vehicle_l : lower[i];   // (:628-633)
        W.u[r] = (i == 0) ? vehicle_l : upper[i];
        if (i < p - 1) {
            const double ds = layer_s[i + 1] - layer_s[i];
            int r1 = 3 * i + 1;
            W.Ac[r1 * kEll + 0] = (int16_t)(3 * i);       W.Av[r1 * kEll + 0] = -1;
            W.Ac[r1 * kEll + 1] = (int16_t)(3 * i + 1);   W.Av[r1 * kEll + 1] = -ds;
            W.Ac[r1 * kEll + 2] = (int16_t)(3 * (i + 1)); W.Av[r1 * kEll + 2] = 1;
            W.l[r1] = W.u[r1] = 0.0;
            r1 = 3 * i + 2;
            W.Ac[r1 * kEll + 0] = (int16_t)(3 * i + 1);       W.Av[r1 * kEll + 0] = -1;
            W.Ac[r1 * kEll + 1] = (int16_t)(3 * i + 2);       W.Av[r1 * kEll + 1] = -ds;
            W.Ac[r1 * kEll + 2] = (int16_t)(3 * (i + 1) + 1); W.Av[r1 * kEll + 2] = 1;
            W.l[r1] = W.u[r1] = 0.0;
        }
    }
    c.sync();
}

// TensionSmoother (tension_smoother.cpp:102-177), variables interleaved per point: x_i, y_i, d_i at 3 i .. 3 i + 2
// (d_i: lateral shift of point i); rows per point: 3 i (x_i - cos(theta_i) d_i = x_list_i), 3 i + 1 (the same in y),
// 3 i + 2 (d_i in its clearance range), theta_i = angle_i + pi / 2. P couples x_i with x_{i+3}: half-bandwidth 9.
// Each entry of P is the sum of the dense blocks that cover it, added in the reference's order (block i ascending,
// the curvature block before the curvature-rate block); P(d_i, d_i) is set, not added.
constexpr double kCartesianDefaultClearance = 2.0;  // tension_smoother.cpp:163
PQS_HD double dds_coef(int k) { return k == 1 ? -2.0 : 1.0; }                                         // [1 -2 1]
PQS_HD double ddds_coef(int k) { return k == 0 ? -1.0 : (k == 1 ? 3.0 : (k == 2 ? -3.0 : 1.0)); }    // [-1 3 -3 1]
template <class Ctx>
PQS_HD void assemble_cartesian(const Ctx &c, Work &W, int p, const double *xl, const double *yl, const double *al,
                               const double *cl, const CartesianWeights &cw) {
    constexpr int S = kHBC + 1;  // row stride of the P band
    const int N = 3 * p, M = 3 * p;
    W.N = N;
    W.M = M;
    for (int j = c.lane(); j < W.Np * S; j += c.lanes()) W.Pb[j] = 0.0;
    for (int r = c.lane(); r < M * kEll; r += c.lanes()) {
        W.Av[r] = 0.0;
        W.Ac[r] = -1;
    }
    c.sync();
    for (int j = c.lane(); j < p; j += c.lanes()) {
        // P(x_j, x_{j+e}) = P(y_j, y_{j+e}), 3 e columns apart
        for (int e = 0; e <= 3 && j + e < p; ++e) {
            double s = 0.0;
            for (int i = (j + e - 3 > 0 ? j + e - 3 : 0); i <= j; ++i) {
                if (i <= p - 3 && j + e <= i + 2) s += dds_coef(j - i) * dds_coef(j + e - i) * cw.curvature;
                if (i <= p - 4) s += ddds_coef(j - i) * ddds_coef(j + e - i) * cw.curvature_rate;   // the i != size - 3 rule
            }
            W.Pb[(size_t)(3 * j) * S + 3 * e] = s;
            W.Pb[(size_t)(3 * j + 1) * S + 3 * e] = s;
        }
        W.Pb[(size_t)(3 * j + 2) * S] = cw.deviation;
        W.q[3 * j] = W.q[3 * j + 1] = W.q[3 * j + 2] = 0.0;
        const double theta = al[j] + M_PI_2;
        int r = 3 * j;
        W.Ac[r * kEll + 0] = (int16_t)(3 * j);      W.Av[r * kEll + 0] = 1;
        W.Ac[r * kEll + 1] = (int16_t)(3 * j + 2);  W.Av[r * kEll + 1] = -cos(theta);
        W.l[r] = W.u[r] = xl[j];
        r = 3 * j + 1;
        W.Ac[r * kEll + 0] = (int16_t)(3 * j + 1);  W.Av[r * kEll + 0] = 1;
        W.Ac[r * kEll + 1] = (int16_t)(3 * j + 2);  W.Av[r * kEll + 1] = -sin(theta);
        W.l[r] = W.u[r] = yl[j];
        r = 3 * j + 2;
        W.Ac[r * kEll] = (int16_t)(3 * j + 2);      W.Av[r * kEll] = 1;
        double lo, hi;
        if (j == 0) {
            lo = hi = 0.0;
        } else if (j == p - 1) {
            lo = -0.5;
            hi = 0.5;
        } else {
            // std::min(clearance, 2): the clearance unless 2 is smaller (Map::getObstacleDistance, 0 off the map)
            const double cr = kCartesianDefaultClearance < cl[j] ? kCartesianDefaultClearance : cl[j];
            lo = -cr;
            hi = cr;
        }
        W.l[r] = lo;
        W.u[r] = hi;
    }
    c.sync();
}

// column lists of A from the row lists; rows are visited in ascending order, so every column's list is sorted by
// row and sums over a column always run in the same order (deterministic rounding)
template <class Ctx>
PQS_HD void build_columns(const Ctx &c, Work &W) {
    for (int j = c.lane(); j < W.N; j += c.lanes()) {
        W.cnt[j] = 0;
        for (int e = 0; e < kEll; ++e) { W.Cr[j * kEll + e] = -1; W.Ce[j * kEll + e] = 0; }
    }
    c.sync();
    if (c.lane() == 0) {
        for (int r = 0; r < W.M; ++r)
            for (int e = 0; e < kEll; ++e) {
                const int col = W.Ac[r * kEll + e];
                if (col < 0) continue;
                const int k = W.cnt[col];
                if (k < kEll) {
                    W.Cr[col * kEll + k] = (int16_t)r;
                    W.Ce[col * kEll + k] = (int8_t)e;
                    W.cnt[col] = (int8_t)(k + 1);
                }
            }
    }
    c.sync();
}

// ------------------------------------------------------------------ small kernels on the working set
template <class Ctx> PQS_HD void mat_vec_A(const Ctx &c, const Work &W, const double *x, double *out) {   // out = A x
    for (int r = c.lane(); r < W.M; r += c.lanes()) {
        double s = 0.0;
        for (int e = 0; e < kEll; ++e) {
            const int col = W.Ac[r * kEll + e];
            if (col >= 0) s += W.Av[r * kEll + e] * x[col];
        }
        out[r] = s;
    }
}
template <class Ctx> PQS_HD void mat_tvec_A(const Ctx &c, const Work &W, const double *y, double *out) {  // out = A' y
    for (int j = c.lane(); j < W.N; j += c.lanes()) {
        double s = 0.0;
        for (int e = 0; e < kEll; ++e) {
            const int r = W.Cr[j * kEll + e];
            if (r >= 0) s += W.Av[r * kEll + W.Ce[j * kEll + e]] * y[r];
        }
        out[j] = s;
    }
}
template <int HBP, class Ctx> PQS_HD void mat_vec_P(const Ctx &c, const Work &W, const double *x, double *out) {   // out = P x (symmetric band)
    for (int j = c.lane(); j < W.N; j += c.lanes()) {
        double s = W.Pb[(size_t)j * (HBP + 1)] * x[j];
        for (int d = 1; d <= HBP; ++d) {
            if (j + d < W.N) s += W.Pb[(size_t)j * (HBP + 1) + d] * x[j + d];
            if (j - d >= 0) s += W.Pb[(size_t)(j - d) * (HBP + 1) + d] * x[j - d];
        }
        out[j] = s;
    }
}
template <class Ctx> PQS_HD double inf_norm(const Ctx &c, const double *v, int n) {
    double m = 0.0;
    for (int i = c.lane(); i < n; i += c.lanes()) m = dmax2(m, dabs(v[i]));
    return c.max(m);
}
template <class Ctx> PQS_HD double inf_norm_scaled(const Ctx &c, const double *s, const double *v, int n, bool inverse) {
    double m = 0.0;
    for (int i = c.lane(); i < n; i += c.lanes()) m = dmax2(m, dabs(inverse ? v[i] / s[i] : v[i] * s[i]));
    return c.max(m);
}

// OSQP scale_data (App. B.2) on band-P / ELL-A
template <int HBP, class Ctx>
PQS_HD void scale_data(const Ctx &c, Work &W, int passes) {
    const int N = W.N, M = W.M;
    for (int j = c.lane(); j < N; j += c.lanes()) W.D[j] = 1.0;
    for (int r = c.lane(); r < M; r += c.lanes()) W.E[r] = 1.0;
    double cs = 1.0;
    c.sync();
    for (int pass = 0; pass < passes; ++pass) {
        // column norms of [P; A] -> t1 (Dt), row norms of A -> t2 (Et)
        for (int j = c.lane(); j < N; j += c.lanes()) {
            double m = dabs(W.Pb[(size_t)j * (HBP + 1)]);
            for (int d = 1; d <= HBP; ++d) {
                if (j + d < N) m = dmax2(m, dabs(W.Pb[(size_t)j * (HBP + 1) + d]));
                if (j - d >= 0) m = dmax2(m, dabs(W.Pb[(size_t)(j - d) * (HBP + 1) + d]));
            }
            for (int e = 0; e < kEll; ++e) {
                const int r = W.Cr[j * kEll + e];
                if (r >= 0) m = dmax2(m, dabs(W.Av[r * kEll + W.Ce[j * kEll + e]]));
            }
            W.t1[j] = 1.0 / sqrt(lim_scaling(m));
        }
        for (int r = c.lane(); r < M; r += c.lanes()) {
            double m = 0.0;
            for (int e = 0; e < kEll; ++e)
                if (W.Ac[r * kEll + e] >= 0) m = dmax2(m, dabs(W.Av[r * kEll + e]));
            W.t2[r] = 1.0 / sqrt(lim_scaling(m));
        }
        c.sync();
        for (int j = c.lane(); j < N; j += c.lanes()) {
            for (int d = 0; d <= HBP; ++d)
                if (j + d < N) W.Pb[(size_t)j * (HBP + 1) + d] *= W.t1[j] * W.t1[j + d];
            W.q[j] *= W.t1[j];
            W.D[j] *= W.t1[j];
        }
        for (int r = c.lane(); r < M; r += c.lanes()) {
            for (int e = 0; e < kEll; ++e) {
                const int col = W.Ac[r * kEll + e];
                if (col >= 0) W.Av[r * kEll + e] *= W.t2[r] * W.t1[col];
            }
            W.E[r] *= W.t2[r];
        }
        c.sync();
        // cost scaling: 1 / max(mean column norm of P, |q|_inf), both limited
        double psum = 0.0, qmax = 0.0;
        for (int j = c.lane(); j < N; j += c.lanes()) {
            double m = dabs(W.Pb[(size_t)j * (HBP + 1)]);
            for (int d = 1; d <= HBP; ++d) {
                if (j + d < N) m = dmax2(m, dabs(W.Pb[(size_t)j * (HBP + 1) + d]));
                if (j - d >= 0) m = dmax2(m, dabs(W.Pb[(size_t)(j - d) * (HBP + 1) + d]));
            }
            psum += m;
            qmax = dmax2(qmax, dabs(W.q[j]));
        }
        psum = c.sum(psum);
        qmax = c.max(qmax);
        double ct = dmax2(psum / N, lim_scaling(qmax));
        ct = 1.0 / lim_scaling(ct);
        for (int j = c.lane(); j < N; j += c.lanes()) {
            for (int d = 0; d <= HBP; ++d) W.Pb[(size_t)j * (HBP + 1) + d] *= ct;
            W.q[j] *= ct;
        }
        cs *= ct;
        c.sync();
    }
    W.c = cs;
    for (int r = c.lane(); r < M; r += c.lanes()) {
        W.l[r] *= W.E[r];
        W.u[r] *= W.E[r];
    }
    c.sync();
}

template <class Ctx>
PQS_HD void set_rho_vec(const Ctx &c, Work &W, bool classify) {
    for (int r = c.lane(); r < W.M; r += c.lanes()) {
        if (classify) {
            const bool loose = W.l[r] < -1e30 * 1e-4 && W.u[r] > 1e30 * 1e-4;
            W.ctype[r] = loose ? -1 : ((W.u[r] - W.l[r] < 1e-4) ? 1 : 0);
        }
        W.rho_vec[r] = W.ctype[r] == -1 ? 1e-6 : (W.ctype[r] == 1 ? 1e3 * W.rho : W.rho);
    }
    c.sync();
}

// band of P + sigma I + A' diag(rho) A, then LDL' in place; false on a non-positive pivot
template <int HB, int HBP, class Ctx>
PQS_HD bool factor(const Ctx &c, Work &W, double sigma) {
    static_assert(HBP <= HB, "the band of P lies inside the band of the reduced matrix");
    const int N = W.N;
    for (int j = c.lane(); j < W.Np; j += c.lanes()) {
        double *row = W.Lb + (size_t)j * (HB + 1);
        for (int d = 0; d <= HB; ++d) row[d] = 0.0;
        if (j >= N) {
            row[0] = 1.0;  // padding rows: identity
            continue;
        }
        for (int d = 0; d <= HBP; ++d) row[d] = W.Pb[(size_t)j * (HBP + 1) + d];
        row[0] += sigma;
        for (int e = 0; e < kEll; ++e) {
            const int r = W.Cr[j * kEll + e];
            if (r < 0) continue;
            const double aj = W.Av[r * kEll + W.Ce[j * kEll + e]] * W.rho_vec[r];
            for (int f = 0; f < kEll; ++f) {
                const int col = W.Ac[r * kEll + f];
                if (col >= j && col - j <= HB) row[col - j] += aj * W.Av[r * kEll + f];
            }
        }
    }
    c.sync();
    int ok = 1;
    for (int j = 0; j < N; ++j) {
        double *row = W.Lb + (size_t)j * (HB + 1);
        const double dj = row[0];
        if (!(dj > 0.0)) ok = 0;
        // lanes a = 1 .. HB update row j + a with the multipliers of column j
        for (int a = 1 + c.lane(); a <= HB; a += c.lanes()) {
            const double la = row[a] / dj;
            double *ra = W.Lb + (size_t)(j + a) * (HB + 1);
            for (int b = a; b <= HB; ++b) ra[b - a] -= la * row[b];
        }
        c.sync();
        for (int a = 1 + c.lane(); a <= HB; a += c.lanes()) row[a] /= dj;
        c.sync();
    }
    return c.all(ok) != 0;
}

// solve (LDL') w = w in place
template <int HB, class Ctx>
PQS_HD void band_solve(const Ctx &c, Work &W) {
    const int N = W.N;
    for (int j = 0; j < N; ++j) {
        const double bj = W.w[j];
        const double *row = W.Lb + (size_t)j * (HB + 1);
        for (int i = 1 + c.lane(); i <= HB; i += c.lanes()) W.w[j + i] -= row[i] * bj;
        c.sync();
    }
    for (int j = c.lane(); j < N; j += c.lanes()) W.w[j] /= W.Lb[(size_t)j * (HB + 1)];
    c.sync();
    for (int j = N - 1; j >= 0; --j) {
        const double *row = W.Lb + (size_t)j * (HB + 1);
        if (c.lane() == 0) {
            double s = 0.0;
            for (int i = 1; i <= HB; ++i) s += row[i] * W.w[j + i];
            W.w[j] -= s;
        }
        c.sync();
    }
}

struct Result { int status, iters, rho_updates; double pri_res, dua_res, obj; };

// Sizes of a working set for QPs of up to n_max variables and m_max rows, and the carving of one QP's working set
// out of a flat scratch block (8-byte aligned) plus its band block (Lb + w, shared memory in the kernel).
template <int HB>
PQS_HD size_t band_doubles(int n_max) { return (size_t)(n_max + HB) * (HB + 1) + (size_t)(n_max + HB); }  // Lb + w
template <int HB, int HBP>
PQS_HD size_t scratch_bytes(int n_max, int m_max) {
    const size_t N = n_max, M = m_max, Np = N + HB;
    size_t d = Np * (HBP + 1) + N /*q*/ + M * kEll /*Av*/ + 2 * M /*l,u*/ + N + M /*D,E*/ + M /*rho*/ + N + 2 * M /*x,z,y*/ + N /*xp*/ +
               M /*dy*/ + 2 * (N > M ? N : M) /*t1,t2*/;
    size_t b = d * sizeof(double) + (M * kEll + N * kEll) * sizeof(int16_t) + (N * kEll + N + M) * sizeof(int8_t);
    return (b + 15) & ~(size_t)15;
}
template <int HB, int HBP>
PQS_HD void carve(Work &W, unsigned char *base, int n_max, int m_max, double *band) {
    const size_t N = n_max, M = m_max, Np = N + HB, T = N > M ? N : M;
    W.Np = (int)Np;
    double *d = reinterpret_cast<double *>(base);
    W.Pb = d; d += Np * (HBP + 1);
    W.q = d; d += N;
    W.Av = d; d += M * kEll;
    W.l = d; d += M;
    W.u = d; d += M;
    W.D = d; d += N;
    W.E = d; d += M;
    W.rho_vec = d; d += M;
    W.x = d; d += N;
    W.z = d; d += M;
    W.y = d; d += M;
    W.xp = d; d += N;
    W.dy = d; d += M;
    W.t1 = d; d += T;
    W.t2 = d; d += T;
    int16_t *h = reinterpret_cast<int16_t *>(d);
    W.Ac = h; h += M * kEll;
    W.Cr = h; h += N * kEll;
    int8_t *b = reinterpret_cast<int8_t *>(h);
    W.Ce = b; b += N * kEll;
    W.cnt = b; b += N;
    W.ctype = b;
    W.Lb = band;
    W.w = band + Np * (HB + 1);
}

// The two handle shapes. TENSION2 and post (bandwidth 4) share one working set of p_max points / layers (tension:
// N = 4 p - 1, M = 3 p - 1; post: N = 3 p, M = 3 p - 2); the Cartesian QP (bandwidth 9) has N = M = 3 p.
PQS_HD int n_max_of(int p_max) { return 4 * p_max; }
PQS_HD int m_max_of(int p_max) { return 3 * p_max + 2; }
PQS_HD size_t band_doubles(int p_max) { return band_doubles<kHB>(n_max_of(p_max)); }
PQS_HD size_t scratch_bytes(int p_max) { return scratch_bytes<kHB, kHBP>(n_max_of(p_max), m_max_of(p_max)); }
PQS_HD void carve(Work &W, unsigned char *base, int p_max, double *band) {
    carve<kHB, kHBP>(W, base, n_max_of(p_max), m_max_of(p_max), band);
}
PQS_HD size_t cartesian_band_doubles(int p_max) { return band_doubles<kHBC>(3 * p_max); }
PQS_HD size_t cartesian_scratch_bytes(int p_max) { return scratch_bytes<kHBC, kHBC>(3 * p_max, 3 * p_max); }
PQS_HD void cartesian_carve(Work &W, unsigned char *base, int p_max, double *band) {
    carve<kHBC, kHBC>(W, base, 3 * p_max, 3 * p_max, band);
}

// OSQP on the assembled working set (cold start). Follows oracle/osqp_generic.py step for step.
template <int HB, int HBP, class Ctx>
PQS_HD Result solve(const Ctx &c, Work &W, const Settings &st) {
    const int N = W.N, M = W.M;
    Result R;
    R.status = -1;
    R.iters = 0;
    R.rho_updates = 0;
    R.pri_res = R.dua_res = R.obj = 0.0;
    build_columns(c, W);
    scale_data<HBP>(c, W, st.scaling);
    W.rho = dmin2(dmax2(st.rho, 1e-6), 1e6);
    set_rho_vec(c, W, true);
    for (int j = c.lane(); j < W.Np; j += c.lanes()) {
        W.w[j] = 0.0;
        if (j < N) W.x[j] = 0.0;
    }
    for (int r = c.lane(); r < M; r += c.lanes()) W.z[r] = W.y[r] = W.dy[r] = 0.0;
    c.sync();
    if (!factor<HB, HBP>(c, W, st.sigma)) {
        R.status = kNumerical;
        return R;
    }
    const double cinv = 1.0 / W.c;
    bool can_check = false;
    int it = 0;
    double n_rp = 0, n_rd = 0, n_z = 0, n_ax = 0, n_q = 0, n_aty = 0, n_px = 0;         // scaled-space norms (rho estimate)
    double u_rp = 0, u_rd = 0, u_z = 0, u_ax = 0, u_q = 0, u_aty = 0, u_px = 0;         // unscaled norms (termination)
    for (it = 1; it <= st.max_iter; ++it) {
        // rhs = sigma x - q + A'(rho z - y)
        for (int r = c.lane(); r < M; r += c.lanes()) W.t2[r] = W.rho_vec[r] * W.z[r] - W.y[r];
        c.sync();
        mat_tvec_A(c, W, W.t2, W.t1);
        c.sync();
        for (int j = c.lane(); j < N; j += c.lanes()) {
            W.xp[j] = W.x[j];
            W.w[j] = st.sigma * W.x[j] - W.q[j] + W.t1[j];
        }
        c.sync();
        band_solve<HB>(c, W);             // w = x~
        mat_vec_A(c, W, W.w, W.t2);       // t2 = z~ = A x~
        c.sync();
        for (int j = c.lane(); j < N; j += c.lanes()) W.x[j] = st.alpha * W.w[j] + (1.0 - st.alpha) * W.xp[j];
        for (int r = c.lane(); r < M; r += c.lanes()) {
            const double zh = st.alpha * W.t2[r] + (1.0 - st.alpha) * W.z[r];
            const double zn = dmin2(dmax2(zh + W.y[r] / W.rho_vec[r], W.l[r]), W.u[r]);
            W.dy[r] = W.rho_vec[r] * (zh - zn);
            W.y[r] += W.dy[r];
            W.z[r] = zn;
        }
        c.sync();
        can_check = st.check_termination && (it % st.check_termination == 0);
        const bool can_adapt = st.adaptive_rho && st.adaptive_rho_interval && (it % st.adaptive_rho_interval == 0);
        if (!(can_check || can_adapt)) continue;
        // ---- info: residuals on unscaled quantities (t1 = P x, t2 = A x; A'y recomputed into w afterwards)
        mat_vec_A(c, W, W.x, W.t2);
        mat_vec_P<HBP>(c, W, W.x, W.t1);
        c.sync();
        {
            double a = 0, b = 0, d = 0, e = 0, f = 0, g = 0, obj = 0;
            for (int r = c.lane(); r < M; r += c.lanes()) {
                const double rp = W.t2[r] - W.z[r], ei = 1.0 / W.E[r];
                a = dmax2(a, dabs(rp)); b = dmax2(b, dabs(W.z[r])); d = dmax2(d, dabs(W.t2[r]));
                e = dmax2(e, dabs(ei * rp)); f = dmax2(f, dabs(ei * W.z[r])); g = dmax2(g, dabs(ei * W.t2[r]));
            }
            n_rp = c.max(a); n_z = c.max(b); n_ax = c.max(d); u_rp = c.max(e); u_z = c.max(f); u_ax = c.max(g);
            for (int j = c.lane(); j < N; j += c.lanes()) obj += 0.5 * W.x[j] * W.t1[j] + W.q[j] * W.x[j];
            R.obj = cinv * c.sum(obj);
        }
        mat_tvec_A(c, W, W.y, W.w);  // w = A'y (w is free between solves)
        c.sync();
        {
            double a = 0, b = 0, d = 0, e = 0, f = 0, g = 0, hq = 0, hu = 0;
            for (int j = c.lane(); j < N; j += c.lanes()) {
                const double rd = W.t1[j] + W.q[j] + W.w[j], di = 1.0 / W.D[j];
                a = dmax2(a, dabs(rd)); b = dmax2(b, dabs(W.w[j])); d = dmax2(d, dabs(W.t1[j])); hq = dmax2(hq, dabs(W.q[j]));
                e = dmax2(e, dabs(di * rd)); f = dmax2(f, dabs(di * W.w[j])); g = dmax2(g, dabs(di * W.t1[j])); hu = dmax2(hu, dabs(di * W.q[j]));
            }
            n_rd = c.max(a); n_aty = c.max(b); n_px = c.max(d); n_q = c.max(hq);
            u_rd = cinv * c.max(e); u_aty = c.max(f); u_px = c.max(g); u_q = c.max(hu);
        }
        R.pri_res = u_rp;
        R.dua_res = u_rd;
        if (can_check) {
            // check_termination (exact tolerances)
            const double ep = st.eps_abs + st.eps_rel * dmax2(u_z, u_ax);
            const double ed = st.eps_abs + st.eps_rel * cinv * dmax2(u_q, dmax2(u_aty, u_px));
            const bool pok = u_rp < ep, dok = u_rd < ed;
            if (pok && dok) { R.status = kSolved; break; }
            // primal infeasibility (is_primal_infeasible)
            if (!pok) {
                double nrm = 0, lhs = 0;
                for (int r = c.lane(); r < M; r += c.lanes()) {
                    const bool uinf = W.u[r] > 1e30 * 1e-4, linf = W.l[r] < -1e30 * 1e-4;
                    double d = W.dy[r];
                    d = (uinf && linf) ? 0.0 : (uinf ? dmin2(d, 0.0) : (linf ? dmax2(d, 0.0) : d));
                    W.t2[r] = d;
                    nrm = dmax2(nrm, dabs(W.E[r] * d));
                    lhs += (uinf ? 0.0 : W.u[r]) * dmax2(d, 0.0) + (linf ? 0.0 : W.l[r]) * dmin2(d, 0.0);
                }
                nrm = c.max(nrm);
                lhs = c.sum(lhs);
                c.sync();
                if (nrm > st.eps_prim_inf && lhs < -st.eps_prim_inf * nrm) {
                    mat_tvec_A(c, W, W.t2, W.w);
                    c.sync();
                    if (inf_norm_scaled(c, W.D, W.w, N, true) < st.eps_prim_inf * nrm) { R.status = kPrimInf; break; }
                }
            }
            // dual infeasibility (is_dual_infeasible)
            if (!dok) {
                double nrm = 0, qdx = 0;
                for (int j = c.lane(); j < N; j += c.lanes()) {
                    const double dx = W.x[j] - W.xp[j];
                    W.w[j] = dx;
                    nrm = dmax2(nrm, dabs(W.D[j] * dx));
                    qdx += W.q[j] * dx;
                }
                nrm = c.max(nrm);
                qdx = c.sum(qdx);
                c.sync();
                if (nrm > st.eps_dual_inf && qdx < -W.c * st.eps_dual_inf * nrm) {
                    mat_vec_P<HBP>(c, W, W.w, W.t1);
                    c.sync();
                    if (inf_norm_scaled(c, W.D, W.t1, N, true) < W.c * st.eps_dual_inf * nrm) {
                        mat_vec_A(c, W, W.w, W.t2);
                        c.sync();
                        int okc = 1;
                        for (int r = c.lane(); r < M; r += c.lanes()) {
                            const bool uinf = W.u[r] > 1e30 * 1e-4, linf = W.l[r] < -1e30 * 1e-4;
                            const double adx = W.t2[r] / W.E[r];
                            if (!uinf && !(adx < st.eps_dual_inf * nrm)) okc = 0;
                            if (!linf && !(adx > -st.eps_dual_inf * nrm)) okc = 0;
                        }
                        if (c.all(okc)) { R.status = kDualInf; break; }
                    }
                }
            }
        }
        if (can_adapt) {
            const double pri = n_rp / (dmax2(n_z, n_ax) + 1e-10);
            const double dua = n_rd / (dmax2(n_q, dmax2(n_aty, n_px)) + 1e-10);
            const double est = dmin2(dmax2(W.rho * sqrt(pri / (dua + 1e-10)), 1e-6), 1e6);
            if (est > W.rho * st.adaptive_rho_tolerance || est < W.rho / st.adaptive_rho_tolerance) {
                W.rho = est;
                set_rho_vec(c, W, false);
                ++R.rho_updates;
                if (!factor<HB, HBP>(c, W, st.sigma)) { R.status = kNumerical; break; }
            }
        }
    }
    R.iters = it > st.max_iter ? st.max_iter : it;
    if (R.status < 0) {
        // the 10x re-check of osqp_solve after the last iteration on the residuals of the last info (max_iter is
        // a multiple of the check interval with OSQP's defaults). The "inaccurate" infeasibility certificates are not
        // re-evaluated: the QPs are feasible by construction (dynamics rows + a non-empty corridor; in the Cartesian QP
        // x_i, y_i absorb any d_i in its range, which contains 0).
        const double ep = 10 * (st.eps_abs + st.eps_rel * dmax2(u_z, u_ax));
        const double ed = 10 * (st.eps_abs + st.eps_rel * cinv * dmax2(u_q, dmax2(u_aty, u_px)));
        R.status = (u_rp < ep && u_rd < ed) ? kSolvedInacc : kMaxIter;
    }
    return R;
}

// One QP end to end: tension smoother. Outputs in the reference's terms: result_x / result_y (QPSolution(i),
// QPSolution(p + i)), result_s re-accumulated from them (tension_smoother_2.cpp:58-70), optionally the whole primal
// vector in the reference's index order (x block, y block, theta block, k block).
template <class Ctx>
PQS_HD Result tension_smooth(const Ctx &c, Work &W, const Settings &st, const TensionWeights &tw, int p, const double *xl,
                             const double *yl, const double *al, const double *kl, const double *sl, double *rx, double *ry,
                             double *rs, double *x_full) {
    assemble_tension(c, W, p, xl, yl, al, kl, sl, tw);
    const Result R = solve<kHB, kHBP>(c, W, st);
    for (int i = c.lane(); i < p; i += c.lanes()) {
        rx[i] = W.D[4 * i] * W.x[4 * i];
        ry[i] = W.D[4 * i + 1] * W.x[4 * i + 1];
        if (x_full) {
            x_full[i] = rx[i];
            x_full[p + i] = ry[i];
            x_full[2 * p + i] = W.D[4 * i + 2] * W.x[4 * i + 2];
            if (i < p - 1) x_full[3 * p + i] = W.D[4 * i + 3] * W.x[4 * i + 3];
        }
    }
    c.sync();
    if (c.lane() == 0) {
        double tmp_s = 0;
        for (int i = 0; i < p; ++i) {
            if (i != 0) tmp_s += sqrt(pow(rx[i] - rx[i - 1], 2) + pow(ry[i] - ry[i - 1], 2));
            rs[i] = tmp_s;
        }
    }
    c.sync();
    return R;
}

// postSmooth's QP: offsets[i] = QPSolution(i) (the lateral offset of layer i, reference_path_smoother.cpp:566-567);
// x_full optional: x block, dx block, ddx block.
template <class Ctx>
PQS_HD Result post_smooth(const Ctx &c, Work &W, const Settings &st, const PostWeights &pw, int p, const double *layer_s,
                          const double *lower, const double *upper, double vehicle_l, double *offsets, double *x_full) {
    assemble_post(c, W, p, layer_s, lower, upper, vehicle_l, pw);
    const Result R = solve<kHB, kHBP>(c, W, st);
    for (int i = c.lane(); i < p; i += c.lanes()) {
        offsets[i] = W.D[3 * i] * W.x[3 * i];
        if (x_full) {
            x_full[i] = offsets[i];
            x_full[p + i] = W.D[3 * i + 1] * W.x[3 * i + 1];
            x_full[2 * p + i] = W.D[3 * i + 2] * W.x[3 * i + 2];
        }
    }
    c.sync();
    return R;
}

// One QP end to end: Cartesian tension smoother (TensionSmoother::osqpSmooth, tension_smoother.cpp:49-100). Inputs:
// the resampled points, their headings and the obstacle distance at each point (Map::getObstacleDistance; read for
// the interior points only). Outputs as tension_smooth: result_x / result_y (QPSolution(i), QPSolution(p + i)),
// result_s re-accumulated from them, optionally the whole primal vector in the reference's index order (x block,
// y block, d block).
template <class Ctx>
PQS_HD Result cartesian_tension_smooth(const Ctx &c, Work &W, const Settings &st, const CartesianWeights &cw, int p,
                                       const double *xl, const double *yl, const double *al, const double *cl,
                                       double *rx, double *ry, double *rs, double *x_full) {
    assemble_cartesian(c, W, p, xl, yl, al, cl, cw);
    const Result R = solve<kHBC, kHBC>(c, W, st);
    for (int i = c.lane(); i < p; i += c.lanes()) {
        rx[i] = W.D[3 * i] * W.x[3 * i];
        ry[i] = W.D[3 * i + 1] * W.x[3 * i + 1];
        if (x_full) {
            x_full[i] = rx[i];
            x_full[p + i] = ry[i];
            x_full[2 * p + i] = W.D[3 * i + 2] * W.x[3 * i + 2];
        }
    }
    c.sync();
    if (c.lane() == 0) {
        double tmp_s = 0;
        for (int i = 0; i < p; ++i) {
            if (i != 0) tmp_s += sqrt(pow(rx[i] - rx[i - 1], 2) + pow(ry[i] - ry[i - 1], 2));
            rs[i] = tmp_s;
        }
    }
    c.sync();
    return R;
}

}  // namespace pqs
