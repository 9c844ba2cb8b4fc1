// pqp_kernel.cuh — one warp per path-QP: assembly + OSQP-style ADMM, state in shared memory.
//
// What it computes (reference file:line it replaces):
//   assembly of P, A, l, u             /root/reference/src/solver/base_solver.cpp:119-261,290-296
//   OSQP setup (Ruiz scaling, rho vec) base_solver.cpp:87   (osqp_setup through osqp-eigen)
//   OSQP ADMM loop, termination, rho   base_solver.cpp:88,110
//   warm update of A and bounds        base_solver.cpp:102-107
// How (see DESIGN.md):
//   * one warp per QP instance, lane L owns the C consecutive stages [L*C, L*C+C) of the
//     stage chain (stage 0 is a virtual stage whose outgoing rows are the x0 rows, stage
//     g>=1 is knot g-1, the last knot's outgoing rows are the two end-state rows);
//   * all per-stage data lives in shared memory as [field][k][lane] (conflict-free);
//   * the x-update solves the reduced SPD system (P + S + A'RA) x = rhs exactly:
//     controls and slacks are eliminated in closed form, leaving a block-tridiagonal
//     system in (l, psi, kappa) with 3x3 blocks. It is factored as block LDL' in a
//     nested-dissection order: each lane eliminates its C-1 interior stages serially,
//     the 32 separator stages are eliminated by block cyclic reduction across lanes
//     with warp shuffles;
//   * per-stage loops are rolled and the solve vectors live in shared memory so that the hot
//     loop is a few hundred instructions (the unrolled first version was I-cache bound);
//   * iterates are kept in *unscaled* variables; OSQP's Ruiz scaling (D, E, c) appears as
//     per-row weights R_i = rho_i e_i^2 / c and per-variable weights S_j = sigma/(c d_j^2),
//     which is algebraically identical to OSQP's iteration on the scaled problem;
//   * the dual is stored scaled (yhat = y / R) so the z/y update needs no division.
//
// This header is also compiled for the host by tests/emu (PQP_EMU) where a warp is 32
// cooperative fibers; that build exists only to test this source on the GPU-less build
// box and is never linked into the product.
#pragma once

#include <stdint.h>

#ifdef PQP_EMU
#include <cmath>
#include "warp_emu.h"
#define PQP_DEV inline
#define PQP_RESTRICT
struct alignas(16) float4 { float x, y, z, w; };
#else
#include <cuda_runtime.h>
#define PQP_DEV __device__ __forceinline__
#define PQP_RESTRICT __restrict__
#endif

namespace pqp {

// ------------------------------------------------------------------ constants (OSQP 0.6.x)
constexpr double kOsqpInfty = 1e30;
constexpr double kMinScaling = 1e-4;
constexpr double kMaxScaling = 1e4;
constexpr double kRhoMin = 1e-6;
constexpr double kRhoMax = 1e6;
constexpr double kRhoEqOverIneq = 1e3;
constexpr double kRhoTol = 1e-4;

// status codes: keep in sync with include/pqp.h
constexpr int kSolved = 0, kMaxIter = 1, kPrimInf = 2, kDualInf = 3, kSolvedInacc = 4,
              kPrimInfInacc = 5, kNumerical = 7, kUnsolved = 10;

// ------------------------------------------------------------------ shared-memory field map
// Per-stage data is stored as 18 float4 groups; element (group g, local stage k, lane) is the
// float4 at index (g*C + k)*32 + lane, so a warp's access to one group of one stage is one
// conflict-free 512-byte LDS.128/STS.128. The logical field number f = 4*g + component.
// Groups 0-6 are read-only inside the ADMM loop (in the increment form the FS slots of groups 5-6
// are rewritten every iteration), 7-11 are read-write, 12-17 are the factor.
enum : int {
    FA = 0,     // 6: a00 a01 a10 a11 | a12 ds        (stage transition coefficients)
    FE = 6,     // 3: 1/m_u 1/m_s0 | 1/m_s1            (closed-form elimination constants)
    FOB = 9,    // 3: outgoing-row bound (lower; upper = lower [+ end-row width])
    FOR_ = 12,  // 3: outgoing-row weight R
    FKR = 15,   //    kappa-row weight R
    FCLO = 16, FCHI = 18,  // clearance-row bounds (2 each)
    FCR = 20,   // 2: clearance-row weights R
    FS = 22,    // 6: S_j = sigma / (c d_j^2) (proximal weights) in the textbook form; in the
                //    increment form the carried row values A x of the stage's six rows
    FX = 28,    // 6: l, psi, kappa, u | s0, s1        (primal iterate x)
    FKZ = 34, FKY = 35,    // kappa box row: z, yhat
    FOY = 36,   // 3: outgoing-row scaled dual yhat    (+1 pad)
    FCZ = 40, FCY = 42,    // clearance rows: z, yhat (2 each)
    FB = 44,    // 3: rhs of the reduced system / x~ after the solve (+1 pad)
    FDI = 48,   // 6: inverse pivot block (sym)
    FG = 54,    // 9: multiplier to the next stage
    FF = 63,    // 9: multiplier to the left separator (fill)
    NFIELD = 72,
    FT = FDI,   // the 24 factor fields double as input staging and as Ruiz scratch
    // float4 group numbers
    GA0 = 0, GA1 = 1, GB2 = 2, GR3 = 3, GC4 = 4, GR5 = 5, GS6 = 6,
    GX0 = 7, GX1 = 8, GOY = 9, GCZ = 10, GBV = 11, GF0 = 12
};
// global per-QP scratch, same [field][k][lane] layout
enum : int {
    WX = 0,    // 6 scaled primal
    WOZ = 6,   // 3 scaled z of outgoing rows
    WOY = 9,   // 3 scaled y of outgoing rows
    WKZ = 12, WKY = 13,
    WCZ = 14, WCY = 16,
    NWARM = 18,
    GD = 0, GE = 6, GCLS = 12, NSCAL = 13,  // D (6 vars), E (6 rows), row-class bitmask (int)
    NDY = 6
};

struct DevParams {
    double front_length, rear_length, kappa_limit, safety_margin, end_l_lb, end_l_ub;
    double w_l, w_kappa, w_dkappa, w_slack;
    double rho0, sigma, alpha, eps_abs, eps_rel, eps_pinf, eps_dinf, rho_tol;
    int max_iter, check_every, scaling, adaptive_rho, adaptive_interval;
    int reserved0;
};

struct KernelArgs {
    DevParams prm;
    int batch, n_max, mode, use_tma;  // mode bit 0: warm start; bit 1: cold-only handle (no warm state is written back)
    int qp0;                          // index of this launch's first instance in the handle's scratch
    const double *knots, *inst;
    const int *n, *p;
    double *sol, *cost;
    int *status, *iters;
    int *work_counter;  // persistent kernels: next instance to take (zeroed before the launch)
    // streamed launch (host API): the kernel starts before the inputs have landed; instance qp
    // belongs to the chunk c with chunk_lo[c] <= qp < chunk_lo[c + 1], whose H2D copy is followed by a write to ready[c];
    // done[chunk] counts finished instances and host_done[chunk] (mapped host memory) is set
    // when a chunk is complete so the host can start its D2H copy. All null for plain launches.
    const int *ready;
    int *done;
    int *host_done;
    int n_chunks;
    int chunk_lo[9];  // chunk boundaries (n_chunks + 1 entries); chunks need not be equal
    int *flags;  // optional: bit 0 = infeasibility suspected (certificate conditions 1-2 held)
    double *x_full, *y_full, *z_full, *info;
    void *warm, *scal, *dy, *rho_state;  // per-instance scratch in the kernel's scalar type
};

// ------------------------------------------------------------------ warp primitives
#ifdef PQP_EMU
template <typename T> PQP_DEV T shfl_up(T v, int d, int lane) {
    return warp_emu::exchange(v, lane, lane - d);
}
template <typename T> PQP_DEV T shfl_down(T v, int d, int lane) {
    return warp_emu::exchange(v, lane, lane + d);
}
template <typename T> PQP_DEV T shfl_xor(T v, int m, int lane) {
    return warp_emu::exchange(v, lane, lane ^ m);
}
PQP_DEV void sync_warp(int lane) { warp_emu::current()->barrier(lane); }
using std::fabs;
using std::fmax;
using std::fmin;
using std::sqrt;
#else
template <typename T> PQP_DEV T shfl_up(T v, int d, int) { return __shfl_up_sync(0xffffffffu, v, d); }
template <typename T> PQP_DEV T shfl_down(T v, int d, int) { return __shfl_down_sync(0xffffffffu, v, d); }
template <typename T> PQP_DEV T shfl_xor(T v, int m, int) { return __shfl_xor_sync(0xffffffffu, v, m); }
PQP_DEV void sync_warp(int) { __syncwarp(); }
#endif

// scalar-type generic math (the kernel is instantiated for float and for double)
PQP_DEV float xmax(float a, float b) { return fmaxf(a, b); }
PQP_DEV double xmax(double a, double b) { return fmax(a, b); }
PQP_DEV float xmin(float a, float b) { return fminf(a, b); }
PQP_DEV double xmin(double a, double b) { return fmin(a, b); }
PQP_DEV float xabs(float a) { return fabsf(a); }
PQP_DEV double xabs(double a) { return fabs(a); }
PQP_DEV float xsqrt(float a) { return sqrtf(a); }
PQP_DEV double xsqrt(double a) { return sqrt(a); }
template <typename T> PQP_DEV T frsqrt(T x) { return T(1) / xsqrt(x); }
// fast reciprocal square root (MUFU.RSQ in FP32); used only for the scaled norms of the rho estimate
#ifdef PQP_EMU
PQP_DEV float xfast_rsqrt(float a) { return 1.0f / std::sqrt(a); }
#else
PQP_DEV float xfast_rsqrt(float a) { return rsqrtf(a); }
#endif
PQP_DEV double xfast_rsqrt(double a) { return 1.0 / sqrt(a); }

template <typename T> PQP_DEV T warp_max(T v, int lane) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) v = xmax(v, shfl_xor(v, m, lane));
    return v;
}
template <typename T> PQP_DEV T warp_sum(T v, int lane) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) v += shfl_xor(v, m, lane);
    return v;
}

template <typename T> PQP_DEV T limit_scaling(T v) {
    v = v < T(kMinScaling) ? T(1) : v;
    return v > T(kMaxScaling) ? T(kMaxScaling) : v;
}
template <typename T> PQP_DEV T clampf(T v, T lo, T hi) { return xmin(xmax(v, lo), hi); }

// 4-wide vector of the kernel's scalar type (one shared-memory "group")
template <typename T> struct Vec4T;
template <> struct Vec4T<float> { typedef float4 type; };
struct alignas(32) pqp_double4 { double x, y, z, w; };
template <> struct Vec4T<double> { typedef pqp_double4 type; };

// ------------------------------------------------------------------ 3x3 helpers
// symmetric 3x3 as [6] = (00,01,02,11,12,22); general 3x3 row-major [9]
PQP_DEV constexpr int SI(int i, int j) {
    return i <= j ? (i == 0 ? j : (i == 1 ? 2 + j : 5)) : (j == 0 ? i : (j == 1 ? 2 + i : 5));
}

// inverse of an SPD 3x3 through its Cholesky factor; returns false on a non-positive pivot
template <typename T> PQP_DEV bool inv_sym3(const T (&a)[6], T (&o)[6]) {
    bool ok = true;
    T p0 = a[0];
    ok = ok && (p0 > T(0));
    T i00 = T(1) / xsqrt(p0);
    T l10 = a[1] * i00, l20 = a[2] * i00;
    T p1 = a[3] - l10 * l10;
    ok = ok && (p1 > T(0));
    T i11 = T(1) / xsqrt(p1);
    T l21 = (a[4] - l20 * l10) * i11;
    T p2 = a[5] - l20 * l20 - l21 * l21;
    ok = ok && (p2 > T(0));
    T i22 = T(1) / xsqrt(p2);
    T i10 = -l10 * i00 * i11;
    T i21 = -l21 * i11 * i22;
    T i20 = -(l20 * i00 + l21 * i10) * i22;
    o[0] = i00 * i00 + i10 * i10 + i20 * i20;
    o[1] = i10 * i11 + i20 * i21;
    o[2] = i20 * i22;
    o[3] = i11 * i11 + i21 * i21;
    o[4] = i21 * i22;
    o[5] = i22 * i22;
    return ok;
}
// out = M * S (general x symmetric)
template <typename T> PQP_DEV void mul_ms(const T (&m)[9], const T (&s)[6], T (&o)[9]) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            o[3 * r + c] = m[3 * r] * s[SI(0, c)] + m[3 * r + 1] * s[SI(1, c)] + m[3 * r + 2] * s[SI(2, c)];
}
// out = A * B' (general)
template <typename T> PQP_DEV void mul_abt(const T (&a)[9], const T (&b)[9], T (&o)[9]) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            o[3 * r + c] = a[3 * r] * b[3 * c] + a[3 * r + 1] * b[3 * c + 1] + a[3 * r + 2] * b[3 * c + 2];
}
// symmetric part of A * B' when the product is known to be symmetric
template <typename T> PQP_DEV void mul_abt_sym(const T (&a)[9], const T (&b)[9], T (&o)[6]) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c)
            o[SI(r, c)] = a[3 * r] * b[3 * c] + a[3 * r + 1] * b[3 * c + 1] + a[3 * r + 2] * b[3 * c + 2];
}

// ------------------------------------------------------------------ per-stage predicates
// gn and a22 are 0 or +-1; the clearance rows' lever arms h0, h1 are in the kernel's scalar type R (rounded to
// FP32 they would put the FP64 instantiation's A 1e-7 relative off the oracle's whenever front_length or
// rear_length is not a float)
template <typename R>
struct StagePredT {
    bool real, mid, last, act0, act1;
    float gn, a22;
    R h0, h1;
};
template <typename R>
PQP_DEV StagePredT<R> stage_pred(int g, int n, int p, R lf, R lr) {
    StagePredT<R> s;
    s.real = (g >= 1) && (g <= n);
    s.mid = (g >= 1) && (g <= n - 1);
    s.last = (g == n);
    s.act0 = s.real;
    s.act1 = (g >= 1) && (g <= p);
    s.gn = (g <= n - 1) ? -1.0f : 0.0f;
    s.a22 = s.mid ? 1.0f : 0.0f;
    s.h0 = s.act1 ? lf : R(0);  // front row for precise stages, centre row (h = 0) otherwise
    s.h1 = s.act1 ? lr : R(0);
    return s;
}

PQP_DEV void soft_bounds(double lb, double ub, double margin, double &olb, double &oub) {
    const double clearance = ub - lb;
    double remain = clearance - 2 * margin;
    remain = remain > 0.1 ? remain : 0.1;
    double shrink = (clearance - remain) / 2.0;
    shrink = shrink > 0.0 ? shrink : 0.0;
    olb = lb + shrink;
    oub = ub - shrink;
}


// ------------------------------------------------------------------ storage policies
// Where a QP's per-stage state lives. Logical field f = 4*group + component; the policy maps
// (field, local stage k, this lane) to storage. Only the owning lane ever touches an element:
// neighbour values travel by warp shuffle, never by cross-lane loads, so the solver code is
// written against the policy's interface (loads in batches, a stage cursor) rather than raw indexing.
template <int C, typename real>
struct SmemStore {
    typedef typename Vec4T<real>::type Vec4;
    real *sm;
    int lane;
    // cyclic-reduction levels unrolled? Several warps share a scheduler and the hot loop should stay small: unrolled
    // only at C <= 2 in FP32, where the levels are a large share of the work (QpWarp widens this for the increment form)
    static constexpr bool kUnrollCr = C <= 2 && sizeof(real) == 4;
    PQP_DEV SmemStore(real *s, int l) : sm(s), lane(l) {}
    PQP_DEV real ld(int f, int k) const { return sm[(((f >> 2) * C + k) * 32 + lane) * 4 + (f & 3)]; }
    PQP_DEV void st(int f, int k, real v) { sm[(((f >> 2) * C + k) * 32 + lane) * 4 + (f & 3)] = v; }
    PQP_DEV Vec4 ld4(int g, int k) const { return reinterpret_cast<const Vec4 *>(sm)[(g * C + k) * 32 + lane]; }
    PQP_DEV void st4(int g, int k, const Vec4 &v) { reinterpret_cast<Vec4 *>(sm)[(g * C + k) * 32 + lane] = v; }
    // n consecutive groups g0.. of stage k into out[4n] (one latency for all of them)
    template <int N> PQP_DEV void ld4n(int g0, int k, real (&out)[4 * N]) const {
#pragma unroll
        for (int g = 0; g < N; ++g) {
            const Vec4 v = ld4(g0 + g, k);
            out[4 * g] = v.x; out[4 * g + 1] = v.y; out[4 * g + 2] = v.z; out[4 * g + 3] = v.w;
        }
    }
    // split form: issue loads, then wait once for all of them (a no-op split under this policy)
    template <int N> PQP_DEV void ld4n_nowait(int g0, int k, real (&out)[4 * N]) const { ld4n<N>(g0, k, out); }
    PQP_DEV void wait_ld() const {}
    PQP_DEV void fence() {}  // stores of this lane are visible to its later loads
    // stage cursor: plain stage indexing under this policy
    PQP_DEV void seek(int) {}
    template <int G0, int N> PQP_DEV void ld_run_nowait(int k, real (&out)[4 * N]) const { ld4n<N>(G0, k, out); }
    template <int G0, int N> PQP_DEV void ld_run_nowait_cur(int k, real (&out)[4 * N]) const { ld4n<N>(G0, k, out); }
    template <int G0, int N> PQP_DEV void ld_run_nowait_ahead(int k, real (&out)[4 * N]) const { ld4n<N>(G0, k < C - 1 ? k + 1 : k, out); }
    PQP_DEV void st4_cur(int g, int k, const Vec4 &v) { st4(g, k, v); }
    template <int N> PQP_DEV void ld4n_nowait_cur(int g0, int k, real (&out)[4 * N]) const { ld4n<N>(g0, k, out); }
    PQP_DEV void ld4_nowait_next(int g, int k, real (&out)[4]) const { ld4n<1>(g, k < C - 1 ? k + 1 : k, out); }
    template <int N> PQP_DEV void ld4n_nowait_ahead(int g0, int k, real (&out)[4 * N]) const { ld4n<N>(g0, k < C - 1 ? k + 1 : k, out); }
    PQP_DEV void ld4_nowait_ahead_next(int g, int k, real (&out)[4]) const { ld4n<1>(g, k < C - 2 ? k + 2 : C - 1, out); }
};

// =========================================================================================
// Which loops are unrolled:
//  * per-stage loops with large bodies (stage update, residuals, set-up) stay rolled (#pragma unroll 1): unrolled,
//    they make a hot loop of tens of KB that thrashes the instruction cache;
//  * the substitution sweeps are fully unrolled: rolled, much of their instruction stream is register copies of the
//    prefetched factor and address arithmetic;
//  * the cyclic-reduction levels are unrolled per storage policy and form (QpWarp::kUnrollCr);
//  * the hot stage-update loop of the increment form is unrolled by two (admm_update_incr<false, false>).
#define PQP_ROLL _Pragma("unroll 1")
#define PQP_SWEEP_UNROLL _Pragma("unroll")
#define PQP_UPDATE_UNROLL _Pragma("unroll 1")
// QpWarp's last template argument selects the ADMM step in increment form (solve
// K dx = -(r_dual + A'R r_prim), x~ = x + dx, with l carried as l + l_lo) instead of the textbook
// form (solve K x~ = S x + A'(R z - y)): algebraically the same iteration, but its rounding error
// scales with |dx| instead of |x|, so the FP32 kernel follows the FP64 oracle's rho schedule
// (tests/test_gpu_parity.py: same iteration count in >= 95 % of instances) at a few per cent more
// instructions per iteration.

template <int C, typename real, typename Store = SmemStore<C, real>, bool Incr = false>
struct QpWarp {
    typedef typename Vec4T<real>::type Vec4;
    typedef StagePredT<real> StagePred;
    // cyclic-reduction levels unrolled (constant shuffle distances and lane masks, no loop bookkeeping between the
    // dependent levels): as the storage policy asks, and in the FP32 increment form up to C = 8, where at most three
    // QPs fit on an SM and each warp has a scheduler to itself (DESIGN §10: 5 % of a C = 8 launch). The textbook form
    // keeps the rolled levels: unrolled, its persistent and one-CTA-per-instance builds round differently.
    static constexpr bool kUnrollCr = Store::kUnrollCr || (Incr && C <= 8 && sizeof(real) == 4);
    const KernelArgs &ka;
    Store store;
    const int lane, qp;
    int n, p;
    real lf, lr, kmax;
    // end rows (valid on the lane/stage that owns knot n-1)
    real zend[2], endw[2];
    // separator (cyclic reduction) factors of this lane
    real crAinv[6], crGm[9], crGp[9];
    // Ruiz cost scaling and current rho
    real cscale, rho;
    // per-lane partial sums of the primal-infeasibility certificate (last check iteration)
    real cert_nrm, cert_lhs;
    int suspect;  // certificate conditions 1-2 held at the last check (warp-uniform)
    // per-QP global scratch
    real *gwarm, *gscal, *gdy;
    // solver parameters in the kernel's scalar type
    real w_l, w_kappa, w_dkappa, w_slack, sigma, alpha, eps_abs, eps_rel, eps_pinf, rho_tol;

    PQP_DEV QpWarp(const KernelArgs &k, const Store &st, int l, int q) : ka(k), store(st), lane(l), qp(q) {}

    // proxy views of the policy-backed state: S(f,k) behaves like a real&, V(g,k) like a Vec4&
    struct SRef {
        Store &st; int f, k;
        PQP_DEV operator real() const { return st.ld(f, k); }
        PQP_DEV SRef &operator=(real v) { st.st(f, k, v); return *this; }
        PQP_DEV SRef &operator=(const SRef &o) { st.st(f, k, (real)o); return *this; }
        PQP_DEV SRef &operator*=(real v) { st.st(f, k, st.ld(f, k) * v); return *this; }
        PQP_DEV SRef &operator+=(real v) { st.st(f, k, st.ld(f, k) + v); return *this; }
        PQP_DEV SRef &operator-=(real v) { st.st(f, k, st.ld(f, k) - v); return *this; }
    };
    struct VRef {
        Store &st; int g, k;
        PQP_DEV operator Vec4() const { return st.ld4(g, k); }
        PQP_DEV VRef &operator=(const Vec4 &v) { st.st4(g, k, v); return *this; }
    };
    PQP_DEV SRef S(int f, int k) { return SRef{store, f, k}; }
    PQP_DEV VRef V(int g, int k) { return VRef{store, g, k}; }
    struct VcRef {  // stage k = the store's cursor stage
        Store &st; int g, k;
        PQP_DEV VcRef &operator=(const Vec4 &v) { st.st4_cur(g, k, v); return *this; }
    };
    PQP_DEV VcRef Vc(int g, int k) { return VcRef{store, g, k}; }
    PQP_DEV real &G(real *base, int f, int k) { return base[(f * C + k) * 32 + lane]; }
    PQP_DEV real &GL(real *base, int f, int k, int ln) { return base[(f * C + k) * 32 + ln]; }
    // row-class bitmask of stage k, kept in the pad component of the yhat group (exact small integer)
    PQP_DEV int cls_of(int k) { return (int)S(FOY + 3, k); }
    PQP_DEV StagePred pred(int k) const { return stage_pred(lane * C + k, n, p, lf, lr); }

    // -------------------------------------------------------------- assembly
    // base_solver.cpp:150-261 for the stage chain; src = this instance's knot block
    PQP_DEV void assemble(const double *src, int stride) {
        const DevParams &P = ka.prm;
        const double *in = ka.inst + (size_t)qp * 5;
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const int g = lane * C + k;
            real a[6] = {0, 0, 0, 0, 0, 0};
            real ob[3] = {0, 0, 0};
            real clo[2] = {0, 0}, chi[2] = {0, 0};
            if (g == 0) {
                ob[0] = (real)(-in[0]);
                ob[1] = (real)(-in[1]);
                ob[2] = (real)(-in[2]);
            } else if (g <= n - 1) {
                const int i = g - 1;
                const double xl = src[2 * stride + i], xp = src[3 * stride + i], xk = src[4 * stride + i];
                const double xkn = src[4 * stride + i + 1];
                const double ds = src[i + 1] - src[i];
                const double kref = src[1 * stride + i];
                const double cp = cos(xp), tp = tan(xp);
                const double f00 = -xk * tp, f01 = (1 - xk * xl) / (cp * cp);
                const double f10 = -xk * xk / cp, f11 = (1 - xk * xl) * xk * tp / cp,
                             f12 = (1 - xk * xl) / cp;
                a[0] = (real)(ds * f00 + 1.0);
                a[1] = (real)(ds * f01);
                a[2] = (real)(ds * f10);
                a[3] = (real)(ds * f11 + 1.0);
                a[4] = (real)(ds * f12);
                a[5] = (real)ds;
                const double u_in = (xkn - xk) / ds;
                const double g0 = (1 - xk * xl) * tp;
                const double g1 = (1 - xk * xl) * xk / cp - kref;
                const double c0 = ds * (g0 - (f00 * xl + f01 * xp));
                const double c1 = ds * (g1 - (f10 * xl + f11 * xp + f12 * xk));
                const double c2 = ds * (u_in - u_in);
                ob[0] = (real)(-c0);
                ob[1] = (real)(-c1);
                ob[2] = (real)(-c2);
            } else if (g == n) {
                a[0] = real(1.0);  // end-l row:   1 * l_{n-1}
                a[3] = real(1.0);  // end-psi row: 1 * psi_{n-1}
                ob[0] = (real)P.end_l_lb;
                endw[0] = (real)(P.end_l_ub - P.end_l_lb);
                ob[1] = (real)in[3];
                endw[1] = (real)(in[4] - in[3]);
            }
            if (g >= 1 && g <= n) {
                const int i = g - 1;
                double lo, hi;
                soft_bounds(src[5 * stride + i], src[6 * stride + i], P.safety_margin, lo, hi);
                clo[0] = (real)lo;
                chi[0] = (real)hi;
                if (g <= p) {
                    soft_bounds(src[7 * stride + i], src[8 * stride + i], P.safety_margin, lo, hi);
                    clo[1] = (real)lo;
                    chi[1] = (real)hi;
                }
            }
            // whole groups (the elimination constants that share groups 1 and 2 are written by the factorisation)
            Vec4 v;
            v.x = a[0]; v.y = a[1]; v.z = a[2]; v.w = a[3];
            store.st4(GA0, k, v);
            v.x = a[4]; v.y = a[5]; v.z = real(0.0); v.w = real(0.0);
            store.st4(GA1, k, v);
            v.x = real(0.0); v.y = ob[0]; v.z = ob[1]; v.w = ob[2];
            store.st4(GB2, k, v);
            v.x = clo[0]; v.y = clo[1]; v.z = chi[0]; v.w = chi[1];
            store.st4(GC4, k, v);
        }
    }

    // -------------------------------------------------------------- Ruiz equilibration
    // OSQP scale_data (SURVEY.md App. B.2) on the structured matrix. d and e ping-pong between
    // two halves of the (still unused) factor region; D, E end up in global scratch, row
    // weights R / classes / S in shared memory.
    // One Ruiz pass: reads D, E from the three groups GF0 + 3 CUR .. (d0 d1 d2 d3 | d4 d5 e0 e1 | e2 e3 e4 e5), writes
    // the other half. Whole groups, one load batch per stage (the stage's a-coefficients, its D / E, the next stage's D)
    // and three group stores, instead of 24 single-value accesses each with its own round trip.
    template <int CUR>
    PQP_DEV void ruiz_pass(real c, real &psum) {
        constexpr int G0 = GF0 + 3 * CUR, G1 = GF0 + 3 * (1 - CUR);
        // neighbour lanes' boundary values: e of the left lane's last outgoing rows, d of the right lane's first x
        real eLb[3], dRb[3];
        {
            real t[8], u[4];
            store.template ld4n_nowait<2>(G0 + 1, C - 1, t);
            store.template ld4n_nowait<1>(G0, 0, u);
            store.wait_ld();
            const real el[3] = {t[2], t[3], t[4]};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                eLb[r] = shfl_up(el[r], 1, lane);
                dRb[r] = shfl_down(u[r], 1, lane);
                if (lane == 0) eLb[r] = real(0.0);
                if (lane == 31) dRb[r] = real(0.0);
            }
        }
        real eL[3] = {eLb[0], eLb[1], eLb[2]};
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            real ta[8], td[12], tn[4];
            store.template ld4n_nowait<2>(GA0, k, ta);
            store.template ld4n_nowait<3>(G0, k, td);
            store.template ld4n_nowait<1>(G0, k < C - 1 ? k + 1 : k, tn);
            store.wait_ld();
            const real a00 = xabs(ta[0]), a01 = xabs(ta[1]), a10 = xabs(ta[2]), a11 = xabs(ta[3]), a12 = xabs(ta[4]),
                       ds = xabs(ta[5]);
            const real gn = xabs(sp.gn), h0 = xabs(sp.h0), h1 = xabs(sp.h1);
            real dk[6], ek[6], dR[3];
#pragma unroll
            for (int j = 0; j < 6; ++j) { dk[j] = td[j]; ek[j] = td[6 + j]; }
#pragma unroll
            for (int r = 0; r < 3; ++r) dR[r] = (k < C - 1) ? tn[r] : dRb[r];
            // the left stage's rows reach this stage's x with coefficient -1 iff 1 <= g <= n
            const real hasL = sp.real ? real(1.0) : real(0.0);
            const real ec0 = sp.act0 ? ek[4] : real(0.0), ec1 = sp.act1 ? ek[5] : real(0.0);
            const real ekap = sp.real ? ek[3] : real(0.0);
            real cn[6];
            cn[0] = dk[0] * xmax(xmax(a00 * ek[0], a10 * ek[1]), xmax(hasL * eL[0], xmax(ec0, ec1)));
            cn[1] = dk[1] * xmax(xmax(a01 * ek[0], a11 * ek[1]), xmax(hasL * eL[1], xmax(h0 * ec0, h1 * ec1)));
            cn[2] = dk[2] * xmax(xmax(a12 * ek[1], sp.a22 * ek[2]), xmax(hasL * eL[2], ekap));
            cn[3] = dk[3] * ds * ek[2];
            cn[4] = dk[4] * ec0;
            cn[5] = dk[5] * ec1;
            const real pw[6] = {sp.real ? w_l : real(0.0), real(0.0), sp.real ? w_kappa : real(0.0),
                                 sp.mid ? w_dkappa : real(0.0), sp.act0 ? w_slack : real(0.0),
                                 sp.act1 ? w_slack : real(0.0)};
#pragma unroll
            for (int j = 0; j < 6; ++j) cn[j] = xmax(cn[j], c * dk[j] * dk[j] * pw[j]);
            real rn[6];
            rn[0] = ek[0] * xmax(xmax(a00 * dk[0], a01 * dk[1]), gn * dR[0]);
            rn[1] = ek[1] * xmax(xmax(a10 * dk[0], a11 * dk[1]), xmax(a12 * dk[2], gn * dR[1]));
            rn[2] = ek[2] * xmax(xmax(sp.a22 * dk[2], ds * dk[3]), gn * dR[2]);
            rn[3] = ekap * dk[2];
            rn[4] = ec0 * xmax(xmax(dk[0], h0 * dk[1]), dk[4]);
            rn[5] = ec1 * xmax(xmax(dk[0], h1 * dk[1]), dk[5]);
            real dn[6], en[6];
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                // 1/sqrt as one MUFU.RSQ in FP32 (2 ulp): the Ruiz factors are only required to be
                // positive - any D, E give an equivalent problem - and a sqrt + divide pair per entry
                // is costly in the set-up; the FP64 instantiation stays exact
                dn[j] = dk[j] * xfast_rsqrt(limit_scaling(cn[j]));
                en[j] = ek[j] * xfast_rsqrt(limit_scaling(rn[j]));
                psum += dn[j] * dn[j] * pw[j];
            }
            Vec4 v;
            v.x = dn[0]; v.y = dn[1]; v.z = dn[2]; v.w = dn[3];
            store.st4(G1, k, v);
            v.x = dn[4]; v.y = dn[5]; v.z = en[0]; v.w = en[1];
            store.st4(G1 + 1, k, v);
            v.x = en[2]; v.y = en[3]; v.z = en[4]; v.w = en[5];
            store.st4(G1 + 2, k, v);
#pragma unroll
            for (int r = 0; r < 3; ++r) eL[r] = ek[r];  // this stage's outgoing-row e is the next stage's "left" e
        }
        store.fence();
    }

    PQP_DEV void scale_and_classify() {
        const DevParams &P = ka.prm;
        {
            Vec4 one;
            one.x = one.y = one.z = one.w = real(1.0);
            PQP_ROLL
            for (int k = 0; k < C; ++k) {
                store.st4(GF0, k, one);
                store.st4(GF0 + 1, k, one);
                store.st4(GF0 + 2, k, one);
            }
            store.fence();
        }
        real c = real(1.0);
        const real nv_inv = real(1.0) / (real)(3 * n + (n - 1) + (p + n));
        int cur = 0;
        for (int pass = 0; pass < P.scaling; ++pass) {
            sync_warp(lane);
            real psum = real(0.0);
            if (cur == 0) ruiz_pass<0>(c, psum);
            else ruiz_pass<1>(c, psum);
            // cost normalisation: c_temp = 1 / limit(max(mean_j |Pbar_jj|, 1))   (q = 0 -> 1)
            const real mean = c * warp_sum(psum, lane) * nv_inv;
            real ct = xmax(mean, real(1.0));
            ct = limit_scaling(ct);
            c = c / ct;
            cur = 1 - cur;
        }
        sync_warp(lane);
        cscale = c;
        if (cur == 0) classify<0>();
        else classify<1>();
    }

    // D, E to global scratch; proximal weights S, row classes and row weights R onto the chip (whole groups)
    template <int CUR>
    PQP_DEV void classify() {
        constexpr int G0 = GF0 + 3 * CUR;
        const real c = cscale;
        const real cinv = real(1.0) / c;
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            real td[12], tb[4], tc[4];
            store.template ld4n_nowait<3>(G0, k, td);
            store.template ld4n_nowait<1>(GB2, k, tb);   // (1/m_s1 | outgoing-row bounds)
            store.template ld4n_nowait<1>(GC4, k, tc);   // clearance-row bounds
            store.wait_ld();
            int cls = 0;
            real e[6], sw[6];
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const real d = td[j];
                e[j] = td[6 + j];
                G(gscal, GD + j, k) = d;
                G(gscal, GE + j, k) = e[j];
                // dummy variables get an identity pivot (accessor calls stay warp-uniform)
                const bool exists = (j == 3) ? sp.mid : (j == 5 ? sp.act1 : sp.real);
                sw[j] = exists ? sigma * cinv / (d * d) : real(1.0);
            }
            real Rw[6];
#pragma unroll
            for (int r = 0; r < 6; ++r) {
                real lo, hi;
                bool act;
                if (r < 3) {
                    lo = tb[1 + r];
                    hi = lo + ((sp.last && r < 2) ? endw[r] : real(0.0));
                    act = (lane * C + k <= n - 1) || (sp.last && r < 2);
                } else if (r == 3) {
                    lo = -kmax; hi = kmax; act = sp.real;
                } else {
                    lo = tc[r - 4]; hi = tc[2 + r - 4];
                    act = (r == 4) ? sp.act0 : sp.act1;
                }
                const real ls = lo * e[r], hs = hi * e[r];
                int cl;
                if (!act) cl = 3;
                else if (ls < real(-kOsqpInfty * kMinScaling) && hs > real(kOsqpInfty * kMinScaling)) cl = 2;
                else if (hs - ls < real(kRhoTol)) cl = 1;
                else cl = 0;
                cls |= cl << (2 * r);
                const real base = (cl == 3) ? real(0.0) : (cl == 2 ? real(kRhoMin) : (cl == 1 ? real(kRhoEqOverIneq) * rho : rho));
                Rw[r] = base * e[r] * e[r] * cinv;
            }
            Vec4 v;
            v.x = Rw[0]; v.y = Rw[1]; v.z = Rw[2]; v.w = Rw[3];
            store.st4(GR3, k, v);                               // FOR_ (3) + FKR
            v.x = Rw[4]; v.y = Rw[5]; v.z = sw[0]; v.w = sw[1];
            store.st4(GR5, k, v);                               // FCR (2) + FS 0..1
            v.x = sw[2]; v.y = sw[3]; v.z = sw[4]; v.w = sw[5];
            store.st4(GS6, k, v);                               // FS 2..5
            S(FOY + 3, k) = (real)cls;
        }
    }

    // -------------------------------------------------------------- iterates: cold / warm
    PQP_DEV void init_iterates(bool warm) {
        const real c = cscale;
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            if (!warm) {
                // whole groups: x (l psi kappa u | s0 s1), kappa-row z / yhat, clearance z / yhat, outgoing yhat
                Vec4 v;
                v.x = v.y = v.z = v.w = real(0.0);
                store.st4(GX0, k, v);
                store.st4(GX1, k, v);
                store.st4(GCZ, k, v);
                v.w = S(FOY + 3, k);  // the row classes ride in the pad component of the yhat group
                store.st4(GOY, k, v);
                if (sp.last) { zend[0] = real(0.0); zend[1] = real(0.0); }
            } else {
                // scaled iterates of the previous solve are re-interpreted in the NEW scaling
                // (OSQP keeps work->x/z/y untouched across osqp_update_A's re-scaling); whole groups again
                real r3[4], r5[4], oyc[4];
                store.template ld4n_nowait<1>(GR3, k, r3);   // Ro0 Ro1 Ro2 Rk
                store.template ld4n_nowait<1>(GR5, k, r5);   // Rc0 Rc1 | ..
                store.template ld4n_nowait<1>(GOY, k, oyc);  // .w = row classes
                store.wait_ld();
                real xv[6], oyn[3], kz, ky, czn[2], cyn[2];
#pragma unroll
                for (int j = 0; j < 6; ++j) xv[j] = G(gwarm, WX + j, k) * G(gscal, GD + j, k);
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const real e = G(gscal, GE + r, k), R = r3[r];
                    const real y = G(gwarm, WOY + r, k) * e / c;
                    oyn[r] = R > real(0.0) ? y / R : real(0.0);
                }
                {
                    const real e = G(gscal, GE + 3, k), R = r3[3];
                    kz = G(gwarm, WKZ, k) / e;
                    ky = R > real(0.0) ? (G(gwarm, WKY, k) * e / c) / R : real(0.0);
                }
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const real e = G(gscal, GE + 4 + j, k), R = r5[j];
                    czn[j] = G(gwarm, WCZ + j, k) / e;
                    cyn[j] = R > real(0.0) ? (G(gwarm, WCY + j, k) * e / c) / R : real(0.0);
                }
                Vec4 v;
                v.x = xv[0]; v.y = xv[1]; v.z = xv[2]; v.w = xv[3];
                store.st4(GX0, k, v);
                v.x = xv[4]; v.y = xv[5]; v.z = kz; v.w = ky;
                store.st4(GX1, k, v);
                v.x = oyn[0]; v.y = oyn[1]; v.z = oyn[2]; v.w = oyc[3];
                store.st4(GOY, k, v);
                v.x = czn[0]; v.y = czn[1]; v.z = cyn[0]; v.w = cyn[1];
                store.st4(GCZ, k, v);
                if (sp.last) {
                    zend[0] = G(gwarm, WOZ + 0, k) / G(gscal, GE + 0, k);
                    zend[1] = G(gwarm, WOZ + 1, k) / G(gscal, GE + 1, k);
                }
            }
        }
    }

    // z of outgoing row r at the start of a (warm) solve, before the first iteration
    PQP_DEV real z0_out(bool warm, int r, int k) {
        return warm ? G(gwarm, WOZ + r, k) / G(gscal, GE + r, k) : real(0.0);
    }

    // -------------------------------------------------------------- factorisation
    // What the factorisation reads of one stage, fetched as whole groups in ONE load batch (~18 values, several of
    // them needed twice).
    struct FacIn {
        real a00, a01, a10, a11, a12, ds, ob[3], Ro[3], Rk, Rc[2], Sw[6];
    };
    PQP_DEV void load_fac(int k, FacIn &q) {
        real t[28];
        store.template ld4n_nowait<7>(GA0, k, t);
        store.wait_ld();
        q.a00 = t[0]; q.a01 = t[1]; q.a10 = t[2]; q.a11 = t[3]; q.a12 = t[4]; q.ds = t[5];
        q.ob[0] = t[9]; q.ob[1] = t[10]; q.ob[2] = t[11];
        q.Ro[0] = t[12]; q.Ro[1] = t[13]; q.Ro[2] = t[14]; q.Rk = t[15];
        q.Rc[0] = t[20]; q.Rc[1] = t[21];
#pragma unroll
        for (int j = 0; j < 6; ++j) q.Sw[j] = t[22 + j];
    }
    // proximal weight of variable j of the stage (the increment form keeps the carried row values in those slots
    // and recomputes S from the Ruiz D in global scratch)
    template <typename T>
    PQP_DEV T fac_weight(const FacIn &q, int j, int k, const StagePred &sp) {
        if (!Incr) return T(q.Sw[j]);
        const bool exists = (j == 3) ? sp.mid : (j == 5 ? sp.act1 : sp.real);
        const T d = T(G(gscal, GD + j, k));
        return exists ? T(sigma) / (T(cscale) * d * d) : T(1.0);
    }
    // effective outgoing-row weights of the stage (row 2 after eliminating u) and 1 / m_u
    template <typename T>
    PQP_DEV void stage_rt(const FacIn &q, int k, const StagePred &sp, T (&Rt)[3], T &miu) {
        const T ds = q.ds;
        const T R2 = q.Ro[2];
        const T pu = sp.mid ? T(w_dkappa) : T(0);
        const T mu = pu + fac_weight<T>(q, 3, k, sp) + R2 * ds * ds;
        miu = T(1) / mu;
        Rt[0] = q.Ro[0];
        Rt[1] = q.Ro[1];
        Rt[2] = R2 - (R2 * ds * miu) * R2 * ds;
    }
    // diagonal block of the reduced system of the stage (own rows + diag(RtL) of the left stage) and 1 / m_s0, 1 / m_s1
    template <typename T>
    PQP_DEV void stage_diag(const FacIn &q, int k, const StagePred &sp, const T (&Rt)[3], const T (&RtL)[3], T (&D)[6],
                            T (&mis)[2]) {
        const T a00 = q.a00, a01 = q.a01, a10 = q.a10, a11 = q.a11, a12 = q.a12, a22 = sp.a22;
        T Rc[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const bool act = j == 0 ? sp.act0 : sp.act1;
            const T ps = act ? T(w_slack) : T(0);
            const T Rcj = q.Rc[j];
            const T ms = ps + fac_weight<T>(q, 4 + j, k, sp) + Rcj;
            mis[j] = T(1) / ms;
            Rc[j] = Rcj - (Rcj * mis[j]) * Rcj;
        }
        const T h0 = sp.h0, h1 = sp.h1;
        const T pk = sp.real ? T(w_kappa) : T(0), pl = sp.real ? T(w_l) : T(0);
        const T hasL = sp.real ? T(1) : T(0);
        D[0] = fac_weight<T>(q, 0, k, sp) + pl + Rt[0] * a00 * a00 + Rt[1] * a10 * a10 + Rc[0] + Rc[1] + hasL * RtL[0];
        D[1] = Rt[0] * a00 * a01 + Rt[1] * a10 * a11 + Rc[0] * h0 + Rc[1] * h1;
        D[2] = Rt[1] * a10 * a12;
        D[3] = fac_weight<T>(q, 1, k, sp) + Rt[0] * a01 * a01 + Rt[1] * a11 * a11 + Rc[0] * h0 * h0 + Rc[1] * h1 * h1 + hasL * RtL[1];
        D[4] = Rt[1] * a11 * a12;
        D[5] = fac_weight<T>(q, 2, k, sp) + pk + Rt[1] * a12 * a12 + Rt[2] * a22 * a22 + T(q.Rk) + hasL * RtL[2];
    }
    // coupling block between the stage and the next: O[r][c] = gn * Rt_r * Ahat[r][c]
    template <typename T>
    PQP_DEV void stage_coupling(const FacIn &q, const StagePred &sp, const T (&Rt)[3], T (&O)[9]) {
        const T gn = sp.gn;
        O[0] = gn * Rt[0] * T(q.a00);
        O[1] = gn * Rt[0] * T(q.a01);
        O[2] = T(0);
        O[3] = gn * Rt[1] * T(q.a10);
        O[4] = gn * Rt[1] * T(q.a11);
        O[5] = gn * Rt[1] * T(q.a12);
        O[6] = T(0);
        O[7] = T(0);
        O[8] = gn * Rt[2] * T(sp.a22);
    }
    // the elimination constants share groups 1 and 2 with the stage's coefficients and bounds: rewrite both groups
    PQP_DEV void store_elim(const FacIn &q, int k, real miu, real mis0, real mis1) {
        Vec4 v;
        v.x = q.a12; v.y = q.ds; v.z = miu; v.w = mis0;
        store.st4(GA1, k, v);
        v.x = mis1; v.y = q.ob[0]; v.z = q.ob[1]; v.w = q.ob[2];
        store.st4(GB2, k, v);
    }

    // Block LDL' of the reduced system in nested-dissection order (see header comment).
    template <typename T>
    PQP_DEV bool factor() {
        bool ok = true;
        // left neighbour's last stage: its Rt (for our first diagonal block) and coupling
        T RtL[3], OL[9];
        {
            const StagePred spl = pred(C - 1);
            T RtLast[3], Olast[9], miu_unused;
            FacIn ql;
            load_fac(C - 1, ql);
            stage_rt<T>(ql, C - 1, spl, RtLast, miu_unused);
            stage_coupling<T>(ql, spl, RtLast, Olast);
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                RtL[r] = shfl_up(RtLast[r], 1, lane);
                if (lane == 0) RtL[r] = T(0);
            }
#pragma unroll
            for (int j = 0; j < 9; ++j) {
                OL[j] = shfl_up(Olast[j], 1, lane);
                if (lane == 0) OL[j] = T(0);
            }
        }
        T Phi[9];  // M~[SL, current]  (rows: left separator, cols: current stage) = OL'
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) Phi[3 * r + c] = OL[3 * c + r];
        T dA[6] = {T(0), T(0), T(0), T(0), T(0), T(0)};
        T Dt[6], Rt[3];
        FacIn qc;  // the current stage's inputs (one load batch per stage)
        {
            const StagePred sp0 = pred(0);
            T miu, mis[2];
            load_fac(0, qc);
            stage_rt<T>(qc, 0, sp0, Rt, miu);
            stage_diag<T>(qc, 0, sp0, Rt, RtL, Dt, mis);
            store_elim(qc, 0, (real)miu, (real)mis[0], (real)mis[1]);
        }
        // interior elimination with fill towards the left separator
        PQP_ROLL
        for (int k = 0; k < C - 1; ++k) {
            const StagePred sp = pred(k);
            T Dinv[6], O[9], Gh[9], Fh[9];
            ok = inv_sym3(Dt, Dinv) && ok;
            stage_coupling<T>(qc, sp, Rt, O);
            mul_ms(O, Dinv, Gh);
            mul_ms(Phi, Dinv, Fh);
            {   // the stage's factor = six whole groups: Dinv[6] G[9] F[9]
                real fv[24];
#pragma unroll
                for (int j = 0; j < 6; ++j) fv[j] = (real)Dinv[j];
#pragma unroll
                for (int j = 0; j < 9; ++j) { fv[6 + j] = (real)Gh[j]; fv[15 + j] = (real)Fh[j]; }
#pragma unroll
                for (int g = 0; g < 6; ++g) {
                    Vec4 v;
                    v.x = fv[4 * g]; v.y = fv[4 * g + 1]; v.z = fv[4 * g + 2]; v.w = fv[4 * g + 3];
                    store.st4(GF0 + g, k, v);
                }
            }
            T t6[6], t9[9];
            mul_abt_sym(Fh, Phi, t6);
#pragma unroll
            for (int j = 0; j < 6; ++j) dA[j] += t6[j];
            mul_abt(Fh, O, t9);
#pragma unroll
            for (int j = 0; j < 9; ++j) Phi[j] = -t9[j];
            mul_abt_sym(Gh, O, t6);
            // next stage's own block (its left neighbour is stage k)
            const StagePred spn = pred(k + 1);
            T RtPrev[3] = {Rt[0], Rt[1], Rt[2]};
            T miu, mis[2], Dn[6];
            load_fac(k + 1, qc);
            stage_rt<T>(qc, k + 1, spn, Rt, miu);
            stage_diag<T>(qc, k + 1, spn, Rt, RtPrev, Dn, mis);
            store_elim(qc, k + 1, (real)miu, (real)mis[0], (real)mis[1]);
#pragma unroll
            for (int j = 0; j < 6; ++j) Dt[j] = Dn[j] - t6[j];
        }
        // separators: A = own Schur complement - fill from the right neighbour's interior
        T Acr[6], Ccr[9];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            T dr = shfl_down(dA[j], 1, lane);
            if (lane == 31) dr = T(0);
            Acr[j] = Dt[j] - dr;
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) Ccr[3 * r + c] = Phi[3 * c + r];  // M^[S_l, S_{l-1}]
        // block cyclic reduction over the 32 separators
        T myAinv[6] = {T(1), T(0), T(0), T(1), T(0), T(1)};
        T myGm[9], myGp[9];
#pragma unroll
        for (int j = 0; j < 9; ++j) { myGm[j] = T(0); myGp[j] = T(0); }
        PQP_ROLL
        for (int t = 0; t < 5; ++t) {
            const int h = 1 << t;
            const bool elim = (lane & (2 * h - 1)) == h;
            const bool surv = (lane & (2 * h - 1)) == 0;
            T Cr[9];  // left coupling of lane+h = M^[l+h, l]
#pragma unroll
            for (int j = 0; j < 9; ++j) {
                Cr[j] = shfl_down(Ccr[j], h, lane);
                if (lane + h > 31) Cr[j] = T(0);
            }
            T Ainv[6], Gm[9], Gp[9], Ct[9];
            const bool okl = inv_sym3(Acr, Ainv);
            if (elim) ok = ok && okl;
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) Ct[3 * r + c] = Ccr[3 * c + r];
            mul_ms(Ct, Ainv, Gm);  // G- = M^[l-h, l] Ainv = C_l' Ainv
            mul_ms(Cr, Ainv, Gp);  // G+ = M^[l+h, l] Ainv = C_{l+h} Ainv
            T Um[6], Up[6], W[9];
            mul_abt_sym(Gm, Ct, Um);  // G- M^[l, l-h]
            mul_abt_sym(Gp, Cr, Up);  // G+ M^[l, l+h]
            mul_abt(Gp, Ct, W);       // G+ C_l
            if (elim) {
#pragma unroll
                for (int j = 0; j < 6; ++j) myAinv[j] = Ainv[j];
#pragma unroll
                for (int j = 0; j < 9; ++j) { myGm[j] = Gm[j]; myGp[j] = Gp[j]; }
            }
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                T fr = shfl_down(elim ? Um[j] : T(0), h, lane);  // from lane+h: its G- C
                T fl = shfl_up(elim ? Up[j] : T(0), h, lane);    // from lane-h: its G+ Cr'
                if (lane + h > 31) fr = T(0);
                if (lane < h) fl = T(0);
                if (surv) Acr[j] -= fr + fl;
            }
#pragma unroll
            for (int j = 0; j < 9; ++j) {
                T w = shfl_up(elim ? W[j] : T(0), h, lane);  // from lane-h: G+ C_{l-h}
                if (lane < h) w = T(0);
                if (surv) Ccr[j] = -w;
            }
        }
        if (lane == 0) {
            T Ainv[6];
            ok = inv_sym3(Acr, Ainv) && ok;
#pragma unroll
            for (int j = 0; j < 6; ++j) myAinv[j] = Ainv[j];
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) crAinv[j] = (real)myAinv[j];
#pragma unroll
        for (int j = 0; j < 9; ++j) { crGm[j] = (real)myGm[j]; crGp[j] = (real)myGp[j]; }
        real bad = ok ? real(0.0) : real(1.0);
        bad = warp_max(bad, lane);
        return bad == real(0.0);
    }

    // -------------------------------------------------------------- solve  M_red x = b
    // b lives in shared memory (group GBV); overwritten by the solution. The factor of one
    // stage is 6 Vec4 (Dinv[6] G[9] F[9] packed contiguously).
    // issues the loads only: the caller waits once (store.wait_ld) for this and whatever else it issued
    PQP_DEV void load_factor(int k, real (&f)[24], bool with_dinv) {
        if (with_dinv) {
            store.template ld_run_nowait<GF0, 6>(k, f);
        } else {
            real t[20];
            store.template ld_run_nowait<GF0 + 1, 5>(k, t);
#pragma unroll
            for (int j = 0; j < 20; ++j) f[4 + j] = t[j];
        }
    }
    // forward sweep over the interior stages: on return bk = rhs of this lane's separator
    // (before the contribution of the right neighbour's interior), acc = sum_k F_k b_k
    PQP_DEV void forward_sweep(real (&bk)[3], real (&acc)[3]) {
        acc[0] = acc[1] = acc[2] = real(0.0);
        real f[24], fnx[24], bvv[4], nvv[4], nnx[4];
        store.template ld4n_nowait<1>(GBV, 0, bvv);
        if (C > 1) {
            load_factor(0, f, false);
            store.template ld4n_nowait<1>(GBV, 1, nvv);
        }
        store.wait_ld();
        bk[0] = bvv[0]; bk[1] = bvv[1]; bk[2] = bvv[2];
        PQP_SWEEP_UNROLL
        for (int k = 0; k < C - 1; ++k) {
            // the next step's factor and rhs are in flight while this step computes; one wait at the end
            if (k + 1 < C - 1) {
                load_factor(k + 1, fnx, false);
                store.template ld4n_nowait<1>(GBV, k + 2, nnx);
            }
            const real *Gm = f + 6, *Fm = f + 15;
            real bn[3] = {nvv[0], nvv[1], nvv[2]};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                bn[r] -= Gm[3 * r] * bk[0] + Gm[3 * r + 1] * bk[1] + Gm[3 * r + 2] * bk[2];
                acc[r] += Fm[3 * r] * bk[0] + Fm[3 * r + 1] * bk[1] + Fm[3 * r + 2] * bk[2];
            }
            Vec4 nv;
            nv.x = bn[0]; nv.y = bn[1]; nv.z = bn[2]; nv.w = nvv[3];
            V(GBV, k + 1) = nv;
#pragma unroll
            for (int r = 0; r < 3; ++r) bk[r] = bn[r];
            store.wait_ld();
#pragma unroll
            for (int j = 4; j < 24; ++j) f[j] = fnx[j];
#pragma unroll
            for (int j = 0; j < 4; ++j) nvv[j] = nnx[j];
        }
    }
    PQP_DEV void solve() {
        real bk[3], acc[3];
        forward_sweep(bk, acc);
        store.fence();  // the backward sweep re-reads the swept rhs
        solve_tail(bk, acc);
        store.fence();  // the update reads x~ from GBV
    }
    // One level of the reduction: the lanes with (lane mod 2h) == h are eliminated, their neighbours at distance h
    // (lane mod 2h == 0) absorb G- b and G+ b of both eliminated neighbours. Every lane computes and sends (the
    // receiver selects: only a surviving lane may change its rhs - an eliminated lane's rhs is what its own back
    // substitution uses); a surviving lane's right neighbour always exists, its left one except for lane 0.
    PQP_DEV void cr_forward_level(int t, real (&bs)[3]) {
        const int h = 1 << t;
        const bool surv = (lane & (2 * h - 1)) == 0;
        real upd[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const real vm = crGm[3 * r] * bs[0] + crGm[3 * r + 1] * bs[1] + crGm[3 * r + 2] * bs[2];
            const real vp = crGp[3 * r] * bs[0] + crGp[3 * r + 1] * bs[1] + crGp[3 * r + 2] * bs[2];
            const real fr = shfl_down(vm, h, lane);
            real fl = shfl_up(vp, h, lane);
            if (lane == 0) fl = real(0.0);
            upd[r] = surv ? (fr + fl) : real(0.0);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) bs[r] -= upd[r];
    }
    // back substitution of the lanes eliminated at level t from their two solved neighbours (branch-free: every
    // lane evaluates, the eliminated ones keep the result)
    PQP_DEV void cr_backward_level(int t, const real (&ts)[3], real (&xs)[3]) {
        const int h = 1 << t;
        const bool elim = (lane & (2 * h - 1)) == h;
        real xl[3], xr[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            xl[r] = shfl_up(xs[r], h, lane);
            xr[r] = shfl_down(xs[r], h, lane);
            if (lane + h > 31) xr[r] = real(0.0);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const real v = ts[c] - (crGm[c] * xl[0] + crGm[3 + c] * xl[1] + crGm[6 + c] * xl[2]) -
                           (crGp[c] * xr[0] + crGp[3 + c] * xr[1] + crGp[6 + c] * xr[2]);
            xs[c] = elim ? v : xs[c];
        }
    }
    // separators (cyclic reduction across lanes) + backward sweep; x~ ends up in GBV
    PQP_DEV void solve_tail(const real (&bk)[3], const real (&acc)[3]) {
        real f[24], fnx[24];
        real bs[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            real fr = shfl_down(acc[r], 1, lane);
            if (lane == 31) fr = real(0.0);
            bs[r] = bk[r] - fr;
        }
        // cyclic reduction over the 32 separators: 5 forward levels, 3x3 solve, 5 backward levels; unrolled with
        // constant shuffle distances and lane masks where kUnrollCr asks for it
        if (kUnrollCr) {
#pragma unroll
            for (int t = 0; t < 5; ++t) cr_forward_level(t, bs);
        } else {
            PQP_ROLL
            for (int t = 0; t < 5; ++t) cr_forward_level(t, bs);
        }
        real ts[3], xs[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            ts[r] = crAinv[SI(r, 0)] * bs[0] + crAinv[SI(r, 1)] * bs[1] + crAinv[SI(r, 2)] * bs[2];
            xs[r] = ts[r];
        }
        if (kUnrollCr) {
#pragma unroll
            for (int t = 4; t >= 0; --t) cr_backward_level(t, ts, xs);
        } else {
            PQP_ROLL
            for (int t = 4; t >= 0; --t) cr_backward_level(t, ts, xs);
        }
        // local backward substitution
        real xSL[3], xn[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            xSL[r] = shfl_up(xs[r], 1, lane);
            if (lane == 0) xSL[r] = real(0.0);
            xn[r] = xs[r];
        }
        {
            Vec4 v;  // the fourth component of the solve vector's group is padding
            v.x = xs[0]; v.y = xs[1]; v.z = xs[2]; v.w = real(0.0);
            V(GBV, C - 1) = v;
        }
        // backward sweep, same prefetch scheme (the rhs of the next stage rides along)
        Vec4 vcur;
        if (C > 1) {
            real t4[4];
            load_factor(C - 2, f, true);
            store.template ld4n_nowait<1>(GBV, C - 2, t4);
            store.wait_ld();
            vcur.x = t4[0]; vcur.y = t4[1]; vcur.z = t4[2]; vcur.w = t4[3];
        }
        PQP_SWEEP_UNROLL
        for (int k = C - 2; k >= 0; --k) {
            // the next step's factor and rhs are in flight while this step computes; one wait at the end
            real t4[4];
            if (k > 0) {
                load_factor(k - 1, fnx, true);
                store.template ld4n_nowait<1>(GBV, k - 1, t4);
            }
            const real *Di = f, *Gm = f + 6, *Fm = f + 15;
            const real b0 = vcur.x, b1 = vcur.y, b2 = vcur.z;
            real xk[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const real t = Di[SI(c, 0)] * b0 + Di[SI(c, 1)] * b1 + Di[SI(c, 2)] * b2;
                xk[c] = t - (Gm[c] * xn[0] + Gm[3 + c] * xn[1] + Gm[6 + c] * xn[2]) -
                        (Fm[c] * xSL[0] + Fm[3 + c] * xSL[1] + Fm[6 + c] * xSL[2]);
            }
            vcur.x = xk[0]; vcur.y = xk[1]; vcur.z = xk[2];
            V(GBV, k) = vcur;
#pragma unroll
            for (int c = 0; c < 3; ++c) xn[c] = xk[c];
            if (k > 0) {
                store.wait_ld();
#pragma unroll
                for (int j = 0; j < 24; ++j) f[j] = fnx[j];
                vcur.x = t4[0]; vcur.y = t4[1]; vcur.z = t4[2]; vcur.w = t4[3];
            }
        }
    }

    // -------------------------------------------------------------- per-stage data in registers
    struct StageRO {  // read-only inside the ADMM loop (7 Vec4)
        real a00, a01, a10, a11, a12, ds, miu, mis0, mis1, ob[3], Ro[3], Rk, clo[2], chi[2], Rc[2], Sw[6];
    };
    PQP_DEV void load_ro(int k, StageRO &q) {
        real t[28];
        store.template ld4n<7>(GA0, k, t);
        q.a00 = t[0]; q.a01 = t[1]; q.a10 = t[2]; q.a11 = t[3];
        q.a12 = t[4]; q.ds = t[5]; q.miu = t[6]; q.mis0 = t[7];
        q.mis1 = t[8]; q.ob[0] = t[9]; q.ob[1] = t[10]; q.ob[2] = t[11];
        q.Ro[0] = t[12]; q.Ro[1] = t[13]; q.Ro[2] = t[14]; q.Rk = t[15];
        q.clo[0] = t[16]; q.clo[1] = t[17]; q.chi[0] = t[18]; q.chi[1] = t[19];
        q.Rc[0] = t[20]; q.Rc[1] = t[21]; q.Sw[0] = t[22]; q.Sw[1] = t[23];
        q.Sw[2] = t[24]; q.Sw[3] = t[25]; q.Sw[4] = t[26]; q.Sw[5] = t[27];
    }
    // the four read-write groups of stage k (x, s/kappa-row, yhat, clearance z/yhat)
    PQP_DEV void load_rw(int k, Vec4 &x0, Vec4 &x1, Vec4 &oy, Vec4 &cz) {
        real t[16];
        store.template ld4n<4>(GX0, k, t);
        x0.x = t[0]; x0.y = t[1]; x0.z = t[2]; x0.w = t[3];
        x1.x = t[4]; x1.y = t[5]; x1.z = t[6]; x1.w = t[7];
        oy.x = t[8]; oy.y = t[9]; oy.z = t[10]; oy.w = t[11];
        cz.x = t[12]; cz.y = t[13]; cz.z = t[14]; cz.w = t[15];
    }

    // -------------------------------------------------------------- right-hand side
    // stage-local part of the rhs from the row vectors w (wo: outgoing, wk: kappa, wc:
    // clearance) and the iterate x; on return wo[2] includes the u-condensation (what the
    // right neighbour sees)
    PQP_DEV void local_rhs(const StageRO &q, const StagePred &sp, const real (&x)[6], real (&wo)[3],
                           real wk, real (&wc)[2], real (&bk)[3]) {
        const real rhs_u = q.Sw[3] * x[3] + q.ds * wo[2];
        wo[2] -= (q.Ro[2] * q.ds * q.miu) * rhs_u;
        const real rhs_s0 = q.Sw[4] * x[4] + wc[0];
        wc[0] -= (q.Rc[0] * q.mis0) * rhs_s0;
        const real rhs_s1 = q.Sw[5] * x[5] + wc[1];
        wc[1] -= (q.Rc[1] * q.mis1) * rhs_s1;
        bk[0] = q.Sw[0] * x[0] + q.a00 * wo[0] + q.a10 * wo[1] + wc[0] + wc[1];
        bk[1] = q.Sw[1] * x[1] + q.a01 * wo[0] + q.a11 * wo[1] + sp.h0 * wc[0] + sp.h1 * wc[1];
        bk[2] = q.Sw[2] * x[2] + q.a12 * wo[1] + sp.a22 * wo[2] + wk;
    }
    // subtract the left neighbour lane's last-stage rows from this lane's first stage
    PQP_DEV void fix_first_stage(const real (&wlast)[3]) {
        const StagePred sp0 = pred(0);
        store.fence();  // GBV(0) was just written by the stage loop
        Vec4 v = V(GBV, 0);
        real wL[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            wL[r] = shfl_up(wlast[r], 1, lane);
            if (lane == 0 || !sp0.real) wL[r] = real(0.0);
        }
        v.x -= wL[0]; v.y -= wL[1]; v.z -= wL[2];
        V(GBV, 0) = v;
        store.fence();  // the solve reads GBV next
    }

    // rhs from the iterates held in shared memory (before the first iteration and after a
    // rho update). `initial`: the outgoing rows' z is z0 (cold: 0, warm: previous z), not yet
    // the bound.
    PQP_DEV void build_rhs(bool initial, bool warm) {
        real wprev[3] = {real(0.0), real(0.0), real(0.0)};
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            StageRO q;
            load_ro(k, q);
            Vec4 x0, x1, oy, cz;
            load_rw(k, x0, x1, oy, cz);
            const real x[6] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y};
            const real oyv[3] = {oy.x, oy.y, oy.z};
            real wo[3], wk, wc[2], bk[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                real z;
                if (sp.last && r < 2) z = zend[r];
                else z = initial ? z0_out(warm, r, k) : q.ob[r];
                wo[r] = q.Ro[r] * (z - oyv[r]);
            }
            wk = q.Rk * (x1.z - x1.w);
            wc[0] = q.Rc[0] * (cz.x - cz.z);
            wc[1] = q.Rc[1] * (cz.y - cz.w);
            local_rhs(q, sp, x, wo, wk, wc, bk);
            Vec4 bv;
            bv.x = bk[0] - ((sp.real && k > 0) ? wprev[0] : real(0.0));
            bv.y = bk[1] - ((sp.real && k > 0) ? wprev[1] : real(0.0));
            bv.z = bk[2] - ((sp.real && k > 0) ? wprev[2] : real(0.0));
            bv.w = real(0.0);
            V(GBV, k) = bv;
#pragma unroll
            for (int r = 0; r < 3; ++r) wprev[r] = wo[r];
        }
        fix_first_stage(wprev);
    }

    // -------------------------------------------------------------- increment form
    // A x of stage k's six rows at the stored iterate x (this stage) / xn (l, psi, kappa of the next
    // stage), and the outgoing rows' residual A x - b with the large terms grouped first
    // ((l - l') + (a00 - 1) l + ...) so that its rounding error is relative to the small terms.
    PQP_DEV void stage_ax(const StageRO &q, const StagePred &sp, const real (&x)[6], const real (&xn)[3], real (&ax)[6]) {
        const real one = real(1.0);
        const real g0 = (x[0] + sp.gn * xn[0]) + (q.a00 - one) * x[0] + q.a01 * x[1];
        const real g1 = (x[1] + sp.gn * xn[1]) + q.a10 * x[0] + (q.a11 - one) * x[1] + q.a12 * x[2];
        const real g2 = (sp.a22 * x[2] + sp.gn * xn[2]) + q.ds * x[3];
        ax[0] = g0; ax[1] = g1; ax[2] = g2;
        ax[3] = sp.real ? x[2] : real(0.0);
        ax[4] = sp.act0 ? (x[0] + sp.h0 * x[1] + x[4]) : real(0.0);
        ax[5] = sp.act1 ? (x[0] + sp.h1 * x[1] + x[5]) : real(0.0);
    }
    // stage-local part of -(P x + A'(y + R (A x - z))) from the row vectors w' = R ((z - A x) - yhat)
    PQP_DEV void local_rhs_incr(const StageRO &q, const StagePred &sp, const real (&x)[6], real (&wo)[3], real wk,
                                real (&wc)[2], real (&bk)[3]) {
        const real pl = sp.real ? w_l : real(0.0), pk = sp.real ? w_kappa : real(0.0), pu = sp.mid ? w_dkappa : real(0.0);
        const real p0 = sp.act0 ? w_slack : real(0.0), p1 = sp.act1 ? w_slack : real(0.0);
        const real rhs_u = q.ds * wo[2] - pu * x[3];
        wo[2] -= (q.Ro[2] * q.ds * q.miu) * rhs_u;
        const real rhs_s0 = wc[0] - p0 * x[4];
        wc[0] -= (q.Rc[0] * q.mis0) * rhs_s0;
        const real rhs_s1 = wc[1] - p1 * x[5];
        wc[1] -= (q.Rc[1] * q.mis1) * rhs_s1;
        bk[0] = q.a00 * wo[0] + q.a10 * wo[1] + wc[0] + wc[1] - pl * x[0];
        bk[1] = q.a01 * wo[0] + q.a11 * wo[1] + sp.h0 * wc[0] + sp.h1 * wc[1];
        bk[2] = q.a12 * wo[1] + sp.a22 * wo[2] + wk - pk * x[2];
    }
    // x (l, psi, kappa) of the right neighbour lane's first stage at the stored iterate
    PQP_DEV void right_x(real (&xr)[3]) {
        const Vec4 v = V(GX0, 0);
        xr[0] = shfl_down(v.x, 1, lane);
        xr[1] = shfl_down(v.y, 1, lane);
        xr[2] = shfl_down(v.z, 1, lane);
        if (lane == 31) { xr[0] = xr[1] = xr[2] = real(0.0); }
    }
    // rhs of the increment solve from the stored iterates. `initial` (start of a solve): the row
    // values A x are evaluated from x (large terms grouped first) and written to the FS slots; later
    // rebuilds (after a rho update) reuse the carried values.
    PQP_DEV void build_rhs_incr(bool initial, bool warm) {
        real wprev[3] = {real(0.0), real(0.0), real(0.0)};
        real xr[3] = {real(0.0), real(0.0), real(0.0)};
        if (initial) right_x(xr);
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            StageRO q;
            Vec4 x0, x1, oy, cz;
            {
                real loaded[44];
                store.template ld4n_nowait<11>(GA0, k, loaded);
                store.wait_ld();
                unpack_stage(loaded, q, x0, x1, oy, cz);
            }
            const real x[6] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y};
            real ax[6];
            if (initial) {
                real xn[3];
                if (k < C - 1) {
                    const Vec4 v = V(GX0, k < C - 1 ? k + 1 : k);
                    xn[0] = v.x; xn[1] = v.y; xn[2] = v.z;
                } else {
                    xn[0] = xr[0]; xn[1] = xr[1]; xn[2] = xr[2];
                }
                stage_ax(q, sp, x, xn, ax);
                Vec4 g5, g6;
                g5.x = q.Rc[0]; g5.y = q.Rc[1]; g5.z = ax[0]; g5.w = ax[1];
                g6.x = ax[2]; g6.y = ax[3]; g6.z = ax[4]; g6.w = ax[5];
                V(GR5, k) = g5;
                V(GS6, k) = g6;
            } else {
#pragma unroll
                for (int j = 0; j < 6; ++j) ax[j] = q.Sw[j];
            }
            const real oyv[3] = {oy.x, oy.y, oy.z};
            real wo[3], wk, wc[2], bk[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                real zmax;  // z - A x
                if (sp.last && r < 2) zmax = zend[r] - ax[r];
                else zmax = (initial ? z0_out(warm, r, k) : q.ob[r]) - ax[r];
                wo[r] = q.Ro[r] * (zmax - oyv[r]);
            }
            wk = q.Rk * ((x1.z - ax[3]) - x1.w);
            wc[0] = q.Rc[0] * ((cz.x - ax[4]) - cz.z);
            wc[1] = q.Rc[1] * ((cz.y - ax[5]) - cz.w);
            local_rhs_incr(q, sp, x, wo, wk, wc, bk);
            Vec4 bv;
            bv.x = bk[0] - ((sp.real && k > 0) ? wprev[0] : real(0.0));
            bv.y = bk[1] - ((sp.real && k > 0) ? wprev[1] : real(0.0));
            bv.z = bk[2] - ((sp.real && k > 0) ? wprev[2] : real(0.0));
            bv.w = real(0.0);
            V(GBV, k) = bv;
#pragma unroll
            for (int r = 0; r < 3; ++r) wprev[r] = wo[r];
        }
        fix_first_stage(wprev);
    }

    // -------------------------------------------------------------- infeasibility certificate terms
    // delta_y of one row (computed without cancellation as R (zt - z+)), projected onto the polar
    // of the recession cone of [lo, hi] (OSQP is_primal_infeasible); a bound counts as infinite
    // when |b| >= 1e29 (OSQP_INFTY = 1e30 is the caller's "no bound" value). Accumulates
    // |dy|_inf and u'max(dy,0) + l'min(dy,0); dy itself goes to global scratch for A'dy.
    PQP_DEV void cert_row(int r, int k, real dy, real lo, real hi) {
        const bool hinf = hi >= real(1e29), linf = lo <= -real(1e29);
        if (hinf) dy = linf ? real(0.0) : xmin(dy, real(0.0));
        else if (linf) dy = xmax(dy, real(0.0));
        G(gdy, r, k) = dy;
        cert_nrm = xmax(cert_nrm, xabs(dy));
        cert_lhs += (dy > real(0.0) ? hi * dy : real(0.0)) + (dy < real(0.0) ? lo * dy : real(0.0));
    }

    // -------------------------------------------------------------- one ADMM update
    // in: GBV = x~ (state part); the rhs of the eliminated variables (u, s0, s1) used by that
    // solve is recomputed from the (still unchanged) iterates instead of being stored.
    // out: iterates advanced in shared memory, GBV = rhs of the next solve.
    // first: first iteration of a solve, where the outgoing equality rows' previous z is
    // z0 (cold: 0, warm: the previous solve's z) rather than their bound.
    // one stage of the ADMM update: advances x, z, yhat of stage k in shared memory from
    // x~_k (xt) and x~_{k+1} (xn); returns the stage-local part of the next rhs (bk) and the
    // outgoing-row vector w (wo, row 2 including the u-condensation)
    template <bool kCheck>
    PQP_DEV void update_stage(int k, bool first, bool warm, const real (&xt)[3], const real (&xn)[3],
                              real (&wo)[3], real (&bk)[3]) {
        const real oma = real(1.0) - alpha;
        const StagePred sp = pred(k);
        StageRO q;
        load_ro(k, q);
        Vec4 x0, x1, oy, cz;
        load_rw(k, x0, x1, oy, cz);
        const real lt = xt[0], pt = xt[1], kt = xt[2];
        const real ln = xn[0], pn = xn[1], kn = xn[2];
        // previous z of the outgoing rows
        real zo_old[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            if (sp.last && r < 2) zo_old[r] = zend[r];
            else zo_old[r] = first ? z0_out(warm, r, k) : q.ob[r];
        }
        const real oyv[3] = {oy.x, oy.y, oy.z};
        // recover the eliminated variables of x~ (rhs recomputed from the old iterates)
        const real aux_u = q.Sw[3] * x0.w + q.ds * (q.Ro[2] * (zo_old[2] - oyv[2]));
        const real aux_s0 = q.Sw[4] * x1.x + q.Rc[0] * (cz.x - cz.z);
        const real aux_s1 = q.Sw[5] * x1.y + q.Rc[1] * (cz.y - cz.w);
        const real ut = q.miu * (aux_u - q.Ro[2] * q.ds * (sp.a22 * kt + sp.gn * kn));
        const real s0t = q.mis0 * (aux_s0 - q.Rc[0] * (lt + sp.h0 * pt));
        const real s1t = q.mis1 * (aux_s1 - q.Rc[1] * (lt + sp.h1 * pt));
        // z~ = A x~
        real zo[3];
        zo[0] = q.a00 * lt + q.a01 * pt + sp.gn * ln;
        zo[1] = q.a10 * lt + q.a11 * pt + q.a12 * kt + sp.gn * pn;
        zo[2] = sp.a22 * kt + q.ds * ut + sp.gn * kn;
        const real zk = sp.real ? kt : real(0.0);
        const real zc0 = sp.act0 ? (lt + sp.h0 * pt + s0t) : real(0.0);
        const real zc1 = sp.act1 ? (lt + sp.h1 * pt + s1t) : real(0.0);
        // x+ = alpha x~ + (1 - alpha) x
        x0.x = alpha * lt + oma * x0.x;
        x0.y = alpha * pt + oma * x0.y;
        x0.z = alpha * kt + oma * x0.z;
        x0.w = alpha * ut + oma * x0.w;
        x1.x = alpha * s0t + oma * x1.x;
        x1.y = alpha * s1t + oma * x1.y;
        // rows: z+ = clamp(alpha z~ + (1-alpha) z + yhat), yhat+ = (..) - z+, w = R (z+ - yhat+)
        real wk, wc[2], oyn[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const real bnd = q.ob[r];
            const real zt = alpha * zo[r] + oma * zo_old[r];
            const real zh = zt + oyv[r];
            real zn;
            if (sp.last && r < 2) {
                zn = clampf(zh, bnd, bnd + endw[r]);
                zend[r] = zn;
            } else {
                zn = bnd;
            }
            oyn[r] = zh - zn;
            wo[r] = q.Ro[r] * (zn - oyn[r]);
            if (kCheck) cert_row(r, k, q.Ro[r] * (zt - zn), bnd, (sp.last && r < 2) ? bnd + endw[r] : bnd);
        }
        oy.x = oyn[0]; oy.y = oyn[1]; oy.z = oyn[2];
        {
            const real zt = alpha * zk + oma * x1.z;
            const real zh = zt + x1.w;
            const real zn = clampf(zh, -kmax, kmax);
            x1.z = zn;
            x1.w = zh - zn;
            wk = q.Rk * (zn - x1.w);
            if (kCheck) cert_row(3, k, q.Rk * (zt - zn), -kmax, kmax);
        }
        {
            const real zt = alpha * zc0 + oma * cz.x;
            const real zh = zt + cz.z;
            const real zn = clampf(zh, q.clo[0], q.chi[0]);
            cz.x = zn;
            cz.z = zh - zn;
            wc[0] = q.Rc[0] * (zn - cz.z);
            if (kCheck) cert_row(4, k, q.Rc[0] * (zt - zn), q.clo[0], q.chi[0]);
        }
        {
            const real zt = alpha * zc1 + oma * cz.y;
            const real zh = zt + cz.w;
            const real zn = clampf(zh, q.clo[1], q.chi[1]);
            cz.y = zn;
            cz.w = zh - zn;
            wc[1] = q.Rc[1] * (zn - cz.w);
            if (kCheck) cert_row(5, k, q.Rc[1] * (zt - zn), q.clo[1], q.chi[1]);
        }
        V(GX0, k) = x0;
        V(GX1, k) = x1;
        V(GOY, k) = oy;
        V(GCZ, k) = cz;
        const real x[6] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y};
        local_rhs(q, sp, x, wo, wk, wc, bk);
    }

    // ADMM update of all stages (ascending; the left neighbour's outgoing rows are carried in
    // registers). It is not fused with the next forward sweep: in-order issue would serialise the sweep
    // step behind each stage's update.
    // in: GBV = x~; out: iterates advanced, GBV = rhs of the next solve.
    template <bool kCheck>
    PQP_DEV void admm_update(bool first, bool warm) {
        real xnb[3];
        {
            const Vec4 v = V(GBV, 0);
            xnb[0] = shfl_down(v.x, 1, lane);
            xnb[1] = shfl_down(v.y, 1, lane);
            xnb[2] = shfl_down(v.z, 1, lane);
            if (lane == 31) { xnb[0] = xnb[1] = xnb[2] = real(0.0); }
        }
        if (kCheck) { cert_nrm = real(0.0); cert_lhs = real(0.0); }
        real wprev[3] = {real(0.0), real(0.0), real(0.0)};
        Vec4 xv = V(GBV, 0);
        PQP_UPDATE_UNROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            const Vec4 xw = V(GBV, k < C - 1 ? k + 1 : k);
            const real xt[3] = {xv.x, xv.y, xv.z};
            real xn[3];
            xn[0] = (k == C - 1) ? xnb[0] : xw.x;
            xn[1] = (k == C - 1) ? xnb[1] : xw.y;
            xn[2] = (k == C - 1) ? xnb[2] : xw.z;
            real wo[3], bk[3];
            update_stage<kCheck>(k, first, warm, xt, xn, wo, bk);
            Vec4 bv;
            bv.x = bk[0] - ((sp.real && k > 0) ? wprev[0] : real(0.0));
            bv.y = bk[1] - ((sp.real && k > 0) ? wprev[1] : real(0.0));
            bv.z = bk[2] - ((sp.real && k > 0) ? wprev[2] : real(0.0));
            bv.w = real(0.0);
            V(GBV, k) = bv;
#pragma unroll
            for (int r = 0; r < 3; ++r) wprev[r] = wo[r];
            xv = xw;
        }
        fix_first_stage(wprev);
    }

    // -------------------------------------------------------------- one ADMM update, increment form
    // in: GBV = dx (state part) of the solve K dx = -(P x + A'(y + R (A x - z))); dt / dn are dx of
    // this / the next stage. The row values A x are carried in the FS slots (q.Sw) and advanced by
    // alpha A dx - never re-evaluated from the rounded x - so their error scales with |dx|.
    // Same outputs as update_stage; the rhs produced is again the increment-form one.
    // the 11 groups of stage k (7 read-only + 4 read-write, consecutive group numbers) unpacked from one load batch
    PQP_DEV void unpack_stage(const real (&t)[44], StageRO &q, Vec4 &x0, Vec4 &x1, Vec4 &oy, Vec4 &cz) {
        q.a00 = t[0]; q.a01 = t[1]; q.a10 = t[2]; q.a11 = t[3];
        q.a12 = t[4]; q.ds = t[5]; q.miu = t[6]; q.mis0 = t[7];
        q.mis1 = t[8]; q.ob[0] = t[9]; q.ob[1] = t[10]; q.ob[2] = t[11];
        q.Ro[0] = t[12]; q.Ro[1] = t[13]; q.Ro[2] = t[14]; q.Rk = t[15];
        q.clo[0] = t[16]; q.clo[1] = t[17]; q.chi[0] = t[18]; q.chi[1] = t[19];
        q.Rc[0] = t[20]; q.Rc[1] = t[21]; q.Sw[0] = t[22]; q.Sw[1] = t[23];
        q.Sw[2] = t[24]; q.Sw[3] = t[25]; q.Sw[4] = t[26]; q.Sw[5] = t[27];
        x0.x = t[28]; x0.y = t[29]; x0.z = t[30]; x0.w = t[31];
        x1.x = t[32]; x1.y = t[33]; x1.z = t[34]; x1.w = t[35];
        oy.x = t[36]; oy.y = t[37]; oy.z = t[38]; oy.w = t[39];
        cz.x = t[40]; cz.y = t[41]; cz.z = t[42]; cz.w = t[43];
    }

    template <bool kCheck>
    PQP_DEV void update_stage_incr(int k, const bool first, bool warm, const real (&dt)[3], const real (&dn)[3],
                                   real (&wo)[3], real (&bk)[3], const real (&loaded)[44], real (&nloaded)[44],
                                   real (&ndwv)[4]) {
        const StagePred sp = pred(k);
        StageRO q;
        Vec4 x0, x1, oy, cz;
        unpack_stage(loaded, q, x0, x1, oy, cz);
        real x[6] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y};
        real ax[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) ax[j] = q.Sw[j];
        const real oyv[3] = {oy.x, oy.y, oy.z};
        // z - A x of the outgoing rows at the old iterate
        real zo_old[3], zmax[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            if (sp.last && r < 2) zo_old[r] = zend[r];
            else zo_old[r] = first ? z0_out(warm, r, k) : q.ob[r];
            zmax[r] = zo_old[r] - ax[r];
        }
        // increments of the eliminated variables (their rhs recomputed from the old iterates)
        const real pu = sp.mid ? w_dkappa : real(0.0);
        const real p0 = sp.act0 ? w_slack : real(0.0), p1 = sp.act1 ? w_slack : real(0.0);
        const real aux_u = q.ds * (q.Ro[2] * (zmax[2] - oyv[2])) - pu * x[3];
        const real aux_s0 = q.Rc[0] * ((cz.x - ax[4]) - cz.z) - p0 * x[4];
        const real aux_s1 = q.Rc[1] * ((cz.y - ax[5]) - cz.w) - p1 * x[5];
        const real du = q.miu * (aux_u - q.Ro[2] * q.ds * (sp.a22 * dt[2] + sp.gn * dn[2]));
        const real ds0 = q.mis0 * (aux_s0 - q.Rc[0] * (dt[0] + sp.h0 * dt[1]));
        const real ds1 = q.mis1 * (aux_s1 - q.Rc[1] * (dt[0] + sp.h1 * dt[1]));
        // alpha A dx
        real dz[6];
        dz[0] = alpha * (q.a00 * dt[0] + q.a01 * dt[1] + sp.gn * dn[0]);
        dz[1] = alpha * (q.a10 * dt[0] + q.a11 * dt[1] + q.a12 * dt[2] + sp.gn * dn[1]);
        dz[2] = alpha * (sp.a22 * dt[2] + q.ds * du + sp.gn * dn[2]);
        dz[3] = sp.real ? alpha * dt[2] : real(0.0);
        dz[4] = sp.act0 ? alpha * (dt[0] + sp.h0 * dt[1] + ds0) : real(0.0);
        dz[5] = sp.act1 ? alpha * (dt[0] + sp.h1 * dt[1] + ds1) : real(0.0);
        // x+ = x + alpha dx
        x[0] += alpha * dt[0]; x[1] += alpha * dt[1]; x[2] += alpha * dt[2];
        x[3] += alpha * du; x[4] += alpha * ds0; x[5] += alpha * ds1;
        x0.x = x[0]; x0.y = x[1]; x0.z = x[2]; x0.w = x[3]; x1.x = x[4]; x1.y = x[5];
        // rows: zt = z_old + alpha (z~ - z_old) = z_old + (alpha A dx - alpha (z_old - A x));
        // afterwards A x+ = A x + alpha A dx
        real wk, wc[2], oyn[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const real bnd = q.ob[r];
            const real step = dz[r] - alpha * zmax[r];
            const real axn = ax[r] + dz[r];
            real zn, dyr;
            if (sp.last && r < 2) {
                const real zt = zo_old[r] + step;
                const real zh = zt + oyv[r];
                zn = clampf(zh, bnd, bnd + endw[r]);
                zend[r] = zn;
                oyn[r] = zh - zn;
                dyr = zt - zn;
            } else {
                // equality row: z+ = b, yhat+ = yhat + (z_old + step - b); z_old = b unless `first`
                zn = bnd;
                dyr = step + (zo_old[r] - bnd);
                oyn[r] = oyv[r] + dyr;
            }
            wo[r] = q.Ro[r] * ((zn - axn) - oyn[r]);
            ax[r] = axn;
            if (kCheck) cert_row(r, k, q.Ro[r] * dyr, bnd, (sp.last && r < 2) ? bnd + endw[r] : bnd);
        }
        oy.x = oyn[0]; oy.y = oyn[1]; oy.z = oyn[2];
        {
            const real zt = x1.z + (dz[3] - alpha * (x1.z - ax[3]));
            const real zh = zt + x1.w;
            const real zn = clampf(zh, -kmax, kmax);
            ax[3] += dz[3];
            x1.z = zn;
            x1.w = zh - zn;
            wk = q.Rk * ((zn - ax[3]) - x1.w);
            if (kCheck) cert_row(3, k, q.Rk * (zt - zn), -kmax, kmax);
        }
        {
            const real zt = cz.x + (dz[4] - alpha * (cz.x - ax[4]));
            const real zh = zt + cz.z;
            const real zn = clampf(zh, q.clo[0], q.chi[0]);
            ax[4] += dz[4];
            cz.x = zn;
            cz.z = zh - zn;
            wc[0] = q.Rc[0] * ((zn - ax[4]) - cz.z);
            if (kCheck) cert_row(4, k, q.Rc[0] * (zt - zn), q.clo[0], q.chi[0]);
        }
        {
            const real zt = cz.y + (dz[5] - alpha * (cz.y - ax[5]));
            const real zh = zt + cz.w;
            const real zn = clampf(zh, q.clo[1], q.chi[1]);
            ax[5] += dz[5];
            cz.y = zn;
            cz.w = zh - zn;
            wc[1] = q.Rc[1] * ((zn - ax[5]) - cz.w);
            if (kCheck) cert_row(5, k, q.Rc[1] * (zt - zn), q.clo[1], q.chi[1]);
        }
        Vc(GX0, k) = x0;
        Vc(GX1, k) = x1;
        Vc(GOY, k) = oy;
        Vc(GCZ, k) = cz;
        {
            Vec4 g5, g6;
            g5.x = q.Rc[0]; g5.y = q.Rc[1]; g5.z = ax[0]; g5.w = ax[1];
            g6.x = ax[2]; g6.y = ax[3]; g6.z = ax[4]; g6.w = ax[5];
            Vc(GR5, k) = g5;
            Vc(GS6, k) = g6;
        }
        // the next stage's load batch is in flight while this stage's rhs part is computed (no wait here)
        store.ld4_nowait_ahead_next(GBV, k, ndwv);
        store.template ld_run_nowait_ahead<GA0, 11>(k, nloaded);
        local_rhs_incr(q, sp, x, wo, wk, wc, bk);
    }

    // kMaybeFirst = false: the caller knows this is not the first iteration of a solve, and the stage loop carries
    // no branch around the z0 code (a taken branch and an instruction refetch in the hottest loop)
    template <bool kCheck, bool kMaybeFirst>
    PQP_DEV void admm_update_incr(bool first_arg, bool warm) {
        const bool first = kMaybeFirst && first_arg;
        Vec4 dv = V(GBV, 0);
        real dnb[3];
        dnb[0] = shfl_down(dv.x, 1, lane);
        dnb[1] = shfl_down(dv.y, 1, lane);
        dnb[2] = shfl_down(dv.z, 1, lane);
        if (lane == 31) { dnb[0] = dnb[1] = dnb[2] = real(0.0); }
        if (kCheck) { cert_nrm = real(0.0); cert_lhs = real(0.0); }
        real wprev[3] = {real(0.0), real(0.0), real(0.0)};
        // one load batch per stage (the next stage's dx and the stage's 11 groups, one wait), issued one stage
        // ahead: stage k+1's batch is in flight while stage k's rhs part is computed
        real dwv[4], loaded[44];
        store.seek(0);
        store.ld4_nowait_next(GBV, 0, dwv);
        store.template ld_run_nowait_cur<GA0, 11>(0, loaded);
        store.wait_ld();
        // the hot instantiation (no check, not the first iteration) is unrolled by two: the prefetched batch then
        // lands in registers the next stage reads directly instead of being copied at every trip (44 + 4 moves),
        // for one more copy of the stage body (DESIGN §10); the check and first-iteration loops stay rolled
        constexpr int kUnroll = (!kCheck && !kMaybeFirst) ? 2 : 1;
#pragma unroll (kUnroll)
        for (int k = 0; k < C; ++k) {
            store.seek(k);
            const StagePred sp = pred(k);
            real ndwv[4], nloaded[44];
            const real dt[3] = {dv.x, dv.y, dv.z};
            real dn[3];
            dn[0] = (k == C - 1) ? dnb[0] : dwv[0];
            dn[1] = (k == C - 1) ? dnb[1] : dwv[1];
            dn[2] = (k == C - 1) ? dnb[2] : dwv[2];
            Vec4 dw;
            dw.x = dwv[0]; dw.y = dwv[1]; dw.z = dwv[2]; dw.w = dwv[3];
            real wo[3], bk[3];
            update_stage_incr<kCheck>(k, first, warm, dt, dn, wo, bk, loaded, nloaded, ndwv);
            Vec4 bv;
            bv.x = bk[0] - ((sp.real && k > 0) ? wprev[0] : real(0.0));
            bv.y = bk[1] - ((sp.real && k > 0) ? wprev[1] : real(0.0));
            bv.z = bk[2] - ((sp.real && k > 0) ? wprev[2] : real(0.0));
            bv.w = real(0.0);
            Vc(GBV, k) = bv;
#pragma unroll
            for (int r = 0; r < 3; ++r) wprev[r] = wo[r];
            dv = dw;
            store.wait_ld();
#pragma unroll
            for (int j = 0; j < 44; ++j) loaded[j] = nloaded[j];
#pragma unroll
            for (int j = 0; j < 4; ++j) dwv[j] = ndwv[j];
        }
        fix_first_stage(wprev);
    }

    // -------------------------------------------------------------- residuals (OSQP update_info)
    struct Norms {
        real pri, ax, z, dua, px, aty;          // unscaled inf-norms
        real spri, sax, sz, sdua, spx, saty;    // scaled (for the rho estimate)
    };
    PQP_DEV Norms residuals() {
        const DevParams &P = ka.prm;
        sync_warp(lane);
        real m[12];
#pragma unroll
        for (int j = 0; j < 12; ++j) m[j] = real(0.0);
        const real c = cscale;
        // e_r = sqrt(R_r) * sqrt(c / base_class), c d_j = sqrt(sigma c) / sqrt(S_j)
        // boundary values of the neighbour lanes (y of the left lane's last outgoing rows, x of the
        // right lane's first stage) travel by shuffle
        real yLb[3], xNb[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            yLb[r] = shfl_up((real)S(FOR_ + r, C - 1) * (real)S(FOY + r, C - 1), 1, lane);
            xNb[r] = shfl_down((real)S(FX + r, 0), 1, lane);
            if (lane == 0) yLb[r] = real(0.0);
            if (lane == 31) xNb[r] = real(0.0);
        }
        const real ke_in = xsqrt(c / rho), ke_eq = xsqrt(c / (real(kRhoEqOverIneq) * rho)),
                   ke_lo = xsqrt(c / real(kRhoMin)), kd = xsqrt(sigma * c);
        real yprev[3] = {yLb[0], yLb[1], yLb[2]};  // y of the previous stage's outgoing rows
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            // the stage's 11 groups and the next stage's x in ONE load batch (one wait), as in the update
            real loaded[44], xn4[4];
            store.template ld4n_nowait<11>(GA0, k, loaded);
            store.template ld4n_nowait<1>(GX0, k < C - 1 ? k + 1 : k, xn4);
            store.wait_ld();
            StageRO q;
            Vec4 x0, x1, oy, cz;
            unpack_stage(loaded, q, x0, x1, oy, cz);
            // Ruiz scalings recovered from the weights held on chip: R_r = base_r e_r^2 / c and
            // S_j = sigma / (c d_j^2)  (no divisions in the check path)
            real ev[6], dv[6];
            {
                const int cls = (int)oy.w;
#pragma unroll
                for (int r = 0; r < 6; ++r) {
                    const int cl = (cls >> (2 * r)) & 3;
                    const real Rr = (r < 3) ? q.Ro[r] : (r == 3 ? q.Rk : q.Rc[r - 4]);
                    const real kc = cl == 1 ? ke_eq : (cl == 0 ? ke_in : ke_lo);
                    ev[r] = (cl == 3 || !(Rr > real(0.0))) ? real(0.0) : Rr * xfast_rsqrt(Rr) * kc;
                }
                if (Incr) {
                    // c d_j straight from the Ruiz D (the increment form keeps no S on chip; recomputing
                    // S = sigma / (c d^2) only to take kd / sqrt(S) = c d cost a division and a rsqrt per entry:
                    // few instructions but long stalls)
#pragma unroll
                    for (int j = 0; j < 6; ++j) {
                        const bool exists = (j == 3) ? sp.mid : (j == 5 ? sp.act1 : sp.real);
                        const real d = G(gscal, GD + j, k);
                        dv[j] = exists ? c * d : kd;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 6; ++j) dv[j] = kd * xfast_rsqrt(q.Sw[j]);  // textbook form: Sw holds S
                }
            }
            const real a00 = q.a00, a01 = q.a01, a10 = q.a10, a11 = q.a11, a12 = q.a12, ds = q.ds;
            const real l = x0.x, ps = x0.y, kp = x0.z, u = x0.w, s0 = x1.x, s1 = x1.y;
            const real ln = (k < C - 1) ? xn4[0] : xNb[0];
            const real pn = (k < C - 1) ? xn4[1] : xNb[1];
            const real kn = (k < C - 1) ? xn4[2] : xNb[2];
            const real yl[3] = {yprev[0], yprev[1], yprev[2]};
            real ax[6], z[6], y[6];
            ax[0] = a00 * l + a01 * ps + sp.gn * ln;
            ax[1] = a10 * l + a11 * ps + a12 * kp + sp.gn * pn;
            ax[2] = sp.a22 * kp + ds * u + sp.gn * kn;
            ax[3] = sp.real ? kp : real(0.0);
            ax[4] = sp.act0 ? (l + sp.h0 * ps + s0) : real(0.0);
            ax[5] = sp.act1 ? (l + sp.h1 * ps + s1) : real(0.0);
            const real oyv[3] = {oy.x, oy.y, oy.z};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                z[r] = (sp.last && r < 2) ? zend[r] : q.ob[r];
                y[r] = q.Ro[r] * oyv[r];
                yprev[r] = y[r];
            }
            z[3] = x1.z; y[3] = q.Rk * x1.w;
            z[4] = cz.x; y[4] = q.Rc[0] * cz.z;
            z[5] = cz.y; y[5] = q.Rc[1] * cz.w;
#pragma unroll
            for (int r = 0; r < 6; ++r) {
                const real e = ev[r];
                const real rp = xabs(ax[r] - z[r]);
                m[0] = xmax(m[0], rp); m[1] = xmax(m[1], xabs(ax[r])); m[2] = xmax(m[2], xabs(z[r]));
                m[6] = xmax(m[6], e * rp); m[7] = xmax(m[7], e * xabs(ax[r])); m[8] = xmax(m[8], e * xabs(z[r]));
            }
            const real hasL = sp.real ? real(1.0) : real(0.0);
            real aty[6], px[6];
            aty[0] = a00 * y[0] + a10 * y[1] + y[4] + y[5] - hasL * yl[0];
            aty[1] = a01 * y[0] + a11 * y[1] + sp.h0 * y[4] + sp.h1 * y[5] - hasL * yl[1];
            aty[2] = a12 * y[1] + sp.a22 * y[2] + y[3] - hasL * yl[2];
            aty[3] = ds * y[2];
            aty[4] = sp.act0 ? y[4] : real(0.0);
            aty[5] = sp.act1 ? y[5] : real(0.0);
            px[0] = sp.real ? w_l * l : real(0.0);
            px[1] = real(0.0);
            px[2] = sp.real ? w_kappa * kp : real(0.0);
            px[3] = sp.mid ? w_dkappa * u : real(0.0);
            px[4] = sp.act0 ? w_slack * s0 : real(0.0);
            px[5] = sp.act1 ? w_slack * s1 : real(0.0);
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const real d = dv[j];
                const real rd = xabs(px[j] + aty[j]);
                m[3] = xmax(m[3], rd); m[4] = xmax(m[4], xabs(px[j])); m[5] = xmax(m[5], xabs(aty[j]));
                m[9] = xmax(m[9], d * rd); m[10] = xmax(m[10], d * xabs(px[j])); m[11] = xmax(m[11], d * xabs(aty[j]));
            }
        }
#pragma unroll
        for (int j = 0; j < 12; ++j) m[j] = warp_max(m[j], lane);
        Norms nr;
        nr.pri = m[0]; nr.ax = m[1]; nr.z = m[2]; nr.dua = m[3]; nr.px = m[4]; nr.aty = m[5];
        nr.spri = m[6]; nr.sax = m[7]; nr.sz = m[8]; nr.sdua = m[9]; nr.spx = m[10]; nr.saty = m[11];
        return nr;
    }

    // OSQP is_primal_infeasible, evaluated once per check: |dy|_inf and the bound term were
    // accumulated by admm_update<true>; |A'dy|_inf is only computed when the first two
    // conditions hold at the normal tolerance. The caller applies the normal and, on the last
    // iteration, the 10x tolerance to the returned raw terms.
    struct Cert { real nrm, lhs, aty; };
    PQP_DEV Cert primal_infeasibility_terms(real eps) {
        Cert ct;
        ct.nrm = warp_max(cert_nrm, lane);
        ct.lhs = warp_sum(cert_lhs, lane);
        ct.aty = real(kOsqpInfty);
        // conditions 1-2 at the normal tolerance (they are only harder at 10x)
        suspect = ((cscale * ct.nrm > eps) && (ct.lhs < -eps * ct.nrm)) ? 1 : 0;
        if (!suspect) return ct;
        sync_warp(lane);
        real mx = real(0.0);
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const StagePred sp = pred(k);
            const real a00 = S(FA + 0, k), a01 = S(FA + 1, k), a10 = S(FA + 2, k), a11 = S(FA + 3, k),
                        a12 = S(FA + 4, k), ds = S(FA + 5, k);
            real y[6], yl[3];
#pragma unroll
            for (int r = 0; r < 6; ++r) y[r] = G(gdy, r, k);
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                if (k > 0) yl[r] = G(gdy, r, k - 1);
                else yl[r] = lane == 0 ? real(0.0) : GL(gdy, r, C - 1, lane - 1);
                if (!sp.real) yl[r] = real(0.0);
            }
            real aty[6];
            aty[0] = a00 * y[0] + a10 * y[1] + y[4] + y[5] - yl[0];
            aty[1] = a01 * y[0] + a11 * y[1] + sp.h0 * y[4] + sp.h1 * y[5] - yl[1];
            aty[2] = a12 * y[1] + sp.a22 * y[2] + y[3] - yl[2];
            aty[3] = ds * y[2];
            aty[4] = y[4];
            aty[5] = y[5];
#pragma unroll
            for (int j = 0; j < 6; ++j) mx = xmax(mx, xabs(aty[j]));
        }
        ct.aty = warp_max(mx, lane);
        return ct;
    }
    PQP_DEV bool cert_holds(const Cert &ct, real eps) const {
        return (cscale * ct.nrm > eps) && (ct.lhs < -eps * ct.nrm) && (ct.aty < eps * ct.nrm);
    }

    // OSQP check_termination (and, when `last`, the 10x "approximate" re-check that osqp_solve
    // performs after the final iteration). Returns a status or kUnsolved.
    PQP_DEV int check_termination(const Norms &nr, bool last) {
        if (!(nr.pri <= real(kOsqpInfty)) || !(nr.dua <= real(kOsqpInfty))) return kNumerical;
        const real mp = xmax(nr.ax, nr.z), md = xmax(nr.px, nr.aty);
        const bool pok = nr.pri < eps_abs + eps_rel * mp, dok = nr.dua < eps_abs + eps_rel * md;
        if (pok && dok) return kSolved;
        // dual infeasibility needs q' dx < 0; q = 0 on this path, so it can never trigger
        Cert ct;
        ct.nrm = ct.lhs = real(0.0);
        ct.aty = real(kOsqpInfty);
        const bool pok10 = nr.pri < real(10.0) * (eps_abs + eps_rel * mp);
        if (!pok) ct = primal_infeasibility_terms(eps_pinf);
        if (!pok && cert_holds(ct, eps_pinf)) return kPrimInf;
        if (!last) return kUnsolved;
        const bool dok10 = nr.dua < real(10.0) * (eps_abs + eps_rel * md);
        if (pok10 && dok10) return kSolvedInacc;
        if (!pok10 && cert_holds(ct, real(10.0) * eps_pinf)) return kPrimInfInacc;
        return kMaxIter;
    }


    // OSQP compute_rho_estimate + update of the weights; returns true if rho changed (the caller
    // refactors and rebuilds the rhs)
    PQP_DEV bool adapt_rho(const Norms &nr) {
        const DevParams &P = ka.prm;
        const real pri = nr.spri / (xmax(nr.sz, nr.sax) + real(1e-10));
        const real dua = nr.sdua / (xmax(nr.saty, nr.spx) + real(1e-10));
        real est = rho * xsqrt(pri / (dua + real(1e-10)));
        est = xmin(xmax(est, real(kRhoMin)), real(kRhoMax));
        if (!(est > rho * rho_tol || est < rho / rho_tol)) return false;
        const real ratio = est / rho, rinv = rho / est;
        rho = est;
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            // the five groups that hold row weights / scaled duals, one load batch, five group stores
            real r3[4], r5[4], x1[4], oy[4], cz[4];
            store.template ld4n_nowait<1>(GR3, k, r3);   // Ro0 Ro1 Ro2 Rk
            store.template ld4n_nowait<1>(GR5, k, r5);   // Rc0 Rc1 | (S or carried A x)
            store.template ld4n_nowait<1>(GX1, k, x1);   // s0 s1 | kappa-row z, yhat
            store.template ld4n_nowait<1>(GOY, k, oy);   // outgoing yhat 0..2 | row classes
            store.template ld4n_nowait<1>(GCZ, k, cz);   // clearance z 0..1 | yhat 0..1
            store.wait_ld();
            const int cls = (int)oy[3];
            real fr[6], fi[6];
#pragma unroll
            for (int r = 0; r < 6; ++r) {
                const int cl = (cls >> (2 * r)) & 3;
                fr[r] = cl <= 1 ? ratio : real(1.0);
                fi[r] = cl <= 1 ? rinv : real(1.0);
            }
            Vec4 v;
            v.x = r3[0] * fr[0]; v.y = r3[1] * fr[1]; v.z = r3[2] * fr[2]; v.w = r3[3] * fr[3];
            store.st4(GR3, k, v);
            v.x = r5[0] * fr[4]; v.y = r5[1] * fr[5]; v.z = r5[2]; v.w = r5[3];
            store.st4(GR5, k, v);
            v.x = x1[0]; v.y = x1[1]; v.z = x1[2]; v.w = x1[3] * fi[3];
            store.st4(GX1, k, v);
            v.x = oy[0] * fi[0]; v.y = oy[1] * fi[1]; v.z = oy[2] * fi[2]; v.w = oy[3];
            store.st4(GOY, k, v);
            v.x = cz[0]; v.y = cz[1]; v.z = cz[2] * fi[4]; v.w = cz[3] * fi[5];
            store.st4(GCZ, k, v);
        }
        store.fence();
        return true;
    }

    // -------------------------------------------------------------- whole solve
    // `scratch`: index of the intra-solve scratch block (Ruiz D/E, delta_y): the instance's slot in the
    // handle for one-CTA-per-instance launches, the resident warp's slot for persistent launches
    // (592 blocks that stay in L2 instead of one per instance streaming out to HBM)
    PQP_DEV void run(const double *src, int stride, size_t scratch) {
        const DevParams &P = ka.prm;
        n = ka.n[qp];
        // the device-pointer entry points cannot inspect n[] on the host: an out-of-range size must not
        // read past the knot block or write past sol[] (the host-pointer calls reject it up front)
        if (n < 2 || n > ka.n_max || n > 32 * C - 1) {
            if (lane == 0) {
                if (ka.status) ka.status[qp] = kNumerical;
                if (ka.iters) ka.iters[qp] = 0;
                if (ka.cost) ka.cost[qp] = 0.0;
                if (ka.flags) ka.flags[qp] = 0;
            }
            return;
        }
        p = ka.p ? ka.p[qp] : n;
        p = p < 0 ? 0 : (p > n ? n : p);
        lf = (real)P.front_length;
        lr = (real)P.rear_length;
        kmax = (real)P.kappa_limit;
        const size_t plane = (size_t)C * 32;
        const size_t slot = (size_t)(qp + ka.qp0);  // per-instance scratch slot in the handle
        gwarm = static_cast<real *>(ka.warm) + slot * NWARM * plane;
        gscal = static_cast<real *>(ka.scal) + scratch * NSCAL * plane;
        gdy = static_cast<real *>(ka.dy) + scratch * NDY * plane;
        w_l = (real)P.w_l; w_kappa = (real)P.w_kappa; w_dkappa = (real)P.w_dkappa; w_slack = (real)P.w_slack;
        sigma = (real)P.sigma; alpha = (real)P.alpha; eps_abs = (real)P.eps_abs; eps_rel = (real)P.eps_rel;
        eps_pinf = (real)P.eps_pinf; rho_tol = (real)P.rho_tol;
        zend[0] = zend[1] = endw[0] = endw[1] = real(0.0);
        cert_nrm = cert_lhs = real(0.0);
        suspect = 0;
        const bool warm = (ka.mode & 1) == 1;
        rho = warm ? static_cast<real *>(ka.rho_state)[qp + ka.qp0] : (real)P.rho0;
        rho = xmin(xmax(rho, real(kRhoMin)), real(kRhoMax));

        assemble(src, stride);
        store.fence();
        sync_warp(lane);
        scale_and_classify();
        store.fence();
        sync_warp(lane);
        init_iterates(warm);

        int status = kUnsolved;
        int iter = 0, rho_updates = 0;
        Norms nr;
        nr.pri = nr.dua = real(0.0);
        int to_check = P.check_every > 0 ? P.check_every : -1;
        int to_adapt = (P.adaptive_rho && P.adaptive_interval > 0) ? P.adaptive_interval : -1;
        bool need_factor = true, initial = true;
        // Heavy, rarely executed pieces (factorisation, rhs rebuild, residuals, termination) have
        // exactly one call site each: instruction-cache footprint matters once the resident
        // warps of an SM drift out of phase.
        PQP_ROLL
        for (;;) {
            if (need_factor) {
                store.fence();
                const bool fok = factor<double>();  // FP64 factorisation, FP32 factors
                store.fence();
                sync_warp(lane);
                if (!fok) { status = kNumerical; break; }
                if (Incr) build_rhs_incr(initial, warm);
                else build_rhs(initial, warm);
                need_factor = false;
                initial = false;
            }
            ++iter;
            solve();
            // iter % interval == 0 without an integer division in the loop
            const bool last = iter >= P.max_iter;
            const bool can_check = (--to_check == 0) || last;
            // OSQP adapts rho on the last iteration too (osqp_solve: the rho update follows the regular
            // termination check inside the loop body): no further solve uses the refactorisation, but the
            // adapted rho is what the next warm solve starts from
            const bool can_adapt = (--to_adapt == 0);
            if (to_check <= 0) to_check = P.check_every > 0 ? P.check_every : -1;
            if (to_adapt <= 0) to_adapt = (P.adaptive_rho && P.adaptive_interval > 0) ? P.adaptive_interval : -1;
            if (Incr) {
                if (can_check) admm_update_incr<true, true>(iter == 1, warm);
                else if (iter == 1) admm_update_incr<false, true>(true, warm);
                else admm_update_incr<false, false>(false, warm);
            } else {
                if (can_check) admm_update<true>(iter == 1, warm);
                else admm_update<false>(iter == 1, warm);
            }
            if (can_check || can_adapt) {
                nr = residuals();
                if (can_check) {
                    status = check_termination(nr, last);
                    // OSQP stops before the rho update only where the scheduled check inside its loop body decides
                    // the run (SOLVED, PRIMAL_INFEASIBLE). At the cap, osqp_solve's after-loop check (made when the
                    // last iteration had no scheduled one) and its 10x re-check follow that update; they see the
                    // same residuals and certificate terms, which the rescaling leaves unchanged. A scheduled check
                    // has just reset to_check to check_every, which an unscheduled iteration never leaves it at.
                    const bool scheduled = to_check == P.check_every;
                    const bool capped = last && status != kNumerical &&
                                        (!scheduled || status == kMaxIter || status == kSolvedInacc || status == kPrimInfInacc);
                    if (status != kUnsolved && !(capped && can_adapt)) break;
                }
                if (can_adapt && adapt_rho(nr)) {
                    ++rho_updates;
                    need_factor = true;
                }
                if (last) break;
            }
        }
        epilogue(status, iter, rho_updates, nr);
    }

    // -------------------------------------------------------------- outputs + warm state
    PQP_DEV void epilogue(int status, int iter, int rho_updates, const Norms &nr) {
        const DevParams &P = ka.prm;
        const int nmax = ka.n_max;
        const real c = cscale;
        double *sol = ka.sol + (size_t)qp * 4 * nmax;
        real cost = real(0.0);
        const int nvm = 6 * nmax - 1, mm = 6 * nmax + 2;
        double *xf = ka.x_full ? ka.x_full + (size_t)qp * nvm : nullptr;
        double *yf = ka.y_full ? ka.y_full + (size_t)qp * mm : nullptr;
        double *zf = ka.z_full ? ka.z_full + (size_t)qp * mm : nullptr;
        PQP_ROLL
        for (int k = 0; k < C; ++k) {
            const int g = lane * C + k;
            const StagePred sp = pred(k);
            StageRO q;
            Vec4 x0, x1, oy, cz;
            {
                real loaded[44];
                store.template ld4n_nowait<11>(GA0, k, loaded);
                store.wait_ld();
                unpack_stage(loaded, q, x0, x1, oy, cz);
            }
            const real l = x0.x, ps = x0.y, kp = x0.z, u = x0.w, s0 = x1.x, s1 = x1.y;
            if (sp.real) {
                const int i = g - 1;
                sol[0 * nmax + i] = (double)l;
                sol[1 * nmax + i] = (double)ps;
                sol[2 * nmax + i] = (double)kp;
                sol[3 * nmax + i] = sp.mid ? (double)u : 0.0;
                cost += real(0.5) * (w_l * l * l + w_kappa * kp * kp + (sp.mid ? w_dkappa * u * u : real(0.0)) +
                                w_slack * s0 * s0 + (sp.act1 ? w_slack * s1 * s1 : real(0.0)));
                if (xf) {
                    xf[3 * i] = l; xf[3 * i + 1] = ps; xf[3 * i + 2] = kp;
                    if (sp.mid) xf[3 * n + i] = u;
                    if (sp.act1) { xf[4 * n - 1 + 2 * i] = s0; xf[4 * n - 1 + 2 * i + 1] = s1; }
                    else xf[4 * n - 1 + 2 * p + (i - p)] = s0;
                }
            }
            // row values, read uniformly (the writes below are lane-divergent)
            real zo_[3], yo_[3];
            const real oyv[3] = {oy.x, oy.y, oy.z};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                zo_[r] = (sp.last && r < 2) ? zend[r] : q.ob[r];
                yo_[r] = q.Ro[r] * oyv[r];
            }
            const real zk_ = x1.z, yk_ = q.Rk * x1.w;
            const real zc0_ = cz.x, zc1_ = cz.y;
            const real yc0_ = q.Rc[0] * cz.z, yc1_ = q.Rc[1] * cz.w;
            // rows in the reference's order (SURVEY.md App. A.3)
            if (yf || zf) {
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    int row = -1;
                    if (g <= n - 1) row = 3 * g + r;           // outgoing rows of stage g = block g
                    else if (sp.last && r < 2) row = (4 * n + p + n) + r;  // m-2, m-1
                    if (row >= 0) {
                        if (yf) yf[row] = (double)yo_[r];
                        if (zf) zf[row] = (double)zo_[r];
                    }
                }
                if (sp.real) {
                    const int i = g - 1;
                    if (yf) yf[3 * n + i] = (double)yk_;
                    if (zf) zf[3 * n + i] = (double)zk_;
                    const int r0 = sp.act1 ? 4 * n + 2 * i : 4 * n + 2 * p + (i - p);
                    if (yf) yf[r0] = (double)yc0_;
                    if (zf) zf[r0] = (double)zc0_;
                    if (sp.act1) {
                        if (yf) yf[r0 + 1] = (double)yc1_;
                        if (zf) zf[r0 + 1] = (double)zc1_;
                    }
                }
            }
            // warm state: scaled iterates (x/d, e z, c y / e); a cold-only handle keeps none
            if (ka.mode & 2) continue;
            const real x6[6] = {l, ps, kp, u, s0, s1};
#pragma unroll
            for (int j = 0; j < 6; ++j) G(gwarm, WX + j, k) = x6[j] / G(gscal, GD + j, k);
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const real e = G(gscal, GE + r, k);
                G(gwarm, WOZ + r, k) = e * zo_[r];
                G(gwarm, WOY + r, k) = c * yo_[r] / e;
            }
            {
                const real e = G(gscal, GE + 3, k);
                G(gwarm, WKZ, k) = e * zk_;
                G(gwarm, WKY, k) = c * yk_ / e;
            }
            {
                const real e0 = G(gscal, GE + 4, k), e1 = G(gscal, GE + 5, k);
                G(gwarm, WCZ + 0, k) = e0 * zc0_;
                G(gwarm, WCY + 0, k) = c * yc0_ / e0;
                G(gwarm, WCZ + 1, k) = e1 * zc1_;
                G(gwarm, WCY + 1, k) = c * yc1_ / e1;
            }
        }
        cost = warp_sum(cost, lane);
        if (lane == 0) {
            if (ka.cost) ka.cost[qp] = (double)cost;
            if (ka.status) ka.status[qp] = status;
            if (ka.iters) ka.iters[qp] = iter;
            if (ka.flags) ka.flags[qp] = (status == kMaxIter || status == kUnsolved) ? suspect : 0;
            if (ka.info) {
                double *inf = ka.info + (size_t)qp * 4;
                inf[0] = nr.pri; inf[1] = nr.dua; inf[2] = rho; inf[3] = rho_updates;
            }
            if (!(ka.mode & 2)) static_cast<real *>(ka.rho_state)[qp + ka.qp0] = rho;
        }
    }
};

}  // namespace pqp
