// pqp_host_common.h — host-side helpers shared by the CUDA library (pqp_api.cu) and the
// test-only emulator driver (tests/emu/emu_driver.cpp): parameter conversion and buffer
// sizing. No device code here.
#pragma once
#include <cmath>
#include <cstddef>

#include "../../include/pqp.h"
#include "pqp_kernel.cuh"

namespace pqp {

inline void default_params(pqp_params *p) {
    p->front_length = 3.9;
    p->rear_length = -1.0;
    p->wheel_base = 2.5;
    p->max_steering_angle = 35.0 * M_PI / 180.0;
    p->expected_safety_margin = 0.6;
    p->weight_l = 0.0;
    p->weight_kappa = 20.0;
    p->weight_dkappa = 100.0;
    p->weight_slack = 10.0;
    p->end_l_lb = -1.0;
    p->end_l_ub = 1.0;
    p->rho = 0.1;
    p->sigma = 1e-6;
    p->alpha = 1.6;
    p->eps_abs = 2e-3;
    p->eps_rel = 2e-3;
    p->eps_prim_inf = 1e-4;
    p->eps_dual_inf = 1e-4;
    p->adaptive_rho_tolerance = 5.0;
    p->max_iter = 4000;
    p->check_termination = 25;
    p->scaling = 10;
    p->adaptive_rho = 1;
    p->adaptive_rho_interval = 25;
    p->reserved = 0;
}

inline DevParams make_dev_params(const pqp_params &p) {
    DevParams d;
    d.front_length = p.front_length;
    d.rear_length = p.rear_length;
    d.kappa_limit = std::tan(p.max_steering_angle) / p.wheel_base;  // base_solver.cpp:226
    d.safety_margin = p.expected_safety_margin;
    d.end_l_lb = p.end_l_lb;
    d.end_l_ub = p.end_l_ub;
    d.w_l = p.weight_l;
    d.w_kappa = p.weight_kappa;
    d.w_dkappa = p.weight_dkappa;
    d.w_slack = p.weight_slack;
    d.rho0 = p.rho;
    d.sigma = p.sigma;
    d.alpha = p.alpha;
    d.eps_abs = p.eps_abs;
    d.eps_rel = p.eps_rel;
    d.eps_pinf = p.eps_prim_inf;
    d.eps_dinf = p.eps_dual_inf;
    d.rho_tol = p.adaptive_rho_tolerance;
    d.max_iter = p.max_iter;
    d.check_every = p.check_termination;
    d.scaling = p.scaling;
    d.adaptive_rho = p.adaptive_rho;
    d.adaptive_interval = p.adaptive_rho_interval;
    d.reserved0 = 0;
    return d;
}

// stages per lane: the chain has n+1 stages (virtual x0 stage + n knots) over 32 lanes
inline int chunk_for(int n_max) {
    int c = 1;
    while (32 * c < n_max + 1) c *= 2;
    return c;
}
constexpr int kMaxChunk = 16;           // n_max <= 511
inline size_t smem_floats(int c) { return (size_t)NFIELD * c * 32; }
inline size_t warm_floats(int c) { return (size_t)NWARM * c * 32; }
inline size_t scal_floats(int c) { return (size_t)NSCAL * c * 32; }
inline size_t dy_floats(int c) { return (size_t)NDY * c * 32; }

// The OSQP settings are checked as OSQP 0.6's validate_settings checks them (as recalled from its sources, which
// are not in this tree); the vehicle and weight fields as the QP needs them: a positive curvature limit
// tan(max_steering_angle) / wheel_base and a positive semidefinite P.
inline bool params_valid(const pqp_params &p) {
    const double fields[] = {p.front_length, p.rear_length, p.wheel_base, p.max_steering_angle,
                             p.expected_safety_margin, p.weight_l, p.weight_kappa, p.weight_dkappa, p.weight_slack,
                             p.end_l_lb, p.end_l_ub, p.rho, p.sigma, p.alpha, p.eps_abs, p.eps_rel, p.eps_prim_inf,
                             p.eps_dual_inf, p.adaptive_rho_tolerance};
    for (double v : fields)
        if (!std::isfinite(v)) return false;
    return p.wheel_base > 0 && p.max_steering_angle > 0 && p.max_steering_angle < M_PI / 2 &&
           p.weight_l >= 0 && p.weight_kappa >= 0 && p.weight_dkappa >= 0 && p.weight_slack >= 0 &&
           p.rho > 0 && p.sigma > 0 && p.alpha > 0 && p.alpha < 2 &&
           p.eps_abs >= 0 && p.eps_rel >= 0 && (p.eps_abs > 0 || p.eps_rel > 0) &&
           p.eps_prim_inf > 0 && p.eps_dual_inf > 0 && p.adaptive_rho_tolerance >= 1 &&
           p.max_iter > 0 && p.check_termination >= 0 && p.scaling >= 0 &&
           (p.adaptive_rho == 0 || p.adaptive_rho == 1) && p.adaptive_rho_interval >= 0;
}

}  // namespace pqp
