// cartesian_driver.cpp — runs the Cartesian tension QP of the CUDA library (pqp_smoother_core.cuh,
// cartesian_tension_smooth: TensionSmoother::osqpSmooth) on the CPU with one lane. TEST ONLY: lets `-m "not gpu"`
// tests check the kernel's source against oracle/cartesian_oracle.py on a GPU-less box. Not part of the product.
#include <vector>

#include "../../path_optimizer_2_b200/csrc/pqp_smoother_core.cuh"

extern "C" {
// weights[3] = curvature, curvature rate, deviation; set[13] = OSQP settings in the order of
// tests/emu/smoother_emu.DEFAULT_SETTINGS; x_full[3 p]; info[6] = status, iters, rho_updates, pri_res, dua_res, obj
int cartesian_emu(int p, const double *xl, const double *yl, const double *al, const double *cl, const double *weights,
                  const double *set, double *rx, double *ry, double *rs, double *x_full, double *info) {
    pqs::Settings st;
    st.rho = set[0]; st.sigma = set[1]; st.alpha = set[2]; st.eps_abs = set[3]; st.eps_rel = set[4]; st.eps_prim_inf = set[5];
    st.eps_dual_inf = set[6]; st.adaptive_rho_tolerance = set[7];
    st.max_iter = (int)set[8]; st.check_termination = (int)set[9]; st.scaling = (int)set[10]; st.adaptive_rho = (int)set[11];
    st.adaptive_rho_interval = (int)set[12];
    std::vector<unsigned char> scratch(pqs::cartesian_scratch_bytes(p));
    std::vector<double> band(pqs::cartesian_band_doubles(p));
    pqs::Work W;
    pqs::cartesian_carve(W, scratch.data(), p, band.data());
    const pqs::CartesianWeights cw = {weights[0], weights[1], weights[2]};
    const pqs::Result R = pqs::cartesian_tension_smooth(pqs::SerialLane(), W, st, cw, p, xl, yl, al, cl, rx, ry, rs, x_full);
    info[0] = R.status; info[1] = R.iters; info[2] = R.rho_updates; info[3] = R.pri_res; info[4] = R.dua_res; info[5] = R.obj;
    return 0;
}
}
