// bspline_driver.cpp — TEST ONLY. Compiles the B-spline stage of the plan glue (pqp_plan_core.cuh: bspline_prepare
// and bspline_eval, the code of bspline_prep_kernel and bspline_eval_kernel) for the host, so its samples, counts and
// degrees can be checked against oracle/bspline_oracle.py on a GPU-less box. Not part of the product.
#include <vector>

#include "../../path_optimizer_2_b200/csrc/pqp_plan_core.cuh"

extern "C" {
// one path as the two kernels run it: info[2] = r, degree; x / y [cap] receive the samples when the status is OK
int bspline_emu(const double *px, const double *py, int m, int m_max, int cap, double *x, double *y, int *info) {
    std::vector<double> t(cap > 0 ? cap : 1);
    int r, degree;
    const int st = pqpl::bspline_prepare(px, py, m, m_max, cap, t.data(), r, degree);
    info[0] = r;
    info[1] = degree;
    if (st == pqpl::kOk)
        for (int j = 0; j < r; ++j) pqpl::bspline_eval(px, py, m, degree, t[j], x[j], y[j]);
    return st;
}

// de Boor at arbitrary parameters (degree 3 to 5, m > degree)
void bspline_emu_eval(const double *px, const double *py, int m, int degree, const double *t, int n, double *x, double *y) {
    for (int j = 0; j < n; ++j) pqpl::bspline_eval(px, py, m, degree, t[j], x[j], y[j]);
}
}
