// Host build of clean_pvnet_b200/csrc/pnp_core.cuh for the CPU test-suite (tests/test_pnp_host_core.py): the same
// arithmetic and the same pnp_solve loop the CUDA kernel runs, with a serial sum over the points as its evaluation instead
// of the warp reduction.  Test infrastructure only -- nothing in the product links or loads this.
#include "../clean_pvnet_b200/csrc/pnp_core.cuh"

static void normal_at(const double *pose, const double *pts2d, const double *pts3d, const double *wgt2d, const double *cam,
                      int pn, pvb::PnpNormal &n)
{
    pvb::pnp_normal_zero(n);
    for (int i = 0; i < pn; ++i) pvb::pnp_accumulate_point(pose, pts3d + 3 * i, pts2d + 2 * i, wgt2d + 3 * i, cam, n);
}

extern "C" int pnp_host_solve(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                              const double *init_rt, double *result_rt, int *info, int pn, int max_num_iterations,
                              double function_tolerance, double gradient_tolerance, double parameter_tolerance)
{
    double cam[4];
    pvb::pnp_camera(K, cam);
    pvb::PnpOptions opt;
    opt.max_num_iterations = max_num_iterations; opt.function_tolerance = function_tolerance;
    opt.gradient_tolerance = gradient_tolerance; opt.parameter_tolerance = parameter_tolerance;
    pvb::PnpState st;
    pvb::pnp_solve(opt, init_rt, [&](const double *pose, pvb::PnpNormal &n) { normal_at(pose, pts2d, pts3d, wgt2d, cam, pn, n); },
                   st);
    for (int i = 0; i < 6; ++i) result_rt[i] = st.x[i];
    if (info) { info[0] = st.iterations; info[1] = st.code; }
    return 0;
}

extern "C" void pnp_host_normal(const double *pose, const double *pts2d, const double *pts3d, const double *wgt2d,
                                const double *K, int pn, double *H21, double *g6, double *cost)
{
    double cam[4];
    pvb::pnp_camera(K, cam);
    pvb::PnpNormal n;
    normal_at(pose, pts2d, pts3d, wgt2d, cam, pn, n);
    for (int i = 0; i < 21; ++i) H21[i] = n.H[i];
    for (int i = 0; i < 6; ++i) g6[i] = n.g[i];
    *cost = n.cost;
}
