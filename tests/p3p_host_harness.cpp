// Host build of clean_pvnet_b200/csrc/p3p_core.cuh for the CPU test-suite (tests/test_p3p_host_core.py).
// Test infrastructure only -- nothing in the product links or loads this.
#include "../clean_pvnet_b200/csrc/p3p_core.cuh"
#include "../clean_pvnet_b200/csrc/pnp_core.cuh"

extern "C" int p3p_host_solve4(const double *pts3d /*[4][3]*/, const double *pts2d /*[4][2]*/, const double *K /*[3][3]*/,
                               double *rt /*[6]*/)
{
    double X[4][3], x2[4][2];
    for (int i = 0; i < 4; ++i) {
        for (int r = 0; r < 3; ++r) X[i][r] = pts3d[i * 3 + r];
        x2[i][0] = pts2d[i * 2]; x2[i][1] = pts2d[i * 2 + 1];
    }
    double cam[4];
    pvb::pnp_camera(K, cam);
    return pvb::p3p_solve4(X, x2, cam, rt);
}

extern "C" int p3p_host_quartic(const double *k, double *roots) { return pvb::p3p_quartic_real_roots(k, roots); }

extern "C" void p3p_host_select4(const double *w, int pn, int *idx) { pvb::p3p_select4(w, pn, idx); }

// the whole start as the kernel runs it: pts2d [pn][2], pts3d [pn][3], w [pn][3] -> rt [6]
extern "C" void p3p_host_start(const double *pts2d, const double *pts3d, const double *w, int pn, const double *K, double *rt)
{
    double cam[4];
    pvb::pnp_camera(K, cam);
    pvb::p3p_start(pts2d, pts3d, w, pn, cam, rt);
}
