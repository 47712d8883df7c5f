// Host build of clean_pvnet_b200/csrc/pnp_iter_core.cuh for the CPU test-suite (tests/test_pnp_iter_host_core.py).
// Test infrastructure only -- nothing in the product links or loads this.
#include "../clean_pvnet_b200/csrc/pnp_iter_core.cuh"

namespace {
struct SerialSum {                       // one "lane" owns every point: the sums are already complete
    template <int C> void sum(double *) const {}
};
}

// n problems, as pvb_pnp_iterative lays them out: pts2d [n][pn][2], pts3d / K at p * pts3d_stride / p * k_stride (doubles);
// pose [n][3][4], rt [n][6], info [n][2] = (iterations, status)
extern "C" void pnp_iter_host_solve(const double *pts2d, const double *pts3d, const double *K, double *pose, double *rt,
                                    int *info, int n, int pn, long long pts3d_stride, long long k_stride)
{
    for (int p = 0; p < n; ++p) {
        double cam[4];
        pvb::pnp_camera(K + p * k_stride, cam);
        int it = 0;
        const int st = pvb::pnp_iter_solve(pts2d + (long long)p * pn * 2, pts3d + p * pts3d_stride, cam, pn, 0, 1, SerialSum(),
                                           rt + 6 * p, it);
        pvb::pnp_iter_pose(rt + 6 * p, pose + 12 * p);
        info[2 * p] = it; info[2 * p + 1] = st;
    }
}

extern "C" void pnp_iter_host_rodrigues(const double *r, double *R, double *dRdr) { pvb::pnp_iter_rodrigues(r, R, dRdr); }

extern "C" void pnp_iter_host_rotation_to_vector(const double *R, double *r) { pvb::pnp_iter_rotation_to_vector(R, r); }
