/*
 * nn_oracle.c -- CPU restatement of clean-pvnet's nearest-neighbour kernel (lib/csrc/nn).
 *
 * TEST INFRASTRUCTURE ONLY, like pvnet_oracle.c: only tests/ build, load or call it; the product never links or
 * imports anything under oracle/.  It is the fallback reference where oracle/_ref/libnn_ref.so (the unmodified kernel,
 * built by oracle/build_nn_ref.py) was not built, and the subject of the CPU known-answer tests.
 *
 *   lib/csrc/nn/src/nearest_neighborhood.cu
 *     :48-117   findNearestPoint{3D,2D}IdxKernel    -> orc_nearest_point_idx
 *
 * The PTX of the reference build (nvcc -O2 -arch=sm_52, lib/csrc/nn/setup.py) computes, per (query p2, point p1):
 *   d? = ref.? - que.? (rounded), 3-D: dist = fma(dz, dz, fma(dx, dx, dy*dy)), 2-D: dist = fma(dx, dx, dy*dy)
 * and keeps the first p1 with dist < min_dist, from min_dist = FLT_MAX and min_idx = 0 (p1 == p2 skipped under
 * exclude_self).  NaN, +inf and FLT_MAX distances therefore never win.  Build with -ffp-contract=off (nn_oracle.py) so
 * the host compiler adds no fusions of its own.
 */
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define ORC_API __attribute__((visibility("default")))
#else
#define ORC_API
#endif

ORC_API void orc_nearest_point_idx(const float *ref, const float *que, int32_t *idxs, int b, int pn1, int pn2, int dim,
                                   int exclude_self)
{
    for (int bi = 0; bi < b; ++bi) {
        const float *r = ref + (size_t)bi * pn1 * dim, *q = que + (size_t)bi * pn2 * dim;
        for (int p2 = 0; p2 < pn2; ++p2) {
            const float x2 = q[(size_t)p2 * dim], y2 = q[(size_t)p2 * dim + 1], z2 = dim == 3 ? q[(size_t)p2 * dim + 2] : 0.f;
            float min_dist = FLT_MAX;
            int min_idx = 0;
            for (int p1 = 0; p1 < pn1; ++p1) {
                if (exclude_self && p1 == p2) continue;
                const float dx = r[(size_t)p1 * dim] - x2, dy = r[(size_t)p1 * dim + 1] - y2;
                float dist = fmaf(dx, dx, dy * dy);
                if (dim == 3) {
                    const float dz = r[(size_t)p1 * dim + 2] - z2;
                    dist = fmaf(dz, dz, dist);
                }
                if (dist < min_dist) { min_dist = dist; min_idx = p1; }
            }
            idxs[(size_t)bi * pn2 + p2] = min_idx;
        }
    }
}
