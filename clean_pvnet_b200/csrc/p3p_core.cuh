// p3p_core.cuh -- closed-form initial pose of the uncertainty PnP: perspective-3-point + a 4th point to choose the root.
//
// Replaces the host step `cv2.solvePnP(points_3d[idxs], points_2d[idxs], K, dist, flags=cv2.SOLVEPNP_P3P)` of
// lib/csrc/uncertainty_pnp/un_pnp_utils.py:25-31 (idxs = the 4 best-weighted keypoints, ascending): the first three
// correspondences give up to four poses, the fourth picks the one that reprojects it best.  OpenCV is a third-party
// dependency of the reference, not part of its sources; this file does NOT restate OpenCV's p3p.cpp but solves the same
// problem by Grunert's elimination written as polynomial arithmetic:
//     depths s1, s2 = u*s1, s3 = v*s1 along the unit bearings f1, f2, f3;  a,b,c = |X2-X3|, |X1-X3|, |X1-X2|
//     q(v) = 1 - 2 cos(b) v + v^2,   N(v) = b^2 (v^2 - 1) + (c^2 - a^2) q(v),   D(v) = 2 b^2 (cos(a) v - cos(g))
//     u = N/D,   quartic:  b^2 N^2 - 2 b^2 cos(g) N D + (b^2 - c^2 q) D^2 = 0,   s1 = b / sqrt(q(v))
// (cos(a) = f2.f3, cos(b) = f1.f3, cos(g) = f1.f2).  Real roots by Ferrari + Newton polishing; rigid alignment of the three
// camera-frame points with the model points by orthonormal frames.  The set of solutions is the same as OpenCV's (it is the
// set of solutions of the P3P problem); tests/test_p3p_host_core.py pins the selected pose against cv2.solvePnP itself.
//
// Plain double arithmetic, compiles as device code and -- for the CPU test-suite only -- as host code.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define PVB_HD __host__ __device__ __forceinline__
#else
#define PVB_HD inline
#endif

namespace pvb {

PVB_HD double p3p_dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
PVB_HD void p3p_cross(const double *a, const double *b, double *c)
{
    c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
PVB_HD bool p3p_normalize(double *a)
{
    const double n = sqrt(p3p_dot(a, a));
    if (!(n > 0.0)) return false;
    a[0] /= n; a[1] /= n; a[2] /= n;
    return true;
}

// real roots of x^3 + b x^2 + c x + d: returns the largest one (always exists)
PVB_HD double p3p_cubic_largest_root(double b, double c, double d)
{
    const double p = c - b * b / 3.0, q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d;
    const double disc = q * q / 4.0 + p * p * p / 27.0;
    double y;
    if (disc > 0.0) {
        const double sq = sqrt(disc);
        y = cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq);
    } else if (p < 0.0) {
        const double m = 2.0 * sqrt(-p / 3.0);
        double arg = 3.0 * q / (p * m);
        arg = fmin(1.0, fmax(-1.0, arg));
        y = m * cos(acos(arg) / 3.0);                  // k = 0 branch is the largest of the three
    } else {
        y = 0.0;                                       // p == q == 0
    }
    double x = y - b / 3.0;
    for (int it = 0; it < 3; ++it) {                   // polish on the original cubic
        const double f = ((x + b) * x + c) * x + d, df = (3.0 * x + 2.0 * b) * x + c;
        if (df != 0.0 && fabs(f) > 0.0) x -= f / df;
    }
    return x;
}

// real roots of k[4] x^4 + ... + k[0]; returns their number (0..4), roots[] unsorted, polished on the original polynomial
PVB_HD int p3p_quartic_real_roots(const double *k, double *roots)
{
    if (!(fabs(k[4]) > 0.0)) return 0;
    const double B = k[3] / k[4], C = k[2] / k[4], Dd = k[1] / k[4], E = k[0] / k[4];
    const double p = C - 3.0 * B * B / 8.0;
    const double q = Dd - B * C / 2.0 + B * B * B / 8.0;
    const double r = E - B * Dd / 4.0 + B * B * C / 16.0 - 3.0 * B * B * B * B / 256.0;
    double y[4];
    int n = 0;
    const double scale = fabs(p) + sqrt(fabs(r)) + 1e-300;
    if (fabs(q) <= 1e-14 * scale * sqrt(scale)) {      // biquadratic  y^4 + p y^2 + r
        const double disc = p * p - 4.0 * r;
        if (disc >= 0.0) {
            const double sq = sqrt(disc);
            const double z1 = (-p + sq) / 2.0, z2 = (-p - sq) / 2.0;
            if (z1 >= 0.0) { y[n++] = sqrt(z1); y[n++] = -sqrt(z1); }
            if (z2 >= 0.0) { y[n++] = sqrt(z2); y[n++] = -sqrt(z2); }
        }
    } else {
        // resolvent  z^3 + 2p z^2 + (p^2 - 4r) z - q^2 = 0 has a positive root z = w^2
        const double z = p3p_cubic_largest_root(2.0 * p, p * p - 4.0 * r, -q * q);
        if (z > 0.0) {
            const double w = sqrt(z);
            const double h1 = (p + z) / 2.0 - q / (2.0 * w), h2 = (p + z) / 2.0 + q / (2.0 * w);
            double disc = w * w - 4.0 * h1;            // y^2 + w y + h1
            if (disc >= 0.0) { const double sq = sqrt(disc); y[n++] = (-w + sq) / 2.0; y[n++] = (-w - sq) / 2.0; }
            disc = w * w - 4.0 * h2;                   // y^2 - w y + h2
            if (disc >= 0.0) { const double sq = sqrt(disc); y[n++] = (w + sq) / 2.0; y[n++] = (w - sq) / 2.0; }
        }
    }
    for (int i = 0; i < n; ++i) {
        double x = y[i] - B / 4.0;
        for (int it = 0; it < 4; ++it) {
            const double f = (((k[4] * x + k[3]) * x + k[2]) * x + k[1]) * x + k[0];
            const double df = ((4.0 * k[4] * x + 3.0 * k[3]) * x + 2.0 * k[2]) * x + k[1];
            if (df != 0.0 && f != 0.0) x -= f / df;
        }
        roots[i] = x;
    }
    return n;
}

// rotation matrix (row-major) -> angle-axis with angle in [0, pi]  (what cv2.Rodrigues returns for a matrix)
PVB_HD void p3p_rotation_to_angle_axis(const double R[3][3], double *aa)
{
    // unit quaternion by the largest-diagonal branch, then the log map
    double qw, qx, qy, qz;
    const double tr = R[0][0] + R[1][1] + R[2][2];
    if (tr > 0.0) {
        const double s = sqrt(tr + 1.0) * 2.0;
        qw = 0.25 * s; qx = (R[2][1] - R[1][2]) / s; qy = (R[0][2] - R[2][0]) / s; qz = (R[1][0] - R[0][1]) / s;
    } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
        const double s = sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]) * 2.0;
        qw = (R[2][1] - R[1][2]) / s; qx = 0.25 * s; qy = (R[0][1] + R[1][0]) / s; qz = (R[0][2] + R[2][0]) / s;
    } else if (R[1][1] > R[2][2]) {
        const double s = sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]) * 2.0;
        qw = (R[0][2] - R[2][0]) / s; qx = (R[0][1] + R[1][0]) / s; qy = 0.25 * s; qz = (R[1][2] + R[2][1]) / s;
    } else {
        const double s = sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]) * 2.0;
        qw = (R[1][0] - R[0][1]) / s; qx = (R[0][2] + R[2][0]) / s; qy = (R[1][2] + R[2][1]) / s; qz = 0.25 * s;
    }
    if (qw < 0.0) { qw = -qw; qx = -qx; qy = -qy; qz = -qz; }
    const double vn = sqrt(qx * qx + qy * qy + qz * qz);
    if (vn < 1e-300) { aa[0] = aa[1] = aa[2] = 0.0; return; }
    const double theta = 2.0 * atan2(vn, qw), f = theta / vn;
    aa[0] = qx * f; aa[1] = qy * f; aa[2] = qz * f;
}

// idx[0..3] = the tail of a stable ascending argsort of key_i = wxx_i + wxy_i (un_pnp_utils.py:25: `np.argsort(...)[-4:]`):
// repeatedly the largest remaining key, the larger index among equals; NaN keys sort last (largest), as in numpy.
PVB_HD void p3p_select4(const double *w /*[pn][3]*/, int pn, int *idx)
{
    idx[0] = idx[1] = idx[2] = idx[3] = -1;
    for (int r = 3; r >= 0; --r) {
        int best = -1;
        double bk = 0.0;
        bool bnan = false;
        for (int i = 0; i < pn; ++i) {
            if (i == idx[0] || i == idx[1] || i == idx[2] || i == idx[3]) continue;
            const double key = w[3 * i] + w[3 * i + 1];
            const bool knan = key != key;
            if (best < 0 || knan || (!bnan && key >= bk)) { best = i; bk = key; bnan = knan; }
        }
        idx[r] = best;
    }
}

// P3P on correspondences 0,1,2; correspondence 3 chooses among the real solutions (smallest reprojection error in pixels).  X: 4 model points [4][3]; x2: 4 image points [4][2]; cam = (fx, fy, px, py).
// Writes rt[6] = (angle-axis, translation).  Returns the number of admissible solutions found (0: rt untouched).
PVB_HD int p3p_solve4(const double X[4][3], const double x2[4][2], const double *cam, double *rt)
{
    // Three coincident image points (an image the voting layer skipped: every keypoint at 0) put the three bearings on one
    // ray, which cannot carry three non-collinear model points: no solution.  Tested up front because with cos = 1 the
    // quartic degenerates and its rounding noise can pass for a root (the device build, with FMA contraction, found one).
    if (x2[0][0] == x2[1][0] && x2[0][1] == x2[1][1] && x2[0][0] == x2[2][0] && x2[0][1] == x2[2][1]) return 0;
    double f[4][3];
    for (int i = 0; i < 4; ++i) {
        f[i][0] = (x2[i][0] - cam[2]) / cam[0]; f[i][1] = (x2[i][1] - cam[3]) / cam[1]; f[i][2] = 1.0;
    }
    const double m3x = f[3][0], m3y = f[3][1];
    for (int i = 0; i < 3; ++i) if (!p3p_normalize(f[i])) return 0;
    const double ca = p3p_dot(f[1], f[2]), cb = p3p_dot(f[0], f[2]), cg = p3p_dot(f[0], f[1]);
    double d12[3], d13[3], d23[3];
    for (int r = 0; r < 3; ++r) { d12[r] = X[1][r] - X[0][r]; d13[r] = X[2][r] - X[0][r]; d23[r] = X[2][r] - X[1][r]; }
    const double a2 = p3p_dot(d23, d23), b2 = p3p_dot(d13, d13), c2 = p3p_dot(d12, d12);
    if (!(a2 > 0.0 && b2 > 0.0 && c2 > 0.0)) return 0;
    // polynomials in v (ascending coefficients)
    const double q[3] = { 1.0, -2.0 * cb, 1.0 };
    const double N[3] = { -b2 + (c2 - a2), (c2 - a2) * q[1], b2 + (c2 - a2) };
    const double D[2] = { -2.0 * b2 * cg, 2.0 * b2 * ca };
    double NN[5] = { 0, 0, 0, 0, 0 }, ND[4] = { 0, 0, 0, 0 }, DD[3] = { 0, 0, 0 }, QDD[5] = { 0, 0, 0, 0, 0 };
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) NN[i + j] += N[i] * N[j];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 2; ++j) ND[i + j] += N[i] * D[j];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) DD[i + j] += D[i] * D[j];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) QDD[i + j] += q[i] * DD[j];
    double k[5];
    for (int i = 0; i < 5; ++i)
        k[i] = b2 * NN[i] - (i < 4 ? 2.0 * b2 * cg * ND[i] : 0.0) + (i < 3 ? b2 * DD[i] : 0.0) - c2 * QDD[i];
    double roots[4];
    const int nr = p3p_quartic_real_roots(k, roots);

    // model frame of the three points
    double ex[3] = { d12[0], d12[1], d12[2] }, ez[3], ey[3];
    if (!p3p_normalize(ex)) return 0;
    p3p_cross(ex, d13, ez);
    if (!p3p_normalize(ez)) return 0;                  // collinear model points
    p3p_cross(ez, ex, ey);

    int found = 0;
    double best = 1.79769313486231570e308;
    for (int ri = 0; ri < nr; ++ri) {
        const double v = roots[ri];
        if (!(v > 0.0)) continue;
        const double qv = (v + q[1]) * v + 1.0, Dv = D[1] * v + D[0], Nv = (N[2] * v + N[1]) * v + N[0];
        if (!(qv > 0.0) || !(fabs(Dv) > 1e-12 * b2)) continue;
        const double u = Nv / Dv;
        if (!(u > 0.0)) continue;
        double s1 = sqrt(b2 / qv), s2 = u * s1, s3 = v * s1;
        // Newton polish of the depths on the three distance equations (the quartic root loses digits when D(v) is small
        // or two roots are close; two or three steps restore them)
        for (int it = 0; it < 3; ++it) {
            const double F0 = s2 * s2 + s3 * s3 - 2.0 * s2 * s3 * ca - a2;
            const double F1 = s1 * s1 + s3 * s3 - 2.0 * s1 * s3 * cb - b2;
            const double F2 = s1 * s1 + s2 * s2 - 2.0 * s1 * s2 * cg - c2;
            const double J[3][3] = { { 0.0, 2.0 * (s2 - s3 * ca), 2.0 * (s3 - s2 * ca) },
                                     { 2.0 * (s1 - s3 * cb), 0.0, 2.0 * (s3 - s1 * cb) },
                                     { 2.0 * (s1 - s2 * cg), 2.0 * (s2 - s1 * cg), 0.0 } };
            const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1]) - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0]) +
                               J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
            if (!(fabs(det) > 1e-300)) break;
            const double d1 = (F0 * (J[1][1] * J[2][2] - J[1][2] * J[2][1]) - J[0][1] * (F1 * J[2][2] - J[1][2] * F2) +
                               J[0][2] * (F1 * J[2][1] - J[1][1] * F2)) / det;
            const double d2 = (J[0][0] * (F1 * J[2][2] - J[1][2] * F2) - F0 * (J[1][0] * J[2][2] - J[1][2] * J[2][0]) +
                               J[0][2] * (J[1][0] * F2 - F1 * J[2][0])) / det;
            const double d3 = (J[0][0] * (J[1][1] * F2 - F1 * J[2][1]) - J[0][1] * (J[1][0] * F2 - F1 * J[2][0]) +
                               F0 * (J[1][0] * J[2][1] - J[1][1] * J[2][0])) / det;
            const double n1 = s1 - d1, n2 = s2 - d2, n3 = s3 - d3;
            if (!(n1 > 0.0 && n2 > 0.0 && n3 > 0.0)) break;
            s1 = n1; s2 = n2; s3 = n3;
        }
        double P[3][3];
        for (int r = 0; r < 3; ++r) { P[0][r] = s1 * f[0][r]; P[1][r] = s2 * f[1][r]; P[2][r] = s3 * f[2][r]; }
        double px[3], pd13[3], pz[3], py[3];
        for (int r = 0; r < 3; ++r) { px[r] = P[1][r] - P[0][r]; pd13[r] = P[2][r] - P[0][r]; }
        if (!p3p_normalize(px)) continue;
        p3p_cross(px, pd13, pz);
        if (!p3p_normalize(pz)) continue;
        p3p_cross(pz, px, py);
        double R[3][3], t[3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[i][j] = px[i] * ex[j] + py[i] * ey[j] + pz[i] * ez[j];
        for (int i = 0; i < 3; ++i) t[i] = P[0][i] - (R[i][0] * X[0][0] + R[i][1] * X[0][1] + R[i][2] * X[0][2]);
        // the fourth point decides
        double c3[3];
        for (int i = 0; i < 3; ++i) c3[i] = R[i][0] * X[3][0] + R[i][1] * X[3][1] + R[i][2] * X[3][2] + t[i];
        const double ex3 = cam[0] * (c3[0] / c3[2] - m3x), ey3 = cam[1] * (c3[1] / c3[2] - m3y);   // pixels, like OpenCV's ranking
        const double err = ex3 * ex3 + ey3 * ey3;
        ++found;
        if (found == 1 || err < best || best != best) {
            best = err;
            p3p_rotation_to_angle_axis(R, rt);
            rt[3] = t[0]; rt[4] = t[1]; rt[5] = t[2];
        }
    }
    return found;
}

} // namespace pvb
