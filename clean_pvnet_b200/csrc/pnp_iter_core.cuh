// pnp_iter_core.cuh -- PVNet's default pose step, `cv2.solvePnP(kpt_3d, kpt_2d, K, zeros(8), flags=SOLVEPNP_ITERATIVE)`
// (lib/utils/pvnet/pvnet_pose_utils.py:5-38, called by lib/evaluators/linemod/pvnet.py:188 and tless_test/pvnet.py:239).
//
// OpenCV's method step for step, for zero distortion and no extrinsic guess (findExtrinsicCameraParams2 and CvLevMarq,
// OpenCV 4.13 calibration_base.cpp; pinned against cv2.solvePnP itself by tests/test_pnp_iter_host_core.py):
//   1. normalise the image points: xn = (u - cx) * (1/fx), yn = (v - cy) * (1/fy); K's skew and bottom row are ignored;
//   2. classify the model: W = singular values of the centred 3x3 scatter matrix; W[2]/W[1] < 1e-3 is planar (OpenCV
//      starts from a homography there: not built, PNP_ITER_PLANAR); a non-planar model needs pn >= 6 for the DLT;
//   3. DLT start: the eigenvector of the smallest eigenvalue of L^T L (L: 2pn x 12, two rows per point) read as [RR | tt],
//      negated when det(RR) < 0; sc = |RR|_F > DBL_EPSILON; R = U V^T of RR's SVD; t = tt |R|_F / sc; rvec = Rodrigues(R);
//   4. Levenberg-Marquardt on (rvec, t), residuals = projection - pixel, Jacobian as projectPoints builds it: each step
//      solves (J^T J with its diagonal times 1 + lambda) d = J^T e, p = p_prev - d, lambda = exp(k log 10), k from -3; a step
//      that raises |e| is retried with k + 1 while k <= 16; afterwards k = max(k - 1, -16); stop after 20 iterations or when
//      |p - p_prev| / (|p_prev| + DBL_EPSILON) < FLT_EPSILON.
// The dense algebra is this file's own: cyclic Jacobi for the 12x12 eigenproblem and the 3x3 SVDs, Cholesky for the 6x6
// step (OpenCV uses an SVD; the step is the same to rounding on the positive definite damped system).
//
// Plain double arithmetic like pnp_core.cuh: compiled as device code (pnp.cu, one warp per problem) and, for the CPU
// test-suite only, as host code (tests/pnp_iter_host_harness.cpp).  Every point loop runs over i = first, first + stride, ...
// and every sum over points goes through `red.template sum<C>(v)`, which adds C numbers across the group in place (an XOR
// butterfly in the kernel, nothing in the serial host build), so every lane ends with the same bits and runs the same code.
#pragma once
#include <math.h>
#include "pnp_core.cuh"

namespace pvb {

// status written to info[1] (pvb_pnp_status in include/pvnet_vote_b200.h)
enum { PNP_ITER_OK = 0, PNP_ITER_LIMIT = 1, PNP_ITER_TOO_FEW = 2, PNP_ITER_PLANAR = 3, PNP_ITER_DEGENERATE = 4 };
constexpr int PNP_ITER_MAX_ITER = 20;                          // findExtrinsicCameraParams2's max_iter
constexpr double PNP_ITER_DBL_EPS = 2.220446049250313e-16;     // DBL_EPSILON
constexpr double PNP_ITER_FLT_EPS = 1.1920928955078125e-07;    // FLT_EPSILON, CvLevMarq's epsilon

// Cyclic Jacobi on the symmetric N x N matrix A (row-major, destroyed: its diagonal ends as the eigenvalues); V gets the
// eigenvectors as columns.  A rotation is skipped where |a_pq| <= DBL_EPSILON sqrt(|a_pp a_qq|), which keeps small
// eigenvalues of a semi-definite matrix to high relative accuracy; the loop ends after a sweep without a rotation.
template <int N>
PVB_HD void pnp_iter_jacobi(double *A, double *V)
{
    for (int i = 0; i < N * N; ++i) V[i] = 0.0;
    for (int i = 0; i < N; ++i) V[i * N + i] = 1.0;
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < N - 1; ++p) {
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[p * N + q], app = A[p * N + p], aqq = A[q * N + q];
                if (!(fabs(apq) > PNP_ITER_DBL_EPS * sqrt(fabs(app) * fabs(aqq)))) continue;
                rotated = true;
                const double theta = (aqq - app) / (2.0 * apq);
                double t = fabs(theta) > 1e150 ? 0.5 / theta
                                               : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                A[p * N + p] = app - t * apq;
                A[q * N + q] = aqq + t * apq;
                A[p * N + q] = A[q * N + p] = 0.0;
                for (int r = 0; r < N; ++r) {
                    if (r != p && r != q) {
                        const double arp = A[r * N + p], arq = A[r * N + q];
                        A[r * N + p] = A[p * N + r] = c * arp - s * arq;
                        A[r * N + q] = A[q * N + r] = s * arp + c * arq;
                    }
                    const double vrp = V[r * N + p], vrq = V[r * N + q];
                    V[r * N + p] = c * vrp - s * vrq;
                    V[r * N + q] = s * vrp + c * vrq;
                }
            }
        }
        if (!rotated) break;
    }
}

// R = U V^T of the SVD A = U W V^T of a 3x3 matrix (row-major), by one-sided Jacobi: plane rotations V orthogonalise the
// columns of B = A V, then w_k = |b_k| and u_k = b_k / w_k.  Working on A itself rather than on A^T A keeps the small
// singular directions accurate (a poor DLT start can be close to rank one).  A rank-deficient A (w_k <= DBL_EPSILON
// max w) takes u_k from the cross product of the other two.
PVB_HD void pnp_iter_orthonormal(const double *A, double *R)
{
    double B[3][3], V[3][3];                           // B[k], V[k]: column k
    for (int k = 0; k < 3; ++k)
        for (int r = 0; r < 3; ++r) { B[k][r] = A[r * 3 + k]; V[k][r] = r == k ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < 2; ++p) {
            for (int q = p + 1; q < 3; ++q) {
                double al = 0.0, be = 0.0, ga = 0.0;
                for (int r = 0; r < 3; ++r) { al += B[p][r] * B[p][r]; be += B[q][r] * B[q][r]; ga += B[p][r] * B[q][r]; }
                if (!(fabs(ga) > PNP_ITER_DBL_EPS * sqrt(al * be))) continue;
                rotated = true;
                const double zeta = (be - al) / (2.0 * ga);
                const double t = fabs(zeta) > 1e150 ? 0.5 / zeta
                                                    : (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(zeta * zeta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int r = 0; r < 3; ++r) {
                    const double bp = B[p][r], bq = B[q][r], vp = V[p][r], vq = V[q][r];
                    B[p][r] = c * bp - s * bq; B[q][r] = s * bp + c * bq;
                    V[p][r] = c * vp - s * vq; V[q][r] = s * vp + c * vq;
                }
            }
        }
        if (!rotated) break;
    }
    double w[3], wmax = 0.0;
    for (int k = 0; k < 3; ++k) { w[k] = sqrt(B[k][0] * B[k][0] + B[k][1] * B[k][1] + B[k][2] * B[k][2]); wmax = fmax(wmax, w[k]); }
    int bad = -1;
    for (int k = 0; k < 3; ++k) {
        if (w[k] > PNP_ITER_DBL_EPS * wmax) for (int r = 0; r < 3; ++r) B[k][r] /= w[k];
        else bad = k;
    }
    if (bad >= 0) {                                    // u_bad = u_a x u_b, signed so that U has V's determinant
        const int a = (bad + 1) % 3, b = (bad + 2) % 3;
        B[bad][0] = B[a][1] * B[b][2] - B[a][2] * B[b][1];
        B[bad][1] = B[a][2] * B[b][0] - B[a][0] * B[b][2];
        B[bad][2] = B[a][0] * B[b][1] - B[a][1] * B[b][0];
        const double detv = V[0][0] * (V[1][1] * V[2][2] - V[1][2] * V[2][1]) - V[0][1] * (V[1][0] * V[2][2] - V[1][2] * V[2][0]) +
                            V[0][2] * (V[1][0] * V[2][1] - V[1][1] * V[2][0]);
        if (detv < 0) for (int r = 0; r < 3; ++r) B[bad][r] = -B[bad][r];
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i * 3 + j] = B[0][i] * V[0][j] + B[1][i] * V[1][j] + B[2][i] * V[2][j];
}

// cv::Rodrigues, vector -> matrix, with OpenCV's 3x9 derivative dRdr[9 j + k] = dR[k] / dr_j (dRdr may be NULL)
PVB_HD void pnp_iter_rodrigues(const double *r, double *R, double *dRdr)
{
    double rx = r[0], ry = r[1], rz = r[2];
    const double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < PNP_ITER_DBL_EPS) {
        for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
        if (dRdr) {
            for (int k = 0; k < 27; ++k) dRdr[k] = 0.0;
            dRdr[5] = dRdr[15] = dRdr[19] = -1.0;
            dRdr[7] = dRdr[11] = dRdr[21] = 1.0;
        }
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1.0 - c, itheta = 1.0 / theta;
    rx *= itheta; ry *= itheta; rz *= itheta;
    const double I[9] = { 1, 0, 0, 0, 1, 0, 0, 0, 1 };
    const double rrt[9] = { rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz };
    const double rx_[9] = { 0, -rz, ry, rz, 0, -rx, -ry, rx, 0 };
    for (int k = 0; k < 9; ++k) R[k] = c * I[k] + c1 * rrt[k] + s * rx_[k];
    if (!dRdr) return;
    const double drrt[27] = { rx + rx, ry, rz, ry, 0, 0, rz, 0, 0,
                              0, rx, 0, rx, ry + ry, rz, 0, rz, 0,
                              0, 0, rx, 0, 0, ry, rx, ry, rz + rz };
    const double drx_[27] = { 0, 0, 0, 0, 0, -1, 0, 1, 0,
                              0, 0, 1, 0, 0, 0, -1, 0, 0,
                              0, -1, 0, 1, 0, 0, 0, 0, 0 };
    for (int i = 0; i < 3; ++i) {
        const double ri = i == 0 ? rx : i == 1 ? ry : rz;
        const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta, a3 = (c - s * itheta) * ri,
                     a4 = s * itheta;
        for (int k = 0; k < 9; ++k)
            dRdr[i * 9 + k] = a0 * I[k] + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * rx_[k] + a4 * drx_[i * 9 + k];
    }
}

// cv::Rodrigues, matrix -> vector: re-orthonormalised by an SVD first, then OpenCV's branches (s < 1e-5: the identity, or
// the near-pi case rebuilt from the diagonal)
PVB_HD void pnp_iter_rotation_to_vector(const double *Rin, double *r)
{
    double R[9];
    pnp_iter_orthonormal(Rin, R);
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : c < -1. ? -1. : c;
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) {
            rx = ry = rz = 0.0;
        } else {
            double t = (R[0] + 1) * 0.5;
            rx = sqrt(fmax(t, 0.));
            t = (R[4] + 1) * 0.5;
            ry = sqrt(fmax(t, 0.)) * (R[1] < 0 ? -1. : 1.);
            t = (R[8] + 1) * 0.5;
            rz = sqrt(fmax(t, 0.)) * (R[2] < 0 ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            rx *= theta; ry *= theta; rz *= theta;
        }
    } else {
        double vth = 1 / (2 * s);
        vth *= theta;
        rx *= vth; ry *= vth; rz *= vth;
    }
    r[0] = rx; r[1] = ry; r[2] = rz;
}

// One point's projection residual (pixels) and its 2x6 Jacobian as cvProjectPoints2 forms them with zero distortion,
// accumulated into n (H = J^T J upper triangle, g = J^T e, cost = 0.5 e.e).  R, dRdr: pnp_iter_rodrigues of the rvec.
PVB_HD void pnp_iter_accumulate_point(const double *R, const double *dRdr, const double *t, const double *M, const double *m,
                                      const double *cam, PnpNormal &n)
{
    const double X = M[0], Y = M[1], Z = M[2];
    double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];
    double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
    double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    z = z ? 1. / z : 1;
    x *= z; y *= z;
    const double e0 = x * cam[0] + cam[2] - m[0], e1 = y * cam[1] + cam[3] - m[1];
    double J0[6], J1[6];
    for (int j = 0; j < 3; ++j) {
        const double dx0 = X * dRdr[9 * j] + Y * dRdr[9 * j + 1] + Z * dRdr[9 * j + 2];
        const double dy0 = X * dRdr[9 * j + 3] + Y * dRdr[9 * j + 4] + Z * dRdr[9 * j + 5];
        const double dz0 = X * dRdr[9 * j + 6] + Y * dRdr[9 * j + 7] + Z * dRdr[9 * j + 8];
        J0[j] = cam[0] * (z * (dx0 - x * dz0));
        J1[j] = cam[1] * (z * (dy0 - y * dz0));
    }
    J0[3] = cam[0] * z; J0[4] = 0.0; J0[5] = cam[0] * (-x * z);
    J1[3] = 0.0; J1[4] = cam[1] * z; J1[5] = cam[1] * (-y * z);
    int q = 0;
    for (int i = 0; i < 6; ++i) {
        for (int j = i; j < 6; ++j) n.H[q++] += J0[i] * J0[j] + J1[i] * J1[j];
        n.g[i] += J0[i] * e0 + J1[i] * e1;
    }
    n.cost += 0.5 * (e0 * e0 + e1 * e1);
}

// normal equations at param = (rvec, t), summed over the group's points
template <class Red>
PVB_HD void pnp_iter_normal_at(const double *param, const double *p2, const double *p3, const double *cam, int pn, int first,
                               int stride, const Red &red, PnpNormal &n)
{
    double R[9], dRdr[27];
    pnp_iter_rodrigues(param, R, dRdr);
    pnp_normal_zero(n);
    for (int i = first; i < pn; i += stride) pnp_iter_accumulate_point(R, dRdr, param + 3, p3 + 3 * i, p2 + 2 * i, cam, n);
    red.template sum<21>(n.H);
    red.template sum<6>(n.g);
    red.template sum<1>(&n.cost);
}

// CvLevMarq::step: param = prev - solve(H with diag * (1 + lambda), g); false when the damped system is not positive definite
PVB_HD bool pnp_iter_step(const PnpNormal &n, const double *prev, int lambda_lg10, double *param)
{
    const double lambda = exp(lambda_lg10 * log(10.));
    double A[6][6], d[6];
    for (int i = 0; i < 6; ++i)
        for (int j = i; j < 6; ++j) A[i][j] = A[j][i] = n.H[pnp_tri(i, j)];
    for (int i = 0; i < 6; ++i) A[i][i] *= 1. + lambda;
    if (!pnp_chol_solve6(A, n.g, d)) return false;
    for (int i = 0; i < 6; ++i) param[i] = prev[i] - d[i];
    return true;
}

// One problem: p2 [pn][2] pixels, p3 [pn][3] model, cam = (fx, fy, cx, cy).  Writes rt = (rvec, t) (all NaN unless the
// status is PNP_ITER_OK or PNP_ITER_LIMIT) and the number of LM iterations; returns the status.
template <class Red>
PVB_HD int pnp_iter_solve(const double *p2, const double *p3, const double *cam, int pn, int first, int stride,
                          const Red &red, double *rt, int &iterations)
{
    const double nan = -(double)NAN;                   // bits 0xfff8000000000000, CUDART_NAN
    for (int i = 0; i < 6; ++i) rt[i] = nan;
    iterations = 0;
    if (pn < 4) return PNP_ITER_TOO_FEW;               // solvePnP asserts npoints >= 4
    // non-finite inputs, image points that all coincide (a skipped image), the model's centroid
    double s0[5] = { 0, 0, 0, 0, 0 };
    for (int i = first; i < pn; i += stride) {
        bool fin = true;
        for (int k = 0; k < 3; ++k) { fin = fin && fabs(p3[3 * i + k]) <= 1.79769313486231570e308; s0[2 + k] += p3[3 * i + k]; }
        fin = fin && fabs(p2[2 * i]) <= 1.79769313486231570e308 && fabs(p2[2 * i + 1]) <= 1.79769313486231570e308;
        s0[0] += fin ? 0.0 : 1.0;
        s0[1] += (p2[2 * i] != p2[0] || p2[2 * i + 1] != p2[1]) ? 1.0 : 0.0;
    }
    red.template sum<5>(s0);
    const bool cam_ok = fabs(cam[0]) <= 1.79769313486231570e308 && fabs(cam[1]) <= 1.79769313486231570e308 &&
                        fabs(cam[2]) <= 1.79769313486231570e308 && fabs(cam[3]) <= 1.79769313486231570e308 &&
                        cam[0] != 0.0 && cam[1] != 0.0;
    if (s0[0] != 0.0 || !cam_ok) return PNP_ITER_DEGENERATE;
    // planarity: singular values of sum (M - Mc)(M - Mc)^T
    const double inv = 1.0 / pn, mc[3] = { s0[2] * inv, s0[3] * inv, s0[4] * inv };
    double sc6[6] = { 0, 0, 0, 0, 0, 0 };
    for (int i = first; i < pn; i += stride) {
        const double d[3] = { p3[3 * i] - mc[0], p3[3 * i + 1] - mc[1], p3[3 * i + 2] - mc[2] };
        sc6[0] += d[0] * d[0]; sc6[1] += d[0] * d[1]; sc6[2] += d[0] * d[2];
        sc6[3] += d[1] * d[1]; sc6[4] += d[1] * d[2]; sc6[5] += d[2] * d[2];
    }
    red.template sum<6>(sc6);
    {
        double S[9] = { sc6[0], sc6[1], sc6[2], sc6[1], sc6[3], sc6[4], sc6[2], sc6[4], sc6[5] }, V[9];
        pnp_iter_jacobi<3>(S, V);
        double w0 = fabs(S[0]), w1 = fabs(S[4]), w2 = fabs(S[8]), x;
        if (w0 < w1) { x = w0; w0 = w1; w1 = x; }
        if (w1 < w2) { x = w1; w1 = w2; w2 = x; }
        if (w0 < w1) { x = w0; w0 = w1; w1 = x; }
        if (w2 / w1 < 1e-3) return PNP_ITER_PLANAR;
    }
    if (pn < 6) return PNP_ITER_TOO_FEW;               // the DLT needs six points; OpenCV raises
    if (s0[1] == 0.0) return PNP_ITER_DEGENERATE;
    // DLT: L^T L (upper triangle, 78 entries) from the normalised points
    const double ifx = 1. / cam[0], ify = 1. / cam[1];
    double LL[78];
    for (int k = 0; k < 78; ++k) LL[k] = 0.0;
    for (int i = first; i < pn; i += stride) {
        const double X = p3[3 * i], Y = p3[3 * i + 1], Z = p3[3 * i + 2];
        const double x = -((p2[2 * i] - cam[2]) * ifx), y = -((p2[2 * i + 1] - cam[3]) * ify);
        const double La[12] = { X, Y, Z, 1., 0, 0, 0, 0, x * X, x * Y, x * Z, x };
        const double Lb[12] = { 0, 0, 0, 0, X, Y, Z, 1., y * X, y * Y, y * Z, y };
        int q = 0;
        for (int a = 0; a < 12; ++a)
            for (int b = a; b < 12; ++b) LL[q++] += La[a] * La[b] + Lb[a] * Lb[b];
    }
    red.template sum<78>(LL);
    double A[144], V[144];
    {
        int q = 0;
        for (int a = 0; a < 12; ++a)
            for (int b = a; b < 12; ++b) { A[a * 12 + b] = A[b * 12 + a] = LL[q]; ++q; }
    }
    pnp_iter_jacobi<12>(A, V);
    int lo = 0;
    for (int k = 1; k < 12; ++k) if (A[k * 13] < A[lo * 13]) lo = k;
    double RRt[12];                                    // [RR | tt], 3 x 4 row-major
    for (int k = 0; k < 12; ++k) RRt[k] = V[k * 12 + lo];
    const double RR[9] = { RRt[0], RRt[1], RRt[2], RRt[4], RRt[5], RRt[6], RRt[8], RRt[9], RRt[10] };
    const double det = RR[0] * (RR[4] * RR[8] - RR[5] * RR[7]) - RR[1] * (RR[3] * RR[8] - RR[5] * RR[6]) +
                       RR[2] * (RR[3] * RR[7] - RR[4] * RR[6]);
    const double sgn = det < 0 ? -1.0 : 1.0;
    double sc = 0.0;
    for (int k = 0; k < 9; ++k) sc += RR[k] * RR[k];
    sc = sqrt(sc);
    if (!(fabs(sc) > PNP_ITER_DBL_EPS)) return PNP_ITER_DEGENERATE;   // OpenCV's CV_Assert
    double RRs[9], R[9];
    for (int k = 0; k < 9; ++k) RRs[k] = sgn * RR[k];
    pnp_iter_orthonormal(RRs, R);
    double nr = 0.0;
    for (int k = 0; k < 9; ++k) nr += R[k] * R[k];
    const double tscale = sqrt(nr) / sc;
    double param[6], prev[6];
    pnp_iter_rotation_to_vector(R, param);
    param[3] = sgn * RRt[3] * tscale; param[4] = sgn * RRt[7] * tscale; param[5] = sgn * RRt[11] * tscale;
    // Levenberg-Marquardt (CvLevMarq's state machine)
    PnpNormal n, nc;
    pnp_iter_normal_at(param, p2, p3, cam, pn, first, stride, red, n);
    double prev_err = sqrt(2.0 * n.cost);
    int lambda_lg10 = -3, status = PNP_ITER_LIMIT;
    for (;;) {
        for (int i = 0; i < 6; ++i) prev[i] = param[i];
        if (!pnp_iter_step(n, prev, lambda_lg10, param)) return PNP_ITER_DEGENERATE;
        pnp_iter_normal_at(param, p2, p3, cam, pn, first, stride, red, nc);
        double err = sqrt(2.0 * nc.cost);
        while (err > prev_err && ++lambda_lg10 <= 16) {
            if (!pnp_iter_step(n, prev, lambda_lg10, param)) return PNP_ITER_DEGENERATE;
            pnp_iter_normal_at(param, p2, p3, cam, pn, first, stride, red, nc);
            err = sqrt(2.0 * nc.cost);
        }
        lambda_lg10 = lambda_lg10 - 1 > -16 ? lambda_lg10 - 1 : -16;
        ++iterations;
        double dp = 0.0, np = 0.0;
        for (int i = 0; i < 6; ++i) { dp += (param[i] - prev[i]) * (param[i] - prev[i]); np += prev[i] * prev[i]; }
        if (sqrt(dp) / (sqrt(np) + PNP_ITER_DBL_EPS) < PNP_ITER_FLT_EPS) { status = PNP_ITER_OK; break; }
        if (iterations >= PNP_ITER_MAX_ITER) break;
        prev_err = err;
        n = nc;
    }
    bool fin = true;
    for (int i = 0; i < 6; ++i) fin = fin && fabs(param[i]) <= 1.79769313486231570e308;
    if (!fin) return PNP_ITER_DEGENERATE;
    for (int i = 0; i < 6; ++i) rt[i] = param[i];
    return status;
}

// [Rodrigues(rvec) | t] as a row-major 3x4 (what pvnet_pose_utils.pnp returns); NaN rt gives a NaN pose
PVB_HD void pnp_iter_pose(const double *rt, double *pose)
{
    double R[9];
    pnp_iter_rodrigues(rt, R, nullptr);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) pose[i * 4 + j] = R[i * 3 + j];
        pose[i * 4 + 3] = rt[3 + i];
    }
}

} // namespace pvb
