// pnp_core.cuh -- arithmetic core of the batched uncertainty-PnP refinement (SURVEY.md 8f row 3).
//
// Replaces, per problem, what lib/csrc/uncertainty_pnp/src/uncertainty_pnp.cpp:61-92 asks Ceres 2.0 to do: minimise
// 0.5 * sum_i |W_i (proj(R(aa) X_i + t) - x_i)|^2 over the 6 pose parameters (angle-axis, translation) with the default
// Levenberg-Marquardt trust-region loop (option defaults: include/ceres/solver.h of the vendored headers).  The residual
// and its forward-mode derivative follow the functor at uncertainty_pnp.cpp:19-37 and ceres/rotation.h:563-607 (same
// small-angle branch, so the derivative there is the one Ceres' jets produce).
//
// Everything here is plain double arithmetic on small fixed-size arrays and compiles both as device code (pnp.cu) and as
// host code (tests/pnp_host_harness.cpp builds it with g++ to check the logic on the CPU box; no product path uses that).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define PVB_HD __host__ __device__ __forceinline__
#else
#define PVB_HD inline
#endif

namespace pvb {

// Ceres 2.0 defaults (include/ceres/solver.h:257-316, :621)
struct PnpOptions {
    int max_num_iterations;          // 50
    double function_tolerance;       // 1e-6
    double gradient_tolerance;       // 1e-10
    double parameter_tolerance;      // 1e-8
};
PVB_HD PnpOptions pnp_default_options()
{
    PnpOptions o;
    o.max_num_iterations = 50; o.function_tolerance = 1e-6; o.gradient_tolerance = 1e-10; o.parameter_tolerance = 1e-8;
    return o;
}

// cam = (fx, fy, px, py) of a row-major 3x3 intrinsic matrix (uncertainty_pnp.cpp:77)
PVB_HD void pnp_camera(const double *K, double *cam)
{
    cam[0] = K[0]; cam[1] = K[4]; cam[2] = K[2]; cam[3] = K[5];
}

// termination codes written to `info` (documented in include/pvnet_vote_b200.h)
enum { PNP_CONV_GRADIENT = 1, PNP_CONV_PARAMETER = 2, PNP_CONV_FUNCTION = 3, PNP_CONV_RADIUS = 4, PNP_NO_CONVERGENCE = 5,
       PNP_FAILURE = 6 };

// Normal equations of one evaluation point: H = J^T J (upper triangle, row-major 21 entries), g = J^T r, cost = 0.5 r.r
struct PnpNormal {
    double H[21], g[6], cost;
};
PVB_HD int pnp_tri(int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); }   // i <= j

PVB_HD void pnp_normal_zero(PnpNormal &n)
{
    for (int i = 0; i < 21; ++i) n.H[i] = 0.0;
    for (int i = 0; i < 6; ++i) n.g[i] = 0.0;
    n.cost = 0.0;
}

// One point's two residuals and their 2x6 Jacobian, accumulated into n.
// pose = (aa[3], t[3]); X = model point; x2 = image point; w = (wxx, wxy, wyy); cam = (fx, fy, px, py)
PVB_HD void pnp_accumulate_point(const double *pose, const double *X, const double *x2, const double *w, const double *cam,
                                 PnpNormal &n)
{
    const double a0 = pose[0], a1 = pose[1], a2 = pose[2];
    double T[3], dT[3][6];        // transformed point and d/d(pose)
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 6; ++c) dT[r][c] = 0.0;
    const double theta2 = a0 * a0 + a1 * a1 + a2 * a2;
    if (theta2 > 2.220446049250313e-16) {        // std::numeric_limits<double>::epsilon(), rotation.h:565
        const double theta = sqrt(theta2), c = cos(theta), s = sin(theta), ti = 1.0 / theta;
        const double aa[3] = { a0, a1, a2 };
        double dtheta[3], dc[3], ds[3], dti[3], wv[3], dw[3][3];
        for (int k = 0; k < 3; ++k) {
            dtheta[k] = aa[k] * ti;               // d theta / d a_k
            dc[k] = -s * dtheta[k]; ds[k] = c * dtheta[k];
            dti[k] = -dtheta[k] / theta2;
            wv[k] = aa[k] * ti;
        }
        for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) dw[r][k] = (r == k ? ti : 0.0) + aa[r] * dti[k];
        const double wxp[3] = { wv[1] * X[2] - wv[2] * X[1], wv[2] * X[0] - wv[0] * X[2], wv[0] * X[1] - wv[1] * X[0] };
        const double wp = wv[0] * X[0] + wv[1] * X[1] + wv[2] * X[2];
        const double tmp = wp * (1.0 - c);
        for (int r = 0; r < 3; ++r) T[r] = X[r] * c + wxp[r] * s + wv[r] * tmp;
        for (int k = 0; k < 3; ++k) {
            const double dwxp[3] = { dw[1][k] * X[2] - dw[2][k] * X[1], dw[2][k] * X[0] - dw[0][k] * X[2],
                                     dw[0][k] * X[1] - dw[1][k] * X[0] };
            const double dwp = dw[0][k] * X[0] + dw[1][k] * X[1] + dw[2][k] * X[2];
            const double dtmp = dwp * (1.0 - c) - wp * dc[k];
            for (int r = 0; r < 3; ++r)
                dT[r][k] = X[r] * dc[k] + dwxp[r] * s + wxp[r] * ds[k] + dw[r][k] * tmp + wv[r] * dtmp;
        }
    } else {                                      // rotation.h:596-607: R ~ I + [aa]x
        T[0] = X[0] + (a1 * X[2] - a2 * X[1]);
        T[1] = X[1] + (a2 * X[0] - a0 * X[2]);
        T[2] = X[2] + (a0 * X[1] - a1 * X[0]);
        dT[0][1] = X[2];  dT[0][2] = -X[1];
        dT[1][0] = -X[2]; dT[1][2] = X[0];
        dT[2][0] = X[1];  dT[2][1] = -X[0];
    }
    T[0] += pose[3]; T[1] += pose[4]; T[2] += pose[5];
    dT[0][3] += 1.0; dT[1][4] += 1.0; dT[2][5] += 1.0;
    const double iz = 1.0 / T[2];
    const double u = cam[0] * T[0] * iz, v = cam[1] * T[1] * iz;
    const double dx = u + cam[2] - x2[0], dy = v + cam[3] - x2[1];
    const double r0 = w[0] * dx + w[1] * dy, r1 = w[1] * dx + w[2] * dy;
    double J0[6], J1[6];
    for (int k = 0; k < 6; ++k) {
        const double du = cam[0] * (dT[0][k] * iz - T[0] * iz * iz * dT[2][k]);
        const double dv = cam[1] * (dT[1][k] * iz - T[1] * iz * iz * dT[2][k]);
        J0[k] = w[0] * du + w[1] * dv;
        J1[k] = w[1] * du + w[2] * dv;
    }
    int q = 0;
    for (int i = 0; i < 6; ++i) {
        for (int j = i; j < 6; ++j) n.H[q++] += J0[i] * J0[j] + J1[i] * J1[j];
        n.g[i] += J0[i] * r0 + J1[i] * r1;
    }
    n.cost += 0.5 * (r0 * r0 + r1 * r1);
}

// Trust-region state of one problem, driven by pnp_solve; result = st.x, st.code, st.iterations
struct PnpState {
    double x[6], x_norm, grad_max;
    PnpNormal n;                 // normal equations at x
    double scale[6];             // jacobi scaling, fixed at iteration 0
    double diag[6];              // clamped squared column norms of the scaled Jacobian (kept while steps are rejected)
    double radius, decrease_factor;
    double step_s[6];            // proposed step in scaled coordinates
    double model_cost_change;
    int reuse_diagonal, iterations, invalid, code;
};

PVB_HD double pnp_max_abs6(const double *g)
{
    double m = 0.0;
    for (int i = 0; i < 6; ++i) { const double a = fabs(g[i]); if (a > m || a != a) m = a; }
    return m;
}
PVB_HD double pnp_norm6(const double *x)
{
    double s = 0.0;
    for (int i = 0; i < 6; ++i) s += x[i] * x[i];
    return sqrt(s);
}

PVB_HD void pnp_init(PnpState &st, const double *init_rt, const PnpNormal &n0)
{
    for (int i = 0; i < 6; ++i) st.x[i] = init_rt[i];
    st.n = n0;
    st.x_norm = pnp_norm6(st.x);
    for (int i = 0; i < 6; ++i) st.scale[i] = 1.0 / (1.0 + sqrt(n0.H[pnp_tri(i, i)]));
    st.grad_max = pnp_max_abs6(n0.g);
    st.radius = 1e4; st.decrease_factor = 2.0;
    st.reuse_diagonal = 0; st.iterations = 0; st.invalid = 0; st.code = 0;
    for (int i = 0; i < 6; ++i) { st.diag[i] = 0.0; st.step_s[i] = 0.0; }
    st.model_cost_change = 0.0;
}

// Cholesky solve of the 6x6 system A y = b (A symmetric, full storage); returns false when A is not positive definite
// or the solution is not finite.
PVB_HD bool pnp_chol_solve6(double A[6][6], const double *b, double *y)
{
    for (int j = 0; j < 6; ++j) {
        double d = A[j][j];
        for (int k = 0; k < j; ++k) d -= A[j][k] * A[j][k];
        if (!(d > 0.0)) return false;
        d = sqrt(d);
        A[j][j] = d;
        for (int i = j + 1; i < 6; ++i) {
            double v = A[i][j];
            for (int k = 0; k < j; ++k) v -= A[i][k] * A[j][k];
            A[i][j] = v / d;
        }
    }
    double z[6];
    for (int i = 0; i < 6; ++i) {
        double v = b[i];
        for (int k = 0; k < i; ++k) v -= A[i][k] * z[k];
        z[i] = v / A[i][i];
    }
    for (int i = 5; i >= 0; --i) {
        double v = z[i];
        for (int k = i + 1; k < 6; ++k) v -= A[k][i] * y[k];
        y[i] = v / A[i][i];
    }
    for (int i = 0; i < 6; ++i) if (!(fabs(y[i]) <= 1.79769313486231570e308)) return false;
    return true;
}

// Termination checks of the previous iteration, then the next Levenberg-Marquardt step.  Returns true with the candidate
// point in cand[6] when one has to be evaluated; false when the solve is over (st.code set).
PVB_HD bool pnp_propose(PnpState &st, const PnpOptions &opt, double *cand)
{
    for (;;) {
        if (st.iterations >= opt.max_num_iterations) { st.code = PNP_NO_CONVERGENCE; return false; }
        if (!(st.grad_max > opt.gradient_tolerance)) { st.code = PNP_CONV_GRADIENT; return false; }
        if (st.radius < 1e-32) { st.code = PNP_CONV_RADIUS; return false; }
        st.iterations++;
        double Hs[6][6], bs[6], A[6][6], y[6];
        for (int i = 0; i < 6; ++i) {
            for (int j = i; j < 6; ++j) Hs[i][j] = Hs[j][i] = st.n.H[pnp_tri(i, j)] * st.scale[i] * st.scale[j];
            bs[i] = st.n.g[i] * st.scale[i];
        }
        if (!st.reuse_diagonal)
            for (int i = 0; i < 6; ++i) st.diag[i] = fmin(fmax(Hs[i][i], 1e-6), 1e32);
        for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) A[i][j] = Hs[i][j] + (i == j ? st.diag[i] / st.radius : 0.0);
        bool ok = pnp_chol_solve6(A, bs, y);
        double mcc = -1.0;
        if (ok) {
            double sb = 0.0, shs = 0.0;
            for (int i = 0; i < 6; ++i) {
                st.step_s[i] = -y[i];
                sb += st.step_s[i] * bs[i];
            }
            for (int i = 0; i < 6; ++i) {
                double v = 0.0;
                for (int j = 0; j < 6; ++j) v += Hs[i][j] * st.step_s[j];
                shs += st.step_s[i] * v;
            }
            mcc = -sb - 0.5 * shs;
        }
        if (!(mcc > 0.0)) {                           // invalid step: shrink and retry (StepIsInvalid)
            if (++st.invalid >= 5) { st.code = PNP_FAILURE; return false; }
            st.radius *= 0.5; st.reuse_diagonal = 1;
            continue;
        }
        st.invalid = 0;
        st.model_cost_change = mcc;
        for (int i = 0; i < 6; ++i) cand[i] = st.x[i] + st.step_s[i] * st.scale[i];
        return true;
    }
}

// The candidate's normal equations are in: convergence tests, then accept or reject.  Returns false when the solve is over.
PVB_HD bool pnp_update(PnpState &st, const PnpOptions &opt, const double *cand, const PnpNormal &nc)
{
    double delta[6];
    for (int i = 0; i < 6; ++i) delta[i] = st.step_s[i] * st.scale[i];
    if (pnp_norm6(delta) <= opt.parameter_tolerance * (st.x_norm + opt.parameter_tolerance)) {
        st.code = PNP_CONV_PARAMETER; return false;                  // the candidate is not adopted
    }
    const double cost_change = st.n.cost - nc.cost;
    if (fabs(cost_change) <= opt.function_tolerance * st.n.cost) {
        st.code = PNP_CONV_FUNCTION; return false;                   // the candidate is not adopted
    }
    const double rho = cost_change / st.model_cost_change;
    if (rho > 1e-3) {                                                // StepAccepted
        for (int i = 0; i < 6; ++i) st.x[i] = cand[i];
        st.n = nc;
        st.x_norm = pnp_norm6(st.x);
        st.grad_max = pnp_max_abs6(nc.g);
        const double q = 2.0 * rho - 1.0;
        st.radius = fmin(1e16, st.radius / fmax(1.0 / 3.0, 1.0 - q * q * q));
        st.decrease_factor = 2.0; st.reuse_diagonal = 0;
    } else {                                                         // StepRejected (also a non-finite candidate cost)
        st.radius /= st.decrease_factor;
        st.decrease_factor *= 2.0;
        st.reuse_diagonal = 1;
    }
    return true;
}

// The whole solve from init_rt.  eval(pose, n) fills n with the normal equations at pose: a warp reduction in the kernel
// (pnp.cu), a serial sum in the host build (tests/pnp_host_harness.cpp).
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <class Eval>
PVB_HD void pnp_solve(const PnpOptions &opt, const double *init_rt, Eval &&eval, PnpState &st)
{
    PnpNormal n;
    eval(init_rt, n);
    pnp_init(st, init_rt, n);
    double cand[6];
    while (pnp_propose(st, opt, cand)) {
        eval(cand, n);
        if (!pnp_update(st, opt, cand, n)) break;
    }
}

} // namespace pvb
