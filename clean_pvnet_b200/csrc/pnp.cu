// pnp.cu -- the uncertainty-PnP tail on the device (SURVEY.md 8f rows 2+3): per-keypoint weights, P3P initial pose and the
// batched Levenberg-Marquardt refinement.
//
// Replaces the per-image CPU call lib/csrc/uncertainty_pnp/src/uncertainty_pnp.cpp:61-92 (ceres::Solve on 6 parameters and
// 2*pn residuals, pn = 9..17 keypoints).  A problem is far too small for more than a warp: lane i owns points i, i+32, ...,
// evaluates their residuals and 2x6 Jacobians (pnp_core.cuh) and the warp adds the 28 numbers of the normal equations with
// an XOR butterfly (every lane ends with the same bits, so all lanes run the identical trust-region state machine without
// divergence or broadcasts).  Everything is fp64 like the reference.  Latency-bound by design: ~10 evaluations per problem.
#include <math_constants.h>
#include "api.h"
#include "common.cuh"
#include "pnp_core.cuh"
#include "p3p_core.cuh"
#include "pnp_iter_core.cuh"

namespace pvb {

// Batched uncertainty PnP: n problems of pn points, one warp per problem, fp64 like the reference.  The 2D inputs are either
// fp64 pts2d + wgt2d, read in place, or (kpt2d != NULL) the voting layer's fp32 keypoints with their covariances or
// weights, converted into shared memory (pn <= PNP_FUSED_MAX_PN).
constexpr int PNP_FUSED_MAX_PN = 64;
struct PnpArgs {
    const double *pts2d;      // [n][pn][2]
    const double *wgt2d;      // [n][pn][3]  (wxx, wxy, wyy)
    const float *kpt2d;       // [n][pn][2]  (the voting layer's kpt_2d)
    const float *cov;         // [n][pn][2][2] (the voting layer's var), or NULL ...
    const float *weights;     // ... then [n][pn][3] precomputed (wxx, wxy, wyy)
    float *weights_out;       // optional [n][pn][3]: the fp32 weights used (kpt2d only)
    const double *pts3d;      // [pn][3], problem p at pts3d + p*pts3d_stride (0: shared)
    const double *K;          // [3][3] row-major, problem p at K + p*k_stride (0: shared)
    const double *init_rt;    // optional [n][6]; NULL: P3P on the four best-weighted points
    double *init_out;         // optional [n][6]: the initial pose that was used
    double *result_rt;        // [n][6]: the refined pose; NULL: the P3P start alone (fp64 inputs, into init_out)
    int *info;                // optional [n][2]: iterations, termination code
    double *pose;             // [n][3][4]: the pose of pvb_pnp_iterative (pnp_iter_kernel only)
    int n, pn;
    long long pts3d_stride, k_stride;
    PnpOptions opt;
};

// ---------------------------------------------------------------------------------
// SURVEY 8f row 2: weights of the uncertainty PnP, inv(sqrtm(cov)) per keypoint packed as (wxx, wxy, wyy)
// (cov_to_weights in common.cuh; pnp_batch_kernel's fp32 inputs use the same function).
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
pnp_weights_kernel(const float *__restrict__ cov, float *__restrict__ w, int n)
{
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= n) return;
    float o0, o1, o2;
    cov_to_weights(__ldg(reinterpret_cast<const float4 *>(cov) + i), o0, o1, o2);
    w[(size_t)i * 3] = o0; w[(size_t)i * 3 + 1] = o1; w[(size_t)i * 3 + 2] = o2;
}

// sum of C numbers over the warp by an XOR butterfly, in place: every lane ends with the same bits
struct PnpWarpSum {
    template <int C> __device__ __forceinline__ void sum(double *v) const
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
            for (int q = 0; q < C; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
        }
    }
};

// normal equations of one problem at `pose`: lane i owns points i, i+32, ...; butterfly sum -> every lane holds the same bits
__device__ __forceinline__ void pnp_warp_normal_at(const double *pose, const double *p2, const double *p3, const double *w,
                                                   const double *cam, int pn, int lane, PnpNormal &n)
{
    pnp_normal_zero(n);
    for (int i = lane; i < pn; i += 32) pnp_accumulate_point(pose, p3 + 3 * i, p2 + 2 * i, w + 3 * i, cam, n);
    const PnpWarpSum red;
    red.sum<21>(n.H);
    red.sum<6>(n.g);
    red.sum<1>(&n.cost);
}

// Problem `prob`'s camera (fx, fy, px, py) and model points: one for the batch (stride 0) or one per problem
__device__ __forceinline__ const double *pnp_model_camera(const PnpArgs &a, int prob, double *cam)
{
    pnp_camera(a.K + (size_t)prob * a.k_stride, cam);
    return a.pts3d + (size_t)prob * a.pts3d_stride;
}

// ---------------------------------------------------------------------------------------------------------------------
// Refinement: one warp per problem, PNP_WARPS problems per CTA.  What lib/evaluators/linemod/pvnet.py:118-130 + un_pnp_utils.
// uncertainty_pnp (:6-57) do per image on the CPU, in the order they do it:
//   - the 2D inputs: fp64 points and weights read in place (Fp64), or the voting layer's fp32 kpt_2d with var (or
//     precomputed weights) converted once into shared memory (Fp32Staged; the weights are rounded to fp32 first, so the
//     result is bit-identical to pvb_uncertainty_weights followed by the Fp64 path);
//   - the start: init_rt, or P3P on the four best-weighted points (un_pnp_utils.py:25-31), a short scalar chain run by
//     lane 0 (p3p_core.cuh); no admissible pose -> NaN, on which the refinement stops at once;
//   - the refinement.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int PNP_WARPS = 4;
enum class PnpInput { Fp64, Fp32Staged };

template <PnpInput IN>
__global__ void __launch_bounds__(PNP_WARPS * 32)
pnp_batch_kernel(PnpArgs a)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int prob = blockIdx.x * PNP_WARPS + wid;
    if (prob >= a.n) return;
    double cam[4];
    const double *p3 = pnp_model_camera(a, prob, cam), *p2, *w;
    if constexpr (IN == PnpInput::Fp32Staged) {
        __shared__ double s_p2[PNP_WARPS][PNP_FUSED_MAX_PN * 2], s_p3[PNP_WARPS][PNP_FUSED_MAX_PN * 3],
            s_w[PNP_WARPS][PNP_FUSED_MAX_PN * 3];
        double *d2 = s_p2[wid], *d3 = s_p3[wid], *dw = s_w[wid];
        for (int i = lane; i < a.pn; i += 32) {
            const float2 q = __ldg(reinterpret_cast<const float2 *>(a.kpt2d) + (size_t)prob * a.pn + i);
            d2[2 * i] = (double)q.x; d2[2 * i + 1] = (double)q.y;
            float w0, w1, w2;
            if (a.cov) cov_to_weights(__ldg(reinterpret_cast<const float4 *>(a.cov) + (size_t)prob * a.pn + i), w0, w1, w2);
            else { const float *ww = a.weights + ((size_t)prob * a.pn + i) * 3; w0 = ww[0]; w1 = ww[1]; w2 = ww[2]; }
            dw[3 * i] = (double)w0; dw[3 * i + 1] = (double)w1; dw[3 * i + 2] = (double)w2;
            if (a.weights_out) { float *wo = a.weights_out + ((size_t)prob * a.pn + i) * 3; wo[0] = w0; wo[1] = w1; wo[2] = w2; }
            d3[3 * i] = p3[3 * i]; d3[3 * i + 1] = p3[3 * i + 1]; d3[3 * i + 2] = p3[3 * i + 2];
        }
        __syncwarp();
        p2 = d2; p3 = d3; w = dw;
    } else {
        p2 = a.pts2d + (size_t)prob * a.pn * 2;
        w = a.wgt2d + (size_t)prob * a.pn * 3;
    }
    double init[6];
    if (a.init_rt) {
#pragma unroll
        for (int i = 0; i < 6; ++i) init[i] = a.init_rt[(size_t)prob * 6 + i];
    } else {
#pragma unroll
        for (int i = 0; i < 6; ++i) init[i] = CUDART_NAN;
        if (lane == 0) p3p_start(p2, p3, w, a.pn, cam, init);
#pragma unroll
        for (int i = 0; i < 6; ++i) init[i] = __shfl_sync(0xffffffffu, init[i], 0);
    }
    if (a.init_out && lane < 6) a.init_out[(size_t)prob * 6 + lane] = init[lane];
    PnpState st;
    pnp_solve(a.opt, init, [&](const double *pose, PnpNormal &n) { pnp_warp_normal_at(pose, p2, p3, w, cam, a.pn, lane, n); },
              st);
    if (lane < 6) a.result_rt[(size_t)prob * 6 + lane] = st.x[lane];
    if (a.info && lane == 0) { a.info[2 * prob] = st.iterations; a.info[2 * prob + 1] = st.code; }
}

// The P3P start alone (pvb_uncertainty_pnp_init), one thread per problem.  The chain is scalar, so a warp per problem would
// leave 31 lanes idle, and without the LM code the kernel needs about 156 registers instead of 254: a batch of 4096
// problems runs in one wave here, in about four as the start of pnp_batch_kernel<Fp64>.
__global__ void __launch_bounds__(64)
p3p_start_kernel(PnpArgs a)
{
    const int prob = blockIdx.x * 64 + threadIdx.x;
    if (prob >= a.n) return;
    double cam[4], rt[6];
    const double *p3 = pnp_model_camera(a, prob, cam);
    p3p_start(a.pts2d + (size_t)prob * a.pn * 2, p3, a.wgt2d + (size_t)prob * a.pn * 3, a.pn, cam, rt);
#pragma unroll
    for (int i = 0; i < 6; ++i) a.init_out[(size_t)prob * 6 + i] = rt[i];
}

// ---------------------------------------------------------------------------------------------------------------------
// PVNet's default pose step, cv2.solvePnP(..., SOLVEPNP_ITERATIVE) (pnp_iter_core.cuh): one warp per problem like
// pnp_batch_kernel.  Lane i owns points i, i+32, ...; every sum over points (the centroid and scatter of the model, the 78
// entries of L^T L, the 28 numbers of J^T J / J^T e / |e|^2) is an XOR butterfly, so every lane holds the same bits and runs
// the identical DLT and Levenberg-Marquardt code without divergence.  No shared memory, no workspace; a problem's result
// depends on nothing but its own inputs.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PNP_WARPS * 32)
pnp_iter_kernel(PnpArgs a)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int prob = blockIdx.x * PNP_WARPS + wid;
    if (prob >= a.n) return;
    double cam[4], rt[6], pose[12];
    const double *p3 = pnp_model_camera(a, prob, cam);
    int iterations;
    const int status = pnp_iter_solve(a.pts2d + (size_t)prob * a.pn * 2, p3, cam, a.pn, lane, 32, PnpWarpSum(), rt, iterations);
    pnp_iter_pose(rt, pose);
#pragma unroll
    for (int i = 0; i < 12; ++i) if (lane == i) a.pose[(size_t)prob * 12 + i] = pose[i];
    if (a.result_rt) {
#pragma unroll
        for (int i = 0; i < 6; ++i) if (lane == 12 + i) a.result_rt[(size_t)prob * 6 + i] = rt[i];
    }
    if (a.info && lane == 31) { a.info[2 * prob] = iterations; a.info[2 * prob + 1] = status; }
}

namespace {

// The checks every PnP entry point makes after its own ones on n and pn: NULL tensors (`given`: every required pointer is
// set), then the strides.
int pnp_check_inputs(int32_t n, bool given, int64_t pts3d_stride, int64_t k_stride)
{
    if (n && !given) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (pts3d_stride < 0 || k_stride < 0) return fail(PVB_ERR_INVALID, "negative stride");
    return PVB_OK;
}

// options == NULL: Ceres' defaults
int pnp_read_options(const pvb_pnp_options *options, PnpOptions &opt)
{
    opt = pnp_default_options();
    if (!options) return PVB_OK;
    if (options->max_num_iterations < 0 || !(options->function_tolerance >= 0.0) || !(options->gradient_tolerance >= 0.0) ||
        !(options->parameter_tolerance >= 0.0))
        return fail(PVB_ERR_INVALID, "pvb_pnp_options: negative or NaN entry");
    opt.max_num_iterations = options->max_num_iterations; opt.function_tolerance = options->function_tolerance;
    opt.gradient_tolerance = options->gradient_tolerance; opt.parameter_tolerance = options->parameter_tolerance;
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_uncertainty_weights(const float *cov, float *weights, int32_t n, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (n && (!cov || !weights)) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (reinterpret_cast<uintptr_t>(cov) & 15u) return fail(PVB_ERR_INVALID, "cov must be 16-byte aligned");
    if (n == 0) return PVB_OK;
    pnp_weights_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(cov, weights, n);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "pnp weights kernel");
}

PVB_API int pvb_uncertainty_pnp(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                const double *init_rt, double *result_rt, int32_t *info, int32_t n, int32_t pn,
                                int64_t pts3d_stride, int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1) return fail(PVB_ERR_INVALID, "pn must be >= 1 (got %d)", pn);
    PnpArgs a = {};
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && wgt2d && K && init_rt && result_rt, pts3d_stride, k_stride)) return rc;
    if (int rc = pnp_read_options(options, a.opt)) return rc;
    if (n == 0) return PVB_OK;
    a.pts2d = pts2d; a.wgt2d = wgt2d; a.pts3d = pts3d; a.K = K; a.init_rt = init_rt; a.result_rt = result_rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    pnp_batch_kernel<PnpInput::Fp64>
        <<<(n + PNP_WARPS - 1) / PNP_WARPS, PNP_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "uncertainty pnp kernel");
}

PVB_API int pvb_uncertainty_pnp_from_votes(const float *kpt_2d, const float *cov, const float *weights, const double *pts3d,
                                           const double *K, const double *init_rt, double *result_rt, double *init_out,
                                           float *weights_out, int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride,
                                           int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1 || pn > PNP_FUSED_MAX_PN) return fail(PVB_ERR_INVALID, "pn must be in [1,%d] (got %d)", PNP_FUSED_MAX_PN, pn);
    if (!init_rt && pn < 4) return fail(PVB_ERR_INVALID, "the P3P initialisation needs pn >= 4 (got %d)", pn);
    const bool given = kpt_2d && pts3d && K && result_rt;
    // before pnp_check_inputs, but only once every required tensor is set: a caller keeps getting "NULL tensor" first,
    // then this, then "negative stride"
    if (n && given && ((cov == nullptr) == (weights == nullptr)))
        return fail(PVB_ERR_INVALID, "pass exactly one of cov / weights");
    PnpArgs a = {};
    if (int rc = pnp_check_inputs(n, given, pts3d_stride, k_stride)) return rc;
    if ((reinterpret_cast<uintptr_t>(kpt_2d) & 7u) || (reinterpret_cast<uintptr_t>(cov) & 15u))
        return fail(PVB_ERR_INVALID, "kpt_2d must be 8-byte and cov 16-byte aligned");
    if (int rc = pnp_read_options(options, a.opt)) return rc;
    if (n == 0) return PVB_OK;
    a.kpt2d = kpt_2d; a.cov = cov; a.weights = weights; a.weights_out = weights_out; a.pts3d = pts3d; a.K = K;
    a.init_rt = init_rt; a.init_out = init_out; a.result_rt = result_rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    pnp_batch_kernel<PnpInput::Fp32Staged>
        <<<(n + PNP_WARPS - 1) / PNP_WARPS, PNP_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "fused uncertainty pnp kernel");
}

PVB_API int pvb_uncertainty_pnp_init(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                     double *init_rt, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                                     pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 4) return fail(PVB_ERR_INVALID, "P3P needs pn >= 4 (got %d)", pn);
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && wgt2d && K && init_rt, pts3d_stride, k_stride)) return rc;
    if (n == 0) return PVB_OK;
    PnpArgs a = {};                    // no result_rt: the P3P start alone, written to init_out
    a.pts2d = pts2d; a.wgt2d = wgt2d; a.pts3d = pts3d; a.K = K; a.init_out = init_rt;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    p3p_start_kernel<<<(n + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "p3p init kernel");
}

PVB_API int pvb_pnp_iterative(const double *pts2d, const double *pts3d, const double *K, double *pose, double *rt,
                              int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                              pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1) return fail(PVB_ERR_INVALID, "pn must be >= 1 (got %d)", pn);
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && K && pose, pts3d_stride, k_stride)) return rc;
    if (n == 0) return PVB_OK;
    PnpArgs a = {};
    a.pts2d = pts2d; a.pts3d = pts3d; a.K = K; a.pose = pose; a.result_rt = rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    pnp_iter_kernel<<<(n + PNP_WARPS - 1) / PNP_WARPS, PNP_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "iterative pnp kernel");
}

} // extern "C"
