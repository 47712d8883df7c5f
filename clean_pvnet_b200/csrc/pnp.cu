// pnp.cu -- the uncertainty-PnP tail on the device (SURVEY.md 8f rows 2+3): per-keypoint weights, P3P initial pose and the
// batched Levenberg-Marquardt refinement.
//
// Replaces the per-image CPU call lib/csrc/uncertainty_pnp/src/uncertainty_pnp.cpp:61-92 (ceres::Solve on 6 parameters and
// 2*pn residuals, pn = 9..17 keypoints).  A problem is far too small for more than a warp: lane i owns points i, i+32, ...,
// evaluates their residuals and 2x6 Jacobians (pnp_core.cuh) and the warp adds the 28 numbers of the normal equations with
// an XOR butterfly (every lane ends with the same bits, so all lanes run the identical trust-region state machine without
// divergence or broadcasts).  Everything is fp64 like the reference.  Latency-bound by design: ~10 evaluations per problem.
#include <math_constants.h>
#include "common.cuh"
#include "kernels.h"
#include "pnp_core.cuh"
#include "p3p_core.cuh"

namespace pvb {

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

cudaError_t launch_pnp_weights(const float *cov, float *w, int n, cudaStream_t st)
{
    if (n <= 0) return cudaSuccess;
    pnp_weights_kernel<<<(n + 127) / 128, 128, 0, st>>>(cov, w, n);
    return cudaGetLastError();
}

// normal equations of one problem at `pose`: lane i owns points i, i+32, ...; butterfly sum -> every lane holds the same bits
__device__ __forceinline__ void pnp_warp_normal_at(const double *pose, const double *p2, const double *p3, const double *w,
                                                   const double *cam, int pn, int lane, PnpNormal &n)
{
    pnp_normal_zero(n);
    for (int i = lane; i < pn; i += 32) pnp_accumulate_point(pose, p3 + 3 * i, p2 + 2 * i, w + 3 * i, cam, n);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int q = 0; q < 21; ++q) n.H[q] += __shfl_xor_sync(0xffffffffu, n.H[q], o);
#pragma unroll
        for (int q = 0; q < 6; ++q) n.g[q] += __shfl_xor_sync(0xffffffffu, n.g[q], o);
        n.cost += __shfl_xor_sync(0xffffffffu, n.cost, o);
    }
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

cudaError_t launch_pnp_batch(const PnpArgs &a, cudaStream_t st)
{
    if (a.n <= 0) return cudaSuccess;
    if (!a.result_rt) {
        p3p_start_kernel<<<(a.n + 63) / 64, 64, 0, st>>>(a);
        return cudaGetLastError();
    }
    const int blocks = (a.n + PNP_WARPS - 1) / PNP_WARPS;
    if (a.kpt2d) pnp_batch_kernel<PnpInput::Fp32Staged><<<blocks, PNP_WARPS * 32, 0, st>>>(a);
    else pnp_batch_kernel<PnpInput::Fp64><<<blocks, PNP_WARPS * 32, 0, st>>>(a);
    return cudaGetLastError();
}

} // namespace pvb
