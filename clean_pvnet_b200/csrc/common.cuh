// common.cuh -- shared device helpers of the H100 RANSAC voting layer.
//
// Exact arithmetic: every floating-point operation the reference kernels perform is
// written with round-to-nearest intrinsics in the contraction pattern nvcc 12.9 gives
// the reference source for sm_100 (read from `cuobjdump -sass` of the unmodified
// reference build, see DESIGN.md "Observed arithmetic").  That is what makes hypotheses
// bit-equal and inlier counts equal to the reference extension.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <utility>

namespace pvb {

// ---------------------------------------------------------------------------------
// Programmatic dependent launch (PDL) of the v3 chain (DESIGN.md 4.3):
//   thin_gather | generate -> [prune_hist -> prune_bound -> vote_kernel (pass 1) -> prune_next -> vote_list_kernel
//   | vote_kernel] -> refit
// thin_gather is launched plainly and never triggers early, so its exit is its trigger.  A chained kernel may start while
// its immediate predecessor is still running.  The dependency rule every chained kernel keeps, so that this is no race:
//   1. it executes grid_dep_wait() before it reads anything its immediate predecessor writes, before it writes anything
//      that predecessor reads, and before it exits (every thread, on every path, early returns included);
//   2. it executes grid_dep_launch_dependents() only after its own grid_dep_wait().
// By induction, when a kernel starts, every kernel two or more launches back has completed and its writes are visible:
// the predecessor has passed its wait (rule 2), which waited for the one before it (rule 1).  Only such data may be read
// before the wait.  A kernel is launched chained only when its predecessor in the stream is a kernel of the chain that keeps
// the rule; after a memset, an event or a foreign kernel it is launched plainly, and the wait returns at once.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Launches kernel<<<grid, block, smem, st>>>(args...), allowed to overlap its predecessor in the stream (PDL) when
// `chained`.  Returns the launch's error.
template <typename... Params, typename... Args>
cudaError_t launch_chained(bool chained, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                           Args &&...args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = chained ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ---------------------------------------------------------------------------------
// Philox4x32-10.  Counter layout of the built-in sampling mode (DESIGN.md "Sampling"):
//   pair indices : ctr = (h, k, image, tag_idx)  -> t0 = out[0] % tn, t1 = out[1] % tn
//   thinning     : ctr = (pixel>>2, 0, image, tag_sel) -> u = (out[pixel&3] >> 8) * 2^-24
// Keyed by (seed_lo, seed_hi).  Results do not depend on grid shape or GPU count.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ float u32_to_unit(uint32_t x) { return (float)(x >> 8) * 5.9604644775390625e-08f; }

// ---------------------------------------------------------------------------------
// Hypothesis from one pixel pair (reference: ransac_voting_kernel.cu:27-48).
// Returns false where the reference thread returns early; the caller writes (0,0).
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool hypothesis_from_pair(float dx0, float dy0, float cx0, float cy0,
                                                     float dx1, float dy1, float cx1, float cy1,
                                                     float &x, float &y)
{
    const float p = __fmul_rn(dy0, dx1);
    const float q = __fmul_rn(dx0, dy1);
    const float det1 = __fsub_rn(p, q);   // nx1*ny0 - nx0*ny1   (.cu:42)
    const float det2 = __fsub_rn(q, p);   // ny1*nx0 - ny0*nx1   (.cu:43)
    if (fabs((double)det1) < 1e-6) return false;
    if (fabs((double)det2) < 1e-6) return false;
    const float e0 = __fmaf_rn(dy0, cx0, -__fmul_rn(dx0, cy0));
    const float e1 = __fmaf_rn(dy1, cx1, -__fmul_rn(dx1, cy1));
    y = __fdiv_rn(__fmaf_rn(dy1, e0, -__fmul_rn(dy0, e1)), det1);   // .cu:44
    x = __fdiv_rn(__fmaf_rn(dx0, e1, -__fmul_rn(dx1, e0)), det2);   // .cu:45
    return true;
}

// ---------------------------------------------------------------------------------
// The reference inlier predicate, exactly (ransac_voting_kernel.cu:107-125).
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool vote_exact(float vx, float vy, float cx, float cy, float hx, float hy,
                                           float thresh)
{
    const float dx = __fsub_rn(hx, cx), dy = __fsub_rn(hy, cy);
    const float n1sq = __fmaf_rn(vx, vx, __fmul_rn(vy, vy));
    const float n2sq = __fmaf_rn(dx, dx, __fmul_rn(dy, dy));
    const float norm1 = __fsqrt_rn(n1sq), norm2 = __fsqrt_rn(n2sq);
    if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) return false;
    const float den = __fmul_rn(norm2, norm1);
    const float dot = __fmaf_rn(vx, dx, __fmul_rn(vy, dy));
    return __fdiv_rn(dot, den) > thresh;
}

// Largest float below 1e-6: (double)n < 1e-6  <=>  n <= below_1e6() for a float n
// (float(1e-6) = 0x358637BD = 9.99999997e-07 < 1e-6 < next float).
__device__ __forceinline__ float below_1e6() { return __int_as_float(0x358637BD); }

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum(int v) { return __reduce_add_sync(0xffffffffu, v); }

// inv(sqrtm(cov)) of one 2x2 covariance, packed (wxx, wxy, wyy) and rounded to fp32 -- SURVEY 8f row 2
// (lib/evaluators/linemod/pvnet.py:118-130: scipy.linalg.sqrtm + np.linalg.inv per keypoint on the CPU).
// Closed form for a symmetric positive definite 2x2 M: sqrt(M) = (M + s I)/t, s = sqrt(det M), t = sqrt(tr M + 2 s),
// so inv(sqrt(M)) = t * adj(M + s I) / det(M + s I).  cov[0,0] < 1e-6 or any NaN -> zeros, like the reference.
__device__ __forceinline__ void cov_to_weights(const float4 c, float &o0, float &o1, float &o2)
{
    o0 = 0.f; o1 = 0.f; o2 = 0.f;
    const bool bad = (c.x < 1e-6f) || (c.x != c.x) || (c.y != c.y) || (c.z != c.z) || (c.w != c.w);
    if (!bad) {
        const double a = c.x, b = 0.5 * ((double)c.y + (double)c.z), d = c.w;
        const double det = a * d - b * b;
        if (det > 0.0) {
            const double s = sqrt(det), t = sqrt(a + d + 2.0 * s);
            const double a2 = a + s, d2 = d + s;
            const double den = a2 * d2 - b * b;
            o0 = (float)(t * d2 / den); o1 = (float)(-t * b / den); o2 = (float)(t * a2 / den);
        }
    }
}

// Parameters of the cone test used by the fast path of the vote kernel (vote.cu).
struct ConeParams {
    float kappa;   // tan(acos(thresh)) = sqrt(1-t^2)/t
    float band;    // guard band per unit of S = |hx-ox|+|hy-oy|+cmax(tile) ; +inf => exact path only
    float floor;   // lower bound of the guard band: flags every test with |h-c| <= 1e-6 (the reference's norm cut)
    float thresh;  // (float)inlier_thresh
};

} // namespace pvb
