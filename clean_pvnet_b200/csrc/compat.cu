// compat.cu -- twins of the reference pybind module `ransac_voting`
// (lib/csrc/ransac_voting/src/ransac_voting.cpp:102-107) on the reference's own tensor layouts:
//   direct [tn,vn,2] f32, coords [tn,2] f32, idxs [hn,vn,2] i32, hyp [hn,vn,2|3] f32, inliers [hn,vn,tn] u8.
// The layer itself never materialises `inliers`; these exist so that code written against the
// reference extension (and the kernel-level parity tests) keeps working.
#include <cstring>
#include "api.h"
#include "common.cuh"
#include "kernels.h"

namespace pvb {

// ransac_voting_kernel.cu:11-49 (plain) and :170-229 (vanishing point).
template <bool VP>
__global__ void __launch_bounds__(256)
compat_generate_kernel(const float *__restrict__ direct, const float *__restrict__ coords,
                       const int32_t *__restrict__ idxs, float *__restrict__ hyp, int tn, int vn, int hn)
{
    const int hvi = blockIdx.x * 256 + threadIdx.x;
    if (hvi >= hn * vn) return;
    const int hi = hvi / vn, vi = hvi - hi * vn;
    const int t0 = idxs[(size_t)hvi * 2], t1 = idxs[(size_t)hvi * 2 + 1];
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if ((unsigned)t0 < (unsigned)tn && (unsigned)t1 < (unsigned)tn) {
        const float dx0 = direct[((size_t)t0 * vn + vi) * 2], dy0 = direct[((size_t)t0 * vn + vi) * 2 + 1];
        const float dx1 = direct[((size_t)t1 * vn + vi) * 2], dy1 = direct[((size_t)t1 * vn + vi) * 2 + 1];
        const float cx0 = coords[(size_t)t0 * 2], cy0 = coords[(size_t)t0 * 2 + 1];
        const float cx1 = coords[(size_t)t1 * 2], cy1 = coords[(size_t)t1 * 2 + 1];
        if (!VP) {
            float x, y;
            if (hypothesis_from_pair(dx0, dy0, cx0, cy0, dx1, dy1, cx1, cy1, x, y)) { o0 = x; o1 = y; }
        } else {
            // l = (dy, -dx, cy*dx - cx*dy); (x,y,z) = l0 x l1   (:199-210), contraction as compiled
            const float lz0 = __fmaf_rn(dx0, cy0, -__fmul_rn(dy0, cx0));
            const float lz1 = __fmaf_rn(dx1, cy1, -__fmul_rn(dy1, cx1));
            float x = __fmaf_rn(dx1, lz0, -__fmul_rn(dx0, lz1));
            float y = __fmaf_rn(dy1, lz0, -__fmul_rn(dy0, lz1));
            float z = __fmaf_rn(dx0, dy1, -__fmul_rn(dy0, dx1));
            const float val_x0 = __fmul_rn(dx0, __fmaf_rn(-cx0, z, x));
            const float val_x1 = __fmul_rn(dx1, __fmaf_rn(-cx1, z, x));
            const float val_y0 = __fmul_rn(dy0, __fmaf_rn(-cy0, z, y));
            const float val_y1 = __fmul_rn(dy1, __fmaf_rn(-cy1, z, y));
            if (val_x0 < 0 && val_x1 < 0 && val_y0 < 0 && val_y1 < 0) { z = -z; x = -x; y = -y; }   // :219-220
            if (__fmul_rn(val_x0, val_x1) < 0 || __fmul_rn(val_y0, val_y1) < 0) { x = 0.f; y = 0.f; z = 0.f; }   // :222-223
            o0 = x; o1 = y; o2 = z;
        }
    }
    if (!VP) { hyp[(size_t)hvi * 2] = o0; hyp[(size_t)hvi * 2 + 1] = o1; }
    else { hyp[(size_t)hvi * 3] = o0; hyp[(size_t)hvi * 3 + 1] = o1; hyp[(size_t)hvi * 3 + 2] = o2; }
}

// ransac_voting_kernel.cu:268-310
__device__ __forceinline__ bool vote_exact_vp(float vx, float vy, float cx, float cy, float hx, float hy, float hz,
                                              float thresh)
{
    const float fx = __fmaf_rn(-cx, hz, hx), fy = __fmaf_rn(-cy, hz, hy);
    const float n1 = __fsqrt_rn(__fmaf_rn(vx, vx, __fmul_rn(vy, vy)));
    const float n2 = __fsqrt_rn(__fmaf_rn(fx, fx, __fmul_rn(fy, fy)));
    if ((double)n1 < 1e-6 || (double)n2 < 1e-6) return false;
    const float valx = __fmul_rn(vx, fx), valy = __fmul_rn(vy, fy);
    const float c = __fdiv_rn(__fadd_rn(valx, valy), __fmul_rn(n2, n1));
    if (valx < 0 || valy < 0) return false;
    return fabsf(c) > thresh;
}

// ransac_voting_kernel.cu:88-126 / :268-310.  Thread per (k,t), loop over h: the pixel's data is
// loaded once and the byte stores of a warp are contiguous in t.
template <bool VP>
__global__ void __launch_bounds__(256)
compat_vote_kernel(const float *__restrict__ direct, const float *__restrict__ coords,
                   const float *__restrict__ hyp, uint8_t *__restrict__ inliers, int tn, int vn, int hn,
                   float thresh, int h_per_block)
{
    const int ti = blockIdx.x * 256 + threadIdx.x;
    const int vi = blockIdx.y;
    if (ti >= tn) return;
    const float vx = direct[((size_t)ti * vn + vi) * 2], vy = direct[((size_t)ti * vn + vi) * 2 + 1];
    const float cx = coords[(size_t)ti * 2], cy = coords[(size_t)ti * 2 + 1];
    const int h0 = blockIdx.z * h_per_block, h1 = min(hn, h0 + h_per_block);
    constexpr int HS = VP ? 3 : 2;
    for (int hi = h0; hi < h1; ++hi) {
        const float *hp = hyp + ((size_t)hi * vn + vi) * HS;
        bool in;
        if (!VP) in = vote_exact(vx, vy, cx, cy, __ldg(hp), __ldg(hp + 1), thresh);
        else in = vote_exact_vp(vx, vy, cx, cy, __ldg(hp), __ldg(hp + 1), __ldg(hp + 2), thresh);
        if (in) inliers[((size_t)hi * vn + vi) * tn + ti] = 1;
    }
}

// reference layouts -> layer layouts, so pvb_vote_count can run the layer's own vote kernel
__global__ void __launch_bounds__(256)
compat_repack_kernel(const float *__restrict__ direct, const float *__restrict__ coords,
                     const float *__restrict__ hyp, int tn, int vn, int hn, float2 *__restrict__ dirs,
                     float2 *__restrict__ xy, float2 *__restrict__ hyp_k, int *__restrict__ meta)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < tn) {
        const float2 c = make_float2(coords[(size_t)i * 2], coords[(size_t)i * 2 + 1]);
        xy[i] = c;
        for (int k = 0; k < vn; ++k)
            dirs[(size_t)k * tn + i] = make_float2(direct[((size_t)i * vn + k) * 2], direct[((size_t)i * vn + k) * 2 + 1]);
    }
    if (i < hn)
        for (int k = 0; k < vn; ++k)
            hyp_k[(size_t)k * hn + i] = make_float2(hyp[((size_t)i * vn + k) * 2], hyp[((size_t)i * vn + k) * 2 + 1]);
    if (i == 0) { meta[0] = tn; meta[1] = 0; }
}

__global__ void __launch_bounds__(256)
compat_unpack_counts_kernel(const int *__restrict__ counts_k, int *__restrict__ counts, int vn, int hn)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= hn * vn) return;
    const int h = i / vn, k = i - h * vn;
    counts[i] = counts_k[(size_t)k * hn + h];
}

namespace {

cudaError_t launch_compat_generate(const float *direct, const float *coords, const int32_t *idxs, float *hyp,
                                   int tn, int vn, int hn, bool vanishing, cudaStream_t st)
{
    const int n = hn * vn;
    if (n == 0) return cudaSuccess;
    if (vanishing) compat_generate_kernel<true><<<(n + 255) / 256, 256, 0, st>>>(direct, coords, idxs, hyp, tn, vn, hn);
    else compat_generate_kernel<false><<<(n + 255) / 256, 256, 0, st>>>(direct, coords, idxs, hyp, tn, vn, hn);
    return cudaGetLastError();
}

cudaError_t launch_compat_vote(const float *direct, const float *coords, const float *hyp, uint8_t *inliers,
                               int tn, int vn, int hn, float thresh, bool vanishing, cudaStream_t st)
{
    if (tn == 0 || vn == 0 || hn == 0) return cudaSuccess;
    const int hpb = 64;
    dim3 g((tn + 255) / 256, vn, (hn + hpb - 1) / hpb);
    if (vanishing) compat_vote_kernel<true><<<g, 256, 0, st>>>(direct, coords, hyp, inliers, tn, vn, hn, thresh, hpb);
    else compat_vote_kernel<false><<<g, 256, 0, st>>>(direct, coords, hyp, inliers, tn, vn, hn, thresh, hpb);
    return cudaGetLastError();
}

int check_compat(const void *a, const void *b, const void *c, const void *d_, int tn, int vn, int hn)
{
    if (tn < 0 || vn < 0 || hn < 0) return fail(PVB_ERR_INVALID, "negative size");
    if ((long long)hn * vn > (1ll << 30) || (long long)tn * vn > (1ll << 30)) return fail(PVB_ERR_INVALID, "problem too large");
    if (((tn && vn) && (!a || !b)) || ((hn && vn) && (!c || !d_))) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (vn > 65535) return fail(PVB_ERR_INVALID, "vn must be <= 65535");
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs, float *hyp, int32_t tn,
                            int32_t vn, int32_t hn, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, idxs, hyp, tn, vn, hn);
    if (rc) return rc;
    cudaError_t e = launch_compat_generate(direct, coords, idxs, hyp, tn, vn, hn, false, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "generate_hypothesis");
}

PVB_API int pvb_generate_hypothesis_vanishing_point(const float *direct, const float *coords, const int32_t *idxs, float *hyp,
                                            int32_t tn, int32_t vn, int32_t hn, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, idxs, hyp, tn, vn, hn);
    if (rc) return rc;
    cudaError_t e = launch_compat_generate(direct, coords, idxs, hyp, tn, vn, hn, true, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "generate_hypothesis_vanishing_point");
}

PVB_API int pvb_voting_for_hypothesis(const float *direct, const float *coords, const float *hyp, uint8_t *inliers, int32_t tn,
                              int32_t vn, int32_t hn, float inlier_thresh, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, inliers, tn, vn, hn);
    if (rc) return rc;
    if (tn && vn && hn && !inliers) return fail(PVB_ERR_INVALID, "NULL tensor");
    cudaError_t e = launch_compat_vote(direct, coords, hyp, inliers, tn, vn, hn, inlier_thresh, false, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "voting_for_hypothesis");
}

PVB_API int pvb_voting_for_hypothesis_vanishing_point(const float *direct, const float *coords, const float *hyp,
                                              uint8_t *inliers, int32_t tn, int32_t vn, int32_t hn,
                                              float inlier_thresh, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, inliers, tn, vn, hn);
    if (rc) return rc;
    if (tn && vn && hn && !inliers) return fail(PVB_ERR_INVALID, "NULL tensor");
    cudaError_t e = launch_compat_vote(direct, coords, hyp, inliers, tn, vn, hn, inlier_thresh, true, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "voting_for_hypothesis_vanishing_point");
}

PVB_API size_t pvb_vote_count_workspace_bytes(int32_t tn, int32_t vn, int32_t hn)
{
    if (tn < 0 || vn < 0 || hn < 0) return 0;
    size_t off = align_up(4 * sizeof(int));
    off += align_up((size_t)tn * sizeof(float2));
    off += align_up((size_t)tn * vn * sizeof(float2));
    off += align_up((size_t)hn * vn * sizeof(float2));
    off += align_up((size_t)hn * vn * sizeof(int));
    return off;
}

PVB_API int pvb_vote_count(const float *direct, const float *coords, const float *hyp, int32_t *counts, int32_t tn, int32_t vn,
                   int32_t hn, float inlier_thresh, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, counts, tn, vn, hn);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (hn == 0 || vn == 0) return PVB_OK;
    if (tn == 0) {
        cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)hn * vn, st);
        return e == cudaSuccess ? PVB_OK : cuda_fail(e, "memset");
    }
    if ((long long)vn * ((hn + 511) / 512) > 65535) return fail(PVB_ERR_INVALID, "vn*ceil(hn/512) must be <= 65535");
    rc = check_workspace(pvb_vote_count_workspace_bytes(tn, vn, hn), workspace, workspace_bytes);
    if (rc) return rc;
    // the reference layout -> the layer's (pixels, directions and hypotheses k-major); meta = { tn, state 0, unused, unused }
    char *w = static_cast<char *>(workspace);
    size_t off = 0;
    int *meta = reinterpret_cast<int *>(w + off); off += align_up(4 * sizeof(int));
    float2 *xy = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)tn * sizeof(float2));
    float2 *dirs = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)tn * vn * sizeof(float2));
    float2 *hyp_k = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)hn * vn * sizeof(float2));
    int *counts_k = reinterpret_cast<int *>(w + off);
    cudaError_t e = cudaMemsetAsync(meta, 0, 4 * sizeof(int), st);
    if (e == cudaSuccess) {
        const int n = tn > hn ? tn : hn;
        compat_repack_kernel<<<(n + 255) / 256 + 1, 256, 0, st>>>(direct, coords, hyp, tn, vn, hn, dirs, xy, hyp_k, meta);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return cuda_fail(e, "repack");
    VoteArgs v;
    memset(&v, 0, sizeof(v));
    v.B = 1; v.K = vn; v.hn = hn; v.cap = tn; v.W = 0; v.H = 0; v.thresh = inlier_thresh;
    v.tn = meta; v.state = meta + 1; v.xy = xy;
    v.dirs = dirs; v.idxs = nullptr; v.hyp = hyp_k; v.counts = counts_k;
    e = launch_vote(v, true, false, st);
    if (e != cudaSuccess) return cuda_fail(e, "vote kernel");
    compat_unpack_counts_kernel<<<(hn * vn + 255) / 256, 256, 0, st>>>(counts_k, counts, vn, hn);
    e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "unpack");
}

} // extern "C"
