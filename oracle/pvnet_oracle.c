/*
 * pvnet_oracle.c -- CPU restatement of clean-pvnet's RANSAC voting layer.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity checker for the CUDA
 * product in clean_pvnet_b200/csrc.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / reference legs may build, load or call it.
 * The product never links or imports anything under oracle/.
 *
 * PARITY PIN: the reference has no tests or golden vectors for this path
 * (SURVEY.md section 4).  The pin is golden vectors produced by the
 * reference's own CUDA extension, compiled unmodified by oracle/build_ref.py,
 * committed under tests/golden/ with the generating scripts: its sm_100a build
 * (kernels.npz etc.: hypotheses bit-equal, inlier counts equal) and its sm_90a
 * build (parity.npz, tests/test_gpu_reference_parity.py).
 *
 * Every function cites the reference file:line it restates (paths relative to
 * /root/reference).  Arithmetic follows the SASS the reference compiles to
 * with nvcc 12.9 (-fmad=true, no fast-math); the contraction pattern was read
 * from `cuobjdump -sass` of oracle/_ref and is written out with explicit
 * fmaf().  Build with -ffp-contract=off so the host compiler adds no fusions.
 *
 *   lib/csrc/ransac_voting/src/ransac_voting_kernel.cu
 *     :11-49    generate_hypothesis_kernel          -> orc_generate_hypothesis
 *     :88-126   voting_for_hypothesis_kernel        -> orc_voting_for_hypothesis
 *     :170-229  generate_hypothesis_vanishing_point -> orc_generate_hypothesis_vp
 *     :268-310  voting_for_hypothesis_vanishing_pt  -> orc_voting_for_hypothesis_vp
 *   lib/csrc/ransac_voting/ransac_voting_gpu.py
 *     :125-143  pixel selection (v3), :207-227 (dist) -> orc_select_pixels
 *     :112-199  ransac_voting_layer_v3              -> orc_ransac_voting_v3
 *     :202-274  estimate_voting_distribution_with_mean -> orc_estimate_voting_distribution
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#if defined(__GNUC__)
#define ORC_API __attribute__((visibility("default")))
#else
#define ORC_API
#endif

/* ------------------------------------------------------------------------ */
/* Philox4x32-10 (Salmon et al., SC'11; same generator curand/ATen use).     */
/* Used only by the "philox" sampling mode, which is this project's own      */
/* counter layout (DESIGN.md "Sampling").  KATs in tests/test_oracle.py.     */
/* ------------------------------------------------------------------------ */
ORC_API void orc_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3];
    uint32_t k0 = key[0], k1 = key[1];
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* Counter layout of the philox sampling mode (mirrored, independently, in
 * clean_pvnet_b200/csrc/common.cuh, philox4x32_10).  tag: 1 = v3 pair indices, 2 = v3
 * thinning, 3 = distribution pair indices, 4 = distribution thinning. */
enum { ORC_TAG_V3_IDX = 1, ORC_TAG_V3_SEL = 2, ORC_TAG_DIST_IDX = 3, ORC_TAG_DIST_SEL = 4 };

static void philox_pair(uint64_t seed, uint32_t tag, uint32_t img, uint32_t k, uint32_t h,
                        uint32_t tn, int32_t *t0, int32_t *t1)
{
    uint32_t ctr[4] = { h, k, img, tag }, key[2] = { (uint32_t)seed, (uint32_t)(seed >> 32) }, o[4];
    orc_philox4x32_10(ctr, key, o);
    *t0 = (int32_t)(o[0] % tn);
    *t1 = (int32_t)(o[1] % tn);
}

static float philox_uniform(uint64_t seed, uint32_t tag, uint32_t img, uint32_t pixel)
{
    uint32_t ctr[4] = { pixel >> 2, 0u, img, tag }, key[2] = { (uint32_t)seed, (uint32_t)(seed >> 32) }, o[4];
    orc_philox4x32_10(ctr, key, o);
    return (float)(o[pixel & 3u] >> 8) * 5.9604644775390625e-08f; /* 2^-24, u in [0,1) */
}

/* ------------------------------------------------------------------------ */
/* Hypothesis from one pixel pair -- ransac_voting_kernel.cu:27-48.          */
/* d? = direct[t?,k,:], c? = coords[t?,:].  Returns 0 when the reference     */
/* thread returns early (output keeps its zero fill, :75).                   */
/* ------------------------------------------------------------------------ */
static int hyp_one(float dx0, float dy0, float cx0, float cy0,
                   float dx1, float dy1, float cx1, float cy1, float *x, float *y)
{
    float p = dy0 * dx1;            /* FMUL  */
    float q = dx0 * dy1;            /* FMUL  */
    float det1 = p - q;             /* FADD  nx1*ny0-nx0*ny1 (:42) */
    float det2 = q - p;             /* FADD  ny1*nx0-ny0*nx1 (:43) */
    if (fabs((double)det1) < 1e-6) return 0;
    if (fabs((double)det2) < 1e-6) return 0;
    float e0 = fmaf(dy0, cx0, -(dx0 * cy0));   /* nx0*cx0+ny0*cy0 */
    float e1 = fmaf(dy1, cx1, -(dx1 * cy1));   /* nx1*cx1+ny1*cy1 */
    *y = fmaf(dy1, e0, -(dy0 * e1)) / det1;    /* :44 */
    *x = fmaf(dx0, e1, -(dx1 * e0)) / det2;    /* :45 */
    return 1;
}

/* generate_hypothesis -- ransac_voting_kernel.cu:11-49, launcher :51-86.
 * direct [tn,vn,2], coords [tn,2] (x,y), idxs [hn,vn,2] -> hyp [hn,vn,2]. */
ORC_API void orc_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs,
                                     float *hyp, int tn, int vn, int hn)
{
    (void)tn;
    memset(hyp, 0, sizeof(float) * (size_t)hn * vn * 2);
    for (int hi = 0; hi < hn; ++hi)
        for (int vi = 0; vi < vn; ++vi) {
            int t0 = idxs[(hi * vn + vi) * 2], t1 = idxs[(hi * vn + vi) * 2 + 1];
            float x, y;
            if (hyp_one(direct[(t0 * vn + vi) * 2], direct[(t0 * vn + vi) * 2 + 1], coords[t0 * 2], coords[t0 * 2 + 1],
                        direct[(t1 * vn + vi) * 2], direct[(t1 * vn + vi) * 2 + 1], coords[t1 * 2], coords[t1 * 2 + 1],
                        &x, &y)) {
                hyp[(hi * vn + vi) * 2] = x;
                hyp[(hi * vn + vi) * 2 + 1] = y;
            }
        }
}

/* One inlier test -- ransac_voting_kernel.cu:107-125. */
static inline int vote_one(float vx, float vy, float cx, float cy, float hx, float hy, float thresh)
{
    float dx = hx - cx, dy = hy - cy;
    float n1sq = fmaf(vx, vx, vy * vy);
    float n2sq = fmaf(dx, dx, dy * dy);
    float norm1 = sqrtf(n1sq), norm2 = sqrtf(n2sq);
    if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) return 0;   /* :121 */
    float den = norm2 * norm1;
    float dot = fmaf(vx, dx, vy * dy);
    float c = dot / den;                                          /* :123 */
    return c > thresh;                                            /* :124 */
}

/* voting_for_hypothesis -- ransac_voting_kernel.cu:88-126, launcher :129-167.
 * Sets inliers[h,k,t]=1 where the test passes; other bytes untouched. */
ORC_API void orc_voting_for_hypothesis(const float *direct, const float *coords, const float *hyp,
                                       uint8_t *inliers, int tn, int vn, int hn, float thresh)
{
    for (int hi = 0; hi < hn; ++hi)
        for (int vi = 0; vi < vn; ++vi) {
            float hx = hyp[(hi * vn + vi) * 2], hy = hyp[(hi * vn + vi) * 2 + 1];
            uint8_t *row = inliers + ((size_t)hi * vn + vi) * tn;
            for (int ti = 0; ti < tn; ++ti)
                if (vote_one(direct[(ti * vn + vi) * 2], direct[(ti * vn + vi) * 2 + 1],
                             coords[ti * 2], coords[ti * 2 + 1], hx, hy, thresh))
                    row[ti] = 1;
        }
}

/* voting + torch.sum(inlier, 2) (ransac_voting_gpu.py:156-159) without the
 * byte tensor: counts [hn,vn] int32. */
ORC_API void orc_vote_count(const float *direct, const float *coords, const float *hyp,
                            int32_t *counts, int tn, int vn, int hn, float thresh)
{
    for (int hi = 0; hi < hn; ++hi)
        for (int vi = 0; vi < vn; ++vi) {
            float hx = hyp[(hi * vn + vi) * 2], hy = hyp[(hi * vn + vi) * 2 + 1];
            int32_t c = 0;
            for (int ti = 0; ti < tn; ++ti)
                c += vote_one(direct[(ti * vn + vi) * 2], direct[(ti * vn + vi) * 2 + 1],
                              coords[ti * 2], coords[ti * 2 + 1], hx, hy, thresh);
            counts[hi * vn + vi] = c;
        }
}

/* generate_hypothesis_vanishing_point -- ransac_voting_kernel.cu:170-229.
 * Arithmetic per the sm_100 SASS of oracle/_ref (see DESIGN.md "Observed arithmetic"). */
ORC_API void orc_generate_hypothesis_vp(const float *direct, const float *coords, const int32_t *idxs,
                                        float *hyp, int tn, int vn, int hn)
{
    (void)tn;
    for (int hi = 0; hi < hn; ++hi)
        for (int vi = 0; vi < vn; ++vi) {
            int id0 = idxs[(hi * vn + vi) * 2], id1 = idxs[(hi * vn + vi) * 2 + 1];
            float dx0 = direct[(id0 * vn + vi) * 2], dy0 = direct[(id0 * vn + vi) * 2 + 1];
            float cx0 = coords[id0 * 2], cy0 = coords[id0 * 2 + 1];
            float dx1 = direct[(id1 * vn + vi) * 2], dy1 = direct[(id1 * vn + vi) * 2 + 1];
            float cx1 = coords[id1 * 2], cy1 = coords[id1 * 2 + 1];
            /* l? = (dy, -dx, cy*dx - cx*dy)   (:199-205) */
            float lz0 = fmaf(cy0, dx0, -(cx0 * dy0));
            float lz1 = fmaf(cy1, dx1, -(cx1 * dy1));
            /* x = ly0*lz1 - lz0*ly1 = -dx0*lz1 + lz0*dx1 (:208) */
            float x = fmaf(lz0, dx1, -(dx0 * lz1));
            /* y = lz0*lx1 - lx0*lz1 = lz0*dy1 - dy0*lz1 (:209) */
            float y = fmaf(lz0, dy1, -(dy0 * lz1));
            /* z = lx0*ly1 - ly0*lx1 = -dy0*dx1 + dx0*dy1 (:210) */
            float z = fmaf(dx0, dy1, -(dy0 * dx1));
            float val_x0 = dx0 * fmaf(-z, cx0, x);
            float val_x1 = dx1 * fmaf(-z, cx1, x);
            float val_y0 = dy0 * fmaf(-z, cy0, y);
            float val_y1 = dy1 * fmaf(-z, cy1, y);
            if (val_x0 < 0 && val_x1 < 0 && val_y0 < 0 && val_y1 < 0) { z = -z; x = -x; y = -y; }
            if (val_x0 * val_x1 < 0 || val_y0 * val_y1 < 0) { x = 0.f; y = 0.f; z = 0.f; }
            hyp[(hi * vn + vi) * 3] = x;
            hyp[(hi * vn + vi) * 3 + 1] = y;
            hyp[(hi * vn + vi) * 3 + 2] = z;
        }
}

/* voting_for_hypothesis_vanishing_point -- ransac_voting_kernel.cu:268-310. */
ORC_API void orc_voting_for_hypothesis_vp(const float *direct, const float *coords, const float *hyp,
                                          uint8_t *inliers, int tn, int vn, int hn, float thresh)
{
    for (int hi = 0; hi < hn; ++hi)
        for (int vi = 0; vi < vn; ++vi) {
            float hx = hyp[(hi * vn + vi) * 3], hy = hyp[(hi * vn + vi) * 3 + 1], hz = hyp[(hi * vn + vi) * 3 + 2];
            uint8_t *row = inliers + ((size_t)hi * vn + vi) * tn;
            for (int ti = 0; ti < tn; ++ti) {
                float cx = coords[ti * 2], cy = coords[ti * 2 + 1];
                float vx = direct[(ti * vn + vi) * 2], vy = direct[(ti * vn + vi) * 2 + 1];
                float fx = fmaf(-cx, hz, hx), fy = fmaf(-cy, hz, hy);
                float n1 = sqrtf(fmaf(vx, vx, vy * vy)), n2 = sqrtf(fmaf(fx, fx, fy * fy));
                if ((double)n1 < 1e-6 || (double)n2 < 1e-6) continue;
                float valx = fx * vx, valy = fy * vy;
                float c = (valx + valy) / (n1 * n2);
                if (valx < 0 || valy < 0) continue;
                if (fabsf(c) > thresh) row[ti] = 1;
            }
        }
}

/* ------------------------------------------------------------------------ */
/* Pixel selection -- ransac_voting_gpu.py:125-143 (v3) / :207-227 (dist).   */
/* mask: contiguous int64 [H*W].  mode 0 (v3): cur_mask = mask.byte(),       */
/* fg = sum of byte VALUES (:126); mode 1 (dist): cur_mask = (mask==1),      */
/* fg = count (:207-208).  selection: optional float [H*W] of U(0,1) draws   */
/* (the reference's `selection`, :136); when NULL and thinning is needed the */
/* philox stream (seed, tag, img) is used.  Outputs pix (row-major order =   */
/* torch.nonzero order, :140) and returns tn, or -1 when fg < min_num.       */
/* Optional (may be NULL): fg_out = fg, nz_out = pixels selected before      */
/* thinning (cur_mask's nonzero count).                                      */
/* ------------------------------------------------------------------------ */
static int select_pixels(const int64_t *mask, int H, int W, int mode, int min_num, int max_num,
                         const float *selection, uint64_t seed, uint32_t tag, uint32_t img,
                         int32_t *pix, int64_t *fg_out, int32_t *nz_out)
{
    const int n = H * W;
    int64_t fg = 0;
    int32_t nz = 0;
    for (int i = 0; i < n; ++i) {
        if (mode == 0) { fg += (uint8_t)mask[i]; nz += ((uint8_t)mask[i] != 0); }
        else { fg += (mask[i] == 1); nz += (mask[i] == 1); }
    }
    if (fg_out) *fg_out = fg;
    if (nz_out) *nz_out = nz;
    if (fg < min_num) return -1;
    int thin = fg > max_num;
    float ratio = 0.f;
    /* max_num / foreground_num.float(): a Python number divided by a tensor is Tensor.__rtruediv__,
     * i.e. reciprocal() * max_num -- two fp32 roundings, not one correctly rounded quotient */
    if (thin) ratio = (1.f / (float)fg) * (float)max_num;
    int tn = 0;
    for (int i = 0; i < n; ++i) {
        int sel = (mode == 0) ? ((uint8_t)mask[i] != 0) : (mask[i] == 1);
        if (!sel) continue;
        if (thin) {
            float u = selection ? selection[i] : philox_uniform(seed, tag, img, (uint32_t)i);
            if (!(u < ratio)) continue;
        }
        pix[tn++] = i;
    }
    return tn;
}

/* Pixel selection alone, batched -- the front of ransac_voting_gpu.py:125-143 (mode 0, tag 2) and :207-227
 * (mode 1, tag 4).  mask int64 [B,H*W]; selection optional float [B,H*W] (NULL: philox stream (seed, tag,
 * img_base+b)).  Per image: fg_out[b], nz_out[b], tn_out[b] (-1 when skipped) and the first tn entries of
 * pix[b*H*W ...] (row-major pixel indices). */
ORC_API void orc_select_pixels(const int64_t *mask, int B, int H, int W, int mode, int min_num, int max_num,
                               const float *selection, uint64_t seed, int img_base, uint32_t tag,
                               int64_t *fg_out, int32_t *nz_out, int32_t *tn_out, int32_t *pix)
{
    const size_t HW = (size_t)H * W;
    for (int b = 0; b < B; ++b)
        tn_out[b] = select_pixels(mask + b * HW, H, W, mode, min_num, max_num, selection ? selection + b * HW : NULL,
                                  seed, tag, (uint32_t)(img_base + b), pix + b * HW, fg_out + b, nz_out + b);
}

/* Least-squares ray intersection of the winner's inliers -- ransac_voting_gpu.py:177-196.
 * The reference accumulates ATA/ATb in fp32 (cuBLAS matmul + torch.sum) and solves with a
 * batched LU; summation order there is unspecified, so the oracle accumulates in double
 * (the value both implementations approximate).  Singular ATA -> identity inverse, the
 * behaviour of b_inv's bare except (:105-108) for the singular k itself (the reference
 * additionally poisons the other keypoints of that image; not restated, see DESIGN.md). */
static void refit_one(const float *dir_k /* [tn] float2 for this k, stride */, int stride,
                      const int32_t *pix, int W, int tn, float wx, float wy, float thresh, float *out)
{
    double a00 = 0, a01 = 0, a11 = 0, b0 = 0, b1 = 0;
    for (int t = 0; t < tn; ++t) {
        float vx = dir_k[(size_t)t * stride], vy = dir_k[(size_t)t * stride + 1];
        float cx = (float)(pix[t] % W), cy = (float)(pix[t] / W);
        if (!vote_one(vx, vy, cx, cy, wx, wy, thresh)) continue;
        double nx = vy, ny = -(double)vx;
        double bb = nx * cx + ny * cy;
        a00 += nx * nx; a01 += nx * ny; a11 += ny * ny;
        b0 += nx * bb;  b1 += ny * bb;
    }
    double det = a00 * a11 - a01 * a01;
    if (det == 0.0 || !isfinite(det)) { out[0] = (float)b0; out[1] = (float)b1; return; }
    out[0] = (float)((a11 * b0 - a01 * b1) / det);
    out[1] = (float)((a00 * b1 - a01 * b0) / det);
}

/* ransac_voting_layer_v3 -- ransac_voting_gpu.py:112-199.
 * mask int64 [B,H,W]; vertex fp32 contiguous [B,H,W,K,2]; out [B,K,2].
 * idxs: optional int32 [B,hn,K,2] (the reference's per-image `idxs`, :145);
 *       NULL -> philox mode.  selection: optional float [B,H,W] (:136).
 * The confidence loop (:150-174) re-evaluates identical hypotheses every
 * round (idxs is drawn once, outside the loop), so one round is exact.
 * Optional debug outputs (may be NULL): tn_out[B], hyp_out[B,K,hn,2],
 * counts_out[B,K,hn], win_out[B,K,2] (winning hypothesis before the refit). */
ORC_API int orc_ransac_voting_v3(const int64_t *mask, const float *vertex, int B, int H, int W, int K,
                                 int hn, float thresh, int min_num, int max_num,
                                 const int32_t *idxs, const float *selection,
                                 uint64_t seed, int img_base,
                                 float *out, int32_t *tn_out, float *hyp_out, int32_t *counts_out,
                                 float *win_out)
{
    const size_t HW = (size_t)H * W;
    int32_t *pix = (int32_t *)malloc(sizeof(int32_t) * HW);
    float *dirs = (float *)malloc(sizeof(float) * HW * K * 2);   /* [tn,K,2] */
    float *hyp = (float *)malloc(sizeof(float) * (size_t)hn * 2);
    if (!pix || !dirs || !hyp) return -1;
    for (int b = 0; b < B; ++b) {
        float *o = out + (size_t)b * K * 2;
        memset(o, 0, sizeof(float) * K * 2);
        if (hyp_out) memset(hyp_out + (size_t)b * K * hn * 2, 0, sizeof(float) * (size_t)K * hn * 2);
        if (counts_out) memset(counts_out + (size_t)b * K * hn, 0, sizeof(int32_t) * (size_t)K * hn);
        if (win_out) memset(win_out + (size_t)b * K * 2, 0, sizeof(float) * K * 2);
        int tn = select_pixels(mask + b * HW, H, W, 0, min_num, max_num,
                               selection ? selection + b * HW : NULL, seed, ORC_TAG_V3_SEL,
                               (uint32_t)(img_base + b), pix, NULL, NULL);
        if (tn_out) tn_out[b] = tn < 0 ? 0 : tn;
        if (tn < 0) continue;                                   /* :129-132 zeros */
        if (tn == 0) continue;   /* unreachable in the reference unless thinning drops everything */
        const float *vb = vertex + (size_t)b * HW * K * 2;
        for (int t = 0; t < tn; ++t)
            memcpy(dirs + (size_t)t * K * 2, vb + (size_t)pix[t] * K * 2, sizeof(float) * K * 2);
        for (int k = 0; k < K; ++k) {
            int best = -1, best_h = 0;
            for (int h = 0; h < hn; ++h) {
                int32_t t0, t1;
                if (idxs) {
                    t0 = idxs[(((size_t)b * hn + h) * K + k) * 2];
                    t1 = idxs[(((size_t)b * hn + h) * K + k) * 2 + 1];
                } else {
                    philox_pair(seed, ORC_TAG_V3_IDX, (uint32_t)(img_base + b), (uint32_t)k, (uint32_t)h,
                                (uint32_t)tn, &t0, &t1);
                }
                float x = 0.f, y = 0.f;
                hyp_one(dirs[((size_t)t0 * K + k) * 2], dirs[((size_t)t0 * K + k) * 2 + 1],
                        (float)(pix[t0] % W), (float)(pix[t0] / W),
                        dirs[((size_t)t1 * K + k) * 2], dirs[((size_t)t1 * K + k) * 2 + 1],
                        (float)(pix[t1] % W), (float)(pix[t1] / W), &x, &y);
                hyp[h * 2] = x; hyp[h * 2 + 1] = y;
                int32_t c = 0;
                for (int t = 0; t < tn; ++t)
                    c += vote_one(dirs[((size_t)t * K + k) * 2], dirs[((size_t)t * K + k) * 2 + 1],
                                  (float)(pix[t] % W), (float)(pix[t] / W), x, y, thresh);
                if (hyp_out) { hyp_out[(((size_t)b * K + k) * hn + h) * 2] = x;
                               hyp_out[(((size_t)b * K + k) * hn + h) * 2 + 1] = y; }
                if (counts_out) counts_out[((size_t)b * K + k) * hn + h] = c;
                if (c > best) { best = c; best_h = h; }          /* torch.max: first maximal index (:160) */
            }
            /* :165-167  all_win_ratio starts at 0 and is replaced only when strictly larger */
            float wx = 0.f, wy = 0.f;
            if (best > 0) { wx = hyp[best_h * 2]; wy = hyp[best_h * 2 + 1]; }
            if (win_out) { win_out[((size_t)b * K + k) * 2] = wx; win_out[((size_t)b * K + k) * 2 + 1] = wy; }
            refit_one(dirs + (size_t)k * 2, K * 2, pix, W, tn, wx, wy, thresh, o + k * 2);
        }
    }
    free(pix); free(dirs); free(hyp);
    return 0;
}

/* estimate_voting_distribution_with_mean -- ransac_voting_gpu.py:202-274.
 * hn_total = round_hyp_num * ceil(min_hyp_num/round_hyp_num) hypotheses per (image,k)
 * (:231-246, concatenated in round order).  idxs optional int32 [B,hn_total,K,2].
 * mean [B,K,2] -> cov [B,K,2,2].  Weighted sums accumulate in double. */
ORC_API int orc_estimate_voting_distribution(const int64_t *mask, const float *vertex, const float *mean,
                                             int B, int H, int W, int K, int hn_total, float thresh,
                                             int min_num, int max_num,
                                             const int32_t *idxs, const float *selection,
                                             uint64_t seed, int img_base,
                                             float *cov, float *hyp_out, float *ratio_out)
{
    const size_t HW = (size_t)H * W;
    int32_t *pix = (int32_t *)malloc(sizeof(int32_t) * HW);
    float *dirs = (float *)malloc(sizeof(float) * HW * K * 2);
    float *hyp = (float *)malloc(sizeof(float) * (size_t)hn_total * 2);
    float *ratio = (float *)malloc(sizeof(float) * (size_t)hn_total);
    if (!pix || !dirs || !hyp || !ratio) return -1;
    for (int b = 0; b < B; ++b) {
        int tn = select_pixels(mask + b * HW, H, W, 1, min_num, max_num,
                               selection ? selection + b * HW : NULL, seed, ORC_TAG_DIST_SEL,
                               (uint32_t)(img_base + b), pix, NULL, NULL);
        const float *vb = vertex + (size_t)b * HW * K * 2;
        if (tn > 0)
            for (int t = 0; t < tn; ++t)
                memcpy(dirs + (size_t)t * K * 2, vb + (size_t)pix[t] * K * 2, sizeof(float) * K * 2);
        for (int k = 0; k < K; ++k) {
            for (int h = 0; h < hn_total; ++h) {
                float x = 0.f, y = 0.f, r = 1.f;            /* :211-216  hyp zeros, ratio ones */
                if (tn > 0) {
                    int32_t t0, t1;
                    if (idxs) {
                        t0 = idxs[(((size_t)b * hn_total + h) * K + k) * 2];
                        t1 = idxs[(((size_t)b * hn_total + h) * K + k) * 2 + 1];
                    } else {
                        philox_pair(seed, ORC_TAG_DIST_IDX, (uint32_t)(img_base + b), (uint32_t)k, (uint32_t)h,
                                    (uint32_t)tn, &t0, &t1);
                    }
                    hyp_one(dirs[((size_t)t0 * K + k) * 2], dirs[((size_t)t0 * K + k) * 2 + 1],
                            (float)(pix[t0] % W), (float)(pix[t0] / W),
                            dirs[((size_t)t1 * K + k) * 2], dirs[((size_t)t1 * K + k) * 2 + 1],
                            (float)(pix[t1] % W), (float)(pix[t1] / W), &x, &y);
                    int32_t c = 0;
                    for (int t = 0; t < tn; ++t)
                        c += vote_one(dirs[((size_t)t * K + k) * 2], dirs[((size_t)t * K + k) * 2 + 1],
                                      (float)(pix[t] % W), (float)(pix[t] / W), x, y, thresh);
                    r = (float)c / (float)tn;               /* :243-244 */
                } else if (tn == 0) {
                    r = 0.f / 0.f;                           /* count 0 / foreground 0 (degenerate) */
                }
                hyp[h * 2] = x; hyp[h * 2 + 1] = y; ratio[h] = r;
                if (hyp_out) { hyp_out[(((size_t)b * K + k) * hn_total + h) * 2] = x;
                               hyp_out[(((size_t)b * K + k) * hn_total + h) * 2 + 1] = y; }
                if (ratio_out) ratio_out[((size_t)b * K + k) * hn_total + h] = r;
            }
            /* :259-269 */
            float mx = ratio[0];
            for (int h = 1; h < hn_total; ++h) if (ratio[h] > mx) mx = ratio[h];
            float th = mx - 0.1f;
            double s00 = 0, s01 = 0, s11 = 0, sw = 0;
            float mx_ = mean[((size_t)b * K + k) * 2], my_ = mean[((size_t)b * K + k) * 2 + 1];
            for (int h = 0; h < hn_total; ++h) {
                float w = ratio[h];
                if (w < th) w = 0.f;
                float ddx = hyp[h * 2] - mx_, ddy = hyp[h * 2 + 1] - my_;
                s00 += (double)ddx * ((double)ddx * w);
                s01 += (double)ddx * ((double)ddy * w);
                s11 += (double)ddy * ((double)ddy * w);
                sw += w;
            }
            float den = (float)sw + 1e-3f;
            float *c = cov + ((size_t)b * K + k) * 4;
            c[0] = (float)(s00 / den); c[1] = (float)(s01 / den);
            c[2] = (float)(s01 / den); c[3] = (float)(s11 / den);
        }
    }
    free(pix); free(dirs); free(hyp); free(ratio);
    return 0;
}
