// crop.cu -- T-LESS's PVNet crop on the device (DESIGN.md section 8g): the crop of tless_test_utils.pvnet_transform
// (lib/utils/tless/tless_test_utils.py:57-77) and of the detector->PVNet cascade's _crop (lib/networks/ct_pvnet/res.py:
// 14-31) for n boxes, cv2.warpAffine(INTER_LINEAR) for n (image, matrix) rows, and the evaluator's un-crop of keypoints
// (lib/evaluators/tless_test/pvnet.py:229-239).
//
// Crop matrix (one thread per box): data_utils.get_affine_transform(center, scale, 0, [w, h]) under numpy 2's
// promotions -- scale rounded to fp32, src[1] = fp32(center + (0, fp32(scale * -0.5))) formed in fp64, the third points
// in fp32 -- then cv2.getAffineTransform's 6x6 system solved as OpenCV's LU does: partial pivoting on |a| (strictly
// greater), elimination with d = -1/pivot, back-substitution by division, all zeros when a pivot is below
// 100 * DBL_EPSILON (cv::solve's answer for a singular system).  Every operation is an explicit _rn intrinsic, so nothing
// contracts into an FMA.
//
// Warp (one CTA per (box, output row)): cv2.warpAffine's fixed-point bilinear.  The forward matrix is inverted as
// warpAffine inverts it (D = 1/(m0 m4 - m1 m3), 0 when singular); row offsets (m1 y + m2) * 1024 and column offsets
// m0 x * 1024 are rounded half to even to int (cvRound, whose out-of-range result is INT_MIN), summed with 16, shifted by
// 5 into 5-bit sub-pixel positions, and the four taps are weighted by 15-bit integer weights with a zero border.  The
// sum is integer arithmetic, so the output byte is exact in any order.  The crop then zeroes what lies outside the
// magnified box (magnify_box of the box corners through the matrix) and normalises (u8 / 255 - mean) / std in fp32,
// writing NCHW, and optionally the uint8 HWC crop.  No intermediate image exists.
#include <cmath>
#include "api.h"

namespace pvb {

// Setup: one thread per box -> centre, scale, forward (and inverse) crop matrix.
struct CropArgs {
    const double *boxes;          // [n][4] xyxy, image coordinates
    int n, out_w, out_h, center_f64;  // center_f64: the cascade's fp64 centre, else pvnet_transform's fp32 one
    double scale_ratio;
    double *center, *scale;       // [n][2], [n]: as the reference computes them (fp64)
    double *M, *Minv;             // [n][6] forward crop matrix; inverse (inv=1) or NULL
};
// Warp: one CTA per (box, output row) over [n][out_h]; the crop variant masks, normalises and writes NCHW fp32.
struct WarpArgs {
    const unsigned char *img;     // [B][H][W][C] at element strides sb, sh, sw, sc
    long long sb, sh, sw, sc;
    int B, H, W, C;
    const double *M;              // [n][6] forward matrices (warpAffine inverts them)
    const int *image_index;       // [n] or NULL (every row reads image 0)
    int n, out_w, out_h;
    const double *boxes;          // crop: [n][4], for the box mask
    int mask;                     // crop: zero what lies outside the magnified box
    double box_ratio;
    float mean[3], stdv[3];       // crop: normalisation
    float *inp;                   // crop: [n][3][out_h][out_w]
    unsigned char *out_u8;        // [n][out_h][out_w][C]: the warp's output; optional for the crop
};
struct UncropArgs {
    const float *kpt;             // [n][K][2], crop frame
    const double *center, *scale; // [n][2], [n]
    int n, K, in_w, in_h;
    double *out;                  // [n][K][2], image frame
};

namespace {

constexpr int CROP_SETUP_THREADS = 128;
constexpr int WARP_THREADS = 128;
constexpr double LU_EPS = 2.220446049250313e-16 * 100;   // hal::LU64f: DBL_EPSILON * 100

// cvRound(v) as saturate_cast<int>(double) computes it on x86-64: half to even, INT_MIN when the result does not fit
__device__ __forceinline__ int cv_round(double v)
{
    return (v >= -2147483648.5 && v < 2147483647.5) ? __double2int_rn(v) : INT_MIN;
}

// cv::getAffineTransform(src, dst) -> M[6]
__device__ __forceinline__ void get_affine(const float sx[3], const float sy[3], const float dx[3], const float dy[3],
                                           double M[6])
{
    double A[6][6], b[6];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double x = sx[i], y = sy[i];
        A[2 * i][0] = x;   A[2 * i][1] = y;   A[2 * i][2] = 1.0; A[2 * i][3] = 0.0; A[2 * i][4] = 0.0; A[2 * i][5] = 0.0;
        A[2 * i + 1][0] = 0.0; A[2 * i + 1][1] = 0.0; A[2 * i + 1][2] = 0.0;
        A[2 * i + 1][3] = x;   A[2 * i + 1][4] = y;   A[2 * i + 1][5] = 1.0;
        b[2 * i] = dx[i];
        b[2 * i + 1] = dy[i];
    }
    bool singular = false;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        int k = i;
        double best = fabs(A[i][i]);
#pragma unroll
        for (int j = i + 1; j < 6; ++j)
            if (fabs(A[j][i]) > best) { best = fabs(A[j][i]); k = j; }
        singular |= best < LU_EPS;
#pragma unroll
        for (int j = i + 1; j < 6; ++j)          // swap rows i and k, columns i.. (static indices: stays in registers)
            if (k == j) {
#pragma unroll
                for (int c = i; c < 6; ++c) { const double t = A[i][c]; A[i][c] = A[j][c]; A[j][c] = t; }
                const double t = b[i]; b[i] = b[j]; b[j] = t;
            }
        const double d = __ddiv_rn(-1.0, A[i][i]);
#pragma unroll
        for (int j = i + 1; j < 6; ++j) {
            const double alpha = __dmul_rn(A[j][i], d);
#pragma unroll
            for (int c = i + 1; c < 6; ++c) A[j][c] = __dadd_rn(A[j][c], __dmul_rn(alpha, A[i][c]));
            b[j] = __dadd_rn(b[j], __dmul_rn(alpha, b[i]));
        }
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double s = b[i];
#pragma unroll
        for (int c = i + 1; c < 6; ++c) s = __dsub_rn(s, __dmul_rn(A[i][c], b[c]));
        b[i] = __ddiv_rn(s, A[i][i]);
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) M[i] = singular ? 0.0 : b[i];
}

// get_affine_transform(center, scale, 0, [ow, oh], inv): center in fp64 (a float32 centre is exact in it)
__device__ __forceinline__ void crop_matrix(double cx, double cy, float scale, int ow, int oh, bool inv, double M[6])
{
    const float v = __fmul_rn(scale, -0.5f);
    float sx[3], sy[3], dx[3], dy[3];
    sx[0] = __double2float_rn(cx);
    sy[0] = __double2float_rn(cy);
    sx[1] = __double2float_rn(__dadd_rn(cx, 0.0));
    sy[1] = __double2float_rn(__dadd_rn(cy, (double)v));
    dx[0] = (float)(ow * 0.5);
    dy[0] = (float)(oh * 0.5);
    dx[1] = dx[0];
    dy[1] = __fadd_rn(dy[0], (float)(ow * -0.5));
    // get_3rd_point(a, b) = b + (-(a.y - b.y), a.x - b.x), in fp32
    sx[2] = __fadd_rn(sx[1], -__fsub_rn(sy[0], sy[1]));
    sy[2] = __fadd_rn(sy[1], __fsub_rn(sx[0], sx[1]));
    dx[2] = __fadd_rn(dx[1], -__fsub_rn(dy[0], dy[1]));
    dy[2] = __fadd_rn(dy[1], __fsub_rn(dx[0], dx[1]));
    if (inv) get_affine(dx, dy, sx, sy, M);
    else get_affine(sx, sy, dx, dy, M);
}

// data_utils.affine_transform's np.dot(pt, M[:, :2].T) + M[:, 2]: x * m0 rounded, y * m1 fused into it (OpenBLAS dgemm)
__device__ __forceinline__ double affine_row(double x, double y, double m0, double m1, double m2)
{
    return __dadd_rn(__fma_rn(y, m1, __dmul_rn(x, m0)), m2);
}

__global__ void __launch_bounds__(CROP_SETUP_THREADS) crop_setup_kernel(const CropArgs a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const double *bx = a.boxes + 4 * (long long)i;
    double cx = __dmul_rn(__dadd_rn(bx[0], bx[2]), 0.5), cy = __dmul_rn(__dadd_rn(bx[1], bx[3]), 0.5);
    if (!a.center_f64) { cx = (double)__double2float_rn(cx); cy = (double)__double2float_rn(cy); }
    const double w = __dsub_rn(bx[2], bx[0]), h = __dsub_rn(bx[3], bx[1]);
    const double s = __dmul_rn(h > w ? h : w, a.scale_ratio);        // Python's max(w, h) keeps w unless h > w
    a.center[2 * i] = cx;
    a.center[2 * i + 1] = cy;
    a.scale[i] = s;
    double M[6];
    crop_matrix(cx, cy, __double2float_rn(s), a.out_w, a.out_h, false, M);
#pragma unroll
    for (int k = 0; k < 6; ++k) a.M[6 * (long long)i + k] = M[k];
    if (a.Minv) {
        crop_matrix(cx, cy, __double2float_rn(s), a.out_w, a.out_h, true, M);
#pragma unroll
        for (int k = 0; k < 6; ++k) a.Minv[6 * (long long)i + k] = M[k];
    }
}

template <bool CROP>
__global__ void __launch_bounds__(WARP_THREADS) warp_kernel(const WarpArgs a)
{
    const int box = blockIdx.x / a.out_h, row = blockIdx.x - box * a.out_h;
    const double *Mf = a.M + 6 * (long long)box;
    const double f0 = Mf[0], f1 = Mf[1], f2 = Mf[2], f3 = Mf[3], f4 = Mf[4], f5 = Mf[5];
    // warpAffine's inversion of the forward matrix
    double D = __dsub_rn(__dmul_rn(f0, f4), __dmul_rn(f1, f3));
    D = D != 0.0 ? __ddiv_rn(1.0, D) : 0.0;
    const double m0 = __dmul_rn(f4, D), m1 = __dmul_rn(f1, -D), m3 = __dmul_rn(f3, -D), m4 = __dmul_rn(f0, D);
    const double m2 = __dsub_rn(__dmul_rn(-m0, f2), __dmul_rn(m1, f5));
    const double m5 = __dsub_rn(__dmul_rn(-m3, f2), __dmul_rn(m4, f5));
    const int X0 = (int)((unsigned)cv_round(__dmul_rn(__dadd_rn(__dmul_rn(m1, (double)row), m2), 1024.0)) + 16u);
    const int Y0 = (int)((unsigned)cv_round(__dmul_rn(__dadd_rn(__dmul_rn(m4, (double)row), m5), 1024.0)) + 16u);

    const int b = a.image_index ? a.image_index[box] : 0;
    const bool have_img = b >= 0 && b < a.B;                  // an index outside [0, B) reads as an all-border image
    const unsigned char *src = a.img + (have_img ? (long long)b * a.sb : 0);

    // magnify_box: the box corners through the forward matrix, scaled about their mean, rounded, clipped to the crop
    int kx0 = 0, ky0 = 0, kx1 = a.out_w - 1, ky1 = a.out_h - 1;
    if (CROP && a.mask) {
        const double *bx = a.boxes + 4 * (long long)box;
        const double px0 = affine_row(bx[0], bx[1], f0, f1, f2), py0 = affine_row(bx[0], bx[1], f3, f4, f5);
        const double px1 = affine_row(bx[2], bx[3], f0, f1, f2), py1 = affine_row(bx[2], bx[3], f3, f4, f5);
        const double mx = __dmul_rn(__dadd_rn(px0, px1), 0.5), my = __dmul_rn(__dadd_rn(py0, py1), 0.5);
        auto mag = [&](double p, double m, int hi) {
            const double r = rint(__dadd_rn(__dmul_rn(__dsub_rn(p, m), a.box_ratio), m));
            const int q = (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;   // astype(int32)
            return q < 0 ? 0 : (q > hi ? hi : q);
        };
        kx0 = mag(px0, mx, a.out_w - 1); ky0 = mag(py0, my, a.out_h - 1);
        kx1 = mag(px1, mx, a.out_w - 1); ky1 = mag(py1, my, a.out_h - 1);
    }
    const bool row_kept = row >= ky0 && row <= ky1;
    const long long plane = (long long)a.out_h * a.out_w;

    for (int x = threadIdx.x; x < a.out_w; x += WARP_THREADS) {
        const int ad = cv_round(__dmul_rn(__dmul_rn(m0, (double)x), 1024.0));
        const int bd = cv_round(__dmul_rn(__dmul_rn(m3, (double)x), 1024.0));
        const int X = (int)((unsigned)X0 + (unsigned)ad) >> 5, Y = (int)((unsigned)Y0 + (unsigned)bd) >> 5;
        const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
        const int w[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
        const bool inx0 = sx >= 0 && sx < a.W, inx1 = sx + 1 >= 0 && sx + 1 < a.W;
        const bool iny0 = sy >= 0 && sy < a.H, iny1 = sy + 1 >= 0 && sy + 1 < a.H;
        const bool in[4] = {have_img && iny0 && inx0, have_img && iny0 && inx1, have_img && iny1 && inx0,
                            have_img && iny1 && inx1};
        const long long off[4] = {sy * a.sh + sx * a.sw, sy * a.sh + (sx + 1) * a.sw, (sy + 1) * a.sh + sx * a.sw,
                                  (sy + 1) * a.sh + (sx + 1) * a.sw};
        const bool kept = !CROP || (row_kept && x >= kx0 && x <= kx1);
        const long long px = (long long)row * a.out_w + x, o = (long long)box * plane + px;
        for (int c = 0; c < a.C; ++c) {
            int acc = 0;
#pragma unroll
            for (int t = 0; t < 4; ++t)
                if (in[t]) acc += w[t] * (int)__ldg(src + off[t] + c * a.sc);
            const int v = kept ? (acc + (1 << 14)) >> 15 : 0;
            if (CROP) {
                const float f = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.0f), a.mean[c]), a.stdv[c]);
                a.inp[((long long)box * 3 + c) * plane + px] = f;                      // NCHW
                if (a.out_u8) a.out_u8[o * 3 + c] = (unsigned char)v;
            } else {
                a.out_u8[o * a.C + c] = (unsigned char)v;
            }
        }
    }
}

__global__ void __launch_bounds__(CROP_SETUP_THREADS) uncrop_kernel(const UncropArgs a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    double M[6];
    crop_matrix(a.center[2 * i], a.center[2 * i + 1], __double2float_rn(a.scale[i]), a.in_w, a.in_h, true, M);
    const float *k = a.kpt + 2 * (long long)i * a.K;
    double *o = a.out + 2 * (long long)i * a.K;
    for (int j = 0; j < a.K; ++j) {
        const double x = k[2 * j], y = k[2 * j + 1];
        o[2 * j] = affine_row(x, y, M[0], M[1], M[2]);
        o[2 * j + 1] = affine_row(x, y, M[3], M[4], M[5]);
    }
}

} // namespace

// External linkage on purpose: nvcc names this file's anonymous namespace, and so its kernels, after the first
// externally visible definition in the file.
cudaError_t launch_crop_setup(const CropArgs &a, cudaStream_t st)
{
    crop_setup_kernel<<<(unsigned)((a.n + CROP_SETUP_THREADS - 1) / CROP_SETUP_THREADS), CROP_SETUP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

namespace {

cudaError_t launch_warp(const WarpArgs &a, bool crop, cudaStream_t st)
{
    const unsigned grid = (unsigned)((long long)a.n * a.out_h);
    if (crop) warp_kernel<true><<<grid, WARP_THREADS, 0, st>>>(a);
    else warp_kernel<false><<<grid, WARP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

// the image and output arguments the crop and the warp share; fills the image and size fields of `a`
int warp_common(WarpArgs &a, const uint8_t *img, int32_t B, int32_t H, int32_t W, int32_t C, const int64_t *img_stride,
                int32_t n, int32_t out_w, int32_t out_h)
{
    if (n < 0 || B < 0) return fail(PVB_ERR_INVALID, "negative size (n=%d B=%d)", n, B);
    if (H < 1 || W < 1 || H > 32767 || W > 32767) return fail(PVB_ERR_INVALID, "image must be 1..32767 pixels a side (got %dx%d)", W, H);
    if (C < 1 || C > 4) return fail(PVB_ERR_INVALID, "C must be in [1,4] (got %d)", C);
    if (out_w < 1 || out_h < 1) return fail(PVB_ERR_INVALID, "output size must be >= 1 (got %dx%d)", out_w, out_h);
    if ((long long)n * out_h > 0x7fffffffll) return fail(PVB_ERR_INVALID, "n * out_h too large (>= 2^31)");
    if (!img_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    for (int i = 0; i < 4; ++i)
        if (img_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
    if (n > 0 && B > 0 && !img) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.img = img; a.sb = img_stride[0]; a.sh = img_stride[1]; a.sw = img_stride[2]; a.sc = img_stride[3];
    a.B = B; a.H = H; a.W = W; a.C = C; a.n = n; a.out_w = out_w; a.out_h = out_h;
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_crop_inputs(const uint8_t *img, int32_t B, int32_t H, int32_t W, const int64_t *img_stride,
                            const double *boxes, const int32_t *image_index, int32_t n, int32_t out_w, int32_t out_h,
                            double scale_ratio, double box_ratio, int32_t flags, const float *mean, const float *std,
                            float *inp, uint8_t *crop_u8, double *center, double *scale, double *matrix,
                            double *matrix_inv, pvb_stream_t stream)
{
    WarpArgs w = {};
    if (int rc = warp_common(w, img, B, H, W, 3, img_stride, n, out_w, out_h)) return rc;
    if (!std::isfinite(scale_ratio) || !std::isfinite(box_ratio))
        return fail(PVB_ERR_INVALID, "scale_ratio and box_ratio must be finite (got %g, %g)", scale_ratio, box_ratio);
    if (box_ratio < 0) return fail(PVB_ERR_INVALID, "box_ratio must be >= 0 (got %g)", box_ratio);
    if (flags & ~(PVB_CROP_MASK_TO_BOX | PVB_CROP_CENTER_F64)) return fail(PVB_ERR_INVALID, "unknown flags 0x%x", flags);
    if (!mean || !std) return fail(PVB_ERR_INVALID, "NULL mean / std");
    for (int c = 0; c < 3; ++c)
        if (!(std[c] != 0.0f) || !std::isfinite(mean[c])) return fail(PVB_ERR_INVALID, "std must be non-zero and mean finite");
    if (!img || !boxes || !inp || !center || !scale || !matrix) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (n == 0) return PVB_OK;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    CropArgs c;
    c.boxes = boxes; c.n = n; c.out_w = out_w; c.out_h = out_h; c.center_f64 = (flags & PVB_CROP_CENTER_F64) != 0;
    c.scale_ratio = scale_ratio; c.center = center; c.scale = scale; c.M = matrix; c.Minv = matrix_inv;
    cudaError_t e = launch_crop_setup(c, st);
    if (e != cudaSuccess) return cuda_fail(e, "crop setup kernel");
    w.M = matrix; w.image_index = image_index; w.boxes = boxes; w.mask = (flags & PVB_CROP_MASK_TO_BOX) != 0;
    w.box_ratio = box_ratio; w.inp = inp; w.out_u8 = crop_u8;
    for (int k = 0; k < 3; ++k) { w.mean[k] = mean[k]; w.stdv[k] = std[k]; }
    e = launch_warp(w, true, st);
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "crop warp kernel");
}

PVB_API int pvb_uncrop_keypoints(const float *kpt_2d, const double *center, const double *scale, int32_t n, int32_t K,
                                 int32_t in_w, int32_t in_h, double *out, pvb_stream_t stream)
{
    if (n < 0 || K < 0) return fail(PVB_ERR_INVALID, "negative size (n=%d K=%d)", n, K);
    if (in_w < 1 || in_h < 1) return fail(PVB_ERR_INVALID, "input size must be >= 1 (got %dx%d)", in_w, in_h);
    if (n == 0 || K == 0) return PVB_OK;
    if (!kpt_2d || !center || !scale || !out) return fail(PVB_ERR_INVALID, "NULL tensor");
    UncropArgs a;
    a.kpt = kpt_2d; a.center = center; a.scale = scale; a.n = n; a.K = K; a.in_w = in_w; a.in_h = in_h; a.out = out;
    uncrop_kernel<<<(unsigned)((n + CROP_SETUP_THREADS - 1) / CROP_SETUP_THREADS), CROP_SETUP_THREADS, 0,
                    static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "uncrop kernel");
}

PVB_API int pvb_warp_affine_linear(const uint8_t *img, int32_t B, int32_t H, int32_t W, int32_t C, const int64_t *img_stride,
                                   const double *M, const int32_t *image_index, int32_t n, int32_t out_w, int32_t out_h,
                                   uint8_t *out, pvb_stream_t stream)
{
    WarpArgs w = {};
    if (int rc = warp_common(w, img, B, H, W, C, img_stride, n, out_w, out_h)) return rc;
    if (n == 0) return PVB_OK;
    if (!img || !M || !out) return fail(PVB_ERR_INVALID, "NULL tensor");
    w.M = M; w.image_index = image_index; w.out_u8 = out;
    cudaError_t e = launch_warp(w, false, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "warp kernel");
}

} // extern "C"
