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
#include "kernels.h"

namespace pvb {
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

cudaError_t launch_crop_setup(const CropArgs &a, cudaStream_t st)
{
    crop_setup_kernel<<<(unsigned)((a.n + CROP_SETUP_THREADS - 1) / CROP_SETUP_THREADS), CROP_SETUP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_warp(const WarpArgs &a, bool crop, cudaStream_t st)
{
    const unsigned grid = (unsigned)((long long)a.n * a.out_h);
    if (crop) warp_kernel<true><<<grid, WARP_THREADS, 0, st>>>(a);
    else warp_kernel<false><<<grid, WARP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_uncrop(const UncropArgs &a, cudaStream_t st)
{
    uncrop_kernel<<<(unsigned)((a.n + CROP_SETUP_THREADS - 1) / CROP_SETUP_THREADS), CROP_SETUP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}

} // namespace pvb
