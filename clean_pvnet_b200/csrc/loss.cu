// loss.cu -- PVNet's vote loss and its gradient from the mask and the keypoints, without the dense target field
// (DESIGN.md section 8e).
//
// The target of pixel (x, y) and keypoint k is clean-pvnet's compute_vertex (lib/utils/pvnet/pvnet_data_utils.py:30-44)
// bit for bit: where mask == 1,
//   d = kpt - (x, y) in fp64;  n = sqrt(RN(dx*dx) + RN(dy*dy));  n < 1e-3 -> n = RN(n + 1e-3);  (dx / n, dy / n) -> fp32
// and 0 elsewhere.  np.linalg.norm is that sqrt, not hypot.  Channel 2k is the x component of keypoint k, 2k + 1 its y.
// vote_target() is the only place that formula lives; all three kernels call it.
//
// The loss is the trainer's expression (lib/train/trainers/pvnet.py:25-27), with w = float(mask):
//   smooth_l1(pred * w, tgt * w, reduction='sum') / w.sum() / 2K
// per element x = RN(RN(p*w) - RN(t*w)), term 0.5 x^2 if |x| < 1 else |x| - 0.5.  The terms are added in fp64 as one
// partial per CTA; vote_loss_final_kernel adds the partials in a fixed order, so the loss is reproducible bit for bit.
// The divisions are CUDA torch's: `/ w.sum()` is an IEEE division by the fp32 weight sum, `/ 2K` (a Python int) is a
// multiplication by RN(1 / 2K), which is how torch divides a CUDA tensor by a CPU scalar.  The backward pass repeats
// autograd's chain:  g2 = RN(RN(g * RN(1/2K)) / wsum);  gin = -g2 if x < -1, g2 if x > 1, else RN(x * g2);  grad = RN(gin*w).
// Every operation is an explicit round-to-nearest intrinsic, so nvcc contracts nothing into an FMA.
#include "common.cuh"
#include "kernels.h"

namespace pvb {

constexpr int VL_THREADS = 256;     // one thread per pixel, consecutive pixels of a row on consecutive lanes

// compute_vertex's vector for keypoint (kx, ky) at column x, row y of a mask == 1 pixel
__device__ __forceinline__ float2 vote_target(double2 kp, int x, int y)
{
    const double dx = __dadd_rn(kp.x, -(double)x), dy = __dadd_rn(kp.y, -(double)y);
    double n = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
    if (n < 1e-3) n = __dadd_rn(n, 1e-3);
    return make_float2(__double2float_rn(__ddiv_rn(dx, n)), __double2float_rn(__ddiv_rn(dy, n)));
}

// x = pred * w - tgt * w, each product rounded on its own (the trainer's two multiplies, then smooth_l1's subtraction)
__device__ __forceinline__ float vote_diff(float p, float t, float w) { return __fsub_rn(__fmul_rn(p, w), __fmul_rn(t, w)); }

// smooth_l1 (beta = 1) of one element, exact in fp64 (x^2 of an fp32 x fits a double)
__device__ __forceinline__ double vote_term(float x)
{
    const float ax = fabsf(x);
    return ax < 1.f ? __dmul_rn(0.5, __dmul_rn((double)x, (double)x)) : __dadd_rn((double)ax, -0.5);
}

// the pixel a thread owns, its mask value and the image's keypoints staged in shared memory
template <typename T>
struct VotePixel {
    int b, p, x, y;
    bool valid;
    T m;
};

template <typename T>
__device__ __forceinline__ VotePixel<T> vote_pixel(const VoteLossArgs &a, double2 *s_kpt)
{
    VotePixel<T> px;
    px.b = blockIdx.y;
    for (int k = threadIdx.x; k < a.K; k += blockDim.x)
        s_kpt[k] = make_double2(a.kpt[((size_t)px.b * a.K + k) * 2], a.kpt[((size_t)px.b * a.K + k) * 2 + 1]);
    __syncthreads();
    const int HW = a.H * a.W;
    px.p = blockIdx.x * VL_THREADS + (int)threadIdx.x;
    px.valid = px.p < HW;
    px.y = px.valid ? px.p / a.W : 0;
    px.x = px.valid ? px.p - px.y * a.W : 0;
    px.m = px.valid ? __ldg(static_cast<const T *>(a.mask) + px.b * a.msb + px.y * a.msy + px.x * a.msx) : T(0);
    return px;
}

// compute_vertex on the device: vertex [B][2K][H][W] contiguous
template <typename T>
__global__ void __launch_bounds__(VL_THREADS) vote_target_kernel(VoteLossArgs a)
{
    extern __shared__ double2 s_kpt[];
    const VotePixel<T> px = vote_pixel<T>(a, s_kpt);
    if (!px.valid) return;
    const bool on = (long long)px.m == 1;
    const size_t HW = (size_t)a.H * a.W;
    float *out = a.out + (size_t)px.b * 2 * a.K * HW + px.p;
    for (int k = 0; k < a.K; ++k) {
        const float2 t = on ? vote_target(s_kpt[k], px.x, px.y) : make_float2(0.f, 0.f);
        out[(size_t)(2 * k) * HW] = t.x;
        out[(size_t)(2 * k + 1) * HW] = t.y;
    }
}

// the CTA's sum of the smooth-l1 terms (fp64) and of the mask values (int64), in a fixed order -> partial[cta], wpart[cta]
template <typename T>
__global__ void __launch_bounds__(VL_THREADS) vote_loss_fwd_kernel(VoteLossArgs a)
{
    extern __shared__ double2 s_kpt[];
    __shared__ double s_s[VL_THREADS / 32];
    __shared__ long long s_w[VL_THREADS / 32];
    const VotePixel<T> px = vote_pixel<T>(a, s_kpt);
    double s = 0.0;
    long long wc = 0;
    if (px.valid) {
        const float w = (float)px.m;                         // .float()
        const bool on = (long long)px.m == 1;
        wc = (long long)px.m;
        const float *pp = a.pred + px.b * a.ps[0] + px.y * a.ps[2] + px.x * a.ps[3];
        for (int k = 0; k < a.K; ++k) {
            // every pixel reads pred: a NaN or inf prediction outside the mask makes the sum NaN (inf * 0), as in torch
            const float2 t = on ? vote_target(s_kpt[k], px.x, px.y) : make_float2(0.f, 0.f);
            s += vote_term(vote_diff(__ldg(pp + (2 * k) * a.ps[1]), t.x, w));
            s += vote_term(vote_diff(__ldg(pp + (2 * k + 1) * a.ps[1]), t.y, w));
        }
    }
    s = warp_sum(s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wc += __shfl_xor_sync(0xffffffffu, wc, o);
    if ((threadIdx.x & 31) == 0) { s_s[threadIdx.x >> 5] = s; s_w[threadIdx.x >> 5] = wc; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; wc = 0;
#pragma unroll
        for (int i = 0; i < VL_THREADS / 32; ++i) { s += s_s[i]; wc += s_w[i]; }
        const size_t cta = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
        a.partial[cta] = s;
        a.wpart[cta] = wc;
    }
}

// one CTA: the partials in a fixed order, then loss = RN(RN(float(S) / wsum) * RN(1 / 2K)); wsum stays for backward
constexpr int VL_FINAL_THREADS = 1024;
__global__ void __launch_bounds__(VL_FINAL_THREADS) vote_loss_final_kernel(const double *partial, const long long *wpart,
                                                                          long long nparts, int K, float *wsum, float *loss)
{
    __shared__ double s_s[VL_FINAL_THREADS / 32];
    __shared__ long long s_w[VL_FINAL_THREADS / 32];
    double s = 0.0;
    long long wc = 0;
    for (long long i = threadIdx.x; i < nparts; i += VL_FINAL_THREADS) { s += partial[i]; wc += wpart[i]; }
    s = warp_sum(s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wc += __shfl_xor_sync(0xffffffffu, wc, o);
    if ((threadIdx.x & 31) == 0) { s_s[threadIdx.x >> 5] = s; s_w[threadIdx.x >> 5] = wc; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; wc = 0;
        for (int i = 0; i < VL_FINAL_THREADS / 32; ++i) { s += s_s[i]; wc += s_w[i]; }
        const float ws = __ll2float_rn(wc);
        *wsum = ws;
        *loss = __fmul_rn(__fdiv_rn(__double2float_rn(s), ws), __fdiv_rn(1.f, (float)(2 * K)));
    }
}

// grad [B][2K][H][W] contiguous from the scalar upstream gradient and the forward pass's wsum
template <typename T>
__global__ void __launch_bounds__(VL_THREADS) vote_loss_bwd_kernel(VoteLossArgs a)
{
    extern __shared__ double2 s_kpt[];
    const VotePixel<T> px = vote_pixel<T>(a, s_kpt);
    if (!px.valid) return;
    const float g2 = __fdiv_rn(__fmul_rn(*a.grad_loss, __fdiv_rn(1.f, (float)(2 * a.K))), *a.wsum);
    const float w = (float)px.m;
    const bool on = (long long)px.m == 1;
    const size_t HW = (size_t)a.H * a.W;
    const float *pp = a.pred + px.b * a.ps[0] + px.y * a.ps[2] + px.x * a.ps[3];
    float *out = a.out + (size_t)px.b * 2 * a.K * HW + px.p;
    for (int k = 0; k < a.K; ++k) {
        const float2 t = on ? vote_target(s_kpt[k], px.x, px.y) : make_float2(0.f, 0.f);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const float x = vote_diff(__ldg(pp + (2 * k + c) * a.ps[1]), c ? t.y : t.x, w);
            const float gin = x < -1.f ? -g2 : (x > 1.f ? g2 : __fmul_rn(x, g2));   // smooth_l1_backward, NaN -> NaN
            out[(size_t)(2 * k + c) * HW] = __fmul_rn(gin, w);
        }
    }
}

size_t vote_loss_workspace_bytes(int B, int H, int W, size_t *partial_offset, size_t *wpart_offset)
{
    const size_t nparts = (size_t)B * (((size_t)H * W + VL_THREADS - 1) / VL_THREADS);
    const size_t po = 256, wo = po + (nparts * sizeof(double) + 255) / 256 * 256;
    if (partial_offset) *partial_offset = po;
    if (wpart_offset) *wpart_offset = wo;
    return wo + (nparts * sizeof(long long) + 255) / 256 * 256;
}

namespace {

enum class VoteOp { Target, Forward, Backward };

template <typename T>
cudaError_t launch_typed(VoteOp op, const VoteLossArgs &a, cudaStream_t st)
{
    const dim3 grid((unsigned)(((long long)a.H * a.W + VL_THREADS - 1) / VL_THREADS), (unsigned)a.B);
    const size_t smem = (size_t)a.K * sizeof(double2);
    switch (op) {
    case VoteOp::Target: vote_target_kernel<T><<<grid, VL_THREADS, smem, st>>>(a); break;
    case VoteOp::Forward: vote_loss_fwd_kernel<T><<<grid, VL_THREADS, smem, st>>>(a); break;
    case VoteOp::Backward: vote_loss_bwd_kernel<T><<<grid, VL_THREADS, smem, st>>>(a); break;
    }
    return cudaGetLastError();
}

cudaError_t launch_vote_op(VoteOp op, const VoteLossArgs &a, cudaStream_t st)
{
    if ((long long)a.B * a.H * a.W == 0) return cudaSuccess;
    switch (a.mask_dtype) {
    case PVB_MASK_U8: return launch_typed<uint8_t>(op, a, st);
    case PVB_MASK_I8: return launch_typed<int8_t>(op, a, st);
    case PVB_MASK_I16: return launch_typed<int16_t>(op, a, st);
    case PVB_MASK_I32: return launch_typed<int32_t>(op, a, st);
    case PVB_MASK_I64: return launch_typed<long long>(op, a, st);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace

cudaError_t launch_vote_target(const VoteLossArgs &a, cudaStream_t st) { return launch_vote_op(VoteOp::Target, a, st); }

cudaError_t launch_vote_loss_forward(const VoteLossArgs &a, cudaStream_t st)
{
    cudaError_t e = launch_vote_op(VoteOp::Forward, a, st);
    if (e != cudaSuccess) return e;
    const long long nparts = (long long)a.B * (((long long)a.H * a.W + VL_THREADS - 1) / VL_THREADS);
    vote_loss_final_kernel<<<1, VL_FINAL_THREADS, 0, st>>>(a.partial, a.wpart, nparts, a.K, a.wsum, a.loss);
    return cudaGetLastError();
}

cudaError_t launch_vote_loss_backward(const VoteLossArgs &a, cudaStream_t st) { return launch_vote_op(VoteOp::Backward, a, st); }

} // namespace pvb
