// Modulated deformable convolution (DCNv2), fp32 NCHW, forward and backward: the device twin of clean-pvnet's
// lib/csrc/dcn_v2 extension (dcn_v2_cuda.cu + dcn_v2_im2col_cuda.cu), which the DLA-34 CenterNet detector runs.
//
// The reference writes the whole column matrix cols[b][c*kh*kw + i*kw + j][ho*Wo + wo] (im2col) and multiplies it by
// the weight with batched SGEMM; its backward loops over the images.  Here the forward is one implicit-GEMM kernel
// whose B-operand tiles are sampled straight into shared memory, so the columns are never stored, and the backward runs
// the whole batch: grad_cols = W^T grad_out in image chunks (the only stored column matrix), one kernel for
// grad_offset + grad_mask, one for grad_input (float atomics, as the reference), grad_weight re-sampling the columns in
// split-K partials reduced in a fixed order, and a fixed-order grad_bias.  Everything but grad_input is bitwise
// reproducible.  All arithmetic is FP32 FFMA (no TF32, no tensor cores).
//
// The TF32 path (DESIGN.md section 8p), which the Python layer takes for fp32 inputs when torch allows TF32 matmuls,
// is a third forward kernel and TF32 twins of the backward's two products, grad_cols and grad_weight: the same sampler
// and tiles, each operand rounded once to TF32 (cvt.rna) and multiplied by mma.sync m16n8k8 with fp32 accumulation.
// The backward's other kernels, its plan and its workspace are shared.
//
// The half-precision forward (fp16 or bf16 operands, DESIGN.md section 8n) is a second implicit-GEMM kernel on the
// tensor cores: the same sampler, fed the up-cast inputs, fills bf16 / fp16 B tiles in shared memory; the weight
// tiles arrive by cp.async; mma.sync m16n8k16 accumulates in fp32.  Its NHWC (channels_last) twin (section 8o) shares
// that body and differs only in where it reads and writes, so its output is the NCHW kernel's bit for bit.  Neither
// has a backward of its own: the Python layer runs the fp32 backward on up-cast copies of the operands the forward used.
//
// A sample point of (pixel, tap, deformable group) has four corner offsets and four bilinear weights that do not depend
// on the channel: they are computed once per tile and reused over the group's channels.  The sampled value is the
// reference kernel's bit for bit: nvcc contracts its `w1*v1 + w2*v2 + w3*v3 + w4*v4` (dcn_v2_im2col_cuda.cu:52) into
// fma(w4,v4, fma(w3,v3, fma(w1,v1, w2*v2))) at sm_90a (read off the reference build's SASS), written out below with
// explicit intrinsics; the mask multiplies after the bilinear sum.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "api.h"

namespace pvb {

// Contiguous fp32 NCHW; shapes validated by dcn_args.
struct DcnArgs {
    const float *input;       // [B][C][H][W]
    const float *offset;      // [B][dg*2*kh*kw][Ho][Wo]
    const float *mask;        // [B][dg*kh*kw][Ho][Wo]
    const float *weight;      // [Co][C][kh][kw]
    const float *bias;        // [Co]
    float *out;               // [B][Co][Ho][Wo] (forward)
    const float *grad_out;    // [B][Co][Ho][Wo] (backward)
    float *grad_input, *grad_offset, *grad_mask, *grad_weight, *grad_bias;   // shaped like their inputs (backward)
    float *cols;              // grad_cols [chunk][C*kh*kw][Ho*Wo] (backward workspace)
    int B, C, H, W, Co, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
};

namespace {

constexpr int BM = 64, BN = 128, BK = 16, NT = 256;   // CTA tile (rows x columns x depth), threads
constexpr int GW_TARGET_CTAS = 528;                    // grad_weight: split the reduction until ~4 CTAs per H100 SM

// The sample point (h, w) of the reference (dcn_v2_im2col_cuda.cu:177-187): used only when h > -1, w > -1, h < H,
// w < W (so NaN gives 0); a corner counts only inside the image.  off = -1 marks a corner that reads as 0.
struct Corners { int off[4]; float wt[4]; };

__device__ __forceinline__ Corners sample_point(float h, float w, int H, int W)
{
    Corners s;
    if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
        const int hl = (int)floorf(h), wl = (int)floorf(w);
        const float lh = __fsub_rn(h, (float)hl), lw = __fsub_rn(w, (float)wl);
        const float hh = __fsub_rn(1.f, lh), hw = __fsub_rn(1.f, lw);
        s.wt[0] = __fmul_rn(hh, hw); s.wt[1] = __fmul_rn(hh, lw); s.wt[2] = __fmul_rn(lh, hw); s.wt[3] = __fmul_rn(lh, lw);
        s.off[0] = (hl >= 0 && wl >= 0) ? hl * W + wl : -1;
        s.off[1] = (hl >= 0 && wl + 1 <= W - 1) ? hl * W + wl + 1 : -1;
        s.off[2] = (hl + 1 <= H - 1 && wl >= 0) ? (hl + 1) * W + wl : -1;
        s.off[3] = (hl + 1 <= H - 1 && wl + 1 <= W - 1) ? (hl + 1) * W + wl + 1 : -1;
    } else {
        for (int q = 0; q < 4; ++q) { s.off[q] = -1; s.wt[q] = 0.f; }
    }
    return s;
}

// one element read as fp32: fp16 and bf16 up-cast exactly, so the sampler sees the value the fp32 path would
__device__ __forceinline__ float ld_f32(const float *p) { return __ldg(p); }
__device__ __forceinline__ float ld_f32(const __half *p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float ld_f32(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

// the bilinear sum of the four corner values v1..v4 (0 for a corner outside the image), in the reference's order
__device__ __forceinline__ float blend(const float wt[4], float v1, float v2, float v3, float v4)
{
    return __fmaf_rn(wt[3], v4, __fmaf_rn(wt[2], v3, __fmaf_rn(wt[0], v1, __fmul_rn(wt[1], v2))));
}

template <typename T>
__device__ __forceinline__ float bilinear(const T *plane, const int off[4], const float wt[4])
{
    const float v1 = off[0] >= 0 ? ld_f32(plane + off[0]) : 0.f;
    const float v2 = off[1] >= 0 ? ld_f32(plane + off[1]) : 0.f;
    const float v3 = off[2] >= 0 ? ld_f32(plane + off[2]) : 0.f;
    const float v4 = off[3] >= 0 ? ld_f32(plane + off[3]) : 0.f;
    return blend(wt, v1, v2, v3, v4);
}

// the sample coordinate of output pixel p at tap (i, j): float(ho*s - p + i*d) + offset, rounded once
template <typename T>
__device__ __forceinline__ void sample_coord(const DcnArgs &a, const T *offset, long long ob, int tap, int p, float &h,
                                             float &w)
{
    const int ho = p / a.Wo, wo = p - (p / a.Wo) * a.Wo;
    const int i = tap / a.kw, j = tap - (tap / a.kw) * a.kw;
    const long long P = (long long)a.Ho * a.Wo;
    const float dy = ld_f32(offset + ob + (2ll * tap) * P + p);
    const float dx = ld_f32(offset + ob + (2ll * tap + 1) * P + p);
    h = __fadd_rn((float)(ho * a.sh - a.ph + i * a.dh), dy);
    w = __fadd_rn((float)(wo * a.sw - a.pw + j * a.dw), dx);
}

// the same on an NHWC offset [B][Ho][Wo][dg*2*kh*kw]: op points at the pixel's (dy, dx) of the tap.  Kept apart from
// sample_coord, whose sharing it would reschedule the fp32 kernels.
template <typename T>
__device__ __forceinline__ void sample_coord_nhwc(const DcnArgs &a, const T *op, int tap, int p, float &h, float &w)
{
    const int ho = p / a.Wo, wo = p - (p / a.Wo) * a.Wo;
    const int i = tap / a.kw, j = tap - (tap / a.kw) * a.kw;
    h = __fadd_rn((float)(ho * a.sh - a.ph + i * a.dh), ld_f32(op));
    w = __fadd_rn((float)(wo * a.sw - a.pw + j * a.dw), ld_f32(op + 1));
}

// shared-memory sample table of one tile: corners, weights and mask of up to BN sample points
struct SampleTable { int off[4][BN]; float wt[4][BN]; float m[BN]; };

__device__ __forceinline__ void store_sample(SampleTable &t, int n, const Corners &s, float m)
{
    for (int q = 0; q < 4; ++q) { t.off[q][n] = s.off[q]; t.wt[q][n] = s.wt[q]; }
    t.m[n] = m;
}

__device__ __forceinline__ float sample_col(const SampleTable &t, int n, const float *plane)
{
    const int off[4] = {t.off[0][n], t.off[1][n], t.off[2][n], t.off[3][n]};
    const float wt[4] = {t.wt[0][n], t.wt[1][n], t.wt[2][n], t.wt[3][n]};
    return __fmul_rn(t.m[n], bilinear(plane, off, wt));
}

// acc[4][8] += As[.][tm*4 + 0..3] x Bs[.][tn*4 + 0..3, 64 + tn*4 + 0..3] over the BK-deep tile, in k order
__device__ __forceinline__ void mma_tile(const float (&As)[BK][BM], const float (&Bs)[BK][BN], float (&acc)[4][8],
                                         int tm, int tn)
{
#pragma unroll
    for (int k = 0; k < BK; ++k) {
        const float4 av = *reinterpret_cast<const float4 *>(&As[k][tm * 4]);
        const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[k][tn * 4]);
        const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[k][64 + tn * 4]);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        const float br[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[r][c] = __fmaf_rn(ar[r], br[c], acc[r][c]);
    }
}

__device__ __forceinline__ int col_of(int tn, int c) { return c < 4 ? tn * 4 + c : 64 + tn * 4 + (c - 4); }

// out[b][o][p] = bias[o] + sum over (g, tap, c in group g) of W[o][c*T + tap] * cols[b][c*T + tap][p]
// grid (ceil(P / BN), ceil(Co / BM), B)
__global__ void __launch_bounds__(NT) dcn_forward_kernel(DcnArgs a)
{
    __shared__ __align__(16) float As[BK][BM];
    __shared__ __align__(16) float Bs[BK][BN];
    __shared__ SampleTable st;
    const int tid = threadIdx.x, tm = tid / 16, tn = tid % 16;
    const int P = a.Ho * a.Wo, p0 = blockIdx.x * BN, o0 = blockIdx.y * BM, b = blockIdx.z;
    const int T = a.kh * a.kw, Cg = a.C / a.dg;
    const long long K = (long long)a.C * T, HW = (long long)a.H * a.W;

    float acc[4][8];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int o = o0 + tm * 4 + r;
        const float bv = o < a.Co ? __ldg(a.bias + o) : 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = bv;
    }

    for (int g = 0; g < a.dg; ++g) {
        const long long ob = ((long long)b * a.dg + g) * 2 * T * P;
        const long long mb = ((long long)b * a.dg + g) * T * P;
        for (int tap = 0; tap < T; ++tap) {
            __syncthreads();                                     // the previous tap's tiles are consumed
            if (tid < BN) {
                const int p = p0 + tid;
                if (p < P) {
                    float h, w;
                    sample_coord(a, a.offset, ob, tap, p, h, w);
                    store_sample(st, tid, sample_point(h, w, a.H, a.W), __ldg(a.mask + mb + (long long)tap * P + p));
                } else {
                    Corners z;
                    for (int q = 0; q < 4; ++q) { z.off[q] = -1; z.wt[q] = 0.f; }
                    store_sample(st, tid, z, 0.f);
                }
            }
            for (int c0 = 0; c0 < Cg; c0 += BK) {
                __syncthreads();                                 // sample table ready; previous tile consumed
#pragma unroll
                for (int r = 0; r < BK * BM / NT; ++r) {
                    const int e = tid + r * NT, k = e / BM, m = e % BM;
                    const int o = o0 + m, c = g * Cg + c0 + k;
                    As[k][m] = (o < a.Co && c0 + k < Cg) ? __ldg(a.weight + (long long)o * K + (long long)c * T + tap) : 0.f;
                }
#pragma unroll
                for (int r = 0; r < BK * BN / NT; ++r) {
                    const int e = tid + r * NT, k = e / BN, n = e % BN;
                    const int c = g * Cg + c0 + k;
                    Bs[k][n] = (c0 + k < Cg && p0 + n < P) ? sample_col(st, n, a.input + ((long long)b * a.C + c) * HW) : 0.f;
                }
                __syncthreads();
                mma_tile(As, Bs, acc, tm, tn);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int o = o0 + tm * 4 + r;
        if (o >= a.Co) continue;
        float *dst = a.out + ((long long)b * a.Co + o) * P;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int p = p0 + col_of(tn, c);
            if (p < P) dst[p] = acc[r][c];
        }
    }
}

// grad_cols[bl][k][p] = sum over o (in order) of W[o][k] * grad_out[b0 + bl][o][p]
// grid (ceil(P / BN), ceil(K / BM), nb)
__global__ void __launch_bounds__(NT) dcn_grad_cols_kernel(DcnArgs a, int b0)
{
    __shared__ __align__(16) float As[BK][BM];
    __shared__ __align__(16) float Bs[BK][BN];
    const int tid = threadIdx.x, tm = tid / 16, tn = tid % 16;
    const int P = a.Ho * a.Wo, p0 = blockIdx.x * BN, k0 = blockIdx.y * BM, bl = blockIdx.z;
    const long long K = (long long)a.C * a.kh * a.kw;
    const float *go = a.grad_out + (long long)(b0 + bl) * a.Co * P;
    float acc[4][8] = {};
    for (int o0 = 0; o0 < a.Co; o0 += BK) {
        __syncthreads();
#pragma unroll
        for (int r = 0; r < BK * BM / NT; ++r) {
            const int e = tid + r * NT, kk = e / BM, m = e % BM;
            As[kk][m] = (o0 + kk < a.Co && k0 + m < K) ? __ldg(a.weight + (long long)(o0 + kk) * K + k0 + m) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < BK * BN / NT; ++r) {
            const int e = tid + r * NT, kk = e / BN, n = e % BN;
            Bs[kk][n] = (o0 + kk < a.Co && p0 + n < P) ? __ldg(go + (long long)(o0 + kk) * P + p0 + n) : 0.f;
        }
        __syncthreads();
        mma_tile(As, Bs, acc, tm, tn);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const long long k = k0 + tm * 4 + r;
        if (k >= K) continue;
        float *dst = a.cols + ((long long)bl * K + k) * P;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int p = p0 + col_of(tn, c);
            if (p < P) dst[p] = acc[r][c];
        }
    }
}

// grad_offset and grad_mask of one (image, group, tap, pixel), summed over the group's channels in order
// (the reference's col2im_coord, dcn_v2_im2col_cuda.cu:256-327).  grid (ceil(P / 256), dg * T, nb)
__global__ void __launch_bounds__(256) dcn_grad_coord_kernel(DcnArgs a, int b0)
{
    const int P = a.Ho * a.Wo, p = blockIdx.x * 256 + threadIdx.x;
    if (p >= P) return;
    const int T = a.kh * a.kw, g = blockIdx.y / T, tap = blockIdx.y % T, bl = blockIdx.z, b = b0 + bl;
    const int Cg = a.C / a.dg;
    const long long HW = (long long)a.H * a.W, K = (long long)a.C * T;
    const long long ob = ((long long)b * a.dg + g) * 2 * T * P, mb = ((long long)b * a.dg + g) * T * P;
    float h, w;
    sample_coord(a, a.offset, ob, tap, p, h, w);
    const float m = __ldg(a.mask + mb + (long long)tap * P + p);
    float gy = 0.f, gx = 0.f, gm = 0.f;
    // a point with h <= -1, w <= -1, h >= H or w >= W contributes nothing (the reference's predicate: NaN passes it)
    if (!(h <= -1.f || w <= -1.f || h >= (float)a.H || w >= (float)a.W)) {
        const Corners s = sample_point(h, w, a.H, a.W);
        const int hl = (int)floorf(h), wl = (int)floorf(w);
        // d(bilinear)/dh and /dw per corner; at integer h the derivative is that of the cell [floor h, floor h + 1]
        const float ah = __fsub_rn((float)(hl + 1), h), bh = __fsub_rn(h, (float)hl);
        const float aw = __fsub_rn((float)(wl + 1), w), bw = __fsub_rn(w, (float)wl);
        const float *cp = a.cols + ((long long)bl * K + (long long)(g * Cg) * T + tap) * P + p;
        const float *ip = a.input + ((long long)b * a.C + (long long)g * Cg) * HW;
        for (int c = 0; c < Cg; ++c, cp += (long long)T * P, ip += HW) {
            const float col = __ldg(cp);
            const float v1 = s.off[0] >= 0 ? __ldg(ip + s.off[0]) : 0.f;
            const float v2 = s.off[1] >= 0 ? __ldg(ip + s.off[1]) : 0.f;
            const float v3 = s.off[2] >= 0 ? __ldg(ip + s.off[2]) : 0.f;
            const float v4 = s.off[3] >= 0 ? __ldg(ip + s.off[3]) : 0.f;
            const float val = __fmaf_rn(s.wt[3], v4, __fmaf_rn(s.wt[2], v3, __fmaf_rn(s.wt[0], v1, __fmul_rn(s.wt[1], v2))));
            const float wy = -aw * v1 - bw * v2 + aw * v3 + bw * v4;
            const float wx = -ah * v1 + ah * v2 - bh * v3 + bh * v4;
            const float cm = col * m;
            gm = __fmaf_rn(col, val, gm);
            gy = __fmaf_rn(wy, cm, gy);
            gx = __fmaf_rn(wx, cm, gx);
        }
    }
    a.grad_offset[ob + (2ll * tap) * P + p] = gy;
    a.grad_offset[ob + (2ll * tap + 1) * P + p] = gx;
    a.grad_mask[mb + (long long)tap * P + p] = gm;
}

// grad_input += the bilinear weights x grad_cols x mask, scattered with float atomics (the reference's col2im,
// dcn_v2_im2col_cuda.cu:197-254).  grid (ceil(P / 256), dg * T, nb)
__global__ void __launch_bounds__(256) dcn_grad_input_kernel(DcnArgs a, int b0)
{
    const int P = a.Ho * a.Wo, p = blockIdx.x * 256 + threadIdx.x;
    if (p >= P) return;
    const int T = a.kh * a.kw, g = blockIdx.y / T, tap = blockIdx.y % T, bl = blockIdx.z, b = b0 + bl;
    const int Cg = a.C / a.dg;
    const long long HW = (long long)a.H * a.W, K = (long long)a.C * T;
    const long long ob = ((long long)b * a.dg + g) * 2 * T * P, mb = ((long long)b * a.dg + g) * T * P;
    float h, w;
    sample_coord(a, a.offset, ob, tap, p, h, w);
    if (!(h > -1.f && w > -1.f && h < (float)a.H && w < (float)a.W)) return;
    const float m = __ldg(a.mask + mb + (long long)tap * P + p);
    const int hl = (int)floorf(h), wl = (int)floorf(w);
    // corner (y, x) gets (1 - |h - y|)(1 - |w - x|) when |h - y| < 1 and |w - x| < 1 and it lies in the image
    const bool hi_h = h > (float)hl, hi_w = w > (float)wl;
    const float ly = __fsub_rn((float)(hl + 1), h), uy = __fsub_rn(__fadd_rn(h, 1.f), (float)(hl + 1));
    const float lx = __fsub_rn((float)(wl + 1), w), ux = __fsub_rn(__fadd_rn(w, 1.f), (float)(wl + 1));
    int off[4]; float wt[4];
    off[0] = (hl >= 0 && wl >= 0) ? hl * a.W + wl : -1;                                     wt[0] = __fmul_rn(ly, lx);
    off[1] = (hl >= 0 && hi_w && wl + 1 < a.W) ? hl * a.W + wl + 1 : -1;                    wt[1] = __fmul_rn(ly, ux);
    off[2] = (hi_h && hl + 1 < a.H && wl >= 0) ? (hl + 1) * a.W + wl : -1;                  wt[2] = __fmul_rn(uy, lx);
    off[3] = (hi_h && hi_w && hl + 1 < a.H && wl + 1 < a.W) ? (hl + 1) * a.W + wl + 1 : -1; wt[3] = __fmul_rn(uy, ux);
    const float *cp = a.cols + ((long long)bl * K + (long long)(g * Cg) * T + tap) * P + p;
    float *gp = a.grad_input + ((long long)b * a.C + (long long)g * Cg) * HW;
    for (int c = 0; c < Cg; ++c, cp += (long long)T * P, gp += HW) {
        const float top = __fmul_rn(__ldg(cp), m);
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (off[q] >= 0) atomicAdd(gp + off[q], __fmul_rn(wt[q], top));
    }
}

// split s of grad_weight: part[s][o][c*T + tap] = sum over the split's (image, pixel) range, in order, of
// grad_out[b][o][p] * cols[b][c*T + tap][p], with the columns re-sampled like the forward.
// grid (ntile_n, ceil(Co / BM), S); tile n covers channels cb .. cb + BN - 1 of group g at tap
__global__ void __launch_bounds__(NT) dcn_grad_weight_kernel(DcnArgs a, long long span, float *part)
{
    __shared__ __align__(16) float As[BK][BM];
    __shared__ __align__(16) float Bs[BK][BN];
    __shared__ int sb[BK], sp[BK];
    __shared__ struct { int off[4][BK]; float wt[4][BK]; float m[BK]; } st;
    const int tid = threadIdx.x, tm = tid / 16, tn = tid % 16;
    const int T = a.kh * a.kw, Cg = a.C / a.dg, nct = (Cg + BN - 1) / BN;
    const int g = blockIdx.x / (T * nct), tap = (blockIdx.x / nct) % T, cb = (blockIdx.x % nct) * BN;
    const int o0 = blockIdx.y * BM, P = a.Ho * a.Wo;
    const long long K = (long long)a.C * T, HW = (long long)a.H * a.W, Q = (long long)a.B * P;
    const long long q0 = (long long)blockIdx.z * span, q1 = min(Q, q0 + span);
    float acc[4][8] = {};
    for (long long qs = q0; qs < q1; qs += BK) {
        __syncthreads();
        if (tid < BK) {
            const long long q = qs + tid;
            Corners s;
            float m = 0.f;
            int b = 0, p = 0;
            if (q < q1) {
                b = (int)(q / P); p = (int)(q - (long long)b * P);
                float h, w;
                sample_coord(a, a.offset, ((long long)b * a.dg + g) * 2 * T * P, tap, p, h, w);
                s = sample_point(h, w, a.H, a.W);
                m = __ldg(a.mask + ((long long)b * a.dg + g) * T * P + (long long)tap * P + p);
            } else {
                for (int k = 0; k < 4; ++k) { s.off[k] = -1; s.wt[k] = 0.f; }
            }
            for (int k = 0; k < 4; ++k) { st.off[k][tid] = s.off[k]; st.wt[k][tid] = s.wt[k]; }
            st.m[tid] = m; sb[tid] = b; sp[tid] = p;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < BK * BM / NT; ++r) {       // pixel-fastest: 16 lanes read 16 consecutive pixels
            const int e = tid + r * NT, kk = e % BK, m = e / BK, o = o0 + m;
            As[kk][m] = (qs + kk < q1 && o < a.Co) ? __ldg(a.grad_out + ((long long)sb[kk] * a.Co + o) * P + sp[kk]) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < BK * BN / NT; ++r) {
            const int e = tid + r * NT, kk = e % BK, n = e / BK, c = cb + n;
            float v = 0.f;
            if (qs + kk < q1 && c < Cg) {
                const int off[4] = {st.off[0][kk], st.off[1][kk], st.off[2][kk], st.off[3][kk]};
                const float wt[4] = {st.wt[0][kk], st.wt[1][kk], st.wt[2][kk], st.wt[3][kk]};
                v = __fmul_rn(st.m[kk], bilinear(a.input + ((long long)sb[kk] * a.C + g * Cg + c) * HW, off, wt));
            }
            Bs[kk][n] = v;
        }
        __syncthreads();
        mma_tile(As, Bs, acc, tm, tn);
    }
    float *dst = part + (long long)blockIdx.z * a.Co * K;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int o = o0 + tm * 4 + r;
        if (o >= a.Co) continue;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int ch = cb + col_of(tn, c);
            if (ch < Cg) dst[(long long)o * K + (long long)(g * Cg + ch) * T + tap] = acc[r][c];
        }
    }
}

// grad_weight[i] = sum over s = 0 .. S-1 (in order) of part[s][i]
__global__ void __launch_bounds__(256) dcn_reduce_splits_kernel(const float *part, float *out, long long n, int S)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    float s = part[i];
    for (int k = 1; k < S; ++k) s = __fadd_rn(s, part[(long long)k * n + i]);
    out[i] = s;
}

// grad_bias[o] = sum over (b, p) of grad_out[b][o][p]: per-thread strided sums, then a fixed reduction tree
__global__ void __launch_bounds__(256) dcn_grad_bias_kernel(DcnArgs a)
{
    __shared__ float red[8];
    const int o = blockIdx.x, P = a.Ho * a.Wo;
    float s = 0.f;
    for (int b = 0; b < a.B; ++b) {
        const float *go = a.grad_out + ((long long)b * a.Co + o) * P;
        for (int p = threadIdx.x; p < P; p += 256) s = __fadd_rn(s, __ldg(go + p));
    }
    for (int d = 16; d > 0; d >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, d));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = red[0];
        for (int w = 1; w < 8; ++w) t = __fadd_rn(t, red[w]);
        a.grad_bias[o] = t;
    }
}

// ---- the half-precision forward: fp16 / bf16 operands on the tensor cores ----------------------------------------
// CTA tile HBM output channels x HBN pixels, K in chunks of HBK channels of one (group, tap); 8 warps as 4 (rows) x 2
// (pixels) of 32 x 32, each an array of 2 x 4 m16n8k16 MMAs.  Tiles are stored [row][k] with a pitch of HKP halves, so
// the eight 16-byte rows an ldmatrix phase reads fall in distinct banks.
constexpr int HBM = 128, HBN = 64, HBK = 32, HKP = HBK + 8;
// split-K: a layer whose tiles would not fill two CTAs per H100 SM splits its K chunks over a cluster of up to
// H_MAX_SPLIT CTAs (each keeping at least H_MIN_CHUNKS chunks), which add their partials through distributed shared
// memory in rank order.  Chosen from the per-image shape only, so an image's output does not depend on the batch.
constexpr int H_TARGET_CTAS = 264, H_MAX_SPLIT = 8, H_MIN_CHUNKS = 4;

// input, offset, mask and out are NCHW for dcn_forward_half_kernel and NHWC (channels_last) for dcn_forward_nhwc_kernel
template <typename T> struct DcnHalfPtrs {
    const T *input, *offset, *mask;
    const T *weight;          // tap-major [Co][kh][kw][C]: a (tap, channel chunk) row is contiguous
    const T *bias;
    T *out;
};

template <typename T> struct HalfSmem {
    union {
        struct { T A[2][HBM][HKP]; T B[2][HBN][HKP]; } t;   // double-buffered weight and column tiles
        float red[HBM][HBN + 4];                           // the fp32 accumulator tile, after the K loop (NCHW)
        float red_t[HBN][HBM + 4];                         // the same, pixel-major (NHWC)
    };
};

__device__ __forceinline__ uint32_t pack2(__half, float x, float y)
{
    const __half2 h = __floats2half2_rn(x, y);
    return *reinterpret_cast<const uint32_t *>(&h);
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16, float x, float y)
{
    const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
    return *reinterpret_cast<const uint32_t *>(&h);
}
// round to nearest even; beyond the format's range the result is +-inf, never the largest finite value
__device__ __forceinline__ __half to_lp(__half, float x) { return __float2half_rn(x); }
__device__ __forceinline__ __nv_bfloat16 to_lp(__nv_bfloat16, float x) { return __float2bfloat16_rn(x); }

__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }

// NHWC sampler: the column entries of channels ch .. ch + 7 at one sample point, px pointing at channel ch of pixel 0
// of the image.  Each corner's 8 channels arrive in one 16-byte load (px 16-byte aligned, C % 8 == 0); the values are
// bilinear()'s on the same up-cast inputs.
template <typename T>
__device__ __forceinline__ void bilinear8(const T *px, long long C, const Corners &s, float m, float (&v)[8])
{
    uint4 r[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
        r[q] = s.off[q] >= 0 ? __ldg(reinterpret_cast<const uint4 *>(px + s.off[q] * C)) : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float c[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) c[q] = to_f32(reinterpret_cast<const T *>(&r[q])[k]);
        v[k] = __fmul_rn(m, blend(s.wt, c[0], c[1], c[2], c[3]));
    }
}

// NHWC sampler, one channel: px points at the channel in pixel 0 of the image
template <typename T>
__device__ __forceinline__ float bilinear_nhwc(const T *px, long long C, const Corners &s)
{
    const float v1 = s.off[0] >= 0 ? ld_f32(px + s.off[0] * C) : 0.f;
    const float v2 = s.off[1] >= 0 ? ld_f32(px + s.off[1] * C) : 0.f;
    const float v3 = s.off[2] >= 0 ? ld_f32(px + s.off[2] * C) : 0.f;
    const float v4 = s.off[3] >= 0 ? ld_f32(px + s.off[3] * C) : 0.f;
    return blend(s.wt, v1, v2, v3, v4);
}

// the rank-ordered sum over a cluster of S CTAs of the partial at x (each CTA's own copy when S == 1)
__device__ __forceinline__ float rank_sum(float *x, int S)
{
    namespace cg = cooperative_groups;
    float v = *x;
    if (S > 1) {
        v = cg::this_cluster().map_shared_rank(x, 0)[0];
        for (int q = 1; q < S; ++q) v = __fadd_rn(v, cg::this_cluster().map_shared_rank(x, q)[0]);
    }
    return v;
}

__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid)   // zero-fills when !valid
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void *p)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}

__device__ __forceinline__ void mma16816(__half, float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma16816(__nv_bfloat16, float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// out[b][o][p] = RN_T(bias[o] + sum over (g, tap, c in group g) of W[o][c*T + tap] * RN_T(cols[b][c*T + tap][p])),
// the sum in fp32 on the tensor cores.  grid (ceil(P / HBN) * S, ceil(Co / HBM), B), clusters of (S, 1, 1) when S > 1;
// CTA rank r of a cluster runs K chunks [r*n/S, (r+1)*n/S) of the n = dg * T * ceil(Cg / HBK).
// NHWC (DESIGN.md section 8o) changes only where the sampler reads a corner's channels and the offset and mask, and
// how the epilogue stores the tile; the tiles, the MMA sequence and the split are the same, so is every output bit.
template <typename T, bool NHWC>
__device__ __forceinline__ void forward_half_body(const DcnArgs &a, const DcnHalfPtrs<T> &t, int S, HalfSmem<T> &sm)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 1, wn = warp & 1;
    const int split = blockIdx.x % S, P = a.Ho * a.Wo, p0 = (int)(blockIdx.x / S) * HBN, o0 = blockIdx.y * HBM;
    const int b = blockIdx.z, T_ = a.kh * a.kw, Cg = a.C / a.dg, nct = (Cg + HBK - 1) / HBK, nchunk = a.dg * T_ * nct;
    const int kb = (int)((long long)split * nchunk / S), ke = (int)((long long)(split + 1) * nchunk / S);
    const long long HW = (long long)a.H * a.W, K = (long long)a.C * T_;
    // every 8-channel run of a weight row is 16-byte aligned, so the weight tile arrives by 16-byte cp.async
    const bool vec = ((a.C | Cg) & 7) == 0 && (reinterpret_cast<uintptr_t>(t.weight) & 15) == 0;
    const bool live = o0 + wm * 32 < a.Co;       // this warp's rows hold at least one output channel
    // the sampler's share of a B tile: pixel sn, channels sk .. sk + 7 of the chunk.  NCHW: a warp reads one channel
    // plane at 32 pixels; NHWC: 4 lanes read a pixel's 32 channels, one 64-byte run per corner
    const int sn = NHWC ? tid / (HBK / 8) : tid % HBN, sk = NHWC ? (tid % (HBK / 8)) * 8 : (tid / HBN) * 8;
    const int sp = p0 + sn;
    const bool vin = NHWC && ((a.C | Cg) & 7) == 0 && (reinterpret_cast<uintptr_t>(t.input) & 15) == 0;

    float acc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int o = o0 + wm * 32 + mt * 16 + hf * 8 + lane / 4;
            const float bv = (split == 0 && o < a.Co) ? ld_f32(t.bias + o) : 0.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) acc[mt][nt][2 * hf] = acc[mt][nt][2 * hf + 1] = bv;
        }

    // the sample point of pixel sp at the current tap: computed once per tap, reused over the group's channels
    Corners s = {};
    float m = 0.f;

    auto stage = [&](int it, int buf) {
        const int g = it / (T_ * nct), tap = (it / nct) % T_, c0 = (it % nct) * HBK;
        if (c0 == 0 || it == kb) {
            if (sp < P) {
                float h, w;
                if constexpr (NHWC) {      // offset [B][Ho][Wo][dg*2*T], mask [B][Ho][Wo][dg*T]
                    const long long px = (long long)b * P + sp;
                    const T *op = t.offset + px * (2 * a.dg * T_) + 2 * (g * T_ + tap);
                    sample_coord_nhwc(a, op, tap, sp, h, w);
                    s = sample_point(h, w, a.H, a.W);
                    m = ld_f32(t.mask + px * (a.dg * T_) + g * T_ + tap);
                } else {
                    sample_coord(a, t.offset, ((long long)b * a.dg + g) * 2 * T_ * P, tap, sp, h, w);
                    s = sample_point(h, w, a.H, a.W);
                    m = ld_f32(t.mask + ((long long)b * a.dg + g) * T_ * P + (long long)tap * P + sp);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < HBM * HBK / 8 / NT; ++r) {     // the weight tile, 8 channels per copy
            const int e = tid + r * NT, row = e / (HBK / 8), v = (e % (HBK / 8)) * 8;
            const int o = o0 + row, c = c0 + v;
            T *dst = &sm.t.A[buf][row][v];
            const T *src = t.weight + (long long)o * K + (long long)tap * a.C + (long long)g * Cg + c;
            if (vec) {
                const bool ok = o < a.Co && c < Cg;
                cp_async16(dst, ok ? src : t.weight, ok);
            } else {
#pragma unroll
                for (int q = 0; q < 8; ++q) dst[q] = (o < a.Co && c + q < Cg) ? src[q] : to_lp(T{}, 0.f);
            }
        }
        cp_async_commit();
        float v[8];
        if constexpr (NHWC) {
            const T *px = t.input + (long long)b * HW * a.C + (long long)g * Cg + c0 + sk;
            if (vin && sp < P && c0 + sk < Cg) {
                bilinear8(px, a.C, s, m, v);
            } else {
#pragma unroll
                for (int q = 0; q < 8; ++q)
                    v[q] = (sp < P && c0 + sk + q < Cg) ? __fmul_rn(m, bilinear_nhwc(px + q, a.C, s)) : 0.f;
            }
        } else {
            const T *plane = t.input + ((long long)b * a.C + (long long)g * Cg + c0 + sk) * HW;
#pragma unroll
            for (int q = 0; q < 8; ++q)
                v[q] = (sp < P && c0 + sk + q < Cg) ? __fmul_rn(m, bilinear(plane + q * HW, s.off, s.wt)) : 0.f;
        }
        uint4 pk;
        pk.x = pack2(T{}, v[0], v[1]); pk.y = pack2(T{}, v[2], v[3]);
        pk.z = pack2(T{}, v[4], v[5]); pk.w = pack2(T{}, v[6], v[7]);
        *reinterpret_cast<uint4 *>(&sm.t.B[buf][sn][sk]) = pk;
    };

    stage(kb, 0);
    cp_async_wait_all();
    __syncthreads();
    for (int it = kb; it < ke; ++it) {
        const int buf = (it - kb) & 1;
        if (it + 1 < ke) stage(it + 1, buf ^ 1);           // the next chunk's tiles load while this one multiplies
        if (live) {
#pragma unroll
            for (int ks = 0; ks < HBK; ks += 16) {
                uint32_t af[2][4], bf[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
                    ldmatrix_x4(af[mt], &sm.t.A[buf][wm * 32 + mt * 16 + (lane & 15)][ks + (lane >> 4) * 8]);
#pragma unroll
                for (int np = 0; np < 2; ++np)
                    ldmatrix_x4(bf[np], &sm.t.B[buf][wn * 32 + np * 16 + (lane & 7) + (lane >> 4) * 8]
                                                    [ks + ((lane >> 3) & 1) * 8]);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt)
                        mma16816(T{}, acc[mt][nt], af[mt], bf[nt >> 1][(nt & 1) * 2], bf[nt >> 1][(nt & 1) * 2 + 1]);
            }
        }
        cp_async_wait_all();
        __syncthreads();
    }

    // the loop ended on a barrier: the tiles are consumed and the accumulator tile may take their place
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int row = wm * 32 + mt * 16 + hf * 8 + lane / 4, col = wn * 32 + nt * 8 + (lane % 4) * 2;
                if constexpr (NHWC) {
                    sm.red_t[col][row] = acc[mt][nt][2 * hf];
                    sm.red_t[col + 1][row] = acc[mt][nt][2 * hf + 1];
                } else {
                    sm.red[row][col] = acc[mt][nt][2 * hf];
                    sm.red[row][col + 1] = acc[mt][nt][2 * hf + 1];
                }
            }
    namespace cg = cooperative_groups;
    if (S > 1) cg::this_cluster().sync(); else __syncthreads();
    // rank `split` stores rows [split*HBM/S, (split+1)*HBM/S) of the tile, adding the ranks' partials in rank order
    const int r0 = split * HBM / S, r1 = (split + 1) * HBM / S;
    if constexpr (NHWC) {                                  // output channels fastest: a warp stores a contiguous run
        const int nr = r1 - r0;
        for (int e = tid; e < nr * HBN; e += NT) {
            const int col = e / nr, row = r0 + e % nr, o = o0 + row, p = p0 + col;
            if (o >= a.Co || p >= P) continue;
            t.out[((long long)b * P + p) * a.Co + o] = to_lp(T{}, rank_sum(&sm.red_t[col][row], S));
        }
    } else {
        for (int e = r0 * HBN + tid; e < r1 * HBN; e += NT) {
            const int row = e / HBN, col = e % HBN, o = o0 + row, p = p0 + col;
            if (o >= a.Co || p >= P) continue;
            t.out[((long long)b * a.Co + o) * P + p] = to_lp(T{}, rank_sum(&sm.red[row][col], S));
        }
    }
    if (S > 1) cg::this_cluster().sync();                  // no CTA leaves while another reads its partials
}

template <typename T>
__global__ void __launch_bounds__(NT, 2) dcn_forward_half_kernel(DcnArgs a, DcnHalfPtrs<T> t, int S)
{
    __shared__ __align__(16) HalfSmem<T> sm;
    forward_half_body<T, false>(a, t, S, sm);
}

// the same forward on NHWC input, offset, mask and output (the name leaves out "forward_half" on purpose: the register
// test counts the NCHW kernels by it)
template <typename T>
__global__ void __launch_bounds__(NT, 2) dcn_forward_nhwc_kernel(DcnArgs a, DcnHalfPtrs<T> t, int S)
{
    __shared__ __align__(16) HalfSmem<T> sm;
    forward_half_body<T, true>(a, t, S, sm);
}

} // namespace

// backward plan: images per grad_cols chunk, and grad_weight's split of the (image, pixel) reduction into `splits`
// ranges of `span` pixels over `ntile_n` column tiles.  Workspace: cols_bytes of grad_cols, then part_bytes of
// grad_weight partials (0 when splits == 1), each 256-byte aligned.  A function of the shapes only.
struct DcnPlan { int chunk, splits; long long span, ntile_n; size_t cols_bytes, part_bytes; };

// External linkage on purpose: nvcc names this file's anonymous namespace, and so its kernels, after the first
// externally visible definition in the file.
DcnPlan dcn_plan(const DcnArgs &a, int chunk)
{
    DcnPlan pl;
    const int T = a.kh * a.kw, Cg = a.C / a.dg;
    const long long K = (long long)a.C * T, P = (long long)a.Ho * a.Wo, Q = (long long)a.B * P;
    pl.chunk = chunk < 1 ? 1 : (chunk > a.B ? a.B : chunk);
    pl.ntile_n = (long long)a.dg * T * ((Cg + BN - 1) / BN);
    const long long tiles = pl.ntile_n * ((a.Co + BM - 1) / BM);
    long long S = (GW_TARGET_CTAS + tiles - 1) / tiles;
    const long long maxS = (Q + 4 * BK - 1) / (4 * BK);       // at least 4 BK-steps per split
    S = S < 1 ? 1 : (S > maxS ? maxS : S);
    if (S > 65535) S = 65535;
    pl.span = ((Q + S - 1) / S + BK - 1) / BK * BK;
    pl.splits = (int)((Q + pl.span - 1) / pl.span);
    pl.cols_bytes = align_up((size_t)pl.chunk * K * P * sizeof(float));
    pl.part_bytes = pl.splits > 1 ? align_up((size_t)pl.splits * a.Co * K * sizeof(float)) : 0;
    return pl;
}

namespace {

size_t dcn_workspace_bytes(const DcnPlan &p) { return p.cols_bytes + p.part_bytes; }

// checks a DCN descriptor and fills the kernels' argument block; PVB_OK or PVB_ERR_INVALID (no CUDA call)
int dcn_args(const pvb_dcn_desc *d, DcnArgs &a)
{
    if (!d) return fail(PVB_ERR_INVALID, "descriptor is NULL");
    if (d->B < 0 || d->C < 1 || d->H < 1 || d->W < 1 || d->C_out < 1 || d->kh < 1 || d->kw < 1)
        return fail(PVB_ERR_INVALID, "bad shape B=%d C=%d H=%d W=%d C_out=%d kh=%d kw=%d", d->B, d->C, d->H, d->W,
                    d->C_out, d->kh, d->kw);
    if (d->stride_h < 1 || d->stride_w < 1 || d->pad_h < 0 || d->pad_w < 0 || d->dilation_h < 1 || d->dilation_w < 1)
        return fail(PVB_ERR_INVALID, "bad stride/pad/dilation (%d,%d)/(%d,%d)/(%d,%d)", d->stride_h, d->stride_w,
                    d->pad_h, d->pad_w, d->dilation_h, d->dilation_w);
    if (d->deformable_groups < 1 || d->C % d->deformable_groups)
        return fail(PVB_ERR_INVALID, "deformable_groups=%d must be >= 1 and divide C=%d", d->deformable_groups, d->C);
    const long long ext_h = (long long)d->dilation_h * (d->kh - 1) + 1, ext_w = (long long)d->dilation_w * (d->kw - 1) + 1;
    const long long span_h = d->H + 2ll * d->pad_h, span_w = d->W + 2ll * d->pad_w;
    if (span_h > (1ll << 30) || span_w > (1ll << 30) || ext_h > (1ll << 30) || ext_w > (1ll << 30))
        return fail(PVB_ERR_INVALID, "padded input or dilated kernel extent >= 2^30");
    if (span_h < ext_h || span_w < ext_w) return fail(PVB_ERR_INVALID, "the dilated kernel does not fit the padded input");
    const long long Ho = (span_h - ext_h) / d->stride_h + 1, Wo = (span_w - ext_w) / d->stride_w + 1;
    const long long K = (long long)d->C * d->kh * d->kw, T = (long long)d->kh * d->kw;
    if (d->B > 65535) return fail(PVB_ERR_INVALID, "B=%d > 65535", d->B);
    if ((long long)d->H * d->W >= (1ll << 31) || Ho * Wo >= (1ll << 31)) return fail(PVB_ERR_INVALID, "H*W or Ho*Wo >= 2^31");
    if (K > 65535ll * 64 || d->C_out > 65535 * 64) return fail(PVB_ERR_INVALID, "C*kh*kw or C_out > 4194240");
    if (T * d->deformable_groups > 65535) return fail(PVB_ERR_INVALID, "deformable_groups*kh*kw > 65535");
    a = DcnArgs{};
    a.B = d->B; a.C = d->C; a.H = d->H; a.W = d->W; a.Co = d->C_out; a.kh = d->kh; a.kw = d->kw;
    a.sh = d->stride_h; a.sw = d->stride_w; a.ph = d->pad_h; a.pw = d->pad_w; a.dh = d->dilation_h; a.dw = d->dilation_w;
    a.dg = d->deformable_groups; a.Ho = (int)Ho; a.Wo = (int)Wo;
    return PVB_OK;
}

// the split-K factor of the half-precision forward: a function of the per-image shape only
int dcn_half_splits(const DcnArgs &a)
{
    const int T = a.kh * a.kw, Cg = a.C / a.dg;
    const long long nchunk = (long long)a.dg * T * ((Cg + HBK - 1) / HBK);
    const long long tiles = ((long long)a.Ho * a.Wo + HBN - 1) / HBN * ((a.Co + HBM - 1) / HBM);
    long long S = (H_TARGET_CTAS + tiles - 1) / tiles;
    if (S > H_MAX_SPLIT) S = H_MAX_SPLIT;
    if (S > nchunk / H_MIN_CHUNKS) S = nchunk / H_MIN_CHUNKS;
    return S < 1 ? 1 : (int)S;
}

template <typename T>
int launch_dcn_forward_half(const DcnArgs &a, const DcnHalfPtrs<T> &t, bool nhwc, cudaStream_t stream)
{
    const int S = dcn_half_splits(a);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(((long long)a.Ho * a.Wo + HBN - 1) / HBN * S), (a.Co + HBM - 1) / HBM, a.B);
    cfg.blockDim = dim3(NT);
    cfg.stream = stream;
    cudaLaunchAttribute cluster;
    cluster.id = cudaLaunchAttributeClusterDimension;
    cluster.val.clusterDim.x = S; cluster.val.clusterDim.y = 1; cluster.val.clusterDim.z = 1;
    cfg.attrs = &cluster;
    cfg.numAttrs = S > 1 ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, nhwc ? dcn_forward_nhwc_kernel<T> : dcn_forward_half_kernel<T>, a, t, S);
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, nhwc ? "dcn nhwc forward kernel" : "dcn half forward kernel");
}

template <typename T>
DcnHalfPtrs<T> half_ptrs(const void *input, const void *offset, const void *mask, const void *weight, const void *bias,
                         void *output)
{
    return DcnHalfPtrs<T>{static_cast<const T *>(input), static_cast<const T *>(offset), static_cast<const T *>(mask),
                          static_cast<const T *>(weight), static_cast<const T *>(bias), static_cast<T *>(output)};
}

// the checks and launch of pvb_dcn_forward_half (nhwc false) and pvb_dcn_forward_half_nhwc (true)
int dcn_forward_half(const pvb_dcn_desc *d, int32_t dtype, const void *input, const void *offset, const void *mask,
                     const void *weight, const void *bias, void *output, bool nhwc, pvb_stream_t stream)
{
    if (dtype != PVB_DCN_F16 && dtype != PVB_DCN_BF16)
        return fail(PVB_ERR_INVALID, "dtype=%d must be PVB_DCN_F16 (%d) or PVB_DCN_BF16 (%d)", dtype, PVB_DCN_F16,
                    PVB_DCN_BF16);
    DcnArgs a;
    if (int rc = dcn_args(d, a)) return rc;
    if (a.B == 0) return PVB_OK;
    if (!input || !offset || !mask || !weight || !bias || !output) return fail(PVB_ERR_INVALID, "NULL tensor");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return dtype == PVB_DCN_F16
               ? launch_dcn_forward_half(a, half_ptrs<__half>(input, offset, mask, weight, bias, output), nhwc, st)
               : launch_dcn_forward_half(a, half_ptrs<__nv_bfloat16>(input, offset, mask, weight, bias, output), nhwc,
                                         st);
}

// ---- the TF32 path: fp32 operands rounded once to TF32 on the tensor cores (DESIGN.md section 8p) -------------------
// The forward and the backward's two products multiply TF_BM x TF_BN tiles over TF_BK-deep steps (the FFMA kernels'
// 64 x 128 x 16, so the backward plan is dcn_plan's) with 8 warps as 2 (rows) x 4 (columns) of 32 x 32, each an array of
// 2 x 4 mma.sync m16n8k8.  Operand tiles are fp32 in shared memory, double-buffered, and rounded to TF32 (cvt.rna) as
// the fragments are loaded.  A tile is stored row-major, [row][k] with a pitch of TF_BK + 4 floats, or k-major,
// [k][row] with a pitch of rows + 8, whichever its global layout fills coalesced; either pitch puts the 32 lanes of a
// fragment load in 32 distinct banks.
constexpr int TF_BM = 64, TF_BN = 128, TF_BK = 16;
// the forward's split-K, chosen as the half-precision forward's: a cluster of up to TF_MAX_SPLIT CTAs, each keeping at
// least TF_MIN_CHUNKS K chunks, when the tiles would not fill two CTAs per H100 SM; a function of the per-image shape
constexpr int TF_TARGET_CTAS = 264, TF_MAX_SPLIT = 8, TF_MIN_CHUNKS = 4;

template <int ROWS, bool KMAJOR> struct TfTile {
    static constexpr int PITCH = KMAJOR ? ROWS + 8 : TF_BK + 4;
    static constexpr int SIZE = KMAJOR ? TF_BK * PITCH : ROWS * PITCH;
    __device__ static __forceinline__ int at(int row, int k) { return KMAJOR ? k * PITCH + row : row * PITCH + k; }
};

// round to the nearest TF32 value (10-bit mantissa), ties away from zero; the result is an fp32 bit pattern
__device__ __forceinline__ uint32_t tf32_rna(float x)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void mma1688(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[mt][nt] += A B^T over one TF_BK-deep step of the tiles A (TF_BM rows) and B (TF_BN rows), for the warp at
// rows wm*32 + mt*16 .., columns wn*32 + nt*8 ..; the m16n8k8 fragments: A (row r, k) at lane 4*(r % 8) + k % 4, B and
// the accumulator alike (PTX ISA, "Matrix Fragments for mma.m16n8k8" with .tf32)
template <typename LA, typename LB>
__device__ __forceinline__ void tf32_step(const float *A, const float *B, float (&acc)[2][4][4], int wm, int wn, int lane)
{
    const int gr = lane >> 2, tg = lane & 3;
#pragma unroll
    for (int ks = 0; ks < TF_BK; ks += 8) {
        uint32_t af[2][4], bf[4][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int r = wm * 32 + mt * 16 + gr;
            af[mt][0] = tf32_rna(A[LA::at(r, ks + tg)]);
            af[mt][1] = tf32_rna(A[LA::at(r + 8, ks + tg)]);
            af[mt][2] = tf32_rna(A[LA::at(r, ks + tg + 4)]);
            af[mt][3] = tf32_rna(A[LA::at(r + 8, ks + tg + 4)]);
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int n = wn * 32 + nt * 8 + gr;
            bf[nt][0] = tf32_rna(B[LB::at(n, ks + tg)]);
            bf[nt][1] = tf32_rna(B[LB::at(n, ks + tg + 4)]);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) mma1688(acc[mt][nt], af[mt], bf[nt][0], bf[nt][1]);
    }
}

using FwA = TfTile<TF_BM, false>;   // forward: weight [o][c]
using FwB = TfTile<TF_BN, false>;   //          columns [p][c]
using GcA = TfTile<TF_BM, true>;    // grad_cols: weight [o][k], k-major
using GcB = TfTile<TF_BN, true>;    //            grad_out [o][p], k-major
using GwA = TfTile<TF_BM, false>;   // grad_weight: grad_out [o][pixel]
using GwB = TfTile<TF_BN, false>;   //              columns [c][pixel]

struct TfFwdSmem {
    union {
        struct { float A[2][FwA::SIZE]; float B[2][FwB::SIZE]; } t;   // double-buffered weight and column tiles
        float red[TF_BM][TF_BN + 8];                                  // the fp32 accumulator tile, after the K loop
    };
};

// out[b][o][p] = bias[o] + sum over (g, tap, c in group g) of RN_tf32(W[o][c*T + tap]) * RN_tf32(cols[b][c*T + tap][p]),
// the sum in fp32 on the tensor cores, from the bias.  a.weight is tap-major, [Co][kh][kw][C].  grid
// (ceil(P / TF_BN) * S, ceil(Co / TF_BM), B), clusters of (S, 1, 1) when S > 1; CTA rank r runs K chunks
// [r*n/S, (r+1)*n/S) of the n = dg * T * ceil(Cg / TF_BK), and the ranks add their partials in rank order.
__global__ void __launch_bounds__(NT, 2) dcn_forward_tf32_kernel(DcnArgs a, int S)
{
    __shared__ __align__(16) TfFwdSmem sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
    const int split = blockIdx.x % S, P = a.Ho * a.Wo, p0 = (int)(blockIdx.x / S) * TF_BN, o0 = blockIdx.y * TF_BM;
    const int b = blockIdx.z, T = a.kh * a.kw, Cg = a.C / a.dg, nct = (Cg + TF_BK - 1) / TF_BK, nchunk = a.dg * T * nct;
    const int kb = (int)((long long)split * nchunk / S), ke = (int)((long long)(split + 1) * nchunk / S);
    const long long HW = (long long)a.H * a.W, K = (long long)a.C * T;
    // every 4-channel run of a weight row is 16-byte aligned, so the weight tile arrives by 16-byte cp.async
    const bool vec = ((a.C | Cg) & 3) == 0 && (reinterpret_cast<uintptr_t>(a.weight) & 15) == 0;
    const bool live = o0 + wm * 32 < a.Co;       // this warp's rows hold at least one output channel
    // the sampler's share of a B tile: pixel sn, channels sk .. sk + 7 of the chunk; a warp reads one plane at 32 pixels
    const int sn = tid % TF_BN, sk = (tid / TF_BN) * 8, sp = p0 + sn;

    float acc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int o = o0 + wm * 32 + mt * 16 + hf * 8 + lane / 4;
            const float bv = (split == 0 && o < a.Co) ? __ldg(a.bias + o) : 0.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) acc[mt][nt][2 * hf] = acc[mt][nt][2 * hf + 1] = bv;
        }

    // the sample point of pixel sp at the current tap: computed once per tap, reused over the group's channels
    Corners s = {};
    float m = 0.f;

    auto stage = [&](int it, int buf) {
        const int g = it / (T * nct), tap = (it / nct) % T, c0 = (it % nct) * TF_BK;
        if ((c0 == 0 || it == kb) && sp < P) {
            float h, w;
            sample_coord(a, a.offset, ((long long)b * a.dg + g) * 2 * T * P, tap, sp, h, w);
            s = sample_point(h, w, a.H, a.W);
            m = __ldg(a.mask + ((long long)b * a.dg + g) * T * P + (long long)tap * P + sp);
        }
        {                                                  // the weight tile, 4 channels per thread
            const int row = tid / (TF_BK / 4), v = (tid % (TF_BK / 4)) * 4, o = o0 + row, c = c0 + v;
            float *dst = &sm.t.A[buf][FwA::at(row, v)];
            const float *src = a.weight + (long long)o * K + (long long)tap * a.C + (long long)g * Cg + c;
            if (vec) {
                const bool ok = o < a.Co && c < Cg;
                cp_async16(dst, ok ? src : a.weight, ok);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) dst[q] = (o < a.Co && c + q < Cg) ? __ldg(src + q) : 0.f;
            }
        }
        cp_async_commit();
        const float *plane = a.input + ((long long)b * a.C + (long long)g * Cg + c0 + sk) * HW;
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q)
            v[q] = (sp < P && c0 + sk + q < Cg) ? __fmul_rn(m, bilinear(plane + q * HW, s.off, s.wt)) : 0.f;
        float4 *dst = reinterpret_cast<float4 *>(&sm.t.B[buf][FwB::at(sn, sk)]);
        dst[0] = make_float4(v[0], v[1], v[2], v[3]);
        dst[1] = make_float4(v[4], v[5], v[6], v[7]);
    };

    stage(kb, 0);
    cp_async_wait_all();
    __syncthreads();
    for (int it = kb; it < ke; ++it) {
        const int buf = (it - kb) & 1;
        if (it + 1 < ke) stage(it + 1, buf ^ 1);           // the next chunk's tiles load while this one multiplies
        if (live) tf32_step<FwA, FwB>(sm.t.A[buf], sm.t.B[buf], acc, wm, wn, lane);
        cp_async_wait_all();
        __syncthreads();
    }

    // the loop ended on a barrier: the tiles are consumed and the accumulator tile may take their place
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int row = wm * 32 + mt * 16 + hf * 8 + lane / 4, col = wn * 32 + nt * 8 + (lane % 4) * 2;
                *reinterpret_cast<float2 *>(&sm.red[row][col]) = make_float2(acc[mt][nt][2 * hf], acc[mt][nt][2 * hf + 1]);
            }
    namespace cg = cooperative_groups;
    if (S > 1) cg::this_cluster().sync(); else __syncthreads();
    // rank `split` stores rows [split*TF_BM/S, (split+1)*TF_BM/S) of the tile, adding the ranks' partials in rank order
    const int r0 = split * TF_BM / S, r1 = (split + 1) * TF_BM / S;
    for (int e = r0 * TF_BN + tid; e < r1 * TF_BN; e += NT) {
        const int row = e / TF_BN, col = e % TF_BN, o = o0 + row, p = p0 + col;
        if (o >= a.Co || p >= P) continue;
        a.out[((long long)b * a.Co + o) * P + p] = rank_sum(&sm.red[row][col], S);
    }
    if (S > 1) cg::this_cluster().sync();                  // no CTA leaves while another reads its partials
}

// grad_cols[bl][k][p] = sum over o of RN_tf32(W[o][k]) * RN_tf32(grad_out[b0 + bl][o][p]) on the tensor cores, in
// TF_BK-deep steps of o.  grid (ceil(P / TF_BN), ceil(K / TF_BM), nb)
__global__ void __launch_bounds__(NT, 2) dcn_grad_cols_tf32_kernel(DcnArgs a, int b0)
{
    __shared__ __align__(16) float As[2][GcA::SIZE];
    __shared__ __align__(16) float Bs[2][GcB::SIZE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
    const int P = a.Ho * a.Wo, p0 = blockIdx.x * TF_BN, k0 = blockIdx.y * TF_BM, bl = blockIdx.z;
    const long long K = (long long)a.C * a.kh * a.kw;
    const float *go = a.grad_out + (long long)(b0 + bl) * a.Co * P;
    float acc[2][4][4] = {};
    float ra[TF_BK * TF_BM / NT], rb[TF_BK * TF_BN / NT];  // the next step's tiles, loaded while this one multiplies
    auto fetch = [&](int o0) {
#pragma unroll
        for (int r = 0; r < TF_BK * TF_BM / NT; ++r) {
            const int e = tid + r * NT, kk = e / TF_BM, m = e % TF_BM;
            ra[r] = (o0 + kk < a.Co && k0 + m < K) ? __ldg(a.weight + (long long)(o0 + kk) * K + k0 + m) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < TF_BK * TF_BN / NT; ++r) {
            const int e = tid + r * NT, kk = e / TF_BN, n = e % TF_BN;
            rb[r] = (o0 + kk < a.Co && p0 + n < P) ? __ldg(go + (long long)(o0 + kk) * P + p0 + n) : 0.f;
        }
    };
    auto put = [&](int buf) {
#pragma unroll
        for (int r = 0; r < TF_BK * TF_BM / NT; ++r) {
            const int e = tid + r * NT;
            As[buf][GcA::at(e % TF_BM, e / TF_BM)] = ra[r];
        }
#pragma unroll
        for (int r = 0; r < TF_BK * TF_BN / NT; ++r) {
            const int e = tid + r * NT;
            Bs[buf][GcB::at(e % TF_BN, e / TF_BN)] = rb[r];
        }
    };
    const int n = (a.Co + TF_BK - 1) / TF_BK;
    fetch(0);
    put(0);
    __syncthreads();
    for (int i = 0; i < n; ++i) {
        const int buf = i & 1;
        if (i + 1 < n) fetch((i + 1) * TF_BK);
        tf32_step<GcA, GcB>(As[buf], Bs[buf], acc, wm, wn, lane);
        if (i + 1 < n) put(buf ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const long long k = k0 + wm * 32 + mt * 16 + hf * 8 + lane / 4;
            if (k >= K) continue;
            float *dst = a.cols + ((long long)bl * K + k) * P;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int p = p0 + wn * 32 + nt * 8 + (lane % 4) * 2;
                if (p < P) dst[p] = acc[mt][nt][2 * hf];
                if (p + 1 < P) dst[p + 1] = acc[mt][nt][2 * hf + 1];
            }
        }
}

// split s of grad_weight: part[s][o][c*T + tap] = sum over the split's (image, pixel) range, in TF_BK-pixel steps, of
// RN_tf32(grad_out[b][o][p]) * RN_tf32(cols[b][c*T + tap][p]), the columns re-sampled like the forward.
// grid (ntile_n, ceil(Co / TF_BM), S) of dcn_plan; tile n covers channels cb .. cb + TF_BN - 1 of group g at tap
__global__ void __launch_bounds__(NT, 2) dcn_grad_weight_tf32_kernel(DcnArgs a, long long span, float *part)
{
    __shared__ __align__(16) float As[2][GwA::SIZE];
    __shared__ __align__(16) float Bs[2][GwB::SIZE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
    const int T = a.kh * a.kw, Cg = a.C / a.dg, nct = (Cg + TF_BN - 1) / TF_BN;
    const int g = blockIdx.x / (T * nct), tap = (blockIdx.x / nct) % T, cb = (blockIdx.x % nct) * TF_BN;
    const int o0 = blockIdx.y * TF_BM, P = a.Ho * a.Wo;
    const long long K = (long long)a.C * T, HW = (long long)a.H * a.W, Q = (long long)a.B * P;
    const long long q0 = (long long)blockIdx.z * span, q1 = min(Q, q0 + span);
    // this thread's pixel of a step, and its first row (output channel) and column (channel); rows and columns go by 16
    const int kk = tid % TF_BK, rn = tid / TF_BK;
    float acc[2][4][4] = {};
    float ra[TF_BM / 16], rb[TF_BN / 16];                  // the next step's tiles, loaded while this one multiplies
    auto fetch = [&](long long qs) {
        const long long q = qs + kk;
        if (q < q1) {
            const int b = (int)(q / P), p = (int)(q - (long long)b * P);
            float h, w;
            sample_coord(a, a.offset, ((long long)b * a.dg + g) * 2 * T * P, tap, p, h, w);
            const Corners s = sample_point(h, w, a.H, a.W);
            const float m = __ldg(a.mask + ((long long)b * a.dg + g) * T * P + (long long)tap * P + p);
#pragma unroll
            for (int r = 0; r < TF_BM / 16; ++r) {
                const int o = o0 + rn + 16 * r;
                ra[r] = o < a.Co ? __ldg(a.grad_out + ((long long)b * a.Co + o) * P + p) : 0.f;
            }
#pragma unroll
            for (int r = 0; r < TF_BN / 16; ++r) {
                const int c = cb + rn + 16 * r;
                rb[r] = c < Cg ? __fmul_rn(m, bilinear(a.input + ((long long)b * a.C + g * Cg + c) * HW, s.off, s.wt))
                               : 0.f;
            }
        } else {
#pragma unroll
            for (int r = 0; r < TF_BM / 16; ++r) ra[r] = 0.f;
#pragma unroll
            for (int r = 0; r < TF_BN / 16; ++r) rb[r] = 0.f;
        }
    };
    auto put = [&](int buf) {
#pragma unroll
        for (int r = 0; r < TF_BM / 16; ++r) As[buf][GwA::at(rn + 16 * r, kk)] = ra[r];
#pragma unroll
        for (int r = 0; r < TF_BN / 16; ++r) Bs[buf][GwB::at(rn + 16 * r, kk)] = rb[r];
    };
    const long long n = (q1 - q0 + TF_BK - 1) / TF_BK;
    fetch(q0);
    put(0);
    __syncthreads();
    for (long long i = 0; i < n; ++i) {
        const int buf = (int)(i & 1);
        if (i + 1 < n) fetch(q0 + (i + 1) * TF_BK);
        tf32_step<GwA, GwB>(As[buf], Bs[buf], acc, wm, wn, lane);
        if (i + 1 < n) put(buf ^ 1);
        __syncthreads();
    }
    float *dst = part + (long long)blockIdx.z * a.Co * K;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int o = o0 + wm * 32 + mt * 16 + hf * 8 + lane / 4;
            if (o >= a.Co) continue;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int ch = cb + wn * 32 + nt * 8 + (lane % 4) * 2 + j;
                    if (ch < Cg) dst[(long long)o * K + (long long)(g * Cg + ch) * T + tap] = acc[mt][nt][2 * hf + j];
                }
        }
}

// the split-K factor of the TF32 forward: a function of the per-image shape only
int dcn_tf32_splits(const DcnArgs &a)
{
    const int T = a.kh * a.kw, Cg = a.C / a.dg;
    const long long nchunk = (long long)a.dg * T * ((Cg + TF_BK - 1) / TF_BK);
    const long long tiles = ((long long)a.Ho * a.Wo + TF_BN - 1) / TF_BN * ((a.Co + TF_BM - 1) / TF_BM);
    long long S = (TF_TARGET_CTAS + tiles - 1) / tiles;
    if (S > TF_MAX_SPLIT) S = TF_MAX_SPLIT;
    if (S > nchunk / TF_MIN_CHUNKS) S = nchunk / TF_MIN_CHUNKS;
    return S < 1 ? 1 : (int)S;
}

// the checks and launches of pvb_dcn_backward (tf32 false: FFMA products) and pvb_dcn_backward_tf32 (true: grad_cols
// and grad_weight on the tensor cores); the plan, and every other kernel, is the same
int dcn_backward(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask, const float *weight,
                 const float *grad_output, float *grad_input, float *grad_offset, float *grad_mask, float *grad_weight,
                 float *grad_bias, int32_t chunk, void *workspace, size_t workspace_bytes, bool tf32,
                 pvb_stream_t stream)
{
    DcnArgs a;
    if (int rc = dcn_args(d, a)) return rc;
    if (a.B == 0) return PVB_OK;
    if (!input || !offset || !mask || !weight || !grad_output || !grad_input || !grad_offset || !grad_mask ||
        !grad_weight || !grad_bias)
        return fail(PVB_ERR_INVALID, "NULL tensor");
    const DcnPlan pl = dcn_plan(a, chunk);
    if (int rc = check_workspace(dcn_workspace_bytes(pl), workspace, workspace_bytes)) return rc;
    a.input = input; a.offset = offset; a.mask = mask; a.weight = weight; a.grad_out = grad_output;
    a.grad_input = grad_input; a.grad_offset = grad_offset; a.grad_mask = grad_mask; a.grad_weight = grad_weight;
    a.grad_bias = grad_bias;
    a.cols = static_cast<float *>(workspace);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int P = a.Ho * a.Wo, T = a.kh * a.kw;
    const long long K = (long long)a.C * T;
    float *part = pl.splits > 1 ? reinterpret_cast<float *>(static_cast<char *>(workspace) + pl.cols_bytes) : a.grad_weight;
    cudaError_t e = cudaMemsetAsync(a.grad_input, 0, (size_t)a.B * a.C * a.H * a.W * sizeof(float), st);
    if (e != cudaSuccess) return cuda_fail(e, "dcn backward kernels");
    for (int b0 = 0; b0 < a.B; b0 += pl.chunk) {
        const int nb = a.B - b0 < pl.chunk ? a.B - b0 : pl.chunk;
        const dim3 grid((P + BN - 1) / BN, (unsigned)((K + BM - 1) / BM), nb);
        if (tf32)
            dcn_grad_cols_tf32_kernel<<<grid, NT, 0, st>>>(a, b0);
        else
            dcn_grad_cols_kernel<<<grid, NT, 0, st>>>(a, b0);
        dcn_grad_coord_kernel<<<dim3((P + 255) / 256, a.dg * T, nb), 256, 0, st>>>(a, b0);
        dcn_grad_input_kernel<<<dim3((P + 255) / 256, a.dg * T, nb), 256, 0, st>>>(a, b0);
    }
    const dim3 gw_grid((unsigned)pl.ntile_n, (a.Co + BM - 1) / BM, pl.splits);
    if (tf32)
        dcn_grad_weight_tf32_kernel<<<gw_grid, NT, 0, st>>>(a, pl.span, part);
    else
        dcn_grad_weight_kernel<<<gw_grid, NT, 0, st>>>(a, pl.span, part);
    if (pl.splits > 1) {
        const long long n = (long long)a.Co * K;
        dcn_reduce_splits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part, a.grad_weight, n, pl.splits);
    }
    dcn_grad_bias_kernel<<<a.Co, 256, 0, st>>>(a);
    e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "dcn backward kernels");
}

static_assert(TF_BM == BM && TF_BN == BN && TF_BK == BK, "the TF32 backward kernels run on dcn_plan's tiles");

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_dcn_forward(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                            const float *weight, const float *bias, float *output, pvb_stream_t stream)
{
    DcnArgs a;
    if (int rc = dcn_args(d, a)) return rc;
    if (a.B == 0) return PVB_OK;
    if (!input || !offset || !mask || !weight || !bias || !output) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.input = input; a.offset = offset; a.mask = mask; a.weight = weight; a.bias = bias; a.out = output;
    const dim3 grid((a.Ho * a.Wo + BN - 1) / BN, (a.Co + BM - 1) / BM, a.B);
    dcn_forward_kernel<<<grid, NT, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "dcn forward kernel");
}

PVB_API int pvb_dcn_forward_half(const pvb_dcn_desc *d, int32_t dtype, const void *input, const void *offset,
                                 const void *mask, const void *weight, const void *bias, void *output,
                                 pvb_stream_t stream)
{
    return dcn_forward_half(d, dtype, input, offset, mask, weight, bias, output, false, stream);
}

PVB_API int pvb_dcn_forward_half_nhwc(const pvb_dcn_desc *d, int32_t dtype, const void *input, const void *offset,
                                      const void *mask, const void *weight, const void *bias, void *output,
                                      pvb_stream_t stream)
{
    return dcn_forward_half(d, dtype, input, offset, mask, weight, bias, output, true, stream);
}

PVB_API size_t pvb_dcn_backward_workspace_bytes(const pvb_dcn_desc *d, int32_t chunk)
{
    DcnArgs a;
    if (!d || d->B < 1 || dcn_args(d, a) != PVB_OK) return 0;
    return dcn_workspace_bytes(dcn_plan(a, chunk));
}

PVB_API int pvb_dcn_backward(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                             const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                             float *grad_mask, float *grad_weight, float *grad_bias, int32_t chunk, void *workspace,
                             size_t workspace_bytes, pvb_stream_t stream)
{
    return dcn_backward(d, input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask, grad_weight,
                        grad_bias, chunk, workspace, workspace_bytes, false, stream);
}

PVB_API int pvb_dcn_forward_tf32(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                                 const float *weight, const float *bias, float *output, pvb_stream_t stream)
{
    DcnArgs a;
    if (int rc = dcn_args(d, a)) return rc;
    if (a.B == 0) return PVB_OK;
    if (!input || !offset || !mask || !weight || !bias || !output) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.input = input; a.offset = offset; a.mask = mask; a.weight = weight; a.bias = bias; a.out = output;
    const int S = dcn_tf32_splits(a);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(((long long)a.Ho * a.Wo + TF_BN - 1) / TF_BN * S), (a.Co + TF_BM - 1) / TF_BM, a.B);
    cfg.blockDim = dim3(NT);
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute cluster;
    cluster.id = cudaLaunchAttributeClusterDimension;
    cluster.val.clusterDim.x = S; cluster.val.clusterDim.y = 1; cluster.val.clusterDim.z = 1;
    cfg.attrs = &cluster;
    cfg.numAttrs = S > 1 ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, dcn_forward_tf32_kernel, a, S);
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "dcn tf32 forward kernel");
}

PVB_API int pvb_dcn_backward_tf32(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                                  const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                                  float *grad_mask, float *grad_weight, float *grad_bias, int32_t chunk, void *workspace,
                                  size_t workspace_bytes, pvb_stream_t stream)
{
    return dcn_backward(d, input, offset, mask, weight, grad_output, grad_input, grad_offset, grad_mask, grad_weight,
                        grad_bias, chunk, workspace, workspace_bytes, true, stream);
}

} // extern "C"
