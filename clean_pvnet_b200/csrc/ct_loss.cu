// ct_loss.cu -- the CenterNet detector's heatmap target and focal loss from its boxes, without the dense target
// (DESIGN.md section 8i).
//
// The target of image b, class c, pixel (x, y) is the ct_hm that lib/datasets/tless*/ct.py draws with
// data_utils.draw_umich_gaussian (lib/utils/data_utils.py:36-64), bit for bit: the maximum, over the image's objects j
// with ct_01 == 1, ct_cls == c, |x - cx| <= r and |y - cy| <= r (cx = ct_ind mod W, cy = ct_ind div W, r = ct_radius),
// of float32(g), and 0 where no object qualifies.  g is gaussian2D's value in fp64, in numpy's operation order:
//   s2 = RN(sigma * sigma), sigma = (2r + 1) / 6;  e = RN(RN(dx*dx / s2) + RN(dy*dy / s2));  g = exp(-e / 2);  g < 2^-52 -> 0
// (gaussian2D's rho term is a signed zero and changes nothing).  ct_gauss() is the only place that formula lives.
//
// The loss is the trainer's FocalLoss on net_utils.sigmoid (lib/utils/net_utils.py:9-39, lib/train/trainers/ct.py:20-21)
// with the fp32 operations CUDA torch runs per element:
//   p = clamp(1 / (1 + expf(-x)), 1e-4f, 0.9999f) (NaN kept);  u = RN(1 - p)
//   pos term = RN(RN(logf(p) * RN(u*u)) * [t == 1]);  neg term = RN(RN(RN(logf(u) * RN(p*p)) * powf(RN(1 - t), 4)) * [t < 1])
// The terms are added in fp64 per CTA; ct_loss_final_kernel adds the partials in a fixed order and rounds each sum once:
//   loss = RN(0 - neg) if no pixel has t == 1, else RN(0 - RN(RN(pos + neg) / num_pos)).
// The backward pass repeats autograd's chain op by op (ct_grad), including the order in which autograd adds the
// gradients of p's four uses: ((pow(p, 2) + (1 - p) of log) + (1 - p) of pow) + log(p).  Every operation is an explicit
// round-to-nearest intrinsic or the libdevice function torch's kernel calls, so nvcc contracts nothing into an FMA.
#include "api.h"
#include "common.cuh"

namespace pvb {

// One CTA per (32x16 pixel tile, class, image); the image's objects of that class whose window meets the tile are staged
// in shared memory.
struct CtArgs {
    const float *logits;      // [B][C][H][W] at element strides ls (forward, backward)
    long long ls[4];
    const long long *ct_ind;  // [B][M] cy * W + cx
    const int *ct_radius;     // [B][M]
    const long long *ct_cls;  // [B][M]
    const float *ct_01;       // [B][M] an object counts where ct_01 == 1
    int B, M, C, H, W;
    float *out;               // contiguous [B][C][H][W]: the target (target) or grad_logits (backward)
    double *pos_part, *neg_part;   // [nparts] per-CTA fp64 sums of the pos and neg terms (forward)
    int *cnt_part;            // [nparts] per-CTA counts of target == 1 (forward)
    long long *num_pos;       // exact count of target == 1: written by the forward pass, read by the backward pass
    float *loss;              // the scalar loss (forward)
    const float *grad_loss;   // the scalar upstream gradient (backward)
};

constexpr int CT_TW = 32, CT_TH = 16;      // one CTA per (32x16 pixel tile, class, image)
constexpr int CT_THREADS = 256;            // each thread owns two pixels of a column: rows ty and ty + 8
constexpr int CT_ROWS = CT_TW * CT_TH / CT_THREADS;
constexpr float CT_LO = 1e-4f, CT_HI = (float)(1.0 - 1e-4);   // torch's clamp bounds, the Python floats cast to fp32

// one object of the tile's list: centre, radius and gaussian2D's RN(sigma * sigma)
struct CtObj { int cx, cy, r; double s2; };

// gaussian2D(2r + 1, sigma = (2r + 1) / 6) at offset (dx, dy) from the centre, |dx|, |dy| <= r, rounded to fp32
__device__ __forceinline__ float ct_gauss(double s2, int dx, int dy)
{
    const double ddx = (double)dx, ddy = (double)dy;
    const double e = __dadd_rn(__ddiv_rn(__dmul_rn(ddx, ddx), s2), __ddiv_rn(__dmul_rn(ddy, ddy), s2));
    const double g = exp(__dmul_rn(-e, 0.5));         // -e / 2, exact
    return g < 0x1p-52 ? 0.f : __double2float_rn(g);
}

// Stages the objects of image b with class c whose window meets the CTA's tile into s_obj; returns their count.
// Any object values are safe: a class outside [0, C), a centre off the image, a negative radius or ct_01 != 1 match
// nothing.  The list's order does not matter (the target is a maximum).
__device__ __forceinline__ int ct_stage(const CtArgs &a, int b, int c, int x0, int y0, CtObj *s_obj, int *s_n)
{
    if (threadIdx.x == 0) *s_n = 0;
    __syncthreads();
    const long long HW = (long long)a.H * a.W;
    for (int j = threadIdx.x; j < a.M; j += blockDim.x) {
        const size_t o = (size_t)b * a.M + j;
        const long long ind = a.ct_ind[o];
        const int r = a.ct_radius[o];
        if (a.ct_01[o] != 1.f || a.ct_cls[o] != (long long)c || r < 0 || ind < 0 || ind >= HW) continue;
        const int cy = (int)(ind / a.W), cx = (int)(ind - (long long)cy * a.W);
        if ((long long)cx + r < x0 || (long long)cx - r > x0 + CT_TW - 1 ||
            (long long)cy + r < y0 || (long long)cy - r > y0 + CT_TH - 1) continue;
        const double sigma = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, (double)r), 1.0), 6.0);   // diameter / 6
        const int k = atomicAdd(s_n, 1);
        s_obj[k] = CtObj{cx, cy, r, __dmul_rn(sigma, sigma)};
    }
    __syncthreads();
    return *s_n;
}

// the target at (x, y) from the staged list
__device__ __forceinline__ float ct_target(const CtObj *s_obj, int n, int x, int y)
{
    float t = 0.f;
    for (int k = 0; k < n; ++k) {
        const CtObj o = s_obj[k];
        const int dx = x - o.cx, dy = y - o.cy;
        if (abs(dx) <= o.r && abs(dy) <= o.r) t = fmaxf(t, ct_gauss(o.s2, dx, dy));
    }
    return t;
}

// net_utils.sigmoid: torch's sigmoid (ct_sigmoid, common.cuh) clamped to [1e-4, 1 - 1e-4], NaN propagated
__device__ __forceinline__ float ct_clamp(float s) { return isnan(s) ? s : fminf(fmaxf(s, CT_LO), CT_HI); }

struct CtTerms { float pos, neg; };

__device__ __forceinline__ CtTerms ct_terms(float x, float t)
{
    const float p = ct_clamp(ct_sigmoid(x));
    const float u = __fsub_rn(1.f, p);
    const float pi = t == 1.f ? 1.f : 0.f, ni = t < 1.f ? 1.f : 0.f;
    const float nw = powf(__fsub_rn(1.f, t), 4.f);
    CtTerms r;
    r.pos = __fmul_rn(__fmul_rn(logf(p), __fmul_rn(u, u)), pi);
    r.neg = __fmul_rn(__fmul_rn(__fmul_rn(logf(u), __fmul_rn(p, p)), nw), ni);
    return r;
}

// autograd's gradient for the logit x, given gy: the gradient of each of the two sums (the same value for both)
__device__ __forceinline__ float ct_grad(float x, float t, float gy, bool with_pos)
{
    const float s = ct_sigmoid(x);
    const float p = ct_clamp(s);
    const float u = __fsub_rn(1.f, p);
    const float pi = t == 1.f ? 1.f : 0.f, ni = t < 1.f ? 1.f : 0.f;
    const float nw = powf(__fsub_rn(1.f, t), 4.f);
    // neg = ((log(u) * p^2) * nw) * ni
    const float g_n2 = __fmul_rn(__fmul_rn(gy, ni), nw);
    const float g_lu = __fmul_rn(g_n2, __fmul_rn(p, p));               // d/d log(u)
    const float g_pp = __fmul_rn(g_n2, logf(u));                       // d/d p^2
    const float gD = __fmul_rn(g_pp, __fmul_rn(2.f, p));               // pow(p, 2): grad * (2 * p^1)
    const float gC = -__fdiv_rn(g_lu, u);                              // log(u) then 1 - p
    float gp = __fadd_rn(gD, gC);
    if (with_pos) {
        // pos = (log(p) * u^2) * pi
        const float g_n6 = __fmul_rn(gy, pi);
        const float g_lp = __fmul_rn(g_n6, __fmul_rn(u, u));           // d/d log(p)
        const float g_q = __fmul_rn(g_n6, logf(p));                    // d/d u^2
        const float gB = -__fmul_rn(g_q, __fmul_rn(2.f, u));           // pow(u, 2) then 1 - p
        const float gA = __fdiv_rn(g_lp, p);                           // log(p)
        gp = __fadd_rn(__fadd_rn(gp, gB), gA);
    }
    const float gs = (s >= CT_LO && s <= CT_HI) ? gp : 0.f;            // clamp_backward
    return __fmul_rn(__fmul_rn(gs, __fsub_rn(1.f, s)), s);             // sigmoid_backward
}

// the tile, class and image a CTA owns, and its staged objects
struct CtTile { int b, c, x, y0; int n; };

__device__ __forceinline__ CtTile ct_tile(const CtArgs &a, CtObj *s_obj, int *s_n)
{
    CtTile t;
    const int tiles_x = (a.W + CT_TW - 1) / CT_TW;
    t.b = blockIdx.z;
    t.c = blockIdx.y;
    const int x0 = (int)(blockIdx.x % tiles_x) * CT_TW, y0 = (int)(blockIdx.x / tiles_x) * CT_TH;
    t.x = x0 + (int)(threadIdx.x % CT_TW);
    t.y0 = y0 + (int)(threadIdx.x / CT_TW);
    t.n = ct_stage(a, t.b, t.c, x0, y0, s_obj, s_n);
    return t;
}

// ct_hm on the device: out [B][C][H][W] contiguous
__global__ void __launch_bounds__(CT_THREADS) ct_target_kernel(CtArgs a)
{
    extern __shared__ CtObj s_obj[];
    __shared__ int s_n;
    const CtTile t = ct_tile(a, s_obj, &s_n);
    if (t.x >= a.W) return;
    float *out = a.out + ((size_t)t.b * a.C + t.c) * ((size_t)a.H * a.W);
#pragma unroll
    for (int i = 0; i < CT_ROWS; ++i) {
        const int y = t.y0 + i * (CT_THREADS / CT_TW);
        if (y < a.H) out[(size_t)y * a.W + t.x] = ct_target(s_obj, t.n, t.x, y);
    }
}

__device__ __forceinline__ const float *ct_logit(const CtArgs &a, int b, int c, int y, int x)
{
    return a.logits + (long long)b * a.ls[0] + (long long)c * a.ls[1] + (long long)y * a.ls[2] + (long long)x * a.ls[3];
}

// the CTA's fp64 sums of the pos and neg terms and its count of t == 1 pixels, in a fixed order -> partials[cta]
__global__ void __launch_bounds__(CT_THREADS) ct_loss_fwd_kernel(CtArgs a)
{
    extern __shared__ CtObj s_obj[];
    __shared__ int s_n;
    __shared__ double s_pos[CT_THREADS / 32], s_neg[CT_THREADS / 32];
    __shared__ int s_cnt[CT_THREADS / 32];
    const CtTile t = ct_tile(a, s_obj, &s_n);
    double pos = 0.0, neg = 0.0;
    int cnt = 0;
    if (t.x < a.W) {
#pragma unroll
        for (int i = 0; i < CT_ROWS; ++i) {
            const int y = t.y0 + i * (CT_THREADS / CT_TW);
            if (y >= a.H) continue;
            const float tg = ct_target(s_obj, t.n, t.x, y);
            const CtTerms r = ct_terms(__ldg(ct_logit(a, t.b, t.c, y, t.x)), tg);
            pos = __dadd_rn(pos, (double)r.pos);
            neg = __dadd_rn(neg, (double)r.neg);
            cnt += tg == 1.f;
        }
    }
    pos = warp_sum(pos);
    neg = warp_sum(neg);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) { s_pos[threadIdx.x >> 5] = pos; s_neg[threadIdx.x >> 5] = neg; s_cnt[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        pos = 0.0; neg = 0.0; cnt = 0;
#pragma unroll
        for (int i = 0; i < CT_THREADS / 32; ++i) { pos += s_pos[i]; neg += s_neg[i]; cnt += s_cnt[i]; }
        const size_t cta = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
        a.pos_part[cta] = pos;
        a.neg_part[cta] = neg;
        a.cnt_part[cta] = cnt;
    }
}

// one CTA: the partials in a fixed order, each sum rounded once to fp32, then the trainer's branch on num_pos
constexpr int CT_FINAL_THREADS = 1024;
__global__ void __launch_bounds__(CT_FINAL_THREADS) ct_loss_final_kernel(const double *pos_part, const double *neg_part,
                                                                        const int *cnt_part, long long nparts,
                                                                        long long *num_pos, float *loss)
{
    __shared__ double s_pos[CT_FINAL_THREADS / 32], s_neg[CT_FINAL_THREADS / 32];
    __shared__ long long s_cnt[CT_FINAL_THREADS / 32];
    double pos = 0.0, neg = 0.0;
    long long cnt = 0;
    for (long long i = threadIdx.x; i < nparts; i += CT_FINAL_THREADS) { pos += pos_part[i]; neg += neg_part[i]; cnt += cnt_part[i]; }
    pos = warp_sum(pos);
    neg = warp_sum(neg);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) { s_pos[threadIdx.x >> 5] = pos; s_neg[threadIdx.x >> 5] = neg; s_cnt[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        pos = 0.0; neg = 0.0; cnt = 0;
        for (int i = 0; i < CT_FINAL_THREADS / 32; ++i) { pos += s_pos[i]; neg += s_neg[i]; cnt += s_cnt[i]; }
        const float pf = __double2float_rn(pos), nf = __double2float_rn(neg);
        *num_pos = cnt;
        *loss = cnt == 0 ? __fsub_rn(0.f, nf) : __fsub_rn(0.f, __fdiv_rn(__fadd_rn(pf, nf), __ll2float_rn(cnt)));
    }
}

// grad [B][C][H][W] contiguous from the scalar upstream gradient and the forward pass's num_pos
__global__ void __launch_bounds__(CT_THREADS) ct_loss_bwd_kernel(CtArgs a)
{
    extern __shared__ CtObj s_obj[];
    __shared__ int s_n;
    const CtTile t = ct_tile(a, s_obj, &s_n);
    if (t.x >= a.W) return;
    // loss = 0 - X: the gradient of X is -g; with positives X = (pos + neg) / num_pos and each sum gets RN(-g / num_pos)
    const long long np = *a.num_pos;
    const float g = -*a.grad_loss;
    const float gy = np == 0 ? g : __fdiv_rn(g, __ll2float_rn(np));
    float *out = a.out + ((size_t)t.b * a.C + t.c) * ((size_t)a.H * a.W);
#pragma unroll
    for (int i = 0; i < CT_ROWS; ++i) {
        const int y = t.y0 + i * (CT_THREADS / CT_TW);
        if (y >= a.H) continue;
        const float tg = ct_target(s_obj, t.n, t.x, y);
        out[(size_t)y * a.W + t.x] = ct_grad(__ldg(ct_logit(a, t.b, t.c, y, t.x)), tg, gy, np != 0);
    }
}

namespace {

dim3 ct_grid(const CtArgs &a)
{
    const unsigned tiles = (unsigned)(((a.W + CT_TW - 1) / CT_TW) * ((a.H + CT_TH - 1) / CT_TH));
    return dim3(tiles, (unsigned)a.C, (unsigned)a.B);
}

long long ct_nparts(int B, int C, int H, int W)
{
    return (long long)B * C * (((long long)W + CT_TW - 1) / CT_TW) * (((long long)H + CT_TH - 1) / CT_TH);
}

// num_pos at offset 0, then the three partial arrays, each 256-byte aligned
size_t ct_loss_workspace_bytes(int B, int C, int H, int W, size_t *pos_offset, size_t *neg_offset, size_t *cnt_offset)
{
    const size_t n = (size_t)ct_nparts(B, C, H, W);
    const size_t po = 256, no = po + (n * sizeof(double) + 255) / 256 * 256, co = no + (n * sizeof(double) + 255) / 256 * 256;
    if (pos_offset) *pos_offset = po;
    if (neg_offset) *neg_offset = no;
    if (cnt_offset) *cnt_offset = co;
    return co + (n * sizeof(int) + 255) / 256 * 256;
}

constexpr int CT_MAX_M = 1024;      // the tile's staged objects take at most 24 KB of shared memory
size_t ct_smem_bytes(int M) { return (size_t)(M > 0 ? M : 1) * sizeof(CtObj); }

// the arguments every CenterNet-loss entry shares; fills the object and size fields of `a`
int ct_common(CtArgs &a, const int64_t *ct_ind, const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01,
              int32_t B, int32_t M, int32_t C, int32_t H, int32_t W)
{
    if (B < 0 || M < 0 || C < 0 || H < 0 || W < 0)
        return fail(PVB_ERR_INVALID, "negative size (B=%d M=%d C=%d H=%d W=%d)", B, M, C, H, W);
    if (M > CT_MAX_M) return fail(PVB_ERR_INVALID, "M must be at most %d objects per image, got %d", CT_MAX_M, M);
    if (B > 65535) return fail(PVB_ERR_INVALID, "B must be at most 65535, got %d", B);
    if (C > 65535) return fail(PVB_ERR_INVALID, "C must be at most 65535, got %d", C);
    if ((long long)H * W > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    if ((long long)B * M > 0 && (!ct_ind || !ct_radius || !ct_cls || !ct_01)) return fail(PVB_ERR_INVALID, "NULL tensor");
    a = CtArgs{};
    a.ct_ind = reinterpret_cast<const long long *>(ct_ind);
    a.ct_radius = ct_radius;
    a.ct_cls = reinterpret_cast<const long long *>(ct_cls);
    a.ct_01 = ct_01;
    a.B = B; a.M = M; a.C = C; a.H = H; a.W = W;
    return PVB_OK;
}

int ct_logits(CtArgs &a, const float *logits, const int64_t *logit_stride)
{
    if (!logit_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    for (int i = 0; i < 4; ++i) {
        if (logit_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
        a.ls[i] = logit_stride[i];
    }
    if ((long long)a.B * a.C * a.H * a.W > 0 && !logits) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.logits = logits;
    return PVB_OK;
}

// checks the workspace and fills the workspace fields of `a`
int ct_workspace(CtArgs &a, const void *workspace, size_t workspace_bytes)
{
    size_t po = 0, no = 0, co = 0;
    if (int rc = check_workspace(ct_loss_workspace_bytes(a.B, a.C, a.H, a.W, &po, &no, &co), workspace, workspace_bytes))
        return rc;
    char *ws = static_cast<char *>(const_cast<void *>(workspace));
    a.num_pos = reinterpret_cast<long long *>(ws);
    a.pos_part = reinterpret_cast<double *>(ws + po);
    a.neg_part = reinterpret_cast<double *>(ws + no);
    a.cnt_part = reinterpret_cast<int *>(ws + co);
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

// lib/datasets/tless*/ct.py ct_hm: data_utils.draw_umich_gaussian per object
PVB_API int pvb_ct_target(const int64_t *ct_ind, const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01,
                          float *ct_hm, int32_t B, int32_t M, int32_t C, int32_t H, int32_t W, pvb_stream_t stream)
{
    CtArgs a;
    if (int rc = ct_common(a, ct_ind, ct_radius, ct_cls, ct_01, B, M, C, H, W)) return rc;
    if ((long long)B * C * H * W == 0) return PVB_OK;
    if (!ct_hm) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.out = ct_hm;
    ct_target_kernel<<<ct_grid(a), CT_THREADS, ct_smem_bytes(M), static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "ct target kernel");
}

PVB_API size_t pvb_ct_loss_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W)
{
    if (B < 0 || C < 0 || H < 0 || W < 0) return 0;
    return ct_loss_workspace_bytes(B, C, H, W, nullptr, nullptr, nullptr);
}

// lib/train/trainers/ct.py:20-21, the forward pass
PVB_API int pvb_ct_loss_forward(const float *logits, const int64_t *logit_stride, const int64_t *ct_ind,
                                const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01, float *loss,
                                int32_t B, int32_t M, int32_t C, int32_t H, int32_t W, void *workspace,
                                size_t workspace_bytes, pvb_stream_t stream)
{
    CtArgs a;
    if (int rc = ct_common(a, ct_ind, ct_radius, ct_cls, ct_01, B, M, C, H, W)) return rc;
    if (int rc = ct_logits(a, logits, logit_stride)) return rc;
    if (!loss) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (int rc = ct_workspace(a, workspace, workspace_bytes)) return rc;
    a.loss = loss;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long nparts = ct_nparts(B, C, H, W);
    if (nparts > 0) ct_loss_fwd_kernel<<<ct_grid(a), CT_THREADS, ct_smem_bytes(M), st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        ct_loss_final_kernel<<<1, CT_FINAL_THREADS, 0, st>>>(a.pos_part, a.neg_part, a.cnt_part, nparts, a.num_pos, loss);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "ct loss forward kernels");
}

// lib/train/trainers/ct.py:20-21, autograd's backward pass of it
PVB_API int pvb_ct_loss_backward(const float *logits, const int64_t *logit_stride, const int64_t *ct_ind,
                                 const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01,
                                 const float *grad_loss, float *grad_logits, int32_t B, int32_t M, int32_t C, int32_t H,
                                 int32_t W, const void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    CtArgs a;
    if (int rc = ct_common(a, ct_ind, ct_radius, ct_cls, ct_01, B, M, C, H, W)) return rc;
    if (int rc = ct_logits(a, logits, logit_stride)) return rc;
    if ((long long)B * C * H * W == 0) return PVB_OK;
    if (!grad_loss || !grad_logits) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (int rc = ct_workspace(a, workspace, workspace_bytes)) return rc;
    a.grad_loss = grad_loss;
    a.out = grad_logits;
    ct_loss_bwd_kernel<<<ct_grid(a), CT_THREADS, ct_smem_bytes(M), static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "ct loss backward kernel");
}

} // extern "C"
