// Deformable PSROI pooling of DCNv2, fp32, forward and backward: the device twin of clean-pvnet's
// lib/csrc/dcn_v2/src/cuda/dcn_v2_psroi_pooling_cuda.cu (DESIGN.md section 8m).
//
// Output (n, c, ph, pw) of [n_roi, C, P, P] averages the bilinear samples of bin (ph, pw) of ROI n, shifted by the
// offset of its part cell and class.  The sample geometry (position, validity, corners, weights) depends on the ROI,
// the bin and the class, never on the channel, so each CTA computes it once into a shared-memory table and every
// channel of the class reads it.  The reference recomputes it, three fp32 divisions and several fp64 operations
// included, in each of its n*C*P^2 threads.
//
// The forward is the reference build's bit for bit, count included.  Its arithmetic, read off the SASS of the
// reference kernel compiled for sm_90a (the source's double expressions are not what runs):
//   start = fma(round(x1), scale, -0.5f)            end = fma(round(x2) + 1.f, scale, -0.5f)
//   roi_w = float(fmax(double(end - start), 0.1))   (the subtraction in fp32; NaN gives 0.1f)
//   bin_w = roi_w / P, sub_w = bin_w / spp          (IEEE divisions)
//   part_w = floor(float(pw) / P * part_size)       trans_x = trans * trans_std (0 with no_trans)
//   wstart = fma(trans_x, roi_w, fma(float(pw), bin_w, start))
//   w = fma(float(iw), sub_w, wstart), skipped when w < -0.5 or w > W - 0.5 (fp64, NaN passes), then
//   clamped to [0, W - 1] in fp64 (NaN becomes 0)
//   value = fma(q11, v22, fma(q10, v21, fma(q00, v11, q01 * v12))), each q a rounded product of (1 - dx), dx, ...
//   sum += value in ih-major order; out = sum / count, 0 when count == 0
// and likewise for h.  The weights are rounded products on their own in the reference too, so the table holds them.
//
// The backward recomputes the counts.  grad_input takes four float atomics per valid sample, as the reference's does,
// so its low bits depend on the order the atomics land in.  grad_trans has no atomics: one CTA owns one (ROI, class,
// part cell) and sums its terms over (channel, bin, sample) in a fixed assignment to threads and a fixed reduction
// tree, so it is bitwise equal run to run and a ROI's value does not depend on the other ROIs.
#include "api.h"

namespace pvb {

namespace {

constexpr int NT = 256;           // threads per CTA
constexpr int TBL = 1024;         // sample-table entries per CTA: every bin chunk holds all samples of its bins
constexpr int MAX_SPP = 32;       // so sample_per_part^2 <= TBL

struct PoolArgs {
    const float *input;           // [B][C][H][W]
    const float *rois;            // [n][5]: batch, x1, y1, x2, y2
    const float *trans;           // [n][2*nc][ps][ps] (unread with no_trans)
    float *out, *count;           // [n][C][P][P] (forward; count may be NULL)
    const float *grad_out;        // [n][C][P][P] (backward)
    float *grad_input, *grad_trans;
    int B, C, H, W, n, P, ps, spp, nc, cec, no_trans;
    int nb, nchunk;               // forward: bins per CTA chunk, chunks per (ROI, class)
    float scale, trans_std;
};

// the per-ROI scalars, as the reference rounds them
struct Roi { int b; float start_w, start_h, roi_w, roi_h, bin_w, bin_h, sub_w, sub_h; };

__device__ __forceinline__ Roi roi_geom(const PoolArgs &a, int n)
{
    const float *r = a.rois + 5ll * n;
    Roi g;
    g.b = __float2int_rz(__ldg(r));                                    // device truncation; NaN gives 0
    const float x1 = roundf(__ldg(r + 1)), y1 = roundf(__ldg(r + 2));
    const float x2 = roundf(__ldg(r + 3)), y2 = roundf(__ldg(r + 4));
    g.start_w = __fmaf_rn(x1, a.scale, -0.5f);
    g.start_h = __fmaf_rn(y1, a.scale, -0.5f);
    const float end_w = __fmaf_rn(__fadd_rn(x2, 1.f), a.scale, -0.5f);
    const float end_h = __fmaf_rn(__fadd_rn(y2, 1.f), a.scale, -0.5f);
    g.roi_w = (float)fmax((double)__fsub_rn(end_w, g.start_w), 0.1);
    g.roi_h = (float)fmax((double)__fsub_rn(end_h, g.start_h), 0.1);
    g.bin_w = __fdiv_rn(g.roi_w, (float)a.P);
    g.bin_h = __fdiv_rn(g.roi_h, (float)a.P);
    g.sub_w = __fdiv_rn(g.bin_w, (float)a.spp);
    g.sub_h = __fdiv_rn(g.bin_h, (float)a.spp);
    return g;
}

__device__ __forceinline__ int part_of(int p, const PoolArgs &a)
{
    const int q = (int)floorf(__fmul_rn(__fdiv_rn((float)p, (float)a.P), (float)a.ps));
    return min(q, a.ps - 1);      // never binds (checked for P, part_size <= 256); keeps the index in bounds
}

// offset into trans of (ROI n, class k, x or y, part cell)
__device__ __forceinline__ long long trans_at(const PoolArgs &a, int n, int k, int xy, int cy, int cx)
{
    return ((((long long)n * a.nc + k) * 2 + xy) * a.ps + cy) * a.ps + cx;
}

// One sample of a bin: `off` is the top-left corner's offset in a plane (-1: skipped), `step` bit 0 says whether the
// right corners are one column over and bit 1 whether the lower ones are one row down (ceil != floor)
struct Sample { int off, step; float q00, q01, q10, q11, dx, dy; };

__device__ __forceinline__ Sample sample_at(const PoolArgs &a, const Roi &g, int n, int k, int ph, int pw, int s)
{
    float tx = 0.f, ty = 0.f;
    if (!a.no_trans) {
        const int cy = part_of(ph, a), cx = part_of(pw, a);
        tx = __fmul_rn(__ldg(a.trans + trans_at(a, n, k, 0, cy, cx)), a.trans_std);
        ty = __fmul_rn(__ldg(a.trans + trans_at(a, n, k, 1, cy, cx)), a.trans_std);
    }
    const float wstart = __fmaf_rn(tx, g.roi_w, __fmaf_rn((float)pw, g.bin_w, g.start_w));
    const float hstart = __fmaf_rn(ty, g.roi_h, __fmaf_rn((float)ph, g.bin_h, g.start_h));
    const int ih = s / a.spp, iw = s - ih * a.spp;
    const float w = __fmaf_rn((float)iw, g.sub_w, wstart);
    const float h = __fmaf_rn((float)ih, g.sub_h, hstart);
    Sample t;
    const double wd = w, hd = h;
    if (wd < -0.5 || wd > a.W - 0.5 || hd < -0.5 || hd > a.H - 0.5) {
        t.off = -1; t.step = 0; t.q00 = t.q01 = t.q10 = t.q11 = t.dx = t.dy = 0.f;
        return t;
    }
    const float wc = (float)fmin(fmax(wd, 0.), a.W - 1.);
    const float hc = (float)fmin(fmax(hd, 0.), a.H - 1.);
    const int x1 = (int)floorf(wc), x2 = (int)ceilf(wc), y1 = (int)floorf(hc), y2 = (int)ceilf(hc);
    t.dx = __fsub_rn(wc, (float)x1);
    t.dy = __fsub_rn(hc, (float)y1);
    const float ux = __fsub_rn(1.f, t.dx), uy = __fsub_rn(1.f, t.dy);
    t.q00 = __fmul_rn(ux, uy); t.q01 = __fmul_rn(ux, t.dy); t.q10 = __fmul_rn(t.dx, uy); t.q11 = __fmul_rn(t.dx, t.dy);
    t.off = y1 * a.W + x1;
    t.step = (x2 - x1) | ((y2 - y1) << 1);
    return t;
}

// shared-memory sample table, entry e = s * nbins + bin (conflict-free for threads on consecutive bins)
struct Table { int off[TBL]; int step[TBL]; float q[4][TBL]; };

__device__ __forceinline__ void put(Table &t, int e, const Sample &s)
{
    t.off[e] = s.off; t.step[e] = s.step;
    t.q[0][e] = s.q00; t.q[1][e] = s.q01; t.q[2][e] = s.q10; t.q[3][e] = s.q11;
}

// grid: n * nc * nchunk CTAs, each (ROI n, class k, bins chunk*nb .. + nb - 1) over every channel of class k;
// threads over (channel, bin) pairs, bin fastest
__global__ void __launch_bounds__(NT) dcn_pool_forward_kernel(PoolArgs a)
{
    __shared__ Table tb;
    const int j = blockIdx.x % a.nchunk, k = (blockIdx.x / a.nchunk) % a.nc, n = blockIdx.x / (a.nchunk * a.nc);
    const int P2 = a.P * a.P, S = a.spp * a.spp, b0 = j * a.nb, nbins = min(a.nb, P2 - b0);
    const Roi g = roi_geom(a, n);
    const bool live = g.b >= 0 && g.b < a.B;
    if (live) {
        for (int e = threadIdx.x; e < nbins * S; e += NT) {
            const int s = e / nbins, bin = b0 + (e - s * nbins);
            put(tb, e, sample_at(a, g, n, k, bin / a.P, bin % a.P, s));
        }
    }
    __syncthreads();
    const long long HW = (long long)a.H * a.W;
    for (int i = threadIdx.x; i < a.cec * nbins; i += NT) {
        const int c = k * a.cec + i / nbins, bl = i % nbins;
        const long long o = ((long long)n * a.C + c) * P2 + b0 + bl;
        float sum = 0.f;
        int cnt = 0;
        if (live) {
            const float *plane = a.input + ((long long)g.b * a.C + c) * HW;
            for (int s = 0; s < S; ++s) {
                const int e = s * nbins + bl, off = tb.off[e];
                if (off < 0) continue;
                const int st = tb.step[e], ox = st & 1, oy = (st >> 1) * a.W;
                const float v11 = __ldg(plane + off), v12 = __ldg(plane + off + oy);
                const float v21 = __ldg(plane + off + ox), v22 = __ldg(plane + off + oy + ox);
                const float val = __fmaf_rn(tb.q[3][e], v22, __fmaf_rn(tb.q[2][e], v21,
                                            __fmaf_rn(tb.q[0][e], v11, __fmul_rn(tb.q[1][e], v12))));
                sum = __fadd_rn(sum, val);
                ++cnt;
            }
        }
        a.out[o] = cnt == 0 ? 0.f : __fdiv_rn(sum, (float)cnt);
        if (a.count) a.count[o] = (float)cnt;
    }
}

// the bins [lo, hi) of one axis whose part index is `cell` (part_of is non-decreasing in the bin)
__device__ __forceinline__ void bins_of_cell(const PoolArgs &a, int cell, int &lo, int &hi)
{
    lo = 0;
    while (lo < a.P && part_of(lo, a) < cell) ++lo;
    hi = lo;
    while (hi < a.P && part_of(hi, a) == cell) ++hi;
}

__device__ __forceinline__ float block_sum(float v, float *red)
{
    for (int d = 16; d > 0; d >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, d));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = red[0];
    for (int w = 1; w < NT / 32; ++w) t = __fadd_rn(t, red[w]);
    return t;
}

// grid: n * nc * ps^2 CTAs, each (ROI n, class k, part cell (cy, cx)) over the bins that read that cell and every
// channel of class k; threads over (channel, bin, sample) terms, sample fastest.  Writes grad_trans of its cell
// (unless no_trans) and adds to grad_input.
__global__ void __launch_bounds__(NT) dcn_pool_backward_kernel(PoolArgs a)
{
    __shared__ Table tb;
    __shared__ float tdx[TBL], tdy[TBL];
    __shared__ int cnt_s[TBL];
    __shared__ float red[NT / 32];
    const int ps2 = a.ps * a.ps;
    const int cell = blockIdx.x % ps2, k = (blockIdx.x / ps2) % a.nc, n = blockIdx.x / (ps2 * a.nc);
    const int cy = cell / a.ps, cx = cell % a.ps;
    int ph0, ph1, pw0, pw1;
    bins_of_cell(a, cy, ph0, ph1);
    bins_of_cell(a, cx, pw0, pw1);
    const int nbw = pw1 - pw0, nbc = (ph1 - ph0) * nbw;
    const int P2 = a.P * a.P, S = a.spp * a.spp, nb = TBL / S;
    const Roi g = roi_geom(a, n);
    const bool live = g.b >= 0 && g.b < a.B;
    const long long HW = (long long)a.H * a.W;
    float gx = 0.f, gy = 0.f;
    for (int cb = 0; live && cb < nbc; cb += nb) {
        const int nbins = min(nb, nbc - cb);
        __syncthreads();                                     // the previous chunk's table is consumed
        for (int e = threadIdx.x; e < nbins; e += NT) cnt_s[e] = 0;
        __syncthreads();
        for (int e = threadIdx.x; e < nbins * S; e += NT) {
            const int s = e / nbins, bl = e - s * nbins, bin = cb + bl;
            const Sample t = sample_at(a, g, n, k, ph0 + bin / nbw, pw0 + bin % nbw, s);
            put(tb, e, t);
            tdx[e] = t.dx; tdy[e] = t.dy;
            if (t.off >= 0) atomicAdd(&cnt_s[bl], 1);       // integer: the count does not depend on the order
        }
        __syncthreads();
        const float *in_b = a.input + (long long)g.b * a.C * HW;
        float *gin_b = a.grad_input + (long long)g.b * a.C * HW;
        for (int i = threadIdx.x; i < a.cec * nbins * S; i += NT) {
            const int s = i % S, r = i / S, bl = r % nbins, c = k * a.cec + r / nbins;
            const int e = s * nbins + bl, off = tb.off[e];
            if (off < 0) continue;
            const int bin = cb + bl, ph = ph0 + bin / nbw, pw = pw0 + bin % nbw;
            const float diff = __fdiv_rn(__ldg(a.grad_out + ((long long)n * a.C + c) * P2 + ph * a.P + pw),
                                         (float)cnt_s[bl]);
            const int st = tb.step[e], ox = st & 1, oy = (st >> 1) * a.W;
            float *gp = gin_b + (long long)c * HW + off;
            atomicAdd(gp, __fmul_rn(tb.q[0][e], diff));
            atomicAdd(gp + oy, __fmul_rn(tb.q[1][e], diff));
            atomicAdd(gp + ox, __fmul_rn(tb.q[2][e], diff));
            atomicAdd(gp + oy + ox, __fmul_rn(tb.q[3][e], diff));
            if (a.no_trans) continue;
            const float *ip = in_b + (long long)c * HW + off;
            const float u00 = __ldg(ip), u01 = __ldg(ip + oy), u10 = __ldg(ip + ox), u11 = __ldg(ip + oy + ox);
            const float dx = tdx[e], dy = tdy[e];
            // d(value)/dw and d(value)/dh, times trans_std * diff * roi_w (roi_h): the reference's terms (:259-262)
            const float dvx = __fmaf_rn(dy, __fsub_rn(u11, u01), __fmul_rn(__fsub_rn(1.f, dy), __fsub_rn(u10, u00)));
            const float dvy = __fmaf_rn(dx, __fsub_rn(u11, u10), __fmul_rn(__fsub_rn(1.f, dx), __fsub_rn(u01, u00)));
            const float sd = __fmul_rn(a.trans_std, diff);
            gx = __fmaf_rn(__fmul_rn(dvx, sd), g.roi_w, gx);
            gy = __fmaf_rn(__fmul_rn(dvy, sd), g.roi_h, gy);
        }
    }
    if (a.no_trans) return;
    gx = block_sum(gx, red);
    gy = block_sum(gy, red);
    if (threadIdx.x == 0) {
        a.grad_trans[trans_at(a, n, k, 0, cy, cx)] = gx;
        a.grad_trans[trans_at(a, n, k, 1, cy, cx)] = gy;
    }
}

// checks a pooling descriptor and fills the kernels' argument block; PVB_OK or PVB_ERR_INVALID (no CUDA call)
int pool_args(const pvb_dcn_pool_desc *d, PoolArgs &a)
{
    if (!d) return fail(PVB_ERR_INVALID, "descriptor is NULL");
    if (d->B < 0 || d->C < 1 || d->H < 1 || d->W < 1 || d->n_roi < 0 || d->pooled_size < 1 || d->part_size < 1)
        return fail(PVB_ERR_INVALID, "bad shape B=%d C=%d H=%d W=%d n_roi=%d pooled_size=%d part_size=%d", d->B, d->C,
                    d->H, d->W, d->n_roi, d->pooled_size, d->part_size);
    if (d->output_dim != d->C)
        return fail(PVB_ERR_INVALID, "output_dim=%d must equal the input's channels C=%d", d->output_dim, d->C);
    if (d->group_size != 1)
        return fail(PVB_ERR_INVALID, "group_size=%d: only group_size 1 is supported (position-sensitive pooling "
                    "needs C = output_dim * group_size^2)", d->group_size);
    if (d->sample_per_part < 1 || d->sample_per_part > MAX_SPP)
        return fail(PVB_ERR_INVALID, "sample_per_part=%d must be in [1, %d]", d->sample_per_part, MAX_SPP);
    const int nc = d->no_trans ? 1 : d->num_classes;
    if (nc < 1 || d->C % nc)
        return fail(PVB_ERR_INVALID, "trans has %d classes (trans.size(1) / 2); output_dim=%d must be a multiple of it",
                    nc, d->C);
    const long long P2 = (long long)d->pooled_size * d->pooled_size;
    if ((long long)d->n_roi * d->C * P2 >= (1ll << 31) || (long long)d->B * d->C * d->H * d->W >= (1ll << 31) ||
        (long long)d->n_roi * 2 * nc * d->part_size * d->part_size >= (1ll << 31))
        return fail(PVB_ERR_INVALID, "n_roi*C*P^2, B*C*H*W or n_roi*2*num_classes*part_size^2 >= 2^31");
    a = PoolArgs{};
    a.B = d->B; a.C = d->C; a.H = d->H; a.W = d->W; a.n = d->n_roi; a.P = d->pooled_size; a.ps = d->part_size;
    a.spp = d->sample_per_part; a.nc = nc; a.cec = d->C / nc; a.no_trans = d->no_trans != 0;
    a.scale = d->spatial_scale; a.trans_std = d->trans_std;
    a.nb = (int)(TBL / (a.spp * a.spp) < P2 ? TBL / (a.spp * a.spp) : P2);
    a.nchunk = (int)((P2 + a.nb - 1) / a.nb);
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_dcn_pool_forward(const pvb_dcn_pool_desc *d, const float *input, const float *rois, const float *trans,
                                 float *out, float *count, pvb_stream_t stream)
{
    PoolArgs a;
    if (int rc = pool_args(d, a)) return rc;
    if (a.n == 0) return PVB_OK;
    if ((!input && a.B) || !rois || (!trans && !a.no_trans) || !out) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.input = input; a.rois = rois; a.trans = trans; a.out = out; a.count = count;
    // n_roi * num_classes * chunks <= n_roi * C * P^2 < 2^31
    dcn_pool_forward_kernel<<<(unsigned)((long long)a.n * a.nc * a.nchunk), NT, 0, static_cast<cudaStream_t>(stream)>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "dcn pool forward kernel");
}

PVB_API int pvb_dcn_pool_backward(const pvb_dcn_pool_desc *d, const float *input, const float *rois, const float *trans,
                                  const float *grad_out, float *grad_input, float *grad_trans, pvb_stream_t stream)
{
    PoolArgs a;
    if (int rc = pool_args(d, a)) return rc;
    const bool any_input = a.B > 0;
    if ((any_input && (!input || !grad_input)) ||
        (a.n > 0 && (!rois || !grad_out || (!a.no_trans && (!trans || !grad_trans)))))
        return fail(PVB_ERR_INVALID, "NULL tensor");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (any_input) {
        cudaError_t e = cudaMemsetAsync(grad_input, 0, (size_t)a.B * a.C * a.H * a.W * sizeof(float), st);
        if (e != cudaSuccess) return cuda_fail(e, "dcn pool backward");
    }
    if (a.n == 0) return PVB_OK;
    a.input = input; a.rois = rois; a.trans = trans; a.grad_out = grad_out; a.grad_input = grad_input;
    a.grad_trans = grad_trans;
    // n_roi * num_classes * part_size^2 is half the size of trans, < 2^31
    dcn_pool_backward_kernel<<<(unsigned)((long long)a.n * a.nc * a.ps * a.ps), NT, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "dcn pool backward kernel");
}

} // extern "C"
