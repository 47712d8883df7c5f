// ct_decode.cu -- the CenterNet detector's decode, Network.decode_detection (lib/networks/ct/dla.py:20-26), for B
// images in two launches (DESIGN.md section 8j).
//
// The reference runs torch.sigmoid, ct_decode.decode_ct_hm (lib/utils/ct/ct_decode.py:6-75) and
// data_utils.clip_to_image (lib/utils/data_utils.py:373-377).  Per image b, class c and pixel i = y * W + x:
//   heat = ct_sigmoid(logit)                                        (common.cuh: CUDA torch's fp32 sigmoid)
//   hmax = max_pool2d(heat, 3, stride 1, pad 1)                     (padding never wins; a NaN in the window wins)
//   v    = heat * (hmax == heat)                                    (peaks keep heat, the rest become 0, a NaN stays NaN)
// then a top-K per class and a top-K over the C*K winners, which is one top-K of the image's C*H*W values under the
// total order (v descending with NaN above +inf, then c ascending, then i ascending), given CUDA torch's tie rule of
// ascending index (pinned on the H100 by tests/test_gpu_ct_decode.py).  Each value is a unique 64-bit key:
//   key = vbits << 32 | (0xffffffff - (c * H*W + i)),   vbits = bits of v (v >= +0), 0xffffffff for NaN
// so a larger key ranks first, and key 0 is free to pad the lists with (c * H*W + i < 2^31).
//
// ct_decode_tile_kernel: one CTA per (32x32 tile, class, image).  It stages the tile's sigmoid with a one-pixel halo in
// shared memory and applies the peak test.  Its list is its Lk = min(K, 1024) largest keys, descending: the non-zero
// values (peaks and NaN), each placed at its rank among them, then the zero values, whose order is the tile's pixel
// order.  The image's top K is inside the union of its lists, and the K-th largest key of any
// one list bounds the image's K-th largest key from below (theta).
// ct_decode_select_kernel: one CTA per image.  A radix select over the list entries >= theta finds the K-th largest
// key; the K keys at or above it are gathered, each ranked by counting the larger ones, and decoded:
//   ys = i div W, xs = i mod W (exact: H*W < 2^24), class = c, score = v;  w = wh[b, 0, ys, xs], h = wh[b, 1, ys, xs]
//   box = (RN(xs - RN(w/2)), RN(ys - RN(h/2)), RN(xs + RN(w/2)), RN(ys + RN(h/2)))
//   clip: x0, y0 = clamp(min=0), x1 = clamp(max=W-1), y1 = clamp(max=H-1), NaN passed through as torch.clamp does.
// Nothing depends on CTA scheduling: the lists are written per CTA, every selection step counts exactly, and the
// output position of a key is its rank.
#include "api.h"
#include "common.cuh"

namespace pvb {

struct CtDecodeArgs {
    const float *hm;          // [B][C][H][W] logits at element strides hs
    long long hs[4];
    const float *wh;          // [B][2][H][W] at element strides ws
    long long ws[4];
    int B, C, H, W, K, clip;
    int T, Lk;                // tiles per class and entries per list
    long long L;              // lists per image, C * T
    unsigned long long *lists;   // workspace [B][L][Lk]: each tile's largest keys, descending
    unsigned long long *sel;     // workspace [B][K]: the image's K selected keys, unordered
    float *ct;                // [B][K][2] (xs, ys)
    float *det;               // [B][K][6] (x0, y0, x1, y1, score, class)
};

constexpr int CD_T = 32;                           // tile side
constexpr int CD_N = CD_T * CD_T;                  // keys per tile
constexpr int CD_THREADS = 256;
constexpr int CD_HALO = CD_T + 2;
constexpr int CD_SEL_THREADS = 1024;
constexpr unsigned long long CD_NAN_BITS = 0xffffffffull;

__global__ void __launch_bounds__(CD_THREADS) ct_decode_tile_kernel(CtDecodeArgs a)
{
    __shared__ float s_heat[CD_HALO][CD_HALO + 1];
    __shared__ unsigned long long s_key[CD_N];       // the tile's non-zero keys, unordered
    __shared__ unsigned s_zc[CD_N / 32];               // zero count of each (iteration, warp) -> its exclusive prefix
    __shared__ int s_np;
    __shared__ unsigned s_nz;
    static_assert(CD_N / 32 == 32, "the zero-count scan is one warp wide");
    const int tiles_x = (a.W + CD_T - 1) / CD_T;
    const int t = blockIdx.x, c = blockIdx.y, b = blockIdx.z;
    const int x0 = (t % tiles_x) * CD_T, y0 = (t / tiles_x) * CD_T;
    const float *hm = a.hm + (long long)b * a.hs[0] + (long long)c * a.hs[1];
    const float NEG = __int_as_float(0xff800000);  // outside the image: max_pool2d's -inf padding

    for (int k = threadIdx.x; k < CD_HALO * CD_HALO; k += CD_THREADS) {
        const int hy = k / CD_HALO, hx = k - hy * CD_HALO;
        const int y = y0 - 1 + hy, x = x0 - 1 + hx;
        float h = NEG;
        if (y >= 0 && y < a.H && x >= 0 && x < a.W) h = ct_sigmoid(__ldg(hm + (long long)y * a.hs[2] + (long long)x * a.hs[3]));
        s_heat[hy][hx] = h;
    }
    __syncthreads();

    // Each pixel's key.  The non-zero values (peaks and NaN) are compacted into s_key; a zero value's key only depends
    // on its position, so the tile's zeros rank after its non-zero values in tile order (ascending pixel index).
    const unsigned base = (unsigned)c * (unsigned)(a.H * a.W);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long mine[CD_N / CD_THREADS];
    unsigned zmask[CD_N / CD_THREADS];
    if (threadIdx.x == 0) s_np = 0;
    __syncthreads();
#pragma unroll
    for (int it = 0; it < CD_N / CD_THREADS; ++it) {
        const int p = it * CD_THREADS + threadIdx.x;
        const int ty = p / CD_T, tx = p - ty * CD_T;
        const int y = y0 + ty, x = x0 + tx;
        unsigned long long key = 0;
        if (y < a.H && x < a.W) {
            float m = NEG;                             // CUDA max_pool2d's scan: val > max || isnan(val)
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const float v = s_heat[ty + dy][tx + dx];
                    if (v > m || isnan(v)) m = v;
                }
            const float h = s_heat[ty + 1][tx + 1];
            const float v = __fmul_rn(h, m == h ? 1.f : 0.f);
            const unsigned long long vb = isnan(v) ? CD_NAN_BITS : (unsigned long long)__float_as_uint(v);
            key = vb << 32 | (unsigned long long)(0xffffffffu - (base + (unsigned)(y * a.W + x)));
        }
        mine[it] = key;
        const bool zero = key != 0 && (key >> 32) == 0;
        zmask[it] = __ballot_sync(0xffffffffu, zero);
        if (lane == 0) s_zc[it * (CD_THREADS / 32) + warp] = __popc(zmask[it]);
        if (key >> 32) s_key[atomicAdd(&s_np, 1)] = key;
    }
    __syncthreads();
    if (warp == 0) {                                   // exclusive scan of the 32 (iteration, warp) zero counts
        const unsigned v = s_zc[lane];
        unsigned inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += u;
        }
        s_zc[lane] = inc - v;
        if (lane == 31) s_nz = inc;
    }
    __syncthreads();

    const int np = s_np, nreal = np + (int)s_nz;
    unsigned long long *out = a.lists + ((size_t)b * a.L + (size_t)c * a.T + t) * a.Lk;
    // the non-zero keys: rank = number of larger ones (keys are unique), written when it is below Lk
    for (int i = threadIdx.x; i < np; i += CD_THREADS) {
        const unsigned long long key = s_key[i];
        int r = 0;
        for (int j = 0; j < np; ++j) r += s_key[j] > key;
        if (r < a.Lk) out[r] = key;
    }
    // the zero keys after them, in tile order
#pragma unroll
    for (int it = 0; it < CD_N / CD_THREADS; ++it)
        if ((zmask[it] >> lane) & 1u) {
            const int r = np + (int)s_zc[it * (CD_THREADS / 32) + warp] + __popc(zmask[it] & ((1u << lane) - 1u));
            if (r < a.Lk) out[r] = mine[it];
        }
    // padding past the tile's pixels
    for (int r = nreal + threadIdx.x; r < a.Lk; r += CD_THREADS) out[r] = 0ull;
}

// calls f(key) for every list entry of image b with key >= lo (lo >= 1), one warp per list; the lists are sorted
// descending, so a warp leaves a list at its first 32-key chunk that is not entirely >= lo
template <class F>
__device__ __forceinline__ void cd_for_each(const CtDecodeArgs &a, int b, unsigned long long lo, F f)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long l = warp; l < a.L; l += CD_SEL_THREADS / 32) {
        const unsigned long long *p = a.lists + ((size_t)b * a.L + l) * a.Lk;
        for (int s = 0; s < a.Lk; s += 32) {
            const unsigned long long key = s + lane < a.Lk ? p[s + lane] : 0ull;
            const bool ok = key >= lo;
            if (ok) f(key);
            if (!__all_sync(0xffffffffu, ok)) break;
        }
    }
}

__global__ void __launch_bounds__(CD_SEL_THREADS) ct_decode_select_kernel(CtDecodeArgs a)
{
    __shared__ unsigned s_hist[256];
    __shared__ unsigned long long s_red[CD_SEL_THREADS / 32];
    __shared__ unsigned long long s_prefix, s_lo;
    __shared__ int s_need, s_done, s_digit, s_count;
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // theta: the largest K-th entry of a full list (a tile holds at most 1024 keys, so only when K <= 1024)
    unsigned long long th = 0;
    if (a.K <= a.Lk)
        for (long long l = threadIdx.x; l < a.L; l += CD_SEL_THREADS)
            th = max(th, a.lists[((size_t)b * a.L + l) * a.Lk + a.K - 1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) th = max(th, __shfl_xor_sync(0xffffffffu, th, o));
    if (lane == 0) s_red[warp] = th;
    if (threadIdx.x == 0) { s_prefix = 0; s_need = a.K; s_done = 0; s_count = 0; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long m = 1;
        for (int w = 0; w < CD_SEL_THREADS / 32; ++w) m = max(m, s_red[w]);
        s_lo = m;
    }
    __syncthreads();
    const unsigned long long lo = s_lo;

    // radix select of the K-th largest key among the entries >= lo, 8 bits a pass from the top; stops as soon as the
    // digit's whole bucket is needed
    unsigned long long hmask = 0;
    for (int shift = 56; shift >= 0 && !s_done; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += CD_SEL_THREADS) s_hist[i] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        cd_for_each(a, b, lo, [&](unsigned long long key) {
            if ((key & hmask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255], 1u);
        });
        __syncthreads();
        if (warp == 0) {
            // lane l owns digits 8l .. 8l + 7; find the digit d where the count above d is < need <= count from d up
            unsigned own = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) own += s_hist[lane * 8 + i];
            unsigned sfx = own;                        // keys in this lane and the lanes above it
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned v = __shfl_down_sync(0xffffffffu, sfx, o);
                if (lane + o < 32) sfx += v;
            }
            const unsigned need = (unsigned)s_need;
            const unsigned up = sfx - own;             // keys in higher lanes
            if (up < need && need <= sfx) {
                unsigned acc = up;
                for (int i = 7; i >= 0; --i) {
                    const unsigned h = s_hist[lane * 8 + i];
                    if (acc + h >= need) {
                        s_digit = lane * 8 + i;
                        s_need = (int)(need - acc);
                        s_done = h == need - acc;
                        break;
                    }
                    acc += h;
                }
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) s_prefix |= (unsigned long long)s_digit << shift;
        hmask |= 0xffull << shift;
        __syncthreads();
    }
    // the selected keys: every entry >= max(lo, kappa), exactly K of them
    const unsigned long long sel_lo = max(lo, s_prefix);
    unsigned long long *sel = a.sel + (size_t)b * a.K;
    cd_for_each(a, b, sel_lo, [&](unsigned long long key) { sel[atomicAdd(&s_count, 1)] = key; });
    __syncthreads();

    const int HW = a.H * a.W;
    for (int i = threadIdx.x; i < a.K; i += CD_SEL_THREADS) {
        const unsigned long long key = sel[i];
        int r = 0;
        for (int j = 0; j < a.K; ++j) r += sel[j] > key;
        const unsigned vb = (unsigned)(key >> 32);
        const unsigned pos = 0xffffffffu - (unsigned)key;
        const int c = (int)(pos / (unsigned)HW), idx = (int)(pos - (unsigned)c * (unsigned)HW);
        const int y = idx / a.W, x = idx - y * a.W;
        const float score = vb == (unsigned)CD_NAN_BITS ? __int_as_float(0x7fffffff) : __uint_as_float(vb);
        const float xs = (float)x, ys = (float)y;
        const float *wp = a.wh + (long long)b * a.ws[0] + (long long)y * a.ws[2] + (long long)x * a.ws[3];
        const float hw = __fmul_rn(__ldg(wp), 0.5f), hh = __fmul_rn(__ldg(wp + a.ws[1]), 0.5f);
        float bx0 = __fsub_rn(xs, hw), by0 = __fsub_rn(ys, hh), bx1 = __fadd_rn(xs, hw), by1 = __fadd_rn(ys, hh);
        if (a.clip) {
            if (!isnan(bx0)) bx0 = fmaxf(bx0, 0.f);
            if (!isnan(by0)) by0 = fmaxf(by0, 0.f);
            if (!isnan(bx1)) bx1 = fminf(bx1, (float)(a.W - 1));
            if (!isnan(by1)) by1 = fminf(by1, (float)(a.H - 1));
        }
        float *ct = a.ct + ((size_t)b * a.K + r) * 2;
        float *det = a.det + ((size_t)b * a.K + r) * 6;
        ct[0] = xs; ct[1] = ys;
        det[0] = bx0; det[1] = by0; det[2] = bx1; det[3] = by1; det[4] = score; det[5] = (float)c;
    }
}

namespace {

// the lists at offset 0, then sel, 256-byte aligned
size_t ct_decode_workspace_bytes(int B, int C, int H, int W, int K, size_t *sel_offset)
{
    const size_t T = (size_t)((W + CD_T - 1) / CD_T) * (size_t)((H + CD_T - 1) / CD_T);
    const size_t Lk = (size_t)(K < CD_N ? K : CD_N);
    const size_t lists = ((size_t)B * C * T * Lk * sizeof(unsigned long long) + 255) / 256 * 256;
    if (sel_offset) *sel_offset = lists;
    return lists + ((size_t)B * K * sizeof(unsigned long long) + 255) / 256 * 256;
}

// the sizes pvb_ct_decode accepts (the limits keep every index exact in fp32 and every key unique)
int ct_decode_sizes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t K)
{
    if (B < 0 || B > 65535) return fail(PVB_ERR_INVALID, "B must be in [0, 65535], got %d", B);
    if (C < 1 || C > 65535 || H < 1 || W < 1)
        return fail(PVB_ERR_INVALID, "C, H and W must be >= 1 and C <= 65535 (got C=%d H=%d W=%d)", C, H, W);
    const long long HW = (long long)H * W;
    if (HW >= (1ll << 24)) return fail(PVB_ERR_INVALID, "H*W must be < 2^24, got %lld", HW);
    if (K < 1 || K > HW) return fail(PVB_ERR_INVALID, "K must be in [1, H*W = %lld], got %d", HW, K);
    if ((long long)C * K >= (1ll << 24)) return fail(PVB_ERR_INVALID, "C*K must be < 2^24, got %lld", (long long)C * K);
    if ((long long)C * HW >= (1ll << 31)) return fail(PVB_ERR_INVALID, "C*H*W must be < 2^31, got %lld", (long long)C * HW);
    return PVB_OK;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API size_t pvb_ct_decode_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t K)
{
    if (B < 0 || C < 0 || H < 0 || W < 0 || K < 0) return 0;
    return ct_decode_workspace_bytes(B, C, H, W, K, nullptr);
}

// lib/networks/ct/dla.py:20-26 Network.decode_detection: sigmoid, ct_decode.decode_ct_hm, data_utils.clip_to_image
PVB_API int pvb_ct_decode(const float *ct_hm, const int64_t *hm_stride, const float *wh, const int64_t *wh_stride,
                          int32_t B, int32_t C, int32_t H, int32_t W, int32_t K, int32_t clip, float *ct,
                          float *detection, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    if (int rc = ct_decode_sizes(B, C, H, W, K)) return rc;
    if (clip != 0 && clip != 1) return fail(PVB_ERR_INVALID, "clip must be 0 or 1 (got %d)", clip);
    if (!hm_stride || !wh_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    CtDecodeArgs a = {};
    for (int i = 0; i < 4; ++i) {
        if (hm_stride[i] < 0 || wh_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
        a.hs[i] = hm_stride[i];
        a.ws[i] = wh_stride[i];
    }
    if (B == 0) return PVB_OK;
    if (!ct_hm || !wh || !ct || !detection) return fail(PVB_ERR_INVALID, "NULL tensor");
    size_t so = 0;
    if (int rc = check_workspace(ct_decode_workspace_bytes(B, C, H, W, K, &so), workspace, workspace_bytes)) return rc;
    char *ws = static_cast<char *>(workspace);
    a.hm = ct_hm; a.wh = wh; a.B = B; a.C = C; a.H = H; a.W = W; a.K = K; a.clip = clip;
    a.lists = reinterpret_cast<unsigned long long *>(ws);
    a.sel = reinterpret_cast<unsigned long long *>(ws + so);
    a.ct = ct; a.det = detection;
    a.T = ((W + CD_T - 1) / CD_T) * ((H + CD_T - 1) / CD_T);
    a.L = (long long)C * a.T;
    a.Lk = K < CD_N ? K : CD_N;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    ct_decode_tile_kernel<<<dim3((unsigned)a.T, (unsigned)C, (unsigned)B), CD_THREADS, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        ct_decode_select_kernel<<<(unsigned)B, CD_SEL_THREADS, 0, st>>>(a);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "ct decode kernels");
}

} // extern "C"
