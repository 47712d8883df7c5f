// prune.cu -- the pruned v3 vote: hypotheses that an angular bound proves cannot be the first maximum are never scored.
//
// For v3 only the first-max winner of each (image, keypoint) and its inliers are observable.  A pixel c with direction u
// votes for h only if angle(u, h-c) < theta = acos(t).  For a set of pixels with bounding box Q and h outside Q, every
// h-c (c in Q) lies in the angular interval [psi_lo, psi_hi] that Q subtends from h (convexity: the extremes are corners),
// so at most #{c in set : angle(u_c) in [psi_lo - theta', psi_hi + theta']} of its pixels vote for h.  The sets are the
// 32x32-pixel cells of the image; summed over the cells this is B(h) >= count(h).  A hypothesis with B(h) < L, L the exact
// count of any hypothesis, cannot be the first maximum.  The argument holds for any partition of the pixels, so pass 2 also
// requires B2(h) >= L, the same bound over the 16x16-pixel sub-cells, which is tighter for cells near h.  DESIGN.md 4.2
// has the argument, including the slack theta' - theta.
//
//   prune_hist_kernel   (band, k, b):   per sub-cell and cell of a 32-row band: bounding box + prefix histogram of
//                                       direction pseudo-angles
//   prune_bound_kernel  (h group, k, b): B(h), three threads per hypothesis -> key; the last CTA of (k, b) takes the
//                                       PRUNE_M largest bounds -> list 0 (pass 1)
//   vote_kernel         list 0
//   prune_next_kernel   (sub-cells, k, b): L = best pass-1 count; B2(h) of {h not in pass 1 : B(h) >= L}; the last CTA
//                                       of (k, b) lists those with B2(h) >= L -> list 1 (pass 2)
//   vote_list_kernel    list 1
#include <cmath>
#include <math_constants.h>
#include "common.cuh"
#include "kernels.h"

namespace pvb {

// Monotone pseudo-angle of a non-zero direction, in [0, 4] counter-clockwise from +x (one unit per quadrant): y / (x + y),
// 1 + -x / (y - x), 2 + -y / (-x - y), 3 + x / (x - y).  The denominator is |x| + |y| and the numerator |y| or |x| in
// every quadrant, the same values bit for bit, so the quadrant only selects them and the offset and one division follows:
// no branch, which matters where a warp's directions lie in different quadrants.  (Quadrant 0 can give +0 where the
// per-quadrant form gives -0; every caller maps both to bin 0.)  The bound divides approximately; the histogram divides
// with IEEE rounding (EXACT), so its bins are reproducible bit for bit.
template <bool EXACT = false>
__device__ __forceinline__ float pseudo_angle(float x, float y)
{
    const bool xn = x < 0.f, yn = y < 0.f;
    const float num = (xn == yn) ? fabsf(y) : fabsf(x), den = fabsf(x) + fabsf(y);
    const float off = yn ? (xn ? 2.f : 3.f) : (xn ? 1.f : 0.f);
    return off + (EXACT ? __fdiv_rn(num, den) : __fdividef(num, den));
}

// First index i in [0, n) with xy[i].y >= y (n if none); xy is sorted by y.  Warp-cooperative 32-ary search: three rounds
// of 32 probes for 30 000 pixels instead of fifteen dependent loads.
__device__ int first_row_at(const float2 *xy, int n, float y)
{
    const int lane = threadIdx.x & 31;
    int lo = 0, hi = n;                                  // the answer lies in [lo, hi]
    while (hi > lo) {
        const int step = (hi - lo + 31) / 32;
        const int p = lo + lane * step;
        const unsigned below = __ballot_sync(0xffffffffu, p < hi && __ldg(&xy[p].y) < y);   // a prefix of the lanes
        const int nb = __popc(below);
        const int nlo = nb ? lo + (nb - 1) * step + 1 : lo;
        hi = min(hi, lo + nb * step);
        lo = nlo;
    }
    return lo;
}

constexpr int HIST_THREADS = 256;
constexpr int HIST_CELLS = 32;                 // cells of a band histogrammed at a time
constexpr int HIST_SUBX = 2 * HIST_CELLS;      // their sub-cell columns; two sub-cell rows per band
constexpr int HIST_SUBS = 2 * HIST_SUBX;       // 128 sub-cells x 64 words of two 16-bit bin counts: 32 KB
static_assert(PRUNE_SUB * PRUNE_SUB < 65536, "a sub-cell's bin counts fit 16 bits");

// One CTA per (band of PRUNE_CELL pixel rows, k, b), chained after generate but independent of it (it waits only at the end).
// The selected-pixel list is in raster (torch.nonzero) order, so the
// band's pixels are one contiguous segment of it.  The histogram and box are taken per sub-cell; every sub-cell and
// every cell of the band gets a record, empty ones with total 0, and a cell's record is the union of its sub-cells'
// (box: min / max of the same float bits; counts: sums), so it is what a histogram over the whole cell gives.
__global__ void __launch_bounds__(HIST_THREADS)
prune_hist_kernel(VoteArgs a, PruneArgs q)
{
    const int band = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
    const int tn = max(0, min(a.tn[b], a.cap));
    const size_t bk = (size_t)b * a.K + k;
    const float2 *xy = a.xy + (size_t)b * a.cap;
    const float2 *dk = a.dirs + bk * a.cap;
    // [sub-cell row][sub-cell column][bin / 2]: bin 2j in the low half of word j, bin 2j + 1 in the high half
    __shared__ __align__(16) int s_hist[2][HIST_SUBX][PRUNE_NBIN / 2];
    __shared__ int s_box[2][HIST_SUBX][4];               // float bits of x0, x1, y0, y1: coordinates are >= 0
    __shared__ int s_seg[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (warp < 2) {
        const int i = first_row_at(xy, tn, (float)((band + warp) * PRUNE_CELL));
        if (lane == 0) s_seg[warp] = i;
    }
    for (int cx0 = 0; cx0 < q.ncx; cx0 += HIST_CELLS) {
        const int nc = min(HIST_CELLS, q.ncx - cx0);
        for (int i = tid; i < HIST_SUBS * PRUNE_NBIN / 8; i += HIST_THREADS)
            reinterpret_cast<int4 *>(&s_hist[0][0][0])[i] = make_int4(0, 0, 0, 0);
        for (int i = tid; i < HIST_SUBS * 4; i += HIST_THREADS)
            (&s_box[0][0][0])[i] = __float_as_int((i & 1) ? -CUDART_INF_F : CUDART_INF_F);
        __syncthreads();
        const int s0 = s_seg[0], s1 = s_seg[1];
        float2 cn = make_float2(0.f, 0.f), vn = make_float2(0.f, 0.f);
        if (s0 + tid < s1) { cn = __ldg(xy + s0 + tid); vn = __ldg(dk + s0 + tid); }
        for (int i0 = s0 + warp * 32; i0 < s1; i0 += HIST_THREADS) {
            const int i = i0 + lane;
            const float2 c = cn, v = vn;
            if (i + HIST_THREADS < s1) { cn = __ldg(xy + i + HIST_THREADS); vn = __ldg(dk + i + HIST_THREADS); }
            int key = -1, hkey = -1, sc = 0;
            if (i < s1) {
                const int sx = (int)c.x / PRUNE_SUB - 2 * cx0, row = (int)c.y - band * PRUNE_CELL;
                // the reference never lets a pixel vote whose norm1 is below 1e-6 or NaN (.cu:121), nor one whose norm1
                // overflows (its cosine is then 0 or NaN): such pixels are left out of the box and the histogram
                const float n1 = __fsqrt_rn(__fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y)));
                if (sx >= 0 && sx < 2 * nc && n1 > below_1e6() && n1 < CUDART_INF_F) {
                    const int bin = min(PRUNE_NBIN - 1, (int)(pseudo_angle<true>(v.x, v.y) * (PRUNE_NBIN / 4)));
                    sc = (row / PRUNE_SUB) * HIST_SUBX + sx;
                    key = row * HIST_SUBX + sx;
                    hkey = sc * PRUNE_NBIN + bin;
                }
            }
            // neighbouring pixels mostly share a sub-cell and a bin, and shared atomics on one address serialise: each
            // run of lanes with equal (sub-cell, bin) adds its length once, to its half of the word
            const int hprev = __shfl_up_sync(0xffffffffu, hkey, 1);
            const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || hprev != hkey);
            if (hkey >= 0 && (lane == 0 || hprev != hkey)) {
                const unsigned later = heads & ~((2u << lane) - 1u);
                atomicAdd(&(&s_hist[0][0][0])[hkey >> 1], ((later ? __ffs(later) - 1 : 32) - lane) << (16 * (hkey & 1)));
            }
            // in raster order the lanes of one (row, sub-cell) form runs sorted by x: only a run's first and last lane
            // update the box
            int *box = &s_box[0][0][0] + 4 * sc;
            const int prev = __shfl_up_sync(0xffffffffu, key, 1), next = __shfl_down_sync(0xffffffffu, key, 1);
            if (key >= 0 && (lane == 0 || prev != key)) {
                atomicMin(box + 0, __float_as_int(c.x));
                atomicMin(box + 2, __float_as_int(c.y));
            }
            if (key >= 0 && (lane == 31 || next != key)) {
                atomicMax(box + 1, __float_as_int(c.x));
                atomicMax(box + 3, __float_as_int(c.y));
            }
        }
        __syncthreads();
        // one warp per cell: inclusive prefix of the 128 bins of each sub-cell, four per lane, stored as 16-bit counts two
        // per word; the cell's record is their sum and the union of their boxes
        for (int cc = warp; cc < nc; cc += HIST_THREADS / 32) {
            const size_t cell = bk * q.ncells + (size_t)band * q.ncx + cx0 + cc;
            int4 sum = make_int4(0, 0, 0, 0);
            int bx = lane & 1 ? __float_as_int(-CUDART_INF_F) : __float_as_int(CUDART_INF_F);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int sr = j >> 1, sx = 2 * cc + (j & 1);
                const int2 w = reinterpret_cast<const int2 *>(s_hist[sr][sx])[lane];
                const int h0 = w.x & 0xffff, h1 = (unsigned)w.x >> 16, h2 = w.y & 0xffff, h3 = (unsigned)w.y >> 16;
                int s = h0 + h1 + h2 + h3;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, s, o);
                    if (lane >= o) s += t;
                }
                const int4 p = make_int4(s - h3 - h2 - h1, s - h3 - h2, s - h3, s);
                int *rec = q.sub + (cell * 4 + j) * PRUNE_REC;
                // most sub-cells of an image are empty: their record is the last word alone (total 0), which is all
                // that prune_next_kernel reads of them
                const bool empty = __shfl_sync(0xffffffffu, s, 31) == 0;
                if (!empty || lane == 31)
                    reinterpret_cast<int2 *>(rec + 4)[lane] = make_int2(p.x | (p.y << 16), p.z | (p.w << 16));
                if (lane < 4) {
                    const int v = s_box[sr][sx][lane];
                    if (!empty) rec[lane] = v;
                    bx = lane & 1 ? max(bx, v) : min(bx, v);
                }
                sum.x += p.x; sum.y += p.y; sum.z += p.z; sum.w += p.w;
            }
            int *rec = q.cells + cell * PRUNE_REC;
            reinterpret_cast<int2 *>(rec + 4)[lane] = make_int2(sum.x | (sum.y << 16), sum.z | (sum.w << 16));
            if (lane < 4) rec[lane] = bx;
        }
        __syncthreads();                                  // s_hist / s_box are reset for the next cells
    }
    // the whole body reads only thin_gather's output and writes nothing generate reads, so it runs alongside generate;
    // the wait keeps the chain's rule for the kernels after this one (common.cuh)
    grid_dep_wait();
    grid_dep_launch_dependents();
}

__device__ __forceinline__ int cell_total(const int *rec) { return (int)((unsigned)rec[PRUNE_REC - 1] >> 16); }

// false for non-finite or huge hypotheses, which get no bound (B(h) = tn)
__device__ __forceinline__ bool bounded(float2 h) { return fabsf(h.x) + fabsf(h.y) <= 1e15f; }

// Pixels of a cell whose direction bin lies in [blo, bhi] (bins taken modulo PRUNE_NBIN; bhi - blo + 1 < PRUNE_NBIN)
__device__ __forceinline__ int bins_between(const unsigned short *P, int blo, int bhi, int tot)
{
    // C(j) = pixels with (unwrapped) bin < j = P[j mod NB - 1] + tot * floor(j / NB); on two's complement the floor
    // division and the modulo are a shift and a mask
    static_assert(PRUNE_NBIN == 128, "bins_between shifts by log2(PRUNE_NBIN)");
    auto C = [&](int j) {
        const int r = j & (PRUNE_NBIN - 1);
        return (r ? (int)P[r - 1] : 0) + tot * (j >> 7);
    };
    return C(bhi + 1) - C(blo);
}

// Adds to `bound` the bound of h over nt cell records `rec` (shared memory).  The window is computed for every record and
// the two whole-record cases (h inside the box, a window of every bin) select the total afterwards, so a warp whose
// hypotheses fall in different cases does not diverge; the window's table reads stay inside the record for any input.
__device__ void count_bound(const PruneArgs &q, const int *rec, int nt, float hx, float hy, int &bound)
{
    const float c = q.cos_w, s = q.sin_w;
    constexpr float EPS = 1e-5f;                            // pseudo-angle rounding (DESIGN.md 4.2)
    for (int t = 0; t < nt; ++t, rec += PRUNE_REC) {
        const float x0 = __int_as_float(rec[0]), x1 = __int_as_float(rec[1]);
        const float y0 = __int_as_float(rec[2]), y1 = __int_as_float(rec[3]);
        const int tot = cell_total(rec);
        const bool inside = hx >= x0 - 0.5f && hx <= x1 + 0.5f && hy >= y0 - 0.5f && hy <= y1 + 0.5f;
        // unless inside, h is at least half a pixel outside the box: the directions h - corner lie in an open
        // half-plane, where "counter-clockwise of" (cross product > 0) orders them; lo / hi are the extreme ones
        float lx = hx - x0, ly = hy - y0, ux = lx, uy = ly;
        const float cx[3] = {x1, x0, x1}, cy[3] = {y0, y1, y1};
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float dx = hx - cx[i], dy = hy - cy[i];
            if (lx * dy - ly * dx < 0.f) { lx = dx; ly = dy; }
            if (ux * dy - uy * dx > 0.f) { ux = dx; uy = dy; }
        }
        // widen by theta': lo turns clockwise, hi counter-clockwise; the widened interval spans less than 2*pi - 0.14
        const float plo = pseudo_angle(c * lx + s * ly, c * ly - s * lx);
        float phi = pseudo_angle(c * ux - s * uy, c * uy + s * ux);
        if (phi < plo) phi += 4.f;
        const int blo = __float2int_rd((plo - EPS) * (PRUNE_NBIN / 4));
        const int bhi = __float2int_rd((phi + EPS) * (PRUNE_NBIN / 4));
        const int win = bins_between(reinterpret_cast<const unsigned short *>(rec + 4), blo, bhi, tot);
        bound += (inside || bhi - blo + 1 >= PRUNE_NBIN) ? tot : win;
    }
}

constexpr int BOUND_HYPS = 64;                 // hypotheses per CTA
constexpr int BOUND_SPLIT = 4;                 // threads per hypothesis, each over a quarter of every staged chunk: one
                                               // thread per hypothesis leaves too few warps to hide the latency
constexpr int BOUND_THREADS = BOUND_HYPS * BOUND_SPLIT;
constexpr int BOUND_WARPS = BOUND_THREADS / 32;
constexpr int STAGE_RECS = 32;                 // non-empty records per staged chunk; two chunks in flight (17 KB)
constexpr int REC_V4 = PRUNE_REC / 4;          // 16-byte pieces of a record
static_assert(PRUNE_REC % 4 == 0, "records are staged in 16-byte pieces");
static_assert(PRUNE_MAX_HN + 256 <= 2 * STAGE_RECS * PRUNE_REC, "the pass-1 selection fits in the record buffers");

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" :: "n"(N) : "memory"); }

// Streams the non-empty ones of the records rec + c * stride (c < nrec; an empty one adds nothing to a bound) through
// shared memory and calls use(records, n) with every thread of the CTA for each chunk of n <= STAGE_RECS of them.  The
// CTA lists the non-empty records 3 x THREADS at a time (empty ones cost one word read), then stages their records with
// cp.async one chunk ahead of the chunk in use.  Within a listing round the order is not the index order, which no
// integer sum over the records sees.  s_rec holds 2 x STAGE_RECS records, s_idx 3 x THREADS ints, s_w THREADS / 32.
template <int THREADS, typename Use>
__device__ __forceinline__ void stream_records(const int *rec, int stride, int nrec, int *s_rec, int *s_idx, int *s_w,
                                               Use use)
{
    constexpr int WARPS = THREADS / 32, SCAN = 3 * THREADS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int c0 = 0; c0 < nrec; c0 += SCAN) {
        bool f[3];
        unsigned bal[3];
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int c = c0 + j * THREADS + tid;
            f[j] = c < nrec && cell_total(rec + (size_t)c * stride) > 0;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) { bal[j] = __ballot_sync(0xffffffffu, f[j]); cnt += __popc(bal[j]); }
        if (lane == 0) s_w[warp] = cnt;
        __syncthreads();
        int base = 0, m = 0;
        for (int w = 0; w < WARPS; ++w) {
            const int c = s_w[w];
            base += (w < warp) ? c : 0;
            m += c;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            if (f[j]) s_idx[base + __popc(bal[j] & ((1u << lane) - 1u))] = c0 + j * THREADS + tid;
            base += __popc(bal[j]);
        }
        __syncthreads();
        const int nch = (m + STAGE_RECS - 1) / STAGE_RECS;
        auto stage = [&](int ch) {
            const int r0 = ch * STAGE_RECS, n = min(STAGE_RECS, m - r0);
            int *dst = s_rec + (ch & 1) * STAGE_RECS * PRUNE_REC;
            for (int i = tid; i < n * REC_V4; i += THREADS) {
                const int r = i / REC_V4, w = (i - r * REC_V4) * 4;
                cp_async16(dst + r * PRUNE_REC + w, rec + (size_t)s_idx[r0 + r] * stride + w);
            }
            cp_async_commit();
        };
        if (nch > 0) stage(0);
        for (int ch = 0; ch < nch; ++ch) {
            if (ch + 1 < nch) { stage(ch + 1); cp_async_wait<1>(); }
            else cp_async_wait<0>();
            __syncthreads();
            use(s_rec + (ch & 1) * STAGE_RECS * PRUNE_REC, min(STAGE_RECS, m - ch * STAGE_RECS));
            __syncthreads();                              // the buffer is restaged two chunks on; s_idx, s_w next round
        }
    }
}

// Pass 1 of (b, k): the PRUNE_M largest bounds, ties in index order, listed in index order; their keys become -1.
// Called by every thread of the CTA once all of the (image, keypoint)'s bounds are in q.key.  s_key holds hn ints,
// s_cnt 256, s_w 2 x BOUND_WARPS, s_sel 2.
__device__ void plan_pass1(const VoteArgs &a, const PruneArgs &q, size_t bk, int *s_key, int *s_cnt, int *s_w, int *s_sel)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int hn = a.hn, M = min(PRUNE_M, hn);
    int *key = q.key + bk * hn;
    int top = 0;
    for (int h = tid; h < hn; h += BOUND_THREADS) {
        const int v = __ldcg(key + h);                    // written by the other CTAs of (b, k)
        s_key[h] = v;
        top = max(top, v);
    }
    top = __reduce_max_sync(0xffffffffu, top);
    if (lane == 0) s_w[warp] = top;
    __syncthreads();
    for (int w = 0; w < BOUND_WARPS; ++w) top = max(top, s_w[w]);
    // thr = the M-th largest bound (bounds are >= 0), by radix selection, at most 8 bits a round from the top: bits
    // [hi, 31] of thr are fixed, and `need` of the M lie among the bounds that agree with thr there
    int thr = 0, need = M;
    for (int hi = 32 - __clz(top | 1); hi > 0;) {
        const int lo = max(0, hi - 8);
        for (int i = tid; i < 256; i += BOUND_THREADS) s_cnt[i] = 0;
        __syncthreads();
        for (int h = tid; h < hn; h += BOUND_THREADS) {
            const int v = s_key[h];
            if ((v >> hi) == (thr >> hi)) atomicAdd(&s_cnt[(v >> lo) & ((1 << (hi - lo)) - 1)], 1);
        }
        __syncthreads();
        if (warp == 0) {                                  // the digit d of thr: the largest with #{digit >= d} >= need
            int c[8], own = 0;
#pragma unroll
            for (int e = 0; e < 8; ++e) { c[e] = s_cnt[8 * lane + e]; own += c[e]; }
            int suf = own;                                // digits >= 8 * lane
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_down_sync(0xffffffffu, suf, o);
                if (lane + o < 32) suf += t;
            }
            const unsigned ok = __ballot_sync(0xffffffffu, suf >= need);   // lane 0 always: every match counts
            if (lane == 31 - __clz(ok)) {
                int above = suf - own;
#pragma unroll
                for (int e = 7; e >= 0; --e) {
                    if (above + c[e] >= need) { s_sel[0] = 8 * lane + e; s_sel[1] = need - above; break; }
                    above += c[e];
                }
            }
        }
        __syncthreads();
        thr |= s_sel[0] << lo;
        need = s_sel[1];
        hi = lo;
    }
    // every bound > thr and the first `need` equal to it, in index order: each warp takes a contiguous range
    const int per = (hn + 32 * BOUND_WARPS - 1) / (32 * BOUND_WARPS) * 32;
    const int h0 = warp * per, h1 = min(hn, h0 + per);
    int gt = 0, eq = 0;
    for (int h = h0 + lane; h - lane < h1; h += 32) {
        const int v = h < h1 ? s_key[h] : -1;
        gt += __popc(__ballot_sync(0xffffffffu, v > thr));
        eq += __popc(__ballot_sync(0xffffffffu, v == thr));
    }
    int *s_gt = s_w, *s_eq = s_w + BOUND_WARPS;
    __syncthreads();                                      // s_w was read above
    if (lane == 0) { s_gt[warp] = gt; s_eq[warp] = eq; }
    __syncthreads();
    gt = eq = 0;
    for (int w = 0; w < warp; ++w) { gt += s_gt[w]; eq += s_eq[w]; }
    int *list = q.list + bk * hn;
    const unsigned below = (1u << lane) - 1u;
    for (int h = h0 + lane; h - lane < h1; h += 32) {
        const int v = h < h1 ? s_key[h] : -1;
        const unsigned mg = __ballot_sync(0xffffffffu, v > thr), me = __ballot_sync(0xffffffffu, v == thr);
        const int g = gt + __popc(mg & below), e = eq + __popc(me & below);
        if (v > thr || (v == thr && e < need)) {
            list[g + min(e, need)] = h;
            key[h] = -1;
        }
        gt += __popc(mg);
        eq += __popc(me);
    }
    if (tid == 0) q.len[bk] = M;
}

// One CTA per (BOUND_HYPS hypotheses, k, b).  The CTA streams the non-empty cells' records (stream_records) and sums
// B(h) over them; the last CTA of (b, k) to finish then picks pass 1 (plan_pass1), so no launch waits for the slowest one.
__global__ void __launch_bounds__(BOUND_THREADS, 2048 / BOUND_THREADS)
prune_bound_kernel(VoteArgs a, PruneArgs q)
{
    const int tid = threadIdx.x;
    const int part = tid / BOUND_HYPS, hl = tid % BOUND_HYPS;
    const int h = blockIdx.x * BOUND_HYPS + hl, k = blockIdx.y, b = blockIdx.z;
    const size_t bk = (size_t)b * a.K + k;
    const int tn = max(0, min(a.tn[b], a.cap));
    __shared__ __align__(16) int s_rec[2][STAGE_RECS * PRUNE_REC];
    __shared__ int s_idx[3 * BOUND_THREADS];
    __shared__ int s_part[BOUND_SPLIT][BOUND_HYPS];
    __shared__ int s_w[2 * BOUND_WARPS];
    __shared__ int s_sel[2];
    const float2 hp = (h < a.hn) ? a.hyp[bk * a.hn + h] : make_float2(0.f, 0.f);   // generate's: before the wait
    grid_dep_wait();                                      // the cell records are prune_hist's output
    grid_dep_launch_dependents();
    int bound = 0;
    stream_records<BOUND_THREADS>(q.cells + bk * q.ncells * PRUNE_REC, PRUNE_REC, q.ncells, &s_rec[0][0], s_idx, s_w,
                                  [&](const int *rec, int n) {
        const int r0 = part * n / BOUND_SPLIT, r1 = (part + 1) * n / BOUND_SPLIT;
        count_bound(q, rec + r0 * PRUNE_REC, r1 - r0, hp.x, hp.y, bound);
    });
    if (part > 0) s_part[part][hl] = bound;
    __syncthreads();
    if (part == 0 && h < a.hn) {
#pragma unroll
        for (int p = 1; p < BOUND_SPLIT; ++p) bound += s_part[p][hl];
        q.key[bk * a.hn + h] = bounded(hp) ? bound : tn;
        q.b2[bk * a.hn + h] = 0;                          // prune_next_kernel's CTAs add their sub-cells' parts to it
    }
    // q.ticket[bk] is 0 when the call starts (it lies in the workspace header) and is left 0 for the refit
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        s_sel[0] = (atomicAdd(q.ticket + bk, 1) == (int)gridDim.x - 1);
        if (s_sel[0]) q.ticket[bk] = 0;
    }
    __syncthreads();
    if (!s_sel[0]) return;
    __threadfence();
    plan_pass1(a, q, bk, &s_rec[0][0], &s_rec[0][0] + PRUNE_MAX_HN, s_w, s_sel);
}

constexpr int NEXT_THREADS = 256;
constexpr int NEXT_CTAS = 8;                   // CTAs per (image, keypoint): CTA x takes the sub-cells s = x mod NEXT_CTAS
                                               // (with 4 sub-cells per cell, one quadrant of every cell or every other)
// per candidate of pass 2 in prune_next_kernel's dynamic shared memory: its hypothesis, its B2 part and its index
constexpr int NEXT_CAND_BYTES = sizeof(float2) + sizeof(int) + sizeof(unsigned short);
static_assert(PRUNE_MAX_HN <= 65536, "candidate indices fit 16 bits");

// exclusive prefix of `flag` over the CTA in thread order; returns it, *total gets the sum.  Every thread calls it.
__device__ __forceinline__ int cta_scan(bool flag, int *s_warp, int *total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    __syncthreads();                                      // s_warp is free
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < NEXT_THREADS / 32; ++w) {
        const int c = s_warp[w];
        before += (w < warp) ? c : 0;
        tot += c;
    }
    *total = tot;
    return before + __popc(m & ((1u << lane) - 1u));
}

// NEXT_CTAS CTAs per (k, b); dynamic shared memory: NEXT_CAND_BYTES x (hn - PRUNE_M).  L = the best exact count of
// pass 1; the candidates of pass 2 are the hypotheses not in pass 1 with B(h) >= L, at most hn - PRUNE_M.  Each CTA
// finds L and the candidates once, keeps their hypotheses in shared memory, streams the non-empty ones of its sub-cells
// (stream_records) and adds, for every candidate, the bound over them to b2 (count_bound over a
// finer partition of the same pixels: DESIGN.md 4.2); the last CTA of (b, k) to finish lists pass 2 = {candidates with
// B2(h) >= L} in index order.  L = 0 excludes nothing and skips the sums.
__global__ void __launch_bounds__(NEXT_THREADS)
prune_next_kernel(VoteArgs a, PruneArgs q)
{
    const int x = blockIdx.x, k = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
    const size_t bk = (size_t)b * a.K + k;
    const int hn = a.hn;
    __shared__ __align__(16) int s_rec[2 * STAGE_RECS * PRUNE_REC];
    __shared__ int s_idx[3 * NEXT_THREADS];
    __shared__ int s_warp[NEXT_THREADS / 32];
    __shared__ int s_last;
    extern __shared__ __align__(16) unsigned char s_dyn[];
    const int ncap = hn - PRUNE_M;
    float2 *s_hyp = reinterpret_cast<float2 *>(s_dyn);
    int *s_b2 = reinterpret_cast<int *>(s_hyp + ncap);
    unsigned short *s_cand = reinterpret_cast<unsigned short *>(s_b2 + ncap);
    const int *key = q.key + bk * hn;
    const float2 *hyp = a.hyp + bk * hn;
    int *b2 = q.b2 + bk * hn;
    // L = the best exact count of pass 1 (0 when nothing was scored: then nothing is excluded).  Pass 1's list is the bound
    // kernel's, two launches back, and is read before the wait; its counts are pass 1's, read after it
    static_assert(PRUNE_M <= NEXT_THREADS, "one pass-1 entry per thread");
    int L = 0;
    {
        const int *counts = a.counts + bk * hn;
        int best = 0;
        const int n1 = q.len[bk];
        const int h1 = tid < n1 ? q.list[bk * hn + tid] : -1;
        grid_dep_wait();
        grid_dep_launch_dependents();
        if (h1 >= 0) best = __ldcg(counts + h1);          // through L2: no L1 holds a line of the counts in a call
        best = __reduce_max_sync(0xffffffffu, best);
        if ((tid & 31) == 0) s_warp[tid >> 5] = best;
        __syncthreads();
        for (int w = 0; w < NEXT_THREADS / 32; ++w) L = max(L, s_warp[w]);
    }
    // the candidates that have a bound (the others stay in pass 2); pass 1's keys are -1 < L
    int nc = 0;
    for (int h0 = 0; h0 < hn && L > 0; h0 += NEXT_THREADS) {
        const int h = h0 + tid;
        const float2 hp = h < hn ? hyp[h] : make_float2(0.f, 0.f);
        const bool f = h < hn && key[h] >= L && bounded(hp);
        int n;
        const int pos = nc + cta_scan(f, s_warp, &n);
        if (f) { s_cand[pos] = (unsigned short)h; s_hyp[pos] = hp; s_b2[pos] = 0; }
        nc += n;
    }
    if (nc > 0) {
        __syncthreads();                                  // s_warp is free, the candidates are in place
        // P threads per candidate, each over a contiguous part of every staged chunk
        const int P = max(1, NEXT_THREADS / nc);
        const int *sub = q.sub + (bk * q.ncells * 4 + x) * PRUNE_REC;
        const int nsub = (4 * q.ncells - x + NEXT_CTAS - 1) / NEXT_CTAS;
        stream_records<NEXT_THREADS>(sub, NEXT_CTAS * PRUNE_REC, nsub, s_rec, s_idx, s_warp, [&](const int *rec, int n) {
            for (int it = tid; it < nc * P; it += NEXT_THREADS) {
                const int j = it % nc, p = it / nc;
                const int r0 = p * n / P, r1 = (p + 1) * n / P;
                if (r1 == r0) continue;
                const float2 hp = s_hyp[j];
                int bound = 0;
                count_bound(q, rec + r0 * PRUNE_REC, r1 - r0, hp.x, hp.y, bound);
                if (bound) atomicAdd(&s_b2[j], bound);
            }
        });
        for (int j = tid; j < nc; j += NEXT_THREADS)
            if (s_b2[j]) atomicAdd(&b2[s_cand[j]], s_b2[j]);
    }
    // q.ticket[bk] is 0 here (the bound step leaves it so) and is left 0 for the refit
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        s_last = (atomicAdd(q.ticket + bk, 1) == (int)gridDim.x - 1);
        if (s_last) q.ticket[bk] = 0;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    int *list = q.list2 + bk * hn;
    int base = 0;
    for (int h0 = 0; h0 < hn; h0 += NEXT_THREADS) {
        const int h = h0 + tid;
        const bool f = h < hn && key[h] >= L && (L == 0 || !bounded(hyp[h]) || __ldcg(b2 + h) >= L);
        int n;
        const int pos = base + cta_scan(f, s_warp, &n);
        if (f) list[pos] = h;
        base += n;
    }
    if (tid == 0) q.len2[bk] = base;
}

bool prune_setup(const VoteArgs &a, PruneArgs &q)
{
    const double t = (double)a.thresh;
    if (!(t > 0.0 && t < 1.0) || a.hn <= PRUNE_M || a.hn > PRUNE_MAX_HN) return false;
    // below PRUNE_MIN_UNITS (image, keypoint) pairs the full vote is short of a wave and latency bound: the extra
    // launches cost more than the skipped tests save (H100, B=1, K=9: 0.104 ms per call in full, 0.151 ms pruned)
    if ((long long)a.B * a.K < PRUNE_MIN_UNITS) return false;
    // the list passes launch grid.y = K (pass 2) and K * 1 slice (pass 1), inside this bound; tests/prune_twin.py states it
    if ((long long)a.K * ((a.hn + 63) / 64) > 65535) return false;
    // theta' >= every angle at which the reference can still count a vote: its fp32 cosine is within 9u of the exact one
    // (DESIGN.md 4.1), so a vote needs cos > t - 9u; 64u and 1e-5 rad on top cover the rounding of the bound itself
    const double u = ldexp(1.0, -24);
    const double w = acos(fmax(-1.0, t - 64.0 * u)) + 1e-5;
    if (!(w < 1.5)) return false;                        // keeps the widened interval below 2*pi - 0.14
    // round the rotation outward: a slightly larger angle only loosens the bound
    q.cos_w = nextafterf((float)cos(w), 0.f);
    q.sin_w = nextafterf((float)sin(w), 1.f);
    return true;
}

cudaError_t launch_vote_pruned(const VoteArgs &a, const PruneArgs &q, cudaStream_t st)
{
    const int nbands = (a.H + PRUNE_CELL - 1) / PRUNE_CELL;
    // every launch is chained (common.cuh); prune_setup guarantees both passes launch (PRUNE_M > 0, hn > PRUNE_M), so
    // each kernel's predecessor is the one before it in this list
    cudaError_t e = launch_chained(true, prune_hist_kernel, dim3(nbands, a.K, a.B), HIST_THREADS, 0, st, a, q);
    if (e == cudaSuccess)
        e = launch_chained(true, prune_bound_kernel, dim3((a.hn + BOUND_HYPS - 1) / BOUND_HYPS, a.K, a.B), BOUND_THREADS, 0, st,
                           a, q);
    if (e == cudaSuccess) e = launch_vote_list_slices(a, q.list, q.len, PRUNE_M, st);
    if (e == cudaSuccess)
        e = launch_chained(true, prune_next_kernel, dim3(NEXT_CTAS, a.K, a.B), NEXT_THREADS,
                           (size_t)(a.hn - PRUNE_M) * NEXT_CAND_BYTES, st, a, q);
    if (e != cudaSuccess) return e;
    return launch_vote_list(a, q.list2, q.len2, a.hn - PRUNE_M, st);
}

} // namespace pvb
