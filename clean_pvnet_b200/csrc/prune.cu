// prune.cu -- the pruned v3 vote: hypotheses that an angular bound proves cannot be the first maximum are never scored.
//
// For v3 only the first-max winner of each (image, keypoint) and its inliers are observable.  A pixel c with direction u
// votes for h only if angle(u, h-c) < theta = acos(t).  For a tile of pixels with bounding box Q and h outside Q, every
// h-c (c in Q) lies in the angular interval [psi_lo, psi_hi] that Q subtends from h (convexity: the extremes are corners),
// so at most #{c in tile : angle(u_c) in [psi_lo - theta', psi_hi + theta']} of its pixels vote for h.  Summed over the
// tiles this is B(h) >= count(h).  A hypothesis with B(h) < L, L the exact count of any hypothesis, cannot be the first
// maximum.  DESIGN.md 4.2 has the argument, including the slack theta' - theta.
//
//   prune_hist_kernel   (tile, k, b): bounding box + prefix histogram of direction pseudo-angles of one tile
//   prune_plan_kernel   (k, b):       B(h) for every hypothesis, the PRUNE_M largest -> list 0 (pass 1)
//   vote_kernel         list 0
//   prune_next_kernel   (k, b):       L = best pass-1 count; {h not in pass 1 : B(h) >= L} -> list 1 (pass 2)
//   vote_kernel         list 1
#include <cmath>
#include <math_constants.h>
#include "common.cuh"
#include "kernels.h"

namespace pvb {

// Monotone pseudo-angle of a non-zero direction, in [0, 4] counter-clockwise from +x (one unit per quadrant).
__device__ __forceinline__ float pseudo_angle(float x, float y)
{
    if (y >= 0.f) return x >= 0.f ? __fdividef(y, x + y) : 1.f + __fdividef(-x, y - x);
    return x < 0.f ? 2.f + __fdividef(-y, -x - y) : 3.f + __fdividef(x, x - y);
}

constexpr int HIST_THREADS = 256;

__global__ void __launch_bounds__(HIST_THREADS)
prune_hist_kernel(VoteArgs a, PruneArgs q)
{
    const int tile = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
    const int tn = min(a.tn[b], a.cap);
    const int t0 = tile * PRUNE_TILE;
    if (t0 >= tn) return;
    const int n = min(PRUNE_TILE, tn - t0);
    const size_t bk = (size_t)b * a.K + k;
    const float2 *xy = a.xy + (size_t)b * a.cap + t0;
    const float2 *dk = a.dirs + bk * a.cap + t0;
    __shared__ int s_hist[PRUNE_NBIN];
    __shared__ float s_box[4][HIST_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < PRUNE_NBIN) s_hist[tid] = 0;
    __syncthreads();
    float x0 = CUDART_INF_F, x1 = -CUDART_INF_F, y0 = CUDART_INF_F, y1 = -CUDART_INF_F;
    for (int i = tid; i < n; i += HIST_THREADS) {
        const float2 c = __ldg(xy + i), v = __ldg(dk + i);
        x0 = fminf(x0, c.x); x1 = fmaxf(x1, c.x); y0 = fminf(y0, c.y); y1 = fmaxf(y1, c.y);
        // the reference never lets a pixel vote whose norm1 is below 1e-6 or NaN (.cu:121), nor one whose norm1
        // overflows (its cosine is then 0 or NaN): such pixels are left out of the histogram
        const float n1 = __fsqrt_rn(__fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y)));
        if (n1 > below_1e6() && n1 < CUDART_INF_F) {
            const int bin = min(PRUNE_NBIN - 1, (int)(pseudo_angle(v.x, v.y) * (PRUNE_NBIN / 4)));
            atomicAdd(&s_hist[bin], 1);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
        y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
    }
    if (lane == 0) { s_box[0][warp] = x0; s_box[1][warp] = x1; s_box[2][warp] = y0; s_box[3][warp] = y1; }
    __syncthreads();
    int *rec = q.tiles + (bk * q.ntiles + tile) * PRUNE_REC;
    if (warp == 0) {
        // inclusive prefix of the 64 bins, two per lane
        const int h0 = s_hist[2 * lane], h1 = s_hist[2 * lane + 1];
        int s = h0 + h1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        rec[4 + 2 * lane] = s - h1;
        rec[4 + 2 * lane + 1] = s;
        if (lane < 4) {
            float e = s_box[lane][0];
            for (int w = 1; w < HIST_THREADS / 32; ++w) e = (lane & 1) ? fmaxf(e, s_box[lane][w]) : fminf(e, s_box[lane][w]);
            rec[lane] = __float_as_int(e);
        }
    }
}

// Pixels of a tile whose direction bin lies in [blo, bhi] (bins taken modulo PRUNE_NBIN; bhi - blo + 1 < PRUNE_NBIN)
__device__ __forceinline__ int bins_between(const int *P, int blo, int bhi, int tot)
{
    // C(j) = pixels with (unwrapped) bin < j = P[j mod NB - 1] + tot * floor(j / NB)
    auto C = [&](int j) {
        const int w = (j >= 0) ? j / PRUNE_NBIN : -((PRUNE_NBIN - 1 - j) / PRUNE_NBIN);
        const int r = j - w * PRUNE_NBIN;
        return (r ? P[r - 1] : 0) + tot * w;
    };
    return C(bhi + 1) - C(blo);
}

// Adds to `bound` the bound of h over nt tile records `rec` (shared memory)
__device__ void count_bound(const PruneArgs &q, const int *rec, int nt, float hx, float hy, int &bound)
{
    const float c = q.cos_w, s = q.sin_w;
    constexpr float EPS = 1e-5f;                            // pseudo-angle rounding (DESIGN.md 4.2)
    for (int t = 0; t < nt; ++t, rec += PRUNE_REC) {
        const float x0 = __int_as_float(rec[0]), x1 = __int_as_float(rec[1]);
        const float y0 = __int_as_float(rec[2]), y1 = __int_as_float(rec[3]);
        const int tot = rec[4 + PRUNE_NBIN - 1];
        if (hx >= x0 - 0.5f && hx <= x1 + 0.5f && hy >= y0 - 0.5f && hy <= y1 + 0.5f) { bound += tot; continue; }
        // h is at least half a pixel outside the box: the directions h - corner lie in an open half-plane, where
        // "counter-clockwise of" (cross product > 0) orders them; lo / hi are the extreme ones
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
        const int blo = (int)floorf((plo - EPS) * (PRUNE_NBIN / 4));
        const int bhi = (int)floorf((phi + EPS) * (PRUNE_NBIN / 4));
        bound += (bhi - blo + 1 >= PRUNE_NBIN) ? tot : bins_between(rec + 4, blo, bhi, tot);
    }
}

constexpr int PLAN_THREADS = 1024;
constexpr int PLAN_HPT = PRUNE_MAX_HN / PLAN_THREADS;
constexpr int PLAN_TILES = 32;                 // tile records staged in shared memory at a time (8.7 KB)

// exclusive prefix of `flag` over the CTA in thread order; returns it, *total gets the sum.  Every thread calls it.
__device__ __forceinline__ int cta_scan(bool flag, int *s_warp, int *total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    __syncthreads();                                      // s_warp is free
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < PLAN_THREADS / 32; ++w) {
        const int c = s_warp[w];
        before += (w < warp) ? c : 0;
        tot += c;
    }
    *total = tot;
    return before + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(PLAN_THREADS)
prune_plan_kernel(VoteArgs a, PruneArgs q)
{
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const size_t bk = (size_t)b * a.K + k;
    const int tn = max(0, min(a.tn[b], a.cap));
    __shared__ int s_warp[PLAN_THREADS / 32];
    __shared__ int s_rec[PLAN_TILES * PRUNE_REC];
    int bnd[PLAN_HPT];
    float2 hp[PLAN_HPT];
#pragma unroll
    for (int j = 0; j < PLAN_HPT; ++j) {
        const int h = j * PLAN_THREADS + tid;
        bnd[j] = (h < a.hn) ? 0 : -1;                     // no hypothesis: -1, never selected
        hp[j] = (h < a.hn) ? a.hyp[bk * a.hn + h] : make_float2(0.f, 0.f);
    }
    const int nt = (tn + PRUNE_TILE - 1) / PRUNE_TILE;
    const int *rec = q.tiles + bk * q.ntiles * PRUNE_REC;
    for (int t0 = 0; t0 < nt; t0 += PLAN_TILES) {
        const int m = min(PLAN_TILES, nt - t0);
        __syncthreads();
        for (int i = tid; i < m * PRUNE_REC; i += PLAN_THREADS) s_rec[i] = __ldg(rec + t0 * PRUNE_REC + i);
        __syncthreads();
#pragma unroll
        for (int j = 0; j < PLAN_HPT; ++j)
            if (bnd[j] >= 0) count_bound(q, s_rec, m, hp[j].x, hp[j].y, bnd[j]);
    }
#pragma unroll
    for (int j = 0; j < PLAN_HPT; ++j)                   // non-finite or huge: not bounded
        if (bnd[j] >= 0 && !(fabsf(hp[j].x) + fabsf(hp[j].y) <= 1e15f)) bnd[j] = tn;
    // pass 1: the M largest bounds (ties in index order).  thr = largest v with #{B >= v} >= M, by bisection over [0, tn]
    const int M = min(PRUNE_M, a.hn);
    int lo = 0, hi = tn + 1;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        int c = 0;
#pragma unroll
        for (int j = 0; j < PLAN_HPT; ++j) c += __syncthreads_count(bnd[j] >= mid);
        if (c >= M) lo = mid; else hi = mid;
    }
    int gt = 0;
#pragma unroll
    for (int j = 0; j < PLAN_HPT; ++j) gt += __syncthreads_count(bnd[j] > lo);
    int *list = q.list + bk * a.hn;
    int base_eq = 0, base_sel = 0;
#pragma unroll
    for (int j = 0; j < PLAN_HPT; ++j) {
        const int h = j * PLAN_THREADS + tid;
        int n_eq, n_sel;
        const int r = base_eq + cta_scan(bnd[j] == lo, s_warp, &n_eq);
        const bool sel = bnd[j] > lo || (bnd[j] == lo && r < M - gt);
        const int pos = base_sel + cta_scan(sel, s_warp, &n_sel);
        if (sel) list[pos] = h;
        if (h < a.hn) q.key[bk * a.hn + h] = sel ? -1 : bnd[j];
        base_eq += n_eq;
        base_sel += n_sel;
    }
    if (tid == 0) q.len[bk] = M;
}

__global__ void __launch_bounds__(PLAN_THREADS)
prune_next_kernel(VoteArgs a, PruneArgs q)
{
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const size_t bk = (size_t)b * a.K + k;
    const size_t BK = (size_t)a.B * a.K;
    __shared__ int s_warp[PLAN_THREADS / 32];
    __shared__ int s_max[PLAN_THREADS / 32];
    const int *counts = a.counts + bk * a.hn;
    // L = the best exact count of pass 1 (0 when nothing was scored: then nothing is excluded)
    int best = 0;
    const int n1 = q.len[bk];
    for (int s = tid; s < n1; s += PLAN_THREADS) best = max(best, counts[q.list[bk * a.hn + s]]);
    best = __reduce_max_sync(0xffffffffu, best);
    if ((tid & 31) == 0) s_max[tid >> 5] = best;
    __syncthreads();
    int L = 0;
    for (int w = 0; w < PLAN_THREADS / 32; ++w) L = max(L, s_max[w]);
    int *list = q.list + (BK + bk) * a.hn;
    int base = 0;
    for (int h0 = 0; h0 < a.hn; h0 += PLAN_THREADS) {
        const int h = h0 + tid;
        const bool f = h < a.hn && q.key[bk * a.hn + h] >= L;
        int n;
        const int pos = base + cta_scan(f, s_warp, &n);
        if (f) list[pos] = h;
        base += n;
    }
    if (tid == 0) q.len[BK + bk] = base;
}

bool prune_setup(const VoteArgs &a, PruneArgs &q)
{
    const double t = (double)a.thresh;
    if (!(t > 0.0 && t < 1.0) || a.hn <= PRUNE_M || a.hn > PRUNE_MAX_HN) return false;
    // below PRUNE_MIN_UNITS (image, keypoint) pairs the full vote is short of a wave and latency bound: the four extra
    // launches cost more than the skipped tests save (H100, B=1, K=9: 0.104 ms per call in full, 0.151 ms pruned)
    if ((long long)a.B * a.K < PRUNE_MIN_UNITS) return false;
    if ((long long)a.K * ((a.hn + PRUNE_M - 1) / PRUNE_M) > 65535) return false;
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
    const size_t BK = (size_t)a.B * a.K;
    prune_hist_kernel<<<dim3(q.ntiles, a.K, a.B), HIST_THREADS, 0, st>>>(a, q);
    prune_plan_kernel<<<dim3(a.K, a.B), PLAN_THREADS, 0, st>>>(a, q);
    cudaError_t e = launch_vote_list(a, q.list, q.len, PRUNE_M, st);
    if (e != cudaSuccess) return e;
    prune_next_kernel<<<dim3(a.K, a.B), PLAN_THREADS, 0, st>>>(a, q);
    return launch_vote_list(a, q.list + BK * a.hn, q.len + BK, a.hn - PRUNE_M, st);
}

} // namespace pvb
