// vote.cu -- hypothesis generation, inlier counting (the hot kernel), winner refit, covariance.
//
// Reference being replaced, per image and per round (ransac_voting_gpu.py:150-196):
//   generate_hypothesis -> zeros u8[hn,vn,tn] -> voting_for_hypothesis -> torch.sum -> torch.max
//   -> voting_for_hypothesis(hn=1) -> matmul/sum/solve
// Here: one launch each for the whole batch, no [hn,vn,tn] byte tensor, no host sync.
//
// vote_kernel design (FP32-issue bound, not HBM bound: hn tests per 16 loaded bytes):
//   * a CTA owns one (image b, keypoint k, hypothesis slice, tile of 512 selected pixels);
//   * every thread keeps HPT hypotheses and their tallies in registers;
//   * the tile is staged once through shared memory as 6-float "cone records", relative to a
//     tile-local origin (centre of the tile's bounding box), and broadcast to all threads
//     (3 LDS.128 per 2 pixels per warp);
//   * the inlier test  cos(angle(v, h-c)) > t  is evaluated in the rotated frame of the pixel's
//     unit vector u:   a = u.(h-c),  p = u_perp.(h-c),   inlier <=> m = kappa*a - |p| > 0,
//     kappa = tan(acos t).  With the record (A1,A2,A3,B1,B2,B3) this is 4 FFMA + 1 FADD per test;
//     the tally is the sign bit of m (LEA.HI), the smallest |m| per 16-pixel block and hypothesis
//     is tracked with FMNMX3: 454 SASS instructions per 64 tests per thread;
//   * m is algebraically, not bitwise, the reference predicate.  A guard band delta = band * S
//     (DESIGN.md 4.1, tools/band_check.c) bounds every rounding difference between the two; blocks
//     whose smallest |m| falls inside it are re-evaluated -- warp-cooperatively -- with the
//     reference's exact operation sequence (vote_exact).  Counts equal the reference's.
//
// No tensor cores: the specification of this path excludes them (a sparse reduction, not a dense contraction).  An mma.sync
// formulation was measured once for what it would buy (+8 %) and dropped.
#include <atomic>
#include <math_constants.h>
#include "common.cuh"
#include "kernels.h"

namespace pvb {

// ---------------------------------------------------------------------------------
// hypotheses: thread per (b,k,h)
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
generate_kernel(VoteArgs a)
{
    // tn, dirs and xy are thin_gather's output.  The trigger comes at once, so prune_hist, which needs none of what this
    // kernel writes, runs alongside it (common.cuh, DESIGN.md 4)
    grid_dep_wait();
    grid_dep_launch_dependents();
    const int h = blockIdx.x * 256 + threadIdx.x;
    if (h >= a.hn) return;
    const int k = blockIdx.y, b = blockIdx.z;
    const int tn = min(a.tn[b], a.cap);
    float x = 0.f, y = 0.f;
    if (tn > 0) {
        int t0, t1;
        if (a.idxs) {
            const int2 t = __ldg(reinterpret_cast<const int2 *>(a.idxs) + ((size_t)b * a.hn + h) * a.K + k);
            t0 = t.x; t1 = t.y;
        } else {
            const uint4 r = philox4x32_10(make_uint4((uint32_t)h, (uint32_t)k, (uint32_t)(a.img_base + b), a.tag_idx),
                                          make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
            t0 = (int)(r.x % (uint32_t)tn);
            t1 = (int)(r.y % (uint32_t)tn);
        }
        if ((unsigned)t0 < (unsigned)tn && (unsigned)t1 < (unsigned)tn) {
            const float2 *dk = a.dirs + ((size_t)b * a.K + k) * a.cap;
            const float2 *xy = a.xy + (size_t)b * a.cap;
            const float2 d0 = dk[t0], d1 = dk[t1], c0 = xy[t0], c1 = xy[t1];
            float hx, hy;
            if (hypothesis_from_pair(d0.x, d0.y, c0.x, c0.y, d1.x, d1.y, c1.x, c1.y, hx, hy)) { x = hx; y = hy; }
        }
    }
    a.hyp[((size_t)b * a.K + k) * a.hn + h] = make_float2(x, y);
    a.counts[((size_t)b * a.K + k) * a.hn + h] = 0;      // the vote kernel accumulates with atomics: saves a memset launch
}

cudaError_t launch_generate(const VoteArgs &a, bool chained, cudaStream_t st)
{
    dim3 g((a.hn + 255) / 256, a.K, a.B);
    return launch_chained(chained, generate_kernel, g, 256, 0, st, a);
}

// ---------------------------------------------------------------------------------
// the vote kernel
// ---------------------------------------------------------------------------------
struct VoteK {
    VoteArgs a;
    ConeParams cone;
    const int *list;   // optional [B][K][hn]: slot s of (b,k) scores hypothesis list[s] (NULL: slot s is hypothesis s)
    const int *len;    // [B][K] slots in use (with list)
    unsigned long long *stats;   // optional, BOX: [3] tests resolved per box as inliers, all tests resolved per box, tests scored
};

constexpr int VOTE_BLOCK = 16;    // pixels per unrolled block (one guard-band check per block)

__device__ __forceinline__ float4 lds128(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

// Cone margin of one pixel record against one hypothesis: m = kappa*u.(h-c) - |u_perp.(h-c)|.
// The same function is used by the fast path and by the guard-band re-check, so both see the
// same value bit for bit.
__device__ __forceinline__ float cone_margin(const float4 ra, const float2 rb, float hxc, float hyc)
{
    const float ap = fmaf(ra.x, hxc, fmaf(ra.y, hyc, ra.z));
    const float pp = fmaf(ra.w, hxc, fmaf(rb.x, hyc, rb.y));
    return ap - fabsf(pp);
}

// Pass 1's per-box classification of one pixel record (DESIGN.md 4.2, "Pass 1 per box"): the record's two affine forms
// a = kappa*u.(h-c) and p = u_perp.(h-c) are evaluated at the four corners (x0|x1, y0|y1) of the box of the CTA's
// hypotheses with cone_margin's operations.  1: every hypothesis of the box is an inlier (m = a - |p| > d at all
// corners: m is concave); -1: none is (a + p or a - p < -d at all corners: both are affine and bound m from above);
// 0: undecided, each hypothesis is tested on its own.  d = inf (an unbounded hypothesis in the box) decides nothing.
__device__ __forceinline__ int box_class(const float4 ra, const float2 rb, float x0, float x1, float y0, float y1, float d)
{
    float mn = CUDART_INF_F, lp = -CUDART_INF_F, lm = -CUDART_INF_F;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float x = (q & 1) ? x1 : x0, y = (q & 2) ? y1 : y0;
        const float ap = fmaf(ra.x, x, fmaf(ra.y, y, ra.z));
        const float pp = fmaf(ra.w, x, fmaf(rb.x, y, rb.y));
        mn = fminf(mn, ap - fabsf(pp));
        lp = fmaxf(lp, ap + pp);
        lm = fmaxf(lm, ap - pp);
    }
    return (mn > d) ? 1 : (lp < -d || lm < -d) ? -1 : 0;
}

// Loads a tile's n pixels, pixel i = threadIdx.x + r*NT to slot r (zeros past n), and returns the tile-local origin (ox, oy),
// the centre of the tile's bounding box, with cmax = max over the tile of |cx-ox|+|cy-oy|.  The guard band scales with
// S = |h-o|_1 + cmax, so a local origin keeps it tight.  Every thread of the CTA calls it.
template <int NT, int PPT>
__device__ __forceinline__ void load_tile(const float2 *dk, const float2 *xy, int n, float2 (&v)[PPT], float2 (&c)[PPT],
                                          float (*s_box)[NT / 32], float &ox, float &oy, float &cmax)
{
    constexpr int NW = NT / 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float x0 = CUDART_INF_F, x1 = -CUDART_INF_F, y0 = CUDART_INF_F, y1 = -CUDART_INF_F;
#pragma unroll
    for (int r = 0; r < PPT; ++r) {
        const int i = tid + r * NT;
        v[r] = make_float2(0.f, 0.f); c[r] = make_float2(0.f, 0.f);
        if (i < n) {
            v[r] = __ldg(dk + i); c[r] = __ldg(xy + i);
            x0 = fminf(x0, c[r].x); x1 = fmaxf(x1, c[r].x); y0 = fminf(y0, c[r].y); y1 = fmaxf(y1, c[r].y);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
        y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
    }
    if (lane == 0) { s_box[0][warp] = x0; s_box[1][warp] = x1; s_box[2][warp] = y0; s_box[3][warp] = y1; }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        x0 = fminf(x0, s_box[0][w]); x1 = fmaxf(x1, s_box[1][w]); y0 = fminf(y0, s_box[2][w]); y1 = fmaxf(y1, s_box[3][w]);
    }
    ox = 0.5f * (x0 + x1); oy = 0.5f * (y0 + y1);
    // half extents, padded against the rounding of ox/oy
    cmax = (0.5f * (x1 - x0) + 0.5f * (y1 - y0)) * 1.000001f + 1e-3f;
}

// Cone record (A1, A2, A3, B1), (B2, B3) of pixel (v, c) relative to the tile origin.  `pixel` false (padding) and a pixel the
// reference never lets vote give margin -1e30 against every hypothesis: negative, never inside a finite band.  A pixel outside
// the domain of the error analysis gives margin 0, always inside the band, so the exact path decides every one of its tests.
__device__ __forceinline__ void cone_record(bool pixel, float2 v, float2 c, float ox, float oy, float cmax, float kappa,
                                            float4 &ra, float2 &rb)
{
    ra = make_float4(0.f, 0.f, -1e30f, 0.f);
    rb = make_float2(0.f, 0.f);
    if (!pixel) return;
    const float n1 = __fsqrt_rn(__fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y)));   // the reference's norm1
    const float cxc = c.x - ox, cyc = c.y - oy;
    if (!(n1 > below_1e6())) {
        // (double)norm1 < 1e-6 or NaN: the reference never votes for this pixel (.cu:121)
    } else if (!(n1 < 1e18f) || !(fabsf(cxc) + fabsf(cyc) <= cmax)) {
        ra.z = 0.f;
    } else {
        const float inv = 1.0f / n1;
        const float ux = v.x * inv, uy = v.y * inv;
        const float a1 = kappa * ux, a2 = kappa * uy;
        ra.x = a1; ra.y = a2; ra.z = -fmaf(a1, cxc, a2 * cyc);
        ra.w = -uy; rb.x = ux; rb.y = fmaf(uy, cxc, -(ux * cyc));
    }
}

// Hypothesis q relative to the tile origin, (hxc, hyc), and its guard band dl.  Non-finite or huge: (0, 0, inf), so every
// test of it takes the exact path.
__device__ __forceinline__ float3 hyp_frame(float2 q, float ox, float oy, float cmax, const ConeParams &cone)
{
    float xc = q.x - ox, yc = q.y - oy;
    const float S = fabsf(xc) + fabsf(yc) + cmax;
    float d = fmaxf(cone.band * S, cone.floor);    // the floor binds only for tiles narrower than ~0.4 px
    if (!(S <= 1e15f) || !(d < CUDART_INF_F)) { xc = 0.f; yc = 0.f; d = CUDART_INF_F; }
    return make_float3(xc, yc, d);
}

// WS = warps that together hold one hypothesis slice (HPT*WS*32 hypotheses).  With fewer than 512 hypotheses per
// keypoint the remaining NT/32/WS warp teams of the CTA split the tile's 16-pixel blocks between them, so every
// thread still owns HPT hypotheses and the inner loop keeps its instruction mix.
// BOX (pass 1): every warp holds the whole slice, so each warp finds the box of its hypotheses on its own.  The tile's
// pixels are classified once against that box (box_class); certain inliers count for every hypothesis without a test,
// certain outliers are dropped, and the undecided ones are compacted to the front of the tile's records, which the inner
// loop then scores as before, guard band and exact path included.
template <int HPT, int NT, int MINB, int VOTE_TILE, int WS, bool BOX>
__global__ void __launch_bounds__(NT, MINB)
vote_kernel(const VoteK p)
{
    static_assert(!BOX || WS == 1, "the box path needs every warp to hold the whole slice");
    constexpr int PPT = VOTE_TILE / NT;               // pixels staged per thread
    constexpr int NW = NT / 32;
    constexpr int TEAM = WS * 32;                     // threads per hypothesis slice
    constexpr int TEAMS = NT / TEAM;                  // teams sharing the staged tile
    __shared__ __align__(16) float4 s_a[VOTE_TILE];   // (A1, A2, A3, B1)
    __shared__ __align__(16) float2 s_b[VOTE_TILE];   // (B2, B3)
    __shared__ float s_box[4][NW];
    __shared__ uint16_t s_idx[BOX ? VOTE_TILE : 1];   // BOX: tile index of each compacted record
    __shared__ int s_nu[BOX ? PPT : 1][NW];           // BOX: undecided pixels per round and warp
    const VoteArgs &a = p.a;
    const int b = blockIdx.z;
    const int k = blockIdx.y % a.K, slice = blockIdx.y / a.K;
    const int tn = min(a.tn[b], a.cap);                 // thin_gather's: two or more launches back (common.cuh)
    const int t0 = blockIdx.x * VOTE_TILE;
    const size_t bk = (size_t)b * a.K + k;
    if (t0 >= tn) { grid_dep_wait(); return; }
    const int *lst = p.list ? p.list + bk * a.hn : nullptr;
    const int n = min(VOTE_TILE, tn - t0);
    const int npad = (n + VOTE_BLOCK - 1) / VOTE_BLOCK * VOTE_BLOCK;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float kappa = p.cone.kappa, thresh = p.cone.thresh;
    const float2 *hyp = a.hyp + bk * a.hn;
    const float2 *xy = a.xy + (size_t)b * a.cap + t0;
    const float2 *dk = a.dirs + ((size_t)b * a.K + k) * a.cap + t0;
    const int team = tid / TEAM;
    const int hbase = slice * (TEAM * HPT) + (tid - team * TEAM);

    // ---- stage 1: load this tile's pixels -> tile-local origin for the fast path.  Stages 1 and 2 read only thin_gather's
    // output, so in pass 1 they run while the bound kernel finishes
    float2 v[PPT], c[PPT];
    float ox, oy, cmax;
    load_tile<NT, PPT>(dk, xy, n, v, c, s_box, ox, oy, cmax);

    // ---- stage 2: cone records
#pragma unroll
    for (int r = 0; r < PPT; ++r) {
        const int i = tid + r * NT;
        if (i < npad) {
            float4 ra;
            float2 rb;
            cone_record(i < n, v[r], c[r], ox, oy, cmax, kappa, ra, rb);
            s_a[i] = ra; s_b[i] = rb;
        }
    }

    // the hypotheses and the list are the predecessors' output, and the counts are zeroed by generate
    grid_dep_wait();
    grid_dep_launch_dependents();
    const int nh = p.list ? __ldcg(p.len + bk) : a.hn;     // hypothesis slots of this (image, keypoint)
    if (slice * (TEAM * HPT) >= nh) return;

    // ---- hypotheses of this thread, relative to the tile origin
    float hxc[HPT], hyc[HPT], dl[HPT];
    int neg[HPT];   // tests whose margin is negative (sign bit) = non-inliers, padding included
#pragma unroll
    for (int j = 0; j < HPT; ++j) {
        const int s = hbase + j * TEAM;
        const float2 q = (s < nh) ? hyp[lst ? __ldcg(lst + s) : s] : make_float2(0.f, 0.f);
        const float3 f = hyp_frame(q, ox, oy, cmax, p.cone);
        hxc[j] = f.x; hyc[j] = f.y; dl[j] = f.z;
        neg[j] = 0;
    }
    __syncthreads();

    int nl = n;     // records scored one hypothesis at a time: the first nl of the tile's (after compaction, with BOX)
    int cin = 0;    // BOX: certain inliers among the pixels this warp classified
    if constexpr (BOX) {
        float x0 = CUDART_INF_F, x1 = -CUDART_INF_F, y0 = CUDART_INF_F, y1 = -CUDART_INF_F;
        bool unb = false;
#pragma unroll
        for (int j = 0; j < HPT; ++j) {
            if (hbase + j * TEAM < nh) {
                x0 = fminf(x0, hxc[j]); x1 = fmaxf(x1, hxc[j]); y0 = fminf(y0, hyc[j]); y1 = fmaxf(y1, hyc[j]);
                unb |= !(dl[j] < CUDART_INF_F);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, o));
            y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, o));
        }
        // the box's guard band: hyp_frame's at the corner of largest |h-o|_1
        const float S = fmaxf(fabsf(x0), fabsf(x1)) + fmaxf(fabsf(y0), fabsf(y1)) + cmax;
        float d = fmaxf(p.cone.band * S, p.cone.floor);
        if (__any_sync(0xffffffffu, unb) || !(d < CUDART_INF_F)) d = CUDART_INF_F;
        int base = 0;
#pragma unroll
        for (int r = 0; r < PPT; ++r) {
            const int i = tid + r * NT;
            float4 ra = make_float4(0.f, 0.f, 0.f, 0.f);
            float2 rb = make_float2(0.f, 0.f);
            int cls = -1;   // beyond the tile: nothing to score
            if (i < n) { ra = s_a[i]; rb = s_b[i]; cls = box_class(ra, rb, x0, x1, y0, y1, d); }
            const unsigned um = __ballot_sync(0xffffffffu, cls == 0);
            cin += __popc(__ballot_sync(0xffffffffu, cls == 1));
            if (lane == 0) s_nu[r][warp] = __popc(um);
            // every read of this round's records comes before the barrier.  The round's writes below go to slots below
            // (r+1)*NT, which no later round reads
            __syncthreads();
            int off = base;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                const int c = s_nu[r][w];
                off += (w < warp) ? c : 0;
                base += c;
            }
            if (cls == 0) {
                const int o = off + __popc(um & ((1u << lane) - 1u));
                s_a[o] = ra; s_b[o] = rb; s_idx[o] = (uint16_t)i;
            }
        }
        nl = base;
        if (p.stats) {   // tooling (pvb_set_pass1_stats): off in production
            if (lane == 0) atomicAdd(p.stats, (unsigned long long)cin * nh);
            if (tid == 0) { atomicAdd(p.stats + 1, (unsigned long long)(n - nl) * nh); atomicAdd(p.stats + 2, (unsigned long long)nl * nh); }
        }
        const int pad = (nl + VOTE_BLOCK - 1) / VOTE_BLOCK * VOTE_BLOCK - nl;
        if (tid < pad) { s_a[nl + tid] = make_float4(0.f, 0.f, -1e30f, 0.f); s_b[nl + tid] = make_float2(0.f, 0.f); }
        __syncthreads();
    }
    const int nlpad = (nl + VOTE_BLOCK - 1) / VOTE_BLOCK * VOTE_BLOCK;

    const uint32_t sa0 = (uint32_t)__cvta_generic_to_shared(s_a);
    const uint32_t sb0 = (uint32_t)__cvta_generic_to_shared(s_b);
    int mine = 0;   // pixels (padding included) this team has scored
    for (int i0 = team * VOTE_BLOCK; i0 < nlpad; i0 += TEAMS * VOTE_BLOCK) {
        mine += VOTE_BLOCK;
        const uint32_t sa = sa0 + (uint32_t)i0 * 16u, sb = sb0 + (uint32_t)i0 * 8u;
        float mn[HPT];   // smallest |margin| of each hypothesis over this block
#pragma unroll
        for (int j = 0; j < HPT; ++j) mn[j] = CUDART_INF_F;
#pragma unroll
        for (int u = 0; u < VOTE_BLOCK; u += 2) {
            const float4 ra0 = lds128(sa + u * 16), ra1 = lds128(sa + u * 16 + 16);
            const float4 rbb = lds128(sb + u * 8);          // (B2,B3) of pixels u and u+1
#pragma unroll
            for (int j = 0; j < HPT; ++j) {
                const float m0 = cone_margin(ra0, make_float2(rbb.x, rbb.y), hxc[j], hyc[j]);
                const float m1 = cone_margin(ra1, make_float2(rbb.z, rbb.w), hxc[j], hyc[j]);
                neg[j] += (int)(__float_as_uint(m0) >> 31);
                neg[j] += (int)(__float_as_uint(m1) >> 31);
                mn[j] = fminf(mn[j], fminf(fabsf(m0), fabsf(m1)));
            }
        }
        bool flag = false;
#pragma unroll
        for (int j = 0; j < HPT; ++j) flag |= mn[j] < dl[j];
        if (__any_sync(0xffffffffu, flag)) {
            // rare, warp-cooperative: for every (lane, j) whose block has a margin inside the guard band, 16 lanes
            // re-test one pixel each against that hypothesis with the reference's exact operation sequence; the
            // reduced correction goes back to the owning lane (fast verdict = sign bit of m)
            const int nb = min(VOTE_BLOCK, nl - i0);     // padding stays "not an inlier"
            float4 ra = make_float4(0.f, 0.f, -1e30f, 0.f);
            float2 rb = make_float2(0.f, 0.f), vv = make_float2(0.f, 0.f), cc = make_float2(0.f, 0.f);
            if (lane < nb) {
                const int px = BOX ? (int)s_idx[i0 + lane] : i0 + lane;
                ra = s_a[i0 + lane]; rb = s_b[i0 + lane];
                vv = __ldg(dk + px); cc = __ldg(xy + px);
            }
#pragma unroll
            for (int j = 0; j < HPT; ++j) {
                unsigned bm = __ballot_sync(0xffffffffu, mn[j] < dl[j]);
                while (bm) {
                    const int L = __ffs(bm) - 1;
                    bm &= bm - 1;
                    const float hx_ = __shfl_sync(0xffffffffu, hxc[j], L), hy_ = __shfl_sync(0xffffffffu, hyc[j], L);
                    const float dl_ = __shfl_sync(0xffffffffu, dl[j], L);
                    const int s = hbase - lane + L + j * TEAM;
                    const float2 q = (s < nh) ? __ldg(hyp + (lst ? __ldcg(lst + s) : s)) : make_float2(0.f, 0.f);
                    int delta = 0;
                    if (lane < nb) {
                        const float m = cone_margin(ra, rb, hx_, hy_);
                        if (fabsf(m) < dl_) {
                            const bool in = vote_exact(vv.x, vv.y, cc.x, cc.y, q.x, q.y, thresh);
                            delta = (in ? 0 : 1) - (int)(__float_as_uint(m) >> 31);
                        }
                    }
                    delta = __reduce_add_sync(0xffffffffu, delta);
                    if (lane == L) neg[j] += delta;
                }
            }
        }
    }
    int *counts = a.counts + bk * a.hn;
#pragma unroll
    for (int j = 0; j < HPT; ++j) {
        const int s = hbase + j * TEAM;
        const int cnt = mine - neg[j] + cin;
        if (s < nh && cnt) atomicAdd(counts + (lst ? __ldcg(lst + s) : s), cnt);
    }
}

// Host side of the guard band (DESIGN.md "Guard band"), u = 2^-24:
//   a test is re-evaluated exactly when |m| < band * S,  S = |hx-ox| + |hy-oy| + max_tile(|cx-ox|+|cy-oy|)
//   band = 1.25 * u * (18 + 22*kappa + 9*G),  kappa = sqrt(1-t^2)/t,  G = 1/(t*sqrt(1-t^2)).
// 2*(9+11*kappa)*u*S bounds twice the rounding error of m itself; 9*G*u*|h-c| is how far the reference's
// fp32 cos can sit from the exact one, mapped into units of m; |h-c| <= S.  tools/band_check.c finds the
// largest |m| of a fast/exact disagreement at 0.35x this bound (1e8 boundary samples).
// The band never falls below floor = 2e-6*(kappa+1): the reference rejects every test with norm2 = |h-c| < 1e-6 whatever
// the angle, and |m| <= (kappa+1)*|h-c| + err with err <= band*S/2.5 <= 0.4*floor, so every such test is flagged.  band*S
// is below the floor only when S < ~0.4 px (t = 0.99), i.e. for tiles whose pixels (nearly) share one position.
ConeParams make_cone(float thresh)
{
    ConeParams c;
    c.thresh = thresh;
    const double t = (double)thresh;
    if (t > 0.0 && t < 1.0) {
        const double s = sqrt(1.0 - t * t);
        const double kappa = s / t, G = 1.0 / (t * s);
        const double band = 1.25 * ldexp(1.0, -24) * (18.0 + 22.0 * kappa + 9.0 * G);
        c.kappa = (float)kappa;
        c.band = nextafterf((float)band, INFINITY);
        c.floor = nextafterf((float)(2e-6 * (kappa + 1.0)), INFINITY);
    } else {
        c.kappa = 0.f;
        c.band = INFINITY;   // threshold outside (0,1): exact path for every test
        c.floor = INFINITY;
    }
    return c;
}

// 0 / 1 -> 1024-pixel tile (the default); 2 / 3 -> 256 / 512-pixel tile (tooling: tools/tune_vote.py).  Up to 256
// hypotheses per keypoint the tile is always 512.  Results do not depend on it.  Atomic: may be flipped while other host
// threads launch.
static std::atomic<int> g_vote_variant{0};

void set_vote_tuning(int variant) { g_vote_variant.store(variant, std::memory_order_relaxed); }

// Tooling: pass 1's per-box test counts (VoteK::stats), summed into a device buffer of 3 words while it is set.  Atomic:
// may be set while other host threads launch.
static std::atomic<unsigned long long *> g_pass1_stats{nullptr};

void set_pass1_stats(unsigned long long *dev) { g_pass1_stats.store(dev, std::memory_order_relaxed); }

cudaError_t launch_vote(const VoteArgs &a, bool zero_counts, bool chained, cudaStream_t st)
{
    if (zero_counts) {     // callers that did not run generate_kernel (which zeroes the counts it creates hypotheses for)
        cudaError_t e = cudaMemsetAsync(a.counts, 0, sizeof(int) * (size_t)a.B * a.K * a.hn, st);
        if (e != cudaSuccess) return e;
    }
    VoteK p;
    p.a = a;
    p.cone = make_cone(a.thresh);
    p.list = nullptr;
    p.len = nullptr;
    p.stats = nullptr;
    const int variant = g_vote_variant.load(std::memory_order_relaxed);
    cudaError_t e = cudaSuccess;
#define PVB_VOTE(HPT, NT, MINB, TILE, WS)                                               \
    do {                                                                                \
        const int slices = (a.hn + (HPT) * (WS) * 32 - 1) / ((HPT) * (WS) * 32);        \
        dim3 g((a.cap + (TILE) - 1) / (TILE), a.K * slices, a.B);                       \
        e = launch_chained(chained, vote_kernel<HPT, NT, MINB, TILE, WS, false>, g, NT, 0, st, p); \
    } while (0)
    if (a.hn <= 32) PVB_VOTE(1, 128, 8, 512, 1);
    else if (a.hn <= 64) PVB_VOTE(2, 128, 8, 512, 1);
    else if (a.hn <= 128) PVB_VOTE(4, 128, 8, 512, 1);
    else if (a.hn <= 256) PVB_VOTE(4, 128, 8, 512, 2);
    else if (variant == 2) PVB_VOTE(4, 128, 8, 256, 4);
    else if (variant == 3) PVB_VOTE(4, 128, 8, 512, 4);
    else PVB_VOTE(4, 128, 8, 1024, 4);    // H100 (400 W), cfg-2: 0.72 ms per launch vs 0.75 ms with 512-pixel tiles
#undef PVB_VOTE
    return e;
}

// The pruned v3 vote's list kernel: vote_kernel turned inside out.  A CTA owns one (image, keypoint, 1024-pixel tile) and
// the whole list; every thread keeps LIST_PPT pixels as cone records in registers, and the list's hypotheses stream
// past as broadcasts from shared memory, staged LIST_CHUNK at a time.  The loop runs over the list's real length, so a list
// of 63 hypotheses costs 63, not a padded slice, and a tile's records are built once for the whole list: the lists of pass 2
// have any length from 0 to hn - PRUNE_M.  Records, origin and guard band are vote_kernel's (load_tile, cone_record,
// hyp_frame), and so is every count.  One CTA per tile and list builds the records once (H100, cfg-2 pass 2: 122 us, against
// 137 us for one CTA per 64 entries and 140 us for two CTAs per list).  A copy of the records in shared memory serves the
// rare exact path (122 us, against 145 us when the path rebuilds the records from v and c).  96 registers, no spills, 5 CTAs per SM.
constexpr int LIST_NT = 128;
constexpr int LIST_PPT = 8;                          // pixels per thread
constexpr int LIST_TILE = LIST_NT * LIST_PPT;
constexpr int LIST_CHUNK = LIST_NT;                  // list entries staged at a time, one per thread
constexpr int LIST_U = 2;                            // hypotheses per loop iteration
static_assert(LIST_CHUNK % LIST_U == 0 && LIST_U % 2 == 0, "");

// Rare: re-tests this thread's pixels whose margin against hypothesis q falls inside its guard band with the reference's exact
// operation sequence (fast verdict = sign bit of m) and returns the correction to the thread's count of non-inliers.  The
// records come from the CTA's copy in shared memory, so the path indexes no register array and finds the pixels inside the
// band with one load and 5 instructions each; padding (i >= n) stays "not an inlier".
__device__ __forceinline__ int list_exact(const float4 q, const float4 *s_a, const float2 *s_b, const float2 *hyp, const float2 *dk,
                                          const float2 *xy, int n, float thresh)
{
    const float2 hq = __ldg(hyp + __float_as_int(q.w));
    int d = 0;
    for (int i = threadIdx.x; i < n; i += LIST_NT) {
        const float m = cone_margin(s_a[i], s_b[i], q.x, q.y);
        if (fabsf(m) < q.z) {
            const float2 vv = __ldg(dk + i), cc = __ldg(xy + i);
            d += (vote_exact(vv.x, vv.y, cc.x, cc.y, hq.x, hq.y, thresh) ? 0 : 1) - (int)(__float_as_uint(m) >> 31);
        }
    }
    return d;
}

__global__ void __launch_bounds__(LIST_NT, 5)
vote_list_kernel(const VoteArgs a, const ConeParams cone, const int *__restrict__ list, const int *__restrict__ len)
{
    constexpr int NW = LIST_NT / 32;
    __shared__ __align__(16) float4 s_a[LIST_TILE];     // the records again, for the exact path
    __shared__ __align__(16) float2 s_b[LIST_TILE];
    __shared__ __align__(16) float4 s_h[LIST_CHUNK];    // (hxc, hyc, dl, hypothesis index bits)
    __shared__ unsigned s_tally[NW][LIST_CHUNK / 2];    // inliers per warp of entries 2i, 2i+1 (16-bit halves)
    __shared__ float s_box[4][NW];
    const int b = blockIdx.z;
    const int k = blockIdx.y;
    // The list is prune_next's output, and a CTA whose list is empty exits before it builds its records: building them
    // before the wait cost more in the CTAs of empty lists than it hid (DESIGN.md 4.3), so the wait comes first
    grid_dep_wait();
    grid_dep_launch_dependents();
    const int tn = min(a.tn[b], a.cap);
    const int t0 = blockIdx.x * LIST_TILE;
    const size_t bk = (size_t)b * a.K + k;
    const int nh = __ldcg(len + bk);
    if (t0 >= tn || nh <= 0) return;
    const int n = min(LIST_TILE, tn - t0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int *lst = list + bk * a.hn;
    const float2 *hyp = a.hyp + bk * a.hn;
    const float2 *xy = a.xy + (size_t)b * a.cap + t0;
    const float2 *dk = a.dirs + bk * a.cap + t0;

    int h = 0;                                          // this thread's first list entry, loaded while the pixels are
    float2 hq = make_float2(0.f, 0.f);
    if (tid < nh) { h = __ldcg(lst + tid); hq = hyp[h]; }
    float4 ra[LIST_PPT];
    float2 rb[LIST_PPT];
    float ox, oy, cmax;
    {
        float2 v[LIST_PPT], c[LIST_PPT];
        load_tile<LIST_NT, LIST_PPT>(dk, xy, n, v, c, s_box, ox, oy, cmax);
#pragma unroll
        for (int r = 0; r < LIST_PPT; ++r) {
            cone_record(tid + r * LIST_NT < n, v[r], c[r], ox, oy, cmax, cone.kappa, ra[r], rb[r]);
            s_a[tid + r * LIST_NT] = ra[r]; s_b[tid + r * LIST_NT] = rb[r];
        }
    }
    unsigned *tally = s_tally[warp];
    for (int c0 = 0; c0 < nh; c0 += LIST_CHUNK) {
        const int ns = min(LIST_CHUNK, nh - c0);
        if (c0 > 0 && tid < ns) { h = __ldcg(lst + c0 + tid); hq = hyp[h]; }
        if (tid < ns) {
            const float3 f = hyp_frame(hq, ox, oy, cmax, cone);
            s_h[tid] = make_float4(f.x, f.y, f.z, __int_as_float(h));
        } else {
            s_h[tid] = make_float4(0.f, 0.f, 0.f, 0.f);   // rounds the loop up to LIST_U: band 0 is never re-tested
        }
        __syncthreads();
        for (int s = 0; s < ns; s += LIST_U) {
            float4 q[LIST_U];
            int neg[LIST_U];            // tests whose margin is negative (sign bit) = non-inliers, padding included
            float mn[LIST_U];           // smallest |margin|
            bool flag = false;
#pragma unroll
            for (int u = 0; u < LIST_U; ++u) {
                q[u] = s_h[s + u];
                neg[u] = 0;
                mn[u] = CUDART_INF_F;
#pragma unroll
                for (int r = 0; r < LIST_PPT; ++r) {
                    const float m = cone_margin(ra[r], rb[r], q[u].x, q[u].y);
                    neg[u] += (int)(__float_as_uint(m) >> 31);
                    mn[u] = fminf(mn[u], fabsf(m));
                }
                flag |= mn[u] < q[u].z;
            }
            if (flag) {
#pragma unroll
                for (int u = 0; u < LIST_U; ++u)
                    if (mn[u] < q[u].z) neg[u] += list_exact(q[u], s_a, s_b, hyp, dk, xy, n, cone.thresh);
            }
            // a thread's tally is at most LIST_PPT, a warp's at most 256: two fit one 32-bit reduction
#pragma unroll
            for (int u = 0; u < LIST_U; u += 2) {
                const unsigned t = __reduce_add_sync(0xffffffffu, (unsigned)(LIST_PPT - neg[u]) | ((unsigned)(LIST_PPT - neg[u + 1]) << 16));
                if (lane == 0) tally[(s + u) / 2] = t;
            }
        }
        __syncthreads();
        if (tid < ns) {
            int cnt = 0;
#pragma unroll
            for (int w = 0; w < NW; ++w) cnt += (int)((s_tally[w][tid / 2] >> (16 * (tid & 1))) & 0xffffu);
            if (cnt) atomicAdd(a.counts + bk * a.hn + __float_as_int(s_h[tid].w), cnt);
        }
        // the next chunk's staging writes only this thread's s_h slot; s_tally is rewritten after the barrier that follows it
    }
}

cudaError_t launch_vote_list(const VoteArgs &a, const int *list, const int *len, int max_len, cudaStream_t st)
{
    if (max_len <= 0) return cudaSuccess;
    dim3 g((a.cap + LIST_TILE - 1) / LIST_TILE, a.K, a.B);
    return launch_chained(true, vote_list_kernel, g, LIST_NT, 0, st, a, make_cone(a.thresh), list, len);
}

// Pass 1: vote_kernel over a full list, in (HPT*32)-hypothesis slices (WS = 1) whose four warps split the 1024-pixel tile.
// With a whole slice per list it scores faster than vote_list_kernel (H100, cfg-2: 192 against 238 us).  BOX: each tile's
// pixels are classified once against the box of the list (box_class); the model predicts 2.1x fewer instructions at cfg-2.
cudaError_t launch_vote_list_slices(const VoteArgs &a, const int *list, const int *len, int max_len, cudaStream_t st)
{
    constexpr int HPT = 4, NT = 128, TILE = 1024;
    static_assert(HPT * 32 == PRUNE_M, "pass 1 is one slice");
    if (max_len <= 0) return cudaSuccess;
    VoteK p;
    p.a = a;
    p.cone = make_cone(a.thresh);
    p.list = list;
    p.len = len;
    p.stats = g_pass1_stats.load(std::memory_order_relaxed);
    const int slices = (max_len + HPT * 32 - 1) / (HPT * 32);
    dim3 g((a.cap + TILE - 1) / TILE, a.K * slices, a.B);
    return launch_chained(true, vote_kernel<HPT, NT, 8, TILE, 1, true>, g, NT, 0, st, p);
}

// Multi-GPU exchange tail shared by the refit and the covariance kernel: one thread stores NV floats of unit `bk` into every
// peer's receive slot (r == own rank: local) as self-validating 8-byte words {float bits, seq} (kernels.h, PeerPush).
template <int NV>
__device__ __forceinline__ void peer_push(const PeerPush &pp, size_t bk, const float (&v)[NV])
{
    for (int r = 0; r < pp.world; ++r) {
        uint2 *dst = pp.recv[r] + bk * NV;
#pragma unroll
        for (int i = 0; i < NV; ++i)
            asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(dst + i), "r"(__float_as_uint(v[i])), "r"(pp.seq) : "memory");
    }
}

// ---------------------------------------------------------------------------------
// winner (torch.max semantics: first maximal index, ransac_voting_gpu.py:160-167) + least-squares
// refit over the winner's inliers (:177-196).  RF_CHUNK pixels per CTA, ticketed deterministic reduction.
// ---------------------------------------------------------------------------------
constexpr int RF_THREADS = 128;
constexpr int RF_CHUNK = 2048;     // pixels per CTA

int refit_splits_for(int cap) { return (cap + RF_CHUNK - 1) / RF_CHUNK; }

// The reference predicate for ONE hypothesis (the winner) against many pixels: same cone test and guard band as the
// vote kernel, with the pixel itself as origin (d = RN(h-c) is the reference's own rounded difference) and without
// normalising v:  m' = kappa*(v.d) - |v x d| = |v|*m,  flagged when m'^2 < (band*|d|_1)^2*|v|^2 (or anything unusual),
// in which case the exact operation sequence decides.  S = |d|_1 >= 2e-6 keeps |d|_2 >= 1.41e-6, clear of the reference's
// norm2 < 1e-6 cut, which the cone test cannot see; closer hypotheses take the exact path.
__device__ __forceinline__ bool vote_winner(float vx, float vy, float cx, float cy, float hx, float hy,
                                            const ConeParams &cone)
{
    const float dx = __fsub_rn(hx, cx), dy = __fsub_rn(hy, cy);
    const float n1sq = fmaf(vx, vx, vy * vy);
    const float S = fabsf(dx) + fabsf(dy);
    const float m = cone.kappa * fmaf(vx, dx, vy * dy) - fabsf(fmaf(vx, dy, -(vy * dx)));
    const float thr = cone.band * S;
    const bool safe = (n1sq > 1e-10f) && (n1sq < 1e8f) && (S >= 2e-6f) && (S <= 1e6f) &&
                      (m * m > thr * thr * n1sq * 1.0001f);
    return safe ? (m > 0.f) : vote_exact(vx, vy, cx, cy, hx, hy, cone.thresh);
}

__global__ void __launch_bounds__(RF_THREADS)
refit_kernel(VoteArgs a, float2 *__restrict__ win, RefitScratch rs, float *__restrict__ out, ConeParams cone, PeerPush pp)
{
    // the counts are the last vote pass's output.  The last kernel of the chain: no dependent to trigger (common.cuh)
    grid_dep_wait();
    const int split = blockIdx.x, k = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = RF_THREADS / 32;
    const int tn = min(a.tn[b], a.cap);
    const size_t bk = (size_t)b * a.K + k;
    __shared__ int s_c[NW], s_h[NW];
    __shared__ double s_acc[NW][5];
    __shared__ int s_last;
    // Exactly one CTA per (image, keypoint) writes out[bk]: CTA 0 of a skipped image, otherwise the CTA that draws the
    // last ticket.  Only those CTAs reach the exchange tail at the bottom.
    float2 res = make_float2(0.f, 0.f);   // this (image, keypoint)'s result, held by thread 0 of the CTA that writes it
    if (a.state[b] != 0 || tn <= 0) {   // :129-132 -> zeros
        if (split != 0) return;
        if (tid == 0) { out[bk * 2] = 0.f; out[bk * 2 + 1] = 0.f; win[bk] = make_float2(0.f, 0.f); }
    } else {
        const int nsplit = (tn + RF_CHUNK - 1) / RF_CHUNK;   // CTAs that have pixels for this image
        if (split >= nsplit) return;
        // winner: every CTA of this (image,keypoint) finds it on its own (hn counts, L2-resident)
        const int *counts = a.counts + bk * a.hn;
        int bc = -1, bh = 0x7fffffff;
        for (int h = tid; h < a.hn; h += RF_THREADS) {
            const int c = counts[h];
            if (c > bc) { bc = c; bh = h; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int oc = __shfl_xor_sync(0xffffffffu, bc, o), oh = __shfl_xor_sync(0xffffffffu, bh, o);
            if (oc > bc || (oc == bc && oh < bh)) { bc = oc; bh = oh; }
        }
        if (lane == 0) { s_c[warp] = bc; s_h[warp] = bh; }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < NW; ++w)
            if (s_c[w] > bc || (s_c[w] == bc && s_h[w] < bh)) { bc = s_c[w]; bh = s_h[w]; }
        // all_win_ratio starts at 0 and is replaced only by a strictly larger ratio (:165-167)
        const float2 wpt = (bc > 0) ? a.hyp[bk * a.hn + bh] : make_float2(0.f, 0.f);
        if (split == 0 && tid == 0) win[bk] = wpt;

        const float2 *xy = a.xy + (size_t)b * a.cap;
        const float2 *dk = a.dirs + bk * a.cap;
        const int t_end = min(tn, (split + 1) * RF_CHUNK);
        double a00 = 0, a01 = 0, a11 = 0, b0 = 0, b1 = 0;
        constexpr int RU = 4;     // loads in flight per thread (the loop is latency bound: 16 pixels per thread)
        for (int t0 = split * RF_CHUNK + tid; t0 < t_end; t0 += RF_THREADS * RU) {
            float2 v[RU], c[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                const int t = t0 + u * RF_THREADS;
                v[u] = make_float2(0.f, 0.f); c[u] = make_float2(0.f, 0.f);
                if (t < t_end) { v[u] = __ldg(dk + t); c[u] = __ldg(xy + t); }
            }
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                if (t0 + u * RF_THREADS < t_end && vote_winner(v[u].x, v[u].y, c[u].x, c[u].y, wpt.x, wpt.y, cone)) {
                    const double nx = (double)v[u].y, ny = -(double)v[u].x;       // normal = (d_y, -d_x)  (:178-180)
                    const double bb = nx * (double)c[u].x + ny * (double)c[u].y;   // b = n . c             (:189)
                    a00 += nx * nx; a01 += nx * ny; a11 += ny * ny;                // ATA                   (:190)
                    b0 += nx * bb; b1 += ny * bb;                                  // ATb                   (:191)
                }
            }
        }
        a00 = warp_sum(a00); a01 = warp_sum(a01); a11 = warp_sum(a11); b0 = warp_sum(b0); b1 = warp_sum(b1);
        if (lane == 0) { s_acc[warp][0] = a00; s_acc[warp][1] = a01; s_acc[warp][2] = a11; s_acc[warp][3] = b0; s_acc[warp][4] = b1; }
        __syncthreads();
        if (tid == 0) {
            double *pq = rs.partial + (bk * rs.splits + split) * 5;
            for (int i = 0; i < 5; ++i) {
                double s = 0;
                for (int w = 0; w < NW; ++w) s += s_acc[w][i];
                __stcg(pq + i, s);
            }
            __threadfence();
            s_last = (atomicAdd(rs.ticket + bk, 1) == nsplit - 1);
        }
        __syncthreads();
        if (!s_last) return;
        if (tid == 0) {
            __threadfence();
            double s[5] = {0, 0, 0, 0, 0};
            for (int sp = 0; sp < nsplit; ++sp)            // fixed order -> deterministic sums
                for (int i = 0; i < 5; ++i) s[i] += __ldcg(rs.partial + (bk * rs.splits + sp) * 5 + i);
            const double det = s[0] * s[2] - s[1] * s[1];
            float x, y;
            if (det == 0.0 || !isfinite(det)) { x = (float)s[3]; y = (float)s[4]; }   // b_inv's identity fallback (:105-108)
            else { x = (float)((s[2] * s[3] - s[1] * s[4]) / det); y = (float)((s[0] * s[4] - s[1] * s[3]) / det); }
            out[bk * 2] = x; out[bk * 2 + 1] = y;
            res = make_float2(x, y);
        }
    }
    // ---- exchange tail (multi-GPU): the thread that produced this (image, keypoint) result stores it into every peer's
    // receive slot over NVLink (r == own rank: local) as two self-validating 8-byte words {float bits, seq}.  Fire and
    // forget: no fence, no counter, no flag (kernels.h, PeerPush).
    if (pp.world <= 0 || tid != 0) return;
    const float v[2] = {res.x, res.y};
    peer_push<2>(pp, bk, v);
}

cudaError_t launch_refit(const VoteArgs &a, float2 *win, const RefitScratch &rs, float *out_kpt, const PeerPush &pp,
                         cudaStream_t st)
{
    dim3 g(rs.splits, a.K, a.B);
    return launch_chained(true, refit_kernel, g, RF_THREADS, 0, st, a, win, rs, out_kpt, make_cone(a.thresh), pp);
}

// ---------------------------------------------------------------------------------
// covariance of the hypothesis cloud (ransac_voting_gpu.py:243-244, 254-269)
// ---------------------------------------------------------------------------------
constexpr int CV_THREADS = 256;

__global__ void __launch_bounds__(CV_THREADS)
covariance_kernel(VoteArgs a, const float *__restrict__ mean, float *__restrict__ cov, PeerPush pp)
{
    const int k = blockIdx.x, b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t bk = (size_t)b * a.K + k;
    const int tn = min(a.tn[b], a.cap);
    const bool skipped = a.state[b] != 0;          // :211-216  hyp zeros, ratio ones
    const int *counts = a.counts + bk * a.hn;
    const float2 *hyp = a.hyp + bk * a.hn;
    const float ftn = (float)tn;
    __shared__ float s_max[CV_THREADS / 32];
    __shared__ double s_acc[CV_THREADS / 32][4];
    float mx = -CUDART_INF_F;
    bool has_nan = false;
    for (int h = tid; h < a.hn; h += CV_THREADS) {
        const float r = skipped ? 1.f : __fdiv_rn((float)counts[h], ftn);
        if (r != r) has_nan = true;
        mx = fmaxf(mx, r);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();
    mx = s_max[0];
    for (int w = 1; w < CV_THREADS / 32; ++w) mx = fmaxf(mx, s_max[w]);
    (void)has_nan;   // tn == 0 without skip cannot happen for min_num >= 1; ratios would be NaN as in the reference
    const float th = __fsub_rn(mx, 0.1f);
    const float mx_ = mean[bk * 2], my_ = mean[bk * 2 + 1];
    double s00 = 0, s01 = 0, s11 = 0, sw = 0;
    for (int h = tid; h < a.hn; h += CV_THREADS) {
        float w = skipped ? 1.f : __fdiv_rn((float)counts[h], ftn);
        if (w < th) w = 0.f;
        const float2 q = skipped ? make_float2(0.f, 0.f) : hyp[h];
        const double dx = (double)__fsub_rn(q.x, mx_), dy = (double)__fsub_rn(q.y, my_);
        s00 += dx * (dx * w); s01 += dx * (dy * w); s11 += dy * (dy * w); sw += w;
    }
    s00 = warp_sum(s00); s01 = warp_sum(s01); s11 = warp_sum(s11); sw = warp_sum(sw);
    if (lane == 0) { s_acc[warp][0] = s00; s_acc[warp][1] = s01; s_acc[warp][2] = s11; s_acc[warp][3] = sw; }
    __syncthreads();
    if (tid == 0) {
        double s[4] = {0, 0, 0, 0};
        for (int w = 0; w < CV_THREADS / 32; ++w)
            for (int i = 0; i < 4; ++i) s[i] += s_acc[w][i];
        const double den = (double)__fadd_rn((float)s[3], 1e-3f);
        float *c = cov + bk * 4;
        const float v[4] = {(float)(s[0] / den), (float)(s[1] / den), (float)(s[1] / den), (float)(s[2] / den)};
        c[0] = v[0]; c[1] = v[1]; c[2] = v[2]; c[3] = v[3];
        if (pp.world > 0) peer_push<4>(pp, bk, v);          // multi-GPU: the 2x2 covariance goes to every peer as it is produced
    }
}

cudaError_t launch_covariance(const VoteArgs &a, const float *mean, float *out_cov, const PeerPush &pp, cudaStream_t st)
{
    dim3 g(a.K, a.B);
    covariance_kernel<<<g, CV_THREADS, 0, st>>>(a, mean, out_cov, pp);
    return cudaGetLastError();
}

} // namespace pvb
