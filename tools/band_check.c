/* band_check.c -- empirical check of the vote kernel's guard band (DESIGN.md "Guard band").
 *
 * Re-states, for the host, the fast cone test of clean_pvnet_b200/csrc/vote.cu (same IEEE operation
 * sequence: fmaf / fp32 mul,add,div,sqrt; build with -ffp-contract=off) next to the reference predicate
 * (oracle vote_one == ransac_voting_kernel.cu:107-125) and searches, with samples concentrated on the
 * cone boundary, for tests where the two disagree.  For every disagreement it records
 *      r = |m| / (u * S),   u = 2^-24,  S = |hx-ox| + |hy-oy| + cmax
 * The kernel flags a test for exact re-evaluation when |m| < band * S; the band constant must stay
 * above max r with margin.   gcc -O2 -mfma -ffp-contract=off tools/band_check.c -lm -o /tmp/band_check
 *
 * A second, exhaustive sweep covers what the boundary sampler cannot reach: hypotheses within a few ulps of (or on) a
 * pixel at small integer coordinates, where 0 < |h-c| < 1e-6 and the reference's norm cut rejects the pixel whatever
 * the angle.  It checks the refit prefilter and the vote kernel's fast path for a tile of one pixel (cmax = 1e-3, the
 * narrowest box), whose band is held up by the floor of make_cone().
 *   usage: band_check [samples [thresh [local]]]     samples = 0 runs the near-pixel sweep only
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

static inline int vote_one(float vx, float vy, float cx, float cy, float hx, float hy, float thresh)
{
    float dx = hx - cx, dy = hy - cy;
    float n1sq = fmaf(vx, vx, vy * vy), n2sq = fmaf(dx, dx, dy * dy);
    float norm1 = sqrtf(n1sq), norm2 = sqrtf(n2sq);
    if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) return 0;
    float den = norm2 * norm1, dot = fmaf(vx, dx, vy * dy);
    return dot / den > thresh;
}

/* the refit's prefilter (vote_winner in vote.cu): 1 = decided without the exact path, verdict in *in */
static inline int winner_fast(float vx, float vy, float cx, float cy, float hx, float hy, float kappa, float bandf, int *in)
{
    float ddx = hx - cx, ddy = hy - cy;
    float n1sq = fmaf(vx, vx, vy * vy);
    float Sd = fabsf(ddx) + fabsf(ddy);
    float mw = kappa * fmaf(vx, ddx, vy * ddy) - fabsf(fmaf(vx, ddy, -(vy * ddx)));
    float thr = bandf * Sd;
    *in = mw > 0.f;
    return (n1sq > 1e-10f) && (n1sq < 1e8f) && (Sd >= 2e-6f) && (Sd <= 1e6f) && (mw * mw > thr * thr * n1sq * 1.0001f);
}

static uint64_t s[2] = {0x9E3779B97F4A7C15ull, 0xD1B54A32D192ED03ull};
static inline uint64_t rnd(void)
{
    uint64_t s1 = s[0], s0 = s[1];
    s[0] = s0; s1 ^= s1 << 23; s[1] = s1 ^ s0 ^ (s1 >> 17) ^ (s0 >> 26);
    return s[1] + s0;
}
static inline double uni(void) { return (rnd() >> 11) * (1.0 / 9007199254740992.0); }

int main(int argc, char **argv)
{
    long n = argc > 1 ? atol(argv[1]) : 200000000L;
    float thresh = argc > 2 ? (float)atof(argv[2]) : 0.99f;
    int W = 640, H = 480;
    const int local = argc > 3 ? atoi(argv[3]) : 1;   /* 1: tile-local origin like the kernel, 0: image centre */
    const double t = (double)thresh, sq = sqrt(1.0 - t * t);
    const float kappa = (float)(sq / t);
    const double G = 1.0 / (t * sq), u = ldexp(1.0, -24), theta = acos(t);
    const float bandf = nextafterf((float)(1.25 * u * (18.0 + 22.0 * kappa + 9.0 * G)), INFINITY);   /* make_cone() */
    const float floorf_ = nextafterf((float)(2e-6 * ((double)kappa + 1.0)), INFINITY);
    double rmax = 0, rmax_d = 0;
    long mism = 0, near = 0, w_total = 0, w_safe = 0;
    for (long it = 0; it < n; ++it) {
        /* pixel, direction (norm around 1 with jitter, like a network output) */
        float cx = (float)(int)(uni() * W), cy = (float)(int)(uni() * H);
        /* tile bounding box containing the pixel: a few rows high, up to the blob width wide */
        float ox, oy, cmax;
        if (local) {
            float bx0 = cx - (float)(int)(uni() * 300), bx1 = cx + (float)(int)(uni() * 300);
            float by0 = cy - (float)(int)(uni() * 4), by1 = cy + (float)(int)(uni() * 4);
            ox = 0.5f * (bx0 + bx1); oy = 0.5f * (by0 + by1);
            cmax = (0.5f * (bx1 - bx0) + 0.5f * (by1 - by0)) * 1.000001f + 1e-3f;
        } else {
            ox = 0.5f * (W - 1); oy = 0.5f * (H - 1); cmax = 0.5f * (W - 1) + 0.5f * (H - 1) + 1.0f;
        }
        double a = uni() * 2 * M_PI, nv = (uni() < 0.8) ? 1.0 : exp((uni() - 0.5) * 8);
        float vx = (float)(cos(a) * nv), vy = (float)(sin(a) * nv);
        /* hypothesis on the cone boundary of this pixel, perturbed by a few ulp-scale amounts */
        double r = exp(uni() * 11.0 - 1.0);                       /* 0.37 .. 22000 px */
        double side = (rnd() & 1) ? 1.0 : -1.0;
        double eps = (uni() - 0.5) * 4e-6 * ((rnd() & 3) ? 1.0 : 50.0);
        double ang = atan2((double)vy, (double)vx) + side * (theta + eps);
        float hx = (float)(cx + r * cos(ang)), hy = (float)(cy + r * sin(ang));
        /* fast path, exactly as vote.cu */
        float n1 = sqrtf(fmaf(vx, vx, vy * vy));
        if (!(n1 > 9.99999997e-7f) || !(n1 < 1e18f)) continue;
        float cxc = cx - ox, cyc = cy - oy;
        float inv = 1.0f / n1, ux = vx * inv, uy = vy * inv;
        float a1 = kappa * ux, a2 = kappa * uy;
        float A3 = -fmaf(a1, cxc, a2 * cyc);
        float B1 = -uy, B2 = ux, B3 = fmaf(uy, cxc, -(ux * cyc));
        /* refit prefilter (vote_winner in vote.cu): pixel-origin, unnormalised */
        {
            int in;
            ++w_total;
            if (winner_fast(vx, vy, cx, cy, hx, hy, kappa, bandf, &in)) {
                ++w_safe;
                if (in != vote_one(vx, vy, cx, cy, hx, hy, thresh)) { printf("WINNER PREFILTER MISMATCH\n"); return 1; }
            }
        }
        float hxc = hx - ox, hyc = hy - oy;
        float ap = fmaf(a1, hxc, fmaf(a2, hyc, A3));
        float pp = fmaf(B1, hxc, fmaf(B2, hyc, B3));
        float m = ap - fabsf(pp);
        int fast = !(m < 0.0f) && !(m == 0.0f && signbit(m));   /* sign bit clear -> tallied as inlier */
        int exact = vote_one(vx, vy, cx, cy, hx, hy, thresh);
        double S = fabs((double)hxc) + fabs((double)hyc) + cmax;
        double d = hypot((double)hx - cx, (double)hy - cy);
        const double band = 1.25 * (18.0 + 22.0 * kappa + 9.0 * G);     /* make_cone() in vote.cu */
        if (fabs(m) < band * u * S) ++near;
        if (fast != exact) {
            ++mism;
            if (!(fabs(m) < band * u * S)) { printf("UNFLAGGED MISMATCH m=%g S=%g\n", m, S); return 1; }
            double rr = fabs((double)m) / (u * S);
            double rd = fabs((double)m) / (u * (S * (9 + 11 * kappa) * 2 + 9.0 * G * d));   /* vs analytic bound */
            if (rr > rmax) rmax = rr;
            if (rd > rmax_d) rmax_d = rd;
        }
    }
    printf("thresh=%.6f kappa=%.6f G=%.3f  samples=%ld  mismatches=%ld  in-band=%ld\n", thresh, kappa, G, n, mism, near);
    printf("max |m|/(u*S) over mismatches = %.3f   (kernel band constant 1.25*(18+22k+9G) = %.1f)\n",
           rmax, 1.25 * (18 + 22 * kappa + 9 * G));
    printf("refit prefilter: %ld of %ld boundary samples decided without the exact path, 0 disagreements\n", w_safe, w_total);
    printf("max |m| / analytic bound [2*err_fast(S) + 9uG|d|] = %.3f (must be < 1)\n", rmax_d);

    /* near-pixel sweep: pixel (cx, cy) in [0,16)^2, hypothesis cx + i ulp, cy + j ulp (|i|, |j| <= 2), 40 directions:
     * towards h, on its cone boundary, random, with norms around 1 */
    long nn = 0, n_cut = 0, n_wsafe = 0, n_flag = 0;
    for (int cy = 0; cy < 16; ++cy)
        for (int cx = 0; cx < 16; ++cx)
            for (int i = -2; i <= 2; ++i)
                for (int j = -2; j <= 2; ++j) {
                    float hx = (float)cx, hy = (float)cy;
                    for (int q = 0; q < (i < 0 ? -i : i); ++q) hx = nextafterf(hx, i < 0 ? -INFINITY : INFINITY);
                    for (int q = 0; q < (j < 0 ? -j : j); ++q) hy = nextafterf(hy, j < 0 ? -INFINITY : INFINITY);
                    const double a0 = atan2((double)hy - cy, (double)hx - cx);
                    for (int r = 0; r < 40; ++r) {
                        double a = r == 0 ? a0 : r < 5 ? a0 + ((r & 1) ? 1 : -1) * theta * (r < 3 ? 1 + 1e-7 : 1 - 1e-7)
                                                       : uni() * 2 * M_PI;
                        double nv = (r & 2) ? 1.0 : exp((uni() - 0.5) * 4);
                        float vx = (float)(cos(a) * nv), vy = (float)(sin(a) * nv);
                        const int exact = vote_one(vx, vy, (float)cx, (float)cy, hx, hy, thresh);
                        ++nn;
                        if (i || j) n_cut += !exact;
                        int in;
                        if (winner_fast(vx, vy, (float)cx, (float)cy, hx, hy, kappa, bandf, &in)) {
                            ++n_wsafe;
                            if (in != exact) { printf("NEAR-PIXEL WINNER PREFILTER MISMATCH c=(%d,%d) h=(%.9g,%.9g)\n", cx, cy, hx, hy); return 1; }
                        }
                        /* vote kernel, a tile of this one pixel: origin = the pixel, cmax = 1e-3 */
                        float n1 = sqrtf(fmaf(vx, vx, vy * vy));
                        if (!(n1 > 9.99999997e-7f) || !(n1 < 1e18f)) continue;
                        float inv = 1.0f / n1, ux = vx * inv, uy = vy * inv;
                        float a1 = kappa * ux, a2 = kappa * uy;
                        float A3 = -fmaf(a1, 0.f, a2 * 0.f), B3 = fmaf(uy, 0.f, -(ux * 0.f));
                        float hxc = hx - (float)cx, hyc = hy - (float)cy;
                        float m = fmaf(a1, hxc, fmaf(a2, hyc, A3)) - fabsf(fmaf(-uy, hxc, fmaf(ux, hyc, B3)));
                        float S = fabsf(hxc) + fabsf(hyc) + ((0.f + 0.f) * 1.000001f + 1e-3f);
                        float d = fmaxf(bandf * S, floorf_);
                        int fast = !signbit(m);
                        if (fabsf(m) < d) { ++n_flag; continue; }
                        if (fast != exact) { printf("NEAR-PIXEL UNFLAGGED MISMATCH c=(%d,%d) h=(%.9g,%.9g) m=%g band=%g\n", cx, cy, hx, hy, m, d); return 1; }
                    }
                }
    printf("near-pixel sweep: %ld tests, %ld rejected by the norm cut, %ld decided by the refit prefilter, "
           "%ld flagged in one-pixel tiles, 0 disagreements\n", nn, n_cut, n_wsafe, n_flag);
    return 0;
}
