/* box_check.c -- empirical check of pass 1's per-box classification (DESIGN.md 4.2, "Pass 1 per box of hypotheses").
 *
 * Re-states, for the host, cone_record, hyp_frame and box_class of clean_pvnet_b200/csrc/vote.cu (same IEEE operation
 * sequence: fmaf / fp32 mul,add,div,sqrt; build with -ffp-contract=off) next to the reference predicate (vote_one, as
 * in tools/band_check.c) and searches adversarial boxes of hypotheses for a pixel the box calls a certain inlier or a
 * certain outlier while the reference disagrees for some hypothesis of the box.  Boxes are drawn around the pixel itself
 * (the apex), on its cone edge, across the back of the cone and at random, from zero or one ulp wide to 50 px.  The
 * hypotheses that span the box and further points inside it are all tested.  Reports the disagreements (exit code 1 if
 * any) and the worst case: the smallest |m| / delta_H of a tested hypothesis of a decided pixel.
 *   gcc -O2 -mfma -ffp-contract=off tools/box_check.c -lm -o /tmp/box_check
 *   usage: box_check [boxes [thresh]]
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

static uint64_t s[2] = {0x9E3779B97F4A7C15ull, 0xD1B54A32D192ED03ull};
static inline uint64_t rnd(void)
{
    uint64_t s1 = s[0], s0 = s[1];
    s[0] = s0; s1 ^= s1 << 23; s[1] = s1 ^ s0 ^ (s1 >> 17) ^ (s0 >> 26);
    return s[1] + s0;
}
static inline double uni(void) { return (rnd() >> 11) * (1.0 / 9007199254740992.0); }

/* cone_record for a pixel inside the analysed domain (the others never reach a decided class) */
static void cone_record(float vx, float vy, float cx, float cy, float ox, float oy, float kappa, float r[6])
{
    const float n1 = sqrtf(fmaf(vx, vx, vy * vy));
    const float cxc = cx - ox, cyc = cy - oy;
    const float inv = 1.0f / n1, ux = vx * inv, uy = vy * inv;
    const float a1 = kappa * ux, a2 = kappa * uy;
    r[0] = a1; r[1] = a2; r[2] = -fmaf(a1, cxc, a2 * cyc);
    r[3] = -uy; r[4] = ux; r[5] = fmaf(uy, cxc, -(ux * cyc));
}

static inline float margin(const float r[6], float x, float y, float *ap, float *pp)
{
    *ap = fmaf(r[0], x, fmaf(r[1], y, r[2]));
    *pp = fmaf(r[3], x, fmaf(r[4], y, r[5]));
    return *ap - fabsf(*pp);
}

static int box_class(const float r[6], float x0, float x1, float y0, float y1, float d)
{
    float mn = INFINITY, lp = -INFINITY, lm = -INFINITY;
    for (int q = 0; q < 4; ++q) {
        const float x = (q & 1) ? x1 : x0, y = (q & 2) ? y1 : y0;
        float ap, pp;
        mn = fminf(mn, margin(r, x, y, &ap, &pp));
        lp = fmaxf(lp, ap + pp);
        lm = fmaxf(lm, ap - pp);
    }
    return (mn > d) ? 1 : (lp < -d || lm < -d) ? -1 : 0;
}

int main(int argc, char **argv)
{
    const long n = argc > 1 ? atol(argv[1]) : 20000000L;
    const float thresh = argc > 2 ? (float)atof(argv[2]) : 0.99f;
    const double t = (double)thresh, sq = sqrt(1.0 - t * t);
    const float kappa = (float)(sq / t);
    const double G = 1.0 / (t * sq), u = ldexp(1.0, -24), theta = acos(t);
    const float bandf = nextafterf((float)(1.25 * u * (18.0 + 22.0 * kappa + 9.0 * G)), INFINITY);   /* make_cone() */
    const float floorf_ = nextafterf((float)(2e-6 * ((double)kappa + 1.0)), INFINITY);
    static const double widths[] = {0.0, 0.0, 1e-6, 1e-3, 0.05, 0.5, 5.0, 50.0};
    enum { NH = 4, NIN = 8 };
    long mism = 0, decided = 0, tested = 0;
    double worst = INFINITY;
    for (long it = 0; it < n; ++it) {
        const float cx = (float)(int)(uni() * 640), cy = (float)(int)(uni() * 480);
        const float bx0 = cx - (float)(int)(uni() * 300), bx1 = cx + (float)(int)(uni() * 300);
        const float by0 = cy - (float)(int)(uni() * 4), by1 = cy + (float)(int)(uni() * 4);
        const float ox = 0.5f * (bx0 + bx1), oy = 0.5f * (by0 + by1);
        const float cmax = (0.5f * (bx1 - bx0) + 0.5f * (by1 - by0)) * 1.000001f + 1e-3f;
        const double a = uni() * 2 * M_PI, nv = (uni() < 0.8) ? 1.0 : exp((uni() - 0.5) * 8);
        const float vx = (float)(cos(a) * nv), vy = (float)(sin(a) * nv);
        float r[6];
        cone_record(vx, vy, cx, cy, ox, oy, kappa, r);
        /* the box's centre: the apex, the cone edge (either side), the back of the cone, or anywhere nearby */
        const int kind = (int)(uni() * 4);
        const double dist = kind == 0 ? uni() * 1e-4 : exp(uni() * log(400.0)) * 0.5;
        const double ang = kind == 1 ? a + (uni() < 0.5 ? -1 : 1) * theta * (1.0 + (uni() - 0.5) * 1e-3)
                         : kind == 2 ? a + M_PI + (uni() - 0.5) * 2 * theta : uni() * 2 * M_PI;
        const double ex = cx + dist * cos(ang), ey = cy + dist * sin(ang);
        const int wi = (int)(uni() * 8);
        const double w = widths[wi];
        float hx[NH + NIN], hy[NH + NIN];
        for (int j = 0; j < NH; ++j) {
            hx[j] = (float)(ex + w * uni()); hy[j] = (float)(ey + w * uni());
            if (wi == 1) {   /* one ulp wide */
                hx[j] = (j & 1) ? nextafterf((float)ex, INFINITY) : (float)ex;
                hy[j] = (j & 2) ? nextafterf((float)ey, INFINITY) : (float)ey;
            }
        }
        /* hyp_frame and the box of the NH spanning hypotheses, as vote_kernel forms it */
        float x0 = INFINITY, x1 = -INFINITY, y0 = INFINITY, y1 = -INFINITY;
        for (int j = 0; j < NH; ++j) {
            const float xc = hx[j] - ox, yc = hy[j] - oy;
            x0 = fminf(x0, xc); x1 = fmaxf(x1, xc); y0 = fminf(y0, yc); y1 = fmaxf(y1, yc);
        }
        const float S = fmaxf(fabsf(x0), fabsf(x1)) + fmaxf(fabsf(y0), fabsf(y1)) + cmax;
        const float d = fmaxf(bandf * S, floorf_);
        const int cls = box_class(r, x0, x1, y0, y1, d);
        if (cls == 0) continue;
        ++decided;
        /* further hypotheses whose frame falls inside the box */
        int nh = NH;
        for (int j = 0; j < NIN; ++j) {
            const float qx = (float)(ex + w * uni()), qy = (float)(ey + w * uni());
            const float xc = qx - ox, yc = qy - oy;
            if (xc >= x0 && xc <= x1 && yc >= y0 && yc <= y1) { hx[nh] = qx; hy[nh] = qy; ++nh; }
        }
        for (int j = 0; j < nh; ++j) {
            float ap, pp;
            const float m = margin(r, hx[j] - ox, hy[j] - oy, &ap, &pp);
            const double q = fabs((double)m) / d;
            if (q < worst) worst = q;
            ++tested;
            if (vote_one(vx, vy, cx, cy, hx[j], hy[j], thresh) != (cls == 1)) {
                if (++mism <= 10)
                    printf("MISMATCH t=%g class %d pixel (%g,%g) v (%.9g,%.9g) h (%.9g,%.9g) m %.3e delta %.3e\n", t, cls, cx, cy,
                           vx, vy, hx[j], hy[j], m, d);
            }
        }
    }
    printf("t=%g boxes=%ld decided=%ld tested=%ld mismatches=%ld worst |m|/delta_H=%.6f\n", t, n, decided, tested, mism,
           worst);
    return mism ? 1 : 0;
}
