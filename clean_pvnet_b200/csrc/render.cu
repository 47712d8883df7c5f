// render.cu -- T-LESS's VSD on the device (DESIGN.md section 8f): a depth rasterizer that renders what the reference's
// OpenGL DepthRender renders (lib/utils/renderer/opengl_utils.py:405-490), and the VSD error of vsd_utils.vsd with the
// 'step' cost (lib/utils/vsd/vsd_utils.py:5-48) for n (estimate, ground truth, image) rows.
//
// Renderer semantics (derived in DESIGN.md 8f): pixel (row r, column c) samples the camera ray through
// (u, v) = (c + 0.5, r + 0.5), u = fx X/Z + s Y/Z + cx, v = fy Y/Z + cy.  The stored value is the camera-frame Z of the
// nearest triangle's plane along that ray, kept when near <= Z <= far, rounded to fp32; 0 where nothing is hit.  R and t
// are rounded to fp32 first, as the shader's float32 view matrix does; the transform itself runs in fp64.
//
// Rasterization is homogeneous (no division by Z before the coverage test), so triangles that cross the near plane or
// lie behind the camera need no polygon clipping: with P' = K P for the three vertices (K-space, third component Z) and
// r' = (u, v, 1), the ray hits the triangle iff the three edge functions E_bc, E_ca, E_ab (E_ab = r' . (P'a x P'b)) all
// have the sign of D = det(P'a, P'b, P'c), and then Z = D / (E_bc + E_ca + E_ab).  Near and far are a per-pixel test on
// that Z, which is what clipping against the two planes keeps.
//
// Watertightness: an edge shared by two triangles is always evaluated from its endpoints in one canonical order (the
// lexicographically smaller model-space vertex first), so both triangles compute the same E bit for bit and each uses
// its sign or its negation.  E == 0 (a pixel centre exactly on the edge) takes the sign E has an infinitesimal step
// along (1, eps) from the pixel centre, i.e. sign(dE/du), else sign(dE/dv).  This is one consistent perturbation of the
// sample point, so every pixel centre on a shared edge or vertex is covered by the triangles on exactly one side.
//
// Depth is kept by atomicMin on the bits of the positive fp32 Z in an image filled with +inf, then +inf becomes 0; the
// minimum does not depend on the order of the atomics, so the output is bit-identical run to run and each pose's image
// depends on nothing else in the batch.
#include <algorithm>
#include <cmath>
#include <vector>
#include "api.h"

namespace pvb {

struct VsdArgs {
    const float *depth_test, *depth_est, *depth_gt;  // [B][H][W], [n_est][H][W], [n_gt][H][W]
    const int *pairs;                                // [n][3]: est index, gt index, image index
    const double *K;                                 // [3][3] per image at K + image * k_stride
    long long k_stride;
    int n, B, n_est, n_gt, est_base, gt_base, H, W;  // rows use est in [est_base, est_base + n_est), likewise gt
    double delta, tau;
    double *e;                                       // [n]: written only for rows within the windows
};

namespace {

constexpr int RENDER_THREADS = 256;
constexpr int RENDER_SMALL_PIXELS = 64;      // a triangle whose clipped screen box has more pixels goes to a CTA of its own
constexpr unsigned RENDER_BG = 0x7f800000u;  // +inf: farther than every covered pixel
constexpr int VSD_THREADS = 256;
constexpr int VSD_PIXELS = VSD_THREADS * 16; // pixels per CTA of the VSD count kernel

struct Tri {
    double3 c[3];      // canonical edge coefficients of edges (b,c), (c,a), (a,b): E = c.x u + c.y v + c.z
    double D;          // det(P'a, P'b, P'c)
    int x0, x1, y0, y1; // inclusive pixel box, clipped to the image; x0 > x1 when empty
    int f[3];          // +1 when the triangle's edge runs in the canonical order, -1 when reversed
    int tie[3];        // the sign a canonical E takes at E == 0
};

__device__ __forceinline__ bool vlt(float3 a, float3 b)
{
    return a.x < b.x || (a.x == b.x && (a.y < b.y || (a.y == b.y && a.z < b.z)));
}

__device__ __forceinline__ double3 cross3(double3 a, double3 b)
{
    return make_double3(__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)),
                        __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
                        __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)));
}

__device__ __forceinline__ double dot3(double3 a, double3 b)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}

// camera-frame point of model point p under the fp32-rounded pose (R row-major, t) in fp64
__device__ __forceinline__ double3 to_camera(const float *R, float3 p)
{
    double3 q;
    q.x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[0], p.x), __dmul_rn(R[1], p.y)), __dmul_rn(R[2], p.z)), (double)R[3]);
    q.y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[4], p.x), __dmul_rn(R[5], p.y)), __dmul_rn(R[6], p.z)), (double)R[7]);
    q.z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[8], p.x), __dmul_rn(R[9], p.y)), __dmul_rn(R[10], p.z)), (double)R[11]);
    return q;
}

// K-space point (fx X + s Y + cx Z, fy Y + cy Z, Z); k = fx, s, cx, fy, cy
__device__ __forceinline__ double3 to_kspace(const double *k, double3 P)
{
    return make_double3(__dadd_rn(__dadd_rn(__dmul_rn(k[0], P.x), __dmul_rn(k[1], P.y)), __dmul_rn(k[2], P.z)),
                        __dadd_rn(__dmul_rn(k[3], P.y), __dmul_rn(k[4], P.z)), P.z);
}

__device__ __forceinline__ void box_add(const double *k, double3 P, double &u0, double &u1, double &v0, double &v1)
{
    const double3 q = to_kspace(k, P);
    const double u = __ddiv_rn(q.x, q.z), v = __ddiv_rn(q.y, q.z);
    u0 = fmin(u0, u); u1 = fmax(u1, u); v0 = fmin(v0, v); v1 = fmax(v1, v);
}

// the point of segment a-b at Z == z (a.z and b.z on either side)
__device__ __forceinline__ double3 at_z(double3 a, double3 b, double z)
{
    const double s = __ddiv_rn(__dsub_rn(z, a.z), __dsub_rn(b.z, a.z));
    return make_double3(__dadd_rn(a.x, __dmul_rn(s, __dsub_rn(b.x, a.x))),
                        __dadd_rn(a.y, __dmul_rn(s, __dsub_rn(b.y, a.y))), z);
}

// Sets up triangle `face` of pose `pose`; returns false when it cannot cover any pixel (bad index, non-finite or
// edge-on, or nothing of it within [near, far] and the image).
__device__ bool tri_setup(const float *__restrict__ pts, int V, const int *__restrict__ faces, int face,
                          const double *__restrict__ pose, const double *__restrict__ K, int H, int W, double znear,
                          double zfar, Tri &t)
{
    int id[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        id[j] = __ldg(faces + 3 * face + j);
        if (id[j] < 0 || id[j] >= V) return false;
    }
    float R[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) R[j] = __double2float_rn(__ldg(pose + j));
    double k[5] = {__ldg(K + 0), __ldg(K + 1), __ldg(K + 2), __ldg(K + 4), __ldg(K + 5)};
    float3 m[3];
    double3 P[3], Q[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        m[j] = make_float3(__ldg(pts + 3 * id[j]), __ldg(pts + 3 * id[j] + 1), __ldg(pts + 3 * id[j] + 2));
        P[j] = to_camera(R, m[j]);
        Q[j] = to_kspace(k, P[j]);
        if (!isfinite(Q[j].x) || !isfinite(Q[j].y) || !isfinite(Q[j].z)) return false;
    }
    // edge j joins vertices (j+1)%3 and (j+2)%3: (b,c), (c,a), (a,b)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const int a = (j + 1) % 3, b = (j + 2) % 3;
        const bool rev = vlt(m[b], m[a]);
        t.f[j] = rev ? -1 : 1;
        t.c[j] = rev ? cross3(Q[b], Q[a]) : cross3(Q[a], Q[b]);
        t.tie[j] = t.c[j].x > 0.0 ? 1 : t.c[j].x < 0.0 ? -1 : t.c[j].y > 0.0 ? 1 : t.c[j].y < 0.0 ? -1 : 0;
    }
    t.D = t.f[0] > 0 ? dot3(Q[0], t.c[0]) : -dot3(Q[0], t.c[0]);
    if (!(t.D != 0.0) || !isfinite(t.D)) return false;
    // screen box of the part of the triangle with near <= Z <= far: its vertices inside the slab and its edges'
    // crossings of the two planes
    double u0 = INFINITY, u1 = -INFINITY, v0 = INFINITY, v1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const double3 a = P[j], b = P[(j + 1) % 3];
        if (a.z >= znear && a.z <= zfar) box_add(k, a, u0, u1, v0, v1);
        if ((a.z < znear) != (b.z < znear)) box_add(k, at_z(a, b, znear), u0, u1, v0, v1);
        if ((a.z > zfar) != (b.z > zfar)) box_add(k, at_z(a, b, zfar), u0, u1, v0, v1);
    }
    if (!(u0 <= u1) || !(v0 <= v1)) return false;
    // pixel c is in the box when c + 0.5 lies in [u0, u1]; the margin keeps a centre the rounded box would miss
    const double mu = 1e-6 + 1e-9 * fmax(fabs(u0), fabs(u1)), mv = 1e-6 + 1e-9 * fmax(fabs(v0), fabs(v1));
    t.x0 = (int)fmax(0.0, ceil(u0 - 0.5 - mu));
    t.x1 = (int)fmin((double)(W - 1), floor(u1 - 0.5 + mu));
    t.y0 = (int)fmax(0.0, ceil(v0 - 0.5 - mv));
    t.y1 = (int)fmin((double)(H - 1), floor(v1 - 0.5 + mv));
    return t.x0 <= t.x1 && t.y0 <= t.y1;
}

__device__ __forceinline__ void tri_pixel(const Tri &t, int x, int y, double znear, double zfar, unsigned *__restrict__ img,
                                          int W)
{
    const double u = (double)x + 0.5, v = (double)y + 0.5;
    const int want = t.D > 0.0 ? 1 : -1;
    double sum = 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const double e = __fma_rn(t.c[j].x, u, __fma_rn(t.c[j].y, v, t.c[j].z));
        const int s = e > 0.0 ? 1 : e < 0.0 ? -1 : t.tie[j];
        if (s * t.f[j] != want) return;
        sum = __dadd_rn(sum, t.f[j] > 0 ? e : -e);
    }
    const double z = __ddiv_rn(t.D, sum);
    if (!(z >= znear && z <= zfar)) return;
    atomicMin(img + (long long)y * W + x, __float_as_uint(__double2float_rn(z)));
}

__global__ void __launch_bounds__(RENDER_THREADS)
render_fill_kernel(unsigned *__restrict__ img, long long total, unsigned value)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        img[i] = value;
}

// one thread per (triangle, pose): small boxes are rasterised here, larger ones queued for render_big_kernel
__global__ void __launch_bounds__(RENDER_THREADS)
render_small_kernel(const float *__restrict__ pts, int V, const int *__restrict__ faces, int F,
                    const double *__restrict__ poses, const double *__restrict__ K, long long k_stride, int H, int W,
                    double znear, double zfar, unsigned *__restrict__ depth, unsigned *__restrict__ queue_len,
                    unsigned *__restrict__ queue)
{
    const int face = blockIdx.x * RENDER_THREADS + threadIdx.x;
    const int pose = blockIdx.y;
    if (face >= F) return;
    Tri t;
    if (!tri_setup(pts, V, faces, face, poses + 12ll * pose, K + k_stride * pose, H, W, znear, zfar, t)) return;
    const int bw = t.x1 - t.x0 + 1, bh = t.y1 - t.y0 + 1;
    if ((long long)bw * bh > RENDER_SMALL_PIXELS) {
        queue[atomicAdd(queue_len, 1u)] = (unsigned)pose * (unsigned)F + (unsigned)face;
        return;
    }
    unsigned *img = depth + (long long)pose * H * W;
    for (int y = t.y0; y <= t.y1; ++y)
        for (int x = t.x0; x <= t.x1; ++x) tri_pixel(t, x, y, znear, zfar, img, W);
}

// one CTA per queued triangle at a time; every thread repeats the (deterministic) setup
__global__ void __launch_bounds__(RENDER_THREADS)
render_big_kernel(const float *__restrict__ pts, int V, const int *__restrict__ faces, int F,
                  const double *__restrict__ poses, const double *__restrict__ K, long long k_stride, int H, int W,
                  double znear, double zfar, unsigned *__restrict__ depth, const unsigned *__restrict__ queue_len,
                  const unsigned *__restrict__ queue)
{
    const unsigned nq = *queue_len;
    for (unsigned q = blockIdx.x; q < nq; q += gridDim.x) {
        const unsigned key = queue[q];
        const int pose = (int)(key / (unsigned)F), face = (int)(key % (unsigned)F);
        Tri t;
        if (!tri_setup(pts, V, faces, face, poses + 12ll * pose, K + k_stride * pose, H, W, znear, zfar, t)) continue;
        unsigned *img = depth + (long long)pose * H * W;
        const int bw = t.x1 - t.x0 + 1;
        const long long area = (long long)bw * (t.y1 - t.y0 + 1);
        for (long long i = threadIdx.x; i < area; i += RENDER_THREADS) {
            const int y = t.y0 + (int)(i / bw), x = t.x0 + (int)(i % bw);
            tri_pixel(t, x, y, znear, zfar, img, W);
        }
    }
}

// +inf (no fragment) -> 0, the reference's background
__global__ void __launch_bounds__(RENDER_THREADS)
render_finish_kernel(unsigned *__restrict__ img, long long total)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        if (img[i] == RENDER_BG) img[i] = 0u;
}

int stream_grid(long long total)
{
    const long long b = (total + RENDER_THREADS - 1) / RENDER_THREADS;
    return (int)(b < 132 * 16 ? (b > 0 ? b : 1) : 132 * 16);
}

// ---------------------------------------------------------------------------------------------------------------------
// VSD, vsd_utils.vsd with cost 'step', per row i = (est, gt, image):
//   dist(d) at (r, c) = sqrt((X*X + Y*Y) + Z*Z), X = ((c - cx) * Z) * (1/fx), Y = ((r - cy) * Z) * (1/fy), Z = double(d)
//   (misc.depth_im_to_dist_im's numpy operations, each rounded on its own; np.linalg.norm sums x^2 + y^2 first)
//   visib(model) = dist_test > 0 & dist_model > 0 & float(dist_model) - float(dist_test) <= float(delta)  (visibility.py)
//   vg = visib(gt);  ve = visib(est) | (vg & dist_est > 0)
//   inter = vg & ve, union = vg | ve, cost = inter & |dist_gt - dist_est| >= tau
//   e = (#cost + #union - #inter) / #union, 1.0 when #union == 0
// The counts are integers, so their atomics are exact and e does not depend on the order of the CTAs.
// ---------------------------------------------------------------------------------------------------------------------
struct VsdCounts { unsigned inter, uni, cost, pad; };

__device__ __forceinline__ double dist_px(float d, double cu, double cv, double ifx, double ify)
{
    const double z = (double)d;
    const double X = __dmul_rn(__dmul_rn(cu, z), ifx), Y = __dmul_rn(__dmul_rn(cv, z), ify);
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, X), __dmul_rn(Y, Y)), __dmul_rn(z, z)));
}

__device__ __forceinline__ bool vsd_row(const int *__restrict__ pairs, int i, const VsdArgs &a, int &ie, int &ig, int &ib)
{
    ie = __ldg(pairs + 3 * i) - a.est_base;
    ig = __ldg(pairs + 3 * i + 1) - a.gt_base;
    ib = __ldg(pairs + 3 * i + 2);
    return ie >= 0 && ie < a.n_est && ig >= 0 && ig < a.n_gt && ib >= 0 && ib < a.B;
}

__global__ void __launch_bounds__(VSD_THREADS)
vsd_count_kernel(VsdArgs a, VsdCounts *__restrict__ counts)
{
    __shared__ unsigned s_red[3][VSD_THREADS / 32];
    const int HW = a.H * a.W;
    const float delta = __double2float_rn(a.delta);
    for (int i = blockIdx.y; i < a.n; i += gridDim.y) {
        int ie, ig, ib;
        if (!vsd_row(a.pairs, i, a, ie, ig, ib)) continue;           // uniform over the CTA
        const double *k = a.K + a.k_stride * ib;
        const double fx = __ldg(k + 0), cx = __ldg(k + 2), fy = __ldg(k + 4), cy = __ldg(k + 5);
        const double ifx = __drcp_rn(fx), ify = __drcp_rn(fy);
        const float *dt = a.depth_test + (long long)ib * HW, *de = a.depth_est + (long long)ie * HW,
                    *dg = a.depth_gt + (long long)ig * HW;
        unsigned n_inter = 0, n_uni = 0, n_cost = 0;
        for (int p = blockIdx.x * VSD_PIXELS + threadIdx.x; p < min(HW, (blockIdx.x + 1) * VSD_PIXELS); p += VSD_THREADS) {
            const float t = __ldg(dt + p), e = __ldg(de + p), g = __ldg(dg + p);
            if (t == 0.0f && e == 0.0f && g == 0.0f) continue;      // every distance 0: no mask holds the pixel
            const int r = p / a.W, c = p - r * a.W;
            const double cu = __dsub_rn((double)c, cx), cv = __dsub_rn((double)r, cy);
            const double xt = dist_px(t, cu, cv, ifx, ify), xe = dist_px(e, cu, cv, ifx, ify),
                         xg = dist_px(g, cu, cv, ifx, ify);
            const float ft = __double2float_rn(xt);
            const bool vg = xt > 0.0 && xg > 0.0 && __fsub_rn(__double2float_rn(xg), ft) <= delta;
            const bool ve = (xt > 0.0 && xe > 0.0 && __fsub_rn(__double2float_rn(xe), ft) <= delta) || (vg && xe > 0.0);
            const bool in = vg && ve;
            n_inter += in;
            n_uni += vg || ve;
            n_cost += in && fabs(__dsub_rn(xg, xe)) >= a.tau;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            n_inter += __shfl_xor_sync(0xffffffffu, n_inter, o);
            n_uni += __shfl_xor_sync(0xffffffffu, n_uni, o);
            n_cost += __shfl_xor_sync(0xffffffffu, n_cost, o);
        }
        const int warp = threadIdx.x >> 5;
        if ((threadIdx.x & 31) == 0) { s_red[0][warp] = n_inter; s_red[1][warp] = n_uni; s_red[2][warp] = n_cost; }
        __syncthreads();
        if (threadIdx.x == 0) {
            n_inter = n_uni = n_cost = 0;
#pragma unroll
            for (int w = 0; w < VSD_THREADS / 32; ++w) { n_inter += s_red[0][w]; n_uni += s_red[1][w]; n_cost += s_red[2][w]; }
            if (n_inter) atomicAdd(&counts[i].inter, n_inter);
            if (n_uni) atomicAdd(&counts[i].uni, n_uni);
            if (n_cost) atomicAdd(&counts[i].cost, n_cost);
        }
        __syncthreads();                                             // s_red is reused by the next row
    }
}

__global__ void vsd_final_kernel(VsdArgs a, const VsdCounts *__restrict__ counts)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    int ie, ig, ib;
    if (i >= a.n || !vsd_row(a.pairs, i, a, ie, ig, ib)) return;
    const VsdCounts c = counts[i];
    a.e[i] = c.uni ? __ddiv_rn((double)(c.cost + (c.uni - c.inter)), (double)c.uni) : 1.0;
}

// ---------------------------------------------------------------------------------------------------------------------
// T-LESS's instance masks (DESIGN.md 8k): handle_test_data.update_mask over an image's instances, in order, on the
// depth opengl_renderer.render returns (the mm depth / 1000 in fp32):
//   key = fp32(d / 1000);  the instance takes the pixel when key != 0 and key < depth_map (which starts at 10.0f), so
//   ties go to the earlier instance and a key of 10 or more (or NaN) never takes it
//   label = obj_id * 1000 + instance_id (int16, 0 where no instance took the pixel)
//   a_pixel_num = #(key != 0), pixel_num = #(label pixels of the instance), box = cv2.boundingRect of those pixels
// One CTA per (MASK_PIXELS pixels, image) keeps its pixels' running key and winner in registers over the image's
// instances; the counts and box extremes go through warp reductions and shared atomics, then one global atomic per
// instance and CTA.  Every sum is an integer, so the result is exact and independent of the order of the atomics.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MASK_THREADS = 256;
constexpr int MASK_PPT = 8;                            // pixels per thread
constexpr int MASK_PIXELS = MASK_THREADS * MASK_PPT;
constexpr int MASK_MAX_INSTANCES = 2048;              // per image: their sums take 48 KB of shared memory

// per-instance sums; the box is kept as maxima of W - x, x + 1, H - y, y + 1, which are all 0 for an empty mask, so the
// sums start from a zero fill
struct MaskAcc { unsigned a, p, x0, x1, y0, y1; };

__global__ void __launch_bounds__(MASK_THREADS)
mask_compose_kernel(const float *__restrict__ depth, const int *__restrict__ table, int B, int m, int H, int W,
                    short *__restrict__ label, MaskAcc *__restrict__ acc)
{
    extern __shared__ unsigned s_acc[];                // [instances of this image][6], a MaskAcc each
    const int b = blockIdx.y;
    const int i0 = __ldg(table + b), mi = __ldg(table + b + 1) - i0;
    const int *slot = table + B + 1 + i0, *lab = table + B + 1 + m + i0;
    const int HW = H * W;
    for (int k = threadIdx.x; k < 6 * mi; k += MASK_THREADS) s_acc[k] = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int p0 = blockIdx.x * MASK_PIXELS + threadIdx.x;
    float key[MASK_PPT];
    int win[MASK_PPT];
#pragma unroll
    for (int q = 0; q < MASK_PPT; ++q) { key[q] = 10.0f; win[q] = -1; }
    for (int j = 0; j < mi; ++j) {
        const float *d = depth + (long long)__ldg(slot + j) * HW;
        unsigned nz = 0;
#pragma unroll
        for (int q = 0; q < MASK_PPT; ++q) {
            const int p = p0 + q * MASK_THREADS;
            if (p < HW) {
                const float k = __fdiv_rn(__ldg(d + p), 1000.0f);
                if (k != 0.0f) {
                    ++nz;
                    if (k < key[q]) { key[q] = k; win[q] = j; }
                }
            }
        }
        nz = __reduce_add_sync(0xffffffffu, nz);
        if (lane == 0 && nz) atomicAdd(&s_acc[6 * j], nz);
    }
    short *out = label + (long long)b * HW;
    int px[MASK_PPT], py[MASK_PPT];
#pragma unroll
    for (int q = 0; q < MASK_PPT; ++q) {
        const int p = p0 + q * MASK_THREADS;
        py[q] = p / W;
        px[q] = p - py[q] * W;
        if (p < HW) out[p] = (short)(win[q] >= 0 ? __ldg(lab + win[q]) : 0);
    }
    for (int j = 0; j < mi; ++j) {
        unsigned c = 0, x0 = 0, x1 = 0, y0 = 0, y1 = 0;
#pragma unroll
        for (int q = 0; q < MASK_PPT; ++q)
            if (win[q] == j) {                         // win is -1 past the end of the image
                ++c;
                x0 = max(x0, (unsigned)(W - px[q])); x1 = max(x1, (unsigned)(px[q] + 1));
                y0 = max(y0, (unsigned)(H - py[q])); y1 = max(y1, (unsigned)(py[q] + 1));
            }
        if (!__any_sync(0xffffffffu, c != 0)) continue;
        c = __reduce_add_sync(0xffffffffu, c);
        x0 = __reduce_max_sync(0xffffffffu, x0); x1 = __reduce_max_sync(0xffffffffu, x1);
        y0 = __reduce_max_sync(0xffffffffu, y0); y1 = __reduce_max_sync(0xffffffffu, y1);
        if (lane == 0) {
            unsigned *s = s_acc + 6 * j;
            atomicAdd(s + 1, c);
            atomicMax(s + 2, x0); atomicMax(s + 3, x1); atomicMax(s + 4, y0); atomicMax(s + 5, y1);
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < mi; j += MASK_THREADS) {
        const unsigned *s = s_acc + 6 * j;
        MaskAcc *g = acc + i0 + j;
        if (s[0]) atomicAdd(&g->a, s[0]);
        if (s[1]) {
            atomicAdd(&g->p, s[1]);
            atomicMax(&g->x0, s[2]); atomicMax(&g->x1, s[3]); atomicMax(&g->y0, s[4]); atomicMax(&g->y1, s[5]);
        }
    }
}

__global__ void mask_finish_kernel(const MaskAcc *__restrict__ acc, int m, int H, int W, long long *__restrict__ a_out,
                                   long long *__restrict__ p_out, int *__restrict__ box_out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const MaskAcc s = acc[i];
    a_out[i] = s.a;
    p_out[i] = s.p;
    const int x = s.p ? W - (int)s.x0 : 0, y = s.p ? H - (int)s.y0 : 0;
    box_out[4 * i + 0] = x;
    box_out[4 * i + 1] = y;
    box_out[4 * i + 2] = s.p ? (int)s.x1 - x : 0;
    box_out[4 * i + 3] = s.p ? (int)s.y1 - y : 0;
}

} // namespace

// a queue counter, then the n * F queue entries
// External linkage on purpose: nvcc names this file's anonymous namespace, and so its kernels, after the first
// externally visible definition in the file.
size_t render_workspace_bytes(int n, int F)
{
    return 256 + (((size_t)n * (size_t)F * sizeof(unsigned) + 255) / 256) * 256;
}

namespace {

// the integer counts of the n rows
size_t vsd_workspace_bytes(int n)
{
    return (((size_t)n * sizeof(VsdCounts) + 255) / 256) * 256;
}

size_t mask_table_bytes(int B, int m)
{
    return (((size_t)B + 1 + 2 * (size_t)m) * sizeof(int) + 255) / 256 * 256;
}

// the table, then the integer sums of the m instances
size_t instance_masks_workspace_bytes(int B, int m)
{
    return mask_table_bytes(B, m) + ((size_t)m * sizeof(MaskAcc) + 255) / 256 * 256;
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API size_t pvb_render_depth_workspace_bytes(int32_t n, int32_t F)
{
    if (n <= 0 || F <= 0 || (long long)n * F > 0x7fffffffll) return 0;
    return render_workspace_bytes(n, F);
}

PVB_API int pvb_render_depth(const float *pts, int32_t V, const int32_t *faces, int32_t F, const double *poses, int32_t n,
                             const double *K, int64_t k_stride, float *depth, int32_t H, int32_t W, double clip_near,
                             double clip_far, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    if (n < 0 || V < 0 || F < 0 || H < 0 || W < 0)
        return fail(PVB_ERR_INVALID, "negative size (n=%d V=%d F=%d H=%d W=%d)", n, V, F, H, W);
    if (!(clip_near > 0.0) || !(clip_far >= clip_near) || !std::isfinite(clip_far))
        return fail(PVB_ERR_INVALID, "need 0 < near <= far < inf (got %g, %g)", clip_near, clip_far);
    if ((long long)H * W > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    if ((long long)n * F > 0x7fffffffll) return fail(PVB_ERR_INVALID, "n * F too large (>= 2^31)");
    if (n > 65535) return fail(PVB_ERR_INVALID, "n must be <= 65535 (got %d)", n);
    if (n == 0 || (long long)H * W == 0) return PVB_OK;
    if (!poses || !K || !depth || (F > 0 && (!faces || (V > 0 && !pts)))) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (k_stride < 0) return fail(PVB_ERR_INVALID, "negative stride");
    if (F > 0)
        if (int rc = check_workspace(render_workspace_bytes(n, F), workspace, workspace_bytes)) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned *img = reinterpret_cast<unsigned *>(depth);
    const long long total = (long long)n * H * W;
    render_fill_kernel<<<stream_grid(total), RENDER_THREADS, 0, st>>>(img, total, RENDER_BG);
    cudaError_t e = cudaSuccess;
    if (F > 0) {
        unsigned *queue_len = static_cast<unsigned *>(workspace);
        unsigned *queue = reinterpret_cast<unsigned *>(static_cast<char *>(workspace) + 256);
        e = cudaMemsetAsync(queue_len, 0, sizeof(unsigned), st);
        if (e == cudaSuccess) {
            render_small_kernel<<<dim3((unsigned)((F + RENDER_THREADS - 1) / RENDER_THREADS), (unsigned)n), RENDER_THREADS,
                                  0, st>>>(pts, V, faces, F, poses, K, k_stride, H, W, clip_near, clip_far, img, queue_len,
                                           queue);
            const long long nq = (long long)n * F;
            render_big_kernel<<<(unsigned)(nq < 132 * 8 ? nq : 132 * 8), RENDER_THREADS, 0, st>>>(
                pts, V, faces, F, poses, K, k_stride, H, W, clip_near, clip_far, img, queue_len, queue);
        }
    }
    if (e == cudaSuccess) {
        render_finish_kernel<<<stream_grid(total), RENDER_THREADS, 0, st>>>(img, total);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "depth render kernels");
}

PVB_API size_t pvb_vsd_workspace_bytes(int32_t n)
{
    if (n <= 0) return 0;
    return vsd_workspace_bytes(n);
}

PVB_API int pvb_vsd(const float *depth_test, int32_t B, const float *depth_est, int32_t n_est, int32_t est_base,
                    const float *depth_gt, int32_t n_gt, int32_t gt_base, const int32_t *pairs, int32_t n, const double *K,
                    int64_t k_stride, int32_t H, int32_t W, double delta, double tau, double *e, void *workspace,
                    size_t workspace_bytes, pvb_stream_t stream)
{
    if (n < 0 || B < 0 || n_est < 0 || n_gt < 0 || H < 0 || W < 0)
        return fail(PVB_ERR_INVALID, "negative size (n=%d B=%d n_est=%d n_gt=%d H=%d W=%d)", n, B, n_est, n_gt, H, W);
    if ((long long)H * W > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    if (std::isnan(delta) || std::isnan(tau)) return fail(PVB_ERR_INVALID, "delta and tau must not be NaN");
    if (n == 0) return PVB_OK;
    const bool px = (long long)H * W > 0;
    if (!pairs || !e || !K || (px && ((B > 0 && !depth_test) || (n_est > 0 && !depth_est) || (n_gt > 0 && !depth_gt))))
        return fail(PVB_ERR_INVALID, "NULL tensor");
    if (k_stride < 0) return fail(PVB_ERR_INVALID, "negative stride");
    if (int rc = check_workspace(vsd_workspace_bytes(n), workspace, workspace_bytes)) return rc;
    VsdArgs a;
    a.depth_test = depth_test; a.depth_est = depth_est; a.depth_gt = depth_gt; a.pairs = pairs; a.K = K;
    a.k_stride = k_stride; a.n = n; a.B = B; a.n_est = n_est; a.n_gt = n_gt; a.est_base = est_base; a.gt_base = gt_base;
    a.H = H; a.W = W; a.delta = delta; a.tau = tau; a.e = e;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    VsdCounts *counts = static_cast<VsdCounts *>(workspace);
    cudaError_t err = cudaMemsetAsync(counts, 0, (size_t)n * sizeof(VsdCounts), st);
    if (err == cudaSuccess) {
        const int chunks = (H * W + VSD_PIXELS - 1) / VSD_PIXELS;
        if (chunks > 0)
            vsd_count_kernel<<<dim3((unsigned)chunks, (unsigned)(n < 65535 ? n : 65535)), VSD_THREADS, 0, st>>>(a, counts);
        vsd_final_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, counts);
        err = cudaGetLastError();
    }
    return err == cudaSuccess ? PVB_OK : cuda_fail(err, "vsd kernels");
}

PVB_API size_t pvb_instance_masks_workspace_bytes(int32_t B, int32_t m)
{
    if (B <= 0 || m <= 0) return 0;
    return instance_masks_workspace_bytes(B, m);
}

PVB_API int pvb_instance_masks(const float *depth, int32_t n_depth, const int32_t *slot, const int32_t *obj_id, int32_t n,
                               const int32_t *image_first, int32_t B, int32_t H, int32_t W, int16_t *label,
                               int64_t *a_pixel_num, int64_t *pixel_num, int32_t *bbox, void *workspace,
                               size_t workspace_bytes, pvb_stream_t stream)
{
    if (n_depth < 0 || n < 0 || B < 0 || H < 0 || W < 0)
        return fail(PVB_ERR_INVALID, "negative size (n_depth=%d n=%d B=%d H=%d W=%d)", n_depth, n, B, H, W);
    if ((long long)H * W > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    if (B > 65535) return fail(PVB_ERR_INVALID, "B must be <= 65535 (got %d)", B);
    if (B == 0) return PVB_OK;
    if (!image_first || !slot || !obj_id) return fail(PVB_ERR_INVALID, "NULL host table");
    const bool px = (long long)H * W > 0;
    if (!a_pixel_num || !pixel_num || !bbox || (px && (!depth || !label))) return fail(PVB_ERR_INVALID, "NULL tensor");
    const int32_t i0 = image_first[0];
    if (i0 < 0) return fail(PVB_ERR_INVALID, "image 0's instances start at %d", i0);
    int max_m = 0;
    for (int32_t b = 0; b < B; ++b) {
        const int32_t lo = image_first[b], hi = image_first[b + 1];
        if (hi <= lo || hi > n)
            return fail(PVB_ERR_INVALID, "image %d's instance range [%d, %d) is empty or outside [0, %d)", b, lo, hi, n);
        if (hi - lo > MASK_MAX_INSTANCES)
            return fail(PVB_ERR_INVALID, "image %d has %d instances (at most %d)", b, hi - lo, MASK_MAX_INSTANCES);
        max_m = std::max(max_m, hi - lo);
    }
    // the kernels' table: image b's instances are [table[b], table[b+1]) (table[0] == 0), then the depth slot of each of
    // the m instances, then its label
    const int32_t m = image_first[B] - i0;
    std::vector<int32_t> table((size_t)B + 1 + 2 * (size_t)m);
    for (int32_t b = 0; b <= B; ++b) table[b] = image_first[b] - i0;
    for (int32_t b = 0; b < B; ++b)
        for (int32_t i = image_first[b]; i < image_first[b + 1]; ++i) {
            if (slot[i] < 0 || slot[i] >= n_depth)
                return fail(PVB_ERR_INVALID, "instance %d reads depth slot %d (outside [0, %d))", i, slot[i], n_depth);
            const long long lab = (long long)obj_id[i] * 1000 + (i - image_first[b]);
            if (lab < -32768 || lab > 32767)
                return fail(PVB_ERR_INVALID, "instance %d's label %lld (obj_id * 1000 + instance_id) does not fit int16", i, lab);
            table[B + 1 + (i - i0)] = slot[i];
            table[B + 1 + m + (i - i0)] = (int32_t)lab;
        }
    if (int rc = check_workspace(instance_masks_workspace_bytes(B, m), workspace, workspace_bytes)) return rc;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    int *d_table = static_cast<int *>(workspace);
    MaskAcc *acc = reinterpret_cast<MaskAcc *>(static_cast<char *>(workspace) + mask_table_bytes(B, m));
    // the table is pageable host memory: the copy stages it before returning, so it may go out of scope at once
    cudaError_t e = cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(acc, 0, (size_t)m * sizeof(MaskAcc), st);
    if (e == cudaSuccess) {
        const int chunks = (H * W + MASK_PIXELS - 1) / MASK_PIXELS;
        if (chunks > 0)
            mask_compose_kernel<<<dim3((unsigned)chunks, (unsigned)B), MASK_THREADS, (size_t)max_m * sizeof(MaskAcc), st>>>(
                depth, d_table, B, m, H, W, reinterpret_cast<short *>(label), acc);
        mask_finish_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(
            acc, m, H, W, reinterpret_cast<long long *>(a_pixel_num) + i0, reinterpret_cast<long long *>(pixel_num) + i0,
            bbox + 4ll * i0);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "instance mask kernels");
}

} // extern "C"
