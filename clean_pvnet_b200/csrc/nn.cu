// nn.cu -- exact brute-force nearest neighbour (the twin of lib/csrc/nn/src/nearest_neighborhood.cu:48-117) and the
// ADD / ADD-S distance of lib/evaluators/linemod/pvnet.py:68-82 (tless_test/pvnet.py:107-117) built on it, and the
// evaluators' other two pose metrics, projection_2d and cm_degree_5 (:59-66, :84-94), on the same transform.
//
// The reference predicate, read from the PTX that `nvcc -O2 -arch=sm_52` (its setup.py) emits for the reference source:
//   d? = RN(ref.? - que.?),  3-D: dist = fma(dz, dz, fma(dx, dx, RN(dy*dy))),  2-D: dist = fma(dx, dx, RN(dy*dy))
//   min_dist = FLT_MAX, min_idx = 0; for p1 in 0..pn1-1 (skipping p1 == p2 under exclude_self): dist < min_dist -> take
// The remaining mul feeds the addend of an fma.rn, so no JIT target can contract it further.  Consequences: the first
// minimum in scan order wins; a NaN, +inf or exactly FLT_MAX distance never wins; a query without a finite distance below
// FLT_MAX gets index 0.  nn_dist spells the predicate out with round-to-nearest intrinsics, so the indices are the
// reference's bit for bit.
//
// Layout of the work: a thread keeps NN_Q queries in registers and a CTA stages NN_TILE reference points at a time in
// shared memory, so every point read from shared memory serves NN_Q distance tests of ~9 FP32-pipe instructions each: the
// kernel is issue-bound like the vote kernel.  When b * ceil(pn2 / NN_QPB) CTAs cannot fill the GPU, pn1 is cut into
// slices over CTAs (nn_plan, from the shapes alone) and the slices meet in a 64-bit atomicMin on
//   key = (float bits of dist) << 32 | idx,   starting from (bits of FLT_MAX) << 32 | 0.
// Why the smallest key is the reference's answer: a slice only reports a distance it took under `dist < best` from
// best = FLT_MAX, i.e. a finite non-negative float below FLT_MAX (a sum of squares rounded to nearest is never -0); NaN
// and +inf never get that far, and their bit patterns would sort above FLT_MAX anyway.  For non-negative floats the bit
// patterns order like the values, so the smallest key carries the smallest distance, and among equal distances the
// lowest index -- the first in scan order, which is what the reference's strict `<` keeps.  A slice's own winner is the
// first minimum of its range for the same reason, and when no slice reports, the initial key gives index 0.
#include <algorithm>
#include <cfloat>
#include "common.cuh"
#include "kernels.h"

namespace pvb {

namespace {

constexpr int NN_THREADS = 256;
constexpr int NN_Q = 8;                         // queries per thread, in registers
constexpr int NN_QPB = NN_THREADS * NN_Q;       // queries per CTA
constexpr int NN_TILE = NN_THREADS;             // reference points per shared-memory tile, one loaded per thread
constexpr int NN_MIN_SLICE = 64;                // shortest slice of pn1 a CTA scans on the split path
constexpr int NN_MIN_CTAS = 3;                  // resident CTAs per SM: <= 85 registers, which the kernels fit unspilled
constexpr int NN_FILL_CTAS = 132 * NN_MIN_CTAS * 2;   // two waves on the H100's 132 SMs

constexpr unsigned long long NN_KEY_INIT = (unsigned long long)0x7f7fffffu << 32;   // (FLT_MAX bits, index 0)

__device__ __forceinline__ float nn_nan() { return __int_as_float(0x7fffffff); }

// the reference's squared distance, ref - que (nearest_neighborhood.cu:72-75 / :106-108)
template <int DIM>
__device__ __forceinline__ float nn_dist(const float4 r, float qx, float qy, float qz)
{
    const float dx = __fsub_rn(r.x, qx), dy = __fsub_rn(r.y, qy);
    float d = __fmaf_rn(dx, dx, __fmul_rn(dy, dy));
    if constexpr (DIM == 3) {
        const float dz = __fsub_rn(r.z, qz);
        d = __fmaf_rn(dz, dz, d);
    }
    return d;
}

// This thread's queries: slot q of CTA chunk qc is query qc * NN_QPB + q * NN_THREADS + tid (consecutive lanes, consecutive
// queries).  A slot past pn2 gets NaN coordinates, so it never takes a point, and is never written.
struct NnQueries {
    float x[NN_Q], y[NN_Q], z[NN_Q], best[NN_Q];
    int i[NN_Q], arg[NN_Q];
};

// The reference loop over the reference points [s0, s1) for this thread's queries; load(p) returns point p as a float4.
template <int DIM, bool EXCL, class Load>
__device__ __forceinline__ void nn_scan(float4 *tile, int s0, int s1, NnQueries &Q, Load load)
{
    for (int t0 = s0; t0 < s1; t0 += NN_TILE) {
        const int p = t0 + (int)threadIdx.x, cnt = min(NN_TILE, s1 - t0);
        __syncthreads();                                  // the previous tile has been read
        if (p < s1) tile[threadIdx.x] = load(p);
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < cnt; ++j) {
            const float4 r = tile[j];
#pragma unroll
            for (int q = 0; q < NN_Q; ++q) {
                const float d = nn_dist<DIM>(r, Q.x[q], Q.y[q], Q.z[q]);
                if (d < Q.best[q] && (!EXCL || t0 + j != Q.i[q])) { Q.best[q] = d; Q.arg[q] = t0 + j; }
            }
        }
    }
}

__device__ __forceinline__ unsigned long long nn_key(float d, int idx)
{
    return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
}

// blockIdx.x = ((problem * nsplit) + slice) * qchunks + query chunk
struct NnBlock { int prob, slice, qc; };
__device__ __forceinline__ NnBlock nn_block(int qchunks, int nsplit)
{
    int x = blockIdx.x;
    NnBlock b;
    b.qc = x % qchunks; x /= qchunks;
    b.slice = x % nsplit; b.prob = x / nsplit;
    return b;
}

struct NnArgs {
    const float *ref, *que;        // [b][pn1][dim], [b][pn2][dim]
    int *idxs;                     // [b][pn2]
    unsigned long long *keys;      // [b][pn2] (split path)
    int pn1, pn2;
    NnPlan plan;
};

template <int DIM, bool EXCL, bool SPLIT>
__global__ void __launch_bounds__(NN_THREADS, NN_MIN_CTAS)
nn_kernel(NnArgs a)
{
    __shared__ float4 tile[NN_TILE];
    const NnBlock blk = nn_block(a.plan.qchunks, a.plan.nsplit);
    const float *ref = a.ref + (size_t)blk.prob * a.pn1 * DIM, *que = a.que + (size_t)blk.prob * a.pn2 * DIM;
    NnQueries Q;
#pragma unroll
    for (int q = 0; q < NN_Q; ++q) {
        const int i = blk.qc * NN_QPB + q * NN_THREADS + (int)threadIdx.x;
        const bool ok = i < a.pn2;
        Q.i[q] = i;
        Q.x[q] = ok ? __ldg(que + (size_t)i * DIM) : nn_nan();
        Q.y[q] = ok ? __ldg(que + (size_t)i * DIM + 1) : nn_nan();
        Q.z[q] = ok && DIM == 3 ? __ldg(que + (size_t)i * DIM + 2) : 0.f;
        Q.best[q] = FLT_MAX; Q.arg[q] = 0;
    }
    const int s0 = blk.slice * a.plan.slice, s1 = min(a.pn1, s0 + a.plan.slice);
    nn_scan<DIM, EXCL>(tile, s0, s1, Q, [&](int p) {
        const float *r = ref + (size_t)p * DIM;
        return make_float4(__ldg(r), __ldg(r + 1), DIM == 3 ? __ldg(r + 2) : 0.f, 0.f);
    });
#pragma unroll
    for (int q = 0; q < NN_Q; ++q) {
        if (Q.i[q] >= a.pn2) continue;
        const size_t o = (size_t)blk.prob * a.pn2 + Q.i[q];
        if constexpr (SPLIT) {
            if (Q.best[q] < FLT_MAX) atomicMin(a.keys + o, nn_key(Q.best[q], Q.arg[q]));
        } else {
            a.idxs[o] = Q.arg[q];
        }
    }
}

__global__ void nn_key_init_kernel(unsigned long long *keys, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        keys[i] = NN_KEY_INIT;
}

__global__ void nn_key_index_kernel(const unsigned long long *keys, int *idxs, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        idxs[i] = (int)(unsigned)(keys[i] & 0xffffffffull);
}

int grid_stride_blocks(size_t n) { return (int)std::min<size_t>((n + 255) / 256, 132 * 16); }

// ---------------------------------------------------------------------------------------------------------------------
// ADD / ADD-S of n pose pairs on one model (Evaluator.add_metric, linemod/pvnet.py:68-82):
//   model_pred = model @ R_pred.T + t_pred, model_targets = model @ R_gt.T + t_gt            (fp64, :70-71)
//   ADD-S: idxs = nearest predicted point of every target point, on both clouds rounded to fp32 (what nn_utils hands
//          the reference kernel); dist_i = |model_pred[idxs[i]] - model_targets[i]|           (fp64, :73-75)
//   ADD:   dist_i = |model_pred[i] - model_targets[i]|                                         (:77)
//   mean_dist = mean_i dist_i                                                                  (fp64)
// The clouds never exist in memory: a CTA transforms the model points it needs (the same fp64 expression everywhere, so
// a point recomputed for its distance has the bits it had when it was rounded for the search).  Every CTA sums the
// distances of its NN_QPB target points into partial[pair][chunk]; add_mean_kernel adds those in a fixed order, so the
// result does not depend on scheduling.
// ---------------------------------------------------------------------------------------------------------------------
struct AddArgs {
    const double *model;           // [pn][3]
    const double *pose_pred, *pose_gt;   // [n][3][4]
    double *mean;                  // [n]
    unsigned long long *keys;      // [n][pn] (ADD-S, split path)
    double *partial;               // [n][qchunks]
    int pn;
    NnPlan plan;
};

// np.dot(model, pose[:, :3].T) + pose[:, 3] for one point, in the summation order of the dot product
__device__ __forceinline__ void pose_apply(const double *P, const double *m, double &x, double &y, double &z)
{
    const double m0 = __ldg(m), m1 = __ldg(m + 1), m2 = __ldg(m + 2);
    x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m0, P[0]), __dmul_rn(m1, P[1])), __dmul_rn(m2, P[2])), P[3]);
    y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m0, P[4]), __dmul_rn(m1, P[5])), __dmul_rn(m2, P[6])), P[7]);
    z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m0, P[8]), __dmul_rn(m1, P[9])), __dmul_rn(m2, P[10])), P[11]);
}

__device__ __forceinline__ void load_poses(const AddArgs &a, int pair, double (*s_pose)[12])
{
    if (threadIdx.x < 24) s_pose[threadIdx.x / 12][threadIdx.x % 12] =
        (threadIdx.x < 12 ? a.pose_pred : a.pose_gt)[(size_t)pair * 12 + threadIdx.x % 12];
    __syncthreads();
}

// |pred(model[src]) - gt(model[dst])| in fp64
__device__ __forceinline__ double add_point_dist(const AddArgs &a, double (*s_pose)[12], int src, int dst)
{
    double px, py, pz, gx, gy, gz;
    pose_apply(s_pose[0], a.model + (size_t)src * 3, px, py, pz);
    pose_apply(s_pose[1], a.model + (size_t)dst * 3, gx, gy, gz);
    const double dx = px - gx, dy = py - gy, dz = pz - gz;
    return sqrt(dx * dx + dy * dy + dz * dz);
}

// sum over the CTA in a fixed order -> partial[pair][qc]
__device__ __forceinline__ void add_block_sum(double v, double *out)
{
    __shared__ double s_w[NN_THREADS / 32];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < NN_THREADS / 32; ++w) s += s_w[w];
        *out = s;
    }
}

// ADD-S search: reference points = the predicted cloud, queries = the target cloud, both rounded to fp32
template <bool SPLIT>
__global__ void __launch_bounds__(NN_THREADS, NN_MIN_CTAS)
adds_kernel(AddArgs a)
{
    __shared__ float4 tile[NN_TILE];
    __shared__ double s_pose[2][12];
    const NnBlock blk = nn_block(a.plan.qchunks, a.plan.nsplit);
    load_poses(a, blk.prob, s_pose);
    NnQueries Q;
#pragma unroll
    for (int q = 0; q < NN_Q; ++q) {
        const int i = blk.qc * NN_QPB + q * NN_THREADS + (int)threadIdx.x;
        Q.i[q] = i; Q.best[q] = FLT_MAX; Q.arg[q] = 0;
        Q.x[q] = Q.y[q] = nn_nan(); Q.z[q] = 0.f;
        if (i < a.pn) {
            double x, y, z;
            pose_apply(s_pose[1], a.model + (size_t)i * 3, x, y, z);
            Q.x[q] = (float)x; Q.y[q] = (float)y; Q.z[q] = (float)z;
        }
    }
    const int s0 = blk.slice * a.plan.slice, s1 = min(a.pn, s0 + a.plan.slice);
    nn_scan<3, false>(tile, s0, s1, Q, [&](int p) {
        double x, y, z;
        pose_apply(s_pose[0], a.model + (size_t)p * 3, x, y, z);
        return make_float4((float)x, (float)y, (float)z, 0.f);
    });
    if constexpr (SPLIT) {
#pragma unroll
        for (int q = 0; q < NN_Q; ++q)
            if (Q.i[q] < a.pn && Q.best[q] < FLT_MAX)
                atomicMin(a.keys + (size_t)blk.prob * a.pn + Q.i[q], nn_key(Q.best[q], Q.arg[q]));
    } else {
        double s = 0.0;
#pragma unroll
        for (int q = 0; q < NN_Q; ++q)
            if (Q.i[q] < a.pn) s += add_point_dist(a, s_pose, Q.arg[q], Q.i[q]);
        add_block_sum(s, a.partial + (size_t)blk.prob * a.plan.qchunks + blk.qc);
    }
}

// the distances of ADD (FROM_KEYS = false: point i to point i) or of a split ADD-S search (the merged keys' indices)
template <bool FROM_KEYS>
__global__ void __launch_bounds__(NN_THREADS, NN_MIN_CTAS)
add_dist_kernel(AddArgs a)
{
    __shared__ double s_pose[2][12];
    const int pair = blockIdx.x / a.plan.qchunks, qc = blockIdx.x % a.plan.qchunks;
    load_poses(a, pair, s_pose);
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NN_Q; ++q) {
        const int i = qc * NN_QPB + q * NN_THREADS + (int)threadIdx.x;
        if (i >= a.pn) continue;
        const int src = FROM_KEYS ? (int)(unsigned)(a.keys[(size_t)pair * a.pn + i] & 0xffffffffull) : i;
        s += add_point_dist(a, s_pose, src, i);
    }
    add_block_sum(s, a.partial + (size_t)pair * a.plan.qchunks + qc);
}

// the sum of one pair's per-CTA partials in a fixed order (on every lane of the calling warp)
__device__ __forceinline__ double pair_partial_sum(const double *partial, int pair, int qchunks, int lane)
{
    double s = 0.0;
    for (int c = lane; c < qchunks; c += 32) s += partial[(size_t)pair * qchunks + c];
    return warp_sum(s);
}

// one warp per pair: mean = (sum of the partials, fixed order) / pn  (pn = 0 gives NaN, like np.mean of nothing)
__global__ void add_mean_kernel(const double *partial, double *mean, int n, int qchunks, int pn)
{
    const int pair = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= n) return;
    const double s = pair_partial_sum(partial, pair, qchunks, lane);
    if (lane == 0) mean[pair] = s / (double)pn;
}

// ---------------------------------------------------------------------------------------------------------------------
// projection_2d and cm_degree_5 of n pose pairs (Evaluator.projection_2d / cm_degree_5_metric, linemod/pvnet.py:59-66 and
// :84-94, on pvnet_pose_utils.project / cm_degree_5, pvnet_pose_utils.py:41-60), fp64:
//   uv = ((model @ R.T + t) @ K.T)[:, :2] / z                   both poses, every product and sum rounded on its own
//   proj2d = mean_i |uv_pred_i - uv_gt_i|                       z <= 0 gives what IEEE division gives (+-inf, NaN)
//   trans_cm = |t_pred - t_gt| * 100
//   trace = trace(R_pred @ R_gt.T); trace = trace if trace <= 3 else 3; trace = trace if trace >= -1 else -1
//   angle_deg = rad2deg(arccos((trace - 1) / 2))                a NaN trace becomes 3, i.e. 0 degrees
// proj_dist_kernel has add_dist_kernel's grid and per-CTA partial sums; pose_final_kernel adds them like add_mean_kernel
// and computes the two pose distances, so a pair's three outputs do not depend on the batch or on scheduling.
// ---------------------------------------------------------------------------------------------------------------------

// uv of one camera-frame point: (x, y, z) @ K.T in the dot product's summation order, then divided by its z
__device__ __forceinline__ void project_point(const double *K, double x, double y, double z, double &u, double &v)
{
    const double X = __dadd_rn(__dadd_rn(__dmul_rn(x, K[0]), __dmul_rn(y, K[1])), __dmul_rn(z, K[2]));
    const double Y = __dadd_rn(__dadd_rn(__dmul_rn(x, K[3]), __dmul_rn(y, K[4])), __dmul_rn(z, K[5]));
    const double Z = __dadd_rn(__dadd_rn(__dmul_rn(x, K[6]), __dmul_rn(y, K[7])), __dmul_rn(z, K[8]));
    u = __ddiv_rn(X, Z);
    v = __ddiv_rn(Y, Z);
}

// K of pair p at K + p * k_stride (0: shared)
__global__ void __launch_bounds__(NN_THREADS, NN_MIN_CTAS)
proj_dist_kernel(AddArgs a, const double *K, long long k_stride)
{
    __shared__ double s_pose[2][12];
    __shared__ double s_K[9];
    const int pair = blockIdx.x / a.plan.qchunks, qc = blockIdx.x % a.plan.qchunks;
    if (threadIdx.x < 9) s_K[threadIdx.x] = K[(size_t)pair * k_stride + threadIdx.x];
    load_poses(a, pair, s_pose);                          // its barrier also publishes s_K
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < NN_Q; ++q) {
        const int i = qc * NN_QPB + q * NN_THREADS + (int)threadIdx.x;
        if (i >= a.pn) continue;
        double px, py, pz, gx, gy, gz, pu, pv, gu, gv;
        pose_apply(s_pose[0], a.model + (size_t)i * 3, px, py, pz);
        pose_apply(s_pose[1], a.model + (size_t)i * 3, gx, gy, gz);
        project_point(s_K, px, py, pz, pu, pv);
        project_point(s_K, gx, gy, gz, gu, gv);
        const double du = __dsub_rn(pu, gu), dv = __dsub_rn(pv, gv);
        s += __dsqrt_rn(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)));
    }
    add_block_sum(s, a.partial + (size_t)pair * a.plan.qchunks + qc);
}

// one warp per pair: proj2d from the partials (pn = 0 gives NaN), trans_cm and angle_deg from the two poses
__global__ void pose_final_kernel(const double *partial, const double *pose_pred, const double *pose_gt, double *proj2d,
                                  double *trans_cm, double *angle_deg, int n, int qchunks, int pn)
{
    const int pair = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= n) return;
    const double s = pair_partial_sum(partial, pair, qchunks, lane);
    if (lane != 0) return;
    proj2d[pair] = s / (double)pn;
    const double *P = pose_pred + (size_t)pair * 12, *G = pose_gt + (size_t)pair * 12;
    const double d0 = __dsub_rn(P[3], G[3]), d1 = __dsub_rn(P[7], G[7]), d2 = __dsub_rn(P[11], G[11]);
    const double sq = __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
    trans_cm[pair] = __dmul_rn(__dsqrt_rn(sq), 100.0);
    double tr = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {                         // (R_pred @ R_gt.T)[r][r] = row r of R_pred . row r of R_gt
        const double *p = P + 4 * r, *g = G + 4 * r;
        const double drr = __dadd_rn(__dadd_rn(__dmul_rn(p[0], g[0]), __dmul_rn(p[1], g[1])), __dmul_rn(p[2], g[2]));
        tr = r == 0 ? drr : __dadd_rn(tr, drr);
    }
    tr = tr <= 3.0 ? tr : 3.0;                            // the reference's comparisons, which send NaN to 3
    tr = tr >= -1.0 ? tr : -1.0;
    angle_deg[pair] = __dmul_rn(acos(__ddiv_rn(__dsub_rn(tr, 1.0), 2.0)), 180.0 / 3.14159265358979323846);
}

} // namespace

NnPlan nn_plan(int b, int pn1, int pn2)
{
    NnPlan p;
    p.qchunks = (pn2 + NN_QPB - 1) / NN_QPB;
    p.nsplit = 1;
    p.slice = pn1;
    const long long ctas = (long long)b * p.qchunks;
    if (ctas > 0 && ctas < NN_FILL_CTAS && pn1 > NN_MIN_SLICE) {
        // whole waves: at most NN_FILL_CTAS CTAs, so the last wave is not a short tail
        const long long want = std::max(1ll, NN_FILL_CTAS / ctas), most = (pn1 + NN_MIN_SLICE - 1) / NN_MIN_SLICE;
        const int ns = (int)std::min(want, most);
        p.slice = (pn1 + ns - 1) / ns;
        p.nsplit = (pn1 + p.slice - 1) / p.slice;
    }
    return p;
}

size_t nn_workspace_bytes(int b, int pn1, int pn2)
{
    const NnPlan p = nn_plan(b, pn1, pn2);
    return p.nsplit > 1 ? (size_t)b * pn2 * sizeof(unsigned long long) : 0;
}

size_t add_metric_workspace_bytes(int n, int pn, int syn, size_t *partial_offset)
{
    const NnPlan p = nn_plan(n, pn, pn);
    const size_t keys = syn && p.nsplit > 1 ? ((size_t)n * pn * sizeof(unsigned long long) + 255) / 256 * 256 : 0;
    if (partial_offset) *partial_offset = keys;
    return keys + (size_t)n * p.qchunks * sizeof(double);
}

size_t pose_metrics_workspace_bytes(int n, int pn)
{
    return (size_t)n * ((pn + NN_QPB - 1) / NN_QPB) * sizeof(double);
}

cudaError_t launch_nearest_point(const float *ref, const float *que, int *idxs, int b, int pn1, int pn2, int dim,
                                 bool exclude_self, void *workspace, cudaStream_t st)
{
    if (b <= 0 || pn2 <= 0) return cudaSuccess;
    NnArgs a;
    a.ref = ref; a.que = que; a.idxs = idxs; a.pn1 = pn1; a.pn2 = pn2;
    a.plan = nn_plan(b, pn1, pn2);
    a.keys = static_cast<unsigned long long *>(workspace);
    const bool split = a.plan.nsplit > 1;
    const size_t nq = (size_t)b * pn2;
    const unsigned grid = (unsigned)((size_t)b * a.plan.nsplit * a.plan.qchunks);
    if (split) nn_key_init_kernel<<<grid_stride_blocks(nq), 256, 0, st>>>(a.keys, nq);
#define PVB_NN_LAUNCH(D, E)                                                                                               \
    (split ? nn_kernel<D, E, true><<<grid, NN_THREADS, 0, st>>>(a) : nn_kernel<D, E, false><<<grid, NN_THREADS, 0, st>>>(a))
    if (dim == 3) { if (exclude_self) PVB_NN_LAUNCH(3, true); else PVB_NN_LAUNCH(3, false); }
    else { if (exclude_self) PVB_NN_LAUNCH(2, true); else PVB_NN_LAUNCH(2, false); }
#undef PVB_NN_LAUNCH
    if (split) nn_key_index_kernel<<<grid_stride_blocks(nq), 256, 0, st>>>(a.keys, idxs, nq);
    return cudaGetLastError();
}

cudaError_t launch_add_metric(const double *model, const double *pose_pred, const double *pose_gt, double *mean_dist, int n,
                              int pn, bool syn, void *workspace, cudaStream_t st)
{
    if (n <= 0) return cudaSuccess;
    AddArgs a;
    a.model = model; a.pose_pred = pose_pred; a.pose_gt = pose_gt; a.mean = mean_dist; a.pn = pn;
    a.plan = nn_plan(n, pn, pn);
    size_t off;
    add_metric_workspace_bytes(n, pn, syn, &off);
    a.keys = static_cast<unsigned long long *>(workspace);
    a.partial = reinterpret_cast<double *>(static_cast<char *>(workspace) + off);
    const unsigned dist_grid = (unsigned)((size_t)n * a.plan.qchunks);
    if (pn > 0) {
        if (!syn) {
            add_dist_kernel<false><<<dist_grid, NN_THREADS, 0, st>>>(a);
        } else if (a.plan.nsplit == 1) {
            adds_kernel<false><<<dist_grid, NN_THREADS, 0, st>>>(a);
        } else {
            const size_t nq = (size_t)n * pn;
            nn_key_init_kernel<<<grid_stride_blocks(nq), 256, 0, st>>>(a.keys, nq);
            adds_kernel<true><<<(unsigned)(dist_grid * a.plan.nsplit), NN_THREADS, 0, st>>>(a);
            add_dist_kernel<true><<<dist_grid, NN_THREADS, 0, st>>>(a);
        }
    }
    add_mean_kernel<<<(n + 7) / 8, 256, 0, st>>>(a.partial, mean_dist, n, a.plan.qchunks, pn);
    return cudaGetLastError();
}

cudaError_t launch_pose_metrics(const double *model, const double *pose_pred, const double *pose_gt, const double *K,
                                long long k_stride, double *proj2d, double *trans_cm, double *angle_deg, int n, int pn,
                                void *workspace, cudaStream_t st)
{
    if (n <= 0) return cudaSuccess;
    AddArgs a = {};
    a.model = model; a.pose_pred = pose_pred; a.pose_gt = pose_gt; a.pn = pn;
    a.plan.qchunks = (pn + NN_QPB - 1) / NN_QPB; a.plan.nsplit = 1; a.plan.slice = pn;
    a.partial = static_cast<double *>(workspace);
    if (pn > 0) proj_dist_kernel<<<(unsigned)((size_t)n * a.plan.qchunks), NN_THREADS, 0, st>>>(a, K, k_stride);
    pose_final_kernel<<<(n + 7) / 8, 256, 0, st>>>(a.partial, pose_pred, pose_gt, proj2d, trans_cm, angle_deg, n,
                                                  a.plan.qchunks, pn);
    return cudaGetLastError();
}

} // namespace pvb
