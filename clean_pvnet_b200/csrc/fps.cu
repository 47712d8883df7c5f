// fps.cu -- batched farthest-point sampling, the device twin of clean-pvnet's `lib/csrc/fps`
// (src/farthest_point_sampling.cpp: farthest_point_sampling and farthest_point_sampling_init_center).
//
// The reference, built by its setup.py with `gcc -O2` and no -march (SSE arithmetic, no FMA contraction):
//   min_dist[i] = FLT_MAX (random start) or std::min(|p_i - centre|^2, FLT_MAX) (init_center, centre = (max + min) * 0.5f
//   over std::max / std::min per component from -FLT_MAX / FLT_MAX); |d|^2 = ((dx*dx) + (dy*dy)) + (dz*dz), each
//   difference rounded first.  cur = the start (random) or the argmax below (init_center); then for i in 0..sn-1:
//   mask[cur] = true; idxs[i] = cur; if (i < sn-1) { for unselected j: dist < min_dist[j] -> take; cur = argmax }.
//   argmax (find_max_dist_idx): max_d = 0.f, max_idx = 0, scan in index order over unselected j with `min_dist[j] > max_d`.
// Consequences the kernel keeps: the smallest index of the largest value wins; a NaN min_dist never wins (and, once NaN,
// is never updated); when no unselected value is > 0 the answer is index 0, selected or not, so sn > pn repeats index 0.
//
// Layout: one thread-block cluster of C CTAs per cloud, C in {1,2,4,8} for the whole launch: the smallest that holds the
// largest cloud on chip, halved while the clusters would not all be resident at once (pvb_farthest_point_sampling).  CTA `rank` keeps points [rank * FPS_CTA_PTS, (rank+1) * FPS_CTA_PTS) in registers, FPS_PTS per
// thread (point rank * FPS_CTA_PTS + j * FPS_THREADS + t in slot j of thread t), with their min_dist.  Points from
// cap = C * FPS_CTA_PTS on are streamed every iteration from the cloud and a min_dist array in the workspace, cap + g +
// k * C * FPS_THREADS by cluster thread g.  A selected point's min_dist becomes -1: no distance is < -1 and -1 is not
// > 0, so it is neither updated nor chosen again, which is what the reference's mask does.
//
// Each iteration: every thread updates its points and keeps its first largest min_dist (strict `>` in index order, from
// 0); candidates (value, index, coordinates) then meet through warp shuffles, a shared-memory slot per warp and one slot
// per CTA, double-buffered by iteration parity.  After one barrier.cluster every warp reads the C CTA slots through
// distributed shared memory and computes the same winner.  Candidate values are never NaN (a NaN never passes `> best`),
// so `b.v > a.v || (b.v == a.v && b.i < a.i)` is a total order and any reduction tree gives the sequential scan's answer.
// The slot of parity p is rewritten two iterations later, after the next barrier.cluster, which every CTA reaches only
// after it has read that slot: one cluster barrier per iteration suffices.
#include <cooperative_groups.h>
#include <algorithm>
#include <atomic>
#include <cfloat>
#include <climits>
#include <vector>
#include "api.h"

namespace cg = cooperative_groups;

namespace pvb {

namespace {

constexpr int FPS_THREADS = 512;
constexpr int FPS_PTS = 16;                                    // register-resident points per thread
constexpr int FPS_CTA_PTS = FPS_THREADS * FPS_PTS;             // 8192 points on chip per CTA
constexpr int FPS_MAX_CLUSTER = 8;                             // the portable cluster size
constexpr int FPS_WARPS = FPS_THREADS / 32;
constexpr unsigned FULL = 0xffffffffu;

struct FpsCand { float v; int i; float x, y, z; };

__device__ __forceinline__ FpsCand fps_none() { return FpsCand{0.f, INT_MAX, 0.f, 0.f, 0.f}; }

// b replaces a: a larger distance, or the same distance at a smaller index
__device__ __forceinline__ bool fps_better(const FpsCand &b, const FpsCand &a)
{
    return b.v > a.v || (b.v == a.v && b.i < a.i);
}

__device__ __forceinline__ FpsCand fps_warp_max(FpsCand c)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        FpsCand d;
        d.v = __shfl_xor_sync(FULL, c.v, o);
        d.i = __shfl_xor_sync(FULL, c.i, o);
        d.x = __shfl_xor_sync(FULL, c.x, o);
        d.y = __shfl_xor_sync(FULL, c.y, o);
        d.z = __shfl_xor_sync(FULL, c.z, o);
        if (fps_better(d, c)) c = d;
    }
    return c;
}

// the reference's Vec3::squared_norm of (p - q), without contraction
__device__ __forceinline__ float fps_dist(float x, float y, float z, float qx, float qy, float qz)
{
    const float dx = __fsub_rn(x, qx), dy = __fsub_rn(y, qy), dz = __fsub_rn(z, qz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// std::max(acc, v) / std::min(acc, v) as max_vec3 / min_vec3 call them: a NaN v never enters
__device__ __forceinline__ float ref_max(float acc, float v) { return acc < v ? v : acc; }
__device__ __forceinline__ float ref_min(float acc, float v) { return v < acc ? v : acc; }

struct FpsShared {
    FpsCand warp_slot[FPS_WARPS];
    FpsCand cta_slot[2];
    float warp_box[FPS_WARPS][6];
    float cta_box[6];
};

// the cluster's winner of the threads' candidates; `parity` picks the CTA slot.  Index INT_MAX (nothing > 0) is index 0.
__device__ FpsCand fps_reduce(FpsCand c, FpsShared &sh, int parity, const cg::cluster_group &cluster, int nranks,
                              float p0x, float p0y, float p0z)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    c = fps_warp_max(c);
    if (lane == 0) sh.warp_slot[warp] = c;
    __syncthreads();
    if (warp == 0) {
        FpsCand d = lane < FPS_WARPS ? sh.warp_slot[lane] : fps_none();
        d = fps_warp_max(d);
        if (lane == 0) sh.cta_slot[parity] = d;
    }
    cluster.sync();
    FpsCand r = fps_none();
    if (lane < nranks) r = *cluster.map_shared_rank(&sh.cta_slot[parity], lane);
    r = fps_warp_max(r);
    if (r.i == INT_MAX) r = FpsCand{0.f, 0, p0x, p0y, p0z};
    return r;
}

// the cluster's bounding box (max xyz, min xyz) under the reference's max / min predicates
__device__ void fps_box(float box[6], FpsShared &sh, const cg::cluster_group &cluster, int nranks)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const float v = __shfl_xor_sync(FULL, box[k], o);
            box[k] = k < 3 ? ref_max(box[k], v) : ref_min(box[k], v);
        }
    if (lane == 0)
        for (int k = 0; k < 6; ++k) sh.warp_box[warp][k] = box[k];
    __syncthreads();
    if (warp == 0) {
        float b[6] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX};
        if (lane < FPS_WARPS)
            for (int k = 0; k < 6; ++k) b[k] = sh.warp_box[lane][k];
#pragma unroll
        for (int o = 16; o; o >>= 1)
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const float v = __shfl_xor_sync(FULL, b[k], o);
                b[k] = k < 3 ? ref_max(b[k], v) : ref_min(b[k], v);
            }
        if (lane == 0)
            for (int k = 0; k < 6; ++k) sh.cta_box[k] = b[k];
    }
    cluster.sync();
    float b[6] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX};
    if (lane < nranks) {
        const float *remote = cluster.map_shared_rank(sh.cta_box, lane);
        for (int k = 0; k < 6; ++k) b[k] = remote[k];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const float v = __shfl_xor_sync(FULL, b[k], o);
            b[k] = k < 3 ? ref_max(b[k], v) : ref_min(b[k], v);
        }
    for (int k = 0; k < 6; ++k) box[k] = b[k];
}

// One cluster per cloud blockIdx.x / C.  table: counts [B], starts [B].  spill: min_dist of points from
// FPS_CTA_PTS on, spill_stride floats per cloud.
__global__ void __launch_bounds__(FPS_THREADS, 1)
fps_kernel(const float *__restrict__ pts, const int *__restrict__ table, int B, int n, int sn, int init_center,
           int *__restrict__ idxs, float *__restrict__ spill, long long spill_stride)
{
    __shared__ FpsShared sh;
    const cg::cluster_group cluster = cg::this_cluster();
    const int nranks = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const int b = blockIdx.x / nranks;
    const int t = threadIdx.x;
    const int count = table[b];
    const float *p = pts + (long long)b * n * 3;
    float *ov = spill + (long long)b * spill_stride - FPS_CTA_PTS;   // ov[i] for i >= cap >= FPS_CTA_PTS
    const int base = rank * FPS_CTA_PTS;
    const int cap = nranks * FPS_CTA_PTS;
    const int g0 = cap + rank * FPS_THREADS + t, gstride = nranks * FPS_THREADS;

    float x[FPS_PTS], y[FPS_PTS], z[FPS_PTS], md[FPS_PTS];
#pragma unroll
    for (int j = 0; j < FPS_PTS; ++j) {
        const int i = base + j * FPS_THREADS + t;
        const bool in = i < count;
        x[j] = in ? p[3ll * i] : 0.f;
        y[j] = in ? p[3ll * i + 1] : 0.f;
        z[j] = in ? p[3ll * i + 2] : 0.f;
        md[j] = in ? FLT_MAX : -1.f;                  // padding behaves like a selected point
    }
    const float p0x = p[0], p0y = p[1], p0z = p[2];

    int parity = 0;
    FpsCand w;                                        // the point selected last
    if (init_center) {
        float box[6] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX};
#pragma unroll
        for (int j = 0; j < FPS_PTS; ++j)
            if (base + j * FPS_THREADS + t < count) {
                box[0] = ref_max(box[0], x[j]); box[1] = ref_max(box[1], y[j]); box[2] = ref_max(box[2], z[j]);
                box[3] = ref_min(box[3], x[j]); box[4] = ref_min(box[4], y[j]); box[5] = ref_min(box[5], z[j]);
            }
        for (int i = g0; i < count; i += gstride) {
            const float px = p[3ll * i], py = p[3ll * i + 1], pz = p[3ll * i + 2];
            box[0] = ref_max(box[0], px); box[1] = ref_max(box[1], py); box[2] = ref_max(box[2], pz);
            box[3] = ref_min(box[3], px); box[4] = ref_min(box[4], py); box[5] = ref_min(box[5], pz);
        }
        fps_box(box, sh, cluster, nranks);
        const float cx = __fmul_rn(__fadd_rn(box[0], box[3]), 0.5f), cy = __fmul_rn(__fadd_rn(box[1], box[4]), 0.5f),
                    cz = __fmul_rn(__fadd_rn(box[2], box[5]), 0.5f);
#pragma unroll
        for (int j = 0; j < FPS_PTS; ++j) {
            const float d = fps_dist(x[j], y[j], z[j], cx, cy, cz);
            if (md[j] >= 0.f) md[j] = FLT_MAX < d ? FLT_MAX : d;   // std::min(d, FLT_MAX); NaN stays NaN
        }
        for (int i = g0; i < count; i += gstride) {
            const float d = fps_dist(p[3ll * i], p[3ll * i + 1], p[3ll * i + 2], cx, cy, cz);
            ov[i] = FLT_MAX < d ? FLT_MAX : d;
        }
        // the first pick is the argmax over the initial min_dist: a selection of "no point" at NaN updates nothing
        w = FpsCand{0.f, -1, __int_as_float(0x7fffffff), __int_as_float(0x7fffffff), __int_as_float(0x7fffffff)};
    } else {
        for (int i = g0; i < count; i += gstride) ov[i] = FLT_MAX;
        const int s = table[B + b];
        w = FpsCand{0.f, s, p[3ll * s], p[3ll * s + 1], p[3ll * s + 2]};
    }

    for (int it = init_center ? -1 : 0;; ++it) {
        if (it >= 0) {
            if (rank == 0 && t == 0) idxs[(long long)b * sn + it] = w.i;
            if (it == sn - 1) break;
        }
        FpsCand c = fps_none();
#pragma unroll
        for (int j = 0; j < FPS_PTS; ++j) {
            const int i = base + j * FPS_THREADS + t;
            const float d = fps_dist(x[j], y[j], z[j], w.x, w.y, w.z);
            if (i == w.i) md[j] = -1.f;
            else if (d < md[j]) md[j] = d;
            if (md[j] > c.v) c = FpsCand{md[j], i, x[j], y[j], z[j]};
        }
#pragma unroll 2
        for (int i = g0; i < count; i += gstride) {
            const float px = p[3ll * i], py = p[3ll * i + 1], pz = p[3ll * i + 2];
            float m = ov[i];
            const float d = fps_dist(px, py, pz, w.x, w.y, w.z);
            if (i == w.i) { m = -1.f; ov[i] = m; }
            else if (d < m) { m = d; ov[i] = m; }
            if (m > c.v) c = FpsCand{m, i, px, py, pz};
        }
        w = fps_reduce(c, sh, parity, cluster, nranks, p0x, p0y, p0z);
        parity ^= 1;
    }
    cluster.sync();                                   // no CTA leaves while another may still read its slots
}

std::atomic<int> g_cluster_cache[64][FPS_MAX_CLUSTER + 1];   // max active clusters per (device, size); 0: not yet asked

size_t fps_table_bytes(int b) { return ((size_t)2 * b * sizeof(int) + 255) / 256 * 256; }

// clusters of `size` CTAs that fit on the device at once
int fps_max_active_clusters(int dev, int size)
{
    std::atomic<int> &slot = g_cluster_cache[dev & 63][size];
    if (int known = slot.load(std::memory_order_relaxed)) return known;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)size);
    cfg.blockDim = dim3(FPS_THREADS);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)size;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, fps_kernel, &cfg) != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    n = std::max(n, 1);
    slot.store(n, std::memory_order_relaxed);
    return n;
}

} // namespace

// the counts [b] and starts [b] (unused under init_center) tables, then the min_dist of every cloud's points past the first
// CTA's on-chip slice
// External linkage on purpose: nvcc names this file's anonymous namespace, and so its kernels, after the first
// externally visible definition in the file.
size_t fps_workspace_bytes(int b, int n)
{
    return fps_table_bytes(b) + (size_t)b * (size_t)std::max(0, n - FPS_CTA_PTS) * sizeof(float);
}

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API size_t pvb_fps_workspace_bytes(int32_t b, int32_t n)
{
    if (b <= 0 || n <= 0) return 0;
    return fps_workspace_bytes(b, n);
}

PVB_API int pvb_farthest_point_sampling(const float *pts, const int32_t *counts, const int32_t *starts, int32_t init_center,
                                        int32_t *idxs, int32_t b, int32_t n, int32_t sn, void *workspace,
                                        size_t workspace_bytes, pvb_stream_t stream)
{
    if (b < 0 || n < 0 || sn < 0) return fail(PVB_ERR_INVALID, "negative size (b=%d n=%d sn=%d)", b, n, sn);
    if (b > 0x7fffffff / 8) return fail(PVB_ERR_INVALID, "b too large (got %d)", b);
    if (b == 0 || sn == 0) return PVB_OK;
    if (!pts || !idxs || !counts || (!init_center && !starts)) return fail(PVB_ERR_INVALID, "NULL pointer");
    for (int32_t i = 0; i < b; ++i) {
        if (counts[i] < 1 || counts[i] > n)
            return fail(PVB_ERR_INVALID, "cloud %d has %d points (must be in [1, %d])", i, counts[i], n);
        if (!init_center && (starts[i] < 0 || starts[i] >= counts[i]))
            return fail(PVB_ERR_INVALID, "cloud %d starts at %d (must be in [0, %d))", i, starts[i], counts[i]);
    }
    if (int rc = check_workspace(fps_workspace_bytes(b, n), workspace, workspace_bytes)) return rc;
    const int init = init_center != 0;
    std::vector<int> table((size_t)2 * b, 0);
    int max_count = 0;
    for (int i = 0; i < b; ++i) {
        table[i] = counts[i];
        table[(size_t)b + i] = init ? 0 : starts[i];
        max_count = std::max(max_count, counts[i]);
    }
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_fail(e, "farthest point sampling kernel");
    int size = 1;
    while (size < FPS_MAX_CLUSTER && (long long)size * FPS_CTA_PTS < max_count) size *= 2;
    // a narrower cluster that streams more of each cloud, rather than a second wave of clusters
    while (size > 1 && b > fps_max_active_clusters(dev, size)) size /= 2;

    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    int *d_table = static_cast<int *>(workspace);
    float *spill = reinterpret_cast<float *>(static_cast<char *>(workspace) + fps_table_bytes(b));
    // the table is pageable host memory: the copy stages it before returning, so it may go out of scope at once
    e = cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)((long long)b * size));
        cfg.blockDim = dim3(FPS_THREADS);
        cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)size;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        e = cudaLaunchKernelEx(&cfg, fps_kernel, pts, (const int *)d_table, b, n, sn, init, idxs, spill,
                               (long long)std::max(0, n - FPS_CTA_PTS));
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "farthest point sampling kernel");
}

} // extern "C"
