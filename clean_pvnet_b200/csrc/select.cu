// select.cu -- foreground selection: mask -> bitmap -> (thinning) -> ordered compaction + gather.
//
// Replaces, for the whole batch and without a host sync, the per-image torch ops of
//   ransac_voting_gpu.py:125-143 (v3)   cur_mask=.byte(); sum; uniform_ thinning; nonzero; masked_select
//   ransac_voting_gpu.py:207-227 (dist) cur_mask=(mask==1); ...
//
// HBM layout produced (see pvb_layout in include/pvnet_vote_b200.h):
//   bits    uint32[B][nwords]      1 bit per pixel, row-major
//   blocktot uint32[B][nblocks]    selected pixels per 128-word block | READY bit -> order-preserving compaction by
//                                  decoupled look-back (thin_gather_kernel)
//   xy      float2[B][cap]         (x,y) of the t-th selected pixel (torch.nonzero order, :140-141)
//   dirs    float2[B][K][cap]      vertex vectors of the selected pixels, keypoint-major so that a
//                                  (image,keypoint) vote CTA streams one contiguous float2 array
//
// Both kernels are HBM/latency bound: the mask is read exactly once (mask_bits), the bitmap (1/256 of an int64 mask)
// is what the second pass touches, and the vertex field is read only at selected pixels.
//
// The evaluator's mask_iou (mask_iou_kernel, at the end) streams a predicted and a ground-truth mask with the same loads.
#include <atomic>
#include "api.h"
#include "common.cuh"
#include "kernels.h"

namespace pvb {

template <typename T>
__device__ __forceinline__ uint32_t mask_byte(T v) { return (uint32_t)(uint8_t)v; }
template <>
__device__ __forceinline__ uint32_t mask_byte<float>(float v) { return (uint32_t)(uint8_t)(long long)v; }
template <>
__device__ __forceinline__ uint32_t mask_byte<double>(double v) { return (uint32_t)(uint8_t)(long long)v; }

constexpr int MB_WARPS = 8;
constexpr int MB_UNROLL = 8;
constexpr int MB_WORDS = 32;     // bitmap words (of 32 pixels) per warp: 1024 pixels, lane i keeps word i

// 16-byte streaming load (ld.global.cs: the mask is read exactly once -- evict-first in L2, so it does not push the
// compacted dirs/xy arrays, which the vote kernel re-reads from L2, out to DRAM).  volatile: the compiler must not
// narrow it to the 32-bit pieces the predicate happens to need (it did: 2x the LSU instructions).
__device__ __forceinline__ uint4 ld_stream16(const void *p)
{
    uint4 v;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// One warp converts 1024 pixels into 32 bitmap words; lane i keeps word i so the words leave as one coalesced store.
//   VEC path (contiguous image, 16-byte aligned, all 1024 pixels in range): every lane loads 16 BYTES per instruction
//   (E = 16/sizeof(T) consecutive pixels: 2 for the int64 mask torch.argmax produces), 8 loads in flight per lane
//   (4 KB per warp), two rounds for int64; the E-bit pieces of the 32/E lanes that share a bitmap word are OR-reduced
//   with one REDUX per load instruction.  The grid is 38 x B CTAs of 8 warps: half a wave at cfg-2, so every CTA is
//   resident from the start (the 512-pixel version needed 1.01 waves: a 16-CTA tail cost a quarter of the kernel).
//   Scalar path (strided masks, image tail): one pixel per lane and load, MB_UNROLL loads in flight, ballots.
template <typename T, int MODE>
__device__ __forceinline__ void mask_pred(T v, bool &sel, uint32_t &val)
{
    if (MODE == PVB_SELECT_BYTE) { val = mask_byte<T>(v); sel = val != 0; }
    else { sel = (v == (T)1); val = sel; }
}

template <typename T, int MODE, bool CONTIG>
__global__ void __launch_bounds__(MB_WARPS * 32)
mask_bits_kernel(const T *__restrict__ mask, long long sb, long long sy, long long sx, int H, int W,
                 int nwords, uint32_t *__restrict__ bits, unsigned long long *__restrict__ fgsum,
                 int *__restrict__ nz, int vec_ok)
{
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w0 = (blockIdx.x * MB_WARPS + warp) * MB_WORDS;
    if (w0 >= nwords) return;
    const int HW = H * W;
    const T *mb = mask + (long long)b * sb;
    const bool full = CONTIG && ((w0 + MB_WORDS) * 32 <= HW);
    uint32_t myword = 0, sum = 0;
    if (full && vec_ok) {
        constexpr int E = 16 / (int)sizeof(T);            // pixels per lane and load
        constexpr int NL = MB_WORDS / E;                  // load instructions per warp (E words each)
        constexpr int NR = NL < 8 ? NL : 8;               // loads in flight per lane and round (8 x 16 B = 4 KB per warp)
        constexpr int LPW = 32 / E;                       // lanes that share one bitmap word
        union V { uint4 u; T t[E]; };
        const uint4 *q = reinterpret_cast<const uint4 *>(mb + (size_t)w0 * 32) + lane;
        const int grp = lane / LPW;                       // word (within one load) this lane contributes to
        const uint32_t gmask = (LPW == 32 ? 0xffffffffu : ((1u << LPW) - 1u)) << (grp * LPW);
#pragma unroll
        for (int r0 = 0; r0 < NL; r0 += NR) {
            V v[NR];
#pragma unroll
            for (int u = 0; u < NR; ++u) v[u].u = ld_stream16(q + (r0 + u) * 32);
#pragma unroll
            for (int u = 0; u < NR; ++u) {
                const int g = r0 + u;                     // this load covers words [g*E, (g+1)*E)
                uint32_t lb = 0;
#pragma unroll
                for (int j = 0; j < E; ++j) {
                    bool sel; uint32_t val;
                    mask_pred<T, MODE>(v[u].t[j], sel, val);
                    lb |= (sel ? 1u : 0u) << j;
                    sum += val;
                }
                const uint32_t word = __reduce_or_sync(gmask, lb << ((lane % LPW) * E));
                // word (g*E + k) was assembled by lane group k; lane (g*E + k) fetches it from that group's first lane
                const uint32_t mine = __shfl_sync(0xffffffffu, word, ((lane - g * E) & (E - 1)) * LPW);
                if (lane >= g * E && lane < (g + 1) * E) myword = mine;
            }
        }
    } else {
        for (int i0 = 0; i0 < MB_WORDS; i0 += MB_UNROLL) {
            T v[MB_UNROLL];
            if (full) {
                const T *q = mb + (size_t)(w0 + i0) * 32 + lane;
#pragma unroll
                for (int u = 0; u < MB_UNROLL; ++u) v[u] = __ldg(q + u * 32);
            } else {
#pragma unroll
                for (int u = 0; u < MB_UNROLL; ++u) {
                    const int p = (w0 + i0 + u) * 32 + lane;
                    v[u] = (T)0;
                    if (p < HW) {
                        long long off = p;
                        if (!CONTIG) { const int y = p / W; off = (long long)y * sy + (long long)(p - y * W) * sx; }
                        v[u] = __ldg(mb + off);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < MB_UNROLL; ++u) {
                uint32_t val;
                bool sel;
                mask_pred<T, MODE>(v[u], sel, val);
                const uint32_t word = __ballot_sync(0xffffffffu, sel);
                if (lane == i0 + u) myword = word;
                sum += val;
            }
        }
    }
    if (lane < MB_WORDS && w0 + lane < nwords) bits[(size_t)b * nwords + w0 + lane] = myword;
    const int s = warp_sum((int)sum);
    const int c = warp_sum(__popc(myword));
    if (lane == 0) {
        atomicAdd(fgsum + b, (unsigned long long)(unsigned)s);
        atomicAdd(nz + b, c);
    }
}

// Fused front end of decode_keypoint (lib/networks/pvnet/resnet18.py:69): the mask is torch.argmax(seg, 1) -- first
// maximal class, NaN counts as maximal like torch -- computed on the fly from the fp32 logits [B,C,H,W]; optionally
// also written out as the int64 mask decode_keypoint returns.  Otherwise identical to mask_bits_kernel.
template <int MODE>
__global__ void __launch_bounds__(MB_WARPS * 32)
seg_bits_kernel(const float *__restrict__ seg, long long sb, long long sc, long long sy, long long sx, int C, int H, int W,
                int nwords, long long *__restrict__ mask_out, uint32_t *__restrict__ bits,
                unsigned long long *__restrict__ fgsum, int *__restrict__ nz)
{
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w0 = (blockIdx.x * MB_WARPS + warp) * MB_WORDS;
    if (w0 >= nwords) return;
    const int HW = H * W;
    const float *sbp = seg + (long long)b * sb;
    const bool contig = (sx == 1 && sy == W);
    uint32_t myword = 0, sum = 0;
    for (int i0 = 0; i0 < MB_WORDS; i0 += MB_UNROLL) {
        long long off[MB_UNROLL];
        float best[MB_UNROLL];
        int idx[MB_UNROLL];
        bool inb[MB_UNROLL];
#pragma unroll
        for (int u = 0; u < MB_UNROLL; ++u) {           // MB_UNROLL class-0 loads in flight per lane
            const int p = (w0 + i0 + u) * 32 + lane;
            inb[u] = p < HW;
            off[u] = p;
            if (!contig && inb[u]) { const int y = p / W; off[u] = (long long)y * sy + (long long)(p - y * W) * sx; }
            best[u] = inb[u] ? __ldg(sbp + off[u]) : 0.f;
            idx[u] = 0;
        }
        for (int c = 1; c < C; ++c) {
            float v[MB_UNROLL];
#pragma unroll
            for (int u = 0; u < MB_UNROLL; ++u) v[u] = inb[u] ? __ldg(sbp + off[u] + (long long)c * sc) : 0.f;
#pragma unroll
            for (int u = 0; u < MB_UNROLL; ++u)
                if (v[u] > best[u] || (v[u] != v[u] && best[u] == best[u])) { best[u] = v[u]; idx[u] = c; }
        }
#pragma unroll
        for (int u = 0; u < MB_UNROLL; ++u) {
            const int p = (w0 + i0 + u) * 32 + lane;
            if (mask_out && inb[u]) mask_out[(size_t)b * HW + p] = idx[u];
            bool sel;
            uint32_t val;
            if (MODE == PVB_SELECT_BYTE) { val = (uint32_t)(uint8_t)idx[u]; sel = val != 0; }
            else { sel = (idx[u] == 1); val = sel; }
            if (!inb[u]) { sel = false; val = 0; }
            const uint32_t word = __ballot_sync(0xffffffffu, sel);
            if (lane == i0 + u) myword = word;
            sum += val;
        }
    }
    if (lane < MB_WORDS && w0 + lane < nwords) bits[(size_t)b * nwords + w0 + lane] = myword;
    const int s = warp_sum((int)sum);
    const int c = warp_sum(__popc(myword));
    if (lane == 0) {
        atomicAdd(fgsum + b, (unsigned long long)(unsigned)s);
        atomicAdd(nz + b, c);
    }
}

// thin_gather_kernel -- thinning decision, ordered compaction and vertex gather of one 128-word block (4096 pixels) in ONE
// launch (round 1/2a: thin_scan_kernel + gather_kernel with wordoff[] in between).
//   * decides skip / thinning for its image (ransac_voting_gpu.py:129-138) and applies the Bernoulli thinning to its words;
//   * in-block exclusive popcount scan -> position of every selected pixel inside the block;
//   * the offset of the block inside the image (torch.nonzero order needs the totals of all preceding blocks) comes from a
//     decoupled look-back: every CTA publishes  total | READY  in blocktot[b][blk] as soon as it has scanned its block and
//     then sums its predecessors' entries, polling the ones that are not there yet.  Block ids are drawn from a per-image
//     ticket counter in arrival order, so a CTA's predecessors have always started (no reliance on the dispatch order);
//     the poll is bounded and reports PVB_ERR_CUDA through the status word instead of hanging;
//   * the block's selected pixels are listed in shared memory and the CTA walks that dense list: one lane per selected
//     pixel, K independent loads in flight per lane, each store instruction of a warp writes 32 consecutive t of one
//     keypoint plane of dirs[] (256 B); pinned HOST input is read row-wise (see set_gather_tuning below).
constexpr int TS_THREADS = 128;
constexpr int GA_THREADS = TS_THREADS;
constexpr unsigned LB_READY = 0x80000000u;          // blocktot entry: bit 31 = published, bits 0..30 = selected pixels

__device__ __forceinline__ unsigned ld_volatile_u32(const unsigned *p)
{
    unsigned v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(GA_THREADS)
thin_gather_kernel(uint32_t *__restrict__ bits, unsigned *__restrict__ blocktot, int *__restrict__ ticket,
                   const unsigned long long *__restrict__ fgsum, int *__restrict__ tn, int *__restrict__ state,
                   int *__restrict__ status, const float *__restrict__ selection, const float *__restrict__ vertex,
                   long long sB, long long sH, long long sW, long long sK, long long sC,
                   float2 *__restrict__ xy, float2 *__restrict__ dirs, int nwords, int nblocks, int K, int cap, int W, int HW,
                   int min_num, int max_num, uint2 key, uint32_t tag, int img_base, int b0, int rowwise)
{
    __shared__ unsigned short s_list[TS_THREADS * 32];   // pixel index inside the block (12 bits)
    __shared__ int s_base, s_blk;
    __shared__ int warp_tot[TS_THREADS / 32];
    const int b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned long long fg = fgsum[b];
    if (fg < (unsigned long long)(min_num < 0 ? 0 : min_num)) {   // :129  (uniform per image): nothing to compact
        if (tid == 0 && blockIdx.x == 0) state[b] = 1;
        return;
    }
    if (tid == 0) s_blk = atomicAdd(ticket + b, 1);             // block id in arrival order (see above)
    __syncthreads();
    const int blk = s_blk;
    const bool thin = fg > (unsigned long long)(max_num < 0 ? 0 : max_num);   // :135
    // max_num / fg.float() is Tensor.__rtruediv__ = fg.float().reciprocal() * max_num: two roundings, as the reference
    const float ratio = thin ? __fmul_rn(__fdiv_rn(1.f, (float)fg), (float)max_num) : 0.f;
    const int w = blk * TS_THREADS + tid;
    uint32_t word = (w < nwords) ? bits[(size_t)b * nwords + w] : 0u;
    if (thin && word) {
        uint32_t keep = 0;
        if (selection) {
            const float *sp = selection + (size_t)b * HW + (size_t)w * 32;
            uint32_t m = word;
            while (m) {
                const int j = __ffs(m) - 1;
                m &= m - 1;
                if (__ldg(sp + j) < ratio) keep |= 1u << j;
            }
        } else {
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const uint32_t nib = (word >> (4 * g)) & 0xfu;
                if (!nib) continue;
                const uint4 r = philox4x32_10(make_uint4((uint32_t)w * 8u + g, 0u, (uint32_t)(img_base + b), tag), key);
                uint32_t kb = 0;
                kb |= (u32_to_unit(r.x) < ratio) ? 1u : 0u;
                kb |= (u32_to_unit(r.y) < ratio) ? 2u : 0u;
                kb |= (u32_to_unit(r.z) < ratio) ? 4u : 0u;
                kb |= (u32_to_unit(r.w) < ratio) ? 8u : 0u;
                keep |= (kb & nib) << (4 * g);
            }
        }
        word = keep;
        bits[(size_t)b * nwords + w] = word;                   // the thinned bitmap stays inspectable (debug / tooling)
    }
    const int c = __popc(word);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int warp_excl = 0, total = 0;
#pragma unroll
    for (int i = 0; i < TS_THREADS / 32; ++i) {
        const int t = warp_tot[i];
        if (i < warp) warp_excl += t;
        total += t;
    }
    if (tid == 0) {
        atomicExch(blocktot + (size_t)b * nblocks + blk, (unsigned)total | LB_READY);   // publish first, then look back
        if (total) atomicAdd(tn + b, total);
    }
    if (total == 0) return;
    if (warp == 0) {   // offset of this block = totals of the preceding blocks (decoupled look-back, bounded poll)
        int base = 0;
        bool ok = true;
        for (int i = lane; i < blk; i += 32) {
            const unsigned *p = blocktot + (size_t)b * nblocks + i;
            unsigned v = ld_volatile_u32(p);
            for (int spin = 0; !(v & LB_READY); ++spin) {
                if (spin > (1 << 22)) { ok = false; break; }
                __nanosleep(20);
                v = ld_volatile_u32(p);
            }
            base += (int)(v & ~LB_READY);
        }
        base = warp_sum(base);
        if (!__all_sync(0xffffffffu, ok) && lane == 0) atomicCAS(status, 0, PVB_ERR_CUDA);
        if (lane == 0) s_base = base;
    }
    {
        int o = warp_excl + incl - c;
        uint32_t m = word;
        while (m) {
            const int j = __ffs(m) - 1;
            m &= m - 1;
            s_list[o++] = (unsigned short)(tid * 32 + j);
        }
    }
    __syncthreads();
    const int base = s_base;
    if (tid == 0 && base + total > cap) {
        // more pixels selected than the workspace holds: report; the walks below stop at cap and every consumer clamps tn
        atomicCAS(status, 0, PVB_ERR_CAPACITY);
        status[1] = b0 + b;
    }
    const bool vec = (sC == 1 && (sK & 1) == 0 && (sW & 1) == 0 && (sH & 1) == 0 && (sB & 1) == 0 &&
                      (reinterpret_cast<uintptr_t>(vertex) & 7u) == 0);
    const float *vimg = vertex + (long long)b * sB;
    if (rowwise && vec && sK == 2) {
        // vertex lives in pinned HOST memory (in-place entry): consecutive lanes read consecutive float2 of the same pixel
        // row so each selected pixel costs one contiguous 8*K-byte PCIe read, not K scattered ones
        const int nel = min(total, max(cap - base, 0)) * K;
        constexpr int U = 4;                       // PCIe reads in flight per thread
        for (int e0 = tid; e0 < nel; e0 += GA_THREADS * U) {
            float2 val[U];
            int tt[U], kk[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int e = e0 + u * GA_THREADS;
                tt[u] = -1;
                if (e < nel) {
                    const int i = e / K, k = e - i * K;
                    const int p = blk * (TS_THREADS * 32) + (int)s_list[i];
                    const int y = p / W, x = p - y * W;
                    tt[u] = base + i; kk[u] = k;
                    if (k == 0) xy[(size_t)b * cap + base + i] = make_float2((float)x, (float)y);
                    val[u] = __ldg(reinterpret_cast<const float2 *>(vimg + (long long)y * sH + (long long)x * sW) + k);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (tt[u] >= 0) dirs[((size_t)b * K + kk[u]) * cap + tt[u]] = val[u];
        }
        return;
    }
    for (int i = tid; i < total; i += GA_THREADS) {
        const int t = base + i;
        if (t >= cap) break;
        const int p = blk * (TS_THREADS * 32) + (int)s_list[i];
        const int y = p / W, x = p - y * W;
        xy[(size_t)b * cap + t] = make_float2((float)x, (float)y);
        const float *vb = vimg + (long long)y * sH + (long long)x * sW;
        float2 *db = dirs + (size_t)b * K * cap + t;
        // plain cached loads: the K loads of one pixel hit the same one or two lines, and an evict-first hint
        // (ld.global.cs) throws those lines out between them -- measured slower on the select stage
        if (vec) {
            for (int k = 0; k < K; ++k)
                db[(size_t)k * cap] = __ldg(reinterpret_cast<const float2 *>(vb + (long long)k * sK));
        } else {
            for (int k = 0; k < K; ++k) {
                const float *q = vb + (long long)k * sK;
                db[(size_t)k * cap] = make_float2(__ldg(q), __ldg(q + sC));
            }
        }
    }
}

// ---------------------------------------------------------------------------------
// gather access pattern for an interleaved vertex tensor ([..,K,2] contiguous) in DEVICE memory: 0 = auto = 1 = pixel-wise
// (one lane per pixel, K independent loads in flight per lane), 2 = row-wise (consecutive lanes read consecutive float2 of
// one pixel's 8*K-byte row).  Pixel-wise was the faster of the two at cfg-2 when it was chosen (not re-measured on the
// H100): the kernel is latency-bound and the pixel-wise walk keeps 9 loads per lane in flight.  Pinned HOST
// memory read in place is always fetched row-wise (a PCIe read is charged per 128-byte line touched, tools/pcie_probe.cu).
// Tooling / A-B measurements; results are identical.
static std::atomic<int> g_gather_mode{0};
void set_gather_tuning(int mode) { g_gather_mode.store(mode, std::memory_order_relaxed); }

cudaError_t launch_select(const SelectArgs &a, cudaStream_t st)
{
    const int nwords = a.nwords;
    dim3 g1((nwords + MB_WARPS * MB_WORDS - 1) / (MB_WARPS * MB_WORDS), a.B);
#define PVB_MB2(T, MODE)                                                                                 \
    do {                                                                                                 \
        const int vec_ok = contig && (reinterpret_cast<uintptr_t>(a.mask) % 16 == 0) &&                  \
                           ((a.msb * (long long)sizeof(T)) % 16 == 0);                                   \
        if (contig)                                                                                      \
            mask_bits_kernel<T, MODE, true><<<g1, MB_WARPS * 32, 0, st>>>(                                \
                (const T *)a.mask, a.msb, a.msy, a.msx, a.H, a.W, nwords, a.bits, a.fgsum, a.nz, vec_ok); \
        else                                                                                             \
            mask_bits_kernel<T, MODE, false><<<g1, MB_WARPS * 32, 0, st>>>(                               \
                (const T *)a.mask, a.msb, a.msy, a.msx, a.H, a.W, nwords, a.bits, a.fgsum, a.nz, 0);     \
    } while (0)
#define PVB_MB(T)                                                                                        \
    do {                                                                                                 \
        if (a.select_mode == PVB_SELECT_BYTE) PVB_MB2(T, PVB_SELECT_BYTE);                               \
        else PVB_MB2(T, PVB_SELECT_EQ1);                                                                 \
    } while (0)
    const bool contig = (a.msx == 1 && a.msy == a.W);
    if (a.seg_classes > 0) {
        if (a.select_mode == PVB_SELECT_BYTE)
            seg_bits_kernel<PVB_SELECT_BYTE><<<g1, MB_WARPS * 32, 0, st>>>((const float *)a.mask, a.msb, a.seg_cs, a.msy, a.msx,
                                                                          a.seg_classes, a.H, a.W, nwords, a.mask_out, a.bits, a.fgsum, a.nz);
        else
            seg_bits_kernel<PVB_SELECT_EQ1><<<g1, MB_WARPS * 32, 0, st>>>((const float *)a.mask, a.msb, a.seg_cs, a.msy, a.msx,
                                                                         a.seg_classes, a.H, a.W, nwords, a.mask_out, a.bits, a.fgsum, a.nz);
    } else
    switch (a.mask_dtype) {
    case PVB_MASK_U8: PVB_MB(uint8_t); break;
    case PVB_MASK_I8: PVB_MB(int8_t); break;
    case PVB_MASK_I16: PVB_MB(int16_t); break;
    case PVB_MASK_I32: PVB_MB(int32_t); break;
    case PVB_MASK_I64: PVB_MB(long long); break;
    case PVB_MASK_F32: PVB_MB(float); break;
    case PVB_MASK_F64: PVB_MB(double); break;
    default: return cudaErrorInvalidValue;
    }
#undef PVB_MB
#undef PVB_MB2
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    dim3 g2(a.nblocks, a.B);
    const int gmode = g_gather_mode.load(std::memory_order_relaxed);
    thin_gather_kernel<<<g2, GA_THREADS, 0, st>>>(a.bits, a.blocktot, a.ticket, a.fgsum, a.tn, a.state, a.status, a.selection,
                                                  a.vertex, a.vs[0], a.vs[1], a.vs[2], a.vs[3], a.vs[4], a.xy, a.dirs, nwords,
                                                  a.nblocks, a.K, a.cap, a.W, a.H * a.W, a.min_num, a.max_num,
                                                  make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)), a.tag_sel, a.img_base,
                                                  a.b0, (a.rowwise_gather || gmode == 2) ? 1 : 0);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// mask_iou of the LINEMOD evaluator (lib/evaluators/linemod/pvnet.py:96-100) for B images:
//   inter[b] = sum(pred & gt), uni[b] = sum(pred | gt)
// It sums the VALUES of the bitwise ops, not pixel counts.  numpy promotes both operands to a common integer type; here
// both are widened to int64 by value (sign-extended if signed, zero-extended if not), which gives the same value, because
// the bits above a narrower promoted result are copies of its top bit in both operands.  The sums are exact modulo 2^64
// like numpy's int64 sum, so the atomics cannot change the result.
// A warp takes IOU_TILE elements at a time.  When both images are contiguous and 16-byte aligned, each operand's tile is
// staged in shared memory with 16-byte evict-first loads (sizeof(T) of them per lane, consecutive lanes on consecutive
// 16 bytes) whatever the two element sizes are; then lane l combines elements l, l + 32, ...  Strided views and the last,
// partial tile of an image are read element by element in the same order.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int IOU_WARPS = 4;
constexpr int IOU_TILE = 32 * 16;                // elements per warp tile: 16 per lane

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <typename TP, typename TG>
__device__ __forceinline__ void iou_add(TP p, TG g, unsigned long long &si, unsigned long long &su)
{
    const long long a = (long long)p, c = (long long)g;
    si += (unsigned long long)(a & c);
    su += (unsigned long long)(a | c);
}

template <typename TP, typename TG>
__global__ void __launch_bounds__(IOU_WARPS * 32)
mask_iou_kernel(const TP *__restrict__ pred, long long psb, long long psy, long long psx, const TG *__restrict__ gt,
                long long gsb, long long gsy, long long gsx, int B, int H, int W, unsigned long long *__restrict__ inter,
                unsigned long long *__restrict__ uni)
{
    __shared__ uint4 s_p[IOU_WARPS][IOU_TILE * sizeof(TP) / 16];
    __shared__ uint4 s_g[IOU_WARPS][IOU_TILE * sizeof(TG) / 16];
    __shared__ unsigned long long s_red[2][IOU_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int HW = H * W, ntiles = (HW + IOU_TILE - 1) / IOU_TILE;
    const bool contig = psx == 1 && psy == W && gsx == 1 && gsy == W;
    for (int b = blockIdx.y; b < B; b += gridDim.y) {
        const TP *pb = pred + (long long)b * psb;
        const TG *gb = gt + (long long)b * gsb;
        const bool vec = contig && ((reinterpret_cast<uintptr_t>(pb) | reinterpret_cast<uintptr_t>(gb)) & 15u) == 0;
        unsigned long long si = 0, su = 0;
        for (int t = blockIdx.x * IOU_WARPS + warp; t < ntiles; t += gridDim.x * IOU_WARPS) {
            const int e0 = t * IOU_TILE;
            if (vec && e0 + IOU_TILE <= HW) {
                const uint4 *qp = reinterpret_cast<const uint4 *>(pb + e0), *qg = reinterpret_cast<const uint4 *>(gb + e0);
                uint4 vp[sizeof(TP)], vg[sizeof(TG)];
#pragma unroll
                for (int j = 0; j < (int)sizeof(TP); ++j) vp[j] = ld_stream16(qp + j * 32 + lane);
#pragma unroll
                for (int j = 0; j < (int)sizeof(TG); ++j) vg[j] = ld_stream16(qg + j * 32 + lane);
#pragma unroll
                for (int j = 0; j < (int)sizeof(TP); ++j) s_p[warp][j * 32 + lane] = vp[j];
#pragma unroll
                for (int j = 0; j < (int)sizeof(TG); ++j) s_g[warp][j * 32 + lane] = vg[j];
                __syncwarp();
                const TP *sp = reinterpret_cast<const TP *>(s_p[warp]);
                const TG *sg = reinterpret_cast<const TG *>(s_g[warp]);
#pragma unroll
                for (int k = 0; k < IOU_TILE / 32; ++k) iou_add(sp[k * 32 + lane], sg[k * 32 + lane], si, su);
                __syncwarp();                            // read before the next tile overwrites it
            } else {
#pragma unroll 4
                for (int k = 0; k < IOU_TILE / 32; ++k) {
                    const int e = e0 + k * 32 + lane;
                    if (e >= HW) break;
                    const int y = e / W, x = e - y * W;
                    iou_add(__ldg(pb + y * psy + x * psx), __ldg(gb + y * gsy + x * gsx), si, su);
                }
            }
        }
        si = warp_sum_u64(si);
        su = warp_sum_u64(su);
        if (lane == 0) { s_red[0][warp] = si; s_red[1][warp] = su; }
        __syncthreads();
        if (threadIdx.x == 0) {
            si = su = 0;
#pragma unroll
            for (int w = 0; w < IOU_WARPS; ++w) { si += s_red[0][w]; su += s_red[1][w]; }
            if (si) atomicAdd(inter + b, si);
            if (su) atomicAdd(uni + b, su);
        }
        __syncthreads();                                 // s_red is reused by the next image
    }
}

namespace {

template <typename TP, typename TG>
void launch_mask_iou_typed(const void *pred, const long long *ps, const void *gt, const long long *gs, long long *inter,
                           long long *uni, int B, int H, int W, cudaStream_t st)
{
    const int ntiles = (int)(((long long)H * W + IOU_TILE - 1) / IOU_TILE);
    const dim3 grid((unsigned)((ntiles + IOU_WARPS - 1) / IOU_WARPS), (unsigned)(B < 65535 ? B : 65535));
    mask_iou_kernel<TP, TG><<<grid, IOU_WARPS * 32, 0, st>>>(
        static_cast<const TP *>(pred), ps[0], ps[1], ps[2], static_cast<const TG *>(gt), gs[0], gs[1], gs[2], B, H, W,
        reinterpret_cast<unsigned long long *>(inter), reinterpret_cast<unsigned long long *>(uni));
}

template <typename TP>
bool launch_mask_iou_gt(const void *pred, const long long *ps, const void *gt, int gt_dtype, const long long *gs,
                        long long *inter, long long *uni, int B, int H, int W, cudaStream_t st)
{
    switch (gt_dtype) {
    case PVB_MASK_U8: launch_mask_iou_typed<TP, uint8_t>(pred, ps, gt, gs, inter, uni, B, H, W, st); return true;
    case PVB_MASK_I8: launch_mask_iou_typed<TP, int8_t>(pred, ps, gt, gs, inter, uni, B, H, W, st); return true;
    case PVB_MASK_I16: launch_mask_iou_typed<TP, int16_t>(pred, ps, gt, gs, inter, uni, B, H, W, st); return true;
    case PVB_MASK_I32: launch_mask_iou_typed<TP, int32_t>(pred, ps, gt, gs, inter, uni, B, H, W, st); return true;
    case PVB_MASK_I64: launch_mask_iou_typed<TP, long long>(pred, ps, gt, gs, inter, uni, B, H, W, st); return true;
    default: return false;
    }
}

} // namespace

} // namespace pvb

using namespace pvb;

extern "C" {

PVB_API int pvb_mask_iou(const void *pred, int32_t pred_dtype, const int64_t *pred_stride, const void *gt, int32_t gt_dtype,
                         const int64_t *gt_stride, int64_t *inter, int64_t *uni, int32_t B, int32_t H, int32_t W,
                         pvb_stream_t stream)
{
    if (B < 0 || H < 0 || W < 0) return fail(PVB_ERR_INVALID, "negative size (B=%d H=%d W=%d)", B, H, W);
    for (int32_t dt : {pred_dtype, gt_dtype})
        if (dt < PVB_MASK_U8 || dt > PVB_MASK_I64)
            return fail(PVB_ERR_INVALID, "mask dtypes must be integer pvb_mask_dtypes (U8..I64), got %d and %d", pred_dtype,
                        gt_dtype);
    if (B == 0) return PVB_OK;
    if (!pred_stride || !gt_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    const long long HW = (long long)H * W;
    if (!inter || !uni || (HW > 0 && (!pred || !gt))) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (HW > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    for (int i = 0; i < 3; ++i)
        if (pred_stride[i] < 0 || gt_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
    const long long ps[3] = {pred_stride[0], pred_stride[1], pred_stride[2]};
    const long long gs[3] = {gt_stride[0], gt_stride[1], gt_stride[2]};
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    long long *in = reinterpret_cast<long long *>(inter), *un = reinterpret_cast<long long *>(uni);
    cudaError_t e = cudaMemsetAsync(in, 0, (size_t)B * sizeof(long long), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(un, 0, (size_t)B * sizeof(long long), st);
    if (e == cudaSuccess && HW > 0) {
        bool ok = false;
        switch (pred_dtype) {
        case PVB_MASK_U8: ok = launch_mask_iou_gt<uint8_t>(pred, ps, gt, gt_dtype, gs, in, un, B, H, W, st); break;
        case PVB_MASK_I8: ok = launch_mask_iou_gt<int8_t>(pred, ps, gt, gt_dtype, gs, in, un, B, H, W, st); break;
        case PVB_MASK_I16: ok = launch_mask_iou_gt<int16_t>(pred, ps, gt, gt_dtype, gs, in, un, B, H, W, st); break;
        case PVB_MASK_I32: ok = launch_mask_iou_gt<int32_t>(pred, ps, gt, gt_dtype, gs, in, un, B, H, W, st); break;
        case PVB_MASK_I64: ok = launch_mask_iou_gt<long long>(pred, ps, gt, gt_dtype, gs, in, un, B, H, W, st); break;
        default: break;
        }
        e = ok ? cudaGetLastError() : cudaErrorInvalidValue;
    }
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "mask iou kernel");
}

} // extern "C"
