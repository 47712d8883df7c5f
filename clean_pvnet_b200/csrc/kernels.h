// kernels.h -- internal launch interface between api.cu and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/pvnet_vote_b200.h"
#include "pnp_core.cuh"

namespace pvb {

struct SelectArgs {
    const void *mask;
    int mask_dtype, select_mode;
    long long msb, msy, msx;      // mask strides (elements)
    const float *vertex;
    long long vs[5];              // vertex strides (elements)
    const float *selection;       // optional [B,H,W]
    int B, H, W, K, nwords, nblocks, cap, min_num, max_num, img_base;
    int rowwise_gather;           // 1: vertex is read in place from pinned host memory: always whole pixel rows per warp
    int seg_classes;              // > 0: `mask` points to fp32 logits [B,C,H,W]; the mask is argmax over C
    long long seg_cs;             // class stride of the logits (elements)
    long long *mask_out;          // optional int64 [B,H,W] argmax output
    uint64_t seed;
    uint32_t tag_sel;
    uint32_t *bits;
    unsigned *blocktot;           // [B][nblocks] block totals | READY bit (zeroed with the header)
    int *ticket;                  // [B] arrival counter of the thin_gather CTAs (zeroed with the header)
    unsigned long long *fgsum;
    int *nz, *tn, *state, *status;
    float2 *xy, *dirs;
};
cudaError_t launch_select(const SelectArgs &a, cudaStream_t st);

struct VoteArgs {
    int B, K, hn, cap, W, H;
    float thresh;
    const int *tn;        // [B]
    const int *state;     // [B]
    const float2 *xy;     // [B][cap]   pixel coordinates (x,y)
    const float2 *dirs;   // [B][K][cap]
    const int32_t *idxs;  // optional [B][hn][K][2]
    uint64_t seed;
    uint32_t tag_idx;
    int img_base;
    float2 *hyp;          // [B][K][hn]
    int *counts;          // [B][K][hn]
};
// hypotheses for every (image, keypoint): explicit idxs or philox; also zeroes counts[b][k][h]
cudaError_t launch_generate(const VoteArgs &a, cudaStream_t st);
// counts[b][k][h] += #pixels voting for hyp[b][k][h]; launch_generate zeroes counts, other callers pass zero_counts = true
cudaError_t launch_vote(const VoteArgs &a, bool zero_counts, cudaStream_t st);
void set_vote_tuning(int variant);   // tooling: pixel-tile size per CTA
void set_gather_tuning(int mode);    // tooling: gather access pattern (select.cu)
// argmax + winner refit -> out_kpt [B][K][2], win [B][K].  The pixels of one (image,keypoint) are split
// over `splits` CTAs; partial normal equations meet in `partial`, the last CTA to arrive (ticket) adds
// them in a fixed order and solves, so the result is deterministic.
struct RefitScratch { double *partial; int *ticket; int splits; };
int refit_splits_for(int cap);
// Multi-GPU result exchange fused into the refit kernel (SURVEY 8e).  The thread that writes an (image, keypoint) result
// also stores it into every peer's receive slot over NVLink as two 8-byte words {float bits, seq}: an aligned 8-byte
// store is single-copy atomic, so the word carries its own validity flag (the protocol NCCL calls LL) and the producer
// needs no fence, no completion counter and no separate flag -- it fires 2*world stores and is done.  Consumers poll the
// words of slot (seq-1) % slots in their OWN memory until every flag equals seq (launch_exchange_wait).
constexpr int PVB_MAX_PEERS = 16;
struct PeerPush {
    int world;                                  // 0: no exchange
    unsigned int seq;                           // low 32 bits of the call's sequence number (never 0)
    uint2 *recv[PVB_MAX_PEERS];                 // peer r: where THIS rank's words of the current slot live in r's memory
};
cudaError_t launch_refit(const VoteArgs &a, float2 *win, const RefitScratch &rs, float *out_kpt, const PeerPush &pp,
                         cudaStream_t st);
// polls the {data, seq} words of one slot -- rank r publishes counts.n[r] floats at recv + r*stride_words -- until every
// flag equals seq (bounded by timeout_ns), writing the data to out[r*stride_words + i]; on timeout sets *status = 1 and
// fills `out` with NaN
struct ExchangeCounts { int n[PVB_MAX_PEERS]; };
cudaError_t launch_exchange_wait(const uint2 *recv, unsigned int seq, float *out, int world, int stride_words,
                                 const ExchangeCounts &counts, unsigned long long timeout_ns, int *status, cudaStream_t st);
// ratio/threshold/weighted covariance -> out_cov [B][K][2][2] (+ the same exchange tail as the refit kernel, 4 floats per unit)
cudaError_t launch_covariance(const VoteArgs &a, const float *mean, float *out_cov, const PeerPush &pp, cudaStream_t st);

// inv(sqrtm(cov)) packed (wxx,wxy,wyy): cov [n][2][2] -> w [n][3]
cudaError_t launch_pnp_weights(const float *cov, float *w, int n, cudaStream_t st);

// batched uncertainty PnP (pnp.cu): n problems of pn points, one warp per problem, fp64 like the reference.  The 2D
// inputs are either fp64 pts2d + wgt2d, read in place, or (kpt2d != NULL) the voting layer's fp32 keypoints with their
// covariances or weights, converted into shared memory (pn <= PNP_FUSED_MAX_PN).
constexpr int PNP_FUSED_MAX_PN = 64;
struct PnpArgs {
    const double *pts2d;      // [n][pn][2]
    const double *wgt2d;      // [n][pn][3]  (wxx, wxy, wyy)
    const float *kpt2d;       // [n][pn][2]  (the voting layer's kpt_2d)
    const float *cov;         // [n][pn][2][2] (the voting layer's var), or NULL ...
    const float *weights;     // ... then [n][pn][3] precomputed (wxx, wxy, wyy)
    float *weights_out;       // optional [n][pn][3]: the fp32 weights used (kpt2d only)
    const double *pts3d;      // [pn][3], problem p at pts3d + p*pts3d_stride (0: shared)
    const double *K;          // [3][3] row-major, problem p at K + p*k_stride (0: shared)
    const double *init_rt;    // optional [n][6]; NULL: P3P on the four best-weighted points
    double *init_out;         // optional [n][6]: the initial pose that was used
    double *result_rt;        // [n][6]: the refined pose; NULL: the P3P start alone (fp64 inputs, into init_out)
    int *info;                // optional [n][2]: iterations, termination code
    int n, pn;
    long long pts3d_stride, k_stride;
    PnpOptions opt;
};
cudaError_t launch_pnp_batch(const PnpArgs &a, cudaStream_t st);

// twins of the reference extension on its own layouts
cudaError_t launch_compat_generate(const float *direct, const float *coords, const int32_t *idxs, float *hyp,
                                   int tn, int vn, int hn, bool vanishing, cudaStream_t st);
cudaError_t launch_compat_vote(const float *direct, const float *coords, const float *hyp, uint8_t *inliers,
                               int tn, int vn, int hn, float thresh, bool vanishing, cudaStream_t st);
// reference layout -> layer layout (pix/dirs/hyp in k-major) for pvb_vote_count
// meta: int[4] = { tn, state(0), unused, unused }
cudaError_t launch_compat_repack(const float *direct, const float *coords, const float *hyp, int tn, int vn,
                                 int hn, float2 *dirs, float2 *xy, float2 *hyp_k, int *meta, cudaStream_t st);
cudaError_t launch_compat_unpack_counts(const int *counts_k, int *counts, int vn, int hn, cudaStream_t st);

} // namespace pvb
