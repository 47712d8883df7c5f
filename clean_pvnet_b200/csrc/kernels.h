// kernels.h -- the voting chain's internal interface: the argument blocks and launches of select.cu, vote.cu, prune.cu and
// exchange.cu, which api.cu's v3 plan, image groups and host pipeline drive.  compat.cu's pvb_vote_count runs launch_vote.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/pvnet_vote_b200.h"

namespace pvb {

struct SelectArgs {
    const void *mask;
    int mask_dtype, select_mode;
    long long msb, msy, msx;      // mask strides (elements)
    const float *vertex;
    long long vs[5];              // vertex strides (elements)
    const float *selection;       // optional [B,H,W]
    int B, H, W, K, nwords, nblocks, cap, min_num, max_num, img_base;
    int b0;                       // index of image 0 in the call (a group's args, api.cu): status[1] reports b0 + b
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
// The v3 chain's launches (select, generate, vote, refit) are programmatic dependent launches (common.cuh states the rule).
// `chained`: the launch directly follows the chain kernel before it in the same stream (thin_gather for generate); pass
// false after anything else (a memset, an event wait) or where chaining measured slower (DESIGN.md 4.3).
// hypotheses for every (image, keypoint): explicit idxs or philox; also zeroes counts[b][k][h]
cudaError_t launch_generate(const VoteArgs &a, bool chained, cudaStream_t st);
// counts[b][k][h] += #pixels voting for hyp[b][k][h]; launch_generate zeroes counts, other callers pass zero_counts = true
// (and chained = false: the memset precedes the kernel)
cudaError_t launch_vote(const VoteArgs &a, bool zero_counts, bool chained, cudaStream_t st);

// Pruned v3 vote (prune.cu, DESIGN.md 4.2): only hypotheses that can still be the first maximum are scored.  A bound
// B(h) >= count(h) comes from per-cell direction histograms; pass 1 scores the PRUNE_M largest bounds, pass 2 every other
// hypothesis whose bound reaches pass 1's best count and whose bound over the cells' four sub-cells reaches it too.  The
// others keep count 0, below the winner's.
constexpr int PRUNE_CELL = 32;              // histogram cells are PRUNE_CELL x PRUNE_CELL pixels of the image
constexpr int PRUNE_SUB = PRUNE_CELL / 2;   // each split into 2 x 2 sub-cells, which refine pass 2
constexpr int PRUNE_NBIN = 128;             // pseudo-angle bins per cell
constexpr int PRUNE_REC = 4 + PRUNE_NBIN / 2;   // words per (image, keypoint, cell): box, 16-bit inclusive prefix counts
constexpr int PRUNE_M = 128;                // pass-1 hypotheses = one slice of the pruned vote shape
constexpr int PRUNE_MAX_HN = 2048;          // pass 1 is picked from every bound staged in shared memory
constexpr int PRUNE_MIN_UNITS = 32;         // fewer (image, keypoint) pairs: the full vote is faster
static_assert(PRUNE_CELL * PRUNE_CELL < 65536, "a cell's prefix counts fit 16 bits");
struct PruneArgs {
    int *cells;          // [B][K][ncells][PRUNE_REC], cell (row band y, column x) at y * ncx + x
    int *sub;            // [B][K][ncells][4][PRUNE_REC], the sub-cells of each cell: top left, top right, bottom left,
                         // bottom right; a cell's record is their union.  Of an empty one only the last word (0) is written
    int *key;            // [B][K][hn]  bound, or -1 for pass-1 hypotheses
    int *b2;             // [B][K][hn]  bound over the sub-cells of pass-2 candidates: zeroed by the bound step, summed by
                         // prune_next_kernel
    int *list;           // [2][B][K][hn]
    int *len;            // [2][B][K]
    int *list2, *len2;   // pass 2's half of each: list + B*K*hn, len + B*K (of the whole call when a group's args)
    int *ticket;         // [B][K] arrival counter of the bound CTAs: 0 at the start of the call, and left 0
    int ncx, ncells;     // ceil(W / PRUNE_CELL), ceil(H / PRUNE_CELL) * ncx
    float cos_w, sin_w;  // rotation by the widened cone half-angle theta'
};
// false when pruning cannot pay (thresholds outside (0,1) or nearly 0, hn <= PRUNE_M, hn > PRUNE_MAX_HN, B*K < PRUNE_MIN_UNITS);
// otherwise fills cos_w / sin_w
bool prune_setup(const VoteArgs &a, PruneArgs &q);
// cell histograms + bounds + pass 1 + pass 2; counts must be zeroed (launch_generate)
cudaError_t launch_vote_pruned(const VoteArgs &a, const PruneArgs &q, cudaStream_t st);
// Both passes score hypothesis lists: entry s of (b,k) is hypothesis list[(b*K+k)*hn + s], s < len[b*K+k] <= max_len.
// Pass 2: vote_list_kernel, pixels in registers, one CTA per (tile, k, b) over the whole list, which costs its real length.
cudaError_t launch_vote_list(const VoteArgs &a, const int *list, const int *len, int max_len, cudaStream_t st);
// Pass 1: vote_kernel, hypotheses in registers, in slices of 128 entries
cudaError_t launch_vote_list_slices(const VoteArgs &a, const int *list, const int *len, int max_len, cudaStream_t st);
void set_vote_tuning(int variant);   // tooling: pixel-tile size per CTA
void set_pass1_stats(unsigned long long *dev);   // tooling: pass 1's per-box test counts (NULL: off)
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

} // namespace pvb
