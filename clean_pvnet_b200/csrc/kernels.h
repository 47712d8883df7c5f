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
    double *pose;             // [n][3][4]: the pose of pvb_pnp_iterative (launch_pnp_iterative only)
    int n, pn;
    long long pts3d_stride, k_stride;
    PnpOptions opt;
};
cudaError_t launch_pnp_batch(const PnpArgs &a, cudaStream_t st);
// PVNet's default pose step, cv2.solvePnP(..., SOLVEPNP_ITERATIVE) (pnp.cu, pnp_iter_core.cuh): reads pts2d, pts3d, K and
// the strides; writes pose [n][3][4], result_rt (optional) and info (optional: iterations, pvb_pnp_status).
cudaError_t launch_pnp_iterative(const PnpArgs &a, cudaStream_t st);

// exact nearest neighbour and ADD / ADD-S (nn.cu).  A problem's pn2 queries go to `qchunks` CTAs, its pn1 reference points
// to `nsplit` slices of `slice` points; nsplit > 1 (chosen from the shapes when b * qchunks CTAs cannot fill the GPU)
// merges the slices through a 64-bit key per query in the workspace.
struct NnPlan { int qchunks, nsplit, slice; };
NnPlan nn_plan(int b, int pn1, int pn2);
size_t nn_workspace_bytes(int b, int pn1, int pn2);
// ADD-S keys [n][pn] (split path only), then the per-CTA partial sums [n][qchunks] at *partial_offset
size_t add_metric_workspace_bytes(int n, int pn, int syn, size_t *partial_offset);
// ref [b][pn1][dim], que [b][pn2][dim] fp32 -> idxs [b][pn2]
cudaError_t launch_nearest_point(const float *ref, const float *que, int *idxs, int b, int pn1, int pn2, int dim,
                                 bool exclude_self, void *workspace, cudaStream_t st);
// model [pn][3], pose_pred / pose_gt [n][3][4] fp64 -> mean_dist [n] fp64
cudaError_t launch_add_metric(const double *model, const double *pose_pred, const double *pose_gt, double *mean_dist, int n,
                              int pn, bool syn, void *workspace, cudaStream_t st);
// projection_2d / cm_degree_5 (nn.cu): the per-CTA partial sums [n][ceil(pn / 2048)] of the reprojection distances
size_t pose_metrics_workspace_bytes(int n, int pn);
// model [pn][3], pose_pred / pose_gt [n][3][4], K [3][3] at K + pair * k_stride, fp64 -> proj2d, trans_cm, angle_deg [n]
cudaError_t launch_pose_metrics(const double *model, const double *pose_pred, const double *pose_gt, const double *K,
                                long long k_stride, double *proj2d, double *trans_cm, double *angle_deg, int n, int pn,
                                void *workspace, cudaStream_t st);
// mask_iou (select.cu): inter[b] = sum(pred & gt), uni[b] = sum(pred | gt) over [B,H,W] masks of integer pvb_mask_dtypes
// with strides ps / gs (elements); zeroes both outputs first
cudaError_t launch_mask_iou(const void *pred, int pred_dtype, const long long *ps, const void *gt, int gt_dtype,
                            const long long *gs, long long *inter, long long *uni, int B, int H, int W, cudaStream_t st);

// T-LESS's VSD (render.cu, DESIGN.md 8f).  Depth rasterizer: pts [V][3] fp32, faces [F][3] int32, poses [n][3][4] fp64,
// K [3][3] fp64 at K + pose * k_stride -> depth [n][H][W] fp32.  Workspace: a queue counter, then n * F queue entries.
size_t render_workspace_bytes(int n, int F);
cudaError_t launch_render_depth(const float *pts, int V, const int *faces, int F, const double *poses, int n,
                                const double *K, long long k_stride, float *depth, int H, int W, double znear,
                                double zfar, void *workspace, cudaStream_t st);
struct VsdArgs {
    const float *depth_test, *depth_est, *depth_gt;  // [B][H][W], [n_est][H][W], [n_gt][H][W]
    const int *pairs;                                // [n][3]: est index, gt index, image index
    const double *K;                                 // [3][3] per image at K + image * k_stride
    long long k_stride;
    int n, B, n_est, n_gt, est_base, gt_base, H, W;  // rows use est in [est_base, est_base + n_est), likewise gt
    double delta, tau;
    double *e;                                       // [n]: written only for rows within the windows
};
// workspace: the integer counts of the n rows
size_t vsd_workspace_bytes(int n);
cudaError_t launch_vsd(const VsdArgs &a, void *workspace, cudaStream_t st);
// T-LESS's instance masks (render.cu, DESIGN.md 8k).  table: HOST int32 [B + 1 + 2m], image b's instances are
// [table[b], table[b+1]) (table[0] == 0), then the depth slot of each of the m instances, then its label.  Writes
// label [B][H][W] int16 and a_out / p_out [m] int64, box_out [m][4] int32 (x, y, w, h).  max_m: the most instances
// of one image (<= MASK_MAX_INSTANCES).  Workspace: the table, then the integer sums of the m instances.
constexpr int MASK_MAX_INSTANCES = 2048;
size_t instance_masks_workspace_bytes(int B, int m);
cudaError_t launch_instance_masks(const float *depth, const int *table, int B, int m, int max_m, int H, int W,
                                  short *label, long long *a_out, long long *p_out, int *box_out, void *workspace,
                                  cudaStream_t st);

// T-LESS's PVNet crop (crop.cu, DESIGN.md 8g).  Setup: one thread per box -> centre, scale, forward (and inverse) crop
// matrix.  Warp: one CTA per (box, output row) over [n][out_h]; the crop variant masks, normalises and writes NCHW fp32.
struct CropArgs {
    const double *boxes;          // [n][4] xyxy, image coordinates
    int n, out_w, out_h, center_f64;  // center_f64: the cascade's fp64 centre, else pvnet_transform's fp32 one
    double scale_ratio;
    double *center, *scale;       // [n][2], [n]: as the reference computes them (fp64)
    double *M, *Minv;             // [n][6] forward crop matrix; inverse (inv=1) or NULL
};
cudaError_t launch_crop_setup(const CropArgs &a, cudaStream_t st);
struct WarpArgs {
    const unsigned char *img;     // [B][H][W][C] at element strides sb, sh, sw, sc
    long long sb, sh, sw, sc;
    int B, H, W, C;
    const double *M;              // [n][6] forward matrices (warpAffine inverts them)
    const int *image_index;       // [n] or NULL (every row reads image 0)
    int n, out_w, out_h;
    const double *boxes;          // crop: [n][4], for the box mask
    int mask;                     // crop: zero what lies outside the magnified box
    double box_ratio;
    float mean[3], stdv[3];       // crop: normalisation
    float *inp;                   // crop: [n][3][out_h][out_w]
    unsigned char *out_u8;        // [n][out_h][out_w][C]: the warp's output; optional for the crop
};
cudaError_t launch_warp(const WarpArgs &a, bool crop, cudaStream_t st);
struct UncropArgs {
    const float *kpt;             // [n][K][2], crop frame
    const double *center, *scale; // [n][2], [n]
    int n, K, in_w, in_h;
    double *out;                  // [n][K][2], image frame
};
cudaError_t launch_uncrop(const UncropArgs &a, cudaStream_t st);

// PVNet's vote loss (loss.cu, DESIGN.md 8e): the target field of compute_vertex, the trainer's smooth-l1 vote loss and its
// gradient, from the mask and the keypoints.  One thread per pixel over a (ceil(H*W / 256), B) grid; the image's keypoints
// are staged in shared memory.
struct VoteLossArgs {
    const float *pred;        // [B][2K][H][W] at element strides ps (forward, backward)
    long long ps[4];
    const void *mask;         // [B][H][W] integer pvb_mask_dtype at element strides msb, msy, msx
    int mask_dtype;
    long long msb, msy, msx;
    const double *kpt;        // [B][K][2] contiguous, (x, y) per keypoint
    int B, H, W, K;
    float *out;               // contiguous [B][2K][H][W]: the target field (target) or grad_pred (backward)
    double *partial;          // [B * ceil(H*W / 256)] per-CTA sums of the smooth-l1 terms (forward)
    long long *wpart;         // [B * ceil(H*W / 256)] per-CTA sums of the mask values (forward)
    float *wsum;              // fp32 weight sum: written by the forward pass, read by the backward pass
    float *loss;              // the scalar loss (forward)
    const float *grad_loss;   // the scalar upstream gradient (backward)
};
// workspace: wsum at offset 0, then the two partial arrays, each 256-byte aligned
size_t vote_loss_workspace_bytes(int B, int H, int W, size_t *partial_offset, size_t *wpart_offset);
cudaError_t launch_vote_target(const VoteLossArgs &a, cudaStream_t st);
cudaError_t launch_vote_loss_forward(const VoteLossArgs &a, cudaStream_t st);
cudaError_t launch_vote_loss_backward(const VoteLossArgs &a, cudaStream_t st);

// The CenterNet heatmap target and focal loss (ct_loss.cu, DESIGN.md 8i), from the boxes.  One CTA per (32x16 pixel
// tile, class, image); the image's objects of that class whose window meets the tile are staged in shared memory.
struct CtArgs {
    const float *logits;      // [B][C][H][W] at element strides ls (forward, backward)
    long long ls[4];
    const long long *ct_ind;  // [B][M] cy * W + cx
    const int *ct_radius;     // [B][M]
    const long long *ct_cls;  // [B][M]
    const float *ct_01;       // [B][M] an object counts where ct_01 == 1
    int B, M, C, H, W;
    float *out;               // contiguous [B][C][H][W]: the target (target) or grad_logits (backward)
    double *pos_part, *neg_part;   // [nparts] per-CTA fp64 sums of the pos and neg terms (forward)
    int *cnt_part;            // [nparts] per-CTA counts of target == 1 (forward)
    long long *num_pos;       // exact count of target == 1: written by the forward pass, read by the backward pass
    float *loss;              // the scalar loss (forward)
    const float *grad_loss;   // the scalar upstream gradient (backward)
};
// workspace: num_pos at offset 0, then the three partial arrays, each 256-byte aligned
size_t ct_loss_workspace_bytes(int B, int C, int H, int W, size_t *pos_offset, size_t *neg_offset, size_t *cnt_offset);
cudaError_t launch_ct_target(const CtArgs &a, cudaStream_t st);
cudaError_t launch_ct_loss_forward(const CtArgs &a, cudaStream_t st);
cudaError_t launch_ct_loss_backward(const CtArgs &a, cudaStream_t st);

// The CenterNet decode (ct_decode.cu, DESIGN.md 8j): sigmoid, 3x3 peak test and top-K per image, then the boxes.
struct CtDecodeArgs {
    const float *hm;          // [B][C][H][W] logits at element strides hs
    long long hs[4];
    const float *wh;          // [B][2][H][W] at element strides ws
    long long ws[4];
    int B, C, H, W, K, clip;
    int T, Lk;                // tiles per class and entries per list (set by launch_ct_decode)
    long long L;              // lists per image, C * T
    unsigned long long *lists;   // workspace [B][L][Lk]: each tile's largest keys, descending
    unsigned long long *sel;     // workspace [B][K]: the image's K selected keys, unordered
    float *ct;                // [B][K][2] (xs, ys)
    float *det;               // [B][K][6] (x0, y0, x1, y1, score, class)
};
// workspace: the lists at offset 0, then sel, 256-byte aligned
size_t ct_decode_workspace_bytes(int B, int C, int H, int W, int K, size_t *sel_offset);
cudaError_t launch_ct_decode(CtDecodeArgs a, cudaStream_t st);

// modulated deformable convolution, DCNv2 (dcn.cu).  Contiguous fp32 NCHW; shapes validated by the C ABI.
struct DcnArgs {
    const float *input;       // [B][C][H][W]
    const float *offset;      // [B][dg*2*kh*kw][Ho][Wo]
    const float *mask;        // [B][dg*kh*kw][Ho][Wo]
    const float *weight;      // [Co][C][kh][kw]
    const float *bias;        // [Co]
    float *out;               // [B][Co][Ho][Wo] (forward)
    const float *grad_out;    // [B][Co][Ho][Wo] (backward)
    float *grad_input, *grad_offset, *grad_mask, *grad_weight, *grad_bias;   // shaped like their inputs (backward)
    float *cols;              // grad_cols [chunk][C*kh*kw][Ho*Wo] (backward workspace)
    int B, C, H, W, Co, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
};
// backward plan: images per grad_cols chunk, and grad_weight's split of the (image, pixel) reduction into `splits`
// ranges of `span` pixels over `ntile_n` column tiles.  Workspace: cols_bytes of grad_cols, then part_bytes of
// grad_weight partials (0 when splits == 1), each 256-byte aligned.  A function of the shapes only.
struct DcnPlan { int chunk, splits; long long span, ntile_n; size_t cols_bytes, part_bytes; };
DcnPlan dcn_plan(const DcnArgs &a, int chunk);
cudaError_t launch_dcn_forward(const DcnArgs &a, cudaStream_t st);
cudaError_t launch_dcn_backward(DcnArgs a, const DcnPlan &plan, void *workspace, cudaStream_t st);

// farthest-point sampling (fps.cu): the counts [b] and starts [b] (unused under init_center) tables, then the min_dist of
// every cloud's points past the first CTA's on-chip slice
size_t fps_workspace_bytes(int b, int n);
// pts [b][n][3] fp32, counts / starts HOST int32 [b] (validated by the caller) -> idxs [b][sn]
cudaError_t launch_fps(const float *pts, const int *counts, const int *starts, int init_center, int *idxs, int b, int n,
                       int sn, void *workspace, cudaStream_t st);

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
