/*
 * pvnet_vote_b200.h -- C ABI of the H100-native RANSAC voting layer.
 *
 * Drop-in boundary for clean-pvnet's `lib/csrc/ransac_voting` (reference paths
 * below are relative to the clean-pvnet checkout):
 *
 *   reference interface                                         replaced by
 *   ----------------------------------------------------------  ---------------------------------
 *   ransac_voting_gpu.py:112  ransac_voting_layer_v3(...)        pvb_ransac_voting_v3
 *   ransac_voting_gpu.py:6    ransac_voting_layer(...)           pvb_ransac_voting_v3 (same result,
 *                                                                 see DESIGN.md "v1 vs v3")
 *   ransac_voting_gpu.py:202  estimate_voting_distribution_...   pvb_estimate_voting_distribution
 *   src/ransac_voting.cpp:20  generate_hypothesis                pvb_generate_hypothesis
 *   src/ransac_voting.cpp:41  voting_for_hypothesis              pvb_voting_for_hypothesis
 *   src/ransac_voting.cpp:64  generate_hypothesis_vanishing_pt   pvb_generate_hypothesis_vanishing_point
 *   src/ransac_voting.cpp:85  voting_for_hypothesis_vanishing_pt pvb_voting_for_hypothesis_vanishing_point
 *
 *   and, for the callers either side of the layer (SURVEY.md section 8f):
 *   lib/networks/pvnet/resnet18.py:65-76  decode_keypoint         pvb_decode_v3 (+ pvb_estimate_voting_distribution)
 *   lib/evaluators/linemod/pvnet.py:118-130  weight loop          pvb_uncertainty_weights
 *   lib/csrc/uncertainty_pnp/src/ext.h  uncertainty_pnp(...)      pvb_uncertainty_pnp (batched)
 *   un_pnp_utils.py:25-31  cv2.solvePnP(..., SOLVEPNP_P3P)        pvb_uncertainty_pnp_init
 *   evaluators/linemod/pvnet.py:118-130 + un_pnp_utils.py:6-57     pvb_uncertainty_pnp_from_votes (all three, one launch)
 *   pvnet_pose_utils.py:5-38  pnp(...) = cv2.solvePnP(ITERATIVE)  pvb_pnp_iterative (batched; the default un_pnp=False path)
 *
 *   and the one native extension of the evaluators (lib/csrc/nn, cffi, imported by both):
 *   lib/csrc/nn/src/ext.h  findNearestPointIdxLauncher(...)       pvb_nearest_point_idx (device pointers, batched)
 *   evaluators/linemod/pvnet.py:68-82  add_metric distance,
 *   evaluators/tless_test/pvnet.py:107-117  adi_metric distance   pvb_add_metric (n pose pairs per call)
 *
 *   and the evaluators' other per-image metrics:
 *   evaluators/linemod/pvnet.py:59-66  projection_2d,
 *   evaluators/linemod/pvnet.py:84-94  cm_degree_5_metric,
 *   evaluators/tless_test/pvnet.py:119-125  cm_degree_5_metric     pvb_pose_metrics (n pose pairs per call)
 *   evaluators/linemod/pvnet.py:96-100  mask_iou                   pvb_mask_iou (B images per call)
 *
 *   and the training side of the vote field:
 *   utils/pvnet/pvnet_data_utils.py:30-44  compute_vertex          pvb_vote_target (B images per call)
 *   train/trainers/pvnet.py:25-27  vote loss                       pvb_vote_loss_forward / pvb_vote_loss_backward
 *
 * Conventions
 *   - plain C: device pointers, sizes, strides (in ELEMENTS), a CUDA stream
 *     handle.  No torch types.  All work is enqueued on `stream`; no entry
 *     point synchronises or allocates (the caller owns the workspace), so the
 *     calls are CUDA-graph capturable.  Exceptions: the *_host variants, which
 *     take HOST buffers and run their own copy/compute pipeline, and the setup
 *     calls of pvb_exchange (create / connect / destroy).
 *   - every function returns PVB_OK (0) or a pvb_status error code;
 *     pvb_last_error() returns a thread-local description.  Nothing calls
 *     exit()/abort() (the reference's gpuErrchk does, cuda_common.h:19-25).
 *   - there is NO CPU implementation behind this ABI.  If no CUDA device is
 *     usable the calls fail with PVB_ERR_CUDA.
 */
#ifndef PVNET_VOTE_B200_H_
#define PVNET_VOTE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PVB_VERSION 200

#if defined(__GNUC__)
#define PVB_API __attribute__((visibility("default")))
#else
#define PVB_API
#endif

typedef void *pvb_stream_t; /* cudaStream_t / CUstream, 0 = legacy default stream */

typedef enum pvb_status {
    PVB_OK = 0,
    PVB_ERR_INVALID = 1,   /* bad argument (null pointer, shape, dtype, stride) */
    PVB_ERR_CUDA = 2,      /* CUDA runtime / launch failure, or no usable device */
    PVB_ERR_WORKSPACE = 3, /* workspace too small or misaligned */
    PVB_ERR_CAPACITY = 4,  /* more pixels selected than `capacity` (reported by pvb_read_status) */
    PVB_ERR_TIMEOUT = 5    /* pvb_exchange_wait gave up: a rank never published its result */
} pvb_status;

/* element type of the mask tensor (reference: any dtype goes through .byte(), ransac_voting_gpu.py:125) */
typedef enum pvb_mask_dtype {
    PVB_MASK_U8 = 0, /* also torch.bool */
    PVB_MASK_I8 = 1,
    PVB_MASK_I16 = 2,
    PVB_MASK_I32 = 3,
    PVB_MASK_I64 = 4, /* torch.argmax output, resnet18.py:69 */
    PVB_MASK_F32 = 5,
    PVB_MASK_F64 = 6
} pvb_mask_dtype;

/* how foreground pixels are picked */
typedef enum pvb_select_mode {
    PVB_SELECT_BYTE = 0, /* v3: (uint8)mask != 0, fg = sum of byte values   (ransac_voting_gpu.py:125-126) */
    PVB_SELECT_EQ1 = 1   /* distribution: mask == 1, fg = pixel count       (ransac_voting_gpu.py:207-208) */
} pvb_select_mode;

/* Problem descriptor shared by the layer-level entry points. */
typedef struct pvb_desc {
    int32_t B, H, W, K;       /* batch, image height/width, keypoints (vn) */
    int32_t hn;               /* hypotheses per (image, keypoint): round_hyp_num for v3,
                                 round_hyp_num*ceil(min_hyp_num/round_hyp_num) for the distribution */
    float inlier_thresh;      /* cos threshold, compared as fp32 like the reference (.cu:124) */
    int32_t min_num, max_num; /* ransac_voting_gpu.py:129,135 */
    int32_t mask_dtype;       /* pvb_mask_dtype */
    int32_t select_mode;      /* pvb_select_mode */
    int64_t mask_stride[3];   /* strides of mask [B,H,W], elements */
    int64_t vertex_stride[5]; /* strides of vertex [B,H,W,K,2], elements (any layout, e.g. the permuted
                                 NCHW view decode_keypoint passes, resnet18.py:66-68) */
    int32_t capacity;         /* max selected pixels per image held by the workspace; 0 = default
                                 (min(H*W, max_num + 8*sqrt(max_num) + 64)); H*W is always safe */
    int32_t img_base;         /* global index of image 0 (multi-GPU shards keep one philox stream) */
    uint64_t seed;            /* philox seed, used when idxs / selection are NULL */
    int32_t rng_tag_idx;      /* philox stream tags (see DESIGN.md "Sampling"); 0 = per-op default */
    int32_t rng_tag_sel;
} pvb_desc;

/* Offsets (bytes from the workspace base) of the intermediate buffers; for tests and tooling. */
typedef struct pvb_layout {
    size_t total;    /* == pvb_workspace_bytes() */
    size_t status;   /* int32[4]: [0] sticky error code (pvb_status), [1] image that overflowed */
    size_t fgsum;    /* uint64[B]  sum of mask bytes (BYTE) / count (EQ1) */
    size_t nz;       /* int32[B]   selected-before-thinning count */
    size_t tn;       /* int32[B]   selected pixel count after thinning (0 when skipped) */
    size_t state;    /* int32[B]   0 ok, 1 skipped (fg < min_num) */
    size_t bits;     /* uint32[B][nwords] selection bitmap (after thinning), bit j of word w = pixel 32*w+j */
    size_t ticket;   /* int32[B] arrival counter of the compaction CTAs (block ids are drawn in arrival order) */
    size_t blocktot; /* uint32[B][nblocks] selected pixels per 128-word block | bit 31 "published" (decoupled look-back) */
    size_t xy;       /* float2[B][capacity]   (x,y) of the t-th selected pixel, row-major (torch.nonzero) order */
    size_t dirs;     /* float2[B][K][capacity] gathered vertex vectors (k-major) */
    size_t hyp;      /* float2[B][K][hn] */
    size_t counts;   /* int32[B][K][hn] */
    size_t win;      /* float2[B][K] winning hypothesis before the refit */
    size_t refit_partial; /* double[B][K][refit_splits][5] partial normal equations */
    size_t refit_ticket;  /* int32[B][K] arrival counters of the refit CTAs */
    size_t prune_cells;   /* int32[B][K][prune_ncells][68] per 32x32-pixel cell of the image (row-major): bounding box
                             (4 floats) of the cell's pixels that can vote, then the inclusive prefix sums of a 128-bin
                             histogram of their direction pseudo-angles as uint16 */
    size_t prune_key;     /* int32[B][K][hn] angular upper bound of each hypothesis's count, -1 if scored in pass 1 */
    size_t prune_list;    /* int32[2][B][K][hn] hypotheses scored by pass 1 / pass 2 of the pruned v3 vote */
    size_t prune_len;     /* int32[2][B][K] lengths of those lists; followed, at the next multiple of 256 bytes, by
                             int32[B][K][prune_ncells][4][68]: the records of each cell's four 16x16-pixel sub-cells (top
                             left, top right, bottom left, bottom right), laid out as prune_cells except that only the
                             last word (0) of an empty one is written; then, at the next multiple of 256 bytes,
                             int32[B][K][hn]: for the pass-2 candidates, the bound over the sub-cells */
    int32_t nwords;  /* ceil(H*W/32) */
    int32_t nblocks; /* ceil(nwords/128) */
    int32_t capacity;
    int32_t refit_splits;
    int32_t prune_ncells; /* ceil(H/32) * ceil(W/32) */
} pvb_layout;

PVB_API int pvb_version(void);
PVB_API const char *pvb_last_error(void);

/* Workspace sizing.  The workspace must be 256-byte aligned device memory. */
PVB_API size_t pvb_workspace_bytes(const pvb_desc *d);
PVB_API int pvb_workspace_layout(const pvb_desc *d, pvb_layout *out);

/* ransac_voting_layer_v3 (ransac_voting_gpu.py:112-199), whole batch, no host sync.
 *   mask    device, [B,H,W] of d->mask_dtype with d->mask_stride
 *   vertex  device fp32, [B,H,W,K,2] with d->vertex_stride
 *   idxs    optional device int32 [B,hn,K,2] contiguous: the reference's per-image `idxs`
 *           (:145).  NULL -> drawn in-kernel from the philox stream (seed, tag, image, k, h).
 *   selection optional device fp32 [B,H,W] contiguous: the reference's U(0,1) `selection`
 *           (:136), consulted only for images with fg > max_num.  NULL -> philox.
 *   out_kpt device fp32 [B,K,2] contiguous.
 * `confidence` / `max_iter` of the reference do not influence its result (idxs is drawn once,
 * outside the loop, :145 vs :150) and therefore have no counterpart here.
 * Only the winners and their inliers are observable, so this entry (like pvb_decode_v3, the _push and the host-buffer
 * entries) does not score hypotheses that an angular bound proves cannot win (DESIGN.md 4.2): their `counts` in the
 * workspace stay 0.  pvb_ransac_voting_v3_all_counts (below) computes the same keypoints and scores every hypothesis. */
PVB_API int pvb_ransac_voting_v3(const pvb_desc *d, const void *mask, const float *vertex,
                         const int32_t *idxs, const float *selection, float *out_kpt,
                         void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* Fused front end of Resnet18.decode_keypoint (lib/networks/pvnet/resnet18.py:65-76): same as
 * pvb_ransac_voting_v3, but the mask is torch.argmax(seg, 1) (:69) computed on the fly from the fp32 logits
 *   seg  device fp32 [B,classes,H,W]; d->mask_stride = its (B,H,W) strides, class_stride its class stride (elements);
 *        d->mask_dtype is ignored.  First maximal class wins, NaN counts as maximal (torch.argmax semantics).
 *   mask_out optional device int64 [B,H,W] contiguous: receives the argmax mask decode_keypoint returns (:73,:76).
 * d->select_mode applies to the class index exactly as it would to the mask tensor. */
PVB_API int pvb_decode_v3(const pvb_desc *d, const float *seg, int32_t classes, int64_t class_stride, int64_t *mask_out,
                          const float *vertex, const int32_t *idxs, const float *selection, float *out_kpt,
                          void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* estimate_voting_distribution_with_mean (ransac_voting_gpu.py:202-274).
 *   mean device fp32 [B,K,2];  out_cov device fp32 [B,K,2,2].  d->select_mode must be
 *   PVB_SELECT_EQ1 to match the reference (:207).  idxs optional int32 [B,hn,K,2] (the 16
 *   per-round draws of :235 concatenated in round order). */
PVB_API int pvb_estimate_voting_distribution(const pvb_desc *d, const void *mask, const float *vertex,
                                     const float *mean, const int32_t *idxs, const float *selection,
                                     float *out_cov, void *workspace, size_t workspace_bytes,
                                     pvb_stream_t stream);

/* Weights of the uncertainty PnP (lib/evaluators/linemod/pvnet.py:118-130, a scipy.linalg.sqrtm + np.linalg.inv loop
 * per keypoint on the CPU): weights[i] = (wxx, wxy, wyy) of inv(sqrtm(cov[i])), zeros where cov[i][0][0] < 1e-6, any
 * entry is NaN or cov[i] is not positive definite.  cov device fp32 [n,2,2] (16-byte aligned), weights device fp32 [n,3].
 * The result is what un_pnp_utils.uncertainty_pnp (lib/csrc/uncertainty_pnp/un_pnp_utils.py:6) takes as weights_2d. */
PVB_API int pvb_uncertainty_weights(const float *cov, float *weights, int32_t n, pvb_stream_t stream);

/* Batched twin of the reference's C entry `uncertainty_pnp(pts2d, pts3d, wgt2d, K, init_rt, result_rt, pn)`
 * (lib/csrc/uncertainty_pnp/src/ext.h:1-9, uncertainty_pnp.cpp:61-92; bound through cffi by un_pnp_utils.py:49-53): refines
 * n poses (angle-axis + translation, 6 doubles) by minimising the weighted reprojection error of pn points each with the
 * Levenberg-Marquardt trust-region loop and the default options of Ceres Solver 2.0 (the reference's minimiser; pinned
 * against the reference's own Ceres binary: tests/golden/ceres_pnp.npz, DESIGN.md section 8).  One warp per problem, fp64
 * like the reference.
 * All pointers are DEVICE memory: pts2d [n,pn,2], wgt2d [n,pn,3] = (wxx,wxy,wyy), init_rt / result_rt [n,6],
 * pts3d [pn,3] and K [3,3] (row-major) per problem at pts3d + p*pts3d_stride / K + p*k_stride (strides in doubles; 0 = one
 * array shared by all problems), info optional int32 [n,2] = (iterations, termination: 1 gradient, 2 parameter, 3 function
 * tolerance, 4 trust region collapsed, 5 iteration limit, 6 five invalid steps in a row).  options NULL = Ceres defaults. */
typedef struct pvb_pnp_options {
    int32_t max_num_iterations;       /* 50   */
    int32_t reserved;                 /* 0    */
    double function_tolerance;        /* 1e-6 */
    double gradient_tolerance;        /* 1e-10 */
    double parameter_tolerance;       /* 1e-8 */
} pvb_pnp_options;
PVB_API int pvb_uncertainty_pnp(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                const double *init_rt, double *result_rt, int32_t *info, int32_t n, int32_t pn,
                                int64_t pts3d_stride, int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream);

/* The whole un_pnp tail of the evaluator in ONE launch, straight from the voting layer's fp32 outputs:
 *   lib/evaluators/linemod/pvnet.py:118-130  weights = inv(sqrtm(var)) per keypoint          (pvb_uncertainty_weights)
 *   un_pnp_utils.py:25-31                    P3P initial pose on the 4 best-weighted points  (pvb_uncertainty_pnp_init)
 *   un_pnp_utils.py:49-53 -> ext.h           Ceres refinement                                (pvb_uncertainty_pnp)
 * kpt_2d device fp32 [n,pn,2]; exactly one of cov (device fp32 [n,pn,2,2], 16-byte aligned) and weights (device fp32
 * [n,pn,3]); pts3d / K as in pvb_uncertainty_pnp; init_rt optional [n,6] (NULL: P3P); result_rt [n,6]; optional outputs:
 * init_out [n,6] (the initial pose used), weights_out fp32 [n,pn,3], info [n,2].  pn <= 64.  Bit-identical to running the
 * three entry points one after the other on the same data (tests/test_gpu_pnp.py). */
PVB_API int pvb_uncertainty_pnp_from_votes(const float *kpt_2d, const float *cov, const float *weights, const double *pts3d,
                                           const double *K, const double *init_rt, double *result_rt, double *init_out,
                                           float *weights_out, int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride,
                                           int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream);

/* Initial poses for pvb_uncertainty_pnp, the reference's recipe on the device (un_pnp_utils.py:25-31:
 * `idxs = argsort(wxx + wxy)[-4:]`, `cv2.solvePnP(points_3d[idxs], points_2d[idxs], K, ..., flags=cv2.SOLVEPNP_P3P)`): P3P on
 * the 2nd..4th best-weighted keypoints, the best-weighted one chooses among the (up to four) poses by its reprojection
 * error.  Same layouts as pvb_uncertainty_pnp; writes init_rt [n,6] (angle-axis, translation); a problem without an
 * admissible solution gets NaNs (what OpenCV returns there).  pn >= 4.  The arithmetic is pinned against cv2.solvePnP on
 * the CPU (tests/test_p3p_host_core.py), the device launch against OpenCV on the GPU box (tests/test_gpu_zz_p3p.py). */
PVB_API int pvb_uncertainty_pnp_init(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                     double *init_rt, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                                     pvb_stream_t stream);

/* PVNet's default pose step for n problems: `pnp(points_3d, points_2d, camera_matrix)` of lib/utils/pvnet/
 * pvnet_pose_utils.py:5-38, i.e. cv2.solvePnP(..., zero distortion, flags=cv2.SOLVEPNP_ITERATIVE) followed by
 * [cv2.Rodrigues(rvec) | tvec], which both evaluators call once per image when cfg.test.un_pnp is False
 * (lib/evaluators/linemod/pvnet.py:188, tless_test/pvnet.py:239).  OpenCV's own method, step for step: its DLT start and
 * its 20-iteration Levenberg-Marquardt loop with OpenCV's damping schedule and stop rule (csrc/pnp_iter_core.cuh).  Pinned
 * against cv2.solvePnP 4.13 itself: rvec and tvec within 1e-8 relative wherever OpenCV's own answer is stable under a
 * 1e-13 relative change of the image points (tests/test_pnp_iter_host_core.py, tests/golden/pnp_iterative.npz).  One warp
 * per problem, fp64, no workspace.
 *   All pointers are DEVICE memory: pts2d [n,pn,2] pixels; pts3d [pn,3] and K [3,3] (row-major; fx, fy, cx, cy are read,
 *   skew and bottom row ignored like OpenCV) per problem at pts3d + p*pts3d_stride / K + p*k_stride (strides in doubles;
 *   0 = shared); pose [n,3,4] = [R | t]; rt optional [n,6] = (rvec, tvec); info optional int32 [n,2] = (LM iterations,
 *   pvb_pnp_status).  Every status but PVB_PNP_OK and PVB_PNP_ITERATION_LIMIT writes an all-NaN pose (and rt).  pn >= 1;
 *   n == 0 is a no-op.  Bad arguments return PVB_ERR_INVALID before any CUDA call. */
typedef enum pvb_pnp_status {
    PVB_PNP_OK = 0,                 /* stopped by |p - p_prev| / (|p_prev| + DBL_EPSILON) < FLT_EPSILON           */
    PVB_PNP_ITERATION_LIMIT = 1,    /* stopped after 20 iterations (OpenCV returns that pose too)                   */
    PVB_PNP_TOO_FEW_POINTS = 2,     /* pn < 4, or a non-planar model with pn < 6: OpenCV raises                     */
    PVB_PNP_PLANAR = 3,             /* W[2]/W[1] < 1e-3: OpenCV's homography start, not built here                   */
    PVB_PNP_DEGENERATE = 4          /* non-finite input, all image points equal, |RR|_F <= DBL_EPSILON, or a step
                                       whose damped system is not positive definite                                 */
} pvb_pnp_status;
PVB_API int pvb_pnp_iterative(const double *pts2d, const double *pts3d, const double *K, double *pose, double *rt,
                              int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                              pvb_stream_t stream);

/* Exact brute-force nearest neighbour, the batched device twin of the reference's
 * `findNearestPointIdxLauncher(ref_pts, que_pts, idxs, b, pn1, pn2, dim, exclude_self)` (lib/csrc/nn/src/ext.h,
 * nearest_neighborhood.cu:48-163, which takes host pointers and allocates, copies and frees on every call).
 *   ref device fp32 [b,pn1,dim], que device fp32 [b,pn2,dim], idxs device int32 [b,pn2]; dim 2 or 3.
 *   idxs[i][q] = the first p (scan order) minimising the reference's fp32 squared distance ref[i][p] - que[i][q]
 *   (exclude_self != 0: p != q), with its rounding; NaN / inf / FLT_MAX distances never win, and a query without any
 *   other distance gets 0.  Bit-equal to the reference kernel (DESIGN.md section 8b).
 *   workspace: pvb_nearest_point_workspace_bytes(b, pn1, pn2) bytes of 256-byte aligned device memory (0 bytes -- and
 *   NULL allowed -- when b * pn2 fills the GPU or pn1 is too short to split).  b == 0 or pn2 == 0 is a no-op.
 * Bad arguments (NULL tensors, dim not 2 or 3, negative sizes) return PVB_ERR_INVALID, a missing or short workspace
 * PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_nearest_point_workspace_bytes(int32_t b, int32_t pn1, int32_t pn2);
PVB_API int pvb_nearest_point_idx(const float *ref, const float *que, int32_t *idxs, int32_t b, int32_t pn1, int32_t pn2,
                                  int32_t dim, int32_t exclude_self, void *workspace, size_t workspace_bytes,
                                  pvb_stream_t stream);

/* The distance of the evaluators' ADD / ADD-S metric for n pose pairs in one call (Evaluator.add_metric,
 * lib/evaluators/linemod/pvnet.py:68-82; T-LESS's adi_metric, tless_test/pvnet.py:107-117, is its caller expanding the
 * (prediction, ground truth) pairs into the n rows):
 *   pred = model @ R_pred.T + t_pred, target = model @ R_gt.T + t_gt in fp64;
 *   syn != 0 (ADD-S): for every target point its nearest predicted point, found like pvb_nearest_point_idx on both clouds
 *   rounded to fp32 (what nn_utils.find_nearest_point_idx hands the reference kernel); syn == 0 (ADD): the same point;
 *   mean_dist[i] = mean over the points of |pred[idx] - target| in fp64.
 *   model device fp64 [pn,3] (shared by all pairs), pose_pred / pose_gt device fp64 [n,3,4] ([R|t]), mean_dist device
 *   fp64 [n].  The `< 0.1 * diameter` test stays with the caller.  pn == 0 gives NaN (the mean of nothing), n == 0 is a
 *   no-op.  workspace: pvb_add_metric_workspace_bytes(n, pn, syn) bytes of 256-byte aligned device memory. */
PVB_API size_t pvb_add_metric_workspace_bytes(int32_t n, int32_t pn, int32_t syn);
PVB_API int pvb_add_metric(const double *model, const double *pose_pred, const double *pose_gt, double *mean_dist, int32_t n,
                           int32_t pn, int32_t syn, void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* projection_2d + cm_degree_5 of the LINEMOD / T-LESS evaluators for n (prediction, ground truth) pose pairs
 * (Evaluator.projection_2d, lib/evaluators/linemod/pvnet.py:59-66, on pvnet_pose_utils.project, pvnet_pose_utils.py:41-50;
 * cm_degree_5_metric, linemod/pvnet.py:84-94 and pvnet_pose_utils.cm_degree_5:53-60), in fp64 with every product and sum
 * rounded on its own:
 *   uv = ((model @ R.T + t) @ K.T)[:, :2] / z for both poses;  proj2d[i] = mean over the points of |uv_pred - uv_gt|
 *   (z <= 0 gives what IEEE division gives; pn == 0 gives NaN, the mean of nothing)
 *   trans_cm[i] = |t_pred - t_gt| * 100
 *   angle_deg[i] = rad2deg(arccos((trace - 1) / 2)), trace = trace(R_pred R_gt^T) clamped like the reference:
 *   `trace if trace <= 3 else 3`, then `trace if trace >= -1 else -1`, so a NaN trace gives 0 degrees.
 *   model device fp64 [pn,3] (shared by all pairs), pose_pred / pose_gt device fp64 [n,3,4] ([R|t]), K device fp64 [3,3]
 *   row-major for pair i at K + i * k_stride (in doubles; 0 = one K for all), outputs device fp64 [n].  The thresholds
 *   (< 5 pixels; < 5 cm and < 5 degrees) stay with the caller.  T-LESS's any-of-all-pairs cm_degree_5_metric
 *   (tless_test/pvnet.py:119-125) is the caller expanding the (prediction, ground truth) pairs into the n rows.
 *   A pair's outputs do not depend on the other pairs.  workspace: pvb_pose_metrics_workspace_bytes(n, pn) bytes of
 *   256-byte aligned device memory (0 -- and NULL allowed -- when pn == 0).  n == 0 is a no-op.
 * Bad arguments return PVB_ERR_INVALID, a missing or short workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_pose_metrics_workspace_bytes(int32_t n, int32_t pn);
PVB_API int pvb_pose_metrics(const double *model, const double *pose_pred, const double *pose_gt, const double *K,
                             int64_t k_stride, double *proj2d, double *trans_cm, double *angle_deg, int32_t n, int32_t pn,
                             void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* mask_iou of the LINEMOD evaluator (lib/evaluators/linemod/pvnet.py:96-100) for B images:
 *   inter[b] = sum (pred & gt), uni[b] = sum (pred | gt)
 * the sums of the VALUES of the bitwise ops, as numpy computes them (with more than two classes, 2 & 1 = 0 and 2 | 1 = 3);
 * both operands are widened to int64 by value, and the int64 sums are exact (modulo 2^64, like numpy's).
 *   pred, gt  device [B,H,W] with element strides pred_stride / gt_stride (HOST int64[3]); pred_dtype / gt_dtype are
 *             integer pvb_mask_dtypes (U8, also for bool, I8, I16, I32, I64); F32 / F64 are rejected, as numpy's `&`
 *             rejects floats.  The evaluator's pair, an int64 prediction and a uint8 ground truth, both contiguous, is
 *             streamed with 16-byte loads.
 *   inter, uni device int64 [B], zeroed by the call itself in stream order (no workspace).  iou = inter / uni is the
 *   caller's (0 / 0 is NaN, as in numpy).  B == 0 is a no-op.
 * Bad arguments (negative sizes, NULL tensors or stride arrays, negative strides, other dtypes, H*W >= 2^31) return
 * PVB_ERR_INVALID before any CUDA call. */
PVB_API int pvb_mask_iou(const void *pred, int32_t pred_dtype, const int64_t *pred_stride, const void *gt, int32_t gt_dtype,
                         const int64_t *gt_stride, int64_t *inter, int64_t *uni, int32_t B, int32_t H, int32_t W,
                         pvb_stream_t stream);

/* ---- training: PVNet's vote loss from the mask and the keypoints (DESIGN.md section 8e) ----------------------------
 * The trainer supervises the unit-vector field with a dense target that every dataset builds on the host
 * (pvnet_data_utils.py:30-44 compute_vertex, called by lib/datasets/{linemod,custom}/pvnet.py:53 and
 * tless_train/pvnet.py:117).  These entries compute that target, and the loss and gradient that consume it, on the device.
 * Shared arguments:
 *   mask       device [B,H,W] of an integer pvb_mask_dtype (U8, also for bool, I8, I16, I32, I64) at element strides
 *              mask_stride (HOST int64[3]).  The target is non-zero only where mask == 1; the loss weight is float(mask).
 *   kpt_2d     device fp64 [B,K,2] contiguous, (x = column, y = row) per keypoint.
 *   B <= 65535, 1 <= K <= 1024, H*W < 2^31.  The target of channel 2k / 2k+1 at (x, y), where mask == 1, is compute_vertex's
 *   bit for bit: d = kpt - (x, y), n = sqrt(RN(dx*dx) + RN(dy*dy)), n < 1e-3 -> n + 1e-3, (dx / n, dy / n) rounded to fp32.
 * Bad arguments (negative sizes, K out of range, NULL pointers or stride arrays, negative strides, other dtypes) return
 * PVB_ERR_INVALID, a missing, short or misaligned workspace PVB_ERR_WORKSPACE, both before any CUDA call.  No entry
 * synchronises with the host. */

/* pvnet_data_utils.py:30-44 compute_vertex for a batch: vertex device fp32 [B,2K,H,W] contiguous, fully written.
 * B, H or W == 0 is a no-op. */
PVB_API int pvb_vote_target(const void *mask, int32_t mask_dtype, const int64_t *mask_stride, const double *kpt_2d,
                            float *vertex, int32_t B, int32_t H, int32_t W, int32_t K, pvb_stream_t stream);

/* The vote loss of lib/train/trainers/pvnet.py:25-27 with batch['vertex'] = compute_vertex(mask, kpt_2d), never built:
 *   w = float(mask);  loss = smooth_l1(pred * w, tgt * w, reduction='sum') / w.sum() / 2K
 * pred device fp32 [B,2K,H,W] at element strides pred_stride (HOST int64[4]), read at every pixel (a NaN or inf prediction
 * where w = 0 gives a NaN loss, as in the reference).  The terms are summed in fp64 and added in a fixed order, so the loss
 * is reproducible bit for bit; w.sum() is the exact int64 sum of the mask values rounded to fp32 (the reference's fp32 sum
 * agrees while its partial sums stay below 2^24).  loss: device fp32 scalar.  workspace:
 * pvb_vote_loss_workspace_bytes(B, H, W) bytes of 256-byte aligned device memory; it keeps the fp32 weight sum for
 * pvb_vote_loss_backward, so pass the same workspace to both.  B, H or W == 0 gives the reference's NaN (0 / 0). */
PVB_API size_t pvb_vote_loss_workspace_bytes(int32_t B, int32_t H, int32_t W);
PVB_API int pvb_vote_loss_forward(const float *pred, const int64_t *pred_stride, const void *mask, int32_t mask_dtype,
                                  const int64_t *mask_stride, const double *kpt_2d, float *loss, int32_t B, int32_t H,
                                  int32_t W, int32_t K, void *workspace, size_t workspace_bytes, pvb_stream_t stream);
/* autograd's gradient of that loss with respect to pred, bit for bit: grad_loss is the device fp32 upstream gradient
 * (read on the device, never by the host), grad_pred device fp32 [B,2K,H,W] contiguous, fully written.  The workspace is
 * the forward call's, after it.  B, H or W == 0 is a no-op. */
PVB_API int pvb_vote_loss_backward(const float *pred, const int64_t *pred_stride, const void *mask, int32_t mask_dtype,
                                   const int64_t *mask_stride, const double *kpt_2d, const float *grad_loss,
                                   float *grad_pred, int32_t B, int32_t H, int32_t W, int32_t K, const void *workspace,
                                   size_t workspace_bytes, pvb_stream_t stream);

/* Reads the sticky status word of a workspace (synchronises `stream`). */
PVB_API int pvb_read_status(const pvb_desc *d, const void *workspace, pvb_stream_t stream);

/* HOST-buffer variant of pvb_ransac_voting_v3: mask/vertex/out_kpt are host pointers
 * (pinned for full speed), contiguous [B,H,W] / [B,H,W,K,2] / [B,K,2].  Splits the batch into
 * `chunk_images`-sized pieces on three internal streams so that one piece's PCIe traffic overlaps the others'
 * kernels.  What crosses the bus is chosen per call by `flags`:
 *   0 (default)            the mask is staged -- one contiguous cudaMemcpyAsync per piece, the copy engine's PCIe
 *                          rate -- and the vertex field is read IN PLACE from the pinned host tensor: gather fetches only the
 *                          SELECTED pixels' rows (tn*K*8 bytes per image instead of the dense H*W*K*8)
 *   PVB_HOST_STAGE_VERTEX  also copy the dense vertex field (pageable inputs are always staged)
 *   PVB_HOST_INPLACE_MASK  read the mask in place as well (no DMA at all; round 1's mode)
 * Stream-ordered after the work already queued on `stream`; `stream` is synchronised before the
 * call returns (the result is in host memory), so CUDA events recorded on `stream` around the call
 * bracket all copies and kernels.  dev_scratch: 256-byte aligned device memory of
 * pvb_host_scratch_bytes(d, chunk_images) bytes.  Thread-safe (per-thread, per-device streams). */
#define PVB_HOST_STAGE_VERTEX 2u
#define PVB_HOST_INPLACE_MASK 4u
PVB_API size_t pvb_host_scratch_bytes(const pvb_desc *d, int32_t chunk_images);
PVB_API int pvb_ransac_voting_v3_host(const pvb_desc *d, const void *mask_host, const float *vertex_host,
                              float *out_kpt_host, int32_t chunk_images, uint32_t flags,
                              void *dev_scratch, size_t dev_scratch_bytes, pvb_stream_t stream);

/* ---- multi-GPU: images are sharded across ranks, one process per GPU (SURVEY.md 8e) --------------------------------
 * The path has no exchange inside the algorithm; what crosses GPUs is each rank's [B_r,K,2] keypoints becoming visible on
 * every rank.  The reference has no counterpart (torch.nn.DataParallel in the trainer only, lib/train/trainers/trainer.py:11).
 * A pvb_exchange is a receive ring in this rank's HBM -- recv[slots][world][floats_per_rank] of 8-byte words
 * {float bits, seq} -- mapped into every peer through CUDA IPC.  pvb_ransac_voting_v3_push is pvb_ransac_voting_v3 whose
 * refit kernel ALSO stores every (image, keypoint) result, as it is produced, into slot (seq-1)%slots of every peer's ring
 * over NVLink: aligned 8-byte stores are single-copy atomic, so every word validates itself and the producer needs no
 * fence, counter or flag and never waits.  pvb_exchange_wait enqueues a one-CTA kernel that polls this rank's own ring
 * until every expected word carries `seq` (bounded by timeout_s) and writes the floats to `out` (device fp32
 * [world][bytes_per_rank/4]; floats_per_rank: HOST array of world counts for ragged shards, NULL = every rank publishes
 * bytes_per_rank/4 floats).  Ring discipline (caller): before call `seq` is launched, the wait of call `seq - slots/2` must
 * already be enqueued on the same stream on every rank; seq starts at 1 and increases by 1 per call on every rank alike.
 * Setup (once): create -> get_handle -> all-gather the 64-byte handles by any means (e.g.
 * torch.distributed.all_gather_object) -> connect.  connect_ptrs takes raw base pointers instead (ranks that live in one
 * process, or memory mapped by other means). */
typedef struct pvb_exchange pvb_exchange;
#define PVB_IPC_HANDLE_BYTES 64
PVB_API int pvb_exchange_create(int32_t rank, int32_t world, int32_t slots, size_t bytes_per_rank, pvb_exchange **out);
PVB_API size_t pvb_exchange_bytes_per_rank(const pvb_exchange *ex); /* bytes_per_rank rounded up to 16 */
PVB_API void *pvb_exchange_base(const pvb_exchange *ex);
PVB_API int pvb_exchange_get_handle(const pvb_exchange *ex, void *handle /* PVB_IPC_HANDLE_BYTES */);
PVB_API int pvb_exchange_connect(pvb_exchange *ex, const void *handles /* world * PVB_IPC_HANDLE_BYTES, rank order */);
PVB_API int pvb_exchange_connect_ptrs(pvb_exchange *ex, void *const *bases /* world base pointers, rank order */);
PVB_API int pvb_ransac_voting_v3_push(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
                                      const float *selection, float *out_kpt, void *workspace, size_t workspace_bytes,
                                      pvb_exchange *exchange, uint64_t seq, pvb_stream_t stream);
/* pvb_ransac_voting_v3 (exchange == NULL) or pvb_ransac_voting_v3_push with every hypothesis scored: afterwards the
 * workspace's `counts` hold the reference's inlier count of every hypothesis (the Python operator's debug=True). */
PVB_API int pvb_ransac_voting_v3_all_counts(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
                                            const float *selection, float *out_kpt, void *workspace, size_t workspace_bytes,
                                            pvb_exchange *exchange, uint64_t seq, pvb_stream_t stream);
/* the same for the second half of the un_pnp pair (resnet18.py:71-72): every [2,2] covariance goes to every peer as the
 * covariance kernel produces it (4 floats per (image, keypoint); use an exchange of its own: bytes_per_rank >= B*K*16) */
PVB_API int pvb_estimate_voting_distribution_push(const pvb_desc *d, const void *mask, const float *vertex, const float *mean,
                                                  const int32_t *idxs, const float *selection, float *out_cov, void *workspace,
                                                  size_t workspace_bytes, pvb_exchange *exchange, uint64_t seq,
                                                  pvb_stream_t stream);
PVB_API int pvb_exchange_wait(pvb_exchange *ex, uint64_t seq, void *out, const int32_t *floats_per_rank, double timeout_s,
                              pvb_stream_t stream);
PVB_API int pvb_exchange_status(pvb_exchange *ex, pvb_stream_t stream); /* synchronises; PVB_ERR_TIMEOUT after a timed-out wait */
PVB_API int pvb_exchange_destroy(pvb_exchange *ex);

/* Stage timing (tooling, used by bench.py).  pvb_profile_enable(n): n = 0 off; n >= 1: every n-th call of a layer entry
 * point records 5 CUDA events on the launching stream at its stage boundaries (an event record drains the pipeline between
 * two kernels, ~3 us each on B200: sample with n > 1 to keep the profile out of a measurement).  pvb_profile_read()
 * synchronises those events and ADDS the elapsed milliseconds of every profiled call since the last pvb_profile_reset()
 * into ms[PVB_STAGE_COUNT], returning the number of calls accumulated.  Per host thread. */
enum { PVB_STAGE_SELECT = 0,   /* mask_bits + thin_gather (thinning, ordered compaction, vertex gather) */
       PVB_STAGE_GENERATE = 1, /* hypothesis generation */
       PVB_STAGE_VOTE = 2,     /* counts memset + vote kernel (the dominant kernel) */
       PVB_STAGE_FINISH = 3,   /* winner + refit, or covariance */
       PVB_STAGE_COUNT = 4 };
PVB_API int pvb_profile_enable(int32_t every);
/* Tuning switches (tooling for A/B measurements; process-wide, atomic).  Results do not depend on them.
 *   gather_mode  access pattern of the gather kernel on an interleaved vertex tensor in device memory: 0 = auto = 1 =
 *                pixel-wise (one lane per pixel), 2 = row-wise (a warp reads whole 8*K-byte pixel rows; what in-place
 *                host reads always use)
 *   vote_variant pixel tile of the vote kernel above 256 hypotheses per keypoint: 0 = 1 = 1024 pixels (default),
 *                2 = 256, 3 = 512; up to 256 hypotheses the tile is always 512 */
PVB_API int pvb_set_tuning(int32_t gather_mode, int32_t vote_variant);
PVB_API int pvb_profile_reset(void);
PVB_API int pvb_profile_read(double *ms, int32_t n);

/* ---- twins of the reference pybind module `ransac_voting` (ransac_voting.cpp:102-107) ---- */
/* direct [tn,vn,2] f32, coords [tn,2] f32, idxs [hn,vn,2] i32 -> hyp [hn,vn,2] f32 (fully written;
 * degenerate pairs give (0,0), the reference's zero fill, .cu:42-43,75) */
PVB_API int pvb_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs, float *hyp,
                            int32_t tn, int32_t vn, int32_t hn, pvb_stream_t stream);
/* sets inliers[h,k,t]=1 (uint8 [hn,vn,tn]) where the test passes; other bytes untouched (.cu:124-125) */
PVB_API int pvb_voting_for_hypothesis(const float *direct, const float *coords, const float *hyp, uint8_t *inliers,
                              int32_t tn, int32_t vn, int32_t hn, float inlier_thresh, pvb_stream_t stream);
/* hyp [hn,vn,3] */
PVB_API int pvb_generate_hypothesis_vanishing_point(const float *direct, const float *coords, const int32_t *idxs,
                                            float *hyp, int32_t tn, int32_t vn, int32_t hn,
                                            pvb_stream_t stream);
PVB_API int pvb_voting_for_hypothesis_vanishing_point(const float *direct, const float *coords, const float *hyp,
                                              uint8_t *inliers, int32_t tn, int32_t vn, int32_t hn,
                                              float inlier_thresh, pvb_stream_t stream);

/* Fused count of the above (voting_for_hypothesis + torch.sum(dim 2), ransac_voting_gpu.py:156-159)
 * on the reference layouts: counts int32 [hn,vn].  Same kernel the layer uses. */
PVB_API int pvb_vote_count(const float *direct, const float *coords, const float *hyp, int32_t *counts,
                   int32_t tn, int32_t vn, int32_t hn, float inlier_thresh,
                   void *workspace, size_t workspace_bytes, pvb_stream_t stream);
PVB_API size_t pvb_vote_count_workspace_bytes(int32_t tn, int32_t vn, int32_t hn);

#ifdef __cplusplus
}
#endif
#endif /* PVNET_VOTE_B200_H_ */
