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
 *   utils/renderer/opengl_utils.py:405-490  DepthRender.render     pvb_render_depth (n poses per call, no OpenGL)
 *   utils/vsd/vsd_utils.py:5-48  vsd (cost 'step'), as
 *   evaluators/tless_test/pvnet.py:66-105  vsd_metric calls it     pvb_vsd (n pose pairs per call)
 *   datasets/tless/handle_test_data.py:81-134  get_mask's
 *     render + update_mask loop, pixel_num.pkl, boundingRect       pvb_instance_masks (B images per call)
 *   lib/csrc/fps/src/ext.h  farthest_point_sampling{,_init_center}  pvb_farthest_point_sampling (b clouds per call)
 *   utils/tless/tless_test_utils.py:57-77  pvnet_transform,
 *   networks/ct_pvnet/res.py:14-31  _crop                           pvb_crop_inputs (n boxes per call)
 *   evaluators/tless_test/pvnet.py:229-239  keypoint un-crop        pvb_uncrop_keypoints (n boxes per call)
 *   cv2.warpAffine(..., INTER_LINEAR)                              pvb_warp_affine_linear (n rows per call)
 *
 *   and the training side of the vote field:
 *   utils/pvnet/pvnet_data_utils.py:30-44  compute_vertex          pvb_vote_target (B images per call)
 *   train/trainers/pvnet.py:25-27  vote loss                       pvb_vote_loss_forward / pvb_vote_loss_backward
 *
 *   and the training side of the detector's heatmap:
 *   datasets/tless{,_ag,_test}/ct.py ct_hm: utils/data_utils.py:36-64
 *     gaussian2D + draw_umich_gaussian                             pvb_ct_target (B images per call)
 *   train/trainers/ct.py:20-21 + utils/net_utils.py:9-39
 *     FocalLoss(sigmoid(output['ct_hm']), ct_hm)                   pvb_ct_loss_forward / pvb_ct_loss_backward
 *
 *   and the detector's decode at inference:
 *   networks/ct/dla.py:20-26  decode_detection: sigmoid +
 *     utils/ct/ct_decode.py:6-75 decode_ct_hm + clip_to_image     pvb_ct_decode (B images per call)
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

/* ---- T-LESS's VSD without OpenGL (DESIGN.md section 8f) ------------------------------------------------------------
 * Depth rendering: replaces lib/utils/renderer/opengl_utils.py:405-490 (DepthRender.render, which the T-LESS evaluator
 * calls as render((720, 540), 100, 10000, K, R, t * 1000) at tless_test/pvnet.py:85, :93) and the depth mode of
 * lib/utils/vsd/renderer.py's render.  For each of n poses:
 *   R, t are rounded to fp32 (the shader's float32 view matrix), model points go to the camera frame in fp64, and pixel
 *   (row r, column c) samples the ray through (u, v) = (c + 0.5, r + 0.5), u = fx X/Z + s Y/Z + cx, v = fy Y/Z + cy.  The
 *   pixel holds the camera-frame Z of the nearest triangle along that ray with clip_near <= Z <= clip_far, rounded to fp32,
 *   or 0.  No culling; triangles crossing the near plane or behind the camera are clipped, never projected through 0.
 *   Coverage is watertight: a pixel centre on an edge or vertex shared by triangles is covered by one of them.
 *   pts device fp32 [V,3], faces device int32 [F,3] (a face with an index outside [0, V) is skipped), poses device fp64
 *   [n,3,4] ([R|t], in the units of pts), K device fp64 [3,3] row-major for pose i at K + i * k_stride (0 = shared; only
 *   fx, s, cx, fy, cy are read, like _compute_calib_proj), depth device fp32 [n,H,W], fully written.  The result is
 *   bit-identical run to run and a pose's image does not depend on the other poses.
 *   n <= 65535, n * F < 2^31, H * W < 2^31, 0 < clip_near <= clip_far < inf.  workspace:
 *   pvb_render_depth_workspace_bytes(n, F) bytes of 256-byte aligned device memory (0 -- and NULL allowed -- when F == 0).
 * Bad arguments return PVB_ERR_INVALID, a missing or short workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_render_depth_workspace_bytes(int32_t n, int32_t F);
PVB_API int pvb_render_depth(const float *pts, int32_t V, const int32_t *faces, int32_t F, const double *poses, int32_t n,
                             const double *K, int64_t k_stride, float *depth, int32_t H, int32_t W, double clip_near,
                             double clip_far, void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* VSD: replaces vsd_utils.vsd (lib/utils/vsd/vsd_utils.py:5-48) with cost 'step', together with the distance images
 * (misc.depth_im_to_dist_im, lib/utils/vsd/misc.py:42-60) and visibility masks (lib/utils/vsd/visibility.py:6-29) that
 * Evaluator.vsd_metric (tless_test/pvnet.py:66-105) builds for it, for n rows (est, gt, image) of `pairs`:
 *   dist = sqrt((X*X + Y*Y) + Z*Z), X = ((c - cx) * Z) * (1/fx), Y = ((r - cy) * Z) * (1/fy) in fp64, each step rounded on
 *   its own as numpy does, at the integer pixel coordinate (c, r);
 *   vg = dist_test > 0 & dist_gt > 0 & float(dist_gt) - float(dist_test) <= float(delta)
 *   ve = (dist_test > 0 & dist_est > 0 & float(dist_est) - float(dist_test) <= float(delta)) | (vg & dist_est > 0)
 *   e  = (#(vg & ve & |dist_gt - dist_est| >= tau) + #(vg | ve) - #(vg & ve)) / #(vg | ve), 1.0 for an empty union.
 *   depth_test device fp32 [B,H,W] (the evaluator's load_depth(path) * 0.1), depth_est fp32 [n_est,H,W] and depth_gt fp32
 *   [n_gt,H,W] (pvb_render_depth), pairs device int32 [n,3], K device fp64 [3,3] of image b at K + b * k_stride.  Row i
 *   uses depth_est[pairs[i][0] - est_base] and depth_gt[pairs[i][1] - gt_base]; a row whose indices fall outside
 *   [est_base, est_base + n_est), [gt_base, gt_base + n_gt) or [0, B) is left untouched in e (device fp64 [n]), so a
 *   caller can render the poses in windows and call once per window pair.  No distance image or mask is stored; the
 *   counts are integers, so e is exact and deterministic.  The `e < 0.3` test and the any-of over an image's rows stay
 *   with the caller.  workspace: pvb_vsd_workspace_bytes(n) bytes of 256-byte aligned device memory.  n == 0 is a no-op.
 * Bad arguments return PVB_ERR_INVALID, a missing or short workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_vsd_workspace_bytes(int32_t n);
PVB_API int pvb_vsd(const float *depth_test, int32_t B, const float *depth_est, int32_t n_est, int32_t est_base,
                    const float *depth_gt, int32_t n_gt, int32_t gt_base, const int32_t *pairs, int32_t n, const double *K,
                    int64_t k_stride, int32_t H, int32_t W, double delta, double tau, double *e, void *workspace,
                    size_t workspace_bytes, pvb_stream_t stream);

/* ---- T-LESS's instance masks without OpenGL (DESIGN.md section 8k) -------------------------------------------------
 * Replaces the per-instance loop of lib/datasets/tless/handle_test_data.py:93-134 (get_mask: opengl_renderer.render
 * + update_mask at :81-90 + np.sum(depth != 0)), and the counts and cv2.boundingRect that test_to_coco (:14-61) and
 * record_scene_ann (:137-194) take from its mask PNGs and pixel_num.pkl, for B images at once.  Image b composes the
 * instances [image_first[b], image_first[b+1]) in order; instance i, the (i - image_first[b])-th of its image, reads
 * depth[slot[i]] (pvb_render_depth's mm depth, e.g. at clip planes 10 / 10000):
 *   key = fp32(depth / 1000) (opengl_renderer.render's division); per pixel the label map starts at 0 and the depth map
 *   at 10.0f, and the instance takes the pixel when key != 0 and key < depth map (ties go to the earlier instance; a key
 *   of 10 or more never takes it); label[b] is then obj_id[i] * 1000 + (i - image_first[b]) where instance i took it.
 *   a_pixel_num[i] = #(key != 0), pixel_num[i] = #(pixels labelled i), bbox[i] = cv2.boundingRect of those pixels as
 *   (x, y, w, h), (0, 0, 0, 0) when there are none.
 *   depth device fp32 [n_depth,H,W]; slot, obj_id HOST int32 [n]; image_first HOST int32 [B+1]; label device int16
 *   [B,H,W], fully written; a_pixel_num, pixel_num device int64 [n] and bbox device int32 [n,4] are written for the
 *   instances [image_first[0], image_first[B]) and left untouched elsewhere, so a caller can render the instances in
 *   windows of whole images and call once per window.  No mask is stored; every output is an integer sum of per-CTA
 *   integer reductions, so the result is exact and bit-identical run to run, and an image's outputs depend on nothing
 *   else in the call.  Each range must be non-empty, within [0, n) and hold at most 2048 instances, each slot in
 *   [0, n_depth), each label must fit int16, B <= 65535 and H * W < 2^31.  The table is copied to the device from host
 *   memory within the call, so unlike the other entries this one cannot be captured into a CUDA graph.  workspace:
 *   pvb_instance_masks_workspace_bytes(B, image_first[B] - image_first[0]) bytes of 256-byte aligned device memory.
 *   B == 0 is a no-op.
 * Bad arguments return PVB_ERR_INVALID, a missing or short workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_instance_masks_workspace_bytes(int32_t B, int32_t m);
PVB_API int pvb_instance_masks(const float *depth, int32_t n_depth, const int32_t *slot, const int32_t *obj_id, int32_t n,
                               const int32_t *image_first, int32_t B, int32_t H, int32_t W, int16_t *label,
                               int64_t *a_pixel_num, int64_t *pixel_num, int32_t *bbox, void *workspace,
                               size_t workspace_bytes, pvb_stream_t stream);

/* ---- farthest-point sampling (DESIGN.md section 8l) ------------------------------------------------------------------
 * The batched device twin of the reference's two cffi entries (lib/csrc/fps/src/ext.h, farthest_point_sampling.cpp)
 *   farthest_point_sampling(pts, idxs, pn, sn)               (random start: rand() % pn after srand(time(0)))
 *   farthest_point_sampling_init_center(pts, idxs, pn, sn)   (start: the point farthest from the bounding box's centre)
 * for b clouds at once.  Cloud i is the first counts[i] rows of pts[i]; idxs[i] are the reference's indices for it, element
 * for element, with its fp32 arithmetic (no contraction), its index-order tie rule and its fallback to index 0 when no
 * unselected point has a distance > 0 (so sn > counts[i] repeats index 0).  init_center == 0 starts cloud i at
 * starts[i], the value the reference draws with rand(); everything after the start is bit-equal.
 *   pts device fp32 [b,n,3]; counts HOST int32 [b], each in [1, n]; starts HOST int32 [b], each in [0, counts[i])
 *   (ignored, and NULL allowed, when init_center != 0); idxs device int32 [b,sn].  workspace:
 *   pvb_fps_workspace_bytes(b, n) bytes of 256-byte aligned device memory.  The tables are copied to the device from host
 *   memory within the call, so, like pvb_instance_masks, it cannot be captured into a CUDA graph; it does not synchronise
 *   with the host.  b == 0 or sn == 0 is a no-op.
 * Bad arguments (NULL pointers, negative sizes, a count or start out of range) return PVB_ERR_INVALID, a missing or short
 * workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
PVB_API size_t pvb_fps_workspace_bytes(int32_t b, int32_t n);
PVB_API int pvb_farthest_point_sampling(const float *pts, const int32_t *counts, const int32_t *starts, int32_t init_center,
                                        int32_t *idxs, int32_t b, int32_t n, int32_t sn, void *workspace,
                                        size_t workspace_bytes, pvb_stream_t stream);

/* ---- T-LESS's PVNet crop and un-crop (DESIGN.md section 8g) ---------------------------------------------------------
 * Shared: img device uint8 [B,H,W,C] at element strides img_stride (HOST int64[4], for B, H, W, C), H, W <= 32767;
 * image_index device int32 [n] or NULL (every row reads image 0; an index outside [0, B) reads as an all-border image).
 * Pixels follow cv2.warpAffine(INTER_LINEAR) with the zero border exactly: the forward matrix inverted as warpAffine
 * inverts it, 10-bit offsets rounded half to even, 5-bit sub-pixel positions, 15-bit integer bilinear weights.
 * n * out_h < 2^31.  Bad arguments return PVB_ERR_INVALID before any CUDA call; n == 0 is a no-op. */
#define PVB_CROP_MASK_TO_BOX 1     /* zero what lies outside the magnified box (pvnet_transform; the cascade does not) */
#define PVB_CROP_CENTER_F64  2     /* the cascade's fp64 centre (res.py _crop), else pvnet_transform's fp32 centre */

/* Replaces tless_test_utils.pvnet_transform (lib/utils/tless/tless_test_utils.py:57-77) and, with flags =
 * PVB_CROP_CENTER_F64, the cascade's _crop (lib/networks/ct_pvnet/res.py:14-31), for n boxes (device fp64 [n,4] xyxy):
 *   center = ((x0 + x2) / 2, (y0 + y2) / 2) (rounded to fp32 unless PVB_CROP_CENTER_F64), scale = max(x2 - x0, y2 - y0) *
 *   scale_ratio; matrix = get_affine_transform(center, scale, 0, [out_w, out_h]) bit for bit with cv2.getAffineTransform
 *   (all zeros for a singular system, as cv2 returns), matrix_inv the same with inv=1 (optional);
 *   crop = cv2.warpAffine(img, matrix, (out_w, out_h)), zeroed outside magnify_box(box corners through matrix,
 *   box_ratio) under PVB_CROP_MASK_TO_BOX; inp = (crop / 255 - mean) / std in fp32 (mean, std HOST float[3], std != 0).
 * Outputs (device): inp fp32 [n,3,out_h,out_w] (NCHW), crop_u8 uint8 [n,out_h,out_w,3] or NULL (the dataset's orig_img),
 * center fp64 [n,2], scale fp64 [n] (the unrounded product; get_affine_transform uses it rounded to fp32), matrix fp64
 * [n,2,3], matrix_inv fp64 [n,2,3] or NULL.  C must be 3.  The output is bit-identical run to run and a box's output
 * does not depend on the other boxes. */
PVB_API int pvb_crop_inputs(const uint8_t *img, int32_t B, int32_t H, int32_t W, const int64_t *img_stride,
                            const double *boxes, const int32_t *image_index, int32_t n, int32_t out_w, int32_t out_h,
                            double scale_ratio, double box_ratio, int32_t flags, const float *mean, const float *std,
                            float *inp, uint8_t *crop_u8, double *center, double *scale, double *matrix,
                            double *matrix_inv, pvb_stream_t stream);

/* Replaces the evaluator's affine_transform(kpt_2d, get_affine_transform(center, scale, 0, [in_w, in_h], inv=1))
 * (lib/evaluators/tless_test/pvnet.py:229-239) for n boxes: kpt_2d device fp32 [n,K,2] in the crop frame, center device
 * fp64 [n,2], scale device fp64 [n] (rounded to fp32, as get_affine_transform does) -> out device fp64 [n,K,2] in the
 * image.  The matrix is bit for bit cv2's; the product follows np.dot's rounding on x86-64 OpenBLAS (y * m1 fused into
 * the rounded x * m0), pinned to <= 1e-12 px. */
PVB_API int pvb_uncrop_keypoints(const float *kpt_2d, const double *center, const double *scale, int32_t n, int32_t K,
                                 int32_t in_w, int32_t in_h, double *out, pvb_stream_t stream);

/* cv2.warpAffine(img[image_index[i]], M[i], (out_w, out_h), flags=INTER_LINEAR) (zero border) for n rows: M device fp64
 * [n,2,3] forward matrices, C in 1..4, out device uint8 [n,out_h,out_w,C].  Also the detector's full-image resize
 * (tless_test_utils.augment, lib/utils/tless/tless_test_utils.py:14-31). */
PVB_API int pvb_warp_affine_linear(const uint8_t *img, int32_t B, int32_t H, int32_t W, int32_t C, const int64_t *img_stride,
                                   const double *M, const int32_t *image_index, int32_t n, int32_t out_w, int32_t out_h,
                                   uint8_t *out, pvb_stream_t stream);

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

/* ---- training the detector: CenterNet's heatmap target and focal loss from the boxes (DESIGN.md section 8i) -----------
 * The CenterNet datasets (lib/datasets/{tless,tless_ag,tless_test}/ct.py) draw a dense [C,H,W] heatmap per sample with
 * data_utils.draw_umich_gaussian; the trainer (lib/train/trainers/ct.py:20-21) takes net_utils.FocalLoss of
 * net_utils.sigmoid(logits) against it.  These entries compute that target, and the loss and gradient that consume it,
 * on the device from the objects.  Shared arguments, each device [B,M] contiguous:
 *   ct_ind     int64, cy * W + cx of the object's centre
 *   ct_radius  int32, r = max(0, int(gaussian_radius((ceil(h), ceil(w))))) from the sample's own float64 box size
 *   ct_cls     int64, the object's class
 *   ct_01      fp32, 1 for an object, anything else for padding
 * An object counts where ct_01 == 1, 0 <= ct_cls < C, 0 <= ct_ind < H*W and r >= 0; any other values match nothing.
 * The target at (b, c, y, x) is the maximum over the counting objects of class c with |x - cx| <= r and |y - cy| <= r of
 * float32(gaussian2D's fp64 value at (x - cx, y - cy)), 0 where none qualifies: draw_umich_gaussian's ct_hm bit for bit.
 * Requirements: B <= 65535, C <= 65535, 0 <= M <= 1024, H*W < 2^31.  Bad arguments (negative sizes, those limits, NULL
 * pointers or stride arrays, negative strides) return PVB_ERR_INVALID, a missing, short or misaligned workspace
 * PVB_ERR_WORKSPACE, both before any CUDA call.  No entry synchronises with the host. */

/* data_utils.draw_umich_gaussian over a batch's objects: ct_hm device fp32 [B,C,H,W] contiguous, fully written.
 * B, C, H or W == 0 is a no-op. */
PVB_API int pvb_ct_target(const int64_t *ct_ind, const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01,
                          float *ct_hm, int32_t B, int32_t M, int32_t C, int32_t H, int32_t W, pvb_stream_t stream);

/* The focal loss of lib/train/trainers/ct.py:20-21 with batch['ct_hm'] = that target, never built:
 *   pred = clamp(sigmoid(logits), 1e-4, 1 - 1e-4);  pos = sum log(pred) (1 - pred)^2 [t == 1];
 *   neg = sum log(1 - pred) pred^2 (1 - t)^4 [t < 1];  loss = -neg if num_pos == 0 else -(pos + neg) / num_pos
 * logits device fp32 [B,C,H,W] at element strides logit_stride (HOST int64[4]).  Each term is CUDA torch's fp32 value;
 * the two sums are fp64, added in a fixed order and rounded once, so the loss is reproducible bit for bit; num_pos is
 * exact.  loss: device fp32 scalar.  workspace: pvb_ct_loss_workspace_bytes(B, C, H, W) bytes of 256-byte aligned device
 * memory; it keeps num_pos for pvb_ct_loss_backward, so pass the same workspace to both. */
PVB_API size_t pvb_ct_loss_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W);
PVB_API int pvb_ct_loss_forward(const float *logits, const int64_t *logit_stride, const int64_t *ct_ind,
                                const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01, float *loss,
                                int32_t B, int32_t M, int32_t C, int32_t H, int32_t W, void *workspace,
                                size_t workspace_bytes, pvb_stream_t stream);
/* autograd's gradient of that loss with respect to the logits, bit for bit: grad_loss is the device fp32 upstream
 * gradient (read on the device, never by the host), grad_logits device fp32 [B,C,H,W] contiguous, fully written.  The
 * workspace is the forward call's, after it.  B, C, H or W == 0 is a no-op. */
PVB_API int pvb_ct_loss_backward(const float *logits, const int64_t *logit_stride, const int64_t *ct_ind,
                                 const int32_t *ct_radius, const int64_t *ct_cls, const float *ct_01,
                                 const float *grad_loss, float *grad_logits, int32_t B, int32_t M, int32_t C, int32_t H,
                                 int32_t W, const void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* ---- the detector's decode: from the output maps to the boxes (DESIGN.md section 8j) --------------------------------
 * Replaces Network.decode_detection (lib/networks/ct/dla.py:20-26): torch.sigmoid, ct_decode.decode_ct_hm
 * (lib/utils/ct/ct_decode.py:6-75) and, with clip = 1, data_utils.clip_to_image (lib/utils/data_utils.py:373-377), for
 * B images.  ct_hm: device fp32 logits [B,C,H,W] at element strides hm_stride (HOST int64[4]); wh: device fp32 [B,2,H,W]
 * at wh_stride.  Per image: heat = sigmoid(logit) in CUDA torch's fp32; a pixel keeps heat where the 3x3 max_pool2d of
 * heat (padding never wins, a NaN in the window wins) equals it and becomes heat * 0 elsewhere; the K largest of the
 * C*H*W values under (value descending, NaN above +inf, class ascending, pixel index ascending) are, in that order,
 *   ct[b][k] = (xs, ys) = (i mod W, i div W);  detection[b][k] = (xs - w/2, ys - h/2, xs + w/2, ys + h/2, value, class)
 * with (w, h) = wh[b, :, ys, xs] and each operation rounded once in fp32; clip = 1 clamps x0, y0 to >= 0, x1 to <= W-1
 * and y1 to <= H-1 (NaN passes).  ct device fp32 [B,K,2] and detection device fp32 [B,K,6], contiguous, fully written.
 * Requirements: 0 <= B <= 65535, 1 <= C <= 65535, H*W < 2^24, 1 <= K <= H*W, C*K < 2^24, C*H*W < 2^31.  workspace:
 * pvb_ct_decode_workspace_bytes(B, C, H, W, K) bytes of 256-byte aligned device memory.  Bad arguments return
 * PVB_ERR_INVALID, a missing, short or misaligned workspace PVB_ERR_WORKSPACE, both before any CUDA call.  The result is
 * bit-identical run to run, an image's result does not depend on the other images, and nothing synchronises with the
 * host.  B == 0 is a no-op. */
PVB_API size_t pvb_ct_decode_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t K);
PVB_API int pvb_ct_decode(const float *ct_hm, const int64_t *hm_stride, const float *wh, const int64_t *wh_stride,
                          int32_t B, int32_t C, int32_t H, int32_t W, int32_t K, int32_t clip, float *ct,
                          float *detection, void *workspace, size_t workspace_bytes, pvb_stream_t stream);

/* ---- the detector: modulated deformable convolution, DCNv2 (DESIGN.md section 8h) -----------------------------------
 * The DLA-34 CenterNet (lib/networks/ct/dla_dcn.py) runs its DCN layers through lib/csrc/dcn_v2, an extension written
 * against THC that does not build on current torch.  Shapes: input [B,C,H,W], offset [B,dg*2*kh*kw,Ho,Wo] ((dy, dx) of
 * tap (i, j) of group g at channels g*2*kh*kw + 2*(i*kw + j) and + 1), mask [B,dg*kh*kw,Ho,Wo], weight [C_out,C,kh,kw],
 * bias [C_out], output [B,C_out,Ho,Wo], Ho = (H + 2*pad_h - (dilation_h*(kh - 1) + 1)) / stride_h + 1 (Wo alike); all
 * device fp32, contiguous.  Channel c belongs to group c / (C / dg).  The sample point of output (ho, wo) at tap (i, j)
 * is h = float(ho*stride_h - pad_h + i*dilation_h) + dy (w alike), used only when h > -1, w > -1, h < H, w < W; its
 * bilinear value over the in-image corners times the mask is the column entry cols[c*kh*kw + i*kw + j][ho*Wo + wo].
 * Requirements: B >= 0 (0 is a no-op), every other size >= 1 (pads >= 0), C % dg == 0, Ho, Wo >= 1, B <= 65535,
 * H*W and Ho*Wo < 2^31, C*kh*kw <= 4194240, C_out <= 4194240, dg*kh*kw <= 65535.  No entry synchronises with the host
 * or allocates.  A malformed descriptor or a NULL tensor returns PVB_ERR_INVALID, a missing, short or misaligned
 * workspace PVB_ERR_WORKSPACE, both before any CUDA call. */
typedef struct pvb_dcn_desc {
    int32_t B, C, H, W, C_out, kh, kw;
    int32_t stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_groups;
} pvb_dcn_desc;

/* Replaces dcn_v2_cuda_forward (lib/csrc/dcn_v2/src/cuda/dcn_v2_cuda.cu:43): output = bias + weight . cols per image in
 * one fused kernel that samples the columns into its operand tiles and never stores them.  The columns are the
 * reference im2col kernel's bit for bit; the product is an fp32 FFMA sum starting from the bias.  The result is
 * bit-identical run to run, and an image's output does not depend on the other images. */
PVB_API int pvb_dcn_forward(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                            const float *weight, const float *bias, float *output, pvb_stream_t stream);

/* The same forward in half precision (DESIGN.md section 8n), for torch.autocast and half models: every tensor is
 * `dtype` (PVB_DCN_F16 = IEEE fp16, PVB_DCN_BF16 = bfloat16), shaped as above except that the weight is tap-major,
 * [C_out][kh][kw][C] (weight.permute(0, 2, 3, 1)), so that a (tap, channel chunk) tile of it is contiguous.  Each
 * column entry is the fp32 forward's, computed from the up-cast inputs and rounded once to `dtype`; output =
 * RN_dtype(bias + weight . cols) with the sum in fp32 on the tensor cores, +-inf where it overflows.  Same descriptor
 * checks, limits and guarantees as pvb_dcn_forward (bit-identical run to run, an image independent of the batch, no
 * host synchronisation, no allocation); an unknown dtype returns PVB_ERR_INVALID before any CUDA call.  There is no
 * half-precision backward: run pvb_dcn_backward on fp32 copies of the operands this call used. */
#define PVB_DCN_F16  1
#define PVB_DCN_BF16 2
PVB_API int pvb_dcn_forward_half(const pvb_dcn_desc *d, int32_t dtype, const void *input, const void *offset,
                                 const void *mask, const void *weight, const void *bias, void *output,
                                 pvb_stream_t stream);

/* Replaces dcn_v2_cuda_forward (dcn_v2_cuda.cu:43) for channels_last models (DESIGN.md section 8o): pvb_dcn_forward_half
 * on NHWC tensors.  input [B][H][W][C], offset [B][Ho][Wo][dg*2*kh*kw], mask [B][Ho][Wo][dg*kh*kw] and output
 * [B][Ho][Wo][C_out] are dense in that order (torch's channels_last layout of the shapes above); weight (tap-major) and
 * bias are as in pvb_dcn_forward_half.  The output's values are pvb_dcn_forward_half's on the same values in NCHW, bit
 * for bit: the columns, the K order, the tensor-core sequence and the split are the same.  When C and C/dg are
 * multiples of 8 and input is 16-byte aligned, each corner's 8 channels arrive in one 16-byte load.  Same checks,
 * refusals (unknown dtype, malformed descriptor, NULL tensor, all before any CUDA call) and guarantees as
 * pvb_dcn_forward_half; B == 0 is a no-op.  The backward is pvb_dcn_backward on NCHW fp32 copies, as for the NCHW call. */
PVB_API int pvb_dcn_forward_half_nhwc(const pvb_dcn_desc *d, int32_t dtype, const void *input, const void *offset,
                                      const void *mask, const void *weight, const void *bias, void *output,
                                      pvb_stream_t stream);

/* Replaces dcn_v2_cuda_backward (dcn_v2_cuda.cu:206) for the whole batch: grad_cols = weight^T . grad_output goes to the
 * workspace `chunk` images at a time (the only column matrix stored); grad_offset / grad_mask (the reference's
 * col2im_coord: grad_mask = sum grad_col * value, grad_offset = sum d(value)/d(h, w) * grad_col * mask, 0 for a point
 * with h <= -1, w <= -1, h >= H or w >= W, the cell [floor h, floor h + 1] at integer h) and grad_input (col2im, float
 * atomics) per chunk; grad_weight = sum over the images of grad_output . cols^T with the columns re-sampled, in split
 * partials added in a fixed order; grad_bias in a fixed order.  All five outputs are fully written (grad_input is
 * zeroed by the call); every one but grad_input is bit-identical run to run.  workspace:
 * pvb_dcn_backward_workspace_bytes(d, chunk) bytes of 256-byte aligned device memory; chunk is clamped to [1, B]. */
PVB_API size_t pvb_dcn_backward_workspace_bytes(const pvb_dcn_desc *d, int32_t chunk);
PVB_API int pvb_dcn_backward(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                             const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                             float *grad_mask, float *grad_weight, float *grad_bias, int32_t chunk, void *workspace,
                             size_t workspace_bytes, pvb_stream_t stream);

/* The fp32 convolution on TF32 tensor cores (DESIGN.md section 8p), what dcn_v2_conv runs for fp32 inputs when torch
 * allows TF32 matmuls.  pvb_dcn_forward_tf32 takes pvb_dcn_forward's tensors except that the weight is tap-major,
 * [C_out][kh][kw][C] (weight.permute(0, 2, 3, 1)), as pvb_dcn_forward_half's; the column entries are pvb_dcn_forward's
 * bit for bit, and output = bias + sum RN_tf32(weight) * RN_tf32(cols) in fp32 on the tensor cores, each operand
 * rounded once (cvt.rna: to nearest, ties away from zero).  pvb_dcn_backward_tf32 takes pvb_dcn_backward's arguments
 * and workspace (pvb_dcn_backward_workspace_bytes: the plan is the same) and runs its kernels, except that grad_cols
 * = RN_tf32(weight)^T . RN_tf32(grad_output) and grad_weight = RN_tf32(grad_output) . RN_tf32(cols)^T run on the
 * tensor cores; grad_bias is pvb_dcn_backward's bit for bit.  Same checks, refusals, limits and guarantees as the
 * fp32 entries: bit-identical run to run (every backward output but grad_input), an image's output independent of the
 * batch, the backward independent of `chunk`, B == 0 a no-op, no host synchronisation, no allocation. */
PVB_API int pvb_dcn_forward_tf32(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                                 const float *weight, const float *bias, float *output, pvb_stream_t stream);
PVB_API int pvb_dcn_backward_tf32(const pvb_dcn_desc *d, const float *input, const float *offset, const float *mask,
                                  const float *weight, const float *grad_output, float *grad_input, float *grad_offset,
                                  float *grad_mask, float *grad_weight, float *grad_bias, int32_t chunk, void *workspace,
                                  size_t workspace_bytes, pvb_stream_t stream);

/* ---- DCNv2's deformable PSROI pooling (DESIGN.md section 8m) -------------------------------------------------------
 * The other half of lib/csrc/dcn_v2 (dcn_v2_psroi_pooling_cuda.cu), behind DCNv2Pooling / DCNPooling.  Shapes: input
 * [B,C,H,W], rois [n_roi,5] = (batch, x1, y1, x2, y2), trans [n_roi, 2*num_classes, part_size, part_size] ((x, y)
 * offsets of class k at channels 2k and 2k + 1; unread with no_trans), out and count [n_roi, C, P, P], P = pooled_size;
 * all device fp32, contiguous.  Output channel c belongs to class c / (C / num_classes).  Bin (ph, pw) of ROI n averages
 * sample_per_part^2 bilinear samples, shifted by trans * trans_std * (ROI width, height) of part cell
 * (floor(ph / P * part_size), floor(pw / P * part_size)); count is the number of samples inside the map.  The rounding
 * is the reference kernel's as its sm_90a build runs it; DESIGN.md 8m tabulates it.
 * Requirements: B, n_roi >= 0, C, H, W, pooled_size, part_size >= 1, output_dim == C, group_size == 1,
 * 1 <= sample_per_part <= 32, num_classes >= 1 dividing C (num_classes is taken as 1 with no_trans),
 * n_roi*C*P^2, B*C*H*W and n_roi*2*num_classes*part_size^2 < 2^31.  A tensor may be NULL only when it is empty or
 * unread.  A bad descriptor or a NULL tensor returns PVB_ERR_INVALID before any CUDA call.
 * Defined where the reference reads out of bounds: a ROI whose batch index (float -> int truncation, NaN -> 0) is
 * outside [0, B) gives output 0, count 0 and no gradient; group_size != 1 and a class count that does not divide C are
 * rejected.  No entry synchronises with the host or allocates; both can be captured in a CUDA graph. */
typedef struct pvb_dcn_pool_desc {
    int32_t B, C, H, W, n_roi, output_dim, pooled_size, part_size, sample_per_part, group_size, num_classes, no_trans;
    float spatial_scale, trans_std;
} pvb_dcn_pool_desc;

/* Replaces dcn_v2_psroi_pooling_cuda_forward (dcn_v2_psroi_pooling_cuda.cu:272): out, and count unless it is NULL,
 * bit-equal to the reference kernel's.  Each CTA computes the sample geometry of its ROI, class and bins once for all
 * the class's channels.  n_roi == 0 is a no-op. */
PVB_API int pvb_dcn_pool_forward(const pvb_dcn_pool_desc *d, const float *input, const float *rois, const float *trans,
                                 float *out, float *count, pvb_stream_t stream);

/* Replaces dcn_v2_psroi_pooling_cuda_backward (dcn_v2_psroi_pooling_cuda.cu:344) and needs no saved count: grad_input
 * [B,C,H,W] is zeroed and then receives each valid sample's bilinear weights times grad_out / count through float
 * atomics, as in the reference; grad_trans (shaped like trans; may be NULL with no_trans) is fully written, each part
 * cell summed in a fixed order, so it is bit-identical run to run and per ROI.  rois get no gradient. */
PVB_API int pvb_dcn_pool_backward(const pvb_dcn_pool_desc *d, const float *input, const float *rois,
                                  const float *trans, const float *grad_out, float *grad_input, float *grad_trans,
                                  pvb_stream_t stream);

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
/* Pass 1's per-box test counts (tooling, DESIGN.md 4.2; process-wide, atomic, results do not depend on it): while
 * dev_counts (device memory, 3 zeroed uint64) is set, pass 1 of the pruned vote adds to it the tests it resolved per box
 * as inliers, all tests it resolved per box, and the tests it scored one hypothesis at a time.  NULL turns it off. */
PVB_API int pvb_set_pass1_stats(void *dev_counts);
/* Grouped launch of the pruned v3 entries (pvb_ransac_voting_v3, _push, pvb_decode_v3; DESIGN.md 4.4): a call whose every
 * group still prunes runs as up to max_groups groups of consecutive images on `streams` internal streams of the calling
 * host thread, joined back into the caller's stream before the entry returns.  0 = the default (2 groups, 2 streams);
 * max_groups = 1 runs every call as one chain on the caller's stream.  Same tooling kind as pvb_set_tuning: process-wide,
 * atomic, and results do not depend on it. */
PVB_API int pvb_set_group_tuning(int32_t max_groups, int32_t streams);
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
