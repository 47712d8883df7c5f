// api.cu -- the C ABI declared in include/pvnet_vote_b200.h.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>
#include <vector>
#include "kernels.h"

using namespace pvb;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int cuda_fail(cudaError_t e, const char *what)
{
    return fail(PVB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// ---- stage timing (pvb_profile_*) --------------------------------------------------------
// stage i runs between boundary events ev[i] and ev[i+1] (5 records per profiled call: every event record is a
// pipeline drain between two kernels, so the profile costs as little as it can and can be sampled)
struct ProfCall {
    cudaEvent_t ev[PVB_STAGE_COUNT + 1];
    bool head;                                                   // first piece of an API call
};
thread_local int g_prof_every = 0;          // 0: off; n: profile every n-th call
thread_local unsigned g_prof_tick = 0;
thread_local std::vector<ProfCall> g_prof_calls;
thread_local std::vector<cudaEvent_t> g_prof_pool;

cudaEvent_t prof_event()
{
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

ProfCall *prof_begin(bool head)
{
    if (g_prof_every <= 0 || (g_prof_tick++ % (unsigned)g_prof_every) != 0) return nullptr;
    ProfCall pc;
    for (auto &e : pc.ev) e = prof_event();
    pc.head = head;
    g_prof_calls.push_back(pc);
    return &g_prof_calls.back();
}

// stage boundaries: prof_start(stage 0) opens the call, prof_end(stage i) closes stage i and opens stage i+1
inline void prof_start(ProfCall *pc, int stage, cudaStream_t st) { if (pc && stage == 0) cudaEventRecord(pc->ev[0], st); }
inline void prof_end(ProfCall *pc, int stage, cudaStream_t st) { if (pc) cudaEventRecord(pc->ev[stage + 1], st); }

int default_capacity(const pvb_desc *d)
{
    const long long HW = (long long)d->H * d->W;
    long long cap = d->capacity;
    if (cap <= 0) {
        const long long mn = d->max_num < 0 ? 0 : d->max_num;
        cap = mn + (long long)ceil(8.0 * sqrt((double)mn)) + 64;
    }
    if (cap > HW) cap = HW;
    cap = (cap + 31) / 32 * 32;
    return (int)cap;
}

int check_desc(const pvb_desc *d)
{
    if (!d) return fail(PVB_ERR_INVALID, "descriptor is NULL");
    if (d->B < 0 || d->H <= 0 || d->W <= 0 || d->K <= 0 || d->hn <= 0)
        return fail(PVB_ERR_INVALID, "bad shape B=%d H=%d W=%d K=%d hn=%d", d->B, d->H, d->W, d->K, d->hn);
    if ((long long)d->H * d->W > (1ll << 30)) return fail(PVB_ERR_INVALID, "image too large (H*W > 2^30)");
    if (d->B > 65535 || d->K > 65535) return fail(PVB_ERR_INVALID, "B and K must be <= 65535");
    if ((long long)d->K * ((d->hn + 511) / 512) > 65535) return fail(PVB_ERR_INVALID, "K*ceil(hn/512) must be <= 65535");
    if (d->mask_dtype < PVB_MASK_U8 || d->mask_dtype > PVB_MASK_F64) return fail(PVB_ERR_INVALID, "bad mask_dtype %d", d->mask_dtype);
    if (d->select_mode != PVB_SELECT_BYTE && d->select_mode != PVB_SELECT_EQ1)
        return fail(PVB_ERR_INVALID, "bad select_mode %d", d->select_mode);
    return PVB_OK;
}

int make_layout(const pvb_desc *d, pvb_layout *L)
{
    const int rc = check_desc(d);
    if (rc) return rc;
    const size_t B = (size_t)d->B, K = (size_t)d->K, hn = (size_t)d->hn;
    const int nwords = (int)(((long long)d->H * d->W + 31) / 32);
    const int nblocks = (nwords + 127) / 128;      // == TS_THREADS of select.cu (one thin_gather CTA per 128 words)
    const int cap = default_capacity(d);
    const int splits = refit_splits_for(cap);
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes); return o; };
    // header: zeroed at the start of every call (everything before `bits`)
    L->status = take(4 * sizeof(int));
    L->fgsum = take(B * sizeof(unsigned long long));
    L->nz = take(B * sizeof(int));
    L->tn = take(B * sizeof(int));
    L->state = take(B * sizeof(int));
    L->refit_ticket = take(B * K * sizeof(int));
    L->ticket = take(B * sizeof(int));
    L->blocktot = take(B * nblocks * sizeof(int));
    L->bits = take(B * nwords * sizeof(uint32_t));
    L->xy = take(B * cap * sizeof(float2));
    L->dirs = take(B * K * cap * sizeof(float2));
    L->hyp = take(B * K * hn * sizeof(float2));
    L->counts = take(B * K * hn * sizeof(int));
    L->win = take(B * K * sizeof(float2));
    L->refit_partial = take(B * K * splits * 5 * sizeof(double));
    const size_t ncells = (size_t)((d->H + PRUNE_CELL - 1) / PRUNE_CELL) * ((d->W + PRUNE_CELL - 1) / PRUNE_CELL);
    L->prune_cells = take(B * K * ncells * PRUNE_REC * sizeof(int));
    L->prune_key = take(B * K * hn * sizeof(int));
    L->prune_list = take(2 * B * K * hn * sizeof(int));
    L->prune_len = take(2 * B * K * sizeof(int));
    // not in pvb_layout (its fields are ABI): the sub-cell records and the pass-2 refinement's bounds follow prune_len
    take(B * K * ncells * 4 * PRUNE_REC * sizeof(int));
    take(B * K * hn * sizeof(int));
    L->total = off;
    L->nwords = nwords;
    L->nblocks = nblocks;
    L->capacity = cap;
    L->refit_splits = splits;
    L->prune_ncells = (int)ncells;
    return PVB_OK;
}

struct Plan {
    pvb_layout L;
    SelectArgs s;
    VoteArgs v;
    float2 *win;
    RefitScratch refit;
    PruneArgs prune;
};

int make_plan(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
              const float *selection, void *ws, size_t ws_bytes, uint32_t tag_idx, uint32_t tag_sel, Plan *P)
{
    int rc = make_layout(d, &P->L);
    if (rc) return rc;
    if (!mask || !vertex) return fail(PVB_ERR_INVALID, "mask/vertex is NULL");
    if (!ws || ws_bytes < P->L.total) return fail(PVB_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", P->L.total, ws_bytes);
    if (reinterpret_cast<uintptr_t>(ws) & 255u) return fail(PVB_ERR_WORKSPACE, "workspace must be 256-byte aligned");
    char *w = static_cast<char *>(ws);
    const pvb_layout &L = P->L;
    SelectArgs &s = P->s;
    s.mask = mask; s.mask_dtype = d->mask_dtype; s.select_mode = d->select_mode;
    s.msb = d->mask_stride[0]; s.msy = d->mask_stride[1]; s.msx = d->mask_stride[2];
    s.vertex = vertex;
    for (int i = 0; i < 5; ++i) s.vs[i] = d->vertex_stride[i];
    s.selection = selection;
    s.B = d->B; s.H = d->H; s.W = d->W; s.K = d->K; s.nwords = L.nwords; s.nblocks = L.nblocks; s.cap = L.capacity;
    s.min_num = d->min_num; s.max_num = d->max_num; s.img_base = d->img_base;
    s.seed = d->seed; s.tag_sel = d->rng_tag_sel ? (uint32_t)d->rng_tag_sel : tag_sel;
    s.rowwise_gather = 0;
    s.seg_classes = 0; s.seg_cs = 0; s.mask_out = nullptr;
    s.bits = reinterpret_cast<uint32_t *>(w + L.bits);
    s.blocktot = reinterpret_cast<unsigned *>(w + L.blocktot);
    s.ticket = reinterpret_cast<int *>(w + L.ticket);
    s.fgsum = reinterpret_cast<unsigned long long *>(w + L.fgsum);
    s.nz = reinterpret_cast<int *>(w + L.nz);
    s.tn = reinterpret_cast<int *>(w + L.tn);
    s.state = reinterpret_cast<int *>(w + L.state);
    s.status = reinterpret_cast<int *>(w + L.status);
    s.xy = reinterpret_cast<float2 *>(w + L.xy);
    s.dirs = reinterpret_cast<float2 *>(w + L.dirs);
    VoteArgs &v = P->v;
    v.B = d->B; v.K = d->K; v.hn = d->hn; v.cap = L.capacity; v.W = d->W; v.H = d->H;
    v.thresh = d->inlier_thresh;
    v.tn = s.tn; v.state = s.state; v.xy = s.xy;
    v.dirs = s.dirs; v.idxs = idxs; v.seed = d->seed;
    v.tag_idx = d->rng_tag_idx ? (uint32_t)d->rng_tag_idx : tag_idx;
    v.img_base = d->img_base;
    v.hyp = reinterpret_cast<float2 *>(w + L.hyp);
    v.counts = reinterpret_cast<int *>(w + L.counts);
    P->win = reinterpret_cast<float2 *>(w + L.win);
    P->refit.partial = reinterpret_cast<double *>(w + L.refit_partial);
    P->refit.ticket = reinterpret_cast<int *>(w + L.refit_ticket);
    P->refit.splits = L.refit_splits;
    P->prune.cells = reinterpret_cast<int *>(w + L.prune_cells);
    P->prune.key = reinterpret_cast<int *>(w + L.prune_key);
    P->prune.list = reinterpret_cast<int *>(w + L.prune_list);
    P->prune.len = reinterpret_cast<int *>(w + L.prune_len);
    const size_t BK = (size_t)d->B * d->K;
    const size_t prune_sub = align_up(L.prune_len + 2 * BK * sizeof(int));
    P->prune.sub = reinterpret_cast<int *>(w + prune_sub);
    P->prune.b2 = reinterpret_cast<int *>(w + align_up(prune_sub + BK * L.prune_ncells * 4 * PRUNE_REC * sizeof(int)));
    P->prune.ticket = P->refit.ticket;               // the bound step leaves it at 0 for the refit
    P->prune.ncx = (d->W + PRUNE_CELL - 1) / PRUNE_CELL;
    P->prune.ncells = L.prune_ncells;
    P->prune.cos_w = P->prune.sin_w = 0.f;
    return PVB_OK;
}

// the vote stage after launch_generate: v3 callers that read no counts (`prune`) score only the hypotheses that can win
cudaError_t run_vote(const Plan &P, bool prune, cudaStream_t st)
{
    PruneArgs q = P.prune;
    if (prune && prune_setup(P.v, q)) return launch_vote_pruned(P.v, q, st);
    // the unpruned vote is launched plainly: chained after generate it measured slower where its grid is a single partial
    // wave (H100, B = 1, K = 17, 720x540: 0.163 against 0.127 ms per call), and no faster at B = 1, K = 9 (DESIGN.md 4.3)
    return launch_vote(P.v, false, false, st);
}

int run_select(const Plan &P, cudaStream_t st)
{
    // status, fgsum, nz, tn, state, refit tickets, thin_gather tickets, block totals: contiguous at the start of the workspace
    cudaError_t e = cudaMemsetAsync(P.s.status, 0, P.L.bits, st);
    if (e != cudaSuccess) return cuda_fail(e, "memset(header)");
    e = launch_select(P.s, st);
    if (e != cudaSuccess) return cuda_fail(e, "select kernels");
    return PVB_OK;
}

int run_front(const Plan &P, bool prune, cudaStream_t st, ProfCall *pc)
{
    prof_start(pc, PVB_STAGE_SELECT, st);
    int rc = run_select(P, st);
    if (rc) return rc;
    prof_end(pc, PVB_STAGE_SELECT, st);
    prof_start(pc, PVB_STAGE_GENERATE, st);
    cudaError_t e = launch_generate(P.v, true, st);     // chained after thin_gather, which exits as its trigger (common.cuh)
    if (e != cudaSuccess) return cuda_fail(e, "generate kernel");
    prof_end(pc, PVB_STAGE_GENERATE, st);
    prof_start(pc, PVB_STAGE_VOTE, st);
    e = run_vote(P, prune, st);
    if (e != cudaSuccess) return cuda_fail(e, "vote kernel");
    prof_end(pc, PVB_STAGE_VOTE, st);
    return PVB_OK;
}

// ---- multi-GPU exchange object (exchange.cu holds the kernels and the design notes) ------------------------------
} // namespace

struct pvb_exchange {
    int rank, world, slots, device;
    size_t bytes_per_rank;      // payload bytes per rank and call (a multiple of 16); the ring holds 2x (8-byte words)
    size_t status_off, total;
    char *local;                // this rank's ring (cudaMalloc)
    char *peer[PVB_MAX_PEERS];  // every rank's ring as seen from this device (peer[rank] == local)
    bool ipc_opened[PVB_MAX_PEERS];
    bool connected;
};

namespace {

int exchange_push_args(pvb_exchange *ex, uint64_t seq, size_t nbytes, PeerPush *pp)
{
    memset(pp, 0, sizeof(*pp));
    if (!ex) return PVB_OK;
    if (!ex->connected) return fail(PVB_ERR_INVALID, "exchange is not connected (pvb_exchange_connect*)");
    if (seq == 0 || (uint32_t)seq == 0) return fail(PVB_ERR_INVALID, "seq must be >= 1 and not a multiple of 2^32");
    if (nbytes > ex->bytes_per_rank) return fail(PVB_ERR_INVALID, "result block (%zu bytes) exceeds the exchange's bytes_per_rank (%zu)", nbytes, ex->bytes_per_rank);
    const size_t slot = (size_t)((seq - 1) % (uint64_t)ex->slots);
    const size_t words = ex->bytes_per_rank / sizeof(float);             // 8-byte words per rank and slot
    pp->world = ex->world;
    pp->seq = (uint32_t)seq;
    for (int r = 0; r < ex->world; ++r)
        pp->recv[r] = reinterpret_cast<uint2 *>(ex->peer[r]) + (slot * ex->world + ex->rank) * words;
    return PVB_OK;
}

size_t mask_elt_bytes(int dt)
{
    switch (dt) {
    case PVB_MASK_U8: case PVB_MASK_I8: return 1;
    case PVB_MASK_I16: return 2;
    case PVB_MASK_I32: case PVB_MASK_F32: return 4;
    default: return 8;
    }
}

} // namespace

extern "C" {

PVB_API int pvb_version(void) { return PVB_VERSION; }
PVB_API const char *pvb_last_error(void) { return g_err; }

PVB_API size_t pvb_workspace_bytes(const pvb_desc *d)
{
    pvb_layout L;
    if (make_layout(d, &L)) return 0;
    return L.total;
}

PVB_API int pvb_workspace_layout(const pvb_desc *d, pvb_layout *out)
{
    if (!out) return fail(PVB_ERR_INVALID, "out is NULL");
    return make_layout(d, out);
}

static int run_v3(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs, const float *selection,
                  float *out_kpt, void *workspace, size_t workspace_bytes, const float *seg, int32_t classes,
                  int64_t class_stride, int64_t *mask_out, pvb_exchange *ex, uint64_t seq, bool prune, cudaStream_t st)
{
    Plan P;
    int rc = make_plan(d, seg ? static_cast<const void *>(seg) : mask, vertex, idxs, selection, workspace, workspace_bytes, 1u, 2u, &P);
    if (rc) return rc;
    if (!out_kpt) return fail(PVB_ERR_INVALID, "out_kpt is NULL");
    PeerPush pp;
    rc = exchange_push_args(ex, seq, (size_t)d->B * d->K * 2 * sizeof(float), &pp);
    if (rc) return rc;
    if (d->B == 0) {
        if (pp.world > 0) return fail(PVB_ERR_INVALID, "an exchanging call needs B >= 1 on every rank");
        return PVB_OK;
    }
    if (seg) {
        P.s.seg_classes = classes;
        P.s.seg_cs = class_stride;
        P.s.mask_out = reinterpret_cast<long long *>(mask_out);
    }
    ProfCall *pc = prof_begin(true);
    rc = run_front(P, prune, st, pc);
    if (rc) return rc;
    prof_start(pc, PVB_STAGE_FINISH, st);
    cudaError_t e = launch_refit(P.v, P.win, P.refit, out_kpt, pp, st);
    if (e != cudaSuccess) return cuda_fail(e, "refit kernel");
    prof_end(pc, PVB_STAGE_FINISH, st);
    return PVB_OK;
}

PVB_API int pvb_ransac_voting_v3(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
                         const float *selection, float *out_kpt, void *workspace, size_t workspace_bytes,
                         pvb_stream_t stream)
{
    return run_v3(d, mask, vertex, idxs, selection, out_kpt, workspace, workspace_bytes, nullptr, 0, 0, nullptr, nullptr, 0,
                  true, static_cast<cudaStream_t>(stream));
}

PVB_API int pvb_ransac_voting_v3_all_counts(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
                                            const float *selection, float *out_kpt, void *workspace, size_t workspace_bytes,
                                            pvb_exchange *exchange, uint64_t seq, pvb_stream_t stream)
{
    return run_v3(d, mask, vertex, idxs, selection, out_kpt, workspace, workspace_bytes, nullptr, 0, 0, nullptr, exchange, seq,
                  false, static_cast<cudaStream_t>(stream));
}

PVB_API int pvb_ransac_voting_v3_push(const pvb_desc *d, const void *mask, const float *vertex, const int32_t *idxs,
                                      const float *selection, float *out_kpt, void *workspace, size_t workspace_bytes,
                                      pvb_exchange *exchange, uint64_t seq, pvb_stream_t stream)
{
    if (!exchange) return fail(PVB_ERR_INVALID, "exchange is NULL");
    return run_v3(d, mask, vertex, idxs, selection, out_kpt, workspace, workspace_bytes, nullptr, 0, 0, nullptr, exchange, seq,
                  true, static_cast<cudaStream_t>(stream));
}

PVB_API int pvb_decode_v3(const pvb_desc *d, const float *seg, int32_t classes, int64_t class_stride, int64_t *mask_out,
                          const float *vertex, const int32_t *idxs, const float *selection, float *out_kpt,
                          void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    if (classes < 1 || classes > 4096) return fail(PVB_ERR_INVALID, "classes must be in [1,4096]");
    if (!seg) return fail(PVB_ERR_INVALID, "seg is NULL");
    return run_v3(d, nullptr, vertex, idxs, selection, out_kpt, workspace, workspace_bytes, seg, classes, class_stride, mask_out,
                  nullptr, 0, true, static_cast<cudaStream_t>(stream));
}

static int run_distribution(const pvb_desc *d, const void *mask, const float *vertex, const float *mean, const int32_t *idxs,
                            const float *selection, float *out_cov, void *workspace, size_t workspace_bytes, pvb_exchange *ex,
                            uint64_t seq, cudaStream_t st)
{
    Plan P;
    int rc = make_plan(d, mask, vertex, idxs, selection, workspace, workspace_bytes, 3u, 4u, &P);
    if (rc) return rc;
    if (!mean || !out_cov) return fail(PVB_ERR_INVALID, "mean/out_cov is NULL");
    PeerPush pp;
    rc = exchange_push_args(ex, seq, (size_t)d->B * d->K * 4 * sizeof(float), &pp);
    if (rc) return rc;
    if (d->B == 0) {
        if (pp.world > 0) return fail(PVB_ERR_INVALID, "an exchanging call needs B >= 1 on every rank");
        return PVB_OK;
    }
    ProfCall *pc = prof_begin(true);
    rc = run_front(P, false, st, pc);
    if (rc) return rc;
    prof_start(pc, PVB_STAGE_FINISH, st);
    cudaError_t e = launch_covariance(P.v, mean, out_cov, pp, st);
    if (e != cudaSuccess) return cuda_fail(e, "covariance kernel");
    prof_end(pc, PVB_STAGE_FINISH, st);
    return PVB_OK;
}

PVB_API int pvb_estimate_voting_distribution(const pvb_desc *d, const void *mask, const float *vertex, const float *mean,
                                     const int32_t *idxs, const float *selection, float *out_cov, void *workspace,
                                     size_t workspace_bytes, pvb_stream_t stream)
{
    return run_distribution(d, mask, vertex, mean, idxs, selection, out_cov, workspace, workspace_bytes, nullptr, 0,
                            static_cast<cudaStream_t>(stream));
}

PVB_API int pvb_estimate_voting_distribution_push(const pvb_desc *d, const void *mask, const float *vertex, const float *mean,
                                                  const int32_t *idxs, const float *selection, float *out_cov, void *workspace,
                                                  size_t workspace_bytes, pvb_exchange *exchange, uint64_t seq,
                                                  pvb_stream_t stream)
{
    if (!exchange) return fail(PVB_ERR_INVALID, "exchange is NULL");
    return run_distribution(d, mask, vertex, mean, idxs, selection, out_cov, workspace, workspace_bytes, exchange, seq,
                            static_cast<cudaStream_t>(stream));
}

PVB_API int pvb_uncertainty_weights(const float *cov, float *weights, int32_t n, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (n && (!cov || !weights)) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (reinterpret_cast<uintptr_t>(cov) & 15u) return fail(PVB_ERR_INVALID, "cov must be 16-byte aligned");
    cudaError_t e = launch_pnp_weights(cov, weights, n, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "pnp weights kernel");
}

namespace {

// The checks every PnP entry point makes after its own ones on n and pn: NULL tensors (`given`: every required pointer is
// set), then the strides.
int pnp_check_inputs(int32_t n, bool given, int64_t pts3d_stride, int64_t k_stride)
{
    if (n && !given) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (pts3d_stride < 0 || k_stride < 0) return fail(PVB_ERR_INVALID, "negative stride");
    return PVB_OK;
}

// options == NULL: Ceres' defaults
int pnp_read_options(const pvb_pnp_options *options, PnpOptions &opt)
{
    opt = pnp_default_options();
    if (!options) return PVB_OK;
    if (options->max_num_iterations < 0 || !(options->function_tolerance >= 0.0) || !(options->gradient_tolerance >= 0.0) ||
        !(options->parameter_tolerance >= 0.0))
        return fail(PVB_ERR_INVALID, "pvb_pnp_options: negative or NaN entry");
    opt.max_num_iterations = options->max_num_iterations; opt.function_tolerance = options->function_tolerance;
    opt.gradient_tolerance = options->gradient_tolerance; opt.parameter_tolerance = options->parameter_tolerance;
    return PVB_OK;
}

} // namespace

PVB_API int pvb_uncertainty_pnp(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                const double *init_rt, double *result_rt, int32_t *info, int32_t n, int32_t pn,
                                int64_t pts3d_stride, int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1) return fail(PVB_ERR_INVALID, "pn must be >= 1 (got %d)", pn);
    PnpArgs a = {};
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && wgt2d && K && init_rt && result_rt, pts3d_stride, k_stride)) return rc;
    if (int rc = pnp_read_options(options, a.opt)) return rc;
    a.pts2d = pts2d; a.wgt2d = wgt2d; a.pts3d = pts3d; a.K = K; a.init_rt = init_rt; a.result_rt = result_rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    cudaError_t e = launch_pnp_batch(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "uncertainty pnp kernel");
}

PVB_API int pvb_uncertainty_pnp_from_votes(const float *kpt_2d, const float *cov, const float *weights, const double *pts3d,
                                           const double *K, const double *init_rt, double *result_rt, double *init_out,
                                           float *weights_out, int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride,
                                           int64_t k_stride, const pvb_pnp_options *options, pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1 || pn > PNP_FUSED_MAX_PN) return fail(PVB_ERR_INVALID, "pn must be in [1,%d] (got %d)", PNP_FUSED_MAX_PN, pn);
    if (!init_rt && pn < 4) return fail(PVB_ERR_INVALID, "the P3P initialisation needs pn >= 4 (got %d)", pn);
    const bool given = kpt_2d && pts3d && K && result_rt;
    // before pnp_check_inputs, but only once every required tensor is set: a caller keeps getting "NULL tensor" first,
    // then this, then "negative stride"
    if (n && given && ((cov == nullptr) == (weights == nullptr)))
        return fail(PVB_ERR_INVALID, "pass exactly one of cov / weights");
    PnpArgs a = {};
    if (int rc = pnp_check_inputs(n, given, pts3d_stride, k_stride)) return rc;
    if ((reinterpret_cast<uintptr_t>(kpt_2d) & 7u) || (reinterpret_cast<uintptr_t>(cov) & 15u))
        return fail(PVB_ERR_INVALID, "kpt_2d must be 8-byte and cov 16-byte aligned");
    if (int rc = pnp_read_options(options, a.opt)) return rc;
    a.kpt2d = kpt_2d; a.cov = cov; a.weights = weights; a.weights_out = weights_out; a.pts3d = pts3d; a.K = K;
    a.init_rt = init_rt; a.init_out = init_out; a.result_rt = result_rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    cudaError_t e = launch_pnp_batch(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "fused uncertainty pnp kernel");
}

PVB_API int pvb_uncertainty_pnp_init(const double *pts2d, const double *pts3d, const double *wgt2d, const double *K,
                                     double *init_rt, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                                     pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 4) return fail(PVB_ERR_INVALID, "P3P needs pn >= 4 (got %d)", pn);
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && wgt2d && K && init_rt, pts3d_stride, k_stride)) return rc;
    PnpArgs a = {};                    // no result_rt: the P3P start alone, written to init_out
    a.pts2d = pts2d; a.wgt2d = wgt2d; a.pts3d = pts3d; a.K = K; a.init_out = init_rt;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    cudaError_t e = launch_pnp_batch(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "p3p init kernel");
}

PVB_API int pvb_pnp_iterative(const double *pts2d, const double *pts3d, const double *K, double *pose, double *rt,
                              int32_t *info, int32_t n, int32_t pn, int64_t pts3d_stride, int64_t k_stride,
                              pvb_stream_t stream)
{
    if (n < 0) return fail(PVB_ERR_INVALID, "n < 0");
    if (pn < 1) return fail(PVB_ERR_INVALID, "pn must be >= 1 (got %d)", pn);
    if (int rc = pnp_check_inputs(n, pts2d && pts3d && K && pose, pts3d_stride, k_stride)) return rc;
    PnpArgs a = {};
    a.pts2d = pts2d; a.pts3d = pts3d; a.K = K; a.pose = pose; a.result_rt = rt; a.info = info;
    a.n = n; a.pn = pn; a.pts3d_stride = pts3d_stride; a.k_stride = k_stride;
    cudaError_t e = launch_pnp_iterative(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "iterative pnp kernel");
}

namespace {

// the workspace checks of the nearest-neighbour entries; `need` may be 0 (then NULL is fine)
int nn_check_workspace(size_t need, const void *workspace, size_t workspace_bytes)
{
    if (!need) return PVB_OK;
    if (!workspace || workspace_bytes < need)
        return fail(PVB_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace ? workspace_bytes : 0);
    if (reinterpret_cast<uintptr_t>(workspace) & 255u) return fail(PVB_ERR_WORKSPACE, "workspace must be 256-byte aligned");
    return PVB_OK;
}

// CTAs of the widest launch; the grid is one-dimensional
bool nn_grid_fits(int b, int pn1, int pn2)
{
    const NnPlan p = nn_plan(b, pn1, pn2);
    return (long long)b * p.nsplit * p.qchunks <= 0x7fffffffll;
}

} // namespace

PVB_API size_t pvb_nearest_point_workspace_bytes(int32_t b, int32_t pn1, int32_t pn2)
{
    if (b <= 0 || pn1 < 0 || pn2 <= 0) return 0;
    return nn_workspace_bytes(b, pn1, pn2);
}

PVB_API int pvb_nearest_point_idx(const float *ref, const float *que, int32_t *idxs, int32_t b, int32_t pn1, int32_t pn2,
                                  int32_t dim, int32_t exclude_self, void *workspace, size_t workspace_bytes,
                                  pvb_stream_t stream)
{
    if (b < 0 || pn1 < 0 || pn2 < 0) return fail(PVB_ERR_INVALID, "negative size (b=%d pn1=%d pn2=%d)", b, pn1, pn2);
    if (dim != 2 && dim != 3) return fail(PVB_ERR_INVALID, "dim must be 2 or 3 (got %d)", dim);
    if (b == 0 || pn2 == 0) return PVB_OK;
    if (!que || !idxs || (pn1 > 0 && !ref)) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (!nn_grid_fits(b, pn1, pn2)) return fail(PVB_ERR_INVALID, "b * pn2 too large");
    if (int rc = nn_check_workspace(nn_workspace_bytes(b, pn1, pn2), workspace, workspace_bytes)) return rc;
    cudaError_t e = launch_nearest_point(ref, que, idxs, b, pn1, pn2, dim, exclude_self != 0, workspace,
                                         static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "nearest point kernels");
}

PVB_API size_t pvb_add_metric_workspace_bytes(int32_t n, int32_t pn, int32_t syn)
{
    if (n <= 0 || pn < 0 || (syn != 0 && syn != 1)) return 0;
    return add_metric_workspace_bytes(n, pn, syn, nullptr);
}

PVB_API int pvb_add_metric(const double *model, const double *pose_pred, const double *pose_gt, double *mean_dist, int32_t n,
                           int32_t pn, int32_t syn, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    if (n < 0 || pn < 0) return fail(PVB_ERR_INVALID, "negative size (n=%d pn=%d)", n, pn);
    if (syn != 0 && syn != 1) return fail(PVB_ERR_INVALID, "syn must be 0 or 1 (got %d)", syn);
    if (n == 0) return PVB_OK;
    if (!pose_pred || !pose_gt || !mean_dist || (pn > 0 && !model)) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (!nn_grid_fits(n, pn, pn)) return fail(PVB_ERR_INVALID, "n * pn too large");
    if (int rc = nn_check_workspace(add_metric_workspace_bytes(n, pn, syn, nullptr), workspace, workspace_bytes)) return rc;
    cudaError_t e = launch_add_metric(model, pose_pred, pose_gt, mean_dist, n, pn, syn != 0, workspace,
                                      static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "add metric kernels");
}

PVB_API size_t pvb_pose_metrics_workspace_bytes(int32_t n, int32_t pn)
{
    if (n <= 0 || pn < 0) return 0;
    return pose_metrics_workspace_bytes(n, pn);
}

PVB_API int pvb_pose_metrics(const double *model, const double *pose_pred, const double *pose_gt, const double *K,
                             int64_t k_stride, double *proj2d, double *trans_cm, double *angle_deg, int32_t n, int32_t pn,
                             void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    if (n < 0 || pn < 0) return fail(PVB_ERR_INVALID, "negative size (n=%d pn=%d)", n, pn);
    if (n == 0) return PVB_OK;
    if (!pose_pred || !pose_gt || !K || !proj2d || !trans_cm || !angle_deg || (pn > 0 && !model))
        return fail(PVB_ERR_INVALID, "NULL tensor");
    if (k_stride < 0) return fail(PVB_ERR_INVALID, "negative stride");
    if (!nn_grid_fits(n, pn, pn)) return fail(PVB_ERR_INVALID, "n * pn too large");
    if (int rc = nn_check_workspace(pose_metrics_workspace_bytes(n, pn), workspace, workspace_bytes)) return rc;
    cudaError_t e = launch_pose_metrics(model, pose_pred, pose_gt, K, k_stride, proj2d, trans_cm, angle_deg, n, pn, workspace,
                                        static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "pose metric kernels");
}

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
    cudaError_t e = launch_mask_iou(pred, pred_dtype, ps, gt, gt_dtype, gs, reinterpret_cast<long long *>(inter),
                                    reinterpret_cast<long long *>(uni), B, H, W, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "mask iou kernel");
}

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
        if (int rc = nn_check_workspace(render_workspace_bytes(n, F), workspace, workspace_bytes)) return rc;
    cudaError_t e = launch_render_depth(pts, V, faces, F, poses, n, K, k_stride, depth, H, W, clip_near, clip_far, workspace,
                                        static_cast<cudaStream_t>(stream));
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
    if (int rc = nn_check_workspace(vsd_workspace_bytes(n), workspace, workspace_bytes)) return rc;
    VsdArgs a;
    a.depth_test = depth_test; a.depth_est = depth_est; a.depth_gt = depth_gt; a.pairs = pairs; a.K = K;
    a.k_stride = k_stride; a.n = n; a.B = B; a.n_est = n_est; a.n_gt = n_gt; a.est_base = est_base; a.gt_base = gt_base;
    a.H = H; a.W = W; a.delta = delta; a.tau = tau; a.e = e;
    cudaError_t err = launch_vsd(a, workspace, static_cast<cudaStream_t>(stream));
    return err == cudaSuccess ? PVB_OK : cuda_fail(err, "vsd kernels");
}

namespace {

constexpr int VOTE_LOSS_MAX_K = 1024;      // the image's keypoints live in 16 KB of shared memory

// the arguments every vote-loss entry shares; fills the mask, keypoint and size fields of `a`
int vote_loss_common(VoteLossArgs &a, const void *mask, int32_t mask_dtype, const int64_t *mask_stride, const double *kpt_2d,
                     int32_t B, int32_t H, int32_t W, int32_t K)
{
    if (B < 0 || H < 0 || W < 0) return fail(PVB_ERR_INVALID, "negative size (B=%d H=%d W=%d)", B, H, W);
    if (K < 1 || K > VOTE_LOSS_MAX_K) return fail(PVB_ERR_INVALID, "K must be in [1, %d], got %d", VOTE_LOSS_MAX_K, K);
    if (B > 65535) return fail(PVB_ERR_INVALID, "B must be at most 65535, got %d", B);
    if ((long long)H * W > 0x7fffffffll) return fail(PVB_ERR_INVALID, "image too large (H*W >= 2^31)");
    if (mask_dtype < PVB_MASK_U8 || mask_dtype > PVB_MASK_I64)
        return fail(PVB_ERR_INVALID, "mask dtype must be an integer pvb_mask_dtype (U8..I64), got %d", mask_dtype);
    if (!mask_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    for (int i = 0; i < 3; ++i)
        if (mask_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
    if ((long long)B * H * W > 0 && (!mask || !kpt_2d)) return fail(PVB_ERR_INVALID, "NULL tensor");
    a = VoteLossArgs{};
    a.mask = mask; a.mask_dtype = mask_dtype;
    a.msb = mask_stride[0]; a.msy = mask_stride[1]; a.msx = mask_stride[2];
    a.kpt = kpt_2d;
    a.B = B; a.H = H; a.W = W; a.K = K;
    return PVB_OK;
}

int vote_loss_pred(VoteLossArgs &a, const float *pred, const int64_t *pred_stride)
{
    if (!pred_stride) return fail(PVB_ERR_INVALID, "NULL stride array");
    for (int i = 0; i < 4; ++i) {
        if (pred_stride[i] < 0) return fail(PVB_ERR_INVALID, "negative stride");
        a.ps[i] = pred_stride[i];
    }
    if ((long long)a.B * a.H * a.W > 0 && !pred) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.pred = pred;
    return PVB_OK;
}

// fills the workspace fields of `a` from a checked workspace
int vote_loss_workspace(VoteLossArgs &a, const void *workspace, size_t workspace_bytes)
{
    size_t po = 0, wo = 0;
    const size_t need = vote_loss_workspace_bytes(a.B, a.H, a.W, &po, &wo);
    if (!workspace || workspace_bytes < need)
        return fail(PVB_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace ? workspace_bytes : 0);
    if (reinterpret_cast<uintptr_t>(workspace) & 255u) return fail(PVB_ERR_WORKSPACE, "workspace must be 256-byte aligned");
    char *ws = static_cast<char *>(const_cast<void *>(workspace));
    a.wsum = reinterpret_cast<float *>(ws);
    a.partial = reinterpret_cast<double *>(ws + po);
    a.wpart = reinterpret_cast<long long *>(ws + wo);
    return PVB_OK;
}

} // namespace

// pvnet_data_utils.py:30-44 compute_vertex
PVB_API int pvb_vote_target(const void *mask, int32_t mask_dtype, const int64_t *mask_stride, const double *kpt_2d,
                            float *vertex, int32_t B, int32_t H, int32_t W, int32_t K, pvb_stream_t stream)
{
    VoteLossArgs a;
    if (int rc = vote_loss_common(a, mask, mask_dtype, mask_stride, kpt_2d, B, H, W, K)) return rc;
    if ((long long)B * H * W > 0 && !vertex) return fail(PVB_ERR_INVALID, "NULL tensor");
    a.out = vertex;
    cudaError_t e = launch_vote_target(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "vote target kernel");
}

PVB_API size_t pvb_vote_loss_workspace_bytes(int32_t B, int32_t H, int32_t W)
{
    if (B < 0 || H < 0 || W < 0) return 0;
    return vote_loss_workspace_bytes(B, H, W, nullptr, nullptr);
}

// lib/train/trainers/pvnet.py:25-27, the forward pass
PVB_API int pvb_vote_loss_forward(const float *pred, const int64_t *pred_stride, const void *mask, int32_t mask_dtype,
                                  const int64_t *mask_stride, const double *kpt_2d, float *loss, int32_t B, int32_t H,
                                  int32_t W, int32_t K, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    VoteLossArgs a;
    if (int rc = vote_loss_common(a, mask, mask_dtype, mask_stride, kpt_2d, B, H, W, K)) return rc;
    if (int rc = vote_loss_pred(a, pred, pred_stride)) return rc;
    if (!loss) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (int rc = vote_loss_workspace(a, workspace, workspace_bytes)) return rc;
    a.loss = loss;
    cudaError_t e = launch_vote_loss_forward(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "vote loss forward kernels");
}

// lib/train/trainers/pvnet.py:25-27, autograd's backward pass of it
PVB_API int pvb_vote_loss_backward(const float *pred, const int64_t *pred_stride, const void *mask, int32_t mask_dtype,
                                   const int64_t *mask_stride, const double *kpt_2d, const float *grad_loss,
                                   float *grad_pred, int32_t B, int32_t H, int32_t W, int32_t K, const void *workspace,
                                   size_t workspace_bytes, pvb_stream_t stream)
{
    VoteLossArgs a;
    if (int rc = vote_loss_common(a, mask, mask_dtype, mask_stride, kpt_2d, B, H, W, K)) return rc;
    if (int rc = vote_loss_pred(a, pred, pred_stride)) return rc;
    if ((long long)B * H * W == 0) return PVB_OK;
    if (!grad_loss || !grad_pred) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (int rc = vote_loss_workspace(a, workspace, workspace_bytes)) return rc;
    a.grad_loss = grad_loss;
    a.out = grad_pred;
    cudaError_t e = launch_vote_loss_backward(a, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "vote loss backward kernel");
}

PVB_API int pvb_read_status(const pvb_desc *d, const void *workspace, pvb_stream_t stream)
{
    pvb_layout L;
    int rc = make_layout(d, &L);
    if (rc) return rc;
    if (!workspace) return fail(PVB_ERR_INVALID, "workspace is NULL");
    int host[4] = {0, 0, 0, 0};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemcpyAsync(host, static_cast<const char *>(workspace) + L.status, sizeof(host), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(e, "read status");
    if (host[0] == PVB_ERR_CAPACITY)
        return fail(PVB_ERR_CAPACITY, "image %d selected more than capacity=%d pixels; pass capacity=H*W", host[1], L.capacity);
    if (host[0]) return fail(host[0], "device status %d", host[0]);
    return PVB_OK;
}

// ---- host-buffer pipeline ---------------------------------------------------------------
struct HostSlot { size_t mask, vertex, out, ws, end; };

static int host_slot_layout(const pvb_desc *d, int chunk, HostSlot *S, pvb_desc *dc)
{
    if (chunk <= 0) return fail(PVB_ERR_INVALID, "chunk_images must be > 0");
    *dc = *d;
    dc->B = chunk;
    const size_t HW = (size_t)d->H * d->W;
    dc->mask_stride[0] = (int64_t)HW; dc->mask_stride[1] = d->W; dc->mask_stride[2] = 1;
    dc->vertex_stride[0] = (int64_t)(HW * d->K * 2); dc->vertex_stride[1] = (int64_t)d->W * d->K * 2;
    dc->vertex_stride[2] = (int64_t)d->K * 2; dc->vertex_stride[3] = 2; dc->vertex_stride[4] = 1;
    pvb_layout L;
    int rc = make_layout(dc, &L);
    if (rc) return rc;
    size_t off = 0;
    S->mask = off; off = align_up(off + (size_t)chunk * HW * mask_elt_bytes(d->mask_dtype));
    S->vertex = off; off = align_up(off + (size_t)chunk * HW * d->K * 2 * sizeof(float));
    S->out = off; off = align_up(off + (size_t)chunk * d->K * 2 * sizeof(float));
    S->ws = off; off = align_up(off + L.total);
    S->end = off;
    return PVB_OK;
}

constexpr int HOST_SLOTS = 4;     // pieces in flight: the mask DMA runs up to HOST_SLOTS-1 pieces ahead of the compute

PVB_API size_t pvb_host_scratch_bytes(const pvb_desc *d, int32_t chunk_images)
{
    HostSlot S; pvb_desc dc;
    if (check_desc(d) || host_slot_layout(d, chunk_images, &S, &dc)) return 0;
    return HOST_SLOTS * S.end;
}

namespace {
// streams and events of the host pipeline: one set per (host thread, device), created on first use and kept
struct HostPipe {
    cudaStream_t copy = nullptr, in = nullptr, cmp = nullptr;
    cudaEvent_t user = nullptr, end = nullptr, dma[HOST_SLOTS] = {}, sel[HOST_SLOTS] = {}, done[HOST_SLOTS] = {};
    bool ready = false;
};
constexpr int MAX_DEVICES = 64;

int host_pipe(int dev, HostPipe **out)
{
    static thread_local HostPipe pipes[MAX_DEVICES];
    if (dev < 0 || dev >= MAX_DEVICES) return fail(PVB_ERR_CUDA, "device index %d out of range", dev);
    HostPipe &p = pipes[dev];
    if (!p.ready) {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);   // lo = least, hi = greatest priority (numerically lower)
        cudaError_t e = cudaStreamCreateWithPriority(&p.copy, cudaStreamNonBlocking, hi);
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&p.in, cudaStreamNonBlocking, hi);
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&p.cmp, cudaStreamNonBlocking, lo);
        if (e != cudaSuccess) return cuda_fail(e, "cudaStreamCreate");
        cudaEvent_t *single[] = {&p.user, &p.end};
        for (cudaEvent_t *pe : single)
            if ((e = cudaEventCreateWithFlags(pe, cudaEventDisableTiming)) != cudaSuccess) return cuda_fail(e, "cudaEventCreate");
        for (int i = 0; i < HOST_SLOTS; ++i) {
            e = cudaEventCreateWithFlags(&p.dma[i], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p.sel[i], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p.done[i], cudaEventDisableTiming);
            if (e != cudaSuccess) return cuda_fail(e, "cudaEventCreate");
        }
        p.ready = true;
    }
    *out = &p;
    return PVB_OK;
}

// device-visible alias of a pinned host pointer, or NULL when `p` is not mapped host memory
const void *mapped_alias(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (a.type != cudaMemoryTypeHost || !a.devicePointer) return nullptr;
    return a.devicePointer;
}
} // namespace

PVB_API int pvb_ransac_voting_v3_host(const pvb_desc *d, const void *mask_host, const float *vertex_host,
                              float *out_kpt_host, int32_t chunk_images, uint32_t flags, void *dev_scratch,
                              size_t dev_scratch_bytes, pvb_stream_t stream)
{
    int rc = check_desc(d);
    if (rc) return rc;
    if (!mask_host || !vertex_host || !out_kpt_host) return fail(PVB_ERR_INVALID, "host buffer is NULL");
    if (flags & ~(uint32_t)(PVB_HOST_INPLACE_MASK | PVB_HOST_STAGE_VERTEX)) return fail(PVB_ERR_INVALID, "unknown flags 0x%x", flags);
    HostSlot S; pvb_desc dc;
    rc = host_slot_layout(d, chunk_images, &S, &dc);
    if (rc) return rc;
    if (!dev_scratch || dev_scratch_bytes < HOST_SLOTS * S.end) return fail(PVB_ERR_WORKSPACE, "device scratch too small: need %zu", HOST_SLOTS * S.end);
    if (reinterpret_cast<uintptr_t>(dev_scratch) & 255u) return fail(PVB_ERR_WORKSPACE, "device scratch must be 256-byte aligned");
    // Software pipeline over `chunk_images`-sized pieces, HOST_SLOTS of them in flight, on three streams:
    //   copy (high priority): cudaMemcpyAsync of whatever is STAGED (by default the mask: one contiguous DMA per piece at the
    //                         copy engine's PCIe rate); runs ahead of the kernels as far as the slot ring allows
    //   in   (high priority): the select kernels; whatever is NOT staged is read in place from the pinned host tensor
    //                         (by default the vertex field: gather fetches only the SELECTED pixels' rows, tn*K*8 bytes
    //                         per image instead of the dense H*W*K*8)
    //   cmp  (low priority):  generate, vote, refit, D2H of the keypoints
    // Both PCIe consumers (DMA and in-place reads) share the link, so the pipeline's job is to keep it busy end to end.
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
    HostPipe *hp = nullptr;
    rc = host_pipe(dev, &hp);
    if (rc) return rc;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    e = cudaEventRecord(hp->user, user);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->copy, hp->user, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->in, hp->user, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->cmp, hp->user, 0);
    if (e != cudaSuccess) return cuda_fail(e, "stream wait");
    const size_t HW = (size_t)d->H * d->W;
    const size_t mbytes = HW * mask_elt_bytes(d->mask_dtype), vbytes = HW * d->K * 2 * sizeof(float);
    const size_t obytes = (size_t)d->K * 2 * sizeof(float);
    char *base = static_cast<char *>(dev_scratch);
    pvb_layout Lc;
    rc = make_layout(&dc, &Lc);
    if (rc) return rc;
    // in-place reads need pinned, device-mapped host memory; anything else is staged
    const char *mask_alias = static_cast<const char *>(mapped_alias(mask_host));
    const char *vertex_alias = static_cast<const char *>(mapped_alias(vertex_host));
    const bool stage_mask = !(flags & PVB_HOST_INPLACE_MASK) || !mask_alias;
    const bool stage_vertex = (flags & PVB_HOST_STAGE_VERTEX) || !vertex_alias;
    int piece = 0;
    for (int b0 = 0; b0 < d->B; b0 += chunk_images, ++piece) {
        const int slot = piece % HOST_SLOTS;
        const int c = (d->B - b0 < chunk_images) ? d->B - b0 : chunk_images;
        char *sb = base + (size_t)slot * S.end;
        const void *mptr = sb + S.mask;
        const float *vptr = reinterpret_cast<const float *>(sb + S.vertex);
        // this slot's buffers are free once the piece that used them HOST_SLOTS pieces ago has been computed
        if (piece >= HOST_SLOTS) {
            e = cudaStreamWaitEvent(hp->copy, hp->done[slot], 0);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->in, hp->done[slot], 0);
            if (e != cudaSuccess) return cuda_fail(e, "stream wait");
        }
        if (stage_mask)
            e = cudaMemcpyAsync(sb + S.mask, static_cast<const char *>(mask_host) + (size_t)b0 * mbytes, (size_t)c * mbytes, cudaMemcpyHostToDevice, hp->copy);
        else
            mptr = mask_alias + (size_t)b0 * mbytes;
        if (e == cudaSuccess && stage_vertex)
            e = cudaMemcpyAsync(sb + S.vertex, reinterpret_cast<const char *>(vertex_host) + (size_t)b0 * vbytes, (size_t)c * vbytes, cudaMemcpyHostToDevice, hp->copy);
        else if (e == cudaSuccess)
            vptr = reinterpret_cast<const float *>(vertex_alias + (size_t)b0 * vbytes);
        if (e != cudaSuccess) return cuda_fail(e, "H2D copy");
        if (stage_mask || stage_vertex) {
            e = cudaEventRecord(hp->dma[slot], hp->copy);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->in, hp->dma[slot], 0);
            if (e != cudaSuccess) return cuda_fail(e, "pipeline event");
        }
        pvb_desc di = dc;
        di.B = c;
        di.img_base = d->img_base + b0;
        di.capacity = Lc.capacity;
        Plan P;
        rc = make_plan(&di, mptr, vptr, nullptr, nullptr, sb + S.ws, S.end - S.ws, 1u, 2u, &P);
        if (rc) return rc;
        P.s.rowwise_gather = stage_vertex ? 0 : 1;
        rc = run_select(P, hp->in);
        if (rc) return rc;
        e = cudaEventRecord(hp->sel[slot], hp->in);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(hp->cmp, hp->sel[slot], 0);
        if (e != cudaSuccess) return cuda_fail(e, "pipeline event");
        PeerPush none;
        memset(&none, 0, sizeof(none));
        e = launch_generate(P.v, false, hp->cmp);     // its predecessor on cmp is the event wait, not thin_gather
        if (e == cudaSuccess) e = run_vote(P, true, hp->cmp);
        if (e == cudaSuccess) e = launch_refit(P.v, P.win, P.refit, reinterpret_cast<float *>(sb + S.out), none, hp->cmp);
        if (e != cudaSuccess) return cuda_fail(e, "compute kernels");
        e = cudaMemcpyAsync(reinterpret_cast<char *>(out_kpt_host) + (size_t)b0 * obytes, sb + S.out, (size_t)c * obytes, cudaMemcpyDeviceToHost, hp->cmp);
        if (e == cudaSuccess) e = cudaEventRecord(hp->done[slot], hp->cmp);
        if (e != cudaSuccess) return cuda_fail(e, "D2H copy");
    }
    e = cudaEventRecord(hp->end, hp->cmp);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(user, hp->end, 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(user);
    if (e != cudaSuccess) return cuda_fail(e, "stream sync");
    return PVB_OK;
}

PVB_API int pvb_profile_enable(int32_t every) { g_prof_every = every < 0 ? 0 : every; g_prof_tick = 0; return PVB_OK; }

PVB_API int pvb_set_tuning(int32_t gather_mode, int32_t vote_variant)
{
    if (vote_variant < 0 || vote_variant > 3) return fail(PVB_ERR_INVALID, "vote_variant must be 0..3");
    if (gather_mode < 0 || gather_mode > 2) return fail(PVB_ERR_INVALID, "gather_mode must be 0..2");
    set_gather_tuning(gather_mode);
    set_vote_tuning(vote_variant);
    return PVB_OK;
}

PVB_API int pvb_profile_reset(void)
{
    for (auto &pc : g_prof_calls)
        for (auto e : pc.ev) g_prof_pool.push_back(e);
    g_prof_calls.clear();
    return PVB_OK;
}

PVB_API int pvb_profile_read(double *ms, int32_t n)
{
    if (!ms || n < PVB_STAGE_COUNT) return fail(PVB_ERR_INVALID, "ms must hold PVB_STAGE_COUNT doubles");
    int calls = 0;
    for (auto &pc : g_prof_calls) {
        for (int i = 0; i < PVB_STAGE_COUNT; ++i) {
            cudaError_t e = cudaEventSynchronize(pc.ev[i + 1]);
            float t = 0.f;
            if (e == cudaSuccess) e = cudaEventElapsedTime(&t, pc.ev[i], pc.ev[i + 1]);
            if (e != cudaSuccess) { cuda_fail(e, "profile elapsed"); return -1; }
            ms[i] += (double)t;
        }
        if (pc.head) ++calls;
    }
    pvb_profile_reset();
    return calls;
}

// ---- twins of the reference extension --------------------------------------------------
static int check_compat(const void *a, const void *b, const void *c, const void *d_, int tn, int vn, int hn)
{
    if (tn < 0 || vn < 0 || hn < 0) return fail(PVB_ERR_INVALID, "negative size");
    if ((long long)hn * vn > (1ll << 30) || (long long)tn * vn > (1ll << 30)) return fail(PVB_ERR_INVALID, "problem too large");
    if (((tn && vn) && (!a || !b)) || ((hn && vn) && (!c || !d_))) return fail(PVB_ERR_INVALID, "NULL tensor");
    if (vn > 65535) return fail(PVB_ERR_INVALID, "vn must be <= 65535");
    return PVB_OK;
}

PVB_API int pvb_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs, float *hyp, int32_t tn,
                            int32_t vn, int32_t hn, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, idxs, hyp, tn, vn, hn);
    if (rc) return rc;
    cudaError_t e = launch_compat_generate(direct, coords, idxs, hyp, tn, vn, hn, false, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "generate_hypothesis");
}

PVB_API int pvb_generate_hypothesis_vanishing_point(const float *direct, const float *coords, const int32_t *idxs, float *hyp,
                                            int32_t tn, int32_t vn, int32_t hn, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, idxs, hyp, tn, vn, hn);
    if (rc) return rc;
    cudaError_t e = launch_compat_generate(direct, coords, idxs, hyp, tn, vn, hn, true, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "generate_hypothesis_vanishing_point");
}

PVB_API int pvb_voting_for_hypothesis(const float *direct, const float *coords, const float *hyp, uint8_t *inliers, int32_t tn,
                              int32_t vn, int32_t hn, float inlier_thresh, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, inliers, tn, vn, hn);
    if (rc) return rc;
    if (tn && vn && hn && !inliers) return fail(PVB_ERR_INVALID, "NULL tensor");
    cudaError_t e = launch_compat_vote(direct, coords, hyp, inliers, tn, vn, hn, inlier_thresh, false, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "voting_for_hypothesis");
}

PVB_API int pvb_voting_for_hypothesis_vanishing_point(const float *direct, const float *coords, const float *hyp,
                                              uint8_t *inliers, int32_t tn, int32_t vn, int32_t hn,
                                              float inlier_thresh, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, inliers, tn, vn, hn);
    if (rc) return rc;
    if (tn && vn && hn && !inliers) return fail(PVB_ERR_INVALID, "NULL tensor");
    cudaError_t e = launch_compat_vote(direct, coords, hyp, inliers, tn, vn, hn, inlier_thresh, true, static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "voting_for_hypothesis_vanishing_point");
}

PVB_API size_t pvb_vote_count_workspace_bytes(int32_t tn, int32_t vn, int32_t hn)
{
    if (tn < 0 || vn < 0 || hn < 0) return 0;
    size_t off = align_up(4 * sizeof(int));
    off += align_up((size_t)tn * sizeof(float2));
    off += align_up((size_t)tn * vn * sizeof(float2));
    off += align_up((size_t)hn * vn * sizeof(float2));
    off += align_up((size_t)hn * vn * sizeof(int));
    return off;
}

PVB_API int pvb_vote_count(const float *direct, const float *coords, const float *hyp, int32_t *counts, int32_t tn, int32_t vn,
                   int32_t hn, float inlier_thresh, void *workspace, size_t workspace_bytes, pvb_stream_t stream)
{
    int rc = check_compat(direct, coords, hyp, counts, tn, vn, hn);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (hn == 0 || vn == 0) return PVB_OK;
    if (tn == 0) {
        cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)hn * vn, st);
        return e == cudaSuccess ? PVB_OK : cuda_fail(e, "memset");
    }
    if ((long long)vn * ((hn + 511) / 512) > 65535) return fail(PVB_ERR_INVALID, "vn*ceil(hn/512) must be <= 65535");
    const size_t need = pvb_vote_count_workspace_bytes(tn, vn, hn);
    if (!workspace || workspace_bytes < need) return fail(PVB_ERR_WORKSPACE, "workspace too small: need %zu", need);
    if (reinterpret_cast<uintptr_t>(workspace) & 255u) return fail(PVB_ERR_WORKSPACE, "workspace must be 256-byte aligned");
    char *w = static_cast<char *>(workspace);
    size_t off = 0;
    int *meta = reinterpret_cast<int *>(w + off); off += align_up(4 * sizeof(int));
    float2 *xy = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)tn * sizeof(float2));
    float2 *dirs = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)tn * vn * sizeof(float2));
    float2 *hyp_k = reinterpret_cast<float2 *>(w + off); off += align_up((size_t)hn * vn * sizeof(float2));
    int *counts_k = reinterpret_cast<int *>(w + off);
    cudaError_t e = launch_compat_repack(direct, coords, hyp, tn, vn, hn, dirs, xy, hyp_k, meta, st);
    if (e != cudaSuccess) return cuda_fail(e, "repack");
    VoteArgs v;
    memset(&v, 0, sizeof(v));
    v.B = 1; v.K = vn; v.hn = hn; v.cap = tn; v.W = 0; v.H = 0; v.thresh = inlier_thresh;
    v.tn = meta; v.state = meta + 1; v.xy = xy;
    v.dirs = dirs; v.idxs = nullptr; v.hyp = hyp_k; v.counts = counts_k;
    e = launch_vote(v, true, false, st);
    if (e != cudaSuccess) return cuda_fail(e, "vote kernel");
    e = launch_compat_unpack_counts(counts_k, counts, vn, hn, st);
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "unpack");
}

// ---- multi-GPU exchange ----------------------------------------------------------------
PVB_API int pvb_exchange_create(int32_t rank, int32_t world, int32_t slots, size_t bytes_per_rank, pvb_exchange **out)
{
    if (!out) return fail(PVB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (world < 1 || world > PVB_MAX_PEERS || rank < 0 || rank >= world) return fail(PVB_ERR_INVALID, "bad rank %d / world %d (max %d)", rank, world, PVB_MAX_PEERS);
    if (slots < 2 || slots > 4096) return fail(PVB_ERR_INVALID, "slots must be in [2,4096]");
    if (bytes_per_rank == 0 || bytes_per_rank > ((size_t)1 << 30)) return fail(PVB_ERR_INVALID, "bad bytes_per_rank");
    pvb_exchange *ex = new (std::nothrow) pvb_exchange();
    if (!ex) return fail(PVB_ERR_INVALID, "out of host memory");
    memset(ex, 0, sizeof(*ex));
    ex->rank = rank; ex->world = world; ex->slots = slots;
    ex->bytes_per_rank = (bytes_per_rank + 15) / 16 * 16;
    ex->status_off = align_up((size_t)slots * world * ex->bytes_per_rank * 2);      // ring of {float bits, seq} words
    ex->total = ex->status_off + 256;
    cudaError_t e = cudaGetDevice(&ex->device);
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&ex->local), ex->total);
    if (e == cudaSuccess) e = cudaMemset(ex->local, 0, ex->total);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { if (ex->local) cudaFree(ex->local); delete ex; return cuda_fail(e, "exchange allocation"); }
    ex->peer[rank] = ex->local;
    ex->connected = (world == 1);
    *out = ex;
    return PVB_OK;
}

PVB_API size_t pvb_exchange_bytes_per_rank(const pvb_exchange *ex) { return ex ? ex->bytes_per_rank : 0; }
PVB_API void *pvb_exchange_base(const pvb_exchange *ex) { return ex ? ex->local : nullptr; }

PVB_API int pvb_exchange_get_handle(const pvb_exchange *ex, void *handle)
{
    if (!ex || !handle) return fail(PVB_ERR_INVALID, "NULL argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == PVB_IPC_HANDLE_BYTES, "handle size");
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ex->local);
    if (e != cudaSuccess) return cuda_fail(e, "cudaIpcGetMemHandle");
    memcpy(handle, &h, sizeof(h));
    return PVB_OK;
}

PVB_API int pvb_exchange_connect_ptrs(pvb_exchange *ex, void *const *bases)
{
    if (!ex || !bases) return fail(PVB_ERR_INVALID, "NULL argument");
    for (int r = 0; r < ex->world; ++r) {
        if (r == ex->rank) continue;
        if (!bases[r]) return fail(PVB_ERR_INVALID, "base pointer of rank %d is NULL", r);
        ex->peer[r] = static_cast<char *>(bases[r]);
    }
    ex->connected = true;
    return PVB_OK;
}

PVB_API int pvb_exchange_connect(pvb_exchange *ex, const void *handles)
{
    if (!ex || !handles) return fail(PVB_ERR_INVALID, "NULL argument");
    const char *hb = static_cast<const char *>(handles);
    for (int r = 0; r < ex->world; ++r) {
        if (r == ex->rank || ex->ipc_opened[r]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hb + (size_t)r * PVB_IPC_HANDLE_BYTES, sizeof(h));
        void *p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return cuda_fail(e, "cudaIpcOpenMemHandle (peer memory over NVLink needs P2P access between the GPUs)");
        ex->peer[r] = static_cast<char *>(p);
        ex->ipc_opened[r] = true;
    }
    ex->connected = true;
    return PVB_OK;
}

PVB_API int pvb_exchange_wait(pvb_exchange *ex, uint64_t seq, void *out, const int32_t *floats_per_rank, double timeout_s,
                              pvb_stream_t stream)
{
    if (!ex || !out) return fail(PVB_ERR_INVALID, "NULL argument");
    if (seq == 0 || (uint32_t)seq == 0) return fail(PVB_ERR_INVALID, "seq must be >= 1 and not a multiple of 2^32");
    if (reinterpret_cast<uintptr_t>(out) & 3u) return fail(PVB_ERR_INVALID, "out must be 4-byte aligned");
    if (!(timeout_s > 0.0)) timeout_s = 10.0;
    const int words = (int)(ex->bytes_per_rank / sizeof(float));
    ExchangeCounts counts;
    for (int r = 0; r < PVB_MAX_PEERS; ++r) counts.n[r] = 0;
    for (int r = 0; r < ex->world; ++r) {
        const int n = floats_per_rank ? floats_per_rank[r] : words;
        if (n < 0 || n > words) return fail(PVB_ERR_INVALID, "floats_per_rank[%d] = %d outside [0, %d]", r, n, words);
        counts.n[r] = n;
    }
    const size_t slot = (size_t)((seq - 1) % (uint64_t)ex->slots);
    const uint2 *recv = reinterpret_cast<const uint2 *>(ex->local) + slot * ex->world * words;
    cudaError_t e = launch_exchange_wait(recv, (uint32_t)seq, static_cast<float *>(out), ex->world, words, counts,
                                         (unsigned long long)(timeout_s * 1e9), reinterpret_cast<int *>(ex->local + ex->status_off),
                                         static_cast<cudaStream_t>(stream));
    return e == cudaSuccess ? PVB_OK : cuda_fail(e, "exchange wait kernel");
}

PVB_API int pvb_exchange_status(pvb_exchange *ex, pvb_stream_t stream)
{
    if (!ex) return fail(PVB_ERR_INVALID, "NULL argument");
    int host = 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaError_t e = cudaMemcpyAsync(&host, ex->local + ex->status_off, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return cuda_fail(e, "exchange status");
    if (host) return fail(PVB_ERR_TIMEOUT, "a pvb_exchange_wait timed out: some rank never published its result");
    return PVB_OK;
}

PVB_API int pvb_exchange_destroy(pvb_exchange *ex)
{
    if (!ex) return PVB_OK;
    cudaDeviceSynchronize();
    for (int r = 0; r < ex->world; ++r)
        if (ex->ipc_opened[r]) cudaIpcCloseMemHandle(ex->peer[r]);
    if (ex->local) cudaFree(ex->local);
    delete ex;
    return PVB_OK;
}

} // extern "C"
