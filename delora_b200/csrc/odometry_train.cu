// Training through the C ABI (sm_90a).
//
// delora_odometry_train_step: projection + normals of the 2B scans (with w_pre > 0: at H x w_pre, then re-projected at
// H x W by delora_project_grids_fwd), the trunk forward keeping its activations (trunk.cuh), the tail forward keeping
// its activations, the dense ICP losses with dL/dT, the tail backward (odometry_tail.cu), the trunk backward, one Adam
// update of the fp32 master blob and one re-prep of the bf16 filters from it.  Weight gradients land in a gradient
// blob with the layout of the weight blob: the wgrad kernels write each filter at its blob offset ([Cout, Cin, k, k]
// is both the state_dict layout and theirs), the tail kernels each fc / head tensor at its own.  This file also holds
// _train_eval, the Adam state, the group step, the training geometries and the dropout seed and keep masks.
//
// Kernels here (fixed summation order, no atomics: bit-identical from run to run):
//   odometry_train_normalized_out_kernel (DELORA_TRAIN_NORMALIZATION_SCALING): T with its translation rescaled to the
//     caller's output, the factor to losses[b][6].
//   odometry_icp_rearm_kernel: zeroes the ICP scratch when B differs from the batch size of the previous step (the
//     scratch layout depends on B); otherwise every CTA exits at once.  odometry_icp_batch_kernel records that batch
//     size after a call that runs the ICP without the backward.
//   DELORA_TRAIN_DROPOUT (masks from dropout.cuh, regenerated in the backward): the dropout variants of the trunk-input
//     conversion and odometry_channel_dropout_kernel (trunk.cu), and of the tail's fc launches (odometry_tail.cu).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "odometry.cuh"
#include "projection.cuh"

namespace delora {

// The training step of a normalised model (DELORA_TRAIN_NORMALIZATION_SCALING), after the ICP finalize: T_out [B, 16] =
// the forward's T with T[:3, 3] multiplied by the pair's factor (or no copy when T_out is NULL), losses[b][6] = factor[b].
__global__ void odometry_train_normalized_out_kernel(const float* __restrict__ T16, const float* __restrict__ factor,
                                                     int B, float* __restrict__ T_out, float* __restrict__ losses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 16) return;
    const int b = i >> 4, e = i & 15;
    const float f = factor[b];
    if (T_out) T_out[i] = (e == 3 || e == 7 || e == 11) ? __fmul_rn(T16[i], f) : T16[i];
    if (e == 0) losses[(size_t)b * DELORA_LOSS_ROW + 6] = f;
}

__global__ void odometry_icp_rearm_kernel(float4* __restrict__ s, long long n4, int B, const long long* __restrict__ ctr) {
    if (ctr[1] == B) return;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride)
        s[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

// Two sections.  The model section (master weights, gradient, Adam's m and v, the counters, the bf16 filters) comes
// first and depends only on act, layers, resnet_outputs, single_mlp and the parity of W (the stem's filter layout).
// The geometry section (frames, grids, ICP scratch, activations, tail buffers, the w_pre buffers) starts at f.keys.
// delora_odometry_train_geometries_* rely on this split: one model section serves several geometry sections.
// geometry_at > 0: the geometry section starts at that byte offset instead (delora_odometry_streams_*_geometries: one
// model section and one geometry section per descriptor, each further one after the previous geometry's sections).
void make_train_plan(const delora_odometry_desc* d, TrainPlan* tp, size_t geometry_at) {
    memset(tp, 0, sizeof(TrainPlan));
    plan_model(d, &tp->m);
    const Model& m = tp->m;
    const int MB = d->max_batch, H = d->H, W = d->W, HW = H * W, nout = d->resnet_outputs;
    size_t off = 0;
    const size_t blob = (size_t)m.blob_floats * 4;
    tp->master = take(off, blob); tp->grad = take(off, blob); tp->adam_m = take(off, blob); tp->adam_v = take(off, blob);
    // [0] Adam's step count, [1] the ICP scratch's batch size, [2] the dropout seed (the slot has 256 bytes)
    tp->ctr = take(off, 3 * sizeof(long long));
    tp->w = plan_trunk_weights(m.t, true, off);
    if (geometry_at) off = geometry_at;
    // one key buffer serves both projections of a step, one after the other
    tp->f = plan_frames(d, 2 * MB, 0, false, d->w_pre > W ? d->w_pre : W, off);
    tp->pts_grid = take(off, (size_t)2 * MB * HW * 16);
    tp->nrm_grid = take(off, (size_t)2 * MB * HW * 16);
    tp->icp = take(off, (size_t)delora_icp_scratch_floats(MB, HW) * 4);
    tp->losses = take(off, (size_t)MB * DELORA_LOSS_ROW * 4);
    tp->grad_T = take(off, (size_t)MB * 12 * 4);
    tp->T16 = take(off, (size_t)MB * 16 * 4);
    tp->T12 = take(off, (size_t)MB * 12 * 4);
    tp->t = plan_trunk_acts(m.t, MB, true, off);
    tp->pooled = take(off, (size_t)MB * 512 * 4);
    tp->g_pooled = take(off, (size_t)MB * 512 * 4);
    tp->fc_out = take(off, (size_t)MB * nout * 4);
    tp->dz_fc = take(off, (size_t)MB * nout * 4);
    tp->raw = take(off, (size_t)MB * 7 * 4);
    if (m.n_lin == 4) {
        tp->hid[0] = take(off, (size_t)MB * 2 * kHeadHidden * 4);
        tp->dz_hid[0] = take(off, (size_t)MB * 2 * kHeadHidden * 4);
    } else {
        for (int i = 0; i < m.n_lin - 1; ++i) {
            tp->hid[i] = take(off, (size_t)MB * m.lin[i].N * 4);
            tp->dz_hid[i] = take(off, (size_t)MB * m.lin[i].N * 4);
        }
    }
    if (d->w_pre > 0) {
        const size_t HWp = (size_t)H * d->w_pre;
        tp->pre_image = take(off, (size_t)2 * MB * 4 * HWp * 4);
        tp->pre_index_map = take(off, (size_t)2 * MB * HWp * 4);
        tp->pre_pts_grid = take(off, (size_t)2 * MB * HWp * 16);
        tp->pre_nrm_grid = take(off, (size_t)2 * MB * HWp * 16);
    }
    tp->total = off;
}

// The training step's sections.  A training plan has no cached image (prev_image, has_prev stay 0, unread).
void map_train(SectionMap& s, const delora_odometry_desc* d, const TrainPlan& tp, bool adam, int ctr_role,
               int weights_flags, int model_flags) {
    s.flags = weights_flags;
    s.field("master", tp.master, DELORA_WS_WEIGHTS);
    map_trunk_weights(s, tp.m.t, tp.w);
    s.flags = model_flags;
    // the group step's last bucket ends up to 3 floats past the blob (plan_buckets)
    s.range("grad", tp.grad, (size_t)(tp.m.blob_floats + 3) / 4 * 16, DELORA_WS_OUTPUT);
    if (adam) {
        s.field("adam_m", tp.adam_m, DELORA_WS_STATE);
        s.field("adam_v", tp.adam_v, DELORA_WS_STATE);
    }
    // [0] Adam's step count, [1] the ICP scratch's batch size, [2] the dropout seed; a slot of the fleet section for
    // the adapting streams' geometries g >= 1
    s.range("ctr", tp.ctr, 3 * sizeof(long long), ctr_role);
    s.flags = 0;
    map_frames(s, tp.f, true, true, DELORA_WS_SCRATCH);
    s.field("pts_grid", tp.pts_grid, DELORA_WS_SCRATCH);
    s.field("nrm_grid", tp.nrm_grid, DELORA_WS_SCRATCH);
    // odometry_icp_rearm_kernel zeroes the scratch in whole float4s: up to 12 bytes past its last float
    s.range("icp", tp.icp, (size_t)(delora_icp_scratch_floats(d->max_batch, d->H * d->W) + 3) / 4 * 16,
            DELORA_WS_SCRATCH);
    s.field("losses", tp.losses, DELORA_WS_OUTPUT);
    s.field("grad_T", tp.grad_T, DELORA_WS_SCRATCH);
    s.field("T16", tp.T16, DELORA_WS_OUTPUT);
    s.field("T12", tp.T12, DELORA_WS_SCRATCH);
    s.span("trunk.acts", tp.t.x_in, tp.pooled, DELORA_WS_SCRATCH);
    s.field("pooled", tp.pooled, DELORA_WS_OUTPUT);
    s.field("g_pooled", tp.g_pooled, DELORA_WS_SCRATCH);
    s.field("fc_out", tp.fc_out, DELORA_WS_SCRATCH);
    s.field("dz_fc", tp.dz_fc, DELORA_WS_SCRATCH);
    s.field("raw", tp.raw, DELORA_WS_SCRATCH);
    char name[32];
    for (int i = 0; i < (tp.m.n_lin == 4 ? 1 : tp.m.n_lin - 1); ++i) {       // two heads: one [rot1 | trans1] buffer
        snprintf(name, sizeof name, "hid[%d]", i);
        s.field(name, tp.hid[i], DELORA_WS_SCRATCH);
        snprintf(name, sizeof name, "dz_hid[%d]", i);
        s.field(name, tp.dz_hid[i], DELORA_WS_SCRATCH);
    }
    if (d->w_pre > 0) {
        // pre_image also holds the pair factors of a normalised step
        s.field("pre_image", tp.pre_image, DELORA_WS_SCRATCH);
        s.field("pre_index_map", tp.pre_index_map, DELORA_WS_SCRATCH);
        s.field("pre_pts_grid", tp.pre_pts_grid, DELORA_WS_SCRATCH);
        s.field("pre_nrm_grid", tp.pre_nrm_grid, DELORA_WS_SCRATCH);
    }
}

// DELORA_WS_TRAIN and DELORA_WS_TRAIN_GEOMETRIES.  Each geometry of the latter trains the whole model section (shared)
// on its own geometry section, which _train_use_geometry lays over the same bytes as every other geometry's.
int map_train_kind(SectionMap& s, const delora_odometry_desc* d, int n, int kind, const char* who) {
    if (kind == DELORA_WS_TRAIN ? check_train_desc(d, who) : check_geometries(d, n, who)) return 1;
    const bool shared = kind == DELORA_WS_TRAIN_GEOMETRIES;
    for (int g = 0; g < n; ++g) {
        // the geometry sections start at one offset: each geometry's fields are sized from its own plan's log
        take_log->off.clear();
        take_log->bytes.clear();
        TrainPlan tp;
        make_train_plan(&d[g], &tp);
        s.geometry = g;
        map_train(s, &d[g], tp, true, DELORA_WS_STATE, shared ? DELORA_WS_SHARED : 0, shared ? DELORA_WS_SHARED : 0);
    }
    return 0;
}

// check_desc plus the field only training reads
int check_train_desc(const delora_odometry_desc* d, const char* who) {
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(d->w_pre == 0 || (d->w_pre >= 2 && (long long)d->H * d->w_pre < (1ll << 27)),
                     "%s: w_pre=%d must be 0 or >= 2 with H * w_pre < 2^27 (H=%d)", who, d->w_pre, d->H);
    return 0;
}

int check_train_params(const delora_odometry_train_params* hp, const char* who) {
    DELORA_CHECK_ARG(hp != nullptr, "%s: null hyperparameters", who);
    DELORA_CHECK_ARG(isfinite(hp->lr) && hp->lr >= 0.0f, "%s: lr=%g must be finite and >= 0", who, (double)hp->lr);
    DELORA_CHECK_ARG(hp->beta1 >= 0.0f && hp->beta1 < 1.0f, "%s: beta1=%g must be in [0, 1)", who, (double)hp->beta1);
    DELORA_CHECK_ARG(hp->beta2 >= 0.0f && hp->beta2 < 1.0f, "%s: beta2=%g must be in [0, 1)", who, (double)hp->beta2);
    DELORA_CHECK_ARG(isfinite(hp->eps) && hp->eps > 0.0f, "%s: eps=%g must be > 0", who, (double)hp->eps);
    return check_icp_params(hp->lambda_po2pl, hp->loss_flags, hp->nb_h, hp->nb_w, hp->epsilon_range, hp->min_neighbors,
                            who);
}

static TailIO train_tail_io(const TrainPlan& tp, char* ws) {
    const Model& m = tp.m;
    TailIO io;
    memset(&io, 0, sizeof(io));
    const float* master = reinterpret_cast<const float*>(ws + tp.master);
    io.fc_w = master + m.fc.blob_w; io.fc_b = master + m.fc.blob_b;
    for (int i = 0; i < m.n_lin; ++i) { io.w[i] = master + m.lin[i].blob_w; io.b[i] = master + m.lin[i].blob_b; }
    io.fc_out = reinterpret_cast<float*>(ws + tp.fc_out);
    for (int i = 0; i < m.n_lin - 1; ++i) io.hid[i] = reinterpret_cast<float*>(ws + tp.hid[m.n_lin == 4 ? 0 : i]);
    io.raw = reinterpret_cast<float*>(ws + tp.raw);
    return io;
}

}  // namespace delora

using namespace delora;

extern "C" int64_t delora_odometry_train_workspace_bytes(const delora_odometry_desc* d) {
    if (check_train_desc(d, "delora_odometry_train_workspace_bytes")) return -1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return (int64_t)tp.total;
}

namespace delora {

// _train_init on a workspace of `total` bytes (>= d's size), armed for d
int train_init(const delora_odometry_desc* d, size_t total, const float* weights, void* workspace,
               cudaStream_t st, const char* who) {
    DELORA_CHECK_ARG(weights && workspace, "%s: null pointer", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    char* ws = (char*)workspace;
    int rc = init_workspace(tp.f, total, ws, st, who);
    if (rc) return rc;
    const cudaError_t e = cudaMemcpyAsync(ws + tp.master, weights, (size_t)tp.m.blob_floats * 4, cudaMemcpyDeviceToDevice,
                                          st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return prep_blob_weights(tp.m, tp.w, ws, reinterpret_cast<const float*>(ws + tp.master), st, who);
}

// The descriptors of one shared training workspace: each valid for training, with d[0]'s model fields and W parity,
// so that all of them plan the same model section
int check_geometries(const delora_odometry_desc* d, int n, const char* who) {
    DELORA_CHECK_ARG(d != nullptr, "%s: null descriptor array", who);
    DELORA_CHECK_ARG(n >= 1, "%s: n=%d must be >= 1", who, n);
    for (int g = 0; g < n; ++g) {
        char w[192];
        snprintf(w, sizeof w, "%s: d[%d]", who, g);
        if (check_train_desc(&d[g], w)) return 1;
        const delora_odometry_desc &a = d[0], &b = d[g];
        DELORA_CHECK_ARG(b.act == a.act, "%s: d[%d].act=%d differs from d[0].act=%d", who, g, b.act, a.act);
        for (int s = 0; s < 4; ++s)
            DELORA_CHECK_ARG(b.layers[s] == a.layers[s], "%s: d[%d].layers[%d]=%d differs from d[0].layers[%d]=%d", who,
                             g, s, b.layers[s], s, a.layers[s]);
        DELORA_CHECK_ARG(b.resnet_outputs == a.resnet_outputs, "%s: d[%d].resnet_outputs=%d differs from "
                         "d[0].resnet_outputs=%d", who, g, b.resnet_outputs, a.resnet_outputs);
        DELORA_CHECK_ARG(b.single_mlp == a.single_mlp, "%s: d[%d].single_mlp=%d differs from d[0].single_mlp=%d", who,
                         g, b.single_mlp, a.single_mlp);
        DELORA_CHECK_ARG(b.W % 2 == a.W % 2, "%s: d[%d].W=%d and d[0].W=%d differ in parity: the stem's filter layout, "
                         "and with it the model section, would differ", who, g, b.W, a.W);
    }
    return 0;
}

// The shared workspace: the model section and the largest geometry section, i.e. the largest single-geometry size
static size_t geometries_bytes(const delora_odometry_desc* d, int n) {
    size_t total = 0;
    for (int g = 0; g < n; ++g) {
        TrainPlan tp;
        make_train_plan(&d[g], &tp);
        total = tp.total > total ? tp.total : total;
    }
    return total;
}

}  // namespace delora

extern "C" int delora_odometry_train_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                          void* stream) {
    const char* who = "delora_odometry_train_init";
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return train_init(d, tp.total, weights, workspace, (cudaStream_t)stream, who);
}

extern "C" int64_t delora_odometry_train_geometries_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_geometries(d, n, "delora_odometry_train_geometries_workspace_bytes")) return -1;
    return (int64_t)geometries_bytes(d, n);
}

extern "C" int delora_odometry_train_geometries_init(const delora_odometry_desc* d, int n, const float* weights,
                                                     void* workspace, void* stream) {
    const char* who = "delora_odometry_train_geometries_init";
    if (check_geometries(d, n, who)) return 1;
    return train_init(d, geometries_bytes(d, n), weights, workspace, (cudaStream_t)stream, who);
}

extern "C" int delora_odometry_train_use_geometry(const delora_odometry_desc* d, int n, int g, void* workspace,
                                                  void* stream) {
    const char* who = "delora_odometry_train_use_geometry";
    if (check_geometries(d, n, who)) return 1;
    DELORA_CHECK_ARG(g >= 0 && g < n, "%s: g=%d outside [0, n=%d)", who, g, n);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(&d[g], &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    // the geometry section as _train_init leaves it, then the ICP scratch's batch marker ctr[1] as _train_init's zero
    int rc = init_workspace(tp.f, tp.total, ws, st, who, tp.f.keys);
    if (rc) return rc;
    const cudaError_t e = cudaMemsetAsync(ws + tp.ctr + sizeof(long long), 0, sizeof(long long), st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

namespace delora {

__global__ void odometry_icp_batch_kernel(long long* __restrict__ ctr, int B) { ctr[1] = B; }

// After an ICP without the backward (which records B itself): the ICP scratch now has the layout of B pairs, and the
// next step or eval re-arms it if its batch size differs
int record_icp_batch(const TrainPlan& tp, char* ws, int B, cudaStream_t st) {
    odometry_icp_batch_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(ws + tp.ctr), B);
    DELORA_CHECK_LAUNCH("odometry_icp_batch_kernel");
    return 0;
}

// Stages 1-3 of delora_odometry_train_step and all of delora_odometry_train_eval: the projection + normals of the 2B
// scans, the forward keeping its activations and the ICP losses with dL/dT, into the workspace (losses, grad_T, T16,
// pooled).  dropout: the forward draws this step's masks.  Normalised models: T_out [B, 16] or NULL gets T in metres.
// at (delora_odometry_streams_push_adapt, B = S): stage 1 projects only the B scans of this tick (scan_2 of each pair,
// inactive streams' counts masked to 0) and takes its first half, scan_1's, from the cache; the output kernel divides
// each quaternion by its own row's norm, writes raw for the valid rows only, valid, has_prev and n_valid; then the
// bookkeeping kernel writes at->T, T12, the masked cache write and empties the sources of the rows without a pair.
// With at->info the ICP is the information operator (losses and dL/dT are the same bits), in metres for normalised
// models: their grids were divided by the pair factors, kept in pre_image.
int train_forward_losses(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const TrainPlan& tp,
                         char* ws, const float* points, const int32_t* n_points, int B, bool dropout, float* T_out,
                         cudaStream_t st, const char* who, const AdaptTick* at) {
    const Model& m = tp.m;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    const int H = d->H, W = d->W, HW = H * W;
    const bool normalized = (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u;
    long long* ctr = reinterpret_cast<long long*>(ws + tp.ctr);
    // the forward reads the step count before odometry_out_bwd_kernel advances it
    const DropoutCtr drop_fwd{dropout ? ctr : nullptr, 0};
    int rc;

    // 1. projection + normals of the 2B scans (scan_1 x B, then scan_2 x B).  w_pre > 0: the reference's two stages,
    // projection + normals at H x w_pre (its offline preprocessing), then those grids projected at H x W (Deployer.step)
    // at: only the B scan_2's are projected (from scan index `first` on), and scan_1's stage-1 output is the cache's
    const int n_proj = at ? B : 2 * B;
    const size_t first = at ? (size_t)B : 0;
    if ((rc = clamp_counts(tp.f, ws, n_points, at ? at->active : nullptr, n_proj, d->n_stride, st))) return rc;
    int32_t* counts = reinterpret_cast<int32_t*>(ws + tp.f.counts);
    delora_f4* pts_grid = reinterpret_cast<delora_f4*>(ws + tp.pts_grid);
    delora_f4* nrm_grid = reinterpret_cast<delora_f4*>(ws + tp.nrm_grid);
    float* images = f(tp.f.images);
    uint64_t* keys = reinterpret_cast<uint64_t*>(ws + tp.f.keys);
    const size_t HWc = (size_t)H * (d->w_pre > 0 ? d->w_pre : W);         // cells of a stage-1 grid
    auto from_cache = [&](void* dst, const void* src, size_t bytes) {
        const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
        return 0;
    };
    if (d->w_pre > 0) {
        delora_f4* pre_pts = reinterpret_cast<delora_f4*>(ws + tp.pre_pts_grid);
        delora_f4* pre_nrm = reinterpret_cast<delora_f4*>(ws + tp.pre_nrm_grid);
        if ((rc = project_scan_grids(d, d->w_pre, hp->loss_flags, hp->nb_h, hp->nb_w, hp->epsilon_range,
                                     hp->min_neighbors, points, counts, n_proj, keys, f(tp.pre_image) + first * 4 * HWc,
                                     reinterpret_cast<int32_t*>(ws + tp.pre_index_map) + first * HWc,
                                     pre_pts + first * HWc, pre_nrm + first * HWc, st)))
            return rc;
        if (at && ((rc = from_cache(pre_pts, at->cache_pts, (size_t)B * HWc * 16)) ||
                   (rc = from_cache(pre_nrm, at->cache_nrm, (size_t)B * HWc * 16)))) return rc;
        // normalised: the factor of each pair from its stored points (the valid H x w_pre cells), kept in the H x w_pre
        // image, which nothing reads after delora_project_normals_fwd; the stored points are divided by it before the
        // H x W projection, the normals are not
        float* factor = normalized ? f(tp.pre_image) : nullptr;
        if (normalized && (rc = launch_grid_normalization_factors(pre_pts, B, H * d->w_pre, factor, st))) return rc;
        const GridParams g = make_grid(H, W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
        if ((rc = project_grids_fwd(pre_pts, pre_nrm, 2 * B, d->w_pre, g, keys, images,
                                    reinterpret_cast<int32_t*>(ws + tp.f.index_map), pts_grid, nrm_grid, factor, B, st)))
            return rc;
    } else {
        if ((rc = project_scan_grids(d, W, hp->loss_flags, hp->nb_h, hp->nb_w, hp->epsilon_range, hp->min_neighbors,
                                     points, counts, n_proj, keys, images + first * 4 * HW,
                                     reinterpret_cast<int32_t*>(ws + tp.f.index_map) + first * HW,
                                     pts_grid + first * HW, nrm_grid + first * HW, st)))
            return rc;
        if (at && ((rc = from_cache(images, at->cache_image, (size_t)B * 4 * HW * 4)) ||
                   (rc = from_cache(pts_grid, at->cache_pts, (size_t)B * HW * 16)) ||
                   (rc = from_cache(nrm_grid, at->cache_nrm, (size_t)B * HW * 16)))) return rc;
    }
    // 2. forward, keeping the activations
    if ((rc = trunk_input(m.t, tp.t, ws, images, images + (size_t)B * 4 * HW, B, st, drop_fwd))) return rc;
    if (at) {               // dropout is off: the served T is dropout-free
        if ((rc = streams_forward(m, train_tail_io(tp, ws), tp.t, tp.w, ws, d->act, f(tp.pooled), B, at->active,
                                  at->has_prev, f(tp.T16), at->valid, nullptr, nullptr, nullptr, at->n_valid, st)))
            return rc;
        // T (normalised: the factor of the H x w_pre grids, kept in pre_image as below), T12, the cache, the sources
        float4* cur_pts = reinterpret_cast<float4*>(pts_grid + (size_t)B * HW);
        float4* cur_nrm = reinterpret_cast<float4*>(nrm_grid + (size_t)B * HW);
        const bool pre = d->w_pre > 0;
        if ((rc = streams_pre(f(tp.T16), normalized ? f(tp.pre_image) : nullptr, at->active, at->valid, B, HW, (int)HWc,
                              at->T, f(tp.T12), nullptr, cur_pts, cur_nrm,
                              pre ? reinterpret_cast<const float4*>(ws + tp.pre_pts_grid) + (size_t)B * HWc : cur_pts,
                              pre ? reinterpret_cast<const float4*>(ws + tp.pre_nrm_grid) + (size_t)B * HWc : cur_nrm,
                              reinterpret_cast<float4*>(at->cache_pts), reinterpret_cast<float4*>(at->cache_nrm),
                              pre ? nullptr : reinterpret_cast<const float4*>(images + (size_t)B * 4 * HW),
                              reinterpret_cast<float4*>(at->cache_image), st))) return rc;
    } else {
        if ((rc = trunk_forward(m.t, tp.t, ws, tp.w, ws, d->act, B, f(tp.pooled), nullptr, st, drop_fwd))) return rc;
        if ((rc = run_tail(m, train_tail_io(tp, ws), d->act, f(tp.pooled), B, f(tp.T16), st, nullptr, drop_fwd)))
            return rc;
        const cudaError_t e = cudaMemcpy2DAsync(f(tp.T12), 12 * sizeof(float), f(tp.T16), 16 * sizeof(float),
                                                12 * sizeof(float), B, cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    // 3. ICP losses and dL/dT: source = scan_2 moved by T, target = scan_1.  The identity fit still runs them: the
    // reference logs the ICP losses in that phase too
    const long long icp_n4 = (delora_icp_scratch_floats(B, HW) + 3) / 4;
    odometry_icp_rearm_kernel<<<2 * num_sms(), 256, 0, st>>>(reinterpret_cast<float4*>(ws + tp.icp), icp_n4, B, ctr);
    DELORA_CHECK_LAUNCH("odometry_icp_rearm_kernel");
    // po2po_alone: DELORA_LOSS_PO2PO on the zero normal grids of stage 1
    const uint32_t icp_flags = hp->loss_flags & ~(DELORA_LOSS_IDENTITY_FIT | DELORA_TRAIN_NORMALIZATION_SCALING |
                                                  DELORA_TRAIN_DROPOUT | DELORA_LOSS_PO2PO_ALONE);
    float* info = at ? at->info : nullptr;
    const float* factor = info && normalized ? f(tp.pre_image) : nullptr;
    if ((rc = icp_dense_launch(pts_grid + (size_t)B * HW, nrm_grid + (size_t)B * HW, f(tp.T12), pts_grid, nrm_grid, B,
                               H, W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, hp->lambda_po2pl, icp_flags,
                               f(tp.losses), f(tp.grad_T), f(tp.icp), info, at ? at->info_scratch : nullptr, factor,
                               st, icp_entry(info, factor)))) return rc;
    if (normalized) {               // T in metres for the caller, the factor in losses[b][6]
        odometry_train_normalized_out_kernel<<<(B * 16 + 255) / 256, 256, 0, st>>>(f(tp.T16), f(tp.pre_image), B, T_out,
                                                                                      f(tp.losses));
        DELORA_CHECK_LAUNCH("odometry_train_normalized_out_kernel");
    }
    return 0;
}

// losses, T (not for normalised models: train_forward_losses wrote it) and pooled of B pairs to the caller's buffers
static int train_outputs(const TrainPlan& tp, const char* ws, int B, bool normalized, float* losses, float* T,
                         float* pooled, cudaStream_t st, const char* who) {
    cudaError_t e = cudaSuccess;
    auto out = [&](float* dst, size_t src, size_t n) {
        if (dst && e == cudaSuccess) e = cudaMemcpyAsync(dst, ws + src, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    };
    out(losses, tp.losses, (size_t)B * DELORA_LOSS_ROW);
    if (!normalized) out(T, tp.T16, (size_t)B * 16);
    out(pooled, tp.pooled, (size_t)B * 512);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// what _train_step and _train_eval refuse alike
int check_train_call(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* points,
                     const int32_t* n_points, int B, const void* workspace, const char* who) {
    if (check_train_desc(d, who)) return 1;
    if (check_train_params(hp, who)) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace, "%s: null pointer", who);
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "%s: B=%d outside [1, max_batch=%d]", who, B, d->max_batch);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) == 0u || d->w_pre > 0,
                     "%s: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0 (the reference's recipe: normals from the "
                     "unscaled points at H x w_pre), got w_pre=%d", who, d->w_pre);
    return 0;
}


// The group step's all-reduce schedule (delora_odometry_train_group_buckets): bucket k of kGroupBuckets in launch
// order, i.e. the backward's production order: heads + fc, layer4, layer3, layer2, stem + layer1.  Each boundary is a
// stage boundary rounded up to 4 floats, so a bucket may take up to 3 floats of the section after it in the blob (which
// the backward produced before it) and never one of the section before it (not produced yet).  The last bucket ends
// at most 3 floats past blob_floats, in the gradient section's 256-byte padding, which nothing reads.
static void plan_buckets(const Model& m, long long off[kGroupBuckets], long long cnt[kGroupBuckets]) {
    auto up4 = [](long long x) { return (x + 3) & ~3ll; };
    long long edge[kGroupBuckets + 1];            // stage starts in blob order: stem, layer2, layer3, layer4, fc, end
    edge[0] = 0;
    for (int s = 1; s < 4; ++s) {
        int i = 0;
        while (m.t.block[i].stage < s) ++i;
        edge[s] = up4(m.t.conv[m.t.block[i].c1].blob);
    }
    edge[4] = up4(m.fc.blob_w);
    edge[5] = up4(m.blob_floats);
    for (int k = 0; k < kGroupBuckets; ++k) {
        off[k] = edge[4 - k];
        cnt[k] = edge[5 - k] - edge[4 - k];
    }
}

int check_group(const delora_odometry_train_group* g, const void* workspace, const char* who) {
    DELORA_CHECK_ARG(g != nullptr, "%s: null group", who);
    DELORA_CHECK_ARG(g->world >= 1 && g->world <= kArMaxWorld, "%s: world=%d must be in [1, %d]", who, g->world,
                     kArMaxWorld);
    DELORA_CHECK_ARG(g->rank >= 0 && g->rank < g->world, "%s: rank=%d outside [0, world=%d)", who, g->rank, g->world);
    for (int q = 0; q < g->world; ++q) {
        DELORA_CHECK_ARG(g->peer_ws[q] != 0 && (g->peer_ws[q] & 15) == 0, "%s: peer_ws[%d] is null or not 16-byte aligned",
                         who, q);
        DELORA_CHECK_ARG(g->peer_flags[q] != 0 && (g->peer_flags[q] & 3) == 0,
                         "%s: peer_flags[%d] is null or not 4-byte aligned", who, q);
    }
    DELORA_CHECK_ARG(g->peer_ws[g->rank] == (uint64_t)(uintptr_t)workspace, "%s: peer_ws[rank=%d] is not the workspace",
                     who, g->rank);
    DELORA_CHECK_ARG((g->multicast & 15) == 0, "%s: multicast is not 16-byte aligned", who);
    DELORA_CHECK_ARG(g->status != nullptr, "%s: null status", who);
    DELORA_CHECK_ARG(g->n_ctas >= 1 && g->n_ctas <= kArMaxCtas, "%s: n_ctas=%d outside [1, %d]", who, g->n_ctas,
                     kArMaxCtas);
    DELORA_CHECK_ARG(g->n_threads >= 32 && g->n_threads <= kArMaxThreads && g->n_threads % 32 == 0,
                     "%s: n_threads=%d must be 32, 64, 96 or 128", who, g->n_threads);
    if (g->world > 1) {
        for (int k = 0; k < kGroupBuckets; ++k)
            DELORA_CHECK_ARG(g->fork_events[k] != nullptr, "%s: null fork_events[%d]", who, k);
        DELORA_CHECK_ARG(g->join_event != nullptr, "%s: null join_event", who);
    }
    return 0;
}

// Stage 4 of the step at B pairs: the tail backward (see train_tail_backward for identity, drop, valid and n_valid),
// then the trunk backward of stage 3 down to 0.  With gr, bucket k of plan_buckets' schedule is all-reduced in place in
// every rank's gradient section as soon as the backward has produced it on `st` (bucket 0 after the tail, bucket 4 - s
// after stage s): g->side_stream waits for it through fork_events[k] and runs the all-reduce, and `st` then waits for
// every bucket through join_event.
int step_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, DropoutCtr drop,
                  const int32_t* valid, const int32_t* n_valid, const GroupReduce* gr, cudaStream_t st,
                  const char* who) {
    const delora_odometry_train_group* g = gr ? gr->g : nullptr;
    cudaStream_t side = g ? (cudaStream_t)g->side_stream : nullptr;
    long long b_off[kGroupBuckets], b_cnt[kGroupBuckets];
    uint64_t peer_grad[kArMaxWorld];
    if (g) {
        plan_buckets(tp.m, b_off, b_cnt);
        for (int q = 0; q < g->world; ++q) peer_grad[q] = g->peer_ws[q] + tp.grad;
    }
    auto all_reduce = [&](int k) -> int {
        if (!g) return 0;
        cudaError_t e = cudaEventRecord((cudaEvent_t)g->fork_events[k], st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(side, (cudaEvent_t)g->fork_events[k], 0);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: fork_events[%d]: %s", who, k, cudaGetErrorString(e));
        return grad_allreduce_launch(peer_grad, g->peer_flags, g->multicast ? g->multicast + tp.grad : 0ull, g->rank,
                                     g->world, b_off[k], b_cnt[k], gr->scale, gr->seq_first + (unsigned)k, gr->seq_step,
                                     gr->seq_stride, g->n_ctas, g->n_threads, g->status, side);
    };
    int rc;
    if ((rc = train_tail_backward(tp, ws, act, B, identity, st, drop, valid, n_valid))) return rc;
    if ((rc = all_reduce(0))) return rc;
    float* conv_dw[kMaxConv];
    for (int i = 0; i < tp.m.t.n_conv; ++i) conv_dw[i] = reinterpret_cast<float*>(ws + tp.grad) + tp.m.t.conv[i].blob;
    const float* g_pooled = reinterpret_cast<const float*>(ws + tp.g_pooled);
    for (int s = 3; s >= 0; --s) {
        if ((rc = trunk_backward(tp.m.t, tp.t, ws, tp.w, ws, act, B, g_pooled, conv_dw, s, st, drop))) return rc;
        if ((rc = all_reduce(4 - s))) return rc;
    }
    if (!g) return 0;
    cudaError_t e = cudaEventRecord((cudaEvent_t)g->join_event, side);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, (cudaEvent_t)g->join_event, 0);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: join_event: %s", who, cudaGetErrorString(e));
    return 0;
}

// delora_odometry_train_step, and with g (world > 1) its group form: bucket k is all-reduced on g->side_stream once
// the backward has produced it, and `stream` joins g->side_stream before the gradient is read.
static int train_step(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                      const delora_odometry_train_group* g, const float* points, const int32_t* n_points, int B,
                      void* workspace, float* losses, float* T, float* pooled, float* grads, void* stream,
                      const char* who) {
    const bool normalized = (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u;
    const bool dropout = (hp->loss_flags & DELORA_TRAIN_DROPOUT) != 0u;
    const bool identity = (hp->loss_flags & DELORA_LOSS_IDENTITY_FIT) != 0u;
    TrainPlan tp;
    make_train_plan(d, &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    long long* ctr = reinterpret_cast<long long*>(ws + tp.ctr);
    // the masks of this step, regenerated after odometry_out_bwd_kernel has advanced the step count
    const DropoutCtr drop_bwd{dropout ? ctr : nullptr, 1};
    // the buckets are averaged; seq = the step count (advanced by odometry_out_bwd_kernel before bucket 0) *
    // kGroupBuckets + k
    const GroupReduce gr{g, g ? 1.0f / (float)g->world : 1.0f, ctr, (unsigned)kGroupBuckets, 0u};
    int rc;
    // 1-3. projection + normals, forward, ICP losses and dL/dT
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, B, dropout, T, st, who))) return rc;
    // 4. backward: tail (dL/dT of the ICP mean or of the identity fit), average pool, trunk
    if ((rc = step_backward(tp, ws, d->act, B, identity, drop_bwd, nullptr, nullptr, g ? &gr : nullptr, st, who)))
        return rc;
    // outputs (T: the weights before the update)
    if ((rc = train_outputs(tp, ws, B, normalized, losses, T, pooled, st, who))) return rc;
    if (grads) {
        const cudaError_t e = cudaMemcpyAsync(grads, ws + tp.grad, (size_t)tp.m.blob_floats * sizeof(float),
                                              cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    // 5. Adam on the master blob, then the bf16 filters from the updated weights
    return adam_update(tp, ws, hp, nullptr, st);
}

}  // namespace delora

extern "C" int delora_odometry_train_step(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                          const float* points, const int32_t* n_points, int B, void* workspace,
                                          float* losses, float* T, float* pooled, float* grads, void* stream) {
    const char* who = "delora_odometry_train_step";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    return train_step(d, hp, nullptr, points, n_points, B, workspace, losses, T, pooled, grads, stream, who);
}

extern "C" int delora_odometry_train_step_group(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                                const delora_odometry_train_group* g, const float* points,
                                                const int32_t* n_points, int B, void* workspace, float* losses,
                                                float* T, float* pooled, float* grads, void* stream) {
    const char* who = "delora_odometry_train_step_group";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    if (check_group(g, workspace, who)) return 1;
    return train_step(d, hp, g->world > 1 ? g : nullptr, points, n_points, B, workspace, losses, T, pooled, grads,
                      stream, who);
}

extern "C" int64_t delora_odometry_train_grad_offset(const delora_odometry_desc* d) {
    if (check_train_desc(d, "delora_odometry_train_grad_offset")) return -1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    return (int64_t)tp.grad;
}

extern "C" int delora_odometry_train_group_buckets(const delora_odometry_desc* d, int64_t* offsets, int64_t* counts) {
    const char* who = "delora_odometry_train_group_buckets";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(offsets && counts, "%s: null pointer", who);
    Model m;
    plan_model(d, &m);
    long long off[kGroupBuckets], cnt[kGroupBuckets];
    plan_buckets(m, off, cnt);
    for (int k = 0; k < kGroupBuckets; ++k) { offsets[k] = off[k]; counts[k] = cnt[k]; }
    return 0;
}

extern "C" int delora_odometry_train_eval(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                          const float* points, const int32_t* n_points, int B, void* workspace,
                                          float* losses, float* T, float* pooled, void* stream) {
    const char* who = "delora_odometry_train_eval";
    if (check_train_call(d, hp, points, n_points, B, workspace, who)) return 1;
    TrainPlan tp;
    make_train_plan(d, &tp);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    // dropout is the identity, as at inference; the identity fit's objective belongs to the step's backward
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, B, false, T, st, who))) return rc;
    if ((rc = record_icp_batch(tp, ws, B, st))) return rc;
    return train_outputs(tp, ws, B, (hp->loss_flags & DELORA_TRAIN_NORMALIZATION_SCALING) != 0u, losses, T, pooled, st,
                         who);
}

extern "C" int delora_odometry_train_weights(const delora_odometry_desc* d, const void* workspace, float* weights,
                                             void* stream) {
    const char* who = "delora_odometry_train_weights";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace && weights, "%s: null pointer", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    const cudaError_t e = cudaMemcpyAsync(weights, (const char*)workspace + tp.master, (size_t)tp.m.blob_floats * 4,
                                          cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_train_get_state(const delora_odometry_desc* d, const void* workspace, float* weights,
                                               float* exp_avg, float* exp_avg_sq, int64_t* step, void* stream) {
    const char* who = "delora_odometry_train_get_state";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    const char* ws = (const char*)workspace;
    const size_t blob = (size_t)tp.m.blob_floats * 4;
    cudaError_t e = cudaSuccess;
    auto out = [&](void* dst, size_t src, size_t bytes) {
        if (dst && e == cudaSuccess) e = cudaMemcpyAsync(dst, ws + src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
    };
    out(weights, tp.master, blob);
    out(exp_avg, tp.adam_m, blob);
    out(exp_avg_sq, tp.adam_v, blob);
    out(step, tp.ctr, sizeof(long long));
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

extern "C" int delora_odometry_train_set_state(const delora_odometry_desc* d, const float* weights, const float* exp_avg,
                                               const float* exp_avg_sq, const int64_t* step, void* workspace,
                                               void* stream) {
    const char* who = "delora_odometry_train_set_state";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(weights, "%s: null weights", who);
    DELORA_CHECK_ARG(exp_avg, "%s: null exp_avg", who);
    DELORA_CHECK_ARG(exp_avg_sq, "%s: null exp_avg_sq", who);
    DELORA_CHECK_ARG(step, "%s: null step", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    char* ws = (char*)workspace;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t blob = (size_t)tp.m.blob_floats * 4;
    cudaError_t e = cudaSuccess;
    auto in = [&](size_t dst, const void* src, size_t bytes) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(ws + dst, src, bytes, cudaMemcpyDeviceToDevice, st);
    };
    in(tp.master, weights, blob);
    in(tp.adam_m, exp_avg, blob);
    in(tp.adam_v, exp_avg_sq, blob);
    in(tp.ctr, step, sizeof(long long));            // ctr[0] only: ctr[1], the ICP scratch's batch size, stays
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    // the bf16 filters from the new master weights, through the table _train_init wrote
    return delora_conv_weight_prep_multi(ws + tp.w.table, tp.m.t.n_conv, st);
}

namespace delora {

__global__ void odometry_set_seed_kernel(long long* __restrict__ ctr, unsigned long long seed) {
    ctr[2] = (long long)seed;
}

// keep[i] = 1 if element i of tensor t is kept at (seed, step), else 0; one thread per 4 elements (one Philox block)
__global__ void __launch_bounds__(256)
dropout_keep_mask_kernel(unsigned long long seed, unsigned long long step, int t, long long n, uint8_t* __restrict__ keep) {
    const long long q = (long long)blockIdx.x * 256 + threadIdx.x;
    if (q * 4 >= n) return;
    const Philox4 r = dropout_words(seed, step, t, (uint64_t)q);
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (q * 4 + k < n) keep[q * 4 + k] = dropout_word_keeps(philox_word(r, k)) ? 1 : 0;
}

}  // namespace delora

extern "C" int delora_odometry_train_set_dropout_seed(const delora_odometry_desc* d, uint64_t seed, void* workspace,
                                                      void* stream) {
    const char* who = "delora_odometry_train_set_dropout_seed";
    if (check_train_desc(d, who)) return 1;
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    TrainPlan tp;
    make_train_plan(d, &tp);
    odometry_set_seed_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<long long*>((char*)workspace + tp.ctr),
                                                                (unsigned long long)seed);
    DELORA_CHECK_LAUNCH("odometry_set_seed_kernel");
    return 0;
}

extern "C" int delora_dropout_keep_mask(uint64_t seed, int64_t step, int tensor, int64_t n, uint8_t* keep, void* stream) {
    const char* who = "delora_dropout_keep_mask";
    DELORA_CHECK_ARG(keep, "%s: null keep", who);
    DELORA_CHECK_ARG(n >= 0, "%s: n=%lld must be >= 0", who, (long long)n);
    DELORA_CHECK_ARG(tensor >= 0 && tensor <= 2, "%s: tensor=%d must be 0 (input), 1 (stage-3 channels) or 2 (fc output)",
                     who, tensor);
    if (n == 0) return 0;
    const long long blocks = ((n + 3) / 4 + 255) / 256;
    dropout_keep_mask_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(seed, (unsigned long long)step, tensor, n,
                                                                                keep);
    DELORA_CHECK_LAUNCH("dropout_keep_mask_kernel");
    return 0;
}
