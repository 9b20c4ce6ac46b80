// The adapting streams (sm_90a): streams workspaces that adapt the model while serving it.
//
// delora_odometry_streams_push_adapt: S = max_batch streams served from a training workspace, which takes the training
// step on the pairs it has just served.  The workspace is the training layout of d (max_batch = S) followed by the
// stream section; no training offset moves, so every delora_odometry_train_* entry point works on it unchanged.  Its
// group form sums the update over several GPUs, its information form also serves each frame's ICP information.
//
// delora_odometry_streams_push_adapt_geometries: one model adapted from the streams of n geometries in one workspace.
// Layout: the adapting-streams workspace of d[0], unchanged; then for g = 1 .. n-1 d[g]'s geometry section (its
// training plan with the geometry section at the running offset), its stream section and one gradient slice in blob
// layout; then, for n > 1, the fleet section: the count of valid pairs over every geometry (int32 at +0) and geometry
// g's counters at +8 + 24 (g - 1), in the layout of the model section's (int64 [3]: a backward count nothing reads,
// the batch marker of g's ICP scratch, unused).  Geometry g's plan keeps d[0]'s model-section offsets (check_geometries
// makes them equal) with grad and ctr moved to its slice and counters, so train_forward_losses and step_backward run
// on it unchanged, and geometry 0's plan is _push_adapt's.  The _adapt_geometries_info form appends the information
// section after all of that (see make_geometries_plan), so no other offset moves.
#include <stdio.h>
#include <string.h>

#include <memory>

#include "odometry.cuh"

namespace delora {

struct AdaptPlan {
    size_t cache_image;                // w_pre = 0 only: [S, 4, H, W]
    size_t cache_pts, cache_nrm;       // [S, H, W] (w_pre = 0) or [S, H, w_pre]
    size_t has_prev, n_valid;          // [S], [1]
    size_t cache_cells;                // cells of one stream's cached grid
    size_t total;
    // The group section of delora_odometry_streams_push_adapt_group, one 256-byte block after the adapting-streams
    // layout: the tick counter (int64: group ticks with update = 1 so far), the fleet-wide count of valid pairs of the
    // last such tick (int32) and the count exchange's slots (int32 [2][kArMaxWorld], see count_allreduce_kernel).
    size_t tick, n_fleet, slots;
    size_t group_total;
    // The information section of delora_odometry_streams_push_adapt_info / _group_info, after the group section: the
    // information rows of the S pairs and the operator's info_scratch at B = S
    size_t info, info_scratch;
    size_t info_total;
};

// geometry_at: see make_train_plan; the stream section follows the geometry section wherever that starts
static void make_adapt_plan(const delora_odometry_desc* d, TrainPlan* tp, AdaptPlan* ap, size_t geometry_at = 0) {
    make_train_plan(d, tp, geometry_at);
    memset(ap, 0, sizeof(AdaptPlan));
    const size_t S = (size_t)d->max_batch, HW = (size_t)d->H * d->W;
    size_t off = tp->total;
    ap->cache_cells = d->w_pre > 0 ? (size_t)d->H * d->w_pre : HW;
    if (d->w_pre == 0) ap->cache_image = take(off, S * 4 * HW * 4);
    ap->cache_pts = take(off, S * ap->cache_cells * 16);
    ap->cache_nrm = take(off, S * ap->cache_cells * 16);
    ap->has_prev = take(off, S * 4);
    ap->n_valid = take(off, 4);
    ap->total = off;
    const size_t base = take(off, 8 + 8 + 2 * kArMaxWorld * 4);
    ap->tick = base;
    ap->n_fleet = base + 8;
    ap->slots = base + 16;
    ap->group_total = off;
    ap->info = take(off, S * DELORA_INFO_ROW * 4);
    ap->info_scratch = take(off, (size_t)delora_icp_information_scratch_floats(d->max_batch, d->H, d->W) * 4);
    ap->info_total = off;
}

// The adapting-streams workspace forms: _adapt (total), _adapt_group (group_total), _adapt_info (info_total)
enum class Adapt { plain, group, info };

static size_t adapt_bytes(const AdaptPlan& ap, Adapt form) {
    return form == Adapt::info ? ap.info_total : form == Adapt::group ? ap.group_total : ap.total;
}

// The adapting-streams workspace's size in one of its forms
static int64_t adapt_workspace_bytes(const delora_odometry_desc* d, Adapt form, const char* who) {
    if (check_train_desc(d, who)) return -1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    return (int64_t)adapt_bytes(ap, form);
}

// _streams_adapt_init, _streams_adapt_group_init and _streams_adapt_info_init; the group and information sections are
// zeroed too, and the forms with a group section preload the collective kernels
static int adapt_init(const delora_odometry_desc* d, Adapt form, const float* weights, void* workspace, cudaStream_t st,
                      const char* who) {
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    // _train_init over the whole workspace zeroes the stream section too; the cached grids then start empty
    int rc = train_init(d, adapt_bytes(ap, form), weights, workspace, st, who);
    if (rc) return rc;
    if ((rc = clear_grids((char*)workspace, ap.cache_pts, ap.cache_nrm, (size_t)d->max_batch * ap.cache_cells, st)))
        return rc;
    return form != Adapt::plain ? collective_kernels_preload(who) : 0;
}

// The hyperparameters and update value every adapting tick refuses alike
static int check_adapt_params(const delora_odometry_train_params* hp, int update, const char* who) {
    if (check_train_params(hp, who)) return 1;
    DELORA_CHECK_ARG(update == 0 || update == 1, "%s: update=%d must be 0 or 1", who, update);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_LOSS_IDENTITY_FIT) == 0u,
                     "%s: loss_flags=0x%x has DELORA_LOSS_IDENTITY_FIT, a pre-training phase, not adaptation", who,
                     hp->loss_flags);
    DELORA_CHECK_ARG((hp->loss_flags & DELORA_TRAIN_DROPOUT) == 0u,
                     "%s: loss_flags=0x%x has DELORA_TRAIN_DROPOUT: the served T is dropout-free, and one forward "
                     "cannot be both", who, hp->loss_flags);
    return 0;
}

// What _push_adapt and _push_adapt_group refuse alike
static int check_push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp, int update,
                            const float* points, const int32_t* n_points, void* workspace, float* T, int32_t* valid,
                            float* losses, const char* who) {
    if (check_train_desc(d, who)) return 1;
    if (check_adapt_params(hp, update, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    return check_train_call(d, hp, points, n_points, d->max_batch, workspace, who);
}

// Stages 1-3 of one adapting tick of the S = d->max_batch streams of (tp, ap): T, valid, the loss rows and the cache
// write, with info (an information workspace) the information rows at the served T; update = 0 then records the ICP
// scratch's batch marker
static int serve_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const TrainPlan& tp,
                       const AdaptPlan& ap, int update, const float* points, const int32_t* n_points,
                       const int32_t* active, char* ws, float* T, int32_t* valid, float* losses, float* info,
                       cudaStream_t st, const char* who) {
    const int S = d->max_batch;
    auto f = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
    AdaptTick at;
    at.active = active;
    at.T = T;
    at.valid = valid;
    at.has_prev = reinterpret_cast<int32_t*>(ws + ap.has_prev);
    at.n_valid = reinterpret_cast<int32_t*>(ws + ap.n_valid);
    at.cache_image = d->w_pre == 0 ? f(ap.cache_image) : nullptr;
    at.cache_pts = reinterpret_cast<delora_f4*>(ws + ap.cache_pts);
    at.cache_nrm = reinterpret_cast<delora_f4*>(ws + ap.cache_nrm);
    at.info = info ? f(ap.info) : nullptr;
    at.info_scratch = info ? f(ap.info_scratch) : nullptr;
    int rc;
    // 1-3 at B = S, the first frame of every pair from the cache; T, valid, the cache and the emptied sources
    if ((rc = train_forward_losses(d, hp, tp, ws, points, n_points, S, false, nullptr, st, who, &at))) return rc;
    if ((rc = streams_rows_out(DELORA_LOSS_ROW, valid, S, f(tp.losses), losses, st))) return rc;
    if (info && (rc = streams_rows_out(DELORA_INFO_ROW, valid, S, f(ap.info), info, st))) return rc;
    // update = 0: the ICP scratch now has the layout of S pairs, as after _train_eval
    return update ? 0 : record_icp_batch(tp, ws, S, st);
}

// One tick of _push_adapt, and with g (world > 1, update = 1) of its group form: the count of valid pairs is
// exchanged (collective k = 0) before the backward, which then divides by the fleet-wide count; the gradient buckets
// are summed over the ranks on g->side_stream (collectives k = 1 .. kGroupBuckets); Adam runs where that count is > 0.
// The group's sequence numbers come from its tick counter, seq = tick * (kGroupBuckets + 1) + k, which advances on
// every group tick with update = 1, so a tick without a valid pair still takes new numbers.
// info non-NULL: an information workspace (_push_adapt_info / _push_adapt_group_info).
static int push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                      const delora_odometry_train_group* g, int update, const float* points, const int32_t* n_points,
                      const int32_t* active, void* workspace, float* T, int32_t* valid, float* losses, float* info,
                      void* stream, const char* who) {
    const int S = d->max_batch;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    if ((rc = serve_adapt(d, hp, tp, ap, update, points, n_points, active, ws, T, valid, losses, info, st, who)))
        return rc;
    if (!update) return 0;
    const int32_t* n_valid = reinterpret_cast<const int32_t*>(ws + ap.n_valid);
    long long* tick = reinterpret_cast<long long*>(ws + ap.tick);
    constexpr unsigned kSeqStride = kGroupBuckets + 1;
    if (g) {                // the fleet-wide count of valid pairs, on every rank before its backward
        uint64_t peer_slots[kArMaxWorld];
        for (int q = 0; q < g->world; ++q) peer_slots[q] = g->peer_ws[q] + ap.slots;
        int32_t* n_fleet = reinterpret_cast<int32_t*>(ws + ap.n_fleet);
        if ((rc = count_allreduce_launch(peer_slots, g->peer_flags, g->rank, g->world, kSeqStride, tick, n_valid,
                                         n_fleet, g->status, st))) return rc;
        n_valid = n_fleet;
    }
    // each rank divides by the fleet-wide count, so the buckets are summed (scale 1)
    const GroupReduce gr{g, 1.0f, tick, kSeqStride, 1u};
    // 4. the backward of the mean over the valid pairs (invalid rows: dL/dT = 0), then Adam where n_valid > 0
    if ((rc = step_backward(tp, ws, d->act, S, false, DropoutCtr{nullptr, 0}, valid, n_valid, g ? &gr : nullptr, st,
                            who))) return rc;
    return adam_update(tp, ws, hp, n_valid, st);
}

}  // namespace delora

using namespace delora;

extern "C" int64_t delora_odometry_streams_adapt_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::plain, "delora_odometry_streams_adapt_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_init(const delora_odometry_desc* d, const float* weights, void* workspace,
                                                  void* stream) {
    return adapt_init(d, Adapt::plain, weights, workspace, (cudaStream_t)stream, "delora_odometry_streams_adapt_init");
}

extern "C" int delora_odometry_streams_push_adapt(const delora_odometry_desc* d, const delora_odometry_train_params* hp,
                                                  int update, const float* points, const int32_t* n_points,
                                                  const int32_t* active, void* workspace, float* T, int32_t* valid,
                                                  float* losses, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    return push_adapt(d, hp, nullptr, update, points, n_points, active, workspace, T, valid, losses, nullptr, stream,
                      who);
}

extern "C" int64_t delora_odometry_streams_adapt_group_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::group, "delora_odometry_streams_adapt_group_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_group_init(const delora_odometry_desc* d, const float* weights,
                                                        void* workspace, void* stream) {
    return adapt_init(d, Adapt::group, weights, workspace, (cudaStream_t)stream, "delora_odometry_streams_adapt_group_init");
}

extern "C" int delora_odometry_streams_push_adapt_group(const delora_odometry_desc* d,
                                                        const delora_odometry_train_params* hp,
                                                        const delora_odometry_train_group* g, int update,
                                                        const float* points, const int32_t* n_points,
                                                        const int32_t* active, void* workspace, float* T,
                                                        int32_t* valid, float* losses, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_group";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    if (check_group(g, workspace, who)) return 1;
    return push_adapt(d, hp, g->world > 1 && update ? g : nullptr, update, points, n_points, active, workspace, T,
                      valid, losses, nullptr, stream, who);
}

extern "C" int64_t delora_odometry_streams_adapt_info_workspace_bytes(const delora_odometry_desc* d) {
    return adapt_workspace_bytes(d, Adapt::info, "delora_odometry_streams_adapt_info_workspace_bytes");
}

extern "C" int delora_odometry_streams_adapt_info_init(const delora_odometry_desc* d, const float* weights,
                                                       void* workspace, void* stream) {
    return adapt_init(d, Adapt::info, weights, workspace, (cudaStream_t)stream,
                      "delora_odometry_streams_adapt_info_init");
}

extern "C" int delora_odometry_streams_push_adapt_info(const delora_odometry_desc* d,
                                                       const delora_odometry_train_params* hp, int update,
                                                       const float* points, const int32_t* n_points,
                                                       const int32_t* active, void* workspace, float* T,
                                                       int32_t* valid, float* losses, float* info, void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_info";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return push_adapt(d, hp, nullptr, update, points, n_points, active, workspace, T, valid, losses, info, stream,
                      who);
}

extern "C" int delora_odometry_streams_push_adapt_group_info(const delora_odometry_desc* d,
                                                             const delora_odometry_train_params* hp,
                                                             const delora_odometry_train_group* g, int update,
                                                             const float* points, const int32_t* n_points,
                                                             const int32_t* active, void* workspace, float* T,
                                                             int32_t* valid, float* losses, float* info,
                                                             void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_group_info";
    if (check_push_adapt(d, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    if (check_group(g, workspace, who)) return 1;
    return push_adapt(d, hp, g->world > 1 && update ? g : nullptr, update, points, n_points, active, workspace, T,
                      valid, losses, info, stream, who);
}

extern "C" int delora_odometry_streams_adapt_reset(const delora_odometry_desc* d, const int32_t* mask, void* workspace,
                                                   void* stream) {
    const char* who = "delora_odometry_streams_adapt_reset";
    if (check_train_desc(d, who)) return 1;
    TrainPlan tp;
    AdaptPlan ap;
    make_adapt_plan(d, &tp, &ap);
    return reset_streams(d, mask, workspace, ap.has_prev, stream, who);
}

namespace delora {

struct GeometriesPlan {
    TrainPlan tp[kMaxGeometries];
    AdaptPlan ap[kMaxGeometries];
    int row[kMaxGeometries];           // the first stream of geometry g in the caller's arrays
    size_t fleet;                      // n > 1 only
    size_t total;
    size_t info_total;                 // with the information section of _push_adapt_geometries_info
};

// TrainPlan is large (the trunk plan's tables): the plans of up to kMaxGeometries geometries go on the heap
static std::unique_ptr<GeometriesPlan> make_geometries_plan(const delora_odometry_desc* d, int n) {
    std::unique_ptr<GeometriesPlan> p(new GeometriesPlan);
    make_adapt_plan(&d[0], &p->tp[0], &p->ap[0]);
    size_t off = p->ap[0].total;
    p->row[0] = 0;
    for (int g = 1; g < n; ++g) {
        make_adapt_plan(&d[g], &p->tp[g], &p->ap[g], off);
        off = p->ap[g].total;
        p->tp[g].grad = take(off, (size_t)p->tp[g].m.blob_floats * 4);
        p->row[g] = p->row[g - 1] + d[g - 1].max_batch;
    }
    p->fleet = 0;
    if (n > 1) {
        p->fleet = take(off, 8 + 24 * (size_t)(n - 1));
        for (int g = 1; g < n; ++g) p->tp[g].ctr = p->fleet + 8 + 24 * (size_t)(g - 1);
    }
    p->total = off;
    // the information section of _push_adapt_geometries_info: the rows of all S_total pairs, then one info_scratch
    // sized for the largest geometry (their ICPs run one after another on one stream, and the scratch needs no
    // initialisation).  make_adapt_plan put ap.info / ap.info_scratch after a single-geometry group section, which here
    // lies in the next geometry's sections: every geometry's, g = 0 included, are moved into this section
    const size_t rows = take(off, (size_t)(p->row[n - 1] + d[n - 1].max_batch) * DELORA_INFO_ROW * 4);
    int64_t scratch = 0;
    for (int g = 0; g < n; ++g) {
        const int64_t floats = delora_icp_information_scratch_floats(d[g].max_batch, d[g].H, d[g].W);
        if (floats > scratch) scratch = floats;
    }
    const size_t info_scratch = take(off, (size_t)scratch * 4);
    for (int g = 0; g < n; ++g) {
        p->ap[g].info = rows + (size_t)p->row[g] * DELORA_INFO_ROW * 4;
        p->ap[g].info_scratch = info_scratch;
    }
    p->info_total = off;
    return p;
}

static int check_adapt_geometries(const delora_odometry_desc* d, int n, const char* who) {
    DELORA_CHECK_ARG(n <= kMaxGeometries, "%s: n=%d must be <= %d", who, n, kMaxGeometries);
    return check_geometries(d, n, who);
}

struct FleetCounts {
    const int32_t* n_valid[kMaxGeometries];
    int n;
};

// *fleet = the sum of every geometry's count of valid pairs, in geometry order
__global__ void odometry_fleet_count_kernel(FleetCounts c, int32_t* __restrict__ fleet) {
    int s = 0;
    for (int g = 0; g < c.n; ++g) s += *c.n_valid[g];
    *fleet = s;
}

// One tick of _push_adapt_geometries; info non-NULL: of _push_adapt_geometries_info, each geometry's information rows
// into its rows of info
static int push_adapt_geometries(const delora_odometry_desc* d, int n, const delora_odometry_train_params* hp,
                                 int update, const float* const* points, const int32_t* const* n_points,
                                 const int32_t* active, void* workspace, float* T, int32_t* valid, float* losses,
                                 float* info, void* stream, const char* who) {
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    int rc;
    // 1-3 per geometry at B = S_g into its rows of the caller's arrays
    for (int g = 0; g < n; ++g) {
        const int r = p->row[g];
        if ((rc = serve_adapt(&d[g], hp, p->tp[g], p->ap[g], update, points[g], n_points[g], active ? active + r : nullptr,
                              ws, T + (size_t)r * 16, valid + r, losses + (size_t)r * DELORA_LOSS_ROW,
                              info ? info + (size_t)r * DELORA_INFO_ROW : nullptr, st, who)))
            return rc;
    }
    if (!update) return 0;
    // 4. every geometry's backward divides by the fleet's count of valid pairs, geometry g >= 1 into its slice; Adam
    // sums the slices into the model's gradient section
    const int32_t* fleet = reinterpret_cast<const int32_t*>(ws + p->ap[0].n_valid);
    GradSlices more;
    memset(&more, 0, sizeof(more));
    if (n > 1) {
        FleetCounts c;
        memset(&c, 0, sizeof(c));
        c.n = n;
        for (int g = 0; g < n; ++g) c.n_valid[g] = reinterpret_cast<const int32_t*>(ws + p->ap[g].n_valid);
        odometry_fleet_count_kernel<<<1, 1, 0, st>>>(c, reinterpret_cast<int32_t*>(ws + p->fleet));
        DELORA_CHECK_LAUNCH("odometry_fleet_count_kernel");
        fleet = reinterpret_cast<const int32_t*>(ws + p->fleet);
        more.n = n - 1;
        for (int g = 1; g < n; ++g) more.g[g - 1] = reinterpret_cast<const float*>(ws + p->tp[g].grad);
    }
    for (int g = 0; g < n; ++g)
        if ((rc = step_backward(p->tp[g], ws, d[g].act, d[g].max_batch, false, DropoutCtr{nullptr, 0}, valid + p->row[g],
                                fleet, nullptr, st, who))) return rc;
    return adam_update(p->tp[0], ws, hp, fleet, st, &more);
}

}  // namespace delora

extern "C" int64_t delora_odometry_streams_adapt_geometries_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_adapt_geometries(d, n, "delora_odometry_streams_adapt_geometries_workspace_bytes")) return -1;
    return (int64_t)make_geometries_plan(d, n)->total;
}

extern "C" int delora_odometry_streams_adapt_geometries_init(const delora_odometry_desc* d, int n, const float* weights,
                                                             void* workspace, void* stream) {
    const char* who = "delora_odometry_streams_adapt_geometries_init";
    if (check_adapt_geometries(d, n, who)) return 1;
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    // _train_init over the whole workspace arms geometry 0 and zeroes every other section
    int rc = train_init(&d[0], p->total, weights, workspace, st, who);
    if (rc) return rc;
    for (int g = 0; g < n; ++g) {
        const AdaptPlan& ap = p->ap[g];
        if ((rc = clear_grids(ws, ap.cache_pts, ap.cache_nrm, (size_t)d[g].max_batch * ap.cache_cells, st))) return rc;
        if (g == 0) continue;
        const cudaError_t e = cudaMemsetAsync(ws + p->tp[g].f.keys, 0xFF, p->tp[g].f.keys_bytes, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    return 0;
}

namespace delora {

// What _push_adapt_geometries and _push_adapt_geometries_info refuse alike
static int check_push_adapt_geometries(const delora_odometry_desc* d, int n, const delora_odometry_train_params* hp,
                                       int update, const float* const* points, const int32_t* const* n_points,
                                       void* workspace, float* T, int32_t* valid, float* losses, const char* who) {
    if (check_adapt_geometries(d, n, who)) return 1;
    if (check_adapt_params(hp, update, who)) return 1;
    if (check_tick(points, n_points, workspace, T, valid, losses, "losses", who)) return 1;
    for (int g = 0; g < n; ++g) {
        DELORA_CHECK_ARG(points[g], "%s: points[%d] is null", who, g);
        DELORA_CHECK_ARG(n_points[g], "%s: n_points[%d] is null", who, g);
        char w[192];
        snprintf(w, sizeof w, "%s: d[%d]", who, g);
        if (check_train_call(&d[g], hp, points[g], n_points[g], d[g].max_batch, workspace, w)) return 1;
    }
    return 0;
}

}  // namespace delora

extern "C" int delora_odometry_streams_push_adapt_geometries(const delora_odometry_desc* d, int n,
                                                             const delora_odometry_train_params* hp, int update,
                                                             const float* const* points,
                                                             const int32_t* const* n_points, const int32_t* active,
                                                             void* workspace, float* T, int32_t* valid, float* losses,
                                                             void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_geometries";
    if (check_push_adapt_geometries(d, n, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    return push_adapt_geometries(d, n, hp, update, points, n_points, active, workspace, T, valid, losses, nullptr,
                                 stream, who);
}

extern "C" int64_t delora_odometry_streams_adapt_geometries_info_workspace_bytes(const delora_odometry_desc* d, int n) {
    if (check_adapt_geometries(d, n, "delora_odometry_streams_adapt_geometries_info_workspace_bytes")) return -1;
    return (int64_t)make_geometries_plan(d, n)->info_total;
}

extern "C" int delora_odometry_streams_push_adapt_geometries_info(const delora_odometry_desc* d, int n,
                                                                  const delora_odometry_train_params* hp, int update,
                                                                  const float* const* points,
                                                                  const int32_t* const* n_points,
                                                                  const int32_t* active, void* workspace, float* T,
                                                                  int32_t* valid, float* losses, float* info,
                                                                  void* stream) {
    const char* who = "delora_odometry_streams_push_adapt_geometries_info";
    if (check_push_adapt_geometries(d, n, hp, update, points, n_points, workspace, T, valid, losses, who)) return 1;
    DELORA_CHECK_ARG(info, "%s: null info", who);
    return push_adapt_geometries(d, n, hp, update, points, n_points, active, workspace, T, valid, losses, info, stream,
                                 who);
}

extern "C" int delora_odometry_streams_adapt_geometries_reset(const delora_odometry_desc* d, int n, const int32_t* mask,
                                                              void* workspace, void* stream) {
    const char* who = "delora_odometry_streams_adapt_geometries_reset";
    if (check_adapt_geometries(d, n, who)) return 1;
    DELORA_CHECK_ARG(mask, "%s: null mask", who);
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    for (int g = 0; g < n; ++g) {
        const int rc = reset_streams(&d[g], mask + p->row[g], workspace, p->ap[g].has_prev, stream, who);
        if (rc) return rc;
    }
    return 0;
}

namespace delora {

// One adapting-streams plan's stream section
static void map_adapt_streams(SectionMap& s, const delora_odometry_desc* d, const AdaptPlan& ap) {
    if (d->w_pre == 0) s.field("cache_image", ap.cache_image, DELORA_WS_STATE);
    s.field("cache_pts", ap.cache_pts, DELORA_WS_STATE);
    s.field("cache_nrm", ap.cache_nrm, DELORA_WS_STATE);
    s.field("has_prev", ap.has_prev, DELORA_WS_STATE);
    s.field("n_valid", ap.n_valid, DELORA_WS_SCRATCH);
}

// DELORA_WS_ADAPT*.  Offsets a plan sets but its kind never reads, left out:
//   - _adapt: ap.tick / n_fleet / slots lie past the end of the workspace.  push_adapt forms the tick pointer on every
//     update tick but dereferences it, n_fleet and slots only with a group, which only _push_adapt_group and
//     _push_adapt_group_info pass (and only with world > 1), on the _adapt_group / _adapt_info workspaces.
//   - _adapt and _adapt_group: ap.info / info_scratch lie past the end.  serve_adapt reads them only with info
//     non-NULL, which only _push_adapt_info and _push_adapt_group_info pass.
//   - _adapt_geometries*, geometry g >= 1: ap[g].tick / n_fleet / slots lie inside g's gradient slice (which
//     make_geometries_plan takes at the same offset); push_adapt_geometries passes no group to anything.  ap[g].info /
//     info_scratch, moved into the information section, lie past the end of the _adapt_geometries form, where
//     serve_adapt reads them only with info (only _push_adapt_geometries_info passes it).  tp[g].adam_m / adam_v are
//     geometry 0's: adam_update runs on tp[0] alone.
// Geometry g >= 1's counters are its fleet slot: [0] advances on every update tick and nothing reads it, [1] only
// decides whether its next ICP re-arms the scratch, so they are scratch, not state.
int map_adapt(SectionMap& s, const delora_odometry_desc* d, int n, int kind, const char* who) {
    if (kind == DELORA_WS_ADAPT || kind == DELORA_WS_ADAPT_GROUP || kind == DELORA_WS_ADAPT_INFO) {
        if (check_train_desc(d, who)) return 1;
        TrainPlan tp;
        AdaptPlan ap;
        make_adapt_plan(d, &tp, &ap);
        map_train(s, d, tp, true, DELORA_WS_STATE, 0, 0);
        map_adapt_streams(s, d, ap);
        if (kind == DELORA_WS_ADAPT) return 0;
        s.range("tick", ap.tick, 8, DELORA_WS_STATE);
        s.range("n_fleet", ap.n_fleet, 4, DELORA_WS_SCRATCH);
        s.range("slots", ap.slots, 2 * kArMaxWorld * 4, DELORA_WS_STATE);
        if (kind == DELORA_WS_ADAPT_INFO) {
            s.field("info", ap.info, DELORA_WS_OUTPUT);
            s.field("info_scratch", ap.info_scratch, DELORA_WS_SCRATCH);
        }
        return 0;
    }
    if (check_adapt_geometries(d, n, who)) return 1;
    const std::unique_ptr<GeometriesPlan> p = make_geometries_plan(d, n);
    for (int g = 0; g < n; ++g) {
        s.geometry = g;
        map_train(s, &d[g], p->tp[g], g == 0, g == 0 ? DELORA_WS_STATE : DELORA_WS_SCRATCH, DELORA_WS_SHARED, 0);
        map_adapt_streams(s, &d[g], p->ap[g]);
        if (g == 0 && n > 1) s.range("fleet", p->fleet, 4, DELORA_WS_SCRATCH);      // the fleet count of valid pairs
        if (kind != DELORA_WS_ADAPT_GEOMETRIES_INFO) continue;
        s.range("info", p->ap[g].info, (size_t)d[g].max_batch * DELORA_INFO_ROW * 4, DELORA_WS_OUTPUT);
        s.flags = DELORA_WS_SHARED;
        s.field("info_scratch", p->ap[g].info_scratch, DELORA_WS_SCRATCH);
        s.flags = 0;
    }
    return 0;
}

}  // namespace delora
