// Odometry inference through the C ABI (sm_90a): raw scans -> relative transforms in one call.
//
// Projection, then the encoder trunk of trunk.cuh (the one the Python encoder runs too), then the fully connected tail
// of odometry_tail.cu.  This file holds what every odometry workspace builds on (declared in odometry.cuh): the model
// plan, the descriptor and ICP-setting checks, the frame section, the inference plan, workspace init, weight loading
// and the projection; and the entry points of the pairs / push workspace (delora_odometry_pairs, _pairs_normalized,
// _push).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "odometry.cuh"
#include "projection.cuh"

namespace delora {

// counts[i] = active ? clamp(n_points[i], 0, n_stride) : 0 (active NULL: every scan is): the projection never reads
// past a scan's stride, and an inactive stream's scatter does no work
__global__ void odometry_counts_kernel(const int32_t* __restrict__ n_in, const int32_t* __restrict__ active, int n,
                                       int n_stride, int32_t* __restrict__ n_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) n_out[i] = stream_active(active, i) ? min(max(n_in[i], 0), n_stride) : 0;
}

int check_desc(const delora_odometry_desc* d, const char* who) {
    DELORA_CHECK_ARG(d != nullptr, "%s: null descriptor", who);
    DELORA_CHECK_ARG((long long)d->H * d->W < (1ll << 27), "%s: bad image size H=%d W=%d", who, d->H, d->W);
    if (check_trunk(d->layers, d->H, d->W, who)) return 1;
    DELORA_CHECK_ARG(d->n_stride >= 1, "%s: n_stride=%d must be >= 1", who, d->n_stride);
    DELORA_CHECK_ARG(d->max_batch >= 1 && d->max_batch <= kMaxBatch, "%s: max_batch=%d must be in [1, %d]", who,
                     d->max_batch, kMaxBatch);
    DELORA_CHECK_ARG(d->act == 1 || d->act == 2, "%s: act=%d must be 1 (relu) or 2 (tanh)", who, d->act);
    DELORA_CHECK_ARG(d->resnet_outputs >= 1 && d->resnet_outputs <= 65536, "%s: resnet_outputs=%d must be in [1, 65536]",
                     who, d->resnet_outputs);
    DELORA_CHECK_ARG(d->single_mlp == 0 || d->single_mlp == 1, "%s: single_mlp=%d must be 0 or 1", who, d->single_mlp);
    DELORA_CHECK_ARG(isfinite(d->hfov0) && isfinite(d->hfov1) && isfinite(d->vfov0) && isfinite(d->vfov1) &&
                     d->hfov1 > d->hfov0 && d->vfov1 > d->vfov0, "%s: bad field of view", who);
    return 0;
}

// Walks the model in state_dict order (src/models/resnet_modified.py:49-66 + model.py:58-84).  A pure function of the
// descriptor.
void plan_model(const delora_odometry_desc* d, Model* m) {
    memset(m, 0, sizeof(Model));
    plan_trunk(d->layers, d->H, d->W, &m->t);
    int64_t blob = m->t.conv_floats;
    auto add_lin = [&](Linear& l, int K, int N) {
        l.K = K; l.N = N; l.blob_w = blob; blob += (int64_t)K * N; l.blob_b = blob; blob += N;
    };
    const int nout = d->resnet_outputs;
    add_lin(m->fc, 512, nout);
    if (d->single_mlp) {
        static const int dims[6] = {0, 512, 512, 256, 64, 7};
        int k = nout;
        for (int i = 1; i < 6; ++i) { add_lin(m->lin[m->n_lin++], k, dims[i]); k = dims[i]; }
    } else {
        add_lin(m->lin[0], nout, kHeadHidden); add_lin(m->lin[1], kHeadHidden, 4);     // fully_connected_rotation
        add_lin(m->lin[2], nout, kHeadHidden); add_lin(m->lin[3], kHeadHidden, 3);     // fully_connected_translation
        m->n_lin = 4;
    }
    m->blob_floats = blob;
}

// ---------------------------------------------------------------- workspace sections
// Each workspace kind (pairs / push, streams, training) has a plan: the Model plus the byte offsets of its own
// layout, built from the frame section and the trunk's sections.  Every buffer starts on a 256-byte boundary.

Frames plan_frames(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, int key_w,
                   size_t& off) {
    const size_t HW = (size_t)d->H * d->W;
    Frames f;
    memset(&f, 0, sizeof(f));
    f.keys_bytes = (size_t)n_scans * d->H * key_w * 8;
    f.keys = take(off, f.keys_bytes);
    f.index_map = take(off, (size_t)n_scans * HW * 4);
    f.counts = take(off, (size_t)n_scans * 4);
    f.images = take(off, (size_t)n_scans * 4 * HW * 4);
    if (n_cached > 0) f.prev_image = take(off, (size_t)n_cached * 4 * HW * 4);
    if (has_prev) f.has_prev = take(off, (size_t)n_cached * 4);
    return f;
}

// The frame section (see plan_frames), then the trunk and tail sections that run at up to B = max_batch
void plan_inference(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, InferPlan* p) {
    memset(p, 0, sizeof(InferPlan));
    plan_model(d, &p->m);
    const Model& m = p->m;
    const int MB = d->max_batch, nout = d->resnet_outputs;
    size_t off = 0;
    p->f = plan_frames(d, n_scans, n_cached, has_prev, d->W, off);
    p->t = plan_trunk_acts(m.t, MB, false, off);
    p->pooled = take(off, (size_t)MB * 512 * 4);
    p->fc_out = take(off, (size_t)MB * nout * 4);
    p->hid[0] = take(off, (size_t)MB * 512 * 4);
    p->hid[1] = take(off, (size_t)MB * 512 * 4);
    p->w = plan_trunk_weights(m.t, false, off);
    p->fc_w = take(off, (size_t)m.fc.K * m.fc.N * 4);
    p->fc_b = take(off, (size_t)m.fc.N * 4);
    for (int i = 0; i < m.n_lin; ++i) {
        p->lin_w[i] = take(off, (size_t)m.lin[i].K * m.lin[i].N * 4);
        p->lin_b[i] = take(off, (size_t)m.lin[i].N * 4);
    }
    p->total = off;
}

// pairs / push: 2 * max_batch scans and the one cached image of _push
static void make_infer_plan(const delora_odometry_desc* d, InferPlan* p) {
    plan_inference(d, 2 * d->max_batch, 1, false, p);
}

TailIO inference_tail_io(const InferPlan& p, char* ws) {
    TailIO io;
    memset(&io, 0, sizeof(io));
    auto f = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
    io.fc_w = f(p.fc_w); io.fc_b = f(p.fc_b);
    for (int i = 0; i < p.m.n_lin; ++i) { io.w[i] = f(p.lin_w[i]); io.b[i] = f(p.lin_b[i]); }
    io.fc_out = f(p.fc_out);
    for (int i = 0; i < kMaxLinear; ++i) io.hid[i] = f(p.hid[i & 1]);
    return io;
}

// counts = the clamped n_points of n scans (active: see odometry_counts_kernel)
int clamp_counts(const Frames& f, char* ws, const int32_t* n_points, const int32_t* active, int n, int n_stride,
                 cudaStream_t st) {
    odometry_counts_kernel<<<(n + 255) / 256, 256, 0, st>>>(n_points, active, n, n_stride,
                                                            reinterpret_cast<int32_t*>(ws + f.counts));
    DELORA_CHECK_LAUNCH("odometry_counts_kernel");
    return 0;
}

int project(const Frames& f, const delora_odometry_desc* d, char* ws, const float* points, const int32_t* n_points,
            const int32_t* active, int n_scans, cudaStream_t st) {
    const int rc = clamp_counts(f, ws, n_points, active, n_scans, d->n_stride, st);
    if (rc) return rc;
    return delora_project_fwd(points, reinterpret_cast<int32_t*>(ws + f.counts), n_scans, 3, d->n_stride, d->H, d->W,
                              d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0, reinterpret_cast<uint64_t*>(ws + f.keys),
                              reinterpret_cast<float*>(ws + f.images), reinterpret_cast<int32_t*>(ws + f.index_map), st);
}

// The 2B scans of B pairs divided by their pair's normalisation factor, then projected: the clamped counts, the factor
// of every pair into factor [B], and the scaled instantiations of the projection's two passes.
static int project_normalized(const Frames& f, const delora_odometry_desc* d, char* ws, const float* points,
                              const int32_t* n_points, int B, float* factor, cudaStream_t st) {
    int rc = clamp_counts(f, ws, n_points, nullptr, 2 * B, d->n_stride, st);
    if (rc) return rc;
    const int32_t* counts = reinterpret_cast<const int32_t*>(ws + f.counts);
    if ((rc = launch_normalization_factors(points, counts, B, d->n_stride, factor, st))) return rc;
    const GridParams g = make_grid(d->H, d->W, d->hfov0, d->hfov1, d->vfov0, d->vfov1, 0);
    return project_fwd(points, counts, 2 * B, 3, d->n_stride, g, reinterpret_cast<uint64_t*>(ws + f.keys),
                       reinterpret_cast<float*>(ws + f.images), reinterpret_cast<int32_t*>(ws + f.index_map), factor, B,
                       st);
}

// DELORA_LOSS_PO2PO_ALONE's companions: PO2PO required, the normal-reading bits refused, each named
static int check_po2po_alone(uint32_t loss_flags, const char* field, const char* who) {
    if ((loss_flags & DELORA_LOSS_PO2PO_ALONE) == 0u) return 0;
    DELORA_CHECK_ARG((loss_flags & DELORA_LOSS_PO2PO) != 0u,
                     "%s: %s=0x%x has DELORA_LOSS_PO2PO_ALONE without DELORA_LOSS_PO2PO", who, field, loss_flags);
    static const struct { uint32_t bit; const char* name; } refused[3] = {
        {DELORA_LOSS_PO2PL, "DELORA_LOSS_PO2PL"}, {DELORA_LOSS_PL2PL, "DELORA_LOSS_PL2PL"},
        {DELORA_NORMAL_LINEAR, "DELORA_NORMAL_LINEAR"}};
    for (const auto& r : refused)
        DELORA_CHECK_ARG((loss_flags & r.bit) == 0u, "%s: %s=0x%x has DELORA_LOSS_PO2PO_ALONE with %s (po2po_alone "
                         "reads no normal)", who, field, loss_flags, r.name);
    return 0;
}

// The loss and normals' settings of delora_odometry_train_params and delora_odometry_residual_params
int check_icp_params(float lambda_po2pl, uint32_t loss_flags, int nb_h, int nb_w, float epsilon_range,
                     int min_neighbors, const char* who) {
    DELORA_CHECK_ARG(isfinite(lambda_po2pl), "%s: lambda_po2pl=%g must be finite", who, (double)lambda_po2pl);
    if (check_po2po_alone(loss_flags, "loss_flags", who)) return 1;
    DELORA_CHECK_ARG((loss_flags & (DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL)) != 0,
                     "%s: loss_flags=0x%x sets no loss bit", who, loss_flags);
    DELORA_CHECK_ARG(nb_h >= 1 && nb_h % 2 == 1, "%s: nb_h=%d must be odd and positive", who, nb_h);
    DELORA_CHECK_ARG(nb_w >= 1 && nb_w % 2 == 1, "%s: nb_w=%d must be odd and positive", who, nb_w);
    DELORA_CHECK_ARG(isfinite(epsilon_range) && epsilon_range >= 0.0f, "%s: epsilon_range=%g must be >= 0", who,
                     (double)epsilon_range);
    DELORA_CHECK_ARG(min_neighbors >= 0, "%s: min_neighbors=%d must be >= 0", who, min_neighbors);
    return 0;
}

// The front end of the ICP objectives: n scans projected at H x w with their dense grids.  Under
// DELORA_LOSS_PO2PO_ALONE no normal is estimated and the normal grid is zero; otherwise the normals of the nb_h x nb_w
// neighbourhood.  Image, index map and point grid are the same bits either way.
int project_scan_grids(const delora_odometry_desc* d, int w, uint32_t loss_flags, int nb_h, int nb_w,
                       float epsilon_range, int min_neighbors, const float* points, const int32_t* counts, int n,
                       uint64_t* keys, float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid,
                       cudaStream_t st) {
    if (loss_flags & DELORA_LOSS_PO2PO_ALONE)
        return delora_project_points_fwd(points, counts, n, 3, d->n_stride, d->H, w, d->hfov0, d->hfov1, d->vfov0,
                                         d->vfov1, 0, keys, image, index_map, pts_grid, nrm_grid, st);
    return delora_project_normals_fwd(points, counts, n, 3, d->n_stride, d->H, w, d->hfov0, d->hfov1, d->vfov0,
                                      d->vfov1, 0, keys, image, index_map, nb_h, nb_w, epsilon_range, min_neighbors,
                                      pts_grid, nrm_grid, nullptr, st);
}

// Every workspace starts zeroed, with its depth keys at all ones (the projection's empty key).  from > 0: only bytes
// [from, total) are zeroed (a training workspace's geometry section, delora_odometry_train_use_geometry).
int init_workspace(const Frames& f, size_t total, void* workspace, cudaStream_t st, const char* who,
                   size_t from) {
    char* ws = (char*)workspace;
    cudaError_t e = cudaMemsetAsync(ws + from, 0, total - from, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ws + f.keys, 0xFF, f.keys_bytes, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// The bf16 filters of the weight section w from the fp32 weight blob
int prep_blob_weights(const Model& m, const TrunkWeights& w, char* ws, const float* blob, cudaStream_t st,
                      const char* who) {
    const float* src[kMaxConv];
    for (int i = 0; i < m.t.n_conv; ++i) src[i] = blob + m.t.conv[i].blob;
    return prep_trunk_weights(m.t, w, ws, src, st, who);
}

int load_weights(const InferPlan& p, const float* weights, void* workspace, cudaStream_t st, const char* who) {
    char* ws = (char*)workspace;
    const Model& m = p.m;
    int rc = prep_blob_weights(m, p.w, ws, weights, st, who);
    if (rc) return rc;
    auto copy = [&](size_t dst, int64_t src, int64_t n) {
        return cudaMemcpyAsync(ws + dst, weights + src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    };
    cudaError_t e = copy(p.fc_w, m.fc.blob_w, (int64_t)m.fc.K * m.fc.N);
    if (e == cudaSuccess) e = copy(p.fc_b, m.fc.blob_b, m.fc.N);
    for (int i = 0; i < m.n_lin && e == cudaSuccess; ++i) {
        e = copy(p.lin_w[i], m.lin[i].blob_w, (int64_t)m.lin[i].K * m.lin[i].N);
        if (e == cudaSuccess) e = copy(p.lin_b[i], m.lin[i].blob_b, m.lin[i].N);
    }
    DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    return 0;
}

// ---------------------------------------------------------------- the section map
void SectionMap::add(const char* name, size_t off, size_t bytes, int role, int add_flags) {
    if (n < cap) {
        delora_ws_section& r = out[n];
        memset(&r, 0, sizeof(r));
        r.offset = (int64_t)off;
        r.bytes = (int64_t)bytes;
        r.role = role;
        r.geometry = geometry;
        r.flags = flags | add_flags;
        strncpy(r.name, name, sizeof(r.name) - 1);
    }
    ++n;
}

void SectionMap::field(const char* name, size_t off, int role) {
    for (size_t i = log->off.size(); i-- > 0;)
        if (log->off[i] == off) return add(name, off, log->bytes[i], role, 0);
    if (!missing) missing = name;
}

void SectionMap::range(const char* name, size_t off, size_t bytes, int role) {
    bool starts = false;
    for (size_t o : log->off) starts = starts || o == off;
    add(name, off, bytes, role, starts ? 0 : DELORA_WS_SUBRANGE);
}

// The buffers of a sub-plan whose fields alias one another (the inference trunk's activations): one record per take()
// offset in [begin, end), sized by the last take() there
void SectionMap::span(const char* prefix, size_t begin, size_t end, int role) {
    std::vector<size_t> offs;
    for (size_t o : log->off)
        if (o >= begin && o < end) offs.push_back(o);
    std::sort(offs.begin(), offs.end());
    offs.erase(std::unique(offs.begin(), offs.end()), offs.end());
    char name[64];
    for (size_t k = 0; k < offs.size(); ++k) {
        snprintf(name, sizeof name, "%s[%zu]", prefix, k);
        field(name, offs[k], role);
    }
}

// The projection's keys are all ones between calls (each resolve re-arms them): scratch
void map_frames(SectionMap& s, const Frames& f, bool index_map, bool counts, int prev_role) {
    s.field("keys", f.keys, DELORA_WS_SCRATCH);
    if (index_map) s.field("index_map", f.index_map, DELORA_WS_SCRATCH);
    if (counts) s.field("counts", f.counts, DELORA_WS_SCRATCH);
    s.field("images", f.images, DELORA_WS_SCRATCH);
    if (f.prev_image) s.field("prev_image", f.prev_image, prev_role);
    if (f.has_prev) s.field("has_prev", f.has_prev, DELORA_WS_STATE);
}

void map_trunk_weights(SectionMap& s, const TrunkPlan& m, const TrunkWeights& w) {
    char name[32];
    s.field("trunk.table", w.table, DELORA_WS_WEIGHTS);
    for (int i = 0; i < m.n_conv; ++i) {
        snprintf(name, sizeof name, "trunk.fwd[%d]", i);
        s.field(name, w.w_fwd[i], DELORA_WS_WEIGHTS);
        if (!w.flip || i == 0) continue;
        snprintf(name, sizeof name, "trunk.flip[%d]", i);
        s.field(name, w.w_flip[i], DELORA_WS_WEIGHTS);
    }
}

// The inference trunk's activation fields alias by design (each stage's blocks alternate over three buffers): one
// record per buffer.  hid[0] and hid[1] are the tail's alternating hidden buffers.
void map_inference(SectionMap& s, const InferPlan& p, int pooled_role) {
    s.span("trunk.acts", p.t.x_in, p.pooled, DELORA_WS_SCRATCH);
    s.field("pooled", p.pooled, pooled_role);
    s.field("fc_out", p.fc_out, DELORA_WS_SCRATCH);
    s.field("hid[0]", p.hid[0], DELORA_WS_SCRATCH);
    s.field("hid[1]", p.hid[1], DELORA_WS_SCRATCH);
    map_trunk_weights(s, p.m.t, p.w);
    s.field("fc_w", p.fc_w, DELORA_WS_WEIGHTS);
    s.field("fc_b", p.fc_b, DELORA_WS_WEIGHTS);
    char name[32];
    for (int i = 0; i < p.m.n_lin; ++i) {
        snprintf(name, sizeof name, "lin_w[%d]", i);
        s.field(name, p.lin_w[i], DELORA_WS_WEIGHTS);
        snprintf(name, sizeof name, "lin_b[%d]", i);
        s.field(name, p.lin_b[i], DELORA_WS_WEIGHTS);
    }
}

// Arms take_log for one section-map call and disarms it on every return
struct TakeLogArm {
    TakeLog log;
    TakeLogArm() { take_log = &log; }
    ~TakeLogArm() { take_log = nullptr; }
};

}  // namespace delora

using namespace delora;

// delora_odometry_workspace_sections: 0 with the number of sections in *count, 1 for a refusal
static int workspace_sections(int kind, const delora_odometry_desc* d, int n, delora_ws_section* out, int cap,
                              int* count) {
    const char* who = "delora_odometry_workspace_sections";
    DELORA_CHECK_ARG(kind >= 0 && kind < DELORA_WS_KINDS, "%s: kind=%d outside [0, %d)", who, kind, DELORA_WS_KINDS);
    DELORA_CHECK_ARG(cap >= 0 && (out || cap == 0), "%s: cap=%d with %s out", who, cap, out ? "an" : "a null");
    const bool geometries = kind == DELORA_WS_TRAIN_GEOMETRIES || kind == DELORA_WS_ADAPT_GEOMETRIES ||
                            kind == DELORA_WS_ADAPT_GEOMETRIES_INFO;
    DELORA_CHECK_ARG(geometries || n == 1, "%s: n=%d must be 1 for kind %d", who, n, kind);
    DELORA_CHECK_ARG(n >= 1 && n <= kMaxGeometries, "%s: n=%d outside [1, %d]", who, n, kMaxGeometries);
    TakeLogArm arm;
    SectionMap s{&arm.log, out, cap, 0, 0, 0, nullptr};
    int rc = 0;
    if (kind == DELORA_WS_PAIRS) {
        if (check_desc(d, who)) return 1;
        InferPlan p;
        make_infer_plan(d, &p);
        // _push's cached image carries over to its next call; pairs copies pooled to the caller
        map_frames(s, p.f, true, true, DELORA_WS_STATE);
        map_inference(s, p, DELORA_WS_OUTPUT);
    } else if (kind <= DELORA_WS_STREAMS_PRE_INFO) {
        rc = map_streams(s, d, kind, who);
    } else if (kind <= DELORA_WS_TRAIN_GEOMETRIES) {
        rc = map_train_kind(s, d, n, kind, who);
    } else {
        rc = map_adapt(s, d, n, kind, who);
    }
    if (rc) return 1;
    DELORA_CHECK_ARG(!s.missing, "%s: kind %d: no take() at the offset of %s", who, kind, s.missing);
    *count = s.n;
    return 0;
}

extern "C" int delora_odometry_workspace_sections(int kind, const delora_odometry_desc* d, int n,
                                                  delora_ws_section* out, int cap) {
    int count = 0;
    return workspace_sections(kind, d, n, out, cap, &count) ? -1 : count;
}

extern "C" int delora_odometry_file_objective(const delora_odometry_file_header* h, uint32_t* loss_flags,
                                              float* lambda_po2pl) {
    const char* who = "delora_odometry_file_objective";
    DELORA_CHECK_ARG(h && loss_flags && lambda_po2pl, "%s: null pointer", who);
    const uint32_t f = h->objective_flags;
    if (f == 0u) {                  // written before the field: the shipped objective
        *loss_flags = DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL;
        *lambda_po2pl = 1.0f;
        return 0;
    }
    const uint32_t bits = DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL | DELORA_NORMAL_LINEAR |
                          DELORA_LOSS_PO2PO_ALONE;
    DELORA_CHECK_ARG((f & ~bits) == 0u, "%s: objective_flags=0x%x has a bit other than the ICP losses, "
                     "DELORA_NORMAL_LINEAR and DELORA_LOSS_PO2PO_ALONE", who, f);
    if (check_po2po_alone(f, "objective_flags", who)) return 1;
    DELORA_CHECK_ARG((f & (DELORA_LOSS_PO2PO | DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL)) != 0u,
                     "%s: objective_flags=0x%x sets no loss bit", who, f);
    DELORA_CHECK_ARG(isfinite(h->lambda_po2pl), "%s: lambda_po2pl=%g must be finite", who, (double)h->lambda_po2pl);
    *loss_flags = f;
    *lambda_po2pl = h->lambda_po2pl;
    return 0;
}

extern "C" int64_t delora_odometry_weight_floats(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_weight_floats")) return -1;
    Model m;
    plan_model(d, &m);
    return m.blob_floats;
}

extern "C" int64_t delora_odometry_workspace_bytes(const delora_odometry_desc* d) {
    if (check_desc(d, "delora_odometry_workspace_bytes")) return -1;
    InferPlan p;
    make_infer_plan(d, &p);
    return (int64_t)p.total;
}

extern "C" int delora_odometry_init(const delora_odometry_desc* d, void* workspace, void* stream) {
    if (check_desc(d, "delora_odometry_init")) return 1;
    DELORA_CHECK_ARG(workspace, "delora_odometry_init: null workspace");
    InferPlan p;
    make_infer_plan(d, &p);
    return init_workspace(p.f, p.total, workspace, (cudaStream_t)stream, "delora_odometry_init");
}

extern "C" int delora_odometry_load_weights(const delora_odometry_desc* d, const float* weights, void* workspace,
                                            void* stream) {
    if (check_desc(d, "delora_odometry_load_weights")) return 1;
    DELORA_CHECK_ARG(weights && workspace, "delora_odometry_load_weights: null pointer");
    InferPlan p;
    make_infer_plan(d, &p);
    return load_weights(p, weights, workspace, (cudaStream_t)stream, "delora_odometry_load_weights");
}

// delora_odometry_pairs and, with factor non-NULL, delora_odometry_pairs_normalized (arguments checked by the caller)
static int run_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B, void* workspace,
                     float* T, float* pooled, float* factor, cudaStream_t st, const char* who) {
    InferPlan p;
    make_infer_plan(d, &p);
    char* ws = (char*)workspace;
    float* images = reinterpret_cast<float*>(ws + p.f.images);
    const size_t img = (size_t)4 * d->H * d->W;
    float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
    int rc;
    if (factor) rc = project_normalized(p.f, d, ws, points, n_points, B, factor, st);
    else rc = project(p.f, d, ws, points, n_points, nullptr, 2 * B, st);
    if (rc) return rc;
    if ((rc = trunk_input(p.m.t, p.t, ws, images, images + (size_t)B * img, B, st))) return rc;
    if ((rc = trunk_forward(p.m.t, p.t, ws, p.w, ws, d->act, B, pooled_ws, nullptr, st))) return rc;
    if ((rc = run_tail(p.m, inference_tail_io(p, ws), d->act, pooled_ws, B, T, st, factor))) return rc;
    if (pooled) {
        const cudaError_t e = cudaMemcpyAsync(pooled, pooled_ws, (size_t)B * 512 * sizeof(float), cudaMemcpyDeviceToDevice, st);
        DELORA_CHECK_ARG(e == cudaSuccess, "%s: %s", who, cudaGetErrorString(e));
    }
    return 0;
}

extern "C" int delora_odometry_pairs(const delora_odometry_desc* d, const float* points, const int32_t* n_points, int B,
                                     void* workspace, float* T, float* pooled, void* stream) {
    if (check_desc(d, "delora_odometry_pairs")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace && T, "delora_odometry_pairs: null pointer");
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "delora_odometry_pairs: B=%d outside [1, max_batch=%d]", B,
                     d->max_batch);
    return run_pairs(d, points, n_points, B, workspace, T, pooled, nullptr, (cudaStream_t)stream, "delora_odometry_pairs");
}

extern "C" int delora_odometry_pairs_normalized(const delora_odometry_desc* d, const float* points,
                                                const int32_t* n_points, int B, void* workspace, float* T,
                                                float* pooled, float* factor, void* stream) {
    const char* who = "delora_odometry_pairs_normalized";
    if (check_desc(d, who)) return 1;
    DELORA_CHECK_ARG(points, "%s: null points", who);
    DELORA_CHECK_ARG(n_points, "%s: null n_points", who);
    DELORA_CHECK_ARG(workspace, "%s: null workspace", who);
    DELORA_CHECK_ARG(T, "%s: null T", who);
    DELORA_CHECK_ARG(factor, "%s: null factor", who);
    DELORA_CHECK_ARG(B >= 1 && B <= d->max_batch, "%s: B=%d outside [1, max_batch=%d]", who, B, d->max_batch);
    return run_pairs(d, points, n_points, B, workspace, T, pooled, factor, (cudaStream_t)stream, who);
}

extern "C" int delora_odometry_push(const delora_odometry_desc* d, const float* points, const int32_t* n_points,
                                    void* workspace, float* T, void* stream) {
    if (check_desc(d, "delora_odometry_push")) return 1;
    DELORA_CHECK_ARG(points && n_points && workspace, "delora_odometry_push: null pointer");
    InferPlan p;
    make_infer_plan(d, &p);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    float* image = reinterpret_cast<float*>(ws + p.f.images);
    float* prev = reinterpret_cast<float*>(ws + p.f.prev_image);
    int rc;
    if ((rc = project(p.f, d, ws, points, n_points, nullptr, 1, st))) return rc;
    if (T) {
        float* pooled_ws = reinterpret_cast<float*>(ws + p.pooled);
        if ((rc = trunk_input(p.m.t, p.t, ws, prev, image, 1, st))) return rc;
        if ((rc = trunk_forward(p.m.t, p.t, ws, p.w, ws, d->act, 1, pooled_ws, nullptr, st))) return rc;
        if ((rc = run_tail(p.m, inference_tail_io(p, ws), d->act, pooled_ws, 1, T, st))) return rc;
    }
    const cudaError_t e = cudaMemcpyAsync(prev, image, (size_t)4 * d->H * d->W * sizeof(float), cudaMemcpyDeviceToDevice, st);
    DELORA_CHECK_ARG(e == cudaSuccess, "delora_odometry_push: %s", cudaGetErrorString(e));
    return 0;
}
