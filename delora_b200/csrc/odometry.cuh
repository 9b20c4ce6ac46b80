// The odometry C ABI's internal interface: the model plan, the workspace sections and plans more than one source
// reads, and the host functions one source calls in another.  Each workspace family has a source of its own:
//   odometry.cu          the model plan, the descriptor checks, the frame section, the inference plan, workspace init,
//                        weight loading, projection, and the pairs / push entry points;
//   odometry_tail.cu     the fully connected tail: its forward (batched and per stream), its backward and Adam;
//   odometry_streams.cu  the six streams workspace kinds;
//   odometry_train.cu    the training workspace: step, eval, state, group, geometries, dropout seed;
//   odometry_adapt.cu    the adapting streams, of one geometry and of several.
// Every kernel is private to its source; other sources reach it through the host functions declared here.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"
#include "dropout.cuh"
#include "trunk.cuh"

namespace delora {

constexpr int kTailWarps = 8;
constexpr int kMaxLinear = 5;
constexpr int kMaxBatch = 1024;
constexpr int kHeadHidden = 100;
constexpr int kMaxGeometries = 16;     // descriptors of delora_odometry_streams_push_adapt_geometries
constexpr int kGroupBuckets = DELORA_TRAIN_GROUP_BUCKETS;

struct TailLinear {
    const float* w;        // [N, K] row-major
    const float* bias;     // [N]
    const float* x;        // [B, ldx]
    float* y;              // [B, ldy]
    int K, N, ldx, ldy;
};

__device__ __forceinline__ bool stream_active(const int32_t* __restrict__ active, int s) {
    return active == nullptr || active[s] != 0;
}

// ---------------------------------------------------------------- the model: layer sequence + weight-blob offsets
struct Linear {
    int K, N;
    int64_t blob_w, blob_b;
};
struct Model {
    TrunkPlan t;                       // the trunk's filters open the blob
    int n_lin;
    Linear lin[kMaxLinear];            // two heads: rot1, rot2, trans1, trans2; single MLP: 5 layers
    Linear fc;
    int64_t blob_floats;
};

// The frame section: n_scans projected scans (depth keys, index map, clamped counts, fp32 images), n_cached cached
// previous images and, with has_prev, one "has a previous frame" flag per cached image.  The depth keys are sized for
// images key_w wide (>= W): the training step projects at the preprocessing width in them as well.
struct Frames {
    size_t keys, keys_bytes, index_map, counts, images;
    size_t prev_image;                 // n_cached > 0 only
    size_t has_prev;                   // with has_prev only
};

// The pairs / push and the streams workspaces: the trunk's inference buffers and its weight section without the
// flipped filters.  The tail reads fp32 copies of its weights (256-byte aligned).  The streams kinds append their own
// sections (StreamsPlan, odometry_streams.cu).
struct InferPlan {
    Model m;
    Frames f;
    TrunkActs t;
    size_t pooled, fc_out, hid[2];
    TrunkWeights w;
    size_t fc_w, fc_b, lin_w[kMaxLinear], lin_b[kMaxLinear];
    size_t total;
};

// Where the tail reads its weights and writes its activations.  Inference: the workspace copies of the weights and two
// hidden buffers the layers alternate between; training: the fp32 master blob and one buffer per layer (the backward
// reads every activation).
struct TailIO {
    const float* fc_w;
    const float* fc_b;
    const float* w[kMaxLinear];
    const float* b[kMaxLinear];
    float* fc_out;                     // [B, nout]: act(resnet.fc(pooled))
    float* hid[kMaxLinear];            // output of lin[i], i < n_lin - 1; two heads: hid[0] = [rot1 | trans1], ld 200
    float* raw;                        // [B, 7] head outputs before the normalisation, or NULL
};

// ---------------------------------------------------------------- training plan: workspace layout
struct TrainPlan {
    Model m;
    size_t master, grad, adam_m, adam_v, ctr;
    TrunkWeights w;
    Frames f;                          // 2 * max_batch scans, no cached image
    size_t pts_grid, nrm_grid, icp, losses, grad_T, T16, T12;
    TrunkActs t;                       // the trunk's saving buffers
    // w_pre > 0 only: the preprocessing projection of the 2 * max_batch scans at H x w_pre (image, index map and the
    // dense grids with their normals), placed after every other buffer
    size_t pre_image, pre_index_map, pre_pts_grid, pre_nrm_grid;
    // tail activations and gradients
    size_t pooled, fc_out, hid[kMaxLinear], raw, dz_hid[kMaxLinear], dz_fc, g_pooled;
    size_t total;
};

// One tick of delora_odometry_streams_push_adapt, as train_forward_losses sees it: the caller's arguments and the
// stream section of the workspace.
struct AdaptTick {
    const int32_t* active;             // [S] or NULL (every stream is)
    float* T;                          // [S, 16] the caller's T
    int32_t* valid;                    // [S] the caller's valid
    int32_t* has_prev;                 // [S]
    int32_t* n_valid;                  // [1] the number of valid streams this tick
    float* cache_image;                // [S, 4, H, W] w_pre = 0 only: each stream's previous image
    delora_f4* cache_pts;              // [S, H, W] (w_pre = 0) or [S, H, w_pre]: its previous stage-1 grids
    delora_f4* cache_nrm;
    float* info;                       // [S, DELORA_INFO_ROW] or NULL (_push_adapt_info): the information rows
    float* info_scratch;               // the information operator's info_scratch at B = S, with info
};

// The gradient slices of geometries 1 .. n of delora_odometry_streams_push_adapt_geometries (blob layout each)
struct GradSlices {
    const float* g[kMaxGeometries - 1];
    int n;
};

// How the group form of a step all-reduces its gradient: bucket k times scale, seq = *seq_step * seq_stride +
// seq_first + k
struct GroupReduce {
    const delora_odometry_train_group* g;
    float scale;
    const long long* seq_step;
    unsigned seq_stride, seq_first;
};

// The records of delora_odometry_workspace_sections, from the take() log of the plan builds (take_log armed).
// field: the section at off, sized by the last take() there (a plan that moves a field after its build takes again at
// the new offset, later); range: a section the caller sizes, inside one take().  Each family's source lists the fields
// its entry points dereference (map_* below).
struct SectionMap {
    const TakeLog* log;
    delora_ws_section* out;
    int cap, n, geometry, flags;       // geometry and flags of the records added next
    const char* missing;               // a field with no take() at its offset: the plan and the map disagree
    void add(const char* name, size_t off, size_t bytes, int role, int flags);
    void field(const char* name, size_t off, int role);
    void range(const char* name, size_t off, size_t bytes, int role);
    void span(const char* prefix, size_t begin, size_t end, int role);      // every take() in [begin, end), in order
};

// ---------------------------------------------------------------- odometry.cu
int check_desc(const delora_odometry_desc* d, const char* who);
int check_icp_params(float lambda_po2pl, uint32_t loss_flags, int nb_h, int nb_w, float epsilon_range,
                     int min_neighbors, const char* who);
void plan_model(const delora_odometry_desc* d, Model* m);
Frames plan_frames(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, int key_w, size_t& off);
void plan_inference(const delora_odometry_desc* d, int n_scans, int n_cached, bool has_prev, InferPlan* p);
TailIO inference_tail_io(const InferPlan& p, char* ws);
int clamp_counts(const Frames& f, char* ws, const int32_t* n_points, const int32_t* active, int n, int n_stride,
                 cudaStream_t st);
int project(const Frames& f, const delora_odometry_desc* d, char* ws, const float* points, const int32_t* n_points,
            const int32_t* active, int n_scans, cudaStream_t st);
int project_scan_grids(const delora_odometry_desc* d, int w, uint32_t loss_flags, int nb_h, int nb_w,
                       float epsilon_range, int min_neighbors, const float* points, const int32_t* counts, int n,
                       uint64_t* keys, float* image, int32_t* index_map, delora_f4* pts_grid, delora_f4* nrm_grid,
                       cudaStream_t st);
int init_workspace(const Frames& f, size_t total, void* workspace, cudaStream_t st, const char* who, size_t from = 0);
int prep_blob_weights(const Model& m, const TrunkWeights& w, char* ws, const float* blob, cudaStream_t st,
                      const char* who);
int load_weights(const InferPlan& p, const float* weights, void* workspace, cudaStream_t st, const char* who);
// the section map of a frame section (index_map / counts: whether the kind reads them; prev_role: its cached images'),
// of a weight section, and of everything plan_inference places after the frame section
void map_frames(SectionMap& s, const Frames& f, bool index_map, bool counts, int prev_role);
void map_trunk_weights(SectionMap& s, const TrunkPlan& m, const TrunkWeights& w);
void map_inference(SectionMap& s, const InferPlan& p, int pooled_role);

// ---------------------------------------------------------------- odometry_tail.cu
int run_tail(const Model& m, const TailIO& io, int act, const float* pooled, int B, float* T, cudaStream_t st,
             const float* factor = nullptr, DropoutCtr drop = DropoutCtr{nullptr, 0});
int streams_forward(const Model& m, const TailIO& io, const TrunkActs& t, const TrunkWeights& w, char* ws, int act,
                    float* pooled, int S, const int32_t* active, int32_t* has_prev, float* T, int32_t* valid,
                    const float* factor, float* factor_out, int32_t* counts, int32_t* n_valid, cudaStream_t st);
int train_tail_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, cudaStream_t st,
                        DropoutCtr drop = DropoutCtr{nullptr, 0}, const int32_t* valid = nullptr,
                        const int32_t* n_valid = nullptr);
int adam_update(const TrainPlan& tp, char* ws, const delora_odometry_train_params* hp, const int32_t* run,
                cudaStream_t st, const GradSlices* more = nullptr);

// ---------------------------------------------------------------- odometry_streams.cu
int check_tick(const void* points, const void* n_points, const void* workspace, const float* T, const int32_t* valid,
               const float* extra, const char* extra_name, const char* who);
int clear_grids(char* ws, size_t pts, size_t nrm, size_t n, cudaStream_t st);
int reset_streams(const delora_odometry_desc* d, const int32_t* mask, void* workspace, size_t has_prev, void* stream,
                  const char* who);
const char* icp_entry(const float* info, const float* factor);
int streams_pre(const float* T16, const float* factor, const int32_t* active, const int32_t* valid, int S, int HW,
                int HWp, float* T, float* T12, float* factor_out, float4* cur_pts, float4* cur_nrm,
                const float4* pre_cur_pts, const float4* pre_cur_nrm, float4* pre_prev_pts, float4* pre_prev_nrm,
                const float4* cur_image, float4* cache_image, cudaStream_t st);
int streams_rows_out(int row, const int32_t* valid, int S, const float* rows, float* out, cudaStream_t st);
int map_streams(SectionMap& s, const delora_odometry_desc* d, int kind, const char* who);   // DELORA_WS_STREAMS*

// ---------------------------------------------------------------- odometry_train.cu
void make_train_plan(const delora_odometry_desc* d, TrainPlan* tp, size_t geometry_at = 0);
int check_train_desc(const delora_odometry_desc* d, const char* who);
int check_train_params(const delora_odometry_train_params* hp, const char* who);
int check_train_call(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* points,
                     const int32_t* n_points, int B, const void* workspace, const char* who);
int check_geometries(const delora_odometry_desc* d, int n, const char* who);
int check_group(const delora_odometry_train_group* g, const void* workspace, const char* who);
int train_init(const delora_odometry_desc* d, size_t total, const float* weights, void* workspace, cudaStream_t st,
               const char* who);
int train_forward_losses(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const TrainPlan& tp,
                         char* ws, const float* points, const int32_t* n_points, int B, bool dropout, float* T_out,
                         cudaStream_t st, const char* who, const AdaptTick* at = nullptr);
int step_backward(const TrainPlan& tp, char* ws, int act, int B, bool identity, DropoutCtr drop, const int32_t* valid,
                  const int32_t* n_valid, const GroupReduce* gr, cudaStream_t st, const char* who);
int record_icp_batch(const TrainPlan& tp, char* ws, int B, cudaStream_t st);
// the sections of one training plan: the model section's (the weights under weights_flags; the gradient, with adam
// Adam's moments, and the counters with ctr_role under model_flags), then the geometry section's
void map_train(SectionMap& s, const delora_odometry_desc* d, const TrainPlan& tp, bool adam, int ctr_role,
               int weights_flags, int model_flags);
int map_train_kind(SectionMap& s, const delora_odometry_desc* d, int n, int kind, const char* who);

// ---------------------------------------------------------------- odometry_adapt.cu
int map_adapt(SectionMap& s, const delora_odometry_desc* d, int n, int kind, const char* who);   // DELORA_WS_ADAPT*

}  // namespace delora
