/*
 * The reference's training loop (src/deploy/trainer.py, Trainer.train) from a C host: no Python, no torch.  Links
 * libdelora_b200.so and cudart only.
 *
 *   odometry_train [--lr LR] [--switch-below L] [--dropout-seed S] [--eval-dir DIR] [--gpus N]
 *                  [--geometry DIR,H,W,VFOV0,VFOV1[,W_PRE]]... in.dlt|in.dlw out.dlt epochs B scan_000.bin ...
 *
 * Reads a training checkpoint (.dlt: weights, Adam's state, epoch and phase; layout in include/delora_b200.h) or a
 * weight file (.dlw: a fresh Adam with learning rate --lr, default 1e-5, the reference's learning_rate) and a list of
 * consecutive KITTI velodyne .bin scans ([N, 4] float32 rows: x, y, z, reflectance), then runs `epochs` epochs.  An
 * epoch walks the consecutive pairs (scan k, scan k+1) in order, B pairs per step (the last step takes the rest), and
 * its objective is the mean of the steps' objectives:
 *   - identity pre-training (the .dlt's unsupervised = 0): DELORA_LOSS_IDENTITY_FIT, MSELoss(T_{B-1}, I) / B;
 *   - afterwards: the mean over the step's pairs of po2po + lambda * po2pl + pl2pl.
 * Once an epoch's objective drops below --switch-below (default 1e-2, trainer.py:184-186) the next epoch is
 * unsupervised.  A .dlw, or a .dlt made from a checkpoint, starts unsupervised, as the reference does with a
 * checkpoint.  After every epoch the state goes to out.dlt (written to out.dlt.tmp, then renamed), so a run that
 * stops can resume from it: N epochs in one run and N1 + N2 = N epochs in two give the same bytes.
 * Losses as odometry_finetune.c: the objective the header records (objective_flags, lambda_po2pl; zeros there: po2pl +
 * pl2pl, lambda_po2pl 1), normals at the resolution the header's w_pre names (none under po2po_alone).
 * A model configured with use_dropout (model_flags has DELORA_MODEL_DROPOUT) trains with its dropouts
 * (DELORA_TRAIN_DROPOUT).  The seed of the masks is --dropout-seed, else the DELORA_DROPOUT_SEED environment variable,
 * else the .dlt's (0 for a .dlw); it is written into every out.dlt, so a resumed run draws the masks of an
 * uninterrupted one.
 * --eval-dir DIR: a held-out sequence (the reference's testing_identifiers), the .bin scans of DIR in name order.  After
 * every epoch the mean ICP objective (po2po + lambda * po2pl + pl2pl per pair) over its consecutive pairs, through
 * delora_odometry_train_eval on the training workspace, is appended to the epoch's line as "held-out <mean>".  The
 * evaluation updates nothing: out.dlt has the bytes of a run without the option.
 * --gpus N (N > 1): data-parallel training on GPUs 0 .. N-1 of this process, one host thread per GPU, peer access
 * enabled both ways, delora_odometry_train_step_group on the unicast path (the gradient of every step is the mean over
 * the GPUs).  The pairs are split into N contiguous shards of n_pairs / N pairs (as parallel_grad.shard_pairs does; the
 * remainder is left out so that every GPU steps the same batch sizes), each GPU walks its shard B pairs per step, and
 * the epoch's objective is the mean over the GPUs of their mean objectives.  GPU r draws its dropout masks with seed
 * + r; the .dlt keeps the seed.  GPU 0 writes out.dlt and runs --eval-dir.  Without the option, or with --gpus 1, the
 * program runs on the current GPU through delora_odometry_train_step.
 * --geometry DIR,H,W,VFOV0,VFOV1[,W_PRE] (repeatable, one GPU): one more dataset recorded by another sensor, the
 * reference's `datasets` list.  Its scans are the .bin files of DIR in name order; its descriptor is the header's with
 * H, W, the vertical field of view (degrees) and w_pre (default 0) replaced.  All datasets train one model in one
 * workspace (delora_odometry_train_geometries_*).  Each epoch runs the batches of every dataset (its consecutive pairs,
 * B per step, the last step the rest) in one shuffled order, as the reference's DataLoader shuffles the concatenated
 * datasets; a batch is always from one dataset, and delora_odometry_train_use_geometry re-arms the workspace when the
 * dataset changes.  The order is drawn from the epoch number, so a run resumed from out.dlt steps as an uninterrupted
 * one.  out.dlt keeps the header's descriptor: pass the same --geometry options when resuming.  --eval-dir scores the
 * header's geometry.  Every geometry takes the header's max_batch, and each switch zeroes the workspace's buffers for
 * that many pairs: export with max_batch = B (include/delora_b200.h gives the cost).
 *
 * Build:  cc odometry_train.c -I include -I $CUDA_HOME/include -L delora_b200 -ldelora_b200 \
 *            -L $CUDA_HOME/lib64 -lcudart -lpthread -Wl,-rpath,$PWD/delora_b200 -o odometry_train
 */
#include <dirent.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "delora_b200.h"

static int fail(const char* what) {
    fprintf(stderr, "odometry_train: %s\n", what);
    return 1;
}

/* the ICP objective a host trains, scores or adapts on, as it prints it once at start */
static void print_objective(const char* who, uint32_t f, float lambda_po2pl) {
    fprintf(stderr, "%s: objective%s%s%s%s, lambda_po2pl %g\n", who,
            (f & DELORA_LOSS_PO2PO_ALONE) ? " po2po_alone" : (f & DELORA_LOSS_PO2PO) ? " po2po" : "",
            (f & DELORA_LOSS_PO2PL) ? " po2pl" : "", (f & DELORA_LOSS_PL2PL) ? " pl2pl" : "",
            (f & DELORA_LOSS_PL2PL) ? ((f & DELORA_NORMAL_LINEAR) ? " (linear normal loss)" : " (squared normal loss)")
                                    : "",
            (double)lambda_po2pl);
}

static int by_name(const void* a, const void* b) { return strcmp(*(char* const*)a, *(char* const*)b); }

/* the .bin files of a directory, sorted by name -> *paths (malloc'ed); the count, or -1 */
static int list_scans(const char* dir, char*** paths) {
    DIR* d = opendir(dir);
    if (!d) return -1;
    int cap = 16, n = 0;
    char** out = (char**)malloc(sizeof(char*) * (size_t)cap);
    const struct dirent* e;
    while (out && (e = readdir(d)) != NULL) {
        const size_t len = strlen(e->d_name);
        if (len < 5 || strcmp(e->d_name + len - 4, ".bin") != 0) continue;
        if (n == cap) {
            cap *= 2;
            char** grown = (char**)realloc(out, sizeof(char*) * (size_t)cap);
            if (!grown) { closedir(d); return -1; }
            out = grown;
        }
        out[n] = (char*)malloc(strlen(dir) + len + 2);
        if (!out[n]) { closedir(d); return -1; }
        sprintf(out[n++], "%s/%s", dir, e->d_name);
    }
    closedir(d);
    if (!out) return -1;
    qsort(out, (size_t)n, sizeof(char*), by_name);
    *paths = out;
    return n;
}

#define CUDA_OK(call)                                                                  \
    do {                                                                               \
        cudaError_t e_ = (call);                                                       \
        if (e_ != cudaSuccess) return fail(cudaGetErrorString(e_));                     \
    } while (0)

#define DELORA_OK(call)                                                                \
    do {                                                                               \
        if ((call) != 0) return fail(delora_last_error());                             \
    } while (0)

/* one scan as [3, n_stride] channels-first (x, y, z), zero-padded; returns the point count or -1 */
static int32_t read_scan(const char* path, int n_stride, float* out) {
    FILE* s = fopen(path, "rb");
    if (!s) return -1;
    fseek(s, 0, SEEK_END);
    const long bytes = ftell(s);
    fseek(s, 0, SEEK_SET);
    const int32_t n = (int32_t)(bytes / (4 * sizeof(float)));
    float* rows = (float*)malloc((size_t)n * 4 * sizeof(float) + 1);
    if (n > n_stride || !rows || fread(rows, 4 * sizeof(float), (size_t)n, s) != (size_t)n) {
        free(rows);
        fclose(s);
        return -1;
    }
    fclose(s);
    memset(out, 0, (size_t)3 * n_stride * sizeof(float));
    for (int32_t i = 0; i < n; ++i)
        for (int c = 0; c < 3; ++c) out[(size_t)c * n_stride + i] = rows[(size_t)i * 4 + c];
    free(rows);
    return n;
}

/* n scans -> [n, 3, n_stride] host floats and their counts (both malloc'ed); 0 on success */
static int load_scans(char** paths, int n, int n_stride, float** scans, int32_t** counts) {
    const size_t scan_floats = (size_t)3 * n_stride;
    *scans = (float*)malloc((size_t)(n > 0 ? n : 1) * scan_floats * sizeof(float));
    *counts = (int32_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(int32_t));
    if (!*scans || !*counts) return fail("out of host memory");
    for (int k = 0; k < n; ++k)
        if (((*counts)[k] = read_scan(paths[k], n_stride, *scans + (size_t)k * scan_floats)) < 0)
            return fail("cannot read a scan (missing, truncated, or more points than n_stride)");
    return 0;
}

/* the points of a step or an evaluation on pairs (k0 + b, k0 + b + 1), b < B: scan_1 of pairs 0..B-1, then scan_2 */
static int stage_pairs(const float* h_scans, const int32_t* h_counts, int k0, int B, size_t scan_floats, float* points,
                       int32_t* counts, int32_t* h_step_counts, cudaStream_t stream) {
    for (int b = 0; b < B; ++b) {
        const int k = k0 + b;
        CUDA_OK(cudaMemcpyAsync(points + (size_t)b * scan_floats, h_scans + (size_t)k * scan_floats,
                                scan_floats * sizeof(float), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(points + (size_t)(B + b) * scan_floats, h_scans + (size_t)(k + 1) * scan_floats,
                                scan_floats * sizeof(float), cudaMemcpyHostToDevice, stream));
        h_step_counts[b] = h_counts[k];
        h_step_counts[B + b] = h_counts[k + 1];
    }
    CUDA_OK(cudaMemcpyAsync(counts, h_step_counts, (size_t)2 * B * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    return 0;
}

/* mean over the B rows of po2po + lambda * po2pl + pl2pl */
static double icp_objective(const float* h_losses, int B, float lambda_po2pl) {
    double objective = 0.0;
    for (int b = 0; b < B; ++b) {
        const float* l = h_losses + (size_t)b * DELORA_LOSS_ROW;
        objective += (double)l[0] + (double)lambda_po2pl * l[1] + (double)l[2];
    }
    return objective / B;
}

/* the header and the three host arrays (weights, exp_avg, exp_avg_sq) to path, through path.tmp and a rename */
static int write_dlt(const char* path, const delora_odometry_train_file_header* hdr, float* const* h_state, size_t n) {
    char tmp[4096];
    if (snprintf(tmp, sizeof tmp, "%s.tmp", path) >= (int)sizeof tmp) return fail("output path too long");
    FILE* o = fopen(tmp, "wb");
    if (!o) return fail("cannot create the output file");
    int ok = fwrite(hdr, sizeof *hdr, 1, o) == 1;
    for (int i = 0; i < 3 && ok; ++i) ok = fwrite(h_state[i], sizeof(float), n, o) == n;
    ok = (fclose(o) == 0) && ok;
    if (!ok || rename(tmp, path) != 0) return fail("cannot write the output file");
    return 0;
}

/* the mean ICP objective of the held-out pairs with the workspace's weights (delora_odometry_train_eval); -1 on error */
static int held_out(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* h_eval_scans,
                    const int32_t* h_eval_counts, int n_eval_pairs, int B_max, size_t scan_floats, void* workspace,
                    float* points, int32_t* counts, float* losses, float* h_losses, int32_t* h_step_counts,
                    cudaStream_t stream, double* mean) {
    double held = 0.0;
    for (int k0 = 0; k0 < n_eval_pairs; k0 += B_max) {
        const int B = n_eval_pairs - k0 < B_max ? n_eval_pairs - k0 : B_max;
        if (stage_pairs(h_eval_scans, h_eval_counts, k0, B, scan_floats, points, counts, h_step_counts, stream))
            return 1;
        DELORA_OK(delora_odometry_train_eval(d, hp, points, counts, B, workspace, losses, NULL, NULL, stream));
        CUDA_OK(cudaMemcpyAsync(h_losses, losses, (size_t)B * DELORA_LOSS_ROW * sizeof(float), cudaMemcpyDeviceToHost,
                                stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        held += icp_objective(h_losses, B, hp->lambda_po2pl) * B;
    }
    *mean = held / n_eval_pairs;
    return 0;
}

#define MAX_GEOMETRIES 16
#define DEG_TO_RAD (3.14159265358979323846 / 180.0)

/* one ",value" field at *p: an integer in [0, 1e9] (integral) or a finite number; advances *p; 0 on success */
static int next_field(const char** p, int integral, double* out) {
    if (**p != ',') return 1;
    const char* s = *p + 1;
    char* end;
    if (integral) {
        const long v = strtol(s, &end, 10);
        if (end == s || v < 0 || v > 1000000000L) return 1;
        *out = (double)v;
    } else {
        const double v = strtod(s, &end);
        if (end == s || !(v >= -1e300 && v <= 1e300)) return 1;     /* also refuses nan and inf */
        *out = v;
    }
    if (*end != ',' && *end != '\0') return 1;
    *p = end;
    return 0;
}

/* "DIR,H,W,VFOV0,VFOV1[,W_PRE]" (fields of view in degrees) -> *dir (a copy) and *g: base with H, W, vfov and w_pre
 * replaced; 0 on success.  The library validates the descriptor itself. */
static int parse_geometry(const char* arg, const delora_odometry_desc* base, char** dir, delora_odometry_desc* g) {
    const char* comma = strchr(arg, ',');
    if (!comma || comma == arg) return 1;
    double v[5] = {0, 0, 0, 0, 0};
    const int integral[5] = {1, 1, 0, 0, 1};
    const char* p = comma;
    for (int i = 0; i < 5; ++i) {
        if (i == 4 && *p == '\0') break;                              /* W_PRE is optional */
        if (next_field(&p, integral[i], &v[i])) return 1;
    }
    if (*p != '\0' || v[0] < 1 || v[1] < 2 || !(v[3] > v[2])) return 1;
    *g = *base;
    g->H = (int)v[0];
    g->W = (int)v[1];
    g->vfov0 = v[2] * DEG_TO_RAD;
    g->vfov1 = v[3] * DEG_TO_RAD;
    g->w_pre = (int)v[4];
    *dir = (char*)malloc((size_t)(comma - arg) + 1);
    if (!*dir) return 1;
    memcpy(*dir, arg, (size_t)(comma - arg));
    (*dir)[comma - arg] = '\0';
    return 0;
}

static uint64_t splitmix64(uint64_t* state) {
    uint64_t z = (*state += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* --gpus N: one GPU of the group, and the epoch its thread runs */
typedef struct {
    int rank;
    const delora_odometry_desc* d;
    delora_odometry_train_params hp;
    delora_odometry_train_group g;
    const float* h_scans;
    const int32_t* h_counts;
    int first, n_pairs, B_max, identity;      /* its shard: pairs first .. first + n_pairs - 1 */
    size_t scan_floats;
    cudaStream_t stream, side;
    cudaEvent_t events[DELORA_TRAIN_GROUP_BUCKETS + 1];
    void* workspace;
    float *points, *losses, *h_losses;
    int32_t *counts, *h_step_counts, *flags, *status;
    double mean;                              /* the epoch's mean objective on this GPU */
    int rc;
} rank_state;

static int rank_epoch(rank_state* r) {
    CUDA_OK(cudaSetDevice(r->rank));
    double sum = 0.0;
    int steps = 0;
    for (int k0 = 0; k0 < r->n_pairs; k0 += r->B_max, ++steps) {
        const int B = r->n_pairs - k0 < r->B_max ? r->n_pairs - k0 : r->B_max;
        if (stage_pairs(r->h_scans, r->h_counts, r->first + k0, B, r->scan_floats, r->points, r->counts,
                        r->h_step_counts, r->stream))
            return 1;
        DELORA_OK(delora_odometry_train_step_group(r->d, &r->hp, &r->g, r->points, r->counts, B, r->workspace,
                                                   r->losses, NULL, NULL, NULL, r->stream));
        CUDA_OK(cudaMemcpyAsync(r->h_losses, r->losses, (size_t)B * DELORA_LOSS_ROW * sizeof(float),
                                cudaMemcpyDeviceToHost, r->stream));
        CUDA_OK(cudaStreamSynchronize(r->stream));
        sum += r->identity ? (double)r->h_losses[(size_t)(B - 1) * DELORA_LOSS_ROW + 5]
                           : icp_objective(r->h_losses, B, r->hp.lambda_po2pl);
    }
    int32_t status = 0;
    CUDA_OK(cudaMemcpy(&status, r->status, sizeof status, cudaMemcpyDeviceToHost));
    if (status != 0) return fail("a GPU of the group did not reach the gradient all-reduce in time");
    r->mean = steps > 0 ? sum / steps : 0.0;
    return 0;
}

static void* rank_thread(void* arg) {
    rank_state* r = (rank_state*)arg;
    r->rc = rank_epoch(r);
    return NULL;
}

/* one GPU's workspace, buffers, streams and events, its state from the host arrays; 0 on success */
static int rank_setup(rank_state* r, int world, float* const* h_state, size_t n, int64_t step, uint64_t dropout_seed,
                      int64_t ws_bytes) {
    CUDA_OK(cudaSetDevice(r->rank));
    for (int q = 0; q < world; ++q) {
        int can = 0;
        if (q == r->rank) continue;
        CUDA_OK(cudaDeviceCanAccessPeer(&can, r->rank, q));
        if (!can) return fail("--gpus: a pair of GPUs has no peer access");
        const cudaError_t e = cudaDeviceEnablePeerAccess(q, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else CUDA_OK(e);
    }
    CUDA_OK(cudaStreamCreate(&r->stream));
    CUDA_OK(cudaStreamCreate(&r->side));
    for (int k = 0; k <= DELORA_TRAIN_GROUP_BUCKETS; ++k)
        CUDA_OK(cudaEventCreateWithFlags(&r->events[k], cudaEventDisableTiming));
    float* d_state[3];
    int64_t* d_step;
    for (int i = 0; i < 3; ++i) {
        CUDA_OK(cudaMalloc((void**)&d_state[i], n * sizeof(float)));
        CUDA_OK(cudaMemcpy(d_state[i], h_state[i], n * sizeof(float), cudaMemcpyHostToDevice));
    }
    CUDA_OK(cudaMalloc((void**)&d_step, sizeof(int64_t)));
    CUDA_OK(cudaMemcpy(d_step, &step, sizeof(int64_t), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc(&r->workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc((void**)&r->points, (size_t)2 * r->B_max * r->scan_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&r->counts, (size_t)2 * r->B_max * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&r->losses, (size_t)r->B_max * DELORA_LOSS_ROW * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&r->flags, (size_t)delora_grad_allreduce_flag_words() * sizeof(uint32_t)));
    CUDA_OK(cudaMemset(r->flags, 0, (size_t)delora_grad_allreduce_flag_words() * sizeof(uint32_t)));
    CUDA_OK(cudaMalloc((void**)&r->status, sizeof(int32_t)));
    CUDA_OK(cudaMemset(r->status, 0, sizeof(int32_t)));
    r->h_losses = (float*)malloc((size_t)r->B_max * DELORA_LOSS_ROW * sizeof(float));
    r->h_step_counts = (int32_t*)malloc((size_t)2 * r->B_max * sizeof(int32_t));
    if (!r->h_losses || !r->h_step_counts) return fail("out of host memory");
    DELORA_OK(delora_odometry_train_init(r->d, d_state[0], r->workspace, r->stream));
    DELORA_OK(delora_odometry_train_set_state(r->d, d_state[0], d_state[1], d_state[2], d_step, r->workspace,
                                              r->stream));
    DELORA_OK(delora_odometry_train_set_dropout_seed(r->d, dropout_seed + (uint64_t)r->rank, r->workspace, r->stream));
    CUDA_OK(cudaStreamSynchronize(r->stream));
    for (int i = 0; i < 3; ++i) cudaFree(d_state[i]);
    cudaFree(d_step);
    return 0;
}

static void rank_release(rank_state* r) {
    cudaSetDevice(r->rank);
    free(r->h_step_counts);
    free(r->h_losses);
    cudaFree(r->status);
    cudaFree(r->flags);
    cudaFree(r->losses);
    cudaFree(r->counts);
    cudaFree(r->points);
    cudaFree(r->workspace);
    for (int k = 0; k <= DELORA_TRAIN_GROUP_BUCKETS; ++k) cudaEventDestroy(r->events[k]);
    cudaStreamDestroy(r->side);
    cudaStreamDestroy(r->stream);
}

int main(int argc, char** argv) {
    float lr = 1e-5f;
    double switch_below = 1e-2;
    const char* seed_arg = getenv("DELORA_DROPOUT_SEED");
    const char* eval_dir = NULL;
    int gpus = 1;
    int n_geom = 0;                           /* --geometry datasets, after the header's (dataset 0) */
    const char* geom_args[MAX_GEOMETRIES];
    int a = 1;
    for (; a + 1 < argc && strncmp(argv[a], "--", 2) == 0; a += 2) {
        if (strcmp(argv[a], "--lr") == 0) lr = (float)atof(argv[a + 1]);
        else if (strcmp(argv[a], "--switch-below") == 0) switch_below = atof(argv[a + 1]);
        else if (strcmp(argv[a], "--dropout-seed") == 0) seed_arg = argv[a + 1];
        else if (strcmp(argv[a], "--eval-dir") == 0) eval_dir = argv[a + 1];
        else if (strcmp(argv[a], "--gpus") == 0) gpus = atoi(argv[a + 1]);
        else if (strcmp(argv[a], "--geometry") == 0) {
            if (n_geom == MAX_GEOMETRIES - 1) return fail("too many --geometry options");
            geom_args[n_geom++] = argv[a + 1];
        }
        else return fail("unknown option");
    }
    /* checked before anything is read, against a dummy descriptor; parsed again below against the header's */
    for (int g = 0; g < n_geom; ++g) {
        delora_odometry_desc probe;
        char* dir;
        memset(&probe, 0, sizeof probe);
        if (parse_geometry(geom_args[g], &probe, &dir, &probe))
            return fail("--geometry wants DIR,H,W,VFOV0,VFOV1[,W_PRE]: a directory, integers H >= 1, W >= 2 and "
                        "W_PRE >= 0, and the vertical field of view in degrees with VFOV0 < VFOV1");
        free(dir);
    }
    if (n_geom > 0 && gpus != 1) return fail("--geometry trains on one GPU: it does not combine with --gpus");
    if (argc - a < 6)
        return fail("usage: odometry_train [--lr LR] [--switch-below L] [--dropout-seed S] [--eval-dir DIR] [--gpus N] "
                    "[--geometry DIR,H,W,VFOV0,VFOV1[,W_PRE]]... in.dlt|in.dlw out.dlt epochs B scan.bin scan.bin "
                    "[scan.bin ...]");
    const char* in_path = argv[a];
    const char* out_path = argv[a + 1];
    const int epochs = atoi(argv[a + 2]);
    const int B_max = atoi(argv[a + 3]);
    const int n_scans = argc - a - 4;
    char** scan_paths = argv + a + 4;

    /* the .dlw header is the first 128 bytes of both formats; a .dlt adds Adam's state after it */
    delora_odometry_train_file_header hdr;
    memset(&hdr, 0, sizeof hdr);
    FILE* f = fopen(in_path, "rb");
    if (!f) return fail("cannot open the input file");
    if (fread(&hdr.base, sizeof hdr.base, 1, f) != 1) return fail("truncated header");
    const int is_dlt = memcmp(hdr.base.magic, DELORA_TRAINING_FILE_MAGIC, 8) == 0;
    if (!is_dlt && memcmp(hdr.base.magic, DELORA_ODOMETRY_FILE_MAGIC, 8) != 0) return fail("not a .dlw or .dlt file");
    if (hdr.base.abi_version != delora_abi_version()) return fail("input file and library ABI versions differ");
    const int normalized = (hdr.base.model_flags & DELORA_MODEL_NORMALIZATION_SCALING) != 0;
    if (normalized && hdr.base.desc.w_pre == 0)
        return fail("the model was trained with normalization_scaling, which trains on the reference's recipe only: "
                    "export it with preprocessing normals (w_pre > 0)");
    if (is_dlt && fread((char*)&hdr + sizeof hdr.base, sizeof hdr - sizeof hdr.base, 1, f) != 1)
        return fail("truncated header");
    const delora_odometry_desc* d = &hdr.base.desc;
    const int64_t n_weights = delora_odometry_weight_floats(d);
    if (n_weights < 0) return fail(delora_last_error());
    if (n_weights != hdr.base.blob_floats) return fail("blob length does not match the descriptor");
    const size_t n = (size_t)n_weights;
    float* h_state[3];
    for (int i = 0; i < 3; ++i) {
        h_state[i] = (float*)calloc(n, sizeof(float));
        if (!h_state[i]) return fail("out of host memory");
    }
    for (int i = 0; i < (is_dlt ? 3 : 1); ++i)
        if (fread(h_state[i], sizeof(float), n, f) != n) return fail("truncated blob");
    fclose(f);
    if (!is_dlt) {            /* weights only: a fresh Adam, the ICP objective */
        hdr.step = 0; hdr.epoch = 0; hdr.unsupervised = 1;
        hdr.lr = lr; hdr.beta1 = 0.9f; hdr.beta2 = 0.999f; hdr.eps = 1e-8f; hdr.loss = 0.0f;
    }
    memcpy(hdr.base.magic, DELORA_TRAINING_FILE_MAGIC, 8);
    hdr.base.abi_version = delora_abi_version();
    hdr.base.header_bytes = (int32_t)sizeof hdr;
    memset(hdr.base.reserved, 0, sizeof hdr.base.reserved);
    memset(hdr.reserved, 0, sizeof hdr.reserved);
    if (seed_arg) {
        const unsigned long long s = strtoull(seed_arg, NULL, 0);
        hdr.dropout_seed[0] = (uint32_t)s;
        hdr.dropout_seed[1] = (uint32_t)(s >> 32);
    }
    const uint64_t dropout_seed = (uint64_t)hdr.dropout_seed[0] | ((uint64_t)hdr.dropout_seed[1] << 32);
    const int dropout = (hdr.base.model_flags & DELORA_MODEL_DROPOUT) != 0;
    uint32_t objective;                       /* the file's ICP objective (zeros in the header: the shipped one) */
    float lambda_po2pl;
    if (delora_odometry_file_objective(&hdr.base, &objective, &lambda_po2pl)) return fail(delora_last_error());
    print_objective("odometry_train", objective, lambda_po2pl);

    const int n_pairs = n_scans - 1;
    if (B_max < 1 || B_max > d->max_batch) return fail("B must be in [1, the header's max_batch]");
    if (epochs < 0) return fail("epochs must be >= 0");
    const size_t scan_floats = (size_t)3 * d->n_stride;
    float *h_scans, *h_eval_scans = NULL;
    int32_t *h_counts, *h_eval_counts = NULL;
    if (load_scans(scan_paths, n_scans, d->n_stride, &h_scans, &h_counts)) return 1;
    int n_eval_pairs = 0;
    if (eval_dir) {
        char** eval_paths;
        const int n_eval = list_scans(eval_dir, &eval_paths);
        if (n_eval < 2) return fail("--eval-dir needs a directory with at least two .bin scans");
        if (load_scans(eval_paths, n_eval, d->n_stride, &h_eval_scans, &h_eval_counts)) return 1;
        for (int k = 0; k < n_eval; ++k) free(eval_paths[k]);
        free(eval_paths);
        n_eval_pairs = n_eval - 1;
    }

    delora_odometry_train_params hp;
    hp.lr = hdr.lr; hp.beta1 = hdr.beta1; hp.beta2 = hdr.beta2; hp.eps = hdr.eps;
    hp.lambda_po2pl = lambda_po2pl;
    hp.nb_h = 7; hp.nb_w = 11;
    hp.epsilon_range = 0.5f;
    hp.min_neighbors = 10;

    if (gpus < 1 || gpus > DELORA_GRAD_ALLREDUCE_MAX_WORLD) return fail("--gpus must be in [1, 16]");
    if (gpus > 1) {
        int n_dev = 0;
        CUDA_OK(cudaGetDeviceCount(&n_dev));
        if (gpus > n_dev) return fail("--gpus: more GPUs than the machine has");
        const int per = n_pairs / gpus;
        if (per < 1) return fail("--gpus: fewer pairs than GPUs");
        if (per * gpus < n_pairs)
            fprintf(stderr, "odometry_train: %d GPUs x %d pairs, the last %d pair(s) left out\n", gpus, per,
                    n_pairs - per * gpus);
        const int64_t ws_bytes = delora_odometry_train_workspace_bytes(d);
        if (ws_bytes < 0) return fail(delora_last_error());
        rank_state* ranks = (rank_state*)calloc((size_t)gpus, sizeof *ranks);
        pthread_t* threads = (pthread_t*)calloc((size_t)gpus, sizeof *threads);
        if (!ranks || !threads) return fail("out of host memory");
        for (int r = 0; r < gpus; ++r) {
            rank_state* R = &ranks[r];
            R->rank = r; R->d = d; R->h_scans = h_scans; R->h_counts = h_counts;
            R->first = r * per; R->n_pairs = per; R->B_max = B_max; R->scan_floats = scan_floats;
            if (rank_setup(R, gpus, h_state, n, hdr.step, dropout_seed, ws_bytes)) return 1;
        }
        for (int r = 0; r < gpus; ++r) {
            delora_odometry_train_group* g = &ranks[r].g;
            memset(g, 0, sizeof *g);
            g->rank = r; g->world = gpus;
            for (int q = 0; q < gpus; ++q) {
                g->peer_ws[q] = (uint64_t)(uintptr_t)ranks[q].workspace;
                g->peer_flags[q] = (uint64_t)(uintptr_t)ranks[q].flags;
            }
            g->multicast = 0;
            g->n_ctas = 16; g->n_threads = 128;
            g->status = ranks[r].status;
            g->side_stream = ranks[r].side;
            for (int k = 0; k < DELORA_TRAIN_GROUP_BUCKETS; ++k) g->fork_events[k] = ranks[r].events[k];
            g->join_event = ranks[r].events[DELORA_TRAIN_GROUP_BUCKETS];
        }
        CUDA_OK(cudaSetDevice(0));
        float* d_state[3];
        int64_t* d_step;
        for (int i = 0; i < 3; ++i) CUDA_OK(cudaMalloc((void**)&d_state[i], n * sizeof(float)));
        CUDA_OK(cudaMalloc((void**)&d_step, sizeof(int64_t)));
        if (dropout) fprintf(stderr, "odometry_train: dropout on, seed %llu + GPU\n", (unsigned long long)dropout_seed);
        fprintf(stderr, "odometry_train: epoch %d, Adam step %lld, %s, %d pairs on %d GPUs\n", hdr.epoch,
                (long long)hdr.step, hdr.unsupervised ? "unsupervised" : "identity pre-training", per * gpus, gpus);
        rank_state* R0 = &ranks[0];
        for (int e = 0; e < epochs; ++e) {
            hp.loss_flags = objective | (hdr.unsupervised ? 0u : DELORA_LOSS_IDENTITY_FIT) |
                            (normalized ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u) | (dropout ? DELORA_TRAIN_DROPOUT : 0u);
            for (int r = 0; r < gpus; ++r) {
                ranks[r].hp = hp;
                ranks[r].identity = !hdr.unsupervised;
                if (pthread_create(&threads[r], NULL, rank_thread, &ranks[r]) != 0) return fail("cannot start a thread");
            }
            double mean = 0.0;
            int failed = 0;
            for (int r = 0; r < gpus; ++r) {
                pthread_join(threads[r], NULL);
                failed |= ranks[r].rc;
                mean += ranks[r].mean;
            }
            if (failed) return 1;
            mean /= gpus;
            printf("epoch %d objective %.9g unsupervised %d", hdr.epoch, mean, hdr.unsupervised);
            CUDA_OK(cudaSetDevice(0));
            if (eval_dir) {
                double held;
                if (held_out(d, &hp, h_eval_scans, h_eval_counts, n_eval_pairs, B_max, scan_floats, R0->workspace,
                             R0->points, R0->counts, R0->losses, R0->h_losses, R0->h_step_counts, R0->stream, &held))
                    return 1;
                printf(" held-out %.9g", held);
            }
            printf("\n");
            hdr.epoch += 1;
            hdr.loss = (float)mean;
            if (!hdr.unsupervised && mean < switch_below) {
                hdr.unsupervised = 1;
                fprintf(stderr, "odometry_train: objective below %g, switching to the unsupervised objective\n",
                        switch_below);
            }
            /* every GPU holds the same state: GPU 0's goes to the file */
            DELORA_OK(delora_odometry_train_get_state(d, R0->workspace, d_state[0], d_state[1], d_state[2], d_step,
                                                      R0->stream));
            for (int i = 0; i < 3; ++i)
                CUDA_OK(cudaMemcpyAsync(h_state[i], d_state[i], n * sizeof(float), cudaMemcpyDeviceToHost, R0->stream));
            CUDA_OK(cudaMemcpyAsync(&hdr.step, d_step, sizeof(int64_t), cudaMemcpyDeviceToHost, R0->stream));
            CUDA_OK(cudaStreamSynchronize(R0->stream));
            if (write_dlt(out_path, &hdr, h_state, n)) return 1;
        }
        for (int i = 0; i < 3; ++i) cudaFree(d_state[i]);
        cudaFree(d_step);
        for (int r = 0; r < gpus; ++r) rank_release(&ranks[r]);
        free(threads);
        free(ranks);
        for (int i = 0; i < 3; ++i) free(h_state[i]);
        free(h_eval_counts);
        free(h_eval_scans);
        free(h_counts);
        free(h_scans);
        return 0;
    }

    /* dataset 0: the header's geometry and the listed scans; 1 .. n_geom: the --geometry ones */
    const int n_sets = 1 + n_geom;
    delora_odometry_desc descs[MAX_GEOMETRIES];
    float* set_scans[MAX_GEOMETRIES];
    int32_t* set_counts[MAX_GEOMETRIES];
    int set_pairs[MAX_GEOMETRIES];
    descs[0] = *d; set_scans[0] = h_scans; set_counts[0] = h_counts; set_pairs[0] = n_pairs;
    for (int g = 1; g < n_sets; ++g) {
        char *dir, **paths;
        if (parse_geometry(geom_args[g - 1], d, &dir, &descs[g])) return fail("bad --geometry");
        if (normalized && descs[g].w_pre == 0)
            return fail("--geometry: a model trained with normalization_scaling needs W_PRE > 0 on every geometry");
        const int n_set = list_scans(dir, &paths);
        if (n_set < 2) return fail("--geometry needs a directory with at least two .bin scans");
        if (load_scans(paths, n_set, d->n_stride, &set_scans[g], &set_counts[g])) return 1;
        for (int k = 0; k < n_set; ++k) free(paths[k]);
        free(paths);
        free(dir);
        set_pairs[g] = n_set - 1;
    }
    /* the epoch's batches (dataset, first pair, size), each dataset's in order */
    int n_batches = 0;
    for (int g = 0; g < n_sets; ++g) n_batches += (set_pairs[g] + B_max - 1) / B_max;
    int (*batches)[3] = (int (*)[3])malloc(sizeof(int[3]) * (size_t)(n_batches > 0 ? n_batches : 1));
    if (!batches) return fail("out of host memory");

    cudaStream_t stream;
    CUDA_OK(cudaStreamCreate(&stream));
    float *d_state[3], *points, *losses;
    int64_t* d_step;
    int32_t* counts;
    void* workspace;
    const int64_t ws_bytes = delora_odometry_train_geometries_workspace_bytes(descs, n_sets);
    if (ws_bytes < 0) return fail(delora_last_error());
    for (int i = 0; i < 3; ++i) {
        CUDA_OK(cudaMalloc((void**)&d_state[i], n * sizeof(float)));
        CUDA_OK(cudaMemcpy(d_state[i], h_state[i], n * sizeof(float), cudaMemcpyHostToDevice));
    }
    CUDA_OK(cudaMalloc((void**)&d_step, sizeof(int64_t)));
    CUDA_OK(cudaMemcpy(d_step, &hdr.step, sizeof(int64_t), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc(&workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc((void**)&points, (size_t)2 * B_max * scan_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&counts, (size_t)2 * B_max * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&losses, (size_t)B_max * DELORA_LOSS_ROW * sizeof(float)));
    DELORA_OK(delora_odometry_train_geometries_init(descs, n_sets, d_state[0], workspace, stream));
    DELORA_OK(delora_odometry_train_set_state(d, d_state[0], d_state[1], d_state[2], d_step, workspace, stream));
    DELORA_OK(delora_odometry_train_set_dropout_seed(d, dropout_seed, workspace, stream));
    int armed = 0;                            /* the dataset whose geometry the workspace is armed for */
    if (dropout) fprintf(stderr, "odometry_train: dropout on, seed %llu\n", (unsigned long long)dropout_seed);
    fprintf(stderr, "odometry_train: epoch %d, Adam step %lld, %s, %d pairs\n", hdr.epoch, (long long)hdr.step,
            hdr.unsupervised ? "unsupervised" : "identity pre-training", n_pairs);
    for (int g = 1; g < n_sets; ++g)
        fprintf(stderr, "odometry_train: dataset %d: %d x %d, w_pre %d, %d pairs\n", g, descs[g].H, descs[g].W,
                descs[g].w_pre, set_pairs[g]);

    float* h_losses = (float*)malloc((size_t)B_max * DELORA_LOSS_ROW * sizeof(float));
    int32_t* h_step_counts = (int32_t*)malloc((size_t)2 * B_max * sizeof(int32_t));
    if (!h_losses || !h_step_counts) return fail("out of host memory");
    for (int e = 0; e < epochs; ++e) {
        hp.loss_flags = objective | (hdr.unsupervised ? 0u : DELORA_LOSS_IDENTITY_FIT) |
                        (normalized ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u) | (dropout ? DELORA_TRAIN_DROPOUT : 0u);
        int nb = 0;
        for (int g = 0; g < n_sets; ++g)
            for (int k0 = 0; k0 < set_pairs[g]; k0 += B_max, ++nb) {
                batches[nb][0] = g;
                batches[nb][1] = k0;
                batches[nb][2] = set_pairs[g] - k0 < B_max ? set_pairs[g] - k0 : B_max;
            }
        if (n_sets > 1) {         /* Fisher-Yates, drawn from the epoch number so that a resumed run repeats it */
            uint64_t rng = (uint64_t)hdr.epoch;
            for (int j = n_batches - 1; j > 0; --j) {
                const int i = (int)(splitmix64(&rng) % (uint64_t)(j + 1));
                int t[3];
                memcpy(t, batches[i], sizeof t);
                memcpy(batches[i], batches[j], sizeof t);
                memcpy(batches[j], t, sizeof t);
            }
        }
        double sum = 0.0;
        int steps = 0;
        for (; steps < n_batches; ++steps) {
            const int g = batches[steps][0], k0 = batches[steps][1], B = batches[steps][2];
            if (g != armed) {
                DELORA_OK(delora_odometry_train_use_geometry(descs, n_sets, g, workspace, stream));
                armed = g;
            }
            if (stage_pairs(set_scans[g], set_counts[g], k0, B, scan_floats, points, counts, h_step_counts, stream))
                return 1;
            DELORA_OK(delora_odometry_train_step(&descs[g], &hp, points, counts, B, workspace, losses, NULL, NULL, NULL,
                                                 stream));
            CUDA_OK(cudaMemcpyAsync(h_losses, losses, (size_t)B * DELORA_LOSS_ROW * sizeof(float),
                                    cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            if (!hdr.unsupervised) {
                sum += (double)h_losses[(size_t)(B - 1) * DELORA_LOSS_ROW + 5];
            } else {
                sum += icp_objective(h_losses, B, hp.lambda_po2pl);
            }
        }
        const double mean = steps > 0 ? sum / steps : 0.0;
        printf("epoch %d objective %.9g unsupervised %d", hdr.epoch, mean, hdr.unsupervised);
        if (eval_dir) {         /* the held-out pairs with the weights after the epoch; no update, no dropout */
            double held;
            if (armed != 0) {
                DELORA_OK(delora_odometry_train_use_geometry(descs, n_sets, 0, workspace, stream));
                armed = 0;
            }
            if (held_out(d, &hp, h_eval_scans, h_eval_counts, n_eval_pairs, B_max, scan_floats, workspace, points, counts,
                         losses, h_losses, h_step_counts, stream, &held))
                return 1;
            printf(" held-out %.9g", held);
        }
        printf("\n");
        hdr.epoch += 1;
        hdr.loss = (float)mean;
        if (!hdr.unsupervised && mean < switch_below) {
            hdr.unsupervised = 1;
            fprintf(stderr, "odometry_train: objective below %g, switching to the unsupervised objective\n",
                    switch_below);
        }
        /* the state after the epoch, in the phase the next epoch runs */
        DELORA_OK(delora_odometry_train_get_state(d, workspace, d_state[0], d_state[1], d_state[2], d_step, stream));
        for (int i = 0; i < 3; ++i)
            CUDA_OK(cudaMemcpyAsync(h_state[i], d_state[i], n * sizeof(float), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(&hdr.step, d_step, sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        if (write_dlt(out_path, &hdr, h_state, n)) return 1;
    }

    free(h_step_counts);
    free(h_losses);
    free(h_eval_counts);
    free(h_eval_scans);
    free(batches);
    for (int g = 0; g < n_sets; ++g) {
        free(set_counts[g]);
        free(set_scans[g]);
    }
    for (int i = 0; i < 3; ++i) {
        free(h_state[i]);
        cudaFree(d_state[i]);
    }
    cudaFree(d_step);
    cudaFree(losses);
    cudaFree(counts);
    cudaFree(points);
    cudaFree(workspace);
    cudaStreamDestroy(stream);
    return 0;
}
