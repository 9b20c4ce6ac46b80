/*
 * Several LiDAR streams from a C host, batched in one workspace: no Python, no torch.  Links libdelora_b200.so and
 * cudart only.
 *
 *   odometry_streams [--residual | --information | --preprocessing [--information]] model.dlw stream0_dir ...
 *   odometry_streams --adapt LR --adapt-out adapted.dlw [--gpus N] [--information] model.dlw stream0_dir ...
 *   odometry_streams --adapt LR --adapt-out adapted.dlw [--geometry DIR,H,W,VFOV0,VFOV1[,W_PRE]]... [--information]
 *                    model.dlw stream0_dir ...
 *
 * model.dlw is written by bin/export_odometry_weights.py (layout: include/delora_b200.h); every directory holds one
 * stream's KITTI velodyne .bin files ([N, 4] float32 rows: x, y, z, reflectance), taken in name order.  All streams
 * share the model and the sensor geometry of model.dlw; the number of directories is the number of streams.  Streams
 * of different lengths go inactive once they run out of scans.  Per tick, for every stream with a transform, it prints
 * one line: the stream index, the frame index k, and T_{k-1,k} as 12 floats (the top three rows of the 4x4, row-major).
 * --residual serves the streams through delora_odometry_streams_push_residual and appends to each line the frame's ICP
 * residual against the stream's previous frame: the point-to-plane loss, the plane-to-plane loss and the matched pairs
 * (normals on the model's image, 7 x 11 neighbourhood, the reference's defaults).  The transforms are the same bits.
 * --information serves the streams through delora_odometry_streams_push_info: the --residual columns, then how well the
 * frame determines its transform (the Gauss-Newton information H of the residual's objective at T): H's smallest
 * eigenvalue, its unit eigenvector (x, y, z, rot x, rot y, rot z: the direction the frame constrains least) and the
 * ratio of the largest eigenvalue to the smallest (large in a corridor, an open field or at a flat wall).
 * --information with --preprocessing (delora_odometry_streams_push_pre_info) or with --adapt, --gpus included
 * (delora_odometry_streams_push_adapt_info / _push_adapt_group_info) or with --adapt and --geometry
 * (delora_odometry_streams_push_adapt_geometries_info, every stream of every sensor) appends the same three columns to
 * those modes' lines, for plain and normalization_scaling files alike: the information is always in the metres and
 * radians of the printed T.  The transforms, residual columns and adapted weights are the same bits as without it.
 * Options may come in any order before model.dlw.
 * A model trained with normalization_scaling (model_flags has DELORA_MODEL_NORMALIZATION_SCALING) is served through
 * delora_odometry_streams_push_normalized, with the same output; --residual is refused for such a model.
 * --preprocessing serves the streams on the reference's two-resolution recipe through delora_odometry_streams_push_pre:
 * each frame's normals at the header's w_pre, its points projected again at the model's width (the images the model
 * trained on with --preprocessing-normals, and the reference's Tester's input), and appends the same three residual
 * columns, the training step's ICP in the model's units, for plain and normalization_scaling files alike.  It refuses
 * a file with w_pre = 0 (export it with bin/export_odometry_weights.py --preprocessing-normals).  The recipe adds a
 * projection + normals at H x w_pre per frame, a second H x W projection per pair, the ICP and the cache write to the
 * raw-scan tick: on one H100 80GB HBM3 at 700 W, w_pre 2250, graph-replayed, ms per tick --residual / --preprocessing
 * at 64 x 720: 1.20 / 1.21 (1 stream), 1.41 / 1.47 (4), 5.14 / 5.44 (16); at 64 x 2048: 1.29 / 1.31, 2.31 / 2.38,
 * 8.73 / 8.98 (scripts/gpu_odometry_streams_pre.py, profiles/odometry_streams_pre_h100_700w.json).
 * --adapt LR --adapt-out FILE.dlw serves the streams while the model adapts to them, through
 * delora_odometry_streams_push_adapt with update = 1: every tick serves the streams with the current weights, prints
 * the same three residual columns (the training step's ICP), then takes one Adam step (learning rate LR, betas 0.9 /
 * 0.999) on the mean objective of the pairs it served.  Normals at the header's w_pre when it is > 0, else on the
 * model's image; a normalization_scaling file needs w_pre > 0, and a use_dropout file is refused.  At the end the
 * adapted weights are written to FILE.dlw with the input file's header.  A tick costs one training step at B = S
 * (64 x 720: 3.51 ms for 1 stream, 14.20 ms for 16, on one H100 80GB HBM3 at 700 W; scripts/
 * gpu_odometry_streams_adapt.py, profiles/odometry_streams_adapt_h100_700w.json).
 * --adapt ... --gpus N adapts ONE model from streams served on GPUs 0 .. N-1 of this process, one host thread per GPU,
 * peer access between every pair, through delora_odometry_streams_push_adapt_group: each GPU serves S = ceil(streams /
 * N) streams, stream s on GPU s / S (the streams past the last directory stay inactive), and every tick's update is
 * the mean over the valid pairs of all GPUs, so all GPUs keep the same weights.  GPU 0 writes FILE.dlw.  The output
 * lines are the same as on one GPU; --gpus 1 writes the file a run without the option writes.  --gpus is refused
 * without --adapt.
 * --adapt ... --geometry DIR,H,W,VFOV0,VFOV1[,W_PRE] (repeatable, one GPU; the syntax of odometry_train.c): one more
 * stream, recorded by another sensor: the .bin files of DIR, served at the header's descriptor with H, W, the vertical
 * field of view (degrees) and w_pre (default 0) replaced.  The streams of every sensor adapt ONE model in one
 * workspace through delora_odometry_streams_push_adapt_geometries: the directories after model.dlw are geometry 0
 * (the header's), each --geometry is a geometry of one stream, numbered after them; every tick's update is the mean
 * over the valid pairs of all sensors.  The output lines are as above.  --geometry is refused without --adapt and
 * with --gpus; W must have the parity of the header's W, and a normalization_scaling file needs W_PRE > 0.
 *
 * Build:  cc odometry_streams.c -I include -I $CUDA_HOME/include -L delora_b200 -ldelora_b200 \
 *            -L $CUDA_HOME/lib64 -lcudart -lpthread -Wl,-rpath,$PWD/delora_b200 -o odometry_streams
 */
#include <dirent.h>
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "delora_b200.h"

#define MAX_GEOMETRIES 16
#define DEG_TO_RAD (3.14159265358979323846 / 180.0)

static int fail(const char* what) {
    fprintf(stderr, "odometry_streams: %s\n", what);
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

#define CUDA_OK(call)                                                                  \
    do {                                                                               \
        cudaError_t e_ = (call);                                                       \
        if (e_ != cudaSuccess) return fail(cudaGetErrorString(e_));                     \
    } while (0)

#define DELORA_OK(call)                                                                \
    do {                                                                               \
        if ((call) != 0) return fail(delora_last_error());                             \
    } while (0)

typedef struct {
    char** paths;
    int n;
} scan_list;

static int by_name(const void* a, const void* b) { return strcmp(*(char* const*)a, *(char* const*)b); }

/* the .bin files of one directory, sorted by name; 0 on success */
static int list_scans(const char* dir, scan_list* out) {
    DIR* d = opendir(dir);
    if (!d) return 1;
    int cap = 16;
    out->n = 0;
    out->paths = (char**)malloc(sizeof(char*) * (size_t)cap);
    if (!out->paths) { closedir(d); return 1; }
    const struct dirent* e;
    while ((e = readdir(d)) != NULL) {
        const size_t len = strlen(e->d_name);
        if (len < 5 || strcmp(e->d_name + len - 4, ".bin") != 0) continue;
        if (out->n == cap) {
            cap *= 2;
            char** grown = (char**)realloc(out->paths, sizeof(char*) * (size_t)cap);
            if (!grown) { closedir(d); return 1; }
            out->paths = grown;
        }
        char* p = (char*)malloc(strlen(dir) + len + 2);
        if (!p) { closedir(d); return 1; }
        sprintf(p, "%s/%s", dir, e->d_name);
        out->paths[out->n++] = p;
    }
    closedir(d);
    qsort(out->paths, (size_t)out->n, sizeof(char*), by_name);
    return 0;
}

/* one KITTI .bin -> channels-first x, y, z rows of stride n_stride; the point count, or -1 */
static int32_t read_scan(const char* path, float* dst, int n_stride) {
    FILE* s = fopen(path, "rb");
    if (!s) return -1;
    fseek(s, 0, SEEK_END);
    const long bytes = ftell(s);
    fseek(s, 0, SEEK_SET);
    const int32_t n = (int32_t)(bytes / (4 * sizeof(float)));
    if (n > n_stride) { fclose(s); return -1; }
    float* rows = (float*)malloc((size_t)n * 4 * sizeof(float) + 1);
    if (!rows || fread(rows, 4 * sizeof(float), (size_t)n, s) != (size_t)n) { free(rows); fclose(s); return -1; }
    fclose(s);
    memset(dst, 0, (size_t)3 * n_stride * sizeof(float));
    for (int32_t i = 0; i < n; ++i)
        for (int c = 0; c < 3; ++c) dst[(size_t)c * n_stride + i] = rows[(size_t)i * 4 + c];
    free(rows);
    return n;
}

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

/* --adapt --gpus N: one GPU of the group, serving streams rank * S .. rank * S + S - 1 (those past the last directory
 * stay inactive), and the tick its thread runs */
typedef struct {
    int rank, S, k;
    const delora_odometry_desc* d;
    const delora_odometry_train_params* hp;
    const scan_list* lists;
    int n_lists;
    cudaStream_t stream, side;
    cudaEvent_t events[DELORA_TRAIN_GROUP_BUCKETS + 1];
    delora_odometry_train_group g;
    void* workspace;
    void* flags;
    int32_t* status;
    float *weights, *points, *T, *losses;
    int32_t *count, *active, *valid;
    float *h_points, *h_T, *h_losses;
    int32_t *h_count, *h_active, *h_valid, h_status;
    float *info, *h_info;                     /* --information: the information rows, else NULL */
    int rc;
} rank_state;

/* --information's columns: the smallest eigenvalue of H, its unit eigenvector and the ratio of the largest to it */
static void print_info(const float* r) {    /* [36, 42): eigenvalues ascending; [42, 48): the smallest one's eigenvector */
    printf(" %.9g", r[36]);
    for (int i = 0; i < 6; ++i) printf(" %.6f", r[42 + i]);
    printf(" %.9g", r[36] > 0.0f ? r[41] / r[36] : INFINITY);
}

/* tick k of one rank: its scans up, one group tick with update = 1, T / valid / losses down */
static int rank_tick(rank_state* r) {
    const delora_odometry_desc* d = r->d;
    const int S = r->S;
    const size_t pts_floats = (size_t)S * 3 * d->n_stride;
    CUDA_OK(cudaSetDevice(r->rank));
    for (int s = 0; s < S; ++s) {
        const int gs = r->rank * S + s;
        r->h_active[s] = gs < r->n_lists && r->k < r->lists[gs].n;
        r->h_count[s] = 0;
        if (!r->h_active[s]) continue;
        r->h_count[s] = read_scan(r->lists[gs].paths[r->k], r->h_points + (size_t)s * 3 * d->n_stride, d->n_stride);
        if (r->h_count[s] < 0) return fail("cannot read a scan (missing, truncated or more points than n_stride)");
    }
    CUDA_OK(cudaMemcpyAsync(r->points, r->h_points, pts_floats * sizeof(float), cudaMemcpyHostToDevice, r->stream));
    CUDA_OK(cudaMemcpyAsync(r->count, r->h_count, (size_t)S * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    CUDA_OK(cudaMemcpyAsync(r->active, r->h_active, (size_t)S * sizeof(int32_t), cudaMemcpyHostToDevice, r->stream));
    if (r->info) {
        DELORA_OK(delora_odometry_streams_push_adapt_group_info(d, r->hp, &r->g, 1, r->points, r->count, r->active,
                                                                r->workspace, r->T, r->valid, r->losses, r->info,
                                                                r->stream));
        CUDA_OK(cudaMemcpyAsync(r->h_info, r->info, (size_t)S * DELORA_INFO_ROW * sizeof(float), cudaMemcpyDeviceToHost,
                                r->stream));
    } else {
        DELORA_OK(delora_odometry_streams_push_adapt_group(d, r->hp, &r->g, 1, r->points, r->count, r->active,
                                                           r->workspace, r->T, r->valid, r->losses, r->stream));
    }
    CUDA_OK(cudaMemcpyAsync(r->h_losses, r->losses, (size_t)S * DELORA_LOSS_ROW * sizeof(float), cudaMemcpyDeviceToHost,
                            r->stream));
    CUDA_OK(cudaMemcpyAsync(r->h_T, r->T, (size_t)S * 16 * sizeof(float), cudaMemcpyDeviceToHost, r->stream));
    CUDA_OK(cudaMemcpyAsync(r->h_valid, r->valid, (size_t)S * sizeof(int32_t), cudaMemcpyDeviceToHost, r->stream));
    CUDA_OK(cudaMemcpyAsync(&r->h_status, r->status, sizeof(int32_t), cudaMemcpyDeviceToHost, r->stream));
    CUDA_OK(cudaStreamSynchronize(r->stream));
    if (r->h_status != 0) return fail("--gpus: a peer did not reach the collective within 20 s");
    return 0;
}

static void* rank_thread(void* arg) {
    rank_state* r = (rank_state*)arg;
    r->rc = rank_tick(r);
    return NULL;
}

/* one GPU's workspace (initialised from the host blob), buffers, streams, events and zeroed flag words */
static int rank_setup(rank_state* r, int world, const float* h_blob, int64_t n_weights, int information) {
    const delora_odometry_desc* d = r->d;
    const int S = r->S;
    CUDA_OK(cudaSetDevice(r->rank));
    for (int q = 0; q < world; ++q) {
        if (q == r->rank) continue;
        int can = 0;
        CUDA_OK(cudaDeviceCanAccessPeer(&can, r->rank, q));
        if (!can) return fail("--gpus: a pair of GPUs has no peer access");
        const cudaError_t e = cudaDeviceEnablePeerAccess(q, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else CUDA_OK(e);
    }
    const int64_t ws_bytes = information ? delora_odometry_streams_adapt_info_workspace_bytes(d)
                                         : delora_odometry_streams_adapt_group_workspace_bytes(d);
    if (ws_bytes < 0) return fail(delora_last_error());
    const size_t pts_floats = (size_t)S * 3 * d->n_stride;
    CUDA_OK(cudaStreamCreate(&r->stream));
    CUDA_OK(cudaStreamCreate(&r->side));
    for (int k = 0; k <= DELORA_TRAIN_GROUP_BUCKETS; ++k)
        CUDA_OK(cudaEventCreateWithFlags(&r->events[k], cudaEventDisableTiming));
    CUDA_OK(cudaMalloc(&r->workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc(&r->flags, (size_t)delora_grad_allreduce_flag_words() * sizeof(uint32_t)));
    CUDA_OK(cudaMalloc((void**)&r->status, sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&r->weights, (size_t)n_weights * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&r->points, pts_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&r->count, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&r->active, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&r->valid, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&r->T, (size_t)S * 16 * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&r->losses, (size_t)S * DELORA_LOSS_ROW * sizeof(float)));
    if (information) CUDA_OK(cudaMalloc((void**)&r->info, (size_t)S * DELORA_INFO_ROW * sizeof(float)));
    CUDA_OK(cudaMemset(r->flags, 0, (size_t)delora_grad_allreduce_flag_words() * sizeof(uint32_t)));
    CUDA_OK(cudaMemset(r->status, 0, sizeof(int32_t)));
    CUDA_OK(cudaMemcpy(r->weights, h_blob, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
    if (information) DELORA_OK(delora_odometry_streams_adapt_info_init(d, r->weights, r->workspace, r->stream));
    else DELORA_OK(delora_odometry_streams_adapt_group_init(d, r->weights, r->workspace, r->stream));
    CUDA_OK(cudaStreamSynchronize(r->stream));
    r->h_points = (float*)malloc(pts_floats * sizeof(float));
    r->h_count = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    r->h_active = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    r->h_valid = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    r->h_T = (float*)malloc((size_t)S * 16 * sizeof(float));
    r->h_losses = (float*)calloc((size_t)S * DELORA_LOSS_ROW, sizeof(float));
    r->h_info = (float*)calloc((size_t)S * DELORA_INFO_ROW, sizeof(float));
    if (!r->h_points || !r->h_count || !r->h_active || !r->h_valid || !r->h_T || !r->h_losses || !r->h_info)
        return fail("out of host memory");
    return 0;
}

static void rank_release(rank_state* r) {
    cudaSetDevice(r->rank);
    free(r->h_info); free(r->h_losses); free(r->h_T); free(r->h_valid); free(r->h_active); free(r->h_count); free(r->h_points);
    cudaFree(r->info); cudaFree(r->losses); cudaFree(r->T); cudaFree(r->valid); cudaFree(r->active); cudaFree(r->count);
    cudaFree(r->points); cudaFree(r->weights); cudaFree(r->status); cudaFree(r->flags); cudaFree(r->workspace);
    for (int k = 0; k <= DELORA_TRAIN_GROUP_BUCKETS; ++k) cudaEventDestroy(r->events[k]);
    cudaStreamDestroy(r->side);
    cudaStreamDestroy(r->stream);
}

/* --adapt --gpus N: n_streams streams over GPUs 0 .. N-1, one model adapted from all of them; GPU 0 writes `out` */
static int adapt_group(int gpus, delora_odometry_desc desc, const delora_odometry_file_header* hdr, float* h_blob,
                       int64_t n_weights, const scan_list* lists, int n_streams, int ticks,
                       const delora_odometry_train_params* hp, const char* out, int information) {
    int n_dev = 0;
    CUDA_OK(cudaGetDeviceCount(&n_dev));
    if (gpus > n_dev) return fail("--gpus: more GPUs than the machine has");
    const int S = (n_streams + gpus - 1) / gpus;
    desc.max_batch = S;
    rank_state* ranks = (rank_state*)calloc((size_t)gpus, sizeof *ranks);
    pthread_t* threads = (pthread_t*)calloc((size_t)gpus, sizeof *threads);
    if (!ranks || !threads) return fail("out of host memory");
    for (int r = 0; r < gpus; ++r) {
        rank_state* R = &ranks[r];
        R->rank = r; R->S = S; R->d = &desc; R->hp = hp; R->lists = lists; R->n_lists = n_streams;
        if (rank_setup(R, gpus, h_blob, n_weights, information)) return 1;
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
        g->n_ctas = 8; g->n_threads = 128;
        g->status = ranks[r].status;
        g->side_stream = ranks[r].side;
        for (int k = 0; k < DELORA_TRAIN_GROUP_BUCKETS; ++k) g->fork_events[k] = ranks[r].events[k];
        g->join_event = ranks[r].events[DELORA_TRAIN_GROUP_BUCKETS];
    }
    for (int k = 0; k < ticks; ++k) {
        for (int r = 0; r < gpus; ++r) {
            ranks[r].k = k;
            if (pthread_create(&threads[r], NULL, rank_thread, &ranks[r]) != 0) return fail("cannot start a thread");
        }
        int failed = 0;
        for (int r = 0; r < gpus; ++r) {
            pthread_join(threads[r], NULL);
            failed |= ranks[r].rc;
        }
        if (failed) return 1;
        for (int gs = 0; gs < n_streams; ++gs) {
            const rank_state* R = &ranks[gs / S];
            const int s = gs % S;
            if (!R->h_valid[s]) continue;
            printf("%d %d", gs, k);
            for (int i = 0; i < 12; ++i) printf(" %.9g", R->h_T[(size_t)s * 16 + i]);
            const float* l = R->h_losses + (size_t)s * DELORA_LOSS_ROW;
            printf(" %.9g %.9g %.0f", l[1], l[2], l[3]);
            if (information) print_info(R->h_info + (size_t)s * DELORA_INFO_ROW);
            printf("\n");
        }
    }
    rank_state* R0 = &ranks[0];             /* every rank holds the same weights: GPU 0 writes them */
    CUDA_OK(cudaSetDevice(0));
    DELORA_OK(delora_odometry_train_weights(&desc, R0->workspace, R0->weights, R0->stream));
    CUDA_OK(cudaMemcpyAsync(h_blob, R0->weights, (size_t)n_weights * sizeof(float), cudaMemcpyDeviceToHost, R0->stream));
    CUDA_OK(cudaStreamSynchronize(R0->stream));
    FILE* o = fopen(out, "wb");
    if (!o) return fail("cannot open the --adapt-out file");
    const int ok = fwrite(hdr, sizeof *hdr, 1, o) == 1 &&
                   fwrite(h_blob, sizeof(float), (size_t)n_weights, o) == (size_t)n_weights;
    if (fclose(o) != 0 || !ok) return fail("cannot write the --adapt-out file");
    for (int r = 0; r < gpus; ++r) rank_release(&ranks[r]);
    free(threads);
    free(ranks);
    return 0;
}

/* the learning rate of --adapt: a finite number >= 0, the whole argument */
static int parse_lr(const char* arg, float* lr) {
    char* end;
    const double v = strtod(arg, &end);
    if (end == arg || *end != '\0' || !(v >= 0.0) || v > 3.0e38) return 1;
    *lr = (float)v;
    return 0;
}

int main(int argc, char** argv) {
    const char* adapt_lr = NULL;
    const char* adapt_out = NULL;
    const char* gpus_arg = NULL;
    int n_geom = 0;                           /* --geometry streams, after the directories of the header's geometry */
    const char* geom_args[MAX_GEOMETRIES];
    int information = 0, residual_opt = 0, pre = 0;
    for (;;) {
        if (argc > 1 && (strcmp(argv[1], "--information") == 0 || strcmp(argv[1], "--residual") == 0 ||
                         strcmp(argv[1], "--preprocessing") == 0)) {
            if (strcmp(argv[1], "--information") == 0) information = 1;
            else if (strcmp(argv[1], "--residual") == 0) residual_opt = 1;
            else pre = 1;
            --argc;
            ++argv;
            continue;
        }
        if (!(argc > 2 && (strcmp(argv[1], "--adapt") == 0 || strcmp(argv[1], "--adapt-out") == 0 ||
                           strcmp(argv[1], "--gpus") == 0 || strcmp(argv[1], "--geometry") == 0)))
            break;
        if (strcmp(argv[1], "--adapt") == 0) adapt_lr = argv[2];
        else if (strcmp(argv[1], "--adapt-out") == 0) adapt_out = argv[2];
        else if (strcmp(argv[1], "--gpus") == 0) gpus_arg = argv[2];
        else {
            if (n_geom == MAX_GEOMETRIES - 1) return fail("too many --geometry options");
            geom_args[n_geom++] = argv[2];
        }
        argc -= 2;
        argv += 2;
    }
    const int adapt = adapt_lr != NULL || adapt_out != NULL;
    float lr = 0.0f;
    if (adapt) {
        if (!adapt_lr || !adapt_out) return fail("--adapt LR and --adapt-out FILE.dlw go together");
        if (parse_lr(adapt_lr, &lr)) {
            char msg[256];
            snprintf(msg, sizeof msg, "--adapt: LR must be a finite number >= 0, got '%s'", adapt_lr);
            return fail(msg);
        }
    }
    int gpus = 0;
    if (gpus_arg) {
        if (!adapt) return fail("--gpus adapts one model on several GPUs: it needs --adapt LR --adapt-out FILE.dlw");
        char* end;
        const long v = strtol(gpus_arg, &end, 10);
        if (end == gpus_arg || *end != '\0' || v < 1 || v > DELORA_GRAD_ALLREDUCE_MAX_WORLD)
            return fail("--gpus must be in [1, 16]");
        gpus = (int)v;
    }
    if (n_geom > 0) {
        if (!adapt) return fail("--geometry adapts one model from several sensors: it needs --adapt LR --adapt-out "
                                "FILE.dlw");
        if (gpus) return fail("--geometry serves every sensor on one GPU: it does not combine with --gpus");
        for (int g = 0; g < n_geom; ++g) {         /* checked before anything is read, against a dummy descriptor */
            delora_odometry_desc probe;
            char* dir;
            memset(&probe, 0, sizeof probe);
            if (parse_geometry(geom_args[g], &probe, &dir, &probe))
                return fail("--geometry wants DIR,H,W,VFOV0,VFOV1[,W_PRE]: a directory, integers H >= 1, W >= 2 and "
                            "W_PRE >= 0, and the vertical field of view in degrees with VFOV0 < VFOV1");
            free(dir);
        }
    }
    if (adapt && (residual_opt || pre)) return fail("--adapt serves its own residual: drop --residual / --preprocessing");
    if (residual_opt && pre) return fail("--preprocessing serves its own residual: drop --residual");
    /* the raw-scan residual streams: --residual, or --information on its own */
    const int residual = residual_opt || (information && !pre && !adapt);
    if (argc < 3)
        return fail("usage: odometry_streams [--residual | --information | --preprocessing [--information]] model.dlw "
                    "stream_dir [stream_dir ...]");
    const int S_dirs = argc - 2;              /* the streams of the header's geometry */
    const int S = S_dirs + n_geom;            /* every stream, the --geometry ones last */

    /* weight file: fixed header, then the fp32 blob; the workspace serves S streams (max_batch = S) */
    FILE* f = fopen(argv[1], "rb");
    if (!f) return fail("cannot open the weight file");
    delora_odometry_file_header hdr;
    if (fread(&hdr, sizeof hdr, 1, f) != 1) return fail("truncated header");
    if (memcmp(hdr.magic, DELORA_ODOMETRY_FILE_MAGIC, 8) != 0) return fail("not a .dlw file");
    if (hdr.abi_version != delora_abi_version()) return fail("weight file and library ABI versions differ");
    const int normalized = (hdr.model_flags & DELORA_MODEL_NORMALIZATION_SCALING) != 0;
    if (normalized && residual)
        return fail("--residual is not provided for models trained with normalization_scaling (serve the file "
                    "without it)");
    if (adapt && (hdr.model_flags & DELORA_MODEL_DROPOUT))
        return fail("--adapt does not train with dropout: the served transforms are dropout-free");
    if (pre && hdr.desc.w_pre == 0)
        return fail("--preprocessing needs a file with w_pre > 0: export it with bin/export_odometry_weights.py "
                    "--preprocessing-normals");
    delora_odometry_desc desc = hdr.desc;
    desc.max_batch = S_dirs;
    const delora_odometry_desc* d = &desc;
    /* --geometry: geometry 0 is the header's, geometry g >= 1 serves stream S_dirs + g - 1 */
    const int n_sets = 1 + n_geom;
    delora_odometry_desc descs[MAX_GEOMETRIES];
    char* geom_dirs[MAX_GEOMETRIES];
    descs[0] = desc;
    for (int g = 1; g < n_sets; ++g) {
        if (parse_geometry(geom_args[g - 1], &desc, &geom_dirs[g - 1], &descs[g])) return fail("bad --geometry");
        descs[g].max_batch = 1;
    }
    const int64_t n_weights = delora_odometry_weight_floats(d);
    if (n_weights < 0) return fail(delora_last_error());
    if (n_weights != hdr.blob_floats) return fail("blob length does not match the descriptor");
    float* h_blob = (float*)malloc((size_t)n_weights * sizeof(float));
    if (!h_blob || fread(h_blob, sizeof(float), (size_t)n_weights, f) != (size_t)n_weights) return fail("truncated blob");
    fclose(f);

    scan_list* lists = (scan_list*)calloc((size_t)S, sizeof(scan_list));
    if (!lists) return fail("out of host memory");
    int ticks = 0;
    for (int s = 0; s < S; ++s) {
        if (list_scans(s < S_dirs ? argv[2 + s] : geom_dirs[s - S_dirs], &lists[s]))
            return fail("cannot list a stream directory");
        if (lists[s].n > ticks) ticks = lists[s].n;
    }

    delora_odometry_train_params hp;                       /* --adapt: Adam, and the residual's losses and neighbourhood */
    hp.lr = lr; hp.beta1 = 0.9f; hp.beta2 = 0.999f; hp.eps = 1e-8f;
    uint32_t objective;                       /* the file's ICP objective (zeros in the header: the shipped one) */
    float lambda_po2pl;
    if (delora_odometry_file_objective(&hdr, &objective, &lambda_po2pl)) return fail(delora_last_error());
    if (adapt || residual || pre) print_objective("odometry_streams", objective, lambda_po2pl);
    hp.lambda_po2pl = lambda_po2pl;
    hp.loss_flags = objective | (normalized ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u);
    hp.nb_h = 7; hp.nb_w = 11;
    hp.epsilon_range = 0.5f;
    hp.min_neighbors = 10;
    if (gpus) {
        const int rc = adapt_group(gpus, desc, &hdr, h_blob, n_weights, lists, S, ticks, &hp, adapt_out, information);
        for (int s = 0; s < S; ++s) {
            for (int i = 0; i < lists[s].n; ++i) free(lists[s].paths[i]);
            free(lists[s].paths);
        }
        free(lists);
        free(h_blob);
        return rc;
    }

    cudaStream_t stream;
    CUDA_OK(cudaStreamCreate(&stream));
    const size_t pts_floats = (size_t)S * 3 * d->n_stride;
    float *weights, *points, *T, *losses, *factor, *info;
    delora_odometry_residual_params rp;
    rp.lambda_po2pl = lambda_po2pl;
    rp.loss_flags = objective;
    if (pre && normalized) rp.loss_flags |= DELORA_TRAIN_NORMALIZATION_SCALING;
    rp.nb_h = 7; rp.nb_w = 11;
    rp.epsilon_range = 0.5f;
    rp.min_neighbors = 10;
    int32_t *count, *active, *valid;
    void* workspace;
    const int64_t ws_bytes = n_geom && information
                                 ? delora_odometry_streams_adapt_geometries_info_workspace_bytes(descs, n_sets)
                             : n_geom     ? delora_odometry_streams_adapt_geometries_workspace_bytes(descs, n_sets)
                             : adapt && information ? delora_odometry_streams_adapt_info_workspace_bytes(d)
                             : adapt      ? delora_odometry_streams_adapt_workspace_bytes(d)
                             : pre && information ? delora_odometry_streams_pre_info_workspace_bytes(d)
                             : pre        ? delora_odometry_streams_pre_workspace_bytes(d)
                             : information ? delora_odometry_streams_info_workspace_bytes(d)
                             : residual   ? delora_odometry_streams_residual_workspace_bytes(d)
                             : normalized ? delora_odometry_streams_normalized_workspace_bytes(d)
                                          : delora_odometry_streams_workspace_bytes(d);
    if (ws_bytes < 0) return fail(delora_last_error());
    CUDA_OK(cudaMalloc((void**)&weights, (size_t)n_weights * sizeof(float)));
    CUDA_OK(cudaMalloc(&workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc((void**)&points, pts_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&count, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&active, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&valid, (size_t)S * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&T, (size_t)S * 16 * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&losses, (size_t)S * DELORA_LOSS_ROW * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&factor, (size_t)S * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&info, (size_t)S * DELORA_INFO_ROW * sizeof(float)));
    CUDA_OK(cudaMemcpy(weights, h_blob, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
    /* --geometry: geometry g's scans and counts start at its first stream's row */
    const float* g_points[MAX_GEOMETRIES];
    const int32_t* g_count[MAX_GEOMETRIES];
    for (int g = 0; g < n_sets; ++g) {
        const int row = g == 0 ? 0 : S_dirs + g - 1;
        g_points[g] = points + (size_t)row * 3 * d->n_stride;
        g_count[g] = count + row;
    }
    if (n_geom) {
        DELORA_OK(delora_odometry_streams_adapt_geometries_init(descs, n_sets, weights, workspace, stream));
    } else if (adapt && information) {
        DELORA_OK(delora_odometry_streams_adapt_info_init(d, weights, workspace, stream));
    } else if (adapt) {
        DELORA_OK(delora_odometry_streams_adapt_init(d, weights, workspace, stream));
    } else {
        if (pre && information) DELORA_OK(delora_odometry_streams_pre_info_init(d, workspace, stream));
        else if (pre) DELORA_OK(delora_odometry_streams_pre_init(d, workspace, stream));
        else if (information) DELORA_OK(delora_odometry_streams_info_init(d, workspace, stream));
        else if (residual) DELORA_OK(delora_odometry_streams_residual_init(d, workspace, stream));
        else if (normalized) DELORA_OK(delora_odometry_streams_normalized_init(d, workspace, stream));
        else DELORA_OK(delora_odometry_streams_init(d, workspace, stream));
        DELORA_OK(delora_odometry_streams_load_weights(d, weights, workspace, stream));
    }

    float* h_points = (float*)malloc(pts_floats * sizeof(float));
    int32_t* h_count = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    int32_t* h_active = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    int32_t* h_valid = (int32_t*)malloc((size_t)S * sizeof(int32_t));
    float* h_T = (float*)malloc((size_t)S * 16 * sizeof(float));
    float* h_losses = (float*)calloc((size_t)S * DELORA_LOSS_ROW, sizeof(float));
    float* h_info = (float*)calloc((size_t)S * DELORA_INFO_ROW, sizeof(float));
    if (!h_points || !h_count || !h_active || !h_valid || !h_T || !h_losses || !h_info)
        return fail("out of host memory");
    for (int k = 0; k < ticks; ++k) {
        for (int s = 0; s < S; ++s) {
            h_active[s] = k < lists[s].n;
            h_count[s] = 0;
            if (!h_active[s]) continue;
            h_count[s] = read_scan(lists[s].paths[k], h_points + (size_t)s * 3 * d->n_stride, d->n_stride);
            if (h_count[s] < 0) return fail("cannot read a scan (missing, truncated or more points than n_stride)");
        }
        CUDA_OK(cudaMemcpyAsync(points, h_points, pts_floats * sizeof(float), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(count, h_count, (size_t)S * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
        CUDA_OK(cudaMemcpyAsync(active, h_active, (size_t)S * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
        if (adapt || pre || residual) {
            if (n_geom && information)
                DELORA_OK(delora_odometry_streams_push_adapt_geometries_info(descs, n_sets, &hp, 1, g_points, g_count,
                                                                             active, workspace, T, valid, losses, info,
                                                                             stream));
            else if (n_geom)
                DELORA_OK(delora_odometry_streams_push_adapt_geometries(descs, n_sets, &hp, 1, g_points, g_count, active,
                                                                        workspace, T, valid, losses, stream));
            else if (adapt && information)
                DELORA_OK(delora_odometry_streams_push_adapt_info(d, &hp, 1, points, count, active, workspace, T, valid,
                                                                  losses, info, stream));
            else if (adapt)
                DELORA_OK(delora_odometry_streams_push_adapt(d, &hp, 1, points, count, active, workspace, T, valid,
                                                             losses, stream));
            else if (pre && information)
                DELORA_OK(delora_odometry_streams_push_pre_info(d, &rp, points, count, active, workspace, T, valid,
                                                                losses, normalized ? factor : NULL, info, stream));
            else if (pre)
                DELORA_OK(delora_odometry_streams_push_pre(d, &rp, points, count, active, workspace, T, valid, losses,
                                                           normalized ? factor : NULL, stream));
            else if (information)
                DELORA_OK(delora_odometry_streams_push_info(d, &rp, points, count, active, workspace, T, valid, losses,
                                                            info, stream));
            else
                DELORA_OK(delora_odometry_streams_push_residual(d, &rp, points, count, active, workspace, T, valid,
                                                                losses, stream));
            if (information)
                CUDA_OK(cudaMemcpyAsync(h_info, info, (size_t)S * DELORA_INFO_ROW * sizeof(float),
                                        cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaMemcpyAsync(h_losses, losses, (size_t)S * DELORA_LOSS_ROW * sizeof(float), cudaMemcpyDeviceToHost,
                                    stream));
        } else if (normalized) {
            DELORA_OK(delora_odometry_streams_push_normalized(d, points, count, active, workspace, T, valid, factor,
                                                              stream));
        } else {
            DELORA_OK(delora_odometry_streams_push(d, points, count, active, workspace, T, valid, stream));
        }
        CUDA_OK(cudaMemcpyAsync(h_T, T, (size_t)S * 16 * sizeof(float), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaMemcpyAsync(h_valid, valid, (size_t)S * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        for (int s = 0; s < S; ++s) {
            if (!h_valid[s]) continue;
            printf("%d %d", s, k);
            for (int i = 0; i < 12; ++i) printf(" %.9g", h_T[(size_t)s * 16 + i]);
            if (adapt || pre || residual) {
                const float* l = h_losses + (size_t)s * DELORA_LOSS_ROW;
                printf(" %.9g %.9g %.0f", l[1], l[2], l[3]);
            }
            if (information) print_info(h_info + (size_t)s * DELORA_INFO_ROW);
            printf("\n");
        }
    }
    if (adapt) {            /* the adapted weights, behind the input file's header */
        DELORA_OK(delora_odometry_train_weights(d, workspace, weights, stream));
        CUDA_OK(cudaMemcpyAsync(h_blob, weights, (size_t)n_weights * sizeof(float), cudaMemcpyDeviceToHost, stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        FILE* o = fopen(adapt_out, "wb");
        if (!o) return fail("cannot open the --adapt-out file");
        const int ok = fwrite(&hdr, sizeof hdr, 1, o) == 1 &&
                       fwrite(h_blob, sizeof(float), (size_t)n_weights, o) == (size_t)n_weights;
        if (fclose(o) != 0 || !ok) return fail("cannot write the --adapt-out file");
    }
    for (int s = 0; s < S; ++s) {
        for (int i = 0; i < lists[s].n; ++i) free(lists[s].paths[i]);
        free(lists[s].paths);
    }
    free(lists);
    for (int g = 0; g < n_geom; ++g) free(geom_dirs[g]);
    free(h_info);
    free(h_losses);
    free(h_T);
    free(h_valid);
    free(h_active);
    free(h_count);
    free(h_points);
    free(h_blob);
    cudaFree(info);
    cudaFree(factor);
    cudaFree(losses);
    cudaFree(T);
    cudaFree(valid);
    cudaFree(active);
    cudaFree(count);
    cudaFree(points);
    cudaFree(workspace);
    cudaFree(weights);
    cudaStreamDestroy(stream);
    return 0;
}
