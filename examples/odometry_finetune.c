/*
 * Self-supervised fine-tuning from a C host: no Python, no torch.  Links libdelora_b200.so and cudart only.
 *
 *   odometry_finetune [--dropout-seed S] in.dlw out.dlw steps lr scan_000.bin scan_001.bin ...
 *
 * Reads the weights of in.dlw (written by bin/export_odometry_weights.py, layout: include/delora_b200.h) and a list of
 * consecutive KITTI velodyne .bin scans ([N, 4] float32 rows: x, y, z, reflectance), runs `steps` training steps on the
 * consecutive pairs (scan k, scan k+1), min(max_batch, pairs) pairs per step, cycling through the list, and writes the
 * updated weights to out.dlw (same header).  Prints the objective (mean over the step's pairs of
 * po2po + lambda * po2pl + pl2pl, before that step's update) once per step.  No ground truth is needed.
 * The objective is the one the header records (objective_flags and lambda_po2pl; zeros there: po2pl + pl2pl, lambda_po2pl
 * 1), printed once on stderr.  The normals the losses use are estimated at the resolution the header's w_pre names
 * (export with --preprocessing-normals for the reference's recipe; po2po_alone estimates none); the program says which
 * on stderr.
 * A model configured with use_dropout (model_flags has DELORA_MODEL_DROPOUT) trains with its dropouts
 * (DELORA_TRAIN_DROPOUT); the seed of the masks is --dropout-seed, else the DELORA_DROPOUT_SEED environment variable,
 * else 0.
 *
 * Build:  cc odometry_finetune.c -I include -I $CUDA_HOME/include -L delora_b200 -ldelora_b200 \
 *            -L $CUDA_HOME/lib64 -lcudart -Wl,-rpath,$PWD/delora_b200 -o odometry_finetune
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "delora_b200.h"

static int fail(const char* what) {
    fprintf(stderr, "odometry_finetune: %s\n", what);
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

int main(int argc, char** argv) {
    unsigned long long dropout_seed = 0;
    const char* seed_env = getenv("DELORA_DROPOUT_SEED");
    if (seed_env) dropout_seed = strtoull(seed_env, NULL, 0);
    if (argc > 2 && strcmp(argv[1], "--dropout-seed") == 0) {
        dropout_seed = strtoull(argv[2], NULL, 0);
        argc -= 2;
        argv += 2;
    }
    if (argc < 7)
        return fail("usage: odometry_finetune [--dropout-seed S] in.dlw out.dlw steps lr scan.bin scan.bin [scan.bin ...]");
    const int steps = atoi(argv[3]);
    const float lr = (float)atof(argv[4]);
    const int n_scans = argc - 5;
    char** scan_paths = argv + 5;

    FILE* f = fopen(argv[1], "rb");
    if (!f) return fail("cannot open the weight file");
    delora_odometry_file_header hdr;
    if (fread(&hdr, sizeof hdr, 1, f) != 1) return fail("truncated header");
    if (memcmp(hdr.magic, DELORA_ODOMETRY_FILE_MAGIC, 8) != 0) return fail("not a .dlw file");
    if (hdr.abi_version != delora_abi_version()) return fail("weight file and library ABI versions differ");
    const int normalized = (hdr.model_flags & DELORA_MODEL_NORMALIZATION_SCALING) != 0;
    if (normalized && hdr.desc.w_pre == 0)
        return fail("the model was trained with normalization_scaling, which trains on the reference's recipe only: "
                    "export it with preprocessing normals (w_pre > 0)");
    const delora_odometry_desc* d = &hdr.desc;
    const int64_t n_weights = delora_odometry_weight_floats(d);
    if (n_weights < 0) return fail(delora_last_error());
    if (n_weights != hdr.blob_floats) return fail("blob length does not match the descriptor");
    float* h_blob = (float*)malloc((size_t)n_weights * sizeof(float));
    if (!h_blob || fread(h_blob, sizeof(float), (size_t)n_weights, f) != (size_t)n_weights) return fail("truncated blob");
    fclose(f);

    /* all scans in host memory, [3, n_stride] each */
    const size_t scan_floats = (size_t)3 * d->n_stride;
    float* h_scans = (float*)malloc((size_t)n_scans * scan_floats * sizeof(float));
    int32_t* h_counts = (int32_t*)malloc((size_t)n_scans * sizeof(int32_t));
    if (!h_scans || !h_counts) return fail("out of host memory");
    for (int k = 0; k < n_scans; ++k)
        if ((h_counts[k] = read_scan(scan_paths[k], d->n_stride, h_scans + (size_t)k * scan_floats)) < 0)
            return fail("cannot read a scan (missing, truncated, or more points than n_stride)");
    const int n_pairs = n_scans - 1;
    const int B = n_pairs < d->max_batch ? n_pairs : d->max_batch;
    /* the header's w_pre chooses the objective: 0 = normals at the model's H x W, as the projection the model sees;
     * > 0 = the reference's recipe (normals at H x w_pre, the points then projected at H x W) */
    if (d->w_pre > 0)
        fprintf(stderr, "odometry_finetune: normals at the preprocessing resolution %dx%d, images at %dx%d\n", d->H,
                d->w_pre, d->H, d->W);
    else
        fprintf(stderr, "odometry_finetune: normals at the model resolution %dx%d\n", d->H, d->W);

    delora_odometry_train_params hp;
    hp.lr = lr; hp.beta1 = 0.9f; hp.beta2 = 0.999f; hp.eps = 1e-8f;
    uint32_t objective;                       /* the file's ICP objective (zeros in the header: the shipped one) */
    if (delora_odometry_file_objective(&hdr, &objective, &hp.lambda_po2pl)) return fail(delora_last_error());
    print_objective("odometry_finetune", objective, hp.lambda_po2pl);
    const int dropout = (hdr.model_flags & DELORA_MODEL_DROPOUT) != 0;
    hp.loss_flags = objective | (normalized ? DELORA_TRAIN_NORMALIZATION_SCALING : 0u) |
                    (dropout ? DELORA_TRAIN_DROPOUT : 0u);
    hp.nb_h = 7; hp.nb_w = 11;
    hp.epsilon_range = 0.5f;
    hp.min_neighbors = 10;

    cudaStream_t stream;
    CUDA_OK(cudaStreamCreate(&stream));
    float *weights, *points, *losses;
    int32_t* counts;
    void* workspace;
    const int64_t ws_bytes = delora_odometry_train_workspace_bytes(d);
    if (ws_bytes < 0) return fail(delora_last_error());
    CUDA_OK(cudaMalloc((void**)&weights, (size_t)n_weights * sizeof(float)));
    CUDA_OK(cudaMalloc(&workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc((void**)&points, (size_t)2 * B * scan_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&counts, (size_t)2 * B * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&losses, (size_t)B * DELORA_LOSS_ROW * sizeof(float)));
    CUDA_OK(cudaMemcpy(weights, h_blob, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
    DELORA_OK(delora_odometry_train_init(d, weights, workspace, stream));
    DELORA_OK(delora_odometry_train_set_dropout_seed(d, dropout_seed, workspace, stream));
    if (dropout) fprintf(stderr, "odometry_finetune: dropout on, seed %llu\n", dropout_seed);

    float* h_losses = (float*)malloc((size_t)B * DELORA_LOSS_ROW * sizeof(float));
    int32_t* h_step_counts = (int32_t*)malloc((size_t)2 * B * sizeof(int32_t));
    if (!h_losses || !h_step_counts) return fail("out of host memory");
    int next = 0;
    for (int s = 0; s < steps; ++s) {
        /* points of a step: scan_1 of pairs 0..B-1, then scan_2 of pairs 0..B-1 */
        for (int b = 0; b < B; ++b) {
            const int k = (next + b) % n_pairs;
            CUDA_OK(cudaMemcpyAsync(points + (size_t)b * scan_floats, h_scans + (size_t)k * scan_floats,
                                    scan_floats * sizeof(float), cudaMemcpyHostToDevice, stream));
            CUDA_OK(cudaMemcpyAsync(points + (size_t)(B + b) * scan_floats, h_scans + (size_t)(k + 1) * scan_floats,
                                    scan_floats * sizeof(float), cudaMemcpyHostToDevice, stream));
            h_step_counts[b] = h_counts[k];
            h_step_counts[B + b] = h_counts[k + 1];
        }
        next = (next + B) % n_pairs;
        CUDA_OK(cudaMemcpyAsync(counts, h_step_counts, (size_t)2 * B * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
        DELORA_OK(delora_odometry_train_step(d, &hp, points, counts, B, workspace, losses, NULL, NULL, NULL, stream));
        CUDA_OK(cudaMemcpyAsync(h_losses, losses, (size_t)B * DELORA_LOSS_ROW * sizeof(float), cudaMemcpyDeviceToHost,
                                stream));
        CUDA_OK(cudaStreamSynchronize(stream));
        double objective = 0.0;
        for (int b = 0; b < B; ++b) {
            const float* l = h_losses + (size_t)b * DELORA_LOSS_ROW;
            objective += (double)l[0] + (double)hp.lambda_po2pl * l[1] + (double)l[2];
        }
        printf("step %d objective %.9g\n", s, objective / B);
    }

    DELORA_OK(delora_odometry_train_weights(d, workspace, weights, stream));
    CUDA_OK(cudaMemcpyAsync(h_blob, weights, (size_t)n_weights * sizeof(float), cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    FILE* o = fopen(argv[2], "wb");
    if (!o) return fail("cannot create the output file");
    if (fwrite(&hdr, sizeof hdr, 1, o) != 1 || fwrite(h_blob, sizeof(float), (size_t)n_weights, o) != (size_t)n_weights)
        return fail("cannot write the output file");
    fclose(o);

    free(h_step_counts);
    free(h_losses);
    free(h_counts);
    free(h_scans);
    free(h_blob);
    cudaFree(losses);
    cudaFree(counts);
    cudaFree(points);
    cudaFree(workspace);
    cudaFree(weights);
    cudaStreamDestroy(stream);
    return 0;
}
