/*
 * Odometry from a C host: no Python, no torch.  Links libdelora_b200.so and cudart only.
 *
 *   odometry_stream model.dlw scan_000.bin scan_001.bin ...
 *
 * model.dlw is written by bin/export_odometry_weights.py (layout: include/delora_b200.h); the scans are KITTI
 * velodyne .bin files ([N, 4] float32 rows: x, y, z, reflectance).  For every scan after the first it prints the
 * relative transform T_{k-1,k} as one line of 12 floats (the top three rows of the 4x4, row-major).
 * A model trained with normalization_scaling (model_flags has DELORA_MODEL_NORMALIZATION_SCALING) runs through
 * delora_odometry_pairs_normalized with B = 1 on (previous scan, this scan): the previous scan, not its image, is kept.
 *
 * Build:  cc odometry_stream.c -I include -I $CUDA_HOME/include -L delora_b200 -ldelora_b200 \
 *            -L $CUDA_HOME/lib64 -lcudart -Wl,-rpath,$PWD/delora_b200 -o odometry_stream
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "delora_b200.h"

static int fail(const char* what) {
    fprintf(stderr, "odometry_stream: %s\n", what);
    return 1;
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

int main(int argc, char** argv) {
    if (argc < 3) return fail("usage: odometry_stream model.dlw scan.bin [scan.bin ...]");

    /* weight file: fixed header, then the fp32 blob */
    FILE* f = fopen(argv[1], "rb");
    if (!f) return fail("cannot open the weight file");
    delora_odometry_file_header hdr;
    if (fread(&hdr, sizeof hdr, 1, f) != 1) return fail("truncated header");
    if (memcmp(hdr.magic, DELORA_ODOMETRY_FILE_MAGIC, 8) != 0) return fail("not a .dlw file");
    if (hdr.abi_version != delora_abi_version()) return fail("weight file and library ABI versions differ");
    const delora_odometry_desc* d = &hdr.desc;
    const int normalized = (hdr.model_flags & DELORA_MODEL_NORMALIZATION_SCALING) != 0;
    const int rows_dev = normalized ? 2 : 1;         /* normalised: [previous scan, this scan] */
    const size_t scan_floats = (size_t)3 * d->n_stride;
    const int64_t n_weights = delora_odometry_weight_floats(d);
    if (n_weights < 0) return fail(delora_last_error());
    if (n_weights != hdr.blob_floats) return fail("blob length does not match the descriptor");
    float* h_blob = (float*)malloc((size_t)n_weights * sizeof(float));
    if (!h_blob || fread(h_blob, sizeof(float), (size_t)n_weights, f) != (size_t)n_weights) return fail("truncated blob");
    fclose(f);

    cudaStream_t stream;
    CUDA_OK(cudaStreamCreate(&stream));
    float *weights, *points, *T, *factor;
    int32_t* count;
    void* workspace;
    const int64_t ws_bytes = delora_odometry_workspace_bytes(d);
    CUDA_OK(cudaMalloc((void**)&weights, (size_t)n_weights * sizeof(float)));
    CUDA_OK(cudaMalloc(&workspace, (size_t)ws_bytes));
    CUDA_OK(cudaMalloc((void**)&points, rows_dev * scan_floats * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&count, rows_dev * sizeof(int32_t)));
    CUDA_OK(cudaMalloc((void**)&T, 16 * sizeof(float)));
    CUDA_OK(cudaMalloc((void**)&factor, sizeof(float)));
    CUDA_OK(cudaMemcpy(weights, h_blob, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice));
    DELORA_OK(delora_odometry_init(d, workspace, stream));
    DELORA_OK(delora_odometry_load_weights(d, weights, workspace, stream));

    float* h_points = (float*)malloc((size_t)3 * d->n_stride * sizeof(float));
    if (!h_points) return fail("out of host memory");
    for (int k = 2; k < argc; ++k) {
        FILE* s = fopen(argv[k], "rb");
        if (!s) return fail("cannot open a scan");
        fseek(s, 0, SEEK_END);
        const long bytes = ftell(s);
        fseek(s, 0, SEEK_SET);
        const int32_t n = (int32_t)(bytes / (4 * sizeof(float)));
        if (n > d->n_stride) return fail("scan has more points than n_stride");
        float* rows = (float*)malloc((size_t)n * 4 * sizeof(float) + 1);
        if (!rows || fread(rows, 4 * sizeof(float), (size_t)n, s) != (size_t)n) return fail("truncated scan");
        fclose(s);
        /* [N, 4] rows -> [1, 3, n_stride] channels-first (x, y, z; reflectance is not used by the model) */
        memset(h_points, 0, (size_t)3 * d->n_stride * sizeof(float));
        for (int32_t i = 0; i < n; ++i)
            for (int c = 0; c < 3; ++c) h_points[(size_t)c * d->n_stride + i] = rows[(size_t)i * 4 + c];
        free(rows);
        const int slot = (normalized && k > 2) ? 1 : 0;
        CUDA_OK(cudaMemcpyAsync(points + slot * scan_floats, h_points, scan_floats * sizeof(float), cudaMemcpyHostToDevice,
                                stream));
        CUDA_OK(cudaMemcpyAsync(count + slot, &n, sizeof(int32_t), cudaMemcpyHostToDevice, stream));
        if (!normalized) {
            DELORA_OK(delora_odometry_push(d, points, count, workspace, k == 2 ? NULL : T, stream));
        } else if (k > 2) {
            DELORA_OK(delora_odometry_pairs_normalized(d, points, count, 1, workspace, T, NULL, factor, stream));
            /* this scan becomes the previous one */
            CUDA_OK(cudaMemcpyAsync(points, points + scan_floats, scan_floats * sizeof(float), cudaMemcpyDeviceToDevice,
                                    stream));
            CUDA_OK(cudaMemcpyAsync(count, count + 1, sizeof(int32_t), cudaMemcpyDeviceToDevice, stream));
        }
        if (k > 2) {
            float h_T[16];
            CUDA_OK(cudaMemcpyAsync(h_T, T, sizeof h_T, cudaMemcpyDeviceToHost, stream));
            CUDA_OK(cudaStreamSynchronize(stream));
            for (int i = 0; i < 12; ++i) printf(i ? " %.9g" : "%.9g", h_T[i]);
            printf("\n");
        } else {
            CUDA_OK(cudaStreamSynchronize(stream));
        }
    }
    free(h_points);
    free(h_blob);
    cudaFree(factor);
    cudaFree(T);
    cudaFree(count);
    cudaFree(points);
    cudaFree(workspace);
    cudaFree(weights);
    cudaStreamDestroy(stream);
    return 0;
}
