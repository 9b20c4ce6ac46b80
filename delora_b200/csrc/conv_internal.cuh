// Library-internal functions the convolution sources call across files.  The C ABI is include/delora_b200.h.
#pragma once
#include "tc_common.cuh"

namespace delora {

// conv_rows.cu: row-block kernel (stride-1 fprop, phase-decomposed dgrad)
bool conv_rows_eligible(int Cin, int Cout, int ksize, int Wg);
int conv_rows_launch(const void* x, const void* w, const void* residual, const void* saved, void* y, int B, int Hout,
                     int Wout, int Cin, int Cout, int ksize, int up_h, int up_w, int act, cudaStream_t stream,
                     int residual_on_grid);

// conv_wgrad.cu: second-generation weight gradient, for the 3x3 layers and the stem
bool wgrad2_eligible(int Cin, int Cout, int ksize, int stride_h, int stride_w);
int64_t wgrad2_scratch_floats(int B, int Hout, int Wout, int Cin, int Cout, int sw);
int wgrad2_launch(const void* x, const void* dz, float* dw, float* scratch, int B, int Hin, int Win, int Cin, int Cin_true,
                  int Cout, int stride_h, int stride_w, cudaStream_t st);
int64_t wgrad2_stem_scratch_floats(int B, int H, int Wout);
int wgrad2_launch_stem(const CUtensorMap& map_x, const void* dz, float* dw, float* scratch, int B, int H, int Wout,
                       int Cin_true, cudaStream_t st);

}  // namespace delora
