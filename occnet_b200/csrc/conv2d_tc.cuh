// Implicit-GEMM stride-1 2-D convolution on wgmma (conv2d_tc.cu): NHWC bf16, weights tap-major [Cout][KH*KW*Cin].
#pragma once
#include "common.cuh"

namespace occ {

bool conv2d_tc_supported(int Cin, int Cout, int KH, int KW);

// out = act(conv(in, w) + bias (+ residual)); in [N,H,W,Cin], out / residual [N,H,W,Cout], stride 1, symmetric `pad`
// with H_out = H, W_out = W (pad = KH / 2).  act: ACT_NONE / ACT_RELU (applied after the residual add).
int conv2d_tc(const bf16* in, const bf16* w_tap_major, const float* bias, const bf16* residual, bf16* out, int N, int H,
              int W, int Cin, int Cout, int KH, int KW, int pad, int act, cudaStream_t stream);

}  // namespace occ
