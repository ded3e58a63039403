// wgmma implicit-GEMM kernels of the voxel decoder and the occupancy / flow heads (conv3d_tc.cu, head_tc.cu)
#pragma once
#include "common.cuh"
#include "kernels.cuh"

namespace occ {

// in/out channels-last bf16 [X][Y][Z=16][C]; w_tap_major bf16 [27][32 (cout)][Cin] with BatchNorm folded in
// (tap = (dz*3+dy)*3+dx); bias fp32 [32] (folded BN shift); out = relu(conv + bias)
int launch_conv3d_tc(const bf16* in, const bf16* w_tap_major, const float* bias, int X, int Y, int Z, int Cin,
                     bf16* out, cudaStream_t stream);

// fp32 storage on the tensor cores: split = [hi | lo] bf16 halves of the fp32 input ([nvox][2*Cin]); w_hi / w_lo the bf16 split of
// the folded weights; out_f32 [nvox][32] = relu(hi.W_hi + lo.W_hi + hi.W_lo + bias), three passes accumulated in fp32
int launch_conv3d_tc_split(const bf16* split, const bf16* w_hi, const bf16* w_lo, const float* bias, int X, int Y, int Z, int Cin,
                           float* out_f32, cudaStream_t stream);

// vox bf16 [nvox][32]; w1cat bf16 [128][32] = [predicter.0 ; flow_predicter.0]; w2cat bf16 [32][128] block-diagonal
// [predicter.2 | 0 ; 0 | flow_predicter.2 ; 0]; b1cat f32 [128]; b2cat f32 [ncls + 2]
int launch_occ_head_tc(const bf16* vox, const bf16* w1cat, const bf16* w2cat, const float* b1cat, const float* b2cat,
                       int ncls, int64_t nvox, float* occ_logits, float* flow, uint8_t* cls_u8, int64_t* cls_i64,
                       cudaStream_t stream);

}  // namespace occ
