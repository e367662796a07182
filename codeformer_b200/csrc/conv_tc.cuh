// wgmma (Hopper tensor core) implicit-GEMM convolution engine: interface.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace cfb {
constexpr int TC_TILE_N = 64;                 // output channels of one n-tile of the engine (GEMM N per CTA)
// OIHW fp32 -> [taps][Cout][Cin] fp16 hi / lo of w*2^k (hi = fp16(.), lo = fp16(. - hi)); scale_slot = 2 device floats,
// [1] receives 2^-k for the epilogue
int tc_split_weights(const float* oihw, __half* hi, __half* lo, int Cout, int Cin, int k, float* scale_slot, cudaStream_t st);
// the same for a kh x kw window: OIHW fp32 -> [taps = kh * kw][Cout][Cin], taps in row-major (r, s) order
int tc_split_weights_taps(const float* oihw, __half* hi, __half* lo, int Cout, int Cin, int taps, float* scale_slot, cudaStream_t st);
// Upsample convs: pre-summed 2x2 parity weights [16][Cout][Cin] (hi/lo) -- pass these as wgt_hi/wgt_lo/wscale_inv with mode CONV_UP
int tc_split_weights_up4(const float* oihw3x3, __half* hi, __half* lo, int Cout, int Cin, float* scale_slot, cudaStream_t st);
bool tc_supported(const ConvArgs& a);
// the image is an exact grid of tiles (no ragged last tile row / column): where the automatic engine choice (engine 0, the
// VectorQuantizer) takes the tensor-core engine; ragged grids run there only when the tensor-core engine is asked for
bool tc_tiles_exact(const ConvArgs& a);
bool tc_can_xform(const ConvArgs& a);
size_t tc_scratch_bytes(const ConvArgs& a);   // operand (hi/lo fp16 activation planes) staging
bool tc_can_emit_stats(const ConvArgs& a);    // GroupNorm(32) partial sums available from the epilogue for this shape
int tc_tiles_per_image(const ConvArgs& a);    // 128-pixel tiles per image (GroupNorm partial slots = 4x this)
int conv_tc(const ConvArgs& a, void* scratch, int sm_count, cudaStream_t st);
// channel-major 128 x 64 tile (the MMAs compute the tile transposed, weights as the A operand): the tile kind tc_tile_n()
// reports for it, distinct from the 64 of the pixel-major 128 x 64 tile
constexpr int TC_TILE_CM = -64;
int tc_tile_n(const ConvArgs& a);             // tile conv_tc() uses for this conv: 128, 64 or TC_TILE_CM (64 channels)
// batched GEMM over 16x16-token images on fp16 hi/lo operand planes (attention cores); see conv_tc.cu
struct BmmArgs {
  const void* a_planes = nullptr; int a_pitch = 0, a_c0 = 0;   // A: [N][256][a_pitch] hi | lo
  const void* b_planes = nullptr; int b_pitch = 0, b_c0 = 0, b_rows = 0;   // B: [N][b_rows][b_pitch] hi | lo
  int N = 0, K = 0, Cout = 0;          // Cout: output columns of ONE (image, head) GEMM
  // multi-head attention (codeformer_arch.py:126): one GEMM per (image, head); head h reads channels +h*a_c_head / +h*b_c_head
  // of the A / B planes (scores) or rows +h*b_r_head of B (V^T); A may hold one image per (n, h) (the probabilities)
  int heads = 1, a_c_head = 0, b_c_head = 0, b_r_head = 0;
  bool a_img_per_head = false;
  bool out_per_head = true;            // out = [N*heads][256][Cout]; false: out = [N][256][heads*o_c_head], head h -> its column slice
  int o_c_head = 0;
  const float* scale_dev = nullptr;   // device scalar multiplied into the result
  float* out = nullptr;               // [N][256][Cout] fp32
  void* out_planes = nullptr;         // optional hi | lo planes of out
};
int bmm_tc(const BmmArgs& g, int sm_count, cudaStream_t st);
int concat_planes(const float* a, const float* b, void* planes, int64_t pixels, int Ca, int Cb, cudaStream_t st);
int softmax256_planes(const float* scores, void* planes, int64_t rows, cudaStream_t st);
int transpose_planes(const void* in_planes, int N, int pitch, int c0, int C, void* out_planes, cudaStream_t st);
// VectorQuantizer.forward as one kernel on NCHW tensors (see conv_tc.cu); hist / ticket: zero on entry, left zero
bool vq_fused_supported(int N, int D, int HW, int K);
int vq_fused(const float* z, const float* codebook, const void* whi, const void* wlo, const float* wscale_inv, const float* e2,
             unsigned* hist, unsigned* ticket, double* part, int N, int D, int HW, int K, float beta, float* zq, int64_t* idx,
             float* stats, cudaStream_t st);
}  // namespace cfb
