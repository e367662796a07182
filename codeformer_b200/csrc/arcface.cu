// ResNetArcFace (identity embeddings of restored faces): the SIMT kernels around the conv engine.
//   stem     conv1 (3x3 p1, 1 -> 64) + folded bn1 + PReLU + MaxPool2d(2) at 128 x 128 -> NHWC [N,64,64,64]
//            (basicsr/archs/arcface_arch.py:230-233); input fp32 [N,1,128,128], or uint8 HWC BGR 512 x 512 faces with the
//            caller's normalisation and gray_resize_for_identity fused (basicsr/models/codeformer_model.py:131-135)
//   bn0      the per-(image, channel) scale / shift tables the fused operand transform reads for every IRBlock's bn0
//   fold_fc  bn4 -> view(B,-1) on NCHW -> fc5 -> bn5 (arcface_arch.py:239-243) as one linear on the NHWC flatten (prepare)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

// One gray pixel of the 128 x 128 identity input from a uint8 HWC BGR 512 x 512 face, in the arithmetic of the device chain
//   x = normalize(img2tensor(face / 255.), 0.5, 0.5)            (u8_to_model_input; RGB order)
//   g = 0.2989 * x[0] + 0.5870 * x[1] + 0.1140 * x[2]           (torch: three fp32 products, two fp32 adds, left to right)
//   F.interpolate(g, (128, 128), 'bilinear', align_corners=False)
// The 4x downscale samples source rows 4y+1 and 4y+2 (and columns likewise) with all four lambdas 0.5: every product by 0.5
// is exact, so the torch expression h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d) rounds the same with or without FMA
// contraction, to rn(0.5 * rn(0.5a + 0.5b) + 0.5 * rn(0.5c + 0.5d)).
__device__ __forceinline__ float arc_gray512(const unsigned char* __restrict__ face, int sy, int sx) {
  const unsigned char* p = face + ((int64_t)sy * 512 + sx) * 3;
  const float r = u8_to_model_input(p[2]), g = u8_to_model_input(p[1]), b = u8_to_model_input(p[0]);
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.5870f, g)), __fmul_rn(0.1140f, b));
}
__device__ __forceinline__ float arc_gray_resized(const unsigned char* __restrict__ face, int y, int x) {
  const int sy = 4 * y + 1, sx = 4 * x + 1;
  const float a = arc_gray512(face, sy, sx), b = arc_gray512(face, sy, sx + 1);
  const float c = arc_gray512(face, sy + 1, sx), d = arc_gray512(face, sy + 1, sx + 1);
  const float top = __fadd_rn(__fmul_rn(0.5f, a), __fmul_rn(0.5f, b));
  const float bot = __fadd_rn(__fmul_rn(0.5f, c), __fmul_rn(0.5f, d));
  return __fadd_rn(__fmul_rn(0.5f, top), __fmul_rn(0.5f, bot));
}

// ---- stem: one block = 8 x 8 pooled outputs (16 x 16 conv outputs, an 18 x 18 gray patch) of one image; thread = one pooled
// pixel x 16 channels.  The conv sums its 9 taps in (r, s) order with fmaf from 0 in both variants, so forward_u8 equals
// forward on the gray image bit for bit. ----
template <bool U8>
__global__ void __launch_bounds__(256) arc_stem_kernel(const float* __restrict__ x, const unsigned char* __restrict__ faces,
                                                       const float* __restrict__ wt, const float* __restrict__ bias, float slope,
                                                       float* __restrict__ out) {
  __shared__ float patch[18][19];
  __shared__ float sw[9][64];
  __shared__ float sb[64];
  const int n = blockIdx.z, y0 = blockIdx.y * 16 - 1, x0 = blockIdx.x * 16 - 1;
  for (int i = threadIdx.x; i < 9 * 64; i += 256) sw[i % 9][i / 9] = wt[i];        // folded OIHW [64][1][3][3] -> [tap][co]
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  pdl_launch_dependents();
  pdl_wait();
  for (int i = threadIdx.x; i < 18 * 18; i += 256) {
    const int py = i / 18, px = i - py * 18, gy = y0 + py, gx = x0 + px;
    float v = 0.f;                                                                 // zero padding of conv1
    if ((unsigned)gy < 128u && (unsigned)gx < 128u) {
      if constexpr (U8) v = arc_gray_resized(faces + (int64_t)n * 512 * 512 * 3, gy, gx);
      else v = __ldg(x + ((int64_t)n * 128 + gy) * 128 + gx);
    }
    patch[py][px] = v;
  }
  __syncthreads();
  const int pp = threadIdx.x & 63, c0 = (threadIdx.x >> 6) * 16;
  const int qy = pp >> 3, qx = pp & 7;
  float m[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) m[c] = -INFINITY;
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const int cy = 2 * qy + (d >> 1), cx = 2 * qx + (d & 1);                       // conv output inside the 16 x 16 block
    float g[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) g[t] = patch[cy + t / 3][cx + t % 3];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float acc = 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) acc = fmaf(g[t], sw[t][c0 + c], acc);
      float v = acc + sb[c0 + c];
      v = v > 0.f ? v : slope * v;
      m[c] = fmaxf(m[c], v);
    }
  }
  const int oy = blockIdx.y * 8 + qy, ox = blockIdx.x * 8 + qx;
  float* o = out + (((int64_t)n * 64 + oy) * 64 + ox) * 64 + c0;
#pragma unroll
  for (int c = 0; c < 16; c += 4) *reinterpret_cast<float4*>(o + c) = make_float4(m[c], m[c + 1], m[c + 2], m[c + 3]);
}

int arc_stem(const float* x, const unsigned char* faces_bgr_hwc, const float* wt, const float* bias, float slope, float* out, int N,
             cudaStream_t st) {
  if (N == 0) return 0;
  const dim3 grid(8, 8, (unsigned)N);
  if (faces_bgr_hwc) CFB_LAUNCH_PDL(arc_stem_kernel<true>, grid, dim3(256), 0, st, x, faces_bgr_hwc, wt, bias, slope, out);
  else CFB_LAUNCH_PDL(arc_stem_kernel<false>, grid, dim3(256), 0, st, x, faces_bgr_hwc, wt, bias, slope, out);
  return 0;
}

// ---- bn0 tables: block b's [N][C_b] scale / shift at N * off[b] of the destinations, from the prepared per-channel values
// at off[b] of the sources ----
__global__ void arc_bn0_kernel(const float* __restrict__ scale, const float* __restrict__ shift, ArcBn0Table t, int N,
                               float* __restrict__ dscale, float* __restrict__ dshift) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * t.off[t.blocks];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int b = 0;
    while ((int64_t)N * t.off[b + 1] <= i) ++b;
    const int C = t.off[b + 1] - t.off[b];
    const int c = (int)((i - (int64_t)N * t.off[b]) % C);
    dscale[i] = scale[t.off[b] + c];
    dshift[i] = shift[t.off[b] + c];
  }
}

int arc_bn0_tables(const float* scale, const float* shift, const ArcBn0Table& t, int N, float* dscale, float* dshift,
                   cudaStream_t st) {
  const int64_t total = (int64_t)N * t.off[t.blocks];
  if (total == 0) return 0;
  const int64_t blocks = (total + 255) / 256;
  CFB_LAUNCH_PDL(arc_bn0_kernel, dim3((unsigned)(blocks > 148 * 8 ? 148 * 8 : blocks)), dim3(256), 0, st, scale, shift, t, N, dscale,
                 dshift);
  return 0;
}

// ---- eval-mode BatchNorm as a per-channel affine: scale = gamma / sqrt(var + eps), shift = beta - mean * scale ----
__global__ void arc_bn_affine_kernel(const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ m,
                                     const float* __restrict__ v, float eps, float* __restrict__ scale, float* __restrict__ shift,
                                     int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s = g[c] / sqrtf(v[c] + eps);
  scale[c] = s;
  shift[c] = b[c] - m[c] * s;
}

int arc_bn_affine(const float* g, const float* b, const float* m, const float* v, float eps, float* scale, float* shift, int C,
                  cudaStream_t st) {
  arc_bn_affine_kernel<<<(C + 255) / 256, 256, 0, st>>>(g, b, m, v, eps, scale, shift, C);
  CFB_LAUNCH_CHECK();
  return 0;
}

// ---- bn4 -> flatten (NCHW order, index c * HW + hw) -> fc5 -> bn5 as one linear on the NHWC flatten (index hw * C + c):
//   wout[o][hw * C + c] = s5[o] * (w[o][c * HW + hw] * s4[c])
//   bout[o] = s5[o] * (sum_j w[o][j] * t4[c(j)] + fc_b[o]) + (b5[o] - m5[o] * s5[o])      (the sum in float64)
// bn4 / bn5 arrive as per-channel (scale, shift) from arc_bn_affine.  One block per output row. ----
__global__ void __launch_bounds__(256) arc_fold_fc_kernel(const float* __restrict__ w, const float* __restrict__ fc_b,
                                                          const float* __restrict__ s4, const float* __restrict__ t4,
                                                          const float* __restrict__ s5, const float* __restrict__ t5, int C, int HW,
                                                          float* __restrict__ wout, float* __restrict__ bout) {
  __shared__ double red[256];
  const int o = blockIdx.x;
  const int K = C * HW;
  const float* wr = w + (int64_t)o * K;
  float* dr = wout + (int64_t)o * K;
  const float so = s5[o];
  double acc = 0.0;
  for (int j = threadIdx.x; j < K; j += 256) {
    const int c = j / HW, hw = j - c * HW;
    dr[(int64_t)hw * C + c] = so * (wr[j] * s4[c]);
    acc += (double)wr[j] * (double)t4[c];
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) bout[o] = so * (float)(red[0] + (double)fc_b[o]) + t5[o];
}

int arc_fold_fc(const float* w, const float* fc_b, const float* s4, const float* t4, const float* s5, const float* t5, int Cout, int C,
                int HW, float* wout, float* bout, cudaStream_t st) {
  arc_fold_fc_kernel<<<Cout, 256, 0, st>>>(w, fc_b, s4, t4, s5, t5, C, HW, wout, bout);
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace cfb
