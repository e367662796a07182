// Inception-v3 for the Fréchet Inception Distance (pytorch-fid's InceptionV3(output_blocks=[3]), use_fid_inception=True;
// basicsr/archs/inception.py): the SIMT kernels around the conv engine.
//   input     fp32 NCHW RGB, or uint8 HWC BGR read as RGB v / 255 (ToTensor); bilinear to 299 x 299 with torch's CPU arithmetic
//             for align_corners=False (resize_input), then 2x - 1 (normalize_input); alone, or fused into the stem's load
//   stem      Conv2d_1a_3x3 (3x3 stride 2 valid, 3 -> 32) + folded BatchNorm + ReLU -> NHWC, channels [32, pitch) zero; an
//             image with a NaN among its stem outputs is flagged.  Torch carries that NaN through every later ReLU to all of
//             pool3, but the conv engine's ReLU epilogue (fmaxf) maps NaN to 0, so the flag carries it instead: the global
//             pool writes NaN features for a flagged image
//   pools     max 3x3 stride 2 valid and stride 1 pad 1 (NaN propagates as in torch's CPU max_pool2d), avg 3x3 stride 1 pad 1
//             with count_include_pad=False (the FID blocks' pool branches), the global average pool to the pool3 features
//   stats     float64 mean, then the centred Gram (X - mu)^T (X - mu) * (1 / (N - 1)) as np.cov computes it; every sum runs
//             over the images in order, so the statistics depend only on the feature matrix, not on how it was batched
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

// Source index and weights of output position d along one axis: torch's compute_source_index_and_lambda as its CPU kernel
// evaluates it (the source index scale * (d + 0.5) - 0.5 contracted to one fused multiply-add); equal sizes copy.
struct FidLin { int i0, i1; float l0, l1; };
__device__ __forceinline__ FidLin fid_lin(int d, int in, int out) {
  FidLin r;
  if (in == out) { r.i0 = r.i1 = d; r.l0 = 1.f; r.l1 = 0.f; return r; }
  const float scale = __fdiv_rn((float)in, (float)out);
  float src = __fmaf_rn(scale, __fadd_rn((float)d, 0.5f), -0.5f);
  if (src < 0.f) src = 0.f;
  int i = (int)floorf(src);
  if (i > in - 1) i = in - 1;
  const float lam = fminf(fmaxf(__fsub_rn(src, (float)i), 0.f), 1.f);
  r.i0 = i; r.i1 = i + (i < in - 1 ? 1 : 0); r.l1 = lam; r.l0 = __fsub_rn(1.f, lam);
  return r;
}

__device__ __forceinline__ float fid_src(const FidInput& in, int64_t n, int c, int y, int x) {
  if (in.u8) return __fdiv_rn((float)in.u8[((n * in.H + y) * in.W + x) * 3 + 2 - c], 255.f);   // BGR byte -> RGB, ToTensor
  return __ldg(in.f32 + ((n * 3 + c) * in.H + y) * in.W + x);
}

// One element of the network input: channel c at (oy, ox) of the 299 x 299 (resize) or H x W image.  The bilinear blend is
// torch's CPU form, a * w0 + b * w1 with one fused multiply-add, along W first and then along H.
__device__ __forceinline__ float fid_value(const FidInput& in, int64_t n, int c, int oy, int ox) {
  float v;
  if (in.resize) {
    const FidLin ly = fid_lin(oy, in.H, FID_SIZE), lx = fid_lin(ox, in.W, FID_SIZE);
    const float a = fid_src(in, n, c, ly.i0, lx.i0), b = fid_src(in, n, c, ly.i0, lx.i1);
    const float e = fid_src(in, n, c, ly.i1, lx.i0), f = fid_src(in, n, c, ly.i1, lx.i1);
    const float t0 = __fmaf_rn(a, lx.l0, __fmul_rn(b, lx.l1));
    const float t1 = __fmaf_rn(e, lx.l0, __fmul_rn(f, lx.l1));
    v = __fmaf_rn(t0, ly.l0, __fmul_rn(t1, ly.l1));
  } else {
    v = fid_src(in, n, c, oy, ox);
  }
  if (in.normalize) v = __fsub_rn(__fmul_rn(2.f, v), 1.f);              // 2 * x - 1
  return v;
}

__global__ void __launch_bounds__(256) fid_input_kernel(FidInput in, float* __restrict__ out, int OH, int OW) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t n = blockIdx.z;
  const int oy = blockIdx.y, ox = blockIdx.x * 256 + threadIdx.x;
  if (ox >= OW) return;
  for (int c = 0; c < 3; ++c) out[((n * 3 + c) * OH + oy) * OW + ox] = fid_value(in, n, c, oy, ox);
}

int fid_input(const FidInput& in, float* out, int N, cudaStream_t st) {
  if (N == 0) return 0;
  const int OH = in.resize ? FID_SIZE : in.H, OW = in.resize ? FID_SIZE : in.W;
  CFB_REQUIRE(N <= 65535 && OH <= 65535, "fid_input: at most 65535 images and rows per launch");
  CFB_LAUNCH_PDL(fid_input_kernel, dim3((unsigned)((OW + 255) / 256), (unsigned)OH, (unsigned)N), dim3(256), 0, st, in, out, OH, OW);
  return 0;
}

// ---- stem: one block = 64 output pixels of one row of one image, one thread = one pixel x 32 channels.  The network input of
// the 3 x 3 x 129 window is staged in shared memory; the 27 taps are summed in (ci, r, s) order with fmaf from 0 ----
__global__ void __launch_bounds__(64) fid_stem_kernel(FidInput in, const float* __restrict__ wt, const float* __restrict__ bias,
                                                      float* __restrict__ out, int* __restrict__ nan_flag, int pitch, int OH,
                                                      int OW, int Ho, int Wo) {
  __shared__ float sw[27 * 32];
  __shared__ float sb[32];
  __shared__ float patch[3][3][129];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) sw[i] = wt[(i & 31) * 27 + (i >> 5)];   // OIHW -> [ci,r,s][co]
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  pdl_launch_dependents();
  pdl_wait();
  const int64_t n = blockIdx.z;
  const int oy = blockIdx.y, x0 = blockIdx.x * 128;
  for (int i = threadIdx.x; i < 3 * 3 * 129; i += blockDim.x) {
    const int ci = i / 387, rem = i - ci * 387, r = rem / 129, px = rem - r * 129;
    const int iy = 2 * oy + r, ix = x0 + px;
    patch[ci][r][px] = ix < OW ? fid_value(in, n, ci, iy, ix) : 0.f;
  }
  __syncthreads();
  const int ox = blockIdx.x * 64 + threadIdx.x;
  if (ox >= Wo) return;
  float acc[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) acc[c] = 0.f;
  for (int ci = 0; ci < 3; ++ci)
    for (int r = 0; r < 3; ++r)
      for (int s = 0; s < 3; ++s) {
        const float v = patch[ci][r][2 * threadIdx.x + s];
        const float* wr = sw + ((ci * 3 + r) * 3 + s) * 32;
#pragma unroll
        for (int c = 0; c < 32; ++c) acc[c] = fmaf(v, wr[c], acc[c]);
      }
  bool nan = false;
#pragma unroll
  for (int c = 0; c < 32; ++c) nan |= acc[c] != acc[c];
  if (nan) nan_flag[n] = 1;
  float* o = out + ((n * Ho + oy) * Wo + ox) * pitch;
#pragma unroll
  for (int c = 0; c < 32; c += 4) {
    float4 v;
    v.x = acc[c] + sb[c]; v.y = acc[c + 1] + sb[c + 1]; v.z = acc[c + 2] + sb[c + 2]; v.w = acc[c + 3] + sb[c + 3];
    v.x = v.x < 0.f ? 0.f : v.x; v.y = v.y < 0.f ? 0.f : v.y; v.z = v.z < 0.f ? 0.f : v.z; v.w = v.w < 0.f ? 0.f : v.w;
    *reinterpret_cast<float4*>(o + c) = v;
  }
  for (int c = 32; c < pitch; c += 4) *reinterpret_cast<float4*>(o + c) = make_float4(0.f, 0.f, 0.f, 0.f);
}

int fid_stem(const FidInput& in, const float* wt, const float* bias, float* out, int* nan_flag, int pitch, int N, cudaStream_t st) {
  if (N == 0) return 0;
  const int OH = in.resize ? FID_SIZE : in.H, OW = in.resize ? FID_SIZE : in.W;
  CFB_REQUIRE(OH >= 3 && OW >= 3 && pitch >= 32 && pitch % 4 == 0, "fid_stem: bad size");
  const int Ho = (OH - 3) / 2 + 1, Wo = (OW - 3) / 2 + 1;
  CFB_REQUIRE(N <= 65535 && Ho <= 65535, "fid_stem: at most 65535 images and rows per launch");
  CFB_LAUNCH_PDL(fid_stem_kernel, dim3((unsigned)((Wo + 63) / 64), (unsigned)Ho, (unsigned)N), dim3(64), 0, st, in, wt, bias, out,
                 nan_flag, pitch, OH, OW, Ho, Wo);
  return 0;
}

// ---- pools over NHWC maps, one thread = one output pixel x 4 channels; windows are scanned row by row ----
__device__ __forceinline__ float fid_max(float m, float v) { return (v > m || v != v) ? v : m; }

__global__ void __launch_bounds__(256) fid_maxpool_kernel(const float* __restrict__ in, int in_pitch, float* __restrict__ out,
                                                          int out_pitch, int out_c0, int H, int W, int Ho, int Wo, int C4,
                                                          int stride, int pad, int64_t total) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C4) * 4;
  const int64_t pix = i / C4;
  const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho);
  const int64_t n = pix / ((int64_t)Wo * Ho);
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int r = 0; r < 3; ++r) {
    const int iy = oy * stride - pad + r;
    if ((unsigned)iy >= (unsigned)H) continue;
    for (int s = 0; s < 3; ++s) {
      const int ix = ox * stride - pad + s;
      if ((unsigned)ix >= (unsigned)W) continue;
      const float4 v = __ldg(reinterpret_cast<const float4*>(in + ((n * H + iy) * W + ix) * in_pitch + c));
      m.x = fid_max(m.x, v.x); m.y = fid_max(m.y, v.y); m.z = fid_max(m.z, v.z); m.w = fid_max(m.w, v.w);
    }
  }
  *reinterpret_cast<float4*>(out + pix * out_pitch + out_c0 + c) = m;
}

int fid_maxpool(const float* in, int in_pitch, float* out, int out_pitch, int out_c0, int N, int H, int W, int C, int stride,
                cudaStream_t st) {
  CFB_REQUIRE(stride == 1 || stride == 2, "fid_maxpool: 3x3 stride 2 valid or stride 1 pad 1");
  CFB_REQUIRE(C % 4 == 0 && in_pitch % 4 == 0 && out_pitch % 4 == 0 && out_c0 % 4 == 0 && C <= in_pitch && out_c0 + C <= out_pitch,
              "fid_maxpool: channel counts and offsets must be multiples of 4");
  const int pad = stride == 1 ? 1 : 0;
  CFB_REQUIRE(H + 2 * pad >= 3 && W + 2 * pad >= 3, "fid_maxpool: map smaller than the window");
  const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(fid_maxpool_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, in, in_pitch, out, out_pitch, out_c0, H,
                 W, Ho, Wo, C / 4, stride, pad, total);
  return 0;
}

// avg_pool2d(x, 3, 1, 1, count_include_pad=False): the window's values added in order from 0, divided by their count
__global__ void __launch_bounds__(256) fid_avgpool_kernel(const float* __restrict__ in, int in_pitch, float* __restrict__ out,
                                                          int out_pitch, int H, int W, int C4, int64_t total) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C4) * 4;
  const int64_t pix = i / C4;
  const int ox = (int)(pix % W), oy = (int)((pix / W) % H);
  const int64_t n = pix / ((int64_t)W * H);
  const int y0 = max(oy - 1, 0), y1 = min(oy + 2, H), x0 = max(ox - 1, 0), x1 = min(ox + 2, W);
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int iy = y0; iy < y1; ++iy)
    for (int ix = x0; ix < x1; ++ix) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(in + ((n * H + iy) * W + ix) * in_pitch + c));
      s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w);
    }
  const float cnt = (float)((y1 - y0) * (x1 - x0));
  *reinterpret_cast<float4*>(out + pix * out_pitch + c) =
      make_float4(__fdiv_rn(s.x, cnt), __fdiv_rn(s.y, cnt), __fdiv_rn(s.z, cnt), __fdiv_rn(s.w, cnt));
}

int fid_avgpool(const float* in, int in_pitch, float* out, int out_pitch, int N, int H, int W, int C, cudaStream_t st) {
  CFB_REQUIRE(C % 4 == 0 && in_pitch % 4 == 0 && out_pitch % 4 == 0 && C <= in_pitch && C <= out_pitch,
              "fid_avgpool: channel counts must be multiples of 4");
  const int64_t total = (int64_t)N * H * W * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(fid_avgpool_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, in, in_pitch, out, out_pitch, H, W,
                 C / 4, total);
  return 0;
}

// AdaptiveAvgPool2d(1): the H x W values of a channel added in order from 0, then / H / W (torch's CPU kernel); NaN for an
// image the stem flagged
__global__ void __launch_bounds__(256) fid_global_pool_kernel(const float* __restrict__ in, int pitch, const int* __restrict__ nan_flag,
                                                              float* __restrict__ out, int H, int W, int C4, int64_t total) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C4) * 4;
  const int64_t n = i / C4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = 0; p < H * W; ++p) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(in + (n * H * W + p) * pitch + c));
    s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w);
  }
  const float fh = (float)H, fw = (float)W;
  if (nan_flag && nan_flag[n]) s = make_float4(NAN, NAN, NAN, NAN);
  *reinterpret_cast<float4*>(out + n * C4 * 4 + c) =
      make_float4(__fdiv_rn(__fdiv_rn(s.x, fh), fw), __fdiv_rn(__fdiv_rn(s.y, fh), fw), __fdiv_rn(__fdiv_rn(s.z, fh), fw),
                  __fdiv_rn(__fdiv_rn(s.w, fh), fw));
}

int fid_global_pool(const float* in, int pitch, const int* nan_flag, float* out, int N, int H, int W, int C, cudaStream_t st) {
  CFB_REQUIRE(C % 4 == 0 && pitch % 4 == 0 && C <= pitch, "fid_global_pool: channel counts must be multiples of 4");
  const int64_t total = (int64_t)N * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(fid_global_pool_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, in, pitch, nan_flag, out, H, W, C / 4,
                 total);
  return 0;
}

// ---- statistics of a feature matrix X [N, D] (float32, row-major) ----
// mean: one thread per column, the N values added in row order in float64, / N (np.mean's pairwise order differs by a few ulp)
__global__ void __launch_bounds__(256) fid_mean_kernel(const float* __restrict__ x, int64_t N, int D, double* __restrict__ mu) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  double s = 0.0;
  for (int64_t i = 0; i < N; ++i) s += (double)__ldg(x + i * D + j);
  mu[j] = s / (double)N;
}

// centred Gram of one 64 x 64 tile pair (tj <= tk) of the upper triangle: 256 threads, 4 x 4 entries each; rows of X are taken
// 16 at a time into shared memory, centred in float64, and every entry adds its products in row order from 0.  The tile and its
// mirror are written, times 1 / (N - 1) (np.cov multiplies by the reciprocal)
constexpr int FID_GT = 64, FID_GK = 16;
__global__ void __launch_bounds__(256) fid_gram_kernel(const float* __restrict__ x, int64_t N, int D, const double* __restrict__ mu,
                                                       double* __restrict__ sigma, double inv) {
  __shared__ double sa[FID_GK][FID_GT], sb[FID_GK][FID_GT];
  // tile pair of this block: the b-th (tj, tk), tj <= tk, in row order
  const int T = D / FID_GT;
  int b = blockIdx.x, tj = 0;
  while (b >= T - tj) { b -= T - tj; ++tj; }
  const int tk = tj + b;
  const int j0 = tj * FID_GT, k0 = tk * FID_GT;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
  const int lr = threadIdx.x >> 4, lc = (threadIdx.x & 15) * 4;      // loader: row lr, columns lc..lc+3 of the 16 x 64 slab
  double mj[4], mk[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) { mj[q] = mu[j0 + lc + q]; mk[q] = mu[k0 + lc + q]; }
  for (int64_t i0 = 0; i0 < N; i0 += FID_GK) {
    const int64_t i = i0 + lr;
    if (i < N) {
      const float4 va = __ldg(reinterpret_cast<const float4*>(x + i * D + j0 + lc));
      const float4 vb = __ldg(reinterpret_cast<const float4*>(x + i * D + k0 + lc));
      sa[lr][lc] = (double)va.x - mj[0]; sa[lr][lc + 1] = (double)va.y - mj[1];
      sa[lr][lc + 2] = (double)va.z - mj[2]; sa[lr][lc + 3] = (double)va.w - mj[3];
      sb[lr][lc] = (double)vb.x - mk[0]; sb[lr][lc + 1] = (double)vb.y - mk[1];
      sb[lr][lc + 2] = (double)vb.z - mk[2]; sb[lr][lc + 3] = (double)vb.w - mk[3];
    }
    __syncthreads();
    const int rows = (int)min((int64_t)FID_GK, N - i0);
    for (int r = 0; r < rows; ++r) {
      double a[4], c[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = sa[r][ty + 16 * q]; c[q] = sb[r][tx + 16 * q]; }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = fma(a[p], c[q], acc[p][q]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + ty + 16 * p, k = k0 + tx + 16 * q;
      const double v = acc[p][q] * inv;
      sigma[(int64_t)j * D + k] = v;
      sigma[(int64_t)k * D + j] = v;
    }
}

int fid_stats(const float* x, int64_t N, int D, double* mu, double* sigma, cudaStream_t st) {
  CFB_REQUIRE(((uintptr_t)x & 15) == 0, "fid_stats: the features must be 16-byte aligned (rows are read as float4)");
  CFB_REQUIRE(N >= 2, "fid_stats: at least 2 feature vectors are needed for a covariance");
  CFB_REQUIRE(D >= FID_GT && D % FID_GT == 0, "fid_stats: the feature width must be a multiple of 64");
  fid_mean_kernel<<<(unsigned)((D + 255) / 256), 256, 0, st>>>(x, N, D, mu);
  CFB_LAUNCH_CHECK();
  const int T = D / FID_GT;
  fid_gram_kernel<<<(unsigned)(T * (T + 1) / 2), 256, 0, st>>>(x, N, D, mu, sigma, 1.0 / (double)(N - 1));
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace cfb
