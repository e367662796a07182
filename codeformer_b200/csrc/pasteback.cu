// Whole-image paste-back on the GPU: the face crop warp and FaceRestoreHelper.paste_faces_to_input_image
// (/root/reference/facelib/utils/face_restoration_helper.py:319-349, 372-516) with cv2's arithmetic.
//
//   warpAffine    M is inverted in double; destination pixels map to the source in 1/32 fixed point (AB_BITS 10,
//                 INTER_BITS 5).  u8: 15-bit integer weights (32-fy)(32-fx)*32 ..., (sum + 2^14) >> 15.  f32 / f64:
//                 the same weights as exact dyadic floats, ((v0 w0 + v1 w1) + v2 w2) + v3 w3.  The parse mask's flags=3
//                 is INTER_AREA, which warpAffine runs as INTER_LINEAR.
//   resize        INTER_LINEAR, 11-bit weights (horizontal clamped, vertical not); an exact halving is the 2x2 mean.
//                 float64 (the parse mask): double coordinates fma(d + 0.5, ssize / dsize, -0.5) and lerp FMAs.
//   erode         rectangular k x k, anchor k/2, pixels outside the image never erode, k == 0 means 3x3.
//   GaussianBlur  separable, BORDER_REFLECT_101, cv2 4.13's x86-64 AVX2 arithmetic: which outputs take fused multiply-adds
//                 depends on the SIMD block of their column (k_blur_roi, k_blur_f64).  The float kernel is
//                 cv2.getGaussianKernel; the parse mask's float64 kernel is cv2's own table (kParseKernelHalf).
//
// Every per-face step works on the face's ROI: the bounding box of the face square grown by 2 source pixels, mapped
// to the canvas, grown by 2 pixels and clipped.  Outside it every warp of the face is exactly 0, so the soft mask is 0
// and the blend m*a + (1-m)*b returns b unchanged: restricting to the ROI is exact.  Values outside the ROI but inside
// the canvas are 0, so erosion ignores them (a 0 inside the window already gives the minimum) and the blur reads them as
// 0; at the canvas border both follow cv2 (no erosion, reflect-101).
//
// The steps that do not depend on the blend order run for all faces at once (blockIdx.z = face).  The areas of the first
// erosion are read back once per call (they fix the kernel sizes); then one composite launch per face, in face order.
// cfb_paste_faces_multi runs the same launch sequence over the faces of several equal-size canvases in one call.
//
//   INTER_AREA    (shrinking, cfb_resize_area_u8) integer factors: window sums, a 2 x 2 halving (s + 2) >> 2, otherwise
//                 cvRound(s * (1.f / area)); other factors: computeResizeAreaTab weights in double stored as float, a float
//                 row sum per source row and a float sum of the rows, both in cv2's tap order, then cvRound and clamp.
//   LANCZOS4      (cfb_resize_lanczos4_u8) cv2's fixed point: eight int16 taps per axis (float weights * 2048, not
//                 renormalised), clamped source coordinates, an int32 horizontal pass and a vertical pass (v + 2^21) >> 22.
//   gray images   add_restored_face's adain_npy(bgr2gray(restored), cropped) in float64 (cfb_gray_adain_faces) and the paste
//                 of float64 faces (cfb_paste_faces_f64): warpAffine on CV_64F blends with the float32 weight table in
//                 double, and the canvas is float64 from the first face on.
// Arithmetic that cv2 does unfused is written with _rn intrinsics so nvcc cannot contract it into FMAs; where cv2 fuses,
// the kernels call __fmaf_rn / __fma_rn.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/cfb200.h"
#include "kernels.cuh"

namespace cfb {
namespace {

constexpr int kParse = 512;           // the parsing network's resolution
constexpr int kParseK = 101;          // GaussianBlur(parse_mask, (101, 101), 11), applied twice
constexpr int kRoiPad = 2;
static_assert(kParse % 8 == 0, "k_blur_f64 assumes no SIMD tail columns in cv2's filter");

// cv2.getGaussianKernel(101, 11, CV_64F), taps 0 .. 50 (the rest mirror them).  cv2 exponentiates in its software double,
// whose last bit std::exp does not always reproduce, so the parse mask's kernel is cv2's own values.
constexpr double kParseKernelHalf[kParseK / 2 + 1] = {
  0x1.3d9320997c25bp-20, 0x1.de17a7bf38417p-20, 0x1.64e8ed67fb58cp-19, 0x1.08402ac73792fp-18, 0x1.8412e6ca94be9p-18,
  0x1.1a9d258b611acp-17, 0x1.983ce6e2d8b48p-17, 0x1.246cb61c4022cp-16, 0x1.9f7c2e4f210b2p-16, 0x1.24bcaeb80f233p-15,
  0x1.991c4ec5d6f8ep-15, 0x1.1b85423e811abp-14, 0x1.85bc1908d022ep-14, 0x1.09aa455fcb2a8p-13, 0x1.673421a12de51p-13,
  0x1.e1add23bf2656p-13, 0x1.404c85f10d7b6p-12, 0x1.a677dc2924522p-12, 0x1.1452178d2dfc5p-11, 0x1.667cb15ebc175p-11,
  0x1.cd4230959cfabp-11, 0x1.264dd24853bf3p-10, 0x1.7477bd22f281bp-10, 0x1.d382d89d4adafp-10, 0x1.22fd1739f5a24p-9,
  0x1.6740df70cfe47p-9, 0x1.b7e1e31cfeb7cp-9, 0x1.0b165029af448p-8, 0x1.41ab7619e5c97p-8, 0x1.8037efebc0c46p-8,
  0x1.c727155fbb708p-8, 0x1.0b5f5ae5abc27p-7, 0x1.378ad7eba8e32p-7, 0x1.680578de9fdf6p-7, 0x1.9c9eb782d6717p-7,
  0x1.d502d0b5254c3p-7, 0x1.085c4a7f64ae8p-6, 0x1.27904729ecf7bp-6, 0x1.47bada6c7b599p-6, 0x1.6867edea4945bp-6,
  0x1.8913f51fae714p-6, 0x1.a92eec6952cc7p-6, 0x1.c82029c32f07fp-6, 0x1.e54ae009f9925p-6, 0x1.0009941ac006fp-5,
  0x1.0bf1ac50126f9p-5, 0x1.1618b501c3bf9p-5, 0x1.1e421299af7d2p-5, 0x1.243bea305ece7p-5, 0x1.27e11b8751b9cp-5,
  0x1.291ac05d51e68p-5,
};

struct PbFace {
  double A[6];        // destination (canvas / crop) -> source (face) map: cv2's inverse of the given matrix
  int x0, y0, rw, rh; // ROI on the canvas
  int k2;             // second erosion kernel (0 -> 3x3)
  int r;              // blur radius (w_edge)
  int goff;           // offset of the blur kernel in the coefficient array
  int pad_;
  long long off;      // offset of the face's ROI planes (floats)
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

void invert_affine(const double* M, double* A) {      // cv2.invertAffineTransform / warpAffine's own inversion
  double D = M[0] * M[4] - M[1] * M[3];
  D = D != 0. ? 1. / D : 0.;
  const double A11 = M[4] * D, A22 = M[0] * D, A12 = -M[1] * D, A21 = -M[3] * D;
  A[0] = A11; A[1] = A12; A[2] = -A11 * M[2] - A12 * M[5];
  A[3] = A21; A[4] = A22; A[5] = -A21 * M[2] - A22 * M[5];
}

void face_roi(const double* inv, int S, int H, int W, int* roi) {
  double xmn = 1e300, xmx = -1e300, ymn = 1e300, ymx = -1e300;
  const double c[4][2] = {{-2., -2.}, {S + 2., -2.}, {-2., S + 2.}, {S + 2., S + 2.}};
  for (int i = 0; i < 4; ++i) {
    const double x = c[i][0] * inv[0] + c[i][1] * inv[1] + inv[2];
    const double y = c[i][0] * inv[3] + c[i][1] * inv[4] + inv[5];
    xmn = std::min(xmn, x); xmx = std::max(xmx, x); ymn = std::min(ymn, y); ymx = std::max(ymx, y);
  }
  auto clampd = [](double v, int lo, int hi) { return (int)std::max<double>(lo, std::min<double>(hi, v)); };
  const int x0 = clampd(std::floor(xmn) - kRoiPad, 0, W), y0 = clampd(std::floor(ymn) - kRoiPad, 0, H);
  const int x1 = clampd(std::ceil(xmx) + kRoiPad + 1, 0, W), y1 = clampd(std::ceil(ymx) + kRoiPad + 1, 0, H);
  roi[0] = x0; roi[1] = y0; roi[2] = std::max(x1 - x0, 0); roi[3] = std::max(y1 - y0, 0);
}

// cv2.getGaussianKernel(n, sigma): fixed tables for n <= 9 and sigma <= 0, else the normalised exp
void gaussian_kernel(int n, double sigma, std::vector<double>& k) {
  static const double t3[] = {0.25, 0.5, 0.25}, t5[] = {0.0625, 0.25, 0.375, 0.25, 0.0625},
      t7[] = {0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125},
      t9[] = {0.015625, 0.05078125, 0.1171875, 0.19921875, 0.234375, 0.19921875, 0.1171875, 0.05078125, 0.015625};
  k.assign(n, 0.);
  if (sigma <= 0 && n <= 9) {
    const double* t = n == 1 ? nullptr : n == 3 ? t3 : n == 5 ? t5 : n == 7 ? t7 : t9;
    for (int i = 0; i < n; ++i) k[i] = t ? t[i] : 1.;
    return;
  }
  const double sig = sigma > 0 ? sigma : n * 0.15 + 0.35;
  const double scale2 = -0.125 / (sig * sig);
  const int n2 = (n - 1) / 2;
  std::vector<double> v(n2);
  double sum = 0.;
  for (int i = 0, x = 1 - n; i < n2; ++i, x += 2) { v[i] = std::exp((double)(x * x) * scale2); sum += v[i]; }
  sum = sum * 2 + 1.;
  const double mul = 1. / sum;
  for (int i = 0; i < n2; ++i) k[i] = k[n - 1 - i] = v[i] * mul;
  k[n2] = mul;
}

// ---- device helpers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_coord(const double* A, int x, int y, int& ix, int& iy, int& fx, int& fy) {
  const int ad = __double2int_rn(__dmul_rn(__dmul_rn(A[0], (double)x), 1024.));
  const int bd = __double2int_rn(__dmul_rn(__dmul_rn(A[3], (double)x), 1024.));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(A[1], (double)y), A[2]), 1024.)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(A[4], (double)y), A[5]), 1024.)) + 16;
  const int X = (X0 + ad) >> 5, Y = (Y0 + bd) >> 5;
  ix = min(max(X >> 5, -32768), 32767); iy = min(max(Y >> 5, -32768), 32767);   // cv2 keeps them as int16 (saturate_cast)
  fx = X & 31; fy = Y & 31;
}

__device__ __forceinline__ int border_idx(int p, int n, int mode) {
  if (p >= 0 && p < n) return p;
  if (mode == 0) return -1;
  if (mode == 4) {                         // reflect-101
    if (n == 1) return 0;
    const int per = 2 * (n - 1);
    int q = p % per; if (q < 0) q += per;
    return q >= n ? per - q : q;
  }
  const int per = 2 * n;                   // reflect
  int q = p % per; if (q < 0) q += per;
  return q >= n ? per - 1 - q : q;
}

// bilinear u8 HWC 3-channel sample, cv2 fixed point; mode 0 = constant cval
__device__ __forceinline__ void sample_u8(const uint8_t* src, int h, int w, int ix, int iy, int fx, int fy, int mode,
                                          const int* cval, int* out) {
  const int wt[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int yy = border_idx(iy + (t >> 1), h, mode), xx = border_idx(ix + (t & 1), w, mode);
    if (yy >= 0 && xx >= 0) {
      const uint8_t* p = src + ((size_t)yy * w + xx) * 3;
      acc[0] += p[0] * wt[t]; acc[1] += p[1] * wt[t]; acc[2] += p[2] * wt[t];
    } else {
      acc[0] += cval[0] * wt[t]; acc[1] += cval[1] * wt[t]; acc[2] += cval[2] * wt[t];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = min(max((acc[c] + (1 << 14)) >> 15, 0), 255);
}

// warpAffine's float32 weight table for 1/32 steps: (1-b)(1-a), (1-b)a, b(1-a), ba rounded to float32
__device__ __forceinline__ void bilinear_wt(int fx, int fy, float* wt) {
  const float a = fx * (1.f / 32.f), b = fy * (1.f / 32.f);
  wt[0] = __fmul_rn(1.f - b, 1.f - a); wt[1] = __fmul_rn(1.f - b, a); wt[2] = __fmul_rn(b, 1.f - a); wt[3] = __fmul_rn(b, a);
}

// bilinear f64 sample of `nch` interleaved channels of an S x S image, constant border 0 (cv2.warpAffine on CV_64F):
// products and the left-to-right sum in double
template <int NCH>
__device__ __forceinline__ void sample_f64(const double* src, int S, int ix, int iy, int fx, int fy, double* out) {
  float wt[4];
  bilinear_wt(fx, fy, wt);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int yy = iy + (t >> 1), xx = ix + (t & 1);
    const bool in = yy >= 0 && yy < S && xx >= 0 && xx < S;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const double s = in ? src[((size_t)yy * S + xx) * NCH + c] : 0.;
      out[c] = t == 0 ? __dmul_rn(s, (double)wt[0]) : __dadd_rn(out[c], __dmul_rn(s, (double)wt[t]));
    }
  }
}

// ---- kernels ----------------------------------------------------------------------------------------------------
__global__ void k_warp_crop(const uint8_t* __restrict__ src, int h, int w, const double* __restrict__ maps, int n,
                            uint8_t* __restrict__ out, int oh, int ow, int mode, int c0, int c1, int c2) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh || f >= n) return;
  int ix, iy, fx, fy, v[3];
  const int cval[3] = {c0, c1, c2};
  warp_coord(maps + 6 * f, x, y, ix, iy, fx, fy);
  sample_u8(src, h, w, ix, iy, fx, fy, mode, cval, v);
  uint8_t* o = out + (((size_t)f * oh + y) * ow + x) * 3;
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

// INTER_LINEAR taps of one output coordinate (cv2 resize): source index and float fraction
__device__ __forceinline__ void lin_tap(int d, double scale, int& s, float& f) {
  f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
  const float fl = floorf(f);
  s = (int)fl;
  f = __fsub_rn(f, fl);
}

__global__ void k_resize_u8(const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst, int oh, int ow,
                            double sx_scale, double sy_scale, int n) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh || f >= n) return;
  src += (size_t)f * h * w * 3;
  uint8_t* o = dst + (((size_t)f * oh + y) * ow + x) * 3;
  if (w == 2 * ow && h == 2 * oh) {        // cv2 runs an exact halving as INTER_AREA
    const uint8_t* p = src + ((size_t)(2 * y) * w + 2 * x) * 3;
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)((p[c] + p[c + 3] + p[(size_t)w * 3 + c] + p[(size_t)w * 3 + c + 3] + 2) >> 2);
    return;
  }
  int sx, sy;
  float fx, fy;
  lin_tap(x, sx_scale, sx, fx);
  if (sx < 0) { sx = 0; fx = 0.f; }
  if (sx >= w - 1) { sx = w - 1; fx = 0.f; }
  const int a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f)), a1 = __float2int_rn(__fmul_rn(fx, 2048.f));
  const int sx1 = min(sx + 1, w - 1);
  lin_tap(y, sy_scale, sy, fy);
  const int b0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fy), 2048.f)), b1 = __float2int_rn(__fmul_rn(fy, 2048.f));
  const int y0 = min(max(sy, 0), h - 1), y1 = min(max(sy + 1, 0), h - 1);
  const uint8_t* r0 = src + (size_t)y0 * w * 3;
  const uint8_t* r1 = src + (size_t)y1 * w * 3;
  for (int c = 0; c < 3; ++c) {
    const int s0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1, s1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
    const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
    o[c] = (uint8_t)min(max(v, 0), 255);
  }
}

// INTER_AREA, integer factors (resizeAreaFast): window sums; 2 x 2 rounds as (s + 2) >> 2, others cvRound(s * (1.f / area))
__global__ void k_resize_area_fast_u8(const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst, int oh, int ow,
                                      int sx, int sy, float inv_area, int n) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh || f >= n) return;
  src += (size_t)f * h * w * 3;
  int s[3] = {0, 0, 0};
  for (int i = 0; i < sy; ++i) {
    const uint8_t* p = src + ((size_t)(y * sy + i) * w + (size_t)x * sx) * 3;
    for (int j = 0; j < sx * 3; j += 3) { s[0] += p[j]; s[1] += p[j + 1]; s[2] += p[j + 2]; }
  }
  uint8_t* o = dst + (((size_t)f * oh + y) * ow + x) * 3;
  for (int c = 0; c < 3; ++c)
    o[c] = (uint8_t)(sx == 2 && sy == 2 ? (s[c] + 2) >> 2 : min(max(__float2int_rn(__fmul_rn((float)s[c], inv_area)), 0), 255));
}

// INTER_AREA, general path (resizeArea): per source row the float row sum of the x taps, then the float sum of
// beta * row over the y taps, both in table order; taps padded to kx / ky with weight 0 (adding +0 is exact)
__global__ void k_resize_area_u8(const uint8_t* __restrict__ src, int h, int w, uint8_t* __restrict__ dst, int oh, int ow,
                                 const int* __restrict__ xi, const float* __restrict__ xa, int kx,
                                 const int* __restrict__ yi, const float* __restrict__ ya, int ky, int n) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh || f >= n) return;
  src += (size_t)f * h * w * 3;
  float sum[3] = {0.f, 0.f, 0.f};
  for (int t = 0; t < ky; ++t) {
    const uint8_t* row = src + (size_t)yi[y * ky + t] * w * 3;
    const float beta = ya[y * ky + t];
    float buf[3] = {0.f, 0.f, 0.f};
    for (int u = 0; u < kx; ++u) {
      const uint8_t* p = row + (size_t)xi[x * kx + u] * 3;
      const float a = xa[x * kx + u];
      for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)p[c], a));
    }
    for (int c = 0; c < 3; ++c) sum[c] = __fadd_rn(sum[c], __fmul_rn(beta, buf[c]));
  }
  uint8_t* o = dst + (((size_t)f * oh + y) * ow + x) * 3;
  for (int c = 0; c < 3; ++c) o[c] = (uint8_t)min(max(__float2int_rn(sum[c]), 0), 255);
}

// computeResizeAreaTab in double (cv2's arithmetic), as [dsize, K] source indices and weights padded with weight 0
int area_taps(int ssize, int dsize, double scale, std::vector<int>& idx, std::vector<float>& wt) {
  std::vector<std::vector<std::pair<int, float>>> taps(dsize);
  for (int dx = 0; dx < dsize; ++dx) {
    const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    const double cell = std::min(scale, ssize - fsx1);
    int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
    sx2 = std::min(sx2, ssize - 1);
    sx1 = std::min(sx1, sx2);
    if (sx1 - fsx1 > 1e-3) taps[dx].push_back({sx1 - 1, (float)((sx1 - fsx1) / cell)});
    for (int sx = sx1; sx < sx2; ++sx) taps[dx].push_back({sx, (float)(1.0 / cell)});
    if (fsx2 - sx2 > 1e-3) taps[dx].push_back({sx2, (float)(std::min(std::min(fsx2 - sx2, 1.), cell) / cell)});
  }
  size_t K = 1;
  for (const auto& t : taps) K = std::max(K, t.size());
  idx.assign((size_t)dsize * K, 0);
  wt.assign((size_t)dsize * K, 0.f);
  for (int d = 0; d < dsize; ++d)
    for (size_t t = 0; t < taps[d].size(); ++t) { idx[d * K + t] = taps[d][t].first; wt[d * K + t] = taps[d][t].second; }
  return (int)K;
}

// crops of several equal-size images: crop f samples image img_of[f] (the k_warp_crop arithmetic)
__global__ void k_warp_crop_multi(const uint8_t* __restrict__ src, int h, int w, const double* __restrict__ maps,
                                  const int* __restrict__ img_of, int n, uint8_t* __restrict__ out, int oh, int ow, int mode,
                                  int c0, int c1, int c2) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh || f >= n) return;
  int ix, iy, fx, fy, v[3];
  const int cval[3] = {c0, c1, c2};
  warp_coord(maps + 6 * f, x, y, ix, iy, fx, fy);
  sample_u8(src + (size_t)img_of[f] * h * w * 3, h, w, ix, iy, fx, fy, mode, cval, v);
  uint8_t* o = out + (((size_t)f * oh + y) * ow + x) * 3;
  o[0] = (uint8_t)v[0]; o[1] = (uint8_t)v[1]; o[2] = (uint8_t)v[2];
}

// float64 INTER_LINEAR tap (cv2.resize on CV_64F): source coordinate fma(d + 0.5, ssize / dsize, -0.5) in double, the two
// clamped source indices and the fraction
__device__ __forceinline__ void lin_tap_f64(int d, double scale, int n, int& i0, int& i1, double& t) {
  const double f = __fma_rn((double)d + 0.5, scale, -0.5), fl = floor(f);
  const int i = (int)fl;
  t = __dsub_rn(f, fl);
  i0 = min(max(i, 0), n - 1);
  i1 = min(max(i + 1, 0), n - 1);
}

// rows first, each pass the lerp fma(b - a, t, a); scale = source size / destination size
__global__ void k_resize_f64(const double* __restrict__ src, int h, int w, double* __restrict__ dst, int oh, int ow,
                             double sx_scale, double sy_scale) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, f = blockIdx.z;
  if (x >= ow || y >= oh) return;
  src += (size_t)f * h * w;
  int x0, x1, y0, y1;
  double tx, ty;
  lin_tap_f64(x, sx_scale, w, x0, x1, tx);
  lin_tap_f64(y, sy_scale, h, y0, y1, ty);
  const double* r0 = src + (size_t)y0 * w;
  const double* r1 = src + (size_t)y1 * w;
  const double a = __fma_rn(__dsub_rn(r0[x1], r0[x0]), tx, r0[x0]), b = __fma_rn(__dsub_rn(r1[x1], r1[x0]), tx, r1[x0]);
  dst[((size_t)f * oh + y) * ow + x] = __fma_rn(__dsub_rn(b, a), ty, a);
}

// ones(S x S) warped to the ROI, f32 bilinear with constant 0: the in-bounds weights, exact multiples of 1/1024
__global__ void k_mask_warp(const PbFace* __restrict__ faces, int S, float* __restrict__ ws) {
  const PbFace& F = faces[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= F.rw || y >= F.rh) return;
  int ix, iy, fx, fy;
  warp_coord(F.A, F.x0 + x, F.y0 + y, ix, iy, fx, fy);
  const int wt[4] = {(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx};
  int acc = 0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int yy = iy + (t >> 1), xx = ix + (t & 1);
    if (yy >= 0 && yy < S && xx >= 0 && xx < S) acc += wt[t];
  }
  ws[F.off + (size_t)y * F.rw + x] = (float)acc * (1.f / 1024.f);
}

// one pass of a rectangular erosion on the ROI planes: plane `in` -> plane `out` (0/1/2 within the face's planes)
__global__ void k_erode(const PbFace* __restrict__ faces, float* __restrict__ ws, int in, int out, int k1, bool cols) {
  const PbFace& F = faces[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= F.rw || y >= F.rh) return;
  int k = k1 >= 0 ? k1 : F.k2;
  if (k == 0) k = 3;
  const int a = k / 2;
  const size_t plane = (size_t)F.rw * F.rh;
  const float* src = ws + F.off + in * plane;
  float m = INFINITY;
  if (!cols) {
    const int lo = max(x - a, 0), hi = min(x - a + k, F.rw);
    for (int j = lo; j < hi; ++j) m = fminf(m, src[(size_t)y * F.rw + j]);
  } else {
    const int lo = max(y - a, 0), hi = min(y - a + k, F.rh);
    for (int i = lo; i < hi; ++i) m = fminf(m, src[(size_t)i * F.rw + x]);
  }
  ws[F.off + out * plane + (size_t)y * F.rw + x] = m;
}

// sum of each face's first erosion in fp64: one block per face, fixed-order strided partials and tree
__global__ void k_area(const PbFace* __restrict__ faces, const float* __restrict__ ws, int plane_idx, double* __restrict__ area) {
  const PbFace& F = faces[blockIdx.x];
  const size_t plane = (size_t)F.rw * F.rh;
  const float* p = ws + F.off + plane_idx * plane;
  double s = 0.;
  for (size_t i = threadIdx.x; i < plane; i += blockDim.x) s += (double)p[i];
  __shared__ double red[1024];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) area[blockIdx.x] = red[0];
}

// f32 Gaussian pass on the ROI planes: reflect-101 at the canvas border, 0 outside the ROI inside the canvas.  cv2's
// sepFilter2D (x86-64, AVX2) picks the arithmetic by the output's canvas column gx = F.x0 + x, so the ROI pass does too:
//   rows, n >= 7   gx < W - W % 4: FMA chain in tap order from 0; the last W % 4 columns: k[0] v[0], then the first
//                  4 * ((n - 1) / 4) taps as rounded products and sums, the rest FMA'd
//   rows, n == 5   gx < W - W % 2: fma(v0, k[2], p1 k[3]) + p2 k[4]; an odd width's last column rounds every step
//   rows, n == 3   v0 k[1] + p1 k[2]                                    (p_i = v[+i] + v[-i])
//   columns        the centre product, then fma(p_i, k[r + i], acc); the last W % 8 columns round every step
// The zeros outside the ROI change nothing in any form: fma(0, k, acc) = acc + 0 * k = acc and v + 0 = v exactly.
__global__ void k_blur_roi(const PbFace* __restrict__ faces, float* __restrict__ ws, const float* __restrict__ gk, int in,
                           int out, bool cols, int H, int W) {
  const PbFace& F = faces[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= F.rw || y >= F.rh) return;
  const size_t plane = (size_t)F.rw * F.rh;
  const float* src = ws + F.off + in * plane;
  const float* k = gk + F.goff;
  const int r = F.r, n = 2 * r + 1, gx = F.x0 + x;
  auto tap = [&](int d) -> float {          // the value d taps away along the pass
    if (!cols) {
      const int g = border_idx(gx + d, W, 4) - F.x0;
      return g >= 0 && g < F.rw ? src[(size_t)y * F.rw + g] : 0.f;
    }
    const int g = border_idx(F.y0 + y + d, H, 4) - F.y0;
    return g >= 0 && g < F.rh ? src[(size_t)g * F.rw + x] : 0.f;
  };
  float acc;
  if (cols) {
    const bool fused = gx < W - W % 8;
    acc = __fmul_rn(tap(0), k[r]);
    for (int i = 1; i <= r; ++i) {
      const float p = __fadd_rn(tap(i), tap(-i));
      acc = fused ? __fmaf_rn(p, k[r + i], acc) : __fadd_rn(acc, __fmul_rn(p, k[r + i]));
    }
  } else if (n == 3) {
    acc = __fadd_rn(__fmul_rn(tap(0), k[1]), __fmul_rn(__fadd_rn(tap(-1), tap(1)), k[2]));
  } else if (n == 5) {
    const float c = tap(0), q1 = __fmul_rn(__fadd_rn(tap(-1), tap(1)), k[3]);
    acc = gx < W - W % 2 ? __fmaf_rn(c, k[2], q1) : __fadd_rn(__fmul_rn(c, k[2]), q1);
    acc = __fadd_rn(acc, __fmul_rn(__fadd_rn(tap(-2), tap(2)), k[4]));
  } else if (gx < W - W % 4) {
    acc = 0.f;
    for (int t = 0; t < n; ++t) acc = __fmaf_rn(tap(t - r), k[t], acc);
  } else {
    const int unfused = 4 * ((n - 1) / 4);
    acc = __fmul_rn(tap(-r), k[0]);
    for (int t = 1; t < n; ++t)
      acc = t <= unfused ? __fadd_rn(acc, __fmul_rn(tap(t - r), k[t])) : __fmaf_rn(tap(t - r), k[t], acc);
  }
  ws[F.off + out * plane + (size_t)y * F.rw + x] = acc;
}

__global__ void k_u8_to_f64(const uint8_t* __restrict__ src, double* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (double)src[i];
}

// f64 Gaussian pass over whole 512 x 512 parse masks (blockIdx.z = face), reflect-101, cv2's arithmetic: rows are an FMA
// chain in tap order from 0 (512 is a multiple of cv2's 4-column blocks, so no column takes its scalar tail); columns take
// the centre product, then acc + (v[+i] + v[-i]) k[r + i] with every step rounded
__global__ void k_blur_f64(const double* __restrict__ src, double* __restrict__ dst, const double* __restrict__ k, int ks, bool cols) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= kParse || y >= kParse) return;
  const size_t base = (size_t)blockIdx.z * kParse * kParse;
  src += base;
  const int r = ks / 2;
  double acc;
  if (!cols) {
    acc = 0.;
    for (int t = 0; t < ks; ++t) acc = __fma_rn(src[(size_t)y * kParse + border_idx(x + t - r, kParse, 4)], k[t], acc);
  } else {
    acc = __dmul_rn(src[(size_t)y * kParse + x], k[r]);
    for (int i = 1; i <= r; ++i) {
      const double p = __dadd_rn(src[(size_t)border_idx(y + i, kParse, 4) * kParse + x], src[(size_t)border_idx(y - i, kParse, 4) * kParse + x]);
      acc = __dadd_rn(acc, __dmul_rn(p, k[r + i]));
    }
  }
  dst[base + (size_t)y * kParse + x] = acc;
}

// parse_mask[:10] = ... = 0; parse_mask / 255.
__global__ void k_parse_finish(double* __restrict__ p, int nfaces) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)nfaces * kParse * kParse) return;
  const int x = (int)(i % kParse), y = (int)((i / kParse) % kParse);
  const bool edge = x < 10 || y < 10 || x >= kParse - 10 || y >= kParse - 10;
  p[i] = __ddiv_rn(edge ? 0. : p[i], 255.);
}

template <typename T>
__global__ void k_canvas_in(const uint8_t* __restrict__ src, T* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (T)src[i];
}

// astype(np.uint8) as numpy does it on x86: truncate toward zero, keep the low byte
template <typename T>
__global__ void k_canvas_out(const T* __restrict__ src, uint8_t* __restrict__ dst, float* __restrict__ dbg, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T v = src[i];
  dst[i] = (uint8_t)((long long)v & 255);
  if (dbg) dbg[i] = (float)v;
}

// one face into the canvas: inv_restored (u8 fixed-point warp, or the f64 warp for FT = double), the parse warp (f64
// bilinear), min(parse, soft), the blend.  A float64 face makes the canvas float64 with or without the parse mask; without
// it numpy multiplies (1 - soft) (float32) with the canvas, which is still uint8 for the first face of an image (a float32
// product) and float64 afterwards (`first`).
template <typename T, typename FT>
__global__ void k_composite(const PbFace* __restrict__ faces, int fi, const FT* __restrict__ face, int S,
                            const double* __restrict__ parse, const float* __restrict__ ws, T* __restrict__ canvas, int W,
                            bool first) {
  const PbFace& F = faces[fi];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= F.rw || y >= F.rh) return;
  int ix, iy, fx, fy;
  warp_coord(F.A, F.x0 + x, F.y0 + y, ix, iy, fx, fy);
  const size_t plane = (size_t)F.rw * F.rh, p = (size_t)y * F.rw + x;
  const float ero = ws[F.off + 2 * plane + p], soft = ws[F.off + 1 * plane + p];
  T* c = canvas + ((size_t)(F.y0 + y) * W + F.x0 + x) * 3;
  if constexpr (sizeof(FT) == 8) {
    static_assert(sizeof(T) == 8, "float64 faces blend into a float64 canvas");
    double v[3];
    sample_f64<3>(face, S, ix, iy, fx, fy, v);
    if (parse) {
      double m = (double)soft, acc;
      sample_f64<1>(parse, S, ix, iy, fx, fy, &acc);
      if (acc < m) m = acc;
      const double om = __dsub_rn(1., m);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch)
        c[ch] = __dadd_rn(__dmul_rn(m, __dmul_rn((double)ero, v[ch])), __dmul_rn(om, c[ch]));
    } else {
      const float om = __fsub_rn(1.f, soft);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const double bg = first ? (double)__fmul_rn(om, (float)c[ch]) : __dmul_rn((double)om, c[ch]);
        c[ch] = __dadd_rn(__dmul_rn((double)soft, __dmul_rn((double)ero, v[ch])), bg);
      }
    }
  } else {
    int v[3];
    const int zero[3] = {0, 0, 0};
    sample_u8(face, S, S, ix, iy, fx, fy, 0, zero, v);
    if constexpr (sizeof(T) == 8) {
      double m = (double)soft;
      if (parse) {
        double acc;
        sample_f64<1>(parse, S, ix, iy, fx, fy, &acc);
        if (acc < m) m = acc;
      }
      const double om = __dsub_rn(1., m);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const double pasted = (double)__fmul_rn(ero, (float)v[ch]);
        c[ch] = __dadd_rn(__dmul_rn(m, pasted), __dmul_rn(om, (double)c[ch]));
      }
    } else {
      const float om = __fsub_rn(1.f, soft);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float pasted = __fmul_rn(ero, (float)v[ch]);
        c[ch] = __fadd_rn(__fmul_rn(soft, pasted), __fmul_rn(om, (float)c[ch]));
      }
    }
  }
}

// per-image maximum of a float64 canvas: block (slice, image) -> partial[image * gridDim.x + slice]
__global__ void k_canvas_max(const double* __restrict__ canvas, size_t per_img, double* __restrict__ partial) {
  const double* p = canvas + (size_t)blockIdx.y * per_img;
  double m = -INFINITY;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per_img; i += (size_t)gridDim.x * blockDim.x) m = fmax(m, p[i]);
  __shared__ double red[256];
  red[threadIdx.x] = m;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.y * gridDim.x + blockIdx.x] = red[0];
}

// astype(np.uint16): truncate toward zero, keep the low 16 bits
__global__ void k_canvas_out16(const double* __restrict__ src, uint16_t* __restrict__ dst, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (uint16_t)((long long)src[i] & 65535);
}

inline dim3 grid2(int w, int h, int z, dim3 b) { return dim3((w + b.x - 1) / b.x, (h + b.y - 1) / b.y, z); }

struct Plan {
  std::vector<PbFace> faces;
  size_t roi_floats = 0;
  int max_rw = 0, max_rh = 0;
};

int make_plan(int H, int W, int n, int S, const double* inv, Plan& P) {
  P.faces.assign(n, PbFace{});
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    PbFace& F = P.faces[i];
    invert_affine(inv + 6 * i, F.A);
    int roi[4];
    face_roi(inv + 6 * i, S, H, W, roi);
    F.x0 = roi[0]; F.y0 = roi[1]; F.rw = roi[2]; F.rh = roi[3];
    F.off = (long long)off;
    off += align256((size_t)F.rw * F.rh * 3 * 4) / 4;
    P.max_rw = std::max(P.max_rw, F.rw);
    P.max_rh = std::max(P.max_rh, F.rh);
  }
  P.roi_floats = off;
  return 0;
}

struct Layout {
  size_t canvas, roi, parse0, parse1, parse_rs, faces, area, pgauss, gauss, cmax, total;
};

constexpr int kMaxSlices = 64;        // k_canvas_max partials per image

// f64_faces: float64 restored faces (a gray image), whose canvas is float64 with or without the parse masks
Layout layout(int H, int W, int n, int S, bool use_parse, const Plan& P, int gauss_floats, int n_img = 1, bool f64_faces = false) {
  Layout L{};
  size_t o = 0;
  auto take = [&](size_t b) { const size_t r = o; o += align256(b); return r; };
  L.canvas = take((size_t)n_img * H * W * 3 * (use_parse || f64_faces ? 8 : 4));
  L.roi = take(P.roi_floats * 4);
  const size_t pm = (size_t)n * kParse * kParse * 8;
  L.parse0 = take(use_parse ? pm : 0);
  L.parse1 = take(use_parse ? pm : 0);
  L.parse_rs = take(use_parse && S != kParse ? (size_t)n * S * S * 8 : 0);
  L.faces = take((size_t)std::max(n, 1) * sizeof(PbFace));
  L.area = take((size_t)std::max(n, 1) * 8);
  L.pgauss = take(kParseK * 8);
  L.gauss = take((size_t)gauss_floats * 4);
  L.cmax = take(f64_faces ? (size_t)n_img * kMaxSlices * 8 : 0);
  L.total = o;
  return L;
}

// the largest w_edge a face can get: the first erosion is <= 1 on its ROI
int max_gauss_floats(const Plan& P) {
  int s = 0;
  for (const PbFace& F : P.faces) s += 2 * ((int)std::sqrt((double)F.rw * F.rh) / 20) + 1;
  return s;
}

// n_img canvases [n_img,H,W,3]; face i goes into canvas img_of[i] (img_of == nullptr: all into canvas 0).  Every step
// before the composite is per face, so a face's result does not depend on the other canvases of the batch.
// FT = double (float64 faces): canvas_u16 (optional) receives astype(np.uint16) of every canvas and wide_out[i] (host) tells
// whether canvas i exceeds 256, where the reference returns the uint16 image.
template <typename T, typename FT = uint8_t>
int paste_impl(uint8_t* canvas_u8, int n_img, const int32_t* img_of, int H, int W, const FT* faces, int n, int S,
               const uint8_t* parse_u8, const double* inv, double upscale, float* dbg, int32_t* w_edge_out, char* ws,
               int64_t ws_bytes, cudaStream_t st, uint16_t* canvas_u16 = nullptr, int32_t* wide_out = nullptr) {
  const bool use_parse = parse_u8 != nullptr;
  constexpr bool kF64 = sizeof(FT) == 8;
  Plan P;
  CFB_CHECK(make_plan(H, W, n, S, inv, P));
  const Layout L = layout(H, W, n, S, use_parse, P, max_gauss_floats(P), n_img, kF64);
  CFB_REQUIRE((int64_t)L.total <= ws_bytes, "cfb_paste_faces: workspace too small");
  T* canvas = (T*)(ws + L.canvas);
  float* roi = (float*)(ws + L.roi);
  PbFace* dfaces = (PbFace*)(ws + L.faces);
  double* darea = (double*)(ws + L.area);
  float* dgauss = (float*)(ws + L.gauss);
  double* dpk = (double*)(ws + L.pgauss);
  const size_t npx = (size_t)n_img * H * W * 3;
  k_canvas_in<T><<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(canvas_u8, canvas, npx);
  CFB_LAUNCH_CHECK();
  const dim3 b(32, 8);
  std::vector<double> gk;
  const double* parse_src = nullptr;
  if (n > 0) {
    const int k1 = (int)(2 * upscale);
    CFB_CUDA(cudaMemcpyAsync(dfaces, P.faces.data(), n * sizeof(PbFace), cudaMemcpyHostToDevice, st));
    const dim3 g = grid2(P.max_rw, P.max_rh, n, b);
    k_mask_warp<<<g, b, 0, st>>>(dfaces, S, roi);
    CFB_LAUNCH_CHECK();
    k_erode<<<g, b, 0, st>>>(dfaces, roi, 0, 1, k1, false);
    CFB_LAUNCH_CHECK();
    k_erode<<<g, b, 0, st>>>(dfaces, roi, 1, 2, k1, true);          // plane 2: inv_mask_erosion
    CFB_LAUNCH_CHECK();
    k_area<<<n, 1024, 0, st>>>(dfaces, roi, 2, darea);
    CFB_LAUNCH_CHECK();
    if (use_parse) {                        // independent of the areas: enqueue before the read-back
      double* p0 = (double*)(ws + L.parse0);
      double* p1 = (double*)(ws + L.parse1);
      gk.assign(kParseK, 0.);
      for (int t = 0; t <= kParseK / 2; ++t) gk[t] = gk[kParseK - 1 - t] = kParseKernelHalf[t];
      CFB_CUDA(cudaMemcpyAsync(dpk, gk.data(), kParseK * 8, cudaMemcpyHostToDevice, st));
      const size_t pn = (size_t)n * kParse * kParse;
      k_u8_to_f64<<<(unsigned)((pn + 255) / 256), 256, 0, st>>>(parse_u8, p0, pn);
      CFB_LAUNCH_CHECK();
      const dim3 gp = grid2(kParse, kParse, n, b);
      for (int rep = 0; rep < 2; ++rep) {
        k_blur_f64<<<gp, b, 0, st>>>(p0, p1, dpk, kParseK, false);
        CFB_LAUNCH_CHECK();
        k_blur_f64<<<gp, b, 0, st>>>(p1, p0, dpk, kParseK, true);
        CFB_LAUNCH_CHECK();
      }
      k_parse_finish<<<(unsigned)((pn + 255) / 256), 256, 0, st>>>(p0, n);
      CFB_LAUNCH_CHECK();
      parse_src = p0;
      if (S != kParse) {
        double* rs = (double*)(ws + L.parse_rs);
        const double sc = (double)kParse / S;
        k_resize_f64<<<grid2(S, S, n, b), b, 0, st>>>(p0, kParse, kParse, rs, S, S, sc, sc);
        CFB_LAUNCH_CHECK();
        parse_src = rs;
      }
    }
    std::vector<double> area(n);
    CFB_CUDA(cudaMemcpyAsync(area.data(), darea, n * 8, cudaMemcpyDeviceToHost, st));
    CFB_CUDA(cudaStreamSynchronize(st));
    std::vector<float> gauss;
    for (int i = 0; i < n; ++i) {
      const int w_edge = (int)std::sqrt(area[i]) / 20;
      PbFace& F = P.faces[i];
      F.k2 = 2 * w_edge;
      F.r = w_edge;
      F.goff = (int)gauss.size();
      gaussian_kernel(2 * w_edge + 1, 0., gk);
      for (double v : gk) gauss.push_back((float)v);
      if (w_edge_out) w_edge_out[i] = w_edge;
    }
    CFB_REQUIRE(gauss.size() <= (size_t)max_gauss_floats(P), "cfb_paste_faces: blur kernel larger than its ROI bound");
    CFB_CUDA(cudaMemcpyAsync(dgauss, gauss.data(), gauss.size() * 4, cudaMemcpyHostToDevice, st));
    CFB_CUDA(cudaMemcpyAsync(dfaces, P.faces.data(), n * sizeof(PbFace), cudaMemcpyHostToDevice, st));
    k_erode<<<g, b, 0, st>>>(dfaces, roi, 2, 0, -1, false);
    CFB_LAUNCH_CHECK();
    k_erode<<<g, b, 0, st>>>(dfaces, roi, 0, 1, -1, true);           // plane 1: inv_mask_center
    CFB_LAUNCH_CHECK();
    k_blur_roi<<<g, b, 0, st>>>(dfaces, roi, dgauss, 1, 0, false, H, W);
    CFB_LAUNCH_CHECK();
    k_blur_roi<<<g, b, 0, st>>>(dfaces, roi, dgauss, 0, 1, true, H, W);   // plane 1: inv_soft_mask
    CFB_LAUNCH_CHECK();
    std::vector<char> touched(n_img, 0);      // the canvas of an image is still uint8-valued until its first face
    for (int i = 0; i < n; ++i) {
      const PbFace& F = P.faces[i];
      const int im = img_of ? img_of[i] : 0;
      const bool first = !touched[im];
      touched[im] = 1;
      if (F.rw == 0 || F.rh == 0) continue;
      T* cv = canvas + (size_t)im * H * W * 3;
      k_composite<T, FT><<<grid2(F.rw, F.rh, 1, b), b, 0, st>>>(dfaces, i, faces + (size_t)i * S * S * 3, S,
                                                                 parse_src ? parse_src + (size_t)i * S * S : nullptr, roi, cv, W,
                                                                 first);
      CFB_LAUNCH_CHECK();
    }
  }
  if constexpr (kF64) {
    if (wide_out) {
      double* dmax = (double*)(ws + L.cmax);
      k_canvas_max<<<dim3(kMaxSlices, n_img), 256, 0, st>>>(canvas, (size_t)H * W * 3, dmax);
      CFB_LAUNCH_CHECK();
      std::vector<double> mx((size_t)n_img * kMaxSlices);
      CFB_CUDA(cudaMemcpyAsync(mx.data(), dmax, mx.size() * 8, cudaMemcpyDeviceToHost, st));
      CFB_CUDA(cudaStreamSynchronize(st));
      bool any = false;
      for (int i = 0; i < n_img; ++i) {
        wide_out[i] = *std::max_element(mx.begin() + (size_t)i * kMaxSlices, mx.begin() + (size_t)(i + 1) * kMaxSlices) > 256.;
        any = any || wide_out[i];
      }
      if (any && canvas_u16) {
        k_canvas_out16<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(canvas, canvas_u16, npx);
        CFB_LAUNCH_CHECK();
      }
    }
  }
  k_canvas_out<T><<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(canvas, canvas_u8, dbg, npx);
  CFB_LAUNCH_CHECK();
  return 0;
}


// ---- INTER_LANCZOS4 ------------------------------------------------------------------------------------------------
// cv2's interpolateLanczos4: the window from one sin / cos of -(x + 3) pi / 4 rotated by multiples of 45 degrees, each tap
// divided by its own y * y, normalised by the float sum; x < FLT_EPSILON is the unit tap
void lanczos4_coeffs(float x, float* cf) {
  static const double s45 = 0.70710678118654752440084436210485;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  if (x < 1.1920929e-07f) {
    for (int i = 0; i < 8; ++i) cf[i] = 0.f;
    cf[3] = 1.f;
    return;
  }
  const double pi = 3.1415926535897932384626433832795;
  const double xd = (double)x, y0 = -(xd + 3) * pi * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
  float sum = 0.f;
  for (int i = 0; i < 8; ++i) {
    const double y = (double)(float)(-(xd + 3 - i) * pi * 0.25);
    cf[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    sum += cf[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) cf[i] *= sum;
}

// per output coordinate: floor of the source coordinate (taps at idx - 3 .. idx + 4, clamped by the kernel) and the eight
// weights * 2048 saturated to int16, as cv::resize builds them
void lanczos4_table(int ssize, int dsize, int32_t* idx, int16_t* coef) {
  const double scale = 1. / ((double)dsize / ssize);
  for (int d = 0; d < dsize; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    const int s = (int)std::floor(f);
    f -= s;
    float cf[8];
    lanczos4_coeffs(f, cf);
    idx[d] = s;
    for (int k = 0; k < 8; ++k)
      coef[d * 8 + k] = (int16_t)std::max(-32768.f, std::min(32767.f, std::nearbyint(cf[k] * 2048.f)));
  }
}

// cv2's float path (CV_16U): interpolateLanczos4 as resize builds float weights -- x + 3 summed in float32, each tap's
// y = -((x + 3) - i) pi / 4 in double from the float32 (x + 3) - i, a tap at |(x + 3) - i| < 1e-6 set to 1e30 before the
// normalisation (so x = 0 leaves the unit tap and neighbours of about 1e-31).
void lanczos4_coeffs_f32(float x, float* cf) {
  static const double s45 = 0.70710678118654752440084436210485;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  const double pi = 3.1415926535897932384626433832795;
  const float x3 = x + 3.f;
  const double y0 = -(double)x3 * pi * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
  float sum = 0.f;
  for (int i = 0; i < 8; ++i) {
    const float t = x3 - (float)i;
    if (std::fabs(t) >= 1e-6f) {
      const double y = -(double)t * pi * 0.25;
      cf[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    } else {
      cf[i] = 1e30f;
    }
    sum += cf[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) cf[i] *= sum;
}

void lanczos4_table_f32(int ssize, int dsize, int32_t* idx, float* coef) {
  const double scale = 1. / ((double)dsize / ssize);
  for (int d = 0; d < dsize; ++d) {
    float f = (float)((d + 0.5) * scale - 0.5);
    const int s = (int)std::floor(f);
    f -= s;
    idx[d] = s;
    lanczos4_coeffs_f32(f, coef + (size_t)d * 8);
  }
}

constexpr int kLzTileW = 64;     // output columns of a block
constexpr int kLzRows = 48;      // source rows a block may hold (the host picks the band height to fit)

// The arithmetic of one element type: uint8 sums int16 taps in int32 and rounds with (v + 2^21) >> 22; uint16 sums float32
// products left to right, every product and sum rounded on its own (cv2's SSE code has no fused multiply-add), then rint.
template <class T> struct LzOps;
template <> struct LzOps<uint8_t> {
  using Coef = short;
  using Acc = int;
  static __device__ __forceinline__ int mac(int a, int v, short c) { return a + v * c; }
  static __device__ __forceinline__ uint8_t out(int acc) { return (uint8_t)min(max((acc + (1 << 21)) >> 22, 0), 255); }
};
template <> struct LzOps<uint16_t> {
  using Coef = float;
  using Acc = float;
  static __device__ __forceinline__ float mac(float a, float v, float c) { return __fadd_rn(a, __fmul_rn(v, c)); }
  static __device__ __forceinline__ uint16_t out(float acc) { return (uint16_t)fminf(fmaxf(rintf(acc), 0.f), 65535.f); }
};

// one block: a band of `band` output rows x kLzTileW output columns of image blockIdx.z.  The horizontal pass of every
// source row the band needs goes to shared memory, the vertical pass reads it back: no intermediate image.
template <class T>
__global__ void __launch_bounds__(256) k_resize_lanczos4(const T* __restrict__ src, int h, int w, T* __restrict__ dst, int oh,
                                                         int ow, const int* __restrict__ xi, const typename LzOps<T>::Coef* __restrict__ xt,
                                                         const int* __restrict__ yi, const typename LzOps<T>::Coef* __restrict__ yt,
                                                         int band) {
  using Op = LzOps<T>;
  using Acc = typename Op::Acc;
  __shared__ Acc hbuf[kLzRows][kLzTileW * 3];
  __shared__ typename Op::Coef sxt[kLzTileW * 8];
  __shared__ int sxi[kLzTileW];
  const int x0 = blockIdx.x * kLzTileW, y0 = blockIdx.y * band, y1 = min(y0 + band, oh);
  const int tw = min(kLzTileW, ow - x0);
  src += (size_t)blockIdx.z * h * w * 3;
  dst += (size_t)blockIdx.z * oh * ow * 3;
  const int rlo = yi[y0] - 3, span = yi[y1 - 1] + 4 - rlo + 1;
  for (int i = threadIdx.x; i < tw * 8; i += 256) sxt[i] = xt[(size_t)x0 * 8 + i];
  for (int i = threadIdx.x; i < tw; i += 256) sxi[i] = xi[x0 + i];
  __syncthreads();
  for (int i = threadIdx.x; i < span * tw; i += 256) {
    const int r = i / tw, xl = i - r * tw;
    const T* row = src + (size_t)min(max(rlo + r, 0), h - 1) * w * 3;
    const int s = sxi[xl] - 3;
    Acc a0 = 0, a1 = 0, a2 = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const T* p = row + min(max(s + k, 0), w - 1) * 3;
      const auto c = sxt[xl * 8 + k];
      a0 = Op::mac(a0, p[0], c); a1 = Op::mac(a1, p[1], c); a2 = Op::mac(a2, p[2], c);
    }
    hbuf[r][xl * 3] = a0; hbuf[r][xl * 3 + 1] = a1; hbuf[r][xl * 3 + 2] = a2;
  }
  __syncthreads();
  const int te = tw * 3;
  for (int i = threadIdx.x; i < (y1 - y0) * te; i += 256) {
    const int yl = i / te, e = i - yl * te, y = y0 + yl, r0 = yi[y] - 3 - rlo;
    Acc acc = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc = Op::mac(acc, hbuf[r0 + k][e], yt[y * 8 + k]);
    dst[((size_t)y * ow + x0) * 3 + e] = Op::out(acc);
  }
}

// cfb_resize_lanczos4_u8 / _u16: tap tables of both axes built on the host (`table`), one launch for the n images
template <class T, class Coef>
int resize_lanczos4(const T* src, int n, int h, int w, T* dst, int out_h, int out_w, void (*table)(int, int, int32_t*, Coef*),
                    const char* fn, cudaStream_t st) {
  const std::string f(fn);
  CFB_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, f + ": bad size");
  CFB_REQUIRE(n <= 65535, f + ": at most 65535 images per call");
  CFB_REQUIRE(n == 0 || (src && dst), f + ": NULL argument");
  if (n == 0) return 0;
  if (h == out_h && w == out_w) {                  // cv2.resize to the same size is a copy
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * h * w * 3 * sizeof(T), cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  // one host block: xi[ow] yi[oh] (int32) then xt[ow * 8] yt[oh * 8] (Coef)
  const size_t ni = (size_t)out_w + out_h;
  std::vector<char> host(ni * 4 + ni * 8 * sizeof(Coef));
  int32_t* xi = (int32_t*)host.data();
  int32_t* yi = xi + out_w;
  Coef* xt = (Coef*)(host.data() + ni * 4);
  Coef* yt = xt + (size_t)out_w * 8;
  table(w, out_w, xi, xt);
  table(h, out_h, yi, yt);
  int band = 16;                                   // the tallest band whose source rows fit the shared rows
  for (;; band /= 2) {
    int span = 0;
    for (int y0 = 0; y0 < out_h; y0 += band) span = std::max(span, yi[std::min(y0 + band, out_h) - 1] - yi[y0] + 8);
    if (span <= kLzRows) break;                    // a band of one row needs eight
  }
  CFB_REQUIRE((out_h + band - 1) / band <= 65535, f + ": output too tall");
  char* dtab = nullptr;
  CFB_CUDA(cudaMallocAsync((void**)&dtab, host.size(), st));
  CFB_CUDA(cudaMemcpyAsync(dtab, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  const int* dxi = (const int*)dtab;
  const Coef* dxt = (const Coef*)(dtab + ni * 4);
  k_resize_lanczos4<T><<<dim3((out_w + kLzTileW - 1) / kLzTileW, (out_h + band - 1) / band, n), 256, 0, st>>>(
      src, h, w, dst, out_h, out_w, dxi, dxt, dxi + out_w, dxt + (size_t)out_w * 8, band);
  CFB_LAUNCH_CHECK();
  CFB_CUDA(cudaFreeAsync(dtab, st));
  return 0;
}

// ---- the gray branch of add_restored_face ----------------------------------------------------------------------
constexpr int kGraySlices = 64;

__device__ __forceinline__ double bgr2gray(const uint8_t* p) {      // 0.2989 r + 0.5870 g + 0.1140 b, left to right
  return __dadd_rn(__dadd_rn(__dmul_rn(0.2989, (double)p[2]), __dmul_rn(0.5870, (double)p[1])), __dmul_rn(0.1140, (double)p[0]));
}

// partial sums over slice blockIdx.x of face blockIdx.y of q = {gray(restored), cropped b, g, r}: the values (stats == NULL)
// or their squared deviations from the means in stats[face][0 / 2][.].  Fixed order: strided per thread, then a tree.
__global__ void k_gray_partial(const uint8_t* __restrict__ restored, const uint8_t* __restrict__ cropped, int npx,
                               const double* __restrict__ stats, double* __restrict__ partial) {
  const int f = blockIdx.y;
  const uint8_t* r = restored + (size_t)f * npx * 3;
  const uint8_t* c = cropped + (size_t)f * npx * 3;
  double mean[4] = {0., 0., 0., 0.};
  if (stats) {
    mean[0] = stats[f * 12];
    for (int k = 0; k < 3; ++k) mean[1 + k] = stats[f * 12 + 6 + k];
  }
  const int per = (npx + gridDim.x - 1) / gridDim.x, lo = blockIdx.x * per, hi = min(lo + per, npx);
  double s[4] = {0., 0., 0., 0.};
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const double q[4] = {bgr2gray(r + (size_t)i * 3), (double)c[(size_t)i * 3], (double)c[(size_t)i * 3 + 1], (double)c[(size_t)i * 3 + 2]};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double d = __dsub_rn(q[k], mean[k]);
      s[k] = __dadd_rn(s[k], stats ? __dmul_rn(d, d) : q[k]);
    }
  }
  __shared__ double red[4][256];
#pragma unroll
  for (int k = 0; k < 4; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
      for (int k = 0; k < 4; ++k) red[k][threadIdx.x] = __dadd_rn(red[k][threadIdx.x], red[k][threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x < 4) partial[((size_t)f * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = red[threadIdx.x][0];
}

// the slices of a face summed in order: stats[face] = {content mean, content std, style mean, style std} x 3 channels (the
// three content channels are the same gray).  pass 0 writes the means, pass 1 sqrt(var + 1e-5).
__global__ void k_gray_stats(const double* __restrict__ partial, int slices, int npx, int pass, double* __restrict__ stats) {
  const int f = blockIdx.x, k = threadIdx.x;
  if (k >= 4) return;
  double s = 0.;
  for (int i = 0; i < slices; ++i) s = __dadd_rn(s, partial[((size_t)f * slices + i) * 4 + k]);
  s = __ddiv_rn(s, (double)npx);
  if (pass) s = sqrt(__dadd_rn(s, 1e-5));
  double* o = stats + f * 12 + pass * 3;
  if (k == 0) o[0] = o[1] = o[2] = s;
  else o[6 + k - 1] = s;
}

// (gray - content mean) / content std * style std + style mean
__global__ void k_gray_apply(const uint8_t* __restrict__ restored, int npx, const double* __restrict__ stats, double* __restrict__ out) {
  const int f = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npx) return;
  const double* st = stats + f * 12;
  const double nrm = __ddiv_rn(__dsub_rn(bgr2gray(restored + ((size_t)f * npx + i) * 3), st[0]), st[3]);
  double* o = out + ((size_t)f * npx + i) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = __dadd_rn(__dmul_rn(nrm, st[9 + c]), st[6 + c]);
}

// ---- is_gray (facelib/utils/misc.py:146-158) of a batch: the exact moments of the three channel differences ---------------
// Image blockIdx.y, pixels strided over the x blocks.  sums[img] = {Σd, Σd²} for d = B-G, G-R, R-B (int64, zeroed by the
// caller); integer adds are exact, so the result does not depend on the order of the atomics.
constexpr int kGrayTestBlocks = 512;     // blocks over all images: about four per SM

__global__ void __launch_bounds__(256) k_is_gray_sums(const uint8_t* __restrict__ img, int64_t npx,
                                                      unsigned long long* __restrict__ sums) {
  const uint8_t* p = img + (size_t)blockIdx.y * npx * 3;
  long long s[6] = {0, 0, 0, 0, 0, 0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = p[i * 3], g = p[i * 3 + 1], r = p[i * 3 + 2];
    const int d[3] = {b - g, g - r, r - b};
#pragma unroll
    for (int k = 0; k < 3; ++k) { s[k] += d[k]; s[3 + k] += d[k] * d[k]; }
  }
#pragma unroll
  for (int k = 0; k < 6; ++k)
    for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
  __shared__ long long red[8][6];
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < 6; ++k) red[warp][k] = s[k];
  __syncthreads();
  if (threadIdx.x < 6) {
    long long t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w][threadIdx.x];
    atomicAdd(sums + (size_t)blockIdx.y * 6 + threadIdx.x, (unsigned long long)t);   // two's complement: signed sums too
  }
}

// the parse network's input of a float64 face: astype(float32) / 255, BGR -> RGB, (x - 0.5) / 0.5, HWC -> NCHW
__global__ void k_f64_to_input(const double* __restrict__ img, float* __restrict__ x, int64_t hw, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t n = i / (3 * hw), r = i - n * 3 * hw;
  const int c = (int)(r / hw);
  const int64_t px = r - (int64_t)c * hw;
  const float t = __fdiv_rn(__double2float_rn(img[(n * hw + px) * 3 + (2 - c)]), 255.f);
  x[i] = __fdiv_rn(__fsub_rn(t, 0.5f), 0.5f);
}

}  // namespace
}  // namespace cfb

#define API_BEGIN try {
#define API_END(ret)                                                                                        \
  } catch (const std::exception& e) { cfb::set_error(std::string("exception: ") + e.what()); return ret; } \
  catch (...) { cfb::set_error("unknown exception"); return ret; }

extern "C" {

int cfb_warp_affine_u8(const uint8_t* img, int32_t h, int32_t w, const double* affines, int32_t n, uint8_t* out,
                       int32_t out_h, int32_t out_w, int32_t border_mode, int32_t v0, int32_t v1, int32_t v2, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "cfb_warp_affine_u8: bad size");
  CFB_REQUIRE(n == 0 || (img && affines && out), "cfb_warp_affine_u8: NULL argument");
  CFB_REQUIRE(border_mode == 0 || border_mode == 2 || border_mode == 4, "cfb_warp_affine_u8: border mode must be 0 (constant), 2 (reflect) or 4 (reflect-101)");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<double> maps(6 * (size_t)n);
  for (int i = 0; i < n; ++i) cfb::invert_affine(affines + 6 * i, maps.data() + 6 * i);
  double* dmaps = nullptr;
  CFB_CUDA(cudaMallocAsync((void**)&dmaps, maps.size() * 8, st));
  CFB_CUDA(cudaMemcpyAsync(dmaps, maps.data(), maps.size() * 8, cudaMemcpyHostToDevice, st));
  const dim3 b(32, 8);
  cfb::k_warp_crop<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(img, h, w, dmaps, n, out, out_h, out_w, border_mode, v0, v1, v2);
  CFB_LAUNCH_CHECK();
  CFB_CUDA(cudaFreeAsync(dmaps, st));
  return 0;
  API_END(1)
}

int cfb_resize_linear_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "cfb_resize_linear_u8: bad size");
  CFB_REQUIRE(n == 0 || (src && dst), "cfb_resize_linear_u8: NULL argument");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (h == out_h && w == out_w) {                  // cv2.resize to the same size is a copy
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * h * w * 3, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  const dim3 b(32, 8);
  cfb::k_resize_u8<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(src, h, w, dst, out_h, out_w, 1. / ((double)out_w / w),
                                                                  1. / ((double)out_h / h), n);
  CFB_LAUNCH_CHECK();
  return 0;
  API_END(1)
}

int cfb_resize_area_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "cfb_resize_area_u8: bad size");
  CFB_REQUIRE(out_h <= h && out_w <= w, "cfb_resize_area_u8: shrinking only (use cfb_resize_linear_u8 to enlarge)");
  CFB_REQUIRE(n == 0 || (src && dst), "cfb_resize_area_u8: NULL argument");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (h == out_h && w == out_w) {                  // cv2.resize to the same size is a copy
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * h * w * 3, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  const double scale_x = 1. / ((double)out_w / w), scale_y = 1. / ((double)out_h / h);
  const int isx = (int)std::nearbyint(scale_x), isy = (int)std::nearbyint(scale_y);
  const dim3 b(32, 8);
  if (std::abs(scale_x - isx) < 2.220446049250313e-16 && std::abs(scale_y - isy) < 2.220446049250313e-16) {
    cfb::k_resize_area_fast_u8<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(src, h, w, dst, out_h, out_w, isx, isy,
                                                                             1.f / (float)(isx * isy), n);
    CFB_LAUNCH_CHECK();
    return 0;
  }
  std::vector<int> xi, yi;
  std::vector<float> xa, ya;
  const int kx = cfb::area_taps(w, out_w, scale_x, xi, xa), ky = cfb::area_taps(h, out_h, scale_y, yi, ya);
  const size_t nx = xi.size(), ny = yi.size();
  std::vector<char> host((nx + ny) * 8);
  memcpy(host.data(), xi.data(), nx * 4);
  memcpy(host.data() + nx * 4, xa.data(), nx * 4);
  memcpy(host.data() + nx * 8, yi.data(), ny * 4);
  memcpy(host.data() + nx * 8 + ny * 4, ya.data(), ny * 4);
  char* dtab = nullptr;
  CFB_CUDA(cudaMallocAsync((void**)&dtab, host.size(), st));
  CFB_CUDA(cudaMemcpyAsync(dtab, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  cfb::k_resize_area_u8<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(
      src, h, w, dst, out_h, out_w, (const int*)dtab, (const float*)(dtab + nx * 4), kx, (const int*)(dtab + nx * 8),
      (const float*)(dtab + nx * 8 + ny * 4), ky, n);
  CFB_LAUNCH_CHECK();
  CFB_CUDA(cudaFreeAsync(dtab, st));
  return 0;
  API_END(1)
}

int cfb_resize_linear_scale_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w,
                               double fx, double fy, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "cfb_resize_linear_scale_u8: bad size");
  CFB_REQUIRE(fx >= 1. && fy >= 1., "cfb_resize_linear_scale_u8: enlarging factors (>= 1) only");
  CFB_REQUIRE(n == 0 || (src && dst), "cfb_resize_linear_scale_u8: NULL argument");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (h == out_h && w == out_w && fx == 1. && fy == 1.) {
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)n * h * w * 3, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  const dim3 b(32, 8);
  cfb::k_resize_u8<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(src, h, w, dst, out_h, out_w, 1. / fx, 1. / fy, n);
  CFB_LAUNCH_CHECK();
  return 0;
  API_END(1)
}

int cfb_warp_affine_multi_u8(const uint8_t* imgs, int32_t n_img, int32_t h, int32_t w, const double* affines,
                             const int32_t* img_index, int32_t n, uint8_t* out, int32_t out_h, int32_t out_w,
                             int32_t border_mode, int32_t v0, int32_t v1, int32_t v2, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && n_img > 0 && h > 0 && w > 0 && out_h > 0 && out_w > 0, "cfb_warp_affine_multi_u8: bad size");
  CFB_REQUIRE(n == 0 || (imgs && affines && img_index && out), "cfb_warp_affine_multi_u8: NULL argument");
  CFB_REQUIRE(border_mode == 0 || border_mode == 2 || border_mode == 4, "cfb_warp_affine_multi_u8: border mode must be 0 (constant), 2 (reflect) or 4 (reflect-101)");
  if (n == 0) return 0;
  for (int i = 0; i < n; ++i)
    CFB_REQUIRE(img_index[i] >= 0 && img_index[i] < n_img, "cfb_warp_affine_multi_u8: image index out of range");
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<char> host((size_t)n * (6 * 8 + 4));
  double* maps = (double*)host.data();
  for (int i = 0; i < n; ++i) cfb::invert_affine(affines + 6 * i, maps + 6 * i);
  memcpy(host.data() + (size_t)n * 48, img_index, (size_t)n * 4);
  char* d = nullptr;
  CFB_CUDA(cudaMallocAsync((void**)&d, host.size(), st));
  CFB_CUDA(cudaMemcpyAsync(d, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  const dim3 b(32, 8);
  cfb::k_warp_crop_multi<<<cfb::grid2(out_w, out_h, n, b), b, 0, st>>>(imgs, h, w, (const double*)d, (const int*)(d + (size_t)n * 48),
                                                                        n, out, out_h, out_w, border_mode, v0, v1, v2);
  CFB_LAUNCH_CHECK();
  CFB_CUDA(cudaFreeAsync(d, st));
  return 0;
  API_END(1)
}

int64_t cfb_paste_faces_multi_workspace_bytes(int32_t n_img, int32_t h_up, int32_t w_up, int32_t n, int32_t face_size,
                                              int32_t use_parse, const double* inverse_affines) {
  if (n_img <= 0 || h_up <= 0 || w_up <= 0 || n < 0 || face_size <= 0 || (n > 0 && !inverse_affines)) {
    cfb::set_error("cfb_paste_faces_multi_workspace_bytes: bad argument");
    return -1;
  }
  cfb::Plan P;
  cfb::make_plan(h_up, w_up, n, face_size, inverse_affines, P);
  return (int64_t)cfb::layout(h_up, w_up, n, face_size, use_parse != 0, P, cfb::max_gauss_floats(P), n_img).total;
}

int cfb_paste_faces_multi(uint8_t* canvases, int32_t n_img, int32_t h_up, int32_t w_up, const uint8_t* faces, int32_t n,
                          int32_t face_size, const uint8_t* parse_masks, const double* inverse_affines, const int32_t* img_index,
                          double upscale, int32_t* w_edge_out, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n_img > 0 && h_up > 0 && w_up > 0 && n >= 0 && face_size > 0 && upscale > 0, "cfb_paste_faces_multi: bad size");
  CFB_REQUIRE(canvases && workspace && (n == 0 || (faces && inverse_affines && img_index)), "cfb_paste_faces_multi: NULL argument");
  for (int i = 0; i < n; ++i)
    CFB_REQUIRE(img_index[i] >= 0 && img_index[i] < n_img, "cfb_paste_faces_multi: image index out of range");
  const int64_t need = cfb_paste_faces_multi_workspace_bytes(n_img, h_up, w_up, n, face_size, parse_masks != nullptr, inverse_affines);
  CFB_REQUIRE(need > 0 && workspace_bytes >= need, "cfb_paste_faces_multi: workspace too small (cfb_paste_faces_multi_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  if (parse_masks)
    return cfb::paste_impl<double>(canvases, n_img, img_index, h_up, w_up, faces, n, face_size, parse_masks, inverse_affines,
                                   upscale, nullptr, w_edge_out, (char*)workspace, workspace_bytes, st);
  return cfb::paste_impl<float>(canvases, n_img, img_index, h_up, w_up, faces, n, face_size, nullptr, inverse_affines, upscale,
                                nullptr, w_edge_out, (char*)workspace, workspace_bytes, st);
  API_END(1)
}

int64_t cfb_paste_faces_workspace_bytes(int32_t h_up, int32_t w_up, int32_t n, int32_t face_size, int32_t use_parse,
                                        const double* inverse_affines) {
  if (h_up <= 0 || w_up <= 0 || n < 0 || face_size <= 0 || (n > 0 && !inverse_affines)) {
    cfb::set_error("cfb_paste_faces_workspace_bytes: bad argument");
    return -1;
  }
  cfb::Plan P;
  cfb::make_plan(h_up, w_up, n, face_size, inverse_affines, P);
  const cfb::Layout L = cfb::layout(h_up, w_up, n, face_size, use_parse != 0, P, cfb::max_gauss_floats(P));
  return (int64_t)L.total;
}

int cfb_paste_faces(uint8_t* canvas, int32_t h_up, int32_t w_up, const uint8_t* faces, int32_t n, int32_t face_size,
                    const uint8_t* parse_masks, const double* inverse_affines, double upscale, float* debug_canvas,
                    int32_t* w_edge_out, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(h_up > 0 && w_up > 0 && n >= 0 && face_size > 0 && upscale > 0, "cfb_paste_faces: bad size");
  CFB_REQUIRE(canvas && workspace && (n == 0 || (faces && inverse_affines)), "cfb_paste_faces: NULL argument");
  const int64_t need = cfb_paste_faces_workspace_bytes(h_up, w_up, n, face_size, parse_masks != nullptr, inverse_affines);
  CFB_REQUIRE(need > 0 && workspace_bytes >= need, "cfb_paste_faces: workspace too small (cfb_paste_faces_workspace_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  if (parse_masks)
    return cfb::paste_impl<double>(canvas, 1, nullptr, h_up, w_up, faces, n, face_size, parse_masks, inverse_affines, upscale,
                                   debug_canvas, w_edge_out, (char*)workspace, workspace_bytes, st);
  return cfb::paste_impl<float>(canvas, 1, nullptr, h_up, w_up, faces, n, face_size, nullptr, inverse_affines, upscale,
                                debug_canvas, w_edge_out, (char*)workspace, workspace_bytes, st);
  API_END(1)
}


void cfb_lanczos4_table(int32_t src_len, int32_t dst_len, int32_t* idx, int16_t* coef) {
  if (src_len > 0 && dst_len > 0 && idx && coef) cfb::lanczos4_table(src_len, dst_len, idx, coef);
}

int cfb_resize_lanczos4_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w, void* stream) {
  API_BEGIN
  return cfb::resize_lanczos4<uint8_t, int16_t>(src, n, h, w, dst, out_h, out_w, cfb::lanczos4_table, "cfb_resize_lanczos4_u8",
                                                (cudaStream_t)stream);
  API_END(1)
}

void cfb_lanczos4_table_f32(int32_t src_len, int32_t dst_len, int32_t* idx, float* coef) {
  if (src_len > 0 && dst_len > 0 && idx && coef) cfb::lanczos4_table_f32(src_len, dst_len, idx, coef);
}

int cfb_resize_lanczos4_u16(const uint16_t* src, int32_t n, int32_t h, int32_t w, uint16_t* dst, int32_t out_h, int32_t out_w,
                            void* stream) {
  API_BEGIN
  return cfb::resize_lanczos4<uint16_t, float>(src, n, h, w, dst, out_h, out_w, cfb::lanczos4_table_f32, "cfb_resize_lanczos4_u16",
                                               (cudaStream_t)stream);
  API_END(1)
}

int cfb_gray_adain_faces(const uint8_t* restored, const uint8_t* cropped, int32_t n, int32_t face_size, double* out, double* stats,
                         void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && face_size > 0 && face_size <= 8192, "cfb_gray_adain_faces: bad size");
  CFB_REQUIRE(n <= 65535, "cfb_gray_adain_faces: at most 65535 faces per call");
  CFB_REQUIRE(n == 0 || (restored && cropped && out), "cfb_gray_adain_faces: NULL argument");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int npx = face_size * face_size;
  double* tmp = nullptr;                           // partial[n][slices][4], then stats[n][12] when the caller wants none
  const size_t np = (size_t)n * cfb::kGraySlices * 4;
  CFB_CUDA(cudaMallocAsync((void**)&tmp, (np + (size_t)n * 12) * 8, st));
  double* dstats = stats ? stats : tmp + np;
  const dim3 g(cfb::kGraySlices, n);
  for (int pass = 0; pass < 2; ++pass) {           // means first, then the squared deviations from them
    cfb::k_gray_partial<<<g, 256, 0, st>>>(restored, cropped, npx, pass ? dstats : nullptr, tmp);
    CFB_LAUNCH_CHECK();
    cfb::k_gray_stats<<<n, 32, 0, st>>>(tmp, cfb::kGraySlices, npx, pass, dstats);
    CFB_LAUNCH_CHECK();
  }
  cfb::k_gray_apply<<<dim3((npx + 255) / 256, n), 256, 0, st>>>(restored, npx, dstats, out);
  CFB_LAUNCH_CHECK();
  CFB_CUDA(cudaFreeAsync(tmp, st));
  return 0;
  API_END(1)
}

int cfb_is_gray_u8(const uint8_t* images, int32_t n, int32_t h, int32_t w, int64_t* sums, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && n <= 65535 && h > 0 && w > 0, "cfb_is_gray_u8: bad size");
  CFB_REQUIRE(n == 0 || (images && sums), "cfb_is_gray_u8: NULL argument");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t npx = (int64_t)h * w;
  const int64_t want = (npx + 2047) / 2048;        // at least 8 pixels per thread
  const int bx = (int)std::max<int64_t>(1, std::min<int64_t>(want, std::max(1, cfb::kGrayTestBlocks / n)));
  CFB_CUDA(cudaMemsetAsync(sums, 0, (size_t)n * 6 * sizeof(int64_t), st));
  cfb::k_is_gray_sums<<<dim3(bx, n), 256, 0, st>>>(images, npx, reinterpret_cast<unsigned long long*>(sums));
  CFB_LAUNCH_CHECK();
  return 0;
  API_END(1)
}

int cfb_f64_to_input(const double* img_bgr_hwc, float* x_nchw, int32_t n, int32_t hw, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n >= 0 && hw > 0, "cfb_f64_to_input: bad size");
  CFB_REQUIRE(n == 0 || (img_bgr_hwc && x_nchw), "cfb_f64_to_input: NULL argument");
  const int64_t total = (int64_t)n * 3 * hw;
  if (total == 0) return 0;
  cfb::k_f64_to_input<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img_bgr_hwc, x_nchw, hw, total);
  CFB_LAUNCH_CHECK();
  return 0;
  API_END(1)
}

int64_t cfb_paste_faces_f64_workspace_bytes(int32_t n_img, int32_t h_up, int32_t w_up, int32_t n, int32_t face_size,
                                            int32_t use_parse, const double* inverse_affines) {
  if (n_img <= 0 || h_up <= 0 || w_up <= 0 || n < 0 || face_size <= 0 || (n > 0 && !inverse_affines)) {
    cfb::set_error("cfb_paste_faces_f64_workspace_bytes: bad argument");
    return -1;
  }
  cfb::Plan P;
  cfb::make_plan(h_up, w_up, n, face_size, inverse_affines, P);
  return (int64_t)cfb::layout(h_up, w_up, n, face_size, use_parse != 0, P, cfb::max_gauss_floats(P), n_img, true).total;
}

int cfb_paste_faces_f64(uint8_t* canvases, int32_t n_img, int32_t h_up, int32_t w_up, const double* faces, int32_t n,
                        int32_t face_size, const uint8_t* parse_masks, const double* inverse_affines, const int32_t* img_index,
                        double upscale, uint16_t* canvases_u16, int32_t* wide_out, int32_t* w_edge_out, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n_img > 0 && n_img <= 65535 && h_up > 0 && w_up > 0 && n >= 0 && face_size > 0 && upscale > 0, "cfb_paste_faces_f64: bad size");
  CFB_REQUIRE(canvases && workspace && (n == 0 || (faces && inverse_affines && img_index)), "cfb_paste_faces_f64: NULL argument");
  CFB_REQUIRE(!canvases_u16 || wide_out, "cfb_paste_faces_f64: canvases_u16 needs wide_out");
  for (int i = 0; i < n; ++i)
    CFB_REQUIRE(img_index[i] >= 0 && img_index[i] < n_img, "cfb_paste_faces_f64: image index out of range");
  const int64_t need = cfb_paste_faces_f64_workspace_bytes(n_img, h_up, w_up, n, face_size, parse_masks != nullptr, inverse_affines);
  CFB_REQUIRE(need > 0 && workspace_bytes >= need, "cfb_paste_faces_f64: workspace too small (cfb_paste_faces_f64_workspace_bytes)");
  return cfb::paste_impl<double, double>(canvases, n_img, img_index, h_up, w_up, faces, n, face_size, parse_masks,
                                         inverse_affines, upscale, nullptr, w_edge_out, (char*)workspace, workspace_bytes,
                                         (cudaStream_t)stream, canvases_u16, wide_out);
  API_END(1)
}

}  // extern "C"
