// Synthetic degradations (cfb_degrade_faces): the blur -> downsample -> noise -> JPEG -> resize chain of FFHQBlindDataset
// (basicsr/data/ffhq_blind_dataset.py:210-240) for a batch of uint8 BGR faces of one size, each with its own kernel, small
// size, noise and quality.  One launch per stage for the whole batch, no host synchronisation:
//   blur     per face, the 2-D correlation (BORDER_REFLECT_101; float64 products added in kernel-row, then kernel-column
//            order without contraction, so a test can repeat the sum bit for bit; one float32 rounding) evaluated only at the
//            source rows and columns the INTER_LINEAR downsample reads -- 2 s of them per axis, or all S when 2 s >= S
//   small    the float32 INTER_LINEAR lerps (cv2's arithmetic: float64 coordinates, fma(b - a, t, a), rows first), noise,
//            clip to [0, 1], and for JPEG faces saturate_cast<uchar>(x * 255) (round half to even)
//   jpeg     libjpeg-turbo's baseline 4:2:0 round trip without a bitstream: per 8 x 8 block the colour conversion, h2v2
//            downsampling, islow FDCT, quantisation, dequantisation and islow IDCT; then per pixel the upsampling (fancy,
//            which reads chroma across MCU boundaries, so it is a second kernel; replication for chroma planes at most 2
//            samples wide) and YCbCr -> BGR
//   final    /255, INTER_LINEAR to in_size, * 255, round half to even, clip -> uint8
// cfb_jpeg_roundtrip runs the JPEG stage alone on equal-size images.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "kernels.cuh"

namespace cfb {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxKsize = 63;

struct DegFace {
  int s;            // small size int(S // scale)
  int n;            // side of the blur grid: S (every source pixel) or 2 s (the taps the downsample reads)
  int q;            // JPEG quality, 0 = no JPEG
  int pad;
  int64_t noise;    // offset of the face's noise field in floats, -1 = no noise
  int64_t grid;     // offset of the blur grid [n][n][3] in floats
  int64_t img;      // offset of the small image [s][s][3] in elements
  int64_t fstate;   // offset of the face's float result [in][in][3] for the colour stages, -1 = round to lq here
};

struct JpgImg {
  int h, w, q, pad;
  int64_t src, dst;          // byte offsets of the HWC BGR images
  int64_t ypl, cpl;          // byte offsets of the decoded Y plane and the two chroma planes
};

// ---------------------------------------------------------------------------------------------------- INTER_LINEAR taps
// cv2's float resize: source coordinate fma(d + 0.5, src / dst, -0.5) in double, i = floor, t = the rest as float; taps
// clamped to the image
__device__ __forceinline__ void lin_tap(int d, int src, int dst, int& i0, int& i1, float& t) {
  const double f = fma(d + 0.5, (double)src / dst, -0.5), fl = floor(f);
  const int i = (int)fl;
  t = __double2float_rn(f - fl);
  i0 = min(max(i, 0), src - 1);
  i1 = min(max(i + 1, 0), src - 1);
}

__device__ __forceinline__ float lerp(float a, float b, float t) { return __fmaf_rn(__fsub_rn(b, a), t, a); }

// saturate_cast<uchar>(float): round half to even, clamp
__device__ __forceinline__ uint8_t sat_u8(float v) { return (uint8_t)min(max(__float2int_rn(v), 0), 255); }

__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * (n - 1) - p;
  return p;
}

// blur-grid index j -> source coordinate
__device__ __forceinline__ int grid_pos(int j, const DegFace& f, int S) {
  if (f.n == S) return j;
  int i0, i1;
  float t;
  lin_tap(j >> 1, S, f.s, i0, i1, t);
  return (j & 1) ? i1 : i0;
}

// ---------------------------------------------------------------------------------------------------------------- blur
__global__ void __launch_bounds__(kThreads) blur_grid_kernel(const uint8_t* __restrict__ gt, int S, const DegFace* __restrict__ faces,
                                                             const double* __restrict__ kernels, int ks, float* __restrict__ grid) {
  extern __shared__ double sk[];
  __shared__ double lut[256];
  const int b = blockIdx.y;
  const DegFace f = faces[b];
  for (int i = threadIdx.x; i < ks * ks; i += blockDim.x) sk[i] = kernels[(int64_t)b * ks * ks + i];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = (double)__fdiv_rn((float)i, 255.f);   // img.astype(f32) / 255.
  __syncthreads();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)f.n * f.n) return;
  const int jy = (int)(idx / f.n), jx = (int)(idx % f.n);
  const int py = grid_pos(jy, f, S), px = grid_pos(jx, f, S), r = ks / 2;
  const uint8_t* img = gt + (int64_t)b * S * S * 3;
  double a0 = 0., a1 = 0., a2 = 0.;
  const bool inner_x = px - r >= 0 && px + r < S;
  for (int ky = 0; ky < ks; ++ky) {
    const uint8_t* row = img + (int64_t)reflect101(py + ky - r, S) * S * 3;
    const double* kr = sk + ky * ks;
    if (inner_x) {
      const uint8_t* p = row + (px - r) * 3;
      for (int kx = 0; kx < ks; ++kx, p += 3) {
        const double w = kr[kx];
        a0 = __dadd_rn(a0, __dmul_rn(w, lut[p[0]]));
        a1 = __dadd_rn(a1, __dmul_rn(w, lut[p[1]]));
        a2 = __dadd_rn(a2, __dmul_rn(w, lut[p[2]]));
      }
    } else {
      for (int kx = 0; kx < ks; ++kx) {
        const uint8_t* p = row + reflect101(px + kx - r, S) * 3;
        const double w = kr[kx];
        a0 = __dadd_rn(a0, __dmul_rn(w, lut[p[0]]));
        a1 = __dadd_rn(a1, __dmul_rn(w, lut[p[1]]));
        a2 = __dadd_rn(a2, __dmul_rn(w, lut[p[2]]));
      }
    }
  }
  float* o = grid + f.grid + idx * 3;
  o[0] = __double2float_rn(a0);
  o[1] = __double2float_rn(a1);
  o[2] = __double2float_rn(a2);
}

// ------------------------------------------------------------------------------------------- downsample, noise, uint8
__global__ void __launch_bounds__(kThreads) small_kernel(int S, const DegFace* __restrict__ faces, const float* __restrict__ grid,
                                                         const float* __restrict__ noise, float* __restrict__ fimg,
                                                         uint8_t* __restrict__ uimg, float* __restrict__ cap_a,
                                                         uint8_t* __restrict__ cap_u8) {
  const DegFace f = faces[blockIdx.y];
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)f.s * f.s) return;
  const int oy = (int)(idx / f.s), ox = (int)(idx % f.s);
  int y0, y1, x0, x1;
  float ty, tx;
  lin_tap(oy, S, f.s, y0, y1, ty);
  lin_tap(ox, S, f.s, x0, x1, tx);
  if (f.n != S) {            // sampled grid: row 2 oy holds tap y0, 2 oy + 1 tap y1
    y0 = 2 * oy, y1 = 2 * oy + 1, x0 = 2 * ox, x1 = 2 * ox + 1;
  }
  const float* g = grid + f.grid;
  const int64_t o = f.img + idx * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float h0 = lerp(g[((int64_t)y0 * f.n + x0) * 3 + c], g[((int64_t)y0 * f.n + x1) * 3 + c], tx);
    const float h1 = lerp(g[((int64_t)y1 * f.n + x0) * 3 + c], g[((int64_t)y1 * f.n + x1) * 3 + c], tx);
    float v = lerp(h0, h1, ty);
    if (cap_a) cap_a[o + c] = v;
    if (f.noise >= 0) v = fminf(fmaxf(__fadd_rn(v, noise[f.noise + idx * 3 + c]), 0.f), 1.f);
    fimg[o + c] = v;
    if (f.q > 0) {
      const uint8_t u = sat_u8(__fmul_rn(v, 255.f));
      uimg[o + c] = u;
      if (cap_u8) cap_u8[o + c] = u;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------- JPEG
__constant__ uint8_t kStdLuma[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                     14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                     18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
__constant__ uint8_t kStdChroma[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                       99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                       99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

// libjpeg fixed point (SCALEBITS 16): FIX(x) = (int)(x * 65536 + 0.5)
constexpr int kFix0299 = 19595, kFix0587 = 38470, kFix0114 = 7471, kFix016874 = 11059, kFix033126 = 21709,
              kFix05 = 32768, kFix041869 = 27439, kFix008131 = 5329, kFix1402 = 91881, kFix034414 = 22554,
              kFix071414 = 46802, kFix1772 = 116130;
constexpr int kHalf = 1 << 15, kCbCrOff = 128 << 16;
// islow DCT constants (CONST_BITS 13)
constexpr int c298 = 2446, c390 = 3196, c541 = 4433, c765 = 6270, c899 = 7373, c1175 = 9633, c1501 = 12299, c1847 = 15137,
              c1961 = 16069, c2053 = 16819, c2562 = 20995, c3072 = 25172;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__device__ __forceinline__ int y_of(int b, int g, int r) { return (kFix0299 * r + kFix0587 * g + kFix0114 * b + kHalf) >> 16; }
__device__ __forceinline__ int cb_of(int b, int g, int r) {
  return (-kFix016874 * r - kFix033126 * g + kFix05 * b + kCbCrOff + kHalf - 1) >> 16;
}
__device__ __forceinline__ int cr_of(int b, int g, int r) {
  return (kFix05 * r - kFix041869 * g - kFix008131 * b + kCbCrOff + kHalf - 1) >> 16;
}

// jfdctint: one 1-D pass over d[0], d[st], ..., d[7 st]
template <bool kPass1>
__device__ __forceinline__ void fdct_1d(int* d, int st) {
  const int t0 = d[0] + d[7 * st], t7 = d[0] - d[7 * st], t1 = d[st] + d[6 * st], t6 = d[st] - d[6 * st];
  const int t2 = d[2 * st] + d[5 * st], t5 = d[2 * st] - d[5 * st], t3 = d[3 * st] + d[4 * st], t4 = d[3 * st] - d[4 * st];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  constexpr int sh = kPass1 ? 13 - 2 : 13 + 2;
  d[0] = kPass1 ? (t10 + t11) * 4 : descale(t10 + t11, 2);
  d[4 * st] = kPass1 ? (t10 - t11) * 4 : descale(t10 - t11, 2);
  int z1 = (t12 + t13) * c541;
  d[2 * st] = descale(z1 + t13 * c765, sh);
  d[6 * st] = descale(z1 - t12 * c1847, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * c1175;
  z1 *= -c899;
  z2 *= -c2562;
  z3 = z3 * -c1961 + z5;
  z4 = z4 * -c390 + z5;
  d[7 * st] = descale(t4 * c298 + z1 + z3, sh);
  d[5 * st] = descale(t5 * c2053 + z2 + z4, sh);
  d[3 * st] = descale(t6 * c3072 + z2 + z3, sh);
  d[st] = descale(t7 * c1501 + z1 + z4, sh);
}

// jidctint: one 1-D pass (input dequantised)
template <bool kPass1>
__device__ __forceinline__ void idct_1d(int* d, int st) {
  int z2 = d[2 * st], z3 = d[6 * st];
  int z1 = (z2 + z3) * c541;
  const int t2e = z1 - z3 * c1847, t3e = z1 + z2 * c765;
  const int t0e = (d[0] + d[4 * st]) * 8192, t1e = (d[0] - d[4 * st]) * 8192;
  const int t10 = t0e + t3e, t13 = t0e - t3e, t11 = t1e + t2e, t12 = t1e - t2e;
  int t0 = d[7 * st], t1 = d[5 * st], t2 = d[3 * st], t3 = d[st];
  z1 = t0 + t3;
  z2 = t1 + t2;
  z3 = t0 + t2;
  int z4 = t1 + t3;
  const int z5 = (z3 + z4) * c1175;
  z1 *= -c899;
  z2 *= -c2562;
  z3 = z3 * -c1961 + z5;
  z4 = z4 * -c390 + z5;
  t0 = t0 * c298 + z1 + z3;
  t1 = t1 * c2053 + z2 + z4;
  t2 = t2 * c3072 + z2 + z3;
  t3 = t3 * c1501 + z1 + z4;
  constexpr int sh = kPass1 ? 13 - 2 : 13 + 2 + 3;
  d[0] = descale(t10 + t3, sh);
  d[7 * st] = descale(t10 - t3, sh);
  d[st] = descale(t11 + t2, sh);
  d[6 * st] = descale(t11 - t2, sh);
  d[2 * st] = descale(t12 + t1, sh);
  d[5 * st] = descale(t12 - t1, sh);
  d[3 * st] = descale(t13 + t0, sh);
  d[4 * st] = descale(t13 - t0, sh);
}

// jpeg_set_quality(q, force_baseline) entry k of a table, then libjpeg-turbo's quantisation of x by the reciprocal of
// 8 * quantval (compute_reciprocal: ((|x| + corr) * recip) >> shift) and the decoder's dequantisation
__device__ __forceinline__ int quant_dequant(int x, int basic, int q) {
  const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
  const int qv = min(max((basic * scale + 50) / 100, 1), 255);
  const unsigned div = (unsigned)qv * 8u;
  int r = 16 + (31 - __clz(div));
  unsigned long long fq = (1ull << r) / div;
  const unsigned long long fr = (1ull << r) % div;
  unsigned c = div / 2;
  if (fr == 0) {
    fq >>= 1;
    --r;
  } else if (fr <= div / 2) {
    ++c;
  } else {
    ++fq;
  }
  const int v = (int)((((unsigned long long)(x < 0 ? -x : x) + c) * fq) >> r);
  return (x < 0 ? -v : v) * qv;
}

__device__ __forceinline__ int3 load_bgr(const uint8_t* img, int w, int y, int x) {
  const uint8_t* p = img + ((int64_t)y * w + x) * 3;
  return make_int3(p[0], p[1], p[2]);
}

// one thread per 8 x 8 block of one component: Y blocks first, then Cb, then Cr
__global__ void __launch_bounds__(128) jpeg_block_kernel(const JpgImg* __restrict__ imgs, const uint8_t* __restrict__ src_base,
                                                         uint8_t* __restrict__ plane_base) {
  const JpgImg J = imgs[blockIdx.y];
  const int ybw = (J.w + 7) / 8, ybh = (J.h + 7) / 8, cbw = (J.w + 15) / 16, cbh = (J.h + 15) / 16;
  const int nyb = ybw * ybh, ncb = cbw * cbh;
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= nyb + 2 * ncb) return;
  const uint8_t* src = src_base + J.src;
  int d[64];
  const bool luma = id < nyb;
  const int comp = luma ? 0 : 1 + (id - nyb) / ncb;
  const int bid = luma ? id : (id - nyb) % ncb;
  const int bw = luma ? ybw : cbw;
  const int by = bid / bw, bx = bid % bw;
  if (luma) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int3 p = load_bgr(src, J.w, min(by * 8 + i, J.h - 1), min(bx * 8 + j, J.w - 1));
        d[i * 8 + j] = y_of(p.x, p.y, p.z) - 128;
      }
  } else {
    const int rh = (J.h + 1) / 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int cy = min(by * 8 + i, rh - 1);             // padded chroma rows repeat the last real one
      const int r0 = min(2 * cy, J.h - 1), r1 = min(2 * cy + 1, J.h - 1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cx = bx * 8 + j;
        const int c0 = min(2 * cx, J.w - 1), c1 = min(2 * cx + 1, J.w - 1);
        const int3 p00 = load_bgr(src, J.w, r0, c0), p01 = load_bgr(src, J.w, r0, c1), p10 = load_bgr(src, J.w, r1, c0),
                   p11 = load_bgr(src, J.w, r1, c1);
        int s;
        if (comp == 1)
          s = cb_of(p00.x, p00.y, p00.z) + cb_of(p01.x, p01.y, p01.z) + cb_of(p10.x, p10.y, p10.z) + cb_of(p11.x, p11.y, p11.z);
        else
          s = cr_of(p00.x, p00.y, p00.z) + cr_of(p01.x, p01.y, p01.z) + cr_of(p10.x, p10.y, p10.z) + cr_of(p11.x, p11.y, p11.z);
        d[i * 8 + j] = ((s + 1 + (j & 1)) >> 2) - 128;          // bias 1, 2, 1, 2, ... along the row (cx parity = j parity)
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) fdct_1d<true>(d + i * 8, 1);
#pragma unroll
  for (int j = 0; j < 8; ++j) fdct_1d<false>(d + j, 8);
  const uint8_t* basic = luma ? kStdLuma : kStdChroma;
#pragma unroll
  for (int k = 0; k < 64; ++k) d[k] = quant_dequant(d[k], basic[k], J.q);
#pragma unroll
  for (int j = 0; j < 8; ++j) idct_1d<true>(d + j, 8);
#pragma unroll
  for (int i = 0; i < 8; ++i) idct_1d<false>(d + i * 8, 1);
  const int stride = luma ? ybw * 8 : cbw * 8;
  uint8_t* out = plane_base + (luma ? J.ypl : J.cpl + (int64_t)(comp - 1) * cbw * 8 * cbh * 8);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      out[(int64_t)(by * 8 + i) * stride + bx * 8 + j] = (uint8_t)min(max(d[i * 8 + j] + 128, 0), 255);
}

// the decoder's h2v2 fancy upsampling (triangle filter, biases 8 / 7, edges replicated; plain replication when the chroma
// plane is at most 2 samples wide, as libjpeg-turbo's jinit_upsampler chooses) and YCbCr -> BGR
__global__ void __launch_bounds__(kThreads) jpeg_color_kernel(const JpgImg* __restrict__ imgs, const uint8_t* __restrict__ plane_base,
                                                              uint8_t* __restrict__ dst_base) {
  const JpgImg J = imgs[blockIdx.y];
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)J.h * J.w) return;
  const int y = (int)(idx / J.w), x = (int)(idx % J.w);
  const int ybw = (J.w + 7) / 8, cbw = (J.w + 15) / 16, cbh = (J.h + 15) / 16;
  const int cstride = cbw * 8, rh = (J.h + 1) / 2, rw = (J.w + 1) / 2;
  const int cy = y >> 1, cx = x >> 1;
  const int cyn = (y & 1) ? min(cy + 1, rh - 1) : max(cy - 1, 0);
  const int cxn = (x & 1) ? min(cx + 1, rw - 1) : max(cx - 1, 0);
  const int bias = (x & 1) ? 7 : 8;
  int ch[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const uint8_t* p = plane_base + J.cpl + (int64_t)c * cstride * cbh * 8;
    if (rw <= 2) {           // libjpeg-turbo replicates unless the chroma plane is wider than 2 samples
      ch[c] = p[cy * cstride + cx] - 128;
      continue;
    }
    const int near = 3 * p[cy * cstride + cx] + p[cyn * cstride + cx];
    const int far = 3 * p[cy * cstride + cxn] + p[cyn * cstride + cxn];
    ch[c] = ((3 * near + far + bias) >> 4) - 128;
  }
  const int Y = plane_base[J.ypl + (int64_t)y * ybw * 8 + x];
  const int cb = ch[0], cr = ch[1];
  uint8_t* o = dst_base + J.dst + idx * 3;
  o[0] = (uint8_t)min(max(Y + ((kFix1772 * cb + kHalf) >> 16), 0), 255);
  o[1] = (uint8_t)min(max(Y + ((-kFix034414 * cb + kHalf - kFix071414 * cr) >> 16), 0), 255);
  o[2] = (uint8_t)min(max(Y + ((kFix1402 * cr + kHalf) >> 16), 0), 255);
}

// --------------------------------------------------------------------------------------------------- final resize
__global__ void __launch_bounds__(kThreads) final_kernel(const DegFace* __restrict__ faces, const float* __restrict__ fimg,
                                                         const uint8_t* __restrict__ dimg, int in_size, uint8_t* __restrict__ lq,
                                                         float* __restrict__ fstate) {
  const int b = blockIdx.y;
  const DegFace f = faces[b];
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)in_size * in_size) return;
  const int oy = (int)(idx / in_size), ox = (int)(idx % in_size);
  int y0, y1, x0, x1;
  float ty, tx;
  lin_tap(oy, f.s, in_size, y0, y1, ty);
  lin_tap(ox, f.s, in_size, x0, x1, tx);
  const int64_t p00 = f.img + ((int64_t)y0 * f.s + x0) * 3, p01 = f.img + ((int64_t)y0 * f.s + x1) * 3;
  const int64_t p10 = f.img + ((int64_t)y1 * f.s + x0) * 3, p11 = f.img + ((int64_t)y1 * f.s + x1) * 3;
  uint8_t* o = lq + ((int64_t)b * in_size * in_size + idx) * 3;
  float* fo = f.fstate >= 0 ? fstate + f.fstate + idx * 3 : nullptr;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float a, bb, cc, dd;
    if (f.q > 0) {           // np.float32(imdecode(...)) / 255.
      a = __fdiv_rn((float)dimg[p00 + c], 255.f);
      bb = __fdiv_rn((float)dimg[p01 + c], 255.f);
      cc = __fdiv_rn((float)dimg[p10 + c], 255.f);
      dd = __fdiv_rn((float)dimg[p11 + c], 255.f);
    } else {
      a = fimg[p00 + c], bb = fimg[p01 + c], cc = fimg[p10 + c], dd = fimg[p11 + c];
    }
    const float v = lerp(lerp(a, bb, tx), lerp(cc, dd, tx), ty);
    if (fo)
      fo[c] = v;
    else
      o[c] = sat_u8(__fmul_rn(v, 255.f));
  }
}

// ------------------------------------------------------------------------------------------------------------ planning
inline int64_t align256(int64_t x) { return (x + 255) / 256 * 256; }

int64_t jpeg_plane_bytes(int h, int w) {
  return align256((int64_t)((w + 7) / 8) * 8 * ((h + 7) / 8) * 8) + align256((int64_t)2 * ((w + 15) / 16) * 8 * ((h + 15) / 16) * 8);
}

struct DegPlan {
  std::vector<DegFace> faces;
  std::vector<JpgImg> jpg;
  int64_t desc, jdesc, grid, fimg, uimg, dimg, planes, total;
  int64_t max_grid, max_small, max_blocks, max_px;
};

DegPlan plan_degrade(int batch, int S, const int32_t* sizes, const int32_t* qualities, const int64_t* noise_offsets,
                     const int64_t* fstate = nullptr) {
  DegPlan P;
  P.faces.resize(batch);
  int64_t grid = 0, img = 0, planes = 0;
  P.max_grid = P.max_small = P.max_blocks = P.max_px = 0;
  for (int b = 0; b < batch; ++b) {
    DegFace& f = P.faces[b];
    f.s = sizes[b];
    f.n = 2 * f.s >= S ? S : 2 * f.s;
    f.q = qualities ? qualities[b] : 0;
    f.pad = 0;
    f.noise = noise_offsets ? noise_offsets[b] : -1;
    f.fstate = fstate ? fstate[b] : -1;
    f.grid = grid;
    f.img = img;
    grid += (int64_t)f.n * f.n * 3;
    img += (int64_t)f.s * f.s * 3;
    P.max_grid = std::max(P.max_grid, (int64_t)f.n * f.n);
    P.max_small = std::max(P.max_small, (int64_t)f.s * f.s);
    if (f.q > 0) {
      JpgImg J{f.s, f.s, f.q, 0, f.img, f.img, planes, planes + align256((int64_t)((f.s + 7) / 8) * 8 * ((f.s + 7) / 8) * 8)};
      planes += jpeg_plane_bytes(f.s, f.s);
      P.jpg.push_back(J);
      const int64_t nb = (int64_t)((f.s + 7) / 8) * ((f.s + 7) / 8) + 2 * (int64_t)((f.s + 15) / 16) * ((f.s + 15) / 16);
      P.max_blocks = std::max(P.max_blocks, nb);
      P.max_px = std::max(P.max_px, (int64_t)f.s * f.s);
    }
  }
  P.desc = 0;
  P.jdesc = align256((int64_t)batch * sizeof(DegFace));
  P.grid = P.jdesc + align256((int64_t)P.jpg.size() * sizeof(JpgImg));
  P.fimg = P.grid + align256(grid * 4);
  P.uimg = P.fimg + align256(img * 4);
  P.dimg = P.uimg + align256(img);
  P.planes = P.dimg + align256(img);
  P.total = P.planes + planes;
  return P;
}

int launch_jpeg(const JpgImg* djpg, int n, int64_t max_blocks, int64_t max_px, const uint8_t* src_base, uint8_t* plane_base,
                uint8_t* dst_base, cudaStream_t st) {
  if (n == 0) return 0;
  jpeg_block_kernel<<<dim3((unsigned)((max_blocks + 127) / 128), n), 128, 0, st>>>(djpg, src_base, plane_base);
  CFB_LAUNCH_CHECK();
  jpeg_color_kernel<<<dim3((unsigned)((max_px + kThreads - 1) / kThreads), n), kThreads, 0, st>>>(djpg, plane_base, dst_base);
  CFB_LAUNCH_CHECK();
  return 0;
}

int degrade(const uint8_t* gt, int batch, int S, const double* kernels, int ks, const int32_t* sizes, const int32_t* qualities,
            const float* noise, const int64_t* noise_offsets, int in_size, uint8_t* lq, void* ws, int64_t ws_bytes,
            float* cap_a, uint8_t* cap_u8, cudaStream_t st, const int64_t* fstate_offsets = nullptr,
            float* fstate = nullptr) {
  CFB_REQUIRE(batch >= 0 && batch <= 65535, "cfb_degrade_faces: batch must be 0..65535");
  CFB_REQUIRE(S >= 1 && in_size >= 1 && in_size <= S, "cfb_degrade_faces: need 1 <= in_size <= gt_size");
  CFB_REQUIRE(ks >= 1 && ks % 2 == 1 && ks <= kMaxKsize, "cfb_degrade_faces: the kernel size must be odd and at most 63");
  if (batch == 0) return 0;
  CFB_REQUIRE(gt && kernels && sizes && lq, "cfb_degrade_faces: NULL argument");
  for (int b = 0; b < batch; ++b) {
    CFB_REQUIRE(sizes[b] >= 1 && sizes[b] <= S, "cfb_degrade_faces: small sizes must be 1..gt_size");
    CFB_REQUIRE(!qualities || (qualities[b] >= 0 && qualities[b] <= 100), "cfb_degrade_faces: quality must be 0 (none) or 1..100");
    CFB_REQUIRE(!noise_offsets || noise_offsets[b] < 0 || noise, "cfb_degrade_faces: noise offsets without a noise field");
  }
  const DegPlan P = plan_degrade(batch, S, sizes, qualities, noise_offsets, fstate_offsets);
  CFB_REQUIRE(ws && ws_bytes >= P.total, "cfb_degrade_faces: workspace too small (cfb_degrade_workspace_bytes)");
  char* w = static_cast<char*>(ws);
  DegFace* dfaces = reinterpret_cast<DegFace*>(w + P.desc);
  JpgImg* djpg = reinterpret_cast<JpgImg*>(w + P.jdesc);
  float* grid = reinterpret_cast<float*>(w + P.grid);
  float* fimg = reinterpret_cast<float*>(w + P.fimg);
  uint8_t* uimg = reinterpret_cast<uint8_t*>(w + P.uimg);
  uint8_t* dimg = reinterpret_cast<uint8_t*>(w + P.dimg);
  uint8_t* planes = reinterpret_cast<uint8_t*>(w + P.planes);
  CFB_CUDA(cudaMemcpyAsync(dfaces, P.faces.data(), P.faces.size() * sizeof(DegFace), cudaMemcpyHostToDevice, st));
  if (!P.jpg.empty())
    CFB_CUDA(cudaMemcpyAsync(djpg, P.jpg.data(), P.jpg.size() * sizeof(JpgImg), cudaMemcpyHostToDevice, st));
  const int smem = ks * ks * 8;
  blur_grid_kernel<<<dim3((unsigned)((P.max_grid + kThreads - 1) / kThreads), batch), kThreads, smem, st>>>(gt, S, dfaces, kernels,
                                                                                                            ks, grid);
  CFB_LAUNCH_CHECK();
  small_kernel<<<dim3((unsigned)((P.max_small + kThreads - 1) / kThreads), batch), kThreads, 0, st>>>(S, dfaces, grid, noise, fimg,
                                                                                                     uimg, cap_a, cap_u8);
  CFB_LAUNCH_CHECK();
  CFB_CHECK(launch_jpeg(djpg, (int)P.jpg.size(), P.max_blocks, P.max_px, uimg, planes, dimg, st));
  final_kernel<<<dim3((unsigned)(((int64_t)in_size * in_size + kThreads - 1) / kThreads), batch), kThreads, 0, st>>>(
      dfaces, fimg, dimg, in_size, lq, fstate);
  CFB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------------ colour stages
// FFHQBlindDataset.__getitem__:253-273 on the float image before its clip(round(x * 255)): the shift, cv2's gray, then
// BGR -> RGB and torchvision's adjust_* ops in the drawn order, each with torch's float32 op sequence (separate mul and add
// kernels, so nothing is contracted) and clamps.  adjust_contrast blends with the mean gray of the whole face, so a face's
// ops split there: color_pre_kernel runs the ops before it and writes per-block float64 sums of the gray, color_mean_kernel
// adds them in block order, color_post_kernel runs the rest and rounds.  Mask faces (inpainting) are where(mask, 255, gt).
constexpr int kShift = 1, kGray = 2, kMask = 4;
constexpr int kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3;   // color_jitter_pt's fn_id

struct ColorFace {
  int flags;        // kShift | kGray | kMask
  int nops;         // torchvision ops, 0..4
  int pre;          // ops before the contrast mean: the position of contrast, or nops
  int pad;
  int op[4];
  float jit[3];     // the shift, BGR
  float fac[4];     // each op's factor
  float omf[4];     // float32(1.0 - factor), as _blend's Python double cast to float32
  int64_t state;    // offset of the face's float state [n][3] (RGB after the first kernel) in floats, -1 = no colour stage
};

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

// rgb_to_grayscale: (0.2989 r + 0.587 g) + 0.114 b
__device__ __forceinline__ float tv_gray(float r, float g, float b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// _blend: (ratio * x + (1.0 - ratio) * y).clamp(0, 1)
__device__ __forceinline__ float blend(float x, float y, float f, float omf) {
  return clamp01(__fadd_rn(__fmul_rn(f, x), __fmul_rn(omf, y)));
}

// adjust_hue: _rgb2hsv, (h + f) % 1.0, _hsv2rgb
__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float f) {
  const float maxc = fmaxf(fmaxf(r, g), b), minc = fminf(fminf(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
  const float crd = eqc ? 1.f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd), gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
  const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  const float hr = __fmul_rn(maxc == r ? 1.f : 0.f, __fsub_rn(bc, gc));
  const float hg = __fmul_rn(maxc == g && maxc != r ? 1.f : 0.f, __fsub_rn(__fadd_rn(2.f, rc), bc));
  const float hb = __fmul_rn(maxc != g && maxc != r ? 1.f : 0.f, __fsub_rn(__fadd_rn(4.f, gc), rc));
  float h = fmodf(__fadd_rn(__fdiv_rn(__fadd_rn(__fadd_rn(hr, hg), hb), 6.f), 1.f), 1.f);
  h = fmodf(__fadd_rn(h, f), 1.f);            // torch.remainder: fmod, plus the divisor when the signs differ
  if (h < 0.f) h = __fadd_rn(h, 1.f);
  const float v = maxc, h6 = __fmul_rn(h, 6.f), fi = floorf(h6), fr = __fsub_rn(h6, fi);
  const float p = clamp01(__fmul_rn(v, __fsub_rn(1.f, s)));
  const float q = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, fr))));
  const float t = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, fr)))));
  switch ((int)fi % 6) {
    case 0: r = v, g = t, b = p; break;
    case 1: r = q, g = v, b = p; break;
    case 2: r = p, g = v, b = t; break;
    case 3: r = p, g = q, b = v; break;
    case 4: r = t, g = p, b = v; break;
    default: r = v, g = p, b = q; break;
  }
}

__device__ __forceinline__ void apply_op(const ColorFace& c, int k, float& r, float& g, float& b, float mean) {
  const float f = c.fac[k], omf = c.omf[k];
  switch (c.op[k]) {
    case kBrightness:
      r = blend(r, 0.f, f, omf), g = blend(g, 0.f, f, omf), b = blend(b, 0.f, f, omf);
      break;
    case kContrast:
      r = blend(r, mean, f, omf), g = blend(g, mean, f, omf), b = blend(b, mean, f, omf);
      break;
    case kSaturation: {
      const float y = tv_gray(r, g, b);
      r = blend(r, y, f, omf), g = blend(g, y, f, omf), b = blend(b, y, f, omf);
      break;
    }
    default:
      hue_shift(r, g, b, f);
  }
}

// fixed-order block sum: lanes by shuffle, then the warps' sums in warp order
__device__ __forceinline__ double block_sum(double v) {
  __shared__ double warp_sums[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s = __dadd_rn(s, warp_sums[w]);
  return s;
}

// the shift, gray, BGR -> RGB and the ops before contrast; the gray of the result summed per block when contrast follows.
// gt is the uint8 source of faces without corruption (state then starts as gt / 255), NULL when final_kernel wrote it.
__global__ void __launch_bounds__(kThreads) color_pre_kernel(const ColorFace* __restrict__ faces, const uint8_t* __restrict__ gt,
                                                             int n_px, float* __restrict__ state, double* __restrict__ partials) {
  const int b = blockIdx.y;
  const ColorFace& c = faces[b];       // read in place: the ops are indexed at run time
  if (c.state < 0) return;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double gsum = 0.;
  if (idx < n_px) {
    float* st = state + c.state + idx * 3;
    float x[3];
    if (gt) {
      const uint8_t* p = gt + ((int64_t)b * n_px + idx) * 3;
#pragma unroll
      for (int k = 0; k < 3; ++k) x[k] = __fdiv_rn((float)p[k], 255.f);
    } else {
#pragma unroll
      for (int k = 0; k < 3; ++k) x[k] = st[k];
    }
    if (c.flags & kShift) {
#pragma unroll
      for (int k = 0; k < 3; ++k) x[k] = clamp01(__fadd_rn(x[k], c.jit[k]));
    }
    if (c.flags & kGray)     // cv2.cvtColor(float32, COLOR_BGR2GRAY): fma(r, 0.299, fma(b, 0.114, g * 0.587))
      x[0] = x[1] = x[2] = __fmaf_rn(x[2], 0.299f, __fmaf_rn(x[0], 0.114f, __fmul_rn(x[1], 0.587f)));
    float r = x[2], g = x[1], bl = x[0];
    for (int k = 0; k < c.pre; ++k) apply_op(c, k, r, g, bl, 0.f);
    if (c.pre < c.nops) gsum = (double)tv_gray(r, g, bl);
    st[0] = r, st[1] = g, st[2] = bl;
  }
  if (c.pre < c.nops) {
    const double s = block_sum(gsum);
    if (threadIdx.x == 0) partials[(int64_t)b * gridDim.x + blockIdx.x] = s;
  }
}

// per face, the block sums in block order, / n_px in float64, rounded once to float32 (NaN for faces without contrast)
__global__ void __launch_bounds__(kThreads) color_mean_kernel(const ColorFace* __restrict__ faces, const double* __restrict__ partials,
                                                              int nblk, int n_px, float* __restrict__ means) {
  const int b = blockIdx.x;
  const ColorFace& c = faces[b];
  if (c.state < 0 || c.pre >= c.nops) {
    if (threadIdx.x == 0) means[b] = __int_as_float(0x7fc00000);
    return;
  }
  double v = 0.;
  for (int i = threadIdx.x; i < nblk; i += kThreads) v = __dadd_rn(v, partials[(int64_t)b * nblk + i]);
  const double s = block_sum(v);
  if (threadIdx.x == 0) means[b] = __double2float_rn(s / n_px);
}

// contrast and the ops after it, RGB -> BGR, round half to even, clip; mask faces and faces without colour stages
__global__ void __launch_bounds__(kThreads) color_post_kernel(const ColorFace* __restrict__ faces, const uint8_t* __restrict__ gt,
                                                              const uint8_t* __restrict__ masks, int n_px,
                                                              const float* __restrict__ state, const float* __restrict__ means,
                                                              uint8_t* __restrict__ lq) {
  const int b = blockIdx.y;
  const ColorFace& c = faces[b];       // read in place: the ops are indexed at run time
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_px) return;
  uint8_t* o = lq + ((int64_t)b * n_px + idx) * 3;
  if (c.state < 0) {       // without corruption: clip(round(float32(k / 255) * 255)) = k; corrupted faces: lq is written
    if (!gt) return;
    const uint8_t* p = gt + ((int64_t)b * n_px + idx) * 3;
    const bool m = (c.flags & kMask) && masks[(int64_t)b * n_px + idx];
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = m ? 255 : p[k];
    return;
  }
  const float* st = state + c.state + idx * 3;
  float r = st[0], g = st[1], bl = st[2];
  if (c.pre < c.nops) {
    const float mean = means[b];
    for (int k = c.pre; k < c.nops; ++k) apply_op(c, k, r, g, bl, mean);
  }
  o[0] = sat_u8(__fmul_rn(bl, 255.f));
  o[1] = sat_u8(__fmul_rn(g, 255.f));
  o[2] = sat_u8(__fmul_rn(r, 255.f));
}

struct ColorPlan {
  std::vector<ColorFace> faces;
  std::vector<int64_t> fstate;
  int64_t deg, desc, state, partials, means, total;
  int nblk;
};

// ops: [batch][6] int32 (flags, nops, op[4]); factors: [batch][7] float32 (jit[3], factor[4]); NULL = no colour stages
ColorPlan plan_color(int batch, int S, const int32_t* sizes, const int32_t* qualities, int in_size, const int32_t* ops,
                     const float* factors) {
  ColorPlan P;
  P.faces.resize(batch);
  P.fstate.assign(batch, -1);
  const int64_t n_px = (int64_t)in_size * in_size;
  int64_t state = 0;
  for (int b = 0; b < batch; ++b) {
    ColorFace& c = P.faces[b];
    c = ColorFace{};
    c.state = -1;
    if (ops) {
      c.flags = ops[b * 6];
      c.nops = ops[b * 6 + 1];
      c.pre = c.nops;
      for (int k = 0; k < c.nops; ++k) {
        c.op[k] = ops[b * 6 + 2 + k];
        c.fac[k] = factors[b * 7 + 3 + k];
        c.omf[k] = (float)(1.0 - (double)c.fac[k]);
        if (c.op[k] == kContrast) c.pre = k;
      }
      for (int k = 0; k < 3; ++k) c.jit[k] = factors[b * 7 + k];
    }
    if ((c.flags & (kShift | kGray)) || c.nops > 0) {
      c.state = P.fstate[b] = state;
      state += n_px * 3;
    }
  }
  P.nblk = (int)((n_px + kThreads - 1) / kThreads);
  P.deg = sizes ? align256(plan_degrade(batch, S, sizes, qualities, nullptr).total) : 0;
  P.desc = P.deg;
  P.state = P.desc + align256((int64_t)batch * sizeof(ColorFace));
  P.partials = P.state + align256(state * 4);
  P.means = P.partials + align256((int64_t)batch * P.nblk * 8);
  P.total = P.means + align256((int64_t)batch * 4);
  return P;
}

bool valid_color(int batch, bool corrupt, const int32_t* ops, const float* factors, const uint8_t* masks) {
  if (!ops) return true;
  if (!factors) return false;
  for (int b = 0; b < batch; ++b) {
    const int flags = ops[b * 6], nops = ops[b * 6 + 1];
    if (flags & ~(kShift | kGray | kMask) || nops < 0 || nops > 4) return false;
    if ((flags & kMask) && (corrupt || !masks || (flags & ~kMask) || nops)) return false;
    int seen = 0;
    for (int k = 0; k < nops; ++k) {
      const int op = ops[b * 6 + 2 + k];
      const float f = factors[b * 7 + 3 + k];
      if (op < 0 || op > 3 || (seen >> op & 1) || !isfinite(f)) return false;
      if (op == kHue ? !(f >= -0.5f && f <= 0.5f) : !(f >= 0.f)) return false;
      seen |= 1 << op;
    }
    for (int k = 0; k < 3; ++k)
      if ((flags & kShift) && !isfinite(factors[b * 7 + k])) return false;
  }
  return true;
}

int degrade_color(const uint8_t* gt, int batch, int S, const double* kernels, int ks, const int32_t* sizes, const int32_t* qualities,
                  const float* noise, const int64_t* noise_offsets, const int32_t* ops, const float* factors, const uint8_t* masks,
                  int in_size, uint8_t* lq, void* ws, int64_t ws_bytes, float* means_out, cudaStream_t st) {
  const bool corrupt = kernels != nullptr;
  CFB_REQUIRE(batch >= 0 && batch <= 65535, "cfb_degrade_faces_color: batch must be 0..65535");
  CFB_REQUIRE(S >= 1 && in_size >= 1 && in_size <= S, "cfb_degrade_faces_color: need 1 <= in_size <= gt_size");
  CFB_REQUIRE(corrupt || in_size == S, "cfb_degrade_faces_color: without corruption in_size must equal gt_size");
  CFB_REQUIRE(corrupt == (sizes != nullptr), "cfb_degrade_faces_color: give kernels and small sizes together, or neither");
  if (batch == 0) return 0;
  CFB_REQUIRE(gt && lq, "cfb_degrade_faces_color: NULL argument");
  CFB_REQUIRE(valid_color(batch, corrupt, ops, factors, masks),
              "cfb_degrade_faces_color: bad colour descriptor (flags, op codes, repeated ops, factors, or a mask with "
              "corruption or colour stages)");
  if (corrupt)
    for (int b = 0; b < batch; ++b)
      CFB_REQUIRE(sizes[b] >= 1 && sizes[b] <= S, "cfb_degrade_faces_color: small sizes must be 1..gt_size");
  const ColorPlan P = plan_color(batch, S, sizes, qualities, in_size, ops, factors);
  CFB_REQUIRE(ws && ws_bytes >= P.total, "cfb_degrade_faces_color: workspace too small (cfb_degrade_color_workspace_bytes)");
  char* w = static_cast<char*>(ws);
  ColorFace* dfaces = reinterpret_cast<ColorFace*>(w + P.desc);
  float* state = reinterpret_cast<float*>(w + P.state);
  double* partials = reinterpret_cast<double*>(w + P.partials);
  float* means = means_out ? means_out : reinterpret_cast<float*>(w + P.means);
  if (corrupt)
    CFB_CHECK(degrade(gt, batch, S, kernels, ks, sizes, qualities, noise, noise_offsets, in_size, lq, ws, P.deg, nullptr, nullptr,
                      st, P.fstate.data(), state));
  CFB_CUDA(cudaMemcpyAsync(dfaces, P.faces.data(), P.faces.size() * sizeof(ColorFace), cudaMemcpyHostToDevice, st));
  const int64_t n_px = (int64_t)in_size * in_size;
  const uint8_t* src = corrupt ? nullptr : gt;
  color_pre_kernel<<<dim3((unsigned)P.nblk, batch), kThreads, 0, st>>>(dfaces, src, (int)n_px, state, partials);
  CFB_LAUNCH_CHECK();
  color_mean_kernel<<<batch, kThreads, 0, st>>>(dfaces, partials, P.nblk, (int)n_px, means);
  CFB_LAUNCH_CHECK();
  color_post_kernel<<<dim3((unsigned)P.nblk, batch), kThreads, 0, st>>>(dfaces, src, masks, (int)n_px, state, means, lq);
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace
}  // namespace cfb

#define DEG_API_BEGIN try {
#define DEG_API_END                                                                                          \
  }                                                                                                          \
  catch (const std::exception& e) {                                                                          \
    cfb::set_error(std::string("exception: ") + e.what());                                                   \
    return 1;                                                                                                \
  }

extern "C" {

int64_t cfb_degrade_workspace_bytes(int32_t batch, int32_t gt_size, const int32_t* small_sizes, const int32_t* qualities) {
  if (batch < 0 || gt_size < 1 || (batch > 0 && !small_sizes)) return -1;
  for (int b = 0; b < batch; ++b)
    if (small_sizes[b] < 1 || small_sizes[b] > gt_size || (qualities && (qualities[b] < 0 || qualities[b] > 100))) return -1;
  return cfb::plan_degrade(batch, gt_size, small_sizes, qualities, nullptr).total;
}

int cfb_degrade_faces(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                      const int32_t* small_sizes, const int32_t* qualities, const float* noise, const int64_t* noise_offsets,
                      int32_t in_size, uint8_t* lq, void* workspace, int64_t workspace_bytes, void* stream) {
  DEG_API_BEGIN
  return cfb::degrade(gt, batch, gt_size, kernels, ksize, small_sizes, qualities, noise, noise_offsets, in_size, lq, workspace,
                      workspace_bytes, nullptr, nullptr, (cudaStream_t)stream);
  DEG_API_END
}

int cfb_debug_degrade_faces(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                            const int32_t* small_sizes, const int32_t* qualities, const float* noise,
                            const int64_t* noise_offsets, int32_t in_size, uint8_t* lq, void* workspace, int64_t workspace_bytes,
                            float* stage_a, uint8_t* pre_jpeg, void* stream) {
  DEG_API_BEGIN
  return cfb::degrade(gt, batch, gt_size, kernels, ksize, small_sizes, qualities, noise, noise_offsets, in_size, lq, workspace,
                      workspace_bytes, stage_a, pre_jpeg, (cudaStream_t)stream);
  DEG_API_END
}

int64_t cfb_degrade_color_workspace_bytes(int32_t batch, int32_t gt_size, const int32_t* small_sizes, const int32_t* qualities,
                                          const int32_t* color_ops, int32_t in_size) {
  if (batch < 0 || gt_size < 1 || in_size < 1 || in_size > gt_size || (!small_sizes && in_size != gt_size)) return -1;
  for (int b = 0; b < batch; ++b) {
    if (small_sizes && (small_sizes[b] < 1 || small_sizes[b] > gt_size || (qualities && (qualities[b] < 0 || qualities[b] > 100))))
      return -1;
    if (color_ops && (color_ops[b * 6 + 1] < 0 || color_ops[b * 6 + 1] > 4)) return -1;
  }
  std::vector<float> zeros(color_ops ? (size_t)batch * 7 : 0, 0.f);
  return cfb::plan_color(batch, gt_size, small_sizes, qualities, in_size, color_ops, color_ops ? zeros.data() : nullptr).total;
}

int cfb_degrade_faces_color(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                            const int32_t* small_sizes, const int32_t* qualities, const float* noise, const int64_t* noise_offsets,
                            const int32_t* color_ops, const float* color_factors, const uint8_t* masks, int32_t in_size,
                            uint8_t* lq, void* workspace, int64_t workspace_bytes, void* stream) {
  DEG_API_BEGIN
  return cfb::degrade_color(gt, batch, gt_size, kernels, ksize, small_sizes, qualities, noise, noise_offsets, color_ops,
                            color_factors, masks, in_size, lq, workspace, workspace_bytes, nullptr, (cudaStream_t)stream);
  DEG_API_END
}

int cfb_debug_degrade_faces_color(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                                  const int32_t* small_sizes, const int32_t* qualities, const float* noise,
                                  const int64_t* noise_offsets, const int32_t* color_ops, const float* color_factors,
                                  const uint8_t* masks, int32_t in_size, uint8_t* lq, void* workspace, int64_t workspace_bytes,
                                  float* contrast_means, void* stream) {
  DEG_API_BEGIN
  CFB_REQUIRE(contrast_means || batch == 0, "cfb_debug_degrade_faces_color: NULL contrast_means");
  return cfb::degrade_color(gt, batch, gt_size, kernels, ksize, small_sizes, qualities, noise, noise_offsets, color_ops,
                            color_factors, masks, in_size, lq, workspace, workspace_bytes, contrast_means, (cudaStream_t)stream);
  DEG_API_END
}

int64_t cfb_jpeg_workspace_bytes(int32_t n, int32_t h, int32_t w) {
  if (n < 0 || h < 1 || w < 1) return -1;
  return cfb::align256((int64_t)n * sizeof(cfb::JpgImg)) + (int64_t)n * cfb::jpeg_plane_bytes(h, w);
}

int cfb_jpeg_roundtrip(const uint8_t* src, uint8_t* dst, int32_t n, int32_t h, int32_t w, const int32_t* qualities, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  DEG_API_BEGIN
  CFB_REQUIRE(n >= 0 && n <= 65535 && h >= 1 && w >= 1, "cfb_jpeg_roundtrip: bad size");
  if (n == 0) return 0;
  CFB_REQUIRE(src && dst && qualities, "cfb_jpeg_roundtrip: NULL argument");
  CFB_REQUIRE(src != dst, "cfb_jpeg_roundtrip: src and dst must not alias");
  const int64_t need = cfb_jpeg_workspace_bytes(n, h, w);
  CFB_REQUIRE(workspace && workspace_bytes >= need, "cfb_jpeg_roundtrip: workspace too small (cfb_jpeg_workspace_bytes)");
  const int64_t img = (int64_t)h * w * 3, pb = cfb::jpeg_plane_bytes(h, w);
  const int64_t yb = cfb::align256((int64_t)((w + 7) / 8) * 8 * ((h + 7) / 8) * 8);
  std::vector<cfb::JpgImg> J(n);
  for (int i = 0; i < n; ++i) {
    CFB_REQUIRE(qualities[i] >= 1 && qualities[i] <= 100, "cfb_jpeg_roundtrip: quality must be 1..100");
    J[i] = cfb::JpgImg{h, w, qualities[i], 0, i * img, i * img, i * pb, i * pb + yb};
  }
  char* ws = static_cast<char*>(workspace);
  cfb::JpgImg* dj = reinterpret_cast<cfb::JpgImg*>(ws);
  uint8_t* planes = reinterpret_cast<uint8_t*>(ws + cfb::align256((int64_t)n * sizeof(cfb::JpgImg)));
  cudaStream_t st = (cudaStream_t)stream;
  CFB_CUDA(cudaMemcpyAsync(dj, J.data(), J.size() * sizeof(cfb::JpgImg), cudaMemcpyHostToDevice, st));
  const int64_t nb = (int64_t)((w + 7) / 8) * ((h + 7) / 8) + 2 * (int64_t)((w + 15) / 16) * ((h + 15) / 16);
  return cfb::launch_jpeg(dj, n, nb, (int64_t)h * w, src, planes, dst, st);
  DEG_API_END
}

}  // extern "C"
