// Restoration metrics (cfb_psnr_ssim): basicsr's calculate_psnr / calculate_ssim (basicsr/metrics/psnr_ssim.py,
// metric_util.py) over batches of HWC image pairs; pair p compares a[p] with b[p / k].
//   load    one templated reader per element type (uint8, uint16, float32, float64) reads the images in place: the crop is an
//           offset, and the Y channel of to_y_channel is formed at load in the reference's order
//   psnr    per (pair, block of rows): the sum of squared differences -- int64 for integer images (exact, so the MSE is the
//           one numpy computes), float64 otherwise; on the Y path the squares are float32, as in the reference
//   ssim    per (pair, channel, 32 x 32 output tile): the 42 x 42 halo tile in shared memory as float64, the 11 horizontal
//           taps, then the 11 vertical ones, for a, b, a^2, b^2 and ab; the SSIM map; the tile's sum
//   final   per pair: the partials summed in a fixed order -> PSNR (or the MSE) and the mean SSIM over the channels
// Every sum has a fixed order that depends on the image size only, so results are the same on every run and in any batch.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "kernels.cuh"

namespace cfb {
namespace {

constexpr int kTile = 32;                       // SSIM outputs per CTA side
constexpr int kHalo = kTile + 10;               // input rows / columns the 11-tap window needs
constexpr int kSsimThreads = 256;               // 8 warps; lane = output column
constexpr int kRowsPerWarp = kTile / (kSsimThreads / 32);
constexpr int kSsimSmem = (2 * kHalo * kHalo + 5 * kHalo * kTile) * 8;
constexpr int kPsnrBlocks = 128;                // row blocks per pair (fewer for images of fewer rows)
constexpr int kReduceThreads = 256;

// cv2.getGaussianKernel(11, 1.5); the reference filters with its outer product
__constant__ double kGauss[11] = {0x1.0d956b52a1d6ep-10, 0x1.f1fe01ae5a5b5p-8, 0x1.26eb175d83f66p-5, 0x1.bff0fe8e98418p-4,
                                  0x1.b43c3f52b19f3p-3,  0x1.106560aa892bfp-2, 0x1.b43c3f52b19f3p-3, 0x1.bff0fe8e98418p-4,
                                  0x1.26eb175d83f66p-5,  0x1.f1fe01ae5a5b5p-8, 0x1.0d956b52a1d6ep-10};

// how a value is read: as stored (PLAIN); the Y of three channels (Y3); float32(x) / 255 * 255 for other channel counts on
// the Y path (YKEEP: to_y_channel converts only three channels but rounds every image through float32)
enum ReadMode { PLAIN = 0, Y3 = 1, YKEEP = 2 };

template <typename T>
struct Pairs {
  const T* a;
  const T* b;
  int k, h, w, c, crop, hv, wv, mode;
  __device__ __forceinline__ const T* pixel(const T* img, int p, int y, int x) const {   // (y, x) in the cropped image
    return img + ((int64_t)p * h * w + (int64_t)(y + crop) * w + (x + crop)) * c;
  }
};

// x.astype(np.float32) / 255. in float32
template <typename T>
__device__ __forceinline__ float unit_f32(T v) { return __fdiv_rn((float)v, 255.f); }

// to_y_channel of three channels (metric_util.py:32-45, bgr2ycbcr with y_only): float64 products and sums of the float32
// unit values in numpy's order, / 255 rounded to float32, then * 255 in float32.  No contraction into FMAs.
template <typename T>
__device__ __forceinline__ float y_of(const T* px) {
  const double b = unit_f32(px[0]), g = unit_f32(px[1]), r = unit_f32(px[2]);
  double t = __dadd_rn(__dmul_rn(b, 24.966), __dmul_rn(g, 128.553));
  t = __dadd_rn(__dadd_rn(t, __dmul_rn(r, 65.481)), 16.0);
  return __fmul_rn(__double2float_rn(__ddiv_rn(t, 255.0)), 255.f);
}

template <typename T>
__device__ __forceinline__ double read_value(const T* px, int ch, int mode) {
  if (mode == Y3) return (double)y_of(px);
  if (mode == YKEEP) return (double)__fmul_rn(unit_f32(px[ch]), 255.f);
  return (double)px[ch];
}

// sum over the block in a fixed tree order (blockDim.x == 256); callable repeatedly
template <typename V>
__device__ __forceinline__ V block_sum(V v, V* sh) {
  __syncthreads();
  sh[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = kReduceThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

// Σ (a - b)^2 over rows blockIdx.x, blockIdx.x + gridDim.x, ... of pair blockIdx.y.  INT: integer images without the Y path,
// summed exactly in int64; otherwise float64 sums of float64 squares (float32 squares on the Y path).
template <typename T, bool INT>
__global__ void __launch_bounds__(kReduceThreads) psnr_partial_kernel(Pairs<T> m, int64_t* part_i, double* part_f) {
  __shared__ int64_t shi[INT ? kReduceThreads : 1];
  __shared__ double shf[INT ? 1 : kReduceThreads];
  const int p = blockIdx.y;
  const int per_row = m.mode == Y3 ? m.wv : m.wv * m.c;
  int64_t si = 0;
  double sf = 0.0;
  for (int y = blockIdx.x; y < m.hv; y += gridDim.x) {
    const T* ra = m.pixel(m.a, p, y, 0);
    const T* rb = m.pixel(m.b, p / m.k, y, 0);
    for (int i = threadIdx.x; i < per_row; i += kReduceThreads) {
      if constexpr (INT) {
        const int64_t d = (int64_t)ra[i] - (int64_t)rb[i];
        si += d * d;
      } else if (m.mode == PLAIN) {
        const double d = __dsub_rn((double)ra[i], (double)rb[i]);
        sf = __dadd_rn(sf, __dmul_rn(d, d));
      } else {
        const float va = m.mode == Y3 ? y_of(ra + 3 * i) : __fmul_rn(unit_f32(ra[i]), 255.f);
        const float vb = m.mode == Y3 ? y_of(rb + 3 * i) : __fmul_rn(unit_f32(rb[i]), 255.f);
        const float d = __fsub_rn(va, vb);
        sf = __dadd_rn(sf, (double)__fmul_rn(d, d));
      }
    }
  }
  const int64_t slot = (int64_t)p * gridDim.x + blockIdx.x;
  if constexpr (INT) {
    const int64_t s = block_sum(si, shi);
    if (threadIdx.x == 0) part_i[slot] = s;
  } else {
    const double s = block_sum(sf, shf);
    if (threadIdx.x == 0) part_f[slot] = s;
  }
}

// One 32 x 32 tile of the SSIM map of channel blockIdx.y of pair blockIdx.z (_ssim, psnr_ssim.py:49-80).  Output (i, j) is the
// window at rows i..i+10, columns j..j+10 of the cropped image (the reference's [5:-5, 5:-5]).  Writes the tile's map sum.
template <typename T>
__global__ void __launch_bounds__(kSsimThreads, 2) ssim_tile_kernel(Pairs<T> m, int tiles_x, double* part) {
  extern __shared__ double sm[];
  double* sa = sm;                              // [kHalo][kHalo]
  double* sb = sa + kHalo * kHalo;              // [kHalo][kHalo]
  double* hs = sb + kHalo * kHalo;              // [5][kHalo][kTile]: horizontal sums of a, b, a^2, b^2, ab
  __shared__ double red[kSsimThreads];
  const int tile = blockIdx.x, ch = blockIdx.y, p = blockIdx.z;
  const int y0 = (tile / tiles_x) * kTile, x0 = (tile % tiles_x) * kTile;
  const int ho = m.hv - 10, wo = m.wv - 10;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (int i = threadIdx.x; i < kHalo * kHalo; i += kSsimThreads) {
    const int r = i / kHalo, q = i - r * kHalo, y = y0 + r, x = x0 + q;
    double va = 0.0, vb = 0.0;                  // outside the image: read by no output inside it
    if (y < m.hv && x < m.wv) {
      va = read_value(m.pixel(m.a, p, y, x), ch, m.mode);
      vb = read_value(m.pixel(m.b, p / m.k, y, x), ch, m.mode);
    }
    sa[i] = va;
    sb[i] = vb;
  }
  __syncthreads();

  for (int r = warp; r < kHalo; r += kSsimThreads / 32) {
    double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int t = 0; t < 11; ++t) {
      const double a = sa[r * kHalo + lane + t], b = sb[r * kHalo + lane + t], g = kGauss[t];
      s[0] = fma(g, a, s[0]);
      s[1] = fma(g, b, s[1]);
      s[2] = fma(g, a * a, s[2]);
      s[3] = fma(g, b * b, s[3]);
      s[4] = fma(g, a * b, s[4]);
    }
#pragma unroll
    for (int q = 0; q < 5; ++q) hs[(q * kHalo + r) * kTile + lane] = s[q];
  }
  __syncthreads();

  // each warp: kRowsPerWarp consecutive output rows, every input row loaded once for all of them
  double acc[kRowsPerWarp][5] = {};
  const int r0 = warp * kRowsPerWarp;
#pragma unroll
  for (int rr = 0; rr < kRowsPerWarp + 10; ++rr) {
    double v[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) v[q] = hs[(q * kHalo + r0 + rr) * kTile + lane];
#pragma unroll
    for (int o = 0; o < kRowsPerWarp; ++o) {
      const int t = rr - o;
      if (t >= 0 && t <= 10) {
#pragma unroll
        for (int q = 0; q < 5; ++q) acc[o][q] = fma(kGauss[t], v[q], acc[o][q]);
      }
    }
  }

  // the map in the reference's order of operations (numpy: no FMA), so that identical images give exactly 1
  const double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  double sum = 0.0;
#pragma unroll
  for (int o = 0; o < kRowsPerWarp; ++o) {
    if (y0 + r0 + o < ho && x0 + lane < wo) {
      const double mu1 = acc[o][0], mu2 = acc[o][1];
      const double mu1_sq = __dmul_rn(mu1, mu1), mu2_sq = __dmul_rn(mu2, mu2), mu1_mu2 = __dmul_rn(mu1, mu2);
      const double s1 = __dsub_rn(acc[o][2], mu1_sq), s2 = __dsub_rn(acc[o][3], mu2_sq), s12 = __dsub_rn(acc[o][4], mu1_mu2);
      const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu1_mu2), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
      const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
      sum = __dadd_rn(sum, __ddiv_rn(num, den));
    }
  }
  const double s = block_sum(sum, red);
  if (threadIdx.x == 0) part[((int64_t)p * gridDim.y + ch) * gridDim.x + tile] = s;
}

// per pair: PSNR (psnr_mode 1), or the MSE (psnr_mode 2), from nb row-block partials; the mean SSIM over ce channels from
// ntiles tile sums each
__global__ void __launch_bounds__(kReduceThreads) metrics_final_kernel(const int64_t* part_i, const double* part_f, int nb,
                                                                       int64_t count, int psnr_mode, const double* ssim_part,
                                                                       int ce, int ntiles, int64_t map_count, double* psnr_out,
                                                                       double* ssim_out) {
  __shared__ int64_t shi[kReduceThreads];
  __shared__ double shf[kReduceThreads];
  const int p = blockIdx.x;
  if (psnr_mode) {
    double mse;
    if (part_i) {
      int64_t s = 0;
      for (int i = threadIdx.x; i < nb; i += kReduceThreads) s += part_i[(int64_t)p * nb + i];
      mse = (double)block_sum(s, shi) / (double)count;
    } else {
      double s = 0.0;
      for (int i = threadIdx.x; i < nb; i += kReduceThreads) s += part_f[(int64_t)p * nb + i];
      mse = block_sum(s, shf) / (double)count;
    }
    if (threadIdx.x == 0) psnr_out[p] = psnr_mode == 2 ? mse : (mse == 0.0 ? INFINITY : 20.0 * log10(255.0 / sqrt(mse)));
  }
  if (ssim_out) {
    double mean = 0.0;                          // numpy's mean of the per-channel means: a left-to-right sum, / ce
    for (int ch = 0; ch < ce; ++ch) {
      const double* src = ssim_part + ((int64_t)p * ce + ch) * ntiles;
      double s = 0.0;
      for (int i = threadIdx.x; i < ntiles; i += kReduceThreads) s += src[i];
      mean += block_sum(s, shf) / (double)map_count;
    }
    if (threadIdx.x == 0) ssim_out[p] = mean / ce;
  }
}

struct Plan {
  int hv, wv, ce, mode, nb, tiles_x, ntiles;
  size_t psnr_off, ssim_off, total;
};

Plan plan_of(int pairs, int h, int w, int c, int crop, bool y) {
  Plan P;
  P.hv = h - 2 * crop;
  P.wv = w - 2 * crop;
  P.mode = y ? (c == 3 ? Y3 : YKEEP) : PLAIN;
  P.ce = P.mode == Y3 ? 1 : c;
  P.nb = P.hv > 0 ? (P.hv < kPsnrBlocks ? P.hv : kPsnrBlocks) : 0;
  const int ho = P.hv - 10, wo = P.wv - 10;
  P.tiles_x = wo > 0 ? (wo + kTile - 1) / kTile : 0;
  P.ntiles = ho > 0 && wo > 0 ? P.tiles_x * ((ho + kTile - 1) / kTile) : 0;
  P.psnr_off = 0;
  P.ssim_off = ((size_t)pairs * P.nb * 8 + 255) / 256 * 256;
  P.total = P.ssim_off + (size_t)pairs * P.ce * P.ntiles * 8;
  return P;
}

template <typename T>
int run(const MetricArgs& a, const Plan& P, void* ws, cudaStream_t st) {
  const Pairs<T> m{static_cast<const T*>(a.a), static_cast<const T*>(a.b), a.k, a.h, a.w, a.c, a.crop, P.hv, P.wv, P.mode};
  const bool integer = std::is_integral<T>::value && P.mode == PLAIN;
  int64_t* part_i = integer ? reinterpret_cast<int64_t*>((char*)ws + P.psnr_off) : nullptr;
  double* part_f = integer ? nullptr : reinterpret_cast<double*>((char*)ws + P.psnr_off);
  double* ssim_part = reinterpret_cast<double*>((char*)ws + P.ssim_off);
  if (a.psnr_mode) {
    if constexpr (std::is_integral<T>::value) {
      if (integer)
        psnr_partial_kernel<T, true><<<dim3(P.nb, a.pairs), kReduceThreads, 0, st>>>(m, part_i, part_f);
      else
        psnr_partial_kernel<T, false><<<dim3(P.nb, a.pairs), kReduceThreads, 0, st>>>(m, part_i, part_f);
    } else {
      psnr_partial_kernel<T, false><<<dim3(P.nb, a.pairs), kReduceThreads, 0, st>>>(m, part_i, part_f);
    }
    CFB_LAUNCH_CHECK();
  }
  if (a.ssim) {
    CFB_CUDA(cudaFuncSetAttribute(ssim_tile_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSsimSmem));
    ssim_tile_kernel<T><<<dim3(P.ntiles, P.ce, a.pairs), kSsimThreads, kSsimSmem, st>>>(m, P.tiles_x, ssim_part);
    CFB_LAUNCH_CHECK();
  }
  metrics_final_kernel<<<a.pairs, kReduceThreads, 0, st>>>(part_i, part_f, P.nb, (int64_t)P.hv * P.wv * P.ce, a.psnr_mode,
                                                            ssim_part, P.ce, P.ntiles, (int64_t)(P.hv - 10) * (P.wv - 10),
                                                            a.psnr, a.ssim);
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace

size_t metrics_workspace_bytes(int pairs, int h, int w, int c, int crop, bool y) {
  return plan_of(pairs, h, w, c, crop, y).total;
}

int psnr_ssim(const MetricArgs& a, void* ws, int64_t ws_bytes, cudaStream_t st) {
  const Plan P = plan_of(a.pairs, a.h, a.w, a.c, a.crop, a.y);
  CFB_REQUIRE(P.hv >= 1 && P.wv >= 1, "cfb_psnr_ssim: the crop leaves no pixels");
  CFB_REQUIRE(!a.ssim || (P.hv >= 11 && P.wv >= 11), "cfb_psnr_ssim: SSIM needs at least 11 x 11 pixels after the crop");
  CFB_REQUIRE(P.ce <= 65535, "cfb_psnr_ssim: at most 65535 channels");
  CFB_REQUIRE(ws && ws_bytes >= (int64_t)P.total, "cfb_psnr_ssim: workspace too small (cfb_psnr_ssim_workspace_bytes)");
  switch (a.kind) {
    case IMG_U8: return run<uint8_t>(a, P, ws, st);
    case IMG_U16: return run<uint16_t>(a, P, ws, st);
    case IMG_F32: return run<float>(a, P, ws, st);
    case IMG_F64: return run<double>(a, P, ws, st);
  }
  set_error("cfb_psnr_ssim: unknown element type");
  return 1;
}

}  // namespace cfb
