// CUDA-core (fp32) kernels of the CodeFormer hot path for sm_90a.
//
// Everything here computes in fp32 on NHWC activations.  The dense 3x3 / 1x1 convolutions also have a
// wgmma tensor-core engine (conv_tc.cu); the fp32 implicit GEMM below is the engine for the shapes the
// tensor path does not take (and the cross-check for it in the tests).
//
// Reference semantics implemented (file:line in /root/reference/basicsr/archs):
//   GroupNorm(32,C,1e-6)+swish        vqgan_arch.py:14-20        gn_coef / fused `in_scale,in_shift,in_act`
//   Conv2d 3x3/1x1, Downsample, Upsample vqgan_arch.py:117-138,147-151   conv_f32 (modes SAME/DOWN/UP)
//   AttnBlock / MultiheadAttention core  vqgan_arch.py:209-222, codeformer_arch.py:126   attention
//   LayerNorm, GELU(erf), +pos            codeformer_arch.py:124-133                      layer_norm, OUT_GELU
//   softmax->topk(1)->one-hot@E           codeformer_arch.py:257-259, vqgan_arch.py:72-84 argmax_gather
//   AdaIN                                 codeformer_arch.py:12-43                         adain_nhwc
//   Fuse_sft combine                      codeformer_arch.py:155-156                       conv epilogue (sft_*)
//   VectorQuantizer.forward               vqgan_arch.py:33-70                              vq_nearest
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

__device__ __forceinline__ float silu_f(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float lrelu_f(float x) { return x > 0.f ? x : 0.2f * x; }

// =====================================================================================================
// fp32 implicit-GEMM convolution.  Tile 128 pixels x BN channels x 16 k, 256 threads, 8x(BN/16) per thread.
// =====================================================================================================
constexpr int CF_BM = 128;
constexpr int CF_BK = 16;
constexpr int CF_APITCH = CF_BM + 4;

template <int BN>
__global__ void __launch_bounds__(256) conv_f32_kernel(ConvArgs a) {
  constexpr int TN = BN / 16;  // columns per thread (4 or 8)
  __shared__ __align__(16) float As[2][CF_BK][CF_APITCH];
  __shared__ __align__(16) float Bs[2][CF_BK][BN];

  const int t = threadIdx.x;
  const int64_t M = (int64_t)a.N * a.Ho * a.Wo;
  const int64_t m0 = (int64_t)blockIdx.x * CF_BM;
  const int n0 = blockIdx.y * BN;
  const int taps = a.ksize * a.ksize;
  const int kchunks = a.Cin / CF_BK;
  const int nk = taps * kchunks;

  // ---- A-load role: row = t>>1, 8 consecutive k starting at (t&1)*8
  const int arow = t >> 1;
  const int akq = (t & 1) * 8;
  const int64_t am = m0 + arow;
  const bool arow_ok = am < M;
  int an = 0, aoy = 0, aox = 0;
  if (arow_ok) {
    an = (int)(am / ((int64_t)a.Ho * a.Wo));
    int rem = (int)(am - (int64_t)an * a.Ho * a.Wo);
    aoy = rem / a.Wo;
    aox = rem - aoy * a.Wo;
  }
  const float* in_n = a.in + (int64_t)an * a.H * a.W * a.Cin;
  const float* sc_n = a.in_scale ? a.in_scale + (int64_t)an * a.Cin : nullptr;
  const float* sh_n = a.in_shift ? a.in_shift + (int64_t)an * a.Cin : nullptr;

  // ---- B-load role
  constexpr int BV = (CF_BK * BN / 4) / 256;  // float4 per thread (1 or 2)
  const int bcol = (BN == 128) ? (t & 31) * 4 : (t & 15) * 4;
  const int brow0 = (BN == 128) ? (t >> 5) : (t >> 4);

  float4 ra[2], rb[BV];

  auto load_global = [&](int it) {
    const int tap = it / kchunks;
    const int c0 = (it - tap * kchunks) * CF_BK;
    int r = 0, s = 0;
    if (a.ksize == 3) { r = tap / 3; s = tap - r * 3; }
    bool ok = arow_ok;
    int iy, ix;
    if (a.mode == CONV_DOWN) {
      iy = aoy * 2 + r; ix = aox * 2 + s;
      ok = ok && iy < a.H && ix < a.W;
    } else if (a.mode == CONV_UP) {
      iy = aoy + r - 1; ix = aox + s - 1;
      ok = ok && iy >= 0 && ix >= 0 && iy < 2 * a.H && ix < 2 * a.W;
      iy >>= 1; ix >>= 1;
    } else {
      const int p = a.ksize >> 1;
      iy = aoy + r - p; ix = aox + s - p;
      ok = ok && iy >= 0 && ix >= 0 && iy < a.H && ix < a.W;
    }
    if (ok) {
      const float* p = in_n + ((int64_t)iy * a.W + ix) * a.Cin + c0 + akq;
      ra[0] = __ldg(reinterpret_cast<const float4*>(p));
      ra[1] = __ldg(reinterpret_cast<const float4*>(p + 4));
      if (sc_n) {
        const float4 s0 = __ldg(reinterpret_cast<const float4*>(sc_n + c0 + akq));
        const float4 s1 = __ldg(reinterpret_cast<const float4*>(sc_n + c0 + akq + 4));
        const float4 h0 = __ldg(reinterpret_cast<const float4*>(sh_n + c0 + akq));
        const float4 h1 = __ldg(reinterpret_cast<const float4*>(sh_n + c0 + akq + 4));
        ra[0].x = fmaf(ra[0].x, s0.x, h0.x); ra[0].y = fmaf(ra[0].y, s0.y, h0.y);
        ra[0].z = fmaf(ra[0].z, s0.z, h0.z); ra[0].w = fmaf(ra[0].w, s0.w, h0.w);
        ra[1].x = fmaf(ra[1].x, s1.x, h1.x); ra[1].y = fmaf(ra[1].y, s1.y, h1.y);
        ra[1].z = fmaf(ra[1].z, s1.z, h1.z); ra[1].w = fmaf(ra[1].w, s1.w, h1.w);
      }
      if (a.in_act == IN_SILU) {
        ra[0].x = silu_f(ra[0].x); ra[0].y = silu_f(ra[0].y); ra[0].z = silu_f(ra[0].z); ra[0].w = silu_f(ra[0].w);
        ra[1].x = silu_f(ra[1].x); ra[1].y = silu_f(ra[1].y); ra[1].z = silu_f(ra[1].z); ra[1].w = silu_f(ra[1].w);
      }
    } else {
      ra[0] = make_float4(0.f, 0.f, 0.f, 0.f);
      ra[1] = ra[0];
    }
    const float* wb = a.wgt_f32 + ((int64_t)tap * a.Cin + c0) * a.Cout + n0 + bcol;
#pragma unroll
    for (int i = 0; i < BV; ++i) {
      const int kr = brow0 + i * 8;
      rb[i] = __ldg(reinterpret_cast<const float4*>(wb + (int64_t)kr * a.Cout));
    }
  };
  auto store_smem = [&](int buf) {
    As[buf][akq + 0][arow] = ra[0].x; As[buf][akq + 1][arow] = ra[0].y;
    As[buf][akq + 2][arow] = ra[0].z; As[buf][akq + 3][arow] = ra[0].w;
    As[buf][akq + 4][arow] = ra[1].x; As[buf][akq + 5][arow] = ra[1].y;
    As[buf][akq + 6][arow] = ra[1].z; As[buf][akq + 7][arow] = ra[1].w;
#pragma unroll
    for (int i = 0; i < BV; ++i) {
      const int kr = brow0 + i * 8;
      *reinterpret_cast<float4*>(&Bs[buf][kr][bcol]) = rb[i];
    }
  };

  const int ty = t >> 4, tx = t & 15;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_global(0);
  store_smem(0);
  __syncthreads();
  int buf = 0;
  for (int it = 0; it < nk; ++it) {
    if (it + 1 < nk) load_global(it + 1);
#pragma unroll
    for (int k = 0; k < CF_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[TN];
      {
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
        if (TN == 8) {
          const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][(BN / 2) + tx * 4]);
          bv[TN - 4] = b1.x; bv[TN - 3] = b1.y; bv[TN - 2] = b1.z; bv[TN - 1] = b1.w;
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) store_smem(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4)));
    if (m >= M) continue;
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
      const int col = n0 + h * (BN / 2) + tx * 4;
      float4 v = make_float4(acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]);
      if (a.bias) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(a.bias + col));
        v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
      }
      const int64_t off = m * a.Cout + col;
      if (a.residual) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(a.residual + off));
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      if (a.out_act == OUT_LRELU) {
        v.x = lrelu_f(v.x); v.y = lrelu_f(v.y); v.z = lrelu_f(v.z); v.w = lrelu_f(v.w);
      } else if (a.out_act == OUT_GELU) {
        v.x = gelu_f(v.x); v.y = gelu_f(v.y); v.z = gelu_f(v.z); v.w = gelu_f(v.w);
      }
      if (a.sft_dec) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(a.sft_dec + off));
        const float4 s = __ldg(reinterpret_cast<const float4*>(a.sft_scale + off));
        float sw = a.sft_w;
        if (a.sft_wv) { const float t = __ldg(a.sft_wv + m / ((int64_t)a.Ho * a.Wo)); sw = t > 0.f ? t : 0.f; }
        v.x = d.x + sw * (d.x * s.x + v.x); v.y = d.y + sw * (d.y * s.y + v.y);
        v.z = d.z + sw * (d.z * s.z + v.z); v.w = d.w + sw * (d.w * s.w + v.w);
      }
      *reinterpret_cast<float4*>(a.out + off) = v;
    }
  }
}

int conv_f32(const ConvArgs& a, cudaStream_t st) {
  CFB_REQUIRE(a.Cin % CF_BK == 0, "conv_f32: Cin must be a multiple of 16");
  CFB_REQUIRE(a.Cout % 64 == 0, "conv_f32: Cout must be a multiple of 64");
  CFB_REQUIRE(a.ksize == 1 || a.ksize == 3, "conv_f32: kernel size must be 1 or 3");
  CFB_REQUIRE(a.wgt_f32 && a.in && a.out, "conv_f32: null tensor");
  const int64_t M = (int64_t)a.N * a.Ho * a.Wo;
  if (M == 0) return 0;
  const unsigned gx = (unsigned)((M + CF_BM - 1) / CF_BM);
  if (a.Cout % 128 == 0) {
    conv_f32_kernel<128><<<dim3(gx, a.Cout / 128), 256, 0, st>>>(a);
  } else {
    conv_f32_kernel<64><<<dim3(gx, a.Cout / 64), 256, 0, st>>>(a);
  }
  CFB_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// First conv (3 -> Cout, reads the caller's NCHW image) and last conv (Cin -> 3, writes NCHW).
// =====================================================================================================
// Thread = 4 horizontally adjacent pixels x COUT/4 channels (4 threads cover a pixel quad): every input value and every
// weight read feeds 4 pixels; 16-byte coalesced NHWC stores.
// The caller's image plumbing is u8_to_model_input (kernels.cuh),
// and back (basicsr/utils/img_util.py:66-67,87-90 with min_max=(-1,1)): clamp, (x+1)/2, *255 in fp32, round half to even
__device__ __forceinline__ unsigned model_output_to_u8(float v) {
  float t = fminf(fmaxf(v, -1.f), 1.f);
  t = __fdiv_rn(__fadd_rn(t, 1.f), 2.f);
  return (unsigned)rintf(__fmul_rn(t, 255.f));
}

// U8 = true: x is the caller's uint8 HWC BGR face [N][H][W][3]; the normalisation above is a 256-entry table.
template <int COUT, bool U8>
__global__ void __launch_bounds__(256) conv_first_kernel(const float* __restrict__ x, const float* __restrict__ wgt,
                                                         const float* __restrict__ bias, float* __restrict__ out,
                                                         int N, int H, int W, float* __restrict__ gn_part) {
  __shared__ __align__(16) float ws[27 * COUT];
  __shared__ float bs[COUT];
  __shared__ float lut[U8 ? 256 : 1];
  if constexpr (U8) lut[threadIdx.x] = u8_to_model_input(threadIdx.x);
  pdl_launch_dependents();
  pdl_wait();
  for (int i = threadIdx.x; i < 27 * COUT; i += 256) ws[i] = wgt[i];
  for (int i = threadIdx.x; i < COUT; i += 256) bs[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  constexpr int CPT = COUT / 4;
  const int64_t HW = (int64_t)H * W;
  const int64_t quad = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);      // 64 pixel quads per CTA
  const int cg = threadIdx.x & 3;
  const int64_t pix0 = quad * 4;
  if (pix0 >= (int64_t)N * HW) return;
  const int n = (int)(pix0 / HW);
  const int rem = (int)(pix0 - (int64_t)n * HW);
  const int y = rem / W, x0 = rem - y * W;                                  // W % 4 == 0: the quad shares a row
  float acc[4][CPT];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < CPT; ++j) acc[p][j] = bs[cg * CPT + j];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = y + r - 1;
    const bool rowok = iy >= 0 && iy < H;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v[6];
      if constexpr (U8) {
        const unsigned char* rp8 = reinterpret_cast<const unsigned char*>(x) + ((int64_t)n * HW + (int64_t)iy * W) * 3 + (2 - c);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const int ix = x0 + q - 1;
          v[q] = (rowok && ix >= 0 && ix < W) ? lut[__ldg(rp8 + ix * 3)] : 0.f;
        }
      } else {
        const float* rp = x + ((int64_t)n * 3 + c) * HW + (int64_t)iy * W;
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const int ix = x0 + q - 1;
          v[q] = (rowok && ix >= 0 && ix < W) ? __ldg(rp + ix) : 0.f;
        }
      }
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float* wr = ws + ((r * 3 + s) * 3 + c) * COUT + cg * CPT;
#pragma unroll
        for (int j = 0; j < CPT; j += 4) {
          const float4 w4 = *reinterpret_cast<const float4*>(wr + j);
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            acc[p][j] = fmaf(v[p + s], w4.x, acc[p][j]); acc[p][j + 1] = fmaf(v[p + s], w4.y, acc[p][j + 1]);
            acc[p][j + 2] = fmaf(v[p + s], w4.z, acc[p][j + 2]); acc[p][j + 3] = fmaf(v[p + s], w4.w, acc[p][j + 3]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    float* o = out + (pix0 + p) * COUT + cg * CPT;
#pragma unroll
    for (int j = 0; j < CPT; j += 4) *reinterpret_cast<float4*>(o + j) = make_float4(acc[p][j], acc[p][j + 1], acc[p][j + 2], acc[p][j + 3]);
  }
  if (gn_part != nullptr) {
    // GroupNorm(32) partials of the values just stored, in the layout of the tensor-core epilogue's partials ([slot][32
    // groups][mean, M2], one slot per warp = 32 consecutive pixels; H*W % 256 == 0 keeps a CTA inside one image): the first
    // ResBlock's norm1 then needs no pass over this tensor.  A thread owns 4 pixels x CPT channels = CPT/2 groups of two
    // channels (COUT = 64): their 8 values around the first one, then equal-count merges over the 8 lanes with the same
    // channel slice in a fixed order.
    static_assert(COUT == 64, "GroupNorm partials: two channels per group");
    float gs[CPT / 2], gq[CPT / 2];
#pragma unroll
    for (int g = 0; g < CPT / 2; ++g) {
      const float k = acc[0][2 * g];
      float a = 0.f, b = 0.f;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const float u = acc[p][2 * g] - k, v = acc[p][2 * g + 1] - k;
        a += u + v;
        b += fmaf(u, u, v * v);
      }
      gn_lane_moments(a, b, k, 8.f);
#pragma unroll
      for (int o = 4, n = 8; o < 32; o <<= 1, n <<= 1) gn_merge_xor(a, b, o, (float)n);
      gs[g] = a; gq[g] = b;
    }
    if ((threadIdx.x & 31) < 4) {
      const int64_t slot = pix0 / 32;                       // global slot index = n * (HW / 32) + slot within the image
      float2* dst = reinterpret_cast<float2*>(gn_part) + slot * 32 + cg * (CPT / 2);
#pragma unroll
      for (int g = 0; g < CPT / 2; ++g) dst[g] = make_float2(gs[g], gq[g]);
    }
  }
}

int conv_first(const float* x, const float* wgt, const float* bias, float* out, int N, int H, int W, int Cout,
               cudaStream_t st, float* gn_part) {
  CFB_REQUIRE(Cout == 64, "conv_first: only nf=64 is built");
  CFB_REQUIRE(W % 4 == 0, "conv_first: W must be a multiple of 4");
  const int64_t quads = (int64_t)N * H * W / 4;
  if (quads == 0) return 0;
  CFB_REQUIRE(gn_part == nullptr || ((int64_t)H * W) % 256 == 0, "conv_first: GroupNorm partials need H*W % 256 == 0");
  CFB_LAUNCH_PDL((conv_first_kernel<64, false>), dim3((unsigned)((quads + 63) / 64)), dim3(256), 0, st, x, wgt, bias, out, N, H, W, gn_part);
  return 0;
}
int conv_first_u8(const unsigned char* x_bgr_hwc, const float* wgt, const float* bias, float* out, int N, int H, int W,
                  int Cout, cudaStream_t st, float* gn_part) {
  CFB_REQUIRE(Cout == 64, "conv_first: only nf=64 is built");
  CFB_REQUIRE(W % 4 == 0, "conv_first: W must be a multiple of 4");
  const int64_t quads = (int64_t)N * H * W / 4;
  if (quads == 0) return 0;
  CFB_REQUIRE(gn_part == nullptr || ((int64_t)H * W) % 256 == 0, "conv_first: GroupNorm partials need H*W % 256 == 0");
  CFB_LAUNCH_PDL((conv_first_kernel<64, true>), dim3((unsigned)((quads + 63) / 64)), dim3(256), 0, st,
                 reinterpret_cast<const float*>(x_bgr_hwc), wgt, bias, out, N, H, W, gn_part);
  return 0;
}

// One output pixel per thread, tiles of 4 x 64 pixels.  The GroupNorm-affine input patch of a tile, 6 x 66 pixels x all Cin
// channels, is read once with coalesced loads (a pixel's Cin floats are contiguous) and normalised into shared memory; the
// 9-tap loop then reads it there.  Reading each thread's taps straight from global memory instead (4 pixels 1 KB apart per
// lane and 16 B at a time) fetched every input byte several times over and left the conv far from its DRAM bound.
// The per-pixel sums run in the same order as the plain definition: rows, then channels, then columns, bias first.
constexpr int CL_TH = 4, CL_TW = 64;                 // output tile
constexpr int CL_PH = CL_TH + 2, CL_PW = CL_TW + 2;  // input patch
constexpr int CL_MAX_CIN = 128;                      // shared memory: 9*Cin*16 + 6*66*Cin*4 bytes <= 227 KB
static size_t conv_last_smem(int Cin) { return (size_t)(9 * Cin * 4 + CL_PH * CL_PW * Cin) * sizeof(float); }

// INPAINT (with U8): the blend of inference_inpainting.py:68-75 before the uint8 conversion.  face is the forward's own uint8
// HWC BGR input [N][H][W][3]; only that instantiation reads it.
template <bool U8, bool INPAINT = false>
__global__ void __launch_bounds__(256) conv_last_kernel(const float* __restrict__ in, const float* __restrict__ in_scale,
                                                        const float* __restrict__ in_shift, const float* __restrict__ wgt,
                                                        const float* __restrict__ bias, float* __restrict__ out, int N,
                                                        int H, int W, int Cin, const unsigned char* __restrict__ face) {
  static_assert(U8 || !INPAINT, "conv_last: the inpainting blend writes uint8");
  extern __shared__ __align__(16) float sm[];
  float* ws = sm;                 // [9][Cin][3] padded -> [9][Cin][4]
  // [CL_PH][CL_PW][Cin/4] float4: normalised patch, zero outside the image.  Channel quad q of patch column pc is stored at
  // q ^ (pc & 7): the 8 lanes of one LDS.128 phase read 8 adjacent columns at the same q and hit 8 distinct bank quads.
  float* xs = ws + 9 * Cin * 4;
  const int Q = Cin / 4;
  const int tiles_x = (W + CL_TW - 1) / CL_TW, tiles_y = (H + CL_TH - 1) / CL_TH;
  const int n = (int)(blockIdx.x / (unsigned)(tiles_x * tiles_y));
  const int trem = (int)blockIdx.x - n * tiles_x * tiles_y;
  const int y0 = (trem / tiles_x) * CL_TH, x0 = (trem % tiles_x) * CL_TW;
  pdl_launch_dependents();
  pdl_wait();
  for (int i = threadIdx.x; i < 9 * Cin; i += 256) {
    ws[i * 4 + 0] = wgt[i * 3 + 0]; ws[i * 4 + 1] = wgt[i * 3 + 1]; ws[i * 4 + 2] = wgt[i * 3 + 2]; ws[i * 4 + 3] = 0.f;
  }
  for (int i = threadIdx.x; i < CL_PH * CL_PW * Q; i += 256) {
    const int q = i % Q, pix = i / Q;
    const int pr = pix / CL_PW, pc = pix - pr * CL_PW;
    const int iy = y0 - 1 + pr, ix = x0 - 1 + pc;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);       // zero padding of the *normalised* tensor
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(in + (((int64_t)n * H + iy) * W + ix) * Cin) + q);
      const float4 s4 = in_scale ? __ldg(reinterpret_cast<const float4*>(in_scale + (int64_t)n * Cin) + q) : make_float4(1.f, 1.f, 1.f, 1.f);
      const float4 h4 = in_shift ? __ldg(reinterpret_cast<const float4*>(in_shift + (int64_t)n * Cin) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      v = make_float4(fmaf(t.x, s4.x, h4.x), fmaf(t.y, s4.y, h4.y), fmaf(t.z, s4.z, h4.z), fmaf(t.w, s4.w, h4.w));
    }
    reinterpret_cast<float4*>(xs)[pix * Q + (q ^ (pc & 7))] = v;
  }
  __syncthreads();
  const int tr = threadIdx.x / CL_TW, tc = threadIdx.x % CL_TW;
  const int y = y0 + tr, x = x0 + tc;
  float acc[3];
  acc[0] = bias ? bias[0] : 0.f; acc[1] = bias ? bias[1] : 0.f; acc[2] = bias ? bias[2] : 0.f;
  for (int r = 0; r < 3; ++r) {
    const int iy = y + r - 1;
    if (iy < 0 || iy >= H) continue;
    const float4* prow = reinterpret_cast<const float4*>(xs) + (tr + r) * CL_PW * Q;
    for (int c = 0; c < Cin; c += 4) {
      float4 v[3];
#pragma unroll
      for (int s = 0; s < 3; ++s) v[s] = prow[(tc + s) * Q + ((c >> 2) ^ ((tc + s) & 7))];
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float* wt = ws + ((r * 3 + s) * Cin + c) * 4;
        const float vj[4] = {v[s].x, v[s].y, v[s].z, v[s].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 w4 = *reinterpret_cast<const float4*>(wt + j * 4);
          acc[0] = fmaf(vj[j], w4.x, acc[0]);
          acc[1] = fmaf(vj[j], w4.y, acc[1]);
          acc[2] = fmaf(vj[j], w4.z, acc[2]);
        }
      }
    }
  }
  if (y >= H || x >= W) return;
  const int64_t HW = (int64_t)H * W, pix = (int64_t)y * W + x;
  if constexpr (INPAINT) {
    // mask = (R + G + B of the normalised input == 3), summed in the reference's RGB order; then (1-m)*in + m*out per
    // channel as two fp32 products and one add (no FMA: the reference multiplies and adds separate tensors)
    const unsigned char* f8 = face + ((int64_t)n * HW + pix) * 3;
    const float xi[3] = {u8_to_model_input(__ldg(f8 + 2)), u8_to_model_input(__ldg(f8 + 1)), u8_to_model_input(__ldg(f8 + 0))};
    const float m = __fadd_rn(__fadd_rn(xi[0], xi[1]), xi[2]) == 3.f ? 1.f : 0.f;
    const float keep = __fsub_rn(1.f, m);
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] = __fadd_rn(__fmul_rn(keep, xi[k]), __fmul_rn(m, acc[k]));
  }
  if constexpr (U8) {
    // uint8 HWC BGR
    unsigned char* o8 = reinterpret_cast<unsigned char*>(out) + ((int64_t)n * HW + pix) * 3;
    o8[0] = (unsigned char)model_output_to_u8(acc[2]); o8[1] = (unsigned char)model_output_to_u8(acc[1]);
    o8[2] = (unsigned char)model_output_to_u8(acc[0]);
  } else {
    float* o = out + (int64_t)n * 3 * HW + pix;
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k * HW] = acc[k];
  }
}

template <bool U8, bool INPAINT = false>
static int launch_conv_last(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
                            float* out, int N, int H, int W, int Cin, cudaStream_t st, const unsigned char* face = nullptr) {
  CFB_REQUIRE(Cin % 32 == 0 && Cin <= CL_MAX_CIN, "conv_last: Cin must be a multiple of 32 and at most 128");
  if (N == 0 || H == 0 || W == 0) return 0;
  // the patch needs more than the default 48 KB of dynamic shared memory: a per-device property of the function
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(attr_done.load(std::memory_order_acquire) & bit)) {
    CFB_CUDA(cudaFuncSetAttribute(conv_last_kernel<U8, INPAINT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)conv_last_smem(CL_MAX_CIN)));
    attr_done.fetch_or(bit, std::memory_order_release);
  }
  const int64_t tiles = (int64_t)N * ((H + CL_TH - 1) / CL_TH) * ((W + CL_TW - 1) / CL_TW);
  CFB_REQUIRE(tiles <= 0x7fffffffLL, "conv_last: too many tiles");
  CFB_LAUNCH_PDL((conv_last_kernel<U8, INPAINT>), dim3((unsigned)tiles), dim3(256), conv_last_smem(Cin), st, in, in_scale, in_shift,
                 wgt, bias, out, N, H, W, Cin, face);
  return 0;
}

int conv_last(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
              float* out, int N, int H, int W, int Cin, cudaStream_t st) {
  return launch_conv_last<false>(in, in_scale, in_shift, wgt, bias, out, N, H, W, Cin, st);
}
int conv_last_u8(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
                 unsigned char* out_bgr_hwc, int N, int H, int W, int Cin, cudaStream_t st) {
  return launch_conv_last<true>(in, in_scale, in_shift, wgt, bias, reinterpret_cast<float*>(out_bgr_hwc), N, H, W, Cin, st);
}
int conv_last_u8_inpaint(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
                         const unsigned char* face_bgr_hwc, unsigned char* out_bgr_hwc, int N, int H, int W, int Cin,
                         cudaStream_t st) {
  CFB_REQUIRE(face_bgr_hwc != nullptr, "conv_last: the inpainting blend needs the input faces");
  return launch_conv_last<true, true>(in, in_scale, in_shift, wgt, bias, reinterpret_cast<float*>(out_bgr_hwc), N, H, W, Cin, st,
                                      face_bgr_hwc);
}

// stand-alone plumbing (unit parity + callers that want the fp32 tensor): uint8 HWC BGR <-> fp32 NCHW RGB in [-1,1]
__global__ void u8_to_input_kernel(const unsigned char* __restrict__ img, float* __restrict__ x, int64_t HW, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / (3 * HW);
    const int64_t r = i - n * 3 * HW;
    const int c = (int)(r / HW);
    const int64_t px = r - (int64_t)c * HW;
    x[i] = u8_to_model_input(img[(n * HW + px) * 3 + (2 - c)]);
  }
}
__global__ void output_to_u8_kernel(const float* __restrict__ x, unsigned char* __restrict__ img, int64_t HW, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / (3 * HW);
    const int64_t r = i - n * 3 * HW;
    const int64_t px = r / 3;
    const int k = (int)(r - px * 3);
    img[i] = (unsigned char)model_output_to_u8(x[(n * 3 + (2 - k)) * HW + px]);
  }
}
int u8_to_input(const unsigned char* img_bgr_hwc, float* x_nchw, int N, int64_t HW, cudaStream_t st) {
  const int64_t total = (int64_t)N * 3 * HW;
  if (total == 0) return 0;
  u8_to_input_kernel<<<(unsigned)((total + 255) / 256 > 148 * 16 ? 148 * 16 : (total + 255) / 256), 256, 0, st>>>(img_bgr_hwc, x_nchw, HW, total);
  CFB_LAUNCH_CHECK();
  return 0;
}
int output_to_u8(const float* x_nchw, unsigned char* img_bgr_hwc, int N, int64_t HW, cudaStream_t st) {
  const int64_t total = (int64_t)N * 3 * HW;
  if (total == 0) return 0;
  output_to_u8_kernel<<<(unsigned)((total + 255) / 256 > 148 * 16 ? 148 * 16 : (total + 255) / 256), 256, 0, st>>>(x_nchw, img_bgr_hwc, HW, total);
  CFB_LAUNCH_CHECK();
  return 0;
}

__global__ void relayout_oihw_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int k) {
  const int64_t total = (int64_t)Cout * Cin * k * k;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    // i indexes out [tap][ci][co]
    const int co = (int)(i % Cout);
    const int ci = (int)((i / Cout) % Cin);
    const int tap = (int)(i / ((int64_t)Cout * Cin));
    out[i] = w[((int64_t)co * Cin + ci) * k * k + tap];
  }
}
int relayout_oihw_to_tck(const float* oihw, float* out, int Cout, int Cin, int k, cudaStream_t st) {
  const int64_t total = (int64_t)Cout * Cin * k * k;
  relayout_oihw_kernel<<<(unsigned)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256), 256, 0, st>>>(oihw, out, Cout,
                                                                                                          Cin, k);
  CFB_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// GroupNorm statistics (deterministic two-stage reduction) folded into per-(n,c) scale/shift.
// =====================================================================================================
static inline int gn_chunk_pixels(int HW) { return HW < 2048 ? HW : 2048; }
size_t gn_workspace_bytes(int N, int HW, int C) {
  const int chunks = HW / gn_chunk_pixels(HW);
  return (size_t)N * chunks * 32 * 2 * sizeof(double);
}

// The sums are fp64 from the first value on: a thread adds up to 1024 pixels, and fp32 sums of squares of a group whose mean
// is r times its standard deviation would lose the variance like (1 + r^2) * 2^-24 (the kernel stays bound by its loads).
__global__ void __launch_bounds__(256) gn_partial_kernel(const float* __restrict__ x, double* __restrict__ part, int HW,
                                                         int C, int CP, int groups) {
  __shared__ double ssum[256 * 4];
  __shared__ double ssq[256 * 4];
  __shared__ double csum[1024];
  __shared__ double csq[1024];
  const int t = threadIdx.x;
  const int C4 = C >> 2;
  const int PL = 256 / C4;
  const int c4 = t % C4, pl = t / C4;
  const int chunk = blockIdx.x, n = blockIdx.y, chunks = gridDim.x;
  const float* base = x + ((int64_t)n * HW + (int64_t)chunk * CP) * C + c4 * 4;
  double s[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
  for (int p = pl; p < CP; p += PL) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(base + (int64_t)p * C));
    const double a = v.x, b = v.y, c = v.z, d = v.w;
    s[0] += a; s[1] += b; s[2] += c; s[3] += d;
    q[0] = fma(a, a, q[0]); q[1] = fma(b, b, q[1]); q[2] = fma(c, c, q[2]); q[3] = fma(d, d, q[3]);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { ssum[pl * C + c4 * 4 + j] = s[j]; ssq[pl * C + c4 * 4 + j] = q[j]; }
  __syncthreads();
  for (int c = t; c < C; c += 256) {
    double a = 0.0, b = 0.0;
    for (int l = 0; l < PL; ++l) { a += ssum[l * C + c]; b += ssq[l * C + c]; }
    csum[c] = a; csq[c] = b;
  }
  __syncthreads();
  if (t < groups) {
    const int cpg = C / groups;
    double a = 0.0, b = 0.0;
    for (int c = 0; c < cpg; ++c) { a += csum[t * cpg + c]; b += csq[t * cpg + c]; }
    double* o = part + (((int64_t)n * chunks + chunk) * groups + t) * 2;
    o[0] = a; o[1] = b;
  }
}

__global__ void gn_final_kernel(const double* __restrict__ part, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float* __restrict__ scale, float* __restrict__ shift,
                                int HW, int C, int chunks, int groups, float eps) {
  __shared__ double gmean[64], grstd[64];
  const int n = blockIdx.x, t = threadIdx.x;
  const int cpg = C / groups;
  if (t < groups) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < chunks; ++k) {
      const double* p = part + (((int64_t)n * chunks + k) * groups + t) * 2;
      a += p[0]; b += p[1];
    }
    const double cnt = (double)HW * cpg;
    const double mean = a / cnt;
    double var = b / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    gmean[t] = mean;
    grstd[t] = 1.0 / sqrt(var + (double)eps);
  }
  __syncthreads();
  for (int c = t; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double sc = grstd[g] * (double)gamma[c];
    scale[(int64_t)n * C + c] = (float)sc;
    shift[(int64_t)n * C + c] = (float)((double)beta[c] - gmean[g] * sc);
  }
}

int gn_coef(const float* x, const float* gamma, const float* beta, float* scale, float* shift, int N, int HW, int C,
            int groups, float eps, void* ws, cudaStream_t st) {
  CFB_REQUIRE(C % 4 == 0 && (C / 4) <= 256 && 256 % (C / 4) == 0, "gn_coef: C must be 4*divisor of 256");
  CFB_REQUIRE(groups <= 64 && C % groups == 0, "gn_coef: bad group count");
  const int CP = gn_chunk_pixels(HW);
  CFB_REQUIRE(HW % CP == 0, "gn_coef: H*W must be a multiple of the chunk size");
  if (N == 0) return 0;
  const int chunks = HW / CP;
  gn_partial_kernel<<<dim3(chunks, N), 256, 0, st>>>(x, (double*)ws, HW, C, CP, groups);
  CFB_LAUNCH_CHECK();
  gn_final_kernel<<<N, 256, 0, st>>>((const double*)ws, gamma, beta, scale, shift, HW, C, chunks, groups, eps);
  CFB_LAUNCH_CHECK();
  return 0;
}

// GroupNorm finalize from the conv epilogue's per-tile partial sums.  A 512x512 image has 8192 partial slots (2 MB): one CTA
// per image was latency-bound (11 us per call, 72 calls per forward = 10 % of a single-face forward), so the slots of an
// image are split over G CTAs; each reduces its contiguous range in a fixed order into fp64, publishes 64 doubles, and the
// LAST CTA of the image to finish (ticket counter) adds the G partials in index order and writes scale / shift.  The
// summation tree depends only on (slots, G(slots)) -- not on the batch, not on which CTA happens to be last -- so the result
// is deterministic and batch-invariant.  Counters are zero on entry and reset by the last CTA.
__host__ __device__ inline int gn_final_split(int slots) {
  int g = slots / 256;
  return g < 1 ? 1 : (g > 16 ? 16 : g);
}
__global__ void __launch_bounds__(256) gn_final_f32_kernel(const float* __restrict__ part, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, float* __restrict__ scale,
                                                           float* __restrict__ shift, int HW, int C, int slots, float eps,
                                                           double* __restrict__ part2, unsigned* __restrict__ counters) {
  __shared__ double ps[8][33], pq[8][33];
  __shared__ double gmean[32], grstd[32];
  __shared__ int is_last;
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y, G = gridDim.x, blk = blockIdx.x, t = threadIdx.x;
  const int g = t & 31, stripe = t >> 5;
  const int per = (slots + G - 1) / G;
  const int lo = blk * per, hi = min(slots, lo + per);
  const int cpg = C / 32;
  // slot k holds (mean_k, M2_k) of m values.  With the image's slot 0 mean K as a shift, d_k = mean_k - K:
  //   a = sum d_k,  b = sum (M2_k + m d_k^2) = sum over all values of (x - K)^2
  // so that mean = K + a / slots and var = b / (slots m) - (a / slots)^2 cancel only at the spread of the slot means
  const float2* base = reinterpret_cast<const float2*>(part) + (int64_t)n * slots * 32 + g;
  const double K = (double)__ldg(base).x, m = (double)HW * cpg / slots;
  double a = 0.0, b = 0.0;
  int k = lo + stripe;
  for (; k + 24 < hi; k += 32) {     // 4 independent loads in flight
    const float2 v0 = __ldg(base + (int64_t)k * 32), v1 = __ldg(base + (int64_t)(k + 8) * 32);
    const float2 v2 = __ldg(base + (int64_t)(k + 16) * 32), v3 = __ldg(base + (int64_t)(k + 24) * 32);
    const double d0 = (double)v0.x - K, d1 = (double)v1.x - K, d2 = (double)v2.x - K, d3 = (double)v3.x - K;
    a += (d0 + d1) + (d2 + d3);
    b += (fma(m * d0, d0, (double)v0.y) + fma(m * d1, d1, (double)v1.y)) + (fma(m * d2, d2, (double)v2.y) + fma(m * d3, d3, (double)v3.y));
  }
  for (; k < hi; k += 8) {
    const float2 v = __ldg(base + (int64_t)k * 32);
    const double d = (double)v.x - K;
    a += d; b += fma(m * d, d, (double)v.y);
  }
  ps[stripe][g] = a; pq[stripe][g] = b;
  __syncthreads();
  double sa = 0.0, sb = 0.0;
  if (t < 32) {
    for (int s = 0; s < 8; ++s) { sa += ps[s][t]; sb += pq[s][t]; }
  }
  if (G > 1) {
    if (t < 32) {
      double* dst = part2 + ((int64_t)n * G + blk) * 64;
      dst[2 * t] = sa; dst[2 * t + 1] = sb;
      __threadfence();
    }
    __syncthreads();
    if (t == 0) is_last = (atomicAdd(counters + n, 1u) == (unsigned)(G - 1));
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (t < 32) {
      sa = 0.0; sb = 0.0;
      const double* src = part2 + (int64_t)n * G * 64;
      for (int q = 0; q < G; ++q) { sa += __ldcg(src + q * 64 + 2 * t); sb += __ldcg(src + q * 64 + 2 * t + 1); }
    }
    if (t == 0) counters[n] = 0u;
  }
  if (t < 32) {
    const double dm = sa / slots;
    double var = sb / ((double)HW * cpg) - dm * dm;
    if (var < 0.0) var = 0.0;
    gmean[t] = K + dm;                   // t < 32: K is group t's
    grstd[t] = 1.0 / sqrt(var + (double)eps);
  }
  __syncthreads();
  for (int c = t; c < C; c += 256) {
    const int gg = c / cpg;
    const double sc = grstd[gg] * (double)gamma[c];
    scale[(int64_t)n * C + c] = (float)sc;
    shift[(int64_t)n * C + c] = (float)((double)beta[c] - gmean[gg] * sc);
  }
}
size_t gn_final_scratch_bytes(int N, int slots) {
  const int G = gn_final_split(slots);
  return G > 1 ? (size_t)N * G * 64 * sizeof(double) : 0;
}
int gn_coef_from_partials(const float* part, int slots, const float* gamma, const float* beta, float* scale, float* shift,
                          int N, int HW, int C, int groups, float eps, void* scratch, unsigned* counters, cudaStream_t st) {
  CFB_REQUIRE(groups == 32 && C % 32 == 0, "gn_coef_from_partials: 32 groups only");
  CFB_REQUIRE(slots > 0 && (int64_t)slots * 32 == HW, "gn_coef_from_partials: a slot holds 32 pixels of the image");
  if (N == 0) return 0;
  const int G = gn_final_split(slots);
  CFB_REQUIRE(G == 1 || (scratch && counters), "gn_coef_from_partials: scratch / counters missing");
  CFB_REQUIRE(N <= 65535, "gn_coef_from_partials: batch too large");
  CFB_LAUNCH_PDL(gn_final_f32_kernel, dim3(G, N), dim3(256), 0, st, part, gamma, beta, scale, shift, HW, C, slots, eps, (double*)scratch,
                 counters);
  return 0;
}

__global__ void gn_cat_partials_kernel(const float2* __restrict__ a, const float2* __restrict__ b, float2* __restrict__ out,
                                       int64_t total, float half_cnt) {
  // group g of the concatenated tensor = two adjacent groups of one source: channels/group doubles, 32 groups stay.  The two
  // (mean, M2) of cnt values each merge as  mean = (mu + mv) / 2,  M2 = M2u + M2v + (mu - mv)^2 * cnt / 2
  pdl_launch_dependents();
  pdl_wait();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(i & 31);
    const int64_t slot = i >> 5;
    const float2* src = (g < 16) ? a + slot * 32 + 2 * g : b + slot * 32 + 2 * (g - 16);
    const float2 u = __ldg(src), v = __ldg(src + 1);
    const float d = u.x - v.x;
    out[i] = make_float2(0.5f * (u.x + v.x), (u.y + v.y) + (d * d) * half_cnt);
  }
}
int gn_cat_partials(const float* a_part, const float* b_part, float* out_part, int64_t total_slots, int C, cudaStream_t st) {
  CFB_REQUIRE(C % 32 == 0, "gn_cat_partials: 32 groups of C channels");
  const int64_t total = total_slots * 32;
  if (total == 0) return 0;
  const int64_t blocks = (total + 255) / 256;
  // a slot of a source group holds 32 pixels x C/32 channels = C values
  CFB_LAUNCH_PDL(gn_cat_partials_kernel, dim3((unsigned)(blocks > 2048 ? 2048 : blocks)), dim3(256), 0, st, (const float2*)a_part,
                 (const float2*)b_part, (float2*)out_part, total, 0.5f * (float)C);
  return 0;
}

__global__ void affine_act_kernel(const float4* __restrict__ x, const float* __restrict__ scale,
                                  const float* __restrict__ shift, float4* __restrict__ y, int64_t total4, int64_t HWC4,
                                  int C, int act) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / HWC4);
    const int c = (int)((i * 4) % C);
    float4 v = __ldg(x + i);
    if (scale) {
      const float4 s = __ldg(reinterpret_cast<const float4*>(scale + (int64_t)n * C + c));
      const float4 h = __ldg(reinterpret_cast<const float4*>(shift + (int64_t)n * C + c));
      v.x = fmaf(v.x, s.x, h.x); v.y = fmaf(v.y, s.y, h.y); v.z = fmaf(v.z, s.z, h.z); v.w = fmaf(v.w, s.w, h.w);
    }
    if (act == IN_SILU) { v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w); }
    y[i] = v;
  }
}
int affine_act(const float* x, const float* scale, const float* shift, float* y, int N, int HW, int C, int act,
               cudaStream_t st) {
  CFB_REQUIRE(C % 4 == 0, "affine_act: C must be a multiple of 4");
  const int64_t total4 = (int64_t)N * HW * C / 4;
  if (total4 == 0) return 0;
  const int64_t blocks = (total4 + 255) / 256;
  affine_act_kernel<<<(unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks), 256, 0, st>>>(
      (const float4*)x, scale, shift, (float4*)y, total4, (int64_t)HW * C / 4, C, act);
  CFB_LAUNCH_CHECK();
  return 0;
}

__device__ __forceinline__ void split_store4(__half* __restrict__ hi, __half* __restrict__ lo, int64_t off, const float4& o);

// =====================================================================================================
// Attention core: out = softmax(q k^T * scale) v, S = 256 keys, one CTA per (32 queries, head, batch).
// =====================================================================================================
constexpr int AT_S = 256;
constexpr int AT_QB = 32;

template <int D>
__global__ void __launch_bounds__(256) attention_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                        const float* __restrict__ v, float* __restrict__ out, int q_pitch,
                                                        int k_pitch, int v_pitch, int o_pitch, float scale,
                                                        __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;                       // [32 dd][32 q]
  float* Ks = Qs + 32 * AT_QB;          // [32 dd][256 keys]
  float* P = Ks + 32 * AT_S;            // [32 q][256 keys]
  const int t = threadIdx.x;
  const int q0 = blockIdx.x * AT_QB, h = blockIdx.y, b = blockIdx.z;
  const int qg = t >> 5, kg = t & 31;  // 4 queries x 8 keys per thread
  const float* qb = q + ((int64_t)b * AT_S + q0) * q_pitch + h * D;
  const float* kb = k + ((int64_t)b * AT_S) * k_pitch + h * D;
  const float* vb = v + ((int64_t)b * AT_S) * v_pitch + h * D;

  float s[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) s[i][j] = 0.f;

  for (int d0 = 0; d0 < D; d0 += 32) {
    {  // Q chunk: thread -> query t/8, 4 dd
      const int qi = t >> 3, dd4 = (t & 7) * 4;
      const float4 v4 = __ldg(reinterpret_cast<const float4*>(qb + (int64_t)qi * q_pitch + d0 + dd4));
      Qs[(dd4 + 0) * AT_QB + qi] = v4.x; Qs[(dd4 + 1) * AT_QB + qi] = v4.y;
      Qs[(dd4 + 2) * AT_QB + qi] = v4.z; Qs[(dd4 + 3) * AT_QB + qi] = v4.w;
    }
    {  // K chunk: thread -> key t, 32 dd
      const float* kr = kb + (int64_t)t * k_pitch + d0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 v4 = __ldg(reinterpret_cast<const float4*>(kr + j * 4));
        Ks[(j * 4 + 0) * AT_S + t] = v4.x; Ks[(j * 4 + 1) * AT_S + t] = v4.y;
        Ks[(j * 4 + 2) * AT_S + t] = v4.z; Ks[(j * 4 + 3) * AT_S + t] = v4.w;
      }
    }
    __syncthreads();
#pragma unroll 8
    for (int dd = 0; dd < 32; ++dd) {
      const float4 q4 = *reinterpret_cast<const float4*>(Qs + dd * AT_QB + qg * 4);
      const float4 ka = *reinterpret_cast<const float4*>(Ks + dd * AT_S + kg * 4);
      const float4 kc = *reinterpret_cast<const float4*>(Ks + dd * AT_S + 128 + kg * 4);
      const float qv[4] = {q4.x, q4.y, q4.z, q4.w};
      const float kv[8] = {ka.x, ka.y, ka.z, ka.w, kc.x, kc.y, kc.z, kc.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float* pr = P + (qg * 4 + i) * AT_S;
    *reinterpret_cast<float4*>(pr + kg * 4) = make_float4(s[i][0] * scale, s[i][1] * scale, s[i][2] * scale, s[i][3] * scale);
    *reinterpret_cast<float4*>(pr + 128 + kg * 4) =
        make_float4(s[i][4] * scale, s[i][5] * scale, s[i][6] * scale, s[i][7] * scale);
  }
  __syncthreads();
  // softmax: warp w -> rows 4w..4w+3
  {
    const int w = t >> 5, l = t & 31;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* pr = P + (w * 4 + i) * AT_S;
      float vals[8];
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) { vals[j] = pr[l + 32 * j]; mx = fmaxf(mx, vals[j]); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) { vals[j] = expf(vals[j] - mx); sum += vals[j]; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.f / sum;
#pragma unroll
      for (int j = 0; j < 8; ++j) pr[l + 32 * j] = vals[j] * inv;
    }
  }
  __syncthreads();
  // out = P V
  constexpr int C4 = D / 4;
  constexpr int QPT = (AT_QB * C4) / 256;  // queries per thread: 2 (D=64) or 16 (D=512)
  const int c4 = t % C4, qs = (t / C4) * QPT;
  float acc[QPT][4];
#pragma unroll
  for (int i = 0; i < QPT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  for (int j = 0; j < AT_S; j += 4) {
    float4 vv[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) vv[jj] = __ldg(reinterpret_cast<const float4*>(vb + (int64_t)(j + jj) * v_pitch + c4 * 4));
#pragma unroll
    for (int i = 0; i < QPT; ++i) {
      const float4 p4 = *reinterpret_cast<const float4*>(P + (qs + i) * AT_S + j);
      const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        acc[i][0] = fmaf(pv[jj], vv[jj].x, acc[i][0]); acc[i][1] = fmaf(pv[jj], vv[jj].y, acc[i][1]);
        acc[i][2] = fmaf(pv[jj], vv[jj].z, acc[i][2]); acc[i][3] = fmaf(pv[jj], vv[jj].w, acc[i][3]);
      }
    }
  }
  const int64_t obase = ((int64_t)b * AT_S + q0) * o_pitch + h * D + c4 * 4;
#pragma unroll
  for (int i = 0; i < QPT; ++i) {
    const float4 o = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    const int64_t off = obase + (int64_t)(qs + i) * o_pitch;
    if (out) *reinterpret_cast<float4*>(out + off) = o;
    if (out_hi) split_store4(out_hi, out_lo, off, o);      // operand planes of the out_proj linear (values are convex
  }                                                         // combinations of v: inside the fp16 range whenever v is)
}

int attention(const float* q, const float* k, const float* v, float* out, int B, int S, int heads, int d, int q_pitch,
              int k_pitch, int v_pitch, int o_pitch, float scale, cudaStream_t st, void* out_planes) {
  CFB_REQUIRE(S == AT_S, "attention: token count must be 256 (16x16 latent)");
  CFB_REQUIRE(d == 64 || d == 512, "attention: head width must be 64 or 512");
  if (B == 0) return 0;
  const size_t smem = (size_t)(32 * AT_QB + 32 * AT_S + AT_QB * AT_S) * sizeof(float);
  // the opt-in is a per-device property of the function (several GPUs may be driven from one process)
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(attr_done.load(std::memory_order_acquire) & bit)) {
    CFB_CUDA(cudaFuncSetAttribute(attention_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CFB_CUDA(cudaFuncSetAttribute(attention_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done.fetch_or(bit, std::memory_order_release);
  }
  dim3 grid(S / AT_QB, heads, B);
  __half* ohi = (__half*)out_planes;
  __half* olo = out_planes ? (__half*)((char*)out_planes + (((size_t)B * S * o_pitch * 2 + 1023) / 1024 * 1024)) : nullptr;
  CFB_REQUIRE(out || out_planes, "attention: no output");
  if (d == 64)
    attention_kernel<64><<<grid, 256, smem, st>>>(q, k, v, out, q_pitch, k_pitch, v_pitch, o_pitch, scale, ohi, olo);
  else
    attention_kernel<512><<<grid, 256, smem, st>>>(q, k, v, out, q_pitch, k_pitch, v_pitch, o_pitch, scale, ohi, olo);
  CFB_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// LayerNorm (eps 1e-5), warp per row; optional second output y2 = y + pos[row % pos_rows]
// =====================================================================================================
__device__ __forceinline__ void split_store4(__half* __restrict__ hi, __half* __restrict__ lo, int64_t off, const float4& o) {
  const __half2 h01 = __floats2half2_rn(o.x, o.y), h23 = __floats2half2_rn(o.z, o.w);
  const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  const __half2 l01 = __floats2half2_rn(o.x - f01.x, o.y - f01.y), l23 = __floats2half2_rn(o.z - f23.x, o.w - f23.y);
  uint2 ph, pl;
  ph.x = *reinterpret_cast<const uint32_t*>(&h01); ph.y = *reinterpret_cast<const uint32_t*>(&h23);
  pl.x = *reinterpret_cast<const uint32_t*>(&l01); pl.y = *reinterpret_cast<const uint32_t*>(&l23);
  *reinterpret_cast<uint2*>(hi + off) = ph;
  *reinterpret_cast<uint2*>(lo + off) = pl;
}

// PLANES: y / y2 are written as fp16 hi/lo operand planes (hi = rn(v), lo = rn(v - hi)) for the tensor-core linears that
// consume them -- the LayerNorm output of a TransformerSALayer is only ever a GEMM operand (codeformer_arch.py:124-131),
// so no fp32 copy and no separate operand-preparation pass exist on that path.  |LN output| reaches |gamma| sqrt(C - 1) + |beta|:
// a value past the fp16 range (65504) sets the overflow bit of the status word (`status`, host-mapped), as every other
// producer of operand planes does -- never a silent inf / NaN operand.
template <int C, bool PLANES>
__global__ void __launch_bounds__(256) layer_norm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float* __restrict__ y,
                                                         float* __restrict__ y2, const float* __restrict__ pos,
                                                         int pos_rows, int rows, int64_t plane_elems, unsigned* status) {
  constexpr int V = C / 128;  // float4 per lane
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (int64_t)row * C;
  float4 v[V];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = __ldg(reinterpret_cast<const float4*>(xr + (i * 32 + l) * 4));
    sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum * (1.f / C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    sq += (a * a + b * b) + (c * c + d * d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq * (1.f / C) + 1e-5f);
  float vmax = 0.f;                          // PLANES: largest |value| written to the operand planes
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int c = (i * 32 + l) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c));
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + bb.x; o.y = (v[i].y - mean) * rstd * g.y + bb.y;
    o.z = (v[i].z - mean) * rstd * g.z + bb.z; o.w = (v[i].w - mean) * rstd * g.w + bb.w;
    const int64_t off = (int64_t)row * C + c;
    if (PLANES) {
      if (y) {
        split_store4(reinterpret_cast<__half*>(y), reinterpret_cast<__half*>(y) + plane_elems, off, o);
        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
      }
    } else {
      *reinterpret_cast<float4*>(y + off) = o;
    }
    if (y2) {
      const float4 p = __ldg(reinterpret_cast<const float4*>(pos + (int64_t)(row % pos_rows) * C + c));
      const float4 o2 = make_float4(o.x + p.x, o.y + p.y, o.z + p.z, o.w + p.w);
      if (PLANES) {
        split_store4(reinterpret_cast<__half*>(y2), reinterpret_cast<__half*>(y2) + plane_elems, off, o2);
        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(o2.x), fabsf(o2.y)), fmaxf(fabsf(o2.z), fabsf(o2.w))));
      } else {
        *reinterpret_cast<float4*>(y2 + off) = o2;
      }
    }
  }
  if (PLANES && vmax > 65504.f && status) { atomicOr_system(status, CFB_STATUS_OVERFLOW); __threadfence_system(); }
}
int layer_norm(const float* x, const float* gamma, const float* beta, float* y, float* y2, const float* pos,
               int pos_rows, int rows, int C, cudaStream_t st) {
  CFB_REQUIRE(C == 512, "layer_norm: only dim_embd=512 is built");
  if (rows == 0) return 0;
  CFB_LAUNCH_PDL((layer_norm_kernel<512, false>), dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, st, x, gamma, beta, y, y2, pos,
                 pos_rows > 0 ? pos_rows : 1, rows, (int64_t)0, (unsigned*)nullptr);
  return 0;
}
// outputs as fp16 hi/lo operand planes: [hi plane | lo plane], each align1024(rows*C*2) bytes (the conv engine's layout)
int layer_norm_planes(const float* x, const float* gamma, const float* beta, void* y_planes, void* y2_planes, const float* pos,
                      int pos_rows, int rows, int C, cudaStream_t st) {
  CFB_REQUIRE(C == 512, "layer_norm: only dim_embd=512 is built");
  if (rows == 0) return 0;
  unsigned* status = nullptr;
  CFB_CHECK(async_status_word(&status));
  const int64_t plane_elems = (int64_t)((((size_t)rows * C * 2 + 1023) / 1024 * 1024) / 2);
  CFB_LAUNCH_PDL((layer_norm_kernel<512, true>), dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, st, x, gamma, beta, (float*)y_planes,
                 (float*)y2_planes, pos, pos_rows > 0 ? pos_rows : 1, rows, plane_elems, status);
  return 0;
}

// =====================================================================================================
// Code lookup: argmax over logits (first maximum), gather codebook row
// =====================================================================================================
__global__ void __launch_bounds__(256) argmax_gather_kernel(const float* __restrict__ logits,
                                                            const float* __restrict__ codebook, int64_t* __restrict__ idx,
                                                            float* __restrict__ quant, int T, int K, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (tok >= T) return;
  const float* lr = logits + (int64_t)tok * K;
  // A row of NaN / -inf logits never satisfies `v > best`: the index then stays at a VALID position (this lane's first
  // column), like torch.topk, instead of indexing the codebook out of bounds (a NaN in must not become a sticky fault).
  float best = -INFINITY;
  int bi = l < K ? l : 0;
  for (int i = l; i < K; i += 32) {
    const float v = __ldg(lr + i);
    if (v > best) { best = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  bi = min(max(bi, 0), K - 1);
  if (l == 0 && idx) idx[tok] = (int64_t)bi;
  if (quant) {
    const float* e = codebook + (int64_t)bi * D;
    for (int c = l * 4; c < D; c += 128)
      *reinterpret_cast<float4*>(quant + (int64_t)tok * D + c) = __ldg(reinterpret_cast<const float4*>(e + c));
  }
}
int argmax_gather(const float* logits, const float* codebook, int64_t* idx, float* quant, int T, int K, int D,
                  cudaStream_t st) {
  CFB_REQUIRE(D % 4 == 0, "argmax_gather: D must be a multiple of 4");
  if (T == 0) return 0;
  CFB_LAUNCH_PDL(argmax_gather_kernel, dim3((unsigned)((T + 7) / 8)), dim3(256), 0, st, logits, codebook, idx, quant, T, K, D);
  return 0;
}

__global__ void gather_rows_kernel(const int64_t* __restrict__ idx, const float* __restrict__ codebook,
                                   float* __restrict__ out, int T, int K, int D) {
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (tok >= T) return;
  int64_t i = idx[tok];
  if (i < 0) i = 0;
  if (i >= K) i = K - 1;
  for (int c = l * 4; c < D; c += 128)
    *reinterpret_cast<float4*>(out + (int64_t)tok * D + c) = __ldg(reinterpret_cast<const float4*>(codebook + i * D + c));
}
int gather_rows(const int64_t* idx, const float* codebook, float* out, int T, int K, int D, cudaStream_t st) {
  if (T == 0) return 0;
  gather_rows_kernel<<<(T + 7) / 8, 256, 0, st>>>(idx, codebook, out, T, K, D);
  CFB_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// AdaIN on NHWC [B,HW,C]: per (b,c) mean / unbiased var (+1e-5) of both tensors
// =====================================================================================================
// Statistics are accumulated in double and then rounded to fp32, and the elementwise part replays the reference's
// fp32 operation order with explicit (non-contracted) roundings.  Reason: when most tokens of a face pick the same
// code a content channel is nearly constant, (x - mean)/std then amplifies a 1e-7 error of the mean by 1/std
// (observed 3e-5 relative on quant_feat with sequential fp32 sums); an accurately rounded mean reproduces the
// reference's own fp32 value and the rest is IEEE-deterministic.
// One CTA = 32 channels of one image: lane = channel (128-byte coalesced rows), 8 warps = 8 token stripes; every stripe sum
// and the 8-stripe combine run in a fixed order, so the result does not depend on the batch or the launch.
__global__ void __launch_bounds__(256) adain_kernel(const float* __restrict__ content, const float* __restrict__ style,
                                                    float* __restrict__ out, int HW, int C) {
  __shared__ double red[2][8][33];
  __shared__ float stat[4][32];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, c = blockIdx.x * 32 + (threadIdx.x & 31), stripe = threadIdx.x >> 5, l = threadIdx.x & 31;
  const bool ok = c < C;
  const float* cp = content + (int64_t)b * HW * C + c;
  const float* sp = style + (int64_t)b * HW * C + c;
  double cs = 0.0, ss = 0.0;
  if (ok)
    for (int p = stripe; p < HW; p += 8) { cs += (double)__ldg(cp + (int64_t)p * C); ss += (double)__ldg(sp + (int64_t)p * C); }
  red[0][stripe][l] = cs; red[1][stripe][l] = ss;
  __syncthreads();
  double cmd = 0.0, smd = 0.0;
  for (int k = 0; k < 8; ++k) { cmd += red[0][k][l]; smd += red[1][k][l]; }
  cmd /= HW; smd /= HW;
  __syncthreads();
  double cv = 0.0, sv = 0.0;
  if (ok)
    for (int p = stripe; p < HW; p += 8) {
      const double a = (double)__ldg(cp + (int64_t)p * C) - cmd, d = (double)__ldg(sp + (int64_t)p * C) - smd;
      cv += a * a; sv += d * d;
    }
  red[0][stripe][l] = cv; red[1][stripe][l] = sv;
  __syncthreads();
  if (stripe == 0) {
    double cvt = 0.0, svt = 0.0;
    for (int k = 0; k < 8; ++k) { cvt += red[0][k][l]; svt += red[1][k][l]; }
    stat[0][l] = (float)cmd; stat[1][l] = (float)smd;
    stat[2][l] = sqrtf(__fadd_rn((float)(cvt / (HW - 1)), 1e-5f));    // calc_mean_std: var(unbiased) + eps, sqrt
    stat[3][l] = sqrtf(__fadd_rn((float)(svt / (HW - 1)), 1e-5f));
  }
  __syncthreads();
  if (!ok) return;
  const float cm = stat[0][l], sm = stat[1][l], cstd = stat[2][l], sstd = stat[3][l];
  for (int p = stripe; p < HW; p += 8) {
    const float nrm = __fdiv_rn(__fsub_rn(__ldg(cp + (int64_t)p * C), cm), cstd);      // (content - mean) / std
    out[(int64_t)b * HW * C + (int64_t)p * C + c] = __fadd_rn(__fmul_rn(nrm, sstd), sm);   // * style_std + style_mean
  }
}
int adain_nhwc(const float* content, const float* style, float* out, int B, int HW, int C, cudaStream_t st) {
  if (B == 0) return 0;
  CFB_REQUIRE(B <= 65535, "adain: batch too large");
  CFB_LAUNCH_PDL(adain_kernel, dim3((unsigned)((C + 31) / 32), (unsigned)B), dim3(256), 0, st, content, style, out, HW, C);
  return 0;
}

// =====================================================================================================
// layout plumbing
// =====================================================================================================
// in [n][R][Cc] -> out [n][Cc][R]  (32x32 smem tiles)
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cc) {
  __shared__ float tile[32][33];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.z;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const float* ib = in + (int64_t)n * R * Cc;
  float* ob = out + (int64_t)n * R * Cc;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < R && c < Cc) tile[i][threadIdx.x] = ib[(int64_t)r * Cc + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < Cc) ob[(int64_t)c * R + r] = tile[threadIdx.x][i];
  }
}
static int transpose_batched(const float* in, float* out, int n, int R, int Cc, cudaStream_t st) {
  if (n == 0 || R == 0 || Cc == 0) return 0;
  dim3 grid((Cc + 31) / 32, (R + 31) / 32, n);
  CFB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "transpose: tensor too large");
  CFB_LAUNCH_PDL(transpose_kernel, grid, dim3(32, 8), 0, st, in, out, R, Cc);
  return 0;
}
int nchw_to_nhwc(const float* in, float* out, int N, int C, int HW, cudaStream_t st) {
  return transpose_batched(in, out, N, C, HW, st);
}
int nhwc_to_nchw(const float* in, float* out, int N, int C, int HW, cudaStream_t st) {
  return transpose_batched(in, out, N, HW, C, st);
}

__global__ void concat_kernel(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ out,
                              int64_t pixels, int Ca4, int Cb4) {
  const int64_t total = pixels * (Ca4 + Cb4);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / (Ca4 + Cb4);
    const int c = (int)(i - p * (Ca4 + Cb4));
    out[i] = (c < Ca4) ? __ldg(a + p * Ca4 + c) : __ldg(b + p * Cb4 + (c - Ca4));
  }
}
int concat_channels(const float* a, const float* b, float* out, int64_t pixels, int Ca, int Cb, cudaStream_t st) {
  CFB_REQUIRE(Ca % 4 == 0 && Cb % 4 == 0, "concat: channels must be multiples of 4");
  const int64_t total = pixels * (Ca + Cb) / 4;
  if (total == 0) return 0;
  const int64_t blocks = (total + 255) / 256;
  concat_kernel<<<(unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks), 256, 0, st>>>((const float4*)a, (const float4*)b,
                                                                                   (float4*)out, pixels, Ca / 4, Cb / 4);
  CFB_LAUNCH_CHECK();
  return 0;
}

// Fidelity sweep: buffer d holds B faces of d.bytes each, back to back; face b goes to faces b*K .. b*K+K-1 of its
// destination.  Each 16-byte vector is read once and stored K times.  grid: (x-stride over a face, buffer, source face).
__global__ void expand_faces_kernel(const __grid_constant__ ExpandList L, int B, int K) {
  pdl_launch_dependents();
  pdl_wait();
  const ExpandCopy& d = L.d[blockIdx.y];
  const int64_t nv = d.bytes / 16;
  for (int b = blockIdx.z; b < B; b += gridDim.z) {
    const uint4* src = (const uint4*)d.src + (int64_t)b * nv;
    uint4* dst = (uint4*)d.dst + (int64_t)b * K * nv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
      const uint4 v = __ldg(src + i);
      for (int k = 0; k < K; ++k) dst[(int64_t)k * nv + i] = v;
    }
  }
}
int expand_faces(const ExpandList& L, int B, int K, cudaStream_t st) {
  CFB_REQUIRE(L.n >= 0 && L.n <= EXPAND_MAX, "expand_faces: too many buffers");
  if (B == 0 || L.n == 0) return 0;
  int64_t big = 0;
  for (int i = 0; i < L.n; ++i) {
    const ExpandCopy& d = L.d[i];
    CFB_REQUIRE(d.bytes % 16 == 0 && (uintptr_t)d.src % 16 == 0 && (uintptr_t)d.dst % 16 == 0,
                "expand_faces: buffers must be 16-byte aligned, with a multiple of 16 bytes per face");
    big = std::max(big, d.bytes / 16);
  }
  // about 8 vectors per thread of the largest buffer; the small buffers' surplus blocks exit at once
  const int64_t gx = std::min<int64_t>(std::max<int64_t>((big + 2047) / 2048, 1), 512);
  CFB_LAUNCH_PDL(expand_faces_kernel, dim3((unsigned)gx, (unsigned)L.n, (unsigned)std::min(B, 65535)), dim3(256), 0, st, L, B, K);
  return 0;
}

__global__ void add_pos_kernel(const float4* __restrict__ x, const float4* __restrict__ pos, float4* __restrict__ y,
                               int64_t total4, int64_t pos4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 a = __ldg(x + i), p = __ldg(pos + (i % pos4));
    y[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
  }
}
int add_pos(const float* x, const float* pos, float* y, int rows, int pos_rows, int C, cudaStream_t st) {
  const int64_t total4 = (int64_t)rows * C / 4;
  if (total4 == 0) return 0;
  add_pos_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, st>>>((const float4*)x, (const float4*)pos, (float4*)y, total4,
                                                                   (int64_t)pos_rows * C / 4);
  CFB_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// VectorQuantizer.forward: d = |z|^2 + |e|^2 - 2 z.e ; argmin (first minimum) by warp shuffle over
// shared-memory codebook tiles; straight-through z_q; loss / perplexity / mean_distance.
// One CTA = 32 tokens; codebook streamed in tiles of 256 codes x 32 dims.
// =====================================================================================================
constexpr int VQ_TB = 32;
struct VqWs {
  float* e2;        // [K]
  double* part;     // [ctas][2]  (sum of squared error, sum of distances)
  unsigned* hist;   // [K]
};
static VqWs vq_carve(void* ws, int T, int D, int K) {
  VqWs w;
  char* p = (char*)ws;
  w.e2 = (float*)p; p += ((size_t)K * sizeof(float) + 255) / 256 * 256;
  w.part = (double*)p; p += ((size_t)((T + VQ_TB - 1) / VQ_TB) * 2 * sizeof(double) + 255) / 256 * 256;
  w.hist = (unsigned*)p;
  return w;
}
size_t vq_workspace_bytes(int T, int D, int K) {
  return ((size_t)K * 4 + 255) / 256 * 256 + ((size_t)((T + VQ_TB - 1) / VQ_TB) * 16 + 255) / 256 * 256 + (size_t)K * 4 + 256;
}

__global__ void vq_e2_kernel(const float* __restrict__ E, float* __restrict__ e2, unsigned* __restrict__ hist, int K, int D) {
  const int code = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (code >= K) return;
  float s = 0.f;
  for (int c = l; c < D; c += 32) { const float v = E[(int64_t)code * D + c]; s = fmaf(v, v, s); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (l == 0) { e2[code] = s; hist[code] = 0u; }
}

__global__ void __launch_bounds__(256) vq_nearest_kernel(const float* __restrict__ z, const float* __restrict__ E,
                                                         const float* __restrict__ e2, int T, int D, int K,
                                                         int64_t* __restrict__ idx, float* __restrict__ zq,
                                                         double* __restrict__ part, unsigned* __restrict__ hist) {
  __shared__ __align__(16) float Zs[32 * VQ_TB];     // [32 dd][32 tok]
  __shared__ __align__(16) float Es[32 * 256];       // [32 dd][256 codes]
  __shared__ float z2s[VQ_TB];
  __shared__ int best_idx[VQ_TB];
  __shared__ double red[8][2];
  const int t = threadIdx.x;
  const int tok0 = blockIdx.x * VQ_TB;
  const int qg = t >> 5, kg = t & 31;

  // |z|^2 per token: warp w -> tokens 4w..4w+3
  {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int tok = tok0 + qg * 4 + i;
      float s = 0.f;
      if (tok < T)
        for (int c = kg; c < D; c += 32) { const float v = z[(int64_t)tok * D + c]; s = fmaf(v, v, s); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (kg == 0) z2s[qg * 4 + i] = s;
    }
  }
  __syncthreads();

  float bestd[4];
  int besti[4];
  double dsum = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) { bestd[i] = INFINITY; besti[i] = K - 1; }

  for (int k0 = 0; k0 < K; k0 += 256) {
    float s[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) s[i][j] = 0.f;
    for (int d0 = 0; d0 < D; d0 += 32) {
      {
        const int qi = t >> 3, dd4 = (t & 7) * 4;
        const int tok = tok0 + qi;
        float4 v4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tok < T) v4 = __ldg(reinterpret_cast<const float4*>(z + (int64_t)tok * D + d0 + dd4));
        Zs[(dd4 + 0) * VQ_TB + qi] = v4.x; Zs[(dd4 + 1) * VQ_TB + qi] = v4.y;
        Zs[(dd4 + 2) * VQ_TB + qi] = v4.z; Zs[(dd4 + 3) * VQ_TB + qi] = v4.w;
      }
      {
        const int code = k0 + t;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float4 v4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (code < K) v4 = __ldg(reinterpret_cast<const float4*>(E + (int64_t)code * D + d0 + j * 4));
          Es[(j * 4 + 0) * 256 + t] = v4.x; Es[(j * 4 + 1) * 256 + t] = v4.y;
          Es[(j * 4 + 2) * 256 + t] = v4.z; Es[(j * 4 + 3) * 256 + t] = v4.w;
        }
      }
      __syncthreads();
      float c[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) c[i][j] = 0.f;
#pragma unroll 8
      for (int dd = 0; dd < 32; ++dd) {
        const float4 q4 = *reinterpret_cast<const float4*>(Zs + dd * VQ_TB + qg * 4);
        const float4 ka = *reinterpret_cast<const float4*>(Es + dd * 256 + kg * 4);
        const float4 kc = *reinterpret_cast<const float4*>(Es + dd * 256 + 128 + kg * 4);
        const float qv[4] = {q4.x, q4.y, q4.z, q4.w};
        const float kv[8] = {ka.x, ka.y, ka.z, ka.w, kc.x, kc.y, kc.z, kc.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) c[i][j] = fmaf(qv[i], kv[j], c[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[i][j] += c[i][j];   // chunked accumulation keeps the rounding error small
      __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int code = k0 + ((j < 4) ? (kg * 4 + j) : (128 + kg * 4 + (j - 4)));
      if (code >= K) continue;
      const float ee = __ldg(e2 + code);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float d = (z2s[qg * 4 + i] + ee) - 2.f * s[i][j];
        if (tok0 + qg * 4 + i < T) dsum += (double)d;
        if (d < bestd[i] || (d == bestd[i] && code < besti[i])) { bestd[i] = d; besti[i] = code; }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, bestd[i], o);
      const int oi = __shfl_xor_sync(0xffffffffu, besti[i], o);
      if (od < bestd[i] || (od == bestd[i] && oi < besti[i])) { bestd[i] = od; besti[i] = oi; }
    }
    if (kg == 0) best_idx[qg * 4 + i] = min(max(besti[i], 0), K - 1);   // all-NaN rows: a valid index, never out of bounds
  }
  __syncthreads();
  // outputs: idx, straight-through z_q, squared error, histogram
  double se = 0.0;
  for (int i = 0; i < 4; ++i) {
    const int tl = qg * 4 + i, tok = tok0 + tl;
    if (tok >= T) continue;
    const int bi = best_idx[tl];
    if (kg == 0) {
      idx[tok] = (int64_t)bi;
      atomicAdd(hist + bi, 1u);
    }
    for (int c = kg; c < D; c += 32) {
      const float zz = z[(int64_t)tok * D + c];
      const float e = __ldg(E + (int64_t)bi * D + c);
      const float diff = e - zz;
      se += (double)(diff * diff);
      zq[(int64_t)tok * D + c] = zz + diff;   // z + (z_q - z), vqgan_arch.py:57
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
  }
  if (kg == 0) { red[qg][0] = se; red[qg][1] = dsum; }
  __syncthreads();
  if (t == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < 8; ++w) { a += red[w][0]; b += red[w][1]; }
    part[blockIdx.x * 2] = a;
    part[blockIdx.x * 2 + 1] = b;
  }
}

__global__ void vq_final_kernel(const double* __restrict__ part, const unsigned* __restrict__ hist, int ctas, int T, int D,
                                int K, float beta, float* __restrict__ stats) {
  __shared__ double sred[256];
  const int t = threadIdx.x;
  double ent = 0.0;
  for (int k = t; k < K; k += 256) {
    const float em = (float)hist[k] / (float)T;
    ent += (double)(em * logf(em + 1e-10f));
  }
  sred[t] = ent;
  __syncthreads();
  if (t == 0) {
    double e = 0.0;
    for (int i = 0; i < 256; ++i) e += sred[i];
    double se = 0.0, ds = 0.0;
    for (int i = 0; i < ctas; ++i) { se += part[i * 2]; ds += part[i * 2 + 1]; }
    const float mse = (float)(se / ((double)T * D));
    stats[0] = mse + beta * mse;            // vqgan_arch.py:55
    stats[1] = expf(-(float)e);             // perplexity, :60-61
    stats[2] = (float)(ds / ((double)T * K));  // mean_distance, :42
    stats[3] = 0.f;
  }
}

__global__ void onehot_kernel(const int64_t* __restrict__ idx, float* __restrict__ onehot, int T, int K) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < T) onehot[(int64_t)i * K + idx[i]] = 1.f;
}

int vq_nearest(const float* z, const float* codebook, int T, int D, int K, float beta, int64_t* idx, float* zq,
               float* stats, float* onehot, void* ws, cudaStream_t st) {
  CFB_REQUIRE(D % 32 == 0, "vq_nearest: emb_dim must be a multiple of 32");
  if (T == 0) return 0;
  VqWs w = vq_carve(ws, T, D, K);
  const int ctas = (T + VQ_TB - 1) / VQ_TB;
  vq_e2_kernel<<<(K + 7) / 8, 256, 0, st>>>(codebook, w.e2, w.hist, K, D);
  CFB_LAUNCH_CHECK();
  vq_nearest_kernel<<<ctas, 256, 0, st>>>(z, codebook, w.e2, T, D, K, idx, zq, w.part, w.hist);
  CFB_LAUNCH_CHECK();
  vq_final_kernel<<<1, 256, 0, st>>>(w.part, w.hist, ctas, T, D, K, beta, stats);
  CFB_LAUNCH_CHECK();
  if (onehot) {
    CFB_CUDA(cudaMemsetAsync(onehot, 0, (size_t)T * K * sizeof(float), st));
    onehot_kernel<<<(T + 255) / 256, 256, 0, st>>>(idx, onehot, T, K);
    CFB_LAUNCH_CHECK();
  }
  return 0;
}

// ---- VectorQuantizer on the tensor-core path: the distance GEMM z.E^T comes from the wgmma engine (1x1 conv with the
// codebook as weights); this kernel forms d = |z|^2 + |e|^2 - 2 z.e, takes the first minimum (warp shuffle), and emits
// the straight-through z_q, squared error, distance sum and histogram.  One warp per token, 8 tokens per CTA.
__global__ void __launch_bounds__(256) vq_select_kernel(const float* __restrict__ z, const float* __restrict__ E,
                                                        const float* __restrict__ e2, const float* __restrict__ dots, int T,
                                                        int D, int K, int64_t* __restrict__ idx, float* __restrict__ zq,
                                                        double* __restrict__ part, unsigned* __restrict__ hist) {
  __shared__ double red[8][2];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int tok = blockIdx.x * 8 + w;
  double se = 0.0, dsum = 0.0;
  if (tok < T) {
    float z2 = 0.f;
    for (int c = l; c < D; c += 32) { const float v = z[(int64_t)tok * D + c]; z2 = fmaf(v, v, z2); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z2 += __shfl_xor_sync(0xffffffffu, z2, o);
    float best = INFINITY;
    int bi = l < K ? l : 0;                 // NaN / +inf distances keep a valid index (no out-of-bounds gather or histogram write)
    const float* dr = dots + (int64_t)tok * K;
    for (int k = l; k < K; k += 32) {
      const float d = (z2 + __ldg(e2 + k)) - 2.f * __ldg(dr + k);
      dsum += (double)d;
      if (d < best) { best = d; bi = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (od < best || (od == best && oi < bi)) { best = od; bi = oi; }
    }
    bi = min(max(bi, 0), K - 1);
    if (l == 0) { idx[tok] = (int64_t)bi; atomicAdd(hist + bi, 1u); }
    for (int c = l; c < D; c += 32) {
      const float zz = z[(int64_t)tok * D + c];
      const float diff = __ldg(E + (int64_t)bi * D + c) - zz;
      se += (double)(diff * diff);
      zq[(int64_t)tok * D + c] = zz + diff;      // z + (z_q - z), vqgan_arch.py:57
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { se += __shfl_xor_sync(0xffffffffu, se, o); dsum += __shfl_xor_sync(0xffffffffu, dsum, o); }
  if (l == 0) { red[w][0] = se; red[w][1] = dsum; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < 8; ++i) { a += red[i][0]; b += red[i][1]; }
    part[blockIdx.x * 2] = a; part[blockIdx.x * 2 + 1] = b;
  }
}

size_t vq_select_workspace_bytes(int T, int K) {
  return ((size_t)K * 4 + 255) / 256 * 256 + ((size_t)((T + 7) / 8) * 16 + 255) / 256 * 256 + (size_t)K * 4 + 256;
}
int vq_select_from_dots(const float* z, const float* codebook, const float* dots, int T, int D, int K, float beta, int64_t* idx,
                        float* zq, float* stats, float* onehot, void* ws, cudaStream_t st) {
  if (T == 0) return 0;
  char* p = (char*)ws;
  float* e2 = (float*)p; p += ((size_t)K * 4 + 255) / 256 * 256;
  double* part = (double*)p; p += ((size_t)((T + 7) / 8) * 16 + 255) / 256 * 256;
  unsigned* hist = (unsigned*)p;
  const int ctas = (T + 7) / 8;
  vq_e2_kernel<<<(K + 7) / 8, 256, 0, st>>>(codebook, e2, hist, K, D);
  CFB_LAUNCH_CHECK();
  vq_select_kernel<<<ctas, 256, 0, st>>>(z, codebook, e2, dots, T, D, K, idx, zq, part, hist);
  CFB_LAUNCH_CHECK();
  vq_final_kernel<<<1, 256, 0, st>>>(part, hist, ctas, T, D, K, beta, stats);
  CFB_LAUNCH_CHECK();
  if (onehot) {
    CFB_CUDA(cudaMemsetAsync(onehot, 0, (size_t)T * K * sizeof(float), st));
    onehot_kernel<<<(T + 255) / 256, 256, 0, st>>>(idx, onehot, T, K);
    CFB_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace cfb

// =====================================================================================================
// Thin convolutions of the caller-side networks (SURVEY.md section 8 rows f3 / f4): the first conv of RRDBNet / ParseNet
// (a few image channels -> 64 features, reads the caller's NCHW image, optional pixel-unshuffle) and their last convs
// (64 features -> a few channels, writes NCHW).  ~1 % of those networks' FLOPs: plain CUDA-core kernels, any H x W.
//   /root/reference/basicsr/archs/rrdbnet_arch.py:89,96,101-108,118   /root/reference/basicsr/archs/arch_util.py:190-206
//   /root/reference/facelib/parsing/parsenet.py:93-105,166,188-189
// =====================================================================================================
namespace cfb {

__device__ __forceinline__ int pad_index(int i, int n, int mode, bool& inside) {
  inside = (unsigned)i < (unsigned)n;
  if (inside || mode == 0) return i;
  if (mode == 1) i = i < 0 ? -i : 2 * n - 2 - i;      // ReflectionPad2d
  i = min(max(i, 0), n - 1);                          // replicate / degenerate sizes
  inside = true;
  return i;
}

// Image sources of conv_thin_in: value of image channel c at row y, column x (before pixel_unshuffle) of batch element n.
struct NchwSrc {                 // x [N, Cimg, Hi, Wi] fp32
  const float* x; int Cimg, Hi, Wi;
  __device__ __forceinline__ float operator()(int n, int c, int y, int x_) const {
    return __ldg(x + (((int64_t)n * Cimg + c) * Hi + y) * Wi + x_);
  }
};

// Index of row / column i of an image of n rows after F.pad(.., (0, p), 'reflect') (p < n): the bottom / right pad only.
__device__ __forceinline__ int reflect_tail(int i, int n) { return i < n ? i : 2 * (n - 1) - i; }

// img.astype(np.float32) of one element of a uint8 / uint16 / float32 / float64 image (float64: round to nearest)
__device__ __forceinline__ float img_f32(unsigned char v) { return (float)v; }
__device__ __forceinline__ float img_f32(unsigned short v) { return (float)v; }
__device__ __forceinline__ float img_f32(float v) { return v; }
__device__ __forceinline__ float img_f32(double v) { return __double2float_rn(v); }

// The tiles of RealESRGANer.pre_process + tile_process read from HWC BGR source images of element type T
// (realesrgan_utils.py:71-175): element n is the window at (in_y, in_x) of image `img` after the pre_pad reflect pad (bottom /
// right) and the reflect pad to the pixel-unshuffle multiple; the value is the reference's float32 img / max_range (an IEEE
// division), BGR -> RGB.  range: per-image max_range (image_max_range), or nullptr for 255.
template <class T>
struct TileSrc {
  const T* img; int H, W, Hp, Wp;                    // source size, size after the pre_pad (Hp = H + pre_pad)
  const int* range;
  RrdbU8Tiles tab;                                   // by value: the table travels in the launch's parameters
  __device__ __forceinline__ float operator()(int n, int c, int y, int x_) const {
    const RrdbU8Tile& t = tab.t[n];
    const int sy = reflect_tail(reflect_tail(t.in_y + y, Hp), H), sx = reflect_tail(reflect_tail(t.in_x + x_, Wp), W);
    const float div = range ? (float)__ldg(range + t.img) : 255.f;
    return __fdiv_rn(img_f32(__ldg(img + (((int64_t)t.img * H + sy) * W + sx) * 3 + (2 - c))), div);
  }
};

// ParseNet's input read from uint8 HWC BGR faces [N, H, W, 3] (cfb_parsenet_masks_u8): img2tensor(face / 255.) + normalize(0.5,
// 0.5) of face_restoration_helper.py:458-460, BGR -> RGB, the value cfb_u8_to_input writes (u8_to_model_input).
struct U8FaceSrc {
  const unsigned char* img; int H, W;
  __device__ __forceinline__ float operator()(int n, int c, int y, int x_) const {
    return u8_to_model_input(__ldg(img + (((int64_t)n * H + y) * W + x_) * 3 + (2 - c)));
  }
};

// x [N, Cimg, H*us, W*us] (read through Src) -> out [N, H, W, out_pitch] (channels out_c0 .. out_c0+63), 3x3 pad 1.
// us > 1: pixel_unshuffle(x, us) first -- channel c*us*us + dy*us + dx of the conv input is x[c][y*us+dy][x*us+dx].
// weights: [tap][cin][64] (relayout_oihw_to_tck).
template <class Src>
__global__ void __launch_bounds__(256) conv_thin_in_kernel(const Src x, const float* __restrict__ wgt,
                                                           const float* __restrict__ bias, float* __restrict__ out, int N, int H,
                                                           int W, int Cimg, int us, int pad_mode, int out_pitch, int out_c0) {
  extern __shared__ __align__(16) float wsm[];       // [9 * Cin][64]
  const int Cin = Cimg * us * us;
  for (int i = threadIdx.x; i < 9 * Cin * 64; i += 256) wsm[i] = wgt[i];
  __syncthreads();
  const int cq = threadIdx.x & 15;                   // 4 output channels
  const int64_t pix = (int64_t)blockIdx.x * 16 + (threadIdx.x >> 4);
  if (pix >= (int64_t)N * H * W) return;
  const int n = (int)(pix / ((int64_t)H * W));
  const int rem = (int)(pix - (int64_t)n * H * W);
  const int oy = rem / W, ox = rem - oy * W;
  float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias + cq * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = 0; r < 3; ++r) {
    bool iny;
    const int iy = pad_index(oy + r - 1, H, pad_mode, iny);
    for (int s = 0; s < 3; ++s) {
      bool inx;
      const int ix = pad_index(ox + s - 1, W, pad_mode, inx);
      if (!(iny && inx)) continue;
      for (int ci = 0; ci < Cin; ++ci) {
        const int c = ci / (us * us), d = ci - c * us * us, dy = d / us, dx = d - dy * us;
        const float v = x(n, c, iy * us + dy, ix * us + dx);
        const float4 w4 = *reinterpret_cast<const float4*>(wsm + ((r * 3 + s) * Cin + ci) * 64 + cq * 4);
        acc.x = fmaf(v, w4.x, acc.x); acc.y = fmaf(v, w4.y, acc.y); acc.z = fmaf(v, w4.z, acc.z); acc.w = fmaf(v, w4.w, acc.w);
      }
    }
  }
  *reinterpret_cast<float4*>(out + pix * out_pitch + out_c0 + cq * 4) = acc;
}
template <class Src>
static int launch_thin_in(const Src& x, const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int Cimg, int us,
                          int pad_mode, int out_pitch, int out_c0, cudaStream_t st) {
  const int Cin = Cimg * us * us;
  CFB_REQUIRE(Cin >= 1 && Cin <= 48 && out_pitch % 4 == 0 && out_c0 % 4 == 0, "conv_thin_in: at most 48 input channels");
  const int64_t M = (int64_t)N * H * W;
  if (M == 0) return 0;
  const size_t smem = (size_t)9 * Cin * 64 * sizeof(float);
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load() & (1ull << (dev & 63)))) {
    CFB_CUDA(cudaFuncSetAttribute(conv_thin_in_kernel<Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, 9 * 48 * 64 * 4));
    attr_done.fetch_or(1ull << (dev & 63));
  }
  conv_thin_in_kernel<Src><<<(unsigned)((M + 15) / 16), 256, smem, st>>>(x, wgt_tck, bias, out, N, H, W, Cimg, us, pad_mode, out_pitch, out_c0);
  CFB_LAUNCH_CHECK();
  return 0;
}
int conv_thin_in(const float* x_nchw, const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int Cimg, int us,
                 int pad_mode, int out_pitch, int out_c0, cudaStream_t st) {
  return launch_thin_in(NchwSrc{x_nchw, Cimg, H * us, W * us}, wgt_tck, bias, out, N, H, W, Cimg, us, pad_mode, out_pitch, out_c0, st);
}
template <class T>
static int thin_in_tiles(const void* img, const int* range, int img_h, int img_w, int pre_pad, const RrdbU8Tiles& tiles,
                         const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int us, int out_pitch, int out_c0,
                         cudaStream_t st) {
  const TileSrc<T> x{(const T*)img, img_h, img_w, img_h + pre_pad, img_w + pre_pad, range, tiles};
  return launch_thin_in(x, wgt_tck, bias, out, N, H, W, 3, us, 0, out_pitch, out_c0, st);
}
int conv_thin_in_tiles(const void* img_bgr_hwc, int in_kind, const int* max_range, int img_h, int img_w, int pre_pad,
                       const RrdbU8Tiles& tiles, const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int us,
                       int out_pitch, int out_c0, cudaStream_t st) {
  CFB_REQUIRE(N <= RrdbU8Tiles::kMax, "conv_thin_in_tiles: too many tiles for one launch");
  CFB_REQUIRE(in_kind >= IMG_U8 && in_kind <= IMG_F64, "conv_thin_in_tiles: unknown image kind");
  switch (in_kind) {
    case IMG_U8: return thin_in_tiles<unsigned char>(img_bgr_hwc, max_range, img_h, img_w, pre_pad, tiles, wgt_tck, bias, out, N, H,
                                                     W, us, out_pitch, out_c0, st);
    case IMG_U16: return thin_in_tiles<unsigned short>(img_bgr_hwc, max_range, img_h, img_w, pre_pad, tiles, wgt_tck, bias, out, N,
                                                       H, W, us, out_pitch, out_c0, st);
    case IMG_F32: return thin_in_tiles<float>(img_bgr_hwc, max_range, img_h, img_w, pre_pad, tiles, wgt_tck, bias, out, N, H, W, us,
                                              out_pitch, out_c0, st);
    default: return thin_in_tiles<double>(img_bgr_hwc, max_range, img_h, img_w, pre_pad, tiles, wgt_tck, bias, out, N, H, W, us,
                                          out_pitch, out_c0, st);
  }
}

// max_range of image_max_range: bit 0 of flags[i] = some element of image i above 256, bit 1 = some NaN
template <class T>
__global__ void __launch_bounds__(256) image_range_flags_kernel(const T* __restrict__ img, int64_t count, int* __restrict__ flags) {
  const T* p = img + (int64_t)blockIdx.y * count;
  bool big = false, nan = false;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < count; i += (int64_t)gridDim.x * 256) {
    const float v = img_f32(__ldg(p + i));
    big |= v > 256.f;
    nan |= v != v;
  }
  big = __any_sync(0xffffffffu, big);
  nan = __any_sync(0xffffffffu, nan);
  if ((threadIdx.x & 31) == 0 && (big || nan)) atomicOr(flags + blockIdx.y, (big ? 1 : 0) | (nan ? 2 : 0));
}
__global__ void image_range_finish_kernel(int* r, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r[i] = r[i] == 1 ? 65535 : 255;
}
template <class T>
static void launch_range_flags(const void* img, int n, int64_t count, int* flags, cudaStream_t st) {
  const unsigned gx = (unsigned)std::min<int64_t>((count + 256 * 8 - 1) / (256 * 8), 256);
  image_range_flags_kernel<T><<<dim3(gx, n), 256, 0, st>>>((const T*)img, count, flags);
}
int image_max_range(const void* images, int kind, int n, int64_t count, int* max_range, cudaStream_t st) {
  CFB_REQUIRE(n >= 0 && n <= 65535 && count > 0, "image_max_range: bad image batch");
  CFB_REQUIRE(kind >= IMG_U8 && kind <= IMG_F64, "image_max_range: unknown image kind");
  if (n == 0) return 0;
  CFB_CUDA(cudaMemsetAsync(max_range, 0, (size_t)n * sizeof(int), st));
  switch (kind) {
    case IMG_U8: launch_range_flags<unsigned char>(images, n, count, max_range, st); break;
    case IMG_U16: launch_range_flags<unsigned short>(images, n, count, max_range, st); break;
    case IMG_F32: launch_range_flags<float>(images, n, count, max_range, st); break;
    default: launch_range_flags<double>(images, n, count, max_range, st); break;
  }
  CFB_LAUNCH_CHECK();
  image_range_finish_kernel<<<(n + 255) / 256, 256, 0, st>>>(max_range, n);
  CFB_LAUNCH_CHECK();
  return 0;
}
int conv_thin_in_u8_faces(const unsigned char* faces_bgr_hwc, const float* wgt_tck, const float* bias, float* out, int N, int H, int W,
                          int pad_mode, int out_pitch, int out_c0, cudaStream_t st) {
  return launch_thin_in(U8FaceSrc{faces_bgr_hwc, H, W}, wgt_tck, bias, out, N, H, W, 3, 1, pad_mode, out_pitch, out_c0, st);
}

// Destinations of conv_thin_out: `wants` selects the output pixels to compute, `store` writes one pixel's Cout values.
struct NchwDst {                 // out [N, Cout, H, W] fp32
  float* out;
  __device__ __forceinline__ bool wants(int, int, int) const { return true; }
  template <int CP>
  __device__ __forceinline__ void store(int n, int oy, int ox, int H, int W, int Cout, const float (&acc)[CP]) const {
    for (int c = 0; c < Cout; ++c) out[(((int64_t)n * Cout + c) * H + oy) * W + ox] = acc[c];
  }
};

// The crop-back of tile_process and post_process with the reference's integer conversion (realesrgan_utils.py:147-186,
// 203-243): pixel (oy, ox) of tile n is kept when it lies in the tile's crop and its canvas position (out + offset into the
// crop) lies inside the out_h x out_w canvas of image `img` (the mod pad and pre_pad rows / columns fall outside); it is
// written as HWC BGR of element type T: clamp to [0, 1], float32 * max_range, round half to even, saturated to T.
// range: per-image max_range (image_max_range), or nullptr for 255.
template <class T>
struct TileDst {
  T* canvas; int out_h, out_w;
  const int* range;
  RrdbU8Tiles tab;
  __device__ __forceinline__ bool pos(int n, int oy, int ox, int& Y, int& X) const {
    const RrdbU8Tile& t = tab.t[n];
    const int cy = oy - t.crop_y, cx = ox - t.crop_x;
    Y = t.out_y + cy; X = t.out_x + cx;
    return (unsigned)cy < (unsigned)t.crop_h && (unsigned)cx < (unsigned)t.crop_w && Y < out_h && X < out_w;
  }
  __device__ __forceinline__ bool wants(int n, int oy, int ox) const { int Y, X; return pos(n, oy, ox, Y, X); }
  template <int CP>
  __device__ __forceinline__ void store(int n, int oy, int ox, int, int, int, const float (&acc)[CP]) const {
    int Y, X;
    pos(n, oy, ox, Y, X);
    const int img = tab.t[n].img;
    const float mul = range ? (float)__ldg(range + img) : 255.f;
    const float top = sizeof(T) == 1 ? 255.f : 65535.f;
    T* px = canvas + (((int64_t)img * out_h + Y) * out_w + X) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) px[2 - c] = (T)fminf(rintf(__fmul_rn(fminf(fmaxf(acc[c], 0.f), 1.f), mul)), top);
  }
};

// ParseNet's logits reduced in registers (cfb_parsenet_masks_u8): out.argmax(dim=1) and the MASK_COLORMAP byte of
// face_restoration_helper.py:463-468, uint8 [N, H, W] each (either may be NULL).  The comparison and tie rule are
// parse_argmax_kernel's (first maximum, strict >; a NaN first logit stays class 0), so the bytes equal the unfused chain's.
struct ArgmaxU8Dst {
  unsigned char* cls; unsigned char* mask;
  __device__ __forceinline__ bool wants(int, int, int) const { return true; }
  template <int CP>
  __device__ __forceinline__ void store(int n, int oy, int ox, int H, int W, int Cout, const float (&acc)[CP]) const {
    float best = acc[0];
    int bi = 0;
#pragma unroll
    for (int c = 1; c < CP; ++c)
      if (c < Cout && acc[c] > best) { best = acc[c]; bi = c; }
    const int64_t i = ((int64_t)n * H + oy) * W + ox;
    if (cls) cls[i] = (unsigned char)bi;
    if (mask) mask[i] = ((bi >= 1 && bi <= 13) || bi == 15) ? 255 : 0;      // MASK_COLORMAP = [0, 255 x13, 0, 255, 0, 0, 0]
  }
};

// in [N, H, W, 64] NHWC -> Dst (Cout <= CP channels), 3x3 pad 1; weights [tap][64][CP] (zero-padded columns)
template <int CP, class Dst>
__global__ void __launch_bounds__(128) conv_thin_out_kernel(const float* __restrict__ in, const float* __restrict__ wgt,
                                                            const float* __restrict__ bias, const Dst out, int N, int H,
                                                            int W, int Cout, int pad_mode) {
  extern __shared__ __align__(16) float wsm[];       // [9 * 64][CP]
  for (int i = threadIdx.x; i < 9 * 64 * CP; i += 128) wsm[i] = wgt[i];
  __syncthreads();
  const int64_t pix = (int64_t)blockIdx.x * 128 + threadIdx.x;
  if (pix >= (int64_t)N * H * W) return;
  const int n = (int)(pix / ((int64_t)H * W));
  const int rem = (int)(pix - (int64_t)n * H * W);
  const int oy = rem / W, ox = rem - oy * W;
  if (!out.wants(n, oy, ox)) return;
  float acc[CP];
#pragma unroll
  for (int c = 0; c < CP; ++c) acc[c] = (bias && c < Cout) ? __ldg(bias + c) : 0.f;
  for (int r = 0; r < 3; ++r) {
    bool iny;
    const int iy = pad_index(oy + r - 1, H, pad_mode, iny);
    for (int s = 0; s < 3; ++s) {
      bool inx;
      const int ix = pad_index(ox + s - 1, W, pad_mode, inx);
      if (!(iny && inx)) continue;
      const float4* src = reinterpret_cast<const float4*>(in + (((int64_t)n * H + iy) * W + ix) * 64);
      const float* wt = wsm + (r * 3 + s) * 64 * CP;
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 v = __ldg(src + c4);
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float* wr = wt + (c4 * 4 + k) * CP;
#pragma unroll
          for (int c = 0; c < CP; ++c) acc[c] = fmaf(vv[k], wr[c], acc[c]);
        }
      }
    }
  }
  out.store(n, oy, ox, H, W, Cout, acc);
}
int conv_thin_out(const float* in_nhwc64, const float* wgt_tcp, const float* bias, float* out_nchw, int N, int H, int W, int Cout,
                  int pad_mode, cudaStream_t st) {
  CFB_REQUIRE(Cout >= 1 && Cout <= 20, "conv_thin_out: at most 20 output channels");
  const int64_t M = (int64_t)N * H * W;
  if (M == 0) return 0;
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load() & (1ull << (dev & 63)))) {
    CFB_CUDA(cudaFuncSetAttribute(conv_thin_out_kernel<20, NchwDst>, cudaFuncAttributeMaxDynamicSharedMemorySize, 9 * 64 * 20 * 4));
    attr_done.fetch_or(1ull << (dev & 63));
  }
  const NchwDst dst{out_nchw};
  if (Cout <= 4)
    conv_thin_out_kernel<4><<<(unsigned)((M + 127) / 128), 128, 9 * 64 * 4 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, Cout, pad_mode);
  else
    conv_thin_out_kernel<20><<<(unsigned)((M + 127) / 128), 128, 9 * 64 * 20 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, Cout, pad_mode);
  CFB_LAUNCH_CHECK();
  return 0;
}
int conv_thin_out_tiles(const float* in_nhwc64, const float* wgt_tcp, const float* bias, const RrdbU8Tiles& tiles,
                        void* canvas_bgr_hwc, int out_kind, const int* max_range, int out_h, int out_w, int N, int H, int W,
                        cudaStream_t st) {
  CFB_REQUIRE(N <= RrdbU8Tiles::kMax, "conv_thin_out_tiles: too many tiles for one launch");
  CFB_REQUIRE(out_kind == IMG_U8 || out_kind == IMG_U16, "conv_thin_out_tiles: the output is uint8 or uint16");
  const int64_t M = (int64_t)N * H * W;
  if (M == 0) return 0;
  const unsigned grid = (unsigned)((M + 127) / 128);
  if (out_kind == IMG_U8) {
    const TileDst<unsigned char> dst{(unsigned char*)canvas_bgr_hwc, out_h, out_w, max_range, tiles};
    conv_thin_out_kernel<4><<<grid, 128, 9 * 64 * 4 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, 3, 0);
  } else {
    const TileDst<unsigned short> dst{(unsigned short*)canvas_bgr_hwc, out_h, out_w, max_range, tiles};
    conv_thin_out_kernel<4><<<grid, 128, 9 * 64 * 4 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, 3, 0);
  }
  CFB_LAUNCH_CHECK();
  return 0;
}
int conv_thin_out_argmax(const float* in_nhwc64, const float* wgt_tcp, const float* bias, unsigned char* cls, unsigned char* mask,
                         int N, int H, int W, int Cout, int pad_mode, cudaStream_t st) {
  CFB_REQUIRE(Cout >= 1 && Cout <= 20, "conv_thin_out_argmax: at most 20 output channels");
  const int64_t M = (int64_t)N * H * W;
  if (M == 0) return 0;
  // the weights' column padding (relayout_thin_out) picks the instantiation, as in conv_thin_out; both fit the default
  // 48 KB of dynamic shared memory
  const ArgmaxU8Dst dst{cls, mask};
  if (Cout <= 4)
    conv_thin_out_kernel<4><<<(unsigned)((M + 127) / 128), 128, 9 * 64 * 4 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, Cout, pad_mode);
  else
    conv_thin_out_kernel<20><<<(unsigned)((M + 127) / 128), 128, 9 * 64 * 20 * 4, st>>>(in_nhwc64, wgt_tcp, bias, dst, N, H, W, Cout, pad_mode);
  CFB_LAUNCH_CHECK();
  return 0;
}

// OIHW [Cout][64][3][3] -> [tap][64][CP] with zero columns beyond Cout
__global__ void relayout_thin_out_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int CP) {
  const int total = 9 * 64 * CP;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % CP, ci = (i / CP) % 64, tap = i / (CP * 64);
    out[i] = c < Cout ? w[((int64_t)c * 64 + ci) * 9 + tap] : 0.f;
  }
}
int relayout_thin_out(const float* oihw, float* out, int Cout, cudaStream_t st) {
  const int CP = Cout <= 4 ? 4 : 20;
  relayout_thin_out_kernel<<<64, 256, 0, st>>>(oihw, out, Cout, CP);
  CFB_LAUNCH_CHECK();
  return 0;
}

// y[i] *= f (device scalars of the weight split: folds a constant output scale into 2^-k)
__global__ void scale_scalar_kernel(float* p, float f) { *p *= f; }
int scale_scalar(float* p, float f, cudaStream_t st) {
  scale_scalar_kernel<<<1, 1, 0, st>>>(p, f);
  CFB_LAUNCH_CHECK();
  return 0;
}
__global__ void scale_vec_kernel(float* __restrict__ p, int n, float f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] *= f;
}
int scale_vec(float* p, int n, float f, cudaStream_t st) {
  if (n == 0) return 0;
  scale_vec_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, n, f);
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace cfb

namespace cfb {
// BatchNorm2d in eval mode folded into the preceding bias-free conv (parsenet.py:87-88,98,103-104):
//   w'[co] = w[co] * gamma[co] / sqrt(var[co] + eps),   b'[co] = beta[co] - mean[co] * gamma[co] / sqrt(var[co] + eps)
__global__ void fold_bn_kernel(const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ mean, const float* __restrict__ var, float eps, float* __restrict__ wout,
                               float* __restrict__ bout, int Cout, int per_out) {
  const int co = blockIdx.x;
  const float s = gamma[co] / sqrtf(var[co] + eps);
  for (int i = threadIdx.x; i < per_out; i += blockDim.x) wout[(int64_t)co * per_out + i] = w[(int64_t)co * per_out + i] * s;
  if (threadIdx.x == 0) bout[co] = beta[co] - mean[co] * s;
}
int fold_bn(const float* w, const float* gamma, const float* beta, const float* mean, const float* var, float eps, float* wout,
            float* bout, int Cout, int per_out, cudaStream_t st) {
  if (Cout == 0) return 0;
  fold_bn_kernel<<<Cout, 256, 0, st>>>(w, gamma, beta, mean, var, eps, wout, bout, Cout, per_out);
  CFB_LAUNCH_CHECK();
  return 0;
}

// out.argmax(dim=1) of the parsing logits + the caller's class -> mask value table (face_restoration_helper.py:463-468)
__global__ void parse_argmax_kernel(const float* __restrict__ logits, unsigned char* __restrict__ cls, unsigned char* __restrict__ mask,
                                    int C, int64_t HW, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / HW, px = i - n * HW;
    const float* p = logits + n * C * HW + px;
    float best = p[0];
    int bi = 0;
    for (int c = 1; c < C; ++c) {
      const float v = p[(int64_t)c * HW];
      if (v > best) { best = v; bi = c; }           // first maximum, like torch.argmax
    }
    if (cls) cls[i] = (unsigned char)bi;
    if (mask) {
      // MASK_COLORMAP = [0, 255 x13, 0, 255, 0, 0, 0]
      const bool on = (bi >= 1 && bi <= 13) || bi == 15;
      mask[i] = on ? 255 : 0;
    }
  }
}
int parse_argmax(const float* logits_nchw, unsigned char* cls, unsigned char* mask, int N, int C, int64_t HW, cudaStream_t st) {
  const int64_t total = (int64_t)N * HW;
  if (total == 0) return 0;
  const int64_t blocks = (total + 255) / 256;
  parse_argmax_kernel<<<(unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks), 256, 0, st>>>(logits_nchw, cls, mask, C, HW, total);
  CFB_LAUNCH_CHECK();
  return 0;
}
}  // namespace cfb

namespace cfb {
// ---- VectorQuantizer one-kernel path (cfb_vq_nearest_fast): |e|^2 of the prepared codebook, one-hot rows of the indices ----
__global__ void vq_e2_only_kernel(const float* __restrict__ E, float* __restrict__ e2, int K, int D) {
  const int code = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (code >= K) return;
  float s = 0.f;
  for (int c = l; c < D; c += 32) { const float v = E[(int64_t)code * D + c]; s = fmaf(v, v, s); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (l == 0) e2[code] = s;
}
int vq_e2(const float* codebook, float* e2, int K, int D, cudaStream_t st) {
  vq_e2_only_kernel<<<(K + 7) / 8, 256, 0, st>>>(codebook, e2, K, D);
  CFB_LAUNCH_CHECK();
  return 0;
}
int onehot_from_idx(const int64_t* idx, float* onehot, int T, int K, cudaStream_t st) {
  CFB_CUDA(cudaMemsetAsync(onehot, 0, (size_t)T * K * sizeof(float), st));
  onehot_kernel<<<(T + 255) / 256, 256, 0, st>>>(idx, onehot, T, K);
  CFB_LAUNCH_CHECK();
  return 0;
}
}  // namespace cfb
