// LPIPS-VGG (perceptual distance of restored faces; lpips 0.1 LPIPS(net='vgg'), the perceptual term of basicsr's LPIPSLoss,
// basicsr/losses/losses.py:257-282): the SIMT kernels around the conv engine.
//   stem      conv1_1 (3x3 p1, 3 -> 64) + ReLU -> NHWC [M,H,W,64], with the input transform fused into the load: fp32 NCHW
//             through the element-wise chain (2x - 1 | range_norm, input_norm; then the ScalingLayer), or uint8 HWC BGR through
//             a per-channel 256-entry table.  The conv pads the *transformed* image with zeros, as torch does.
//   head      one pass over relu_k of every image of a group (one reference, G candidates): the channel norms, the per-pixel
//             sum_c w_c (f0 / (|f0| + eps) - f1 / (|f1| + eps))^2 of each candidate, summed per block in a fixed order, and the
//             2 x 2 floor max pool of every image (the next slice's MaxPool2d(2, 2)); NaN propagates as in torch's CPU max_pool2d
//   finalize  per (candidate, layer): the block sums in a fixed order (float64), / (H_k W_k), and the layers summed 0..4
// Image i of a launch is image i % (1 + G) of group i / (1 + G): 0 the reference, j >= 1 candidate j - 1.  No reduction order
// depends on the batch, the number of groups or G, so a value is the same whatever it was batched with.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

__device__ __forceinline__ float lp_relu(float v) { return v < 0.f ? 0.f : v; }          // NaN stays NaN, as torch.relu
__device__ __forceinline__ float lp_max(float m, float v) { return (v > m || v != v) ? v : m; }

// The fp32 input chain of one element of RGB channel c, each step rounded as torch's fp32 ops (no contraction).
__device__ __forceinline__ float lp_xform(float v, int c, const LpipsXform& t) {
  if (t.flags & LPIPS_RANGE_NORM) v = __fdiv_rn(__fadd_rn(v, 1.f), 2.f);                  // (x + 1) / 2
  if (t.flags & LPIPS_INPUT_NORM) v = __fdiv_rn(__fsub_rn(v, t.mean[c]), t.std[c]);       // (x - mean) / std
  if (t.flags & LPIPS_NORMALIZE) v = __fsub_rn(__fmul_rn(2.f, v), 1.f);                    // 2 * x - 1
  return __fdiv_rn(__fsub_rn(v, t.shift[c]), t.scale[c]);                                 // ScalingLayer
}

// ---- stem: one block = 128 output pixels of one row of one image, one thread = one pixel x 64 channels.  The transformed
// 3 x 3 x 130 input patch is staged in shared memory; the 27 taps are summed in (ci, r, s) order with fmaf from 0, so the
// uint8 form equals the fp32 form on the transformed tensor bit for bit. ----
template <bool U8>
__global__ void __launch_bounds__(128) lpips_stem_kernel(const float* __restrict__ ref, const float* __restrict__ cand,
                                                         const unsigned char* __restrict__ ref8, const unsigned char* __restrict__ cand8,
                                                         const float* __restrict__ table, LpipsXform xf, const float* __restrict__ wt,
                                                         const float* __restrict__ bias, float* __restrict__ out, int G, int H, int W) {
  __shared__ float sw[27 * 64];
  __shared__ float sb[64];
  __shared__ float patch[3][3][130];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) sw[i] = wt[(i & 63) * 27 + (i >> 6)];   // OIHW -> [ci,r,s][co]
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  pdl_launch_dependents();
  pdl_wait();
  const int img = blockIdx.z, oy = blockIdx.y, x0 = blockIdx.x * 128 - 1;
  const int q = img / (1 + G), j = img - q * (1 + G);
  const int64_t src = j == 0 ? q : (int64_t)q * G + j - 1;                 // image index in ref / cand
  for (int i = threadIdx.x; i < 3 * 3 * 130; i += blockDim.x) {
    const int ci = i / 390, rem = i - ci * 390, r = rem / 130, px = rem - r * 130;
    const int iy = oy - 1 + r, ix = x0 + px;
    float v = 0.f;                                                         // zero padding of the transformed image
    if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) {
      if constexpr (U8) {
        const unsigned char* p = (j == 0 ? ref8 : cand8) + ((src * H + iy) * W + ix) * 3;
        v = __ldg(table + ci * 256 + p[2 - ci]);                           // BGR byte -> RGB channel ci
      } else {
        v = lp_xform(__ldg((j == 0 ? ref : cand) + ((src * 3 + ci) * H + iy) * W + ix), ci, xf);
      }
    }
    patch[ci][r][px] = v;
  }
  __syncthreads();
  const int ox = blockIdx.x * 128 + threadIdx.x;
  if (ox >= W) return;
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = 0.f;
  for (int ci = 0; ci < 3; ++ci)
    for (int r = 0; r < 3; ++r)
      for (int s = 0; s < 3; ++s) {
        const float v = patch[ci][r][threadIdx.x + s];
        const float* wr = sw + ((ci * 3 + r) * 3 + s) * 64;
#pragma unroll
        for (int c = 0; c < 64; ++c) acc[c] = fmaf(v, wr[c], acc[c]);
      }
  float* o = out + (((int64_t)img * H + oy) * W + ox) * 64;
#pragma unroll
  for (int c = 0; c < 64; c += 4)
    *reinterpret_cast<float4*>(o + c) = make_float4(lp_relu(acc[c] + sb[c]), lp_relu(acc[c + 1] + sb[c + 1]),
                                                    lp_relu(acc[c + 2] + sb[c + 2]), lp_relu(acc[c + 3] + sb[c + 3]));
}

int lpips_stem(const float* ref, const float* cand, const unsigned char* ref8, const unsigned char* cand8, const float* table,
               const LpipsXform& xf, const float* wt, const float* bias, float* out, int groups, int G, int H, int W, cudaStream_t st) {
  const int64_t M = (int64_t)groups * (1 + G);
  if (M == 0) return 0;
  CFB_REQUIRE(M <= 65535 && H <= 65535, "lpips_stem: at most 65535 images and rows per launch");
  const dim3 grid((unsigned)((W + 127) / 128), (unsigned)H, (unsigned)M);
  if (table)
    CFB_LAUNCH_PDL(lpips_stem_kernel<true>, grid, dim3(128), 0, st, ref, cand, ref8, cand8, table, xf, wt, bias, out, G, H, W);
  else
    CFB_LAUNCH_PDL(lpips_stem_kernel<false>, grid, dim3(128), 0, st, ref, cand, ref8, cand8, table, xf, wt, bias, out, G, H, W);
  return 0;
}

// ---- head and pool of one layer: block (b, q) covers quads [b * 64, b * 64 + 64) of group q, warp w the 8 consecutive
// quads from b * 64 + 8 w; a quad is the 2 x 2 pool window at (2 qy, 2 qx) over ceil(H/2) x ceil(W/2) (a ragged last row or
// column has pixels for the head only).  Lane l holds channels l * V + 32 V j (V = 2 for 64 channels, 4 otherwise).  Sums over
// channels: the lane's channels in order, then an xor butterfly (every lane ends with the same bits).  Per candidate, the warp
// adds its pixel values in quad order, pixel order (0,0) (0,1) (1,0) (1,1); the block adds its warps 0..7. ----
template <int C>
__global__ void __launch_bounds__(256) lpips_head_kernel(const float* __restrict__ feat, const float* __restrict__ lin, int G, int H,
                                                         int W, float* __restrict__ pooled, float* __restrict__ partial, int nblk) {
  constexpr int V = C == 64 ? 2 : 4;
  constexpr int NJ = C / (32 * V);
  constexpr int NPL = C / 32;
  extern __shared__ float wsum[];                                          // [8 warps][G]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int q = blockIdx.y, blk = blockIdx.x;
  const int Hq = (H + 1) / 2, Wq = (W + 1) / 2, Hp = H / 2, Wp = W / 2;
  const int64_t nquads = (int64_t)Hq * Wq;
  float w[NPL];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int v = 0; v < V; ++v) w[j * V + v] = __ldg(lin + j * 32 * V + lane * V + v);
  for (int g = lane; g < G; g += 32) wsum[warp * G + g] = 0.f;
  pdl_launch_dependents();
  pdl_wait();
  __syncwarp();
  const int64_t img0 = (int64_t)q * (1 + G);
  auto load = [&](int64_t img, int y, int x, float* f) {
    const float* p = feat + (((img * H) + y) * W + x) * C + lane * V;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if constexpr (V == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + j * 32 * V));
        f[j * 4] = t.x; f[j * 4 + 1] = t.y; f[j * 4 + 2] = t.z; f[j * 4 + 3] = t.w;
      } else {
        const float2 t = __ldg(reinterpret_cast<const float2*>(p + j * 32 * V));
        f[j * 2] = t.x; f[j * 2 + 1] = t.y;
      }
    }
  };
  auto warp_sum = [&](float s) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    return s;
  };
  // f / (sqrt(sum_c f^2) + 1e-10) in place (lpips normalize_tensor)
  auto normalize = [&](float* f) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NPL; ++i) s = __fadd_rn(s, __fmul_rn(f[i], f[i]));
    const float d = __fadd_rn(sqrtf(warp_sum(s)), 1e-10f);
#pragma unroll
    for (int i = 0; i < NPL; ++i) f[i] = __fdiv_rn(f[i], d);
  };
  auto store_pool = [&](int64_t img, int qy, int qx, const float* m) {
    float* p = pooled + (((img * Hp) + qy) * Wp + qx) * C + lane * V;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if constexpr (V == 4) *reinterpret_cast<float4*>(p + j * 32 * V) = make_float4(m[j * 4], m[j * 4 + 1], m[j * 4 + 2], m[j * 4 + 3]);
      else *reinterpret_cast<float2*>(p + j * 32 * V) = make_float2(m[j * 2], m[j * 2 + 1]);
    }
  };
  for (int t = 0; t < 8; ++t) {
    const int64_t quad = (int64_t)blk * 64 + warp * 8 + t;
    if (quad >= nquads) break;
    const int qy = (int)(quad / Wq), qx = (int)(quad - (int64_t)qy * Wq);
    const bool pool = pooled != nullptr && qy < Hp && qx < Wp;
    float f0[4][NPL], m[NPL], f[NPL];
    bool valid[4];
#pragma unroll
    for (int i = 0; i < NPL; ++i) m[i] = -INFINITY;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int y = 2 * qy + (p >> 1), x = 2 * qx + (p & 1);
      valid[p] = y < H && x < W;
      if (!valid[p]) continue;
      load(img0, y, x, f0[p]);
#pragma unroll
      for (int i = 0; i < NPL; ++i) m[i] = lp_max(m[i], f0[p][i]);
      normalize(f0[p]);
    }
    if (pool) store_pool(img0, qy, qx, m);
    for (int g = 0; g < G; ++g) {
      const int64_t img = img0 + 1 + g;
#pragma unroll
      for (int i = 0; i < NPL; ++i) m[i] = -INFINITY;
      float acc = 0.f;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        if (!valid[p]) continue;
        load(img, 2 * qy + (p >> 1), 2 * qx + (p & 1), f);
#pragma unroll
        for (int i = 0; i < NPL; ++i) m[i] = lp_max(m[i], f[i]);
        normalize(f);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NPL; ++i) {
          const float d = __fsub_rn(f0[p][i], f[i]);
          s = __fadd_rn(s, __fmul_rn(w[i], __fmul_rn(d, d)));
        }
        acc = __fadd_rn(acc, warp_sum(s));
      }
      if (lane == 0) wsum[warp * G + g] = __fadd_rn(wsum[warp * G + g], acc);
      if (pool) store_pool(img, qy, qx, m);
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s = __fadd_rn(s, wsum[k * G + g]);
    partial[((int64_t)q * G + g) * nblk + blk] = s;
  }
}

int lpips_head_blocks(int H, int W) { return (int)((((int64_t)(H + 1) / 2) * ((W + 1) / 2) + 63) / 64); }

int lpips_head(const float* feat, const float* lin, int groups, int G, int H, int W, int C, float* pooled, float* partial,
               cudaStream_t st) {
  if (groups == 0 || G == 0) return 0;
  CFB_REQUIRE(groups <= 65535, "lpips_head: at most 65535 groups per launch");
  CFB_REQUIRE(G <= 1024, "lpips_head: at most 1024 candidates per reference");
  const int nblk = lpips_head_blocks(H, W);
  const dim3 grid((unsigned)nblk, (unsigned)groups);
  const size_t smem = (size_t)8 * G * sizeof(float);
  switch (C) {
    case 64: CFB_LAUNCH_PDL(lpips_head_kernel<64>, grid, dim3(256), smem, st, feat, lin, G, H, W, pooled, partial, nblk); break;
    case 128: CFB_LAUNCH_PDL(lpips_head_kernel<128>, grid, dim3(256), smem, st, feat, lin, G, H, W, pooled, partial, nblk); break;
    case 256: CFB_LAUNCH_PDL(lpips_head_kernel<256>, grid, dim3(256), smem, st, feat, lin, G, H, W, pooled, partial, nblk); break;
    case 512: CFB_LAUNCH_PDL(lpips_head_kernel<512>, grid, dim3(256), smem, st, feat, lin, G, H, W, pooled, partial, nblk); break;
    default: CFB_REQUIRE(false, "lpips_head: channels must be 64, 128, 256 or 512");
  }
  return 0;
}

// ---- finalize: one thread per pair; res_k = float(sum_b partial_k[b] / (H_k W_k)) with the sum in float64 in block order,
// val = res_0 + res_1 + ... in float (lpips: val = 0; val += res[l] for l = 0..4) ----
__global__ void lpips_finalize_kernel(LpipsLayers L, int P, float* __restrict__ val, float* __restrict__ per_layer) {
  pdl_launch_dependents();
  pdl_wait();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float v = 0.f;
  for (int k = 0; k < L.n; ++k) {
    const float* part = L.part[k] + (int64_t)p * L.nblk[k];
    double s = 0.0;
    for (int b = 0; b < L.nblk[k]; ++b) s += (double)part[b];
    const float r = (float)(s / (double)L.hw[k]);
    if (per_layer) per_layer[(int64_t)p * L.n + k] = r;
    v = k == 0 ? r : __fadd_rn(v, r);
  }
  if (val) val[p] = v;
}

int lpips_finalize(const LpipsLayers& L, int P, float* val, float* per_layer, cudaStream_t st) {
  if (P == 0) return 0;
  CFB_LAUNCH_PDL(lpips_finalize_kernel, dim3((unsigned)((P + 127) / 128)), dim3(128), 0, st, L, P, val, per_layer);
  return 0;
}

}  // namespace cfb
