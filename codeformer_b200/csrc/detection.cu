// RetinaFace-ResNet50 (face detection of whole-image mode): the SIMT kernels around the conv engine.
//   stem        torchvision resnet50 conv1 (7x7 s2 p3, 3 -> 64) + folded bn1 + ReLU; input fp32 NCHW or uint8 HWC BGR with the
//               detector's (104, 117, 123) mean subtraction fused (facelib/detection/retinaface/retinaface.py:222), or with
//               the face normalisation of u8_to_input fused (BiSeNet's ResNet18 has the same stem)
//   maxpool     resnet50 maxpool (3x3 s2 p1, -inf padding)
//   add_nearest FPN: output_k += F.interpolate(output_{k+1}, size=output_k.shape[2:], mode='nearest') (retinaface_net.py:84-94)
//   heads       per-level head tensors [N,h,w,64] (bbox 8 | class 4 | landmark 20 | 0) -> loc / softmaxed conf / landms in
//               prior order (permute(0,2,3,1).view(B,-1,k) of retinaface_net.py:140-175, softmax of retinaface.py:143)
//   candidates  PriorBox + decode + decode_landm + x scale + `scores > conf_threshold` compaction in prior order
//               (retinaface.py:194-225, retinaface_utils.py:1-40, 254-294)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

// ---- stem: one thread per output pixel, all 64 channels; the folded OIHW weights [64][3][7][7] are read into shared memory
// as [147 taps][64] ----
enum StemIn { STEM_F32 = 0, STEM_U8_DETECT = 1, STEM_U8_FACE = 2 };

template <int IN>
__global__ void __launch_bounds__(128) rf_stem_kernel(const float* __restrict__ x_nchw, const unsigned char* __restrict__ img,
                                                      const float* __restrict__ wt, const float* __restrict__ bias,
                                                      float* __restrict__ out, int H, int W, int Ho, int Wo) {
  __shared__ float sw[147 * 64];
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < 147 * 64; i += blockDim.x) sw[i] = wt[(i & 63) * 147 + (i >> 6)];   // OIHW -> [ci,r,s][co]
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  pdl_launch_dependents();
  pdl_wait();
  __syncthreads();
  const int n = blockIdx.z, oy = blockIdx.y, ox = blockIdx.x * blockDim.x + threadIdx.x;
  if (ox >= Wo) return;
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = 0.f;
  const float mean[3] = {104.f, 117.f, 123.f};
  for (int ci = 0; ci < 3; ++ci) {
    for (int r = 0; r < 7; ++r) {
      const int iy = 2 * oy - 3 + r;
      if ((unsigned)iy >= (unsigned)H) continue;
      for (int s = 0; s < 7; ++s) {
        const int ix = 2 * ox - 3 + s;
        if ((unsigned)ix >= (unsigned)W) continue;
        float v;
        if (IN == STEM_U8_DETECT) v = __fsub_rn((float)img[(((int64_t)n * H + iy) * W + ix) * 3 + ci], mean[ci]);   // exact in fp32
        else if (IN == STEM_U8_FACE) v = u8_to_model_input(img[(((int64_t)n * H + iy) * W + ix) * 3 + (2 - ci)]);   // RGB channel ci
        else v = __ldg(x_nchw + (((int64_t)n * 3 + ci) * H + iy) * W + ix);
        const float* wr = sw + ((ci * 7 + r) * 7 + s) * 64;
#pragma unroll
        for (int c = 0; c < 64; ++c) acc[c] = fmaf(v, wr[c], acc[c]);
      }
    }
  }
  float* o = out + (((int64_t)n * Ho + oy) * Wo + ox) * 64;
#pragma unroll
  for (int c = 0; c < 64; c += 4)
    *reinterpret_cast<float4*>(o + c) = make_float4(fmaxf(acc[c] + sb[c], 0.f), fmaxf(acc[c + 1] + sb[c + 1], 0.f),
                                                    fmaxf(acc[c + 2] + sb[c + 2], 0.f), fmaxf(acc[c + 3] + sb[c + 3], 0.f));
}

int rf_stem(const float* x_nchw, const unsigned char* img_bgr_hwc, const float* wt, const float* bias, float* out, int N, int H,
            int W, cudaStream_t st, bool face_u8) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  if (N == 0) return 0;
  const dim3 grid((unsigned)((Wo + 127) / 128), (unsigned)Ho, (unsigned)N);
  if (img_bgr_hwc && face_u8)
    CFB_LAUNCH_PDL(rf_stem_kernel<STEM_U8_FACE>, grid, dim3(128), 0, st, x_nchw, img_bgr_hwc, wt, bias, out, H, W, Ho, Wo);
  else if (img_bgr_hwc)
    CFB_LAUNCH_PDL(rf_stem_kernel<STEM_U8_DETECT>, grid, dim3(128), 0, st, x_nchw, img_bgr_hwc, wt, bias, out, H, W, Ho, Wo);
  else CFB_LAUNCH_PDL(rf_stem_kernel<STEM_F32>, grid, dim3(128), 0, st, x_nchw, img_bgr_hwc, wt, bias, out, H, W, Ho, Wo);
  return 0;
}

// ---- max-pool 3x3 s2 p1 over NHWC 64 channels: one thread per (output pixel, 4 channels) ----
__global__ void rf_maxpool_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int Ho, int Wo) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * Ho * Wo * 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i & 15);
    const int64_t px = i >> 4;
    const int ox = (int)(px % Wo);
    const int64_t t = px / Wo;
    const int oy = (int)(t % Ho), n = (int)(t / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < 3; ++r) {
      const int iy = 2 * oy - 1 + r;
      if ((unsigned)iy >= (unsigned)H) continue;
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * ox - 1 + s;
        if ((unsigned)ix >= (unsigned)W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(in + (((int64_t)n * H + iy) * W + ix) * 64 + c4 * 4));
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    *reinterpret_cast<float4*>(out + px * 64 + c4 * 4) = m;
  }
}

int rf_maxpool(const float* in, float* out, int N, int H, int W, cudaStream_t st) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t total = (int64_t)N * Ho * Wo * 16;
  if (total == 0) return 0;
  const unsigned blocks = (unsigned)((total + 255) / 256 < 65535 * 4 ? (total + 255) / 256 : 65535 * 4);
  CFB_LAUNCH_PDL(rf_maxpool_kernel, dim3(blocks), dim3(256), 0, st, in, out, N, H, W, Ho, Wo);
  return 0;
}

// ---- FPN top-down add.  The source index is the one upsample_nearest2d computes for a given output size: the identity for
// equal sizes, i >> 1 for an exact doubling, else min((int64)floorf(i * (float)in / out), in - 1) ----
__device__ __forceinline__ int nearest_src(int i, int in, int out) {
  if (in == out) return i;
  if (out == 2 * in) return i >> 1;
  const float scale = (float)in / (float)out;
  const int s = (int)floorf(__fmul_rn((float)i, scale));
  return s < in - 1 ? s : in - 1;
}

__global__ void rf_add_nearest_kernel(float* __restrict__ fine, const float* __restrict__ coarse, int N, int Hf, int Wf, int Hc,
                                      int Wc, int C4) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * Hf * Wf * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t px = i / C4;
    const int x = (int)(px % Wf);
    const int64_t t = px / Wf;
    const int y = (int)(t % Hf), n = (int)(t / Hf);
    const int ys = nearest_src(y, Hc, Hf), xs = nearest_src(x, Wc, Wf);
    float4 a = *reinterpret_cast<float4*>(fine + i * 4);
    const float4 b = __ldg(reinterpret_cast<const float4*>(coarse + ((((int64_t)n * Hc + ys) * Wc + xs) * C4 + c4) * 4));
    a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
    *reinterpret_cast<float4*>(fine + i * 4) = a;
  }
}

int rf_add_nearest(float* fine, const float* coarse, int N, int Hf, int Wf, int Hc, int Wc, int C, cudaStream_t st) {
  const int64_t total = (int64_t)N * Hf * Wf * (C / 4);
  if (total == 0) return 0;
  const unsigned blocks = (unsigned)((total + 255) / 256 < 65535 * 4 ? (total + 255) / 256 : 65535 * 4);
  CFB_LAUNCH_PDL(rf_add_nearest_kernel, dim3(blocks), dim3(256), 0, st, fine, coarse, N, Hf, Wf, Hc, Wc, C / 4);
  return 0;
}

// ---- head tensors -> loc [N,P,4], conf [N,P,2] (softmax over the 2 classes), landms [N,P,10] ----
struct RfLevels { const float* h[3]; int hh[3], ww[3]; };

__device__ __forceinline__ void rf_locate(const RfLevels& L, int p, int& lvl, int& pix, int& a) {
  int q = p;
  lvl = 0;
  while (lvl < 2 && q >= 2 * L.hh[lvl] * L.ww[lvl]) { q -= 2 * L.hh[lvl] * L.ww[lvl]; ++lvl; }
  pix = q >> 1; a = q & 1;
}

// softmax of two logits as torch's CPU kernel forms it: exp(x - max), the sum, then multiplication by its reciprocal
__device__ __forceinline__ void rf_softmax2(float c0, float c1, float& s0, float& s1) {
  const float m = fmaxf(c0, c1);
  const float e0 = expf(__fsub_rn(c0, m)), e1 = expf(__fsub_rn(c1, m));
  const float inv = __frcp_rn(__fadd_rn(e0, e1));
  s0 = __fmul_rn(e0, inv); s1 = __fmul_rn(e1, inv);
  if (c0 != c0 || c1 != c1) { s0 = NAN; s1 = NAN; }
}

__global__ void rf_heads_kernel(RfLevels L, float* __restrict__ loc, float* __restrict__ conf, float* __restrict__ landms, int N, int P) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * P;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / P), p = (int)(i - (int64_t)n * P);
    int lvl, pix, a;
    rf_locate(L, p, lvl, pix, a);
    const float* h = L.h[lvl] + ((int64_t)n * L.hh[lvl] * L.ww[lvl] + pix) * 64;
#pragma unroll
    for (int j = 0; j < 4; ++j) loc[i * 4 + j] = h[a * 4 + j];
    float s0, s1;
    rf_softmax2(h[8 + a * 2], h[8 + a * 2 + 1], s0, s1);
    conf[i * 2] = s0; conf[i * 2 + 1] = s1;
#pragma unroll
    for (int j = 0; j < 10; ++j) landms[i * 10 + j] = h[12 + a * 10 + j];
  }
}

int rf_heads(const float* const h[3], const int hh[3], const int ww[3], float* loc, float* conf, float* landms, int N, int P,
             cudaStream_t st) {
  const int64_t total = (int64_t)N * P;
  if (total == 0) return 0;
  RfLevels L;
  for (int k = 0; k < 3; ++k) { L.h[k] = h[k]; L.hh[k] = hh[k]; L.ww[k] = ww[k]; }
  const unsigned blocks = (unsigned)((total + 255) / 256 < 65535 * 4 ? (total + 255) / 256 : 65535 * 4);
  CFB_LAUNCH_PDL(rf_heads_kernel, dim3(blocks), dim3(256), 0, st, L, loc, conf, landms, N, P);
  return 0;
}

// ---- candidates: one block per image walks the priors in order, 1024 at a time; a thread's prior is kept when its score
// is > conf_threshold (never for NaN), and its row goes to the position an exclusive block scan gives (no atomics) ----
constexpr int RF_CAND_THREADS = 1024;

__global__ void __launch_bounds__(RF_CAND_THREADS) rf_candidates_kernel(const float* __restrict__ loc, const float* __restrict__ conf,
                                                                       const float* __restrict__ landms, int H, int W, int P,
                                                                       float thr, float* __restrict__ rows, int* __restrict__ counts) {
  __shared__ int warp_sum[32];
  __shared__ int base_s;
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int steps[3] = {8, 16, 32}, mins[3][2] = {{16, 32}, {64, 128}, {256, 512}};
  int fh[3], fw[3];
  for (int k = 0; k < 3; ++k) { fh[k] = (H + steps[k] - 1) / steps[k]; fw[k] = (W + steps[k] - 1) / steps[k]; }
  if (t == 0) base_s = 0;
  __syncthreads();
  const float Wf = (float)W, Hf = (float)H;
  for (int p0 = 0; p0 < P; p0 += RF_CAND_THREADS) {
    const int p = p0 + t;
    const int64_t i = (int64_t)n * P + p;
    const float score = p < P ? conf[i * 2 + 1] : 0.f;
    const bool keep = p < P && score > thr;          // false for NaN
    const unsigned ball = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_sum[wid] = __popc(ball);
    __syncthreads();
    if (wid == 0) {
      int v = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      warp_sum[lane] = v;            // inclusive scan over the warps
    }
    __syncthreads();
    const int base = base_s;
    if (keep) {
      const int pos = base + (wid ? warp_sum[wid - 1] : 0) + __popc(ball & ((1u << lane) - 1u));
      // prior of p (PriorBox.forward: float64 arithmetic, then float32)
      int q = p, k = 0;
      while (k < 2 && q >= 2 * fh[k] * fw[k]) { q -= 2 * fh[k] * fw[k]; ++k; }
      const int a = q & 1, pix = q >> 1, iy = pix / fw[k], jx = pix - iy * fw[k];
      const float pcx = (float)__ddiv_rn(__dmul_rn((double)jx + 0.5, (double)steps[k]), (double)W);
      const float pcy = (float)__ddiv_rn(__dmul_rn((double)iy + 0.5, (double)steps[k]), (double)H);
      const float pw = (float)__ddiv_rn((double)mins[k][a], (double)W);
      const float ph = (float)__ddiv_rn((double)mins[k][a], (double)H);
      const float* l = loc + i * 4;
      // decode (retinaface_utils.py:267-271): centre = p + (l * 0.1) * s, size = s * exp(l * 0.2); x1 = cx - w / 2; x2 = w + x1
      const float cx = __fadd_rn(pcx, __fmul_rn(__fmul_rn(l[0], 0.1f), pw));
      const float cy = __fadd_rn(pcy, __fmul_rn(__fmul_rn(l[1], 0.1f), ph));
      const float bw = __fmul_rn(pw, expf(__fmul_rn(l[2], 0.2f)));
      const float bh = __fmul_rn(ph, expf(__fmul_rn(l[3], 0.2f)));
      const float x1 = __fsub_rn(cx, __fdiv_rn(bw, 2.f)), y1 = __fsub_rn(cy, __fdiv_rn(bh, 2.f));
      const float x2 = __fadd_rn(bw, x1), y2 = __fadd_rn(bh, y1);
      float* r = rows + ((int64_t)n * P + pos) * 15;
      r[0] = __fmul_rn(x1, Wf); r[1] = __fmul_rn(y1, Hf); r[2] = __fmul_rn(x2, Wf); r[3] = __fmul_rn(y2, Hf);
      r[4] = score;
      const float* m = landms + i * 10;
#pragma unroll
      for (int j = 0; j < 5; ++j) {       // decode_landm (retinaface_utils.py:286-293)
        r[5 + 2 * j] = __fmul_rn(__fadd_rn(pcx, __fmul_rn(__fmul_rn(m[2 * j], 0.1f), pw)), Wf);
        r[6 + 2 * j] = __fmul_rn(__fadd_rn(pcy, __fmul_rn(__fmul_rn(m[2 * j + 1], 0.1f), ph)), Hf);
      }
    }
    __syncthreads();
    if (t == 0) base_s = base + warp_sum[31];
    __syncthreads();
  }
  if (t == 0) counts[n] = base_s;
}

int rf_candidates(const float* loc, const float* conf, const float* landms, int N, int H, int W, float thr, float* rows, int* counts,
                  cudaStream_t st) {
  if (N == 0) return 0;
  const int P = 2 * (((H + 7) / 8) * ((W + 7) / 8) + ((H + 15) / 16) * ((W + 15) / 16) + ((H + 31) / 32) * ((W + 31) / 32));
  CFB_LAUNCH_PDL(rf_candidates_kernel, dim3((unsigned)N), dim3(RF_CAND_THREADS), 0, st, loc, conf, landms, H, W, P, thr, rows, counts);
  return 0;
}

}  // namespace cfb
