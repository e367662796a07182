// YOLOv5l-face (face detection of whole-image mode, --detection_model YOLOv5l): the SIMT kernels around the conv engine.
//   stem        StemBlock.stem_1 (3x3 s2 p1, 3 -> 64) + folded BatchNorm + SiLU; input fp32 NCHW (RGB / 255) or uint8 HWC BGR,
//               with the BGR -> RGB swap, the letterbox border (114) and the / 255 fused (yolov5face/face_detector.py:50-67,
//               utils/datasets.py:5-35)
//   maxpool2    StemBlock.stem_2p (MaxPool2d(2, 2, ceil_mode=True)) into a channel slice of the stem's concat buffer
//   spp         SPP's three MaxPool2d(k, 1, k // 2) (k = 3, 5, 7; -inf padding) of slice 0 into slices 1..3 (common.py:SPP)
//   copy        one channel block into a channel slice of a concat buffer, optionally nearest x2 (nn.Upsample of the head)
//   decode      Detect (yolo.py:52-86): the per-level head outputs -> raw x_l [B,3,ny,nx,16] (optional) and the decoded
//               pred [B,P,16]
//   candidates  `pred[..., 4] > conf_thres` compaction in prediction order (general.py:non_max_suppression_face)
// Max pools propagate NaN as torch's CPU max_pool2d does.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

__device__ __forceinline__ float yo_silu(float x) { return __fdiv_rn(x, __fadd_rn(1.f, expf(-x))); }
__device__ __forceinline__ float yo_sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }
__device__ __forceinline__ float yo_max(float m, float v) { return (v > m || v != v) ? v : m; }

static unsigned yo_blocks(int64_t total) {
  return (unsigned)((total + 255) / 256 < 65535 * 4 ? (total + 255) / 256 : 65535 * 4);
}

// ---- stem: one thread per output pixel, all 64 channels; the folded OIHW weights [64][3][3][3] go to shared memory as
// [27 taps][64].  The uint8 path places the [ih, iw] image at (top, left) of the H x W letterbox canvas; every other canvas
// pixel is 114.  Its value is channel (2 - c) of the BGR pixel divided by 255 (__fdiv_rn: torch's float division), so it
// equals the fp32 path fed with the preprocessed tensor bit for bit. ----
template <bool U8>
__global__ void __launch_bounds__(128) yolo_stem_kernel(const float* __restrict__ x_nchw, const unsigned char* __restrict__ img,
                                                        const float* __restrict__ wt, const float* __restrict__ bias,
                                                        float* __restrict__ out, int H, int W, int ih, int iw, int top,
                                                        int left, int Ho, int Wo) {
  __shared__ float sw[27 * 64];
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) sw[i] = wt[(i & 63) * 27 + (i >> 6)];   // OIHW -> [ci,r,s][co]
  if (threadIdx.x < 64) sb[threadIdx.x] = bias[threadIdx.x];
  pdl_launch_dependents();
  pdl_wait();
  __syncthreads();
  const int n = blockIdx.z, oy = blockIdx.y, ox = blockIdx.x * blockDim.x + threadIdx.x;
  if (ox >= Wo) return;
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = 0.f;
  for (int ci = 0; ci < 3; ++ci) {
    for (int r = 0; r < 3; ++r) {
      const int iy = 2 * oy - 1 + r;
      if ((unsigned)iy >= (unsigned)H) continue;
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * ox - 1 + s;
        if ((unsigned)ix >= (unsigned)W) continue;
        float v;
        if (U8) {
          const int y = iy - top, x = ix - left;
          const unsigned u = ((unsigned)y < (unsigned)ih && (unsigned)x < (unsigned)iw)
                                 ? img[(((int64_t)n * ih + y) * iw + x) * 3 + (2 - ci)] : 114u;
          v = __fdiv_rn((float)u, 255.f);
        } else {
          v = __ldg(x_nchw + (((int64_t)n * 3 + ci) * H + iy) * W + ix);
        }
        const float* wr = sw + ((ci * 3 + r) * 3 + s) * 64;
#pragma unroll
        for (int c = 0; c < 64; ++c) acc[c] = fmaf(v, wr[c], acc[c]);
      }
    }
  }
  float* o = out + (((int64_t)n * Ho + oy) * Wo + ox) * 64;
#pragma unroll
  for (int c = 0; c < 64; c += 4)
    *reinterpret_cast<float4*>(o + c) = make_float4(yo_silu(acc[c] + sb[c]), yo_silu(acc[c + 1] + sb[c + 1]),
                                                    yo_silu(acc[c + 2] + sb[c + 2]), yo_silu(acc[c + 3] + sb[c + 3]));
}

int yolo_stem(const float* x_nchw, const unsigned char* img_bgr_hwc, const float* wt, const float* bias, float* out, int N, int H,
              int W, int ih, int iw, int top, int left, cudaStream_t st) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  if (N == 0) return 0;
  const dim3 grid((unsigned)((Wo + 127) / 128), (unsigned)Ho, (unsigned)N);
  if (img_bgr_hwc)
    CFB_LAUNCH_PDL(yolo_stem_kernel<true>, grid, dim3(128), 0, st, x_nchw, img_bgr_hwc, wt, bias, out, H, W, ih, iw, top, left, Ho, Wo);
  else
    CFB_LAUNCH_PDL(yolo_stem_kernel<false>, grid, dim3(128), 0, st, x_nchw, img_bgr_hwc, wt, bias, out, H, W, ih, iw, top, left, Ho, Wo);
  return 0;
}

// ---- MaxPool2d(2, 2, ceil_mode=True) of NHWC C channels into a channel slice: one thread per (output pixel, 4 channels) ----
__global__ void yolo_maxpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int Ho, int Wo,
                                     int C4, int out_pitch, int out_c0) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * Ho * Wo * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t px = i / C4;
    const int ox = (int)(px % Wo);
    const int64_t t = px / Wo;
    const int oy = (int)(t % Ho), n = (int)(t / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < 2; ++r) {
      const int iy = 2 * oy + r;
      if (iy >= H) continue;
      for (int s = 0; s < 2; ++s) {
        const int ix = 2 * ox + s;
        if (ix >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(in + (((int64_t)n * H + iy) * W + ix) * C4 * 4 + c4 * 4));
        m.x = yo_max(m.x, v.x); m.y = yo_max(m.y, v.y); m.z = yo_max(m.z, v.z); m.w = yo_max(m.w, v.w);
      }
    }
    *reinterpret_cast<float4*>(out + px * out_pitch + out_c0 + c4 * 4) = m;
  }
}

int yolo_maxpool2(const float* in, float* out, int N, int H, int W, int C, int out_pitch, int out_c0, cudaStream_t st) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(yolo_maxpool2_kernel, dim3(yo_blocks(total)), dim3(256), 0, st, in, out, N, H, W, Ho, Wo, C / 4, out_pitch, out_c0);
  return 0;
}

// ---- SPP: buf [N,H,W,4C]; channels [0, C) hold cv1's output, [C, 2C), [2C, 3C), [3C, 4C) receive its 3x3, 5x5, 7x7 stride-1
// max pools.  One thread per (pixel, 4 channels) walks the 7x7 window once; the smaller windows are its centred parts. ----
__global__ void yolo_spp_kernel(float* __restrict__ buf, int N, int H, int W, int C4) {
  pdl_launch_dependents();
  pdl_wait();
  const int pitch = 16 * C4;
  const int64_t total = (int64_t)N * H * W * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t px = i / C4;
    const int x = (int)(px % W);
    const int64_t t = px / W;
    const int y = (int)(t % H), n = (int)(t / H);
    float4 m[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) m[k] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = -3; dy <= 3; ++dy) {
      const int iy = y + dy;
      if ((unsigned)iy >= (unsigned)H) continue;
      for (int dx = -3; dx <= 3; ++dx) {
        const int ix = x + dx;
        if ((unsigned)ix >= (unsigned)W) continue;
        const float4 v = *reinterpret_cast<const float4*>(buf + (((int64_t)n * H + iy) * W + ix) * pitch + c4 * 4);
        const int r = max(abs(dy), abs(dx));
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (r <= k + 1) { m[k].x = yo_max(m[k].x, v.x); m[k].y = yo_max(m[k].y, v.y); m[k].z = yo_max(m[k].z, v.z); m[k].w = yo_max(m[k].w, v.w); }
        }
      }
    }
    float* o = buf + px * pitch + c4 * 4;
#pragma unroll
    for (int k = 0; k < 3; ++k) *reinterpret_cast<float4*>(o + (k + 1) * 4 * C4) = m[k];
  }
}

int yolo_spp(float* buf, int N, int H, int W, int C, cudaStream_t st) {
  const int64_t total = (int64_t)N * H * W * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(yolo_spp_kernel, dim3(yo_blocks(total)), dim3(256), 0, st, buf, N, H, W, C / 4);
  return 0;
}

// ---- copy C channels of src (pitch, offset) into a channel slice of dst; up2: nearest x2 (dst is 2H x 2W, source y >> 1,
// which is upsample_nearest2d's index for scale_factor 2) ----
__global__ void yolo_copy_kernel(const float* __restrict__ src, int src_pitch, int src_c0, float* __restrict__ dst, int dst_pitch,
                                 int dst_c0, int N, int Hs, int Ws, int C4, int up) {
  pdl_launch_dependents();
  pdl_wait();
  const int Hd = Hs << up, Wd = Ws << up;
  const int64_t total = (int64_t)N * Hd * Wd * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int64_t px = i / C4;
    const int x = (int)(px % Wd);
    const int64_t t = px / Wd;
    const int y = (int)(t % Hd), n = (int)(t / Hd);
    const int64_t sp = ((int64_t)n * Hs + (y >> up)) * Ws + (x >> up);
    *reinterpret_cast<float4*>(dst + px * dst_pitch + dst_c0 + c4 * 4) =
        __ldg(reinterpret_cast<const float4*>(src + sp * src_pitch + src_c0 + c4 * 4));
  }
}

int yolo_copy(const float* src, int src_pitch, int src_c0, float* dst, int dst_pitch, int dst_c0, int N, int Hs, int Ws, int C,
              bool up2, cudaStream_t st) {
  const int64_t total = (int64_t)N * Hs * Ws * (up2 ? 4 : 1) * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(yolo_copy_kernel, dim3(yo_blocks(total)), dim3(256), 0, st, src, src_pitch, src_c0, dst, dst_pitch, dst_c0, N, Hs,
                 Ws, C / 4, up2 ? 1 : 0);
  return 0;
}

// ---- Detect: head level l is NHWC [N, ny, nx, 64] (channel a*16 + f, 48 real).  raw_l[n][a][y][x][f] is the view/permute
// of yolo.py:58; pred rows are (level, anchor, y, x).  The decode follows yolo.py:63-84 operation by operation:
//   sigmoid on fields 0-4 and 15; xy = (s * 2 - 0.5 + grid) * stride; wh = (s * 2) ** 2 * anchor_grid;
//   landmarks = raw * anchor_grid + grid * stride.  anchor_grid [3 levels][3 anchors][w, h] in pixels (the state buffer). ----
struct YoLevels { const float* h[3]; float* raw[3]; int ny[3], nx[3]; };

__global__ void yolo_decode_kernel(YoLevels L, const float* __restrict__ anchor_grid, float* __restrict__ pred, int N, int P) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * P;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / P);
    int q = (int)(i - (int64_t)n * P), l = 0;
    while (l < 2 && q >= 3 * L.ny[l] * L.nx[l]) { q -= 3 * L.ny[l] * L.nx[l]; ++l; }
    const int hw = L.ny[l] * L.nx[l];
    const int a = q / hw, pix = q - a * hw, y = pix / L.nx[l], x = pix - y * L.nx[l];
    const float* h = L.h[l] + ((int64_t)n * hw + pix) * 64 + a * 16;
    float* r = L.raw[l] ? L.raw[l] + (((int64_t)n * 3 + a) * hw + pix) * 16 : nullptr;
    float* o = pred + i * 16;
    const float stride = (float)(8 << l), gx = (float)x, gy = (float)y;
    const float aw = anchor_grid[(l * 3 + a) * 2], ah = anchor_grid[(l * 3 + a) * 2 + 1];
    float v[16];
#pragma unroll
    for (int f = 0; f < 16; ++f) v[f] = h[f];
    if (r) {
#pragma unroll
      for (int f = 0; f < 16; ++f) r[f] = v[f];
    }
    const float s0 = yo_sigmoid(v[0]), s1 = yo_sigmoid(v[1]), s2 = yo_sigmoid(v[2]), s3 = yo_sigmoid(v[3]);
    o[0] = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(s0, 2.f), 0.5f), gx), stride);
    o[1] = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(s1, 2.f), 0.5f), gy), stride);
    const float tw = __fmul_rn(s2, 2.f), th = __fmul_rn(s3, 2.f);
    o[2] = __fmul_rn(__fmul_rn(tw, tw), aw);
    o[3] = __fmul_rn(__fmul_rn(th, th), ah);
    o[4] = yo_sigmoid(v[4]);
    const float gxs = __fmul_rn(gx, stride), gys = __fmul_rn(gy, stride);
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      o[5 + 2 * j] = __fadd_rn(__fmul_rn(v[5 + 2 * j], aw), gxs);
      o[6 + 2 * j] = __fadd_rn(__fmul_rn(v[6 + 2 * j], ah), gys);
    }
    o[15] = yo_sigmoid(v[15]);
  }
}

int yolo_decode(const float* const h[3], float* const raw[3], const int ny[3], const int nx[3], const float* anchor_grid, float* pred,
                int N, int P, cudaStream_t st) {
  const int64_t total = (int64_t)N * P;
  if (total == 0) return 0;
  YoLevels L;
  for (int k = 0; k < 3; ++k) { L.h[k] = h[k]; L.raw[k] = raw[k]; L.ny[k] = ny[k]; L.nx[k] = nx[k]; }
  CFB_LAUNCH_PDL(yolo_decode_kernel, dim3(yo_blocks(total)), dim3(256), 0, st, L, anchor_grid, pred, N, P);
  return 0;
}

// ---- candidates: one block per image walks the predictions in order, 1024 at a time; a row is kept when its objectness is
// > thr (never for NaN) and goes to the position an exclusive block scan gives (no atomics) ----
constexpr int YO_CAND_THREADS = 1024;

__global__ void __launch_bounds__(YO_CAND_THREADS) yolo_candidates_kernel(const float* __restrict__ pred, int P, float thr,
                                                                         float* __restrict__ rows, int* __restrict__ counts) {
  __shared__ int warp_sum[32];
  __shared__ int base_s;
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  if (t == 0) base_s = 0;
  __syncthreads();
  for (int p0 = 0; p0 < P; p0 += YO_CAND_THREADS) {
    const int p = p0 + t;
    const int64_t i = (int64_t)n * P + p;
    const bool keep = p < P && pred[i * 16 + 4] > thr;          // false for NaN
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
      const float4* s = reinterpret_cast<const float4*>(pred + i * 16);
      float4* d = reinterpret_cast<float4*>(rows + ((int64_t)n * P + pos) * 16);
#pragma unroll
      for (int j = 0; j < 4; ++j) d[j] = s[j];
    }
    __syncthreads();
    if (t == 0) base_s = base + warp_sum[31];
    __syncthreads();
  }
  if (t == 0) counts[n] = base_s;
}

int yolo_candidates(const float* pred, int N, int P, float thr, float* rows, int* counts, cudaStream_t st) {
  if (N == 0) return 0;
  CFB_LAUNCH_PDL(yolo_candidates_kernel, dim3((unsigned)N), dim3(YO_CAND_THREADS), 0, st, pred, P, thr, rows, counts);
  return 0;
}

}  // namespace cfb
