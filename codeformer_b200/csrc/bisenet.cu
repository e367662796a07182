// BiSeNet (face parsing of the paste-back step): the SIMT kernels around the conv engine.  Every reduction has a fixed order
// per image, so an image's results do not depend on the batch it runs in.
//   mean        F.avg_pool2d over the whole map of an NHWC tensor -> [N, C] (ARM, FFM, the context path's global average)
//   attention   the 1x1 convs on a pooled vector, one CTA per image: ARM conv_atten + bn_atten + sigmoid, FFM conv1 + ReLU +
//               conv2 + sigmoid, conv_avg + bn + ReLU (BatchNorm folded at prepare)
//   scale_add   feat * att[n, c] + add, add a per-(n, c) vector (arm32 + the broadcast avg_up), a same-size tensor
//               (arm16 + feat32_up) or feat itself (FFM): the reference's torch.mul, then the addition
//   bilinear    F.interpolate(mode='bilinear', align_corners=True) of the head logits (NHWC, zero-padded channels) to NCHW,
//               with the source indices, weights and fused multiply-adds of torch's CPU kernel
//   argmax      that bilinear fused with out.argmax(dim=1) and MASK_COLORMAP (face_restoration_helper.py:463-468)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.cuh"

namespace cfb {

static unsigned grid_of(int64_t total, int threads) {
  const int64_t b = (total + threads - 1) / threads;
  return (unsigned)(b < 65535 * 4 ? b : 65535 * 4);
}

// ---- mean: block (32-channel group, image), 256 threads = 8 pixel rows x 32 channels; row r sums pixels r, r + 8, .. in order,
// then thread r = 0 adds the 8 row sums in order ----
__global__ void __launch_bounds__(256) bise_mean_kernel(const float* __restrict__ in, float* __restrict__ out, int HW, int C) {
  __shared__ float part[8][33];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y, c = blockIdx.x * 32 + (threadIdx.x & 31), r = threadIdx.x >> 5;
  const float* p = in + (int64_t)n * HW * C + c;
  float s = 0.f;
  if (c < C)
    for (int px = r; px < HW; px += 8) s = __fadd_rn(s, __ldg(p + (int64_t)px * C));
  part[r][threadIdx.x & 31] = s;
  __syncthreads();
  if (r == 0 && c < C) {
    float t = part[0][threadIdx.x];
#pragma unroll
    for (int k = 1; k < 8; ++k) t = __fadd_rn(t, part[k][threadIdx.x]);
    out[(int64_t)n * C + c] = __fdiv_rn(t, (float)HW);
  }
}

int bise_mean(const float* in, float* out, int N, int HW, int C, cudaStream_t st) {
  if (N == 0) return 0;
  CFB_LAUNCH_PDL(bise_mean_kernel, dim3((unsigned)((C + 31) / 32), (unsigned)N), dim3(256), 0, st, in, out, HW, C);
  return 0;
}

// ---- attention: one CTA per image; y = act1(W1 v + b1) (c0 -> c1), then optionally z = act2(W2 y + b2) (c1 -> c2).  One
// thread per output channel, the input channels summed in order.  act: 0 none, 1 ReLU, 2 sigmoid (torch's 1 / (1 + exp(-x))) ----
__device__ __forceinline__ float bise_act(float s, int act) {
  if (act == 1) return fmaxf(s, 0.f);
  if (act == 2) return __frcp_rn(__fadd_rn(1.f, expf(-s)));
  return s;
}

__device__ __forceinline__ void bise_matvec(const float* __restrict__ w, const float* __restrict__ b, const float* v, float* y, int cin,
                                            int cout, int act) {
  for (int co = threadIdx.x; co < cout; co += blockDim.x) {
    const float* wr = w + (int64_t)co * cin;
    float s = 0.f;
    for (int ci = 0; ci < cin; ++ci) s = fmaf(__ldg(wr + ci), v[ci], s);
    y[co] = bise_act(b ? __fadd_rn(s, __ldg(b + co)) : s, act);
  }
}

constexpr int BISE_ATT_MAX = 512;

__global__ void __launch_bounds__(256) bise_attention_kernel(BiseAttention a, const float* __restrict__ v, float* __restrict__ out) {
  __shared__ float sv[BISE_ATT_MAX], sh[BISE_ATT_MAX];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < a.c0; i += blockDim.x) sv[i] = v[(int64_t)n * a.c0 + i];
  __syncthreads();
  if (!a.w2) {
    bise_matvec(a.w1, a.b1, sv, out + (int64_t)n * a.c1, a.c0, a.c1, a.act1);
    return;
  }
  bise_matvec(a.w1, a.b1, sv, sh, a.c0, a.c1, a.act1);
  __syncthreads();
  bise_matvec(a.w2, a.b2, sh, out + (int64_t)n * a.c2, a.c1, a.c2, a.act2);
}

int bise_attention(const BiseAttention& a, const float* v, float* out, int N, cudaStream_t st) {
  CFB_REQUIRE(a.c0 <= BISE_ATT_MAX && a.c1 <= BISE_ATT_MAX && a.c2 <= BISE_ATT_MAX, "bise_attention: at most 512 channels");
  if (N == 0) return 0;
  CFB_LAUNCH_PDL(bise_attention_kernel, dim3((unsigned)N), dim3(256), 0, st, a, v, out);
  return 0;
}

// ---- scale_add: out = feat * att[n, c] + add (add_vec [N, C], add_t [N, HW, C], or feat when both are null); out may be feat ----
__global__ void bise_scale_add_kernel(const float* feat, const float* __restrict__ att, const float* __restrict__ add_vec,
                                      const float* add_t, float* out, int N, int64_t HW, int C4) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * HW * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const int n = (int)(i / (HW * C4));
    const int64_t nc = (int64_t)n * C4 + c4;
    const float4 f = reinterpret_cast<const float4*>(feat)[i];
    const float4 a = __ldg(reinterpret_cast<const float4*>(att) + nc);
    const float4 d = add_vec ? __ldg(reinterpret_cast<const float4*>(add_vec) + nc) : add_t ? reinterpret_cast<const float4*>(add_t)[i] : f;
    reinterpret_cast<float4*>(out)[i] = make_float4(__fadd_rn(__fmul_rn(f.x, a.x), d.x), __fadd_rn(__fmul_rn(f.y, a.y), d.y),
                                                    __fadd_rn(__fmul_rn(f.z, a.z), d.z), __fadd_rn(__fmul_rn(f.w, a.w), d.w));
  }
}

int bise_scale_add(const float* feat, const float* att, const float* add_vec, const float* add_t, float* out, int N, int64_t HW, int C,
                   cudaStream_t st) {
  CFB_REQUIRE(C % 4 == 0, "bise_scale_add: channels must be a multiple of 4");
  const int64_t total = (int64_t)N * HW * (C / 4);
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(bise_scale_add_kernel, dim3(grid_of(total, 256)), dim3(256), 0, st, feat, att, add_vec, add_t, out, N, HW, C / 4);
  return 0;
}

// ---- bilinear, align_corners=True, as torch's CPU kernel forms it (aten/src/ATen/native/UpSample.h): scale = float(in - 1) /
// (out - 1), src = scale * i, i0 = min(floor(src), in - 1), i1 = i0 + (i0 < in - 1), l1 = clamp(src - i0, 0, 1), l0 = 1 - l1;
// each dimension combines its two terms as fma(t0, l0, t1 * l1), width inside, height outside ----
struct BiseTap { int i0, i1; float l0, l1; };

__device__ __forceinline__ BiseTap bise_tap(int i, int in, int out) {
  const float scale = out > 1 ? __fdiv_rn((float)(in - 1), (float)(out - 1)) : 0.f;
  const float src = __fmul_rn(scale, (float)i);
  BiseTap t;
  t.i0 = min((int)floorf(src), in - 1);
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = fminf(fmaxf(__fsub_rn(src, (float)t.i0), 0.f), 1.f);
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}

// the logit of channel c at the output pixel of (ty, tx): the one expression both kernels below evaluate
__device__ __forceinline__ float bise_logit(const float* __restrict__ img, int pitch, int w, const BiseTap& ty, const BiseTap& tx, int c) {
  const float* r0 = img + (int64_t)ty.i0 * w * pitch + c;
  const float* r1 = img + (int64_t)ty.i1 * w * pitch + c;
  const float t0 = fmaf(__ldg(r0 + (int64_t)tx.i0 * pitch), tx.l0, __fmul_rn(__ldg(r0 + (int64_t)tx.i1 * pitch), tx.l1));
  const float t1 = fmaf(__ldg(r1 + (int64_t)tx.i0 * pitch), tx.l0, __fmul_rn(__ldg(r1 + (int64_t)tx.i1 * pitch), tx.l1));
  return fmaf(t0, ty.l0, __fmul_rn(t1, ty.l1));
}

__global__ void bise_bilinear_kernel(const float* __restrict__ in, int pitch, int h, int w, int C, float* __restrict__ out, int N, int H,
                                     int W) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * H * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int64_t t = i / W;
    const int y = (int)(t % H), n = (int)(t / H);
    const BiseTap ty = bise_tap(y, h, H), tx = bise_tap(x, w, W);
    const float* img = in + (int64_t)n * h * w * pitch;
    float* o = out + (int64_t)n * C * H * W + (int64_t)y * W + x;
    for (int c = 0; c < C; ++c) o[(int64_t)c * H * W] = bise_logit(img, pitch, w, ty, tx, c);
  }
}

int bise_bilinear(const float* in, int pitch, int h, int w, int C, float* out, int N, int H, int W, cudaStream_t st) {
  const int64_t total = (int64_t)N * H * W;
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(bise_bilinear_kernel, dim3(grid_of(total, 256)), dim3(256), 0, st, in, pitch, h, w, C, out, N, H, W);
  return 0;
}

// first maximum with a strict >, as parse_argmax_kernel (a NaN first logit stays class 0)
__global__ void bise_bilinear_argmax_kernel(const float* __restrict__ in, int pitch, int h, int w, int C, unsigned char* __restrict__ cls,
                                            unsigned char* __restrict__ mask, int N, int H, int W) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)N * H * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int64_t t = i / W;
    const int y = (int)(t % H), n = (int)(t / H);
    const BiseTap ty = bise_tap(y, h, H), tx = bise_tap(x, w, W);
    const float* img = in + (int64_t)n * h * w * pitch;
    float best = bise_logit(img, pitch, w, ty, tx, 0);
    int bi = 0;
    for (int c = 1; c < C; ++c) {
      const float v = bise_logit(img, pitch, w, ty, tx, c);
      if (v > best) { best = v; bi = c; }
    }
    if (cls) cls[i] = (unsigned char)bi;
    if (mask) mask[i] = ((bi >= 1 && bi <= 13) || bi == 15) ? 255 : 0;      // MASK_COLORMAP = [0, 255 x13, 0, 255, 0, 0, 0]
  }
}

int bise_bilinear_argmax(const float* in, int pitch, int h, int w, int C, unsigned char* cls, unsigned char* mask, int N, int H, int W,
                         cudaStream_t st) {
  const int64_t total = (int64_t)N * H * W;
  if (total == 0) return 0;
  CFB_LAUNCH_PDL(bise_bilinear_argmax_kernel, dim3(grid_of(total, 256)), dim3(256), 0, st, in, pitch, h, w, C, cls, mask, N, H, W);
  return 0;
}

}  // namespace cfb
