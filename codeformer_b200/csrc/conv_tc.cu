// wgmma implicit-GEMM convolution engine for sm_90a (H100).
//
// Computes the 3x3 / 1x1 convolutions and linears of the CodeFormer hot path
//   nn.Conv2d call sites      /root/reference/basicsr/archs/vqgan_arch.py:120,132,147-151,173-200,243,266,292,314
//   Fuse_sft convs, Linear    /root/reference/basicsr/archs/codeformer_arch.py:104-106,141-149,183,192
// as GEMMs  D[M = 128 output pixels, N = 64 or 128 output channels (TcCfg; 64-channel halo tiles are computed transposed, CM)]
// += A[M, K] * B[N, K]^T  with K = taps * Cin, on
// the Hopper tensor cores:
//   * operands are error-compensated fp16 pairs  x = hi + lo  (hi = fp16(x), lo = fp16(x - hi)); the products
//     lo*hi + hi*lo + hi*hi are three wgmma.mma_async m64n64k16 per 64-row half and k-step, fp32 accumulation in registers
//     (>= 21 effective mantissa bits; the 1e-3 parity bar needs >= 16, SURVEY.md Appendix B);
//   * the tensor core truncates when it adds into its accumulator, so the MMA warpgroup only accumulates `chunk` k-blocks
//     before it hands the partial sum to the epilogue warps through a shared-memory slot; they fold it into fp32 registers
//     with round-to-nearest adds (cfull / cempty barriers);
//   * A tiles are fetched by TMA straight from the NHWC operand planes: one 4-D box {64 ch, BW, BH, 1} per filter tap at
//     shifted (x+s-1, y+r-1) coordinates -- out-of-bounds rows/cols are zero-filled by the TMA unit, which *is* the conv
//     padding; the box lands in shared memory as 128 rows x 128 B in the 128B-swizzled K-major layout the wgmma
//     descriptors read (no im2col buffer anywhere).  Stride-2 Downsample = TMA traversal strides (elementStrides 2);
//     Upsample = four 2x2 parity convs on the low-res planes with pre-summed weights;
//   * B tiles ([tap][Cout][Cin] fp16) by 3-D TMA boxes {64, 64, 1};
//   * warp-specialised persistent CTAs (1 per SM): one TMA producer warp (one elected lane issues), one MMA warpgroup,
//     8 epilogue warps (fold -> per-warp swizzled smem transpose -> bias / residual / activation / SFT -> coalesced fp32 NHWC
//     stores, optional fp16 hi/lo planes for a raw-input consumer, GroupNorm(32) partial sums), all hand-offs on mbarriers;
//   * halo engine (HALO): 8x16-pixel tiles; the (10x18) input patch of a 64-channel block is fetched ONCE and the taps read
//     it through row-shifted 128B-swizzled descriptors (see the MMA warpgroup and tc_geometry);
//   * in-kernel operand transform (XF, the default for every GroupNorm(+SiLU) consumer): the patch of a 64-channel block
//     arrives as the fp32 ACTIVATION itself (own loader warp, two 32-channel TMA boxes) and 4 transform warps apply
//     GroupNorm-affine + SiLU + the fp16 hi/lo split in place before the MMAs read it -- no operand planes in HBM, no
//     separate preparation pass (tc_can_xform says where it is used); GEN = the same for any H x W with reflection /
//     replicate padding (ParseNet, RRDBNet); the kernel also runs the attention GEMMs (bmm_tc);
//   * every kernel of the forward is launched with programmatic stream serialization (PDL, kernels.cuh).
// Diagnostics are BUILD options (-DCFB_TC_STAMPS=1): stamp tests inside the role loops cost time in every conv kernel, so
// production builds omit them and keep TcParams compact.

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "conv_tc.cuh"

namespace cfb {

// ------------------------------------------------------------------------------------------------------
// weight split: OIHW fp32 -> [tap][Cout][Cin] fp16 hi/lo of (w * 2^k), k chosen so max|w| lands in [2^13,2^14)
// (keeps `lo` out of the fp16 subnormal range); scale_slot[0] = |w|max bits, scale_slot[1] = 2^-k for the epilogue
// ------------------------------------------------------------------------------------------------------
__global__ void tc_absmax_kernel(const float* __restrict__ w, int64_t total, unsigned* __restrict__ slot) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(slot, __float_as_uint(m));
}

__global__ void tc_split_weights_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo,
                                        int Cout, int Cin, int taps, float* __restrict__ slot) {
  const float amax = __uint_as_float(reinterpret_cast<const unsigned*>(slot)[0]);
  int e = 0;
  if (amax > 0.f && isfinite(amax)) frexpf(amax, &e);
  const float scale = exp2f((float)(14 - e));
  const int64_t total = (int64_t)Cout * Cin * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cin);
    const int co = (int)((i / Cin) % Cout);
    const int tap = (int)(i / ((int64_t)Cout * Cin));
    const float v = w[((int64_t)co * Cin + ci) * taps + tap] * scale;
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) slot[1] = exp2f((float)(e - 14));
}

int tc_split_weights(const float* oihw, __half* hi, __half* lo, int Cout, int Cin, int k, float* scale_slot,
                     cudaStream_t st) {
  return tc_split_weights_taps(oihw, hi, lo, Cout, Cin, k * k, scale_slot, st);
}

int tc_split_weights_taps(const float* oihw, __half* hi, __half* lo, int Cout, int Cin, int taps, float* scale_slot,
                          cudaStream_t st) {
  const int64_t total = (int64_t)Cout * Cin * taps;
  const int64_t blocks = (total + 255) / 256;
  const unsigned g = (unsigned)(blocks > 1024 ? 1024 : blocks);
  CFB_CUDA(cudaMemsetAsync(scale_slot, 0, 2 * sizeof(float), st));
  tc_absmax_kernel<<<g, 256, 0, st>>>(oihw, total, reinterpret_cast<unsigned*>(scale_slot));
  CFB_LAUNCH_CHECK();
  tc_split_weights_kernel<<<g, 256, 0, st>>>(oihw, hi, lo, Cout, Cin, taps, scale_slot);
  CFB_LAUNCH_CHECK();
  return 0;
}

// Upsample (nearest x2) followed by a 3x3 conv == four 2x2 convs on the LOW-resolution tensor, one per output parity
// (py,px): out[2y+py][2x+px] = sum_{dy,dx in {0,1}} W'[py][px][dy][dx] . in[y+dy+py-1][x+dx+px-1], where W' pre-sums the 3x3
// taps that read the same source pixel (rows: py=0 -> {r0 | r1+r2}, py=1 -> {r0+r1 | r2}; same for columns).  2.25x fewer
// MACs and the operand planes stay at the low resolution.  Sums are formed in fp32 before the hi/lo split.
__device__ __forceinline__ void up4_range(int parity, int d, int& lo, int& hi) {
  if (parity == 0) { lo = d == 0 ? 0 : 1; hi = d == 0 ? 0 : 2; }
  else { lo = d == 0 ? 0 : 2; hi = d == 0 ? 1 : 2; }
}
__device__ __forceinline__ float up4_weight(const float* __restrict__ w, int co, int ci, int Cin, int tap16) {
  const int ph = tap16 >> 2, py = ph >> 1, px = ph & 1, dy = (tap16 >> 1) & 1, dx = tap16 & 1;
  int r0, r1, s0, s1;
  up4_range(py, dy, r0, r1);
  up4_range(px, dx, s0, s1);
  float v = 0.f;
  for (int r = r0; r <= r1; ++r)
    for (int q = s0; q <= s1; ++q) v += w[(((int64_t)co * Cin + ci) * 3 + r) * 3 + q];
  return v;
}
__global__ void tc_absmax_up4_kernel(const float* __restrict__ w, int Cout, int Cin, unsigned* __restrict__ slot) {
  const int64_t total = (int64_t)16 * Cout * Cin;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cin), co = (int)((i / Cin) % Cout), tap = (int)(i / ((int64_t)Cout * Cin));
    m = fmaxf(m, fabsf(up4_weight(w, co, ci, Cin, tap)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(slot, __float_as_uint(m));
}
__global__ void tc_split_up4_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo, int Cout,
                                    int Cin, float* __restrict__ slot) {
  const float amax = __uint_as_float(reinterpret_cast<const unsigned*>(slot)[0]);
  int e = 0;
  if (amax > 0.f && isfinite(amax)) frexpf(amax, &e);
  const float scale = exp2f((float)(14 - e));
  const int64_t total = (int64_t)16 * Cout * Cin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cin), co = (int)((i / Cin) % Cout), tap = (int)(i / ((int64_t)Cout * Cin));
    const float v = up4_weight(w, co, ci, Cin, tap) * scale;
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(v - __half2float(h));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) slot[1] = exp2f((float)(e - 14));
}
int tc_split_weights_up4(const float* oihw3x3, __half* hi, __half* lo, int Cout, int Cin, float* scale_slot, cudaStream_t st) {
  const int64_t total = (int64_t)16 * Cout * Cin;
  const int64_t blocks = (total + 255) / 256;
  const unsigned g = (unsigned)(blocks > 1024 ? 1024 : blocks);
  CFB_CUDA(cudaMemsetAsync(scale_slot, 0, 2 * sizeof(float), st));
  tc_absmax_up4_kernel<<<g, 256, 0, st>>>(oihw3x3, Cout, Cin, reinterpret_cast<unsigned*>(scale_slot));
  CFB_LAUNCH_CHECK();
  tc_split_up4_kernel<<<g, 256, 0, st>>>(oihw3x3, hi, lo, Cout, Cin, scale_slot);
  CFB_LAUNCH_CHECK();
  return 0;
}

__device__ void report_overflow();       // status word, defined with the barrier helpers below

// ------------------------------------------------------------------------------------------------------
// operand preparation: fp32 NHWC (+ fused GroupNorm affine, SiLU, nearest x2) -> fp16 hi / lo NHWC planes
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float tc_silu(float x) { return x / (1.f + expf(-x)); }
// output SiLU of the epilogues (YOLOv5 Conv): the fast exponential and division keep the epilogue's register budget; __expf
// is within 2 + 1.173 |x| ulp, far inside the fp32 parity bars of the detector
__device__ __forceinline__ float tc_silu_out(float x) { return __fdividef(x, 1.f + __expf(-x)); }

// One block = PB consecutive output pixels of ONE image; a thread keeps the same 8-channel slice for all its pixels, so
// the per-(n,c) GroupNorm scale/shift is loaded once per block instead of once per element.
__global__ void __launch_bounds__(256) tc_prep_kernel(const float* __restrict__ in, const float* __restrict__ scale,
                                                      const float* __restrict__ shift, int act, int up, int N, int H, int W,
                                                      int C, int PB, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int C8 = C >> 3;
  const int Hp = H << up, Wp = W << up;
  const int64_t img_px = (int64_t)Hp * Wp;
  const int64_t pix0 = (int64_t)blockIdx.x * PB;          // PB divides Hp*Wp: the block stays inside image n
  const int n = (int)(pix0 / img_px);
  const int c = (threadIdx.x % C8) * 8;
  const int pstep = 256 / C8;
  float sv[8], hv[8];
  if (scale) {
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + (int64_t)n * C + c));
    const float4 s1 = __ldg(reinterpret_cast<const float4*>(scale + (int64_t)n * C + c + 4));
    const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + (int64_t)n * C + c));
    const float4 h1 = __ldg(reinterpret_cast<const float4*>(shift + (int64_t)n * C + c + 4));
    sv[0] = s0.x; sv[1] = s0.y; sv[2] = s0.z; sv[3] = s0.w; sv[4] = s1.x; sv[5] = s1.y; sv[6] = s1.z; sv[7] = s1.w;
    hv[0] = h0.x; hv[1] = h0.y; hv[2] = h0.z; hv[3] = h0.w; hv[4] = h1.x; hv[5] = h1.y; hv[6] = h1.z; hv[7] = h1.w;
  }
  float vmax = 0.f;
  for (int pl = threadIdx.x / C8; pl < PB; pl += pstep) {
    const int64_t pix = pix0 + pl;
    const int64_t rem = pix - (int64_t)n * img_px;
    const int oy = (int)(rem / Wp), ox = (int)(rem - (int64_t)oy * Wp);
    const float* src = in + (((int64_t)n * H + (oy >> up)) * W + (ox >> up)) * C + c;
    const float4 a = __ldg(reinterpret_cast<const float4*>(src));
    const float4 b = __ldg(reinterpret_cast<const float4*>(src + 4));
    float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    if (scale) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], sv[j], hv[j]);
    }
    if (act == IN_SILU) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = tc_silu(v[j]);
    }
    __align__(16) __half hh[8];
    __align__(16) __half ll[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      vmax = fmaxf(vmax, fabsf(v[j]));
      hh[j] = __float2half_rn(v[j]);
      ll[j] = __float2half_rn(v[j] - __half2float(hh[j]));
    }
    *reinterpret_cast<uint4*>(hi + pix * C + c) = *reinterpret_cast<const uint4*>(hh);
    *reinterpret_cast<uint4*>(lo + pix * C + c) = *reinterpret_cast<const uint4*>(ll);
  }
  if (vmax > 65504.f) report_overflow();       // fp16 operand range guard: reported through the status word, never silent
}

// The raw split of activations whose channel count is a multiple of 64 but not 64 * 2^k (Inception-v3's 192, 320, 448, 768,
// 1280): one thread per 8 channels of a pixel, the same values as tc_prep_kernel without an affine.
__global__ void __launch_bounds__(256) tc_prep_raw_kernel(const float* __restrict__ in, int64_t items, __half* __restrict__ hi,
                                                          __half* __restrict__ lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float vmax = 0.f;
  if (i < items) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(in + i * 8));
    const float4 b = __ldg(reinterpret_cast<const float4*>(in + i * 8 + 4));
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    __align__(16) __half hh[8];
    __align__(16) __half ll[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      vmax = fmaxf(vmax, fabsf(v[j]));
      hh[j] = __float2half_rn(v[j]);
      ll[j] = __float2half_rn(v[j] - __half2float(hh[j]));
    }
    *reinterpret_cast<uint4*>(hi + i * 8) = *reinterpret_cast<const uint4*>(hh);
    *reinterpret_cast<uint4*>(lo + i * 8) = *reinterpret_cast<const uint4*>(ll);
  }
  if (vmax > 65504.f) report_overflow();
}

// torch.cat([enc_feat, dec], dim=1) of Fuse_sft_block (codeformer_arch.py:152) written directly as RAW fp16 hi/lo operand
// planes: the fused ResBlock reads the concatenation only through the tensor engine (conv1 transforms it in-kernel, the
// 1x1 conv_out takes it raw) and its GroupNorm statistics come from the sources' partial sums, so no fp32 copy is needed.
__global__ void __launch_bounds__(256) concat_planes_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                            __half* __restrict__ hi, __half* __restrict__ lo, int64_t pixels,
                                                            int Ca, int Cb) {
  pdl_launch_dependents();
  pdl_wait();
  const int C8 = (Ca + Cb) >> 3;
  const int64_t total = pixels * C8;
  float vmax = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i / C8;
    const int c = (int)(i - px * C8) * 8;
    const float* src = c < Ca ? a + px * Ca + c : b + px * Cb + (c - Ca);
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(src)), v1 = __ldg(reinterpret_cast<const float4*>(src + 4));
    const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
    __align__(16) __half hh[8];
    __align__(16) __half ll[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      vmax = fmaxf(vmax, fabsf(v[j]));
      hh[j] = __float2half_rn(v[j]);
      ll[j] = __float2half_rn(v[j] - __half2float(hh[j]));
    }
    *reinterpret_cast<uint4*>(hi + px * (Ca + Cb) + c) = *reinterpret_cast<const uint4*>(hh);
    *reinterpret_cast<uint4*>(lo + px * (Ca + Cb) + c) = *reinterpret_cast<const uint4*>(ll);
  }
  if (vmax > 65504.f) report_overflow();
}
int concat_planes(const float* a, const float* b, void* planes, int64_t pixels, int Ca, int Cb, cudaStream_t st) {
  CFB_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "concat_planes: channel counts must be multiples of 8");
  if (pixels == 0) return 0;
  const size_t plane = ((size_t)pixels * (Ca + Cb) * 2 + 1023) / 1024 * 1024;
  const int64_t total = pixels * ((Ca + Cb) >> 3);
  const int64_t blocks = (total + 255) / 256;
  CFB_LAUNCH_PDL(concat_planes_kernel, dim3((unsigned)(blocks > 148 * 32 ? 148 * 32 : blocks)), dim3(256), 0, st, a, b, (__half*)planes,
                 (__half*)((char*)planes + plane), pixels, Ca, Cb);
  return 0;
}

// ------------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive when `pred` holds (a predicated instruction, no branch)
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
               ::"r"(bar), "r"((uint32_t)pred) : "memory");
}
// Bounded wait without a trap.  A protocol bug (or an injected fault) must surface as a Python exception, never as a hung
// GPU and never as a sticky context error (SURVEY.md section 8(b) "Errors": the reference's callers catch RuntimeError and
// fall back to the input face, inference_codeformer.py:209-211).  On time-out the waiting thread raises the device-wide
// abort flag and reports through the host-mapped status word; every other wait loop sees the flag after its next failed
// try_wait; a warp that has seen it leaves its role loop at once (no further TMA / MMA / barrier traffic), all warps meet at
// the kernel's tear-down, the kernel exits normally and the host turns the status word into an error (runtime.cu:
// async_status_check).  The results of that launch are garbage by contract.
__device__ unsigned g_abort = 0;                 // per device: set on a barrier time-out, cleared by the host when it reports it
__device__ unsigned* g_status_host = nullptr;    // host-mapped status word (bit 0: barrier time-out, bit 1: fp16 operand overflow)
__device__ long long g_wait_limit = 4000000000LL;   // cycles (~2 s); the fault-injection test lowers it

__device__ __noinline__ void mbar_timeout() {
  atomicExch(&g_abort, 1u);
  if (g_status_host) { atomicOr_system(g_status_host, CFB_STATUS_TIMEOUT); __threadfence_system(); }
}
__device__ __noinline__ void report_overflow() {
  if (g_status_host) { atomicOr_system(g_status_host, CFB_STATUS_OVERFLOW); __threadfence_system(); }
}
// RELAX_NS > 0: a producer / helper role whose wake-up latency is not critical sleeps between polls, leaving the issue slots
// to the working warps of its scheduler (a failed try_wait comes back after a few hundred cycles, whatever the hint says:
// in the round-2 profile the poll loops of 19 warps were 40 % of all executed instructions).  The abort flag and the
// time-out clock are only looked at every 128 failed polls.
template <int RELAX_NS = 0>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, bool& aborted) {
  uint32_t done = 0;
  uint32_t polls = 0;
  long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(0x989680u)
        : "memory");
    if (done) break;
    if (RELAX_NS > 0) __nanosleep(RELAX_NS);
    if ((++polls & 127u) == 0u) {
      if (*(volatile unsigned*)&g_abort) { aborted = true; break; }
      if (t0 == 0) t0 = clock64();
      else if (clock64() - t0 > *(volatile long long*)&g_wait_limit) { mbar_timeout(); aborted = true; break; }
    }
  }
  aborted = __any_sync(0xffffffffu, aborted);      // the whole (converged) warp takes the same decision
}
// diagnostics kernels: plain bounded wait
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(0x989680u)
        : "memory");
    if (!done && clock64() - t0 > *(volatile long long*)&g_wait_limit) { mbar_timeout(); break; }
  }
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// the same with an L2 cache policy (createpolicy): the weight slices every CTA of a conv streams stay resident in L2 while the
// activations stream through it
__device__ __forceinline__ void tma_load_3d_hint(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                                 uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_last_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// One leader lane of a fully converged warp (same lane every time).  Keeping the role warps converged and predicating
// only the issue instructions lets ptxas hold descriptors / addresses in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- warpgroup MMA (wgmma, sm_90a) ----
// K-major, 128B-swizzled operand tile (rows of 128 B, 8-row core-matrix groups `sbo` bytes apart): start address >> 4 in
// bits [0,14), leading-byte offset 1 (unused by swizzled K-major layouts), stride-byte offset >> 4 in bits [32,46), layout
// SWIZZLE_128B (1) in bits [62,64).  Stepping K by 16 elements inside the 128-byte row = +32 B on the start address.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers:
// thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8*j + 2*(t%4) (+1), j = 0..7
__device__ __forceinline__ void wg_mma_64x64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accum)
      : "memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T: same register layout with j = 0..15
__device__ __forceinline__ void wg_mma_64x128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accum)
      : "memory");
}
__device__ __forceinline__ void wg_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// Per-warpgroup register limit (.sync.aligned: every thread of the warpgroup executes it).  `inc` blocks until other
// warpgroups have released enough registers with `dec`.
template <int N> __device__ __forceinline__ void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// Warpgroup-uniform decision (named barrier `bar_id` over the 128 threads of one MMA warpgroup: 2 for physical warps 0..3, 3
// for warps 4..7): true when `v` holds in any thread.  The wgmma instructions are .sync.aligned over the warpgroup, so after a
// barrier wait that may have been abandoned (time-out / device-wide abort flag) the four warps must agree before any of them
// issues the next one.
__device__ __forceinline__ bool wg_any(bool v, uint32_t bar_id = 2) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.or.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r)
      : "r"((uint32_t)v), "r"(bar_id)
      : "memory");
  return r != 0;
}

// ------------------------------------------------------------------------------------------------------
// fused operand transform: per-patch worker of the transform warps (see conv_tc_kernel, XF)
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_ftz(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_ftz(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {      // {hi:16 | lo:16}, round to nearest even
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// float(h) - c with one rounding (the fp16 -> fp32 conversion is exact); h = fp16 bits
__device__ __forceinline__ float f16_minus_f32(uint32_t h, float c) {
  return __half2float(__ushort_as_half((unsigned short)h)) - c;
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// float4 forms for the epilogue's transpose patches.  The dynamic shared-memory base is realigned through an integer cast, so
// plain pointer accesses compile to GENERIC ld/st (LD.E / ST.E with 64-bit address arithmetic); these stay in the shared window.
// No "memory" clobber: volatile asms keep their mutual order and every write -> read hand-off of a patch crosses a
// __syncwarp(), while the compiler stays free to move the residual / SFT global loads of a row batch ahead of them.
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128f(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d));
}
// 8 raw values -> y = act(x * sc + sh) -> fp16 hi / lo words.  MODE 2: affine + SiLU, 1: affine, 0: plain split.
// SiLU = y / (1 + 2^(-y log2 e)) with ex2.approx / rcp.approx (~2^-21 relative: below the hi/lo operand error of 2^-22..2^-21).
// lo = rn(y - hi) is formed as -(hi - y) with one subtract per element and a sign flip of the packed pair.
// LO = false (single-pass fp16 variant): hi only, lv is left unwritten.
template <int MODE, bool LO = true>
__device__ __forceinline__ void xf_chunk(const uint4& a, const uint4& b, const float (&sc)[8], const float (&sh)[8], uint4& hv,
                                         uint4& lv, float& amax) {
  const uint32_t raw[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float y[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = __uint_as_float(raw[2 * q + e]);
      if (MODE >= 1) v = fmaf(v, sc[2 * q + e], sh[2 * q + e]);
      if (MODE == 2) v = v * rcp_ftz(1.f + ex2_ftz(v * -1.4426950408889634f));
      y[e] = v;
    }
    amax = fmaxf(amax, fmaxf(fabsf(y[0]), fabsf(y[1])));
    hw[q] = pack_f16x2(y[0], y[1]);
    if constexpr (LO) {
      const float d0 = f16_minus_f32(hw[q] & 0xffffu, y[0]);    // hi - y = -lo
      const float d1 = f16_minus_f32(hw[q] >> 16, y[1]);
      lw[q] = pack_f16x2(d0, d1) ^ 0x80008000u;
    }
  }
  hv = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  if constexpr (LO) lv = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}
// One patch: RPP rows per pass (8 lanes per row), two passes in flight per iteration.  LO = false: the hi plane only.
// The 2 transform warps of the 128-wide tiles (RPP = 8) run on 96 registers: their 12 iterations stay a loop, which
// ptxas would otherwise interleave into spills.
template <int MODE, int RPP, int NPASS, int PW, int ROWS, bool LO = true>
__device__ __forceinline__ void xf_patch(uint32_t src_base, uint32_t hi_base, uint32_t lo_base, int c0, int j, int rsub,
                                         const float (&sc)[8], const float (&sh)[8], bool border, int y0, int x0, int Hin,
                                         int Win, float& amax) {
#pragma unroll (RPP >= 16 ? 64 : 1)
  for (int it = 0; it < NPASS; it += 2) {
    uint4 a[2], b[2];
    bool act[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int r = rsub + (it + u) * RPP;
      act[u] = (it + u < NPASS) && (r < ROWS);                 // warp-uniform: a warp owns 4 consecutive rows and ROWS % 4 == 0
      if (act[u]) {
        const uint32_t row = src_base + (uint32_t)r * 128u;
        const uint32_t sw = (row >> 7) & 7u;                    // swizzle phase = absolute address bits [7,10)
        a[u] = lds128(row + (((uint32_t)c0 ^ sw) << 4));
        b[u] = lds128(row + (((uint32_t)(c0 + 1) ^ sw) << 4));
      }
    }
    __syncwarp();                                              // every lane of the row has loaded before any lane stores
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (act[u]) {
        const int r = rsub + (it + u) * RPP;
        uint4 hv, lv;
        xf_chunk<MODE, LO>(a[u], b[u], sc, sh, hv, lv, amax);
        if (border) {
          const int py = r / PW, px = r - py * PW;
          if (!((unsigned)(y0 + py) < (unsigned)Hin && (unsigned)(x0 + px) < (unsigned)Win)) {
            hv = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (LO) lv = make_uint4(0u, 0u, 0u, 0u);
          }
        }
        const uint32_t hrow = hi_base + (uint32_t)r * 128u, lrow = lo_base + (uint32_t)r * 128u;
        sts128(hrow + ((((uint32_t)j) ^ ((hrow >> 7) & 7u)) << 4), hv);
        if constexpr (LO) sts128(lrow + ((((uint32_t)j) ^ ((lrow >> 7) & 7u)) << 4), lv);
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------
// Phase stamps are a BUILD option: -DCFB_TC_STAMPS=1 (production builds omit the tests and the struct field).
#ifndef CFB_TC_STAMPS
#define CFB_TC_STAMPS 0
#endif
struct TcParams {
  int N, Ho, Wo, Cout;
  int taps, pad, stride;  // 9/1/1 (3x3 'same'), 1/0/1 (1x1), 9/0/2 (Downsample: pad right/bottom = TMA OOB zero fill)
  int kw, pad_w;          // per-tap engine: taps per kernel row and the left padding (pad = the top padding); square: 3|1, pad
  int BW, BH;             // pixel tile = BH rows x BW cols = 128
  int tiles_x, tiles_y;   // per image
  int m_tiles, n_tiles;
  int kblocks;            // Cin / 64
  int chunk;              // k-blocks accumulated by the MMA warpgroup before the partial sum is folded by the epilogue
  int a_c0, b_c0;         // channel offsets of the A / B operand inside their planes (batched-GEMM mode)
  int b_batched;          // B operand is a per-image activation plane: third TMA coordinate = image index, not the tap
  // batched GEMM over (image, head) pairs (multi-head attention): the "image" index nb of an m-tile is n * heads + h
  int heads;              // 1: plain
  int a_c_head, b_c_head; // channel offset per head inside the A / B planes
  int a_img_per_head;     // A planes hold one image per (n, h) (softmax probabilities) instead of one per n
  int b_r_head;           // row offset per head inside the B planes (V^T: rows = h*64 + c)
  int out_per_head;       // 1: out is [n*heads + h][256][Cout]; 0: out is [n][256][Cout] and head h owns columns [h*o_c_head, ..)
  int o_c_head;
  int up4;                // Upsample as four 2x2 convs: m-tile = (low-res tile, output parity), 4 taps, weights [16][Cout][Cin]
  int PW, PH;             // halo engine: input patch (BW+k-1) x (BH+k-1) pixels fetched once per 64-channel block
  // GEN variant (XF only; ParseNet / RRDBNet): true image sizes with ragged tiles, padding mode of the halo patch, output
  // placement into a wider buffer, a second (scaled) residual, stride-2 by subsampling
  int Hin, Win;           // true input height / width (tiles are ceil-divided; out-of-image patch pixels follow pad_mode)
  int pad_mode;           // 0 zero, 1 reflect (ReflectionPad2d), 2 replicate (reflection padding of a nearest-x2 upsampled tensor)
  int sub;                // 1: keep only the even output positions (3x3 stride-2 pad-1 conv == its stride-1 result subsampled)
  int out_pitch, out_c0, cout_valid;   // destination: channels per pixel, channel offset, number of real output channels
  int res_pitch;          // channels per pixel of `residual`
  const float* residual2; // out = (conv + bias + residual) * post_scale + residual2
  int res2_pitch;
  float post_scale;
  int fault;              // test hook (cfb_debug_inject_fault): CTA 0 drops the weight load of its first stage -> barrier time-out
  int xform;              // XF kernel variant requested (in_scale may be null: raw split)
  int a_split;            // XF: k-blocks [0, a_split) are read from fp32 source 0 (tmA_hi), the rest from source 1 (tmA_lo)
  const float* in_scale;    // XF: per-(n, cin) affine of the fused operand transform (GroupNorm folded), and its activation
  const float* in_shift;
  int in_act;
  const float* bias;
  const float* residual;
  int out_act;
  const float* sft_dec;
  const float* sft_scale;
  union {
    float sft_w;
    float prelu;            // PRELU kernels (ResNetArcFace, no SFT epilogue): the PReLU slope
  };
  const float* wscale_inv;  // device scalar: 2^-k of the weight split
  float* out;
  __half* pl_hi;            // optional: `out` again as fp16 hi / lo planes (operand of a following raw-input conv)
  __half* pl_lo;
  float* gn_part;           // optional GroupNorm(32) partials of `out`: [m_tile*4 + warp][32][mean, M2]
  int gn_cpg;               // channels per group = Cout/32
  const float* sft_wv;      // [N] per-image w in place of sft_w | null (ConvArgs::sft_wv; raw-input kernels only, !XF)
#if CFB_TC_STAMPS
  long long* dbg;           // diagnostics (cfb_debug_set_stamps): CTA 0 writes clock64() at its role hand-offs; null in production
#endif
};
// phase stamps of CTA 0: one lane per role writes the SM cycle counter
// Wait counters of the 128 x 128 tiles (same build option): every CTA adds the cycles its roles spend in each wait to
// dbg[TC_CNT0 + blockIdx.x * TC_NCNT + k], summed over the warps of the role (lane 0 of each warp adds):
//   MMA warpgroups  0 weight `full`, 1 patch `afull`, 2 `cempty` before the tile hand-off, 3 whole role
//   epilogue warps  4 `cfull`, 5 residual / SFT loads (issue until the last value of the batch has arrived), 6 stores
//                   (output, operand planes, GroupNorm partials), 7 whole role
// TC_T0 / TC_ADD expand to nothing in production builds.
#if CFB_TC_STAMPS
constexpr int TC_CNT0 = 32, TC_NCNT = 8;
#define TC_STAMP(i) do { if (p.dbg != nullptr && blockIdx.x == 0) p.dbg[i] = clock64(); } while (0)
#define TC_T0(t) const long long t = clock64()
#define TC_ADD(k, t) do { if (WIDE && p.dbg != nullptr && lane == 0) \
    atomicAdd(reinterpret_cast<unsigned long long*>(p.dbg + TC_CNT0 + blockIdx.x * TC_NCNT + (k)), \
              (unsigned long long)(clock64() - (t))); } while (0)
#else
#define TC_STAMP(i) do { } while (0)
#define TC_T0(t) do { } while (0)
#define TC_ADD(k, t) do { } while (0)
#endif
// the same with a running sum in a register, added to counter k once per tile (TC_FLUSH)
#if CFB_TC_STAMPS
#define TC_VAR(v) long long v = 0
#define TC_SUM(v, t) v += clock64() - (t)
#define TC_FLUSH(k, v) do { if (WIDE && p.dbg != nullptr && lane == 0) \
    atomicAdd(reinterpret_cast<unsigned long long*>(p.dbg + TC_CNT0 + blockIdx.x * TC_NCNT + (k)), (unsigned long long)(v)); \
    v = 0; } while (0)
#else
#define TC_VAR(v) do { } while (0)
#define TC_SUM(v, t) do { } while (0)
#define TC_FLUSH(k, v) do { } while (0)
#endif
#if CFB_TC_STAMPS
// diagnostics: a warp vote that reads `v`, so a clock read after it is taken once the load of `v` has completed
__device__ __forceinline__ void tc_arrived(float v) {
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.eq.f32 p, %0, 0f00000000;\n\tvote.sync.any.pred q, p, 0xffffffff;\n\t}" ::"f"(v));
}
#endif

// XF (fused operand transform): the warps after the epilogue warps transform the A patches, the warp after them loads the raw
// patches.
constexpr int XF_SKEW = 128;                          // byte skew of the second patch plane (see the transform warps)
constexpr int TC_A_BYTES = 128 * 128;                 // 128 pixels x 64 fp16

// Tiles are 128 output pixels x BN output channels.
//   BN = 64 (every engine): one MMA warpgroup issues the wgmma of the whole 128-row tile into 2 x 32 fp32 registers per thread
//     and hands every partial sum to 8 epilogue warps (4 row quadrants x 2 column halves), which fold it into registers.
//   BN = 128 (halo engine, 3x3 and Upsample convs with Cout % 128 == 0): two MMA warpgroups, one per 64-pixel half, issue
//     m64n128k16 into 64 fp32 registers per thread and fold their partial sums themselves into a 64-float running sum in
//     registers; the finished tile goes through the shared fp32 tile slot once, and 4 epilogue warps (one per row quadrant,
//     all 128 columns) read it from there.  A 64-channel patch is transformed once per 128 output channels instead of once
//     per 64, and each A byte read from shared memory feeds twice the MACs.  16 warps (8 MMA, TMA, 4 epilogue, 2 transform,
//     patch loader; without the transform 3 idle warps) in 4 warpgroups: the MMA warpgroups run on 160 registers, the
//     others on 96 (setmaxnreg).
template <int BN>
struct TcCfg {
  static_assert(BN == 64 || BN == 128, "the wgmma engine runs 64- or 128-wide n-tiles");
  static constexpr bool WIDE = BN == 128;
  static constexpr int MMA_WARPS = WIDE ? 8 : 4;
  static constexpr int EPI_WARPS = WIDE ? 4 : 8;
  // MMA warpgroup(s), TMA warp, epilogue warps; BN = 128 runs whole warpgroups (setmaxnreg), padded with 3 idle warps
  static constexpr int THREADS = WIDE ? 512 : 32 * (MMA_WARPS + 1 + EPI_WARPS);
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = 2 * TC_A_BYTES + 2 * B_BYTES;
  static constexpr int STAGES = 3;
  // Partial-sum hand-off (128 rows, padded by 4 floats against bank conflicts).  BN = 64: the MMA warpgroup stores each
  // partial sum here and goes on with the next chunk while the epilogue warps fold the slot into their fp32 registers with
  // round-to-nearest adds.  BN = 128: the MMA warpgroups store the finished tile here once (their running sum in registers:
  // first chunk 0 + sum, later chunks added with round-to-nearest adds, the same sums in the same order), the epilogue reads
  // it once.
  static constexpr int SLOT_PITCH = BN + 4;
  static constexpr int SLOT_BYTES = 128 * SLOT_PITCH * 4;
  static constexpr int SLOTS = 1;
  static constexpr int STG_BYTES = WIDE ? 0 : 8 * 4096;    // per-epilogue-warp 32x32-float transpose patches
  static constexpr int TAIL_BYTES = SLOT_BYTES + 1024 /*align slack*/ + 512 /*barriers*/ + STG_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + TAIL_BYTES;
  // halo engine: 16x8-pixel tiles; the (16+2)x(8+2) input patch of one 64-channel block is fetched ONCE (hi and lo
  // planes) and all 9 taps read it through row-shifted wgmma descriptors; weights stream through their own ring.
  static constexpr int H_A_PLANE = 23 * 1024;              // >= 18*10*128 B, 1024-aligned
  static constexpr int H_A_SLOT = 2 * H_A_PLANE;
  static constexpr int H_A_SLOTS = 2;
  static constexpr int H_B_SLOT = 2 * B_BYTES;
  static constexpr int H_B_SLOTS = WIDE ? 2 : 4;           // 2 x 32 KB: a refill has one k-block (1536 MMA clocks) to land
                                                           // (single pass: 4 x 16 KB hi-only slots in the same memory)
  static constexpr int H_SMEM_BYTES = H_A_SLOTS * H_A_SLOT + H_B_SLOTS * H_B_SLOT + TAIL_BYTES;
  // fused operand transform (XF, halo engine only): the A patches arrive as the RAW fp32 activation (two 32-channel planes per
  // slot) and the transform warps apply GroupNorm-affine + SiLU + the hi/lo split in place before the MMAs read them
  static constexpr int XF_WARPS = WIDE ? 2 : 4;             // a BN = 128 patch feeds twice the MMA time of a BN = 64 one
  static constexpr int XF_THREADS = 32 * (MMA_WARPS + 1 + EPI_WARPS + XF_WARPS + 1);
  static_assert(!WIDE || XF_THREADS == THREADS, "the 128-wide transform variant fills the pad warps exactly");
  static constexpr int X_A_SLOTS = 2;
  static constexpr int X_A_PLANE2 = H_A_PLANE + XF_SKEW;   // second plane of an XF slot (ends at 46720 <= H_A_SLOT)
  static constexpr int X_B_SLOTS = H_B_SLOTS;
  static constexpr int X_SMEM_BYTES = X_A_SLOTS * H_A_SLOT + X_B_SLOTS * H_B_SLOT + TAIL_BYTES;
};

// Accumulation scheme (why the partial-sum slot): the tensor core adds into its fp32 accumulator with truncation, so a long
// K loop into one accumulator drifts by ~(#MMAs)*2^-25 relative (2e-5 at K=4608 -- too much for the 1e-3 end-to-end bar).
// The MMA warpgroup therefore only accumulates `chunk` k-blocks (64 K-elements each) per partial sum, issuing the small
// cross terms (lo*hi, hi*lo) of every k-step before hi*hi, and the epilogue warps fold every finished partial sum into fp32
// registers with round-to-nearest adds.
// CPG > 0: the epilogue also emits GroupNorm(32) partials (mean, M2) of the stored tile (CPG = Cout/32 channels per group).
// CM (channel-major, BN = 64 only): the MMA warpgroup computes the tile transposed, D^T[64 channels x 128 pixels] =
// W[64 x K] * X[128 x K]^T, as one m64n128k16 per product and k-step (weights = A operand, halo patch = B operand), and stores
// each partial sum into the slot as [pixel][channel]: the epilogue is that of the pixel-major 128 x 64 tile.
// P1 (single-pass fp16): one product A_hi B_hi per k-step instead of three.  Only the hi weight plane fp16(w * 2^k) is
// loaded, the transform warps write only the hi plane fp16(y), and a raw-planes input has only its hi plane fp16(x) loaded;
// accumulation, chunked partial sums and their round-to-nearest folds are those of the split scheme, and wscale_inv undoes
// 2^k exactly.  Built for GEN without SiLU (RRDBNet), the 128-wide and channel-major halo tiles and the per-tap engine
// (CodeFormer's generator and Fuse_sft_block convs); K1 and the SiLU epilogue stay split.
// PRELU: the epilogue activation is v > 0 ? v : p.prelu * v (ResNetArcFace); built for the generalised engine and the plain
// per-tap engine, so that no other variant carries the branch.
template <int BN, int CPG, bool HALO, bool XF, bool GEN = false, bool K1 = false, bool CM = false, bool SILU = false,
          bool P1 = false, bool PRELU = false>
__global__ void __launch_bounds__(XF ? TcCfg<BN>::XF_THREADS : TcCfg<BN>::THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo, const TcParams p) {
  static_assert(!XF || HALO, "the fused operand transform exists for the halo engine only");
  static_assert(!GEN || (XF && CPG == 0), "the generalised addressing exists for the fused-transform engine only");
  static_assert(!PRELU || (BN == 64 && CPG == 0 && !K1 && !CM && !SILU && !P1 && (GEN || !HALO)),
                "the PReLU epilogue is built for the generalised and the per-tap engines");
  static_assert(!K1 || (XF && !GEN && CPG == 0), "K1 = fused transform of a 1x1 conv (patch = tile): its own instantiation");
  using Cfg = TcCfg<BN>;
  constexpr bool WIDE = Cfg::WIDE;
  static_assert(!WIDE || (HALO && !GEN && !K1 && CPG != 2), "128-wide tiles exist for the 3x3 / Upsample halo engine");
  static_assert(!CM || (BN == 64 && HALO && !GEN && !K1), "channel-major tiles exist for the 64-channel 3x3 / Upsample halo convs");
  static_assert(!P1 || (!SILU && !K1 && (GEN || WIDE || CM || !HALO)),
                "the single-pass fp16 variant is built for the generalised, 128-wide, channel-major and per-tap engines");
  constexpr int MMA_WARPS = Cfg::MMA_WARPS, EPI_WARPS = Cfg::EPI_WARPS;
  constexpr int A_SLOTS = XF ? Cfg::X_A_SLOTS : Cfg::H_A_SLOTS;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;
  const int first_tile = (int)blockIdx.x;
  const int tile_step = (int)gridDim.x;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // ring "full/empty": per-tap engine = STAGES k-block stages; halo engine = weight (B) slots.  "afull/aempty": halo A slots.
  // single-pass 128-wide tiles load only the hi weight plane: the same ring memory holds twice as many slots of half the size,
  // so a refill has two k-blocks of MMA time to land instead of one (their MMAs waited on `full` for 29-44 % of their cycles
  // with the 2-slot ring, tools/epilogue_waits.py)
  constexpr bool HALF_B = HALO && WIDE && P1;
  constexpr int NRING = HALO ? (XF ? Cfg::X_B_SLOTS : Cfg::H_B_SLOTS) * (HALF_B ? 2 : 1) : STAGES;
  constexpr int RING_BYTES = HALO ? (HALF_B ? Cfg::B_BYTES : Cfg::H_B_SLOT) : STAGE_BYTES;
  uint8_t* ring_base = HALO ? smem + A_SLOTS * Cfg::H_A_SLOT : smem;
  float* acc_slot = reinterpret_cast<float*>(ring_base + NRING * RING_BYTES);       // partial sums, [128][SLOT_PITCH]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring_base + NRING * RING_BYTES + Cfg::SLOT_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + NRING;
  uint64_t* cfull = bars + 2 * NRING;
  uint64_t* cempty = bars + 2 * NRING + Cfg::SLOTS;
  uint64_t* afull = bars + 2 * NRING + 2 * Cfg::SLOTS;
  uint64_t* aempty = afull + 3;
  uint64_t* araw = aempty + 3;                       // XF: raw patch landed (TMA -> transform warps)
  uint8_t* stage_buf = reinterpret_cast<uint8_t*>(bars) + 512;      // epilogue transpose patches (16-byte aligned)

  // Roles are numbered logically (0 TMA, 1 MMA, 2.. epilogue, then transform, then the patch loader).  The MMA role is the
  // warpgroup(s) of physical warps 0..MMA_WARPS-1 (wgmma needs aligned warpgroups); the other roles sit on the remaining warp
  // ids in REVERSE order: the sub-partition arbiter favours the highest warp id among its eligible warps, and the TMA producer
  // must never wait for an issue slot, then the epilogue; the instruction-heavy transform warps come last.
  constexpr int NWARPS = (XF ? Cfg::XF_THREADS : Cfg::THREADS) / 32;
  const int pwarp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform
  const int ridx = NWARPS - 1 - pwarp;
  const int warp = pwarp < MMA_WARPS ? 1 : (ridx == 0 ? 0 : ridx + 1);
  const int lane = threadIdx.x & 31;
  bool aborted = false;      // set when a barrier wait timed out anywhere on the device: leave the role loop (see mbar_wait)
  if constexpr (WIDE) {
    // 16 warps cap every thread at 128 registers; the MMA warpgroups (0-1) hold 64 accumulators and the 64-float running sum
    // of their tile, so they take 160 (`inc` at the top of the MMA role) from warpgroups 2-3 (TMA, epilogue, transform,
    // patch loader or idle pad warps), which give theirs back here, before the first barrier of the kernel, and run on 96:
    // 2 x 128 x 160 + 2 x 128 x 96 = 65 536.  `inc` never waits on a warpgroup that is itself waiting (abort path included).
    if (pwarp >= MMA_WARPS) wg_regs_dec<96>();
  }
  if (threadIdx.x == 0) TC_STAMP(0);

  if (warp == 0 && lane == 0) {
    for (int a = 0; a < 3; ++a) {
      mbar_init(smem_u32(afull + a), XF ? Cfg::XF_WARPS : 1);      // XF: every transform warp arrives
      mbar_init(smem_u32(aempty + a), MMA_WARPS);
      mbar_init(smem_u32(araw + a), 1);
    }
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA_lo) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    for (int s = 0; s < NRING; ++s) { mbar_init(smem_u32(full + s), 1); mbar_init(smem_u32(empty + s), MMA_WARPS); }
    for (int a = 0; a < Cfg::SLOTS; ++a) {
      mbar_init(smem_u32(cfull + a), MMA_WARPS);
      mbar_init(smem_u32(cempty + a), EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: everything above touched only this CTA's shared memory and the kernel parameters.
  // The next grid of the stream may start its own set-up now; this one waits here until the previous grid has completed.
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) TC_STAMP(1);

  const int total_tiles = p.m_tiles * p.n_tiles;
  const int nk = p.taps * p.kblocks;

  if (warp == 0) {
    // ============================ TMA producer (warp converged, one elected lane issues) ============================
    {
      int stage = 0;
      uint32_t phase = 0;
      int aslot = 0;
      uint32_t aphase = 0;
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
        const int mtl = p.up4 ? (mt >> 2) : mt;            // low-res tile; (mt & 3) = output parity (py,px)
        const int par_y = p.up4 ? ((mt & 3) >> 1) : 0, par_x = p.up4 ? (mt & 1) : 0;
        const int per_img = p.tiles_x * p.tiles_y;
        const int n = mtl / per_img;
        const int rem = mtl - n * per_img;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        const int y0 = ty * p.BH * p.stride, x0 = tx * p.BW * p.stride;
        if constexpr (HALO) {
          for (int kb = 0; kb < p.kblocks; ++kb) {
            if constexpr (!XF) {
              mbar_wait<500>(smem_u32(aempty + aslot), aphase ^ 1, aborted); if (aborted) goto teardown;
              if (elect_one()) {
                const uint32_t sa = smem_u32(smem + aslot * Cfg::H_A_SLOT);
                const uint32_t ab = smem_u32(afull + aslot);
                mbar_expect_tx(ab, (uint32_t)((P1 ? 1 : 2) * p.PW * p.PH * 128));
                tma_load_4d(sa, &tmA_hi, ab, kb * 64, x0 - p.pad, y0 - p.pad, n);
                if constexpr (!P1) tma_load_4d(sa + Cfg::H_A_PLANE, &tmA_lo, ab, kb * 64, x0 - p.pad, y0 - p.pad, n);
              }
              __syncwarp();
              if (++aslot == A_SLOTS) { aslot = 0; aphase ^= 1; }
            }
            for (int tap = 0; tap < p.taps; ++tap) {
              const int btap = p.up4 ? (mt & 3) * 4 + tap : tap;      // Upsample: weight slice of this output parity
              mbar_wait<500>(smem_u32(empty + stage), phase ^ 1, aborted); if (aborted) goto teardown;
              if (elect_one()) {
                if (tile == first_tile && tap == 0 && kb == 0) TC_STAMP(2);
                const uint32_t sb = smem_u32(ring_base + stage * RING_BYTES);
                const uint32_t fb = smem_u32(full + stage);
                const bool drop = p.fault && blockIdx.x == 0 && tile == first_tile && kb == 0 && tap == 0;   // injected fault
                mbar_expect_tx(fb, (uint32_t)(P1 ? Cfg::B_BYTES : Cfg::H_B_SLOT));
                if constexpr (WIDE && !P1) {
                  // split 128 x 128 tiles: their 2-slot ring gives a refill one k-block to land, and their MMAs waited on
                  // `full` for 32-56 % of their cycles, most with a residual / SFT epilogue streaming activations through L2
                  // (tools/epilogue_waits.py).  The weights every CTA of the conv reads are marked evict_last so that stream
                  // does not push them out.  The single-pass tiles (4 slots) measured slower with the hint.
                  const uint64_t pol = l2_evict_last_policy();
                  if (!drop) tma_load_3d_hint(sb, &tmB_hi, fb, kb * 64, nt * BN, btap, pol);
                  tma_load_3d_hint(sb + Cfg::B_BYTES, &tmB_lo, fb, kb * 64, nt * BN, btap, pol);
                } else {
                  if (!drop) tma_load_3d(sb, &tmB_hi, fb, kb * 64, nt * BN, btap);
                  if constexpr (!P1) tma_load_3d(sb + Cfg::B_BYTES, &tmB_lo, fb, kb * 64, nt * BN, btap);
                }
              }
              __syncwarp();
              if (++stage == NRING) { stage = 0; phase ^= 1; }
            }
          }
        } else {
          for (int tap = 0; tap < p.taps; ++tap) {
            // source offset of this tap and its weight slice: 3x3 -> (r,s)-pad; 2x2 parity conv -> (dy+py-1, dx+px-1)
            int r, s, btap = tap;
            if (p.up4) { r = (tap >> 1) + par_y; s = (tap & 1) + par_x; btap = (mt & 3) * 4 + tap; }
            else { r = tap / p.kw; s = tap - r * p.kw; }          // kh x kw window, row-major taps (OIHW order)
            for (int kb = 0; kb < p.kblocks; ++kb) {
              mbar_wait<500>(smem_u32(empty + stage), phase ^ 1, aborted); if (aborted) goto teardown;
              if (elect_one()) {
                if (tile == first_tile && tap == 0 && kb == 0) TC_STAMP(2);
                const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
                // multi-head batched GEMM: image index n = n_img * heads + head
                const int hh = p.heads > 1 ? n % p.heads : 0, nimg = p.heads > 1 ? n / p.heads : n;
                const int a_img = p.a_img_per_head ? n : nimg;
                const int ac = p.a_c0 + hh * p.a_c_head + kb * 64, bc = p.b_c0 + hh * p.b_c_head + kb * 64;
                const int brow = nt * BN + hh * p.b_r_head;
                const int b3 = p.b_batched ? nimg : btap;
                const uint32_t fb = smem_u32(full + stage);
                const bool drop = p.fault && blockIdx.x == 0 && tile == first_tile && kb == 0 && tap == 0;   // injected fault
                mbar_expect_tx(fb, (uint32_t)(P1 ? TC_A_BYTES + Cfg::B_BYTES : Cfg::STAGE_BYTES));
                tma_load_4d(sa, &tmA_hi, fb, ac, x0 + s - p.pad_w, y0 + r - p.pad, a_img);
                if constexpr (!P1) tma_load_4d(sa + TC_A_BYTES, &tmA_lo, fb, ac, x0 + s - p.pad_w, y0 + r - p.pad, a_img);
                if (!drop) tma_load_3d(sa + 2 * TC_A_BYTES, &tmB_hi, fb, bc, brow, b3);
                if constexpr (!P1) tma_load_3d(sa + 2 * TC_A_BYTES + Cfg::B_BYTES, &tmB_lo, fb, bc, brow, b3);
              }
              __syncwarp();
              if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else if (warp == 1) {
    // ============================ MMA warpgroup(s) (physical warps 0..MMA_WARPS-1) ============================
    // Per k-block (64 K-elements) and 64-row half of the tile: 4 k-steps x {A_lo B_hi, A_hi B_lo, A_hi B_hi}.  BN = 64: one
    // warpgroup issues both halves (m64n64k16); BN = 128: warpgroup `wg` issues half `wg` (m64n128k16); CM: one warpgroup
    // issues the whole transposed tile (m64n128k16, weights as A: W_hi X_lo, W_lo X_hi, W_hi X_hi -- the same products in
    // the same order).  P1: A_hi B_hi (CM: W_hi X_hi) only.
    // A descriptors: per-tap engine = 128 rows of 128 B in 8-row groups 1024 B apart (rows 64..127 start 8 KB in).  Halo
    // engine: rows of the tile are pixels (h, w) of a 16x8 patch; patch row h is one 8-row core-matrix group that starts
    // (h + r) * PW + s rows into the halo buffer => group stride PW*128 B and a start address that is only 128-byte
    // aligned.  The tensor core applies the 128B swizzle on absolute shared-memory address bits, i.e. exactly the pattern
    // the TMA unit used when it wrote the buffer.
    // CM: the same descriptor is the B operand and spans the whole 128-pixel tile: its 16 core-matrix groups are the 16 patch
    // rows, PW*128 B apart, and the second 64-row half starts a_half = 8 groups in.
    if constexpr (WIDE) wg_regs_inc<160>();
    TC_T0(t_mma);
    {
      constexpr bool N128 = WIDE || CM;                 // m64n128k16 issue: one accumulator of 64 fp32 per thread
      constexpr int MH = N128 ? 1 : 2;                  // 64-row halves issued by this warpgroup
      const uint32_t a_sbo = HALO ? (uint32_t)(p.PW * 128) : 1024u;
      const uint32_t a_half = HALO ? (uint32_t)(8 * p.PW * 128) : 8192u;
      const int wq = (int)(threadIdx.x >> 5) & 3;      // 16-row group of this warp inside each 64-row half
      const int wg = (int)(threadIdx.x >> 7);          // BN = 128: the 64-row half of this warpgroup
      const uint32_t bar_id = 2u + (uint32_t)wg;       // named barrier of this warpgroup's abort decision
      const uint32_t slot_base = smem_u32(acc_slot);
      int stage = 0;
      uint32_t phase = 0;
      int slot = 0;
      uint32_t slot_phase = 0;
      int aslot = 0;
      uint32_t aphase = 0;
      float acc[MH][N128 ? 64 : 32];
      if constexpr (N128) {
        // BN = 128 and CM: per chunk of k-blocks, every k-block's group is committed with one earlier group still in flight
        // (wait_group 1, a fixed depth), after which the weight slot (and, after its last tap, the patch) of the PREVIOUS
        // k-block is released; wait_group 0 only after the chunk's last k-block, where the partial sum is folded into the
        // running sum in registers (BN = 128) or handed to the epilogue warps (CM).
        // BN = 128: `run` is the tile's running sum (first chunk 0 + sum, later chunks added with round-to-nearest: the sums
        // of the 128 x 64 path in the same order).  A finished tile is stored into the slot once, after the next tile's first
        // k-block has been issued, so the store runs under that k-block's MMAs and the epilogue has a whole tile of MMA time
        // to drain the slot.
        float run[64];                                               // BN = 128 only (CM never touches it)
        // run -> slot [row][SLOT_PITCH] -> epilogue warps; true when the wait for the slot was abandoned (abort)
        auto hand_off = [&]() -> bool {
          TC_T0(t_h);
          mbar_wait(smem_u32(cempty + slot), slot_phase ^ 1, aborted);
          if (wg_any(aborted, bar_id)) return true;
          TC_ADD(2, t_h);
          const int row = wg * 64 + wq * 16 + (lane >> 2);
          // this thread's first slot element, formed anew per hand-off (opaque move): otherwise the compiler keeps the 32
          // store addresses live across the tile loop and spills them; this way they are immediate offsets of one register
          uint32_t e0;
          asm volatile("mov.b32 %0, %1;" : "=r"(e0)
                       : "r"(slot_base + (uint32_t)(slot * Cfg::SLOT_BYTES) + (uint32_t)((row * Cfg::SLOT_PITCH + 2 * (lane & 3)) * 4)));
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int h8 = 0; h8 < 2; ++h8) {
              const uint32_t e = e0 + (uint32_t)((8 * h8 * Cfg::SLOT_PITCH + 8 * j) * 4);
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(e), "f"(run[4 * j + 2 * h8]), "f"(run[4 * j + 2 * h8 + 1])
                           : "memory");
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(cfull + slot));
          if (++slot == Cfg::SLOTS) { slot = 0; slot_phase ^= 1; }
          return false;
        };
        for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
          const int par = p.up4 ? ((tile / p.n_tiles) & 3) : 0;    // output parity of this tile
          const int par_y = par >> 1, par_x = par & 1;
          for (int c0 = 0; c0 < nk; c0 += p.chunk) {
            const int c1 = min(c0 + p.chunk, nk);
            uint32_t prev_empty = 0, prev_aempty = 0;                // barriers the previous k-block releases (0: none)
            for (int it = c0; it < c1; ++it) {
              const int kb = it / p.taps;
              const int tap = it - kb * p.taps;
              if (tap == 0) {
                TC_T0(t_a);
                mbar_wait(smem_u32(afull + aslot), aphase, aborted);
                if (wg_any(aborted, bar_id)) { wg_wait_all(); aborted = true; goto teardown; }
                TC_ADD(1, t_a);
              }
              int r = (p.taps == 9) ? tap / 3 : 0;
              int sft = (p.taps == 9) ? tap - r * 3 : 0;
              if (p.up4) { r = (tap >> 1) + par_y; sft = (tap & 1) + par_x; }
              const uint32_t a_hi0 = smem_u32(smem + aslot * Cfg::H_A_SLOT) + (uint32_t)((r * p.PW + sft) * 128) +
                                     (uint32_t)wg * a_half;
              const uint32_t a_lo0 = a_hi0 + (uint32_t)(XF ? Cfg::X_A_PLANE2 : Cfg::H_A_PLANE);
              const uint32_t bsm = smem_u32(ring_base + stage * RING_BYTES);
              TC_T0(t_b);
              mbar_wait(smem_u32(full + stage), phase, aborted);
              if (wg_any(aborted, bar_id)) { wg_wait_all(); aborted = true; goto teardown; }
              TC_ADD(0, t_b);
              wg_fence();
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const uint64_t db_hi = wg_desc(bsm + 32 * k, 1024u), db_lo = wg_desc(bsm + Cfg::B_BYTES + 32 * k, 1024u);
                const uint64_t da_hi = wg_desc(a_hi0 + 32 * k, a_sbo), da_lo = wg_desc(a_lo0 + 32 * k, a_sbo);
                if constexpr (P1 && CM) {
                  wg_mma_64x128(acc[0], db_hi, da_hi, (it == c0 && k == 0) ? 0u : 1u);
                } else if constexpr (P1) {
                  wg_mma_64x128(acc[0], da_hi, db_hi, (it == c0 && k == 0) ? 0u : 1u);
                } else if constexpr (CM) {
                  wg_mma_64x128(acc[0], db_hi, da_lo, (it == c0 && k == 0) ? 0u : 1u);
                  wg_mma_64x128(acc[0], db_lo, da_hi, 1u);
                  wg_mma_64x128(acc[0], db_hi, da_hi, 1u);
                } else {
                  wg_mma_64x128(acc[0], da_lo, db_hi, (it == c0 && k == 0) ? 0u : 1u);
                  wg_mma_64x128(acc[0], da_hi, db_lo, 1u);
                  wg_mma_64x128(acc[0], da_hi, db_hi, 1u);
                }
              }
              wg_commit();
              if constexpr (WIDE) {
                if (it == 0 && tile != first_tile) {                 // previous tile -> slot under this k-block's MMAs
                  if (hand_off()) { wg_wait_all(); aborted = true; goto teardown; }
                }
              }
              wg_wait_1();
              __syncwarp();
              mbar_arrive_if(prev_empty, lane == 0 && prev_empty != 0);
              mbar_arrive_if(prev_aempty, lane == 0 && prev_aempty != 0);
              prev_empty = smem_u32(empty + stage);
              prev_aempty = tap == p.taps - 1 ? smem_u32(aempty + aslot) : 0u;
              if (++stage == NRING) { stage = 0; phase ^= 1; }
              if (tap == p.taps - 1 && ++aslot == A_SLOTS) { aslot = 0; aphase ^= 1; }
            }
            wg_wait_all();
            __syncwarp();
            mbar_arrive_if(prev_empty, lane == 0);
            mbar_arrive_if(prev_aempty, lane == 0 && prev_aempty != 0);
            if constexpr (CM) {
              // partial sum -> slot[pixel][channel], folded by the epilogue warps as on the pixel-major tile.  Thread t holds
              // channels 16*(t/32) + (t%32)/4 (+8) and pixels 8j + 2(t%4) (+1); with SLOT_PITCH = 68 the 32 scalar stores of
              // one instruction fall on 32 distinct banks, (4*pixel + channel) mod 32.
              mbar_wait(smem_u32(cempty + slot), slot_phase ^ 1, aborted);
              if (wg_any(aborted, bar_id)) { aborted = true; goto teardown; }
              const uint32_t st0 = slot_base + (uint32_t)(slot * Cfg::SLOT_BYTES) +
                                   (uint32_t)((2 * (lane & 3) * Cfg::SLOT_PITCH + wq * 16 + (lane >> 2)) * 4);
#pragma unroll
              for (int j = 0; j < 16; ++j) {
#pragma unroll
                for (int h8 = 0; h8 < 2; ++h8) {
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const uint32_t a = st0 + (uint32_t)(((8 * j + e) * Cfg::SLOT_PITCH + 8 * h8) * 4);
                    asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(acc[0][4 * j + 2 * h8 + e]) : "memory");
                  }
                }
              }
              __syncwarp();
              if (lane == 0) mbar_arrive(smem_u32(cfull + slot));
              if (++slot == Cfg::SLOTS) { slot = 0; slot_phase ^= 1; }
              continue;
            }
            if constexpr (WIDE) {      // fold: the first chunk gives 0 + sum (+0 for a -0 sum, as the epilogue's fold from 0 would)
#pragma unroll
              for (int i = 0; i < 64; ++i) run[i] = __fadd_rn(c0 == 0 ? 0.f : run[i], acc[0][i]);
            }
          }
        }
        if constexpr (WIDE) {
          if (first_tile < total_tiles && hand_off()) { aborted = true; goto teardown; }      // the last tile
          TC_ADD(3, t_mma);
        }
      } else {
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        const int par = p.up4 ? ((tile / p.n_tiles) & 3) : 0;      // output parity of this tile
        const int par_y = par >> 1, par_x = par & 1;
        for (int it = 0; it < nk; ++it) {
          uint32_t a_hi0, a_lo0, bsm;
          int tap = 0;
          if constexpr (HALO) {
            const int kb = it / p.taps;
            tap = it - kb * p.taps;
            if (tap == 0) { mbar_wait(smem_u32(afull + aslot), aphase, aborted); if (wg_any(aborted)) { aborted = true; goto teardown; } }
            int r = (p.taps == 9) ? tap / 3 : 0;
            int sft = (p.taps == 9) ? tap - r * 3 : 0;
            if (p.up4) { r = (tap >> 1) + par_y; sft = (tap & 1) + par_x; }
            const uint32_t aoff = (uint32_t)((r * p.PW + sft) * 128);
            a_hi0 = smem_u32(smem + aslot * Cfg::H_A_SLOT) + aoff;
            a_lo0 = a_hi0 + (uint32_t)(XF ? Cfg::X_A_PLANE2 : Cfg::H_A_PLANE);
            bsm = smem_u32(ring_base + stage * RING_BYTES);
          } else {
            a_hi0 = smem_u32(smem + stage * STAGE_BYTES);
            a_lo0 = a_hi0 + TC_A_BYTES;
            bsm = a_hi0 + 2 * TC_A_BYTES;
          }
          mbar_wait(smem_u32(full + stage), phase, aborted); if (wg_any(aborted)) { aborted = true; goto teardown; }
          if (blockIdx.x == 0 && threadIdx.x == 0 && tile == first_tile && it == 0) TC_STAMP(3);
          const uint32_t first = (it % p.chunk) == 0 ? 1u : 0u;
          wg_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t db_hi = wg_desc(bsm + 32 * k, 1024u), db_lo = wg_desc(bsm + Cfg::B_BYTES + 32 * k, 1024u);
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
              const uint64_t da_hi = wg_desc(a_hi0 + mh * a_half + 32 * k, a_sbo), da_lo = wg_desc(a_lo0 + mh * a_half + 32 * k, a_sbo);
              if constexpr (P1) {
                wg_mma_64x64(acc[mh], da_hi, db_hi, (first && k == 0) ? 0u : 1u);
              } else {
                wg_mma_64x64(acc[mh], da_lo, db_hi, (first && k == 0) ? 0u : 1u);
                wg_mma_64x64(acc[mh], da_hi, db_lo, 1u);
                wg_mma_64x64(acc[mh], da_hi, db_hi, 1u);
              }
            }
          }
          wg_commit();
          wg_wait_all();
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(empty + stage));           // this stage / weight slot has been read
          if (++stage == NRING) { stage = 0; phase ^= 1; }
          if constexpr (HALO) {
            if (tap == p.taps - 1) {                                         // every tap of this block has read the patch
              if (lane == 0) mbar_arrive(smem_u32(aempty + aslot));
              if (++aslot == A_SLOTS) { aslot = 0; aphase ^= 1; }
            }
          }
          if ((it % p.chunk) == p.chunk - 1 || it == nk - 1) {
            // partial sum complete -> shared-memory slot -> epilogue warps fold it
            mbar_wait(smem_u32(cempty + slot), slot_phase ^ 1, aborted); if (wg_any(aborted)) { aborted = true; goto teardown; }
            const uint32_t sbase = slot_base + (uint32_t)(slot * Cfg::SLOT_BYTES);
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
              const int row = mh * 64 + wq * 16 + (lane >> 2);
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const uint32_t e = sbase + (uint32_t)((row * Cfg::SLOT_PITCH + 8 * j + 2 * (lane & 3)) * 4);
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(e), "f"(acc[mh][4 * j]), "f"(acc[mh][4 * j + 1]) : "memory");
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(e + 8 * Cfg::SLOT_PITCH * 4), "f"(acc[mh][4 * j + 2]),
                             "f"(acc[mh][4 * j + 3]) : "memory");
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(cfull + slot));
            if (++slot == Cfg::SLOTS) { slot = 0; slot_phase ^= 1; }
          }
        }
      }
      }
    }
  } else if (XF && warp == 2 + EPI_WARPS + Cfg::XF_WARPS) {
    // ============================ XF: A-patch loader (own warp: patches must be requested a whole patch ahead) ==========
    // The patch of one 64-channel block arrives as RAW fp32 NHWC values of the producing conv's output: two TMA boxes of
    // 32 channels (128 B rows, 128B swizzle) into the two planes of the slot.  tmA_hi / tmA_lo are the fp32 tensor maps of
    // source 0 / source 1: the k-blocks [0, a_split) come from source 0, the rest from source 1 -- torch.cat([enc, dec])
    // of Fuse_sft_block (codeformer_arch.py:152) never exists in memory.
    if constexpr (XF) {
      int aslot = 0;
      uint32_t aphase = 0;
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        const int mt0 = tile / p.n_tiles;
        const int mt = p.up4 ? (mt0 >> 2) : mt0;           // Upsample: the four output parities read the same low-res patch
        const int per_img = p.tiles_x * p.tiles_y;
        const int n = mt / per_img;
        const int rem = mt - n * per_img;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        const int y0 = ty * p.BH, x0 = tx * p.BW;
        for (int kb = 0; kb < p.kblocks; ++kb) {
          mbar_wait<500>(smem_u32(aempty + aslot), aphase ^ 1, aborted); if (aborted) goto teardown;       // every MMA that read this slot has completed
          if (elect_one()) {
            const uint32_t sa = smem_u32(smem + aslot * Cfg::H_A_SLOT);
            const uint32_t rb = smem_u32(araw + aslot);
            const bool src0 = kb < p.a_split;
            const CUtensorMap* src = src0 ? &tmA_hi : &tmA_lo;
            const int c0 = (src0 ? kb : kb - p.a_split) * 64;
            if (tile == first_tile && kb == 0) TC_STAMP(10);
            mbar_expect_tx(rb, (uint32_t)(2 * p.PW * p.PH * 128));
            tma_load_4d(sa, src, rb, c0, x0 - p.pad, y0 - p.pad, n);
            tma_load_4d(sa + Cfg::X_A_PLANE2, src, rb, c0 + 32, x0 - p.pad, y0 - p.pad, n);
          }
          __syncwarp();
          if (++aslot == A_SLOTS) { aslot = 0; aphase ^= 1; }
        }
      }
    }
  } else if ((XF || WIDE) && warp >= 2 + EPI_WARPS) {        // BN = 128 without XF: the 3 pad warps have no role

    // ============================ XF: operand transform (warps 10..) ============================
    // raw fp32 patch (zero outside the image: TMA out-of-bounds fill) -> y = act(x * scale[n,c] + shift[n,c]) (GroupNorm folded
    // into scale/shift, vqgan_arch.py:14-20,153-160) -> fp16 hi = rn(y), lo = rn(y - hi), written back IN PLACE in the
    // 128B-swizzled K-major layout the MMA descriptors read: plane 0 (raw channels 0..31 of the block) becomes the hi plane
    // (64 channels x fp16), plane 1 (raw channels 32..63) the lo plane.  A patch row (one pixel, 256 B raw) is handled by 8
    // lanes of ONE warp -- lane j owns channels 8j..8j+7 -- and every lane loads before any lane stores (__syncwarp), which
    // is what makes the in-place rewrite safe.  Plane 1 is skewed by 128 B so that, with the swizzle being a function of
    // absolute shared-memory address bits, the 16-byte chunks {0,2,4,6} of plane-0 lanes and plane-1 lanes of the same row
    // fall on different banks: each warp-wide LDS.128 / STS.128 is 4 conflict-free wavefronts.  Pixels outside the image
    // stay exactly zero (the conv pads the NORMALISED tensor).  fence.proxy.async publishes the writes to the tensor core.
    if constexpr (XF) {
      constexpr int XFW = Cfg::XF_WARPS;
      constexpr int RPP = 4 * XFW;                                  // patch rows per pass (8 lanes per row)
      constexpr int XF_PW = 10, XF_PH = 18, XF_ROWS = XF_PW * XF_PH;   // halo patch of an 8 x 16 tile and a 3 x 3 filter
      constexpr int NPASS = (XF_ROWS + RPP - 1) / RPP;
      constexpr int NPASS1 = (128 + RPP - 1) / RPP;                     // 1x1 convs: the patch is the 8 x 16 tile itself
      const int t = (warp - (2 + EPI_WARPS)) * 32 + lane;
      const int j = t & 7, rsub = t >> 3;
      const int pl = j >> 2, c0 = 2 * (j & 3);                      // source plane and first 16-byte chunk of this lane's 8 channels
      const int mode = p.in_scale ? (p.in_act == IN_SILU ? 2 : 1) : 0;   // 2: affine + SiLU, 1: affine, 0: raw split
      const int Hin = GEN ? p.Hin : p.tiles_y * p.BH, Win = GEN ? p.Win : p.tiles_x * p.BW;
      const int Cin = p.kblocks * 64;
      float amax = 0.f;
      int aslot = 0;
      uint32_t aphase = 0;
      for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
        const int mt0 = tile / p.n_tiles;
        const int mt = p.up4 ? (mt0 >> 2) : mt0;
        const int per_img = p.tiles_x * p.tiles_y;
        const int n = mt / per_img;
        const int rem = mt - n * per_img;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        const int y0 = ty * p.BH - p.pad, x0 = tx * p.BW - p.pad;
        const bool border = !K1 && (y0 < 0 || x0 < 0 || y0 + XF_PH > Hin || x0 + XF_PW > Win);
        for (int kb = 0; kb < p.kblocks; ++kb) {
          float sc[8], sh[8];
          if (mode) {
            const int nn = GEN ? min(n, p.N - 1) : n;       // GEN: the tile count is padded to an even number (dummy tile)
            const float* sp = p.in_scale + (int64_t)nn * Cin + kb * 64 + j * 8;
            const float* hp = p.in_shift + (int64_t)nn * Cin + kb * 64 + j * 8;
            const float4 s0 = __ldg(reinterpret_cast<const float4*>(sp)), s1 = __ldg(reinterpret_cast<const float4*>(sp + 4));
            const float4 h0 = __ldg(reinterpret_cast<const float4*>(hp)), h1 = __ldg(reinterpret_cast<const float4*>(hp + 4));
            sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
            sh[0] = h0.x; sh[1] = h0.y; sh[2] = h0.z; sh[3] = h0.w; sh[4] = h1.x; sh[5] = h1.y; sh[6] = h1.z; sh[7] = h1.w;
          } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) { sc[k] = 1.f; sh[k] = 0.f; }
          }
          mbar_wait<250>(smem_u32(araw + aslot), aphase, aborted); if (aborted) goto teardown;
          if (t == 0 && tile == first_tile && kb == 0) TC_STAMP(11);
          if (t == 0 && tile == first_tile + tile_step && kb == 0) TC_STAMP(19);
          const uint32_t base0 = smem_u32(smem + aslot * Cfg::H_A_SLOT);
          const uint32_t src_base = base0 + (pl ? (uint32_t)Cfg::X_A_PLANE2 : 0u);
          const uint32_t lo_base = base0 + (uint32_t)Cfg::X_A_PLANE2;
          if constexpr (K1) {
            if (mode == 2) xf_patch<2, RPP, NPASS1, 8, 128>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
            else if (mode == 1) xf_patch<1, RPP, NPASS1, 8, 128>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
            else xf_patch<0, RPP, NPASS1, 8, 128>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
          } else {
            if (mode == 2) xf_patch<2, RPP, NPASS, XF_PW, XF_ROWS, !P1>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
            else if (mode == 1) xf_patch<1, RPP, NPASS, XF_PW, XF_ROWS, !P1>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
            else xf_patch<0, RPP, NPASS, XF_PW, XF_ROWS, !P1>(src_base, base0, lo_base, c0, j, rsub, sc, sh, border, y0, x0, Hin, Win, amax);
          }
          if constexpr (GEN) {
            if (p.pad_mode && border) {
              // ReflectionPad2d / replicate padding: an out-of-image pixel of the patch equals an in-image pixel of the SAME
              // patch (index -1 -> 1 or 0, index H -> H-2 or H-1), so after every warp has written its rows the outside rows
              // are copied from their source rows (transformed values: the per-channel affine is position independent)
              asm volatile("bar.sync 1, %0;" ::"r"(32 * XFW) : "memory");
#pragma unroll 1
              for (int r = rsub; r < XF_ROWS; r += RPP) {
                const int py = r / XF_PW, px = r - py * XF_PW;
                const int gy = y0 + py, gx = x0 + px;
                if ((unsigned)gy < (unsigned)Hin && (unsigned)gx < (unsigned)Win) continue;
                int sy = gy, sx = gx;
                if (p.pad_mode == 1) {
                  sy = sy < 0 ? -sy : (sy >= Hin ? 2 * Hin - 2 - sy : sy);
                  sx = sx < 0 ? -sx : (sx >= Win ? 2 * Win - 2 - sx : sx);
                }
                sy = min(max(sy, max(y0, 0)), min(Hin, y0 + XF_PH) - 1);      // inside the image AND inside this patch
                sx = min(max(sx, max(x0, 0)), min(Win, x0 + XF_PW) - 1);
                const int rs = (sy - y0) * XF_PW + (sx - x0);
                const uint32_t hs = base0 + (uint32_t)rs * 128u, hd = base0 + (uint32_t)r * 128u;
                const uint32_t ls = lo_base + (uint32_t)rs * 128u, ld = lo_base + (uint32_t)r * 128u;
                const uint4 hv = lds128(hs + ((((uint32_t)j) ^ ((hs >> 7) & 7u)) << 4));
                if constexpr (P1) {
                  sts128(hd + ((((uint32_t)j) ^ ((hd >> 7) & 7u)) << 4), hv);
                } else {
                  const uint4 lv = lds128(ls + ((((uint32_t)j) ^ ((ls >> 7) & 7u)) << 4));
                  sts128(hd + ((((uint32_t)j) ^ ((hd >> 7) & 7u)) << 4), hv);
                  sts128(ld + ((((uint32_t)j) ^ ((ld >> 7) & 7u)) << 4), lv);
                }
              }
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(afull + aslot));
          if (t == 0 && tile == first_tile && kb == 0) TC_STAMP(12);
          if (t == 0 && tile == first_tile + tile_step && kb == 0) TC_STAMP(20);
          if (++aslot == A_SLOTS) { aslot = 0; aphase ^= 1; }
        }
      }
      if (amax > 65504.f) report_overflow();      // an operand left the fp16 range: the host turns the status word into an error
    }
  } else {
    // ============================ epilogue (warps 2..EPI_WARPS+1) ============================
    constexpr int HC = BN * 4 / EPI_WARPS;   // columns owned by this warp: 32 (BN = 64), all 128 (BN = 128)
    const int lg = (warp - 2) & 3;           // row quadrant of this warp: rows [32*lg, 32*lg+32) of the tile
    const int half = (warp - 2) >> 2;        // BN = 64: which half of the tile's columns (logical warps e and e+4 share a quadrant)
    const int row = lg * 32 + lane;          // pixel row of the tile
    const int cbase = half * HC;
    const float wsi = __ldg(p.wscale_inv);
    // tile geometry: 8 x 16 pixels on the halo engine (compile-time), else BW = 2^bw_shift columns (or any BW: division)
    const int BW = HALO ? 8 : p.BW, BH = HALO ? 16 : p.BH;
    const int bw_shift = HALO ? 3 : ((BW & (BW - 1)) == 0 ? __ffs(BW) - 1 : -1);   // log2(BW) when BW is a power of two
    // element strides of one tile row / column in `out` (Upsample tiles write every second pixel of the output).  On the
    // per-tap engine out_pitch is Cout unless the conv writes a channel slice of a wider buffer (then residual, SFT, planes and
    // statistics are off, and the host has moved p.out to the slice's first channel)
    const int64_t SW = (int64_t)(p.up4 ? 2 : 1) * (HALO ? p.Cout : p.out_pitch), SH = SW * p.Wo;
    // every tile lies inside the image unless the image size is not a multiple of the tile (per-tap engine only): then the
    // outside rows / columns of the last tiles are not stored (such convs emit no GroupNorm partials)
    const int ts = p.up4 ? 2 : 1;
    const bool whole_tiles = HALO || (p.tiles_y * BH * ts == p.Ho && p.tiles_x * BW * ts == p.Wo);
    int slot = 0;
    uint32_t slot_phase = 0;
    float omax = 0.f;                        // largest magnitude emitted into fp16 operand planes (range guard)
    TC_T0(t_epi);
    TC_VAR(c_ld);
    TC_VAR(c_st);
    for (int tile = first_tile; tile < total_tiles; tile += tile_step) {
      const int pm = tile / p.n_tiles, nt = tile - pm * p.n_tiles;
      const int mt = pm;
      const int mtl = p.up4 ? (mt >> 2) : mt;
      const int per_img = p.tiles_x * p.tiles_y;
      const int nb = mtl / per_img;
      const int rem = mtl - nb * per_img;
      // multi-head batched GEMM writing [n][token][heads * o_c_head]: head h of image n owns its column slice
      const bool hsplit = !HALO && p.heads > 1 && !p.out_per_head;       // batched-GEMM kernels only (per-tap engine)
      const int n = hsplit ? nb / p.heads : nb;
      const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
      const int h = bw_shift >= 0 ? (row >> bw_shift) : row / BW, w = row - h * BW;
      int oy = ty * BH + h, ox = tx * BW + w;
      if (p.up4) { oy = 2 * oy + ((mt & 3) >> 1); ox = 2 * ox + (mt & 1); }   // this tile writes one output parity
      const int64_t pix = ((int64_t)n * p.Ho + oy) * p.Wo + ox;
      // first pixel of the tile in `out` (elements); the (row, chunk) items of the store loop are hh * SH + ww * SW away
      const int64_t off_tile = (((int64_t)n * p.Ho + (p.up4 ? 2 * ty * BH + ((mt & 3) >> 1) : ty * BH)) * p.Wo +
                                (p.up4 ? 2 * tx * BW + (mt & 1) : tx * BW)) * (HALO ? p.Cout : p.out_pitch);
      const int col0 = nt * BN + cbase + (hsplit ? (nb % p.heads) * p.o_c_head : 0);
      const int64_t off0 = pix * (HALO ? p.Cout : p.out_pitch) + col0;
      // pull this thread's residual / SFT row slices towards L2 now: they are consumed only after the whole K loop
      const bool row_in = whole_tiles || (oy < p.Ho && ox < p.Wo);
      if (!GEN && p.residual && row_in) {
#pragma unroll
        for (int j = 0; j < HC; j += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + off0 + j));
      }
      if (p.sft_dec && row_in) {
#pragma unroll
        for (int j = 0; j < HC; j += 32) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(p.sft_dec + off0 + j));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(p.sft_scale + off0 + j));
        }
      }
      float acc[WIDE ? 1 : HC];
      if constexpr (WIDE) {
        // the MMA warpgroups have stored the finished tile (every partial sum folded) into the slot; the store loop reads it
        TC_T0(t_c);
        mbar_wait<250>(smem_u32(cfull + slot), slot_phase, aborted); if (aborted) goto teardown;
        TC_ADD(4, t_c);
      } else {
#pragma unroll
        for (int j = 0; j < HC; ++j) acc[j] = 0.f;
        for (int it0 = 0; it0 < nk; it0 += p.chunk) {
          mbar_wait<250>(smem_u32(cfull + slot), slot_phase, aborted); if (aborted) goto teardown;
          const uint32_t srow = smem_u32(acc_slot) + (uint32_t)(slot * Cfg::SLOT_BYTES) + (uint32_t)((row * Cfg::SLOT_PITCH + cbase) * 4);
#pragma unroll
          for (int c0 = 0; c0 < HC; c0 += 4) {          // round-to-nearest adds of the partial sum
            const float4 v = lds128f(srow + (uint32_t)(c0 * 4));
            acc[c0] += v.x; acc[c0 + 1] += v.y; acc[c0 + 2] += v.z; acc[c0 + 3] += v.w;
          }
          asm volatile("" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(smem_u32(cempty + slot));
          if (++slot == Cfg::SLOTS) { slot = 0; slot_phase ^= 1; }
        }
      }
      if (warp == 2 && lane == 0 && tile == first_tile) TC_STAMP(7);
      if (warp == 2 && lane == 0 && tile == first_tile + tile_step) TC_STAMP(17);
      // ---- finalize this tile: scale, bias, residual, activation, SFT, store (fp32 NHWC), GroupNorm partials.
      // A thread owns a pixel ROW, so storing straight from registers would touch 32 different 128-byte lines per
      // instruction.  Each warp instead transposes 32x32-float blocks through a private 4 KB XOR-swizzled smem patch (BN = 128:
      // reads the tile slot directly): afterwards lane l holds the 16-byte chunk (l & 7) of row (l >> 3) + 4*it, i.e. 8 lanes
      // cover one full 128-byte line and every global access (residual / SFT loads, the store) is a fully used line.
      const uint32_t stg = smem_u32(stage_buf) + (uint32_t)(warp - 2) * 4096u;     // 32 rows x 8 chunks of 16 B
      const uint32_t stg_w = stg + (uint32_t)lane * 128u;                          // this lane's row (write side)
      const int cch = lane & 7, rsub = lane >> 3;
      if constexpr (GEN) {
        // generalised placement (ParseNet / RRDBNet): ragged tiles (only pixels inside the true image are stored), destination
        // with its own channel pitch / offset (dense-block buffers), optional even-position subsampling (stride 2), and
        //   out = act(conv * 2^-k + bias + residual) * post_scale + residual2
        const int Hs = p.sub ? (p.Ho >> 1) : p.Ho, Ws = p.sub ? (p.Wo >> 1) : p.Wo;
#pragma unroll
        for (int q = 0; q < HC; q += 32) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            sts128f(stg_w + (uint32_t)((j ^ (lane & 7)) << 4), acc[q + 4 * j] * wsi, acc[q + 4 * j + 1] * wsi, acc[q + 4 * j + 2] * wsi,
                    acc[q + 4 * j + 3] * wsi);
          __syncwarp();
          const int colq = col0 + q + cch * 4;
          const bool col_ok = colq < p.cout_valid;
          float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
          if (p.bias) bv = __ldg(reinterpret_cast<const float4*>(p.bias + colq));
          int64_t pixs[8];
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int trow = lg * 32 + it * 4 + rsub;
            const int hh = trow / BW, ww = trow - hh * BW;
            int oy2 = ty * BH + hh, ox2 = tx * BW + ww;
            if (p.up4) { oy2 = 2 * oy2 + ((mt & 3) >> 1); ox2 = 2 * ox2 + (mt & 1); }
            bool ok = col_ok && n < p.N && oy2 < p.Ho && ox2 < p.Wo;
            if (p.sub) { ok = ok && (((oy2 | ox2) & 1) == 0); oy2 >>= 1; ox2 >>= 1; }
            pixs[it] = ok ? ((int64_t)n * Hs + oy2) * Ws + ox2 : (int64_t)-1;
          }
          float4 rres[8];
#pragma unroll
          for (int it = 0; it < 8; ++it)
            rres[it] = (p.residual && pixs[it] >= 0) ? __ldg(reinterpret_cast<const float4*>(p.residual + pixs[it] * p.res_pitch + colq))
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int r = it * 4 + rsub;
            float4 v = lds128f(stg + (uint32_t)(r * 128 + ((cch ^ (r & 7)) << 4)));
            v.x += bv.x + rres[it].x; v.y += bv.y + rres[it].y; v.z += bv.z + rres[it].z; v.w += bv.w + rres[it].w;
            if constexpr (PRELU) {
              v.x = v.x > 0.f ? v.x : p.prelu * v.x; v.y = v.y > 0.f ? v.y : p.prelu * v.y;
              v.z = v.z > 0.f ? v.z : p.prelu * v.z; v.w = v.w > 0.f ? v.w : p.prelu * v.w;
            } else if (p.out_act == OUT_LRELU || p.out_act == OUT_RELU) {      // ReLU = slope 0 (a negative value becomes -0.0)
              const float sl = p.out_act == OUT_LRELU ? 0.2f : 0.f;
              v.x = v.x > 0.f ? v.x : sl * v.x; v.y = v.y > 0.f ? v.y : sl * v.y;
              v.z = v.z > 0.f ? v.z : sl * v.z; v.w = v.w > 0.f ? v.w : sl * v.w;
            } else if (SILU) {
              v.x = tc_silu_out(v.x); v.y = tc_silu_out(v.y); v.z = tc_silu_out(v.z); v.w = tc_silu_out(v.w);
            }
            if (pixs[it] >= 0) {
              if (p.residual2) {
                const float4 r2 = __ldg(reinterpret_cast<const float4*>(p.residual2 + pixs[it] * p.res2_pitch + colq));
                v.x = fmaf(v.x, p.post_scale, r2.x); v.y = fmaf(v.y, p.post_scale, r2.y);
                v.z = fmaf(v.z, p.post_scale, r2.z); v.w = fmaf(v.w, p.post_scale, r2.w);
              }
              *reinterpret_cast<float4*>(p.out + pixs[it] * p.out_pitch + p.out_c0 + colq) = v;
            }
          }
          __syncwarp();
        }
      } else {
      // BN = 128: this warp's 32 rows of the tile slot, 16-byte chunk (lane & 7) of row (lane >> 3) + 4*it
      const uint32_t slot_q = smem_u32(acc_slot) + (uint32_t)(slot * Cfg::SLOT_BYTES) +
                              (uint32_t)(((lg * 32 + rsub) * Cfg::SLOT_PITCH + cbase + cch * 4) * 4);
#pragma unroll
      for (int q = 0; q < HC; q += 32) {
        if constexpr (!WIDE) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            sts128f(stg_w + (uint32_t)((j ^ (lane & 7)) << 4), acc[q + 4 * j] * wsi, acc[q + 4 * j + 1] * wsi, acc[q + 4 * j + 2] * wsi,
                    acc[q + 4 * j + 3] * wsi);
          __syncwarp();
        }
        const int colq = col0 + q + cch * 4;                  // first of this lane's 4 channels
        float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.bias) bv = __ldg(reinterpret_cast<const float4*>(p.bias + colq));
        // global offsets of the (row, chunk) items of this lane, then their residual loads in flight at once: all 8 rows, or two
        // batches of 4 in the register-capped (96-register) transform variants
        constexpr int RB = (XF || WIDE) ? 4 : 8;
        // GroupNorm partials: sums of deviations from the first value of the group this lane sees (k0, k1), so that a large
        // group mean does not cancel against the sum of squares (statistics need whole tiles: every value is inside)
        float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f, k0 = 0.f, k1 = 0.f;
#pragma unroll
        for (int ib = 0; ib < 8; ib += RB) {
        int64_t offs[RB];
        bool inside[RB];
#pragma unroll
        for (int k = 0; k < RB; ++k) {
          const int it = ib + k;
          const int trow = lg * 32 + it * 4 + rsub;
          const int hh = bw_shift >= 0 ? (trow >> bw_shift) : trow / BW, ww = trow - hh * BW;
          offs[k] = off_tile + colq + hh * SH + ww * SW;
          inside[k] = whole_tiles || ((ty * BH + hh) * ts < p.Ho && (tx * BW + ww) * ts < p.Wo);
        }
        TC_T0(t_l);
        float4 rres[RB];
#pragma unroll
        for (int k = 0; k < RB; ++k)
          rres[k] = (p.residual && inside[k]) ? __ldg(reinterpret_cast<const float4*>(p.residual + offs[k])) : make_float4(0.f, 0.f, 0.f, 0.f);
#if CFB_TC_STAMPS
        if (WIDE && p.residual) { tc_arrived(rres[RB - 1].w); TC_SUM(c_ld, t_l); }
#endif
#pragma unroll
        for (int k = 0; k < RB; ++k) {
          const int it = ib + k;
          const int r = it * 4 + rsub;                        // row within this warp's 32-row quadrant
          float4 v;
          if constexpr (WIDE) {      // scaled here as the BN = 64 path scales before its transpose (__fmul_rn: never contracted)
            v = lds128f(slot_q + (uint32_t)((it * 4 * Cfg::SLOT_PITCH + q) * 4));
            v.x = __fmul_rn(v.x, wsi); v.y = __fmul_rn(v.y, wsi); v.z = __fmul_rn(v.z, wsi); v.w = __fmul_rn(v.w, wsi);
          } else {
            v = lds128f(stg + (uint32_t)(r * 128 + ((cch ^ (r & 7)) << 4)));
          }
          const int64_t off = offs[k];
          v.x += bv.x + rres[k].x; v.y += bv.y + rres[k].y; v.z += bv.z + rres[k].z; v.w += bv.w + rres[k].w;
          if constexpr (PRELU) {
            v.x = v.x > 0.f ? v.x : p.prelu * v.x; v.y = v.y > 0.f ? v.y : p.prelu * v.y;
            v.z = v.z > 0.f ? v.z : p.prelu * v.z; v.w = v.w > 0.f ? v.w : p.prelu * v.w;
          } else if (p.out_act == OUT_LRELU) {
            v.x = v.x > 0.f ? v.x : 0.2f * v.x; v.y = v.y > 0.f ? v.y : 0.2f * v.y;
            v.z = v.z > 0.f ? v.z : 0.2f * v.z; v.w = v.w > 0.f ? v.w : 0.2f * v.w;
          } else if (p.out_act == OUT_GELU) {
            v.x = 0.5f * v.x * (1.f + erff(v.x * 0.70710678118654752440f));
            v.y = 0.5f * v.y * (1.f + erff(v.y * 0.70710678118654752440f));
            v.z = 0.5f * v.z * (1.f + erff(v.z * 0.70710678118654752440f));
            v.w = 0.5f * v.w * (1.f + erff(v.w * 0.70710678118654752440f));
          } else if (p.out_act == OUT_RELU) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          } else if (SILU) {
            v.x = tc_silu_out(v.x); v.y = tc_silu_out(v.y); v.z = tc_silu_out(v.z); v.w = tc_silu_out(v.w);
          }
          if (p.sft_dec && inside[k]) {
            TC_T0(t_s);
            const float4 d = __ldg(reinterpret_cast<const float4*>(p.sft_dec + off));
            const float4 sc = __ldg(reinterpret_cast<const float4*>(p.sft_scale + off));
#if CFB_TC_STAMPS
            if (WIDE) { tc_arrived(d.w); tc_arrived(sc.w); TC_SUM(c_ld, t_s); }
#endif
            float sw = p.sft_w;     // per image (a tile never spans two): max(w, 0), so w <= 0 or NaN leaves dec unchanged
            if constexpr (!XF) { if (p.sft_wv) { const float t = __ldg(p.sft_wv + n); sw = t > 0.f ? t : 0.f; } }
            v.x = d.x + sw * (d.x * sc.x + v.x); v.y = d.y + sw * (d.y * sc.y + v.y);
            v.z = d.z + sw * (d.z * sc.z + v.z); v.w = d.w + sw * (d.w * sc.w + v.w);
          }
          if (!inside[k]) v = make_float4(0.f, 0.f, 0.f, 0.f);          // outside the image: no store, no statistics
          TC_T0(t_st);
          // per-tap engine: the zero-padded weight columns from cout_valid on are not stored (a channel slice of a concatenation)
          const bool col_in = HALO || colq < p.cout_valid;
          if (p.out && inside[k] && col_in) *reinterpret_cast<float4*>(p.out + off) = v;      // null: only the operand planes are consumed
          if (p.pl_hi && inside[k]) {
            omax = fmaxf(omax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
            const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
            const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
            uint2 ph, pl;
            ph.x = *reinterpret_cast<const uint32_t*>(&h01); ph.y = *reinterpret_cast<const uint32_t*>(&h23);
            pl.x = *reinterpret_cast<const uint32_t*>(&l01); pl.y = *reinterpret_cast<const uint32_t*>(&l23);
            *reinterpret_cast<uint2*>(p.pl_hi + off) = ph;
            *reinterpret_cast<uint2*>(p.pl_lo + off) = pl;
          }
          TC_SUM(c_st, t_st);
          if constexpr (CPG == 2) {
            if (it == 0) { k0 = v.x; k1 = v.z; }
            const float a = v.x - k0, b = v.y - k0, c = v.z - k1, d = v.w - k1;
            s0 += a + b; q0 += fmaf(a, a, b * b);
            s1 += c + d; q1 += fmaf(c, c, d * d);
          } else if constexpr (CPG >= 4) {
            if (it == 0) k0 = v.x;
            const float a = v.x - k0, b = v.y - k0, c = v.z - k0, d = v.w - k0;
            s0 += (a + b) + (c + d);
            q0 += fmaf(a, a, b * b) + fmaf(c, c, d * d);
          }
        }
        }
        if constexpr (CPG > 0) {
          // GroupNorm partials of the values just stored, as (mean, M2 = sum of squared deviations from the mean) of each
          // slot: this lane's 8 rows x (CPG >= 4 ? 4 : 2) values first, then equal-count merges over the 4 row-lanes (xor 8,
          // 16) and, for groups wider than one chunk, over the chunk-lanes of the group; fixed order => deterministic
          constexpr float NL = CPG == 2 ? 16.f : 32.f;
          gn_lane_moments(s0, q0, k0, NL);
          if constexpr (CPG == 2) gn_lane_moments(s1, q1, k1, NL);
          gn_merge_xor(s0, q0, 8, NL); gn_merge_xor(s0, q0, 16, 2.f * NL);
          if constexpr (CPG == 2) { gn_merge_xor(s1, q1, 8, NL); gn_merge_xor(s1, q1, 16, 2.f * NL); }
          if constexpr (CPG >= 8) gn_merge_xor(s0, q0, 1, 4.f * NL);
          if constexpr (CPG >= 16) gn_merge_xor(s0, q0, 2, 8.f * NL);
          constexpr int CL = (CPG >= 4) ? CPG / 4 : 1;         // chunk-lanes per group
          TC_T0(t_gs);
          if (rsub == 0 && (cch & (CL - 1)) == 0) {
            float* gp = p.gn_part + ((int64_t)mt * 4 + lg) * 64;
            if constexpr (CPG == 2) {
              *reinterpret_cast<float4*>(gp + (colq / 2) * 2) = make_float4(s0, q0, s1, q1);
            } else {
              *reinterpret_cast<float2*>(gp + (colq / CPG) * 2) = make_float2(s0, q0);
            }
          }
          TC_SUM(c_st, t_gs);
        }
        __syncwarp();
      }
      }
      if constexpr (WIDE) {          // every read of the tile slot is done: the MMA warpgroups may store the next tile
        if (lane == 0) mbar_arrive(smem_u32(cempty + slot));
        if (++slot == Cfg::SLOTS) { slot = 0; slot_phase ^= 1; }
        TC_FLUSH(5, c_ld);
        TC_FLUSH(6, c_st);
      }
      if (warp == 2 && lane == 0 && tile == first_tile) TC_STAMP(16);
      if (warp == 2 && lane == 0 && tile == first_tile + tile_step) TC_STAMP(18);
    }
    if (omax > 65504.f) report_overflow();   // a value left the fp16 range of the operand planes: reported, never silent
    TC_ADD(7, t_epi);
    if (warp == 2 && lane == 0) TC_STAMP(13);
  }

teardown:
  if (aborted) {             // error path only: let the bulk copies / MMAs that are still in flight finish before the CTA's
    const long long t0 = clock64();          // shared and tensor memory are handed back
    while (clock64() - t0 < 400000) {}
  }
  __syncthreads();
  if (threadIdx.x == 0) TC_STAMP(8);
}

// ------------------------------------------------------------------------------------------------------
// asynchronous status word: binding of this device's symbols (called once per device by runtime.cu)
// ------------------------------------------------------------------------------------------------------
int tc_bind_status_word(unsigned* host_mapped_dev_ptr, long long wait_limit_cycles) {
  const unsigned zero = 0;
  CFB_CUDA(cudaMemcpyToSymbol(g_status_host, &host_mapped_dev_ptr, sizeof(host_mapped_dev_ptr)));
  CFB_CUDA(cudaMemcpyToSymbol(g_wait_limit, &wait_limit_cycles, sizeof(wait_limit_cycles)));
  CFB_CUDA(cudaMemcpyToSymbol(g_abort, &zero, sizeof(zero)));
  return 0;
}
static std::atomic<int> g_inject_fault{0};
static std::atomic<long long*> g_stamps{nullptr};      // diagnostics: device buffer of >= 32 int64 (cfb_debug_set_stamps)
int tc_set_stamps(long long* dev_ptr) { g_stamps.store(dev_ptr); return 0; }
int tc_inject_fault(int kind) { g_inject_fault.store(kind); return 0; }
int tc_clear_abort() {
  const unsigned zero = 0;
  CFB_CUDA(cudaMemcpyToSymbol(g_abort, &zero, sizeof(zero)));
  return 0;
}

// ------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

static int make_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, int spatial_stride = 1, bool f32 = false) {
  EncodeTiledFn fn = get_encode_fn();
  CFB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
  // traversal stride 2 along W and H turns the box into the stride-2 sampling pattern of Downsample
  cuuint32_t estr[5] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1, 1};
  const CUresult rc = fn(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                         reinterpret_cast<const cuuint64_t*>(dims), reinterpret_cast<const cuuint64_t*>(strides_bytes),
                         reinterpret_cast<const cuuint32_t*>(box), estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  CFB_REQUIRE(rc == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)rc) + ")");
  return 0;
}

// tile width: the power of two >= W up to 128 (tiles hold 128 pixels; the last tile row / column of an image whose size is not
// a multiple of the tile is ragged -- its outside pixels read TMA zero fill and are never stored)
static inline int tile_bw(int W) {
  int bw = 1;
  while (bw < W && bw < 128) bw <<= 1;
  return bw;
}

// k-blocks (64 K-elements) per partial sum; env CFB_TC_CHUNK overrides for experiments (1..64)
static int tc_chunk_kblocks() {
  static int v = [] {
    const char* e = getenv("CFB_TC_CHUNK");
    int c = e ? atoi(e) : 8;
    return c < 1 ? 1 : (c > 4096 ? 4096 : c);
  }();
  return v;
}

// halo engine (one patch fetch per 64-channel block, taps via shifted descriptors): 3x3 stride-1 convs and the 2x2 parity
// convs of Upsample, on 8x16-pixel tiles; it halves the L2 -> SM operand traffic of the per-tap engine and is the only engine
// with the fused operand transform and the generalised (ParseNet / RRDBNet) addressing.  CFB_TC_HALO=0 switches it off.
static bool halo_enabled() {
  static bool v = [] { const char* e = getenv("CFB_TC_HALO"); return !(e && atoi(e) == 0); }();
  return v;
}
struct TcGeom { int BW, BH; bool halo; };
static TcGeom tc_geometry(const ConvArgs& a) {
  TcGeom g;
  const int Wt = a.mode == CONV_UP ? a.W : a.Wo, Ht = a.mode == CONV_UP ? a.H : a.Ho;   // grid the tiles live on
  g.halo = halo_enabled() && a.kh == 0 && (a.ksize == 3 || (a.ksize == 1 && a.halo1x1 && a.mode == CONV_SAME)) &&
           (a.mode == CONV_SAME || a.mode == CONV_UP) &&
           ((Wt % 8 == 0 && Ht % 16 == 0) || a.gen);      // gen: ragged tiles, stores are bounds-checked
  if (g.halo) { g.BW = 8; g.BH = 16; }
  else { g.BW = tile_bw(a.mode == CONV_UP ? a.W : a.Wo); g.BH = 128 / g.BW; }   // Upsample: tiles live on the low-res grid
  return g;
}

int tc_tiles_per_image(const ConvArgs& a) {
  const TcGeom g = tc_geometry(a);
  if (a.mode == CONV_UP) return 4 * ((a.W + g.BW - 1) / g.BW) * ((a.H + g.BH - 1) / g.BH);
  return ((a.Wo + g.BW - 1) / g.BW) * ((a.Ho + g.BH - 1) / g.BH);
}

// the window of a conv: the explicit kh x kw form (ConvArgs::kh > 0) or the square ksize forms
struct TcWin { int kh, kw, ph, pw, stride; };
static TcWin tc_window(const ConvArgs& a) {
  const int s = a.mode == CONV_DOWN ? 2 : 1;
  if (a.kh > 0) return {a.kh, a.kw, a.pad_h, a.pad_w, s};
  const int p = a.mode == CONV_DOWN ? a.down_pad : a.ksize / 2;
  return {a.ksize, a.ksize, p, p, s};
}

bool tc_supported(const ConvArgs& a) {
  if (a.Cin % 64 != 0 || a.Cout % 64 != 0) return false;
  if (a.kh > 0) {
    // explicit window: per-tap engine, raw input, stride 1 or 2, Ho = (H + 2 pad_h - kh) / stride + 1 (likewise Wo)
    const int s = a.mode == CONV_DOWN ? 2 : 1;
    if (a.gen || a.xform || a.mode == CONV_UP || a.kh > 7 || a.kw < 1 || a.kw > 7) return false;
    if (a.pad_h < 0 || a.pad_w < 0 || a.pad_h >= a.kh || a.pad_w >= a.kw) return false;
    if (a.H + 2 * a.pad_h < a.kh || a.W + 2 * a.pad_w < a.kw) return false;
    if (a.Ho != (a.H + 2 * a.pad_h - a.kh) / s + 1 || a.Wo != (a.W + 2 * a.pad_w - a.kw) / s + 1) return false;
  } else {
    if (!(a.ksize == 1 || a.ksize == 3)) return false;
    if (a.mode == CONV_DOWN && a.ksize != 3 && !(a.ksize == 1 && a.down_pad == 0 && a.Ho == (a.H + 1) / 2)) return false;
    if (a.mode == CONV_DOWN && a.down_pad != 0 && !(a.down_pad == 1 && a.ksize == 3)) return false;
  }
  if (a.Wo < 1 || a.Ho < 1) return false;
  const TcGeom g = tc_geometry(a);
  if (a.gen) return g.halo && a.ksize == 3;
  const int BW = g.BW, BH = g.BH;
  if (a.mode == CONV_UP && a.ksize != 3) return false;
  if (128 % BW != 0) return false;
  if ((int64_t)a.N * (a.Ho / BH + 1) * (a.Wo / BW + 1) * (a.Cout / 64) > 0x7fffffffLL) return false;
  return true;
}

bool tc_tiles_exact(const ConvArgs& a) {
  if (!tc_supported(a)) return false;
  const TcGeom g = tc_geometry(a);
  const int Wt = a.mode == CONV_UP ? a.W : a.Wo, Ht = a.mode == CONV_UP ? a.H : a.Ho;   // grid the tiles live on
  return Wt % g.BW == 0 && Ht % g.BH == 0;
}

// fused operand transform: available for 3x3 stride-1 convs (and GroupNorm-affine 1x1 convs) on the halo engine.  It reads
// the fp32 activation itself (no planes written by the producer, no prep pass), so it is used wherever the engine exists.
// CFB_TC_XFORM=0 disables it, =3 keeps it to the 128-wide layers at >= 64x64.
bool tc_can_xform(const ConvArgs& a) {
  static const int mode = [] { const char* e = getenv("CFB_TC_XFORM"); return e ? atoi(e) : 1; }();
  if (a.gen) return tc_supported(a);      // generalised variant: CONV_UP included
  if (mode == 0 || !tc_supported(a) || a.mode != CONV_SAME || !(a.ksize == 3 || (a.ksize == 1 && a.halo1x1 && a.Cout % 128 == 0))) return false;
  if (mode == 3 && !(a.Cout % 128 == 0 && a.Cin >= 128 && (int64_t)a.Ho * a.Wo >= 4096)) return false;
  return tc_geometry(a).halo;
}

size_t tc_scratch_bytes(const ConvArgs& a) {
  if (!tc_supported(a)) return 0;
  const bool same = a.mode == CONV_SAME && a.kh == 0;
  const int Hp = same ? a.Ho : a.H, Wp = same ? a.Wo : a.W;   // operand plane = input resolution
  const size_t plane = ((size_t)a.N * Hp * Wp * a.Cin * 2 + 1023) / 1024 * 1024;
  return 2 * plane;
}

struct TcMaps { CUtensorMap a_hi, a_lo, b_hi, b_lo; };

template <int BN, int CPG, bool HALO, bool XF = false, bool GEN = false, bool K1 = false, bool CM = false, bool SILU = false,
          bool P1 = false, bool PRELU = false>
static int launch_tc2(const TcMaps& m, const TcParams& p, int sm_count, cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  constexpr int SMEM = XF ? Cfg::X_SMEM_BYTES : (HALO ? Cfg::H_SMEM_BYTES : Cfg::SMEM_BYTES);
  constexpr int THREADS = XF ? Cfg::XF_THREADS : Cfg::THREADS;
  static_assert(SMEM <= 232448, "shared memory budget");
  // cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE property of the function: remember it per device
  // (one process may drive several GPUs from several threads)
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(attr_done.load(std::memory_order_acquire) & bit)) {
    CFB_CUDA(cudaFuncSetAttribute(conv_tc_kernel<BN, CPG, HALO, XF, GEN, K1, CM, SILU, P1, PRELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_done.fetch_or(bit, std::memory_order_release);
  }
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count ? total : sm_count;
  CFB_LAUNCH_PDL((conv_tc_kernel<BN, CPG, HALO, XF, GEN, K1, CM, SILU, P1, PRELU>), dim3((unsigned)grid), dim3(THREADS), (size_t)SMEM, st,
                 m.a_hi, m.a_lo, m.b_hi, m.b_lo, p);
  return 0;
}
// Single-pass fp16 (ConvArgs::single_pass) exists only for the convs that run in fp16 mode: the generalised convs of RRDBNet,
// and the generator / Fuse_sft_block convs of CodeFormer -- 128-wide halo tiles (fused transform with GroupNorm partials, or
// raw planes), channel-major halo tiles (fused transform with partials, or raw planes) and the per-tap 1x1 conv on raw planes.
// Anything else is an error: a conv never runs split when single pass was asked for.
template <int CPG>
static int launch_tc_p1(const TcMaps& m, const TcParams& p, int sm_count, cudaStream_t st, bool gen, int tile) {
  constexpr bool T = true, F = false;
  const bool halo3 = p.PW == 10 && p.PH == 18;
  if (p.out_act != OUT_SILU) {
    if (gen) {
      if constexpr (CPG == 0) {
        if (p.xform && halo3) return launch_tc2<64, 0, T, T, T, F, F, F, T>(m, p, sm_count, st);
      }
    } else if (tile == 128 && halo3) {
      if constexpr (CPG == 4 || CPG == 8 || CPG == 16) {
        if (p.xform) return launch_tc2<128, CPG, T, T, F, F, F, F, T>(m, p, sm_count, st);
      }
      if constexpr (CPG != 2) {
        if (!p.xform) return launch_tc2<128, CPG, T, F, F, F, F, F, T>(m, p, sm_count, st);
      }
    } else if (tile == TC_TILE_CM && halo3) {
      if constexpr (CPG == 2) {
        if (p.xform) return launch_tc2<64, 2, T, T, F, F, T, F, T>(m, p, sm_count, st);
      }
      if constexpr (CPG <= 2) {
        if (!p.xform) return launch_tc2<64, CPG, T, F, F, F, T, F, T>(m, p, sm_count, st);
      }
    } else if (tile == TC_TILE_N && !p.xform && p.PW == 0 && p.taps == 1) {
      if constexpr (CPG == 0) return launch_tc2<64, 0, F, F, F, F, F, F, T>(m, p, sm_count, st);
    }
  }
  CFB_REQUIRE(false, "conv_tc: single-pass fp16 is built for the generalised engine, the 128-wide and channel-major halo tiles "
                     "and the per-tap 1x1 conv, without the SiLU epilogue");
  return 1;
}

template <int CPG>
static int launch_tc(const TcMaps& m, const TcParams& p, int sm_count, cudaStream_t st, bool gen = false, int tile = TC_TILE_N,
                     bool single_pass = false) {
  // the SiLU epilogue (YOLOv5) is built into two variants only, so the others keep their register budgets
  CFB_REQUIRE(p.out_act != OUT_SILU || (CPG == 0 && (gen || (!p.xform && p.PW == 0))),
              "conv_tc: the SiLU epilogue is built for the per-tap and generalised engines without statistics");
  if (p.out_act == OUT_PRELU) {     // ResNetArcFace: split precision, no statistics, no SFT / planes (conv_tc checks those)
    CFB_REQUIRE(!single_pass && CPG == 0 && (gen || (!p.xform && p.PW == 0)),
                "conv_tc: the PReLU epilogue is built for the split per-tap and generalised engines without statistics");
    if constexpr (CPG == 0) {
      if (gen) return launch_tc2<64, 0, true, true, true, false, false, false, false, true>(m, p, sm_count, st);
      return launch_tc2<64, 0, false, false, false, false, false, false, false, true>(m, p, sm_count, st);
    }
  }
  if (single_pass) return launch_tc_p1<CPG>(m, p, sm_count, st, gen, tile);
  if (tile == TC_TILE_CM) {    // channel-major 128 x 64 tiles: conv_tc() only asks for them where tc_tile_kind() says so
    if constexpr (CPG <= 2) {
      CFB_REQUIRE(p.PW == 10 && p.PH == 18, "conv_tc: channel-major tiles need the 3x3 / Upsample halo engine");
      if (p.xform) return launch_tc2<64, CPG, true, true, false, false, true>(m, p, sm_count, st);
      return launch_tc2<64, CPG, true, false, false, false, true>(m, p, sm_count, st);
    } else {
      CFB_REQUIRE(false, "conv_tc: channel-major tiles need Cout % 128 == 64");
    }
  }
  if (tile == 128) {     // 128-wide n-tiles: conv_tc() only asks for them where tc_tile_kind() says so
    if constexpr (CPG != 2) {
      CFB_REQUIRE(p.PW == 10 && p.PH == 18, "conv_tc: 128-wide tiles need the 3x3 / Upsample halo engine");
      if (p.xform) return launch_tc2<128, CPG, true, true>(m, p, sm_count, st);
      return launch_tc2<128, CPG, true>(m, p, sm_count, st);
    } else {
      CFB_REQUIRE(false, "conv_tc: 128-wide tiles need Cout % 128 == 0");
    }
  }
  if constexpr (CPG == 0) {
    if (gen) {
      CFB_REQUIRE(p.xform && p.PW == 10 && p.PH == 18, "conv_tc: generalised variant needs the halo + transform engine");
      if (p.out_act == OUT_SILU) return launch_tc2<64, 0, true, true, true, false, false, true>(m, p, sm_count, st);
      return launch_tc2<64, 0, true, true, true>(m, p, sm_count, st);
    }
    if (p.out_act == OUT_SILU) return launch_tc2<64, 0, false, false, false, false, false, true>(m, p, sm_count, st);
  }
  if (p.xform) {         // fused operand transform: conv_tc() only asks for it when tc_can_xform() holds
    CFB_REQUIRE((p.PW == 10 && p.PH == 18) || (p.PW == 8 && p.PH == 16 && p.taps == 1),
                "conv_tc: fused operand transform needs the halo engine");
    if (p.taps == 1) {      // 1x1 conv with a GroupNorm-affine input (AttnBlock q,k,v): patch = tile
      if constexpr (CPG == 0) return launch_tc2<64, 0, true, true, false, true>(m, p, sm_count, st);
      else { CFB_REQUIRE(false, "conv_tc: the 1x1 fused transform is built without statistics"); }
    }
    return launch_tc2<64, CPG, true, true>(m, p, sm_count, st);
  }
  if (p.PW > 0) return launch_tc2<64, CPG, true>(m, p, sm_count, st);
  return launch_tc2<64, CPG, false>(m, p, sm_count, st);
}

// Tile of the 3x3 and Upsample convs of the halo engine (not GEN): 128-output-channel tiles (two MMA warpgroups, see TcCfg)
// when Cout % 128 == 0, channel-major 128 x 64 tiles (TC_TILE_CM, see conv_tc_kernel) otherwise; every other conv runs on
// pixel-major 128 x 64 tiles.  CFB_TC_BN=64 keeps every conv on the pixel-major 128 x 64 tiles (same results bit for bit:
// A/B comparisons in one build).
static int tc_tile_kind(const ConvArgs& a, const TcGeom& g) {
  static const bool on = [] { const char* e = getenv("CFB_TC_BN"); return !(e && atoi(e) == 64); }();
  if (!(on && g.halo && !a.gen && a.ksize == 3 && (a.mode == CONV_SAME || a.mode == CONV_UP))) return TC_TILE_N;
  return a.Cout % 128 == 0 ? 128 : TC_TILE_CM;
}

int tc_tile_n(const ConvArgs& a) { return tc_tile_kind(a, tc_geometry(a)); }

// GroupNorm partials can be emitted for Cout in {64, 128, 256, 512} on whole tiles (2 .. 16 channels per group inside a 64-wide n-tile)
bool tc_can_emit_stats(const ConvArgs& a) {
  // every slot must hold 32 pixels of the image: (mean, M2) slots cannot skip the outside rows of a ragged tile
  if (!tc_tiles_exact(a)) return false;
  if (a.Cout % 128 == 0) return a.Cout == 128 || a.Cout == 256 || a.Cout == 512;
  return a.Cout == 64;
}

int conv_tc(const ConvArgs& a, void* scratch, int sm_count, cudaStream_t st) {
  CFB_REQUIRE(tc_supported(a), "conv_tc: unsupported shape");
  CFB_REQUIRE(a.wgt_hi && a.wgt_lo && a.wscale_inv, "conv_tc: split weights missing");
  const int64_t M = (int64_t)a.N * a.Ho * a.Wo;
  if (M == 0) return 0;
  // ---- operand planes (fp16 hi/lo NHWC; at the output resolution, or the input resolution for Downsample / explicit windows)
  const bool same = a.mode == CONV_SAME && a.kh == 0;
  const int Hp = same ? a.Ho : a.H, Wp = same ? a.Wo : a.W;
  const int64_t Mp = (int64_t)a.N * Hp * Wp;
  const size_t plane = ((size_t)Mp * a.Cin * 2 + 1023) / 1024 * 1024;
  __half* hi = (__half*)scratch;
  __half* lo = (__half*)((char*)scratch + plane);
  if (!a.skip_prep && a.kh > 0 && (a.Cin / 8 > 256 || 256 % (a.Cin / 8) != 0)) {
    CFB_REQUIRE(!a.in_scale && a.in_act == IN_NONE, "conv_tc: an input affine needs Cin = 64 * 2^k (<= 2048)");
    const int64_t items = Mp * (a.Cin / 8);
    tc_prep_raw_kernel<<<(unsigned)((items + 255) / 256), 256, 0, st>>>(a.in, items, hi, lo);
    CFB_LAUNCH_CHECK();
  } else if (!a.skip_prep) {
    const int C8 = a.Cin / 8;
    CFB_REQUIRE(C8 <= 256 && 256 % C8 == 0, "conv_tc: Cin must be 64 * 2^k (<= 2048)");
    const int64_t img_px = (int64_t)Hp * Wp;
    // pixels per thread: up to 32 (amortises the per-block affine loads) but never so many that the grid drops
    // below ~16 blocks per SM -- the small 16x16 / 32x32 layers are latency-bound otherwise
    const int pstep = 256 / C8;
    int iters = 32;
    while (iters > 1 && Mp / ((int64_t)pstep * iters) < 148 * 16) iters >>= 1;
    int64_t PB = (int64_t)pstep * iters;
    while (PB > 1 && img_px % PB != 0) PB >>= 1;
    CFB_REQUIRE(PB >= 1 && img_px % PB == 0 && Mp % PB == 0, "conv_tc: image size not supported by the operand prep kernel");
    tc_prep_kernel<<<(unsigned)(Mp / PB), 256, 0, st>>>(a.in, a.in_scale, a.in_shift, a.in_act, 0, a.N, a.H,
                                                        a.W, a.Cin, (int)PB, hi, lo);
    CFB_LAUNCH_CHECK();
  }
  // ---- tensor maps
  const TcGeom geo = tc_geometry(a);
  const int BW = geo.BW, BH = geo.BH;
  const int PW = geo.halo ? BW + a.ksize - 1 : 0, PH = geo.halo ? BH + a.ksize - 1 : 0;
  const int tile = tc_tile_kind(a, geo);
  const int BN = tile == 128 ? 128 : TC_TILE_N;
  TcMaps mp;
  CUtensorMap &mA_hi = mp.a_hi, &mA_lo = mp.a_lo, &mB_hi = mp.b_hi, &mB_lo = mp.b_lo;
  if (a.xform) {
    // fused operand transform: the A operand is read straight from the fp32 NHWC activation(s); boxes of 32 channels
    // (128 B rows) x the halo patch.  Source 1 is the second half of a channel concatenation (or source 0 again).
    CFB_REQUIRE(a.in != nullptr && geo.halo, "conv_tc: fused operand transform needs the fp32 input and the halo engine");
    // gen: `in` points into a wider NHWC buffer of in_pitch channels; the 64-aligned window [0, Cin) is read (channels beyond
    // the buffer are zero-filled by the TMA unit, channels beyond the real Cin meet zero weights)
    const int C0 = a.in2 ? a.Cin1 : (a.gen && a.in_pitch ? a.in_pitch : a.Cin), C1 = a.in2 ? a.Cin - a.Cin1 : C0;
    CFB_REQUIRE(!(a.gen && a.in2), "conv_tc: the generalised variant reads one source");
    CFB_REQUIRE(a.gen || (C0 % 64 == 0 && C1 % 64 == 0 && C0 > 0 && C1 > 0), "conv_tc: concatenated sources must be multiples of 64 channels");
    CFB_REQUIRE(C0 % 4 == 0 && C0 > 0, "conv_tc: source channel pitch must be a multiple of 4");
    const uint32_t box[4] = {32, (uint32_t)PW, (uint32_t)PH, 1};
    {
      const uint64_t dims[4] = {(uint64_t)C0, (uint64_t)Wp, (uint64_t)Hp, (uint64_t)a.N};
      const uint64_t str[3] = {(uint64_t)C0 * 4, (uint64_t)Wp * C0 * 4, (uint64_t)Hp * Wp * C0 * 4};
      CFB_CHECK(make_map(&mA_hi, a.in, 4, dims, str, box, 1, true));
    }
    {
      const uint64_t dims[4] = {(uint64_t)C1, (uint64_t)Wp, (uint64_t)Hp, (uint64_t)a.N};
      const uint64_t str[3] = {(uint64_t)C1 * 4, (uint64_t)Wp * C1 * 4, (uint64_t)Hp * Wp * C1 * 4};
      CFB_CHECK(make_map(&mA_lo, a.in2 ? a.in2 : a.in, 4, dims, str, box, 1, true));
    }
  } else {
    const int sp = a.mode == CONV_DOWN ? 2 : 1;
    const uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)Wp, (uint64_t)Hp, (uint64_t)a.N};
    const uint64_t str[3] = {(uint64_t)a.Cin * 2, (uint64_t)Wp * a.Cin * 2, (uint64_t)Hp * Wp * a.Cin * 2};
    // per-tap engine: ceil(box/stride) = BW x BH pixels land; halo engine: the whole (BW+k-1) x (BH+k-1) patch
    const uint32_t box[4] = {64, (uint32_t)(geo.halo ? PW : BW * sp), (uint32_t)(geo.halo ? PH : BH * sp), 1};
    CFB_CHECK(make_map(&mA_hi, hi, 4, dims, str, box, sp));
    CFB_CHECK(make_map(&mA_lo, lo, 4, dims, str, box, sp));
  }
  const TcWin win = tc_window(a);
  {
    const int taps = a.mode == CONV_UP ? 16 : win.kh * win.kw;
    const uint64_t dims[3] = {(uint64_t)a.Cin, (uint64_t)a.Cout, (uint64_t)taps};
    const uint64_t str[2] = {(uint64_t)a.Cin * 2, (uint64_t)a.Cout * a.Cin * 2};
    const uint32_t box[3] = {64, (uint32_t)BN, 1};
    CFB_CHECK(make_map(&mB_hi, a.wgt_hi, 3, dims, str, box));
    CFB_CHECK(make_map(&mB_lo, a.wgt_lo, 3, dims, str, box));
  }
  TcParams p;
  p.N = a.N; p.Ho = a.Ho; p.Wo = a.Wo; p.Cout = a.Cout;
  p.taps = win.kh * win.kw; p.kw = win.kw; p.pad = win.ph; p.pad_w = win.pw; p.stride = win.stride;
  p.up4 = a.mode == CONV_UP ? 1 : 0;
  p.a_c0 = 0; p.b_c0 = 0; p.b_batched = 0;
  p.heads = 1; p.a_c_head = 0; p.b_c_head = 0; p.a_img_per_head = 0; p.b_r_head = 0; p.out_per_head = 1; p.o_c_head = 0;
  if (p.up4) { p.taps = 4; p.pad = 1; p.pad_w = 1; }
  p.chunk = tc_chunk_kblocks();
  p.PW = PW; p.PH = PH;
  p.BW = BW; p.BH = BH;
  p.tiles_x = ((p.up4 ? a.W : a.Wo) + BW - 1) / BW; p.tiles_y = ((p.up4 ? a.H : a.Ho) + BH - 1) / BH;   // exact unless gen (ragged)
  {
    int64_t lowres_tiles = (int64_t)a.N * p.tiles_x * p.tiles_y;
    p.m_tiles = (int)(lowres_tiles * (p.up4 ? 4 : 1));
  }
  p.n_tiles = a.Cout / BN; p.kblocks = a.Cin / 64;
  p.Hin = Hp; p.Win = Wp; p.pad_mode = a.pad_mode; p.sub = a.subsample ? 1 : 0;
  p.out_pitch = a.out_pitch ? a.out_pitch : a.Cout; p.out_c0 = a.out_c0; p.cout_valid = a.cout_valid ? a.cout_valid : a.Cout;
  p.res_pitch = a.res_pitch ? a.res_pitch : p.out_pitch; p.residual2 = a.residual2;
  p.res2_pitch = a.res2_pitch ? a.res2_pitch : p.out_pitch; p.post_scale = a.post_scale;
  if (a.gen) {
    CFB_REQUIRE(a.xform && !a.gn_part && !a.out_planes && !a.sft_dec, "conv_tc: generalised variant = fused transform, fp32 output only");
    CFB_REQUIRE(p.out_pitch % 4 == 0 && p.out_c0 % 4 == 0 && p.cout_valid % 4 == 0 && p.res_pitch % 4 == 0 && p.res2_pitch % 4 == 0,
                "conv_tc: channel pitches / offsets must be multiples of 4");
    CFB_REQUIRE(!a.subsample || (a.mode == CONV_SAME && a.Ho % 2 == 0 && a.Wo % 2 == 0), "conv_tc: subsampling needs even sizes");
    CFB_REQUIRE(a.out_act == OUT_NONE || a.out_act == OUT_LRELU || a.out_act == OUT_RELU || a.out_act == OUT_SILU ||
                    a.out_act == OUT_PRELU,
                "conv_tc: generalised variant has bias / residual / LeakyReLU / ReLU / SiLU / PReLU epilogues");
  } else if (p.out_pitch != a.Cout || p.out_c0 != 0 || a.cout_valid != 0) {
    // per-tap engine writing a channel slice: the tile offsets use the destination pitch, which only the plain store follows;
    // cout_valid < Cout leaves the destination channels after the slice's real ones untouched
    CFB_REQUIRE(!geo.halo && p.out_pitch % 4 == 0 && p.out_c0 % 4 == 0 && p.cout_valid % 4 == 0 && p.cout_valid <= a.Cout &&
                    p.out_c0 + p.cout_valid <= p.out_pitch,
                "conv_tc: a destination slice needs the per-tap engine, 4-aligned and inside the pitch");
    CFB_REQUIRE(!a.residual && !a.sft_dec && !a.out_planes && !a.gn_part && !a.residual2,
                "conv_tc: a destination slice of the per-tap engine takes bias and activation only");
  }
  if (p.taps * p.kblocks <= 12) p.chunk = p.taps * p.kblocks;   // short K (Cin = 64): one partial sum, no 8+1 split
  p.in_scale = nullptr; p.in_shift = nullptr; p.in_act = IN_NONE; p.xform = a.xform ? 1 : 0;
  p.fault = g_inject_fault.exchange(0);
#if CFB_TC_STAMPS
  p.dbg = g_stamps.load();
#endif
  p.a_split = a.in2 ? a.Cin1 / 64 : a.Cin / 64;
  if (a.xform) {
    CFB_REQUIRE(a.skip_prep && tc_can_xform(a), "conv_tc: fused operand transform not available for this conv");
    CFB_REQUIRE((a.in_scale != nullptr) == (a.in_shift != nullptr) && (a.in_scale || a.in_act == IN_NONE),
                "conv_tc: fused operand transform takes scale and shift together");
    p.in_scale = a.in_scale; p.in_shift = a.in_shift; p.in_act = a.in_act;
  } else {
    CFB_REQUIRE(a.in2 == nullptr, "conv_tc: a two-source input needs the fused operand transform");
  }
  p.bias = a.bias; p.residual = a.residual; p.out_act = a.out_act;
  // per-image SFT weights are read by the raw-input kernels only (the Fuse_sft_block's shift.2 conv reads shift.0's planes): the
  // fused-transform variants keep their register budgets
  CFB_REQUIRE(!a.sft_wv || (a.sft_dec && !a.xform), "conv_tc: per-image SFT weights need the SFT epilogue of a raw-input conv");
  p.sft_dec = a.sft_dec; p.sft_scale = a.sft_scale; p.sft_w = a.sft_w; p.sft_wv = a.sft_wv; p.wscale_inv = a.wscale_inv;
  if (a.out_act == OUT_PRELU) {
    CFB_REQUIRE(!a.sft_dec && !a.gn_part && !a.out_planes && !a.residual2 && (a.gen || !geo.halo),
                "conv_tc: the PReLU epilogue takes bias and residual only, on the generalised or the per-tap engine");
    p.prelu = a.prelu_slope;
  }
  p.out = a.gen || !a.out ? a.out : a.out + a.out_c0;      // per-tap engine: the slice offset is folded into the base pointer
  p.gn_part = a.gn_part; p.gn_cpg = a.Cout / 32;
  p.pl_hi = (__half*)a.out_planes;
  p.pl_lo = a.out_planes ? (__half*)((char*)a.out_planes + (((size_t)a.N * a.Ho * a.Wo * a.Cout * 2 + 1023) / 1024 * 1024)) : nullptr;
  const int cpg = a.gn_part ? a.Cout / 32 : 0;
  CFB_REQUIRE(!a.gn_part || tc_can_emit_stats(a), "conv_tc: GroupNorm partials are not available for this Cout");
  if (a.gen) return launch_tc<0>(mp, p, sm_count, st, true, TC_TILE_N, a.single_pass);
  switch (cpg) {
    case 0: return launch_tc<0>(mp, p, sm_count, st, false, tile, a.single_pass);
    case 2: return launch_tc<2>(mp, p, sm_count, st, false, tile, a.single_pass);
    case 4: return launch_tc<4>(mp, p, sm_count, st, false, tile, a.single_pass);
    case 8: return launch_tc<8>(mp, p, sm_count, st, false, tile, a.single_pass);
    case 16: return launch_tc<16>(mp, p, sm_count, st, false, tile, a.single_pass);
  }
  CFB_REQUIRE(false, "conv_tc: no kernel variant for this configuration");
  return 1;
}


// ------------------------------------------------------------------------------------------------------
// Batched GEMM on the same engine (attention cores): per image n
//     out[n][t][j] = scale * sum_k A[n][t][a_c0 + k] * B[n][j][b_c0 + k],   t in 0..255 (16x16 tokens), j in 0..Cout-1
// A and B are fp16 hi/lo operand planes (token-major, channel pitch a_pitch / b_pitch); B is addressed per image
// through the third TMA coordinate.  Used for  scores = q k^T * C^-1/2  and  out = P v  of AttnBlock
// (/root/reference/basicsr/archs/vqgan_arch.py:209-222).
// ------------------------------------------------------------------------------------------------------
int bmm_tc(const BmmArgs& g, int sm_count, cudaStream_t st) {
  constexpr int BN = TC_TILE_N;
  CFB_REQUIRE(g.K % 64 == 0 && g.Cout % 64 == 0 && g.N >= 0 && g.heads >= 1, "bmm_tc: K and Cout must be multiples of 64");
  CFB_REQUIRE(g.a_c0 % 64 == 0 && g.b_c0 % 64 == 0 && g.a_pitch % 8 == 0 && g.b_pitch % 8 == 0 && g.a_c_head % 64 == 0 &&
                  g.b_c_head % 64 == 0 && g.b_r_head % BN == 0 && g.o_c_head % 4 == 0,
              "bmm_tc: unaligned operand slice");
  if (g.N == 0) return 0;
  const int a_imgs = g.a_img_per_head ? g.N * g.heads : g.N;
  const size_t a_plane = ((size_t)a_imgs * 256 * g.a_pitch * 2 + 1023) / 1024 * 1024;
  const size_t b_plane = ((size_t)g.N * g.b_rows * g.b_pitch * 2 + 1023) / 1024 * 1024;
  TcMaps mp;
  CUtensorMap &mA_hi = mp.a_hi, &mA_lo = mp.a_lo, &mB_hi = mp.b_hi, &mB_lo = mp.b_lo;
  {
    const uint64_t dims[4] = {(uint64_t)g.a_pitch, 16, 16, (uint64_t)a_imgs};
    const uint64_t str[3] = {(uint64_t)g.a_pitch * 2, (uint64_t)16 * g.a_pitch * 2, (uint64_t)256 * g.a_pitch * 2};
    const uint32_t box[4] = {64, 16, 8, 1};
    CFB_CHECK(make_map(&mA_hi, g.a_planes, 4, dims, str, box));
    CFB_CHECK(make_map(&mA_lo, (const char*)g.a_planes + a_plane, 4, dims, str, box));
  }
  {
    const uint64_t dims[3] = {(uint64_t)g.b_pitch, (uint64_t)g.b_rows, (uint64_t)g.N};
    const uint64_t str[2] = {(uint64_t)g.b_pitch * 2, (uint64_t)g.b_rows * g.b_pitch * 2};
    const uint32_t box[3] = {64, (uint32_t)BN, 1};
    CFB_CHECK(make_map(&mB_hi, g.b_planes, 3, dims, str, box));
    CFB_CHECK(make_map(&mB_lo, (const char*)g.b_planes + b_plane, 3, dims, str, box));
  }
  const int out_pitch = g.out_per_head ? g.Cout : g.heads * g.o_c_head;      // channels per token row of `out`
  const int out_imgs = g.out_per_head ? g.N * g.heads : g.N;
  CFB_REQUIRE(g.heads == 1 || g.out_per_head || g.o_c_head == g.Cout, "bmm_tc: a head's column slice must equal its Cout");
  TcParams p;
  p.N = g.N * g.heads; p.Ho = 16; p.Wo = 16; p.Cout = out_pitch;
  p.taps = 1; p.kw = 1; p.pad = 0; p.pad_w = 0; p.stride = 1; p.up4 = 0;
  p.a_c0 = g.a_c0; p.b_c0 = g.b_c0; p.b_batched = 1;
  p.heads = g.heads; p.a_c_head = g.a_c_head; p.b_c_head = g.b_c_head; p.a_img_per_head = g.a_img_per_head ? 1 : 0;
  p.b_r_head = g.b_r_head; p.out_per_head = g.out_per_head ? 1 : 0; p.o_c_head = g.o_c_head;
  p.chunk = tc_chunk_kblocks();
  p.PW = 0; p.PH = 0;
  p.BW = 16; p.BH = 8; p.tiles_x = 1; p.tiles_y = 2;
  p.m_tiles = g.N * g.heads * 2; p.n_tiles = g.Cout / BN; p.kblocks = g.K / 64;
  if (p.kblocks <= 12) p.chunk = p.kblocks;
  p.in_scale = nullptr; p.in_shift = nullptr; p.in_act = IN_NONE; p.xform = 0; p.a_split = 0; p.fault = 0;
#if CFB_TC_STAMPS
  p.dbg = g_stamps.load();
#endif
  p.Hin = 16; p.Win = 16; p.pad_mode = 0; p.sub = 0; p.out_pitch = out_pitch; p.out_c0 = 0; p.cout_valid = out_pitch; p.res_pitch = out_pitch;
  p.residual2 = nullptr; p.res2_pitch = out_pitch; p.post_scale = 1.f;
  p.bias = nullptr; p.residual = nullptr; p.out_act = OUT_NONE; p.sft_dec = nullptr; p.sft_scale = nullptr; p.sft_w = 0.f; p.sft_wv = nullptr;
  p.wscale_inv = g.scale_dev; p.out = g.out;
  p.gn_part = nullptr; p.gn_cpg = 0;
  p.pl_hi = (__half*)g.out_planes;
  p.pl_lo = g.out_planes ? (__half*)((char*)g.out_planes + (((size_t)out_imgs * 256 * out_pitch * 2 + 1023) / 1024 * 1024)) : nullptr;
  return launch_tc<0>(mp, p, sm_count, st);
}

// softmax over rows of 256 fp32 scores -> fp16 hi/lo operand planes of the probabilities (one warp per row)
__global__ void __launch_bounds__(256) softmax256_planes_kernel(const float* __restrict__ s, __half* __restrict__ hi,
                                                                __half* __restrict__ lo, int64_t rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (row >= rows) return;
  const float4 a = __ldg(reinterpret_cast<const float4*>(s + row * 256 + l * 8));
  const float4 b = __ldg(reinterpret_cast<const float4*>(s + row * 256 + l * 8 + 4));
  float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  float mx = v[0];
#pragma unroll
  for (int j = 1; j < 8; ++j) mx = fmaxf(mx, v[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { v[j] = expf(v[j] - mx); sum += v[j]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;
  __align__(16) __half hh[8];
  __align__(16) __half ll[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float pv = v[j] * inv;
    hh[j] = __float2half_rn(pv);
    ll[j] = __float2half_rn(pv - __half2float(hh[j]));
  }
  *reinterpret_cast<uint4*>(hi + row * 256 + l * 8) = *reinterpret_cast<const uint4*>(hh);
  *reinterpret_cast<uint4*>(lo + row * 256 + l * 8) = *reinterpret_cast<const uint4*>(ll);
}
int softmax256_planes(const float* scores, void* planes, int64_t rows, cudaStream_t st) {
  if (rows == 0) return 0;
  const size_t plane = ((size_t)rows * 256 * 2 + 1023) / 1024 * 1024;
  CFB_LAUNCH_PDL(softmax256_planes_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, st, scores, (__half*)planes,
                 (__half*)((char*)planes + plane), rows);
  return 0;
}

// V^T operand planes: in planes [N][256 tokens][pitch] (channels c0..c0+C) -> out planes [N][C][256], hi and lo
__global__ void transpose_planes_kernel(const __half* __restrict__ in, __half* __restrict__ out, int pitch, int c0, int C) {
  __shared__ __half tile[32][34];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.z, t0 = blockIdx.y * 32, cb = blockIdx.x * 32;
  const __half* ib = in + (int64_t)n * 256 * pitch;
  __half* ob = out + (int64_t)n * C * 256;
  for (int i = threadIdx.y; i < 32; i += 8) tile[i][threadIdx.x] = ib[(int64_t)(t0 + i) * pitch + c0 + cb + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) ob[(int64_t)(cb + i) * 256 + t0 + threadIdx.x] = tile[threadIdx.x][i];
}
int transpose_planes(const void* in_planes, int N, int pitch, int c0, int C, void* out_planes, cudaStream_t st) {
  CFB_REQUIRE(C % 32 == 0, "transpose_planes: C must be a multiple of 32");
  if (N == 0) return 0;
  const size_t ip = ((size_t)N * 256 * pitch * 2 + 1023) / 1024 * 1024;
  const size_t op = ((size_t)N * C * 256 * 2 + 1023) / 1024 * 1024;
  dim3 grid(C / 32, 8, N);
  CFB_REQUIRE(N <= 65535, "transpose_planes: batch too large");
  for (int h = 0; h < 2; ++h) {
    CFB_LAUNCH_PDL(transpose_planes_kernel, grid, dim3(32, 8), 0, st, (const __half*)((const char*)in_planes + h * ip),
                   (__half*)((char*)out_planes + h * op), pitch, c0, C);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------------
// VectorQuantizer.forward as ONE kernel (BASELINE configs[2]; /root/reference/basicsr/archs/vqgan_arch.py:33-70)
//   d = |z|^2 + |e|^2 - 2 z.E^T ; argmin ; z_q = z + (E[idx] - z) ; loss ; perplexity ; mean_distance
// on the caller's NCHW tensors.  One CTA owns 128 consecutive tokens of one image and ALL codes:
//   phase 0  every thread reads its (token, 8-channel) items of z straight from NCHW (coalesced along the tokens), splits them
//            into fp16 hi / lo and writes them into shared memory in the K-major 128B-swizzled layout the wgmma descriptors
//            read (the whole 128 x D A tile stays resident: <= 128 KB), accumulates |z|^2;
//   phase 1  warp 4 streams the prepared codebook planes (B_hi | B_lo of 64 codes x one 64-channel k-block) through a 4-stage
//            TMA ring; the MMA warpgroup (warps 0..3) accumulates the 128 x 64 dot products of a 64-code chunk in registers
//            with the split-fp16 wgmma sequence of the conv engine and keeps (first minimum, index) per token row;
//   phase 2  all threads gather E[idx], write the straight-through z_q in NCHW and the squared-error partial sums; the last CTA
//            of the grid (ticket) turns the partial sums and the code histogram into the three statistics and clears them.
// The [tokens, codes] distance matrix never leaves registers; no other kernel, copy or transpose runs.
// ------------------------------------------------------------------------------------------------------
struct VqParams {
  const float* z; const float* codebook; const float* e2; const float* wscale_inv;
  float* zq; int64_t* idx; float* stats;
  double* part;          // [ctas][2]: squared error, sum of all distances
  unsigned* hist;        // [K]: zero on entry, cleared again by the last CTA
  unsigned* ticket;      // zero on entry
  int N, D, HW, K, kblocks, nchunks;
  float beta;
};
constexpr int VQ_THREADS = 512;      // 16 warps: 0..3 MMA warpgroup, 4 TMA; all 16 move z / z_q in phases 0 and 2
constexpr int VQ_B = 64 * 128, VQ_STAGE = 2 * VQ_B, VQ_STAGES = 4;
constexpr int VQ_A_KB = 128 * 128;      // one 64-channel k-block of one plane: 128 token rows x 128 B

__global__ void __launch_bounds__(VQ_THREADS, 1)
vq_fused_kernel(const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo, const VqParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_hi = smem;                                   // [kblocks][128][128 B]
  uint8_t* a_lo = smem + 4 * VQ_A_KB;
  uint8_t* ring = smem + 8 * VQ_A_KB;                     // VQ_STAGES x (B_hi | B_lo)
  float* e2s = reinterpret_cast<float*>(ring + VQ_STAGES * VQ_STAGE);      // [K <= 1024]
  float* z2p = e2s + 1024;                                // [4 k-blocks][128 tokens]
  int* bidx = reinterpret_cast<int*>(z2p + 512);          // [128]
  double* red = reinterpret_cast<double*>(bidx + 128);    // [4]
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + 8);
  uint64_t* full = bars;
  uint64_t* empty = bars + VQ_STAGES;
  int* s_flags = reinterpret_cast<int*>(empty + VQ_STAGES);   // [0] abort seen, [1] last CTA

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int per_img = p.HW / 128;
  const int n = blockIdx.x / per_img;
  const int hw0 = (blockIdx.x - n * per_img) * 128;
  bool aborted = false;

  if (threadIdx.x == 0) {
    for (int s = 0; s < VQ_STAGES; ++s) { mbar_init(smem_u32(full + s), 1); mbar_init(smem_u32(empty + s), 4); }
    s_flags[0] = 0; s_flags[1] = 0;
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB_lo) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // ---- phase 0: z (NCHW) -> fp16 hi / lo operand tile in shared memory, |z|^2, |e|^2 table
  // One warp item = 16 tokens x one 64-channel k-block: lane (a = lane>>3, b = lane&7) reads 8 channels (b*8..) of 4 consecutive
  // tokens (a) with 16-byte loads along the token axis (64 B segments: every sector fully used) and writes, per token, the
  // 16-byte chunk b of that token's row -- 8 lanes cover a 128 B row, 4 rows per instruction: conflict-free STS.128.
  {
    const int la = lane >> 3, lb = lane & 7;
    for (int k = threadIdx.x; k < p.K; k += VQ_THREADS) e2s[k] = __ldg(p.e2 + k);
    const int items = 8 * p.kblocks;                      // 8 groups of 16 tokens x kblocks
    const float* zn = p.z + (int64_t)n * p.D * p.HW + hw0;
    for (int it0 = warp; it0 < items; it0 += 32) {        // two items in flight per warp (all of them at D = 256)
      float4 v[2][8];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int item = it0 + 16 * u;
        if (item < items) {
          const int kb = item % p.kblocks, t4 = ((item / p.kblocks) * 4 + la) * 4;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            v[u][j] = __ldg(reinterpret_cast<const float4*>(zn + (int64_t)(kb * 64 + lb * 8 + j) * p.HW + t4));
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int item = it0 + 16 * u;
        if (item < items) {
          const int kb = item % p.kblocks, t4 = ((item / p.kblocks) * 4 + la) * 4;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int tl = t4 + k;
            float y[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = k == 0 ? v[u][j].x : (k == 1 ? v[u][j].y : (k == 2 ? v[u][j].z : v[u][j].w));
            uint32_t hw_[4], lw_[4];
            float ss = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float y0 = y[2 * q], y1 = y[2 * q + 1];
              ss = fmaf(y0, y0, ss); ss = fmaf(y1, y1, ss);
              hw_[q] = pack_f16x2(y0, y1);
              const float d0 = f16_minus_f32(hw_[q] & 0xffffu, y0), d1 = f16_minus_f32(hw_[q] >> 16, y1);
              lw_[q] = pack_f16x2(d0, d1) ^ 0x80008000u;
            }
            const uint32_t off = (uint32_t)(kb * VQ_A_KB + tl * 128 + ((((uint32_t)lb) ^ ((uint32_t)tl & 7u)) << 4));
            sts128(smem_u32(a_hi) + off, make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]));
            sts128(smem_u32(a_lo) + off, make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]));
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            ss += __shfl_xor_sync(0xffffffffu, ss, 4);
            if (lb == 0) z2p[kb * 128 + tl] = ss;           // one writer per (k-block, token)
          }
        }
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes of the A tile -> tensor core
  __syncthreads();

  // ---- phase 1
  if (warp == 4) {
    int stage = 0;
    uint32_t phase = 0;
    for (int ch = 0; ch < p.nchunks; ++ch) {
      for (int kb = 0; kb < p.kblocks; ++kb) {
        mbar_wait<200>(smem_u32(empty + stage), phase ^ 1, aborted); if (aborted) goto role_done;
        if (elect_one()) {
          const uint32_t sb = smem_u32(ring + stage * VQ_STAGE), fb = smem_u32(full + stage);
          mbar_expect_tx(fb, (uint32_t)VQ_STAGE);
          tma_load_3d(sb, &tmB_hi, fb, kb * 64, ch * 64, 0);
          tma_load_3d(sb + VQ_B, &tmB_lo, fb, kb * 64, ch * 64, 0);
        }
        __syncwarp();
        if (++stage == VQ_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp < 4) {
    // the MMA warpgroup: thread t holds rows 16*warp + lane/4 (+8) of each 64-row half and codes 8j + 2*(lane%4) (+1) of the
    // chunk; the same k-step order as conv_tc_kernel (per k-step and half: A_lo B_hi, A_hi B_lo, A_hi B_hi), so the dot products
    // equal the stored ones of cfb_vq_nearest bit for bit
    const float wsi = __ldg(p.wscale_inv);
    float z2[4], best[4], dsum = 0.f;
    int bi[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int tl = (r >> 1) * 64 + warp * 16 + (lane >> 2) + (r & 1) * 8;
      z2[r] = 0.f;
      for (int kb = 0; kb < p.kblocks; ++kb) z2[r] += z2p[kb * 128 + tl];
      best[r] = INFINITY; bi[r] = 0x7fffffff;
    }
    int stage = 0;
    uint32_t phase = 0;
    float acc[2][32];
    for (int ch = 0; ch < p.nchunks; ++ch) {
      for (int kb = 0; kb < p.kblocks; ++kb) {
        mbar_wait(smem_u32(full + stage), phase, aborted); if (wg_any(aborted)) { aborted = true; goto role_done; }
        const uint32_t sb = smem_u32(ring + stage * VQ_STAGE);
        const uint32_t ah = smem_u32(a_hi) + kb * VQ_A_KB, al = smem_u32(a_lo) + kb * VQ_A_KB;
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t db_hi = wg_desc(sb + 32 * k, 1024u), db_lo = wg_desc(sb + VQ_B + 32 * k, 1024u);
#pragma unroll
          for (int mh = 0; mh < 2; ++mh) {
            const uint64_t da_hi = wg_desc(ah + mh * 8192 + 32 * k, 1024u), da_lo = wg_desc(al + mh * 8192 + 32 * k, 1024u);
            wg_mma_64x64(acc[mh], da_lo, db_hi, (kb == 0 && k == 0) ? 0u : 1u);
            wg_mma_64x64(acc[mh], da_hi, db_lo, 1u);
            wg_mma_64x64(acc[mh], da_hi, db_hi, 1u);
          }
        }
        wg_commit();
        wg_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(empty + stage));
        if (++stage == VQ_STAGES) { stage = 0; phase ^= 1; }
      }
      // distances of this chunk (the reference's operation order, vqgan_arch.py:40-41); ascending codes, strict <
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int code = ch * 64 + 8 * j + 2 * (lane & 3) + e;
            const float d = (z2[r] + e2s[code]) - 2.f * (acc[r >> 1][4 * j + 2 * (r & 1) + e] * wsi);
            dsum += d;
            if (d < best[r]) { best[r] = d; bi[r] = code; }
          }
        }
      }
    }
    // the four lanes of a row: lowest index among equal minima (torch.argmin)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best[r], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[r], o);
        if (ob < best[r] || (ob == best[r] && oi < bi[r])) { best[r] = ob; bi[r] = oi; }
      }
      if ((lane & 3) == 0) {
        const int tl = (r >> 1) * 64 + warp * 16 + (lane >> 2) + (r & 1) * 8;
        const int b = min(max(bi[r], 0), p.K - 1);
        bidx[tl] = b;
        p.idx[(int64_t)n * p.HW + hw0 + tl] = (int64_t)b;
        atomicAdd(p.hist + b, 1u);
      }
    }
    double ds = (double)dsum;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ds += __shfl_xor_sync(0xffffffffu, ds, o);
    if (lane == 0) red[warp] = ds;
  }
role_done:
  if (aborted && lane == 0) s_flags[0] = 1;
  __syncthreads();
  // ---- phase 2: straight-through z_q (NCHW) and the squared error, all threads
  if (!s_flags[0]) {
    // same item shape as phase 0: (4 consecutive tokens) x (8 channels); 16-byte loads / stores along the token axis
    const int la = lane >> 3, lb = lane & 7;
    const int items = 8 * p.kblocks;
    const float* zn = p.z + (int64_t)n * p.D * p.HW + hw0;
    float* qn = p.zq + (int64_t)n * p.D * p.HW + hw0;
    double se = 0.0;
    for (int item = warp; item < items; item += VQ_THREADS / 32) {
      const int kb = item % p.kblocks, t4 = ((item / p.kblocks) * 4 + la) * 4;
      const int c0 = kb * 64 + lb * 8;
      float4 zz[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) zz[j] = __ldg(reinterpret_cast<const float4*>(zn + (int64_t)(c0 + j) * p.HW + t4));
      float ev[4][8];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float* er = p.codebook + (int64_t)bidx[t4 + k] * p.D + c0;
        const float4 e0 = __ldg(reinterpret_cast<const float4*>(er)), e1 = __ldg(reinterpret_cast<const float4*>(er + 4));
        ev[k][0] = e0.x; ev[k][1] = e0.y; ev[k][2] = e0.z; ev[k][3] = e0.w; ev[k][4] = e1.x; ev[k][5] = e1.y; ev[k][6] = e1.z; ev[k][7] = e1.w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 o;
        float diff;
        diff = ev[0][j] - zz[j].x; se += (double)(diff * diff); o.x = zz[j].x + diff;      // z + (z_q - z), vqgan_arch.py:57
        diff = ev[1][j] - zz[j].y; se += (double)(diff * diff); o.y = zz[j].y + diff;
        diff = ev[2][j] - zz[j].z; se += (double)(diff * diff); o.z = zz[j].z + diff;
        diff = ev[3][j] - zz[j].w; se += (double)(diff * diff); o.w = zz[j].w + diff;
        *reinterpret_cast<float4*>(qn + (int64_t)(c0 + j) * p.HW + t4) = o;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    __shared__ double se_w[VQ_THREADS / 32];
    if (lane == 0) se_w[warp] = se;
    __syncthreads();
    if (threadIdx.x == 0) {
      double a = 0.0, b = 0.0;
      for (int i = 0; i < VQ_THREADS / 32; ++i) a += se_w[i];
      for (int i = 0; i < 4; ++i) b += red[i];
      p.part[(int64_t)blockIdx.x * 2] = a;
      p.part[(int64_t)blockIdx.x * 2 + 1] = b;
      __threadfence();
      s_flags[1] = (atomicAdd(p.ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_flags[1]) {
      // last CTA of the grid: statistics (vqgan_arch.py:42,55,60-61) from the partial sums and the histogram, then clear both
      __threadfence();
      __shared__ double sred[3][VQ_THREADS];
      const int T = p.N * p.HW;
      double ent = 0.0, s_se = 0.0, s_d = 0.0;
      for (int k = threadIdx.x; k < p.K; k += VQ_THREADS) {
        const float em = (float)__ldcg(p.hist + k) / (float)T;
        ent += (double)(em * logf(em + 1e-10f));
        p.hist[k] = 0u;
      }
      for (int i = threadIdx.x; i < (int)gridDim.x; i += VQ_THREADS) { s_se += __ldcg(p.part + 2 * i); s_d += __ldcg(p.part + 2 * i + 1); }
      sred[0][threadIdx.x] = ent; sred[1][threadIdx.x] = s_se; sred[2][threadIdx.x] = s_d;
      __syncthreads();
      if (threadIdx.x == 0) {
        double e = 0.0, s2 = 0.0, d2 = 0.0;
        for (int i = 0; i < VQ_THREADS; ++i) { e += sred[0][i]; s2 += sred[1][i]; d2 += sred[2][i]; }      // fixed order
        const float mse = (float)(s2 / ((double)T * p.D));
        p.stats[0] = mse + p.beta * mse;
        p.stats[1] = expf(-(float)e);
        p.stats[2] = (float)(d2 / ((double)T * p.K));
        p.stats[3] = 0.f;
        *p.ticket = 0u;
      }
    }
  }
  if (aborted) {             // error path only: let the bulk copies still in flight finish before the CTA's shared memory is handed back
    const long long t0 = clock64();
    while (clock64() - t0 < 400000) {}
  }
  __syncthreads();
}

bool vq_fused_supported(int N, int D, int HW, int K) {
  return N >= 0 && D % 64 == 0 && D >= 64 && D <= 256 && HW % 128 == 0 && K % 64 == 0 && K <= 1024;
}

int vq_fused(const float* z, const float* codebook, const void* whi, const void* wlo, const float* wscale_inv, const float* e2,
             unsigned* hist, unsigned* ticket, double* part, int N, int D, int HW, int K, float beta, float* zq, int64_t* idx,
             float* stats, cudaStream_t st) {
  CFB_REQUIRE(vq_fused_supported(N, D, HW, K), "vq_fused: shape not supported");
  if (N == 0) return 0;
  TcMaps mp;
  {
    const uint64_t dims[3] = {(uint64_t)D, (uint64_t)K, 1};
    const uint64_t str[2] = {(uint64_t)D * 2, (uint64_t)K * D * 2};
    const uint32_t box[3] = {64, 64, 1};
    CFB_CHECK(make_map(&mp.b_hi, whi, 3, dims, str, box));
    CFB_CHECK(make_map(&mp.b_lo, wlo, 3, dims, str, box));
  }
  VqParams p;
  p.z = z; p.codebook = codebook; p.e2 = e2; p.wscale_inv = wscale_inv; p.zq = zq; p.idx = idx; p.stats = stats; p.part = part;
  p.hist = hist; p.ticket = ticket; p.N = N; p.D = D; p.HW = HW; p.K = K; p.kblocks = D / 64; p.nchunks = K / 64; p.beta = beta;
  constexpr int SMEM = 8 * VQ_A_KB + VQ_STAGES * VQ_STAGE + 1024 * 4 + 512 * 4 + 128 * 4 + 8 * 8 + 2 * VQ_STAGES * 8 + 64 + 1024;
  static_assert(SMEM <= 232448, "shared memory budget");
  static std::atomic<uint64_t> attr_done{0};
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(attr_done.load(std::memory_order_acquire) & bit)) {
    CFB_CUDA(cudaFuncSetAttribute(vq_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_done.fetch_or(bit, std::memory_order_release);
  }
  vq_fused_kernel<<<(unsigned)(N * (HW / 128)), VQ_THREADS, SMEM, st>>>(mp.b_hi, mp.b_lo, p);
  CFB_LAUNCH_CHECK();
  return 0;
}

}  // namespace cfb
