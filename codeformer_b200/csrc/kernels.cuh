// Internal launcher interface between the host runtime (runtime.cu / capi.cu) and the kernels.
// Every launcher enqueues on `st` and returns the launch status; none synchronises.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

namespace cfb {

// ---- error plumbing --------------------------------------------------------------------------
void set_error(const std::string& msg);
#define CFB_CUDA(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::cfb::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                       std::to_string(__LINE__));                                                 \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)
#define CFB_LAUNCH_CHECK()                                                                        \
  do {                                                                                            \
    cudaError_t _e = cudaGetLastError();                                                          \
    if (_e != cudaSuccess) {                                                                      \
      ::cfb::set_error(std::string("kernel launch failed: ") + cudaGetErrorString(_e) + " @" +    \
                       __FILE__ + ":" + std::to_string(__LINE__));                                \
      return 1;                                                                                   \
    }                                                                                             \
    ::cfb::count_launch();                                                                        \
  } while (0)
#define CFB_CHECK(x)                                                                              \
  do {                                                                                            \
    if ((x) != 0) return 1;                                                                       \
  } while (0)
#define CFB_REQUIRE(cond, msg)                                                                    \
  do {                                                                                            \
    if (!(cond)) {                                                                                \
      ::cfb::set_error(std::string(msg) + " [" #cond "] @" + __FILE__ + ":" + std::to_string(__LINE__)); \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

// asynchronous device status word (host-mapped): kernels report a barrier time-out or an fp16 operand overflow here instead
// of trapping; the host turns it into an error without poisoning the context (runtime.cu)
#define CFB_STATUS_TIMEOUT 1u
#define CFB_STATUS_OVERFLOW 2u
#define CFB_STATUS_INDEX 4u      // a code index outside the codebook was given (cfb_code_scores)
int async_status_init(cudaStream_t st);      // per-device one-time setup (idempotent)
int async_status_check(const char* where);   // non-zero + set_error() when a kernel reported a failure since the last check
// device pointer of the current device's status word (bound on first use), for kernels outside conv_tc.cu: they take it as
// an argument (the library is linked without -rdc, so conv_tc.cu's device symbols are not visible to them)
int async_status_word(unsigned** dev_word);
int tc_bind_status_word(unsigned* host_mapped_dev_ptr, long long wait_limit_cycles);   // conv_tc.cu: device symbols of this device
int tc_clear_abort();
int tc_set_stamps(long long* dev_ptr);     // diagnostics: phase stamps of CTA 0 (cfb_debug_set_stamps)
int tc_inject_fault(int kind);               // test hook: the next wgmma conv launch drops one TMA load (-> barrier time-out)

void count_launch();
int64_t launch_count();
void reset_launch_count();

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------
// The forward is a chain of ~340 dependent launches; with plain stream order each one pays the launch latency and its own
// set-up (barrier init, tensor-map prefetch) after the previous grid has
// drained.  Kernels launched through CFB_LAUNCH_PDL carry cudaLaunchAttributeProgrammaticStreamSerialization: their CTAs may
// start as soon as every CTA of the previous grid has executed pdl_launch_dependents() (SM resources permitting), do their
// set-up, and block in pdl_wait() until the previous grid has COMPLETED and its memory is visible.  Rules kept everywhere:
//   * every thread calls pdl_wait() before its first access to global memory another kernel may have written (and before its
//     own first global write), and before any early return;
//   * a kernel without the attribute behaves as before (the instructions are no-ops there), so the two kinds mix freely.
// CFB_PDL=0 switches the attribute off (A/B timing).
bool pdl_enabled();
#ifdef __CUDACC__
#ifndef CFB_PDL_DEVICE
#define CFB_PDL_DEVICE 1
#endif
#if CFB_PDL_DEVICE
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#else      // A/B builds without the device side (the host side then never sets the attribute: pdl_enabled() is false)
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_launch_dependents() {}
#endif
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
// launch + error plumbing + launch counter (kernel must call pdl_wait())
#define CFB_LAUNCH_PDL(kernel, grid, block, smem, st, ...)                                          \
  do {                                                                                              \
    cudaError_t _e = ::cfb::launch_pdl(kernel, grid, block, smem, st, __VA_ARGS__);                 \
    if (_e != cudaSuccess) {                                                                        \
      ::cfb::set_error(std::string("kernel launch failed: ") + cudaGetErrorString(_e) + " @" +      \
                       __FILE__ + ":" + std::to_string(__LINE__));                                  \
      return 1;                                                                                     \
    }                                                                                               \
    ::cfb::count_launch();                                                                          \
  } while (0)

// ---- GroupNorm partial slots ----------------------------------------------------------------------
// A slot holds (mean, M2) of its values, M2 = sum of squared deviations from the slot mean, never (sum, sum of squares): with
// a group mean r times its standard deviation, fp32 sums of squares lose the variance to cancellation like (1 + r^2) * 2^-24,
// the moments only like r * 2^-24 (through the rounding of the mean).  Producers sum the deviations from one value k of the
// lane (s = sum (x - k), q = sum (x - k)^2 over n values) and turn them into moments ...
__device__ __forceinline__ void gn_lane_moments(float& s, float& q, float k, float n) {
  const float d = s * (1.f / n);          // n is a power of two: exact
  q = fmaxf(fmaf(-s, d, q), 0.f);
  s = k + d;
}
// ... then merge equal counts (n values each) with lane ^ o (Chan et al.): mean = (ma + mb) / 2, M2 = M2a + M2b +
// (ma - mb)^2 * 2n / 4.  Symmetric in the two lanes, so both hold the same bits afterwards.
__device__ __forceinline__ void gn_merge_xor(float& mean, float& m2, int o, float n) {
  const float om = __shfl_xor_sync(0xffffffffu, mean, o), oq = __shfl_xor_sync(0xffffffffu, m2, o);
  const float d = mean - om;
  m2 = (m2 + oq) + (d * d) * (0.5f * n);
  mean = 0.5f * (mean + om);
}
// The caller's image plumbing of a uint8 face, bit for bit (inference_codeformer.py:199-200 + basicsr/utils/img_util.py:22-29):
//   t = float32(u8 / 255.)  [numpy float64 division, then astype float32];  x = (t - 0.5) / 0.5  [torchvision normalize, fp32]
__device__ __forceinline__ float u8_to_model_input(int u) {
  const float t = (float)((double)u / 255.0);
  return __fdiv_rn(__fsub_rn(t, 0.5f), 0.5f);
}
#endif

enum InAct { IN_NONE = 0, IN_SILU = 1 };
enum OutAct { OUT_NONE = 0, OUT_LRELU = 1, OUT_GELU = 2, OUT_RELU = 3, OUT_SILU = 4, OUT_PRELU = 5 };
enum ConvMode { CONV_SAME = 0, CONV_DOWN = 1, CONV_UP = 2 };

// Convolution / linear layer as an implicit GEMM over NHWC fp32 activations.
//   M = N*Ho*Wo output pixels (tokens), N = Cout, K = taps*Cin.
struct ConvArgs {
  const float* in = nullptr;        // [N,H,W,Cin]  (H,W are the stored dims; CONV_UP reads (y>>1,x>>1))
  int N = 0, H = 0, W = 0, Cin = 0;
  int Ho = 0, Wo = 0, Cout = 0;
  int ksize = 3;                    // 1 | 3
  int mode = CONV_SAME;
  int down_pad = 0;                 // CONV_DOWN (per-tap engine): zero padding before the window; 0 = the Downsample's (0,1,0,1)
                                    // padding (Ho = H/2), 1 = a torchvision-style 3x3 stride-2 pad-1 conv (Ho = ceil(H/2))
  // per-tap engine, explicit window (kh > 0; ksize and down_pad are then not read): a kh x kw kernel (1..7 each) with zero
  // padding pad_h / pad_w on both sides, stride 1 (CONV_SAME) or 2 (CONV_DOWN); Ho = (H + 2 pad_h - kh) / stride + 1, likewise Wo.
  // Weights [kh * kw][Cout][Cin] (tc_split_weights_taps).  Inception-v3's 1x7 / 7x1 / 1x3 / 3x1 / 5x5 and valid 3x3 convs
  int kh = 0, kw = 0, pad_h = 0, pad_w = 0;
  const float* wgt_f32 = nullptr;   // [taps][Cin][Cout] fp32 (CUDA-core engine)
  const void* wgt_hi = nullptr;     // [taps][Cout][Cin] fp16 hi   (tensor-core engine)
  const void* wgt_lo = nullptr;     // [taps][Cout][Cin] fp16 lo
  const float* wscale_inv = nullptr; // device scalar 2^-k undoing the power-of-two scaling of the fp16 weight split
  const float* bias = nullptr;      // [Cout] | null
  const float* in_scale = nullptr;  // [N,Cin] fused per-sample affine (GroupNorm folded) | null
  const float* in_shift = nullptr;
  int in_act = IN_NONE;
  const float* residual = nullptr;  // [N,Ho,Wo,Cout] | null
  int out_act = OUT_NONE;
  // SFT epilogue (codeformer_arch.py:155-156): out = dec + w*(dec*scale + conv)
  const float* sft_dec = nullptr;
  const float* sft_scale = nullptr;
  float sft_w = 0.f;
  const float* sft_wv = nullptr;    // [N] per-image w (device) in place of sft_w | null; w <= 0 or NaN blends with 0 (out = dec)
  float* out = nullptr;             // [N,Ho,Wo,Cout]
  float prelu_slope = 0.f;          // OUT_PRELU (ResNetArcFace): out = v > 0 ? v : slope * v; generalised and per-tap engines
  // tensor-core engine only: GroupNorm(32) partials of `out`, [N*tiles_per_image*4][32 groups][mean, M2] floats
  float* gn_part = nullptr;
  // tensor-core engine only: also emit `out` as fp16 hi/lo operand planes for a following conv that consumes it raw
  void* out_planes = nullptr;       // [hi plane | lo plane], each align1024(N*Ho*Wo*Cout*2) bytes
  bool skip_prep = false;           // operand planes in `scratch` are already valid (kernel-only timing)
  bool xform = false;      // tensor engine: read the fp32 activation `in` directly and apply in_scale/in_shift/in_act + the fp16 hi/lo
                           // split inside the conv kernel (tc_can_xform); in_scale == null: plain split of the raw values
  bool halo1x1 = false;    // 1x1 conv with a GroupNorm-affine input (AttnBlock q,k,v): run it on the halo engine (patch = tile, one
                           // tap) so that the fused operand transform applies -- no separate operand-preparation pass
  const float* in2 = nullptr;   // xform only: channels [Cin1, Cin) come from this second NHWC tensor (torch.cat of Fuse_sft_block)
  int Cin1 = 0;
  // ---- generalised addressing (xform only; ParseNet / RRDBNet rows f3 / f4): any H x W (ragged tiles), padding mode of the
  // 3x3 window, source / destination inside wider NHWC buffers (dense blocks), stride 2 by subsampling, second residual
  bool gen = false;
  int in_pitch = 0;             // channels per pixel of the buffer `in` points into (0: Cin); Cin is the 64-aligned window read
  int pad_mode = 0;             // 0 zero, 1 reflect, 2 replicate
  bool subsample = false;       // keep the even output positions only: out is [N, Ho/2, Wo/2, ...] (Ho, Wo even)
  int out_pitch = 0, out_c0 = 0;   // destination channels per pixel (0: Cout) and channel offset
  int cout_valid = 0;           // real output channels (0: Cout); Cout itself is the 64-aligned padded count of the weights
                                // (also read by the per-tap engine: columns from cout_valid on are not stored)
  int res_pitch = 0;            // channels per pixel of `residual` (0: out_pitch)
  const float* residual2 = nullptr;   // out = act(conv + bias + residual) * post_scale + residual2
  int res2_pitch = 0;
  float post_scale = 1.f;
  // opt-in: fp16 operands, one A_hi*B_hi wgmma product per k-step instead of the split scheme's three (fp32 accumulation and
  // output as before); the lo weight plane stays prepared but is not read, nor is the lo plane of a raw-planes input.  Built
  // for gen, the 128-wide and channel-major halo tiles and the per-tap 1x1 conv (conv_tc raises elsewhere)
  bool single_pass = false;
};

int conv_f32(const ConvArgs& a, cudaStream_t st);                       // CUDA-core fp32 implicit GEMM
// first conv: x NCHW [N,3,H,W] -> NHWC [N,H,W,Cout], 3x3 p1; weight [27][Cout] (tap-major, then cin)
// gn_part (optional): GroupNorm(32) partials of `out`, [N * H*W/32 slots][32 groups][mean, M2] (the layout
// gn_coef_from_partials reads; slots per image = H*W/32)
int conv_first(const float* x_nchw, const float* wgt, const float* bias, float* out, int N, int H, int W, int Cout,
               cudaStream_t st, float* gn_part = nullptr);
// last conv: NHWC [N,H,W,Cin] (+ fused affine) -> NCHW [N,3,H,W], 3x3 p1; weight [9][Cin][3]
int conv_last(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
              float* out_nchw, int N, int H, int W, int Cin, cudaStream_t st);
// the same two kernels with the caller's image plumbing fused in (inference_codeformer.py:199-206,
// basicsr/utils/img_util.py:9-35,38-94): uint8 HWC BGR face in, uint8 HWC BGR restored face out
// n_orig in (0, N): images n >= n_orig are face n - n_orig mirrored left-right (cv2.flip(face, 1)); 0 = no mirror
int conv_first_u8(const unsigned char* x_bgr_hwc, const float* wgt, const float* bias, float* out, int N, int H, int W,
                  int Cout, cudaStream_t st, float* gn_part = nullptr, int n_orig = 0);
int conv_last_u8(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
                 unsigned char* out_bgr_hwc, int N, int H, int W, int Cin, cudaStream_t st);
// conv_last_u8 with the inpainting blend of inference_inpainting.py:68-75 before the conversion: where the normalised input
// face (the forward's own uint8 input, face_bgr_hwc) sums to 3 over its channels the output is the network's, elsewhere the input
int conv_last_u8_inpaint(const float* in, const float* in_scale, const float* in_shift, const float* wgt, const float* bias,
                         const unsigned char* face_bgr_hwc, unsigned char* out_bgr_hwc, int N, int H, int W, int Cin,
                         cudaStream_t st);
int u8_to_input(const unsigned char* img_bgr_hwc, float* x_nchw, int N, int64_t HW, cudaStream_t st);
int output_to_u8(const float* x_nchw, unsigned char* img_bgr_hwc, int N, int64_t HW, cudaStream_t st);

// thin convolutions of the caller-side networks (rows f3 / f4): image channels -> 64 features and 64 features -> image channels
int conv_thin_in(const float* x_nchw, const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int Cimg, int us,
                 int pad_mode, int out_pitch, int out_c0, cudaStream_t st);
int conv_thin_out(const float* in_nhwc64, const float* wgt_tcp, const float* bias, float* out_nchw, int N, int H, int W, int Cout,
                  int pad_mode, cudaStream_t st);
// RRDBNet's tiles read from / written to images (cfb_rrdb_forward_u8_tiles, cfb_rrdb_forward_tiles): one row of its tile table.  The table of
// one launch travels by value in the kernel parameters (9 * 4 * 64 bytes, under the 4 KB parameter limit).
struct RrdbU8Tile {
  int img;                       // source image / canvas index
  int in_y, in_x;                // input window origin, in the coordinates of the pre_pad + mod-padded image
  int crop_y, crop_x, crop_h, crop_w;   // kept rectangle of the tile's output
  int out_y, out_x;              // its canvas position
};
struct RrdbU8Tiles {
  static constexpr int kMax = 64;
  RrdbU8Tile t[kMax];
};
// Element type of the images those tiles are read from and written to (the CFB_IMG_* values of include/cfb200.h).
enum ImgKind { IMG_U8 = 0, IMG_U16 = 1, IMG_F32 = 2, IMG_F64 = 3 };
// max_range: the reference's per-image divisor, device int32 [images] from image_max_range, or nullptr for 255 (uint8 images).
// The input is float32(v) / max_range, the output clamp(v, 0, 1) * max_range rounded half to even (saturated in a uint8 canvas).
int conv_thin_in_tiles(const void* img_bgr_hwc, int in_kind, const int* max_range, int img_h, int img_w, int pre_pad,
                       const RrdbU8Tiles& tiles, const float* wgt_tck, const float* bias, float* out, int N, int H, int W, int us,
                       int out_pitch, int out_c0, cudaStream_t st);
int conv_thin_out_tiles(const float* in_nhwc64, const float* wgt_tcp, const float* bias, const RrdbU8Tiles& tiles,
                        void* canvas_bgr_hwc, int out_kind, const int* max_range, int out_h, int out_w, int N, int H, int W,
                        cudaStream_t st);
// RealESRGANer.enhance's `max_range = 65535 if np.max(img.astype(np.float32)) > 256 else 255` of each of n images of `count`
// elements, into device int32 max_range[n]; a NaN makes np.max NaN, hence 255.  No host synchronisation.
int image_max_range(const void* images, int kind, int n, int64_t count, int* max_range, cudaStream_t st);
// ParseNet's ends for cfb_parsenet_masks_u8: the input conv reads uint8 HWC BGR faces [N, H, W, 3] (the value of
// u8_to_input); the output conv writes the argmax classes and / or the 0/255 face mask, uint8 [N, H, W] (either may be NULL)
int conv_thin_in_u8_faces(const unsigned char* faces_bgr_hwc, const float* wgt_tck, const float* bias, float* out, int N, int H, int W,
                          int pad_mode, int out_pitch, int out_c0, cudaStream_t st);
int conv_thin_out_argmax(const float* in_nhwc64, const float* wgt_tcp, const float* bias, unsigned char* cls, unsigned char* mask,
                         int N, int H, int W, int Cout, int pad_mode, cudaStream_t st);
int relayout_thin_out(const float* oihw, float* out, int Cout, cudaStream_t st);
int fold_bn(const float* w, const float* gamma, const float* beta, const float* mean, const float* var, float eps, float* wout,
            float* bout, int Cout, int per_out, cudaStream_t st);
// RetinaFace-ResNet50 (detection.cu): stem conv + max-pool, FPN top-down add, head gather, candidate compaction
// face_u8: the uint8 input is a BGR face normalised like u8_to_input (RGB, (x / 255 - 0.5) / 0.5; BiSeNet) instead of the
// detector's mean-subtracted BGR image
int rf_stem(const float* x_nchw, const unsigned char* img_bgr_hwc, const float* wt, const float* bias, float* out, int N, int H,
            int W, cudaStream_t st, bool face_u8 = false);
int rf_maxpool(const float* in, float* out, int N, int H, int W, cudaStream_t st);
int rf_add_nearest(float* fine, const float* coarse, int N, int Hf, int Wf, int Hc, int Wc, int C, cudaStream_t st);
int rf_heads(const float* const h[3], const int hh[3], const int ww[3], float* loc, float* conf, float* landms, int N, int P,
             cudaStream_t st);
int rf_candidates(const float* loc, const float* conf, const float* landms, int N, int H, int W, float thr, float* rows, int* counts,
                  cudaStream_t st);
// YOLOv5l-face (yolo.cu): stem conv, StemBlock / SPP max pools, concat-slice copy, Detect decode, candidate compaction
int yolo_stem(const float* x_nchw, const unsigned char* img_bgr_hwc, const float* wt, const float* bias, float* out, int N, int H,
              int W, int ih, int iw, int top, int left, cudaStream_t st);
int yolo_maxpool2(const float* in, float* out, int N, int H, int W, int C, int out_pitch, int out_c0, cudaStream_t st);
int yolo_spp(float* buf, int N, int H, int W, int C, cudaStream_t st);
int yolo_copy(const float* src, int src_pitch, int src_c0, float* dst, int dst_pitch, int dst_c0, int N, int Hs, int Ws, int C,
              bool up2, cudaStream_t st);
int yolo_decode(const float* const h[3], float* const raw[3], const int ny[3], const int nx[3], const float* anchor_grid, float* pred,
                int N, int P, cudaStream_t st);
int yolo_candidates(const float* pred, int N, int P, float thr, float* rows, int* counts, cudaStream_t st);
// ResNetArcFace (arcface.cu): stem conv + PReLU + max pool (fp32 [N,1,128,128], or uint8 BGR 512 x 512 faces with the gray
// resize fused) -> NHWC [N,64,64,64]; the per-image bn0 tables of the IRBlocks; the prepare-time BatchNorm folds
int arc_stem(const float* x, const unsigned char* faces_bgr_hwc, const float* wt, const float* bias, float slope, float* out, int N,
             cudaStream_t st);
struct ArcBn0Table {               // block b's channels are [off[b], off[b + 1]) of the prepared per-channel tables
  static constexpr int kMax = 128;
  int blocks = 0;
  int off[kMax + 1] = {};
};
int arc_bn0_tables(const float* scale, const float* shift, const ArcBn0Table& t, int N, float* dscale, float* dshift,
                   cudaStream_t st);
int arc_bn_affine(const float* g, const float* b, const float* m, const float* v, float eps, float* scale, float* shift, int C,
                  cudaStream_t st);
int arc_fold_fc(const float* w, const float* fc_b, const float* s4, const float* t4, const float* s5, const float* t5, int Cout, int C,
                int HW, float* wout, float* bout, cudaStream_t st);
// BiSeNet (bisenet.cu): whole-map mean of an NHWC tensor -> [N, C]; the 1x1 attention convs on it (one CTA per image); the
// channel-scale combine; bilinear (align_corners=True) upsampling of the head logits, alone or fused with the parse argmax
int bise_mean(const float* in, float* out, int N, int HW, int C, cudaStream_t st);
struct BiseAttention {             // y = act1(w1 v + b1) [c0 -> c1], then z = act2(w2 y + b2) [c1 -> c2] when w2 is set
  const float* w1; const float* b1; int c0, c1, act1;      // act: 0 none, 1 ReLU, 2 sigmoid; weights [cout][cin]
  const float* w2; const float* b2; int c2, act2;
};
int bise_attention(const BiseAttention& a, const float* v, float* out, int N, cudaStream_t st);
int bise_scale_add(const float* feat, const float* att, const float* add_vec, const float* add_t, float* out, int N, int64_t HW, int C,
                   cudaStream_t st);
int bise_bilinear(const float* in, int pitch, int h, int w, int C, float* out, int N, int H, int W, cudaStream_t st);
int bise_bilinear_argmax(const float* in, int pitch, int h, int w, int C, unsigned char* cls, unsigned char* mask, int N, int H, int W,
                         cudaStream_t st);
// LPIPS-VGG (lpips.cu): image i of a launch is image i % (1 + G) of group i / (1 + G), 0 the reference, j >= 1 candidate j - 1
//   stem      conv1_1 + ReLU -> NHWC [M,H,W,64] from fp32 NCHW ref [groups] / cand [groups * G] through the LpipsXform chain, or
//             from uint8 HWC BGR ref8 / cand8 through `table` ([3][256], RGB channel order) when table is set
//   head      relu_k [M,H,W,C] -> pooled [M,H/2,W/2,C] (null: none) and partial [groups][G][lpips_head_blocks(H, W)]
//   finalize  partials of L.n layers -> val [P] (the sum over the layers) and per_layer [P][L.n] (either may be null)
enum { LPIPS_NORMALIZE = 1, LPIPS_RANGE_NORM = 2, LPIPS_INPUT_NORM = 4 };
struct LpipsXform {                // applied in the order range_norm, input_norm, normalize, ScalingLayer
  int flags = 0;
  float mean[3] = {}, std[3] = {}, shift[3] = {}, scale[3] = {};
};
struct LpipsLayers {
  static constexpr int kMax = 5;
  int n = 0;
  const float* part[kMax] = {};
  int nblk[kMax] = {};
  int64_t hw[kMax] = {};
};
int lpips_stem(const float* ref, const float* cand, const unsigned char* ref8, const unsigned char* cand8, const float* table,
               const LpipsXform& xf, const float* wt, const float* bias, float* out, int groups, int G, int H, int W, cudaStream_t st);
int lpips_head_blocks(int H, int W);
int lpips_head(const float* feat, const float* lin, int groups, int G, int H, int W, int C, float* pooled, float* partial,
               cudaStream_t st);
int lpips_finalize(const LpipsLayers& L, int P, float* val, float* per_layer, cudaStream_t st);
// Inception-v3 for FID (fid.cu).  The input stage: fp32 NCHW RGB (f32) or uint8 HWC BGR (u8, read as RGB v / 255) of H x W;
// resize: bilinear (align_corners=False) to FID_SIZE x FID_SIZE, else the source size; normalize: 2x - 1 afterwards
constexpr int FID_SIZE = 299;
struct FidInput {
  const float* f32 = nullptr;
  const unsigned char* u8 = nullptr;
  int H = 0, W = 0;
  int resize = 0, normalize = 0;
};
int fid_input(const FidInput& in, float* out_nchw, int N, cudaStream_t st);
// Conv2d_1a_3x3 (3x3 stride 2 valid, weights [32][27] with the BatchNorm folded) + ReLU on the input stage's values -> NHWC
// [N, Ho, Wo, pitch], channels [32, pitch) zero; nan_flag[n] (zero on entry) is set when a stem output of image n is NaN
int fid_stem(const FidInput& in, const float* wt, const float* bias, float* out, int* nan_flag, int pitch, int N, cudaStream_t st);
// 3x3 max pool, stride 2 valid or stride 1 pad 1, of channels [0, C) into channels [out_c0, out_c0 + C) of the destination
int fid_maxpool(const float* in, int in_pitch, float* out, int out_pitch, int out_c0, int N, int H, int W, int C, int stride,
                cudaStream_t st);
int fid_avgpool(const float* in, int in_pitch, float* out, int out_pitch, int N, int H, int W, int C, cudaStream_t st);
// -> [N, C]; NaN for the images whose nan_flag is set (nan_flag may be null)
int fid_global_pool(const float* in, int pitch, const int* nan_flag, float* out, int N, int H, int W, int C, cudaStream_t st);
// float64 mean mu [D] and covariance sigma [D, D] (np.cov(x, rowvar=False)) of x [N, D]; D a multiple of 64, N >= 2
int fid_stats(const float* x, int64_t N, int D, double* mu, double* sigma, cudaStream_t st);
int parse_argmax(const float* logits_nchw, unsigned char* cls, unsigned char* mask, int N, int C, int64_t HW, cudaStream_t st);
int scale_scalar(float* p, float f, cudaStream_t st);
int scale_vec(float* p, int n, float f, cudaStream_t st);

// Restoration metrics (metrics.cu; cfb_psnr_ssim): pair p compares a[p] with b[p / k], HWC images [h, w, c] of element type
// `kind` (ImgKind); psnr_mode 0 none, 1 PSNR in dB, 2 the MSE; ssim (optional) the mean SSIM.  Outputs: device double [pairs].
struct MetricArgs {
  const void* a; const void* b; int kind;
  int pairs, k, h, w, c, crop;
  bool y;                           // test_y_channel
  int psnr_mode; double* psnr; double* ssim;
};
size_t metrics_workspace_bytes(int pairs, int h, int w, int c, int crop, bool y);
int psnr_ssim(const MetricArgs& a, void* ws, int64_t ws_bytes, cudaStream_t st);

// weight re-layout: OIHW -> [taps][Cin][Cout]
int relayout_oihw_to_tck(const float* oihw, float* out, int Cout, int Cin, int k, cudaStream_t st);

// GroupNorm statistics -> per-(n,c) scale/shift.  partials: workspace of gn_partial_count() doubles
size_t gn_workspace_bytes(int N, int HW, int C);
int gn_coef(const float* x, const float* gamma, const float* beta, float* scale, float* shift, int N, int HW, int C,
            int groups, float eps, void* ws, cudaStream_t st);
// finalize from the (mean, M2) slots of the tensor-core epilogue or conv_first (slots per image = H*W/32)
// scratch: gn_final_scratch_bytes(N, slots) bytes; counters: N zero-initialised unsigned (left zero again by the kernel)
size_t gn_final_scratch_bytes(int N, int slots);
int gn_coef_from_partials(const float* part, int slots, const float* gamma, const float* beta, float* scale, float* shift,
                          int N, int HW, int C, int groups, float eps, void* scratch, unsigned* counters, cudaStream_t st);
// partials of cat([a,b]) (2C channels, 32 groups) from the partials of a and b (C channels each)
int gn_cat_partials(const float* a_part, const float* b_part, float* out_part, int64_t total_slots, int C, cudaStream_t st);
int affine_act(const float* x, const float* scale, const float* shift, float* y, int N, int HW, int C, int act,
               cudaStream_t st);

// out (fp32) and/or out_planes (fp16 hi | lo operand planes of the same [B*S, o_pitch] matrix) receive the result
int attention(const float* q, const float* k, const float* v, float* out, int B, int S, int heads, int d, int q_pitch,
              int k_pitch, int v_pitch, int o_pitch, float scale, cudaStream_t st, void* out_planes = nullptr);
int layer_norm(const float* x, const float* gamma, const float* beta, float* y, float* y2, const float* pos,
               int pos_rows, int rows, int C, cudaStream_t st);
int layer_norm_planes(const float* x, const float* gamma, const float* beta, void* y_planes, void* y2_planes, const float* pos,
                      int pos_rows, int rows, int C, cudaStream_t st);
int add_pos(const float* x, const float* pos, float* y, int rows, int pos_rows, int C, cudaStream_t st);
// logits [T,K] -> idx [T] (first max), quant [T,D] = E[idx]
int argmax_gather(const float* logits, const float* codebook, int64_t* idx, float* quant, int T, int K, int D,
                  cudaStream_t st);
int gather_rows(const int64_t* idx, const float* codebook, float* out, int T, int K, int D, cudaStream_t st);
// code-prediction scores per image of S tokens, in float64 (cfb_code_scores): out[b] = {mean CE, tokens with top_idx == gt, mean
// squared distance of lq [B*S,D] (NHWC) to E[gt]}.  A gt index outside [0,K) is not read: it sets CFB_STATUS_INDEX, and that
// image's three values are NaN.
int code_scores(const float* logits, const int64_t* top_idx, const int64_t* gt, const float* lq, const float* codebook, int B,
                int S, int K, int D, double* out, cudaStream_t st);
int adain_nhwc(const float* content, const float* style, float* out, int B, int HW, int C, cudaStream_t st);
int nchw_to_nhwc(const float* in, float* out, int N, int C, int HW, cudaStream_t st);
int nhwc_to_nchw(const float* in, float* out, int N, int C, int HW, cudaStream_t st);
int concat_channels(const float* a, const float* b, float* out, int64_t pixels, int Ca, int Cb, cudaStream_t st);
// fidelity sweep (cfb_codeformer_sweep_u8): for each listed buffer of B faces of `bytes` each, face b is copied to faces
// b*K .. b*K+K-1 of dst (face-major).  bytes, src and dst 16-byte aligned.
constexpr int EXPAND_MAX = 16;
struct ExpandCopy { const void* src; void* dst; int64_t bytes; };
struct ExpandList { ExpandCopy d[EXPAND_MAX]; int n = 0; };
int expand_faces(const ExpandList& L, int B, int K, cudaStream_t st);

// VectorQuantizer.forward core on token-major z [T,D] (NHWC); writes idx, zq_st = z + (E[idx]-z) [T,D],
// stats = {loss, perplexity, mean_distance, 0}; onehot optional [T,K]
size_t vq_workspace_bytes(int T, int D, int K);
int vq_nearest(const float* z, const float* codebook, int T, int D, int K, float beta, int64_t* idx, float* zq,
               float* stats, float* onehot, void* ws, cudaStream_t st);

// one-kernel path (cfb_vq_nearest_fast): |e_k|^2 of the prepared codebook, and the one-hot rows of its indices
int vq_e2(const float* codebook, float* e2, int K, int D, cudaStream_t st);
int onehot_from_idx(const int64_t* idx, float* onehot, int T, int K, cudaStream_t st);

// tensor-core variant: dots [T,K] = z . E^T already computed (wgmma 1x1 conv); selects the nearest code per token
size_t vq_select_workspace_bytes(int T, int K);
int vq_select_from_dots(const float* z, const float* codebook, const float* dots, int T, int D, int K, float beta, int64_t* idx,
                        float* zq, float* stats, float* onehot, void* ws, cudaStream_t st);
}  // namespace cfb
