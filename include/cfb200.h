/*
 * cfb200.h -- C ABI of libcfb200.so, the H100-native (sm_90a) replacement of CodeFormer's
 * core forward pass.
 *
 * Drop-in boundary.  The reference has no FFI on this path: the arithmetic is reached
 * through PyTorch nn.Modules looked up in a registry
 *   ARCH_REGISTRY.get('CodeFormer') / .get('VQAutoEncoder')   basicsr/utils/registry.py:62-66,79
 *   CodeFormer.forward(x, w, detach_16, code_only, adain)      basicsr/archs/codeformer_arch.py:223-280
 *   VQAutoEncoder.forward(x)                                   basicsr/archs/vqgan_arch.py:385-389
 *   VectorQuantizer.forward(z) / get_codebook_feat             basicsr/archs/vqgan_arch.py:33-84
 * and the only native-extension convention the reference has is the pybind11 `m.def` modules
 * of basicsr/ops/{dcn,fused_act,upfirdn2d}/src/*.cpp built by basicsr/setup.py:118-135.
 * This header is what a maintainer binds instead (ctypes stub in INTEGRATION.md): plain C,
 * raw device/host pointers + sizes + a cudaStream_t passed as void*, int status returns
 * (0 = ok; cfb_last_error() gives the message).  No torch types cross this boundary.
 *
 * All tensors are fp32 and contiguous.  "NCHW" tensors use the reference's layout; internal
 * activations are NHWC and never leave the library.  Every call enqueues on `stream` and
 * returns without synchronising unless stated.
 */
#ifndef CFB200_H_
#define CFB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CFB_VERSION 100

typedef struct cfb_net cfb_net;

/* Constructor arguments of the reference classes.
 * CodeFormer(dim_embd, n_head, n_layers, codebook_size, latent_size, connect_list)  codeformer_arch.py:162-166
 * VQAutoEncoder(img_size, nf, ch_mult, 'nearest', res_blocks, attn_resolutions, codebook_size, emb_dim, beta)
 *                                                                                    vqgan_arch.py:328-329 */
typedef struct cfb_config {
  int32_t kind;            /* 0 = VQAutoEncoder, 1 = CodeFormer */
  int32_t img_size;        /* 512 */
  int32_t nf;              /* 64 */
  int32_t n_ch_mult;       /* 6 */
  int32_t ch_mult[8];      /* 1,2,2,4,4,8 */
  int32_t res_blocks;      /* 2 */
  int32_t n_attn_res;      /* 1 */
  int32_t attn_res[4];     /* 16 */
  int32_t codebook_size;   /* 1024 */
  int32_t emb_dim;         /* 256 */
  float   beta;            /* 0.25 */
  /* CodeFormer only */
  int32_t dim_embd;        /* 512 */
  int32_t n_head;          /* 8 */
  int32_t n_layers;        /* 9 */
  int32_t latent_size;     /* 256 */
  int32_t n_connect;       /* 4 */
  int32_t connect[6];      /* 32,64,128,256 (feature sizes of connect_list) */
} cfb_config;

/* ---- library ---- */
int         cfb_version(void);
const char* cfb_last_error(void);             /* thread-local message of the last failing call */
int         cfb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- network life cycle (replaces nn.Module construction + load_state_dict) ---- */
cfb_net* cfb_net_create(const cfb_config* cfg);                 /* NULL on error */
void     cfb_net_destroy(cfb_net* net);
/* Hand one state_dict tensor (reference key name, reference layout e.g. OIHW) as a DEVICE
 * fp32 pointer; it is copied/re-laid-out at cfb_net_prepare and need not outlive it. */
int      cfb_net_set_param(cfb_net* net, const char* name, const float* dev_ptr, int64_t numel);
int      cfb_net_prepare(cfb_net* net, void* stream);          /* errors if any key is missing */
int64_t  cfb_workspace_bytes(cfb_net* net, int32_t batch);     /* scratch needed for a forward at this batch; <0 on error */
/* engine of the dense convolutions / linears: 0 = auto (wgmma tensor cores wherever the shape allows, default),
 * 1 = fp32 CUDA-core implicit GEMM everywhere, 2 = wgmma only (unsupported shapes are an error) */
int      cfb_net_set_engine(cfb_net* net, int32_t engine);
/* Precision of the generator and Fuse_sft_block convs (the decoder: everything after the code lookup / quantizer except the
 * AttnBlocks' q,k,v / proj_out and conv_last): 0 = fp32 (default; split fp16 x3 operands, fp32 parity), 1 = fp16 (fp16
 * operands, one tensor-core product per k-step, fp32 accumulation and fp32 activations).  The encoder, the Transformer, the
 * quantizer and so logits, lq_feat and the code indices are the same in both.  fp16 needs engine 0 or 2 on an sm_90 device
 * (the forward raises otherwise).  Other values are an error.  Takes effect at the next forward; no re-prepare. */
int      cfb_net_set_precision(cfb_net* net, int32_t precision);
/* parity hook: after stage `name` ("enc.<i>", "gen.<i>", "fuse.<size>", "ft.<l>", "quant") of the next forwards, copy
 * that NHWC fp32 activation to dst (device, `capacity` floats).  dst = NULL removes the hook. */
int      cfb_net_capture(cfb_net* net, const char* stage, float* dst, int64_t capacity);
/* number of kernel launches the last forward on this net enqueued (bench.py "gpu_launches") */
int64_t  cfb_last_launch_count(cfb_net* net);

/* ---- CodeFormer.forward (codeformer_arch.py:223-280) ----
 * x [B,3,512,512] NCHW in [-1,1]; out [B,3,512,512] NCHW (unclamped; may be NULL when code_only);
 * logits [B,256,K]; lq_feat [B,256,16,16] NCHW; top_idx [B,256] int64 (may be NULL).
 * All DEVICE pointers.  `w` is the fidelity weight (branch w>0, :276). */
int cfb_codeformer_forward(cfb_net* net, const float* x, float* out, float* logits, float* lq_feat,
                           int64_t* top_idx, int32_t batch, float w, int32_t adain, int32_t code_only,
                           void* workspace, int64_t workspace_bytes, void* stream);
/* Per-face fidelity weights: the *_wv entry points take w_dev, a DEVICE float [batch] (one w per face, on `stream`), in place of
 * `w`.  Face i equals the scalar call on that face alone with w = w_dev[i], bit for bit; a face with w_dev[i] <= 0 or NaN gets
 * the skipped-fusion result of w <= 0.  The Fuse_sft_blocks run for every face whatever the values (their blend multiplies by
 * max(w, 0)), so in fp16 precision their operand range guard may also fail a batch whose faces all have w <= 0. */
int cfb_codeformer_forward_wv(cfb_net* net, const float* x, float* out, float* logits, float* lq_feat,
                              int64_t* top_idx, int32_t batch, const float* w_dev, int32_t adain, int32_t code_only,
                              void* workspace, int64_t workspace_bytes, void* stream);

/* Same call with HOST buffers (pinned recommended): H2D of x, forward, D2H of out/logits/lq_feat,
 * all on `stream`, then one stream synchronise.  dev_scratch must hold the device copies:
 * cfb_host_io_bytes(net,batch) bytes, in addition to the workspace. */
int64_t cfb_host_io_bytes(cfb_net* net, int32_t batch);
int cfb_codeformer_forward_host(cfb_net* net, const float* x_host, float* out_host, float* logits_host,
                                float* lq_feat_host, int32_t batch, float w, int32_t adain,
                                void* dev_scratch, int64_t dev_scratch_bytes,
                                void* workspace, int64_t workspace_bytes, void* stream);

/* f1 (SURVEY.md section 8f): the forward with the caller's image plumbing fused into the first and last conv.
 * faces_bgr / restored_bgr: DEVICE uint8 [batch,512,512,3] HWC BGR, i.e. face_helper.cropped_faces as they are
 * (inference_codeformer.py:197).  Replaces img2tensor(face/255.) + normalize(0.5,0.5) -> net(x,w,adain)[0] ->
 * tensor2img(rgb2bgr, min_max=(-1,1)).astype(uint8)   (inference_codeformer.py:199-213, basicsr/utils/img_util.py:9-35,38-94)
 * with the same fp32 arithmetic and rounding (round-half-even).  logits / lq_feat / top_idx are optional. */
int cfb_codeformer_forward_u8(cfb_net* net, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                              int64_t* top_idx, int32_t batch, float w, int32_t adain,
                              void* workspace, int64_t workspace_bytes, void* stream);
/* cfb_codeformer_forward_u8 for face inpainting (inference_inpainting.py:64-75; there w = 1, adain = 0 on the codebook-512,
 * 3-connect net): same arguments, launches and precision, but before the uint8 conversion every pixel where the normalised input
 * face sums to 3 over its channels (only (255,255,255)) takes the network's output and every other pixel keeps the input:
 * (1-mask)*input + mask*output in fp32, then tensor2img.  Restored faces are the script's save_face, byte for byte. */
int cfb_codeformer_inpaint_u8(cfb_net* net, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                              int64_t* top_idx, int32_t batch, float w, int32_t adain,
                              void* workspace, int64_t workspace_bytes, void* stream);
/* the two uint8 forwards with one w per face (w_dev: DEVICE float [batch], see cfb_codeformer_forward_wv) */
int cfb_codeformer_forward_u8_wv(cfb_net* net, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                                 int64_t* top_idx, int32_t batch, const float* w_dev, int32_t adain,
                                 void* workspace, int64_t workspace_bytes, void* stream);
int cfb_codeformer_inpaint_u8_wv(cfb_net* net, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                                 int64_t* top_idx, int32_t batch, const float* w_dev, int32_t adain,
                                 void* workspace, int64_t workspace_bytes, void* stream);
/* Fidelity sweep: `batch` faces, each at `k` fidelity weights, with one encoder / Transformer / code-lookup pass at batch
 * `batch` and the decoder at batch batch*k.  w_dev: DEVICE float [batch*k], face-major (w_dev[b*k + j] is face b's j-th
 * weight); restored_bgr: DEVICE uint8 [batch,k,512,512,3].  restored_bgr[b][j] equals cfb_codeformer_forward_u8_wv on face b
 * alone with w = w_dev[b*k + j], byte for byte (so also cfb_codeformer_forward_u8 with that w); the fp16 caveat of the *_wv
 * entry points applies.  logits / lq_feat / top_idx are optional and hold the batch-`batch` results.  No inpainting and no
 * code_only.  workspace >= cfb_sweep_workspace_bytes(net, batch, k) (<0 on error). */
int64_t cfb_sweep_workspace_bytes(cfb_net* net, int32_t batch, int32_t k);
int cfb_codeformer_sweep_u8(cfb_net* net, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                            int64_t* top_idx, int32_t batch, int32_t k, const float* w_dev, int32_t adain,
                            void* workspace, int64_t workspace_bytes, void* stream);
/* the same with HOST uint8 buffers (0.79 MB per face each way instead of 3.1 MB): H2D, forward, D2H, stream sync.
 * dev_scratch >= cfb_host_io_bytes(net, batch). */
int cfb_codeformer_restore_host(cfb_net* net, const uint8_t* faces_host, uint8_t* restored_host, int32_t batch, float w,
                                int32_t adain, void* dev_scratch, int64_t dev_scratch_bytes,
                                void* workspace, int64_t workspace_bytes, void* stream);
/* the plumbing alone (unit parity): uint8 HWC BGR [n,hw,3] <-> fp32 NCHW RGB [n,3,hw] in [-1,1] */
int cfb_u8_to_input(const uint8_t* img_bgr_hwc, float* x_nchw, int32_t n, int32_t hw, void* stream);
int cfb_output_to_u8(const float* x_nchw, uint8_t* img_bgr_hwc, int32_t n, int32_t hw, void* stream);
/* ---- VQAutoEncoder.forward (vqgan_arch.py:385-389) ----
 * out [B,3,512,512]; idx [B*256] int64; stats[4] = {codebook_loss, perplexity, mean_distance, 0};
 * min_encodings [B*256,K] one-hot fp32 or NULL (materialised only when asked). */
int cfb_vqae_forward(cfb_net* net, const float* x, float* out, int64_t* idx, float* stats,
                     float* min_encodings, int32_t batch,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* ---- Encoder.forward alone (vqgan_arch.py:269-273), for both network kinds: the generator, the fusion and the Transformer
 * never run, and the workspace is that of the encoder (cfb_encoder_workspace_bytes(net, n) for n ENCODED images; <0 on error).
 * The latent equals the one the fused forwards quantize (VQAutoEncoder) or return as lq_feat (CodeFormer), bit for bit.
 * cfb_encoder_forward: x [batch,3,S,S] NCHW in [-1,1] -> latent [batch,emb_dim,S/2^(n-1),S/2^(n-1)] NCHW. */
int64_t cfb_encoder_workspace_bytes(cfb_net* net, int32_t batch);
int cfb_encoder_forward(cfb_net* net, const float* x, float* latent, int32_t batch, void* workspace, int64_t workspace_bytes,
                        void* stream);
/* Latent codes of uint8 faces (scripts/generate_latent_gt.py): faces_bgr DEVICE uint8 [batch,S,S,3] HWC BGR, read with the
 * input arithmetic of cfb_codeformer_forward_u8.  The encoder runs once at batch + mirror images: images 0..batch-1 are the
 * faces, images batch + j (j < mirror <= batch) face j flipped left-right (cv2.flip(face, 1)), read mirrored by the first conv.
 * idx [(batch+mirror)*h*w] int64 gets the code selection of VectorQuantizer.forward on each latent -- the same entry that module
 * calls (cfb_vq_nearest_fast where cfb_vq_fast_supported, else cfb_vq_nearest) -- so the indices equal quantize(encoder(x)) of
 * the fp32 chain bit for bit.  latent [(batch+mirror),emb_dim,h,w] NCHW is optional.  Workspace: cfb_encoder_workspace_bytes(net,
 * batch + mirror). */
int cfb_latent_codes_u8(cfb_net* net, const uint8_t* faces_bgr, int64_t* idx, float* latent, int32_t batch, int32_t mirror,
                        void* workspace, int64_t workspace_bytes, void* stream);
/* CodeFormer.forward(code_only=True) from uint8 faces (codeformer_arch.py:247-249) with no restored-image buffer: logits
 * [batch,256,K] (required), lq_feat [batch,256,16,16] NCHW and top_idx [batch,256] int64 (the argmax of the logits) optional.
 * Equal, bit for bit, to cfb_codeformer_forward on the fp32 chain of the faces with code_only = 1.  Workspace: cfb_workspace_bytes. */
int cfb_codeformer_code_only_u8(cfb_net* net, const uint8_t* faces_bgr, float* logits, float* lq_feat, int64_t* top_idx,
                                int32_t batch, void* workspace, int64_t workspace_bytes, void* stream);
/* Code-prediction scores of CodeFormer's stage 2 (codeformer_idx_model.py:100-115), per image, in float64: logits [batch,tokens,
 * codes], top_idx [batch,tokens] int64 (the net's argmax, not recomputed), gt_idx [batch,tokens] int64, lq_feat_nhwc
 * [batch,tokens,dim], codebook [codes,dim]; all DEVICE.  scores [batch][3] double: the mean over tokens of
 * logsumexp(logits_t) - logits_t[gt_t], the number of tokens with top_idx == gt, and the mean over tokens x dim of
 * (codebook[gt_t] - lq_feat_t)^2.  Every sum runs in a fixed order that does not depend on the batch.  A NaN logit makes that
 * image's cross-entropy NaN.  A gt index outside [0, codes) is never read: that image's three scores are NaN and the status word
 * reports it (cfb_check_async_status, or the next forward). */
int cfb_code_scores(const float* logits, const int64_t* top_idx, const int64_t* gt_idx, const float* lq_feat_nhwc,
                    const float* codebook, int32_t batch, int32_t tokens, int32_t codes, int32_t dim, double* scores, void* stream);

/* ---- VectorQuantizer.forward (vqgan_arch.py:33-70), standalone (config 3 microbench) ----
 * z [B,D,H,W] NCHW, codebook [K,D]; z_q [B,D,H,W] NCHW (= z + (E[idx]-z), :57); idx [B*H*W] int64;
 * stats[4] as above; min_encodings optional.  workspace >= cfb_vq_workspace_bytes. */
int64_t cfb_vq_workspace_bytes(int32_t batch, int32_t hw, int32_t dim, int32_t codes);
int cfb_vq_nearest(const float* z, const float* codebook, int32_t batch, int32_t h, int32_t w,
                   int32_t dim, int32_t codes, float beta, float* z_q, int64_t* idx, float* stats,
                   float* min_encodings, void* workspace, int64_t workspace_bytes, void* stream);

/* VectorQuantizer.forward, fused path (vqgan_arch.py:33-70; BASELINE configs[2]): the codebook is split for the tensor cores and
 * its |e|^2 computed ONCE (cfb_vq_prepare, redo when the embedding changes).  A call is then ONE kernel on the caller's NCHW
 * tensors (vq_fused_kernel: z tile -> shared-memory operand planes, codebook through TMA, distances on wgmma with the argmin
 * taken from the register accumulators, gather + straight-through z_q + loss, statistics by the last CTA; the prepared buffer
 * also holds the kernel's self-cleaning histogram, so calls sharing one prepared buffer must not overlap).  The [tokens, codes]
 * matrix is never stored.  Same outputs as cfb_vq_nearest.
 * cfb_vq_fast_supported: sm_90, 16x16-style latents (h*w % 128 == 0, exact tensor-core tiles), dim % 64 == 0 and
 * 64 <= dim <= 256, codes % 64 == 0 and codes <= 1024; other shapes go to cfb_vq_nearest. */
int32_t cfb_vq_fast_supported(int32_t batch, int32_t h, int32_t w, int32_t dim, int32_t codes);
int64_t cfb_vq_prepared_bytes(int32_t codes, int32_t dim);
int     cfb_vq_prepare(const float* codebook, int32_t codes, int32_t dim, void* prepared, int64_t prepared_bytes, void* stream);
int64_t cfb_vq_fast_workspace_bytes(int32_t batch, int32_t hw, int32_t dim, int32_t codes);
int     cfb_vq_nearest_fast(const float* z, const float* codebook, const void* prepared, int32_t batch, int32_t h, int32_t w,
                            int32_t dim, int32_t codes, float beta, float* z_q, int64_t* idx, float* stats, float* min_encodings,
                            void* workspace, int64_t workspace_bytes, void* stream);
/* ---- VectorQuantizer.get_codebook_feat (vqgan_arch.py:72-84) ---- idx [n] int64 -> z_q [B,D,H,W] NCHW */
int cfb_codebook_lookup(const int64_t* idx, const float* codebook, int32_t batch, int32_t h, int32_t w,
                        int32_t dim, int32_t codes, float* z_q, void* stream);

/* ---- per-kernel entry points (unit-parity tests; NHWC fp32 device tensors) ---- */
/* conv2d: in [N,H,W,Cin] NHWC, weight OIHW [Cout,Cin,k,k] (reference layout), bias [Cout] or NULL.
 * mode: 0 = 'same' k=1|3 stride 1 (nn.Conv2d padding=k/2); 1 = Downsample (pad right/bottom 1, 3x3 s2 p0,
 * vqgan_arch.py:122-126); 2 = Upsample (nearest x2 then 3x3 p1, vqgan_arch.py:134-138).
 * in_scale/in_shift [N,Cin] optional fused per-sample affine (GroupNorm), in_act 0|1(SiLU);
 * residual [N,Ho,Wo,Cout] optional; out_act 0 | 1 LeakyReLU(0.2) | 2 GELU(erf).
 * engine: 0 = auto, 1 = fp32 CUDA-core implicit GEMM, 2 = wgmma split-fp16 tensor-core implicit GEMM. */
int cfb_conv2d_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out,
                    int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t mode,
                    const float* in_scale, const float* in_shift, int32_t in_act,
                    const float* residual, int32_t out_act, int32_t engine,
                    void* workspace, int64_t workspace_bytes, void* stream);
int64_t cfb_conv2d_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t mode);
/* GroupNorm(32,C,eps) statistics folded with the affine: scale[n,c] = rstd*gamma, shift[n,c] = beta - mean*rstd*gamma
 * (vqgan_arch.py:14-15).  x [N,HW,C] NHWC.  workspace >= cfb_gn_workspace_bytes. */
int64_t cfb_gn_workspace_bytes(int32_t n, int32_t hw, int32_t c);
int cfb_group_norm_coef(const float* x, const float* gamma, const float* beta, float* scale, float* shift,
                        int32_t n, int32_t hw, int32_t c, int32_t groups, float eps,
                        void* workspace, int64_t workspace_bytes, void* stream);
/* y = act(x*scale[n,c]+shift[n,c]) materialised (NHWC) */
int cfb_affine_act(const float* x, const float* scale, const float* shift, float* y,
                   int32_t n, int32_t hw, int32_t c, int32_t act, void* stream);
/* softmax(q k^T * scale) v for `heads` heads of width d packed in rows of pitch (in floats); S tokens per batch */
int cfb_attention(const float* q, const float* k, const float* v, float* out,
                  int32_t batch, int32_t tokens, int32_t heads, int32_t d,
                  int32_t q_pitch, int32_t k_pitch, int32_t v_pitch, int32_t o_pitch, float scale, void* stream);
/* LayerNorm over the last dim (eps 1e-5); y2 (optional) = y + pos[t % pos_rows] */
int cfb_layer_norm(const float* x, const float* gamma, const float* beta, float* y, float* y2,
                   const float* pos, int32_t pos_rows, int32_t rows, int32_t c, void* stream);
/* AdaIN of codeformer_arch.py:29-43 on NHWC [B,HW,C] */
int cfb_adain_nhwc(const float* content, const float* style, float* out, int32_t batch, int32_t hw, int32_t c, void* stream);
/* diagnostics / bench: average device time (CUDA events on `stream`) of the wgmma conv KERNEL alone over `reps` launches
 * (bench.py roofline).  With in_scale/in_shift (per-(n,cin) GroupNorm affine) and in_act the kernel is the one the forward
 * launches for a GroupNorm+SiLU consumer: the fused-operand-transform variant reading the fp32 activation (all-in, no prep
 * pass exists); without them the weights are split and the raw operand planes prepared once outside the timed region. */
int cfb_debug_time_conv(const float* in, const float* weight_oihw, float* out, int32_t n, int32_t h, int32_t w, int32_t cin,
                        int32_t cout, int32_t ksize, int32_t mode, int32_t reps, void* workspace, int64_t workspace_bytes,
                        void* stream, const float* in_scale, const float* in_shift, int32_t in_act, float* ms_per_launch);
/* diagnostics / tests: one conv on the wgmma engine with every epilogue of the forward exposed.  mode 0 ('same', 3x3) | 2
 * (Upsample); xform 1 = fused operand transform (in_scale/in_shift optional: null = plain hi/lo split of the raw values), with
 * in2 != null channels [cin1, cin) read from in2 (torch.cat of Fuse_sft_block); residual, SFT (out = sft_dec + sft_w *
 * (sft_dec * sft_scale + conv)), out_planes (fp16 hi | lo planes of out, each align1024(n*Ho*Wo*cout*2) bytes) and gn_part
 * (GroupNorm(32) partials, per 32-pixel slot and group the (mean, M2) of its values: 4 * 32 * 2 floats per 128-pixel tile)
 * optional.  *tile_n receives the tile of the launched
 * kernel: 128 (128 pixels x 128 channels), 64 (128 pixels x 64 channels, pixel-major) or -64 (128 pixels x 64 channels,
 * channel-major: computed transposed with the weights as the wgmma A operand).
 * workspace >= cfb_conv2d_workspace_bytes(n, h, w, cin, cout, 3, mode). */
int cfb_debug_conv_tc(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias, float* out,
                      int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                      const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                      const float* sft_dec, const float* sft_scale, float sft_w, void* out_planes, float* gn_part,
                      void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n);
/* The same with the kernel size, the activation epilogue and the operand precision of cfb_net_set_precision: ksize 3, or 1
 * (mode 0, xform 0: the per-tap engine on raw planes, *tile_n = 64); out_act 0 none | 1 LeakyReLU(0.2) (Fuse_sft_block's
 * scale.0 / shift.0); precision 0 fp32 (split; == cfb_debug_conv_tc with out_act 0), 1 fp16 (single pass; built for the
 * 128-wide and channel-major 3x3 / Upsample tiles and the 1x1 conv -- other forms are an error).
 * workspace >= cfb_conv2d_workspace_bytes(n, h, w, cin, cout, ksize, mode). */
int cfb_debug_conv_tc_prec(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias,
                           float* out, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                           const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                           const float* sft_dec, const float* sft_scale, float sft_w, void* out_planes, float* gn_part,
                           void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n, int32_t ksize,
                           int32_t out_act, int32_t precision);
/* cfb_debug_conv_tc_prec with one SFT weight per image: sft_wv (DEVICE float [n], required with sft_dec) in place of sft_w;
 * image i blends with max(sft_wv[i], 0) (NaN: 0). */
int cfb_debug_conv_tc_prec_wv(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias,
                              float* out, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                              const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                              const float* sft_dec, const float* sft_scale, const float* sft_wv, void* out_planes,
                              float* gn_part, void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n,
                              int32_t ksize, int32_t out_act, int32_t precision);
/* diagnostics / tests: the attention core of the forward on the wgmma engine (bmm_tc: scores, softmax256_planes, bmm_tc: P v)
 * from fp32 inputs.  q, k, v, out: [n][256 tokens][heads * d] (the 16x16 latent), out = softmax(q_h k_h^T d^-1/2) v_h per head h
 * (channels [h*d, (h+1)*d)); out_planes (optional): fp16 hi | lo planes of out, each align1024(n*256*heads*d*2) bytes.  heads 1
 * is the AttnBlock core (d = C), heads > 1 the Transformer's nn.MultiheadAttention core; d a multiple of 64.  q, k and v are
 * split into operand planes as their producing convs write them.  workspace >= cfb_debug_bmm_tc_workspace_bytes(n, heads, d). */
int64_t cfb_debug_bmm_tc_workspace_bytes(int32_t n, int32_t heads, int32_t d);
int cfb_debug_bmm_tc(const float* q, const float* k, const float* v, float* out, void* out_planes, int32_t n, int32_t heads,
                     int32_t d, void* workspace, int64_t workspace_bytes, void* stream);
/* diagnostics / tests: the LayerNorm of the forward on the wgmma engine (cfb_layer_norm's arithmetic, eps 1e-5), which writes
 * its outputs only as fp16 operand planes: y_planes (optional) of y, y2_planes (optional; needs pos, pos_rows > 0) of
 * y + pos[t % pos_rows].  Each is hi | lo, hi = fp16(v), lo = fp16(v - hi), each plane align1024(rows * c * 2) bytes, as
 * cfb_debug_bmm_tc's out_planes.  A value past 65504 sets the fp16 overflow bit of the status word (cfb_check_async_status). */
int cfb_debug_layer_norm_planes(const float* x, const float* gamma, const float* beta, void* y_planes, void* y2_planes,
                                const float* pos, int32_t pos_rows, int32_t rows, int32_t c, void* stream);
/* diagnostics / tests: the code lookup of the forward (codeformer_arch.py:257-259): idx[t] (optional) = the first maximum of
 * logits[t] ([T][K]), quant[t] (optional, [T][D]) = codebook[idx[t]] ([K][D]; D a multiple of 4).  NaN logits never win; a row
 * without a maximum (all NaN or -inf) gives index 0. */
int cfb_debug_code_lookup(const float* logits, const float* codebook, int64_t* idx, float* quant, int32_t T, int32_t K,
                          int32_t D, void* stream);
/* diagnostics / tests: the GroupNorm(32) finalize of the forward on partials in the layout cfb_debug_conv_tc writes (slots of
 * 32 pixels, [n][slots][32 groups][2] floats): scale[n,c] = rstd*gamma, shift[n,c] = beta - mean*rstd*gamma over hw pixels
 * of c channels.  The workspace (>= cfb_debug_gn_partials_workspace_bytes) holds the split-finalize scratch and the ticket
 * counters; the call zeroes the counters.  cfb_debug_gn_cat_partials merges the partials of two sources of c channels each
 * into those of torch.cat([a, b], 1) (2c channels, the same slots), as Fuse_sft_block's GroupNorm takes them. */
int64_t cfb_debug_gn_partials_workspace_bytes(int32_t n, int32_t slots);
int cfb_debug_gn_coef_from_partials(const float* part, int32_t slots, const float* gamma, const float* beta, float* scale,
                                    float* shift, int32_t n, int32_t hw, int32_t c, float eps, void* workspace,
                                    int64_t workspace_bytes, void* stream);
int cfb_debug_gn_cat_partials(const float* a_part, const float* b_part, float* out_part, int64_t total_slots, int32_t c,
                              void* stream);
/* ---- RRDBNet (SURVEY.md section 8 row f4): the upsampler behind RealESRGANer.enhance ----
 * /root/reference/basicsr/archs/rrdbnet_arch.py:67-120 (constructor :86, forward :103-119); the caller's tiling loop
 * (basicsr/utils/realesrgan_utils.py:100-175) stays in Python (codeformer_b200/upsampler.py).
 * Parameters are the reference's state-dict names (conv_first, body.{i}.rdb{1,2,3}.conv{1..5}, conv_body, conv_up1, conv_up2,
 * conv_hr, conv_last; .weight OIHW / .bias).  x: [batch, num_in_ch, h, w] fp32 NCHW, any h, w (multiples of 2 for scale 2, of 4
 * for scale 1: pixel_unshuffle); out: [batch, num_out_ch, h*scale, w*scale].  Built for num_feat = 64, num_grow_ch = 32. */
typedef struct cfb_rrdb cfb_rrdb;
cfb_rrdb* cfb_rrdb_create(int32_t num_in_ch, int32_t num_out_ch, int32_t scale, int32_t num_feat, int32_t num_block, int32_t num_grow_ch);
void      cfb_rrdb_destroy(cfb_rrdb* net);
int       cfb_rrdb_set_param(cfb_rrdb* net, const char* name, const float* dev_ptr, int64_t numel);
int       cfb_rrdb_prepare(cfb_rrdb* net, void* stream);
/* Precision of the 3x3 / Upsample convs (every conv except conv_first and conv_last, which stay fp32): 0 = fp32 (default;
 * split fp16 x3 operands, fp32 parity), 1 = fp16 (the reference's half=True: fp16 operands, one tensor-core product per
 * k-step, fp32 accumulation and fp32 activations).  Other values are an error.  Takes effect at the next forward; no
 * re-prepare. */
int       cfb_rrdb_set_precision(cfb_rrdb* net, int32_t precision);
int64_t   cfb_rrdb_workspace_bytes(cfb_rrdb* net, int32_t batch, int32_t h, int32_t w);
int       cfb_rrdb_forward(cfb_rrdb* net, const float* x, float* out, int32_t batch, int32_t h, int32_t w,
                           void* workspace, int64_t workspace_bytes, void* stream);
/* RealESRGANer's pre_process + tile_process + post_process and its uint8 conversion (realesrgan_utils.py:71-210) for tiles of
 * equal size, from uint8 HWC BGR images to uint8 HWC BGR images, as one forward at batch num_tiles.
 * images_bgr: [num_images, img_h, img_w, 3] on the device; the padded image is img_h + pre_pad (+ the reflect pad to the
 * pixel-unshuffle multiple) high, likewise wide; each pad must be smaller than the dimension it reflects.
 * tiles: host int32 [num_tiles][9] = image, in_y, in_x (window origin in the padded image), crop_y, crop_x, crop_h, crop_w
 * (kept rectangle of the tile's tile_h*scale x tile_w*scale output), out_y, out_x (its place in the output); tile_h and tile_w
 * must be multiples of the pixel-unshuffle factor.  out_bgr: [num_images, img_h*scale, img_w*scale, 3]; pixels past it (the
 * pads) are discarded.  The input value is float32 u8 / 255, the output clamp(v, 0, 1) * 255 rounded half to even.  Built for
 * 3 channels in and out; honours cfb_rrdb_set_precision; workspace: cfb_rrdb_workspace_bytes(net, num_tiles, tile_h, tile_w).
 * The table travels in the launch parameters: no host synchronisation. */
int       cfb_rrdb_forward_u8_tiles(cfb_rrdb* net, const uint8_t* images_bgr, int32_t num_images, int32_t img_h, int32_t img_w,
                                    int32_t pre_pad, const int32_t* tiles, int32_t num_tiles, int32_t tile_h, int32_t tile_w,
                                    uint8_t* out_bgr, void* workspace, int64_t workspace_bytes, void* stream);
/* cfb_rrdb_forward_u8_tiles for the other images RealESRGANer.enhance takes (realesrgan_utils.py:190-243): images_bgr of element
 * type in_kind (uint8, uint16, float32 or float64), out_bgr of out_kind (CFB_IMG_U8 or CFB_IMG_U16); the same tile table, pads,
 * checks and workspace.  Per image, as the reference: img.astype(np.float32) (float64 rounded to nearest first),
 * max_range = 65535 if its float32 maximum exceeds 256 else 255 (a NaN makes numpy's maximum NaN: 255), the input value
 * float32 v / max_range (an IEEE division), the output clamp(v, 0, 1) * max_range in float32 rounded half to even (saturated
 * to 255 in a uint8 canvas).  max_range: device int32 [num_images], written by the call (a device reduction over every image,
 * before the forward; no host synchronisation) when num_tiles > 0 -- the caller reads it back to pick each result's dtype
 * (uint16 where it is 65535).  num_images <= 65535. */
#define CFB_IMG_U8  0
#define CFB_IMG_U16 1
#define CFB_IMG_F32 2
#define CFB_IMG_F64 3
int       cfb_rrdb_forward_tiles(cfb_rrdb* net, const void* images_bgr, int32_t in_kind, int32_t num_images, int32_t img_h,
                                 int32_t img_w, int32_t pre_pad, const int32_t* tiles, int32_t num_tiles, int32_t tile_h, int32_t tile_w,
                                 void* out_bgr, int32_t out_kind, int32_t* max_range, void* workspace, int64_t workspace_bytes,
                                 void* stream);

/* ---- ParseNet (SURVEY.md section 8 row f3): face parsing of the restored face for the paste-back blend ----
 * /root/reference/facelib/parsing/parsenet.py:140-194; built by init_parsing_model('parsenet') as ParseNet(in_size=512,
 * out_size=512, parsing_ch=19) (facelib/parsing/__init__.py:13) and called at facelib/utils/face_restoration_helper.py:457-462.
 * Parameters are the reference's state-dict names (encoder.0.conv2d, {encoder,body,decoder}.{i}.{shortcut_func,conv1,conv2}.
 * conv2d.{weight,bias}, ...norm.norm.{weight,bias,running_mean,running_var}); eval-mode BatchNorm is folded at prepare.
 * x: [batch,3,h,w] fp32 NCHW in [-1,1]; out_mask: [batch, parsing_ch, h, w] logits; out_img (optional): [batch,3,h,w].
 * cfb_parse_argmax: classes = out_mask.argmax(1) (first maximum) and/or the caller's 0/255 face mask of
 * face_restoration_helper.py:463-468 (MASK_COLORMAP), both uint8 [batch, h*w]. */
typedef struct cfb_parsenet cfb_parsenet;
cfb_parsenet* cfb_parsenet_create(int32_t in_size, int32_t out_size, int32_t min_feat_size, int32_t base_ch, int32_t parsing_ch,
                                  int32_t res_depth, int32_t ch_min, int32_t ch_max);
void      cfb_parsenet_destroy(cfb_parsenet* net);
int       cfb_parsenet_set_param(cfb_parsenet* net, const char* name, const float* dev_ptr, int64_t numel);
int       cfb_parsenet_prepare(cfb_parsenet* net, void* stream);
int64_t   cfb_parsenet_workspace_bytes(cfb_parsenet* net, int32_t batch, int32_t h, int32_t w);
int       cfb_parsenet_forward(cfb_parsenet* net, const float* x, float* out_mask, float* out_img, int32_t batch, int32_t h, int32_t w,
                               void* workspace, int64_t workspace_bytes, void* stream);
int       cfb_parse_argmax(const float* logits_nchw, uint8_t* classes, uint8_t* mask, int32_t batch, int32_t channels, int64_t hw,
                           void* stream);
/* Precision of the GEN convs (shortcut, conv1 and conv2 of every encoder, body and decoder block; encoder.0 and the two heads
 * stay fp32 in both): 0 = fp32 (default; split fp16 x3 operands, fp32 parity), 1 = fp16 (fp16 operands, one tensor-core
 * product per k-step, fp32 accumulation and fp32 activations).  Other values are an error.  Takes effect at the next forward;
 * no re-prepare.  Honoured by cfb_parsenet_forward and cfb_parsenet_masks_u8. */
int       cfb_parsenet_set_precision(cfb_parsenet* net, int32_t precision);
/* The parse masks straight from uint8 faces: faces_bgr [batch, h, w, 3] HWC BGR (the value cfb_u8_to_input makes of them)
 * -> classes and / or mask, uint8 [batch, h, w] (either may be NULL, not both), byte-equal to cfb_u8_to_input +
 * cfb_parsenet_forward + cfb_parse_argmax.  out_img_conv is not run.  workspace: cfb_parsenet_workspace_bytes(net, batch,
 * h, w). */
int       cfb_parsenet_masks_u8(cfb_parsenet* net, const uint8_t* faces_bgr, uint8_t* classes, uint8_t* mask, int32_t batch,
                                int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);

/* One 3x3 conv of the generalised fused-transform engine (the building block of RRDBNet / ParseNet; test entry point).
 * in: NHWC buffer of in_pitch channels per pixel, channels [0, cin) are read; any h x w.  upsample != 0: nearest x2 first.
 * pad_mode 0 zero / 1 reflect / 2 replicate (of the low-resolution tensor when upsampling).  subsample != 0: stride 2 (the
 * even output positions of the stride-1 result; h, w even).  out: NHWC buffer of out_pitch channels, the cout real channels
 * go to [out_c0, out_c0 + cout).  out = act(conv + bias + residual) * post_scale + residual2 (post only with residual2);
 * out_act 0 none / 1 LeakyReLU(0.2) / 3 ReLU / 4 SiLU. */
int64_t cfb_conv2d_gen_workspace_bytes(int32_t cin, int32_t cout);
int cfb_conv2d_gen_nhwc(const float* in, int32_t in_pitch, const float* weight_oihw, const float* bias, float* out,
                        int32_t out_pitch, int32_t out_c0, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout,
                        int32_t upsample, int32_t pad_mode, int32_t subsample, int32_t out_act, const float* residual,
                        int32_t res_pitch, const float* residual2, int32_t res2_pitch, float post_scale, void* workspace,
                        int64_t workspace_bytes, void* stream);
/* The same with the operand precision of cfb_rrdb_set_precision: 0 fp32 (split; == cfb_conv2d_gen_nhwc), 1 fp16 (out_act 4,
 * SiLU, is not built for it). */
int cfb_conv2d_gen_nhwc_prec(const float* in, int32_t in_pitch, const float* weight_oihw, const float* bias, float* out,
                             int32_t out_pitch, int32_t out_c0, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout,
                             int32_t upsample, int32_t pad_mode, int32_t subsample, int32_t out_act, const float* residual,
                             int32_t res_pitch, const float* residual2, int32_t res2_pitch, float post_scale, void* workspace,
                             int64_t workspace_bytes, void* stream, int32_t precision);

/* One 1x1 or 3x3 conv of the per-tap engine on any h x w (test entry point for the detector's conv forms).  stride 2 computes
 * only the output positions, ceil(h/2) x ceil(w/2): 3x3 with padding 1, 1x1 without.  in / out / residual NHWC, cin and cout
 * multiples of 64.  out = act(conv + bias + residual), act 0 none / 3 ReLU. */
int64_t cfb_conv2d_pertap_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t stride);
int cfb_conv2d_pertap_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h, int32_t w,
                           int32_t cin, int32_t cout, int32_t ksize, int32_t stride, int32_t out_act, const float* residual,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* The same per-tap engine with the YOLOv5 epilogue (test entry point): 1x1 (stride 1 or 2) or 3x3 stride-2 pad-1 conv,
 * out_act 0 none / 4 SiLU, written into channels [out_c0, out_c0 + cout) of an NHWC buffer with out_pitch channels per pixel
 * (multiples of 4); the other channels are left as they are.  Workspace: cfb_conv2d_pertap_workspace_bytes. */
int cfb_conv2d_pertap_slice_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                                 int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t stride, int32_t out_act,
                                 int32_t out_pitch, int32_t out_c0, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- RetinaFace-ResNet50 face detector (facelib/detection/retinaface; detection.cu + the conv engine) ----
 * Parameters by the reference's state-dict names (BatchNorm folded at prepare).  forward: x fp32 NCHW [batch,3,h,w] (the
 * mean-subtracted image) -> loc [batch,P,4], conf [batch,P,2] (softmaxed), landms [batch,P,10], P = cfb_retinaface_priors(h, w).
 * forward_u8: uint8 HWC BGR images [batch,h,w,3] with the (104,117,123) mean subtraction fused.
 * candidates: per image, the rows [x1,y1,x2,y2,score,10 landmark coordinates] (pixels) of the priors whose score is
 * > conf_threshold, in prior order, into rows [batch,P,15]; counts [batch] (device int32). */
typedef struct cfb_retinaface cfb_retinaface;
int64_t   cfb_retinaface_priors(int32_t h, int32_t w);
cfb_retinaface* cfb_retinaface_create(void);
void      cfb_retinaface_destroy(cfb_retinaface* net);
int       cfb_retinaface_set_param(cfb_retinaface* net, const char* name, const float* dev_ptr, int64_t numel);
int       cfb_retinaface_prepare(cfb_retinaface* net, void* stream);
int64_t   cfb_retinaface_workspace_bytes(cfb_retinaface* net, int32_t batch, int32_t h, int32_t w);
int       cfb_retinaface_forward(cfb_retinaface* net, const float* x_nchw, float* loc, float* conf, float* landms, int32_t batch,
                                 int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int       cfb_retinaface_forward_u8(cfb_retinaface* net, const uint8_t* img_bgr_hwc, float* loc, float* conf, float* landms,
                                    int32_t batch, int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int       cfb_retinaface_candidates(const float* loc, const float* conf, const float* landms, int32_t batch, int32_t h, int32_t w,
                                    float conf_threshold, float* rows, int32_t* counts, void* stream);

/* ---- BiSeNet(num_class) face parser (facelib/parsing/bisenet.py; bisenet.cu + the conv engine) ----
 * Parameters by the reference's state-dict names (BatchNorm folded at prepare), 1 <= num_class <= 64.  h and w must be
 * multiples of 32.  forward: x fp32 NCHW [batch,3,h,w] -> out, out16, out32, each fp32 NCHW [batch,num_class,h,w].
 * masks_u8: uint8 HWC BGR faces [batch,h,w,3] (the normalisation of cfb_u8_to_input fused) -> classes = out.argmax(dim=1) and
 * the 0/255 MASK_COLORMAP mask, uint8 [batch,h,w] each (either may be NULL), byte-equal to cfb_u8_to_input + forward +
 * cfb_parse_argmax; out16 / out32 are not computed.  Workspace (both): cfb_bisenet_workspace_bytes.
 * cfb_debug_bisenet_bilinear: NHWC [n,h,w,pitch] (first c channels) -> NCHW [n,c,out_h,out_w], bilinear, align_corners=True.
 * cfb_debug_bisenet_attention: mean [n,c] of NHWC feat [n,hw,c], att = act2(w2 act1(w1 mean + b1) + b2) (w2 NULL: one layer),
 * weights [cout][cin], act 0 none / 1 ReLU / 2 sigmoid, one CTA per image. */
typedef struct cfb_bisenet cfb_bisenet;
cfb_bisenet* cfb_bisenet_create(int32_t num_class);
void         cfb_bisenet_destroy(cfb_bisenet* net);
int          cfb_bisenet_set_param(cfb_bisenet* net, const char* name, const float* dev_ptr, int64_t numel);
int          cfb_bisenet_prepare(cfb_bisenet* net, void* stream);
int64_t      cfb_bisenet_workspace_bytes(cfb_bisenet* net, int32_t batch, int32_t h, int32_t w);
int          cfb_bisenet_forward(cfb_bisenet* net, const float* x_nchw, float* out, float* out16, float* out32, int32_t batch,
                                 int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int          cfb_bisenet_masks_u8(cfb_bisenet* net, const uint8_t* faces_bgr, uint8_t* classes, uint8_t* mask, int32_t batch,
                                  int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int          cfb_debug_bisenet_bilinear(const float* in_nhwc, int32_t pitch, int32_t n, int32_t h, int32_t w, int32_t c,
                                        float* out_nchw, int32_t out_h, int32_t out_w, void* stream);
int          cfb_debug_bisenet_attention(const float* feat_nhwc, int32_t n, int32_t hw, int32_t c, const float* w1, const float* b1,
                                         int32_t c1, int32_t act1, const float* w2, const float* b2, int32_t c2, int32_t act2,
                                         float* mean, float* att, void* stream);

/* ---- ResNetArcFace('IRBlock', layers, use_se=False) identity embeddings (basicsr/archs/arcface_arch.py; arcface.cu + the
 * conv engine) ----
 * create: the four block counts of `layers` (each >= 1).  Parameters by the reference's state-dict names (BatchNorm folded at
 * prepare, the PReLU slopes read there).  forward: x fp32 [batch,1,128,128] (the gray identity input) -> emb [batch,512].
 * forward_u8: uint8 HWC BGR faces [batch,512,512,3]; img2tensor(face / 255.) + normalize(0.5, 0.5), the gray conversion and the
 * bilinear resize to 128 x 128 of gray_resize_for_identity are fused into the stem, and the result equals those steps as
 * separate fp32 device passes followed by forward, bit for bit.  Workspace: cfb_arcface_workspace_bytes(net, batch).
 * debug_conv (test entry point): one conv of the network's forms on NHWC fp32 -- 3x3 stride 1 on the generalised engine, with
 * the optional per-(image, channel) input affine in_scale / in_shift [n][cin] (no activation; zero padding outside the image),
 * or 1x1 / 3x3 stride 2 on the per-tap engine; out_act 0 none / 5 PReLU (prelu_slope), optional residual added before it.
 * Workspace: cfb_conv2d_gen_workspace_bytes(cin, cout) for 3x3 stride 1, cfb_conv2d_pertap_workspace_bytes otherwise. */
typedef struct cfb_arcface cfb_arcface;
cfb_arcface* cfb_arcface_create(int32_t l1, int32_t l2, int32_t l3, int32_t l4);
void         cfb_arcface_destroy(cfb_arcface* net);
int          cfb_arcface_set_param(cfb_arcface* net, const char* name, const float* dev_ptr, int64_t numel);
int          cfb_arcface_prepare(cfb_arcface* net, void* stream);
int64_t      cfb_arcface_workspace_bytes(cfb_arcface* net, int32_t batch);
int          cfb_arcface_forward(cfb_arcface* net, const float* x, float* emb, int32_t batch, void* workspace, int64_t workspace_bytes,
                                 void* stream);
int          cfb_arcface_forward_u8(cfb_arcface* net, const uint8_t* faces_bgr_hwc, float* emb, int32_t batch, void* workspace,
                                    int64_t workspace_bytes, void* stream);
int          cfb_debug_arcface_conv(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                                    int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t stride, const float* in_scale,
                                    const float* in_shift, int32_t out_act, float prelu_slope, const float* residual,
                                    void* workspace, int64_t workspace_bytes, void* stream);

/* ---- LPIPS(net='vgg', version='0.1') perceptual distance (lpips 0.1; the perceptual term of basicsr's LPIPSLoss; lpips.cu +
 * the conv engine) ----
 * Parameters by lpips' state-dict names: scaling_layer.shift / .scale [3], net.slice<s>.<i>.weight / .bias (torchvision
 * vgg16().features index i), lin<k>.model.1.weight [C_k].  A launch holds `batch` groups of one reference and `group` (>= 1)
 * candidates: ref [batch], cand [batch * group] (candidate j of group q at q * group + j); pair p = q * group + j.  h, w >= 16.
 * forward: fp32 NCHW RGB images; xform = flags applied to every element before the ScalingLayer, in this order: 2 range_norm
 *   (x + 1) / 2, 4 input_norm (x - [0.485, 0.456, 0.406]) / [0.229, 0.224, 0.225], 1 normalize 2x - 1 (each a torch fp32 op).
 * forward_u8: uint8 HWC BGR images; convention 0 'lpips' (im2tensor: u / 127.5 - 1) or 1 'codeformer' (float32(u / 255.),
 *   normalize(0.5, 0.5), then LPIPSLoss's range_norm and input_norm), through the table cfb_lpips_u8_table gives; it equals
 *   forward on those transformed images bit for bit.
 * Outputs: val [P] float32 (the sum over the five layers, in order) and, when per_layer is set, per_layer [P][5].  Results do
 * not depend on the batch or the group size.  Workspace: cfb_lpips_workspace_bytes(net, batch, h, w, group); it grows with
 * batch * (1 + group) * h * w * 512 bytes (two relu1 maps).
 * u8_table (host only): the [3][256] stem inputs of a convention by RGB channel, for ScalingLayer shift / scale [3].
 * debug_stem (test entry point): conv1_1 + ReLU of the prepared net -> NHWC [batch * (1 + group), h, w, 64] in the launch's
 *   image order; u8 selects the input form, mode is xform (fp32) or the convention (uint8).
 * debug_head (test entry point): the head-and-pool pass of one layer on NHWC feat [batch * (1 + group), h, w, c] (c 64, 128,
 *   256 or 512) with lin [c]: pooled (optional) [batch * (1 + group), h / 2, w / 2, c], res [P] the layer's values.  Workspace:
 *   cfb_debug_lpips_head_workspace_bytes. */
typedef struct cfb_lpips cfb_lpips;
cfb_lpips* cfb_lpips_create(void);
void       cfb_lpips_destroy(cfb_lpips* net);
int        cfb_lpips_set_param(cfb_lpips* net, const char* name, const float* dev_ptr, int64_t numel);
int        cfb_lpips_prepare(cfb_lpips* net, void* stream);
int64_t    cfb_lpips_workspace_bytes(cfb_lpips* net, int32_t batch, int32_t h, int32_t w, int32_t group);
int        cfb_lpips_forward(cfb_lpips* net, const float* ref_nchw, const float* cand_nchw, int32_t batch, int32_t h, int32_t w,
                             int32_t group, int32_t xform, float* val, float* per_layer, void* workspace, int64_t workspace_bytes,
                             void* stream);
int        cfb_lpips_forward_u8(cfb_lpips* net, const uint8_t* ref_bgr, const uint8_t* cand_bgr, int32_t batch, int32_t h, int32_t w,
                                int32_t group, int32_t convention, float* val, float* per_layer, void* workspace,
                                int64_t workspace_bytes, void* stream);
int        cfb_lpips_u8_table(int32_t convention, const float* shift, const float* scale, float* table);
int        cfb_debug_lpips_stem(cfb_lpips* net, const void* ref, const void* cand, int32_t u8, int32_t mode, float* out, int32_t batch,
                                int32_t h, int32_t w, int32_t group, void* stream);
int64_t    cfb_debug_lpips_head_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t group);
int        cfb_debug_lpips_head(const float* feat, const float* lin, float* pooled, float* res, int32_t batch, int32_t h, int32_t w,
                                int32_t group, int32_t c, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- InceptionV3 for the Fréchet Inception Distance (pytorch-fid InceptionV3(output_blocks=[3]), use_fid_inception=True;
 * fid.cu + the conv engine) ----
 * Parameters by the state-dict names of pytorch-fid's wrapper (blocks.<i>.<j>.conv.weight, .bn.weight / bias / running_mean /
 * running_var; BatchNorm eps 1e-3 folded at prepare).
 * forward: x fp32 NCHW [batch,3,h,w] RGB -> feat [batch,2048] float32, the pool3 features; resize: bilinear (align_corners=False,
 *   torch's CPU arithmetic) to 299 x 299 first, normalize: 2x - 1 after it.  The network input must be at least 75 x 75.
 *   An image with a NaN in a value the first conv reads gets NaN features, as in torch.  feat is 16-byte aligned.
 * forward_u8: uint8 HWC BGR faces [batch,h,w,3] through pytorch-fid's path (RGB v / 255, resize, 2x - 1), fused into the stem;
 *   equal to cfb_fid_input followed by forward with both flags off, bit for bit.  Workspace: cfb_fid_workspace_bytes.
 * input: the input stage alone, fp32 NCHW [batch,3,h,w] or (u8) uint8 HWC BGR [batch,h,w,3] -> out fp32 NCHW [batch,3,299,299]
 *   (resize) or [batch,3,h,w].
 * stats: float64 mu [d] and sigma [d,d] = np.cov(feat, rowvar=False) of feat [n,d] (n >= 2, d a multiple of 64, feat 16-byte
 *   aligned); every sum runs
 *   over the rows in order, so the result depends only on the matrix.
 * debug_fid_pool (test entry point): NHWC [n,h,w,c] -> 3x3 max pool stride 2 valid (kind 0), max pool stride 1 pad 1 (1), or avg
 *   pool stride 1 pad 1 with count_include_pad=False (2); c a multiple of 4. */
typedef struct cfb_fid cfb_fid;
cfb_fid* cfb_fid_create(void);
void     cfb_fid_destroy(cfb_fid* net);
int      cfb_fid_set_param(cfb_fid* net, const char* name, const float* dev_ptr, int64_t numel);
int      cfb_fid_prepare(cfb_fid* net, void* stream);
int64_t  cfb_fid_workspace_bytes(cfb_fid* net, int32_t batch, int32_t h, int32_t w, int32_t resize);
int      cfb_fid_forward(cfb_fid* net, const float* x_nchw, int32_t batch, int32_t h, int32_t w, int32_t resize, int32_t normalize,
                         float* feat, void* workspace, int64_t workspace_bytes, void* stream);
int      cfb_fid_forward_u8(cfb_fid* net, const uint8_t* faces_bgr, int32_t batch, int32_t h, int32_t w, float* feat, void* workspace,
                            int64_t workspace_bytes, void* stream);
int      cfb_fid_input(const void* src, int32_t u8, int32_t batch, int32_t h, int32_t w, int32_t resize, int32_t normalize, float* out,
                       void* stream);
int      cfb_fid_stats(const float* feat, int64_t n, int32_t d, double* mu, double* sigma, void* stream);
int      cfb_debug_fid_pool(const float* in, float* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t kind, void* stream);
/* Test entry point of the per-tap engine's explicit windows: a kh x kw conv (1..7 each), zero padding (pad_h, pad_w), stride 1
 * or 2, of NHWC in [n,h,w,cin] (cin a multiple of 64) with OIHW weights [cout,cin,kh,kw] and bias [cout] (may be NULL), into
 * channels [out_c0, out_c0 + cout) of out [n,ho,wo,out_pitch], ho = (h + 2 pad_h - kh) / stride + 1; the other channels are
 * not written.  Workspace: cfb_conv2d_pertap_window_workspace_bytes. */
int64_t  cfb_conv2d_pertap_window_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw,
                                                  int32_t stride, int32_t pad_h, int32_t pad_w);
int      cfb_conv2d_pertap_window_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                                       int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw, int32_t stride, int32_t pad_h,
                                       int32_t pad_w, int32_t out_act, int32_t out_pitch, int32_t out_c0, void* workspace,
                                       int64_t workspace_bytes, void* stream);

/* ---- YOLOv5l-face detector (facelib/detection/yolov5face, models/yolov5l.yaml; yolo.cu + the conv engine) ----
 * Parameters by the reference's state-dict names (BatchNorm folded at prepare; the Detect anchor_grid buffer gives the anchor
 * sizes in pixels).  h and w are multiples of 32; P = cfb_yolov5face_predictions(h, w) = 3 (hw/64 + hw/256 + hw/1024).
 * forward: x fp32 NCHW [batch,3,h,w] (RGB / 255) -> pred [batch,P,16] (Detect's decoded output, rows ordered by level, anchor,
 * y, x) and, where not NULL, the raw head outputs raw_l [batch,3,h/s_l,w/s_l,16] for s_l = 8, 16, 32.
 * forward_u8: uint8 HWC BGR images [batch,img_h,img_w,3] placed at (top, left) of the h x w letterbox canvas, whose other
 * pixels are 114; the BGR -> RGB swap and the / 255 are fused (the result equals forward on that canvas bit for bit).
 * candidates: per image, the pred rows whose objectness (field 4) is > conf_threshold, in prediction order, into rows
 * [batch,P,16]; counts [batch] (device int32). */
typedef struct cfb_yolov5face cfb_yolov5face;
int64_t         cfb_yolov5face_predictions(int32_t h, int32_t w);
cfb_yolov5face* cfb_yolov5face_create(void);
void            cfb_yolov5face_destroy(cfb_yolov5face* net);
int             cfb_yolov5face_set_param(cfb_yolov5face* net, const char* name, const float* dev_ptr, int64_t numel);
int             cfb_yolov5face_prepare(cfb_yolov5face* net, void* stream);
int64_t         cfb_yolov5face_workspace_bytes(cfb_yolov5face* net, int32_t batch, int32_t h, int32_t w);
int             cfb_yolov5face_forward(cfb_yolov5face* net, const float* x_nchw, float* pred, float* raw0, float* raw1, float* raw2,
                                       int32_t batch, int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int             cfb_yolov5face_forward_u8(cfb_yolov5face* net, const uint8_t* img_bgr_hwc, int32_t img_h, int32_t img_w, int32_t top,
                                          int32_t left, float* pred, float* raw0, float* raw1, float* raw2, int32_t batch, int32_t h,
                                          int32_t w, void* workspace, int64_t workspace_bytes, void* stream);
int             cfb_yolov5face_candidates(const float* pred, int32_t batch, int32_t h, int32_t w, float conf_threshold, float* rows,
                                          int32_t* counts, void* stream);

/* ---- Restoration metrics: basicsr's calculate_psnr / calculate_ssim (basicsr/metrics/psnr_ssim.py) on the device ----
 * Pair p compares a[p] with b[p / k] (a holds pairs images, b pairs / k: a sweep's K candidates per face against one ground
 * truth each), HWC images [h, w, c] of element type dtype (CFB_IMG_U8 / _U16 / _F32 / _F64) read in place.  crop_border pixels
 * are dropped from each edge.  y_channel: to_y_channel (metric_util.py:32-45) at load -- v = float32(x) / 255; for c == 3
 * Y = (v0 * 24.966 + v1 * 128.553) + v2 * 65.481 + 16 in float64 (channel 0 blue), / 255 rounded to float32; then * 255 in float32.
 * want_psnr: 0 none, 1 psnr_out[p] = 20 log10(255 / sqrt(mse)) (inf for mse == 0; peak 255 for every dtype), 2 psnr_out[p] =
 *   mse, the mean of (a - b)^2 -- summed exactly in int64 for integer images without y_channel (so it equals numpy's mean), in
 *   float64 otherwise, of float32 squares on the Y path.
 * want_ssim: ssim_out[p] = the mean over channels of the mean SSIM map (Gaussian window 11, sigma 1.5, valid region only,
 *   C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2), filtered in float64 (the 11 horizontal taps, then the 11 vertical ones).
 * psnr_out / ssim_out: device double [pairs].  Needs at least one pixel (PSNR) or 11 x 11 (SSIM) after the crop;
 * pairs <= 65535.  Every sum has a fixed order that depends on the image size only: the results are the same on every run and
 * whatever the batch.  NaN or inf values give NaN / inf results.  workspace: cfb_psnr_ssim_workspace_bytes bytes. */
int64_t cfb_psnr_ssim_workspace_bytes(int32_t pairs, int32_t h, int32_t w, int32_t c, int32_t crop_border, int32_t y_channel);
int     cfb_psnr_ssim(const void* a, const void* b, int32_t dtype, int32_t pairs, int32_t k, int32_t h, int32_t w, int32_t c,
                      int32_t crop_border, int32_t y_channel, int32_t want_psnr, int32_t want_ssim, double* psnr_out,
                      double* ssim_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- Synthetic degradations: FFHQBlindDataset's blur -> downsample -> noise -> JPEG -> resize chain on the device ----
 * (basicsr/data/ffhq_blind_dataset.py:210-240) for gt uint8 BGR faces [batch, gt_size, gt_size, 3], one launch per stage.
 * Per face b: kernels [batch, ksize, ksize] float64 (device; odd ksize <= 63) correlated with BORDER_REFLECT_101 in float64
 * and rounded once to float32, only where the downsample reads; small_sizes[b] (host, 1..gt_size) the INTER_LINEAR
 * downsample (cv2's float arithmetic); noise_offsets[b] (host; -1 = none) the float offset of its [s, s, 3] field in the
 * packed device array noise, added before the clip to [0, 1]; qualities[b] (host; 0 = none, else 1..100) the cv2 JPEG
 * round trip (libjpeg-turbo baseline 4:2:0, islow) of saturate_cast<uchar>(x * 255); then / 255, INTER_LINEAR to in_size
 * (<= gt_size) and clip(round(x * 255)) -> lq uint8 BGR [batch, in_size, in_size, 3].  Workspace:
 * cfb_degrade_workspace_bytes (-1 for bad arguments).
 * debug_degrade_faces (test entry point): also stage_a float32, the image after the downsample, and pre_jpeg uint8, the JPEG
 *   input (faces with a quality only), each packed as the faces' [s, s, 3] images one after another.
 * jpeg_roundtrip: dst = cv2.imdecode(cv2.imencode('.jpg', src, [IMWRITE_JPEG_QUALITY, q]), 1) for n uint8 BGR images
 *   [n, h, w, 3], qualities (host) 1..100 per image; src and dst must not alias.  Workspace: cfb_jpeg_workspace_bytes. */
int64_t cfb_degrade_workspace_bytes(int32_t batch, int32_t gt_size, const int32_t* small_sizes, const int32_t* qualities);
int     cfb_degrade_faces(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                          const int32_t* small_sizes, const int32_t* qualities, const float* noise, const int64_t* noise_offsets,
                          int32_t in_size, uint8_t* lq, void* workspace, int64_t workspace_bytes, void* stream);
int     cfb_debug_degrade_faces(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                                const int32_t* small_sizes, const int32_t* qualities, const float* noise,
                                const int64_t* noise_offsets, int32_t in_size, uint8_t* lq, void* workspace,
                                int64_t workspace_bytes, float* stage_a, uint8_t* pre_jpeg, void* stream);
/* ---- Colorization and inpainting inputs: FFHQBlindDataset's colour and mask stages (ffhq_blind_dataset.py:242-273) ----
 * applied to the dataset's float32 image before its clip(round(x * 255)), so each face rounds once, as the dataset does.
 * With kernels and small_sizes (both or neither), that image is the corruption chain's final INTER_LINEAR (arguments as
 * cfb_degrade_faces); without them it is gt / 255 and in_size must equal gt_size (the dataset does not resize then).
 * color_ops (host; NULL = no colour stages) [batch][6] int32: flags (1 shift, 2 gray, 4 mask), the number of torchvision ops
 * n (0..4), then n op codes in application order (0 brightness, 1 contrast, 2 saturation, 3 hue; each at most once).
 * color_factors (host) [batch][7] float32: the shift in BGR order, then the n factors (>= 0; hue in [-0.5, 0.5]).  Per face:
 *   shift   x + shift[c] in float32, clip to [0, 1]
 *   gray    cv2.cvtColor(float32, COLOR_BGR2GRAY) bit for bit, fma(r, 0.299f, fma(b, 0.114f, g * 0.587f)), on 3 channels
 *   ops     on RGB, torchvision's adjust_brightness / _contrast / _saturation / _hue with torch's float32 op sequence:
 *           _blend = clamp(f * x + float32(1.0 - f) * y, 0, 1) without contraction, gray = (0.2989 r + 0.587 g) + 0.114 b,
 *           hue = _rgb2hsv, (h + f) % 1.0, _hsv2rgb
 *   output  round half to even of x * 255, clip -> lq uint8 BGR [batch, in_size, in_size, 3]
 * The contrast mean is the mean gray of the whole face just before the contrast op: float64 sums per 256-pixel block, added
 * in block order, / n in float64, rounded once to float32 -- the same whatever the batch and on every run.
 * Mask faces (flags 4 alone, no corruption): masks is a device uint8 [batch, gt_size, gt_size] array, and lq is 255 where
 * the face's mask is nonzero and gt elsewhere.  Faces without any stage give cfb_degrade_faces' bytes (with corruption)
 * or gt (without).  Mixed stages and op orders run in the same four launches after the chain, without host synchronisation.
 * Workspace: cfb_degrade_color_workspace_bytes (-1 for bad arguments).
 * debug_degrade_faces_color (test entry point): also each face's contrast mean (device float32 [batch]; NaN without one). */
int64_t cfb_degrade_color_workspace_bytes(int32_t batch, int32_t gt_size, const int32_t* small_sizes, const int32_t* qualities,
                                          const int32_t* color_ops, int32_t in_size);
int     cfb_degrade_faces_color(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                                const int32_t* small_sizes, const int32_t* qualities, const float* noise,
                                const int64_t* noise_offsets, const int32_t* color_ops, const float* color_factors,
                                const uint8_t* masks, int32_t in_size, uint8_t* lq, void* workspace, int64_t workspace_bytes,
                                void* stream);
int     cfb_debug_degrade_faces_color(const uint8_t* gt, int32_t batch, int32_t gt_size, const double* kernels, int32_t ksize,
                                      const int32_t* small_sizes, const int32_t* qualities, const float* noise,
                                      const int64_t* noise_offsets, const int32_t* color_ops, const float* color_factors,
                                      const uint8_t* masks, int32_t in_size, uint8_t* lq, void* workspace,
                                      int64_t workspace_bytes, float* contrast_means, void* stream);
int64_t cfb_jpeg_workspace_bytes(int32_t n, int32_t h, int32_t w);
int     cfb_jpeg_roundtrip(const uint8_t* src, uint8_t* dst, int32_t n, int32_t h, int32_t w, const int32_t* qualities,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* Asynchronous failures.  Kernels never trap and never leave a sticky CUDA error behind (the reference's callers catch
 * RuntimeError and fall back to the input face, inference_codeformer.py:209-211; web-demos/hugging_face/app.py:176): a
 * barrier time-out of the tensor-core pipeline, an activation outside the fp16 operand range (|x| > 65504) or a code index
 * outside the codebook given to cfb_code_scores sets a bit in a host-mapped status word.  It is reported (status 1 + cfb_last_error) by the NEXT forward on that device, by the
 * *_host entry points right after their stream synchronisation, and by this call -- use it after synchronising the stream
 * of an asynchronous forward.  The context stays usable; the reporting call clears the condition. */
int cfb_check_async_status(void);
/* test hooks: barrier time-out in SM cycles (default 4e9, about 2 s); kind != 0 makes the next wgmma conv launch drop one
 * TMA load so that its pipeline times out (tests/test_gpu_faults.py) */
int cfb_debug_set_wait_limit(int64_t cycles);
int cfb_debug_inject_fault(int32_t kind);
/* diagnostics: while `stamps` (device memory, >= 32 int64) is non-NULL, CTA 0 of every wgmma conv launch
 * writes the SM cycle counter at its role hand-offs ([0] entry, [1] set-up done, [2] first TMA, [3] first MMA, [4] last MMA
 * issued, [5]/[6] first/last accumulator seen by the epilogue, [7] epilogue K loop done, [13] epilogue done, [8]/[9] tear-down,
 * [10..12] transform roles, [14]/[15] %globaltimer at entry / exit), and every CTA of a 128x128-tile conv adds the cycles its
 * roles wait to stamps[32 + 8 * cta + k] (k: MMA weight / patch / tile hand-off waits and whole role, epilogue cfull wait,
 * residual/SFT loads, stores and whole role; zero them first; the buffer then needs 32 + 8 * grid int64).  NULL switches it
 * off.  The stamps exist only in builds of the library with -DCFB_TC_STAMPS=1 (they slow every conv kernel); the production
 * build accepts the call and ignores it. */
int cfb_debug_set_stamps(int64_t* stamps);
/* layout plumbing */
int cfb_nchw_to_nhwc(const float* in, float* out, int32_t n, int32_t c, int32_t hw, void* stream);
int cfb_nhwc_to_nchw(const float* in, float* out, int32_t n, int32_t c, int32_t hw, void* stream);

/* ---- whole-image paste-back (face_restoration_helper.py:319-349, 372-516; pasteback.cu) ----
 * cv2 arithmetic throughout (fixed-point warpAffine coordinates, 11-bit INTER_LINEAR resize, rect erosion, reflect-101
 * Gaussian blur).  All images are uint8 HWC, 3 channels, device memory; matrices are host double[6] (row-major 2x3).
 * cfb_warp_affine_u8: n crops [n,out_h,out_w,3] of one image with cv2.warpAffine(img, affines[i], (out_w, out_h), INTER_LINEAR,
 *   border_mode, (v0, v1, v2)); border_mode 0 = constant, 2 = reflect, 4 = reflect-101 (cv2's numbering).
 * cfb_resize_linear_u8: cv2.resize(src[i], (out_w, out_h), INTER_LINEAR) for n images [n,h,w,3].
 * cfb_paste_faces: pastes n restored faces [n,S,S,3] into `canvas` [h_up,w_up,3] (the resized background; overwritten with the
 *   result) in face order.  inverse_affines are the matrices paste_faces_to_input_image passes to warpAffine (after its offset
 *   adjustments); upscale sets the first erosion (int(2*upscale)).  parse_masks [n,512,512] (0/255, MASK_COLORMAP of the
 *   parsing network's argmax) selects use_parse (float64 blend); NULL blends in float32.  debug_canvas (optional, device
 *   [h_up,w_up,3] f32) receives the canvas before the uint8 cast; w_edge_out (optional, host int32[n]) the fusion edge per
 *   face.  The areas that fix the kernel sizes are read back once, so the call synchronises `stream`. */
int cfb_warp_affine_u8(const uint8_t* img, int32_t h, int32_t w, const double* affines, int32_t n, uint8_t* out,
                       int32_t out_h, int32_t out_w, int32_t border_mode, int32_t v0, int32_t v1, int32_t v2, void* stream);
int cfb_resize_linear_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w,
                         void* stream);
int64_t cfb_paste_faces_workspace_bytes(int32_t h_up, int32_t w_up, int32_t n, int32_t face_size, int32_t use_parse,
                                        const double* inverse_affines);
int cfb_paste_faces(uint8_t* canvas, int32_t h_up, int32_t w_up, const uint8_t* faces, int32_t n, int32_t face_size,
                    const uint8_t* parse_masks, const double* inverse_affines, double upscale, float* debug_canvas,
                    int32_t* w_edge_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- whole-image mode over batches of equal-size images ----
 * cfb_resize_area_u8: cv2.resize(src[i], (out_w, out_h), INTER_AREA) for n images [n,h,w,3], shrinking only (out_h <= h,
 *   out_w <= w): resizeAreaFast's integer sums for integer factors, computeResizeAreaTab weights with float sums otherwise.
 * cfb_resize_linear_scale_u8: cv2.resize(src[i], (0, 0), fx=fx, fy=fy, INTER_LINEAR) for enlarging factors (>= 1), the
 *   output size being the caller's (cv2: round(w * fx), round(h * fy)); the taps follow fx / fy, not the size ratio.
 * cfb_warp_affine_multi_u8: cfb_warp_affine_u8 over a batch imgs [n_img,h,w,3]; crop i samples image img_index[i] (host).
 * cfb_paste_faces_multi: cfb_paste_faces over n_img canvases [n_img,h_up,w_up,3]; face i goes into canvas img_index[i]
 *   (host int32[n]).  Each canvas ends byte for byte as cfb_paste_faces of its own faces would leave it; composites run in
 *   face order, and the areas of all faces are read back in one synchronisation of `stream`. */
int cfb_resize_area_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w,
                       void* stream);
int cfb_resize_linear_scale_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w,
                               double fx, double fy, void* stream);
int cfb_warp_affine_multi_u8(const uint8_t* imgs, int32_t n_img, int32_t h, int32_t w, const double* affines,
                             const int32_t* img_index, int32_t n, uint8_t* out, int32_t out_h, int32_t out_w,
                             int32_t border_mode, int32_t v0, int32_t v1, int32_t v2, void* stream);
int64_t cfb_paste_faces_multi_workspace_bytes(int32_t n_img, int32_t h_up, int32_t w_up, int32_t n, int32_t face_size,
                                              int32_t use_parse, const double* inverse_affines);
int cfb_paste_faces_multi(uint8_t* canvases, int32_t n_img, int32_t h_up, int32_t w_up, const uint8_t* faces, int32_t n,
                          int32_t face_size, const uint8_t* parse_masks, const double* inverse_affines, const int32_t* img_index,
                          double upscale, int32_t* w_edge_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- whole-image mode: any output scale, and gray images ----
 * cfb_resize_lanczos4_u8: cv2.resize(src[i], (out_w, out_h), INTER_LANCZOS4) for n images [n,h,w,3], any factors, byte for byte:
 *   what RealESRGANer.enhance does for outscale != scale (realesrgan_utils.py:245-250) and paste_faces_to_input_image does to
 *   the upsampled background (face_restoration_helper.py:381).  The tap tables are built on the host per call.
 * cfb_lanczos4_table: those tables for one axis (host only, no device needed): idx[dst_len] = floor of the source coordinate
 *   (taps at idx-3 .. idx+4, clamped to the image), coef[dst_len*8] = the weights * 2048 as int16.
 * cfb_resize_lanczos4_u16: cv2.resize on CV_16U [n,h,w,3], byte for byte: cv2's float path, not the int16 taps of uint8 --
 *   float32 weights, a horizontal then a vertical pass of float32 products summed left to right (no fused multiply-add),
 *   rounded half to even and saturated.  What enhance does to a 16-bit result for outscale != scale.
 * cfb_lanczos4_table_f32: its tables for one axis (host only): idx as above, coef[dst_len*8] the float32 weights.
 * cfb_gray_adain_faces: add_restored_face on a gray image (face_restoration_helper.py:364-369): out[i] [S,S,3] float64 =
 *   adain_npy(bgr2gray(restored[i]), cropped[i]) (facelib/utils/misc.py:169-202), both inputs uint8 [n,S,S,3] BGR.  stats
 *   (optional, device double [n,4,3]) receives content mean, content std, style mean, style std per channel.  float64, two-pass
 *   variance, fixed summation order (equal to numpy's up to rounding; the same on every run, whatever n is).
 * cfb_is_gray_u8: the moments behind is_gray(img, threshold) (facelib/utils/misc.py:146-158) of n images [n,h,w,3] BGR in one
 *   launch: sums (device int64 [n][6]) = {Σd1, Σd2, Σd3, Σd1², Σd2², Σd3²} for d1 = B-G, d2 = G-R, d3 = R-B, exact.  The caller
 *   decides: mean over k of (h*w*Σdk² - (Σdk)²) / (h*w)² <= threshold.
 * cfb_f64_to_input: cfb_u8_to_input for float64 faces: astype(float32) / 255, BGR -> RGB, (x - 0.5) / 0.5 (:459-461).
 * cfb_paste_faces_f64: cfb_paste_faces_multi for float64 faces [n,S,S,3] (the restored faces of a gray image): warpAffine as
 *   cv2 runs it on CV_64F (the fixed-point coordinates, float32 weights, sums in double) and a float64 canvas from the first
 *   face on.  wide_out (optional, host int32[n_img]) tells which canvases exceed 256, where the reference returns
 *   astype(np.uint16) (:496-499); canvases_u16 (optional, needs wide_out) receives that cast of every canvas when any does.
 *   `canvases` always receives astype(np.uint8). */
int cfb_resize_lanczos4_u8(const uint8_t* src, int32_t n, int32_t h, int32_t w, uint8_t* dst, int32_t out_h, int32_t out_w,
                           void* stream);
void cfb_lanczos4_table(int32_t src_len, int32_t dst_len, int32_t* idx, int16_t* coef);
int cfb_resize_lanczos4_u16(const uint16_t* src, int32_t n, int32_t h, int32_t w, uint16_t* dst, int32_t out_h, int32_t out_w,
                            void* stream);
void cfb_lanczos4_table_f32(int32_t src_len, int32_t dst_len, int32_t* idx, float* coef);
int cfb_gray_adain_faces(const uint8_t* restored, const uint8_t* cropped, int32_t n, int32_t face_size, double* out, double* stats,
                         void* stream);
int cfb_is_gray_u8(const uint8_t* images, int32_t n, int32_t h, int32_t w, int64_t* sums, void* stream);
int cfb_f64_to_input(const double* img_bgr_hwc, float* x_nchw, int32_t n, int32_t hw, void* stream);
int64_t cfb_paste_faces_f64_workspace_bytes(int32_t n_img, int32_t h_up, int32_t w_up, int32_t n, int32_t face_size,
                                            int32_t use_parse, const double* inverse_affines);
int cfb_paste_faces_f64(uint8_t* canvases, int32_t n_img, int32_t h_up, int32_t w_up, const double* faces, int32_t n,
                        int32_t face_size, const uint8_t* parse_masks, const double* inverse_affines, const int32_t* img_index,
                        double upscale, uint16_t* canvases_u16, int32_t* wide_out, int32_t* w_edge_out, void* workspace,
                        int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CFB200_H_ */
