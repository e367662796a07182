// Host runtime of libcfb200: the network plan (block lists of the reference constructors), weight
// preparation, the stream-ordered workspace arena, and the forward passes that enqueue the kernels.
//
// Mirrors, block for block:
//   Encoder / Generator block lists      /root/reference/basicsr/archs/vqgan_arch.py:229-323
//   VQAutoEncoder.forward                vqgan_arch.py:385-389
//   CodeFormer.forward                   /root/reference/basicsr/archs/codeformer_arch.py:223-280
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/cfb200.h"
#include "kernels.cuh"
#include "conv_tc.cuh"

namespace cfb {

// ---- error / counters --------------------------------------------------------------------------
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const std::string& last_error() { return g_err; }
static std::atomic<int64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool pdl_enabled() {
#if defined(CFB_PDL_DEVICE) && !CFB_PDL_DEVICE
  return false;
#endif
  static const bool v = [] { const char* e = getenv("CFB_PDL"); return !(e && atoi(e) == 0); }();
  return v;
}
int64_t launch_count() { return g_launches.load(); }
void reset_launch_count() { g_launches.store(0); }

// ---- asynchronous device status (barrier time-out / fp16 operand overflow) ---------------------------------
// One host-mapped word per device.  Kernels never trap: they set bits here (conv_tc.cu) and the host reports them as an
// ordinary error at the next check point -- the CUDA context stays usable, the caller's per-face fallback keeps working
// (SURVEY.md section 8(b) "Errors"; /root/reference/inference_codeformer.py:209-211).
static std::mutex g_status_mu;
static unsigned* g_status_words = nullptr;            // host pointer of a mapped, portable allocation: [64] words
static unsigned* g_status_dev_word[64] = {};          // device pointer of word `dev`, as bound on device `dev`
static uint64_t g_status_bound = 0;                   // devices whose symbols are bound
static long long g_wait_limit_cycles = 4000000000LL;

int async_status_init(cudaStream_t) {
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_REQUIRE(dev >= 0 && dev < 64, "more than 64 CUDA devices are not supported");
  std::lock_guard<std::mutex> lk(g_status_mu);
  if (g_status_bound & (1ull << dev)) return 0;
  if (!g_status_words) {
    CFB_CUDA(cudaHostAlloc((void**)&g_status_words, 64 * sizeof(unsigned), cudaHostAllocMapped | cudaHostAllocPortable));
    memset(g_status_words, 0, 64 * sizeof(unsigned));
  }
  unsigned* dptr = nullptr;
  CFB_CUDA(cudaHostGetDevicePointer((void**)&dptr, g_status_words, 0));
  g_status_dev_word[dev] = dptr + dev;
  CFB_CHECK(tc_bind_status_word(dptr + dev, g_wait_limit_cycles));
  g_status_bound |= 1ull << dev;
  return 0;
}

int async_status_word(unsigned** dev_word) {
  CFB_CHECK(async_status_init(nullptr));      // after the first call per device: a lock and a bit test, no CUDA call
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_status_mu);
  *dev_word = g_status_dev_word[dev];
  return 0;
}

int async_status_check(const char* where) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); return 0; }
  unsigned bits = 0;
  {
    std::lock_guard<std::mutex> lk(g_status_mu);
    if (!g_status_words || !(g_status_bound & (1ull << dev))) return 0;
    bits = __atomic_exchange_n(g_status_words + dev, 0u, __ATOMIC_ACQ_REL);
  }
  if (!bits) return 0;
  std::string msg = std::string(where) + ": a kernel of an earlier launch on this device reported";
  if (bits & CFB_STATUS_TIMEOUT) msg += " [barrier time-out: the tensor-core pipeline was aborted, results of that launch are invalid]";
  if (bits & CFB_STATUS_OVERFLOW) msg += " [fp16 operand overflow: an activation exceeded 65504 on the fp16 tensor-core operand path]";
  if (bits & CFB_STATUS_INDEX) msg += " [code index out of range: a ground-truth code given to cfb_code_scores is outside [0, codebook_size)]";
  if (bits & CFB_STATUS_TIMEOUT) {
    if (cudaDeviceSynchronize() != cudaSuccess) cudaGetLastError();   // the aborted launch has drained; the context is healthy
    tc_clear_abort();
  }
  set_error(msg);
  return 1;
}

// ---- stream-ordered arena over the caller's workspace ---------------------------------------------
// All work of one forward is enqueued on one stream, so a block can be handed out again as soon as the
// host has *enqueued* its last reader.  First-fit with coalescing; `dry` mode only tracks the high-water mark.
class Arena {
 public:
  void reset(void* base, size_t cap, bool dry) {
    base_ = (char*)base; cap_ = cap; dry_ = dry; high_ = 0; free_.clear(); used_.clear();
    if (dry) { base_ = (char*)(uintptr_t)0x10000; cap_ = (size_t)1 << 46; }
    free_[0] = cap_;
  }
  void* alloc(size_t bytes) {
    bytes = (bytes + 1023) / 1024 * 1024;   // 1 KiB granularity keeps every tensor TMA/float4 aligned
    if (bytes == 0) bytes = 1024;
    for (auto it = free_.begin(); it != free_.end(); ++it) {
      if (it->second >= bytes) {
        const size_t off = it->first, sz = it->second;
        free_.erase(it);
        if (sz > bytes) free_[off + bytes] = sz - bytes;
        used_[off] = bytes;
        if (off + bytes > high_) high_ = off + bytes;
        return base_ + off;
      }
    }
    return nullptr;
  }
  void release(void* p) {
    if (!p) return;
    const size_t off = (size_t)((char*)p - base_);
    auto u = used_.find(off);
    if (u == used_.end()) return;
    size_t sz = u->second;
    used_.erase(u);
    auto nxt = free_.lower_bound(off);
    if (nxt != free_.end() && off + sz == nxt->first) { sz += nxt->second; nxt = free_.erase(nxt); }
    if (nxt != free_.begin()) {
      auto prv = std::prev(nxt);
      if (prv->first + prv->second == off) { prv->second += sz; return; }
    }
    free_[off] = sz;
  }
  size_t high() const { return high_; }
  bool dry() const { return dry_; }

 private:
  char* base_ = nullptr;
  size_t cap_ = 0, high_ = 0;
  bool dry_ = false;
  std::map<size_t, size_t> free_, used_;
};

// ---- what every network handle shares ----------------------------------------------------------------
// The parameters the caller registered (device pointers it keeps alive), the slab with the prepared weights on the device
// that was current at prepare time, the workspace arena and the conv precision.  `label` names the network in error
// messages, `api` is the infix of its C functions (cfb_<api>_prepare, ...).
struct NetCore {
  std::mutex mu;
  std::unordered_map<std::string, std::pair<const float*, int64_t>> raw;
  float* slab = nullptr;
  size_t slab_bytes = 0;
  int device = -1;                    // CUDA device the slab / prepared weights live on
  int sm_count = 148;
  bool prepared = false;
  int precision = 0;                  // of the convs each forward names: 0 split fp16 x3 (fp32 parity), 1 single-pass fp16
  Arena arena;
  const char* label;
  const char* api;

  NetCore(const char* label_, const char* api_) : label(label_), api(api_) {}
  ~NetCore() { release_slab(); }

  int set_param(const char* name, const float* dev_ptr, int64_t numel) {
    std::lock_guard<std::mutex> lk(mu);
    raw[name] = {dev_ptr, numel};
    prepared = false;
    return 0;
  }

  // cfb_<api>_set_precision: host state only, read by the next forward
  int set_precision(int32_t precision) {
    CFB_REQUIRE(precision == 0 || precision == 1,
                "cfb_" + std::string(api) + "_set_precision: precision must be 0 (fp32, split) or 1 (fp16)");
    std::lock_guard<std::mutex> lk(mu);
    this->precision = precision;
    return 0;
  }

  const float* param(const std::string& name, int64_t numel) const {
    auto it = raw.find(name);
    if (it == raw.end()) { set_error("missing parameter '" + name + "'"); return nullptr; }
    if (it->second.second != numel) {
      set_error("parameter '" + name + "' has " + std::to_string(it->second.second) + " elements, expected " +
                std::to_string(numel));
      return nullptr;
    }
    return it->second.first;
  }

  // a slab of at least `bytes` on the current device: the net follows the device that is current at prepare time
  // (net.to(other_gpu) -> a new prepare), so a slab on another device is freed there first
  int reserve_slab(size_t bytes) {
    int dev = 0;
    CFB_CUDA(cudaGetDevice(&dev));
    if (slab && (device != dev || slab_bytes < bytes)) {
      if (device != dev && device >= 0) { cudaSetDevice(device); cudaFree(slab); cudaSetDevice(dev); }
      else cudaFree(slab);
      slab = nullptr; slab_bytes = 0;
    }
    if (!slab) { CFB_CUDA(cudaMalloc((void**)&slab, bytes)); slab_bytes = bytes; }
    device = dev;
    return 0;
  }

  void release_slab() {
    if (!slab) return;
    int cur = -1;
    const bool sw = cudaGetDevice(&cur) == cudaSuccess && device >= 0 && cur != device;
    if (sw) cudaSetDevice(device);
    cudaFree(slab);
    if (sw) cudaSetDevice(cur);
    slab = nullptr; slab_bytes = 0;
  }

  // the networks that have only the wgmma path: device check, SM count, the device's status word
  int begin_prepare(cudaStream_t st) {
    int dev = 0, major = 0, sms = 148;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CFB_REQUIRE(major == 9, std::string(label) + ": the wgmma engine needs an sm_90 device (there is no other path)");
    CFB_CHECK(async_status_init(st));
    sm_count = sms > 0 ? sms : 148;
    return 0;
  }

  // a dry run (workspace sizing) needs neither prepared weights nor a device
  int begin_forward(bool dry) {
    CFB_REQUIRE(dry || prepared, "cfb_" + std::string(api) + "_prepare has not been called");
    if (dry) return 0;
    int dev = -1;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_REQUIRE(dev == device, std::string(label) + " was prepared on another CUDA device");
    return async_status_check(("cfb_" + std::string(api) + "_forward").c_str());
  }

  std::string ws_error() const { return "workspace too small (cfb_" + std::string(api) + "_workspace_bytes)"; }

  int alloc(float** p, size_t elems) {
    *p = (float*)arena.alloc(elems * sizeof(float));
    CFB_REQUIRE(*p != nullptr, ws_error());
    return 0;
  }

  // host-only dry run of a forward: the arena's high-water mark is the workspace it needs
  template <class F> int64_t dry_run(F&& forward) {
    std::lock_guard<std::mutex> lk(mu);
    if (forward() != 0) return -1;
    return (int64_t)arena.high() + 4096;
  }
};

struct Tensor {
  float* p = nullptr;
  int N = 0, H = 0, W = 0, C = 0;
  bool owned = true;  // false: caller memory or kept-alive tap
  float* gn_part = nullptr;   // GroupNorm partial sums emitted by the producing tensor-core conv (or null)
  int gn_slots = 0;           // partial slots per image
  void* planes = nullptr;     // fp16 hi/lo operand planes of this tensor emitted by the producing conv (raw values)
  const float* p2 = nullptr;  // channel concatenation held as two tensors: channels [0,C1) live in p, [C1,C) in p2 (Fuse_sft_block)
  int C1 = 0;
  int64_t numel() const { return (int64_t)N * H * W * C; }
};

struct ConvW {
  std::string name;
  int cin = 0, cout = 0, k = 0;
  bool has_bias = true;
  const float* src_w = nullptr;  // reference-layout source (row offset into a larger OIHW tensor allowed)
  const float* src_b = nullptr;
  float* w_f32 = nullptr;        // [taps][cin][cout]
  __half* w_hi = nullptr;        // [taps][cout][cin]
  __half* w_lo = nullptr;
  float* bias = nullptr;
  float* wscale = nullptr;       // 2 floats: [0] scratch |w|max, [1] 2^-k of the fp16 split
  bool is_up = false;            // conv of an Upsample block: also keep the 4-parity 2x2 weights for the tensor-core engine
  __half* u_hi = nullptr;        // [16][cout][cin]
  __half* u_lo = nullptr;
  float* uscale = nullptr;
};
struct NormW { std::string name; int c = 0; const float* gamma = nullptr; const float* beta = nullptr; };
struct ResW { NormW n1, n2; ConvW c1, c2, co; bool has_out = false; };
struct AttnW { NormW n; ConvW qkv, proj; float* consts = nullptr; /* device: [0] = C^-1/2, [1] = 1 */ };
struct FuseW { ResW enc; ConvW s0, s2, h0, h2; };
struct LayerW { NormW n1, n2; ConvW qk, v, o, l1, l2; };
struct Block { int kind; int cin, cout, res; ConvW conv; ResW res_w; AttnW attn; NormW norm; };
enum { B_CONV = 0, B_RES, B_ATTN, B_DOWN, B_UP, B_NORM };

}  // namespace cfb

using namespace cfb;

constexpr int GN_COUNTERS = 1 << 16;

struct cfb_net : cfb::NetCore {
  cfb_net() : NetCore("CodeFormer", "net") {}
  cfb_config cfg;
  std::vector<Block> enc, gen;
  std::map<int, FuseW> fuse;          // keyed by feature size
  std::vector<LayerW> layers;
  ConvW feat_emb, idx_lin;
  ConvW vq_code;                      // codebook as a 1x1 'conv' (distance GEMM of VectorQuantizer.forward on tensor cores)
  NormW idx_norm;
  const float* position_emb = nullptr;
  const float* codebook = nullptr;    // points into slab copy
  int64_t last_launches = 0;
  bool tc_ok = false;                 // device is sm_90 => wgmma engine usable
  cudaStream_t st = nullptr;
  // small owned copies of norm params etc. live in the slab too
  std::vector<std::pair<const float**, std::pair<std::string, int64_t>>> vec_params;  // (dst, (name, numel))
  std::vector<ConvW*> convs;
  float* mha_consts = nullptr;        // device: [0] = head_dim^-1/2, [1] = 1
  unsigned* gn_counters = nullptr;    // ticket-counter ring of the split GroupNorm finalize (in the slab, zero between uses)
  int gn_ctr_pos = 0;
  std::map<int, int64_t> ws_memo;     // batch -> cfb_workspace_bytes (16 host-side dry runs per miss)
  std::map<std::pair<int, int>, int64_t> sweep_ws_memo;   // (batch, k) -> cfb_sweep_workspace_bytes
  int engine = 0;                     // 0 auto (wgmma where the shape allows), 1 fp32 CUDA cores, 2 wgmma only
  std::map<std::string, std::pair<float*, int64_t>> captures;   // stage name -> (device dst, capacity in floats)
};

namespace cfb {

// ---- plan construction (mirrors the reference constructors) -----------------------------------------
static void mk_conv(cfb_net* n, ConvW& c, const std::string& name, int cin, int cout, int k, bool bias = true) {
  c.name = name; c.cin = cin; c.cout = cout; c.k = k; c.has_bias = bias;
  n->convs.push_back(&c);
}
static void mk_norm(cfb_net* n, NormW& w, const std::string& name, int c) {
  w.name = name; w.c = c;
  n->vec_params.push_back({&w.gamma, {name + ".weight", c}});
  n->vec_params.push_back({&w.beta, {name + ".bias", c}});
}
static void mk_res(cfb_net* n, ResW& r, const std::string& p, int cin, int cout) {
  mk_norm(n, r.n1, p + ".norm1", cin);
  mk_conv(n, r.c1, p + ".conv1", cin, cout, 3);
  mk_norm(n, r.n2, p + ".norm2", cout);
  mk_conv(n, r.c2, p + ".conv2", cout, cout, 3);
  r.has_out = cin != cout;
  if (r.has_out) mk_conv(n, r.co, p + ".conv_out", cin, cout, 1);
}
static bool in_list(const int32_t* l, int n, int v) {
  for (int i = 0; i < n; ++i) if (l[i] == v) return true;
  return false;
}

static void build_blocks(cfb_net* n, std::vector<Block>& blocks, const std::string& prefix,
                         const std::vector<std::array<int, 4>>& plan) {
  blocks.resize(plan.size());   // resize first: ConvW addresses are registered in n->convs
  for (size_t i = 0; i < plan.size(); ++i) {
    Block& b = blocks[i];
    b.kind = plan[i][0]; b.cin = plan[i][1]; b.cout = plan[i][2]; b.res = plan[i][3];
    const std::string p = prefix + ".blocks." + std::to_string(i);
    switch (b.kind) {
      case B_CONV: mk_conv(n, b.conv, p, b.cin, b.cout, 3); break;
      case B_RES: mk_res(n, b.res_w, p, b.cin, b.cout); break;
      case B_ATTN:
        mk_norm(n, b.attn.n, p + ".norm", b.cin);
        mk_conv(n, b.attn.qkv, p + ".qkv", b.cin, 3 * b.cin, 1);   // q,k,v fused along Cout (special-cased in prepare)
        mk_conv(n, b.attn.proj, p + ".proj_out", b.cin, b.cin, 1);
        break;
      case B_DOWN: case B_UP: mk_conv(n, b.conv, p + ".conv", b.cin, b.cout, 3); b.conv.is_up = (b.kind == B_UP); break;
      case B_NORM: mk_norm(n, b.norm, p, b.cin); break;
    }
  }
}

static int build_plan(cfb_net* n) {
  const cfb_config& c = n->cfg;
  CFB_REQUIRE(c.n_ch_mult >= 1 && c.n_ch_mult <= 8, "config: bad ch_mult length");
  CFB_REQUIRE(c.nf == 64, "config: only nf=64 is built (first/last conv kernels)");
  // Encoder.__init__  vqgan_arch.py:241-267
  std::vector<std::array<int, 4>> ep, gp;
  int curr = c.img_size;
  ep.push_back({B_CONV, 3, c.nf, curr});
  int cin = c.nf;
  for (int i = 0; i < c.n_ch_mult; ++i) {
    cin = c.nf * (i == 0 ? 1 : c.ch_mult[i - 1]);
    const int cout = c.nf * c.ch_mult[i];
    for (int r = 0; r < c.res_blocks; ++r) {
      ep.push_back({B_RES, cin, cout, curr});
      cin = cout;
      if (in_list(c.attn_res, c.n_attn_res, curr)) ep.push_back({B_ATTN, cin, cin, curr});
    }
    if (i != c.n_ch_mult - 1) { curr /= 2; ep.push_back({B_DOWN, cin, cin, curr}); }
  }
  ep.push_back({B_RES, cin, cin, curr});
  ep.push_back({B_ATTN, cin, cin, curr});
  ep.push_back({B_RES, cin, cin, curr});
  ep.push_back({B_NORM, cin, cin, curr});
  ep.push_back({B_CONV, cin, c.emb_dim, curr});
  // Generator.__init__  vqgan_arch.py:287-316
  cin = c.nf * c.ch_mult[c.n_ch_mult - 1];
  curr = c.img_size >> (c.n_ch_mult - 1);
  gp.push_back({B_CONV, c.emb_dim, cin, curr});
  gp.push_back({B_RES, cin, cin, curr});
  gp.push_back({B_ATTN, cin, cin, curr});
  gp.push_back({B_RES, cin, cin, curr});
  for (int i = c.n_ch_mult - 1; i >= 0; --i) {
    const int cout = c.nf * c.ch_mult[i];
    for (int r = 0; r < c.res_blocks; ++r) {
      gp.push_back({B_RES, cin, cout, curr});
      cin = cout;
      if (in_list(c.attn_res, c.n_attn_res, curr)) gp.push_back({B_ATTN, cin, cin, curr});
    }
    if (i != 0) { curr *= 2; gp.push_back({B_UP, cin, cin, curr}); }
  }
  gp.push_back({B_NORM, cin, cin, curr});
  gp.push_back({B_CONV, cin, 3, curr});
  build_blocks(n, n->enc, "encoder", ep);
  mk_conv(n, n->vq_code, "quantize.embedding", c.emb_dim, c.codebook_size, 1, false);
  build_blocks(n, n->gen, "generator", gp);
  if (c.kind == 1) {
    CFB_REQUIRE(c.img_size == 512 && c.emb_dim == 256, "config: CodeFormer is defined for 512x512 / emb 256");
    CFB_REQUIRE(c.dim_embd == 512 && c.dim_embd % c.n_head == 0 && c.dim_embd / c.n_head == 64,
                "config: only dim_embd=512 with 64-wide heads is built");
    mk_conv(n, n->feat_emb, "feat_emb", c.emb_dim, c.dim_embd, 1);
    n->layers.resize(c.n_layers);
    for (int l = 0; l < c.n_layers; ++l) {
      LayerW& L = n->layers[l];
      const std::string p = "ft_layers." + std::to_string(l);
      const int E = c.dim_embd;
      mk_conv(n, L.qk, p + ".self_attn.in_proj#qk", E, 2 * E, 1);
      mk_conv(n, L.v, p + ".self_attn.in_proj#v", E, E, 1);
      mk_conv(n, L.o, p + ".self_attn.out_proj", E, E, 1);
      mk_conv(n, L.l1, p + ".linear1", E, 2 * E, 1);
      mk_conv(n, L.l2, p + ".linear2", 2 * E, E, 1);
      mk_norm(n, L.n1, p + ".norm1", E);
      mk_norm(n, L.n2, p + ".norm2", E);
    }
    mk_norm(n, n->idx_norm, "idx_pred_layer.0", c.dim_embd);
    mk_conv(n, n->idx_lin, "idx_pred_layer.1", c.dim_embd, c.codebook_size, 1, false);
    static const int chan_of[6][2] = {{16, 512}, {32, 256}, {64, 256}, {128, 128}, {256, 128}, {512, 64}};
    for (int i = 0; i < c.n_connect; ++i) {
      int ch = 0;
      for (auto& e : chan_of) if (e[0] == c.connect[i]) ch = e[1];
      CFB_REQUIRE(ch != 0, "config: connect_list entries must be one of 16..512");
      FuseW& f = n->fuse[c.connect[i]];
      const std::string p = "fuse_convs_dict." + std::to_string(c.connect[i]);
      mk_res(n, f.enc, p + ".encode_enc", 2 * ch, ch);
      mk_conv(n, f.s0, p + ".scale.0", ch, ch, 3);
      mk_conv(n, f.s2, p + ".scale.2", ch, ch, 3);
      mk_conv(n, f.h0, p + ".shift.0", ch, ch, 3);
      mk_conv(n, f.h2, p + ".shift.2", ch, ch, 3);
    }
  }
  return 0;
}

// ---- weight preparation --------------------------------------------------------------------------------
static int resolve_conv_sources(cfb_net* n, ConvW& c, float* qkv_scratch_w, float* qkv_scratch_b, cudaStream_t st) {
  const int64_t wn = (int64_t)c.cout * c.cin * c.k * c.k;
  const size_t hash = c.name.find('#');
  if (c.name.size() > 4 && c.name.compare(c.name.size() - 4, 4, ".qkv") == 0) {
    // AttnBlock q,k,v (vqgan_arch.py:173-193) stacked along Cout so one GEMM feeds the attention core
    const std::string p = c.name.substr(0, c.name.size() - 4);
    const int C = c.cin;
    const char* nm[3] = {".q", ".k", ".v"};
    for (int i = 0; i < 3; ++i) {
      const float* w = n->param(p + nm[i] + ".weight", (int64_t)C * C);
      const float* b = n->param(p + nm[i] + ".bias", C);
      if (!w || !b) return 1;
      CFB_CUDA(cudaMemcpyAsync(qkv_scratch_w + (int64_t)i * C * C, w, (size_t)C * C * 4, cudaMemcpyDeviceToDevice, st));
      CFB_CUDA(cudaMemcpyAsync(qkv_scratch_b + (int64_t)i * C, b, (size_t)C * 4, cudaMemcpyDeviceToDevice, st));
    }
    c.src_w = qkv_scratch_w; c.src_b = qkv_scratch_b;
    return 0;
  }
  if (hash != std::string::npos) {
    // nn.MultiheadAttention in_proj_weight [3E,E] rows = [Wq;Wk;Wv]  (codeformer_arch.py:102)
    const std::string base = c.name.substr(0, hash);
    const std::string part = c.name.substr(hash + 1);
    const int E = c.cin;
    const float* w = n->param(base + "_weight", (int64_t)3 * E * E);
    const float* b = n->param(base + "_bias", (int64_t)3 * E);
    if (!w || !b) return 1;
    const int row0 = part == "qk" ? 0 : 2 * E;
    c.src_w = w + (int64_t)row0 * E; c.src_b = b + row0;
    return 0;
  }
  c.src_w = n->param(c.name + ".weight", wn);
  if (!c.src_w) return 1;
  if (c.has_bias) { c.src_b = n->param(c.name + ".bias", c.cout); if (!c.src_b) return 1; }
  return 0;
}

static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

static int prepare(cfb_net* n, cudaStream_t st) {
  // slab size
  size_t total = 0;
  for (ConvW* c : n->convs) {
    const size_t wn = (size_t)c->cout * c->cin * c->k * c->k;
    total += align256(wn * 4) + 2 * align256(wn * 2) + align256((size_t)c->cout * 4) + 256;
    if (c->is_up) total += 2 * align256((size_t)16 * c->cout * c->cin * 2) + 256;
  }
  for (auto& v : n->vec_params) total += align256((size_t)v.second.second * 4);
  total += align256((size_t)n->cfg.codebook_size * n->cfg.emb_dim * 4);
  if (n->cfg.kind == 1) total += align256((size_t)n->cfg.latent_size * n->cfg.dim_embd * 4);
  const size_t scratch = align256((size_t)3 * 512 * 512 * 4) + align256(3 * 512 * 4);
  total += scratch;
  total += 256 * (n->enc.size() + n->gen.size());      // per-AttnBlock device constants
  total += align256((size_t)GN_COUNTERS * sizeof(unsigned)) + 256;
  // the net lives on the device that is current at prepare time (net.to(other_gpu) -> a new prepare): slab, SM count and
  // engine availability all follow it
  int dev = 0, major = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CFB_CHECK(n->reserve_slab(total));
  n->sm_count = sms > 0 ? sms : 148;
  n->tc_ok = (major == 9);
  n->ws_memo.clear();
  n->sweep_ws_memo.clear();
  CFB_CHECK(async_status_init(st));
  char* p = (char*)n->slab;
  auto take = [&](size_t bytes) { char* r = p; p += align256(bytes); return r; };
  n->mha_consts = (float*)take(256);
  {
    const float hc[2] = {n->cfg.kind == 1 ? 1.0f / sqrtf((float)(n->cfg.dim_embd / n->cfg.n_head)) : 1.0f, 1.0f};
    CFB_CUDA(cudaMemcpyAsync(n->mha_consts, hc, sizeof(hc), cudaMemcpyHostToDevice, st));
  }
  n->gn_counters = (unsigned*)take((size_t)GN_COUNTERS * sizeof(unsigned));
  n->gn_ctr_pos = 0;
  CFB_CUDA(cudaMemsetAsync(n->gn_counters, 0, (size_t)GN_COUNTERS * sizeof(unsigned), st));
  float* qkv_w = (float*)take((size_t)3 * 512 * 512 * 4);
  float* qkv_b = (float*)take(3 * 512 * 4);
  for (ConvW* c : n->convs) {
    if (c->name.size() > 4 && c->name.compare(c->name.size() - 4, 4, ".qkv") == 0)
      CFB_REQUIRE(c->cin <= 512, "AttnBlock wider than 512 channels is not built");
    CFB_CHECK(resolve_conv_sources(n, *c, qkv_w, qkv_b, st));
    const size_t wn = (size_t)c->cout * c->cin * c->k * c->k;
    c->w_f32 = (float*)take(wn * 4);
    c->w_hi = (__half*)take(wn * 2);
    c->w_lo = (__half*)take(wn * 2);
    c->bias = (float*)take((size_t)c->cout * 4);
    c->wscale = (float*)take(8);
    CFB_CHECK(relayout_oihw_to_tck(c->src_w, c->w_f32, c->cout, c->cin, c->k, st));
    CFB_CHECK(tc_split_weights(c->src_w, c->w_hi, c->w_lo, c->cout, c->cin, c->k, c->wscale, st));
    if (c->is_up) {
      c->u_hi = (__half*)take((size_t)16 * c->cout * c->cin * 2);
      c->u_lo = (__half*)take((size_t)16 * c->cout * c->cin * 2);
      c->uscale = (float*)take(8);
      CFB_CHECK(tc_split_weights_up4(c->src_w, c->u_hi, c->u_lo, c->cout, c->cin, c->uscale, st));
    }
    if (c->has_bias) CFB_CUDA(cudaMemcpyAsync(c->bias, c->src_b, (size_t)c->cout * 4, cudaMemcpyDeviceToDevice, st));
    else CFB_CUDA(cudaMemsetAsync(c->bias, 0, (size_t)c->cout * 4, st));
  }
  for (auto& v : n->vec_params) {
    const float* src = n->param(v.second.first, v.second.second);
    if (!src) return 1;
    float* dst = (float*)take((size_t)v.second.second * 4);
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)v.second.second * 4, cudaMemcpyDeviceToDevice, st));
    *v.first = dst;
  }
  {
    const int64_t ne = (int64_t)n->cfg.codebook_size * n->cfg.emb_dim;
    const float* src = n->param("quantize.embedding.weight", ne);
    if (!src) return 1;
    float* dst = (float*)take((size_t)ne * 4);
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)ne * 4, cudaMemcpyDeviceToDevice, st));
    n->codebook = dst;
  }
  if (n->cfg.kind == 1) {
    const int64_t ne = (int64_t)n->cfg.latent_size * n->cfg.dim_embd;
    const float* src = n->param("position_emb", ne);
    if (!src) return 1;
    float* dst = (float*)take((size_t)ne * 4);
    CFB_CUDA(cudaMemcpyAsync(dst, src, (size_t)ne * 4, cudaMemcpyDeviceToDevice, st));
    n->position_emb = dst;
  }
  for (std::vector<Block>* bl : {&n->enc, &n->gen})
    for (Block& b : *bl)
      if (b.kind == B_ATTN) {
        b.attn.consts = (float*)take(8);
        const float hc[2] = {1.0f / sqrtf((float)b.cin), 1.0f};
        CFB_CUDA(cudaMemcpyAsync(b.attn.consts, hc, sizeof(hc), cudaMemcpyHostToDevice, st));
      }
  // the qkv scratch is read by kernels enqueued above: the sources must stay valid until they ran
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// ---- forward building blocks ----------------------------------------------------------------------------
struct Fwd {
  cfb_net* n;
  cudaStream_t st;
  Arena& ar;
  bool dry;
  int engine;   // 0 auto, 1 f32, 2 tc
  // caller-side image plumbing fused into the first / last conv (cfb_codeformer_forward_u8): uint8 HWC BGR faces
  const unsigned char* in_u8 = nullptr;
  int in_u8_orig = 0;         // in (0, N): images n >= in_u8_orig are face n - in_u8_orig mirrored (cfb_latent_codes_u8)
  unsigned char* out_u8 = nullptr;
  bool inpaint = false;       // conv_last blends out_u8 with in_u8 as inference_inpainting.py does (cfb_codeformer_inpaint_u8)
  bool single_pass = false;   // the convs issued now run single-pass fp16 (ConvArgs::single_pass): set by generator()

  int alloc(Tensor& t, int N, int H, int W, int C) {
    t.N = N; t.H = H; t.W = W; t.C = C; t.owned = true; t.gn_part = nullptr; t.gn_slots = 0; t.planes = nullptr;
    t.p2 = nullptr; t.C1 = 0;
    t.p = (float*)ar.alloc((size_t)t.numel() * 4);
    CFB_REQUIRE(t.p != nullptr, "workspace too small (use cfb_workspace_bytes)");
    return 0;
  }
  int alloc_raw(void** p, size_t bytes) {
    *p = ar.alloc(bytes);
    CFB_REQUIRE(*p != nullptr, "workspace too small (use cfb_workspace_bytes)");
    return 0;
  }
  void release(Tensor& t) {
    if (t.owned) {
      if (t.p) ar.release(t.p);
      if (t.gn_part) ar.release(t.gn_part);
      if (t.planes) ar.release(t.planes);
    }
    t.p = nullptr; t.gn_part = nullptr; t.planes = nullptr;
  }
  void release_raw(void* p) { ar.release(p); }

  // debug/parity hook: copy a stage's NHWC activation out (cfb_net_capture)
  int capture(const std::string& stage, const Tensor& t) {
    if (dry || n->captures.empty()) return 0;
    auto it = n->captures.find(stage);
    if (it == n->captures.end()) return 0;
    CFB_REQUIRE(it->second.second >= t.numel(), "capture buffer too small for stage " + stage);
    CFB_CUDA(cudaMemcpyAsync(it->second.first, t.p, (size_t)t.numel() * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  }

  struct ConvOpt {
    int mode = CONV_SAME;
    const float* in_scale = nullptr; const float* in_shift = nullptr; int in_act = IN_NONE;
    const float* residual = nullptr; int out_act = OUT_NONE;
    const float* sft_dec = nullptr; const float* sft_scale = nullptr; float sft_w = 0.f;
    const float* sft_wv = nullptr;   // [N] per-image w on the device in place of sft_w
    float* out_ptr = nullptr;   // write into caller memory instead of the arena
    bool want_stats = false;    // consumer is a GroupNorm: let the tensor-core epilogue emit the partial sums
    bool want_planes = false;   // a following conv reads this output raw: emit its fp16 hi/lo operand planes too
    bool planes_only = false;   // ... and nothing reads the fp32 tensor: skip its store (tensor engine only)
  };

  int conv(const ConvW& w, const Tensor& in, Tensor& out, const ConvOpt& o) {
    CFB_REQUIRE(in.C == w.cin, "conv: channel mismatch for " + w.name);
    int Ho = in.H, Wo = in.W;
    if (o.mode == CONV_DOWN) { Ho = in.H / 2; Wo = in.W / 2; }
    if (o.mode == CONV_UP) { Ho = in.H * 2; Wo = in.W * 2; }
    ConvArgs a;
    a.in = in.p; a.N = in.N; a.H = in.H; a.W = in.W; a.Cin = in.C; a.Ho = Ho; a.Wo = Wo; a.Cout = w.cout;
    a.ksize = w.k; a.mode = o.mode; a.wgt_f32 = w.w_f32; a.wgt_hi = w.w_hi; a.wgt_lo = w.w_lo; a.wscale_inv = w.wscale + 1; a.bias = w.bias;
    a.in_scale = o.in_scale; a.in_shift = o.in_shift; a.in_act = o.in_act; a.residual = o.residual;
    a.out_act = o.out_act; a.sft_dec = o.sft_dec; a.sft_scale = o.sft_scale; a.sft_w = o.sft_w; a.sft_wv = o.sft_wv;
    bool use_tc = engine == 2 || (engine == 0 && n->tc_ok && tc_tiles_exact(a));
    CFB_REQUIRE(dry || !single_pass || use_tc, "conv: precision fp16 runs on the wgmma engine only: " + w.name);
    a.single_pass = single_pass;
    const bool no_f32 = o.planes_only && o.want_planes && use_tc && !o.out_ptr;
    if (o.out_ptr) {
      out.p = o.out_ptr; out.N = in.N; out.H = Ho; out.W = Wo; out.C = w.cout; out.owned = false;
      out.gn_part = nullptr; out.gn_slots = 0; out.planes = nullptr; out.p2 = nullptr; out.C1 = 0;
    } else if (no_f32) {
      out.p = nullptr; out.N = in.N; out.H = Ho; out.W = Wo; out.C = w.cout; out.owned = true;
      out.gn_part = nullptr; out.gn_slots = 0; out.planes = nullptr; out.p2 = nullptr; out.C1 = 0;
    } else {
      CFB_CHECK(alloc(out, in.N, Ho, Wo, w.cout));
    }
    a.out = out.p;
    if (use_tc && o.mode == CONV_UP) { a.wgt_hi = w.u_hi; a.wgt_lo = w.u_lo; a.wscale_inv = w.uscale + 1; }
    if (use_tc) {
      CFB_REQUIRE(tc_supported(a), "conv: shape not supported by the wgmma engine: " + w.name);
      if (o.want_stats && !o.out_ptr && tc_can_emit_stats(a)) {
        out.gn_slots = tc_tiles_per_image(a) * 4;
        CFB_CHECK(alloc_raw((void**)&out.gn_part, (size_t)in.N * out.gn_slots * 64 * sizeof(float)));
        a.gn_part = out.gn_part;
      }
      if (o.want_planes && !o.out_ptr) {
        const size_t pb = (((size_t)in.N * Ho * Wo * w.cout * 2 + 1023) / 1024 * 1024) * 2;
        CFB_CHECK(alloc_raw(&out.planes, pb));
        a.out_planes = out.planes;
      }
      // Three ways the A operand reaches the tensor core:
      //  xf   GroupNorm-affine (+ SiLU) consumers on the halo + pair engine read the fp32 activation itself -- or the two
      //       halves of a channel concatenation -- and transform + split it inside the conv kernel (tc_can_xform);
      //  raw  the producer already emitted this tensor's fp16 hi/lo planes and the consumer takes it untransformed;
      //  prep everything else: a separate operand-preparation pass over the fp32 tensor.
      const bool plain = !o.in_scale && !o.in_shift && o.in_act == IN_NONE;
      a.halo1x1 = w.k == 1 && o.mode == CONV_SAME && o.in_scale && o.in_shift && in.p;     // AttnBlock q,k,v on GroupNorm(x)
      if (a.halo1x1 && !tc_can_xform(a)) a.halo1x1 = false;
      const bool xf = in.p && tc_can_xform(a) && ((o.in_scale && o.in_shift) || (plain && !in.planes));   // plain: in-kernel split only
      const bool raw = !xf && in.planes && plain;
      const bool reuse = raw || xf;
      void* scratch = raw ? in.planes : nullptr;
      if (!reuse) CFB_CHECK(alloc_raw(&scratch, tc_scratch_bytes(a)));
      CFB_REQUIRE(in.p != nullptr || raw, "conv: planes-only input without a planes consumer: " + w.name);
      CFB_REQUIRE(in.p2 == nullptr || reuse, "conv: a two-source tensor needs the fused operand transform or its planes: " + w.name);
      if (xf) { a.in2 = in.p2; a.Cin1 = in.C1; }
      a.skip_prep = reuse;
      a.xform = xf;
      if (!dry) CFB_CHECK(conv_tc(a, scratch, n->sm_count, st));
      if (!reuse) release_raw(scratch);
    } else {
      CFB_REQUIRE(in.p != nullptr && out.p != nullptr && in.p2 == nullptr, "conv: planes-only / two-source tensor reached the fp32 engine: " + w.name);
      if (!dry) CFB_CHECK(conv_f32(a, st));
    }
    return 0;
  }

  // GroupNorm(32, C, 1e-6) statistics -> scale/shift [N,C]
  int gn(const NormW& w, const Tensor& x, float** scale, float** shift) {
    CFB_REQUIRE(x.C == w.c, "norm: channel mismatch for " + w.name);
    CFB_REQUIRE(x.p || x.gn_part, "norm: planes-only tensor without partial sums for " + w.name);
    CFB_CHECK(alloc_raw((void**)scale, (size_t)x.N * x.C * 4));
    CFB_CHECK(alloc_raw((void**)shift, (size_t)x.N * x.C * 4));
    if (x.gn_part) {   // statistics already reduced per tile by the producing conv's epilogue
      void* scr = nullptr;
      const size_t sb = gn_final_scratch_bytes(x.N, x.gn_slots);
      if (sb) CFB_CHECK(alloc_raw(&scr, sb));
      if (!dry) {
        CFB_REQUIRE(x.N <= GN_COUNTERS / 2, "GroupNorm finalize: batch larger than the ticket-counter ring");
        // ticket counters: a ring in the net's slab, zero between uses (the kernel resets them); every call takes the next N
        // so that forwards in flight on other streams never share a counter
        if (n->gn_ctr_pos + x.N > GN_COUNTERS) n->gn_ctr_pos = 0;
        unsigned* ctr = n->gn_counters + n->gn_ctr_pos;
        n->gn_ctr_pos += x.N;
        CFB_CHECK(gn_coef_from_partials(x.gn_part, x.gn_slots, w.gamma, w.beta, *scale, *shift, x.N, x.H * x.W, x.C, 32, 1e-6f, scr, ctr, st));
      }
      if (scr) release_raw(scr);
      return 0;
    }
    void* ws = nullptr;
    CFB_CHECK(alloc_raw(&ws, gn_workspace_bytes(x.N, x.H * x.W, x.C)));
    if (!dry) CFB_CHECK(gn_coef(x.p, w.gamma, w.beta, *scale, *shift, x.N, x.H * x.W, x.C, 32, 1e-6f, ws, st));
    release_raw(ws);
    return 0;
  }

  // ResBlock.forward  vqgan_arch.py:153-164
  int resblock(const ResW& r, const Tensor& x, Tensor& y, bool out_planes = false) {
    float *s1, *h1, *s2, *h2;
    CFB_CHECK(gn(r.n1, x, &s1, &h1));
    Tensor h;
    ConvOpt o1; o1.in_scale = s1; o1.in_shift = h1; o1.in_act = IN_SILU; o1.want_stats = true;
    CFB_CHECK(conv(r.c1, x, h, o1));      // conv2 reads h as fp32 (fused operand transform or prep pass): no planes of h
    release_raw(s1); release_raw(h1);
    CFB_CHECK(gn(r.n2, h, &s2, &h2));
    Tensor skip = x; skip.owned = false;
    if (r.has_out) { ConvOpt oo; CFB_CHECK(conv(r.co, x, skip, oo)); }
    ConvOpt o2; o2.in_scale = s2; o2.in_shift = h2; o2.in_act = IN_SILU; o2.residual = skip.p; o2.want_stats = true;
    o2.want_planes = out_planes;
    CFB_CHECK(conv(r.c2, h, y, o2));
    release_raw(s2); release_raw(h2);
    release(h);
    if (r.has_out) release(skip);
    return 0;
  }

  // AttnBlock.forward  vqgan_arch.py:202-226
  int attnblock(const AttnW& w, const Tensor& x, Tensor& y, bool out_planes = false) {
    CFB_REQUIRE(x.H * x.W == 256, "AttnBlock: built for the 16x16 latent");
    float *s, *h;
    CFB_CHECK(gn(w.n, x, &s, &h));
    const int C = x.C;
    const bool tc_attn = engine != 1 && n->tc_ok && x.H == 16 && x.W == 16 && C % 128 == 0;
    Tensor qkv;
    ConvOpt o; o.in_scale = s; o.in_shift = h; o.want_planes = tc_attn;
    CFB_CHECK(conv(w.qkv, x, qkv, o));
    release_raw(s); release_raw(h);
    Tensor a;
    CFB_CHECK(alloc(a, x.N, x.H, x.W, x.C));
    if (tc_attn && qkv.planes) {
      // attention core on the wgmma engine: scores = q k^T C^-1/2 and out = P v as per-image GEMMs on operand planes
      const int64_t T = (int64_t)x.N * 256;
      float* scores = nullptr;
      void *pp = nullptr, *vt = nullptr;
      CFB_CHECK(alloc_raw((void**)&scores, (size_t)T * 256 * 4));
      CFB_CHECK(alloc_raw(&pp, 2 * (((size_t)T * 256 * 2 + 1023) / 1024 * 1024)));
      CFB_CHECK(alloc_raw(&vt, 2 * (((size_t)x.N * C * 256 * 2 + 1023) / 1024 * 1024)));
      CFB_CHECK(alloc_raw(&a.planes, 2 * (((size_t)T * C * 2 + 1023) / 1024 * 1024)));
      if (!dry) {
        BmmArgs g1;
        g1.a_planes = qkv.planes; g1.a_pitch = 3 * C; g1.a_c0 = 0;
        g1.b_planes = qkv.planes; g1.b_pitch = 3 * C; g1.b_c0 = C; g1.b_rows = 256;
        g1.N = x.N; g1.K = C; g1.Cout = 256; g1.scale_dev = w.consts; g1.out = scores;
        CFB_CHECK(bmm_tc(g1, n->sm_count, st));
        CFB_CHECK(softmax256_planes(scores, pp, T, st));
        CFB_CHECK(transpose_planes(qkv.planes, x.N, 3 * C, 2 * C, C, vt, st));
        BmmArgs g2;
        g2.a_planes = pp; g2.a_pitch = 256; g2.a_c0 = 0;
        g2.b_planes = vt; g2.b_pitch = 256; g2.b_c0 = 0; g2.b_rows = C;
        g2.N = x.N; g2.K = 256; g2.Cout = C; g2.scale_dev = w.consts + 1; g2.out = a.p; g2.out_planes = a.planes;
        CFB_CHECK(bmm_tc(g2, n->sm_count, st));
      }
      release_raw(scores); release_raw(pp); release_raw(vt);
    } else {
      if (!dry)
        CFB_CHECK(attention(qkv.p, qkv.p + C, qkv.p + 2 * C, a.p, x.N, 256, 1, C, 3 * C, 3 * C, 3 * C, C,
                            1.0f / sqrtf((float)C), st));
    }
    release(qkv);
    ConvOpt op; op.residual = x.p; op.want_stats = true; op.want_planes = out_planes;
    CFB_CHECK(conv(w.proj, a, y, op));
    release(a);
    return 0;
  }

  // Fuse_sft_block.forward  codeformer_arch.py:151-157; wv: per-image w (device, [N]) in place of wgt, or null
  int fuse(const FuseW& f, const Tensor& enc_feat, const Tensor& dec, float wgt, const float* wv, Tensor& y) {
    Tensor cat;
    const bool stats_from_parts = enc_feat.gn_part && dec.gn_part && enc_feat.gn_slots == dec.gn_slots && enc_feat.C == dec.C;
    bool two_src = false;
    if (stats_from_parts && (engine == 2 || (engine == 0 && n->tc_ok))) {
      ConvArgs a1;      // conv1 of the fused ResBlock: does it run the in-kernel operand transform?
      a1.N = dec.N; a1.H = dec.H; a1.W = dec.W; a1.Cin = f.enc.c1.cin; a1.Ho = dec.H; a1.Wo = dec.W; a1.Cout = f.enc.c1.cout;
      a1.ksize = f.enc.c1.k; a1.mode = CONV_SAME;
      two_src = f.enc.has_out && tc_can_xform(a1) && enc_feat.C % 64 == 0 && dec.C % 64 == 0;
    }
    void* cat_planes = nullptr;
    if (two_src) {
      // torch.cat([enc_feat, dec]) (codeformer_arch.py:152) is never materialised in fp32: conv1 of the fused ResBlock reads the
      // two tensors through two tensor maps (fused operand transform), GroupNorm statistics come from the sources' partial
      // sums, and only the raw 1x1 conv_out needs the concatenation -- as fp16 hi/lo operand planes
      cat.p = enc_feat.p; cat.p2 = dec.p; cat.C1 = enc_feat.C;
      cat.N = dec.N; cat.H = dec.H; cat.W = dec.W; cat.C = enc_feat.C + dec.C; cat.owned = false;
      cat.gn_part = nullptr; cat.gn_slots = 0; cat.planes = nullptr;
      CFB_CHECK(alloc_raw(&cat_planes, 2 * (((size_t)cat.numel() * 2 + 1023) / 1024 * 1024)));
      cat.planes = cat_planes;
      if (!dry) CFB_CHECK(concat_planes(enc_feat.p, dec.p, cat.planes, (int64_t)dec.N * dec.H * dec.W, enc_feat.C, dec.C, st));
    } else {
      CFB_CHECK(alloc(cat, dec.N, dec.H, dec.W, enc_feat.C + dec.C));
      if (!dry) CFB_CHECK(concat_channels(enc_feat.p, dec.p, cat.p, (int64_t)dec.N * dec.H * dec.W, enc_feat.C, dec.C, st));
    }
    float* cat_part = nullptr;
    if (stats_from_parts) {
      // GroupNorm statistics of the concatenation follow from the two sources' partial sums (no extra pass)
      cat.gn_slots = dec.gn_slots;
      CFB_CHECK(alloc_raw((void**)&cat_part, (size_t)dec.N * cat.gn_slots * 64 * sizeof(float)));
      cat.gn_part = cat_part;
      if (!dry) CFB_CHECK(gn_cat_partials(enc_feat.gn_part, dec.gn_part, cat.gn_part, (int64_t)dec.N * cat.gn_slots, dec.C, st));
    }
    Tensor e;
    CFB_CHECK(resblock(f.enc, cat, e, true));      // scale.0 / shift.0 both read `e` raw: one set of planes, no prep
    if (two_src) { release_raw(cat_planes); if (cat_part) release_raw(cat_part); cat.planes = nullptr; cat.gn_part = nullptr; }
    else release(cat);
    Tensor s0, sc, h0;
    ConvOpt ol; ol.out_act = OUT_LRELU; ol.want_planes = true;      // s0 / h0 feed scale.2 / shift.2 raw
    CFB_CHECK(conv(f.s0, e, s0, ol));
    ConvOpt on;
    CFB_CHECK(conv(f.s2, s0, sc, on));
    release(s0);
    CFB_CHECK(conv(f.h0, e, h0, ol));
    release(e);
    ConvOpt of; of.sft_dec = dec.p; of.sft_scale = sc.p; of.sft_w = wgt; of.sft_wv = wv; of.want_stats = true; of.want_planes = true;
    CFB_CHECK(conv(f.h2, h0, y, of));
    release(h0); release(sc);
    return 0;
  }

  // Fidelity sweep: the decoder runs at batch N*K on the encoder results of N faces; decoder face b*K+k gets face b's
  // generator input and encoder taps, in one expand_faces launch.  Of a tap, fuse() reads the fp32 activation p and, through
  // stats_from_parts, gn_part / gn_slots; it never reads the tap's operand planes (the concatenation's planes are rebuilt
  // from p), so those are not copied.  Every copied buffer is contiguous per face, which makes face b one run of bytes at
  // b * bytes-per-face: p is NHWC [N][H][W][C]; gn_part is [N][gn_slots][64] (gn_coef_from_partials reads image n's slots at
  // n * gn_slots).  The batch-N buffers are released here, the expanded taps after their fusion (generator()).
  int expand_for_sweep(Tensor& quant, std::map<int, Tensor>& taps, int K) {
    ExpandList L;
    std::vector<std::pair<Tensor*, Tensor>> grown;      // (batch-N tensor, its expansion)
    auto grow = [&](Tensor& t) -> int {
      CFB_REQUIRE(t.p && !t.p2 && L.n + 2 <= EXPAND_MAX, "sweep: unexpected decoder input");
      Tensor e;
      CFB_CHECK(alloc(e, t.N * K, t.H, t.W, t.C));
      L.d[L.n++] = {t.p, e.p, (int64_t)t.H * t.W * t.C * 4};
      if (t.gn_part) {
        const int64_t pb = (int64_t)t.gn_slots * 64 * sizeof(float);
        e.gn_slots = t.gn_slots;
        CFB_CHECK(alloc_raw((void**)&e.gn_part, (size_t)e.N * pb));
        L.d[L.n++] = {t.gn_part, e.gn_part, pb};
      }
      grown.push_back({&t, e});
      return 0;
    };
    const int N = quant.N;
    CFB_CHECK(grow(quant));
    for (auto& kv : taps) CFB_CHECK(grow(kv.second));
    if (!dry) CFB_CHECK(expand_faces(L, N, K, st));
    for (auto& g : grown) {       // the sources are free once their one reader is enqueued
      release(*g.first);
      *g.first = g.second;
    }
    return 0;
  }

  // conv1 of a fused ResBlock at this shape: fused operand transform available?
  bool xf_ok(int N, int H, int W, const ConvW& w) const {
    if (!(engine == 2 || (engine == 0 && n->tc_ok))) return false;
    ConvArgs a;
    a.N = N; a.H = H; a.W = W; a.Ho = H; a.Wo = W; a.Cin = w.cin; a.Cout = w.cout; a.ksize = w.k; a.mode = CONV_SAME;
    return tc_can_xform(a);
  }
  // Does a consumer of block i's output read it RAW through the tensor engine (then the producer also emits its fp16 hi/lo
  // operand planes)?  Down/Upsample convs and a ResBlock's 1x1 conv_out do.  GroupNorm (+SiLU) consumers -- a ResBlock's
  // conv1, a norm -> conv pair -- read the fp32 tensor itself (fused operand transform or prep pass).
  bool next_takes_planes(const std::vector<Block>& bl, size_t i) const {
    if (!(engine == 2 || (engine == 0 && n->tc_ok))) return false;
    if (i + 1 >= bl.size()) return false;
    const Block& nb = bl[i + 1];
    if (nb.kind == B_DOWN || nb.kind == B_UP) return true;
    if (nb.kind == B_RES) return nb.res_w.has_out;
    return false;
  }

  // Encoder.forward (+ the taps of codeformer_arch.py:226-230).  x_nchw is the caller's image.
  int encoder(const float* x_nchw, int B, Tensor& z, std::map<int, Tensor>* taps, const std::vector<int>& tap_blocks) {
    const cfb_config& c = n->cfg;
    Tensor x;
    CFB_CHECK(alloc(x, B, c.img_size, c.img_size, c.nf));
    // on the tensor-core path every GroupNorm takes its statistics from partial sums of the producing kernel's epilogue: the
    // first conv emits them too (no pass over the 64-channel full-resolution tensor for the first ResBlock's norm1)
    const int64_t hw = (int64_t)c.img_size * c.img_size;
    if (engine != 1 && n->tc_ok && c.nf == 64 && hw % 256 == 0 && B <= GN_COUNTERS / 2) {
      x.gn_slots = (int)(hw / 32);
      CFB_CHECK(alloc_raw((void**)&x.gn_part, (size_t)B * x.gn_slots * 64 * sizeof(float)));
    }
    if (!dry) {
      if (in_u8)
        CFB_CHECK(conv_first_u8(in_u8, n->enc[0].conv.w_f32, n->enc[0].conv.bias, x.p, B, c.img_size, c.img_size, c.nf, st, x.gn_part,
                                in_u8_orig));
      else CFB_CHECK(conv_first(x_nchw, n->enc[0].conv.w_f32, n->enc[0].conv.bias, x.p, B, c.img_size, c.img_size, c.nf, st, x.gn_part));
    }
    CFB_CHECK(capture("enc.0", x));
    float *ps = nullptr, *ph = nullptr;   // pending GroupNorm of a 'norm' block
    for (size_t i = 1; i < n->enc.size(); ++i) {
      const Block& b = n->enc[i];
      const bool pl = next_takes_planes(n->enc, i);
      Tensor y;
      switch (b.kind) {
        case B_RES: CFB_CHECK(resblock(b.res_w, x, y, pl)); break;
        case B_ATTN: CFB_CHECK(attnblock(b.attn, x, y, pl)); break;
        case B_DOWN: { ConvOpt o; o.mode = CONV_DOWN; o.want_stats = true; o.want_planes = pl; CFB_CHECK(conv(b.conv, x, y, o)); break; }
        case B_NORM: CFB_CHECK(gn(b.norm, x, &ps, &ph)); continue;   // consumed by the next conv
        case B_CONV: {
          ConvOpt o; o.in_scale = ps; o.in_shift = ph;
          o.want_planes = (i + 1 == n->enc.size()) && n->cfg.kind == 1;   // lq_feat feeds feat_emb raw
          CFB_CHECK(conv(b.conv, x, y, o));
          if (ps) { release_raw(ps); release_raw(ph); ps = ph = nullptr; }
          break;
        }
        default: CFB_REQUIRE(false, "encoder: unexpected block kind");
      }
      release(x);
      x = y;
      CFB_CHECK(capture("enc." + std::to_string(i), x));
      for (int tb : tap_blocks)
        if ((int)i == tb && taps) { x.owned = false; (*taps)[x.W] = x; (*taps)[x.W].owned = true; }
    }
    z = x;
    return 0;
  }

  // Generator.forward with the SFT fusion of codeformer_arch.py:272-277; writes NCHW into out_nchw.  wv (device, [N]): one w
  // per image; the fusion then runs whatever the values, and an image with w <= 0 (or NaN) blends with 0, i.e. keeps dec
  int generator(Tensor x, float* out_nchw, std::map<int, Tensor>* taps, const std::vector<int>& fuse_blocks, float w,
                const float* wv = nullptr) {
    const bool fusing = taps && (w > 0.f || wv);
    // fp16 precision: the convs of every generator block and of the fusion run single pass, except the AttnBlocks' q,k,v and
    // proj_out (about 2 of 586 GF per face); conv_last is the fp32 SIMT conv in both precisions
    const bool p1 = n->precision == 1;
    float *ps = nullptr, *ph = nullptr;
    for (size_t i = 0; i < n->gen.size(); ++i) {
      const Block& b = n->gen[i];
      single_pass = p1 && b.kind != B_ATTN;
      bool pl = next_takes_planes(n->gen, i);
      if (fusing)
        for (int fb : fuse_blocks)
          if ((int)i == fb) pl = false;      // consumed by the fusion (concat + SFT read fp32); the fused output emits its own
      Tensor y;
      switch (b.kind) {
        case B_RES: CFB_CHECK(resblock(b.res_w, x, y, pl)); break;
        case B_ATTN: CFB_CHECK(attnblock(b.attn, x, y, pl)); break;
        case B_UP: { ConvOpt o; o.mode = CONV_UP; o.want_stats = true; o.want_planes = pl; CFB_CHECK(conv(b.conv, x, y, o)); break; }
        case B_NORM: CFB_CHECK(gn(b.norm, x, &ps, &ph)); continue;
        case B_CONV:
          if (i + 1 == n->gen.size()) {
            if (!dry) {
              if (out_u8 && inpaint)
                CFB_CHECK(conv_last_u8_inpaint(x.p, ps, ph, b.conv.w_f32, b.conv.bias, in_u8, out_u8, x.N, x.H, x.W, x.C, st));
              else if (out_u8) CFB_CHECK(conv_last_u8(x.p, ps, ph, b.conv.w_f32, b.conv.bias, out_u8, x.N, x.H, x.W, x.C, st));
              else CFB_CHECK(conv_last(x.p, ps, ph, b.conv.w_f32, b.conv.bias, out_nchw, x.N, x.H, x.W, x.C, st));
            }
            if (ps) { release_raw(ps); release_raw(ph); ps = ph = nullptr; }
            release(x);
            return 0;
          } else {
            ConvOpt o; o.in_scale = ps; o.in_shift = ph; o.want_stats = true; o.want_planes = pl;
            CFB_CHECK(conv(b.conv, x, y, o));
            if (ps) { release_raw(ps); release_raw(ph); ps = ph = nullptr; }
          }
          break;
        default: CFB_REQUIRE(false, "generator: unexpected block kind");
      }
      release(x);
      x = y;
      CFB_CHECK(capture("gen." + std::to_string(i), x));
      if (fusing)
        for (int fb : fuse_blocks)
          if ((int)i == fb) {
            auto it = taps->find(x.W);
            CFB_REQUIRE(it != taps->end(), "fusion: encoder feature missing");
            auto fw = n->fuse.find(x.W);
            CFB_REQUIRE(fw != n->fuse.end(), "fusion: no Fuse_sft_block for this size");
            Tensor fz;
            single_pass = p1;
            CFB_CHECK(fuse(fw->second, it->second, x, w, wv, fz));
            release(x);
            release(it->second);
            x = fz;
            CFB_CHECK(capture("fuse." + std::to_string(x.W), x));
          }
    }
    CFB_REQUIRE(false, "generator: plan does not end with a conv");
    return 1;
  }

  // TransformerSALayer.forward x9 + idx_pred_layer  codeformer_arch.py:235-245
  int transformer(const Tensor& lq, float* logits_out) {
    const cfb_config& c = n->cfg;
    const int B = lq.N, S = lq.H * lq.W, E = c.dim_embd, T = B * S;
    CFB_REQUIRE(S == c.latent_size, "transformer: token count != latent_size");
    Tensor tok = lq; tok.owned = false;   // [B,16,16,256] == tokens [T,256]
    Tensor x;
    { ConvOpt o; CFB_CHECK(conv(n->feat_emb, tok, x, o)); }
    // On the tensor engine every LayerNorm / attention / GELU output of a layer is only ever a GEMM operand: the producing
    // kernel writes it straight as fp16 hi/lo operand planes (no fp32 copy, no operand-preparation pass).
    const bool tcp = engine != 1 && n->tc_ok;
    const size_t plE = 2 * (((size_t)T * E * 2 + 1023) / 1024 * 1024);
    auto planes_tensor = [&](Tensor& t, int C, size_t bytes) -> int {
      t.p = nullptr; t.N = B; t.H = lq.H; t.W = lq.W; t.C = C; t.owned = true; t.gn_part = nullptr; t.gn_slots = 0;
      t.p2 = nullptr; t.C1 = 0; t.planes = nullptr;
      return alloc_raw(&t.planes, bytes);
    };
    for (const LayerW& L : n->layers) {
      Tensor t2, qkin, qk, v, a, x2, hdn, x3;
      if (tcp) {
        CFB_CHECK(planes_tensor(t2, E, plE));
        CFB_CHECK(planes_tensor(qkin, E, plE));
        if (!dry) CFB_CHECK(layer_norm_planes(x.p, L.n1.gamma, L.n1.beta, t2.planes, qkin.planes, n->position_emb, S, T, E, st));
      } else {
        CFB_CHECK(alloc(t2, B, lq.H, lq.W, E));
        CFB_CHECK(alloc(qkin, B, lq.H, lq.W, E));
        if (!dry) CFB_CHECK(layer_norm(x.p, L.n1.gamma, L.n1.beta, t2.p, qkin.p, n->position_emb, S, T, E, st));
      }
      { ConvOpt o; o.want_planes = tcp; o.planes_only = tcp; CFB_CHECK(conv(L.qk, qkin, qk, o)); }
      { ConvOpt o; o.want_planes = tcp; o.planes_only = tcp; CFB_CHECK(conv(L.v, t2, v, o)); }
      release(qkin); release(t2);
      if (tcp) {
        // nn.MultiheadAttention core (codeformer_arch.py:126) on the wgmma engine: per (image, head) GEMMs on operand planes --
        // scores = (q_h k_h^T) * d^-1/2 (K = 64, the power-of-two scale commutes exactly with the product), softmax -> planes
        // of the probabilities, out_h = P v_h written as the operand planes of out_proj (no fp32 copy of anything)
        const int Hh = c.n_head, dh = E / c.n_head;
        CFB_CHECK(planes_tensor(a, E, plE));
        float* scores = nullptr;
        void *pp = nullptr, *vt = nullptr;
        const int64_t rows = (int64_t)B * Hh * S;
        CFB_CHECK(alloc_raw((void**)&scores, (size_t)rows * S * 4));
        CFB_CHECK(alloc_raw(&pp, 2 * (((size_t)rows * S * 2 + 1023) / 1024 * 1024)));
        CFB_CHECK(alloc_raw(&vt, 2 * (((size_t)B * E * S * 2 + 1023) / 1024 * 1024)));
        if (!dry) {
          BmmArgs g1;
          g1.a_planes = qk.planes; g1.a_pitch = 2 * E; g1.a_c0 = 0; g1.a_c_head = dh;
          g1.b_planes = qk.planes; g1.b_pitch = 2 * E; g1.b_c0 = E; g1.b_c_head = dh; g1.b_rows = S;
          g1.N = B; g1.heads = Hh; g1.K = dh; g1.Cout = S; g1.scale_dev = n->mha_consts; g1.out = scores; g1.out_per_head = true;
          CFB_CHECK(bmm_tc(g1, n->sm_count, st));
          CFB_CHECK(softmax256_planes(scores, pp, rows, st));
          CFB_CHECK(transpose_planes(v.planes, B, E, 0, E, vt, st));
          BmmArgs g2;
          g2.a_planes = pp; g2.a_pitch = S; g2.a_c0 = 0; g2.a_img_per_head = true;
          g2.b_planes = vt; g2.b_pitch = S; g2.b_c0 = 0; g2.b_rows = E; g2.b_r_head = dh;
          g2.N = B; g2.heads = Hh; g2.K = S; g2.Cout = dh; g2.scale_dev = n->mha_consts + 1; g2.out = nullptr; g2.out_planes = a.planes;
          g2.out_per_head = false; g2.o_c_head = dh;
          CFB_CHECK(bmm_tc(g2, n->sm_count, st));
        }
        release_raw(scores); release_raw(pp); release_raw(vt);
      } else {
        CFB_CHECK(alloc(a, B, lq.H, lq.W, E));
        if (!dry)
          CFB_CHECK(attention(qk.p, qk.p + E, v.p, a.p, B, S, c.n_head, E / c.n_head, 2 * E, 2 * E, E, E,
                              sqrtf(1.0f / (float)(E / c.n_head)), st, nullptr));
      }
      release(qk); release(v);
      { ConvOpt o; o.residual = x.p; CFB_CHECK(conv(L.o, a, x2, o)); }
      release(a); release(x);
      if (tcp) {
        CFB_CHECK(planes_tensor(t2, E, plE));
        if (!dry) CFB_CHECK(layer_norm_planes(x2.p, L.n2.gamma, L.n2.beta, t2.planes, nullptr, nullptr, 0, T, E, st));
      } else {
        CFB_CHECK(alloc(t2, B, lq.H, lq.W, E));
        if (!dry) CFB_CHECK(layer_norm(x2.p, L.n2.gamma, L.n2.beta, t2.p, nullptr, nullptr, 0, T, E, st));
      }
      { ConvOpt o; o.out_act = OUT_GELU; o.want_planes = tcp; o.planes_only = tcp; CFB_CHECK(conv(L.l1, t2, hdn, o)); }
      release(t2);
      { ConvOpt o; o.residual = x2.p; CFB_CHECK(conv(L.l2, hdn, x3, o)); }
      release(hdn); release(x2);
      x = x3;
      CFB_CHECK(capture("ft." + std::to_string((int)(&L - &n->layers[0])), x));
    }
    Tensor t2, lg;
    if (tcp) {
      CFB_CHECK(planes_tensor(t2, E, plE));
      if (!dry) CFB_CHECK(layer_norm_planes(x.p, n->idx_norm.gamma, n->idx_norm.beta, t2.planes, nullptr, nullptr, 0, T, E, st));
    } else {
      CFB_CHECK(alloc(t2, B, lq.H, lq.W, E));
      if (!dry) CFB_CHECK(layer_norm(x.p, n->idx_norm.gamma, n->idx_norm.beta, t2.p, nullptr, nullptr, 0, T, E, st));
    }
    release(x);
    { ConvOpt o; o.out_ptr = logits_out; CFB_CHECK(conv(n->idx_lin, t2, lg, o)); }
    release(t2);
    return 0;
  }
};

// The prepared weights live on ONE device; a forward issued while another device is current would launch kernels there
// on foreign memory.  Also the place where an asynchronous failure of an earlier launch is reported (never silently lost).
static int check_device(cfb_net* n) {
  int dev = -1;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_REQUIRE(dev == n->device, "the net was prepared on CUDA device " + std::to_string(n->device) + " but device " +
                                    std::to_string(dev) + " is current (call net.to(device) / cfb_net_prepare again)");
  return async_status_check("forward");
}

static std::vector<int> tap_blocks_of(const cfb_config& c, bool encoder) {
  // fuse_encoder_block / fuse_generator_block  codeformer_arch.py:204-206
  static const int enc_of[6][2] = {{512, 2}, {256, 5}, {128, 8}, {64, 11}, {32, 14}, {16, 18}};
  static const int gen_of[6][2] = {{16, 6}, {32, 9}, {64, 12}, {128, 15}, {256, 18}, {512, 21}};
  std::vector<int> r;
  for (int i = 0; i < c.n_connect; ++i)
    for (auto& e : (encoder ? enc_of : gen_of))
      if (e[0] == c.connect[i]) r.push_back(e[1]);
  return r;
}

static int codeformer_forward_impl(cfb_net* n, const float* x, float* out, float* logits, float* lq_feat,
                                   int64_t* top_idx, int B, float w, int adain, int code_only, void* ws, int64_t ws_bytes,
                                   cudaStream_t st, bool dry, const unsigned char* x_u8 = nullptr,
                                   unsigned char* out_u8 = nullptr, bool inpaint = false, const float* w_dev = nullptr,
                                   int sweep_k = 1) {
  CFB_REQUIRE(n->cfg.kind == 1, "net was created as VQAutoEncoder");
  CFB_REQUIRE(dry || n->prepared, "cfb_net_prepare has not been called");
  if (!dry) CFB_CHECK(check_device(n));
  CFB_REQUIRE(dry || n->precision == 0 || (n->engine != 1 && n->tc_ok),
              "precision fp16 (single pass) runs on the wgmma engine only: use engine 'auto' or 'tc' on an sm_90 device");
  CFB_REQUIRE(B >= 0, "negative batch");
  if (B == 0) return 0;
  n->arena.reset(ws, (size_t)ws_bytes, dry);
  Fwd f{n, st, n->arena, dry, n->engine};
  f.in_u8 = x_u8; f.out_u8 = out_u8; f.inpaint = inpaint;
  const cfb_config& c = n->cfg;
  std::map<int, Tensor> taps;
  Tensor lq;
  // codeformer_arch.py:276 -- features are only consumed when w>0; a per-image w (w_dev) always runs the fusion
  const bool want_taps = (w > 0.f || w_dev) && !code_only;
  CFB_CHECK(f.encoder(x, B, lq, want_taps ? &taps : nullptr, tap_blocks_of(c, true)));
  const int T = B * lq.H * lq.W;
  float* logits_buf = logits;
  if (!logits_buf) CFB_CHECK(f.alloc_raw((void**)&logits_buf, (size_t)T * c.codebook_size * 4));
  CFB_CHECK(f.transformer(lq, logits_buf));
  if (lq_feat && !dry) CFB_CHECK(nhwc_to_nchw(lq.p, lq_feat, B, lq.C, lq.H * lq.W, st));
  if (code_only) {                                     // codeformer_arch.py:247-249
    if (top_idx && !dry) CFB_CHECK(argmax_gather(logits_buf, n->codebook, top_idx, nullptr, T, c.codebook_size, c.emb_dim, st));
    return 0;
  }
  CFB_REQUIRE(out != nullptr || out_u8 != nullptr, "out must not be NULL unless code_only");
  // softmax -> topk(1) -> get_codebook_feat  (:257-259)
  Tensor quant;
  CFB_CHECK(f.alloc(quant, B, lq.H, lq.W, c.emb_dim));
  if (!dry) CFB_CHECK(argmax_gather(logits_buf, n->codebook, top_idx, quant.p, T, c.codebook_size, c.emb_dim, st));
  if (adain) {                                         // :265-266
    Tensor q2;
    CFB_CHECK(f.alloc(q2, B, lq.H, lq.W, c.emb_dim));
    if (!dry) CFB_CHECK(adain_nhwc(quant.p, lq.p, q2.p, B, lq.H * lq.W, c.emb_dim, st));
    f.release(quant);
    quant = q2;
  }
  CFB_CHECK(f.capture("quant", quant));
  f.release(lq);
  // fidelity sweep (cfb_codeformer_sweep_u8): w_dev holds B*K weights, face-major; the decoder runs at batch B*K
  if (sweep_k > 1) CFB_CHECK(f.expand_for_sweep(quant, taps, sweep_k));
  CFB_CHECK(f.generator(quant, out, want_taps ? &taps : nullptr, tap_blocks_of(c, false), w, w_dev));
  return 0;
}

static int vqae_forward_impl(cfb_net* n, const float* x, float* out, int64_t* idx, float* stats, float* onehot, int B,
                             void* ws, int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_REQUIRE(dry || n->prepared, "cfb_net_prepare has not been called");
  if (B == 0) return 0;
  if (!dry) CFB_CHECK(check_device(n));
  CFB_REQUIRE(dry || n->precision == 0 || (n->engine != 1 && n->tc_ok),
              "precision fp16 (single pass) runs on the wgmma engine only: use engine 'auto' or 'tc' on an sm_90 device");
  n->arena.reset(ws, (size_t)ws_bytes, dry);
  Fwd f{n, st, n->arena, dry, n->engine};
  const cfb_config& c = n->cfg;
  Tensor z;
  CFB_CHECK(f.encoder(x, B, z, nullptr, {}));
  const int T = B * z.H * z.W;
  Tensor zq;
  CFB_CHECK(f.alloc(zq, B, z.H, z.W, z.C));
  int64_t* idx_buf = idx;
  float* stats_buf = stats;
  if (!idx_buf) CFB_CHECK(f.alloc_raw((void**)&idx_buf, (size_t)T * 8));
  if (!stats_buf) CFB_CHECK(f.alloc_raw((void**)&stats_buf, 16));
  bool tc_vq = false;
  {
    ConvArgs probe;
    probe.N = B; probe.H = z.H; probe.W = z.W; probe.Cin = z.C; probe.Ho = z.H; probe.Wo = z.W; probe.Cout = c.codebook_size;
    probe.ksize = 1; probe.mode = CONV_SAME;
    tc_vq = n->engine != 1 && n->tc_ok && tc_tiles_exact(probe);
  }
  if (tc_vq) {
    // distance GEMM z.E^T on the wgmma engine, then the warp-shuffle argmin over the dot products
    Tensor dots;
    Fwd::ConvOpt o;
    CFB_CHECK(f.conv(n->vq_code, z, dots, o));
    void* vws = nullptr;
    CFB_CHECK(f.alloc_raw(&vws, vq_select_workspace_bytes(T, c.codebook_size)));
    if (!dry)
      CFB_CHECK(vq_select_from_dots(z.p, n->codebook, dots.p, T, z.C, c.codebook_size, c.beta, idx_buf, zq.p, stats_buf, onehot, vws, st));
    f.release(dots);
  } else {
    void* vws = nullptr;
    CFB_CHECK(f.alloc_raw(&vws, vq_workspace_bytes(T, z.C, c.codebook_size)));
    if (!dry) CFB_CHECK(vq_nearest(z.p, n->codebook, T, z.C, c.codebook_size, c.beta, idx_buf, zq.p, stats_buf, onehot, vws, st));
  }
  f.release(z);
  CFB_CHECK(f.generator(zq, out, nullptr, {}, 0.f));
  return 0;
}

// Encoder.forward alone (vqgan_arch.py:269-273) for either network kind; the generator and, for CodeFormer, the Transformer
// never run.  B images are encoded.  x_u8 (uint8 HWC BGR faces) replaces x; with n_orig in (0, B), images b >= n_orig are face
// b - n_orig mirrored (conv_first_u8).  latent_nchw [B,D,h,w] is optional when idx is given.  idx [B*h*w]: the code selection
// of VectorQuantizer.forward on that latent, through the same library entry that module calls (cfb_vq_nearest_fast where
// cfb_vq_fast_supported, else cfb_vq_nearest), so the indices equal quantize(encoder(x)) bit for bit.
static int encoder_impl(cfb_net* n, const float* x, const unsigned char* x_u8, int n_orig, float* latent_nchw, int64_t* idx,
                        int B, void* ws, int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_REQUIRE(dry || n->prepared, "cfb_net_prepare has not been called");
  CFB_REQUIRE(B >= 0, "negative batch");
  if (B == 0) return 0;
  if (!dry) CFB_CHECK(check_device(n));
  n->arena.reset(ws, (size_t)ws_bytes, dry);
  Fwd f{n, st, n->arena, dry, n->engine};
  f.in_u8 = x_u8;
  f.in_u8_orig = n_orig;
  const cfb_config& c = n->cfg;
  Tensor z;
  CFB_CHECK(f.encoder(x, B, z, nullptr, {}));
  const int H = z.H, W = z.W, D = z.C, K = c.codebook_size;
  float* zn = latent_nchw;
  if (!zn) CFB_CHECK(f.alloc_raw((void**)&zn, (size_t)B * D * H * W * 4));
  if (!dry) CFB_CHECK(nhwc_to_nchw(z.p, zn, B, D, H * W, st));
  f.release(z);
  if (!idx) return 0;
  // the quantizer's z_q and statistics are scratch here; the workspace holds either selection path
  const size_t zq_b = ((size_t)B * D * H * W * 4 + 1023) / 1024 * 1024;
  const size_t prep_b = ((size_t)cfb_vq_prepared_bytes(K, D) + 1023) / 1024 * 1024;
  const size_t fast_b = prep_b + (size_t)cfb_vq_fast_workspace_bytes(B, H * W, D, K);
  const size_t slow_b = (size_t)cfb_vq_workspace_bytes(B, H * W, D, K);
  char* scratch = nullptr;
  CFB_CHECK(f.alloc_raw((void**)&scratch, zq_b + 1024 + std::max(fast_b, slow_b)));
  if (dry) return 0;
  float* zq = (float*)scratch;
  float* stats = (float*)(scratch + zq_b);
  char* vws = scratch + zq_b + 1024;
  if (cfb_vq_fast_supported(B, H, W, D, K)) {
    CFB_CHECK(cfb_vq_prepare(n->codebook, K, D, vws, (int64_t)prep_b, st));
    CFB_CHECK(cfb_vq_nearest_fast(zn, n->codebook, vws, B, H, W, D, K, c.beta, zq, idx, stats, nullptr, vws + prep_b,
                                  (int64_t)(fast_b - prep_b), st));
  } else {
    CFB_CHECK(cfb_vq_nearest(zn, n->codebook, B, H, W, D, K, c.beta, zq, idx, stats, nullptr, vws, (int64_t)slow_b, st));
  }
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// RRDBNet (SURVEY.md section 8 row f4): the background / face upsampler behind RealESRGANer.enhance
//   /root/reference/basicsr/archs/rrdbnet_arch.py:9-120, call sites /root/reference/basicsr/utils/realesrgan_utils.py:100-175
// 23 RRDBs of three ResidualDenseBlocks: every 3x3 conv runs on the wgmma engine in its generalised fused-transform form
// (fp32 activation read in place, fp16 hi/lo split inside the kernel, any H x W, zero padding by TMA out-of-bounds fill).
// The dense concatenations torch.cat((x, x1, ..)) never exist: one NHWC buffer of 192 channels per block holds
// [x | x1 | x2 | x3 | x4]; conv_k reads its 64-aligned channel window (weights are zero beyond the real Cin) and writes its
// 32 growth channels at their offset; conv5 writes `x5*0.2 + x` (0.2 folded into the weight scale and bias) into the next
// block's buffer, and the third block of an RRDB also applies `*0.2 + x_rrdb` in the same epilogue.
// =========================================================================================================
namespace cfb {
// One conv of the plan of a network on the wgmma engines (RRDBNet, ParseNet, RetinaFace, YOLOv5-face).  The split weights
// are zero-padded to 64-aligned channel counts; the per-tap engine and the generalised halo engine both read those.
struct GenConv {
  std::string name;
  int cin = 0, cout = 0;            // real sizes
  int cin_p = 0, cout_p = 0;        // 64-aligned sizes of the split weights
  int k = 3, stride = 1;
  bool gen = true;                  // generalised halo engine (3x3 stride 1); otherwise the per-tap engine
  std::string bn;                   // detectors: prefix of the BatchNorm folded into the weights ("": none)
  float out_scale = 1.f;            // constant folded into 2^-k and the bias
  bool up = false;                  // nearest x2 + conv (four parity convs)
  int kh = 0, kw = 0, pad_h = 0, pad_w = 0;   // explicit kh x kw window (kh > 0, per-tap engine; k is then not read)
  __half* w_hi = nullptr; __half* w_lo = nullptr; float* bias = nullptr; float* wscale = nullptr;
  int taps() const { return kh > 0 ? kh * kw : k * k; }
};

static GenConv plan_conv(const std::string& name, int cin, int cout, int k = 3, int stride = 1) {
  GenConv c;
  c.name = name; c.cin = cin; c.cout = cout; c.k = k; c.stride = stride; c.gen = k == 3 && stride == 1;
  c.cin_p = (cin + 63) / 64 * 64; c.cout_p = (cout + 63) / 64 * 64;
  return c;
}

// slab space of the planned convs: their split weights, the largest zero-padded fp32 weight (the size of the pad and the
// BatchNorm-fold scratch) and the widest output (the folded-bias scratch)
struct SlabPlan {
  size_t convs = 0, padmax = 0;
  int cout_max = 0;
  void add(const GenConv& c) {
    const size_t wn = (size_t)c.cout_p * c.cin_p * (c.up ? 16 : c.taps());
    convs += 2 * align256(wn * 2) + align256((size_t)c.cout_p * 4) + 256;
    padmax = std::max(padmax, (size_t)c.cout_p * c.cin_p * c.taps() * 4);
    cout_max = std::max(cout_max, c.cout_p);
  }
  size_t bytes() const { return convs + 2 * align256(padmax) + align256((size_t)cout_max * 4); }
};

// The split weights of one conv, carved from `p`: zero-pad the [cout][cin][k][k] fp32 weight to [cout_p][cin_p][k][k], split
// it into the engine's fp16 hi/lo planes (the four parity 2x2 sets for `up`), copy the bias (b == null: zero) and fold
// out_scale into 2^-k and the bias.
static int prepare_conv(GenConv& c, const float* w, const float* b, float* pad, char*& p, cudaStream_t st) {
  auto take = [&](size_t bytes) { char* r = p; p += align256(bytes); return r; };
  const int taps = c.taps();
  const size_t wn = (size_t)c.cout_p * c.cin_p * (c.up ? 16 : taps);
  c.w_hi = (__half*)take(wn * 2); c.w_lo = (__half*)take(wn * 2);
  c.bias = (float*)take((size_t)c.cout_p * 4); c.wscale = (float*)take(8);
  CFB_CUDA(cudaMemsetAsync(pad, 0, (size_t)c.cout_p * c.cin_p * taps * 4, st));
  CFB_CUDA(cudaMemcpy2DAsync(pad, (size_t)c.cin_p * taps * 4, w, (size_t)c.cin * taps * 4, (size_t)c.cin * taps * 4, c.cout,
                             cudaMemcpyDeviceToDevice, st));
  if (c.up) CFB_CHECK(tc_split_weights_up4(pad, c.w_hi, c.w_lo, c.cout_p, c.cin_p, c.wscale, st));
  else CFB_CHECK(tc_split_weights_taps(pad, c.w_hi, c.w_lo, c.cout_p, c.cin_p, taps, c.wscale, st));
  CFB_CUDA(cudaMemsetAsync(c.bias, 0, (size_t)c.cout_p * 4, st));
  if (b) CFB_CUDA(cudaMemcpyAsync(c.bias, b, (size_t)c.cout * 4, cudaMemcpyDeviceToDevice, st));
  if (c.out_scale != 1.f) {
    CFB_CHECK(scale_scalar(c.wscale + 1, c.out_scale, st));
    CFB_CHECK(scale_vec(c.bias, c.cout, c.out_scale, st));
  }
  return 0;
}

// The slab of one prepare call, carved in order; it starts with the scratch of the weight preparation.
struct WeightPrep {
  NetCore& net;
  cudaStream_t st;
  char* p;
  float *pad, *fold_w, *fold_b;
  WeightPrep(NetCore& n, const SlabPlan& plan, cudaStream_t s) : net(n), st(s), p((char*)n.slab) {
    pad = (float*)take(plan.padmax);
    fold_w = (float*)take(plan.padmax);
    fold_b = (float*)take((size_t)plan.cout_max * 4);
  }
  char* take(size_t bytes) { char* r = p; p += align256(bytes); return r; }
  // eval-mode BatchNorm `bn` (weight, bias, running_mean, running_var) folded into the conv weight `w_name` -> fold_w, fold_b
  int fold(const std::string& w_name, const std::string& bn, int cout, int per_out, float eps = 1e-5f) {
    const float* w = net.param(w_name, (int64_t)cout * per_out);
    const float* g = net.param(bn + "weight", cout);
    const float* be = net.param(bn + "bias", cout);
    const float* mu = net.param(bn + "running_mean", cout);
    const float* var = net.param(bn + "running_var", cout);
    if (!w || !g || !be || !mu || !var) return 1;
    return fold_bn(w, g, be, mu, var, eps, fold_w, fold_b, cout, per_out, st);     // nn.BatchNorm2d default eps 1e-5
  }
  int conv(GenConv& c, const float* w, const float* b) { return prepare_conv(c, w, b, pad, p, st); }
};
}  // namespace cfb

struct cfb_rrdb : cfb::NetCore {
  cfb_rrdb() : NetCore("RRDBNet", "rrdb") {}
  int in_ch = 3, out_ch = 3, scale = 4, feat = 64, blocks = 23, grow = 32;
  std::vector<cfb::GenConv> convs;      // [blocks*15] dense convs, then conv_body, conv_up1, conv_up2, conv_hr
  float* first_w = nullptr; float* first_b = nullptr;   // conv_first  [tap][cin][64]
  float* last_w = nullptr; float* last_b = nullptr;     // conv_last   [tap][64][4]
};

namespace cfb {

static int rrdb_prepare(cfb_rrdb* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  n->convs.clear();
  const int us = n->scale == 2 ? 2 : (n->scale == 1 ? 4 : 1);
  const int cin_first = n->in_ch * us * us;
  for (int b = 0; b < n->blocks; ++b)
    for (int r = 1; r <= 3; ++r)
      for (int k = 1; k <= 5; ++k) {
        const std::string nm = "body." + std::to_string(b) + ".rdb" + std::to_string(r) + ".conv" + std::to_string(k);
        n->convs.push_back(plan_conv(nm, n->feat + (k - 1) * n->grow, k == 5 ? n->feat : n->grow));
        n->convs.back().out_scale = k == 5 ? 0.2f : 1.f;
      }
  for (const std::string nm : {"conv_body", "conv_up1", "conv_up2", "conv_hr"}) {
    n->convs.push_back(plan_conv(nm, n->feat, n->feat));
    n->convs.back().up = nm == "conv_up1" || nm == "conv_up2";
  }
  SlabPlan plan;
  for (const GenConv& c : n->convs) plan.add(c);
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256((size_t)9 * cin_first * 64 * 4) + 256 + align256((size_t)9 * 64 * 4 * 4) + 256));
  WeightPrep wp(*n, plan, st);
  for (GenConv& c : n->convs) {
    const float* w = n->param(c.name + ".weight", (int64_t)c.cout * c.cin * 9);
    const float* b = n->param(c.name + ".bias", c.cout);
    if (!w || !b) return 1;
    CFB_CHECK(wp.conv(c, w, b));
  }
  {
    const float* w = n->param("conv_first.weight", (int64_t)n->feat * cin_first * 9);
    const float* b = n->param("conv_first.bias", n->feat);
    if (!w || !b) return 1;
    n->first_w = (float*)wp.take((size_t)9 * cin_first * 64 * 4); n->first_b = (float*)wp.take(256);
    CFB_CHECK(relayout_oihw_to_tck(w, n->first_w, n->feat, cin_first, 3, st));
    CFB_CUDA(cudaMemcpyAsync(n->first_b, b, (size_t)n->feat * 4, cudaMemcpyDeviceToDevice, st));
  }
  {
    const float* w = n->param("conv_last.weight", (int64_t)n->out_ch * n->feat * 9);
    const float* b = n->param("conv_last.bias", n->out_ch);
    if (!w || !b) return 1;
    n->last_w = (float*)wp.take((size_t)9 * 64 * 4 * 4); n->last_b = (float*)wp.take(256);
    CFB_CHECK(relayout_thin_out(w, n->last_w, n->out_ch, st));
    CFB_CUDA(cudaMemcpyAsync(n->last_b, b, (size_t)n->out_ch * 4, cudaMemcpyDeviceToDevice, st));
  }
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

struct GenLaunch {          // one generalised conv: src window -> destination slice
  const GenConv* c; const float* in; int in_pitch; int H, W; int N;
  float* out; int out_pitch, out_c0; int act;
  const float* res = nullptr; int res_pitch = 0; const float* res2 = nullptr; int res2_pitch = 0; float post = 1.f;
  int pad_mode = 0; bool sub = false;
  bool single_pass = false;   // fp16 operands, one product per k-step (ConvArgs::single_pass)
  const float* in_scale = nullptr; const float* in_shift = nullptr;   // per-(image, channel) affine of the input (no activation)
  float prelu = 0.f;          // act == OUT_PRELU: the slope
};
static int gen_conv(const GenLaunch& g, int sm_count, cudaStream_t st) {
  ConvArgs a;
  a.in = g.in; a.N = g.N; a.H = g.H; a.W = g.W; a.Cin = g.c->cin_p;
  a.Ho = g.c->up ? 2 * g.H : g.H; a.Wo = g.c->up ? 2 * g.W : g.W; a.Cout = g.c->cout_p; a.ksize = 3;
  a.mode = g.c->up ? CONV_UP : CONV_SAME;
  a.wgt_hi = g.c->w_hi; a.wgt_lo = g.c->w_lo; a.wscale_inv = g.c->wscale + 1; a.bias = g.c->bias;
  a.residual = g.res; a.out_act = g.act; a.out = g.out;
  a.skip_prep = true; a.xform = true; a.gen = true;
  a.in_pitch = g.in_pitch; a.pad_mode = g.pad_mode; a.subsample = g.sub;
  a.out_pitch = g.out_pitch; a.out_c0 = g.out_c0; a.cout_valid = g.c->cout;
  a.res_pitch = g.res_pitch; a.residual2 = g.res2; a.res2_pitch = g.res2_pitch; a.post_scale = g.post;
  a.single_pass = g.single_pass;
  a.in_scale = g.in_scale; a.in_shift = g.in_shift; a.prelu_slope = g.prelu;
  return conv_tc(a, nullptr, sm_count, st);
}

// A conv on the per-tap engine, weights not set: 1x1 or 3x3, stride 1 or 2 (only the ceil(H/2) x ceil(W/2) outputs; 3x3 pads
// by 1), written at channel out_c0 of a destination with out_pitch channels per pixel (out_pitch == cout: a dense output).
static ConvArgs pertap_args(const float* in, int N, int h, int w, int cin, int cout, int k, int stride, float* out, int out_pitch,
                            int out_c0, int act, const float* res) {
  ConvArgs a;
  a.in = in; a.N = N; a.H = h; a.W = w; a.Cin = cin; a.Cout = cout; a.ksize = k;
  a.Ho = stride == 2 ? (h + 1) / 2 : h; a.Wo = stride == 2 ? (w + 1) / 2 : w;
  a.mode = stride == 2 ? CONV_DOWN : CONV_SAME; a.down_pad = (stride == 2 && k == 3) ? 1 : 0;
  a.residual = res; a.out_act = act; a.out = out;
  a.out_pitch = out_pitch == cout ? 0 : out_pitch; a.out_c0 = out_c0;
  return a;
}

// A conv with an explicit kh x kw window (GenConv::kh > 0) on the per-tap engine, weights not set: zero padding (pad_h, pad_w),
// stride c.stride, written at channel out_c0 of a destination with out_pitch channels per pixel; into a slice (out_pitch != cout_p
// or out_c0 != 0) only the c.cout real channels are stored.
static ConvArgs pertap_window_args(const float* in, int N, int h, int w, const GenConv& c, float* out, int out_pitch, int out_c0,
                                   int act) {
  ConvArgs a = pertap_args(in, N, h, w, c.cin_p, c.cout_p, 1, 1, out, out_pitch, out_c0, act, nullptr);
  a.kh = c.kh; a.kw = c.kw; a.pad_h = c.pad_h; a.pad_w = c.pad_w;
  a.mode = c.stride == 2 ? CONV_DOWN : CONV_SAME; a.down_pad = 0;
  a.Ho = (h + 2 * c.pad_h - c.kh) / c.stride + 1; a.Wo = (w + 2 * c.pad_w - c.kw) / c.stride + 1;
  if (out_pitch != c.cout_p || out_c0 != 0) a.cout_valid = c.cout;
  return a;
}

// A planned conv of a network forward on the per-tap engine: its operand planes live in the arena until the launch is enqueued.
static int pertap_conv(NetCore& n, ConvArgs a, const GenConv& c, bool dry, cudaStream_t st) {
  a.wgt_hi = c.w_hi; a.wgt_lo = c.w_lo; a.wscale_inv = c.wscale + 1; a.bias = c.bias;
  CFB_REQUIRE(tc_supported(a), std::string(n.label) + ": conv not supported by the wgmma engine: " + c.name);
  void* scratch = n.arena.alloc(tc_scratch_bytes(a));
  CFB_REQUIRE(scratch != nullptr, n.ws_error());
  if (!dry) CFB_CHECK(conv_tc(a, scratch, n.sm_count, st));
  n.arena.release(scratch);
  return 0;
}

static size_t rrdb_ws_bytes(const cfb_rrdb* n, int N, int H, int W) {
  const int us = n->scale == 2 ? 2 : (n->scale == 1 ? 4 : 1);
  const size_t px = (size_t)N * (H / us) * (W / us);
  // F (64) + three dense buffers (192) + body (64) at low resolution; up1 (64 @2x); up2 + hr (64 @4x)
  return (px * (64 + 3 * 192 + 64) + px * 4 * 64 + px * 16 * 64 * 2) * sizeof(float) + 8 * 1024;
}

// The image ends of cfb_rrdb_forward_u8_tiles / cfb_rrdb_forward_tiles: conv_first reads the tiles from the source images,
// conv_last writes their crops into the canvases; the launches take the host tile table in slices of RrdbU8Tiles::kMax tiles.
// range: the per-image max_range (device), nullptr for the uint8 entry point (255).
struct RrdbTileIo {
  const void* img; int in_kind, img_h, img_w, pre_pad;
  const RrdbU8Tile* tiles;
  void* canvas; int out_kind, out_h, out_w;
  const int* range;
  template <class F>
  int each_slice(int N, F f) const {
    for (int t0 = 0; t0 < N; t0 += RrdbU8Tiles::kMax) {
      const int cnt = std::min(RrdbU8Tiles::kMax, N - t0);
      RrdbU8Tiles tab{};
      std::copy(tiles + t0, tiles + t0 + cnt, tab.t);
      CFB_CHECK(f(t0, cnt, tab));
    }
    return 0;
  }
};

static int rrdb_forward(cfb_rrdb* n, const float* x, float* out, int N, int H, int W, void* ws, int64_t ws_bytes, cudaStream_t st,
                        const RrdbTileIo* io = nullptr) {
  CFB_CHECK(n->begin_forward(false));
  const int us = n->scale == 2 ? 2 : (n->scale == 1 ? 4 : 1);
  CFB_REQUIRE(H % us == 0 && W % us == 0, "RRDBNet: H and W must be multiples of the pixel-unshuffle factor (arch_util.py:202)");
  if (N == 0 || H == 0 || W == 0) return 0;
  CFB_REQUIRE((size_t)ws_bytes >= rrdb_ws_bytes(n, N, H, W), "workspace too small (cfb_rrdb_workspace_bytes)");
  const int h = H / us, w = W / us;
  const size_t px = (size_t)N * h * w;
  float* p = (float*)(((uintptr_t)ws + 1023) / 1024 * 1024);
  float* F = p; p += px * 64;
  float* D[3]; for (int i = 0; i < 3; ++i) { D[i] = p; p += px * 192; }
  float* Bd = p; p += px * 64;
  float* U1 = p; p += px * 4 * 64;
  float* U2 = p; p += px * 16 * 64;
  float* HR = p; p += px * 16 * 64;
  // dense buffers start at zero: every channel a conv window can touch is finite from the first launch on
  CFB_CUDA(cudaMemsetAsync(D[0], 0, px * 192 * 3 * sizeof(float), st));
  if (io) {
    CFB_CHECK(io->each_slice(N, [&](int t0, int cnt, const RrdbU8Tiles& tab) {
      const size_t o = (size_t)t0 * h * w;
      CFB_CHECK(conv_thin_in_tiles(io->img, io->in_kind, io->range, io->img_h, io->img_w, io->pre_pad, tab, n->first_w, n->first_b,
                                   F + o * 64, cnt, h, w, us, 64, 0, st));
      return conv_thin_in_tiles(io->img, io->in_kind, io->range, io->img_h, io->img_w, io->pre_pad, tab, n->first_w, n->first_b,
                                D[0] + o * 192, cnt, h, w, us, 192, 0, st);
    }));
  } else {
    CFB_CHECK(conv_thin_in(x, n->first_w, n->first_b, F, N, h, w, n->in_ch, us, 0, 64, 0, st));
    CFB_CHECK(conv_thin_in(x, n->first_w, n->first_b, D[0], N, h, w, n->in_ch, us, 0, 192, 0, st));
  }
  // every GEN conv runs in the handle's precision; conv_first / conv_last are the fp32 SIMT thin convs in both
  auto conv = [&](GenLaunch& g) { g.single_pass = n->precision == 1; return gen_conv(g, n->sm_count, st); };
  int X = 0, Y = 1;            // x of the current RRDB lives in D[X]; D[2] is the middle buffer
  const int Z = 2;
  for (int b = 0; b < n->blocks; ++b) {
    const int src[3] = {X, Y, Z}, dst[3] = {Y, Z, Y};
    for (int r = 0; r < 3; ++r) {
      float* S = D[src[r]];
      for (int k = 0; k < 5; ++k) {
        const GenConv& c = n->convs[(b * 3 + r) * 5 + k];
        GenLaunch g{&c, S, 192, h, w, N, nullptr, 192, 0, OUT_NONE};
        if (k < 4) { g.out = S; g.out_c0 = 64 + 32 * k; g.act = OUT_LRELU; }           // x_{k+1} = lrelu(conv_k(cat(x, x1..xk)))
        else {
          g.out = D[dst[r]]; g.out_c0 = 0; g.res = S; g.res_pitch = 192;               // x5 * 0.2 + x   (rrdbnet_arch.py:40)
          if (r == 2) { g.res2 = D[X]; g.res2_pitch = 192; g.post = 0.2f; }            // out * 0.2 + x  (rrdbnet_arch.py:63)
        }
        CFB_CHECK(conv(g));
      }
    }
    std::swap(X, Y);
  }
  const size_t nb = (size_t)n->blocks * 15;
  { GenLaunch g{&n->convs[nb + 0], D[X], 192, h, w, N, Bd, 64, 0, OUT_NONE}; g.res = F; g.res_pitch = 64;   // feat + conv_body(body(feat))
    CFB_CHECK(conv(g)); }
  { GenLaunch g{&n->convs[nb + 1], Bd, 64, h, w, N, U1, 64, 0, OUT_LRELU}; CFB_CHECK(conv(g)); }
  { GenLaunch g{&n->convs[nb + 2], U1, 64, 2 * h, 2 * w, N, U2, 64, 0, OUT_LRELU}; CFB_CHECK(conv(g)); }
  { GenLaunch g{&n->convs[nb + 3], U2, 64, 4 * h, 4 * w, N, HR, 64, 0, OUT_LRELU}; CFB_CHECK(conv(g)); }
  if (io)
    return io->each_slice(N, [&](int t0, int cnt, const RrdbU8Tiles& tab) {
      return conv_thin_out_tiles(HR + (size_t)t0 * 16 * h * w * 64, n->last_w, n->last_b, tab, io->canvas, io->out_kind, io->range,
                                 io->out_h, io->out_w, cnt, 4 * h, 4 * w, st);
    });
  CFB_CHECK(conv_thin_out(HR, n->last_w, n->last_b, out, N, 4 * h, 4 * w, n->out_ch, 0, st));
  return 0;
}

// Checks of cfb_rrdb_forward_u8_tiles / cfb_rrdb_forward_tiles (`fn`) before any launch: the reflect pads of pre_process must be
// valid (each pad smaller than the dimension it reflects, as F.pad requires), every tile window must lie in the padded image and
// every crop in the tile's output, so that no launch reads or writes outside the images.  range (device int32 [B]) is filled
// by image_max_range first, or nullptr: 255 for every image (the uint8 entry point).
static int rrdb_tiles(const char* fn, cfb_rrdb* n, const void* images, int in_kind, int B, int H, int W, int pre_pad,
                      const int32_t* tiles, int T, int th, int tw, void* out, int out_kind, int* range, void* ws, int64_t ws_bytes,
                      cudaStream_t st) {
  const std::string f(fn);
  CFB_REQUIRE(n->in_ch == 3 && n->out_ch == 3, f + ": built for 3 image channels in and out");
  CFB_REQUIRE(B >= 0 && H > 0 && W > 0 && T >= 0, f + ": bad image batch");
  CFB_REQUIRE(pre_pad >= 0 && pre_pad < H && pre_pad < W,
              f + ": pre_pad must be smaller than the image height and width (reflect pad)");
  const int us = n->scale == 2 ? 2 : (n->scale == 1 ? 4 : 1);
  const int Hp = H + pre_pad, Wp = W + pre_pad;
  const int mh = (us - Hp % us) % us, mw = (us - Wp % us) % us;
  CFB_REQUIRE(mh < Hp && mw < Wp, f + ": the pad to the pixel-unshuffle multiple must be smaller than the padded image (reflect pad)");
  CFB_REQUIRE(th > 0 && tw > 0 && th % us == 0 && tw % us == 0,
              "RRDBNet: H and W must be multiples of the pixel-unshuffle factor (arch_util.py:202)");
  const int Hm = Hp + mh, Wm = Wp + mw, oth = th * n->scale, otw = tw * n->scale;
  std::vector<RrdbU8Tile> tab(T);
  for (int i = 0; i < T; ++i) {
    const int32_t* r = tiles + (size_t)i * 9;
    RrdbU8Tile& t = tab[i];
    t = RrdbU8Tile{r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], r[8]};
    CFB_REQUIRE(t.img >= 0 && t.img < B, f + ": tile image index out of range");
    CFB_REQUIRE(t.in_y >= 0 && t.in_x >= 0 && t.in_y + th <= Hm && t.in_x + tw <= Wm, f + ": tile window outside the padded image");
    CFB_REQUIRE(t.crop_y >= 0 && t.crop_x >= 0 && t.crop_h >= 0 && t.crop_w >= 0 && t.crop_y + t.crop_h <= oth &&
                t.crop_x + t.crop_w <= otw && t.out_y >= 0 && t.out_x >= 0,
                f + ": tile crop outside the tile's output or negative output origin");
  }
  if (T == 0) return 0;
  if (range) CFB_CHECK(image_max_range(images, in_kind, B, (int64_t)H * W * 3, range, st));
  const RrdbTileIo io{images, in_kind, H, W, pre_pad, tab.data(), out, out_kind, H * n->scale, W * n->scale, range};
  return rrdb_forward(n, nullptr, nullptr, T, th, tw, ws, ws_bytes, st, &io);
}

}  // namespace cfb

// =========================================================================================================
// ParseNet (SURVEY.md section 8 row f3): the face-parsing network the paste-back step runs on every restored face
//   /root/reference/facelib/parsing/parsenet.py:140-194 (constructor :142-186, forward :188-194), caller
//   /root/reference/facelib/utils/face_restoration_helper.py:457-487.
// Every ConvLayer = ReflectionPad2d(1) + 3x3 conv (+ eval-mode BatchNorm, folded into the weights at prepare) (+ LeakyReLU 0.2).
// The 64..256-channel convs run on the generalised fused-transform wgmma engine: reflection padding is produced inside the
// kernel (border pixels of the halo patch are copies of patch pixels), 'down' layers (stride 2) keep the even positions of the
// stride-1 result, 'up' layers (nearest x2 + reflection pad) are four parity convs on the low-resolution tensor with replicate
// padding, and the residual sums `identity + res` / `feat + body(feat)` are epilogue residuals.
// =========================================================================================================
namespace cfb {
struct PnBlock { int kind; int cin, cout; GenConv sc, c1, c2; };     // kind: 0 none, 1 down, 2 up
}
struct cfb_parsenet : cfb::NetCore {
  cfb_parsenet() : NetCore("ParseNet", "parsenet") {}
  int in_size = 512, out_size = 512, min_feat = 32, base_ch = 64, parsing_ch = 19, res_depth = 10, ch_min = 32, ch_max = 256;
  std::vector<cfb::PnBlock> blocks;       // encoder[1:], body, decoder in order
  int n_enc = 0, n_body = 0, n_dec = 0, head_ch = 64;
  float *first_w = nullptr, *first_b = nullptr, *mask_w = nullptr, *mask_b = nullptr, *img_w = nullptr, *img_b = nullptr;
};
namespace cfb {

static int pn_build(cfb_parsenet* n) {       // ParseNet.__init__  parsenet.py:151-186
  auto clip = [&](int x) { return std::max(n->ch_min, std::min(x, n->ch_max)); };
  const int mfs = std::min(n->in_size, n->min_feat);
  const int down = (int)std::lround(std::floor(std::log2((double)(n->in_size / mfs))));
  const int up = (int)std::lround(std::floor(std::log2((double)(n->out_size / mfs))));
  n->blocks.clear();
  int head = n->base_ch;
  auto add = [&](const std::string& p, int kind, int cin, int cout) {
    PnBlock b; b.kind = kind; b.cin = cin; b.cout = cout;
    b.sc = plan_conv(p + ".shortcut_func", cin, cout); b.sc.up = kind == 2;
    b.c1 = plan_conv(p + ".conv1", cin, cout); b.c1.up = kind == 2;
    b.c2 = plan_conv(p + ".conv2", cout, cout);
    n->blocks.push_back(b);
  };
  for (int i = 0; i < down; ++i) { add("encoder." + std::to_string(i + 1), 1, clip(head), clip(head * 2)); head *= 2; }
  n->n_enc = down;
  for (int i = 0; i < n->res_depth; ++i) add("body." + std::to_string(i), 0, clip(head), clip(head));
  n->n_body = n->res_depth;
  for (int i = 0; i < up; ++i) { add("decoder." + std::to_string(i), 2, clip(head), clip(head / 2)); head /= 2; }
  n->n_dec = up;
  n->head_ch = clip(head);
  CFB_REQUIRE(n->base_ch == 64 && n->head_ch == 64, "ParseNet: built for base_ch = 64 and a 64-channel head (in_size == out_size)");
  for (const PnBlock& b : n->blocks) {
    CFB_REQUIRE(b.cin % 64 == 0 && b.cout % 64 == 0, "ParseNet: channel counts must be multiples of 64");
    CFB_REQUIRE(b.kind != 0 || b.cin == b.cout, "ParseNet: a body block with a channel change (conv shortcut) is not built");
  }
  CFB_REQUIRE(n->parsing_ch >= 1 && n->parsing_ch <= 20, "ParseNet: at most 20 parsing classes");
  return 0;
}

static int pn_prepare(cfb_parsenet* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  CFB_CHECK(pn_build(n));
  SlabPlan plan;
  for (const PnBlock& b : n->blocks) { if (b.kind) plan.add(b.sc); plan.add(b.c1); plan.add(b.c2); }
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256((size_t)27 * 64 * 4) + 256 + 2 * (align256((size_t)9 * 64 * 20 * 4) + 256)));
  WeightPrep wp(*n, plan, st);
  auto prep = [&](GenConv& c, bool bn) -> int {
    if (bn) {
      CFB_CHECK(wp.fold(c.name + ".conv2d.weight", c.name + ".norm.norm.", c.cout, c.cin * 9));
      return wp.conv(c, wp.fold_w, wp.fold_b);
    }
    const float* w = n->param(c.name + ".conv2d.weight", (int64_t)c.cout * c.cin * 9);
    const float* b = n->param(c.name + ".conv2d.bias", c.cout);
    if (!w || !b) return 1;
    return wp.conv(c, w, b);
  };
  for (PnBlock& b : n->blocks) {
    if (b.kind) CFB_CHECK(prep(b.sc, false));
    CFB_CHECK(prep(b.c1, true));
    CFB_CHECK(prep(b.c2, true));
  }
  {
    const float* w = n->param("encoder.0.conv2d.weight", (int64_t)64 * 3 * 9);
    const float* b = n->param("encoder.0.conv2d.bias", 64);
    if (!w || !b) return 1;
    n->first_w = (float*)wp.take((size_t)27 * 64 * 4); n->first_b = (float*)wp.take(256);
    CFB_CHECK(relayout_oihw_to_tck(w, n->first_w, 64, 3, 3, st));
    CFB_CUDA(cudaMemcpyAsync(n->first_b, b, 64 * 4, cudaMemcpyDeviceToDevice, st));
  }
  for (int which = 0; which < 2; ++which) {
    const std::string nm = which ? "out_img_conv" : "out_mask_conv";
    const int co = which ? 3 : n->parsing_ch;
    const float* w = n->param(nm + ".conv2d.weight", (int64_t)co * 64 * 9);
    const float* b = n->param(nm + ".conv2d.bias", co);
    if (!w || !b) return 1;
    float* wd = (float*)wp.take((size_t)9 * 64 * 20 * 4);
    float* bd = (float*)wp.take(256);
    CFB_CHECK(relayout_thin_out(w, wd, co, st));
    CFB_CUDA(cudaMemcpyAsync(bd, b, (size_t)co * 4, cudaMemcpyDeviceToDevice, st));
    if (which) { n->img_w = wd; n->img_b = bd; } else { n->mask_w = wd; n->mask_b = bd; }
  }
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// The uint8 ends of cfb_parsenet_masks_u8: encoder.0 reads the faces, out_mask_conv writes classes / mask; out_img_conv is
// not run (the caller drops out_img, face_restoration_helper.py:464).
struct PnU8Io { const unsigned char* faces; unsigned char* cls; unsigned char* mask; };

static int pn_forward(cfb_parsenet* n, const float* x, float* out_mask, float* out_img, int N, int H, int W, void* ws, int64_t ws_bytes,
                      cudaStream_t st, bool dry, const PnU8Io* u8 = nullptr) {
  CFB_CHECK(n->begin_forward(dry));
  const int div = 1 << n->n_enc;
  CFB_REQUIRE(H % div == 0 && W % div == 0 && H >= 2 * div && W >= 2 * div, "ParseNet: H and W must be multiples of 2^down_steps");
  if (N == 0) return 0;
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  float* t = nullptr;
  int h = H, w = W, c = 64;
  CFB_CHECK(n->alloc(&t, (size_t)N * h * w * 64));
  if (!dry) {
    if (u8) CFB_CHECK(conv_thin_in_u8_faces(u8->faces, n->first_w, n->first_b, t, N, h, w, 1, 64, 0, st));
    else CFB_CHECK(conv_thin_in(x, n->first_w, n->first_b, t, N, h, w, 3, 1, 1, 64, 0, st));
  }
  // every GEN conv runs in the handle's precision; encoder.0 and the heads are the fp32 SIMT thin convs in both
  auto conv = [&](GenLaunch& g) { g.single_pass = n->precision == 1; return gen_conv(g, n->sm_count, st); };
  float* feat = nullptr;           // encoder output, added back after the body (parsenet.py:190)
  for (size_t i = 0; i < n->blocks.size(); ++i) {
    const PnBlock& b = n->blocks[i];
    CFB_REQUIRE(b.cin == c, "ParseNet: channel plan mismatch");
    const bool last_body = (int)i == n->n_enc + n->n_body - 1 && n->n_body > 0;
    if ((int)i == n->n_enc) feat = t;
    float *s = nullptr, *c1 = nullptr, *o = nullptr;
    int ho = h, wo = w;
    if (b.kind == 1) { ho = h / 2; wo = w / 2; } else if (b.kind == 2) { ho = 2 * h; wo = 2 * w; }
    const int h1 = b.kind == 2 ? ho : h, w1 = b.kind == 2 ? wo : w;          // resolution of conv1's output
    if (b.kind) {
      CFB_CHECK(n->alloc(&s, (size_t)N * ho * wo * b.cout));
      GenLaunch g{&b.sc, t, b.cin, h, w, N, s, b.cout, 0, OUT_NONE};
      g.pad_mode = b.kind == 2 ? 2 : 1; g.sub = b.kind == 1;
      if (!dry) CFB_CHECK(conv(g));
    }
    CFB_CHECK(n->alloc(&c1, (size_t)N * h1 * w1 * b.cout));
    {
      GenLaunch g{&b.c1, t, b.cin, h, w, N, c1, b.cout, 0, OUT_LRELU};
      g.pad_mode = b.kind == 2 ? 2 : 1;
      if (!dry) CFB_CHECK(conv(g));
    }
    CFB_CHECK(n->alloc(&o, (size_t)N * ho * wo * b.cout));
    {
      GenLaunch g{&b.c2, c1, b.cout, h1, w1, N, o, b.cout, 0, OUT_NONE};
      g.pad_mode = 1; g.sub = b.kind == 1;
      g.res = b.kind ? s : t; g.res_pitch = b.cout;
      if (last_body) { g.res2 = feat; g.res2_pitch = b.cout; g.post = 1.f; }      // x = feat + body(feat)
      if (!dry) CFB_CHECK(conv(g));
    }
    ar.release(c1);
    if (s) ar.release(s);
    if (t != feat) ar.release(t);
    if (last_body && feat) { ar.release(feat); feat = nullptr; }
    t = o; h = ho; w = wo; c = b.cout;
  }
  if (n->n_body == 0) feat = nullptr;
  CFB_REQUIRE(c == 64, "ParseNet: head must have 64 channels");
  if (!dry) {
    if (u8) {
      CFB_CHECK(conv_thin_out_argmax(t, n->mask_w, n->mask_b, u8->cls, u8->mask, N, h, w, n->parsing_ch, 1, st));
    } else {
      CFB_CHECK(conv_thin_out(t, n->mask_w, n->mask_b, out_mask, N, h, w, n->parsing_ch, 1, st));
      if (out_img) CFB_CHECK(conv_thin_out(t, n->img_w, n->img_b, out_img, N, h, w, 3, 1, st));
    }
  }
  ar.release(t);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// RetinaFace-ResNet50: the face detector of whole-image mode
//   /root/reference/facelib/detection/retinaface/retinaface.py:77-145 (RetinaFace, cfg_re50), retinaface_net.py (FPN, SSH,
//   heads), torchvision resnet50 conv1 .. layer4 (body, return layers layer2/3/4).
// Eval-mode BatchNorm is folded into every conv at prepare.  Engines per conv form:
//   stem (7x7 s2 + max-pool)            SIMT (detection.cu), fp32 or uint8 BGR input
//   3x3 stride 1 (layer conv2, FPN merge, SSH)   generalised fused-transform halo engine (ragged tiles, destination slices
//                                        of the SSH concat, ReLU epilogue)
//   1x1 (bottleneck conv1 / conv3 + residual, downsample, FPN output_k, heads), 3x3 stride 2 pad 1
//                                        per-tap engine on operand planes (ragged tiles; stride 2 computes only the output
//                                        positions: element-strided TMA boxes, ceil(H/2) outputs)
//   FPN top-down add (after the ReLU)   SIMT, torch's nearest index
// =========================================================================================================
struct cfb_retinaface : cfb::NetCore {
  cfb_retinaface() : NetCore("RetinaFace", "retinaface") {}
  std::vector<cfb::GenConv> convs;       // body blocks (conv1, conv2, conv3[, downsample]), fpn, ssh, heads: see rf_build
  int blocks[4] = {3, 4, 6, 3};
  float *stem_w = nullptr, *stem_b = nullptr;
};
namespace cfb {

static void rf_build(cfb_retinaface* n) {
  n->convs.clear();
  auto add = [&](const std::string& w, const std::string& bn, int cin, int cout, int k, int stride) {
    n->convs.push_back(plan_conv(w, cin, cout, k, stride));
    n->convs.back().bn = bn;
  };
  const int widths[4] = {64, 128, 256, 512};
  int cin = 64;
  for (int l = 0; l < 4; ++l) {
    const int wd = widths[l];
    for (int b = 0; b < n->blocks[l]; ++b) {
      const std::string p = "body.layer" + std::to_string(l + 1) + "." + std::to_string(b) + ".";
      const int s = (b == 0 && l > 0) ? 2 : 1;
      add(p + "conv1.weight", p + "bn1.", cin, wd, 1, 1);
      add(p + "conv2.weight", p + "bn2.", wd, wd, 3, s);
      add(p + "conv3.weight", p + "bn3.", wd, 4 * wd, 1, 1);
      if (b == 0) add(p + "downsample.0.weight", p + "downsample.1.", cin, 4 * wd, 1, s);
      cin = 4 * wd;
    }
  }
  const int ins[3] = {512, 1024, 2048};
  for (int k = 0; k < 3; ++k) {
    const std::string p = "fpn.output" + std::to_string(k + 1) + ".";
    add(p + "0.weight", p + "1.", ins[k], 256, 1, 1);
  }
  add("fpn.merge1.0.weight", "fpn.merge1.1.", 256, 256, 3, 1);
  add("fpn.merge2.0.weight", "fpn.merge2.1.", 256, 256, 3, 1);
  for (int k = 0; k < 3; ++k) {
    const std::string p = "ssh" + std::to_string(k + 1) + ".";
    add(p + "conv3X3.0.weight", p + "conv3X3.1.", 256, 128, 3, 1);
    add(p + "conv5X5_1.0.weight", p + "conv5X5_1.1.", 256, 64, 3, 1);
    add(p + "conv5X5_2.0.weight", p + "conv5X5_2.1.", 64, 64, 3, 1);
    add(p + "conv7X7_2.0.weight", p + "conv7X7_2.1.", 64, 64, 3, 1);
    add(p + "conv7x7_3.0.weight", p + "conv7x7_3.1.", 64, 64, 3, 1);
  }
  for (int k = 0; k < 3; ++k) add("heads." + std::to_string(k), "", 256, 64, 1, 1);   // bbox 8 | class 4 | landmark 20 | 0
}

static int rf_prepare(cfb_retinaface* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  rf_build(n);
  SlabPlan plan;
  for (const GenConv& c : n->convs) plan.add(c);
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256((size_t)64 * 147 * 4) + align256(256)));
  WeightPrep wp(*n, plan, st);
  for (GenConv& c : n->convs) {
    if (c.bn.empty()) {        // heads: [bbox 8 | class 4 | landmark 20 | zero 32] x 256, with their biases
      CFB_CUDA(cudaMemsetAsync(wp.fold_w, 0, (size_t)c.cout * c.cin * 4, st));
      CFB_CUDA(cudaMemsetAsync(wp.fold_b, 0, 64 * 4, st));
      const std::string lv = c.name.substr(6);
      const struct { const char* head; int rows, row0; } parts[3] = {{"BboxHead.", 8, 0}, {"ClassHead.", 4, 8}, {"LandmarkHead.", 20, 12}};
      for (const auto& h : parts) {
        const std::string base = std::string(h.head) + lv + ".conv1x1.";
        const float* w = n->param(base + "weight", (int64_t)h.rows * 256);
        const float* b = n->param(base + "bias", h.rows);
        if (!w || !b) return 1;
        CFB_CUDA(cudaMemcpyAsync(wp.fold_w + (size_t)h.row0 * 256, w, (size_t)h.rows * 256 * 4, cudaMemcpyDeviceToDevice, st));
        CFB_CUDA(cudaMemcpyAsync(wp.fold_b + h.row0, b, (size_t)h.rows * 4, cudaMemcpyDeviceToDevice, st));
      }
    } else {
      CFB_CHECK(wp.fold(c.name, c.bn, c.cout, c.cin * c.k * c.k));
    }
    CFB_CHECK(wp.conv(c, wp.fold_w, wp.fold_b));
  }
  n->stem_w = (float*)wp.take((size_t)64 * 147 * 4); n->stem_b = (float*)wp.take(256);
  CFB_CHECK(wp.fold("body.conv1.weight", "body.bn1.", 64, 147));
  CFB_CUDA(cudaMemcpyAsync(n->stem_w, wp.fold_w, (size_t)64 * 147 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaMemcpyAsync(n->stem_b, wp.fold_b, 64 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// number of priors of an h x w input (PriorBox: two anchors per cell of the /8, /16, /32 maps, ceil-divided)
static int64_t rf_priors(int H, int W) {
  int64_t P = 0;
  for (int s : {8, 16, 32}) P += 2 * (int64_t)((H + s - 1) / s) * ((W + s - 1) / s);
  return P;
}

static int rf_forward(cfb_retinaface* n, const float* x, const unsigned char* img, float* loc, float* conf, float* landms, int N,
                      int H, int W, void* ws, int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_CHECK(n->begin_forward(dry));
  CFB_REQUIRE(H >= 1 && W >= 1 && N >= 0, "RetinaFace: empty image");
  CFB_REQUIRE(rf_priors(H, W) * N < ((int64_t)1 << 31) / 16, "RetinaFace: image too large");
  if (N == 0) return 0;
  if (n->convs.empty()) rf_build(n);
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  // one conv of the plan: 3x3 stride 1 on the generalised engine, everything else on the per-tap engine
  auto conv = [&](const GenConv& c, const float* in, int h, int w, float* out, int act, const float* res, int out_pitch = 0,
                  int out_c0 = 0) -> int {
    if (c.gen) {
      GenLaunch g{&c, in, c.cin_p, h, w, N, out, out_pitch ? out_pitch : c.cout, out_c0, act};
      g.res = res; g.res_pitch = c.cout;
      return dry ? 0 : gen_conv(g, n->sm_count, st);
    }
    return pertap_conv(*n, pertap_args(in, N, h, w, c.cin_p, c.cout_p, c.k, c.stride, out, out_pitch, out_c0, act, res), c, dry, st);
  };
  const int H2 = (H - 1) / 2 + 1, W2 = (W - 1) / 2 + 1;
  int h = (H2 - 1) / 2 + 1, w = (W2 - 1) / 2 + 1;
  float *s0 = nullptr, *cur = nullptr;
  CFB_CHECK(n->alloc(&s0, (size_t)N * H2 * W2 * 64));
  if (!dry) CFB_CHECK(rf_stem(x, img, n->stem_w, n->stem_b, s0, N, H, W, st));
  CFB_CHECK(n->alloc(&cur, (size_t)N * h * w * 64));
  if (!dry) CFB_CHECK(rf_maxpool(s0, cur, N, H2, W2, st));
  ar.release(s0);
  size_t ci = 0;
  float* C[3] = {nullptr, nullptr, nullptr};
  int ch[3] = {0, 0, 0}, cw[3] = {0, 0, 0};
  for (int l = 0; l < 4; ++l) {
    for (int b = 0; b < n->blocks[l]; ++b) {
      const GenConv& c1 = n->convs[ci++];
      const GenConv& c2 = n->convs[ci++];
      const GenConv& c3 = n->convs[ci++];
      const GenConv* ds = b == 0 ? &n->convs[ci++] : nullptr;
      const int ho = c2.stride == 2 ? (h + 1) / 2 : h, wo = c2.stride == 2 ? (w + 1) / 2 : w;
      float *t1 = nullptr, *t2 = nullptr, *res = cur, *y = nullptr;
      CFB_CHECK(n->alloc(&t1, (size_t)N * h * w * c1.cout));
      CFB_CHECK(conv(c1, cur, h, w, t1, OUT_RELU, nullptr));
      CFB_CHECK(n->alloc(&t2, (size_t)N * ho * wo * c2.cout));
      CFB_CHECK(conv(c2, t1, h, w, t2, OUT_RELU, nullptr));
      ar.release(t1);
      if (ds) {
        CFB_CHECK(n->alloc(&res, (size_t)N * ho * wo * ds->cout));
        CFB_CHECK(conv(*ds, cur, h, w, res, OUT_NONE, nullptr));
      }
      CFB_CHECK(n->alloc(&y, (size_t)N * ho * wo * c3.cout));
      CFB_CHECK(conv(c3, t2, ho, wo, y, OUT_RELU, res));          // relu(bn3(conv3(.)) + identity)
      ar.release(t2);
      if (res != cur) ar.release(res);
      if (l < 2 || b > 0) ar.release(cur);       // the input of layer3.0 / layer4.0 is a kept pyramid level (C3 / C4)
      cur = y; h = ho; w = wo;
    }
    if (l >= 1) { C[l - 1] = cur; ch[l - 1] = h; cw[l - 1] = w; }      // layer2/3/4 outputs; still the next layer's input
  }
  // FPN (retinaface_net.py:76-96): output_k = relu(bn(conv1x1(C_k))); output_2 += nearest(output_3); merge2; output_1 += ...
  float* O[3];
  for (int k = 0; k < 3; ++k) {
    CFB_CHECK(n->alloc(&O[k], (size_t)N * ch[k] * cw[k] * 256));
    CFB_CHECK(conv(n->convs[ci + k], C[k], ch[k], cw[k], O[k], OUT_RELU, nullptr));
    ar.release(C[k]);
  }
  const GenConv& merge1 = n->convs[ci + 3];
  const GenConv& merge2 = n->convs[ci + 4];
  ci += 5;
  float *m2 = nullptr, *m1 = nullptr;
  if (!dry) CFB_CHECK(rf_add_nearest(O[1], O[2], N, ch[1], cw[1], ch[2], cw[2], 256, st));
  CFB_CHECK(n->alloc(&m2, (size_t)N * ch[1] * cw[1] * 256));
  CFB_CHECK(conv(merge2, O[1], ch[1], cw[1], m2, OUT_RELU, nullptr));
  ar.release(O[1]);
  if (!dry) CFB_CHECK(rf_add_nearest(O[0], m2, N, ch[0], cw[0], ch[1], cw[1], 256, st));
  CFB_CHECK(n->alloc(&m1, (size_t)N * ch[0] * cw[0] * 256));
  CFB_CHECK(conv(merge1, O[0], ch[0], cw[0], m1, OUT_RELU, nullptr));
  ar.release(O[0]);
  float* fpn[3] = {m1, m2, O[2]};
  // SSH (retinaface_net.py:47-59): relu(cat[conv3X3, conv5X5, conv7X7]) written as three destination slices with ReLU
  // epilogues; then the three 1x1 heads of the level in one conv
  float* hd[3];
  for (int k = 0; k < 3; ++k) {
    const GenConv* s = &n->convs[ci + 5 * k];
    const int hk = ch[k], wk = cw[k];
    float *f = nullptr, *t5 = nullptr, *t7 = nullptr;
    CFB_CHECK(n->alloc(&f, (size_t)N * hk * wk * 256));
    CFB_CHECK(conv(s[0], fpn[k], hk, wk, f, OUT_RELU, nullptr, 256, 0));
    CFB_CHECK(n->alloc(&t5, (size_t)N * hk * wk * 64));
    CFB_CHECK(conv(s[1], fpn[k], hk, wk, t5, OUT_RELU, nullptr));
    CFB_CHECK(conv(s[2], t5, hk, wk, f, OUT_RELU, nullptr, 256, 128));
    CFB_CHECK(n->alloc(&t7, (size_t)N * hk * wk * 64));
    CFB_CHECK(conv(s[3], t5, hk, wk, t7, OUT_RELU, nullptr));
    CFB_CHECK(conv(s[4], t7, hk, wk, f, OUT_RELU, nullptr, 256, 192));
    ar.release(t5); ar.release(t7);
    ar.release(fpn[k]);
    CFB_CHECK(n->alloc(&hd[k], (size_t)N * hk * wk * 64));
    CFB_CHECK(conv(n->convs[ci + 15 + k], f, hk, wk, hd[k], OUT_NONE, nullptr));
    ar.release(f);
  }
  if (!dry) CFB_CHECK(rf_heads(hd, ch, cw, loc, conf, landms, N, (int)rf_priors(H, W), st));
  for (int k = 0; k < 3; ++k) ar.release(hd[k]);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// BiSeNet(num_class): the light face parser of the paste-back step (facelib's default parser)
//   /root/reference/facelib/parsing/bisenet.py:104-140 (BiSeNet, ContextPath, ARM, FFM), resnet.py (ResNet18).
// Eval-mode BatchNorm is folded into every conv at prepare (eps 1e-5).  H and W are multiples of 32, so every nearest resize of
// the context path is an exact x2 or a broadcast of the 1 x 1 global average.  Engines per conv form:
//   stem (7x7 s2 + bn1 + ReLU + max-pool)      SIMT (detection.cu, RetinaFace's), fp32 or uint8 BGR faces (normalisation fused)
//   3x3 stride 1 (BasicBlock convs, ARM and    generalised halo engine: ReLU epilogue, residual + ReLU epilogue
//     head ConvBNReLU)
//   conv_head32 / conv_head16 on nearest x2   generalised halo engine, up form (four parity convs on the low-resolution map)
//   3x3 stride 2, 1x1 downsample, FFM convblk, per-tap engine (conv_out zero-padded to 64 output channels)
//     conv_out 1x1
//   avg pool, attention vectors, feat * att + add, bilinear (+ argmax)    SIMT (bisenet.cu)
// FFM's torch.cat([feat8, feat_cp8]) is one 256-channel buffer: conv_head16 writes channels [128, 256), feat8 is copied to
// [0, 128) (layer3 reads feat8 dense on the per-tap engine, which has no input pitch), and conv_out16 reads [128, 256) in place.
// =========================================================================================================
struct cfb_bisenet : cfb::NetCore {
  cfb_bisenet() : NetCore("BiSeNet", "bisenet") {}
  int num_class = 19;
  std::vector<cfb::GenConv> res;          // ResNet18 layer1..4: conv1, conv2[, downsample] per BasicBlock
  cfb::GenConv arm[2], head32, head16, convblk, outc[3], outp[3];   // arm16, arm32; conv_out / 16 / 32: ConvBNReLU, conv_out
  float *stem_w = nullptr, *stem_b = nullptr;
  float *att_w[2] = {nullptr, nullptr}, *att_b[2] = {nullptr, nullptr};   // arm16 / arm32 conv_atten + bn_atten [128][128]
  float *avg_w = nullptr, *avg_b = nullptr;                             // conv_avg + bn [128][512]
  float *ffm_w1 = nullptr, *ffm_w2 = nullptr;                           // ffm.conv1 [64][256], ffm.conv2 [256][64]
  std::vector<cfb::GenConv*> all() {
    std::vector<cfb::GenConv*> v;
    for (cfb::GenConv& c : res) v.push_back(&c);
    for (cfb::GenConv* c : {&arm[0], &arm[1], &head32, &head16, &convblk, &outc[0], &outc[1], &outc[2], &outp[0], &outp[1], &outp[2]})
      v.push_back(c);
    return v;
  }
};
namespace cfb {

static void bs_build(cfb_bisenet* n) {
  auto mk = [](const std::string& p, const std::string& bn, int cin, int cout, int k, int stride) {
    GenConv c = plan_conv(p + "weight", cin, cout, k, stride);
    c.bn = bn;
    return c;
  };
  n->res.clear();
  int cin = 64;
  for (int l = 0; l < 4; ++l) {
    const int cout = 64 << l;
    for (int b = 0; b < 2; ++b) {
      const std::string p = "cp.resnet.layer" + std::to_string(l + 1) + "." + std::to_string(b) + ".";
      const int s = (b == 0 && l > 0) ? 2 : 1;
      n->res.push_back(mk(p + "conv1.", p + "bn1.", cin, cout, 3, s));
      n->res.push_back(mk(p + "conv2.", p + "bn2.", cout, cout, 3, 1));
      if (cin != cout) n->res.push_back(mk(p + "downsample.0.", p + "downsample.1.", cin, cout, 1, s));
      cin = cout;
    }
  }
  n->arm[0] = mk("cp.arm16.conv.conv.", "cp.arm16.conv.bn.", 256, 128, 3, 1);
  n->arm[1] = mk("cp.arm32.conv.conv.", "cp.arm32.conv.bn.", 512, 128, 3, 1);
  n->head32 = mk("cp.conv_head32.conv.", "cp.conv_head32.bn.", 128, 128, 3, 1);
  n->head16 = mk("cp.conv_head16.conv.", "cp.conv_head16.bn.", 128, 128, 3, 1);
  n->head32.up = n->head16.up = true;
  n->convblk = mk("ffm.convblk.conv.", "ffm.convblk.bn.", 256, 256, 1, 1);
  const char* heads[3] = {"conv_out.", "conv_out16.", "conv_out32."};
  const int hin[3] = {256, 128, 128}, mid[3] = {256, 64, 64};
  for (int k = 0; k < 3; ++k) {
    const std::string p = heads[k];
    n->outc[k] = mk(p + "conv.conv.", p + "conv.bn.", hin[k], mid[k], 3, 1);
    n->outp[k] = mk(p + "conv_out.", "", mid[k], n->num_class, 1, 1);
  }
}

static int bs_prepare(cfb_bisenet* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  bs_build(n);
  SlabPlan plan;
  for (const GenConv* c : n->all()) plan.add(*c);
  const size_t extra = align256((size_t)64 * 147 * 4) + align256(256) + 2 * (align256((size_t)128 * 128 * 4) + align256(128 * 4)) +
                       align256((size_t)128 * 512 * 4) + align256(128 * 4) + 2 * align256((size_t)64 * 256 * 4);
  CFB_CHECK(n->reserve_slab(plan.bytes() + extra));
  WeightPrep wp(*n, plan, st);
  for (GenConv* c : n->all()) {
    if (c->bn.empty()) {       // conv_out: no BatchNorm, no bias
      const float* w = n->param(c->name, (int64_t)c->cout * c->cin);
      if (!w) return 1;
      CFB_CHECK(wp.conv(*c, w, nullptr));
    } else {
      CFB_CHECK(wp.fold(c->name, c->bn, c->cout, c->cin * c->k * c->k));
      CFB_CHECK(wp.conv(*c, wp.fold_w, wp.fold_b));
    }
  }
  // a folded weight [cout][per_out] + bias kept in the slab
  auto keep = [&](const std::string& w, const std::string& bn, int cout, int per_out, float*& wd, float*& bd) -> int {
    CFB_CHECK(wp.fold(w, bn, cout, per_out));
    wd = (float*)wp.take((size_t)cout * per_out * 4); bd = (float*)wp.take((size_t)std::max(cout, 64) * 4);
    CFB_CUDA(cudaMemcpyAsync(wd, wp.fold_w, (size_t)cout * per_out * 4, cudaMemcpyDeviceToDevice, st));
    CFB_CUDA(cudaMemcpyAsync(bd, wp.fold_b, (size_t)cout * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  CFB_CHECK(keep("cp.resnet.conv1.weight", "cp.resnet.bn1.", 64, 147, n->stem_w, n->stem_b));
  CFB_CHECK(keep("cp.arm16.conv_atten.weight", "cp.arm16.bn_atten.", 128, 128, n->att_w[0], n->att_b[0]));
  CFB_CHECK(keep("cp.arm32.conv_atten.weight", "cp.arm32.bn_atten.", 128, 128, n->att_w[1], n->att_b[1]));
  CFB_CHECK(keep("cp.conv_avg.conv.weight", "cp.conv_avg.bn.", 128, 512, n->avg_w, n->avg_b));
  for (int k = 0; k < 2; ++k) {
    const float* w = n->param(k ? "ffm.conv2.weight" : "ffm.conv1.weight", 64 * 256);
    if (!w) return 1;
    float*& wd = k ? n->ffm_w2 : n->ffm_w1;
    wd = (float*)wp.take((size_t)64 * 256 * 4);
    CFB_CUDA(cudaMemcpyAsync(wd, w, (size_t)64 * 256 * 4, cudaMemcpyDeviceToDevice, st));
  }
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// The uint8 ends of cfb_bisenet_masks_u8: the stem reads the faces, and the upsampling of `out` is fused with the argmax;
// conv_out16 / conv_out32 are not run (the caller keeps `out` only, face_restoration_helper.py:462).
struct BsU8Io { const unsigned char* faces; unsigned char* cls; unsigned char* mask; };

static int bs_forward(cfb_bisenet* n, const float* x, float* const out[3], int N, int H, int W, void* ws, int64_t ws_bytes,
                      cudaStream_t st, bool dry, const BsU8Io* u8 = nullptr) {
  CFB_CHECK(n->begin_forward(dry));
  CFB_REQUIRE(N >= 0 && H >= 32 && W >= 32 && H % 32 == 0 && W % 32 == 0, "BiSeNet: H and W must be positive multiples of 32");
  if (N == 0) return 0;
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  // one conv of the plan: 3x3 stride 1 on the generalised engine (the up form for the heads of the context path), everything
  // else on the per-tap engine.  h, w: the input resolution.
  auto conv = [&](const GenConv& c, const float* in, int in_pitch, int h, int w, float* o, int out_pitch, int out_c0, int act,
                  const float* resid) -> int {
    if (c.gen) {
      GenLaunch g{&c, in, in_pitch, h, w, N, o, out_pitch, out_c0, act};
      g.res = resid; g.res_pitch = c.cout;
      return dry ? 0 : gen_conv(g, n->sm_count, st);
    }
    return pertap_conv(*n, pertap_args(in, N, h, w, c.cin_p, c.cout_p, c.k, c.stride, o, out_pitch, out_c0, act, resid), c, dry, st);
  };
  auto px = [&](int h, int w) { return (size_t)N * h * w; };
  const int H2 = H / 2, W2 = W / 2;
  int h = H / 4, w = W / 4;
  float *s0 = nullptr, *cur = nullptr;
  CFB_CHECK(n->alloc(&s0, px(H2, W2) * 64));
  if (!dry) CFB_CHECK(rf_stem(x, u8 ? u8->faces : nullptr, n->stem_w, n->stem_b, s0, N, H, W, st, true));
  CFB_CHECK(n->alloc(&cur, px(h, w) * 64));
  if (!dry) CFB_CHECK(rf_maxpool(s0, cur, N, H2, W2, st));
  ar.release(s0);
  // ResNet18: relu(shortcut + bn2(conv2(relu(bn1(conv1(x))))))
  float* F[3] = {nullptr, nullptr, nullptr};      // feat8, feat16, feat32
  int fh[3] = {0, 0, 0}, fw[3] = {0, 0, 0};
  size_t ci = 0;
  for (int l = 0; l < 4; ++l) {
    for (int b = 0; b < 2; ++b) {
      const GenConv& c1 = n->res[ci++];
      const GenConv& c2 = n->res[ci++];
      const GenConv* ds = c1.cin != c1.cout ? &n->res[ci++] : nullptr;
      const int ho = c1.stride == 2 ? h / 2 : h, wo = c1.stride == 2 ? w / 2 : w;
      float *t1 = nullptr, *sc = cur, *y = nullptr;
      CFB_CHECK(n->alloc(&t1, px(ho, wo) * c1.cout));
      CFB_CHECK(conv(c1, cur, c1.cin_p, h, w, t1, c1.cout, 0, OUT_RELU, nullptr));
      if (ds) {
        CFB_CHECK(n->alloc(&sc, px(ho, wo) * ds->cout));
        CFB_CHECK(conv(*ds, cur, ds->cin_p, h, w, sc, ds->cout, 0, OUT_NONE, nullptr));
      }
      CFB_CHECK(n->alloc(&y, px(ho, wo) * c2.cout));
      CFB_CHECK(conv(c2, t1, c2.cin_p, ho, wo, y, c2.cout, 0, OUT_RELU, sc));
      ar.release(t1);
      if (sc != cur) ar.release(sc);
      if (l < 2 || b > 0) ar.release(cur);      // the inputs of layer3.0 / layer4.0 are feat8 / feat16, kept
      cur = y; h = ho; w = wo;
    }
    if (l >= 1) { F[l - 1] = cur; fh[l - 1] = h; fw[l - 1] = w; }
  }
  const int h8 = fh[0], w8 = fw[0], h16 = fh[1], w16 = fw[1], h32 = fh[2], w32 = fw[2];
  // ContextPath: avg = conv_avg(avg_pool(feat32)); feat32_sum = arm32(feat32) + avg_up; feat_cp16 = conv_head32(up(feat32_sum))
  float *v512 = nullptr, *avg = nullptr, *m = nullptr, *att = nullptr;
  CFB_CHECK(n->alloc(&v512, (size_t)N * 512));
  CFB_CHECK(n->alloc(&avg, (size_t)N * 128));
  CFB_CHECK(n->alloc(&m, (size_t)N * 256));
  CFB_CHECK(n->alloc(&att, (size_t)N * 256));
  if (!dry) {
    CFB_CHECK(bise_mean(F[2], v512, N, h32 * w32, 512, st));
    CFB_CHECK(bise_attention(BiseAttention{n->avg_w, n->avg_b, 512, 128, 1, nullptr, nullptr, 0, 0}, v512, avg, N, st));
  }
  // ARM k (0: arm16, 1: arm32) on its feature map, combined with `add_vec` or `add_t` in place
  auto arm = [&](int k, const float* in, int hh, int ww, float* a, const float* add_vec, const float* add_t) -> int {
    CFB_CHECK(conv(n->arm[k], in, n->arm[k].cin_p, hh, ww, a, 128, 0, OUT_RELU, nullptr));
    if (dry) return 0;
    CFB_CHECK(bise_mean(a, m, N, hh * ww, 128, st));
    CFB_CHECK(bise_attention(BiseAttention{n->att_w[k], n->att_b[k], 128, 128, 2, nullptr, nullptr, 0, 0}, m, att, N, st));
    return bise_scale_add(a, att, add_vec, add_t, a, N, (int64_t)hh * ww, 128, st);
  };
  float *a32 = nullptr, *cp16 = nullptr, *a16 = nullptr, *fcat = nullptr;
  CFB_CHECK(n->alloc(&a32, px(h32, w32) * 128));
  CFB_CHECK(arm(1, F[2], h32, w32, a32, avg, nullptr));
  ar.release(F[2]); ar.release(v512); ar.release(avg);
  CFB_CHECK(n->alloc(&cp16, px(h16, w16) * 128));
  CFB_CHECK(conv(n->head32, a32, 128, h32, w32, cp16, 128, 0, OUT_RELU, nullptr));
  ar.release(a32);
  // feat16_sum = arm16(feat16) + feat32_up; feat_cp8 = conv_head16(up(feat16_sum)) -> fcat[128:256)
  CFB_CHECK(n->alloc(&a16, px(h16, w16) * 128));
  CFB_CHECK(arm(0, F[1], h16, w16, a16, nullptr, cp16));
  ar.release(F[1]);
  CFB_CHECK(n->alloc(&fcat, px(h8, w8) * 256));
  CFB_CHECK(conv(n->head16, a16, 128, h16, w16, fcat, 256, 128, OUT_RELU, nullptr));
  ar.release(a16);
  if (!dry) CFB_CHECK(yolo_copy(F[0], 128, 0, fcat, 256, 0, N, h8, w8, 128, false, st));
  ar.release(F[0]);
  // FFM: feat = convblk(fcat); feat * sigmoid(conv2(relu(conv1(avg_pool(feat))))) + feat
  float* ff = nullptr;
  CFB_CHECK(n->alloc(&ff, px(h8, w8) * 256));
  CFB_CHECK(conv(n->convblk, fcat, 256, h8, w8, ff, 256, 0, OUT_RELU, nullptr));
  if (!dry) {
    CFB_CHECK(bise_mean(ff, m, N, h8 * w8, 256, st));
    CFB_CHECK(bise_attention(BiseAttention{n->ffm_w1, nullptr, 256, 64, 1, n->ffm_w2, nullptr, 256, 2}, m, att, N, st));
    CFB_CHECK(bise_scale_add(ff, att, nullptr, nullptr, ff, N, (int64_t)h8 * w8, 256, st));
  }
  ar.release(m); ar.release(att);
  // BiSeNetOutput k on `in`: ConvBNReLU 3x3, conv_out 1x1 (64 padded channels), bilinear to H x W
  auto head = [&](int k, const float* in, int in_pitch, int hh, int ww) -> int {
    const GenConv &c = n->outc[k], &p = n->outp[k];
    float *t = nullptr, *lo = nullptr;
    CFB_CHECK(n->alloc(&t, px(hh, ww) * c.cout));
    CFB_CHECK(conv(c, in, in_pitch, hh, ww, t, c.cout, 0, OUT_RELU, nullptr));
    CFB_CHECK(n->alloc(&lo, px(hh, ww) * p.cout_p));
    CFB_CHECK(conv(p, t, p.cin_p, hh, ww, lo, p.cout_p, 0, OUT_NONE, nullptr));
    ar.release(t);
    if (!dry) {
      if (u8) CFB_CHECK(bise_bilinear_argmax(lo, p.cout_p, hh, ww, n->num_class, u8->cls, u8->mask, N, H, W, st));
      else CFB_CHECK(bise_bilinear(lo, p.cout_p, hh, ww, n->num_class, out[k], N, H, W, st));
    }
    ar.release(lo);
    return 0;
  };
  CFB_CHECK(head(0, ff, 256, h8, w8));
  ar.release(ff);
  if (!u8) {
    CFB_CHECK(head(1, fcat + 128, 256, h8, w8));
    CFB_CHECK(head(2, cp16, 128, h16, w16));
  }
  ar.release(fcat); ar.release(cp16);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// ResNetArcFace('IRBlock', layers, use_se=False): identity embeddings of faces (scoring a fidelity sweep)
//   /root/reference/basicsr/archs/arcface_arch.py:56-100 (IRBlock), 171-245 (ResNetArcFace); the gray 128 x 128 input of
//   basicsr/models/codeformer_model.py:131-135 (gray_resize_for_identity).
// Eval-mode BatchNorm after a conv is folded into its weights at prepare; the PReLU slopes (one scalar per module, shared by
// both activations of an IRBlock) are read from the parameters at prepare.  Engines per conv form:
//   stem (conv1 + bn1 + PReLU + MaxPool2d(2))          SIMT (arcface.cu), fp32 or uint8 BGR 512 x 512 faces (gray resize fused)
//   IRBlock bn0 -> conv1 3x3 + bn1 + PReLU            generalised halo engine: bn0 is the fused operand transform (affine
//                                                      without activation, applied inside the image only: the conv pads the
//                                                      normalised tensor with zeros, which a weight fold would not), PReLU
//                                                      epilogue
//   conv2 3x3 + bn2 + residual + PReLU, stride 1      generalised halo engine, residual + PReLU epilogue
//   conv2 3x3 stride 2 pad 1 (+ the same epilogue)    per-tap engine, PReLU epilogue
//   downsample 1x1 stride 2 + BN                      per-tap engine
//   bn4 -> flatten (NCHW) -> fc5 -> bn5               one linear (both BatchNorms folded, fc5's columns permuted to the NHWC
//                                                      flatten at prepare) as a per-tap 1x1 conv over the B rows
// 8 x 8 maps (layer4) are smaller than one 128-pixel tile: both engines run them as ragged tiles.
// =========================================================================================================
namespace cfb {
struct ArcBlock {
  int cin = 0, cout = 0, stride = 1;
  GenConv c1, c2, ds;
  bool has_ds = false;
  float slope = 0.f;
};
}
struct cfb_arcface : cfb::NetCore {
  cfb_arcface() : NetCore("ResNetArcFace", "arcface") {}
  int layers[4] = {2, 2, 2, 2};
  std::vector<cfb::ArcBlock> blocks;
  cfb::ArcBn0Table bn0;                    // channel offsets of each block's bn0 in bn0_scale / bn0_shift
  float *bn0_scale = nullptr, *bn0_shift = nullptr;
  float *stem_w = nullptr, *stem_b = nullptr;
  float stem_slope = 0.f;
  cfb::GenConv fc;                         // [512][8 * 8 * 512] on the NHWC flatten
};
namespace cfb {

constexpr int ARC_FEAT = 8 * 8 * 512;      // fc5's input: layer4 at 8 x 8 for a 128 x 128 input

static int arc_build(cfb_arcface* n) {     // ResNetArcFace.__init__ / _make_layer, arcface_arch.py:183-227
  n->blocks.clear();
  int inplanes = 64, total = 0;
  for (int l = 0; l < 4; ++l) {
    CFB_REQUIRE(n->layers[l] >= 1, "ResNetArcFace: every layer needs at least one block");
    total += n->layers[l];
  }
  CFB_REQUIRE(total <= ArcBn0Table::kMax, "ResNetArcFace: at most " + std::to_string(ArcBn0Table::kMax) + " blocks");
  n->bn0 = ArcBn0Table{};
  for (int l = 0; l < 4; ++l) {
    const int planes = 64 << l;
    for (int b = 0; b < n->layers[l]; ++b) {
      const std::string p = "layer" + std::to_string(l + 1) + "." + std::to_string(b) + ".";
      ArcBlock k;
      k.cin = inplanes; k.cout = planes; k.stride = (b == 0 && l > 0) ? 2 : 1;
      k.c1 = plan_conv(p + "conv1.weight", inplanes, inplanes, 3, 1); k.c1.bn = p + "bn1.";
      k.c2 = plan_conv(p + "conv2.weight", inplanes, planes, 3, k.stride); k.c2.bn = p + "bn2.";
      k.has_ds = b == 0 && (k.stride != 1 || inplanes != planes);
      if (k.has_ds) { k.ds = plan_conv(p + "downsample.0.weight", inplanes, planes, 1, k.stride); k.ds.bn = p + "downsample.1."; }
      n->bn0.off[n->bn0.blocks + 1] = n->bn0.off[n->bn0.blocks] + inplanes;
      ++n->bn0.blocks;
      n->blocks.push_back(k);
      inplanes = planes;
    }
  }
  n->fc = plan_conv("fc5.weight", ARC_FEAT, 512, 1, 1);
  return 0;
}

static int arc_prepare(cfb_arcface* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  CFB_CHECK(arc_build(n));
  SlabPlan plan;
  for (const ArcBlock& b : n->blocks) { plan.add(b.c1); plan.add(b.c2); if (b.has_ds) plan.add(b.ds); }
  const int C0 = n->bn0.off[n->bn0.blocks];
  const size_t fc_wn = (size_t)512 * ARC_FEAT;
  CFB_CHECK(n->reserve_slab(plan.bytes() + 2 * align256((size_t)C0 * 4) + align256(64 * 9 * 4) + align256(64 * 4) +
                            2 * align256(fc_wn * 2) + align256(512 * 4) + 256 + 4 * align256(512 * 4)));
  WeightPrep wp(*n, plan, st);
  n->bn0_scale = (float*)wp.take((size_t)C0 * 4); n->bn0_shift = (float*)wp.take((size_t)C0 * 4);
  auto bn_affine = [&](const std::string& bn, int c, float* scale, float* shift) -> int {
    const float* g = n->param(bn + "weight", c);
    const float* be = n->param(bn + "bias", c);
    const float* mu = n->param(bn + "running_mean", c);
    const float* var = n->param(bn + "running_var", c);
    if (!g || !be || !mu || !var) return 1;
    return arc_bn_affine(g, be, mu, var, 1e-5f, scale, shift, c, st);      // nn.BatchNorm2d / BatchNorm1d default eps
  };
  std::vector<float> slopes(n->blocks.size() + 1, 0.f);
  auto slope = [&](const std::string& name, float* dst) -> int {
    const float* s = n->param(name, 1);
    if (!s) return 1;
    CFB_CUDA(cudaMemcpyAsync(dst, s, 4, cudaMemcpyDeviceToHost, st));
    return 0;
  };
  auto folded = [&](GenConv& c) -> int {
    CFB_CHECK(wp.fold(c.name, c.bn, c.cout, c.cin * c.k * c.k));
    return wp.conv(c, wp.fold_w, wp.fold_b);
  };
  for (size_t i = 0; i < n->blocks.size(); ++i) {
    ArcBlock& b = n->blocks[i];
    const std::string p = b.c1.name.substr(0, b.c1.name.size() - std::string("conv1.weight").size());
    CFB_CHECK(bn_affine(p + "bn0.", b.cin, n->bn0_scale + n->bn0.off[i], n->bn0_shift + n->bn0.off[i]));
    CFB_CHECK(folded(b.c1));
    CFB_CHECK(folded(b.c2));
    if (b.has_ds) CFB_CHECK(folded(b.ds));
    CFB_CHECK(slope(p + "prelu.weight", &slopes[i]));
  }
  n->stem_w = (float*)wp.take(64 * 9 * 4); n->stem_b = (float*)wp.take(64 * 4);
  CFB_CHECK(wp.fold("conv1.weight", "bn1.", 64, 9));
  CFB_CUDA(cudaMemcpyAsync(n->stem_w, wp.fold_w, 64 * 9 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaMemcpyAsync(n->stem_b, wp.fold_b, 64 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CHECK(slope("prelu.weight", &slopes.back()));
  // the head: bn4 / bn5 as per-channel affines, folded with fc5 into a temporary fp32 weight, then split into the slab
  GenConv& fc = n->fc;
  fc.w_hi = (__half*)wp.take(fc_wn * 2); fc.w_lo = (__half*)wp.take(fc_wn * 2);
  fc.bias = (float*)wp.take(512 * 4); fc.wscale = (float*)wp.take(8);
  float* s4 = (float*)wp.take(512 * 4); float* t4 = (float*)wp.take(512 * 4);
  float* s5 = (float*)wp.take(512 * 4); float* t5 = (float*)wp.take(512 * 4);
  CFB_CHECK(bn_affine("bn4.", 512, s4, t4));
  CFB_CHECK(bn_affine("bn5.", 512, s5, t5));
  const float* w5 = n->param("fc5.weight", (int64_t)fc_wn);
  const float* b5 = n->param("fc5.bias", 512);
  if (!w5 || !b5) return 1;
  float* tmp = nullptr;
  CFB_CUDA(cudaMalloc((void**)&tmp, fc_wn * 4));
  int rc = arc_fold_fc(w5, b5, s4, t4, s5, t5, 512, 512, 64, tmp, fc.bias, st);
  if (rc == 0) rc = tc_split_weights(tmp, fc.w_hi, fc.w_lo, 512, ARC_FEAT, 1, fc.wscale, st);
  const cudaError_t se = cudaStreamSynchronize(st);
  cudaFree(tmp);
  if (rc) return rc;
  CFB_REQUIRE(se == cudaSuccess, std::string("ResNetArcFace prepare: ") + cudaGetErrorString(se));
  for (size_t i = 0; i < n->blocks.size(); ++i) n->blocks[i].slope = slopes[i];
  n->stem_slope = slopes.back();
  n->prepared = true;
  return 0;
}

// x: fp32 [N,1,128,128] or faces: uint8 HWC BGR [N,512,512,3] -> emb [N,512]
static int arc_forward(cfb_arcface* n, const float* x, const unsigned char* faces, float* emb, int N, void* ws, int64_t ws_bytes,
                       cudaStream_t st, bool dry) {
  CFB_CHECK(n->begin_forward(dry));
  CFB_REQUIRE(N >= 0, "ResNetArcFace: negative batch");
  if (N == 0) return 0;
  if (n->blocks.empty()) CFB_CHECK(arc_build(n));
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  float *sc = nullptr, *sh = nullptr, *cur = nullptr;
  CFB_CHECK(n->alloc(&sc, (size_t)N * n->bn0.off[n->bn0.blocks]));
  CFB_CHECK(n->alloc(&sh, (size_t)N * n->bn0.off[n->bn0.blocks]));
  if (!dry) CFB_CHECK(arc_bn0_tables(n->bn0_scale, n->bn0_shift, n->bn0, N, sc, sh, st));
  CFB_CHECK(n->alloc(&cur, (size_t)N * 64 * 64 * 64));
  if (!dry) CFB_CHECK(arc_stem(x, faces, n->stem_w, n->stem_b, n->stem_slope, cur, N, st));
  int h = 64;
  for (size_t i = 0; i < n->blocks.size(); ++i) {
    const ArcBlock& b = n->blocks[i];
    const int ho = b.stride == 2 ? h / 2 : h;
    float *t1 = nullptr, *res = cur, *y = nullptr;
    CFB_CHECK(n->alloc(&t1, (size_t)N * h * h * b.cin));
    {   // prelu(bn1(conv1(bn0(x))))
      GenLaunch g{&b.c1, cur, b.cin, h, h, N, t1, b.cin, 0, OUT_PRELU};
      g.in_scale = sc + (size_t)N * n->bn0.off[i]; g.in_shift = sh + (size_t)N * n->bn0.off[i]; g.prelu = b.slope;
      if (!dry) CFB_CHECK(gen_conv(g, n->sm_count, st));
    }
    if (b.has_ds) {
      CFB_CHECK(n->alloc(&res, (size_t)N * ho * ho * b.cout));
      CFB_CHECK(pertap_conv(*n, pertap_args(cur, N, h, h, b.cin, b.cout, 1, b.stride, res, 0, 0, OUT_NONE, nullptr), b.ds, dry, st));
    }
    CFB_CHECK(n->alloc(&y, (size_t)N * ho * ho * b.cout));
    if (b.c2.gen) {   // prelu(bn2(conv2(.)) + residual)
      GenLaunch g{&b.c2, t1, b.cin, h, h, N, y, b.cout, 0, OUT_PRELU};
      g.res = res; g.res_pitch = b.cout; g.prelu = b.slope;
      if (!dry) CFB_CHECK(gen_conv(g, n->sm_count, st));
    } else {
      ConvArgs a = pertap_args(t1, N, h, h, b.cin, b.cout, 3, 2, y, 0, 0, OUT_PRELU, res);
      a.prelu_slope = b.slope;
      CFB_CHECK(pertap_conv(*n, a, b.c2, dry, st));
    }
    ar.release(t1);
    if (res != cur) ar.release(res);
    ar.release(cur);
    cur = y; h = ho;
  }
  CFB_REQUIRE(h == 8 && n->blocks.back().cout == 512, "ResNetArcFace: layer4 must end at 8 x 8 x 512");
  // the head: the N flattened NHWC rows as one 1 x N image of ARC_FEAT channels; its operand planes are the plain fp16 split of
  // the rows (concat_planes with one source), as the per-tap engine's own operand pass builds them for at most 2048 channels
  ConvArgs a = pertap_args(cur, 1, 1, N, ARC_FEAT, 512, 1, 1, emb, 0, 0, OUT_NONE, nullptr);
  a.wgt_hi = n->fc.w_hi; a.wgt_lo = n->fc.w_lo; a.wscale_inv = n->fc.wscale + 1; a.bias = n->fc.bias; a.skip_prep = true;
  CFB_REQUIRE(tc_supported(a), "ResNetArcFace: head not supported by the wgmma engine");
  void* planes = ar.alloc(tc_scratch_bytes(a));
  CFB_REQUIRE(planes != nullptr, n->ws_error());
  if (!dry) {
    CFB_CHECK(concat_planes(cur, nullptr, planes, N, ARC_FEAT, 0, st));
    CFB_CHECK(conv_tc(a, planes, n->sm_count, st));
  }
  ar.release(planes);
  ar.release(cur);
  ar.release(sc); ar.release(sh);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// LPIPS(net='vgg', version='0.1'): the perceptual distance of restored faces (lpips 0.1; basicsr/losses/losses.py:257-282,
// LPIPSLoss, the perceptual term of every CodeFormer training config).
//   ScalingLayer -> torchvision vgg16().features cut after relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 -> per layer k:
//   f / (|f|_c + 1e-10) of both images, (f0 - f1)^2, lin_k (1x1, C -> 1, no bias), mean over H x W -> val = sum over k.
// Engines:
//   conv1_1 (3 -> 64) + ReLU                    SIMT stem (lpips.cu), the input transform fused into its load
//   the 12 other 3x3 convs + ReLU               generalised halo engine (biases kept; no BatchNorm)
//   head of relu_k + MaxPool2d(2, 2) into the next slice      one SIMT pass over relu_k (lpips.cu), then a finalize
// A launch holds `groups` groups of one reference and G candidates; every relu_k is released after its head-and-pool pass, so
// the workspace peaks at two relu1 maps of the launch's images.
// =========================================================================================================
struct cfb_lpips : cfb::NetCore {
  cfb_lpips() : NetCore("LPIPS", "lpips") {}
  cfb::GenConv convs[12];                  // conv1_2 .. conv5_3
  float *stem_w = nullptr, *stem_b = nullptr;
  float* lin[5] = {};
  float* tables = nullptr;                 // [LPIPS_U8_CONVENTIONS][3][256] uint8 -> stem input, RGB channel order
  float shift[3] = {}, scale[3] = {};      // ScalingLayer, read at prepare
};
namespace cfb {

// torchvision vgg16().features: index, cin, cout of the 13 convs; the conv count that ends each LPIPS slice
static const int kLpConv[13][3] = {{0, 3, 64},     {2, 64, 64},     {5, 64, 128},    {7, 128, 128},  {10, 128, 256},
                                   {12, 256, 256}, {14, 256, 256},  {17, 256, 512},  {19, 512, 512}, {21, 512, 512},
                                   {24, 512, 512}, {26, 512, 512},  {28, 512, 512}};
static const int kLpSliceEnd[5] = {2, 4, 7, 10, 13};
constexpr int LPIPS_U8_CONVENTIONS = 2;

static std::string lp_conv_name(int i) {   // net.slice<s>.<index>. (lpips pretrained_networks.vgg16: features[x] in slice s)
  const int idx = kLpConv[i][0];
  const int s = idx < 4 ? 1 : idx < 9 ? 2 : idx < 16 ? 3 : idx < 23 ? 4 : 5;
  return "net.slice" + std::to_string(s) + "." + std::to_string(idx) + ".";
}

// The per-channel table of a uint8 convention, on the host in each step's own precision (x86-64 SSE: IEEE single / double,
// no contraction), RGB channel order:
//   0 'lpips'       lpips.im2tensor: float32(u / 127.5 - 1) [numpy float64], then the ScalingLayer in fp32
//   1 'codeformer'  float32(u / 255.) [float64 division] and normalize(0.5, 0.5) (the training pipeline's image tensors), then
//                   LPIPSLoss(use_input_norm=True, range_norm=True): (x + 1) / 2, (x - mean) / std, then the ScalingLayer
static int lp_u8_table(int convention, const float shift[3], const float scale[3], float* t) {
  CFB_REQUIRE(convention >= 0 && convention < LPIPS_U8_CONVENTIONS, "LPIPS: unknown uint8 convention");
  const float mean[3] = {(float)0.485, (float)0.456, (float)0.406}, stdv[3] = {(float)0.229, (float)0.224, (float)0.225};
  for (int c = 0; c < 3; ++c)
    for (int u = 0; u < 256; ++u) {
      float x;
      if (convention == 0) {
        x = (float)((double)u / 127.5 - 1.0);
      } else {
        const float v = (float)((double)u / 255.0);
        x = (v - 0.5f) / 0.5f;
        x = (x + 1.f) / 2.f;
        x = (x - mean[c]) / stdv[c];
      }
      t[c * 256 + u] = (x - shift[c]) / scale[c];
    }
  return 0;
}

static LpipsXform lp_xform(const cfb_lpips* n, int flags) {
  LpipsXform x;
  x.flags = flags;
  const float mean[3] = {(float)0.485, (float)0.456, (float)0.406}, stdv[3] = {(float)0.229, (float)0.224, (float)0.225};
  for (int c = 0; c < 3; ++c) { x.mean[c] = mean[c]; x.std[c] = stdv[c]; x.shift[c] = n->shift[c]; x.scale[c] = n->scale[c]; }
  return x;
}

static int lp_prepare(cfb_lpips* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  SlabPlan plan;
  for (int i = 0; i < 12; ++i) {
    n->convs[i] = plan_conv(lp_conv_name(i + 1) + "weight", kLpConv[i + 1][1], kLpConv[i + 1][2]);
    plan.add(n->convs[i]);
  }
  const size_t tbytes = (size_t)LPIPS_U8_CONVENTIONS * 3 * 256 * 4;
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256(64 * 27 * 4) + align256(64 * 4) + 5 * align256(512 * 4) + align256(tbytes)));
  WeightPrep wp(*n, plan, st);
  for (int i = 0; i < 12; ++i) {
    GenConv& c = n->convs[i];
    const std::string p = lp_conv_name(i + 1);
    const float* w = n->param(p + "weight", (int64_t)c.cout * c.cin * 9);
    const float* b = n->param(p + "bias", c.cout);
    if (!w || !b) return 1;
    CFB_CHECK(wp.conv(c, w, b));
  }
  const float* w0 = n->param("net.slice1.0.weight", 64 * 27);
  const float* b0 = n->param("net.slice1.0.bias", 64);
  const float* sh = n->param("scaling_layer.shift", 3);
  const float* sc = n->param("scaling_layer.scale", 3);
  if (!w0 || !b0 || !sh || !sc) return 1;
  n->stem_w = (float*)wp.take(64 * 27 * 4); n->stem_b = (float*)wp.take(64 * 4);
  CFB_CUDA(cudaMemcpyAsync(n->stem_w, w0, 64 * 27 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaMemcpyAsync(n->stem_b, b0, 64 * 4, cudaMemcpyDeviceToDevice, st));
  for (int k = 0; k < 5; ++k) {
    const int C = kLpConv[kLpSliceEnd[k] - 1][2];
    const float* l = n->param("lin" + std::to_string(k) + ".model.1.weight", C);
    if (!l) return 1;
    n->lin[k] = (float*)wp.take(512 * 4);
    CFB_CUDA(cudaMemcpyAsync(n->lin[k], l, (size_t)C * 4, cudaMemcpyDeviceToDevice, st));
  }
  CFB_CUDA(cudaMemcpyAsync(n->shift, sh, 12, cudaMemcpyDeviceToHost, st));
  CFB_CUDA(cudaMemcpyAsync(n->scale, sc, 12, cudaMemcpyDeviceToHost, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  std::vector<float> t((size_t)LPIPS_U8_CONVENTIONS * 768);
  for (int c = 0; c < LPIPS_U8_CONVENTIONS; ++c) CFB_CHECK(lp_u8_table(c, n->shift, n->scale, t.data() + (size_t)c * 768));
  n->tables = (float*)wp.take(tbytes);
  CFB_CUDA(cudaMemcpyAsync(n->tables, t.data(), tbytes, cudaMemcpyHostToDevice, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// The inputs of a launch: fp32 NCHW ref [groups,3,H,W] / cand [groups*G,3,H,W] with the LpipsXform flags, or uint8 HWC BGR
// ref8 [groups,H,W,3] / cand8 [groups*G,H,W,3] with a convention.
struct LpIn {
  const float* ref = nullptr; const float* cand = nullptr; int flags = 0;
  const unsigned char* ref8 = nullptr; const unsigned char* cand8 = nullptr; int convention = -1;
};

static int lp_stem(cfb_lpips* n, const LpIn& in, float* out, int groups, int G, int H, int W, cudaStream_t st) {
  const float* table = nullptr;
  if (in.ref8) {
    CFB_REQUIRE(in.convention >= 0 && in.convention < LPIPS_U8_CONVENTIONS, "LPIPS: unknown uint8 convention");
    table = n->tables + (size_t)in.convention * 768;
  }
  CFB_REQUIRE(in.flags >= 0 && in.flags < 8, "LPIPS: unknown input transform flags");
  return lpips_stem(in.ref, in.cand, in.ref8, in.cand8, table, lp_xform(n, in.flags), n->stem_w, n->stem_b, out, groups, G, H, W, st);
}

static int lp_forward(cfb_lpips* n, const LpIn& in, int groups, int G, int H, int W, float* val, float* per_layer, void* ws,
                      int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_CHECK(n->begin_forward(dry));
  CFB_REQUIRE(groups >= 0 && G >= 1, "LPIPS: a group needs at least one candidate");
  CFB_REQUIRE(H >= 16 && W >= 16, "LPIPS: H and W must be at least 16 (relu5_3 is at 1/16 of the input)");
  if (groups == 0) return 0;
  const int64_t M = (int64_t)groups * (1 + G), P = (int64_t)groups * G;
  CFB_REQUIRE(M <= 65535, "LPIPS: at most 65535 images per launch");
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  LpipsLayers L;
  L.n = 5;
  float* part[5] = {};
  for (int k = 0, h = H, w = W; k < 5; ++k, h /= 2, w /= 2) {
    L.nblk[k] = lpips_head_blocks(h, w);
    L.hw[k] = (int64_t)h * w;
    CFB_CHECK(n->alloc(&part[k], (size_t)P * L.nblk[k]));
    L.part[k] = part[k];
  }
  float* cur = nullptr;
  CFB_CHECK(n->alloc(&cur, (size_t)M * H * W * 64));
  if (!dry) CFB_CHECK(lp_stem(n, in, cur, groups, G, H, W, st));
  int h = H, w = W, ci = 1;
  for (int s = 0; s < 5; ++s) {
    for (; ci < kLpSliceEnd[s]; ++ci) {
      const GenConv& c = n->convs[ci - 1];
      float* y = nullptr;
      CFB_CHECK(n->alloc(&y, (size_t)M * h * w * c.cout));
      GenLaunch g{&c, cur, c.cin, h, w, (int)M, y, c.cout, 0, OUT_RELU};
      if (!dry) CFB_CHECK(gen_conv(g, n->sm_count, st));
      ar.release(cur);
      cur = y;
    }
    const int C = kLpConv[ci - 1][2];
    float* pooled = nullptr;
    if (s < 4) CFB_CHECK(n->alloc(&pooled, (size_t)M * (h / 2) * (w / 2) * C));
    if (!dry) CFB_CHECK(lpips_head(cur, n->lin[s], groups, G, h, w, C, pooled, part[s], st));
    ar.release(cur);
    cur = pooled; h /= 2; w /= 2;
  }
  if (!dry) CFB_CHECK(lpips_finalize(L, (int)P, val, per_layer, st));
  for (float* p : part) ar.release(p);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// YOLOv5l-face: the other large detector of whole-image mode (--detection_model YOLOv5l)
//   facelib/detection/yolov5face/models/yolov5l.yaml, common.py (Conv, StemBlock, C3, Bottleneck, SPP), yolo.py (Detect).
// Every Conv is conv (no bias) + BatchNorm2d (folded at prepare) + SiLU.  Engines per conv form:
//   stem_1 (3x3 s2, 3 -> 64)                      SIMT (yolo.cu), fp32 or uint8 BGR input with the letterbox fused
//   3x3 stride 1 (Bottleneck cv2)                 generalised halo engine, SiLU epilogue; the shortcut enters as residual2
//                                                 after the activation (x + silu(bn(conv)))
//   1x1, 3x3 stride 2 pad 1, Detect (48 -> 64)   per-tap engine, SiLU epilogue (none for Detect), destination slices
// The concatenations never run as copies of both halves: C3's m-chain and cv2 write the two halves of cv3's input, the stem's
// stem_2b and max pool the two halves of stem_3's input, SPP's cv1 and pools the four quarters of cv2's input, and the head's
// convs 9 / 13 / 17 / 20 write into the concat buffers of layers 21 / 18 / 18 / 21.  The copy kernel fills the rest: the
// nearest x2 upsamples (layers 10, 14) and the backbone features of layers 11 and 15.
// =========================================================================================================
struct cfb_yolov5face : cfb::NetCore {
  cfb_yolov5face() : NetCore("YOLOv5-face", "yolov5face") {}
  std::unordered_map<std::string, cfb::GenConv> convs;     // by module prefix, e.g. "model.1.m.0.cv2"
  float *stem_w = nullptr, *stem_b = nullptr, *anchor_grid = nullptr;
};
namespace cfb {

// (layer, c1, c2, bottlenecks, shortcut) of the eight C3 blocks of yolov5l.yaml
struct YoC3 { int i, c1, c2, n; bool sc; };
static const YoC3 kYoC3[8] = {{1, 64, 128, 3, true},     {3, 256, 256, 9, true},
                                                               {5, 512, 512, 9, true},    {8, 1024, 1024, 3, false},
                                                               {12, 1024, 512, 3, false}, {16, 512, 256, 3, false},
                                                               {19, 512, 512, 3, false},  {22, 1024, 1024, 3, false}};

static void yo_build(cfb_yolov5face* n) {
  n->convs.clear();
  auto add = [&](const std::string& name, int cin, int cout, int k, int stride, bool bn = true) {
    GenConv c = plan_conv(name, cin, cout, k, stride);
    if (bn) c.bn = name + ".bn.";
    n->convs[name] = c;
  };
  add("model.0.stem_2a", 64, 32, 1, 1);
  add("model.0.stem_2b", 32, 64, 3, 2);
  add("model.0.stem_3", 128, 64, 1, 1);
  for (const auto& b : kYoC3) {
    const std::string p = "model." + std::to_string(b.i) + ".";
    const int c_ = b.c2 / 2;
    add(p + "cv1", b.c1, c_, 1, 1);
    add(p + "cv2", b.c1, c_, 1, 1);
    add(p + "cv3", 2 * c_, b.c2, 1, 1);
    for (int j = 0; j < b.n; ++j) {
      add(p + "m." + std::to_string(j) + ".cv1", c_, c_, 1, 1);
      add(p + "m." + std::to_string(j) + ".cv2", c_, c_, 3, 1);
    }
  }
  add("model.2", 128, 256, 3, 2);
  add("model.4", 256, 512, 3, 2);
  add("model.6", 512, 1024, 3, 2);
  add("model.7.cv1", 1024, 512, 1, 1);
  add("model.7.cv2", 2048, 1024, 1, 1);
  add("model.9", 1024, 512, 1, 1);
  add("model.13", 512, 256, 1, 1);
  add("model.17", 256, 256, 3, 2);
  add("model.20", 512, 512, 3, 2);
  const int ch[3] = {256, 512, 1024};
  for (int l = 0; l < 3; ++l) add("model.23.m." + std::to_string(l), ch[l], 48, 1, 1, false);
}

static int yo_prepare(cfb_yolov5face* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  yo_build(n);
  SlabPlan plan;
  for (const auto& kv : n->convs) plan.add(kv.second);
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256((size_t)64 * 27 * 4) + align256(256) + align256(18 * 4)));
  WeightPrep wp(*n, plan, st);
  for (auto& kv : n->convs) {
    GenConv& c = kv.second;
    if (!c.bn.empty()) {
      CFB_CHECK(wp.fold(c.name + ".conv.weight", c.bn, c.cout, c.cin * c.k * c.k));
    } else {                 // Detect: plain conv with bias
      const float* w = n->param(c.name + ".weight", (int64_t)c.cout * c.cin);
      const float* b = n->param(c.name + ".bias", c.cout);
      if (!w || !b) return 1;
      CFB_CUDA(cudaMemcpyAsync(wp.fold_w, w, (size_t)c.cout * c.cin * 4, cudaMemcpyDeviceToDevice, st));
      CFB_CUDA(cudaMemcpyAsync(wp.fold_b, b, (size_t)c.cout * 4, cudaMemcpyDeviceToDevice, st));
    }
    CFB_CHECK(wp.conv(c, wp.fold_w, wp.fold_b));      // stem_2a / stem_2b / Detect: zero-padded to 64 channels
  }
  n->stem_w = (float*)wp.take((size_t)64 * 27 * 4); n->stem_b = (float*)wp.take(256);
  CFB_CHECK(wp.fold("model.0.stem_1.conv.weight", "model.0.stem_1.bn.", 64, 27));
  CFB_CUDA(cudaMemcpyAsync(n->stem_w, wp.fold_w, (size_t)64 * 27 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaMemcpyAsync(n->stem_b, wp.fold_b, 64 * 4, cudaMemcpyDeviceToDevice, st));
  const float* ag = n->param("model.23.anchor_grid", 18);
  if (!ag) return 1;
  n->anchor_grid = (float*)wp.take(18 * 4);
  CFB_CUDA(cudaMemcpyAsync(n->anchor_grid, ag, 18 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

// predictions of an h x w input: 3 anchors per cell of the /8, /16, /32 maps
static int64_t yo_predictions(int H, int W) {
  return 3 * ((int64_t)(H / 8) * (W / 8) + (int64_t)(H / 16) * (W / 16) + (int64_t)(H / 32) * (W / 32));
}

static int yo_forward(cfb_yolov5face* n, const float* x, const unsigned char* img, int ih, int iw, int top, int left, float* pred,
                      float* const raw[3], int N, int H, int W, void* ws, int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_CHECK(n->begin_forward(dry));
  CFB_REQUIRE(H >= 32 && W >= 32 && H % 32 == 0 && W % 32 == 0 && N >= 0, "YOLOv5-face: H and W must be positive multiples of 32");
  CFB_REQUIRE(!img || (ih >= 1 && iw >= 1 && top >= 0 && left >= 0 && top + ih <= H && left + iw <= W),
              "YOLOv5-face: the image must lie inside the letterbox canvas");
  CFB_REQUIRE(yo_predictions(H, W) * N < ((int64_t)1 << 31) / 16 && (int64_t)H * W <= ((int64_t)1 << 26), "YOLOv5-face: image too large");
  if (N == 0) return 0;
  if (n->convs.empty()) yo_build(n);
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  auto alloc = [&](float** p, int h, int w, int c) { return n->alloc(p, (size_t)N * h * w * c); };
  // one conv: 3x3 stride 1 on the generalised engine (res2: the Bottleneck shortcut), everything else on the per-tap engine
  auto conv = [&](const std::string& name, const float* in, int h, int w, float* out, int out_pitch, int out_c0, int act,
                  const float* res2 = nullptr, int res2_pitch = 0) -> int {
    const GenConv& c = n->convs.at(name);
    if (c.gen) {
      GenLaunch g{&c, in, c.cin_p, h, w, N, out, out_pitch, out_c0, act};
      g.res2 = res2; g.res2_pitch = res2_pitch;
      return dry ? 0 : gen_conv(g, n->sm_count, st);
    }
    return pertap_conv(*n, pertap_args(in, N, h, w, c.cin_p, c.cout_p, c.k, c.stride, out, out_pitch, out_c0, act, nullptr), c, dry, st);
  };
  // C3 (common.py): cv3(cat(m(cv1(x)), cv2(x))) with the cat as one [2c_] buffer; out: a dense [c2] buffer
  auto c3 = [&](int i, const float* in, int h, int w, float** out) -> int {
    const YoC3& b = *std::find_if(std::begin(kYoC3), std::end(kYoC3), [&](const YoC3& e) { return e.i == i; });
    const std::string p = "model." + std::to_string(i) + ".";
    const int c_ = b.c2 / 2;
    float *cat = nullptr, *a = nullptr, *t = nullptr;
    CFB_CHECK(alloc(&cat, h, w, 2 * c_));
    CFB_CHECK(conv(p + "cv2", in, h, w, cat, 2 * c_, c_, OUT_SILU));
    CFB_CHECK(alloc(&a, h, w, c_));
    CFB_CHECK(conv(p + "cv1", in, h, w, a, c_, 0, OUT_SILU));
    CFB_CHECK(alloc(&t, h, w, c_));
    for (int j = 0; j < b.n; ++j) {
      const std::string m = p + "m." + std::to_string(j) + ".";
      CFB_CHECK(conv(m + "cv1", a, h, w, t, c_, 0, OUT_SILU));
      float* dst = nullptr;
      if (j == b.n - 1) dst = cat;
      else CFB_CHECK(alloc(&dst, h, w, c_));
      CFB_CHECK(conv(m + "cv2", t, h, w, dst, j == b.n - 1 ? 2 * c_ : c_, 0, OUT_SILU, b.sc ? a : nullptr, c_));
      ar.release(a);
      a = dst;
    }
    ar.release(t);
    CFB_CHECK(alloc(out, h, w, b.c2));
    CFB_CHECK(conv(p + "cv3", cat, h, w, *out, b.c2, 0, OUT_SILU));
    ar.release(cat);
    return 0;
  };
  const int H2 = H / 2, W2 = W / 2, H4 = H / 4, W4 = W / 4, H8 = H / 8, W8 = W / 8, H16 = H / 16, W16 = W / 16, H32 = H / 32,
            W32 = W / 32;
  // StemBlock
  float *s1 = nullptr, *t = nullptr, *sc = nullptr, *x0 = nullptr;
  CFB_CHECK(alloc(&s1, H2, W2, 64));
  if (!dry) CFB_CHECK(yolo_stem(x, img, n->stem_w, n->stem_b, s1, N, H, W, ih, iw, top, left, st));
  CFB_CHECK(alloc(&t, H2, W2, 64));
  CFB_CHECK(conv("model.0.stem_2a", s1, H2, W2, t, 64, 0, OUT_SILU));          // 32 channels + 32 zero channels
  CFB_CHECK(alloc(&sc, H4, W4, 128));
  CFB_CHECK(conv("model.0.stem_2b", t, H2, W2, sc, 128, 0, OUT_SILU));
  ar.release(t);
  if (!dry) CFB_CHECK(yolo_maxpool2(s1, sc, N, H2, W2, 64, 128, 64, st));
  ar.release(s1);
  CFB_CHECK(alloc(&x0, H4, W4, 64));
  CFB_CHECK(conv("model.0.stem_3", sc, H4, W4, x0, 64, 0, OUT_SILU));
  ar.release(sc);
  // backbone
  float *x1 = nullptr, *x2 = nullptr, *x3 = nullptr, *x4 = nullptr, *x5 = nullptr, *x6 = nullptr, *sp = nullptr, *x7 = nullptr,
        *x8 = nullptr;
  CFB_CHECK(c3(1, x0, H4, W4, &x1));
  ar.release(x0);
  CFB_CHECK(alloc(&x2, H8, W8, 256));
  CFB_CHECK(conv("model.2", x1, H4, W4, x2, 256, 0, OUT_SILU));
  ar.release(x1);
  CFB_CHECK(c3(3, x2, H8, W8, &x3));
  ar.release(x2);
  CFB_CHECK(alloc(&x4, H16, W16, 512));
  CFB_CHECK(conv("model.4", x3, H8, W8, x4, 512, 0, OUT_SILU));
  CFB_CHECK(c3(5, x4, H16, W16, &x5));
  ar.release(x4);
  CFB_CHECK(alloc(&x6, H32, W32, 1024));
  CFB_CHECK(conv("model.6", x5, H16, W16, x6, 1024, 0, OUT_SILU));
  CFB_CHECK(alloc(&sp, H32, W32, 2048));                                   // SPP: [cv1 | mp3 | mp5 | mp7]
  CFB_CHECK(conv("model.7.cv1", x6, H32, W32, sp, 2048, 0, OUT_SILU));
  ar.release(x6);
  if (!dry) CFB_CHECK(yolo_spp(sp, N, H32, W32, 512, st));
  CFB_CHECK(alloc(&x7, H32, W32, 1024));
  CFB_CHECK(conv("model.7.cv2", sp, H32, W32, x7, 1024, 0, OUT_SILU));
  ar.release(sp);
  CFB_CHECK(c3(8, x7, H32, W32, &x8));
  ar.release(x7);
  // head: cat21 = [20 | 9] at /32, cat11 = [up(9) | 5] at /16, cat18 = [17 | 13] at /16, cat15 = [up(13) | 3] at /8
  float *cat21 = nullptr, *cat11 = nullptr, *cat18 = nullptr, *cat15 = nullptr, *x12 = nullptr, *p3 = nullptr, *p4 = nullptr,
        *p5 = nullptr;
  CFB_CHECK(alloc(&cat21, H32, W32, 1024));
  CFB_CHECK(conv("model.9", x8, H32, W32, cat21, 1024, 512, OUT_SILU));
  ar.release(x8);
  CFB_CHECK(alloc(&cat11, H16, W16, 1024));
  if (!dry) CFB_CHECK(yolo_copy(cat21, 1024, 512, cat11, 1024, 0, N, H32, W32, 512, true, st));
  if (!dry) CFB_CHECK(yolo_copy(x5, 512, 0, cat11, 1024, 512, N, H16, W16, 512, false, st));
  ar.release(x5);
  CFB_CHECK(c3(12, cat11, H16, W16, &x12));
  ar.release(cat11);
  CFB_CHECK(alloc(&cat18, H16, W16, 512));
  CFB_CHECK(conv("model.13", x12, H16, W16, cat18, 512, 256, OUT_SILU));
  ar.release(x12);
  CFB_CHECK(alloc(&cat15, H8, W8, 512));
  if (!dry) CFB_CHECK(yolo_copy(cat18, 512, 256, cat15, 512, 0, N, H16, W16, 256, true, st));
  if (!dry) CFB_CHECK(yolo_copy(x3, 256, 0, cat15, 512, 256, N, H8, W8, 256, false, st));
  ar.release(x3);
  CFB_CHECK(c3(16, cat15, H8, W8, &p3));
  ar.release(cat15);
  CFB_CHECK(conv("model.17", p3, H8, W8, cat18, 512, 0, OUT_SILU));
  CFB_CHECK(c3(19, cat18, H16, W16, &p4));
  ar.release(cat18);
  CFB_CHECK(conv("model.20", p4, H16, W16, cat21, 1024, 0, OUT_SILU));
  CFB_CHECK(c3(22, cat21, H32, W32, &p5));
  ar.release(cat21);
  // Detect
  const float* P[3] = {p3, p4, p5};
  const int ny[3] = {H8, H16, H32}, nx[3] = {W8, W16, W32};
  float* hd[3];
  for (int l = 0; l < 3; ++l) {
    CFB_CHECK(alloc(&hd[l], ny[l], nx[l], 64));
    CFB_CHECK(conv("model.23.m." + std::to_string(l), P[l], ny[l], nx[l], hd[l], 64, 0, OUT_NONE));
  }
  if (!dry) CFB_CHECK(yolo_decode(hd, raw, ny, nx, n->anchor_grid, pred, N, (int)yo_predictions(H, W), st));
  for (int l = 0; l < 3; ++l) ar.release(hd[l]);
  ar.release(p3); ar.release(p4); ar.release(p5);
  return 0;
}

}  // namespace cfb

// =========================================================================================================
// C ABI
// =========================================================================================================
// =========================================================================================================
// InceptionV3 for FID: pytorch-fid's InceptionV3(output_blocks=[3]) with use_fid_inception=True (basicsr/archs/inception.py),
// the pool3 features of restored faces.  torchvision's Inception3 with the FID blocks: Mixed_5b..5d FIDInceptionA (pool
// features 32 / 64 / 64), Mixed_6b..6e FIDInceptionC (channels_7x7 128 / 160 / 160 / 192), Mixed_7b FIDInceptionE_1, Mixed_7c
// FIDInceptionE_2; the pool branches of A, C and E_1 are avg_pool2d(3, 1, 1, count_include_pad=False), that of E_2
// max_pool2d(3, 1, 1).  Every BasicConv2d is conv (no bias) + BatchNorm(eps 1e-3, folded at prepare) + ReLU.  Engines:
//   Conv2d_1a_3x3 (3x3 s2 valid, 3 -> 32)        SIMT stem (fid.cu), the input stage (bilinear to 299, 2x - 1) fused into its load
//   3x3 pad 1 stride 1                            generalised halo engine
//   1x1, 3x3 valid (stride 1 and 2), 5x5, 1x7, 7x1, 1x3, 3x1     per-tap engine, explicit windows
//   max / avg pools, global average pool         SIMT (fid.cu)
// Maps are NHWC with a 64-aligned channel pitch whose pad channels are zero (zero weights and bias + ReLU, or a memset).  Each
// block's branches write their channel slices of one concatenation buffer, in torchvision's order.
// =========================================================================================================
struct cfb_fid : cfb::NetCore {
  cfb_fid() : NetCore("InceptionV3", "fid") {}
  std::vector<cfb::GenConv> convs;        // the 93 convs after the stem, in plan order
  float *stem_w = nullptr, *stem_b = nullptr;
};
namespace cfb {

constexpr float FID_BN_EPS = 1e-3f;
constexpr int FID_FEATURES = 2048;

// block prefixes of the wrapper's state dict (blocks.<i>.<j>.) for the convs after the stem
static void fid_build(cfb_fid* n) {
  std::vector<GenConv>& v = n->convs;
  v.clear();
  auto add = [&](const std::string& name, int cin, int cout, int kh, int kw, int ph, int pw, int stride) {
    GenConv c = plan_conv(name, cin, cout, kh == kw ? kh : 1, stride);
    c.gen = kh == 3 && kw == 3 && ph == 1 && pw == 1 && stride == 1;
    if (!c.gen) { c.kh = kh; c.kw = kw; c.pad_h = ph; c.pad_w = pw; }
    v.push_back(c);
  };
  add("blocks.0.1.", 32, 32, 3, 3, 0, 0, 1);          // Conv2d_2a_3x3
  add("blocks.0.2.", 32, 64, 3, 3, 1, 1, 1);          // Conv2d_2b_3x3
  add("blocks.1.0.", 64, 80, 1, 1, 0, 0, 1);          // Conv2d_3b_1x1
  add("blocks.1.1.", 80, 192, 3, 3, 0, 0, 1);         // Conv2d_4a_3x3
  const int pf[3] = {32, 64, 64};
  int cin = 192;
  for (int i = 0; i < 3; ++i) {                       // Mixed_5b..5d (InceptionA)
    const std::string p = "blocks.2." + std::to_string(i) + ".";
    add(p + "branch1x1.", cin, 64, 1, 1, 0, 0, 1);
    add(p + "branch5x5_1.", cin, 48, 1, 1, 0, 0, 1);
    add(p + "branch5x5_2.", 48, 64, 5, 5, 2, 2, 1);
    add(p + "branch3x3dbl_1.", cin, 64, 1, 1, 0, 0, 1);
    add(p + "branch3x3dbl_2.", 64, 96, 3, 3, 1, 1, 1);
    add(p + "branch3x3dbl_3.", 96, 96, 3, 3, 1, 1, 1);
    add(p + "branch_pool.", cin, pf[i], 1, 1, 0, 0, 1);
    cin = 224 + pf[i];
  }
  add("blocks.2.3.branch3x3.", 288, 384, 3, 3, 0, 0, 2);           // Mixed_6a (InceptionB)
  add("blocks.2.3.branch3x3dbl_1.", 288, 64, 1, 1, 0, 0, 1);
  add("blocks.2.3.branch3x3dbl_2.", 64, 96, 3, 3, 1, 1, 1);
  add("blocks.2.3.branch3x3dbl_3.", 96, 96, 3, 3, 0, 0, 2);
  const int c7s[4] = {128, 160, 160, 192};
  for (int i = 0; i < 4; ++i) {                       // Mixed_6b..6e (InceptionC)
    const std::string p = "blocks.2." + std::to_string(4 + i) + ".";
    const int c7 = c7s[i];
    add(p + "branch1x1.", 768, 192, 1, 1, 0, 0, 1);
    add(p + "branch7x7_1.", 768, c7, 1, 1, 0, 0, 1);
    add(p + "branch7x7_2.", c7, c7, 1, 7, 0, 3, 1);
    add(p + "branch7x7_3.", c7, 192, 7, 1, 3, 0, 1);
    add(p + "branch7x7dbl_1.", 768, c7, 1, 1, 0, 0, 1);
    add(p + "branch7x7dbl_2.", c7, c7, 7, 1, 3, 0, 1);
    add(p + "branch7x7dbl_3.", c7, c7, 1, 7, 0, 3, 1);
    add(p + "branch7x7dbl_4.", c7, c7, 7, 1, 3, 0, 1);
    add(p + "branch7x7dbl_5.", c7, 192, 1, 7, 0, 3, 1);
    add(p + "branch_pool.", 768, 192, 1, 1, 0, 0, 1);
  }
  add("blocks.3.0.branch3x3_1.", 768, 192, 1, 1, 0, 0, 1);         // Mixed_7a (InceptionD)
  add("blocks.3.0.branch3x3_2.", 192, 320, 3, 3, 0, 0, 2);
  add("blocks.3.0.branch7x7x3_1.", 768, 192, 1, 1, 0, 0, 1);
  add("blocks.3.0.branch7x7x3_2.", 192, 192, 1, 7, 0, 3, 1);
  add("blocks.3.0.branch7x7x3_3.", 192, 192, 7, 1, 3, 0, 1);
  add("blocks.3.0.branch7x7x3_4.", 192, 192, 3, 3, 0, 0, 2);
  cin = 1280;
  for (int i = 0; i < 2; ++i) {                       // Mixed_7b, 7c (InceptionE)
    const std::string p = "blocks.3." + std::to_string(1 + i) + ".";
    add(p + "branch1x1.", cin, 320, 1, 1, 0, 0, 1);
    add(p + "branch3x3_1.", cin, 384, 1, 1, 0, 0, 1);
    add(p + "branch3x3_2a.", 384, 384, 1, 3, 0, 1, 1);
    add(p + "branch3x3_2b.", 384, 384, 3, 1, 1, 0, 1);
    add(p + "branch3x3dbl_1.", cin, 448, 1, 1, 0, 0, 1);
    add(p + "branch3x3dbl_2.", 448, 384, 3, 3, 1, 1, 1);
    add(p + "branch3x3dbl_3a.", 384, 384, 1, 3, 0, 1, 1);
    add(p + "branch3x3dbl_3b.", 384, 384, 3, 1, 1, 0, 1);
    add(p + "branch_pool.", cin, 192, 1, 1, 0, 0, 1);
    cin = 2048;
  }
}

static int fid_prepare(cfb_fid* n, cudaStream_t st) {
  CFB_CHECK(n->begin_prepare(st));
  SlabPlan plan;
  for (const GenConv& c : n->convs) plan.add(c);
  CFB_CHECK(n->reserve_slab(plan.bytes() + align256(32 * 27 * 4) + align256(32 * 4)));
  WeightPrep wp(*n, plan, st);
  for (GenConv& c : n->convs) {
    CFB_CHECK(wp.fold(c.name + "conv.weight", c.name + "bn.", c.cout, c.cin * c.taps(), FID_BN_EPS));
    CFB_CHECK(wp.conv(c, wp.fold_w, wp.fold_b));
  }
  CFB_CHECK(wp.fold("blocks.0.0.conv.weight", "blocks.0.0.bn.", 32, 27, FID_BN_EPS));
  n->stem_w = (float*)wp.take(32 * 27 * 4); n->stem_b = (float*)wp.take(32 * 4);
  CFB_CUDA(cudaMemcpyAsync(n->stem_w, wp.fold_w, 32 * 27 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaMemcpyAsync(n->stem_b, wp.fold_b, 32 * 4, cudaMemcpyDeviceToDevice, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  n->prepared = true;
  return 0;
}

static int pad64(int c) { return (c + 63) / 64 * 64; }

// pool3 features [N, 2048] of N images through the input stage `in`
static int fid_forward(cfb_fid* n, const FidInput& in, int N, float* feat, void* ws, int64_t ws_bytes, cudaStream_t st, bool dry) {
  CFB_CHECK(n->begin_forward(dry));
  const int OH = in.resize ? FID_SIZE : in.H, OW = in.resize ? FID_SIZE : in.W;
  CFB_REQUIRE(N >= 0 && in.H >= 1 && in.W >= 1, "InceptionV3: bad input size");
  CFB_REQUIRE(OH >= 75 && OW >= 75, "InceptionV3: the network input must be at least 75 x 75 (resize_input=True gives 299 x 299)");
  if (N == 0) return 0;
  Arena& ar = n->arena;
  ar.reset(ws, (size_t)ws_bytes, dry);
  struct Map { float* p; int h, w, c, pitch; };       // c real channels, pitch >= c (pad channels zero)
  auto alloc = [&](Map& m, int h, int w, int c, int pitch) -> int {
    m.h = h; m.w = w; m.c = c; m.pitch = pitch;
    CFB_CHECK(n->alloc(&m.p, (size_t)N * h * w * pitch));
    if (!dry && (pitch != c)) CFB_CUDA(cudaMemsetAsync(m.p, 0, (size_t)N * h * w * pitch * 4, st));
    return 0;
  };
  auto out_hw = [](const GenConv& c, int h, int w, int& oh, int& ow) {
    if (c.gen) { oh = h; ow = w; return; }
    oh = (h + 2 * c.pad_h - c.kh) / c.stride + 1; ow = (w + 2 * c.pad_w - c.kw) / c.stride + 1;
  };
  // conv + ReLU of x into channels [c0, c0 + cout) of `o` (o.pitch channels per pixel)
  auto conv = [&](const GenConv& c, const Map& x, const Map& o, int c0) -> int {
    CFB_REQUIRE(x.c == c.cin, "InceptionV3: channel mismatch at " + c.name);
    if (c.gen) {
      GenLaunch g{&c, x.p, x.pitch, x.h, x.w, N, o.p, o.pitch, c0, OUT_RELU};
      return dry ? 0 : gen_conv(g, n->sm_count, st);
    }
    CFB_REQUIRE(x.pitch == c.cin_p, "InceptionV3: per-tap input pitch at " + c.name);
    return pertap_conv(*n, pertap_window_args(x.p, N, x.h, x.w, c, o.p, o.pitch, c0, OUT_RELU), c, dry, st);
  };
  // conv into a new map of its own (pitch cout_p; the generalised engine stores only the real channels, so the pad is zeroed)
  auto conv_new = [&](const GenConv& c, const Map& x, Map& o) -> int {
    int oh = 0, ow = 0;
    out_hw(c, x.h, x.w, oh, ow);
    CFB_CHECK(alloc(o, oh, ow, c.cout, c.cout_p));
    return conv(c, x, o, 0);
  };
  auto pool_conv = [&](const GenConv& c, const Map& x, bool max_pool, const Map& o, int c0) -> int {
    Map pm;
    CFB_CHECK(alloc(pm, x.h, x.w, x.c, x.pitch));
    if (!dry) {
      if (max_pool) CFB_CHECK(fid_maxpool(x.p, x.pitch, pm.p, x.pitch, 0, N, x.h, x.w, x.pitch, 1, st));
      else CFB_CHECK(fid_avgpool(x.p, x.pitch, pm.p, x.pitch, N, x.h, x.w, x.pitch, st));
    }
    CFB_CHECK(conv(c, pm, o, c0));
    ar.release(pm.p);
    return 0;
  };
  // a chain of convs from x, the last one into channels [c0, ..) of o
  auto chain = [&](std::initializer_list<const GenConv*> cs, const Map& x, const Map& o, int c0) -> int {
    Map cur = x;
    size_t i = 0;
    for (const GenConv* c : cs) {
      if (++i == cs.size()) { CFB_CHECK(conv(*c, cur, o, c0)); break; }
      Map nx;
      CFB_CHECK(conv_new(*c, cur, nx));
      if (cur.p != x.p) ar.release(cur.p);
      cur = nx;
    }
    if (cur.p != x.p) ar.release(cur.p);
    return 0;
  };
  const std::vector<GenConv>& C = n->convs;
  // stem: Conv2d_1a (SIMT, input stage fused), 2a, 2b, max pool, 3b, 4a, max pool
  Map x, y;
  // per-image NaN flags of the stem, read by the global pool (the engine's ReLU epilogue maps NaN to 0, torch's keeps it)
  int* nan_flag = (int*)ar.alloc((size_t)N * sizeof(int));
  CFB_REQUIRE(nan_flag != nullptr, n->ws_error());
  if (!dry) CFB_CUDA(cudaMemsetAsync(nan_flag, 0, (size_t)N * sizeof(int), st));
  CFB_CHECK(alloc(x, (OH - 3) / 2 + 1, (OW - 3) / 2 + 1, 32, 64));
  if (!dry) CFB_CHECK(fid_stem(in, n->stem_w, n->stem_b, x.p, nan_flag, 64, N, st));
  CFB_CHECK(conv_new(C[0], x, y)); ar.release(x.p); x = y;
  CFB_CHECK(conv_new(C[1], x, y)); ar.release(x.p); x = y;
  CFB_CHECK(alloc(y, (x.h - 3) / 2 + 1, (x.w - 3) / 2 + 1, x.c, x.pitch));
  if (!dry) CFB_CHECK(fid_maxpool(x.p, x.pitch, y.p, y.pitch, 0, N, x.h, x.w, x.pitch, 2, st));
  ar.release(x.p); x = y;
  CFB_CHECK(conv_new(C[2], x, y)); ar.release(x.p); x = y;
  CFB_CHECK(conv_new(C[3], x, y)); ar.release(x.p); x = y;
  CFB_CHECK(alloc(y, (x.h - 3) / 2 + 1, (x.w - 3) / 2 + 1, x.c, x.pitch));
  if (!dry) CFB_CHECK(fid_maxpool(x.p, x.pitch, y.p, y.pitch, 0, N, x.h, x.w, x.pitch, 2, st));
  ar.release(x.p); x = y;
  size_t k = 4;
  for (int i = 0; i < 3; ++i, k += 7) {               // Mixed_5b..5d: [1x1 64 | 5x5 64 | 3x3dbl 96 | pool pf]
    const int c = 224 + C[k + 6].cout;
    CFB_CHECK(alloc(y, x.h, x.w, c, pad64(c)));
    CFB_CHECK(conv(C[k], x, y, 0));
    CFB_CHECK(chain({&C[k + 1], &C[k + 2]}, x, y, 64));
    CFB_CHECK(chain({&C[k + 3], &C[k + 4], &C[k + 5]}, x, y, 128));
    CFB_CHECK(pool_conv(C[k + 6], x, false, y, 224));
    ar.release(x.p); x = y;
  }
  {                                                   // Mixed_6a: [3x3 s2 384 | 3x3dbl s2 96 | max pool 288]
    const int h = (x.h - 3) / 2 + 1, w = (x.w - 3) / 2 + 1;
    CFB_CHECK(alloc(y, h, w, 768, 768));
    CFB_CHECK(conv(C[k], x, y, 0));
    CFB_CHECK(chain({&C[k + 1], &C[k + 2], &C[k + 3]}, x, y, 384));
    if (!dry) CFB_CHECK(fid_maxpool(x.p, x.pitch, y.p, y.pitch, 480, N, x.h, x.w, x.c, 2, st));
    ar.release(x.p); x = y; k += 4;
  }
  for (int i = 0; i < 4; ++i, k += 10) {              // Mixed_6b..6e: [1x1 192 | 7x7 192 | 7x7dbl 192 | pool 192]
    CFB_CHECK(alloc(y, x.h, x.w, 768, 768));
    CFB_CHECK(conv(C[k], x, y, 0));
    CFB_CHECK(chain({&C[k + 1], &C[k + 2], &C[k + 3]}, x, y, 192));
    CFB_CHECK(chain({&C[k + 4], &C[k + 5], &C[k + 6], &C[k + 7], &C[k + 8]}, x, y, 384));
    CFB_CHECK(pool_conv(C[k + 9], x, false, y, 576));
    ar.release(x.p); x = y;
  }
  {                                                   // Mixed_7a: [3x3 s2 320 | 7x7x3 s2 192 | max pool 768]
    const int h = (x.h - 3) / 2 + 1, w = (x.w - 3) / 2 + 1;
    CFB_CHECK(alloc(y, h, w, 1280, 1280));
    CFB_CHECK(chain({&C[k], &C[k + 1]}, x, y, 0));
    CFB_CHECK(chain({&C[k + 2], &C[k + 3], &C[k + 4], &C[k + 5]}, x, y, 320));
    if (!dry) CFB_CHECK(fid_maxpool(x.p, x.pitch, y.p, y.pitch, 512, N, x.h, x.w, x.c, 2, st));
    ar.release(x.p); x = y; k += 6;
  }
  for (int i = 0; i < 2; ++i, k += 9) {               // Mixed_7b, 7c: [1x1 320 | 3x3 2a 2b 768 | 3x3dbl 3a 3b 768 | pool 192]
    CFB_CHECK(alloc(y, x.h, x.w, 2048, 2048));
    CFB_CHECK(conv(C[k], x, y, 0));
    Map t, u;
    CFB_CHECK(conv_new(C[k + 1], x, t));
    CFB_CHECK(conv(C[k + 2], t, y, 320));
    CFB_CHECK(conv(C[k + 3], t, y, 704));
    ar.release(t.p);
    CFB_CHECK(conv_new(C[k + 4], x, t));
    CFB_CHECK(conv_new(C[k + 5], t, u));
    ar.release(t.p);
    CFB_CHECK(conv(C[k + 6], u, y, 1088));
    CFB_CHECK(conv(C[k + 7], u, y, 1472));
    ar.release(u.p);
    CFB_CHECK(pool_conv(C[k + 8], x, i == 1, y, 1856));     // FIDInceptionE_2 pools with max_pool2d(3, 1, 1)
    ar.release(x.p); x = y;
  }
  if (!dry) CFB_CHECK(fid_global_pool(x.p, x.pitch, nan_flag, feat, N, x.h, x.w, FID_FEATURES, st));
  ar.release(x.p);
  ar.release(nan_flag);
  return 0;
}

}  // namespace cfb

#define API_BEGIN try {
#define API_END(ret)                                                             \
  } catch (const std::exception& e) { cfb::set_error(std::string("exception: ") + e.what()); return ret; } \
  catch (...) { cfb::set_error("unknown exception"); return ret; }

extern "C" {

int cfb_version(void) { return CFB_VERSION; }
const char* cfb_last_error(void) { return cfb::last_error().c_str(); }

int cfb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  API_BEGIN
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  CFB_CUDA(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  return 0;
  API_END(1)
}

cfb_net* cfb_net_create(const cfb_config* cfg) {
  API_BEGIN
  if (!cfg) { cfb::set_error("cfb_net_create: NULL config"); return nullptr; }
  cfb_net* n = new cfb_net();
  n->cfg = *cfg;
  n->convs.reserve(512);
  if (cfb::build_plan(n) != 0) { delete n; return nullptr; }
  int dev = 0, major = 0, sms = 148;
  if (cudaGetDevice(&dev) == cudaSuccess) {
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  } else {
    cudaGetLastError();
  }
  n->sm_count = sms > 0 ? sms : 148;
  n->tc_ok = (major == 9);
  n->device = dev;
  return n;
  API_END(nullptr)
}

void cfb_net_destroy(cfb_net* n) { delete n; }     // ~NetCore frees the slab on its device

cfb_rrdb* cfb_rrdb_create(int32_t num_in_ch, int32_t num_out_ch, int32_t scale, int32_t num_feat, int32_t num_block, int32_t num_grow_ch) {
  API_BEGIN
  if (num_feat != 64 || num_grow_ch != 32 || num_in_ch < 1 || num_in_ch > 3 || num_out_ch < 1 || num_out_ch > 4 || num_block < 1 ||
      !(scale == 1 || scale == 2 || scale == 4)) {
    cfb::set_error("cfb_rrdb_create: built for num_feat=64, num_grow_ch=32, <=3 image channels, scale 1/2/4");
    return nullptr;
  }
  cfb_rrdb* n = new cfb_rrdb();
  n->in_ch = num_in_ch; n->out_ch = num_out_ch; n->scale = scale; n->feat = num_feat; n->blocks = num_block; n->grow = num_grow_ch;
  return n;
  API_END(nullptr)
}
void cfb_rrdb_destroy(cfb_rrdb* n) { delete n; }
int cfb_rrdb_set_param(cfb_rrdb* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_rrdb_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_rrdb_prepare(cfb_rrdb* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_rrdb_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rrdb_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int cfb_rrdb_set_precision(cfb_rrdb* n, int32_t precision) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_rrdb_set_precision: NULL net");
  return n->set_precision(precision);
  API_END(1)
}
int64_t cfb_rrdb_workspace_bytes(cfb_rrdb* n, int32_t batch, int32_t h, int32_t w) {
  if (!n || batch < 0 || h < 0 || w < 0) return -1;
  return (int64_t)cfb::rrdb_ws_bytes(n, batch, h, w);
}
int cfb_rrdb_forward(cfb_rrdb* n, const float* x, float* out, int32_t batch, int32_t h, int32_t w, void* workspace,
                     int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x && out && workspace)), "cfb_rrdb_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rrdb_forward(n, x, out, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}
int cfb_rrdb_forward_u8_tiles(cfb_rrdb* n, const uint8_t* images_bgr, int32_t num_images, int32_t img_h, int32_t img_w,
                              int32_t pre_pad, const int32_t* tiles, int32_t num_tiles, int32_t tile_h, int32_t tile_w,
                              uint8_t* out_bgr, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (num_tiles <= 0 || (images_bgr && tiles && out_bgr && workspace)), "cfb_rrdb_forward_u8_tiles: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rrdb_tiles("cfb_rrdb_forward_u8_tiles", n, images_bgr, cfb::IMG_U8, num_images, img_h, img_w, pre_pad, tiles,
                         num_tiles, tile_h, tile_w, out_bgr, cfb::IMG_U8, nullptr, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}
int cfb_rrdb_forward_tiles(cfb_rrdb* n, const void* images_bgr, int32_t in_kind, int32_t num_images, int32_t img_h, int32_t img_w,
                           int32_t pre_pad, const int32_t* tiles, int32_t num_tiles, int32_t tile_h, int32_t tile_w, void* out_bgr,
                           int32_t out_kind, int32_t* max_range, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (num_tiles <= 0 || (images_bgr && tiles && out_bgr && max_range && workspace)),
              "cfb_rrdb_forward_tiles: NULL argument");
  CFB_REQUIRE(in_kind >= CFB_IMG_U8 && in_kind <= CFB_IMG_F64, "cfb_rrdb_forward_tiles: in_kind must be a CFB_IMG_* value");
  CFB_REQUIRE(out_kind == CFB_IMG_U8 || out_kind == CFB_IMG_U16, "cfb_rrdb_forward_tiles: out_kind must be CFB_IMG_U8 or CFB_IMG_U16");
  CFB_REQUIRE(num_images <= 65535, "cfb_rrdb_forward_tiles: at most 65535 images per call");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rrdb_tiles("cfb_rrdb_forward_tiles", n, images_bgr, in_kind, num_images, img_h, img_w, pre_pad, tiles, num_tiles,
                         tile_h, tile_w, out_bgr, out_kind, max_range, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}

cfb_parsenet* cfb_parsenet_create(int32_t in_size, int32_t out_size, int32_t min_feat_size, int32_t base_ch, int32_t parsing_ch,
                                  int32_t res_depth, int32_t ch_min, int32_t ch_max) {
  API_BEGIN
  cfb_parsenet* n = new cfb_parsenet();
  n->in_size = in_size; n->out_size = out_size; n->min_feat = min_feat_size; n->base_ch = base_ch; n->parsing_ch = parsing_ch;
  n->res_depth = res_depth; n->ch_min = ch_min; n->ch_max = ch_max;
  if (in_size < 1 || out_size < 1 || min_feat_size < 1 || cfb::pn_build(n) != 0) { delete n; return nullptr; }
  return n;
  API_END(nullptr)
}
void cfb_parsenet_destroy(cfb_parsenet* n) { delete n; }
int cfb_parsenet_set_param(cfb_parsenet* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_parsenet_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_parsenet_prepare(cfb_parsenet* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_parsenet_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::pn_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_parsenet_workspace_bytes(cfb_parsenet* n, int32_t batch, int32_t h, int32_t w) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_parsenet_workspace_bytes: NULL net"); return -1; }
  return n->dry_run([&] {
    return cfb::pn_forward(n, (const float*)0x1000, (float*)0x1000, (float*)0x1000, batch, h, w, nullptr, 0, nullptr, true);
  });
  API_END(-1)
}
int cfb_parsenet_forward(cfb_parsenet* n, const float* x, float* out_mask, float* out_img, int32_t batch, int32_t h, int32_t w,
                         void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x && out_mask && workspace)), "cfb_parsenet_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::pn_forward(n, x, out_mask, out_img, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_parsenet_set_precision(cfb_parsenet* n, int32_t precision) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_parsenet_set_precision: NULL net");
  return n->set_precision(precision);
  API_END(1)
}
int cfb_parsenet_masks_u8(cfb_parsenet* n, const uint8_t* faces_bgr, uint8_t* classes, uint8_t* mask, int32_t batch, int32_t h,
                          int32_t w, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (classes || mask) && (batch == 0 || (faces_bgr && workspace)), "cfb_parsenet_masks_u8: NULL argument");
  CFB_REQUIRE(batch >= 0 && h > 0 && w > 0, "cfb_parsenet_masks_u8: bad face batch");
  std::lock_guard<std::mutex> lk(n->mu);
  const cfb::PnU8Io io{faces_bgr, classes, mask};
  return cfb::pn_forward(n, nullptr, nullptr, nullptr, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream, false, &io);
  API_END(1)
}
int cfb_parse_argmax(const float* logits_nchw, uint8_t* classes, uint8_t* mask, int32_t batch, int32_t channels, int64_t hw, void* stream) {
  API_BEGIN
  CFB_REQUIRE(logits_nchw && (classes || mask), "cfb_parse_argmax: NULL argument");
  return cfb::parse_argmax(logits_nchw, classes, mask, batch, channels, hw, (cudaStream_t)stream);
  API_END(1)
}

int64_t cfb_conv2d_gen_workspace_bytes(int32_t cin, int32_t cout) {
  const size_t cin_p = (size_t)(cin + 63) / 64 * 64, cout_p = (size_t)(cout + 63) / 64 * 64;
  return (int64_t)(align256(cout_p * cin_p * 9 * 4) + 2 * align256(cout_p * cin_p * 16 * 2) + align256(cout_p * 4) + 256 + 4096);
}

int cfb_conv2d_gen_nhwc(const float* in, int32_t in_pitch, const float* weight_oihw, const float* bias, float* out,
                        int32_t out_pitch, int32_t out_c0, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout,
                        int32_t upsample, int32_t pad_mode, int32_t subsample, int32_t out_act, const float* residual,
                        int32_t res_pitch, const float* residual2, int32_t res2_pitch, float post_scale, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  return cfb_conv2d_gen_nhwc_prec(in, in_pitch, weight_oihw, bias, out, out_pitch, out_c0, n, h, w, cin, cout, upsample, pad_mode,
                                  subsample, out_act, residual, res_pitch, residual2, res2_pitch, post_scale, workspace,
                                  workspace_bytes, stream, 0);
}

int cfb_conv2d_gen_nhwc_prec(const float* in, int32_t in_pitch, const float* weight_oihw, const float* bias, float* out,
                             int32_t out_pitch, int32_t out_c0, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout,
                             int32_t upsample, int32_t pad_mode, int32_t subsample, int32_t out_act, const float* residual,
                             int32_t res_pitch, const float* residual2, int32_t res2_pitch, float post_scale, void* workspace,
                             int64_t workspace_bytes, void* stream, int32_t precision) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace, "cfb_conv2d_gen_nhwc: NULL argument");
  CFB_REQUIRE(precision == 0 || precision == 1, "cfb_conv2d_gen_nhwc_prec: precision must be 0 (fp32, split) or 1 (fp16)");
  CFB_REQUIRE(workspace_bytes >= cfb_conv2d_gen_workspace_bytes(cin, cout), "cfb_conv2d_gen_nhwc: workspace too small");
  CFB_REQUIRE(cin >= 1 && cout >= 1 && cout % 4 == 0, "cfb_conv2d_gen_nhwc: cout must be a multiple of 4");
  cudaStream_t st = (cudaStream_t)stream;
  CFB_CHECK(cfb::async_status_init(st));
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cfb::GenConv c = cfb::plan_conv("", cin, cout);
  c.up = upsample != 0;
  char* p = (char*)(((uintptr_t)workspace + 255) / 256 * 256);
  float* pad = (float*)p; p += align256((size_t)c.cout_p * c.cin_p * 9 * 4);
  CFB_CHECK(cfb::prepare_conv(c, weight_oihw, bias, pad, p, st));
  cfb::GenLaunch g{&c, in, in_pitch, h, w, n, out, out_pitch, out_c0, out_act};
  g.res = residual; g.res_pitch = res_pitch; g.res2 = residual2; g.res2_pitch = res2_pitch; g.post = post_scale;
  g.pad_mode = pad_mode; g.sub = subsample != 0; g.single_pass = precision == 1;
  return cfb::gen_conv(g, sms, st);
  API_END(1)
}

// body of the two per-tap test entry points (after their own argument checks): split the weight into the workspace, run
static int pertap_nhwc(const char* fn, cfb::ConvArgs a, const float* weight_oihw, const float* bias, int32_t stride, void* workspace,
                       int64_t workspace_bytes, cudaStream_t st) {
  CFB_CHECK(cfb::async_status_init(st));
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CFB_REQUIRE(cfb::tc_supported(a), std::string(fn) + ": shape not supported by the wgmma engine");
  CFB_REQUIRE(workspace_bytes >= cfb_conv2d_pertap_workspace_bytes(a.N, a.H, a.W, a.Cin, a.Cout, a.ksize, stride),
              std::string(fn) + ": workspace too small");
  const size_t wn = (size_t)a.Cout * a.Cin * a.ksize * a.ksize;
  char* p = (char*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  __half* whi = (__half*)p; p += align256(wn * 2);
  __half* wlo = (__half*)p; p += align256(wn * 2);
  float* wsc = (float*)p; p += 256;
  p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
  CFB_CHECK(cfb::tc_split_weights(weight_oihw, whi, wlo, a.Cout, a.Cin, a.ksize, wsc, st));
  a.wgt_hi = whi; a.wgt_lo = wlo; a.wscale_inv = wsc + 1; a.bias = bias;
  return cfb::conv_tc(a, p, sms, st);
}

int cfb_conv2d_pertap_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h, int32_t w,
                           int32_t cin, int32_t cout, int32_t ksize, int32_t stride, int32_t out_act, const float* residual,
                           void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace, "cfb_conv2d_pertap_nhwc: NULL argument");
  CFB_REQUIRE(stride == 1 || stride == 2, "cfb_conv2d_pertap_nhwc: stride must be 1 or 2");
  CFB_REQUIRE(out_act == cfb::OUT_NONE || out_act == cfb::OUT_RELU, "cfb_conv2d_pertap_nhwc: activation must be none or ReLU");
  return pertap_nhwc("cfb_conv2d_pertap_nhwc", cfb::pertap_args(in, n, h, w, cin, cout, ksize, stride, out, 0, 0, out_act, residual),
                     weight_oihw, bias, stride, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}

int cfb_conv2d_pertap_slice_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                                 int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t stride, int32_t out_act,
                                 int32_t out_pitch, int32_t out_c0, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace, "cfb_conv2d_pertap_slice_nhwc: NULL argument");
  CFB_REQUIRE(stride == 1 || stride == 2, "cfb_conv2d_pertap_slice_nhwc: stride must be 1 or 2");
  CFB_REQUIRE(ksize == 1 || stride == 2, "cfb_conv2d_pertap_slice_nhwc: 3x3 convs run stride 2 on the per-tap engine");
  CFB_REQUIRE(out_act == cfb::OUT_NONE || out_act == cfb::OUT_SILU, "cfb_conv2d_pertap_slice_nhwc: activation must be none or SiLU");
  return pertap_nhwc("cfb_conv2d_pertap_slice_nhwc",
                     cfb::pertap_args(in, n, h, w, cin, cout, ksize, stride, out, out_pitch, out_c0, out_act, nullptr), weight_oihw,
                     bias, stride, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}

int64_t cfb_conv2d_pertap_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t stride) {
  if (n < 0 || h < 1 || w < 1 || cin < 1 || cout < 1 || !(ksize == 1 || ksize == 3) || !(stride == 1 || stride == 2)) return -1;
  const cfb::ConvArgs a = cfb::pertap_args(nullptr, n, h, w, cin, cout, ksize, stride, nullptr, 0, 0, cfb::OUT_NONE, nullptr);
  const size_t wn = (size_t)cout * cin * ksize * ksize;
  return (int64_t)(2 * align256(wn * 2) + 256 + cfb::tc_scratch_bytes(a) + 4096);
}

int64_t cfb_retinaface_priors(int32_t h, int32_t w) { return h < 1 || w < 1 ? -1 : cfb::rf_priors(h, w); }

cfb_retinaface* cfb_retinaface_create(void) {
  API_BEGIN
  cfb_retinaface* n = new cfb_retinaface();
  cfb::rf_build(n);
  return n;
  API_END(nullptr)
}
void cfb_retinaface_destroy(cfb_retinaface* n) { delete n; }
int cfb_retinaface_set_param(cfb_retinaface* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_retinaface_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_retinaface_prepare(cfb_retinaface* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_retinaface_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rf_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_retinaface_workspace_bytes(cfb_retinaface* n, int32_t batch, int32_t h, int32_t w) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_retinaface_workspace_bytes: NULL net"); return -1; }
  return n->dry_run([&] {
    return cfb::rf_forward(n, (const float*)0x1000, nullptr, nullptr, nullptr, nullptr, batch, h, w, nullptr, 0, nullptr, true);
  });
  API_END(-1)
}
int cfb_retinaface_forward(cfb_retinaface* n, const float* x_nchw, float* loc, float* conf, float* landms, int32_t batch, int32_t h,
                           int32_t w, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x_nchw && loc && conf && landms && workspace)), "cfb_retinaface_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rf_forward(n, x_nchw, nullptr, loc, conf, landms, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_retinaface_forward_u8(cfb_retinaface* n, const uint8_t* img_bgr_hwc, float* loc, float* conf, float* landms, int32_t batch,
                              int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (img_bgr_hwc && loc && conf && landms && workspace)), "cfb_retinaface_forward_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::rf_forward(n, nullptr, img_bgr_hwc, loc, conf, landms, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream,
                         false);
  API_END(1)
}
int cfb_retinaface_candidates(const float* loc, const float* conf, const float* landms, int32_t batch, int32_t h, int32_t w,
                              float conf_threshold, float* rows, int32_t* counts, void* stream) {
  API_BEGIN
  CFB_REQUIRE(batch == 0 || (loc && conf && landms && rows && counts), "cfb_retinaface_candidates: NULL argument");
  CFB_REQUIRE(h >= 1 && w >= 1 && batch >= 0, "cfb_retinaface_candidates: empty image");
  return cfb::rf_candidates(loc, conf, landms, batch, h, w, conf_threshold, rows, counts, (cudaStream_t)stream);
  API_END(1)
}

cfb_bisenet* cfb_bisenet_create(int32_t num_class) {
  API_BEGIN
  if (num_class < 1 || num_class > 64) { cfb::set_error("cfb_bisenet_create: built for 1..64 classes"); return nullptr; }
  cfb_bisenet* n = new cfb_bisenet();
  n->num_class = num_class;
  cfb::bs_build(n);
  return n;
  API_END(nullptr)
}
void cfb_bisenet_destroy(cfb_bisenet* n) { delete n; }
int cfb_bisenet_set_param(cfb_bisenet* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_bisenet_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_bisenet_prepare(cfb_bisenet* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_bisenet_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::bs_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_bisenet_workspace_bytes(cfb_bisenet* n, int32_t batch, int32_t h, int32_t w) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_bisenet_workspace_bytes: NULL net"); return -1; }
  float* const outs[3] = {(float*)0x1000, (float*)0x1000, (float*)0x1000};
  return n->dry_run([&] { return cfb::bs_forward(n, (const float*)0x1000, outs, batch, h, w, nullptr, 0, nullptr, true); });
  API_END(-1)
}
int cfb_bisenet_forward(cfb_bisenet* n, const float* x_nchw, float* out, float* out16, float* out32, int32_t batch, int32_t h, int32_t w,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x_nchw && out && out16 && out32 && workspace)), "cfb_bisenet_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  float* const outs[3] = {out, out16, out32};
  return cfb::bs_forward(n, x_nchw, outs, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_bisenet_masks_u8(cfb_bisenet* n, const uint8_t* faces_bgr, uint8_t* classes, uint8_t* mask, int32_t batch, int32_t h, int32_t w,
                         void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (classes || mask) && (batch == 0 || (faces_bgr && workspace)), "cfb_bisenet_masks_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  float* const outs[3] = {nullptr, nullptr, nullptr};
  const cfb::BsU8Io io{faces_bgr, classes, mask};
  return cfb::bs_forward(n, nullptr, outs, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream, false, &io);
  API_END(1)
}
int cfb_debug_bisenet_bilinear(const float* in_nhwc, int32_t pitch, int32_t n, int32_t h, int32_t w, int32_t c, float* out_nchw,
                               int32_t out_h, int32_t out_w, void* stream) {
  API_BEGIN
  CFB_REQUIRE(in_nhwc && out_nchw, "cfb_debug_bisenet_bilinear: NULL argument");
  CFB_REQUIRE(n >= 0 && h >= 1 && w >= 1 && c >= 1 && c <= pitch && out_h >= 1 && out_w >= 1, "cfb_debug_bisenet_bilinear: bad shape");
  return cfb::bise_bilinear(in_nhwc, pitch, h, w, c, out_nchw, n, out_h, out_w, (cudaStream_t)stream);
  API_END(1)
}
int cfb_debug_bisenet_attention(const float* feat_nhwc, int32_t n, int32_t hw, int32_t c, const float* w1, const float* b1, int32_t c1,
                                int32_t act1, const float* w2, const float* b2, int32_t c2, int32_t act2, float* mean, float* att,
                                void* stream) {
  API_BEGIN
  CFB_REQUIRE(feat_nhwc && w1 && mean && att, "cfb_debug_bisenet_attention: NULL argument");
  CFB_REQUIRE(n >= 0 && hw >= 1 && c >= 1 && c1 >= 1 && (!w2 || c2 >= 1), "cfb_debug_bisenet_attention: bad shape");
  const cudaStream_t st = (cudaStream_t)stream;
  CFB_CHECK(cfb::bise_mean(feat_nhwc, mean, n, hw, c, st));
  return cfb::bise_attention(cfb::BiseAttention{w1, b1, c, c1, act1, w2, b2, c2, act2}, mean, att, n, st);
  API_END(1)
}

cfb_arcface* cfb_arcface_create(int32_t l1, int32_t l2, int32_t l3, int32_t l4) {
  API_BEGIN
  cfb_arcface* n = new cfb_arcface();
  const int32_t l[4] = {l1, l2, l3, l4};
  std::copy(l, l + 4, n->layers);
  if (cfb::arc_build(n) != 0) { delete n; return nullptr; }
  return n;
  API_END(nullptr)
}
void cfb_arcface_destroy(cfb_arcface* n) { delete n; }
int cfb_arcface_set_param(cfb_arcface* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_arcface_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_arcface_prepare(cfb_arcface* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_arcface_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::arc_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_arcface_workspace_bytes(cfb_arcface* n, int32_t batch) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_arcface_workspace_bytes: NULL net"); return -1; }
  return n->dry_run([&] { return cfb::arc_forward(n, (const float*)0x1000, nullptr, nullptr, batch, nullptr, 0, nullptr, true); });
  API_END(-1)
}
int cfb_arcface_forward(cfb_arcface* n, const float* x, float* emb, int32_t batch, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x && emb && workspace)), "cfb_arcface_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::arc_forward(n, x, nullptr, emb, batch, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_arcface_forward_u8(cfb_arcface* n, const uint8_t* faces_bgr_hwc, float* emb, int32_t batch, void* workspace,
                           int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (faces_bgr_hwc && emb && workspace)), "cfb_arcface_forward_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::arc_forward(n, nullptr, faces_bgr_hwc, emb, batch, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_debug_arcface_conv(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h, int32_t w,
                           int32_t cin, int32_t cout, int32_t ksize, int32_t stride, const float* in_scale, const float* in_shift,
                           int32_t out_act, float prelu_slope, const float* residual, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace, "cfb_debug_arcface_conv: NULL argument");
  CFB_REQUIRE(out_act == cfb::OUT_NONE || out_act == cfb::OUT_PRELU, "cfb_debug_arcface_conv: activation must be none or PReLU");
  CFB_REQUIRE((in_scale != nullptr) == (in_shift != nullptr), "cfb_debug_arcface_conv: scale and shift go together");
  cudaStream_t st = (cudaStream_t)stream;
  if (ksize == 3 && stride == 1) {
    CFB_REQUIRE(workspace_bytes >= cfb_conv2d_gen_workspace_bytes(cin, cout), "cfb_debug_arcface_conv: workspace too small");
    CFB_REQUIRE(cin % 64 == 0 && cout % 64 == 0, "cfb_debug_arcface_conv: channel counts must be multiples of 64");
    CFB_CHECK(cfb::async_status_init(st));
    int dev = 0, sms = 148;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cfb::GenConv c = cfb::plan_conv("", cin, cout);
    char* p = (char*)(((uintptr_t)workspace + 255) / 256 * 256);
    float* pad = (float*)p; p += align256((size_t)c.cout_p * c.cin_p * 9 * 4);
    CFB_CHECK(cfb::prepare_conv(c, weight_oihw, bias, pad, p, st));
    cfb::GenLaunch g{&c, in, cin, h, w, n, out, cout, 0, out_act};
    g.res = residual; g.res_pitch = cout; g.in_scale = in_scale; g.in_shift = in_shift; g.prelu = prelu_slope;
    return cfb::gen_conv(g, sms, st);
  }
  CFB_REQUIRE(in_scale == nullptr, "cfb_debug_arcface_conv: the input affine is built for 3x3 stride-1 convs");
  CFB_REQUIRE(stride == 1 || stride == 2, "cfb_debug_arcface_conv: stride must be 1 or 2");
  cfb::ConvArgs a = cfb::pertap_args(in, n, h, w, cin, cout, ksize, stride, out, 0, 0, out_act, residual);
  a.prelu_slope = prelu_slope;
  return pertap_nhwc("cfb_debug_arcface_conv", a, weight_oihw, bias, stride, workspace, workspace_bytes, st);
  API_END(1)
}

int64_t cfb_yolov5face_predictions(int32_t h, int32_t w) {
  return h < 32 || w < 32 || h % 32 || w % 32 ? -1 : cfb::yo_predictions(h, w);
}

cfb_yolov5face* cfb_yolov5face_create(void) {
  API_BEGIN
  cfb_yolov5face* n = new cfb_yolov5face();
  cfb::yo_build(n);
  return n;
  API_END(nullptr)
}
void cfb_yolov5face_destroy(cfb_yolov5face* n) { delete n; }
int cfb_yolov5face_set_param(cfb_yolov5face* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_yolov5face_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_yolov5face_prepare(cfb_yolov5face* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_yolov5face_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::yo_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_yolov5face_workspace_bytes(cfb_yolov5face* n, int32_t batch, int32_t h, int32_t w) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_yolov5face_workspace_bytes: NULL net"); return -1; }
  float* const raw[3] = {nullptr, nullptr, nullptr};
  return n->dry_run([&] {
    return cfb::yo_forward(n, (const float*)0x1000, nullptr, 0, 0, 0, 0, nullptr, raw, batch, h, w, nullptr, 0, nullptr, true);
  });
  API_END(-1)
}
int cfb_yolov5face_forward(cfb_yolov5face* n, const float* x_nchw, float* pred, float* raw0, float* raw1, float* raw2, int32_t batch,
                           int32_t h, int32_t w, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x_nchw && pred && workspace)), "cfb_yolov5face_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  float* const raw[3] = {raw0, raw1, raw2};
  return cfb::yo_forward(n, x_nchw, nullptr, 0, 0, 0, 0, pred, raw, batch, h, w, workspace, workspace_bytes, (cudaStream_t)stream,
                         false);
  API_END(1)
}
int cfb_yolov5face_forward_u8(cfb_yolov5face* n, const uint8_t* img_bgr_hwc, int32_t img_h, int32_t img_w, int32_t top, int32_t left,
                              float* pred, float* raw0, float* raw1, float* raw2, int32_t batch, int32_t h, int32_t w,
                              void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (img_bgr_hwc && pred && workspace)), "cfb_yolov5face_forward_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  float* const raw[3] = {raw0, raw1, raw2};
  return cfb::yo_forward(n, nullptr, img_bgr_hwc, img_h, img_w, top, left, pred, raw, batch, h, w, workspace, workspace_bytes,
                         (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_yolov5face_candidates(const float* pred, int32_t batch, int32_t h, int32_t w, float conf_threshold, float* rows,
                              int32_t* counts, void* stream) {
  API_BEGIN
  CFB_REQUIRE(batch == 0 || (pred && rows && counts), "cfb_yolov5face_candidates: NULL argument");
  const int64_t P = cfb_yolov5face_predictions(h, w);
  CFB_REQUIRE(P > 0 && batch >= 0 && P * batch < ((int64_t)1 << 31) / 16, "cfb_yolov5face_candidates: bad size");
  return cfb::yolo_candidates(pred, batch, (int)P, conf_threshold, rows, counts, (cudaStream_t)stream);
  API_END(1)
}

cfb_lpips* cfb_lpips_create(void) {
  API_BEGIN
  return new cfb_lpips();
  API_END(nullptr)
}
void cfb_lpips_destroy(cfb_lpips* n) { delete n; }
int cfb_lpips_set_param(cfb_lpips* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_lpips_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_lpips_prepare(cfb_lpips* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_lpips_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::lp_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_lpips_workspace_bytes(cfb_lpips* n, int32_t batch, int32_t h, int32_t w, int32_t group) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_lpips_workspace_bytes: NULL net"); return -1; }
  cfb::LpIn in;
  in.ref = in.cand = (const float*)0x1000;
  return n->dry_run([&] { return cfb::lp_forward(n, in, batch, group, h, w, nullptr, nullptr, nullptr, 0, nullptr, true); });
  API_END(-1)
}
int cfb_lpips_forward(cfb_lpips* n, const float* ref_nchw, const float* cand_nchw, int32_t batch, int32_t h, int32_t w, int32_t group,
                      int32_t xform, float* val, float* per_layer, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (ref_nchw && cand_nchw && val && workspace)), "cfb_lpips_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  cfb::LpIn in;
  in.ref = ref_nchw; in.cand = cand_nchw; in.flags = xform;
  return cfb::lp_forward(n, in, batch, group, h, w, val, per_layer, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_lpips_forward_u8(cfb_lpips* n, const uint8_t* ref_bgr, const uint8_t* cand_bgr, int32_t batch, int32_t h, int32_t w,
                         int32_t group, int32_t convention, float* val, float* per_layer, void* workspace, int64_t workspace_bytes,
                         void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (ref_bgr && cand_bgr && val && workspace)), "cfb_lpips_forward_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  cfb::LpIn in;
  in.ref8 = ref_bgr; in.cand8 = cand_bgr; in.convention = convention;
  return cfb::lp_forward(n, in, batch, group, h, w, val, per_layer, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_lpips_u8_table(int32_t convention, const float* shift, const float* scale, float* table) {
  API_BEGIN
  CFB_REQUIRE(shift && scale && table, "cfb_lpips_u8_table: NULL argument");
  return cfb::lp_u8_table(convention, shift, scale, table);
  API_END(1)
}
int cfb_debug_lpips_stem(cfb_lpips* n, const void* ref, const void* cand, int32_t u8, int32_t mode, float* out, int32_t batch,
                         int32_t h, int32_t w, int32_t group, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && ref && cand && out, "cfb_debug_lpips_stem: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  CFB_CHECK(n->begin_forward(false));
  CFB_REQUIRE(batch >= 0 && group >= 1 && h >= 1 && w >= 1, "cfb_debug_lpips_stem: bad size");
  cfb::LpIn in;
  if (u8) { in.ref8 = (const uint8_t*)ref; in.cand8 = (const uint8_t*)cand; in.convention = mode; }
  else { in.ref = (const float*)ref; in.cand = (const float*)cand; in.flags = mode; }
  return cfb::lp_stem(n, in, out, batch, group, h, w, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_debug_lpips_head_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t group) {
  if (batch < 0 || group < 1 || h < 1 || w < 1) return -1;
  return (int64_t)batch * group * cfb::lpips_head_blocks(h, w) * 4 + 256;
}
int cfb_debug_lpips_head(const float* feat, const float* lin, float* pooled, float* res, int32_t batch, int32_t h, int32_t w,
                         int32_t group, int32_t c, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(feat && lin && res && workspace, "cfb_debug_lpips_head: NULL argument");
  const int64_t need = cfb_debug_lpips_head_workspace_bytes(batch, h, w, group);
  CFB_REQUIRE(need >= 0 && workspace_bytes >= need, "cfb_debug_lpips_head: bad size or workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  CFB_CHECK(cfb::async_status_init(st));
  float* part = (float*)(((uintptr_t)workspace + 255) / 256 * 256);
  CFB_CHECK(cfb::lpips_head(feat, lin, batch, group, h, w, c, pooled, part, st));
  cfb::LpipsLayers L;
  L.n = 1; L.part[0] = part; L.nblk[0] = cfb::lpips_head_blocks(h, w); L.hw[0] = (int64_t)h * w;
  return cfb::lpips_finalize(L, batch * group, nullptr, res, st);
  API_END(1)
}

int64_t cfb_psnr_ssim_workspace_bytes(int32_t pairs, int32_t h, int32_t w, int32_t c, int32_t crop_border, int32_t y_channel) {
  if (pairs < 0 || h <= 0 || w <= 0 || c <= 0 || crop_border < 0) {
    cfb::set_error("cfb_psnr_ssim_workspace_bytes: bad size");
    return -1;
  }
  return (int64_t)cfb::metrics_workspace_bytes(pairs, h, w, c, crop_border, y_channel != 0);
}
int cfb_psnr_ssim(const void* a, const void* b, int32_t dtype, int32_t pairs, int32_t k, int32_t h, int32_t w, int32_t c,
                  int32_t crop_border, int32_t y_channel, int32_t want_psnr, int32_t want_ssim, double* psnr_out, double* ssim_out,
                  void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(dtype >= CFB_IMG_U8 && dtype <= CFB_IMG_F64, "cfb_psnr_ssim: dtype must be one of CFB_IMG_*");
  CFB_REQUIRE(pairs >= 0 && pairs <= 65535 && k >= 1 && pairs % k == 0, "cfb_psnr_ssim: bad pair count");
  CFB_REQUIRE(h > 0 && w > 0 && c > 0 && crop_border >= 0, "cfb_psnr_ssim: bad size");
  CFB_REQUIRE(want_psnr >= 0 && want_psnr <= 2, "cfb_psnr_ssim: want_psnr must be 0, 1 or 2");
  CFB_REQUIRE(!want_psnr || psnr_out, "cfb_psnr_ssim: NULL psnr_out");
  CFB_REQUIRE(!want_ssim || ssim_out, "cfb_psnr_ssim: NULL ssim_out");
  if (pairs == 0 || (!want_psnr && !want_ssim)) return 0;
  CFB_REQUIRE(a && b, "cfb_psnr_ssim: NULL image");
  const cfb::MetricArgs m{a, b, dtype, pairs, k, h, w, c, crop_border, y_channel != 0, want_psnr, want_psnr ? psnr_out : nullptr,
                          want_ssim ? ssim_out : nullptr};
  return cfb::psnr_ssim(m, workspace, workspace_bytes, (cudaStream_t)stream);
  API_END(1)
}

int cfb_check_async_status(void) {
  API_BEGIN
  return cfb::async_status_check("cfb_check_async_status");
  API_END(1)
}

int cfb_debug_set_wait_limit(int64_t cycles) {
  API_BEGIN
  CFB_REQUIRE(cycles > 0, "cfb_debug_set_wait_limit: cycles must be positive");
  CFB_CHECK(cfb::async_status_init(nullptr));
  {
    std::lock_guard<std::mutex> lk(cfb::g_status_mu);
    cfb::g_wait_limit_cycles = cycles;
  }
  int dev = 0;
  CFB_CUDA(cudaGetDevice(&dev));
  unsigned* dptr = nullptr;
  CFB_CUDA(cudaHostGetDevicePointer((void**)&dptr, cfb::g_status_words, 0));
  return cfb::tc_bind_status_word(dptr + dev, cycles);
  API_END(1)
}

int cfb_debug_inject_fault(int32_t kind) {
  API_BEGIN
  return cfb::tc_inject_fault(kind);
  API_END(1)
}
int cfb_debug_set_stamps(int64_t* stamps) {
  API_BEGIN
  return cfb::tc_set_stamps((long long*)stamps);
  API_END(1)
}

int cfb_net_set_param(cfb_net* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_net_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}

int cfb_net_prepare(cfb_net* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_net_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::prepare(n, (cudaStream_t)stream);
  API_END(1)
}

int64_t cfb_workspace_bytes(cfb_net* n, int32_t batch) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_workspace_bytes: NULL net"); return -1; }
  std::lock_guard<std::mutex> lk(n->mu);
  {
    auto it = n->ws_memo.find(batch);      // 16 host-side dry-run plans per miss: remember the answer per batch size
    if (it != n->ws_memo.end()) return it->second;
  }
  // The arena is first-fit, so the peak depends on the exact allocation sequence, which the call flags change (fusion on
  // or off, AdaIN, code_only, caller-provided logits or not): size for the worst of all of them (host-only dry runs).
  size_t high = 0;
  if (n->cfg.kind == 1) {
    for (int m = 0; m < 16; ++m) {
      const float w = (m & 1) ? 1.f : 0.f;
      float* lg = (m & 8) ? (float*)0x1000 : nullptr;
      if (cfb::codeformer_forward_impl(n, (const float*)0x1000, (float*)0x1000, lg, (float*)0x1000, nullptr, batch, w, (m >> 1) & 1,
                                       (m >> 2) & 1, nullptr, 0, nullptr, true) != 0)
        return -1;
      if (n->arena.high() > high) high = n->arena.high();
    }
  } else {
    for (int m = 0; m < 2; ++m) {
      if (cfb::vqae_forward_impl(n, (const float*)0x1000, (float*)0x1000, m ? (int64_t*)0x1000 : nullptr, m ? (float*)0x1000 : nullptr,
                                 nullptr, batch, nullptr, 0, nullptr, true) != 0)
        return -1;
      if (n->arena.high() > high) high = n->arena.high();
    }
  }
  n->ws_memo[batch] = (int64_t)high + 4096;
  return (int64_t)high + 4096;
  API_END(-1)
}

int64_t cfb_sweep_workspace_bytes(cfb_net* n, int32_t batch, int32_t k) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_sweep_workspace_bytes: NULL net"); return -1; }
  if (n->cfg.kind != 1 || batch < 0 || k < 1 || (int64_t)batch * k > INT32_MAX) {
    cfb::set_error("cfb_sweep_workspace_bytes: needs a CodeFormer net, batch >= 0 and k >= 1");
    return -1;
  }
  std::lock_guard<std::mutex> lk(n->mu);
  {
    auto it = n->sweep_ws_memo.find({batch, k});
    if (it != n->sweep_ws_memo.end()) return it->second;
  }
  // the worst of the flags a sweep takes: AdaIN on or off, caller-provided logits or not
  size_t high = 0;
  for (int m = 0; m < 4; ++m) {
    float* lg = (m & 2) ? (float*)0x1000 : nullptr;
    if (cfb::codeformer_forward_impl(n, nullptr, nullptr, lg, (float*)0x1000, nullptr, batch, 0.f, m & 1, 0, nullptr, 0, nullptr,
                                     true, (const unsigned char*)0x1000, (unsigned char*)0x1000, false, (const float*)0x1000,
                                     k) != 0)
      return -1;
    if (n->arena.high() > high) high = n->arena.high();
  }
  n->sweep_ws_memo[{batch, k}] = (int64_t)high + 4096;
  return (int64_t)high + 4096;
  API_END(-1)
}

int64_t cfb_last_launch_count(cfb_net* n) { return n ? n->last_launches : 0; }

int cfb_net_set_engine(cfb_net* n, int32_t engine) {
  API_BEGIN
  CFB_REQUIRE(n && engine >= 0 && engine <= 2, "cfb_net_set_engine: engine must be 0 (auto), 1 (fp32) or 2 (wgmma)");
  std::lock_guard<std::mutex> lk(n->mu);
  n->engine = engine;
  n->ws_memo.clear();
  n->sweep_ws_memo.clear();
  return 0;
  API_END(1)
}

int cfb_net_set_precision(cfb_net* n, int32_t precision) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_net_set_precision: NULL net");
  return n->set_precision(precision);
  API_END(1)
}

int cfb_net_capture(cfb_net* n, const char* stage, float* dst, int64_t capacity) {
  API_BEGIN
  CFB_REQUIRE(n && stage, "cfb_net_capture: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  if (dst) n->captures[stage] = {dst, capacity};
  else n->captures.erase(stage);
  n->ws_memo.clear();
  n->sweep_ws_memo.clear();
  return 0;
  API_END(1)
}

static int codeformer_f32(const char* what, cfb_net* n, const float* x, float* out, float* logits, float* lq_feat,
                          int64_t* top_idx, int32_t batch, float w, const float* w_dev, int32_t adain, int32_t code_only,
                          void* workspace, int64_t workspace_bytes, void* stream) {
  CFB_REQUIRE(n, std::string(what) + ": NULL net");
  if (batch == 0) return 0;
  CFB_REQUIRE(x, std::string(what) + ": NULL input");
  std::lock_guard<std::mutex> lk(n->mu);   // two caller threads may share one net (web-demos/hugging_face/app.py:282)
  const int64_t before = cfb::launch_count();
  const int rc = cfb::codeformer_forward_impl(n, x, out, logits, lq_feat, top_idx, batch, w, adain, code_only, workspace,
                                              workspace_bytes, (cudaStream_t)stream, false, nullptr, nullptr, false, w_dev);
  n->last_launches = cfb::launch_count() - before;
  return rc;
}

int cfb_codeformer_forward(cfb_net* n, const float* x, float* out, float* logits, float* lq_feat, int64_t* top_idx,
                           int32_t batch, float w, int32_t adain, int32_t code_only, void* workspace,
                           int64_t workspace_bytes, void* stream) {
  API_BEGIN
  return codeformer_f32("cfb_codeformer_forward", n, x, out, logits, lq_feat, top_idx, batch, w, nullptr, adain, code_only,
                        workspace, workspace_bytes, stream);
  API_END(1)
}

int cfb_codeformer_forward_wv(cfb_net* n, const float* x, float* out, float* logits, float* lq_feat, int64_t* top_idx,
                              int32_t batch, const float* w_dev, int32_t adain, int32_t code_only, void* workspace,
                              int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(w_dev || batch == 0, "cfb_codeformer_forward_wv: NULL w_dev");
  return codeformer_f32("cfb_codeformer_forward_wv", n, x, out, logits, lq_feat, top_idx, batch, 0.f, w_dev, adain, code_only,
                        workspace, workspace_bytes, stream);
  API_END(1)
}

static int codeformer_u8(const char* what, cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits,
                         float* lq_feat, int64_t* top_idx, int32_t batch, float w, int32_t adain, void* workspace,
                         int64_t workspace_bytes, void* stream, bool inpaint, const float* w_dev = nullptr, int sweep_k = 1) {
  CFB_REQUIRE(n, std::string(what) + ": NULL net");
  if (batch == 0) return 0;
  CFB_REQUIRE(faces_bgr && restored_bgr, std::string(what) + ": NULL image pointer");
  std::lock_guard<std::mutex> lk(n->mu);
  const int64_t before = cfb::launch_count();
  const int rc = cfb::codeformer_forward_impl(n, nullptr, nullptr, logits, lq_feat, top_idx, batch, w, adain, 0, workspace,
                                              workspace_bytes, (cudaStream_t)stream, false, faces_bgr, restored_bgr, inpaint,
                                              w_dev, sweep_k);
  n->last_launches = cfb::launch_count() - before;
  return rc;
}

int cfb_codeformer_forward_u8(cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                              int64_t* top_idx, int32_t batch, float w, int32_t adain, void* workspace,
                              int64_t workspace_bytes, void* stream) {
  API_BEGIN
  return codeformer_u8("cfb_codeformer_forward_u8", n, faces_bgr, restored_bgr, logits, lq_feat, top_idx, batch, w, adain,
                       workspace, workspace_bytes, stream, false);
  API_END(1)
}

int cfb_codeformer_inpaint_u8(cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                              int64_t* top_idx, int32_t batch, float w, int32_t adain, void* workspace,
                              int64_t workspace_bytes, void* stream) {
  API_BEGIN
  return codeformer_u8("cfb_codeformer_inpaint_u8", n, faces_bgr, restored_bgr, logits, lq_feat, top_idx, batch, w, adain,
                       workspace, workspace_bytes, stream, true);
  API_END(1)
}

int cfb_codeformer_forward_u8_wv(cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                                 int64_t* top_idx, int32_t batch, const float* w_dev, int32_t adain, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(w_dev || batch == 0, "cfb_codeformer_forward_u8_wv: NULL w_dev");
  return codeformer_u8("cfb_codeformer_forward_u8_wv", n, faces_bgr, restored_bgr, logits, lq_feat, top_idx, batch, 0.f, adain,
                       workspace, workspace_bytes, stream, false, w_dev);
  API_END(1)
}

int cfb_codeformer_inpaint_u8_wv(cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                                 int64_t* top_idx, int32_t batch, const float* w_dev, int32_t adain, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(w_dev || batch == 0, "cfb_codeformer_inpaint_u8_wv: NULL w_dev");
  return codeformer_u8("cfb_codeformer_inpaint_u8_wv", n, faces_bgr, restored_bgr, logits, lq_feat, top_idx, batch, 0.f, adain,
                       workspace, workspace_bytes, stream, true, w_dev);
  API_END(1)
}

int cfb_codeformer_sweep_u8(cfb_net* n, const uint8_t* faces_bgr, uint8_t* restored_bgr, float* logits, float* lq_feat,
                            int64_t* top_idx, int32_t batch, int32_t k, const float* w_dev, int32_t adain, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(k >= 1, "cfb_codeformer_sweep_u8: k must be >= 1");
  CFB_REQUIRE((int64_t)batch * k <= INT32_MAX, "cfb_codeformer_sweep_u8: batch * k too large");
  CFB_REQUIRE(w_dev || batch == 0, "cfb_codeformer_sweep_u8: NULL w_dev");
  return codeformer_u8("cfb_codeformer_sweep_u8", n, faces_bgr, restored_bgr, logits, lq_feat, top_idx, batch, 0.f, adain,
                       workspace, workspace_bytes, stream, false, w_dev, k);
  API_END(1)
}

int cfb_codeformer_restore_host(cfb_net* n, const uint8_t* faces_host, uint8_t* restored_host, int32_t batch, float w,
                                int32_t adain, void* dev_scratch, int64_t dev_scratch_bytes, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && faces_host && restored_host && dev_scratch, "cfb_codeformer_restore_host: NULL argument");
  CFB_REQUIRE(dev_scratch_bytes >= cfb_host_io_bytes(n, batch), "dev_scratch too small (cfb_host_io_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t img = (size_t)batch * 3 * n->cfg.img_size * n->cfg.img_size;
  uint8_t* din = (uint8_t*)dev_scratch;
  uint8_t* dout = din + (img + 1023) / 1024 * 1024;
  CFB_CUDA(cudaMemcpyAsync(din, faces_host, img, cudaMemcpyHostToDevice, st));
  CFB_CHECK(cfb_codeformer_forward_u8(n, din, dout, nullptr, nullptr, nullptr, batch, w, adain, workspace, workspace_bytes, stream));
  CFB_CUDA(cudaMemcpyAsync(restored_host, dout, img, cudaMemcpyDeviceToHost, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  return cfb::async_status_check("cfb_codeformer_restore_host");
  API_END(1)
}

int cfb_u8_to_input(const uint8_t* img_bgr_hwc, float* x_nchw, int32_t n, int32_t hw, void* stream) {
  API_BEGIN
  CFB_REQUIRE((img_bgr_hwc && x_nchw) || n == 0, "cfb_u8_to_input: NULL argument");
  return cfb::u8_to_input(img_bgr_hwc, x_nchw, n, hw, (cudaStream_t)stream);
  API_END(1)
}
int cfb_output_to_u8(const float* x_nchw, uint8_t* img_bgr_hwc, int32_t n, int32_t hw, void* stream) {
  API_BEGIN
  CFB_REQUIRE((img_bgr_hwc && x_nchw) || n == 0, "cfb_output_to_u8: NULL argument");
  return cfb::output_to_u8(x_nchw, img_bgr_hwc, n, hw, (cudaStream_t)stream);
  API_END(1)
}

int64_t cfb_host_io_bytes(cfb_net* n, int32_t batch) {
  if (!n) return -1;
  const cfb_config& c = n->cfg;
  const int64_t img = (int64_t)batch * 3 * c.img_size * c.img_size * 4;
  const int64_t lat = (int64_t)batch * c.latent_size;
  return 2 * (img + 1024) + lat * c.codebook_size * 4 + lat * c.emb_dim * 4 + 4096;
}

int cfb_codeformer_forward_host(cfb_net* n, const float* x_host, float* out_host, float* logits_host, float* lq_host,
                                int32_t batch, float w, int32_t adain, void* dev_scratch, int64_t dev_scratch_bytes,
                                void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && x_host && out_host && dev_scratch, "cfb_codeformer_forward_host: NULL argument");
  CFB_REQUIRE(dev_scratch_bytes >= cfb_host_io_bytes(n, batch), "dev_scratch too small (cfb_host_io_bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  const cfb_config& c = n->cfg;
  const size_t img = (size_t)batch * 3 * c.img_size * c.img_size * 4;
  const size_t lat = (size_t)batch * c.latent_size;
  char* p = (char*)dev_scratch;
  float* dx = (float*)p; p += (img + 1023) / 1024 * 1024;
  float* dout = (float*)p; p += (img + 1023) / 1024 * 1024;
  float* dlog = (float*)p; p += lat * c.codebook_size * 4;
  float* dlq = (float*)p;
  CFB_CUDA(cudaMemcpyAsync(dx, x_host, img, cudaMemcpyHostToDevice, st));
  CFB_CHECK(cfb_codeformer_forward(n, dx, dout, dlog, dlq, nullptr, batch, w, adain, 0, workspace, workspace_bytes, stream));
  CFB_CUDA(cudaMemcpyAsync(out_host, dout, img, cudaMemcpyDeviceToHost, st));
  if (logits_host) CFB_CUDA(cudaMemcpyAsync(logits_host, dlog, lat * c.codebook_size * 4, cudaMemcpyDeviceToHost, st));
  if (lq_host) CFB_CUDA(cudaMemcpyAsync(lq_host, dlq, lat * c.emb_dim * 4, cudaMemcpyDeviceToHost, st));
  CFB_CUDA(cudaStreamSynchronize(st));
  return cfb::async_status_check("cfb_codeformer_forward_host");
  API_END(1)
}

int cfb_vqae_forward(cfb_net* n, const float* x, float* out, int64_t* idx, float* stats, float* min_encodings,
                     int32_t batch, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_vqae_forward: NULL net");
  if (batch == 0) return 0;
  CFB_REQUIRE(x && out, "cfb_vqae_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  const int64_t before = cfb::launch_count();
  const int rc = cfb::vqae_forward_impl(n, x, out, idx, stats, min_encodings, batch, workspace, workspace_bytes,
                                        (cudaStream_t)stream, false);
  n->last_launches = cfb::launch_count() - before;
  return rc;
  API_END(1)
}

int64_t cfb_encoder_workspace_bytes(cfb_net* n, int32_t batch) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_encoder_workspace_bytes: NULL net"); return -1; }
  std::lock_guard<std::mutex> lk(n->mu);
  // the worst of the call forms: latent out alone, codes alone, both (host-only dry runs of the encoder)
  size_t high = 0;
  for (int m = 1; m < 4; ++m) {
    if (cfb::encoder_impl(n, (const float*)0x1000, nullptr, 0, (m & 1) ? (float*)0x1000 : nullptr, (m & 2) ? (int64_t*)0x1000 : nullptr,
                          batch, nullptr, 0, nullptr, true) != 0)
      return -1;
    if (n->arena.high() > high) high = n->arena.high();
  }
  return (int64_t)high + 4096;
  API_END(-1)
}

int cfb_encoder_forward(cfb_net* n, const float* x, float* latent, int32_t batch, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_encoder_forward: NULL net");
  if (batch == 0) return 0;
  CFB_REQUIRE(x && latent, "cfb_encoder_forward: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  const int64_t before = cfb::launch_count();
  const int rc = cfb::encoder_impl(n, x, nullptr, 0, latent, nullptr, batch, workspace, workspace_bytes, (cudaStream_t)stream, false);
  n->last_launches = cfb::launch_count() - before;
  return rc;
  API_END(1)
}

int cfb_latent_codes_u8(cfb_net* n, const uint8_t* faces_bgr, int64_t* idx, float* latent, int32_t batch, int32_t mirror,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_latent_codes_u8: NULL net");
  CFB_REQUIRE(batch >= 0 && mirror >= 0 && mirror <= batch, "cfb_latent_codes_u8: needs 0 <= mirror <= batch");
  CFB_REQUIRE((int64_t)batch + mirror <= INT32_MAX / 2, "cfb_latent_codes_u8: batch too large");
  if (batch == 0) return 0;
  CFB_REQUIRE(faces_bgr && idx, "cfb_latent_codes_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  const int64_t before = cfb::launch_count();
  const int rc = cfb::encoder_impl(n, nullptr, faces_bgr, mirror ? batch : 0, latent, idx, batch + mirror, workspace,
                                   workspace_bytes, (cudaStream_t)stream, false);
  n->last_launches = cfb::launch_count() - before;
  return rc;
  API_END(1)
}

int cfb_codeformer_code_only_u8(cfb_net* n, const uint8_t* faces_bgr, float* logits, float* lq_feat, int64_t* top_idx,
                                int32_t batch, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_codeformer_code_only_u8: NULL net");
  if (batch == 0) return 0;
  CFB_REQUIRE(faces_bgr && logits, "cfb_codeformer_code_only_u8: NULL argument");
  std::lock_guard<std::mutex> lk(n->mu);
  const int64_t before = cfb::launch_count();
  const int rc = cfb::codeformer_forward_impl(n, nullptr, nullptr, logits, lq_feat, top_idx, batch, 0.f, 0, 1, workspace,
                                              workspace_bytes, (cudaStream_t)stream, false, faces_bgr);
  n->last_launches = cfb::launch_count() - before;
  return rc;
  API_END(1)
}

int cfb_code_scores(const float* logits, const int64_t* top_idx, const int64_t* gt_idx, const float* lq_feat_nhwc,
                    const float* codebook, int32_t batch, int32_t tokens, int32_t codes, int32_t dim, double* scores, void* stream) {
  API_BEGIN
  CFB_REQUIRE(batch >= 0 && tokens > 0 && codes > 0 && dim > 0, "cfb_code_scores: bad shape");
  if (batch == 0) return 0;
  CFB_REQUIRE(logits && top_idx && gt_idx && lq_feat_nhwc && codebook && scores, "cfb_code_scores: NULL argument");
  return cfb::code_scores(logits, top_idx, gt_idx, lq_feat_nhwc, codebook, batch, tokens, codes, dim, scores, (cudaStream_t)stream);
  API_END(1)
}

static bool vq_tc_args(cfb::ConvArgs& a, int batch, int h, int w, int dim, int codes) {
  a = cfb::ConvArgs();
  a.N = batch; a.H = h; a.W = w; a.Cin = dim; a.Ho = h; a.Wo = w; a.Cout = codes; a.ksize = 1; a.mode = cfb::CONV_SAME;
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return major == 9 && cfb::tc_tiles_exact(a);
}

int64_t cfb_vq_workspace_bytes(int32_t batch, int32_t hw, int32_t dim, int32_t codes) {
  const int64_t T = (int64_t)batch * hw;
  const int64_t tok = 2 * ((T * dim * 4 + 1023) / 1024 * 1024);
  const int64_t simt = (int64_t)cfb::vq_workspace_bytes((int)T, dim, codes);
  // tensor-core path (16x16-style latents): split codebook + operand planes + the [T,K] dot products
  const int64_t wsplit = 2 * (int64_t)align256((size_t)codes * dim * 2) + 256;
  const int64_t planes = 2 * ((T * dim * 2 + 1023) / 1024 * 1024);
  const int64_t dots = (T * codes * 4 + 1023) / 1024 * 1024;
  const int64_t tc = wsplit + planes + dots + (int64_t)cfb::vq_select_workspace_bytes((int)T, codes) + 4096;
  return tok + (simt > tc ? simt : tc) + 8192;
}

int cfb_vq_nearest(const float* z, const float* codebook, int32_t batch, int32_t h, int32_t w, int32_t dim, int32_t codes,
                   float beta, float* z_q, int64_t* idx, float* stats, float* min_encodings, void* workspace,
                   int64_t workspace_bytes, void* stream) {
  API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t T = (int64_t)batch * h * w;
  if (T == 0) return 0;                     // empty batch: nothing to do (stats are left untouched)
  CFB_REQUIRE(z && codebook && z_q && idx && stats && workspace, "cfb_vq_nearest: NULL argument");
  CFB_REQUIRE(workspace_bytes >= cfb_vq_workspace_bytes(batch, h * w, dim, codes), "cfb_vq_nearest: workspace too small");
  const size_t tb = ((size_t)T * dim * 4 + 1023) / 1024 * 1024;
  char* p = (char*)workspace;
  float* zt = (float*)p; p += tb;
  float* zqt = (float*)p; p += tb;
  CFB_CHECK(cfb::nchw_to_nhwc(z, zt, batch, dim, h * w, st));
  cfb::ConvArgs a;
  // conv_tc's operand prep takes dim = 64 * 2^k (<= 2048); other widths (e.g. 320) run on the SIMT kernel
  if (vq_tc_args(a, batch, h, w, dim, codes) && dim >= 64 && dim <= 2048 && 256 % (dim / 8) == 0) {
    __half* whi = (__half*)p; p += align256((size_t)codes * dim * 2);
    __half* wlo = (__half*)p; p += align256((size_t)codes * dim * 2);
    float* wsc = (float*)p; p += 256;
    p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
    void* planes = p; p += 2 * (((size_t)T * dim * 2 + 1023) / 1024 * 1024);
    float* dots = (float*)p; p += ((size_t)T * codes * 4 + 1023) / 1024 * 1024;
    a.in = zt; a.out = dots; a.wgt_hi = whi; a.wgt_lo = wlo; a.wscale_inv = wsc + 1;
    int dev = 0, sms = 148;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CFB_CHECK(cfb::tc_split_weights(codebook, whi, wlo, codes, dim, 1, wsc, st));
    CFB_CHECK(cfb::conv_tc(a, planes, sms, st));
    CFB_CHECK(cfb::vq_select_from_dots(zt, codebook, dots, (int)T, dim, codes, beta, idx, zqt, stats, min_encodings, p, st));
  } else {
    CFB_CHECK(cfb::vq_nearest(zt, codebook, (int)T, dim, codes, beta, idx, zqt, stats, min_encodings, p, st));
  }
  CFB_CHECK(cfb::nhwc_to_nchw(zqt, z_q, batch, dim, h * w, st));
  return 0;
  API_END(1)
}

// ---- VectorQuantizer.forward, fused path (BASELINE config 3): ONE kernel (conv_tc.cu: vq_fused_kernel) on NCHW tensors ------
int32_t cfb_vq_fast_supported(int32_t batch, int32_t h, int32_t w, int32_t dim, int32_t codes) {
  cfb::ConvArgs a;
  return vq_tc_args(a, batch, h, w, dim, codes) && cfb::vq_fused_supported(batch, dim, h * w, codes) ? 1 : 0;
}
int64_t cfb_vq_prepared_bytes(int32_t codes, int32_t dim) {
  // split codebook (hi, lo), weight scale, |e|^2, and the self-cleaning code histogram + ticket of the one-kernel path
  return (int64_t)(2 * align256((size_t)codes * dim * 2) + 256 + 2 * align256((size_t)codes * 4) + 256);
}
int cfb_vq_prepare(const float* codebook, int32_t codes, int32_t dim, void* prepared, int64_t prepared_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(codebook && prepared && prepared_bytes >= cfb_vq_prepared_bytes(codes, dim), "cfb_vq_prepare: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  char* p = (char*)prepared;
  __half* whi = (__half*)p; p += align256((size_t)codes * dim * 2);
  __half* wlo = (__half*)p; p += align256((size_t)codes * dim * 2);
  float* wsc = (float*)p; p += 256;
  float* e2 = (float*)p;
  CFB_CHECK(cfb::tc_split_weights(codebook, whi, wlo, codes, dim, 1, wsc, st));
  CFB_CHECK(cfb::vq_e2(codebook, e2, codes, dim, st));
  CFB_CUDA(cudaMemsetAsync((char*)e2 + align256((size_t)codes * 4), 0, align256((size_t)codes * 4) + 256, st));   // histogram + ticket
  return 0;
  API_END(1)
}
int64_t cfb_vq_fast_workspace_bytes(int32_t batch, int32_t hw, int32_t dim, int32_t codes) {
  // vq_fused's partial sums (squared error, sum of distances: 2 doubles per CTA of 128 tokens) behind the 1024-byte alignment
  // cfb_vq_nearest_fast applies to the workspace pointer
  const int64_t ctas = (int64_t)batch * ((hw + 127) / 128);
  return ctas * 16 + 1024;
}
int cfb_vq_nearest_fast(const float* z, const float* codebook, const void* prepared, int32_t batch, int32_t h, int32_t w, int32_t dim,
                        int32_t codes, float beta, float* z_q, int64_t* idx, float* stats, float* min_encodings, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  API_BEGIN
  cudaStream_t st = (cudaStream_t)stream;
  const int HW = h * w;
  const int64_t T = (int64_t)batch * HW;
  if (T == 0) return 0;
  CFB_REQUIRE(z && codebook && prepared && z_q && idx && stats && workspace, "cfb_vq_nearest_fast: NULL argument");
  CFB_REQUIRE(cfb_vq_fast_supported(batch, h, w, dim, codes), "cfb_vq_nearest_fast: shape not on the fused path (use cfb_vq_nearest)");
  CFB_REQUIRE(workspace_bytes >= cfb_vq_fast_workspace_bytes(batch, HW, dim, codes), "cfb_vq_nearest_fast: workspace too small");
  CFB_CHECK(cfb::async_status_init(st));
  const char* q = (const char*)prepared;
  const __half* whi = (const __half*)q; q += align256((size_t)codes * dim * 2);
  const __half* wlo = (const __half*)q; q += align256((size_t)codes * dim * 2);
  const float* wsc = (const float*)q; q += 256;
  const float* e2 = (const float*)q;
  // the code histogram and the last-CTA ticket live in the prepared buffer (zero between calls)
  unsigned* hist = (unsigned*)((char*)e2 + align256((size_t)codes * 4));
  unsigned* ticket = (unsigned*)((char*)hist + align256((size_t)codes * 4));
  double* part = (double*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  CFB_CHECK(cfb::vq_fused(z, codebook, whi, wlo, wsc + 1, e2, hist, ticket, part, batch, dim, HW, codes, beta, z_q, idx, stats, st));
  if (min_encodings) CFB_CHECK(cfb::onehot_from_idx(idx, min_encodings, (int)T, codes, st));
  return 0;
  API_END(1)
}

int cfb_codebook_lookup(const int64_t* idx, const float* codebook, int32_t batch, int32_t h, int32_t w, int32_t dim,
                        int32_t codes, float* z_q, void* stream) {
  API_BEGIN
  CFB_REQUIRE(idx && codebook && z_q, "cfb_codebook_lookup: NULL argument");
  // gather token-major then transpose in place is not possible; gather straight into NCHW order instead
  // (small: B*256 tokens) via a temporary-free two-step is avoided by a strided gather kernel:
  cudaStream_t st = (cudaStream_t)stream;
  const int T = batch * h * w;
  if (T == 0) return 0;
  float* tmp = nullptr;
  CFB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)T * dim * 4, st));
  int rc = cfb::gather_rows(idx, codebook, tmp, T, codes, dim, st);
  if (rc == 0) rc = cfb::nhwc_to_nchw(tmp, z_q, batch, dim, h * w, st);
  cudaFreeAsync(tmp, st);
  return rc;
  API_END(1)
}

int64_t cfb_conv2d_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t mode) {
  cfb::ConvArgs a;
  a.N = n; a.H = h; a.W = w; a.Cin = cin; a.Cout = cout; a.ksize = ksize; a.mode = mode;
  a.Ho = mode == cfb::CONV_DOWN ? h / 2 : (mode == cfb::CONV_UP ? h * 2 : h);
  a.Wo = mode == cfb::CONV_DOWN ? w / 2 : (mode == cfb::CONV_UP ? w * 2 : w);
  const size_t wn = (size_t)cout * cin * ksize * ksize;
  const size_t wsplit = mode == cfb::CONV_UP ? (size_t)16 * cout * cin : wn;
  return (int64_t)(align256(wn * 4) + 2 * align256(wsplit * 2) + 256 + cfb::tc_scratch_bytes(a) + 8192);
}

int cfb_conv2d_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                    int32_t w, int32_t cin, int32_t cout, int32_t ksize, int32_t mode, const float* in_scale,
                    const float* in_shift, int32_t in_act, const float* residual, int32_t out_act, int32_t engine,
                    void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace, "cfb_conv2d_nhwc: NULL argument");
  CFB_CHECK(cfb::async_status_init(nullptr));
  CFB_REQUIRE(workspace_bytes >= cfb_conv2d_workspace_bytes(n, h, w, cin, cout, ksize, mode), "cfb_conv2d_nhwc: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  cfb::ConvArgs a;
  a.in = in; a.N = n; a.H = h; a.W = w; a.Cin = cin; a.Cout = cout; a.ksize = ksize; a.mode = mode;
  a.Ho = mode == cfb::CONV_DOWN ? h / 2 : (mode == cfb::CONV_UP ? h * 2 : h);
  a.Wo = mode == cfb::CONV_DOWN ? w / 2 : (mode == cfb::CONV_UP ? w * 2 : w);
  a.bias = bias; a.in_scale = in_scale; a.in_shift = in_shift; a.in_act = in_act; a.residual = residual;
  a.out_act = out_act; a.out = out;
  const size_t wn = (size_t)cout * cin * ksize * ksize;
  char* p = (char*)workspace;
  float* wf = (float*)p; p += align256(wn * 4);
  const size_t wsplit = mode == cfb::CONV_UP ? (size_t)16 * cout * cin : wn;
  __half* whi = (__half*)p; p += align256(wsplit * 2);
  __half* wlo = (__half*)p; p += align256(wsplit * 2);
  float* wsc = (float*)p; p += 256;
  p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
  a.wgt_f32 = wf; a.wgt_hi = whi; a.wgt_lo = wlo; a.wscale_inv = wsc + 1;
  bool use_tc = engine == 2;
  if (engine == 0) {
    int dev = 0, major = 0;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    use_tc = major == 9 && cfb::tc_tiles_exact(a);
  }
  if (use_tc) {
    CFB_REQUIRE(cfb::tc_supported(a), "cfb_conv2d_nhwc: shape not supported by the wgmma engine");
    int dev = 0, sms = 148;
    CFB_CUDA(cudaGetDevice(&dev));
    CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (mode == cfb::CONV_UP) CFB_CHECK(cfb::tc_split_weights_up4(weight_oihw, whi, wlo, cout, cin, wsc, st));
    else CFB_CHECK(cfb::tc_split_weights(weight_oihw, whi, wlo, cout, cin, ksize, wsc, st));
    // same choice as the network runtime (Fwd::conv): a GroupNorm-affine (+SiLU) input goes through the in-kernel operand
    // transform wherever the engine has it, so the kernel tests exercise the path the forward ships
    if (in_scale && in_shift && cfb::tc_can_xform(a)) { a.xform = true; a.skip_prep = true; }
    CFB_CHECK(cfb::conv_tc(a, p, sms, st));
  } else {
    CFB_CHECK(cfb::relayout_oihw_to_tck(weight_oihw, wf, cout, cin, ksize, st));
    CFB_CHECK(cfb::conv_f32(a, st));
  }
  return 0;
  API_END(1)
}

int cfb_debug_conv_tc(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias, float* out,
                      int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                      const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                      const float* sft_dec, const float* sft_scale, float sft_w, void* out_planes, float* gn_part,
                      void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n) {
  return cfb_debug_conv_tc_prec(in, in2, cin1, weight_oihw, bias, out, n, h, w, cin, cout, mode, xform, in_scale, in_shift, in_act,
                                residual, sft_dec, sft_scale, sft_w, out_planes, gn_part, workspace, workspace_bytes, stream,
                                tile_n, 3, cfb::OUT_NONE, 0);
}

static int debug_conv_tc(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias,
                         float* out, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                         const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                         const float* sft_dec, const float* sft_scale, float sft_w, const float* sft_wv, void* out_planes,
                         float* gn_part, void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n, int32_t ksize,
                         int32_t out_act, int32_t precision) {
  CFB_REQUIRE(in && weight_oihw && out && workspace && tile_n, "cfb_debug_conv_tc: NULL argument");
  CFB_REQUIRE(mode == cfb::CONV_SAME || mode == cfb::CONV_UP, "cfb_debug_conv_tc: mode must be 0 or 2");
  CFB_REQUIRE(ksize == 3 || (ksize == 1 && mode == cfb::CONV_SAME && !xform), "cfb_debug_conv_tc_prec: ksize 3, or 1 (raw, mode 0)");
  CFB_REQUIRE(precision == 0 || precision == 1, "cfb_debug_conv_tc_prec: precision must be 0 (fp32, split) or 1 (fp16)");
  CFB_REQUIRE(out_act == cfb::OUT_NONE || out_act == cfb::OUT_LRELU, "cfb_debug_conv_tc_prec: out_act must be 0 or 1 (LeakyReLU)");
  CFB_REQUIRE(workspace_bytes >= cfb_conv2d_workspace_bytes(n, h, w, cin, cout, ksize, mode), "cfb_debug_conv_tc: workspace too small");
  CFB_CHECK(cfb::async_status_init(nullptr));
  cudaStream_t st = (cudaStream_t)stream;
  cfb::ConvArgs a;
  a.in = in; a.N = n; a.H = h; a.W = w; a.Cin = cin; a.Cout = cout; a.ksize = ksize; a.mode = mode;
  a.Ho = mode == cfb::CONV_UP ? h * 2 : h;
  a.Wo = mode == cfb::CONV_UP ? w * 2 : w;
  a.bias = bias; a.in_scale = in_scale; a.in_shift = in_shift; a.in_act = in_act; a.residual = residual; a.out = out;
  a.sft_dec = sft_dec; a.sft_scale = sft_scale; a.sft_w = sft_w; a.sft_wv = sft_wv; a.out_planes = out_planes; a.gn_part = gn_part;
  a.in2 = in2; a.Cin1 = in2 ? cin1 : 0;
  a.out_act = out_act; a.single_pass = precision == 1;
  CFB_REQUIRE(cfb::tc_supported(a), "cfb_debug_conv_tc: shape not on the wgmma engine");
  const size_t wn = (size_t)cout * cin * ksize * ksize;
  const size_t wsplit = mode == cfb::CONV_UP ? (size_t)16 * cout * cin : wn;
  char* p = (char*)workspace + align256(wn * 4);
  __half* whi = (__half*)p; p += align256(wsplit * 2);
  __half* wlo = (__half*)p; p += align256(wsplit * 2);
  float* wsc = (float*)p; p += 256;
  p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
  a.wgt_hi = whi; a.wgt_lo = wlo; a.wscale_inv = wsc + 1;
  if (xform) {
    CFB_REQUIRE(cfb::tc_can_xform(a), "cfb_debug_conv_tc: no fused operand transform for this conv");
    a.xform = true; a.skip_prep = true;
  }
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (mode == cfb::CONV_UP) CFB_CHECK(cfb::tc_split_weights_up4(weight_oihw, whi, wlo, cout, cin, wsc, st));
  else CFB_CHECK(cfb::tc_split_weights(weight_oihw, whi, wlo, cout, cin, ksize, wsc, st));
  *tile_n = cfb::tc_tile_n(a);
  CFB_CHECK(cfb::conv_tc(a, p, sms, st));
  return 0;
}

int cfb_debug_conv_tc_prec(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias,
                           float* out, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                           const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                           const float* sft_dec, const float* sft_scale, float sft_w, void* out_planes, float* gn_part,
                           void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n, int32_t ksize,
                           int32_t out_act, int32_t precision) {
  API_BEGIN
  return debug_conv_tc(in, in2, cin1, weight_oihw, bias, out, n, h, w, cin, cout, mode, xform, in_scale, in_shift, in_act, residual,
                       sft_dec, sft_scale, sft_w, nullptr, out_planes, gn_part, workspace, workspace_bytes, stream, tile_n, ksize,
                       out_act, precision);
  API_END(1)
}

int cfb_debug_conv_tc_prec_wv(const float* in, const float* in2, int32_t cin1, const float* weight_oihw, const float* bias,
                              float* out, int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t mode, int32_t xform,
                              const float* in_scale, const float* in_shift, int32_t in_act, const float* residual,
                              const float* sft_dec, const float* sft_scale, const float* sft_wv, void* out_planes,
                              float* gn_part, void* workspace, int64_t workspace_bytes, void* stream, int32_t* tile_n,
                              int32_t ksize, int32_t out_act, int32_t precision) {
  API_BEGIN
  CFB_REQUIRE(sft_wv || !sft_dec, "cfb_debug_conv_tc_prec_wv: NULL sft_wv with an SFT epilogue");
  return debug_conv_tc(in, in2, cin1, weight_oihw, bias, out, n, h, w, cin, cout, mode, xform, in_scale, in_shift, in_act, residual,
                       sft_dec, sft_scale, 0.f, sft_wv, out_planes, gn_part, workspace, workspace_bytes, stream, tile_n, ksize,
                       out_act, precision);
  API_END(1)
}

static size_t align1024(size_t b) { return (b + 1023) / 1024 * 1024; }
int64_t cfb_debug_bmm_tc_workspace_bytes(int32_t n, int32_t heads, int32_t d) {
  const size_t T = (size_t)n * 256, E = (size_t)heads * d;
  return (int64_t)(1024 + 2 * align1024(T * 2 * E * 2) + 2 * align1024(T * E * 2) + align1024(T * heads * 256 * 4) +
                   2 * align1024(T * heads * 256 * 2) + 2 * align1024(T * E * 2));
}
int cfb_debug_bmm_tc(const float* q, const float* k, const float* v, float* out, void* out_planes, int32_t n, int32_t heads,
                     int32_t d, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(q && k && v && out && workspace, "cfb_debug_bmm_tc: NULL argument");
  CFB_REQUIRE(n >= 0 && heads >= 1 && d >= 64 && d % 64 == 0, "cfb_debug_bmm_tc: d must be a positive multiple of 64");
  CFB_REQUIRE(workspace_bytes >= cfb_debug_bmm_tc_workspace_bytes(n, heads, d), "cfb_debug_bmm_tc: workspace too small");
  CFB_CHECK(cfb::async_status_init(nullptr));
  cudaStream_t st = (cudaStream_t)stream;
  const int E = heads * d;
  const int64_t T = (int64_t)n * 256, rows = T * heads;
  char* p = (char*)workspace;
  float* consts = (float*)p; p += 1024;
  void* qk = p; p += 2 * align1024((size_t)T * 2 * E * 2);
  void* vp = p; p += 2 * align1024((size_t)T * E * 2);
  float* scores = (float*)p; p += align1024((size_t)rows * 256 * 4);
  void* pp = p; p += 2 * align1024((size_t)rows * 256 * 2);
  void* vt = p;
  // the scale of each core as the forward holds it: C^-1/2 (AttnBlock, one head), head_dim^-1/2 (nn.MultiheadAttention)
  const float hc[2] = {1.0f / sqrtf((float)d), 1.0f};
  CFB_CUDA(cudaMemcpyAsync(consts, hc, sizeof(hc), cudaMemcpyHostToDevice, st));
  // q | k and v as the operand planes their producing convs write (one [T][2E] plane pair, one [T][E])
  CFB_CHECK(cfb::concat_planes(q, k, qk, T, E, E, st));
  CFB_CHECK(cfb::concat_planes(v, nullptr, vp, T, E, 0, st));
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  // the launch sequence of Fwd::attnblock (heads 1) and of the Transformer layer (several heads), with an fp32 output added
  cfb::BmmArgs g1;
  g1.a_planes = qk; g1.a_pitch = 2 * E; g1.a_c0 = 0;
  g1.b_planes = qk; g1.b_pitch = 2 * E; g1.b_c0 = E; g1.b_rows = 256;
  g1.N = n; g1.K = d; g1.Cout = 256; g1.scale_dev = consts; g1.out = scores;
  if (heads > 1) { g1.heads = heads; g1.a_c_head = d; g1.b_c_head = d; g1.out_per_head = true; }
  CFB_CHECK(cfb::bmm_tc(g1, sms, st));
  CFB_CHECK(cfb::softmax256_planes(scores, pp, rows, st));
  CFB_CHECK(cfb::transpose_planes(vp, n, E, 0, E, vt, st));
  cfb::BmmArgs g2;
  g2.a_planes = pp; g2.a_pitch = 256; g2.a_c0 = 0;
  g2.b_planes = vt; g2.b_pitch = 256; g2.b_c0 = 0; g2.b_rows = E;
  g2.N = n; g2.K = 256; g2.Cout = heads > 1 ? d : E; g2.scale_dev = consts + 1; g2.out = out; g2.out_planes = out_planes;
  if (heads > 1) { g2.heads = heads; g2.a_img_per_head = true; g2.b_r_head = d; g2.out_per_head = false; g2.o_c_head = d; }
  CFB_CHECK(cfb::bmm_tc(g2, sms, st));
  return 0;
  API_END(1)
}

int cfb_debug_time_conv(const float* in, const float* weight_oihw, float* out, int32_t n, int32_t h, int32_t w, int32_t cin,
                        int32_t cout, int32_t ksize, int32_t mode, int32_t reps, void* workspace, int64_t workspace_bytes,
                        void* stream, const float* in_scale, const float* in_shift, int32_t in_act, float* ms_per_launch) {
  API_BEGIN
  CFB_REQUIRE(in && weight_oihw && out && workspace && ms_per_launch && reps > 0, "cfb_debug_time_conv: bad argument");
  CFB_REQUIRE(workspace_bytes >= cfb_conv2d_workspace_bytes(n, h, w, cin, cout, ksize, mode), "cfb_debug_time_conv: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  cfb::ConvArgs a;
  a.in = in; a.N = n; a.H = h; a.W = w; a.Cin = cin; a.Cout = cout; a.ksize = ksize; a.mode = mode;
  a.Ho = mode == cfb::CONV_DOWN ? h / 2 : (mode == cfb::CONV_UP ? h * 2 : h);
  a.Wo = mode == cfb::CONV_DOWN ? w / 2 : (mode == cfb::CONV_UP ? w * 2 : w);
  a.out = out;
  CFB_REQUIRE(cfb::tc_supported(a), "cfb_debug_time_conv: shape not on the wgmma engine");
  const size_t wn = (size_t)cout * cin * ksize * ksize;
  const size_t wsplit = mode == cfb::CONV_UP ? (size_t)16 * cout * cin : wn;
  char* p = (char*)workspace + align256(wn * 4);
  __half* whi = (__half*)p; p += align256(wsplit * 2);
  __half* wlo = (__half*)p; p += align256(wsplit * 2);
  float* wsc = (float*)p; p += 256;
  p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
  a.wgt_hi = whi; a.wgt_lo = wlo; a.wscale_inv = wsc + 1;
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (mode == cfb::CONV_UP) CFB_CHECK(cfb::tc_split_weights_up4(weight_oihw, whi, wlo, cout, cin, wsc, st));
  else CFB_CHECK(cfb::tc_split_weights(weight_oihw, whi, wlo, cout, cin, ksize, wsc, st));
  CFB_CHECK(cfb::async_status_init(nullptr));
  a.in_scale = in_scale; a.in_shift = in_shift; a.in_act = in_act;
  // a GroupNorm-affine (+SiLU) input: the kernel timed is the one the forward ships -- fused operand transform where the
  // engine has it (all-in: no separate prep pass exists), otherwise prep once outside the timed region
  if (in_scale && in_shift && cfb::tc_can_xform(a)) { a.xform = true; a.skip_prep = true; }
  CFB_CHECK(cfb::conv_tc(a, p, sms, st));          // operand prep + one warm-up launch
  a.skip_prep = true;
  for (int i = 0; i < 2; ++i) CFB_CHECK(cfb::conv_tc(a, p, sms, st));
  cudaEvent_t e0, e1;
  CFB_CUDA(cudaEventCreate(&e0));
  CFB_CUDA(cudaEventCreate(&e1));
  CFB_CUDA(cudaEventRecord(e0, st));               // events on the launching stream: only the conv kernel is between them
  for (int i = 0; i < reps; ++i) CFB_CHECK(cfb::conv_tc(a, p, sms, st));
  CFB_CUDA(cudaEventRecord(e1, st));
  CFB_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  CFB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ms_per_launch = ms / reps;
  return 0;
  API_END(1)
}

int64_t cfb_gn_workspace_bytes(int32_t n, int32_t hw, int32_t c) { return (int64_t)cfb::gn_workspace_bytes(n, hw, c) + 256; }
int cfb_group_norm_coef(const float* x, const float* gamma, const float* beta, float* scale, float* shift, int32_t n,
                        int32_t hw, int32_t c, int32_t groups, float eps, void* workspace, int64_t workspace_bytes,
                        void* stream) {
  API_BEGIN
  CFB_REQUIRE(x && gamma && beta && scale && shift && workspace, "cfb_group_norm_coef: NULL argument");
  CFB_REQUIRE(workspace_bytes >= (int64_t)cfb::gn_workspace_bytes(n, hw, c), "cfb_group_norm_coef: workspace too small");
  return cfb::gn_coef(x, gamma, beta, scale, shift, n, hw, c, groups, eps, workspace, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_debug_gn_partials_workspace_bytes(int32_t n, int32_t slots) {
  return (int64_t)(align256(cfb::gn_final_scratch_bytes(n, slots)) + align256((size_t)n * sizeof(unsigned)));
}
int cfb_debug_gn_coef_from_partials(const float* part, int32_t slots, const float* gamma, const float* beta, float* scale,
                                    float* shift, int32_t n, int32_t hw, int32_t c, float eps, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(part && gamma && beta && scale && shift && workspace && n >= 0 && slots > 0,
              "cfb_debug_gn_coef_from_partials: bad argument");
  CFB_REQUIRE(workspace_bytes >= cfb_debug_gn_partials_workspace_bytes(n, slots), "cfb_debug_gn_coef_from_partials: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  // finalize scratch, then the ticket counters, which the kernel needs zero on entry
  unsigned* ctr = (unsigned*)((char*)workspace + align256(cfb::gn_final_scratch_bytes(n, slots)));
  CFB_CUDA(cudaMemsetAsync(ctr, 0, (size_t)n * sizeof(unsigned), st));
  return cfb::gn_coef_from_partials(part, slots, gamma, beta, scale, shift, n, hw, c, 32, eps, workspace, ctr, st);
  API_END(1)
}
int cfb_debug_gn_cat_partials(const float* a_part, const float* b_part, float* out_part, int64_t total_slots, int32_t c,
                              void* stream) {
  API_BEGIN
  CFB_REQUIRE(a_part && b_part && out_part && total_slots >= 0 && c > 0 && c % 32 == 0, "cfb_debug_gn_cat_partials: bad argument");
  return cfb::gn_cat_partials(a_part, b_part, out_part, total_slots, c, (cudaStream_t)stream);
  API_END(1)
}
int cfb_affine_act(const float* x, const float* scale, const float* shift, float* y, int32_t n, int32_t hw, int32_t c,
                   int32_t act, void* stream) {
  API_BEGIN
  return cfb::affine_act(x, scale, shift, y, n, hw, c, act, (cudaStream_t)stream);
  API_END(1)
}
int cfb_attention(const float* q, const float* k, const float* v, float* out, int32_t batch, int32_t tokens, int32_t heads,
                  int32_t d, int32_t q_pitch, int32_t k_pitch, int32_t v_pitch, int32_t o_pitch, float scale, void* stream) {
  API_BEGIN
  return cfb::attention(q, k, v, out, batch, tokens, heads, d, q_pitch, k_pitch, v_pitch, o_pitch, scale, (cudaStream_t)stream);
  API_END(1)
}
int cfb_layer_norm(const float* x, const float* gamma, const float* beta, float* y, float* y2, const float* pos,
                   int32_t pos_rows, int32_t rows, int32_t c, void* stream) {
  API_BEGIN
  return cfb::layer_norm(x, gamma, beta, y, y2, pos, pos_rows, rows, c, (cudaStream_t)stream);
  API_END(1)
}
int cfb_debug_layer_norm_planes(const float* x, const float* gamma, const float* beta, void* y_planes, void* y2_planes,
                                const float* pos, int32_t pos_rows, int32_t rows, int32_t c, void* stream) {
  API_BEGIN
  CFB_REQUIRE(x && gamma && beta && (y_planes || y2_planes), "cfb_debug_layer_norm_planes: NULL argument");
  CFB_REQUIRE(!y2_planes || (pos && pos_rows > 0), "cfb_debug_layer_norm_planes: y2_planes needs pos and pos_rows > 0");
  return cfb::layer_norm_planes(x, gamma, beta, y_planes, y2_planes, pos, pos_rows, rows, c, (cudaStream_t)stream);
  API_END(1)
}
int cfb_debug_code_lookup(const float* logits, const float* codebook, int64_t* idx, float* quant, int32_t T, int32_t K,
                          int32_t D, void* stream) {
  API_BEGIN
  CFB_REQUIRE(logits && codebook && (idx || quant) && T >= 0 && K > 0 && D > 0, "cfb_debug_code_lookup: bad argument");
  return cfb::argmax_gather(logits, codebook, idx, quant, T, K, D, (cudaStream_t)stream);
  API_END(1)
}
int cfb_adain_nhwc(const float* content, const float* style, float* out, int32_t batch, int32_t hw, int32_t c, void* stream) {
  API_BEGIN
  return cfb::adain_nhwc(content, style, out, batch, hw, c, (cudaStream_t)stream);
  API_END(1)
}
int cfb_nchw_to_nhwc(const float* in, float* out, int32_t n, int32_t c, int32_t hw, void* stream) {
  API_BEGIN
  return cfb::nchw_to_nhwc(in, out, n, c, hw, (cudaStream_t)stream);
  API_END(1)
}
int cfb_nhwc_to_nchw(const float* in, float* out, int32_t n, int32_t c, int32_t hw, void* stream) {
  API_BEGIN
  return cfb::nhwc_to_nchw(in, out, n, c, hw, (cudaStream_t)stream);
  API_END(1)
}


cfb_fid* cfb_fid_create(void) {
  API_BEGIN
  cfb_fid* n = new cfb_fid();
  cfb::fid_build(n);           // the plan: workspace queries need no prepared weights
  return n;
  API_END(nullptr)
}
void cfb_fid_destroy(cfb_fid* n) { delete n; }
int cfb_fid_set_param(cfb_fid* n, const char* name, const float* dev_ptr, int64_t numel) {
  API_BEGIN
  CFB_REQUIRE(n && name && dev_ptr, "cfb_fid_set_param: NULL argument");
  return n->set_param(name, dev_ptr, numel);
  API_END(1)
}
int cfb_fid_prepare(cfb_fid* n, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n, "cfb_fid_prepare: NULL net");
  std::lock_guard<std::mutex> lk(n->mu);
  return cfb::fid_prepare(n, (cudaStream_t)stream);
  API_END(1)
}
int64_t cfb_fid_workspace_bytes(cfb_fid* n, int32_t batch, int32_t h, int32_t w, int32_t resize) {
  API_BEGIN
  if (!n) { cfb::set_error("cfb_fid_workspace_bytes: NULL net"); return -1; }
  cfb::FidInput in;
  in.f32 = (const float*)0x1000; in.H = h; in.W = w; in.resize = resize != 0;
  return n->dry_run([&] { return cfb::fid_forward(n, in, batch, nullptr, nullptr, 0, nullptr, true); });
  API_END(-1)
}
int cfb_fid_forward(cfb_fid* n, const float* x_nchw, int32_t batch, int32_t h, int32_t w, int32_t resize, int32_t normalize,
                    float* feat, void* workspace, int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (x_nchw && feat && workspace)), "cfb_fid_forward: NULL argument");
  CFB_REQUIRE(((uintptr_t)feat & 15) == 0, "cfb_fid_forward: feat must be 16-byte aligned");
  std::lock_guard<std::mutex> lk(n->mu);
  cfb::FidInput in;
  in.f32 = x_nchw; in.H = h; in.W = w; in.resize = resize != 0; in.normalize = normalize != 0;
  return cfb::fid_forward(n, in, batch, feat, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_fid_forward_u8(cfb_fid* n, const uint8_t* faces_bgr, int32_t batch, int32_t h, int32_t w, float* feat, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  API_BEGIN
  CFB_REQUIRE(n && (batch == 0 || (faces_bgr && feat && workspace)), "cfb_fid_forward_u8: NULL argument");
  CFB_REQUIRE(((uintptr_t)feat & 15) == 0, "cfb_fid_forward_u8: feat must be 16-byte aligned");
  std::lock_guard<std::mutex> lk(n->mu);
  cfb::FidInput in;
  in.u8 = faces_bgr; in.H = h; in.W = w; in.resize = 1; in.normalize = 1;
  return cfb::fid_forward(n, in, batch, feat, workspace, workspace_bytes, (cudaStream_t)stream, false);
  API_END(1)
}
int cfb_fid_input(const void* src, int32_t u8, int32_t batch, int32_t h, int32_t w, int32_t resize, int32_t normalize, float* out,
                  void* stream) {
  API_BEGIN
  CFB_REQUIRE(batch == 0 || (src && out), "cfb_fid_input: NULL argument");
  CFB_REQUIRE(batch >= 0 && h >= 1 && w >= 1, "cfb_fid_input: bad size");
  cfb::FidInput in;
  if (u8) in.u8 = (const uint8_t*)src; else in.f32 = (const float*)src;
  in.H = h; in.W = w; in.resize = resize != 0; in.normalize = normalize != 0;
  return cfb::fid_input(in, out, batch, (cudaStream_t)stream);
  API_END(1)
}
int cfb_fid_stats(const float* feat, int64_t n, int32_t d, double* mu, double* sigma, void* stream) {
  API_BEGIN
  CFB_REQUIRE(feat && mu && sigma, "cfb_fid_stats: NULL argument");
  return cfb::fid_stats(feat, n, d, mu, sigma, (cudaStream_t)stream);
  API_END(1)
}
int cfb_debug_fid_pool(const float* in, float* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t kind, void* stream) {
  API_BEGIN
  CFB_REQUIRE(in && out, "cfb_debug_fid_pool: NULL argument");
  CFB_REQUIRE(n >= 0 && h >= 1 && w >= 1 && c >= 4 && kind >= 0 && kind <= 2, "cfb_debug_fid_pool: bad size or kind");
  cudaStream_t st = (cudaStream_t)stream;
  if (kind == 2) return cfb::fid_avgpool(in, c, out, c, n, h, w, c, st);
  return cfb::fid_maxpool(in, c, out, c, 0, n, h, w, c, kind == 0 ? 2 : 1, st);
  API_END(1)
}

int64_t cfb_conv2d_pertap_window_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw,
                                                 int32_t stride, int32_t pad_h, int32_t pad_w) {
  if (n < 0 || h < 1 || w < 1 || cin < 1 || cout < 1 || kh < 1 || kw < 1 || kh > 7 || kw > 7 || !(stride == 1 || stride == 2) ||
      pad_h < 0 || pad_w < 0)
    return -1;
  cfb::GenConv c = cfb::plan_conv("", cin, cout, 1, stride);
  c.kh = kh; c.kw = kw; c.pad_h = pad_h; c.pad_w = pad_w;
  if (h + 2 * pad_h < kh || w + 2 * pad_w < kw) return -1;
  const cfb::ConvArgs a = cfb::pertap_window_args(nullptr, n, h, w, c, nullptr, c.cout_p, 0, cfb::OUT_NONE);
  const size_t wn = (size_t)c.cout_p * c.cin_p * c.taps();
  return (int64_t)(align256(wn * 4) + 2 * align256(wn * 2) + align256((size_t)c.cout_p * 4) + 256 + cfb::tc_scratch_bytes(a) + 8192);
}

int cfb_conv2d_pertap_window_nhwc(const float* in, const float* weight_oihw, const float* bias, float* out, int32_t n, int32_t h,
                                  int32_t w, int32_t cin, int32_t cout, int32_t kh, int32_t kw, int32_t stride, int32_t pad_h,
                                  int32_t pad_w, int32_t out_act, int32_t out_pitch, int32_t out_c0, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  API_BEGIN
  const char* fn = "cfb_conv2d_pertap_window_nhwc";
  CFB_REQUIRE(in && weight_oihw && out && workspace, std::string(fn) + ": NULL argument");
  CFB_REQUIRE(cin % 64 == 0 && cout % 4 == 0, std::string(fn) + ": cin must be a multiple of 64 and cout of 4");
  CFB_REQUIRE(out_act == cfb::OUT_NONE || out_act == cfb::OUT_RELU, std::string(fn) + ": activation must be none or ReLU");
  const int64_t need = cfb_conv2d_pertap_window_workspace_bytes(n, h, w, cin, cout, kh, kw, stride, pad_h, pad_w);
  CFB_REQUIRE(need > 0 && workspace_bytes >= need, std::string(fn) + ": bad shape or workspace too small");
  CFB_REQUIRE(out_pitch >= cout && out_c0 >= 0 && out_c0 + cout <= out_pitch, std::string(fn) + ": slice outside the pitch");
  cudaStream_t st = (cudaStream_t)stream;
  CFB_CHECK(cfb::async_status_init(st));
  int dev = 0, sms = 148;
  CFB_CUDA(cudaGetDevice(&dev));
  CFB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cfb::GenConv c = cfb::plan_conv("", cin, cout, 1, stride);
  c.kh = kh; c.kw = kw; c.pad_h = pad_h; c.pad_w = pad_w;
  char* p = (char*)(((uintptr_t)workspace + 1023) / 1024 * 1024);
  float* pad = (float*)p; p += align256((size_t)c.cout_p * c.cin_p * c.taps() * 4);
  CFB_CHECK(cfb::prepare_conv(c, weight_oihw, bias, pad, p, st));
  p = (char*)(((uintptr_t)p + 1023) / 1024 * 1024);
  cfb::ConvArgs a = cfb::pertap_window_args(in, n, h, w, c, out, out_pitch, out_c0, out_act);
  if (out_pitch == c.cout_p && out_c0 == 0 && cout != c.cout_p) a.cout_valid = cout;
  a.wgt_hi = c.w_hi; a.wgt_lo = c.w_lo; a.wscale_inv = c.wscale + 1; a.bias = c.bias;
  CFB_REQUIRE(cfb::tc_supported(a), std::string(fn) + ": shape not supported by the wgmma engine");
  return cfb::conv_tc(a, p, sms, st);
  API_END(1)
}
}  // extern "C"
