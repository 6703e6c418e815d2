// C ABI of libamphion_b200: handles, parameter arena, forward plans.
// See include/amphion_b200.h for the contract and the reference citations.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "ab_common.cuh"
#include "ab_tc.cuh"

namespace ab {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

}  // namespace ab

using namespace ab;

// ---------------------------------------------------------------------------
// generator handle
// ---------------------------------------------------------------------------
namespace {

enum SlotKind { SLOT_CONV_W, SLOT_CONVT_W, SLOT_VEC };

struct Slot {
  std::string name;
  SlotKind kind;
  int64_t shape[3];   // reference state-dict shape
  int ndim;
  size_t offset;      // into the arena (fp32 repacked image)
  size_t bytes;
  bool loaded;
  // 16-bit weight image for the wgmma kernel (built by finalize when precision != fp32); tc_bytes > 0 iff the conv
  // runs there (tc_image_bytes)
  size_t tc_offset;
  size_t tc_bytes;
  int stride;         // ConvTranspose1d stride (SLOT_CONVT_W)
  int dilation;       // Conv1d dilation (SLOT_CONV_W)
  float gain = 1.0f;  // applied to the fp32 image at load time (NSF-HiFiGAN: 2 on every ups weight / bias)
};

struct ConvRef {   // one weight-normed conv of the model
  int w = -1, b = -1;
  int cin = 0, cout = 0, k = 0, d = 1;
};

struct ActRef {    // one Activation1d module
  int alpha = -1, beta = -1, fup = -1, fdown = -1;
};

struct BlockRef {  // one ResBlock / AMPBlock
  int k = 0;
  std::vector<int> dil;
  std::vector<ConvRef> c1, c2;  // c2 empty for ResBlock2 / AMPBlock2
  std::vector<ActRef> acts;     // 2*nd (type 1) or nd (type 2); empty for HiFi-GAN
};

struct StageRef {
  ConvRef up;   // cin/cout/k, d unused; stride in `u`
  int u = 1;
  int ch = 0;
  bool has_up = true;   // false: AB_GEN_TRUNK's single stage (no transposed conv in front of the blocks)
  std::vector<BlockRef> blocks;
};

}  // namespace

struct ab_generator {
  ab_generator_config cfg;
  std::vector<Slot> slots;
  std::unordered_map<std::string, int> index;
  size_t fp32_bytes = 0;    // arena part holding fp32 images
  size_t arena_need = 0;    // total (fp32 + worst-case tensor-core images)
  char* arena = nullptr;
  size_t arena_bytes = 0;
  bool finalized = false;
  int precision = AB_PREC_FP32;
  int hop = 1;
  int launches = 0;
  int rb_mode = 2;          // "resblock_fusion" option
  std::vector<cudaEvent_t> tail_events;   // ab_generator_set_tail_events: consumed by the next forward
  int64_t source_frames = 0;              // NSF-HiFiGAN: frames of the f0 track of the next forward (0 = covers the mel)

  std::unordered_map<int, SnakeCoef> act_coef;   // by up-filter slot: host copy of the 12+12 taps, packed (finalize)

  ConvRef conv_pre, conv_post;
  int cond_w = -1, cond_b = -1;   // HiFiGAN_vits global conditioning (hifigan.py:424-425)
  ActRef act_post;
  std::vector<StageRef> stages;

  // profiling (ab_generator_set_profiling)
  bool profiling = false;
  struct ProfRec { int cls; cudaEvent_t e0, e1; double flops, bytes; };
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> event_pool;
  cudaEvent_t get_event() {
    if (!event_pool.empty()) { cudaEvent_t e = event_pool.back(); event_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
  }
  ~ab_generator() {
    for (auto& r : prof_recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    for (auto e : event_pool) cudaEventDestroy(e);
  }

  int add_slot(const std::string& name, SlotKind kind, std::initializer_list<int64_t> shape) {
    Slot s;
    s.name = name;
    s.kind = kind;
    s.ndim = (int)shape.size();
    size_t n = 1;
    int i = 0;
    for (auto v : shape) {
      s.shape[i++] = v;
      n *= (size_t)v;
    }
    s.offset = fp32_bytes;
    s.bytes = n * sizeof(float);
    s.loaded = false;
    s.tc_offset = 0;
    s.tc_bytes = 0;
    s.stride = 1;
    s.dilation = 1;
    fp32_bytes += align_up(s.bytes, 256);
    slots.push_back(s);
    index[name] = (int)slots.size() - 1;
    return (int)slots.size() - 1;
  }
  float* fptr(int slot) const { return slot < 0 ? nullptr : reinterpret_cast<float*>(arena + slots[slot].offset); }
  void* tcptr(int slot) const { return arena + slots[slot].tc_offset; }
};

namespace {

ConvRef make_conv(ab_generator* g, const std::string& name, int cin, int cout, int k, int d, bool transposed,
                  bool has_bias = true) {
  ConvRef c;
  c.cin = cin;
  c.cout = cout;
  c.k = k;
  c.d = d;
  if (transposed)
    c.w = g->add_slot(name + ".weight", SLOT_CONVT_W, {cin, cout, k});
  else
    c.w = g->add_slot(name + ".weight", SLOT_CONV_W, {cout, cin, k});
  g->slots[c.w].dilation = d;
  c.b = has_bias ? g->add_slot(name + ".bias", SLOT_VEC, {cout}) : -1;
  return c;
}

ActRef make_act(ab_generator* g, const std::string& prefix, int ch, bool has_beta) {
  ActRef a;
  a.alpha = g->add_slot(prefix + ".act.alpha", SLOT_VEC, {ch});
  a.beta = has_beta ? g->add_slot(prefix + ".act.beta", SLOT_VEC, {ch}) : a.alpha;
  a.fup = g->add_slot(prefix + ".upsample.filter", SLOT_VEC, {1, 1, 12});
  a.fdown = g->add_slot(prefix + ".downsample.lowpass.filter", SLOT_VEC, {1, 1, 12});
  return a;
}

int validate_config(const ab_generator_config& c) {
  if (c.kind != AB_GEN_HIFIGAN && c.kind != AB_GEN_BIGVGAN && c.kind != AB_GEN_NSFHIFIGAN && c.kind != AB_GEN_TRUNK)
    return fail(AB_ERR_ARG, "config: unknown generator kind %d", c.kind);
  const bool trunk = c.kind == AB_GEN_TRUNK;
  if (trunk) {
    if (c.num_upsamples != 0) return fail(AB_ERR_ARG, "config: a trunk has no upsampling stages");
    if (c.trunk_out_channels <= 0 || c.trunk_out_channels > 65536) return fail(AB_ERR_ARG, "config: trunk_out_channels %d out of range", c.trunk_out_channels);
    if (c.trunk_in_kernel <= 0 || !(c.trunk_in_kernel & 1) || c.trunk_out_kernel <= 0 || !(c.trunk_out_kernel & 1))
      return fail(AB_ERR_UNSUPPORTED, "config: trunk conv kernels must be odd (got %d, %d)", c.trunk_in_kernel, c.trunk_out_kernel);
    if (c.resblock != 1) return fail(AB_ERR_UNSUPPORTED, "config: the trunk uses ResBlock1 blocks (apnet.py:113-278)");
  } else if (c.trunk_out_channels || c.trunk_in_kernel || c.trunk_out_kernel) {
    return fail(AB_ERR_ARG, "config: trunk_* fields belong to AB_GEN_TRUNK");
  }
  if (c.n_mel <= 0 || c.upsample_initial_channel <= 0) return fail(AB_ERR_ARG, "config: n_mel / upsample_initial_channel must be positive");
  if ((!trunk && c.num_upsamples <= 0) || c.num_upsamples > AB_MAX_STAGES) return fail(AB_ERR_ARG, "config: num_upsamples %d out of range", c.num_upsamples);
  if (c.num_kernels <= 0 || c.num_kernels > AB_MAX_KERNELS) return fail(AB_ERR_ARG, "config: num_kernels %d out of range", c.num_kernels);
  if (c.resblock != 1 && c.resblock != 2) return fail(AB_ERR_ARG, "config: resblock must be 1 or 2");
  if ((c.upsample_initial_channel >> c.num_upsamples) <= 0) return fail(AB_ERR_ARG, "config: upsample_initial_channel too small for %d stages", c.num_upsamples);
  for (int i = 0; i < c.num_upsamples; ++i) {
    const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i];
    if (u <= 0 || k < u || ((k - u) & 1)) return fail(AB_ERR_UNSUPPORTED, "config: stage %d: kernel %d / rate %d (need k >= u, k-u even)", i, k, u);
  }
  for (int j = 0; j < c.num_kernels; ++j) {
    if (c.num_dilations[j] <= 0 || c.num_dilations[j] > AB_MAX_DILATIONS) return fail(AB_ERR_ARG, "config: num_dilations[%d] out of range", j);
    const int k = c.resblock_kernel_sizes[j];
    if (k <= 0 || !(k & 1)) return fail(AB_ERR_UNSUPPORTED, "config: resblock kernel size %d must be odd", k);
    for (int p = 0; p < c.num_dilations[j]; ++p)
      if (c.resblock_dilation_sizes[j][p] <= 0) return fail(AB_ERR_ARG, "config: dilation must be positive");
  }
  if (c.kind == AB_GEN_BIGVGAN && c.activation != AB_ACT_SNAKE && c.activation != AB_ACT_SNAKEBETA)
    return fail(AB_ERR_ARG, "config: BigVGAN activation must be snake or snakebeta");
  if (c.gin_channels < 0 || c.gin_channels > 65536) return fail(AB_ERR_ARG, "config: gin_channels %d out of range", c.gin_channels);
  if ((c.gin_channels > 0 || c.conv_post_no_bias) && c.kind != AB_GEN_HIFIGAN)
    return fail(AB_ERR_ARG, "config: gin_channels / conv_post_no_bias belong to the HiFi-GAN kind (HiFiGAN_vits)");
  return AB_OK;
}

// Routing at tensor-core precision: the size of the slot's 16-bit weight image, 0 when its conv runs on the fp32
// CUDA-core kernels instead of the wgmma kernel.
//   ConvTranspose1d and the (square) ResBlock / AMPBlock convs run on the wgmma kernel whenever the shape has an
//   image; a block of tc_conv_supported convs (C <= 256, k <= 31) runs as pairs or whole blocks, any other as single
//   convs.  conv_pre / conv_post run there iff C_in != C_out, C_in <= 512 and C_out > 4: the C -> 1 conv_post is
//   HBM-bound and the last layer, so it stays exact.
size_t tc_image_bytes(const Slot& s, bool pre_or_post) {
  if (s.kind == SLOT_CONVT_W) return tc_weight_image_bytes(1, (int)s.shape[0], (int)s.shape[1], (int)s.shape[2], s.stride);
  if (s.kind != SLOT_CONV_W) return 0;
  const int cout = (int)s.shape[0], cin = (int)s.shape[1], k = (int)s.shape[2];
  if (pre_or_post && (cin == cout || cin > 512 || cout <= 4)) return 0;
  return tc_weight_image_bytes(0, cin, cout, k, s.dilation);
}

}  // namespace

extern "C" {

const char* ab_last_error(void) { return g_err; }
int ab_version(void) { return 100; }

int ab_device_is_sm90(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9;
}

int ab_generator_create(const ab_generator_config* cfg, ab_generator** out) {
  if (!cfg || !out) return fail(AB_ERR_ARG, "ab_generator_create: null argument");
  int rc = validate_config(*cfg);
  if (rc != AB_OK) return rc;
  ab_generator* g = new ab_generator();
  g->cfg = *cfg;
  const bool big = cfg->kind == AB_GEN_BIGVGAN;
  const bool has_beta = cfg->activation == AB_ACT_SNAKEBETA;
  const int c0 = cfg->upsample_initial_channel;
  const bool trunk = cfg->kind == AB_GEN_TRUNK;
  g->conv_pre = make_conv(g, "conv_pre", cfg->n_mel, c0, trunk ? cfg->trunk_in_kernel : 7, 1, false);
  g->hop = 1;
  int ch = c0;
  if (trunk) {   // one stage at the input rate: no transposed conv, the ResBlock branches read conv_pre's output
    StageRef st;
    st.ch = c0;
    st.u = 1;
    st.has_up = false;
    for (int j = 0; j < cfg->num_kernels; ++j) {
      BlockRef blk;
      blk.k = cfg->resblock_kernel_sizes[j];
      const std::string pre = "resblocks." + std::to_string(j);
      for (int p = 0; p < cfg->num_dilations[j]; ++p) {
        const int d = cfg->resblock_dilation_sizes[j][p];
        blk.dil.push_back(d);
        blk.c1.push_back(make_conv(g, pre + ".convs1." + std::to_string(p), ch, ch, blk.k, d, false));
        blk.c2.push_back(make_conv(g, pre + ".convs2." + std::to_string(p), ch, ch, blk.k, 1, false));
      }
      st.blocks.push_back(blk);
    }
    g->stages.push_back(st);
  }
  for (int i = 0; i < cfg->num_upsamples; ++i) {
    StageRef st;
    const int cin = c0 >> i;
    ch = c0 >> (i + 1);
    st.ch = ch;
    st.u = cfg->upsample_rates[i];
    g->hop *= st.u;
    // BigVGAN wraps each transposed conv in a ModuleList: key "ups.{i}.0" (bigvgan.py:254-276)
    const std::string upname = "ups." + std::to_string(i) + (big ? ".0" : "");
    st.up = make_conv(g, upname, cin, ch, cfg->upsample_kernel_sizes[i], 1, true);
    g->slots[st.up.w].stride = st.u;
    if (cfg->kind == AB_GEN_NSFHIFIGAN) g->slots[st.up.w].gain = g->slots[st.up.b].gain = 2.0f;   // x = x + x (:269-271)
    for (int j = 0; j < cfg->num_kernels; ++j) {
      BlockRef blk;
      blk.k = cfg->resblock_kernel_sizes[j];
      const std::string pre = "resblocks." + std::to_string(i * cfg->num_kernels + j);
      for (int p = 0; p < cfg->num_dilations[j]; ++p) {
        const int d = cfg->resblock_dilation_sizes[j][p];
        blk.dil.push_back(d);
        if (cfg->resblock == 1) {
          blk.c1.push_back(make_conv(g, pre + ".convs1." + std::to_string(p), ch, ch, blk.k, d, false));
          blk.c2.push_back(make_conv(g, pre + ".convs2." + std::to_string(p), ch, ch, blk.k, 1, false));
        } else {
          blk.c1.push_back(make_conv(g, pre + ".convs." + std::to_string(p), ch, ch, blk.k, d, false));
        }
      }
      if (big) {
        const int na = cfg->resblock == 1 ? 2 * cfg->num_dilations[j] : cfg->num_dilations[j];
        for (int a = 0; a < na; ++a)
          blk.acts.push_back(make_act(g, pre + ".activations." + std::to_string(a), ch, has_beta));
      }
      st.blocks.push_back(blk);
    }
    g->stages.push_back(st);
  }
  if (big) g->act_post = make_act(g, "activation_post", ch, has_beta);
  g->conv_post = make_conv(g, "conv_post", ch, trunk ? cfg->trunk_out_channels : 1, trunk ? cfg->trunk_out_kernel : 7, 1, false,
                           !cfg->conv_post_no_bias);
  if (cfg->gin_channels > 0) {
    g->cond_w = g->add_slot("cond.weight", SLOT_VEC, {c0, cfg->gin_channels, 1});
    g->cond_b = g->add_slot("cond.bias", SLOT_VEC, {c0});
  }

  // tensor-core weight images live behind the fp32 images
  size_t tc = 0;
  for (size_t i = 0; i < g->slots.size(); ++i) {
    Slot& s = g->slots[i];
    s.tc_bytes = tc_image_bytes(s, (int)i == g->conv_pre.w || (int)i == g->conv_post.w);
    s.tc_offset = g->fp32_bytes + tc;
    tc += align_up(s.tc_bytes, 256);
  }
  g->arena_need = g->fp32_bytes + tc;
  *out = g;
  return AB_OK;
}

void ab_generator_destroy(ab_generator* g) { delete g; }

size_t ab_generator_param_bytes(const ab_generator* g) { return g ? g->arena_need : 0; }

int ab_generator_bind_params(ab_generator* g, void* dev_arena, size_t bytes) {
  if (!g || !dev_arena) return fail(AB_ERR_ARG, "bind_params: null argument");
  if (bytes < g->arena_need) return fail(AB_ERR_WORKSPACE, "bind_params: arena %zu B < required %zu B", bytes, g->arena_need);
  if (reinterpret_cast<uintptr_t>(dev_arena) & 255) return fail(AB_ERR_ARG, "bind_params: arena must be 256-byte aligned");
  g->arena = static_cast<char*>(dev_arena);
  g->arena_bytes = bytes;
  g->finalized = false;
  for (auto& s : g->slots) s.loaded = false;
  return AB_OK;
}

int ab_generator_num_tensors(const ab_generator* g) { return g ? (int)g->slots.size() : 0; }

const char* ab_generator_tensor_name(const ab_generator* g, int i) {
  if (!g || i < 0 || i >= (int)g->slots.size()) return nullptr;
  return g->slots[i].name.c_str();
}

static int load_common(ab_generator* g, const char* name, const float* dev_g, const float* dev_v,
                       const int64_t* shape, int32_t ndim, void* stream) {
  if (!g || !name || !dev_v || !shape) return fail(AB_ERR_ARG, "load_tensor: null argument");
  if (!g->arena) return fail(AB_ERR_STATE, "load_tensor: bind_params first");
  auto it = g->index.find(name);
  if (it == g->index.end()) return fail(AB_ERR_ARG, "load_tensor: unknown tensor '%s'", name);
  Slot& s = g->slots[it->second];
  size_t n_ref = 1, n_in = 1;
  for (int i = 0; i < s.ndim; ++i) n_ref *= (size_t)s.shape[i];
  for (int i = 0; i < ndim; ++i) n_in *= (size_t)shape[i];
  bool same = ndim == s.ndim;
  for (int i = 0; same && i < ndim; ++i) same = shape[i] == s.shape[i];
  // vectors may come with any shape of the right size (e.g. filter [1,1,12] or [12])
  if (!(same || (s.kind == SLOT_VEC && n_in == n_ref)))
    return fail(AB_ERR_ARG, "load_tensor: '%s' has the wrong shape (%d dims, %zu elements; expected %zu)", name, ndim, n_in, n_ref);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* dst = g->fptr(it->second);
  if (s.kind == SLOT_VEC) {
    if (dev_g) return fail(AB_ERR_ARG, "load_weight_norm: '%s' is not a convolution weight", name);
    AB_CUDA_TRY(cudaMemcpyAsync(dst, dev_v, s.bytes, cudaMemcpyDeviceToDevice, st));
  } else {
    int rc = launch_repack_weight(dev_v, dev_g, dst, (int)s.shape[0], (int)s.shape[1], (int)s.shape[2],
                                  s.kind == SLOT_CONVT_W ? 1 : 0, st);
    if (rc != AB_OK) return rc;
  }
  if (s.gain != 1.0f) {
    int rc = launch_scale_inplace(dst, s.bytes / sizeof(float), s.gain, st);
    if (rc != AB_OK) return rc;
  }
  s.loaded = true;
  g->finalized = false;
  return AB_OK;
}

int ab_generator_load_tensor(ab_generator* g, const char* name, const float* dev_src,
                             const int64_t* shape, int32_t ndim, void* stream) {
  return load_common(g, name, nullptr, dev_src, shape, ndim, stream);
}

int ab_generator_load_weight_norm(ab_generator* g, const char* name, const float* dev_g,
                                  const float* dev_v, const int64_t* shape, int32_t ndim, void* stream) {
  if (!dev_g) return fail(AB_ERR_ARG, "load_weight_norm: null weight_g");
  return load_common(g, name, dev_g, dev_v, shape, ndim, stream);
}

int ab_generator_finalize(ab_generator* g, int32_t precision, void* stream) {
  if (!g) return fail(AB_ERR_ARG, "finalize: null handle");
  if (!g->arena) return fail(AB_ERR_STATE, "finalize: bind_params first");
  for (auto& s : g->slots)
    if (!s.loaded) return fail(AB_ERR_STATE, "finalize: tensor '%s' was never loaded", s.name.c_str());
  if (precision != AB_PREC_FP32 && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "finalize: unknown precision %d", precision);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (precision != AB_PREC_FP32) {
    if (!ab_device_is_sm90()) return fail(AB_ERR_UNSUPPORTED, "finalize: tensor-core precision needs an sm_90 (Hopper) device");
    for (size_t i = 0; i < g->slots.size(); ++i) {
      const Slot& s = g->slots[i];
      if (!s.tc_bytes) continue;
      const bool t = s.kind == SLOT_CONVT_W;   // state-dict shape: ConvTranspose1d [C_in, C_out, k], Conv1d [C_out, C_in, k]
      int rc = launch_tc_pack_weight(g->fptr((int)i), g->tcptr((int)i), t ? 1 : 0, (int)s.shape[t ? 0 : 1],
                                     (int)s.shape[t ? 1 : 0], (int)s.shape[2], t ? s.stride : s.dilation, precision, st);
      if (rc != AB_OK) return rc;
    }
  }
  // Activation1d taps: 24 floats per activation go to the host once, so that every later launch carries them by value
  // (uniform-register operands of the packed FMAs).  The only synchronising step of the handle's life.
  g->act_coef.clear();
  {
    const std::string up_suffix = ".upsample.filter";
    std::vector<int> ups;
    for (size_t i = 0; i + 1 < g->slots.size(); ++i) {
      const std::string& n = g->slots[i].name;
      if (n.size() > up_suffix.size() && n.compare(n.size() - up_suffix.size(), up_suffix.size(), up_suffix) == 0) ups.push_back((int)i);
    }
    std::vector<float> host(ups.size() * 24);
    for (size_t j = 0; j < ups.size(); ++j) {     // make_act: the down filter is the slot after the up filter
      if (cudaMemcpyAsync(&host[j * 24], g->fptr(ups[j]), 12 * sizeof(float), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
          cudaMemcpyAsync(&host[j * 24 + 12], g->fptr(ups[j] + 1), 12 * sizeof(float), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return fail(AB_ERR_CUDA, "finalize: reading the anti-aliasing filters failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    if (!ups.empty()) {
      if (cudaStreamSynchronize(st) != cudaSuccess)
        return fail(AB_ERR_CUDA, "finalize: %s", cudaGetErrorString(cudaGetLastError()));
      for (size_t j = 0; j < ups.size(); ++j) pack_snake_coef(&host[j * 24], &host[j * 24 + 12], &g->act_coef[ups[j]]);
    }
  }
  g->precision = precision;
  g->finalized = true;
  return AB_OK;
}

// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
namespace {
constexpr int NBUF = 7;  // fp32: R0 R1 U P0 P1 TMP ACT
constexpr int NIMG = 4;  // 16-bit operand images: U P0 P1 R (stage output, HiFi-GAN)

size_t stage_max_image_bytes(const ab_generator* g, int64_t B, int64_t T) {
  size_t mx = 0;
  int64_t t = T;
  for (auto& st : g->stages) {
    t *= st.u;
    mx = std::max(mx, tc_act_image_bytes(B, st.ch, t));
  }
  return mx;
}

size_t stage_max_elems(const ab_generator* g, int64_t B, int64_t T) {
  size_t mx = (size_t)B * g->cfg.upsample_initial_channel * T;
  int64_t t = T;
  for (auto& st : g->stages) {
    t *= st.u;
    mx = std::max(mx, (size_t)B * st.ch * t);
  }
  return mx;
}
}  // namespace

// NSF-HiFiGAN: length of stage i's output after `length = min(x.shape[-1], x_source.shape[-1])` (nsfhifigan.py:264-268).
// noise_convs[i] = Conv1d(1, C, 2s, stride s, padding s/2), s = prod(rates[i+1:]) (:223-236; kernel 1 for the last stage),
// applied to a source of source_frames * prod(rates) samples; Tn = length of the stage's transposed-conv output.
static int64_t nsf_stage_length(const ab_generator* g, int stage, int64_t Tn, int64_t source_frames) {
  if (g->cfg.kind != AB_GEN_NSFHIFIGAN || source_frames <= 0) return Tn;
  int64_t upp = 1, sfac = 1;
  for (int j = 0; j < g->cfg.num_upsamples; ++j) upp *= g->cfg.upsample_rates[j];
  for (int j = stage + 1; j < g->cfg.num_upsamples; ++j) sfac *= g->cfg.upsample_rates[j];
  const int64_t src = source_frames * upp;
  const int64_t xs = stage + 1 < g->cfg.num_upsamples ? (src + 2 * (sfac / 2) - 2 * sfac) / sfac + 1 : src;
  return std::max<int64_t>(std::min(Tn, xs), 0);
}

size_t ab_generator_workspace_bytes(const ab_generator* g, int64_t B, int64_t T) {
  if (!g || B <= 0 || T <= 0) return 0;
  return NBUF * align_up(stage_max_elems(g, B, T) * sizeof(float), 256) +
         NIMG * align_up(stage_max_image_bytes(g, B, T), 256);
}

int ab_generator_last_launches(const ab_generator* g) { return g ? g->launches : 0; }

int ab_generator_set_profiling(ab_generator* g, int32_t enable) {
  if (!g) return fail(AB_ERR_ARG, "set_profiling: null handle");
  g->profiling = enable != 0;
  return AB_OK;
}

int ab_generator_set_tail_events(ab_generator* g, void* const* events, int32_t n) {
  if (!g || n < 0 || (n > 0 && !events)) return fail(AB_ERR_ARG, "set_tail_events: bad argument");
  g->tail_events.clear();
  for (int i = 0; i < n; ++i) {
    if (!events[i]) return fail(AB_ERR_ARG, "set_tail_events: null event %d", i);
    g->tail_events.push_back(static_cast<cudaEvent_t>(events[i]));
  }
  return AB_OK;
}

int64_t ab_generator_output_samples(const ab_generator* g, int64_t frames, int64_t source_frames) {
  if (!g || frames <= 0) return 0;
  int64_t Tn = frames;
  for (int i = 0; i < g->cfg.num_upsamples; ++i) Tn = nsf_stage_length(g, i, Tn * g->cfg.upsample_rates[i], source_frames);
  return Tn;
}

int ab_generator_set_option(ab_generator* g, const char* key, int32_t value) {
  if (!g || !key) return fail(AB_ERR_ARG, "set_option: null argument");
  if (strcmp(key, "nsf_source_frames") == 0) {   // one-shot: consumed by the next forward
    if (value < 0) return fail(AB_ERR_ARG, "set_option: nsf_source_frames must be >= 0");
    if (value > 0 && g->cfg.kind != AB_GEN_NSFHIFIGAN) return fail(AB_ERR_ARG, "set_option: nsf_source_frames belongs to NSF-HiFiGAN");
    g->source_frames = value;
    return AB_OK;
  }
  if (strcmp(key, "resblock_fusion") == 0) {
    if (value < 0 || value > 4) return fail(AB_ERR_ARG, "set_option: resblock_fusion must be 0..4 (got %d)", value);
    g->rb_mode = value;
    return AB_OK;
  }
  return fail(AB_ERR_ARG, "set_option: unknown key '%s'", key);
}

int ab_generator_get_profile(ab_generator* g, ab_profile_entry* out, int32_t max_entries, int32_t* n_out) {
  if (!g || !out || !n_out) return fail(AB_ERR_ARG, "get_profile: null argument");
  static const char* kNames[5] = {"tc_conv", "conv1d_fp32", "conv_transpose1d_fp32", "activation1d", "tc_gemmconv"};
  if (max_entries < 5) return fail(AB_ERR_ARG, "get_profile: need room for 5 entries");
  for (int i = 0; i < 5; ++i) {
    memset(&out[i], 0, sizeof(out[i]));
    strncpy(out[i].name, kNames[i], sizeof(out[i].name) - 1);
  }
  for (auto& r : g->prof_recs) {
    AB_CUDA_TRY(cudaEventSynchronize(r.e1));
    float ms = 0.f;
    AB_CUDA_TRY(cudaEventElapsedTime(&ms, r.e0, r.e1));
    out[r.cls].launches += 1;
    out[r.cls].ms += ms;
    out[r.cls].flops += r.flops;
    out[r.cls].bytes += r.bytes;
    g->event_pool.push_back(r.e0);
    g->event_pool.push_back(r.e1);
  }
  g->prof_recs.clear();
  *n_out = 5;
  return AB_OK;
}


// block mode (resblock_fusion 2) is chosen when it computes at most this many tile rows per output row
static constexpr double kChainMaxRecompute = 1.5;

static int forward_impl(ab_generator* g, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3],
                        const float* dev_g, int64_t g_batch_stride, float* dev_wav, void* dev_workspace,
                        size_t workspace_bytes, void* stream) {
  if (!g || !dev_mel || !dev_wav || !mel_strides) return fail(AB_ERR_ARG, "forward: null argument");
  if (dev_g != nullptr && g->cond_w < 0) return fail(AB_ERR_STATE, "forward: conditioning given but the generator has gin_channels == 0");
  if (dev_g != nullptr && g_batch_stride < g->cfg.gin_channels) return fail(AB_ERR_ARG, "forward: g row stride < gin_channels");
  if (!g->finalized) return fail(AB_ERR_STATE, "forward: finalize() the generator first");
  if (B <= 0 || T <= 0) return fail(AB_ERR_ARG, "forward: batch and frames must be positive (got %lld, %lld)", (long long)B, (long long)T);
  if (B > 65535) return fail(AB_ERR_UNSUPPORTED, "forward: batch %lld > 65535", (long long)B);
  if ((int64_t)T * g->hop > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "forward: sequence too long");
  const size_t need = ab_generator_workspace_bytes(g, B, T);
  if (!dev_workspace || workspace_bytes < need) return fail(AB_ERR_WORKSPACE, "forward: workspace %zu B < required %zu B", workspace_bytes, need);
  if (reinterpret_cast<uintptr_t>(dev_workspace) & 255) return fail(AB_ERR_ARG, "forward: workspace must be 256-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bufsz = align_up(stage_max_elems(g, B, T) * sizeof(float), 256);
  const size_t imgsz = align_up(stage_max_image_bytes(g, B, T), 256);
  float* buf[NBUF];
  for (int i = 0; i < NBUF; ++i) buf[i] = reinterpret_cast<float*>(static_cast<char*>(dev_workspace) + i * bufsz);
  uint16_t* img[NIMG];
  for (int i = 0; i < NIMG; ++i)
    img[i] = reinterpret_cast<uint16_t*>(static_cast<char*>(dev_workspace) + NBUF * bufsz + i * imgsz);
  uint16_t *U16 = img[0], *P16[2] = {img[1], img[2]}, *R16 = img[3];
  const uint16_t* r_img = nullptr;   // operand image of lrelu(stage input, 0.1) when the previous stage emitted it
  float *R[2] = {buf[0], buf[1]}, *U = buf[2], *P[2] = {buf[3], buf[4]}, *TMP = buf[5], *ACT = buf[6];
  const bool big = g->cfg.kind == AB_GEN_BIGVGAN;
  const bool tc = g->precision != AB_PREC_FP32;
  const int nk = g->cfg.num_kernels;
  int launches = 0;
  int rc;
  // optional per-launch device timing
  auto prof_begin = [&](int cls, double flops, double bytes) {
    if (!g->profiling) return;
    ab_generator::ProfRec r;
    r.cls = cls; r.flops = flops; r.bytes = bytes;
    r.e0 = g->get_event(); r.e1 = g->get_event();
    cudaEventRecord(r.e0, st);
    g->prof_recs.push_back(r);
  };
  auto prof_end = [&]() {
    if (!g->profiling) return;
    cudaEventRecord(g->prof_recs.back().e1, st);
  };

  // algorithmic HBM bytes of a Conv1d launch with fp32 activations and weights (profile)
  auto conv_bytes = [&](const ConvRef& c, int Tn, const float* residual, const float* acc_prev) {
    const double el = (double)B * Tn;
    return 4.0 * (el * c.cin + el * c.cout * (1 + (residual != nullptr) + (acc_prev != nullptr)) + (double)c.cin * c.cout * c.k);
  };
  // fp32 CUDA-core Conv1d
  auto conv = [&](const ConvRef& c, const float* x, int64_t xsb, int64_t xsc, int64_t xst, float* y,
                  int Tn, float pre_slope, const float* residual, const float* acc_prev, float out_div,
                  int post_tanh) -> int {
    ConvParams p;
    p.x = x; p.xsb = xsb; p.xsc = xsc; p.xst = xst;
    p.w_t = g->fptr(c.w); p.bias = g->fptr(c.b);
    p.residual = residual; p.acc_prev = acc_prev; p.y = y;
    p.B = (int)B; p.Cin = c.cin; p.Cout = c.cout; p.T = Tn; p.k = c.k; p.d = c.d;
    p.pre_slope = pre_slope; p.out_div = out_div; p.post_tanh = post_tanh;
    ++launches;
    prof_begin(1, 2.0 * B * Tn * c.cout * c.cin * c.k, conv_bytes(c, Tn, residual, acc_prev));
    const int r = launch_conv1d_fp32(p, st);
    prof_end();
    return r;
  };
  // whether conv c runs on the wgmma kernel (tc_image_bytes decided it at create)
  auto on_tc = [&](const ConvRef& c) { return tc && g->slots[c.w].tc_bytes > 0; };
  // Conv1d c on the wgmma kernel, from fp32 x (lrelu(., pre_slope) in the loader) or the operand image ximg; with c2
  // the ResBlock1 pair c -> lrelu(., pre_slope) -> c2 in one launch.  bytes: the launch's algorithmic HBM bytes (profile)
  auto tc_conv = [&](const ConvRef& c, const ConvRef* c2, const float* x, int64_t xsb, int64_t xsc, int64_t xst,
                     const uint16_t* ximg, float* y, uint16_t* yimg, int Tn, float pre_slope, const float* residual,
                     const float* acc_prev, float out_div, int post_tanh, double bytes) -> int {
    TcConvParams p;
    p.x = x; p.xsb = xsb; p.xsc = xsc; p.xst = xst; p.ximg = ximg; p.pre_slope = pre_slope;
    p.w = g->tcptr(c.w); p.bias = g->fptr(c.b);
    if (c2) { p.w2 = g->tcptr(c2->w); p.b2 = g->fptr(c2->b); p.mid_slope = pre_slope; }
    p.residual = residual; p.acc_prev = acc_prev; p.out_div = out_div; p.post_tanh = post_tanh;
    p.y = y; p.yimg = yimg; p.img_slope = 0.1f;
    p.B = (int)B; p.Cin = c.cin; p.Cout = c.cout; p.T = Tn; p.k = c.k; p.d_or_u = c.d;
    p.precision = g->precision;
    ++launches;
    const bool rb = c.cin == c.cout && tc_conv_supported(c.cin, c.k);   // pair / block-mode capable ResBlock conv
    prof_begin(rb ? 0 : 4, 2.0 * B * Tn * c.cout * c.cin * c.k * (c2 ? 2 : 1), bytes);
    const int r = launch_tc_conv(p, st);
    prof_end();
    return r;
  };
  auto snake = [&](const ActRef& a, const float* x, float* y, int C, int Tn, uint16_t* yimg = nullptr) -> int {
    SnakeParams p;
    p.yimg = yimg; p.bf16 = g->precision == AB_PREC_TC_BF16;
    p.x = x; p.y = y; p.alpha = g->fptr(a.alpha); p.beta = g->fptr(a.beta);
    p.f_up = g->fptr(a.fup); p.f_down = g->fptr(a.fdown);
    auto kc = g->act_coef.find(a.fup);
    if (kc != g->act_coef.end()) { p.kc = kc->second; p.have_kc = 1; }
    p.fast_snake = g->precision != AB_PREC_FP32;
    p.B = (int)B; p.C = C; p.T = Tn; p.logscale = g->cfg.snake_logscale;
    ++launches;
    prof_begin(3, 0.0, (double)B * C * Tn * (4.0 + (y ? 4.0 : 0.0) + (yimg ? 2.0 : 0.0)));
    const int r = launch_activation1d(p, st);
    prof_end();
    return r;
  };
  // conv_pre (hifigan.py:204, bigvgan.py:314)
  const int C0 = g->cfg.upsample_initial_channel;
  const ConvRef& cpre = g->conv_pre;
  rc = on_tc(cpre) ? tc_conv(cpre, nullptr, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], nullptr, R[0], nullptr,
                             (int)T, 1.0f, nullptr, nullptr, 1.0f, 0, conv_bytes(cpre, (int)T, nullptr, nullptr))
                   : conv(cpre, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], R[0], (int)T, 1.0f,
                          nullptr, nullptr, 1.0f, 0);
  if (rc != AB_OK) return rc;
  if (dev_g != nullptr) {   // x = x + cond(g)  (hifigan.py:429-430)
    ++launches;
    rc = launch_cond_add(R[0], dev_g, g_batch_stride, g->fptr(g->cond_w), g->fptr(g->cond_b), (int)B, C0,
                         g->cfg.gin_channels, (int)T, st);
    if (rc != AB_OK) return rc;
  }
  int cur_r = 0;
  int Tn = (int)T;
  int cin = C0;
  for (size_t i = 0; i < g->stages.size(); ++i) {
    const StageRef& sg = g->stages[i];
    // x = leaky_relu(x, 0.1) (HiFi-GAN only) ; x = ups[i](x)   (hifigan.py:206-207, bigvgan.py:316-318)
    uint16_t* u_img = nullptr;
    if (!sg.has_up) {
      std::swap(U, R[cur_r]);   // AB_GEN_TRUNK: the blocks read conv_pre's output in place
    } else {
      const bool up_tc = on_tc(sg.up);
      const float pre_slope = big ? 1.0f : 0.1f;
      ++launches;
      const double eo = (double)B * sg.ch * Tn * sg.u;
      prof_begin(up_tc ? 4 : 2, 2.0 * eo * cin * ((double)sg.up.k / sg.u),
                 4.0 * ((double)B * cin * Tn + eo + (double)cin * sg.ch * sg.up.k));
      if (up_tc) {
        TcConvParams p;
        p.mode = 1;
        p.x = R[cur_r]; p.xsb = (int64_t)cin * Tn; p.xsc = Tn; p.xst = 1; p.pre_slope = pre_slope;
        p.ximg = (r_img != nullptr && (cin % 16) == 0) ? r_img : nullptr;
        p.w = g->tcptr(sg.up.w); p.bias = g->fptr(sg.up.b); p.y = U;
        // HiFi-GAN: every consumer of U applies lrelu(., 0.1) first (hifigan.py:95) -> emit that operand image
        u_img = (!big && tc_can_emit_image(1, cin, sg.ch, sg.up.k, sg.u)) ? U16 : nullptr;
        p.yimg = u_img; p.img_slope = 0.1f;
        p.B = (int)B; p.Cin = cin; p.Cout = sg.ch; p.T = Tn; p.k = sg.up.k; p.d_or_u = sg.u; p.precision = g->precision;
        rc = launch_tc_conv(p, st);
      } else {
        ConvTParams tp;
        tp.x = R[cur_r]; tp.w_t = g->fptr(sg.up.w); tp.bias = g->fptr(sg.up.b); tp.y = U;
        tp.B = (int)B; tp.Cin = cin; tp.Cout = sg.ch; tp.Tin = Tn; tp.k = sg.up.k; tp.u = sg.u; tp.pre_slope = pre_slope;
        rc = launch_conv_transpose1d_fp32(tp, st);
      }
      prof_end();
      if (rc != AB_OK) return rc;
    }
    Tn *= sg.u;
    const int C = sg.ch;
    {
      // NSF-HiFiGAN with a source shorter than this stage (short f0, odd source stride): the reference truncates x
      // to the source length before the ResBlocks (nsfhifigan.py:264-268).  Compact the rows; the operand image
      // (laid out for the untruncated length) is dropped for this stage.
      const int64_t Lt = nsf_stage_length(g, (int)i, Tn, g->source_frames);
      if (Lt < Tn) {
        if (Lt <= 0) return fail(AB_ERR_ARG, "forward: the f0 track leaves no samples in stage %d", (int)i);
        AB_CUDA_TRY(cudaMemcpy2DAsync(TMP, (size_t)Lt * sizeof(float), U, (size_t)Tn * sizeof(float), (size_t)Lt * sizeof(float),
                                      (size_t)B * C, cudaMemcpyDeviceToDevice, st));
        std::swap(U, TMP);
        u_img = nullptr;
        Tn = (int)Lt;
      }
    }
    float* Rout = R[cur_r ^ 1];
    const int64_t sb = (int64_t)C * Tn, sc = Tn;
    bool stage_img_written = false;
    for (int j = 0; j < nk; ++j) {
      const BlockRef& blk = sg.blocks[j];
      const float* cur = U;
      const uint16_t* cur_img = u_img;
      int pp = 0;
      const int nd = (int)blk.dil.size();
      const bool pair = !blk.c2.empty();
      const int ncv = pair ? 2 : 1;
      // every conv of a block has a weight image or none; fused: pair / block mode (HiFi-GAN) and tc_conv launch class
      const bool blk_tc = on_tc(blk.c1[0]);
      const bool fused = blk_tc && tc_conv_supported(C, blk.k);
      if (fused && !big && g->rb_mode >= 2 && nd <= AB_TC_CHAIN_MAX_PAIRS) {
        // whole block in one launch when the halo recompute costs less than the per-pair HBM round trips of x
        const double recompute = tc_chain_recompute(C, blk.k, blk.dil.data(), nd, ncv);
        if (recompute > 0.0 && (g->rb_mode >= 3 || recompute <= kChainMaxRecompute)) {
          const bool stage_img = j == nk - 1 && i + 1 < g->stages.size();
          TcChainParams cp;
          memset(&cp, 0, sizeof(cp));
          cp.x = U; cp.ximg = u_img; cp.y = Rout; cp.acc_prev = j > 0 ? Rout : nullptr;
          cp.yimg = stage_img ? R16 : nullptr;
          for (int q = 0; q < nd; ++q) {
            cp.dil[q] = blk.dil[q];
            cp.w[q * ncv] = g->tcptr(blk.c1[q].w);
            cp.bias[q * ncv] = g->fptr(blk.c1[q].b);
            if (ncv == 2) {
              cp.w[q * 2 + 1] = g->tcptr(blk.c2[q].w);
              cp.bias[q * 2 + 1] = g->fptr(blk.c2[q].b);
            }
          }
          cp.npairs = nd; cp.nconv = ncv; cp.B = (int)B; cp.C = C; cp.T = Tn; cp.k = blk.k;
          cp.slope = 0.1f; cp.img_slope = 0.1f; cp.out_div = j == nk - 1 ? (float)nk : 1.0f;
          cp.precision = g->precision;
          ++launches;
          const double el = (double)B * C * Tn;
          prof_begin(0, 2.0 * el * C * blk.k * ncv * nd, 4.0 * (el * (2 + (j > 0)) + (double)ncv * nd * C * C * blk.k));
          rc = launch_tc_chain(cp, st);
          prof_end();
          if (rc != AB_OK) return rc;
          if (stage_img) stage_img_written = true;
          continue;
        }
      }
      // algorithmic HBM bytes of one tensor-core launch (profile): a fused launch counts fp32 activations in and out,
      // a single conv of a wider or longer-kernel block a 16-bit input
      auto rb_bytes = [&](const ConvRef& c, int nconv, const float* x, const float* residual, const float* acc_prev) {
        const double el = (double)B * Tn;
        if (fused)
          return 4.0 * (el * C * (2 + (residual != nullptr && residual != x) + (acc_prev != nullptr)) + (double)nconv * C * C * c.k);
        return 4.0 * el * c.cout * (1 + (residual != nullptr) + (acc_prev != nullptr)) + 2.0 * el * c.cin + 4.0 * c.cin * c.cout * c.k;
      };
      // one conv: y = (c(act(x)) + residual + acc_prev) / out_div, act = the AMPBlock's anti-aliased snake
      // (bigvgan.py:137-146, :222-228; on tensor cores its kernel writes the 16-bit operand image only) or
      // lrelu(., 0.1) in the conv's loader (hifigan.py:95-99)
      auto single = [&](const ConvRef& c, const ActRef* a, const float* x, float* y, const float* residual,
                        const float* acc_prev, float out_div) -> int {
        const float* in = x;
        const uint16_t* img = nullptr;
        float slope = 0.1f;
        if (a) {
          img = blk_tc ? P16[0] : nullptr;
          in = blk_tc ? x : ACT;
          slope = 1.0f;
          const int r = blk_tc ? snake(*a, x, nullptr, C, Tn, P16[0]) : snake(*a, x, ACT, C, Tn);
          if (r != AB_OK) return r;
        }
        if (!blk_tc) return conv(c, in, sb, sc, 1, y, Tn, slope, residual, acc_prev, out_div, 0);
        return tc_conv(c, nullptr, in, sb, sc, 1, img, y, nullptr, Tn, slope, residual, acc_prev, out_div, 0,
                       rb_bytes(c, 1, x, residual, acc_prev));
      };
      for (int p = 0; p < nd; ++p) {
        const bool last = p == nd - 1;
        float* dst = last ? Rout : P[pp];
        uint16_t* dst_img = (last || big) ? nullptr : P16[pp];
        // the stage output feeds the next ConvTranspose through lrelu(., 0.1) (hifigan.py:206): emit that image
        const bool stage_img = last && j == nk - 1 && !big && i + 1 < g->stages.size();
        if (stage_img) dst_img = R16;
        if (!last) pp ^= 1;
        // xs = rb_0(x) ; xs += rb_j(x) ; x = xs / num_kernels  (hifigan.py:208-214)
        const float* accp = (last && j > 0) ? Rout : nullptr;
        const float div = (last && j == nk - 1) ? (float)nk : 1.0f;
        if (fused && !big) {
          rc = tc_conv(blk.c1[p], pair ? &blk.c2[p] : nullptr, cur, sb, sc, 1, cur_img, dst, dst_img, Tn, 0.1f, cur, accp,
                       div, 0, rb_bytes(blk.c1[p], ncv, cur, cur, accp));
          if (rc != AB_OK) return rc;
          cur_img = dst_img;
          if (stage_img) stage_img_written = true;
        } else if (pair) {
          rc = single(blk.c1[p], big ? &blk.acts[2 * p] : nullptr, cur, TMP, nullptr, nullptr, 1.0f);
          if (rc != AB_OK) return rc;
          rc = single(blk.c2[p], big ? &blk.acts[2 * p + 1] : nullptr, TMP, dst, cur, accp, div);
          if (rc != AB_OK) return rc;
          cur_img = nullptr;
        } else {
          rc = single(blk.c1[p], big ? &blk.acts[p] : nullptr, cur, dst, cur, accp, div);
          if (rc != AB_OK) return rc;
          cur_img = nullptr;
        }
        cur = dst;
      }
    }
    cur_r ^= 1;
    cin = C;
    r_img = stage_img_written ? R16 : nullptr;
  }
  // post: leaky_relu(x) with the DEFAULT slope 0.01 (hifigan.py:215) or
  // activation_post (bigvgan.py:327); conv_post; tanh
  const float* xin = R[cur_r];
  const int64_t sb = (int64_t)cin * Tn, sc = Tn;
  if (big) {
    rc = snake(g->act_post, xin, ACT, cin, Tn);
    if (rc != AB_OK) return rc;
    xin = ACT;
  }
  // conv_post in contiguous batch chunks, an event after each (ab_generator_set_tail_events): the caller's
  // final gather of chunk i then runs under conv_post of chunk i+1
  const int nchunk = g->tail_events.empty() ? 1 : (int)std::min<int64_t>((int64_t)g->tail_events.size(), B);
  const int64_t Bfull = B;
  const ConvRef& cpost = g->conv_post;
  const float post_slope = big ? 1.0f : 0.01f;
  const int post_tanh = g->cfg.kind == AB_GEN_TRUNK ? 0 : 1;
  for (int ci = 0; ci < nchunk; ++ci) {
    const int64_t b0 = Bfull * ci / nchunk, b1 = Bfull * (ci + 1) / nchunk;
    B = b1 - b0;
    const float* x = xin + b0 * sb;
    float* y = dev_wav + b0 * cpost.cout * Tn;
    rc = on_tc(cpost) ? tc_conv(cpost, nullptr, x, sb, sc, 1, nullptr, y, nullptr, Tn, post_slope, nullptr, nullptr, 1.0f,
                                post_tanh, conv_bytes(cpost, Tn, nullptr, nullptr))
                      : conv(cpost, x, sb, sc, 1, y, Tn, post_slope, nullptr, nullptr, 1.0f, post_tanh);
    B = Bfull;
    if (rc != AB_OK) break;
    if (!g->tail_events.empty()) {
      // when there are more events than utterances the surplus events fire with the last chunk
      const size_t e0 = g->tail_events.size() * (size_t)ci / nchunk, e1 = g->tail_events.size() * (size_t)(ci + 1) / nchunk;
      for (size_t e = e0; e < e1; ++e) cudaEventRecord(g->tail_events[e], st);
    }
  }
  g->tail_events.clear();
  g->source_frames = 0;
  if (rc != AB_OK) return rc;
  g->launches = launches;
  return AB_OK;
}

int ab_generator_forward(ab_generator* g, const float* dev_mel, int64_t B, int64_t T,
                         const int64_t mel_strides[3], float* dev_wav, void* dev_workspace,
                         size_t workspace_bytes, void* stream) {
  return forward_impl(g, dev_mel, B, T, mel_strides, nullptr, 0, dev_wav, dev_workspace, workspace_bytes, stream);
}

int ab_generator_forward_cond(ab_generator* g, const float* dev_x, int64_t B, int64_t T, const int64_t x_strides[3],
                              const float* dev_g, int64_t g_batch_stride, float* dev_wav, void* dev_workspace,
                              size_t workspace_bytes, void* stream) {
  return forward_impl(g, dev_x, B, T, x_strides, dev_g, g_batch_stride, dev_wav, dev_workspace, workspace_bytes, stream);
}

// ---------------------------------------------------------------------------
// standalone building blocks
// ---------------------------------------------------------------------------
int ab_activation1d_forward(const float* dev_x, float* dev_y, int64_t B, int64_t C, int64_t T,
                            const float* dev_alpha, const float* dev_beta, int32_t logscale,
                            const float* f_up, const float* f_down, void* stream) {
  if (!dev_x || !dev_y || !dev_alpha || !dev_beta || !f_up || !f_down) return fail(AB_ERR_ARG, "activation1d: null argument");
  if (T > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "activation1d: sequence too long");
  SnakeParams p;
  p.x = dev_x; p.y = dev_y; p.alpha = dev_alpha; p.beta = dev_beta; p.f_up = f_up; p.f_down = f_down;
  p.B = (int)B; p.C = (int)C; p.T = (int)T; p.logscale = logscale;
  p.yimg = nullptr; p.bf16 = 0;
  return launch_activation1d(p, static_cast<cudaStream_t>(stream));
}

size_t ab_conv1d_workspace_bytes(int64_t cin, int64_t cout, int32_t k, int32_t precision) {
  size_t n = align_up((size_t)cin * cout * k * sizeof(float), 256);
  if (precision != AB_PREC_FP32) n += align_up(tc_weight_image_bytes(0, (int)cin, (int)cout, k, 1), 256);
  return n;
}

int ab_conv1d_forward(const float* dev_x, const float* dev_w, const float* dev_bias,
                      const float* dev_residual, float* dev_y, int64_t B, int64_t cin, int64_t cout,
                      int64_t T, int32_t k, int32_t d, float pre_slope, int32_t post_tanh,
                      int32_t precision, void* ws, size_t ws_bytes, void* stream) {
  if (!dev_x || !dev_w || !dev_y || !ws) return fail(AB_ERR_ARG, "conv1d: null argument");
  if (ws_bytes < ab_conv1d_workspace_bytes(cin, cout, k, precision)) return fail(AB_ERR_WORKSPACE, "conv1d: workspace too small");
  if (T > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "conv1d: sequence too long");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* w_t = static_cast<float*>(ws);
  int rc = launch_repack_weight(dev_w, nullptr, w_t, (int)cout, (int)cin, k, 0, st);
  if (rc != AB_OK) return rc;
  if (precision == AB_PREC_FP32) {
    ConvParams p;
    p.x = dev_x; p.xsb = cin * T; p.xsc = T; p.xst = 1; p.w_t = w_t; p.bias = dev_bias;
    p.residual = dev_residual; p.acc_prev = nullptr; p.y = dev_y;
    p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)T; p.k = k; p.d = d;
    p.pre_slope = pre_slope; p.out_div = 1.0f; p.post_tanh = post_tanh;
    return launch_conv1d_fp32(p, st);
  }
  void* img = static_cast<char*>(ws) + align_up((size_t)cin * cout * k * sizeof(float), 256);
  if (tc_weight_image_bytes(0, (int)cin, (int)cout, k, d) == 0) return fail(AB_ERR_UNSUPPORTED, "conv1d: %s", ab_last_error());
  rc = launch_tc_pack_weight(w_t, img, 0, (int)cin, (int)cout, k, d, precision, st);
  if (rc != AB_OK) return rc;
  TcConvParams p;
  p.x = dev_x; p.xsb = cin * T; p.xsc = T; p.xst = 1; p.pre_slope = pre_slope;
  p.w = img; p.bias = dev_bias; p.residual = dev_residual; p.post_tanh = post_tanh; p.y = dev_y;
  p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)T; p.k = k; p.d_or_u = d; p.precision = precision;
  return launch_tc_conv(p, st);
}

size_t ab_conv_transpose1d_workspace_bytes(int64_t cin, int64_t cout, int32_t k, int32_t u, int32_t precision) {
  size_t n = align_up((size_t)cin * cout * k * sizeof(float), 256);
  if (precision != AB_PREC_FP32) n += align_up(tc_weight_image_bytes(1, (int)cin, (int)cout, k, u), 256);
  return n;
}

int ab_conv_transpose1d_forward(const float* dev_x, const float* dev_w, const float* dev_bias,
                                float* dev_y, int64_t B, int64_t cin, int64_t cout, int64_t Tin,
                                int32_t k, int32_t u, float pre_slope, int32_t precision, void* ws,
                                size_t ws_bytes, void* stream) {
  if (!dev_x || !dev_w || !dev_y || !ws) return fail(AB_ERR_ARG, "conv_transpose1d: null argument");
  if (ws_bytes < ab_conv_transpose1d_workspace_bytes(cin, cout, k, u, precision)) return fail(AB_ERR_WORKSPACE, "conv_transpose1d: workspace too small");
  if (Tin * u > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: sequence too long");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* w_t = static_cast<float*>(ws);
  int rc = launch_repack_weight(dev_w, nullptr, w_t, (int)cin, (int)cout, k, 1, st);
  if (rc != AB_OK) return rc;
  if (precision != AB_PREC_FP32) {
    void* img = static_cast<char*>(ws) + align_up((size_t)cin * cout * k * sizeof(float), 256);
    if (tc_weight_image_bytes(1, (int)cin, (int)cout, k, u) == 0) return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: %s", ab_last_error());
    rc = launch_tc_pack_weight(w_t, img, 1, (int)cin, (int)cout, k, u, precision, st);
    if (rc != AB_OK) return rc;
    TcConvParams p;
    p.mode = 1;
    p.x = dev_x; p.xsb = cin * Tin; p.xsc = Tin; p.xst = 1; p.pre_slope = pre_slope;
    p.w = img; p.bias = dev_bias; p.y = dev_y;
    p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)Tin; p.k = k; p.d_or_u = u; p.precision = precision;
    return launch_tc_conv(p, st);
  }
  ConvTParams p;
  p.x = dev_x; p.w_t = w_t; p.bias = dev_bias; p.y = dev_y;
  p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.Tin = (int)Tin; p.k = k; p.u = u; p.pre_slope = pre_slope;
  return launch_conv_transpose1d_fp32(p, st);
}

}  // extern "C"
