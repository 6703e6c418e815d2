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
  bool head_cols = false;   // Vocos' head.out: the weight image pairs each bin's magnitude and phase rows
  bool no_tc = false;       // never runs on the wgmma kernel (FACodec's out_proj, read by the vq2emb kernel)
  bool strided = false;     // Conv1d of stride `stride` (the FACodec encoder's downsampling convs)
};

struct ConvRef {   // one weight-normed conv of the model
  int w = -1, b = -1;
  int cin = 0, cout = 0, k = 0, d = 1;
  bool reflect = false;   // ReflectionPad1d((k-1)*d/2) in front of it instead of zero padding (MelGAN)
};

struct ActRef {    // one Activation1d module
  int alpha = -1, beta = -1, fup = -1, fdown = -1;
};

struct BlockRef {  // one ResBlock / AMPBlock
  int k = 0;
  std::vector<int> dil;
  std::vector<ConvRef> c1, c2;  // c2 empty for ResBlock2 / AMPBlock2
  std::vector<ActRef> acts;     // 2*nd (type 1) or nd (type 2); empty for HiFi-GAN
  ConvRef sc;                   // MelGAN ResnetBlock: the 1x1 shortcut (c1, c2 then hold one conv each)
};

// Vocos (AB_GEN_VOCOS) and VocosBackbone + nn.Linear (AB_GEN_VOCOS_LINEAR): slot indices of the backbone and head;
// the Linear layers are k = 1 convs
struct VocosBlockRef {   // one ConvNeXtBlock (vocos.py:469-527)
  int dw_w = -1, dw_b = -1, ln_w = -1, ln_b = -1, gamma = -1;
  ConvRef pw1, pw2;
};

struct VocosRef {
  int norm_w = -1, norm_b = -1, final_w = -1, final_b = -1, window = -1;
  std::vector<VocosBlockRef> blocks;
  ConvRef head;   // head.out: [n_fft + 2, dim]; AB_GEN_VOCOS_LINEAR: the Linear "1" [out, dim]
};

// DiffWave (AB_GEN_DIFFWAVE): slot indices; every tensor is a SLOT_VEC copied as is, the layer weights are repacked
// into the arena's packed region at finalize (launch_dw_pack)
struct DiffWaveLayerRef {   // one ResidualBlock (diffwave.py:90-122)
  int dil = 1;
  int wdil = -1, bdil = -1, wdp = -1, bdp = -1, wcond = -1, bcond = -1, wout = -1, bout = -1;
};

struct DiffWaveRef {
  int win = -1, bin = -1, table = -1, wp1 = -1, bp1 = -1, wp2 = -1, bp2 = -1;
  int wup[2] = {-1, -1}, bup[2] = {-1, -1};
  int wsk = -1, bsk = -1, wo = -1, bo = -1;
  std::vector<DiffWaveLayerRef> layers;
  size_t packed_offset = 0;   // arena offset of the packed region (diffwave_packed_floats)
  int64_t cond_B = 0, cond_T = 0;   // shapes of the last ab_diffwave_condition (0: none yet)
  int cond_rows = 0;
};

struct StageRef {
  ConvRef up;   // cin/cout/k, d unused; stride in `u`
  int u = 1;
  int ch = 0;
  bool has_up = true;   // false: AB_GEN_TRUNK's single stage (no transposed conv in front of the blocks)
  ActRef act;           // AB_GEN_FACODEC: the DecoderBlock's Activation1d in front of the transposed conv;
                        // AB_GEN_FACODEC_ENCODER: the EncoderBlock's Activation1d in front of the strided conv
  int down = 0;         // AB_GEN_FACODEC_ENCODER: `up` is the strided Conv1d (stride down) that closes the stage
  std::vector<BlockRef> blocks;
};

// FACodec (AB_GEN_FACODEC): timbre_linear and the codebook layers of the three ResidualVQs, in code-row order;
// AB_GEN_FACODEC_REDECODER: timbre_linear and the embedding tables (cb, rows) of the three groups, in code-row order
struct FacodecLayerRef {
  int cb = -1;
  ConvRef out_proj;
  int64_t rows = 0;
  ConvRef in_proj;          // facodec_quantize only
  size_t cbn_offset = 0;    // facodec_quantize: arena offset of the normalised rows [rows][16], then their squared norms
};
struct TimbreLayerRef {     // one TransformerEncoderLayer (transformer.py:84-151)
  int ln1_w = -1, ln1_b = -1, ln2_w = -1, ln2_b = -1;   // LayerNorm weight / bias, or with use_cln the style Linear's
  ConvRef qkv, out_proj, ffn_1, ffn_2;
};
struct FacodecRef {
  int style_w = -1, style_b = -1;
  std::vector<FacodecLayerRef> layers;
  // facodec_quantize: the timbre encoder (transformer.py:154-217); the redecoder: its prosody encoder (use_cln)
  int pe = -1, last_w = -1, last_b = -1;
  std::vector<TimbreLayerRef> timbre;
  // facodec_prosody_encoder (FACodecDecoderV2): melspec_linear and the prosody transformer melspec_encoder
  int mel_w = -1, mel_b = -1, pros_pe = -1, pros_last_w = -1, pros_last_b = -1;
  std::vector<TimbreLayerRef> prosody;
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
  VocosRef vocos;
  DiffWaveRef dw;
  FacodecRef fac;
  ab_mel* istft = nullptr;   // Vocos: the iSTFT plan (cuFFT C2R + overlap-add of ab_istft_forward)

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
    ab_mel_destroy(istft);
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

// AB_GEN_VOCOS: only its own fields; the ISTFT needs what ab_istft_forward serves.  AB_GEN_VOCOS_LINEAR: the backbone's
// fields and trunk_out_channels (the Linear's out_features)
int validate_vocos_config(const ab_generator_config& c) {
  const bool linear = c.kind == AB_GEN_VOCOS_LINEAR;
  if (c.num_upsamples || c.resblock || c.num_kernels || c.activation || c.snake_logscale || c.gin_channels ||
      c.conv_post_no_bias || (!linear && c.trunk_out_channels) || c.trunk_in_kernel || c.trunk_out_kernel ||
      (linear && (c.istft_n_fft || c.istft_hop)))
    return fail(AB_ERR_ARG, linear ? "config: VocosBackbone + Linear uses only n_mel, upsample_initial_channel, ffn_channels, "
                                     "num_layers and trunk_out_channels (every other field must be 0)"
                                   : "config: Vocos uses only n_mel, upsample_initial_channel, ffn_channels, num_layers, "
                                     "istft_n_fft and istft_hop (every other field must be 0)");
  const int lim = 1 << 16;
  if (c.n_mel <= 0 || c.n_mel > lim || c.upsample_initial_channel <= 0 || c.upsample_initial_channel > lim ||
      c.ffn_channels <= 0 || c.ffn_channels > lim || c.num_layers <= 0 || c.num_layers > 4096)
    return fail(AB_ERR_ARG, "config: Vocos input_channels %d, dim %d, intermediate_dim %d, num_layers %d out of range", c.n_mel,
                c.upsample_initial_channel, c.ffn_channels, c.num_layers);
  if (linear) {
    if (c.trunk_out_channels <= 0 || c.trunk_out_channels > lim)
      return fail(AB_ERR_ARG, "config: the Linear's out_features %d out of range", c.trunk_out_channels);
    return AB_OK;
  }
  if (c.istft_n_fft <= 0 || c.istft_hop <= 0 || c.istft_n_fft > lim)
    return fail(AB_ERR_ARG, "config: Vocos n_fft %d / hop %d out of range", c.istft_n_fft, c.istft_hop);
  if ((c.istft_n_fft & 1) || c.istft_hop > c.istft_n_fft || ((c.istft_n_fft - c.istft_hop) & 1))
    return fail(AB_ERR_UNSUPPORTED, "config: Vocos iSTFT needs an even n_fft, hop <= n_fft and n_fft - hop even (n_fft %d, hop %d)",
                c.istft_n_fft, c.istft_hop);
  return AB_OK;
}

// AB_GEN_DIFFWAVE: only its own fields
int validate_diffwave_config(const ab_generator_config& c) {
  if (c.resblock || c.num_kernels || c.activation || c.snake_logscale || c.gin_channels || c.conv_post_no_bias ||
      c.trunk_out_channels || c.trunk_in_kernel || c.trunk_out_kernel || c.ffn_channels || c.istft_n_fft || c.istft_hop)
    return fail(AB_ERR_ARG, "config: DiffWave uses only n_mel, upsample_initial_channel, num_layers, num_upsamples, "
                            "upsample_rates, dilation_cycle and embedding_rows (every other field must be 0)");
  if (c.n_mel <= 0 || c.n_mel > 512 || c.num_layers <= 0 || c.num_layers > 256 || c.dilation_cycle <= 0 ||
      c.dilation_cycle > 20 || c.embedding_rows <= 0 || c.embedding_rows > (1 << 20) || c.num_upsamples != 2)
    return fail(AB_ERR_ARG, "config: DiffWave n_mel %d (1..512), residual_layers %d (1..256), dilation_cycle %d (1..20), "
                "embedding rows %d or upsample factors (%d, need 2) out of range", c.n_mel, c.num_layers, c.dilation_cycle,
                c.embedding_rows, c.num_upsamples);
  if (c.upsample_initial_channel != DW_CHANNELS)
    return fail(AB_ERR_UNSUPPORTED, "config: DiffWave runs residual_channels = %d only (got %d)", DW_CHANNELS,
                c.upsample_initial_channel);
  for (int i = 0; i < 2; ++i)   // an odd factor makes the upsampled mel one sample longer than the audio
    if (c.upsample_rates[i] <= 0 || (c.upsample_rates[i] & 1) || c.upsample_rates[i] > 4096)
      return fail(AB_ERR_UNSUPPORTED, "config: DiffWave upsample factor %d must be even and positive", c.upsample_rates[i]);
  return AB_OK;
}

// FACodec's DecoderBlocks / EncoderBlocks: three ResidualUnits k = 7, dilations (1, 3, 9), SnakeBeta with logscale
// (facodec.py:121-154), or with snake1d the codec encoder's plain Snake1d (amphion_codec/codec.py:42-97, no logscale).
// blocks and model name them in the messages.
int check_facodec_units(const ab_generator_config& c, const char* blocks, const char* model, bool snake1d = false) {
  if (c.resblock != 1 || c.num_kernels != 1 || c.resblock_kernel_sizes[0] != 7 || c.num_dilations[0] != 3 ||
      c.resblock_dilation_sizes[0][0] != 1 || c.resblock_dilation_sizes[0][1] != 3 || c.resblock_dilation_sizes[0][2] != 9)
    return fail(AB_ERR_ARG, "config: %s hold ResidualUnits k = 7, dilations (1, 3, 9): resblock 1, num_kernels 1, kernel 7, "
                            "3 dilations", blocks);
  if (snake1d && c.activation == AB_ACT_SNAKE1D) {
    if (c.snake_logscale != 0) return fail(AB_ERR_ARG, "config: Snake1d has no logscale (snake_logscale must be 0)");
    return AB_OK;
  }
  if (c.activation != AB_ACT_SNAKEBETA || c.snake_logscale != 1)
    return fail(AB_ERR_ARG, snake1d ? "config: %s uses SnakeBeta with alpha_logscale = True, or Snake1d"
                                    : "config: %s uses SnakeBeta with alpha_logscale = True", model);
  return AB_OK;
}

// The three code groups (prosody, content, residual) of FACodec's decoder and redecoder: vq_num_q and the table sizes.
// model and table name them in the messages.
int check_facodec_groups(const ab_generator_config& c, const char* model, const char* table) {
  if (c.vq_num_q[0] <= 0 || c.vq_num_q[1] <= 0 || c.vq_num_q[2] < 0 ||
      c.vq_num_q[0] + c.vq_num_q[1] + c.vq_num_q[2] > AB_FACODEC_MAX_Q)
    return fail(AB_ERR_ARG, "config: %s vq_num_q (%d, %d, %d): prosody and content >= 1, residual >= 0, at most %d in all",
                model, c.vq_num_q[0], c.vq_num_q[1], c.vq_num_q[2], AB_FACODEC_MAX_Q);
  for (int i = 0; i < 3; ++i)
    if (c.vq_codebook_bits[i] <= 0 || c.vq_codebook_bits[i] > 24)
      return fail(AB_ERR_ARG, "config: %s size 2^%d out of range (bits 1..24)", table, c.vq_codebook_bits[i]);
  return AB_OK;
}

// The generator of FACodec's decoder and redecoder: the fixed block structure (facodec.py:121-133, :220-240)
int validate_facodec_generator_config(const ab_generator_config& c) {
  if (c.gin_channels || c.conv_post_no_bias || c.trunk_out_channels || c.trunk_in_kernel || c.trunk_out_kernel ||
      c.ffn_channels || c.num_layers || c.istft_n_fft || c.istft_hop || c.dilation_cycle || c.embedding_rows)
    return fail(AB_ERR_ARG, "config: FACodec uses only the generator fields and vq_* (gin / trunk / Vocos / DiffWave fields must be 0)");
  const int lim = 1 << 16;
  if (c.n_mel <= 0 || c.n_mel > lim || c.upsample_initial_channel <= 0 || c.upsample_initial_channel > lim)
    return fail(AB_ERR_ARG, "config: FACodec in_channels %d / upsample_initial_channel %d out of range", c.n_mel,
                c.upsample_initial_channel);
  if (c.num_upsamples <= 0 || c.num_upsamples > AB_MAX_STAGES || (c.upsample_initial_channel >> c.num_upsamples) <= 0)
    return fail(AB_ERR_ARG, "config: FACodec up_ratios: %d stages for %d channels", c.num_upsamples, c.upsample_initial_channel);
  for (int i = 0; i < c.num_upsamples; ++i)
    if (c.upsample_rates[i] <= 0 || c.upsample_rates[i] > 64 || c.upsample_kernel_sizes[i] != 2 * c.upsample_rates[i])
      return fail(AB_ERR_ARG, "config: FACodec stage %d: ratio %d (1..64) with kernel %d (must be 2 x ratio)", i,
                  c.upsample_rates[i], c.upsample_kernel_sizes[i]);
  return check_facodec_units(c, "FACodec DecoderBlocks", "FACodec");
}

// AB_GEN_FACODEC: the generator and the ResidualVQ geometry
int validate_facodec_config(const ab_generator_config& c) {
  int rc = validate_facodec_generator_config(c);
  if (rc != AB_OK) return rc;
  if ((rc = check_facodec_groups(c, "FACodec", "FACodec codebook")) != AB_OK) return rc;
  if (c.vq_codebook_dim <= 0 || c.vq_codebook_dim > FAC_MAX_CODEBOOK_DIM || c.vq_codebook_dim == c.n_mel)
    return fail(AB_ERR_UNSUPPORTED, "config: FACodec codebook_dim %d (1..%d, != vq_dim: out_proj must be a Linear)",
                c.vq_codebook_dim, FAC_MAX_CODEBOOK_DIM);
  if (c.facodec_quantize != 0 && c.facodec_quantize != 1)
    return fail(AB_ERR_ARG, "config: facodec_quantize must be 0 or 1 (got %d)", c.facodec_quantize);
  // the timbre encoder is always 256 wide (facodec.py:363) and reads x directly
  if (c.facodec_quantize && c.n_mel != FAC_TIMBRE_C)
    return fail(AB_ERR_UNSUPPORTED, "config: FACodec quantization needs in_channels == %d (the timbre encoder's width; "
                "got %d)", FAC_TIMBRE_C, c.n_mel);
  // FACodecDecoderV2: the prosody transformer feeds the quantizer, so it comes with facodec_quantize
  if (c.facodec_prosody_encoder != 0 && (c.facodec_prosody_encoder != 1 || !c.facodec_quantize))
    return fail(AB_ERR_ARG, "config: facodec_prosody_encoder must be 0, or 1 with facodec_quantize = 1 (got %d, %d)",
                c.facodec_prosody_encoder, c.facodec_quantize);
  return AB_OK;
}

// AB_GEN_FACODEC_REDECODER: the generator and the embedding tables (facodec.py:602-689)
int validate_facodec_redecoder_config(const ab_generator_config& c) {
  int rc = validate_facodec_generator_config(c);
  if (rc != AB_OK) return rc;
  // the prosody transformer is 256 wide, and its output is summed with the vq_dim-wide embeddings
  if (c.n_mel != FAC_TIMBRE_C)
    return fail(AB_ERR_UNSUPPORTED, "config: the FACodec redecoder needs in_channels == vq_dim == %d (the prosody "
                "transformer's width; got %d)", FAC_TIMBRE_C, c.n_mel);
  if ((rc = check_facodec_groups(c, "FACodec redecoder", "FACodec redecoder table")) != AB_OK) return rc;
  if (c.vq_codebook_dim != 0 || c.facodec_quantize != 0 || c.facodec_prosody_encoder != 0)
    return fail(AB_ERR_ARG, "config: the FACodec redecoder has no codebook_dim, facodec_quantize or "
                            "facodec_prosody_encoder (all must be 0)");
  return AB_OK;
}

// AB_GEN_FACODEC_ENCODER: the encoder's fixed block structure (facodec.py:121-194)
int validate_facodec_encoder_config(const ab_generator_config& c) {
  if (c.gin_channels || c.conv_post_no_bias || c.trunk_in_kernel || c.trunk_out_kernel || c.ffn_channels || c.num_layers ||
      c.istft_n_fft || c.istft_hop)
    return fail(AB_ERR_ARG, "config: the FACodec encoder uses only the generator fields and trunk_out_channels "
                            "(gin / trunk kernels / Vocos fields must be 0)");
  if (c.n_mel != 1) return fail(AB_ERR_ARG, "config: the FACodec encoder reads one waveform channel (n_mel must be 1, got %d)", c.n_mel);
  const int lim = 1 << 16;
  if (c.upsample_initial_channel <= 0 || c.trunk_out_channels <= 0 || c.trunk_out_channels > lim)
    return fail(AB_ERR_ARG, "config: FACodec encoder ngf %d / out_channels %d out of range", c.upsample_initial_channel,
                c.trunk_out_channels);
  if (c.num_upsamples <= 0 || c.num_upsamples > AB_MAX_STAGES || ((int64_t)c.upsample_initial_channel << c.num_upsamples) > lim)
    return fail(AB_ERR_ARG, "config: FACodec encoder up_ratios: %d stages from ngf %d", c.num_upsamples, c.upsample_initial_channel);
  // strides beyond the tensor-core strided conv's (AB_TC_MAX_STRIDE) are refused rather than served at fp32
  for (int i = 0; i < c.num_upsamples; ++i)
    if (c.upsample_rates[i] <= 0 || c.upsample_rates[i] > AB_TC_MAX_STRIDE ||
        c.upsample_kernel_sizes[i] != 2 * c.upsample_rates[i])
      return fail(AB_ERR_UNSUPPORTED, "config: FACodec encoder stage %d: stride %d (1..%d) with kernel %d (must be 2 x stride)",
                  i, c.upsample_rates[i], AB_TC_MAX_STRIDE, c.upsample_kernel_sizes[i]);
  return check_facodec_units(c, "FACodec EncoderBlocks", "the FACodec encoder", true);
}

// AB_GEN_RVQ: a ResidualVQ of FactorizedVectorQuantize layers (amphion_codec/quantize/residual_vq.py,
// factorized_vector_quantize.py) and nothing else
int validate_rvq_config(const ab_generator_config& c) {
  ab_generator_config z;
  memset(&z, 0, sizeof(z));
  z.kind = c.kind; z.n_mel = c.n_mel; z.vq_num_q[0] = c.vq_num_q[0]; z.vq_codebook_dim = c.vq_codebook_dim;
  z.vq_codebook_size = c.vq_codebook_size;
  if (memcmp(&z, &c, sizeof(z)) != 0)
    return fail(AB_ERR_ARG, "config: a residual VQ uses only n_mel (input_dim), vq_num_q[0] (num_quantizers), "
                            "vq_codebook_size and vq_codebook_dim (every other field must be 0)");
  if (c.n_mel <= 0 || c.n_mel > 4096 || c.vq_num_q[0] <= 0 || c.vq_num_q[0] > AB_FACODEC_MAX_Q || c.vq_codebook_size <= 0 ||
      c.vq_codebook_size > (1 << 24))
    return fail(AB_ERR_ARG, "config: residual VQ input_dim %d (1..4096), num_quantizers %d (1..%d) or codebook_size %d "
                "(1..2^24) out of range", c.n_mel, c.vq_num_q[0], AB_FACODEC_MAX_Q, c.vq_codebook_size);
  // the quantize kernel keeps the residual and the running sum of a 16-frame tile in shared memory
  if (c.n_mel > AB_RVQ_MAX_INPUT_DIM)
    return fail(AB_ERR_UNSUPPORTED, "config: residual VQ input_dim %d does not fit the quantize kernel's shared memory "
                "(at most %d)", c.n_mel, AB_RVQ_MAX_INPUT_DIM);
  if (c.vq_codebook_dim <= 0 || c.vq_codebook_dim > FAC_MAX_CODEBOOK_DIM || c.vq_codebook_dim == c.n_mel)
    return fail(AB_ERR_UNSUPPORTED, "config: residual VQ codebook_dim %d (1..%d, != input_dim: the projections must be "
                "convolutions)", c.vq_codebook_dim, FAC_MAX_CODEBOOK_DIM);
  return AB_OK;
}

int validate_config(const ab_generator_config& c) {
  if (c.kind != AB_GEN_HIFIGAN && c.kind != AB_GEN_BIGVGAN && c.kind != AB_GEN_NSFHIFIGAN && c.kind != AB_GEN_TRUNK &&
      c.kind != AB_GEN_MELGAN && c.kind != AB_GEN_VOCOS && c.kind != AB_GEN_DIFFWAVE && c.kind != AB_GEN_FACODEC &&
      c.kind != AB_GEN_FACODEC_ENCODER && c.kind != AB_GEN_FACODEC_REDECODER && c.kind != AB_GEN_RVQ &&
      c.kind != AB_GEN_VOCOS_LINEAR)
    return fail(AB_ERR_ARG, "config: unknown generator kind %d", c.kind);
  if (c.kind == AB_GEN_RVQ) return validate_rvq_config(c);
  if (c.vq_codebook_size) return fail(AB_ERR_ARG, "config: vq_codebook_size belongs to AB_GEN_RVQ");
  if (c.kind == AB_GEN_FACODEC) return validate_facodec_config(c);
  if (c.kind == AB_GEN_FACODEC_REDECODER) return validate_facodec_redecoder_config(c);
  if (c.activation == AB_ACT_SNAKE1D && c.kind != AB_GEN_FACODEC_ENCODER)
    return fail(AB_ERR_ARG, "config: Snake1d is served in the FACodec encoder kind only");
  if (c.facodec_quantize || c.facodec_prosody_encoder)
    return fail(AB_ERR_ARG, "config: facodec_quantize / facodec_prosody_encoder belong to AB_GEN_FACODEC");
  for (int i = 0; i < 3; ++i)
    if (c.vq_num_q[i] || c.vq_codebook_bits[i]) return fail(AB_ERR_ARG, "config: vq_* fields belong to AB_GEN_FACODEC");
  if (c.vq_codebook_dim) return fail(AB_ERR_ARG, "config: vq_* fields belong to AB_GEN_FACODEC");
  if (c.kind == AB_GEN_DIFFWAVE) return validate_diffwave_config(c);
  if (c.dilation_cycle || c.embedding_rows) return fail(AB_ERR_ARG, "config: dilation_cycle / embedding_rows belong to AB_GEN_DIFFWAVE");
  if (c.kind == AB_GEN_FACODEC_ENCODER) return validate_facodec_encoder_config(c);
  if (c.kind == AB_GEN_VOCOS || c.kind == AB_GEN_VOCOS_LINEAR) return validate_vocos_config(c);
  if (c.ffn_channels || c.num_layers || c.istft_n_fft || c.istft_hop)
    return fail(AB_ERR_ARG, "config: ffn_channels / num_layers / istft_* belong to AB_GEN_VOCOS");
  const bool trunk = c.kind == AB_GEN_TRUNK;
  const bool melgan = c.kind == AB_GEN_MELGAN;
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
    if (melgan) {
      if (u <= 0 || k != 2 * u) return fail(AB_ERR_ARG, "config: MelGAN stage %d: kernel %d must be 2 x ratio %d", i, k, u);
    } else if (u <= 0 || k < u || ((k - u) & 1)) {
      return fail(AB_ERR_UNSUPPORTED, "config: stage %d: kernel %d / rate %d (need k >= u, k-u even)", i, k, u);
    }
  }
  for (int j = 0; j < c.num_kernels; ++j) {
    if (c.num_dilations[j] <= 0 || c.num_dilations[j] > AB_MAX_DILATIONS) return fail(AB_ERR_ARG, "config: num_dilations[%d] out of range", j);
    const int k = c.resblock_kernel_sizes[j];
    if (k <= 0 || !(k & 1)) return fail(AB_ERR_UNSUPPORTED, "config: resblock kernel size %d must be odd", k);
    for (int p = 0; p < c.num_dilations[j]; ++p)
      if (c.resblock_dilation_sizes[j][p] <= 0) return fail(AB_ERR_ARG, "config: dilation must be positive");
  }
  if (melgan) {   // ResnetBlock(dim, dilation = 3^j), j < n_residual_layers (melgan.py:34-47, :82-85)
    if (c.num_kernels != 1 || c.resblock_kernel_sizes[0] != 3)
      return fail(AB_ERR_ARG, "config: MelGAN has one block kind with kernel 3 (num_kernels %d, kernel %d)", c.num_kernels,
                  c.resblock_kernel_sizes[0]);
    for (int p = 0, d = 1; p < c.num_dilations[0]; ++p, d *= 3)
      if (c.resblock_dilation_sizes[0][p] != d)
        return fail(AB_ERR_ARG, "config: MelGAN residual layer %d must have dilation %d (got %d)", p, d, c.resblock_dilation_sizes[0][p]);
    if ((c.upsample_initial_channel >> c.num_upsamples) << c.num_upsamples != c.upsample_initial_channel)
      return fail(AB_ERR_ARG, "config: MelGAN upsample_initial_channel %d must be ngf * 2^%d", c.upsample_initial_channel, c.num_upsamples);
    if (c.activation != AB_ACT_LRELU) return fail(AB_ERR_ARG, "config: MelGAN uses LeakyReLU(0.2)");
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
  if (s.strided) return tc_weight_image_bytes(2, cin, cout, k, s.stride);
  if (pre_or_post && (cin == cout || cin > 512 || cout <= 4)) return 0;
  return tc_weight_image_bytes(0, cin, cout, k, s.dilation);
}

// HiFi-GAN, BigVGAN, NSF-HiFiGAN and trunk tensors (reference state-dict names)
void add_gan_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const bool big = cfg->kind == AB_GEN_BIGVGAN;
  const bool has_beta = cfg->activation == AB_ACT_SNAKEBETA;
  const int c0 = cfg->upsample_initial_channel;
  const bool trunk = cfg->kind == AB_GEN_TRUNK;
  g->conv_pre = make_conv(g, "conv_pre", cfg->n_mel, c0, trunk ? cfg->trunk_in_kernel : 7, 1, false);
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
}

// MelGAN tensors (AB_GEN_MELGAN)
void add_melgan_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int c0 = cfg->upsample_initial_channel;
  // one nn.Sequential "model" (melgan.py:57-98): [pad, conv_pre], per stage i [lrelu, ConvTranspose, R ResnetBlocks],
  // [lrelu, pad, conv_post, tanh]; a ResnetBlock's convs are block.2 (k = 3, dilation 3^j), block.4 and shortcut (1x1)
  const int R = cfg->num_dilations[0], n = cfg->num_upsamples;
  auto mod = [](int i) { return "model." + std::to_string(i); };
  g->conv_pre = make_conv(g, mod(1), cfg->n_mel, c0, 7, 1, false);
  g->conv_pre.reflect = true;
  for (int i = 0; i < n; ++i) {
    StageRef st;
    const int base = 2 + i * (2 + R), cin = c0 >> i;
    st.ch = c0 >> (i + 1);
    st.u = cfg->upsample_rates[i];
    g->hop *= st.u;
    st.up = make_conv(g, mod(base + 1), cin, st.ch, 2 * st.u, 1, true);
    g->slots[st.up.w].stride = st.u;
    for (int j = 0; j < R; ++j) {
      BlockRef blk;
      blk.k = 3;
      const int d = cfg->resblock_dilation_sizes[0][j];
      blk.dil.push_back(d);
      const std::string pre = mod(base + 2 + j);
      blk.c1.push_back(make_conv(g, pre + ".block.2", st.ch, st.ch, 3, d, false));
      blk.c1.back().reflect = true;
      blk.c2.push_back(make_conv(g, pre + ".block.4", st.ch, st.ch, 1, 1, false));
      blk.sc = make_conv(g, pre + ".shortcut", st.ch, st.ch, 1, 1, false);
      st.blocks.push_back(blk);
    }
    g->stages.push_back(st);
  }
  g->conv_post = make_conv(g, mod(2 + n * (2 + R) + 2), c0 >> n, 1, 7, 1, false);
  g->conv_post.reflect = true;
}

ConvRef make_linear(ab_generator* g, const std::string& name, int cin, int cout);   // below

// The generator and timbre_linear of FACodec's decoder and redecoder, the reference's names (facodec.py:121-133,
// :220-240): model.* and timbre_linear.*
void add_facodec_generator_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int c0 = cfg->upsample_initial_channel, n = cfg->num_upsamples;
  auto mod = [](int i) { return "model." + std::to_string(i); };
  g->conv_pre = make_conv(g, mod(0), cfg->n_mel, c0, 7, 1, false);
  int ch = c0;
  for (int i = 0; i < n; ++i) {
    StageRef st;
    const std::string base = mod(1 + i) + ".block.";
    const int cin = c0 >> i;
    ch = st.ch = c0 >> (i + 1);
    st.u = cfg->upsample_rates[i];
    g->hop *= st.u;
    st.act = make_act(g, base + "0", cin, true);
    st.up = make_conv(g, base + "1", cin, ch, 2 * st.u, 1, true);
    g->slots[st.up.w].stride = st.u;
    BlockRef blk;   // the three ResidualUnits as one AMPBlock1-like block: act, k = 7 conv, act, k = 1 conv per unit
    blk.k = 7;
    for (int p = 0; p < 3; ++p) {
      const int d = cfg->resblock_dilation_sizes[0][p];
      const std::string pre = base + std::to_string(2 + p) + ".block.";
      blk.dil.push_back(d);
      blk.acts.push_back(make_act(g, pre + "0", ch, true));
      blk.c1.push_back(make_conv(g, pre + "1", ch, ch, 7, d, false));
      blk.acts.push_back(make_act(g, pre + "2", ch, true));
      blk.c2.push_back(make_conv(g, pre + "3", ch, ch, 1, 1, false));
    }
    st.blocks.push_back(blk);
    g->stages.push_back(st);
  }
  g->act_post = make_act(g, mod(1 + n), ch, true);
  g->conv_post = make_conv(g, mod(2 + n), ch, 1, 7, 1, false);
  const int C = cfg->n_mel;
  g->fac.style_w = g->add_slot("timbre_linear.weight", SLOT_VEC, {2 * C, C});
  g->fac.style_b = g->add_slot("timbre_linear.bias", SLOT_VEC, {2 * C});
}

// A FACodec transformer (transformer.py:154-234) under `prefix`: pe, four layers, last_ln, into pe / layers / last_w /
// last_b.  use_cln: each LayerNorm is a StyleAdaptiveLayerNorm, listed as its style Linear [2H, H] / [2H]
// (transformer.py:13-32).  fp32_only: the GEMMs run on the CUDA cores at every precision (no tensor-core image).
void add_facodec_transformer_tensors(ab_generator* g, const std::string& prefix, bool use_cln, int* pe,
                                     std::vector<TimbreLayerRef>* layers, int* last_w, int* last_b,
                                     bool fp32_only = false) {
  const int H = FAC_TIMBRE_C;
  *pe = g->add_slot(prefix + "position_emb.pe", SLOT_VEC, {FAC_PE_ROWS, 1, H});
  auto ln = [&](const std::string& name, int* w, int* b) {
    if (use_cln) {
      *w = g->add_slot(name + ".style.weight", SLOT_VEC, {2 * H, H});
      *b = g->add_slot(name + ".style.bias", SLOT_VEC, {2 * H});
    } else {
      *w = g->add_slot(name + ".weight", SLOT_VEC, {H});
      *b = g->add_slot(name + ".bias", SLOT_VEC, {H});
    }
  };
  for (int i = 0; i < 4; ++i) {
    const std::string pre = prefix + "layers." + std::to_string(i) + ".";
    TimbreLayerRef t;
    ln(pre + "ln_1", &t.ln1_w, &t.ln1_b);
    ln(pre + "ln_2", &t.ln2_w, &t.ln2_b);
    // nn.MultiheadAttention packs q, k and v into in_proj_weight [3H, H] / in_proj_bias [3H]
    t.qkv.cin = H; t.qkv.cout = 3 * H; t.qkv.k = 1;
    t.qkv.w = g->add_slot(pre + "self_attn.in_proj_weight", SLOT_CONV_W, {3 * H, H});
    g->slots[t.qkv.w].shape[2] = 1;
    t.qkv.b = g->add_slot(pre + "self_attn.in_proj_bias", SLOT_VEC, {3 * H});
    t.out_proj = make_linear(g, pre + "self_attn.out_proj", H, H);
    t.ffn_1 = make_conv(g, pre + "ffn.ffn_1", H, 4 * H, 5, 1, false);
    t.ffn_2 = make_linear(g, pre + "ffn.ffn_2", 4 * H, H);
    if (fp32_only)
      for (const ConvRef* c : {&t.qkv, &t.out_proj, &t.ffn_1, &t.ffn_2}) g->slots[c->w].no_tc = true;
    layers->push_back(t);
  }
  ln(prefix + "last_ln", last_w, last_b);
}

// FACodec decoder tensors (AB_GEN_FACODEC), the reference's names (facodec.py:121-133, :220-240, :286-369, fvq.py:23-29)
void add_facodec_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  add_facodec_generator_tensors(g);
  FacodecRef& f = g->fac;
  const int C = cfg->n_mel, D = cfg->vq_codebook_dim;
  for (int q = 0; q < 3; ++q)
    for (int j = 0; j < cfg->vq_num_q[q]; ++j) {
      const std::string pre = "quantizer." + std::to_string(q) + ".layers." + std::to_string(j) + ".";
      FacodecLayerRef l;
      l.rows = (int64_t)1 << cfg->vq_codebook_bits[q];
      l.cb = g->add_slot(pre + "_codebook.weight", SLOT_VEC, {l.rows, D});
      l.out_proj = make_linear(g, pre + "out_proj", D, C);
      g->slots[l.out_proj.w].no_tc = true;
      f.layers.push_back(l);
    }
  if (!cfg->facodec_quantize) return;
  // FACodecDecoder.forward(vq=True): the quantizers' in_proj (read by the RVQ kernel) and the timbre encoder
  size_t li = 0;
  for (int q = 0; q < 3; ++q)
    for (int j = 0; j < cfg->vq_num_q[q]; ++j, ++li) {
      FacodecLayerRef& l = f.layers[li];
      l.in_proj = make_linear(g, "quantizer." + std::to_string(q) + ".layers." + std::to_string(j) + ".in_proj", C, D);
      g->slots[l.in_proj.w].no_tc = true;
    }
  add_facodec_transformer_tensors(g, "timbre_encoder.", false, &f.pe, &f.timbre, &f.last_w, &f.last_b);
  if (!cfg->facodec_prosody_encoder) return;
  // FACodecDecoderV2 (facodec.py:1006-1017): melspec_linear (read by the prosody input kernel in its nn.Linear layout)
  // and melspec_encoder, which runs in fp32 at every precision because its output is quantized
  f.mel_w = g->add_slot("melspec_linear.weight", SLOT_VEC, {FAC_TIMBRE_C, FAC_PROSODY_BINS});
  f.mel_b = g->add_slot("melspec_linear.bias", SLOT_VEC, {FAC_TIMBRE_C});
  add_facodec_transformer_tensors(g, "melspec_encoder.", false, &f.pros_pe, &f.prosody, &f.pros_last_w, &f.pros_last_b,
                                  true);
}

// FACodec redecoder tensors (AB_GEN_FACODEC_REDECODER), the reference's names (facodec.py:602-689): the embedding
// tables "{prosody,content,residual}_embs.{j}.weight" [2^bits, 256], the generator and timbre_linear, and the prosody
// transformer "timbre_cond_prosody_enc.*" with style-adaptive LayerNorms
void add_facodec_redecoder_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  static const char* kTables[3] = {"prosody_embs.", "content_embs.", "residual_embs."};
  for (int q = 0; q < 3; ++q)
    for (int j = 0; j < cfg->vq_num_q[q]; ++j) {
      FacodecLayerRef l;
      l.rows = (int64_t)1 << cfg->vq_codebook_bits[q];
      l.cb = g->add_slot(kTables[q] + std::to_string(j) + ".weight", SLOT_VEC, {l.rows, cfg->n_mel});
      g->fac.layers.push_back(l);
    }
  add_facodec_generator_tensors(g);
  FacodecRef& f = g->fac;
  add_facodec_transformer_tensors(g, "timbre_cond_prosody_enc.", true, &f.pe, &f.timbre, &f.last_w, &f.last_b);
}

// FACodec encoder tensors (AB_GEN_FACODEC_ENCODER), the reference's names (facodec.py:121-194): "block.0" (conv_pre,
// 1 -> ngf, k = 7), per stride i "block.{1+i}.block.{0,1,2}.block.{0..3}" (three ResidualUnits at C = ngf 2^i),
// ".block.3" (Activation1d) and ".block.4" (the strided conv C -> 2C, k = 2s), "block.{1+n}" (final Activation1d),
// "block.{2+n}" (conv_post, k = 3).  With AB_ACT_SNAKE1D (the codec's CodecEncoder, codec.py:60-143) each activation
// is a Snake1d whose one tensor is "<module>.alpha" [1, C, 1].
void add_facodec_encoder_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int n = cfg->num_upsamples;
  auto mod = [](int i) { return "block." + std::to_string(i); };
  auto act = [&](const std::string& prefix, int ch) {
    if (cfg->activation != AB_ACT_SNAKE1D) return make_act(g, prefix, ch, true);
    ActRef a;
    a.alpha = g->add_slot(prefix + ".alpha", SLOT_VEC, {1, ch, 1});
    return a;
  };
  g->conv_pre = make_conv(g, mod(0), 1, cfg->upsample_initial_channel, 7, 1, false);
  g->slots[g->conv_pre.w].no_tc = true;   // one input channel: 31 of the wgmma kernel's 32 K lanes would be zero
  int ch = cfg->upsample_initial_channel;
  for (int i = 0; i < n; ++i) {
    StageRef st;
    const std::string base = mod(1 + i) + ".block.";
    st.ch = ch;
    st.u = 1;
    st.has_up = false;
    st.down = cfg->upsample_rates[i];
    g->hop *= st.down;
    BlockRef blk;   // the three ResidualUnits, as FACodec's decoder holds them
    blk.k = 7;
    for (int p = 0; p < 3; ++p) {
      const int d = cfg->resblock_dilation_sizes[0][p];
      const std::string pre = base + std::to_string(p) + ".block.";
      blk.dil.push_back(d);
      blk.acts.push_back(act(pre + "0", ch));
      blk.c1.push_back(make_conv(g, pre + "1", ch, ch, 7, d, false));
      blk.acts.push_back(act(pre + "2", ch));
      blk.c2.push_back(make_conv(g, pre + "3", ch, ch, 1, 1, false));
    }
    st.blocks.push_back(blk);
    st.act = act(base + "3", ch);
    st.up = make_conv(g, base + "4", ch, 2 * ch, 2 * st.down, 1, false);
    g->slots[st.up.w].stride = st.down;
    g->slots[st.up.w].strided = true;
    g->stages.push_back(st);
    ch *= 2;
  }
  g->act_post = act(mod(1 + n), ch);
  g->conv_post = make_conv(g, mod(2 + n), ch, cfg->trunk_out_channels, 3, 1, false);
}

// nn.Linear(cin, cout) as a k = 1 conv: weight [out, in] (state-dict shape), repacked as [in][1][out]
ConvRef make_linear(ab_generator* g, const std::string& name, int cin, int cout) {
  ConvRef c;
  c.cin = cin;
  c.cout = cout;
  c.k = 1;
  c.w = g->add_slot(name + ".weight", SLOT_CONV_W, {cout, cin});
  g->slots[c.w].shape[2] = 1;
  c.b = g->add_slot(name + ".bias", SLOT_VEC, {cout});
  return c;
}

// The codec's ResidualVQ (AB_GEN_RVQ), the reference's names (residual_vq.py:55-66, factorized_vector_quantize.py:40-50):
// per layer i "quantizers.{i}.in_project" (WNConv1d input_dim -> codebook_dim, k = 1), ".out_project" (WNConv1d
// codebook_dim -> input_dim, k = 1) and ".codebook.weight" [codebook_size, codebook_dim].  Repacked as every k = 1 conv,
// in_project is [input_dim][codebook_dim] and out_project [codebook_dim][input_dim], the layouts the RVQ kernels read.
void add_rvq_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int C = cfg->n_mel, D = cfg->vq_codebook_dim;
  for (int i = 0; i < cfg->vq_num_q[0]; ++i) {
    const std::string pre = "quantizers." + std::to_string(i) + ".";
    FacodecLayerRef l;
    l.rows = cfg->vq_codebook_size;
    l.in_proj = make_conv(g, pre + "in_project", C, D, 1, 1, false);
    l.out_proj = make_conv(g, pre + "out_project", D, C, 1, 1, false);
    l.cb = g->add_slot(pre + "codebook.weight", SLOT_VEC, {l.rows, D});
    g->slots[l.in_proj.w].no_tc = g->slots[l.out_proj.w].no_tc = true;
    g->fac.layers.push_back(l);
  }
}

// Vocos tensors (AB_GEN_VOCOS), the reference's state-dict names (vocos.py:469-527, :720-783, :314-361, :824-881);
// AB_GEN_VOCOS_LINEAR: nn.Sequential(VocosBackbone, nn.Linear)'s, "0.*" and "1.{weight,bias}" (repcodec_model.py:108-127)
void add_vocos_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int D = cfg->upsample_initial_channel, F = cfg->ffn_channels;
  const bool linear = cfg->kind == AB_GEN_VOCOS_LINEAR;
  const std::string bb = linear ? "0." : "backbone.";
  VocosRef& v = g->vocos;
  g->conv_pre = make_conv(g, bb + "embed", cfg->n_mel, D, 7, 1, false);
  v.norm_w = g->add_slot(bb + "norm.weight", SLOT_VEC, {D});
  v.norm_b = g->add_slot(bb + "norm.bias", SLOT_VEC, {D});
  for (int i = 0; i < cfg->num_layers; ++i) {
    const std::string pre = bb + "convnext." + std::to_string(i);
    VocosBlockRef b;
    b.dw_w = g->add_slot(pre + ".dwconv.weight", SLOT_VEC, {D, 1, 7});
    b.dw_b = g->add_slot(pre + ".dwconv.bias", SLOT_VEC, {D});
    b.ln_w = g->add_slot(pre + ".norm.weight", SLOT_VEC, {D});
    b.ln_b = g->add_slot(pre + ".norm.bias", SLOT_VEC, {D});
    b.pw1 = make_linear(g, pre + ".pwconv1", D, F);
    b.pw2 = make_linear(g, pre + ".pwconv2", F, D);
    b.gamma = g->add_slot(pre + ".gamma", SLOT_VEC, {D});
    v.blocks.push_back(b);
  }
  v.final_w = g->add_slot(bb + "final_layer_norm.weight", SLOT_VEC, {D});
  v.final_b = g->add_slot(bb + "final_layer_norm.bias", SLOT_VEC, {D});
  if (linear) {
    v.head = make_linear(g, "1", D, cfg->trunk_out_channels);
    return;
  }
  v.head = make_linear(g, "head.out", D, cfg->istft_n_fft + 2);
  g->slots[v.head.w].head_cols = true;
  v.window = g->add_slot("head.istft.window", SLOT_VEC, {cfg->istft_n_fft});
  g->hop = cfg->istft_hop;
}

// DiffWave tensors (AB_GEN_DIFFWAVE), the reference's names (diffwave.py:28-66, :90-110, :127-162)
void add_diffwave_tensors(ab_generator* g) {
  const ab_generator_config* cfg = &g->cfg;
  const int C = cfg->upsample_initial_channel, nm = cfg->n_mel;
  DiffWaveRef& d = g->dw;
  d.win = g->add_slot("input_projection.weight", SLOT_VEC, {C, 1, 1});
  d.bin = g->add_slot("input_projection.bias", SLOT_VEC, {C});
  d.table = g->add_slot("diffusion_embedding.embedding", SLOT_VEC, {cfg->embedding_rows, 128});
  d.wp1 = g->add_slot("diffusion_embedding.projection1.weight", SLOT_VEC, {512, 128});
  d.bp1 = g->add_slot("diffusion_embedding.projection1.bias", SLOT_VEC, {512});
  d.wp2 = g->add_slot("diffusion_embedding.projection2.weight", SLOT_VEC, {512, 512});
  d.bp2 = g->add_slot("diffusion_embedding.projection2.bias", SLOT_VEC, {512});
  for (int i = 0; i < 2; ++i) {   // ConvTranspose2d weight [1, 1, 3, 2f]: any shape of 6f elements loads
    const std::string pre = "spectrogram_upsampler.conv" + std::to_string(i + 1);
    d.wup[i] = g->add_slot(pre + ".weight", SLOT_VEC, {1, 3, 2 * cfg->upsample_rates[i]});
    d.bup[i] = g->add_slot(pre + ".bias", SLOT_VEC, {1});
    g->hop *= cfg->upsample_rates[i];
  }
  for (int i = 0; i < cfg->num_layers; ++i) {
    const std::string pre = "residual_layers." + std::to_string(i);
    DiffWaveLayerRef l;
    l.dil = 1 << (i % cfg->dilation_cycle);
    l.wdil = g->add_slot(pre + ".dilated_conv.weight", SLOT_VEC, {2 * C, C, 3});
    l.bdil = g->add_slot(pre + ".dilated_conv.bias", SLOT_VEC, {2 * C});
    l.wdp = g->add_slot(pre + ".diffusion_projection.weight", SLOT_VEC, {C, 512});
    l.bdp = g->add_slot(pre + ".diffusion_projection.bias", SLOT_VEC, {C});
    l.wcond = g->add_slot(pre + ".conditioner_projection.weight", SLOT_VEC, {2 * C, nm, 1});
    l.bcond = g->add_slot(pre + ".conditioner_projection.bias", SLOT_VEC, {2 * C});
    l.wout = g->add_slot(pre + ".output_projection.weight", SLOT_VEC, {2 * C, C, 1});
    l.bout = g->add_slot(pre + ".output_projection.bias", SLOT_VEC, {2 * C});
    d.layers.push_back(l);
  }
  d.wsk = g->add_slot("skip_projection.weight", SLOT_VEC, {C, C, 1});
  d.bsk = g->add_slot("skip_projection.bias", SLOT_VEC, {C});
  d.wo = g->add_slot("output_projection.weight", SLOT_VEC, {1, C, 1});
  d.bo = g->add_slot("output_projection.bias", SLOT_VEC, {1});
}

// Packed region of a DiffWave handle, in floats: per layer w1p [3C + n_mel][2C], b1p [2C], w2p [C][2C], b2p [2C], then
// the 16-bit images of the tensor-core kernel w1h [2C][dw_k1p] and w2h [2C][C] (each part 64-float aligned; the images
// are written only at tensor-core precision), then every layer's diffusion_projection [layers][C][512] and bias
// [layers][C] back to back.
size_t dw_layer_packed_floats(int n_mel) {
  const size_t C = DW_CHANNELS;
  return align_up((3 * C + n_mel) * 2 * C, 64) + align_up(2 * C, 64) + align_up(C * 2 * C, 64) + align_up(2 * C, 64) +
         align_up(C * dw_k1p(n_mel), 64) + align_up(C * C, 64);
}
// layer l's parts of the packed region
struct DwLayerPack {
  float *w1, *b1, *w2, *b2;
  uint16_t *w1h, *w2h;
};
DwLayerPack dw_layer_pack(char* packed, int n_mel, int l) {
  const size_t C = DW_CHANNELS;
  DwLayerPack r;
  r.w1 = reinterpret_cast<float*>(packed) + l * dw_layer_packed_floats(n_mel);
  r.b1 = r.w1 + align_up((3 * C + n_mel) * 2 * C, 64);
  r.w2 = r.b1 + align_up(2 * C, 64);
  r.b2 = r.w2 + align_up(C * 2 * C, 64);
  r.w1h = reinterpret_cast<uint16_t*>(r.b2 + align_up(2 * C, 64));
  r.w2h = reinterpret_cast<uint16_t*>(r.b2 + align_up(2 * C, 64) + align_up(C * dw_k1p(n_mel), 64));
  return r;
}
size_t diffwave_packed_floats(const ab_generator_config& c) {
  return c.num_layers * (dw_layer_packed_floats(c.n_mel) + (size_t)DW_CHANNELS * 513);
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
  g->hop = 1;
  if (cfg->kind == AB_GEN_MELGAN) {
    add_melgan_tensors(g);
  } else if (cfg->kind == AB_GEN_VOCOS) {
    add_vocos_tensors(g);
    const ab_mel_config mc = {cfg->istft_n_fft, cfg->istft_hop, cfg->istft_n_fft, 0, 0, 0.0f, 0.0f};
    rc = ab_mel_create(&mc, &g->istft);
    if (rc != AB_OK) {
      delete g;
      return rc;
    }
  } else if (cfg->kind == AB_GEN_VOCOS_LINEAR) {
    add_vocos_tensors(g);
  } else if (cfg->kind == AB_GEN_DIFFWAVE) {
    add_diffwave_tensors(g);
  } else if (cfg->kind == AB_GEN_FACODEC) {
    add_facodec_tensors(g);
  } else if (cfg->kind == AB_GEN_FACODEC_ENCODER) {
    add_facodec_encoder_tensors(g);
  } else if (cfg->kind == AB_GEN_FACODEC_REDECODER) {
    add_facodec_redecoder_tensors(g);
  } else if (cfg->kind == AB_GEN_RVQ) {
    add_rvq_tensors(g);
  } else {
    add_gan_tensors(g);
  }

  // tensor-core weight images live behind the fp32 images
  size_t tc = 0;
  for (size_t i = 0; i < g->slots.size(); ++i) {
    Slot& s = g->slots[i];
    s.tc_bytes = s.no_tc ? 0 : tc_image_bytes(s, (int)i == g->conv_pre.w || (int)i == g->conv_post.w);
    s.tc_offset = g->fp32_bytes + tc;
    tc += align_up(s.tc_bytes, 256);
  }
  g->arena_need = g->fp32_bytes + tc;
  if (cfg->kind == AB_GEN_DIFFWAVE) {
    g->dw.packed_offset = g->arena_need;
    g->arena_need += align_up(diffwave_packed_floats(*cfg) * sizeof(float), 256);
  }
  if ((cfg->kind == AB_GEN_FACODEC && cfg->facodec_quantize) || cfg->kind == AB_GEN_RVQ) {   // normalised codebooks, built at finalize
    for (auto& l : g->fac.layers) {
      l.cbn_offset = g->arena_need;
      g->arena_need += align_up((size_t)l.rows * FAC_MAX_CODEBOOK_DIM * sizeof(float), 256) +
                       align_up((size_t)l.rows * sizeof(float), 256);
    }
  }
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
  if (g->cfg.kind == AB_GEN_DIFFWAVE) {
    if (precision != AB_PREC_FP32 && !ab_device_is_sm90())
      return fail(AB_ERR_UNSUPPORTED, "finalize: tensor-core precision needs an sm_90 (Hopper) device");
    const int nl = g->cfg.num_layers, nm = g->cfg.n_mel, C = DW_CHANNELS;
    float* pk = reinterpret_cast<float*>(g->arena + g->dw.packed_offset);
    float* proj = pk + nl * dw_layer_packed_floats(nm);
    for (int l = 0; l < nl; ++l) {
      const DiffWaveLayerRef& L = g->dw.layers[l];
      DwPackParams p;
      p.wdil = g->fptr(L.wdil); p.bdil = g->fptr(L.bdil); p.wcond = g->fptr(L.wcond); p.bcond = g->fptr(L.bcond);
      p.wout = g->fptr(L.wout); p.bout = g->fptr(L.bout);
      const DwLayerPack lp = dw_layer_pack(g->arena + g->dw.packed_offset, nm, l);
      p.w1p = lp.w1; p.b1p = lp.b1; p.w2p = lp.w2; p.b2p = lp.b2;
      p.w1h = precision != AB_PREC_FP32 ? lp.w1h : nullptr; p.w2h = lp.w2h;
      p.bf16 = precision == AB_PREC_TC_BF16;
      p.n_mel = nm;
      const int rc = launch_dw_pack(p, st);
      if (rc != AB_OK) return rc;
      AB_CUDA_TRY(cudaMemcpyAsync(proj + (size_t)l * C * 512, g->fptr(L.wdp), (size_t)C * 512 * 4, cudaMemcpyDeviceToDevice, st));
      AB_CUDA_TRY(cudaMemcpyAsync(proj + (size_t)nl * C * 512 + l * C, g->fptr(L.bdp), C * 4, cudaMemcpyDeviceToDevice, st));
    }
    g->dw.cond_B = g->dw.cond_T = 0;
    g->precision = precision;
    g->finalized = true;
    return AB_OK;
  }
  if (precision != AB_PREC_FP32) {
    if (!ab_device_is_sm90()) return fail(AB_ERR_UNSUPPORTED, "finalize: tensor-core precision needs an sm_90 (Hopper) device");
    for (size_t i = 0; i < g->slots.size(); ++i) {
      const Slot& s = g->slots[i];
      if (!s.tc_bytes) continue;
      const bool t = s.kind == SLOT_CONVT_W;   // state-dict shape: ConvTranspose1d [C_in, C_out, k], Conv1d [C_out, C_in, k]
      if (s.head_cols) {
        int rc = launch_tc_pack_head_weight(g->fptr((int)i), g->tcptr((int)i), (int)s.shape[1], (int)s.shape[0], precision, st);
        if (rc != AB_OK) return rc;
        continue;
      }
      int rc = launch_tc_pack_weight(g->fptr((int)i), g->tcptr((int)i), t ? 1 : s.strided ? 2 : 0, (int)s.shape[t ? 0 : 1],
                                     (int)s.shape[t ? 1 : 0], (int)s.shape[2], t || s.strided ? s.stride : s.dilation,
                                     precision, st);
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
  // the transformers' GEMMs (the timbre encoder's, the prosody encoder's) all run on the wgmma kernel at 16 bits
  for (const auto& t : g->fac.timbre)
    for (const ConvRef* c : {&t.qkv, &t.out_proj, &t.ffn_1, &t.ffn_2})
      if (precision != AB_PREC_FP32 && g->slots[c->w].tc_bytes == 0)
        return fail(AB_ERR_UNSUPPORTED, "finalize: '%s' has no tensor-core image", g->slots[c->w].name.c_str());
  if ((g->cfg.kind == AB_GEN_FACODEC && g->cfg.facodec_quantize) || g->cfg.kind == AB_GEN_RVQ) {
    for (const auto& l : g->fac.layers) {
      float* cbn = reinterpret_cast<float*>(g->arena + l.cbn_offset);
      float* cbn2 = reinterpret_cast<float*>(g->arena + l.cbn_offset +
                                             align_up((size_t)l.rows * FAC_MAX_CODEBOOK_DIM * sizeof(float), 256));
      const int rc = launch_facodec_cbnorm(g->fptr(l.cb), cbn, cbn2, l.rows, g->cfg.vq_codebook_dim, st);
      if (rc != AB_OK) return rc;
    }
  }
  g->precision = precision;
  g->finalized = true;
  return AB_OK;
}

// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
extern "C++" {
namespace {
constexpr int NBUF = 7;  // fp32: R0 R1 U P0 P1 TMP ACT
constexpr int NIMG = 4;  // 16-bit operand images: U P0 P1 R (stage output, HiFi-GAN)

double rup16(int c) { return (double)((c + 15) / 16 * 16); }

// Bump allocator over a workspace: take(bytes) returns the next 256-byte-aligned region, nullptr when base is null
// (sizes only); off is the size of everything taken so far
struct Carve {
  char* base;
  size_t off = 0;
  template <class P = float>
  P* take(size_t bytes) {
    P* p = base ? reinterpret_cast<P*>(base + off) : nullptr;
    off += align_up(bytes, 256);
    return p;
  }
};

int check_workspace(const char* what, const void* ws, size_t bytes, size_t need) {
  if (!ws || bytes < need) return fail(AB_ERR_WORKSPACE, "%s: workspace %zu B < required %zu B", what, bytes, need);
  if (reinterpret_cast<uintptr_t>(ws) & 255) return fail(AB_ERR_ARG, "%s: workspace must be 256-byte aligned", what);
  return AB_OK;
}

// One Activation1d launch as a generator issues it: the taps packed on the host (kc; null: the kernel reads f_up /
// f_down), and at 16 bits the short snake, which launch_activation1d takes on image-only launches.  Shared by
// Launch::snake and ab_activation1d_packed_forward, so that the standalone entry point runs the generator's launch.
SnakeParams generator_snake_params(const SnakeCoef* kc, int precision, const float* x, float* y, uint16_t* yimg,
                                   const float* alpha, const float* beta, const float* f_up, const float* f_down,
                                   int logscale, int B, int C, int T) {
  SnakeParams p;
  if (kc) { p.kc = *kc; p.have_kc = 1; }
  p.fast_snake = precision != AB_PREC_FP32;
  p.yimg = yimg; p.bf16 = precision == AB_PREC_TC_BF16;
  p.x = x; p.y = y; p.alpha = alpha; p.beta = beta; p.f_up = f_up; p.f_down = f_down;
  p.B = B; p.C = C; p.T = T; p.logscale = logscale;
  return p;
}

// The launches of one entry-point call: counts them (ab_generator_last_launches), times each one when profiling is on
// (ab_generator_set_profiling), and runs the layers the model kinds share
struct Launch {
  ab_generator* g;
  cudaStream_t st;
  int launches = 0;

  template <class F>
  int timed(int cls, double flops, double bytes, F launch) {
    ++launches;
    if (!g->profiling) return launch();
    const ab_generator::ProfRec r{cls, g->get_event(), g->get_event(), flops, bytes};
    cudaEventRecord(r.e0, st);
    g->prof_recs.push_back(r);
    const int rc = launch();
    cudaEventRecord(g->prof_recs.back().e1, st);
    return rc;
  }
  // n launches that are counted but not timed
  template <class F>
  int counted(int n, F launch) {
    launches += n;
    return launch();
  }
  // the count becomes ab_generator_last_launches when the call succeeds
  int done(int rc) {
    if (rc == AB_OK) g->launches = launches;
    return rc;
  }

  // whether conv c runs on the wgmma kernel (tc_image_bytes decided it at create)
  bool on_tc(const ConvRef& c) const { return g->precision != AB_PREC_FP32 && g->slots[c.w].tc_bytes > 0; }

  // algorithmic HBM bytes of a Conv1d launch with fp32 activations and weights (profile)
  static double conv_bytes(const ConvRef& c, int64_t B, int Tn, const float* residual, const float* acc_prev) {
    const double el = (double)B * Tn;
    return 4.0 * (el * c.cin + el * c.cout * (1 + (residual != nullptr) + (acc_prev != nullptr)) + (double)c.cin * c.cout * c.k);
  }

  // fp32 CUDA-core Conv1d; epi / gamma: Vocos' GELU or layer-scale residual epilogue in place of the branch mix
  int conv(const ConvRef& c, int64_t B, const float* x, int64_t xsb, int64_t xsc, int64_t xst, float* y, int Tn,
           float pre_slope, const float* residual, const float* acc_prev, float out_div, int post_tanh,
           int epi = CONV_EPI_NONE, const float* gamma = nullptr) {
    ConvParams p;
    p.x = x; p.xsb = xsb; p.xsc = xsc; p.xst = xst;
    p.w_t = g->fptr(c.w); p.bias = g->fptr(c.b);
    p.residual = residual; p.acc_prev = acc_prev; p.y = y;
    p.B = (int)B; p.Cin = c.cin; p.Cout = c.cout; p.T = Tn; p.k = c.k; p.d = c.d;
    p.pre_slope = pre_slope; p.out_div = out_div; p.post_tanh = post_tanh; p.reflect = c.reflect;
    p.epi = epi; p.gamma = gamma;
    return timed(1, 2.0 * B * Tn * c.cout * c.cin * c.k, conv_bytes(c, B, Tn, residual, acc_prev),
                 [&] { return launch_conv1d_fp32(p, st); });
  }

  // Conv1d c on the wgmma kernel, from fp32 x (lrelu(., pre_slope) in the loader) or the operand image ximg; with c2
  // the ResBlock1 pair c -> lrelu(., pre_slope) -> c2 in one launch.  yimg: the image of lrelu(y, img_slope).  bytes:
  // the launch's algorithmic HBM bytes; cls: the profile class, -1 for 0 on a pair / block-mode capable ResBlock conv
  // and 4 on any other
  int tc_conv(const ConvRef& c, const ConvRef* c2, int64_t B, const float* x, int64_t xsb, int64_t xsc, int64_t xst,
              const uint16_t* ximg, float* y, uint16_t* yimg, int Tn, float pre_slope, const float* residual,
              const float* acc_prev, float out_div, int post_tanh, double bytes, int cls = -1, float img_slope = 0.1f) {
    TcConvParams p;
    p.x = x; p.xsb = xsb; p.xsc = xsc; p.xst = xst; p.ximg = ximg; p.pre_slope = pre_slope;
    p.w = g->tcptr(c.w); p.bias = g->fptr(c.b);
    if (c2) { p.w2 = g->tcptr(c2->w); p.b2 = g->fptr(c2->b); p.mid_slope = pre_slope; }
    p.residual = residual; p.acc_prev = acc_prev; p.out_div = out_div; p.post_tanh = post_tanh;
    p.y = y; p.yimg = yimg; p.img_slope = img_slope;
    p.B = (int)B; p.Cin = c.cin; p.Cout = c.cout; p.T = Tn; p.k = c.k; p.d_or_u = c.d;
    p.precision = g->precision; p.reflect = c.reflect;
    if (cls < 0) cls = c.cin == c.cout && tc_conv_supported(c.cin, c.k) ? 0 : 4;
    return timed(cls, 2.0 * B * Tn * c.cout * c.cin * c.k * (c2 ? 2 : 1), bytes, [&] { return launch_tc_conv(p, st); });
  }

  // Activation1d, or the codec encoder's Snake1d: fp32 y and / or the 16-bit operand image yimg
  int snake(const ActRef& a, int64_t B, const float* x, float* y, int C, int Tn, uint16_t* yimg = nullptr) {
    if (g->cfg.activation == AB_ACT_SNAKE1D)
      return timed(3, 0.0, (double)B * C * Tn * (4.0 + (y ? 4.0 : 0.0)) + (yimg ? 2.0 * B * rup16(C) * Tn : 0.0), [&] {
        return launch_snake1d(x, y, yimg, g->precision == AB_PREC_TC_BF16, g->fptr(a.alpha), (int)B, C, Tn, st);
      });
    auto kc = g->act_coef.find(a.fup);
    const SnakeParams p = generator_snake_params(kc != g->act_coef.end() ? &kc->second : nullptr, g->precision, x, y,
                                                 yimg, g->fptr(a.alpha), g->fptr(a.beta), g->fptr(a.fup),
                                                 g->fptr(a.fdown), g->cfg.snake_logscale, (int)B, C, Tn);
    return timed(3, 0.0, (double)B * C * Tn * (4.0 + (y ? 4.0 : 0.0) + (yimg ? 2.0 : 0.0)),
                 [&] { return launch_activation1d(p, st); });
  }

  // LayerNorm over channels [after Vocos' depthwise conv, slots dw_w / dw_b >= 0] -> fp32 y or the operand image yimg
  int norm(int64_t B, int C, int Tn, const float* x, int dw_w, int dw_b, int ln_w, int ln_b, float eps, float* y,
           uint16_t* yimg) {
    NormParams p;
    p.x = x; p.dw_w = g->fptr(dw_w); p.dw_b = g->fptr(dw_b); p.ln_w = g->fptr(ln_w); p.ln_b = g->fptr(ln_b);
    p.y = y; p.yimg = yimg; p.bf16 = g->precision == AB_PREC_TC_BF16;
    p.B = (int)B; p.C = C; p.T = Tn; p.eps = eps;
    const double el = (double)B * Tn;
    return timed(6, el * C * ((dw_w >= 0 ? 14.0 : 0.0) + 8.0), 4.0 * el * C + (y ? 4.0 * el * C : 2.0 * el * rup16(C)),
                 [&] { return launch_vocos_norm(p, st); });
  }

  // The last layer of a forward in contiguous batch chunks, chunk(b0, nb) each, and an event after each
  // (ab_generator_set_tail_events): the caller's final gather of chunk i then runs under chunk i+1.  Runs nothing when
  // rc is an error; consumes the tail events and nsf_source_frames either way.
  template <class F>
  int tail(int64_t B, int rc, F chunk) {
    const size_t ne = g->tail_events.size();
    const int nchunk = ne == 0 ? 1 : (int)std::min<int64_t>((int64_t)ne, B);
    for (int ci = 0; rc == AB_OK && ci < nchunk; ++ci) {
      const int64_t b0 = B * ci / nchunk, b1 = B * (ci + 1) / nchunk;
      rc = chunk(b0, b1 - b0);
      // when there are more events than utterances the surplus events fire with the last chunk
      if (rc == AB_OK)
        for (size_t e = ne * ci / nchunk; e < ne * (ci + 1) / nchunk; ++e) cudaEventRecord(g->tail_events[e], st);
    }
    g->tail_events.clear();
    g->source_frames = 0;
    return rc;
  }
};

// Output length of the FACodec encoder's strided conv (k = 2s, padding s//2 + s%2) over t samples; 0 when the input is
// empty or the padded input is shorter than the kernel (Conv1d raises), so an emptied stage stays empty
int64_t encoder_stage_length(int64_t t, int s) {
  if (t <= 0) return 0;
  const int64_t padded = t + 2 * (s / 2 + s % 2);
  return padded < 2 * s ? 0 : (padded - 2 * s) / s + 1;
}

// Largest stage tensor of a forward of T frames (T samples for the encoder), in elements (image = false) or as a
// 16-bit operand image in bytes: conv_pre's output, each stage's blocks and, for the encoder, its strided conv's output
size_t stage_max(const ab_generator* g, int64_t B, int64_t T, bool image) {
  auto size = [&](int c, int64_t t) { return image ? tc_act_image_bytes(B, c, t) : (size_t)B * c * t; };
  size_t mx = size(g->cfg.upsample_initial_channel, T);
  int64_t t = T;
  for (auto& st : g->stages) {
    t *= st.u;
    mx = std::max(mx, size(st.ch, t));
    if (st.down) {
      t = encoder_stage_length(t, st.down);
      mx = std::max(mx, size(st.up.cout, t));
    }
  }
  return mx;
}

// Workspace of the generator pipeline: NBUF fp32 stage buffers and NIMG 16-bit operand images; FACodec's decoder and
// redecoder then the FiLM output (fp32, or conv_pre's operand image) and the style [B][2C].  Returns its size.
struct GanWs {
  float* buf[NBUF];
  uint16_t* img[NIMG];
  char* film;
  float* style;
};

size_t gan_layout(const ab_generator* g, int64_t B, int64_t T, char* base, GanWs* w) {
  Carve c{base};
  GanWs v = {};
  const size_t bufsz = stage_max(g, B, T, false) * sizeof(float), imgsz = stage_max(g, B, T, true);
  for (float*& b : v.buf) b = c.take(bufsz);
  for (uint16_t*& i : v.img) i = c.take<uint16_t>(imgsz);
  if (g->cfg.kind == AB_GEN_FACODEC || g->cfg.kind == AB_GEN_FACODEC_REDECODER) {
    const int C = g->cfg.n_mel;
    v.film = c.take<char>(std::max((size_t)B * C * T * sizeof(float), tc_act_image_bytes(B, C, T)));
    v.style = c.take((size_t)B * 2 * C * sizeof(float));
  }
  if (w) *w = v;
  return c.off;
}

// Vocos workspace: the fp32 residual stream X, the embed / final-norm output Y (fp32), the block input H and the
// intermediate I (fp32 at AB_PREC_FP32, else 16-bit operand images; I also holds the fp32 head output), the spectrum S
// [B*T][bins] complex and the iSTFT's workspace.  base == nullptr: sizes only.  0 when the iSTFT plan fails.
// AB_GEN_VOCOS_LINEAR: X, Y, H and I only (the Linear writes the output).
struct VocosWs {
  float *X, *Y, *H, *I, *S;
  void* ist;
  size_t ist_bytes;
};

size_t vocos_layout(const ab_generator* g, int64_t B, int64_t T, char* base, VocosWs* w) {
  const int D = g->cfg.upsample_initial_channel, F = g->cfg.ffn_channels, bins = g->cfg.istft_n_fft / 2 + 1;
  const bool fp32 = g->precision == AB_PREC_FP32, linear = g->cfg.kind == AB_GEN_VOCOS_LINEAR;
  const size_t el = (size_t)B * T;
  Carve c{base};
  VocosWs v = {};
  v.X = c.take(el * D * 4);
  v.Y = c.take(el * D * 4);
  v.H = c.take(fp32 ? el * D * 4 : tc_act_image_bytes(B, D, T));
  if (linear) {
    v.I = c.take(fp32 ? el * F * 4 : tc_act_image_bytes(B, F, T));
    if (w) *w = v;
    return c.off;
  }
  const size_t ist = ab_istft_workspace_bytes(g->istft, B, T);
  if (ist == 0) return 0;
  v.I = c.take(fp32 ? el * std::max(F, 2 * bins) * 4 : tc_act_image_bytes(B, F, T));
  v.S = c.take(el * bins * 8);
  v.ist = c.take<char>(ist);
  v.ist_bytes = align_up(ist, 256);
  if (w) *w = v;
  return c.off;
}
}  // namespace
}  // extern "C++"

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
  if (g->cfg.kind == AB_GEN_VOCOS || g->cfg.kind == AB_GEN_VOCOS_LINEAR) return vocos_layout(g, B, T, nullptr, nullptr);
  if (g->cfg.kind == AB_GEN_DIFFWAVE || g->cfg.kind == AB_GEN_RVQ) return 0;
  return gan_layout(g, B, T, nullptr, nullptr);
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
  if (g->cfg.kind == AB_GEN_FACODEC_ENCODER) return ab_facodec_encoder_frames(g, frames);
  if (g->cfg.kind == AB_GEN_VOCOS || g->cfg.kind == AB_GEN_DIFFWAVE) return frames * g->hop;
  int64_t Tn = frames;
  for (int i = 0; i < g->cfg.num_upsamples; ++i) Tn = nsf_stage_length(g, i, Tn * g->cfg.upsample_rates[i], source_frames);
  return Tn;
}

int ab_generator_set_option(ab_generator* g, const char* key, int32_t value) {
  if (!g || !key) return fail(AB_ERR_ARG, "set_option: null argument");
  if (g->cfg.kind == AB_GEN_VOCOS || g->cfg.kind == AB_GEN_VOCOS_LINEAR)
    return fail(AB_ERR_ARG, "set_option: Vocos has no execution-plan option ('%s')", key);
  if (g->cfg.kind == AB_GEN_DIFFWAVE) return fail(AB_ERR_ARG, "set_option: DiffWave has no execution-plan option ('%s')", key);
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
  static const char* kNames[14] = {"tc_conv", "conv1d_fp32", "conv_transpose1d_fp32", "activation1d", "tc_gemmconv",
                                   "tc_pointwise", "vocos_norm", "diffwave_cond", "diffwave_input", "diffwave_layer",
                                   "diffwave_tail", "facodec_prologue", "facodec_quantize", "timbre_attention"};
  // classes 5-6 are Vocos' kernels (and the Linear head's), 7-10 DiffWave's, 11 FACodec's, 12-13 FACodec's quantization and timbre encoder; the
  // redecoder's prosody transformer reports its attention in class 13; a residual VQ handle reports vq2emb in 11 and
  // quantization in 12
  const int n = g->cfg.kind == AB_GEN_FACODEC_REDECODER ? 14
                : g->cfg.kind == AB_GEN_RVQ ? 13
                : g->cfg.kind == AB_GEN_FACODEC ? (g->cfg.facodec_quantize ? 14 : 12)
                : g->cfg.kind == AB_GEN_DIFFWAVE ? 11
                : g->cfg.kind == AB_GEN_VOCOS || g->cfg.kind == AB_GEN_VOCOS_LINEAR ? 7 : 5;
  if (max_entries < n) return fail(AB_ERR_ARG, "get_profile: need room for %d entries", n);
  for (int i = 0; i < n; ++i) {
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
  *n_out = n;
  return AB_OK;
}


// block mode (resblock_fusion 2) is chosen when it computes at most this many tile rows per output row.  On HiFi-GAN
// V1 that is the k = 3 blocks at 128, 64 and 32 channels (1.23, 1.10, 1.05), the k = 7 blocks at 64 and 32 (1.39,
// 1.16) and the k = 11 block at 32 (1.31); the 64-channel k = 11 (1.88) and 128-channel k = 7 (2.29) blocks were
// slower in block mode than as pairs on an H100 (DESIGN.md §6).
static constexpr double kChainMaxRecompute = 1.5;

extern "C++" {
namespace {
// Checks every generator forward shares (ab_generator_forward[_cond], ab_facodec_inference, ab_facodec_encode)
int check_forward(const ab_generator* g, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3],
                  const float* dev_g, int64_t g_batch_stride, const float* dev_wav, const void* dev_workspace,
                  size_t workspace_bytes) {
  if (!g || !dev_mel || !dev_wav || !mel_strides) return fail(AB_ERR_ARG, "forward: null argument");
  if (dev_g != nullptr && g->cond_w < 0) return fail(AB_ERR_STATE, "forward: conditioning given but the generator has gin_channels == 0");
  if (dev_g != nullptr && g_batch_stride < g->cfg.gin_channels) return fail(AB_ERR_ARG, "forward: g row stride < gin_channels");
  if (!g->finalized) return fail(AB_ERR_STATE, "forward: finalize() the generator first");
  if (g->cfg.kind == AB_GEN_DIFFWAVE) return fail(AB_ERR_ARG, "forward: a DiffWave handle runs through ab_diffwave_forward");
  if (g->cfg.kind == AB_GEN_RVQ) return fail(AB_ERR_ARG, "forward: a residual VQ handle runs through ab_rvq_*");
  if (B <= 0 || T <= 0) return fail(AB_ERR_ARG, "forward: batch and frames must be positive (got %lld, %lld)", (long long)B, (long long)T);
  if (B > 65535) return fail(AB_ERR_UNSUPPORTED, "forward: batch %lld > 65535", (long long)B);
  // FACodec's encoder: T counts input samples, and the stages shorten the sequence
  const bool enc = g->cfg.kind == AB_GEN_FACODEC_ENCODER;
  if ((int64_t)T * (enc ? 1 : g->hop) > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "forward: sequence too long");
  const int rc = check_workspace("forward", dev_workspace, workspace_bytes, ab_generator_workspace_bytes(g, B, T));
  if (rc != AB_OK) return rc;
  if (g->cfg.kind == AB_GEN_MELGAN) {   // ReflectionPad1d(p) needs more than p samples (the reference raises a RuntimeError)
    if (T <= 3) return fail(AB_ERR_ARG, "forward: conv_pre's ReflectionPad1d(3) needs more than 3 mel frames (got %lld)", (long long)T);
    int64_t t = T;
    for (size_t i = 0; i < g->stages.size(); ++i) {
      t *= g->stages[i].u;
      for (auto& blk : g->stages[i].blocks)
        if (t <= blk.dil[0])
          return fail(AB_ERR_ARG, "forward: stage %d ResnetBlock's ReflectionPad1d(%d) needs more than %lld samples", (int)i,
                      blk.dil[0], (long long)t);
    }
  }
  return AB_OK;
}

// Vocos' layers on one workspace (vocos_layout): the backbone and the Linear heads
struct VocosForward {
  Launch& L;
  ab_generator* g;
  int64_t B;
  int Tn;
  bool tc;
  VocosWs w;
  uint16_t *Himg, *Iimg;

  VocosForward(Launch& l, int64_t b, int64_t T, const VocosWs& ws)
      : L(l), g(l.g), B(b), Tn((int)T), tc(l.g->precision != AB_PREC_FP32), w(ws),
        Himg(reinterpret_cast<uint16_t*>(ws.H)), Iimg(reinterpret_cast<uint16_t*>(ws.I)) {}

  int norm(const float* x, int dw_w, int dw_b, int ln_w, int ln_b, float* y, uint16_t* yimg) {
    return L.norm(B, g->cfg.upsample_initial_channel, Tn, x, dw_w, dw_b, ln_w, ln_b, 1e-6f, y, yimg);
  }
  // fp32 Linear over channels (k = 1 conv) of nb utterances with the GELU, layer-scale residual or time-major epilogue
  int linear_fp32(const ConvRef& c, int64_t nb, const float* x, float* y, int epi, const float* gamma) {
    return L.conv(c, nb, x, (int64_t)c.cin * Tn, Tn, 1, y, Tn, 1.0f, epi == CONV_EPI_GAMMA_RESIDUAL ? y : nullptr, nullptr,
                  1.0f, 0, epi, gamma);
  }
  // Linear over channels of nb utterances on the pointwise wgmma GEMM, from the operand image ximg
  int pointwise(const ConvRef& c, int epi, int64_t nb, const uint16_t* ximg, uint16_t* yimg, float* y,
                const float* gamma, float* spec) {
    TcPwParams p;
    p.epilogue = epi; p.ximg = ximg; p.w = g->tcptr(c.w); p.bias = g->fptr(c.b); p.gamma = gamma;
    p.yimg = yimg; p.y = y; p.spec = spec;
    p.B = (int)nb; p.Cin = c.cin; p.Cout = c.cout; p.T = Tn; p.precision = g->precision;
    const double el = (double)nb * Tn;
    const double out = epi == AB_PW_GELU ? 2.0 * el * rup16(c.cout) : epi == AB_PW_GAMMA_RESIDUAL ? 8.0 * el * c.cout
                       : epi == AB_PW_LINEAR ? 4.0 * el * c.cout : 8.0 * el * (c.cout / 2);
    return L.timed(5, 2.0 * el * c.cin * c.cout, 2.0 * el * rup16(c.cin) + 2.0 * c.cin * c.cout + out,
                   [&] { return launch_tc_pointwise(p, L.st); });
  }

  // VocosBackbone.forward (vocos.py:764-783): x = norm(embed(x)), the ConvNeXt blocks and final_layer_norm, whose output
  // is left in w.Y (fp32) or, at 16 bits, as the operand image in w.H
  int backbone(const float* dev_mel, const int64_t mel_strides[3]) {
    const VocosRef& v = g->vocos;
    const ConvRef& cpre = g->conv_pre;
    // x = norm(embed(x)) (vocos.py:764-772)
    int rc = L.on_tc(cpre) ? L.tc_conv(cpre, nullptr, B, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], nullptr,
                                       w.Y, nullptr, Tn, 1.0f, nullptr, nullptr, 1.0f, 0,
                                       Launch::conv_bytes(cpre, B, Tn, nullptr, nullptr))
                           : L.conv(cpre, B, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], w.Y, Tn, 1.0f, nullptr,
                                    nullptr, 1.0f, 0);
    if (rc == AB_OK) rc = norm(w.Y, -1, -1, v.norm_w, v.norm_b, w.X, nullptr);
    // x = x + gamma * pwconv2(gelu(pwconv1(norm(dwconv(x))))) (vocos.py:509-527)
    for (size_t i = 0; rc == AB_OK && i < v.blocks.size(); ++i) {
      const VocosBlockRef& blk = v.blocks[i];
      if (tc) {
        rc = norm(w.X, blk.dw_w, blk.dw_b, blk.ln_w, blk.ln_b, nullptr, Himg);
        if (rc == AB_OK) rc = pointwise(blk.pw1, AB_PW_GELU, B, Himg, Iimg, nullptr, nullptr, nullptr);
        if (rc == AB_OK) rc = pointwise(blk.pw2, AB_PW_GAMMA_RESIDUAL, B, Iimg, nullptr, w.X, g->fptr(blk.gamma), nullptr);
      } else {
        rc = norm(w.X, blk.dw_w, blk.dw_b, blk.ln_w, blk.ln_b, w.H, nullptr);
        if (rc == AB_OK) rc = linear_fp32(blk.pw1, B, w.H, w.I, CONV_EPI_GELU, nullptr);
        if (rc == AB_OK) rc = linear_fp32(blk.pw2, B, w.I, w.X, CONV_EPI_GAMMA_RESIDUAL, g->fptr(blk.gamma));
      }
    }
    // final_layer_norm (:781)
    if (rc == AB_OK) rc = norm(w.X, -1, -1, v.final_w, v.final_b, tc ? nullptr : w.Y, tc ? Himg : nullptr);
    return rc;
  }
};

// Vocos: the backbone, the head's Linear with S = min(exp(mag), 1e2) (cos p + i sin p) (vocos.py:343-360) and the iSTFT
int forward_vocos(Launch& L, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3], float* dev_wav,
                  void* dev_workspace) {
  ab_generator* g = L.g;
  const VocosRef& v = g->vocos;
  const int bins = g->cfg.istft_n_fft / 2 + 1;
  VocosWs w;
  if (vocos_layout(g, B, T, static_cast<char*>(dev_workspace), &w) == 0) return fail(AB_ERR_CUDA, "forward: iSTFT plan: %s", g_err);
  VocosForward f(L, B, T, w);
  int rc = f.backbone(dev_mel, mel_strides);
  if (rc == AB_OK && f.tc) rc = f.pointwise(v.head, AB_PW_SPECTRUM, B, f.Himg, nullptr, nullptr, nullptr, w.S);
  if (rc == AB_OK && !f.tc) {
    rc = f.linear_fp32(v.head, B, w.Y, w.I, CONV_EPI_NONE, nullptr);
    // [B, 2 bins, T]: the magnitude and phase halves of one utterance are bins * T apart
    for (int64_t b = 0; rc == AB_OK && b < B; ++b) {
      const float* hb = w.I + b * 2 * bins * T;
      rc = L.counted(1, [&] {
        return ab_spectral_head_forward(hb, hb + (int64_t)bins * T, nullptr, 1, bins, T, 1e2f, nullptr, nullptr, nullptr,
                                        w.S + b * T * bins * 2, L.st);
      });
    }
  }
  // ISTFT "same" (:142-167)
  return L.tail(B, rc, [&](int64_t b0, int64_t nb) {
    return L.counted(2, [&] {
      return ab_istft_forward(g->istft, w.S + b0 * T * bins * 2, nb, T, g->fptr(v.window), dev_wav + b0 * T * g->hop, w.ist,
                              w.ist_bytes, L.st);
    });
  });
}

// nn.Sequential(VocosBackbone, nn.Linear) (repcodec_model.py:108-127): the backbone, then y [B, T, out] = Linear(x), on
// the GEMM's time-major epilogue or, in fp32, the k = 1 conv's; with tail events the Linear runs in the batch chunks
int forward_vocos_linear(Launch& L, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3], float* dev_y,
                         void* dev_workspace) {
  ab_generator* g = L.g;
  const ConvRef& head = g->vocos.head;
  VocosWs w;
  vocos_layout(g, B, T, static_cast<char*>(dev_workspace), &w);
  VocosForward f(L, B, T, w);
  const int rc = f.backbone(dev_mel, mel_strides);
  const size_t img = tc_act_image_bytes(1, head.cin, T) / sizeof(uint16_t);   // one utterance's operand image
  return L.tail(B, rc, [&](int64_t b0, int64_t nb) {
    float* y = dev_y + b0 * T * head.cout;
    return f.tc ? f.pointwise(head, AB_PW_LINEAR, nb, f.Himg + b0 * img, nullptr, y, nullptr, nullptr)
                : f.linear_fp32(head, nb, w.Y + b0 * head.cin * T, y, CONV_EPI_LINEAR, nullptr);
  });
}

// The generator pipeline (HiFi-GAN, BigVGAN, NSF-HiFiGAN, the trunks, MelGAN, FACodec's generators and encoder), one
// stage helper per step.  Between stages the stage input is R[cur_r]: cin channels of Tn samples.
struct GanForward {
  Launch& L;
  ab_generator* g;
  int64_t B;
  // FACodec's generator is BigVGAN's pipeline with an activation in front of each transposed conv; its encoder the same
  // ResidualUnits with an activation and a strided conv closing each stage
  bool melgan, fac, enc, big;
  float *R[2], *U, *P[2], *TMP, *ACT;
  uint16_t *U16, *P16[2], *R16;
  const uint16_t* r_img = nullptr;   // operand image of lrelu(stage input, 0.1) when the previous stage emitted it
  uint16_t* u_img = nullptr;         // operand image of lrelu(U, 0.1) when the ConvTranspose emitted it
  int cur_r = 0, Tn, cin;

  GanForward(Launch& l, int64_t b, int64_t T, const GanWs& w) : L(l), g(l.g), B(b), Tn((int)T), cin(g->cfg.upsample_initial_channel) {
    melgan = g->cfg.kind == AB_GEN_MELGAN;
    fac = g->cfg.kind == AB_GEN_FACODEC || g->cfg.kind == AB_GEN_FACODEC_REDECODER;
    enc = g->cfg.kind == AB_GEN_FACODEC_ENCODER;
    big = g->cfg.kind == AB_GEN_BIGVGAN || fac || enc;
    R[0] = w.buf[0]; R[1] = w.buf[1]; U = w.buf[2]; P[0] = w.buf[3]; P[1] = w.buf[4]; TMP = w.buf[5]; ACT = w.buf[6];
    U16 = w.img[0]; P16[0] = w.img[1]; P16[1] = w.img[2]; R16 = w.img[3];
  }

  // conv_pre (hifigan.py:204, bigvgan.py:314), then HiFiGAN_vits' x = x + cond(g) (hifigan.py:429-430)
  int pre(const float* dev_mel, const int64_t mel_strides[3], const uint16_t* x_img, const float* dev_g, int64_t g_batch_stride) {
    const ConvRef& cpre = g->conv_pre;
    const int C0 = cin;
    // HiFi-GAN: a tensor-core stage-0 ConvTranspose reads lrelu(x, 0.1) -> conv_pre emits that operand image, unless the
    // conditioning add changes x after it
    const bool pre_img = !big && !melgan && dev_g == nullptr && L.on_tc(cpre) && !g->stages.empty() && g->stages[0].has_up &&
                         L.on_tc(g->stages[0].up) && (C0 % 16) == 0 && tc_can_emit_image(0, cpre.cin, cpre.cout, cpre.k, cpre.d);
    int rc = L.on_tc(cpre) ? L.tc_conv(cpre, nullptr, B, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], x_img, R[0],
                                       pre_img ? R16 : nullptr, Tn, 1.0f, nullptr, nullptr, 1.0f, 0,
                                       Launch::conv_bytes(cpre, B, Tn, nullptr, nullptr) + (pre_img ? 2.0 * B * Tn * C0 : 0.0))
                           : L.conv(cpre, B, dev_mel, mel_strides[0], mel_strides[1], mel_strides[2], R[0], Tn, 1.0f, nullptr,
                                    nullptr, 1.0f, 0);
    if (rc != AB_OK) return rc;
    if (dev_g != nullptr) {
      rc = L.counted(1, [&] {
        return launch_cond_add(R[0], dev_g, g_batch_stride, g->fptr(g->cond_w), g->fptr(g->cond_b), (int)B, C0,
                               g->cfg.gin_channels, Tn, L.st);
      });
      if (rc != AB_OK) return rc;
    }
    if (pre_img) r_img = R16;
    return AB_OK;
  }

  // x = leaky_relu(x, 0.1) (HiFi-GAN only) ; x = ups[i](x)   (hifigan.py:206-207, bigvgan.py:316-318) into U, FACodec's
  // Activation1d in front (facodec.py:224-232); MelGAN: leaky_relu(x, 0.2), padding u//2 + u%2 (melgan.py:72-80)
  int up(const StageRef& sg) {
    u_img = nullptr;
    if (!sg.has_up) {
      std::swap(U, R[cur_r]);   // AB_GEN_TRUNK: the blocks read conv_pre's output in place
      return AB_OK;
    }
    const bool up_tc = L.on_tc(sg.up);
    const float* up_x = R[cur_r];
    if (fac) {   // the activation writes the operand image the tensor-core ConvTranspose reads, or fp32
      const bool img = up_tc && (cin % 16) == 0;
      const int rc = img ? L.snake(sg.act, B, R[cur_r], nullptr, cin, Tn, P16[0]) : L.snake(sg.act, B, R[cur_r], ACT, cin, Tn);
      if (rc != AB_OK) return rc;
      r_img = img ? P16[0] : nullptr;
      up_x = ACT;
    }
    const float pre_slope = big ? 1.0f : melgan ? 0.2f : 0.1f;
    const int pad = melgan || fac ? sg.u / 2 + sg.u % 2 : (sg.up.k - sg.u) / 2;
    // HiFi-GAN: every consumer of U applies lrelu(., 0.1) first (hifigan.py:95) -> emit that operand image
    if (up_tc) u_img = (!big && !melgan && tc_can_emit_image(1, cin, sg.ch, sg.up.k, sg.u)) ? U16 : nullptr;
    const double eo = (double)B * sg.ch * Tn * sg.u;
    return L.timed(up_tc ? 4 : 2, 2.0 * eo * cin * ((double)sg.up.k / sg.u),
                   4.0 * ((double)B * cin * Tn + eo + (double)cin * sg.ch * sg.up.k), [&] {
                     if (up_tc) {
                       TcConvParams p;
                       p.mode = 1;
                       p.x = up_x; p.xsb = (int64_t)cin * Tn; p.xsc = Tn; p.xst = 1; p.pre_slope = pre_slope;
                       p.ximg = (r_img != nullptr && (cin % 16) == 0) ? r_img : nullptr;
                       p.w = g->tcptr(sg.up.w); p.bias = g->fptr(sg.up.b); p.y = U;
                       p.yimg = u_img; p.img_slope = 0.1f;
                       p.B = (int)B; p.Cin = cin; p.Cout = sg.ch; p.T = Tn; p.k = sg.up.k; p.d_or_u = sg.u;
                       p.precision = g->precision; p.pad = pad;
                       return launch_tc_conv(p, L.st);
                     }
                     ConvTParams tp;
                     tp.x = up_x; tp.w_t = g->fptr(sg.up.w); tp.bias = g->fptr(sg.up.b); tp.y = U;
                     tp.B = (int)B; tp.Cin = cin; tp.Cout = sg.ch; tp.Tin = Tn; tp.k = sg.up.k; tp.u = sg.u;
                     tp.pre_slope = pre_slope; tp.pad = pad;
                     return launch_conv_transpose1d_fp32(tp, L.st);
                   });
  }

  // NSF-HiFiGAN with a source shorter than stage i (short f0, odd source stride): the reference truncates x to the
  // source length before the ResBlocks (nsfhifigan.py:264-268).  Compact the rows of U (C channels); the operand image
  // (laid out for the untruncated length) is dropped for this stage.
  int nsf_truncate(int i, int C) {
    const int64_t Lt = nsf_stage_length(g, i, Tn, g->source_frames);
    if (Lt >= Tn) return AB_OK;
    if (Lt <= 0) return fail(AB_ERR_ARG, "forward: the f0 track leaves no samples in stage %d", i);
    AB_CUDA_TRY(cudaMemcpy2DAsync(TMP, (size_t)Lt * sizeof(float), U, (size_t)Tn * sizeof(float), (size_t)Lt * sizeof(float),
                                  (size_t)B * C, cudaMemcpyDeviceToDevice, L.st));
    std::swap(U, TMP);
    u_img = nullptr;
    Tn = (int)Lt;
    return AB_OK;
  }

  // MelGAN: x <- shortcut(x) + c2(lrelu(c1(lrelu(x, 0.2), reflect-padded, dilation 3^j), 0.2)) for each ResnetBlock
  // (melgan.py:34-47), as three launches: c1 -> TMP, c2 -> P0, shortcut + P0 -> the block output.  The outputs
  // alternate between P1 and Rout so that the stage's last block writes Rout.
  int melgan_blocks(const StageRef& sg, float* Rout) {
    const int64_t sb = (int64_t)sg.ch * Tn;
    auto run = [&](const ConvRef& c, const float* x, float* y, float slope, const float* acc_prev) -> int {
      if (!L.on_tc(c)) return L.conv(c, B, x, sb, Tn, 1, y, Tn, slope, nullptr, acc_prev, 1.0f, 0);
      const double el = (double)B * Tn;
      return L.tc_conv(c, nullptr, B, x, sb, Tn, 1, nullptr, y, nullptr, Tn, slope, nullptr, acc_prev, 1.0f, 0,
                       4.0 * el * c.cout * (1 + (acc_prev != nullptr)) + 4.0 * el * c.cin + 2.0 * c.cin * c.cout * c.k);
    };
    for (size_t j = 0; j < sg.blocks.size(); ++j) {
      const BlockRef& blk = sg.blocks[j];
      const float* cur = j == 0 ? U : ((sg.blocks.size() - j) % 2 == 0 ? Rout : P[1]);
      float* dst = (sg.blocks.size() - 1 - j) % 2 == 0 ? Rout : P[1];
      int rc = run(blk.c1[0], cur, TMP, 0.2f, nullptr);
      if (rc == AB_OK) rc = run(blk.c2[0], TMP, P[0], 0.2f, nullptr);
      if (rc == AB_OK) rc = run(blk.sc, cur, dst, 1.0f, P[0]);   // shortcut(x) + block(x)
      if (rc != AB_OK) return rc;
    }
    return AB_OK;
  }

  // The ResBlocks / AMPBlocks of stage i on U into Rout: xs = rb_0(x) ; xs += rb_j(x) ; x = xs / num_kernels
  // (hifigan.py:208-214), each block in one launch (block mode), as fused pairs or as single convs.  Sets r_img for the
  // next stage.
  int blocks(size_t i, const StageRef& sg, float* Rout) {
    const int C = sg.ch, nk = g->cfg.num_kernels;
    const int64_t sb = (int64_t)C * Tn, sc = Tn;
    bool stage_img_written = false;
    int rc;
    for (int j = 0; j < nk; ++j) {
      const BlockRef& blk = sg.blocks[j];
      const float* cur = U;
      const uint16_t* cur_img = u_img;
      int pp = 0;
      const int nd = (int)blk.dil.size();
      const bool pair = !blk.c2.empty();
      const int ncv = pair ? 2 : 1;
      // every conv of a block has a weight image or none; fused: pair / block mode (HiFi-GAN) and tc_conv launch class
      const bool blk_tc = L.on_tc(blk.c1[0]);
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
          const double el = (double)B * C * Tn;
          rc = L.timed(0, 2.0 * el * C * blk.k * ncv * nd, 4.0 * (el * (2 + (j > 0)) + (double)ncv * nd * C * C * blk.k),
                       [&] { return launch_tc_chain(cp, L.st); });
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
          const int r = blk_tc ? L.snake(*a, B, x, nullptr, C, Tn, P16[0]) : L.snake(*a, B, x, ACT, C, Tn);
          if (r != AB_OK) return r;
        }
        if (!blk_tc) return L.conv(c, B, in, sb, sc, 1, y, Tn, slope, residual, acc_prev, out_div, 0);
        return L.tc_conv(c, nullptr, B, in, sb, sc, 1, img, y, nullptr, Tn, slope, residual, acc_prev, out_div, 0,
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
        const float* accp = (last && j > 0) ? Rout : nullptr;
        const float div = (last && j == nk - 1) ? (float)nk : 1.0f;
        if (fused && !big) {
          rc = L.tc_conv(blk.c1[p], pair ? &blk.c2[p] : nullptr, B, cur, sb, sc, 1, cur_img, dst, dst_img, Tn, 0.1f, cur, accp,
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
    r_img = stage_img_written ? R16 : nullptr;
    return AB_OK;
  }

  // FACodec encoder: x = Conv1d(C, 2C, k = 2s, stride s, padding s//2 + s%2)(Activation1d(SnakeBeta)(x))
  // (facodec.py:136-154); the activation writes the operand image the tensor-core conv reads, or fp32
  int down(const StageRef& sg) {
    const ConvRef& dc = sg.up;
    const int C = cin, sd = sg.down, pad = sd / 2 + sd % 2;
    const bool dtc = L.on_tc(dc), img = dtc && (C % 16) == 0;
    int rc = img ? L.snake(sg.act, B, R[cur_r], nullptr, C, Tn, P16[0]) : L.snake(sg.act, B, R[cur_r], ACT, C, Tn);
    if (rc != AB_OK) return rc;
    const int To = (int)encoder_stage_length(Tn, sd);
    float* dst = R[cur_r ^ 1];
    rc = L.timed(dtc ? 4 : 1, 2.0 * B * To * dc.cout * dc.cin * dc.k,
                 4.0 * ((double)B * C * Tn + (double)B * dc.cout * To + (double)dc.cin * dc.cout * dc.k), [&] {
                   if (dtc) {
                     TcConvParams p;
                     p.mode = 2;
                     p.x = ACT; p.xsb = (int64_t)C * Tn; p.xsc = Tn; p.xst = 1; p.ximg = img ? P16[0] : nullptr;
                     p.w = g->tcptr(dc.w); p.bias = g->fptr(dc.b); p.y = dst;
                     p.B = (int)B; p.Cin = C; p.Cout = dc.cout; p.T = Tn; p.k = dc.k; p.d_or_u = sd; p.pad = pad;
                     p.precision = g->precision;
                     return launch_tc_conv(p, L.st);
                   }
                   ConvParams p;
                   p.x = ACT; p.xsb = (int64_t)C * Tn; p.xsc = Tn; p.xst = 1;
                   p.w_t = g->fptr(dc.w); p.bias = g->fptr(dc.b); p.residual = nullptr; p.acc_prev = nullptr; p.y = dst;
                   p.B = (int)B; p.Cin = C; p.Cout = dc.cout; p.T = Tn; p.k = dc.k; p.d = 1;
                   p.pre_slope = 1.0f; p.out_div = 1.0f; p.post_tanh = 0;
                   return launch_conv1d_strided_fp32(p, sd, pad, L.st);
                 });
    if (rc != AB_OK) return rc;
    cur_r ^= 1;
    Tn = To;
    cin = dc.cout;
    return AB_OK;
  }

  // post: leaky_relu(x) with the DEFAULT slope 0.01 (hifigan.py:215) or activation_post (bigvgan.py:327); conv_post;
  // tanh.  conv_post runs in the tail chunks (Launch::tail).
  int post(float* dev_wav) {
    const float* xin = R[cur_r];
    const int64_t sb = (int64_t)cin * Tn, sc = Tn;
    if (big) {
      const int rc = L.snake(g->act_post, B, xin, ACT, cin, Tn);
      if (rc != AB_OK) return rc;
      xin = ACT;
    }
    const ConvRef& cpost = g->conv_post;
    const float post_slope = big ? 1.0f : melgan ? 0.2f : 0.01f;
    const int post_tanh = g->cfg.kind == AB_GEN_TRUNK || enc ? 0 : 1;
    return L.tail(B, AB_OK, [&](int64_t b0, int64_t nb) {
      const float* x = xin + b0 * sb;
      float* y = dev_wav + b0 * cpost.cout * Tn;
      return L.on_tc(cpost) ? L.tc_conv(cpost, nullptr, nb, x, sb, sc, 1, nullptr, y, nullptr, Tn, post_slope, nullptr, nullptr,
                                        1.0f, post_tanh, Launch::conv_bytes(cpost, nb, Tn, nullptr, nullptr))
                            : L.conv(cpost, nb, x, sb, sc, 1, y, Tn, post_slope, nullptr, nullptr, 1.0f, post_tanh);
    });
  }
};

// A checked forward of any generator kind but DiffWave.  x_img (FACodec at tensor-core precision): conv_pre's input as
// an operand image, in place of dev_mel.
int forward_generator(Launch& L, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3], const float* dev_g,
                      int64_t g_batch_stride, float* dev_wav, void* dev_workspace, size_t workspace_bytes,
                      const uint16_t* x_img = nullptr) {
  ab_generator* g = L.g;
  int rc = check_forward(g, dev_mel, B, T, mel_strides, dev_g, g_batch_stride, dev_wav, dev_workspace, workspace_bytes);
  if (rc != AB_OK) return rc;
  if (g->cfg.kind == AB_GEN_VOCOS) return forward_vocos(L, dev_mel, B, T, mel_strides, dev_wav, dev_workspace);
  if (g->cfg.kind == AB_GEN_VOCOS_LINEAR) return forward_vocos_linear(L, dev_mel, B, T, mel_strides, dev_wav, dev_workspace);
  GanWs w;
  gan_layout(g, B, T, static_cast<char*>(dev_workspace), &w);
  GanForward f(L, B, T, w);
  if ((rc = f.pre(dev_mel, mel_strides, x_img, dev_g, g_batch_stride)) != AB_OK) return rc;
  for (size_t i = 0; i < g->stages.size(); ++i) {
    const StageRef& sg = g->stages[i];
    if ((rc = f.up(sg)) != AB_OK) return rc;
    f.Tn *= sg.u;
    if ((rc = f.nsf_truncate((int)i, sg.ch)) != AB_OK) return rc;
    float* Rout = f.R[f.cur_r ^ 1];
    if ((rc = f.melgan ? f.melgan_blocks(sg, Rout) : f.blocks(i, sg, Rout)) != AB_OK) return rc;
    f.cur_r ^= 1;
    f.cin = sg.ch;
    if (sg.down && (rc = f.down(sg)) != AB_OK) return rc;
  }
  return f.post(dev_wav);
}
}  // namespace
}  // extern "C++"

int ab_generator_forward(ab_generator* g, const float* dev_mel, int64_t B, int64_t T,
                         const int64_t mel_strides[3], float* dev_wav, void* dev_workspace,
                         size_t workspace_bytes, void* stream) {
  if (g && (g->cfg.kind == AB_GEN_FACODEC || g->cfg.kind == AB_GEN_FACODEC_REDECODER))
    return fail(AB_ERR_ARG, "forward: a FACodec handle runs through ab_facodec_inference");
  if (g && g->cfg.kind == AB_GEN_FACODEC_ENCODER)
    return fail(AB_ERR_ARG, "forward: a FACodec encoder handle runs through ab_facodec_encode");
  Launch L{g, static_cast<cudaStream_t>(stream)};
  return L.done(forward_generator(L, dev_mel, B, T, mel_strides, nullptr, 0, dev_wav, dev_workspace, workspace_bytes));
}

int ab_generator_forward_cond(ab_generator* g, const float* dev_x, int64_t B, int64_t T, const int64_t x_strides[3],
                              const float* dev_g, int64_t g_batch_stride, float* dev_wav, void* dev_workspace,
                              size_t workspace_bytes, void* stream) {
  if (g && (g->cfg.kind == AB_GEN_FACODEC || g->cfg.kind == AB_GEN_FACODEC_REDECODER))
    return fail(AB_ERR_ARG, "forward: a FACodec handle runs through ab_facodec_inference");
  if (g && g->cfg.kind == AB_GEN_FACODEC_ENCODER)
    return fail(AB_ERR_ARG, "forward: a FACodec encoder handle runs through ab_facodec_encode");
  Launch L{g, static_cast<cudaStream_t>(stream)};
  return L.done(forward_generator(L, dev_x, B, T, x_strides, dev_g, g_batch_stride, dev_wav, dev_workspace, workspace_bytes));
}

// ---------------------------------------------------------------------------
// DiffWave
// ---------------------------------------------------------------------------
extern "C++" {
namespace {
// Workspace: the fp32 residual stream in two buffers X0 / X1 (layer l reads one and writes the other), the skip sum,
// the upsampled mel [B, n_mel, L], then the diffusion projections [n_steps][layers][C] and the step values.
struct DiffWaveWs {
  float *X[2], *S, *M, *D, *steps;
};

size_t diffwave_layout(const ab_generator* g, int64_t B, int64_t T, int n_steps, char* base, DiffWaveWs* w) {
  const size_t L = (size_t)T * g->hop;
  Carve c{base};
  DiffWaveWs v;
  for (float*& x : v.X) x = c.take(B * DW_CHANNELS * L * 4);
  v.S = c.take(B * DW_CHANNELS * L * 4);
  v.M = c.take(B * (size_t)g->cfg.n_mel * L * 4);
  v.D = c.take((size_t)n_steps * g->cfg.num_layers * DW_CHANNELS * 4);
  v.steps = c.take((size_t)n_steps * 4);
  if (w) *w = v;
  return c.off;
}

int diffwave_check(const ab_generator* g, int64_t B, int64_t T, int n_steps, void* ws, size_t ws_bytes, const char* what) {
  if (!g) return fail(AB_ERR_ARG, "%s: null handle", what);
  if (g->cfg.kind != AB_GEN_DIFFWAVE) return fail(AB_ERR_ARG, "%s: not a DiffWave handle", what);
  if (!g->finalized) return fail(AB_ERR_STATE, "%s: finalize() the generator first", what);
  if (B <= 0 || T <= 0 || B > 65535) return fail(AB_ERR_ARG, "%s: batch %lld / frames %lld out of range", what, (long long)B, (long long)T);
  if (T * g->hop > (1ll << 30) || B * (int64_t)std::max(DW_CHANNELS, g->cfg.n_mel) * T * g->hop > (1ll << 40))
    return fail(AB_ERR_UNSUPPORTED, "%s: sequence too long", what);
  return check_workspace(what, ws, ws_bytes, diffwave_layout(g, B, T, n_steps, nullptr, nullptr));
}

// ab_diffwave_condition: the upsampled mel and the diffusion projections of every step
int diffwave_condition(Launch& L, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3],
                       const float* host_steps, int32_t n_steps, void* ws, size_t ws_bytes) {
  ab_generator* g = L.g;
  if (!dev_mel || !mel_strides || !host_steps) return fail(AB_ERR_ARG, "diffwave_condition: null argument");
  if (n_steps <= 0 || n_steps > 65535) return fail(AB_ERR_ARG, "diffwave_condition: n_steps %d out of range", n_steps);
  int rc = diffwave_check(g, B, T, n_steps, ws, ws_bytes, "diffwave_condition");
  if (rc != AB_OK) return rc;
  for (int i = 0; i < n_steps; ++i)   // the reference indexes the table at floor(t) and ceil(t)
    if (!(host_steps[i] >= 0.f) || !(ceilf(host_steps[i]) < (float)g->cfg.embedding_rows))
      return fail(AB_ERR_ARG, "diffwave_condition: diffusion step %g outside the embedding table [0, %d)", host_steps[i],
                  g->cfg.embedding_rows);
  cudaStream_t st = L.st;
  DiffWaveWs w;
  diffwave_layout(g, B, T, n_steps, static_cast<char*>(ws), &w);
  const DiffWaveRef& d = g->dw;
  const int nm = g->cfg.n_mel, nl = g->cfg.num_layers, C = DW_CHANNELS;
  g->dw.cond_B = 0;
  AB_CUDA_TRY(cudaMemcpyAsync(w.steps, host_steps, (size_t)n_steps * 4, cudaMemcpyHostToDevice, st));
  DwUpsampleParams up;
  up.mel = dev_mel; up.msb = mel_strides[0]; up.msc = mel_strides[1]; up.mst = mel_strides[2];
  up.w1 = g->fptr(d.wup[0]); up.b1 = g->fptr(d.bup[0]); up.w2 = g->fptr(d.wup[1]); up.b2 = g->fptr(d.bup[1]);
  up.out = w.M; up.B = (int)B; up.n_mel = nm; up.F = (int)T; up.f1 = g->cfg.upsample_rates[0]; up.f2 = g->cfg.upsample_rates[1];
  const double Ls = (double)T * g->hop;
  rc = L.timed(7, 2.0 * B * nm * Ls * 36.0, 4.0 * B * nm * (T + Ls), [&] { return launch_dw_upsample(up, st); });
  if (rc != AB_OK) return rc;
  DwEmbedParams e;
  const float* proj = reinterpret_cast<const float*>(g->arena + d.packed_offset) + nl * dw_layer_packed_floats(nm);
  e.steps = w.steps; e.table = g->fptr(d.table); e.w1 = g->fptr(d.wp1); e.b1 = g->fptr(d.bp1);
  e.w2 = g->fptr(d.wp2); e.b2 = g->fptr(d.bp2); e.wd = proj; e.bd = proj + (size_t)nl * C * 512; e.d = w.D; e.layers = nl;
  rc = L.timed(7, 2.0 * n_steps * (128.0 * 512 + 512.0 * 512 + (double)nl * C * 512),
               4.0 * (128.0 * 512 + 512.0 * 512 + (double)nl * C * 512 + (double)n_steps * nl * C),
               [&] { return launch_dw_embed(e, n_steps, st); });
  if (rc != AB_OK) return rc;
  g->dw.cond_B = B; g->dw.cond_T = T; g->dw.cond_rows = n_steps;
  return AB_OK;
}

// ab_diffwave_step: one pass of the network and the sampler update
int diffwave_step(Launch& L, float* dev_audio, int64_t B, int64_t T, int32_t step_row, float c1, float c2, float sigma,
                  const float* dev_noise, float* dev_eps, void* ws, size_t ws_bytes) {
  ab_generator* g = L.g;
  if (!dev_audio) return fail(AB_ERR_ARG, "diffwave_step: null audio");
  if (!g || g->cfg.kind != AB_GEN_DIFFWAVE) return fail(AB_ERR_ARG, "diffwave_step: not a DiffWave handle");
  if (g->dw.cond_B != B || g->dw.cond_T != T)
    return fail(AB_ERR_STATE, "diffwave_step: run ab_diffwave_condition for this batch (%lld x %lld frames) first", (long long)B,
                (long long)T);
  const int rows = g->dw.cond_rows;
  int rc = diffwave_check(g, B, T, rows, ws, ws_bytes, "diffwave_step");
  if (rc != AB_OK) return rc;
  if (step_row < -1 || step_row >= rows || (step_row == -1 && rows != B))
    return fail(AB_ERR_ARG, "diffwave_step: step row %d with %d conditioned steps and batch %lld", step_row, rows, (long long)B);
  cudaStream_t st = L.st;
  DiffWaveWs w;
  diffwave_layout(g, B, T, rows, static_cast<char*>(ws), &w);
  const DiffWaveRef& d = g->dw;
  const int nm = g->cfg.n_mel, nl = g->cfg.num_layers, C = DW_CHANNELS;
  const int64_t Ls = T * g->hop;
  const double el = (double)B * Ls;
  rc = L.timed(8, 2.0 * el * C, 4.0 * el * (1 + C),
               [&] { return launch_dw_input(dev_audio, g->fptr(d.win), g->fptr(d.bin), w.X[0], (int)B, Ls, st); });
  for (int l = 0; rc == AB_OK && l < nl; ++l) {
    DwLayerParams p;
    p.x_in = w.X[l & 1]; p.x_out = w.X[(l + 1) & 1]; p.skip = w.S; p.cond = w.M;
    p.d = w.D + ((size_t)(step_row < 0 ? 0 : step_row) * nl + l) * C;
    p.d_bstride = step_row < 0 ? (int64_t)nl * C : 0;
    const DwLayerPack lp = dw_layer_pack(g->arena + d.packed_offset, nm, l);
    p.w1 = lp.w1; p.b1 = lp.b1; p.w2 = lp.w2; p.b2 = lp.b2; p.w1h = lp.w1h; p.w2h = lp.w2h; p.precision = g->precision;
    p.B = (int)B; p.n_mel = nm; p.dil = d.layers[l].dil; p.first = l == 0; p.L = Ls;
    // x read (3 taps, once from HBM), x written, skip read + written (stored by the first layer), mel read
    rc = L.timed(9, 2.0 * el * 2 * C * (3 * C + nm + C), 4.0 * el * (C * (l == 0 ? 3 : 4) + nm),
                 [&] { return launch_dw_layer(p, st); });
  }
  if (rc != AB_OK) return rc;
  DwTailParams t;
  t.skip = w.S; t.wsk = g->fptr(d.wsk); t.bsk = g->fptr(d.bsk); t.wo = g->fptr(d.wo); t.bo = g->fptr(d.bo);
  t.skip_div = (float)sqrt((double)nl);
  t.B = (int)B; t.L = Ls; t.eps = dev_eps; t.audio = dev_audio; t.noise = dev_noise; t.c1 = c1; t.c2 = c2; t.sigma = sigma;
  return L.timed(10, 2.0 * el * (C * C + C), 4.0 * el * (C + (dev_eps ? 1 : 2) + (dev_noise ? 1 : 0)),
                 [&] { return launch_dw_tail(t, st); });
}
}  // namespace
}  // extern "C++"

size_t ab_diffwave_workspace_bytes(const ab_generator* g, int64_t B, int64_t T, int32_t n_steps) {
  if (!g || g->cfg.kind != AB_GEN_DIFFWAVE || B <= 0 || T <= 0 || n_steps <= 0) return 0;
  return diffwave_layout(g, B, T, n_steps, nullptr, nullptr);
}

int ab_diffwave_condition(ab_generator* g, const float* dev_mel, int64_t B, int64_t T, const int64_t mel_strides[3],
                          const float* host_steps, int32_t n_steps, void* ws, size_t ws_bytes, void* stream) {
  Launch L{g, static_cast<cudaStream_t>(stream)};
  return L.done(diffwave_condition(L, dev_mel, B, T, mel_strides, host_steps, n_steps, ws, ws_bytes));
}

int ab_diffwave_step(ab_generator* g, float* dev_audio, int64_t B, int64_t T, int32_t step_row, float c1, float c2,
                     float sigma, const float* dev_noise, float* dev_eps, void* ws, size_t ws_bytes, void* stream) {
  Launch L{g, static_cast<cudaStream_t>(stream)};
  return L.done(diffwave_step(L, dev_audio, B, T, step_row, c1, c2, sigma, dev_noise, dev_eps, ws, ws_bytes));
}

int ab_diffwave_forward(ab_generator* g, const float* dev_audio, int64_t B, int64_t T, const float* dev_mel,
                        const int64_t mel_strides[3], const float* host_steps, int32_t n_steps, float* dev_eps, void* ws,
                        size_t ws_bytes, void* stream) {
  if (!dev_eps || !dev_audio) return fail(AB_ERR_ARG, "diffwave_forward: null argument");
  if (n_steps != 1 && n_steps != B)
    return fail(AB_ERR_ARG, "diffwave_forward: %d diffusion steps for a batch of %lld (need 1 or the batch)", n_steps, (long long)B);
  Launch L{g, static_cast<cudaStream_t>(stream)};
  // the conditioning's count stands when the step then fails
  const int rc = L.done(diffwave_condition(L, dev_mel, B, T, mel_strides, host_steps, n_steps, ws, ws_bytes));
  if (rc != AB_OK) return rc;
  // the audio is only read when eps is given
  return L.done(diffwave_step(L, const_cast<float*>(dev_audio), B, T, n_steps == 1 ? 0 : -1, 1.f, 0.f, 0.f, nullptr, dev_eps,
                              ws, ws_bytes));
}

// ---------------------------------------------------------------------------
// FACodec decoder
// ---------------------------------------------------------------------------
// redecoder: 0 the entry serves the decoder only, 1 the decoder and the redecoder, 2 the redecoder only
static int facodec_check(const ab_generator* g, int64_t B, int64_t T, const char* what, int redecoder = 0) {
  if (!g) return fail(AB_ERR_ARG, "%s: null handle", what);
  const bool ok = redecoder == 2 ? g->cfg.kind == AB_GEN_FACODEC_REDECODER
                  : g->cfg.kind == AB_GEN_FACODEC || (redecoder == 1 && g->cfg.kind == AB_GEN_FACODEC_REDECODER);
  if (!ok)
    return fail(AB_ERR_ARG, "%s: not a FACodec %shandle", what,
                redecoder == 2 ? "redecoder " : redecoder == 1 ? "decoder or redecoder " : "");
  if (!g->finalized) return fail(AB_ERR_STATE, "%s: finalize() the generator first", what);
  if (B <= 0 || T <= 0 || B > 65535) return fail(AB_ERR_ARG, "%s: batch %lld / frames %lld out of range", what, (long long)B, (long long)T);
  if (T * g->hop > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "%s: sequence too long", what);
  return AB_OK;
}

int ab_facodec_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_q, int64_t B,
                      int64_t T, int32_t use_residual, float* dev_out, void* stream) {
  int rc = facodec_check(g, B, T, "facodec_vq2emb");
  if (rc != AB_OK) return rc;
  if (!dev_codes || !codes_strides || !dev_out) return fail(AB_ERR_ARG, "facodec_vq2emb: null argument");
  const int* nq = g->cfg.vq_num_q;
  const int n_all = nq[0] + nq[1] + nq[2], n_pc = nq[0] + nq[1];
  // facodec.py:564: the residual group joins when the decoder has one and use_residual_code is set
  const bool resid = use_residual && nq[2] > 0;
  if (n_q != n_all && !(!use_residual && n_q == n_pc))
    return fail(AB_ERR_ARG, "facodec_vq2emb: %d code rows; the decoder has %d (%d prosody, %d content, %d residual)", n_q,
                n_all, nq[0], nq[1], nq[2]);
  FacVqParams p;
  memset(&p, 0, sizeof(p));
  p.codes = dev_codes; p.cs0 = codes_strides[0]; p.cs1 = codes_strides[1]; p.cs2 = codes_strides[2];
  p.nq = resid ? n_all : n_pc;
  for (int q = 0; q < p.nq; ++q) {
    const FacodecLayerRef& l = g->fac.layers[q];
    p.cb[q] = g->fptr(l.cb); p.w[q] = g->fptr(l.out_proj.w); p.bias[q] = g->fptr(l.out_proj.b); p.rows[q] = l.rows;
  }
  p.group_end[0] = nq[0]; p.group_end[1] = n_pc; p.group_end[2] = n_all;
  p.ngroups = resid ? 3 : 2;
  p.B = (int)B; p.C = g->cfg.n_mel; p.T = (int)T; p.D = g->cfg.vq_codebook_dim; p.out = dev_out;
  Launch L{g, static_cast<cudaStream_t>(stream)};
  const double el = (double)B * T;
  rc = L.timed(11, 2.0 * el * p.nq * p.C * p.D, 8.0 * el * p.nq + 4.0 * el * p.C + 4.0 * p.nq * (double)p.C * (p.D + 1),
               [&] { return launch_facodec_vq2emb(p, L.st); });
  return L.done(rc);
}

int ab_facodec_inference(ab_generator* g, const float* dev_x, int64_t B, int64_t T, const int64_t x_strides[3],
                         const float* dev_spk, int64_t spk_row_stride, float* dev_wav, void* dev_workspace,
                         size_t workspace_bytes, void* stream) {
  int rc = facodec_check(g, B, T, "facodec_inference", 1);
  if (rc == AB_OK && (!dev_x || !x_strides || !dev_spk || !dev_wav))
    rc = fail(AB_ERR_ARG, "facodec_inference: null argument");
  const int C = g ? g->cfg.n_mel : 0;
  if (rc == AB_OK && spk_row_stride < C) rc = fail(AB_ERR_ARG, "facodec_inference: speaker-embedding row stride < %d", C);
  if (rc == AB_OK)
    rc = check_workspace("facodec_inference", dev_workspace, workspace_bytes, ab_generator_workspace_bytes(g, B, T));
  if (rc != AB_OK) {
    if (g) g->tail_events.clear();
    return rc;
  }
  Launch L{g, static_cast<cudaStream_t>(stream)};
  GanWs w;
  gan_layout(g, B, T, static_cast<char*>(dev_workspace), &w);
  // conv_pre reads the FiLM output as its operand image when it runs on the wgmma kernel
  const bool img = L.on_tc(g->conv_pre);
  const double el = (double)B * T;
  rc = L.timed(11, 4.0 * B * C * C, 4.0 * (2.0 * C * C + B * 3.0 * C), [&] {
    return launch_facodec_style(dev_spk, spk_row_stride, g->fptr(g->fac.style_w), g->fptr(g->fac.style_b), w.style, (int)B, C,
                                L.st);
  });
  if (rc == AB_OK) {
    FacFilmParams p;
    p.x = dev_x; p.xsb = x_strides[0]; p.xsc = x_strides[1]; p.xst = x_strides[2];
    p.style = w.style; p.y = img ? nullptr : reinterpret_cast<float*>(w.film);
    p.yimg = img ? reinterpret_cast<uint16_t*>(w.film) : nullptr; p.bf16 = g->precision == AB_PREC_TC_BF16;
    p.B = (int)B; p.C = C; p.T = (int)T;
    rc = L.timed(11, 10.0 * el * C, 4.0 * el * C + (img ? 2.0 * el * rup16(C) : 4.0 * el * C),
                 [&] { return launch_facodec_film(p, L.st); });
  }
  if (rc != AB_OK) {
    g->tail_events.clear();
    return rc;
  }
  const int64_t strides[3] = {(int64_t)C * T, T, 1};
  return L.done(forward_generator(L, reinterpret_cast<const float*>(w.film), B, T, strides, nullptr, 0, dev_wav, dev_workspace,
                                  workspace_bytes, img ? reinterpret_cast<const uint16_t*>(w.film) : nullptr));
}

// FACodecDecoder.forward(vq=True): workspace of the timbre encoder.  S the fp32 stream [B, 256, T]; H a LayerNorm's
// output (fp32, or the operand image at 16 bits) and last_ln's output; QKV [B, 768, T]; A the attention output (fp32 or
// image); F ffn_1's fp32 output [B, 1024, T] and FI the image of its ReLU.
struct TimbreWs {
  float *S, *H, *QKV, *A, *F;
  uint16_t* FI;
};
extern "C++" {
static TimbreWs timbre_layout(Carve& c, int64_t B, int64_t T) {
  const size_t el = (size_t)B * T, C = FAC_TIMBRE_C;
  TimbreWs w;
  w.S = c.take(el * C * 4);
  w.H = c.take(el * C * 4);
  w.QKV = c.take(el * 3 * C * 4);
  w.A = c.take(el * C * 4);
  w.F = c.take(el * 4 * C * 4);
  w.FI = c.take<uint16_t>(tc_act_image_bytes(B, 4 * C, T));
  return w;
}

// FACodecRedecoder.vq2emb: the prosody transformer's workspace (TimbreWs), then the nine style vectors [9][B][2C]
// (layer l's ln_1 at 2l, its ln_2 at 2l + 1, last_ln at 8)
static TimbreWs redecoder_layout(Carve& c, int64_t B, int64_t T, float** styles) {
  const TimbreWs w = timbre_layout(c, B, T);
  *styles = c.take((size_t)9 * B * 2 * FAC_TIMBRE_C * sizeof(float));
  return w;
}

// The four pre-LN layers of a FACodec transformer on the fp32 stream w.S (transformer.py:122-151): the decoder's timbre
// encoder and the redecoder's prosody encoder differ only in their LayerNorms.  norm(layer, i, y, yimg) runs the
// layer's ln_1 (i = 0) or ln_2 (i = 1) on w.S into y (fp32) or the operand image yimg.  Per layer: ln_1, the QKV GEMM,
// the attention, out_proj onto S, ln_2, ffn_1 (k = 5; at 16 bits it also writes the image of its ReLU), ffn_2 onto S.
// tc: the GEMMs take 16-bit operands (the handle's precision); false runs them and the attention in fp32 on CUDA cores.
template <class Norm>
static int facodec_transformer_layers(Launch& L, const TimbreWs& w, int64_t B, int Tn,
                                      const std::vector<TimbreLayerRef>& layers, bool tc, Norm norm) {
  ab_generator* g = L.g;
  const int C = FAC_TIMBRE_C;
  const double el = (double)B * Tn;
  const uint16_t* Himg = reinterpret_cast<const uint16_t*>(w.H);
  // a GEMM (k = 1) or the k = 5 ffn_1 conv: x fp32 or ximg, y = (bias + W x) [+ residual = y]; all in profile class 0 at
  // 16 bits, and the image of relu(y)
  auto gemm = [&](const ConvRef& c, const float* x, const uint16_t* ximg, float* y, bool residual, float pre_slope,
                  uint16_t* yimg) -> int {
    // residual in place: each output element is read and then written by the same thread
    if (!tc) return L.conv(c, B, x, (int64_t)c.cin * Tn, Tn, 1, y, Tn, pre_slope, residual ? y : nullptr, nullptr, 1.0f, 0);
    return L.tc_conv(c, nullptr, B, nullptr, 0, 0, 0, ximg, y, yimg, Tn, 1.0f, nullptr, residual ? y : nullptr, 1.0f, 0,
                     el * c.cin * 2.0 + 4.0 * el * c.cout * (residual ? 2 : 1) + (yimg ? 2.0 * el * c.cout : 0.0) +
                         2.0 * c.cin * c.cout * c.k,
                     0, 0.0f);
  };
  int rc;
  for (const TimbreLayerRef& t : layers) {
    // x = x + out_proj(MHA(LN1(x)))
    if ((rc = norm(t, 0, tc ? nullptr : w.H, tc ? reinterpret_cast<uint16_t*>(w.H) : nullptr)) != AB_OK) return rc;
    if ((rc = gemm(t.qkv, w.H, Himg, w.QKV, false, 1.0f, nullptr)) != AB_OK) return rc;
    rc = L.timed(13, 4.0 * B * (double)Tn * Tn * C, 4.0 * el * 3 * C + (tc ? 2.0 : 4.0) * el * C, [&] {
      return launch_facodec_attention(w.QKV, tc ? nullptr : w.A, tc ? reinterpret_cast<uint16_t*>(w.A) : nullptr,
                                      g->precision == AB_PREC_TC_BF16, (int)B, Tn, L.st);
    });
    if (rc != AB_OK) return rc;
    if ((rc = gemm(t.out_proj, w.A, reinterpret_cast<const uint16_t*>(w.A), w.S, true, 1.0f, nullptr)) != AB_OK) return rc;
    // x = x + ffn_2(relu(ffn_1(LN2(x))))
    if ((rc = norm(t, 1, tc ? nullptr : w.H, tc ? reinterpret_cast<uint16_t*>(w.H) : nullptr)) != AB_OK) return rc;
    if ((rc = gemm(t.ffn_1, w.H, Himg, w.F, false, 1.0f, tc ? w.FI : nullptr)) != AB_OK) return rc;
    if ((rc = gemm(t.ffn_2, w.F, w.FI, w.S, true, 0.0f, nullptr)) != AB_OK) return rc;
  }
  return AB_OK;
}
}  // extern "C++"

size_t ab_facodec_quantize_workspace_bytes(const ab_generator* g, int64_t B, int64_t T) {
  if (!g || g->cfg.kind != AB_GEN_FACODEC || !g->cfg.facodec_quantize || B <= 0 || T <= 0) return 0;
  Carve c{nullptr};
  timbre_layout(c, B, T);
  if (g->cfg.facodec_prosody_encoder) c.take((size_t)B * T * FAC_TIMBRE_C * sizeof(float));   // melspec_encoder's output
  return c.off;
}

// FACodecDecoder.forward(vq=True) (dev_pf null) and FACodecDecoderV2.forward(vq=True) (dev_pf: the prosody feature)
static int facodec_quantize_impl(ab_generator* g, const char* what, const float* dev_x, const int64_t x_strides[3],
                                 const float* dev_pf, const int64_t pf_strides[3], int64_t B, int64_t T,
                                 int32_t n_quantizers, float* dev_emb_out, int64_t* dev_codes_out,
                                 float* dev_quantized_out, float* dev_spk_out, void* dev_workspace,
                                 size_t workspace_bytes, void* stream) {
  int rc = facodec_check(g, B, T, what);
  if (rc != AB_OK) return rc;
  if (!g->cfg.facodec_quantize) return fail(AB_ERR_STATE, "%s: the handle was created without facodec_quantize", what);
  const bool v2 = g->cfg.facodec_prosody_encoder != 0;
  if (v2 && !dev_pf)
    return fail(AB_ERR_STATE, "%s: the handle serves FACodecDecoderV2, whose forward reads the prosody feature "
                              "(ab_facodec_quantize_prosody)", what);
  if (!v2 && dev_pf)
    return fail(AB_ERR_STATE, "%s: the handle was created without facodec_prosody_encoder", what);
  if (!dev_x || !x_strides || (v2 && !pf_strides) || !dev_emb_out || !dev_codes_out || !dev_quantized_out || !dev_spk_out)
    return fail(AB_ERR_ARG, "%s: null argument", what);
  if (n_quantizers < 1) return fail(AB_ERR_ARG, "%s: n_quantizers %d < 1 (no layer would run)", what, n_quantizers);
  if (B > FAC_PE_ROWS)   // PositionalEncoding adds pe[:B] (transformer.py:43-45)
    return fail(AB_ERR_ARG, "%s: batch %lld > %d, the rows of the positional encoding", what, (long long)B, FAC_PE_ROWS);
  rc = check_workspace(what, dev_workspace, workspace_bytes, ab_facodec_quantize_workspace_bytes(g, B, T));
  if (rc != AB_OK) return rc;
  Launch L{g, static_cast<cudaStream_t>(stream)};
  Carve ws{static_cast<char*>(dev_workspace)};
  const TimbreWs w = timbre_layout(ws, B, T);
  const int C = g->cfg.n_mel, D = g->cfg.vq_codebook_dim, Tn = (int)T;
  const double el = (double)B * T;
  auto norm = [&](int lw, int lb, float* y, uint16_t* yimg) { return L.norm(B, C, Tn, w.S, -1, -1, lw, lb, 1e-5f, y, yimg); };

  // FACodecDecoderV2 (facodec.py:1034-1038): melspec_encoder(melspec_linear(prosody_feature^T)) into P, all fp32: the
  // input projection and pe into S, four layers on S, last_ln into P
  float* P = nullptr;
  if (v2) {
    const FacodecRef& f = g->fac;
    P = ws.take((size_t)B * T * C * sizeof(float));
    FacProsodyInParams q;
    q.x = dev_pf; q.xsb = pf_strides[0]; q.xsi = pf_strides[1]; q.xst = pf_strides[2];
    q.w = g->fptr(f.mel_w); q.bias = g->fptr(f.mel_b); q.pe = g->fptr(f.pros_pe); q.y = w.S;
    q.B = (int)B; q.T = Tn;
    rc = L.timed(11, el * C * (2.0 * FAC_PROSODY_BINS + 2.0), 4.0 * el * (FAC_PROSODY_BINS + C) + 4.0 * C * (FAC_PROSODY_BINS + 2.0),
                 [&] { return launch_facodec_prosody_input(q, L.st); });
    if (rc != AB_OK) return rc;
    rc = facodec_transformer_layers(L, w, B, Tn, f.prosody, false,
                                    [&](const TimbreLayerRef& t, int i, float* y, uint16_t* yimg) {
      return i == 0 ? norm(t.ln1_w, t.ln1_b, y, yimg) : norm(t.ln2_w, t.ln2_b, y, yimg);
    });
    if (rc != AB_OK) return rc;
    if ((rc = norm(f.pros_last_w, f.pros_last_b, P, nullptr)) != AB_OK) return rc;
  }

  // the quantizers (all groups, one launch) and the positional add into S
  FacRvqParams p;
  memset(&p, 0, sizeof(p));
  p.x = dev_x; p.xsb = x_strides[0]; p.xsc = x_strides[1]; p.xst = x_strides[2];
  int n_used = 0, nq_run = 0;
  for (int gi = 0, l0 = 0; gi < 3; l0 += g->cfg.vq_num_q[gi], ++gi) {
    p.layer0[gi] = l0;
    p.nused[gi] = std::min(n_quantizers, g->cfg.vq_num_q[gi]);   // rvq.py:50-52
    p.code_row0[gi] = n_used;
    n_used += p.nused[gi];
    for (int j = 0; j < p.nused[gi]; ++j) {
      const FacodecLayerRef& l = g->fac.layers[l0 + j];
      const int q = l0 + j;
      p.w_in[q] = g->fptr(l.in_proj.w); p.b_in[q] = g->fptr(l.in_proj.b);
      p.w_out[q] = g->fptr(l.out_proj.w); p.b_out[q] = g->fptr(l.out_proj.b);
      p.cb[q] = g->fptr(l.cb);
      p.cbn[q] = reinterpret_cast<const float*>(g->arena + l.cbn_offset);
      p.cbn2[q] = reinterpret_cast<const float*>(g->arena + l.cbn_offset +
                                                 align_up((size_t)l.rows * FAC_MAX_CODEBOOK_DIM * sizeof(float), 256));
      p.rows[q] = l.rows;
      nq_run += 1;
    }
  }
  p.ngroups = g->cfg.vq_num_q[2] > 0 ? 3 : 2;
  p.B = (int)B; p.C = C; p.T = Tn; p.D = D;
  p.emb = dev_emb_out; p.codes = dev_codes_out; p.quantized = dev_quantized_out;
  p.pe = g->fptr(g->fac.pe); p.stream = w.S;
  double cb_flops = 0.0, cb_bytes = 0.0;
  for (int q = 0; q < AB_FACODEC_MAX_Q; ++q)
    if (p.cb[q]) { cb_flops += 2.0 * el * p.rows[q] * D; cb_bytes += 4.0 * p.rows[q] * (FAC_MAX_CODEBOOK_DIM + 1); }
  rc = L.timed(12, 4.0 * el * nq_run * C * D + cb_flops,
               4.0 * el * C * (2 + p.ngroups + 1 + (v2 ? 1 : 0)) + 8.0 * el * n_used + cb_bytes + 8.0 * nq_run * (double)C * D,
               [&] { return launch_facodec_rvq(p, L.st, P); });
  if (rc != AB_OK) return rc;

  // the timbre encoder on S (transformer.py:206-217)
  rc = facodec_transformer_layers(L, w, B, Tn, g->fac.timbre, g->precision != AB_PREC_FP32,
                                  [&](const TimbreLayerRef& t, int i, float* y, uint16_t* yimg) {
    return i == 0 ? norm(t.ln1_w, t.ln1_b, y, yimg) : norm(t.ln2_w, t.ln2_b, y, yimg);
  });
  if (rc != AB_OK) return rc;
  if ((rc = norm(g->fac.last_w, g->fac.last_b, w.H, nullptr)) != AB_OK) return rc;
  rc = L.timed(12, el * C, 4.0 * el * C + 4.0 * B * C, [&] { return launch_facodec_time_mean(w.H, dev_spk_out, (int)B, C, Tn, L.st); });
  return L.done(rc);
}

int ab_facodec_quantize(ab_generator* g, const float* dev_x, const int64_t x_strides[3], int64_t B, int64_t T,
                        int32_t n_quantizers, float* dev_emb_out, int64_t* dev_codes_out, float* dev_quantized_out,
                        float* dev_spk_out, void* dev_workspace, size_t workspace_bytes, void* stream) {
  return facodec_quantize_impl(g, "facodec_quantize", dev_x, x_strides, nullptr, nullptr, B, T, n_quantizers, dev_emb_out,
                               dev_codes_out, dev_quantized_out, dev_spk_out, dev_workspace, workspace_bytes, stream);
}

int ab_facodec_quantize_prosody(ab_generator* g, const float* dev_x, const int64_t x_strides[3], const float* dev_prosody,
                                const int64_t prosody_strides[3], int64_t B, int64_t T, int32_t n_quantizers,
                                float* dev_emb_out, int64_t* dev_codes_out, float* dev_quantized_out, float* dev_spk_out,
                                void* dev_workspace, size_t workspace_bytes, void* stream) {
  if (g && !dev_prosody) return fail(AB_ERR_ARG, "facodec_quantize_prosody: null argument");
  return facodec_quantize_impl(g, "facodec_quantize_prosody", dev_x, x_strides, dev_prosody, prosody_strides, B, T,
                               n_quantizers, dev_emb_out, dev_codes_out, dev_quantized_out, dev_spk_out, dev_workspace,
                               workspace_bytes, stream);
}

int ab_facodec_prosody_input_forward(const float* dev_x, const int64_t x_strides[3], const float* dev_w,
                                     const float* dev_bias, const float* dev_pe, int64_t B, int64_t T, float* dev_y,
                                     void* stream) {
  if (!x_strides) return fail(AB_ERR_ARG, "facodec_prosody_input_forward: null argument");
  if (B <= 0 || T <= 0 || B > FAC_PE_ROWS || T > (1ll << 30))
    return fail(AB_ERR_ARG, "facodec_prosody_input_forward: batch %lld / frames %lld out of range", (long long)B,
                (long long)T);
  FacProsodyInParams p;
  p.x = dev_x; p.xsb = x_strides[0]; p.xsi = x_strides[1]; p.xst = x_strides[2];
  p.w = dev_w; p.bias = dev_bias; p.pe = dev_pe; p.y = dev_y;
  p.B = (int)B; p.T = (int)T;
  return launch_facodec_prosody_input(p, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------
// FACodec redecoder
// ---------------------------------------------------------------------------
size_t ab_facodec_redecoder_vq2emb_workspace_bytes(const ab_generator* g, int64_t B, int64_t T) {
  if (!g || g->cfg.kind != AB_GEN_FACODEC_REDECODER || B <= 0 || T <= 0) return 0;
  Carve c{nullptr};
  float* styles;
  redecoder_layout(c, B, T, &styles);
  return c.off;
}

int ab_facodec_redecoder_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_q,
                                int64_t B, int64_t T, const float* dev_spk, int64_t spk_row_stride, int32_t use_residual,
                                float* dev_out, void* dev_workspace, size_t workspace_bytes, void* stream) {
  const char* what = "facodec_redecoder_vq2emb";
  if (g && B > FAC_PE_ROWS)   // PositionalEncoding adds pe[:B] (transformer.py:43-45)
    return fail(AB_ERR_ARG, "%s: batch %lld > %d, the rows of the positional encoding", what, (long long)B, FAC_PE_ROWS);
  int rc = facodec_check(g, B, T, what, 2);
  if (rc != AB_OK) return rc;
  if (!dev_codes || !codes_strides || !dev_spk || !dev_out) return fail(AB_ERR_ARG, "%s: null argument", what);
  const int C = FAC_TIMBRE_C, Tn = (int)T;
  if (spk_row_stride < C) return fail(AB_ERR_ARG, "%s: speaker-embedding row stride < %d", what, C);
  const int* nq = g->cfg.vq_num_q;
  // code rows are read by position (facodec.py:739-756); extra rows are not read
  const int rows = nq[0] + nq[1] + (use_residual ? nq[2] : 0);
  if (n_q < rows)
    return fail(AB_ERR_ARG, "%s: %d code rows; vq2emb reads %d (%d prosody, %d content, %d residual)", what, n_q, rows,
                nq[0], nq[1], use_residual ? nq[2] : 0);
  rc = check_workspace(what, dev_workspace, workspace_bytes, ab_facodec_redecoder_vq2emb_workspace_bytes(g, B, T));
  if (rc != AB_OK) return rc;
  Launch L{g, static_cast<cudaStream_t>(stream)};
  Carve ws{static_cast<char*>(dev_workspace)};
  float* styles = nullptr;
  const TimbreWs w = redecoder_layout(ws, B, T, &styles);
  const FacodecRef& f = g->fac;
  const double el = (double)B * T;

  // (gamma, beta) of every StyleAdaptiveLayerNorm from the speaker embedding (transformer.py:25): the condition is the
  // embedding expanded over time, whose time mean is the embedding itself
  auto style_of = [&](int i) { return styles + (size_t)i * B * 2 * C; };
  for (int i = 0; i < 9; ++i) {
    const int sw = i == 8 ? f.last_w : (i & 1) ? f.timbre[i / 2].ln2_w : f.timbre[i / 2].ln1_w;
    const int sb = i == 8 ? f.last_b : (i & 1) ? f.timbre[i / 2].ln2_b : f.timbre[i / 2].ln1_b;
    rc = L.timed(11, 4.0 * B * C * C, 4.0 * (2.0 * C * C + B * 3.0 * C), [&] {
      return launch_facodec_style(dev_spk, spk_row_stride, g->fptr(sw), g->fptr(sb), style_of(i), (int)B, C, L.st);
    });
    if (rc != AB_OK) return rc;
  }
  // gamma * LayerNorm(S) + beta (transformer.py:29-31) into y (fp32) or the operand image yimg
  auto film = [&](int i, float* y, uint16_t* yimg) -> int {
    FacFilmParams p;
    p.x = w.S; p.xsb = (int64_t)C * T; p.xsc = T; p.xst = 1;
    p.style = style_of(i); p.y = y; p.yimg = yimg; p.bf16 = g->precision == AB_PREC_TC_BF16;
    p.B = (int)B; p.C = C; p.T = Tn;
    return L.timed(11, 10.0 * el * C, 4.0 * el * C + (y ? 4.0 : 2.0) * el * C, [&] { return launch_facodec_film(p, L.st); });
  };
  // the gathers: prev + the tables' rows (+ pe) -> out
  auto embed = [&](const float* prev, int row0, int ntab, const float* pe, float* out) -> int {
    FacEmbedParams p;
    memset(&p, 0, sizeof(p));
    p.codes = dev_codes; p.cs0 = codes_strides[0]; p.cs1 = codes_strides[1]; p.cs2 = codes_strides[2];
    p.row0 = row0; p.ntab = ntab;
    for (int j = 0; j < ntab; ++j) { p.tab[j] = g->fptr(f.layers[row0 + j].cb); p.rows[j] = f.layers[row0 + j].rows; }
    p.prev = prev; p.pe = pe; p.out = out;
    p.B = (int)B; p.C = C; p.T = Tn;
    return L.timed(11, el * C * (ntab + (prev ? 1 : 0) + (pe ? 1 : 0) - 1), 8.0 * el * ntab + 4.0 * el * C * (ntab + 1 + (prev ? 1 : 0)),
                   [&] { return launch_facodec_embed(p, L.st); });
  };
  // facodec.py:739-744: per prosody table, x_t = transformer(x_t + emb(codes)); the transformer adds pe each time
  for (int i = 0; i < nq[0]; ++i) {
    if ((rc = embed(i == 0 ? nullptr : w.H, i, 1, g->fptr(f.pe), w.S)) != AB_OK) return rc;
    rc = facodec_transformer_layers(L, w, B, Tn, f.timbre, g->precision != AB_PREC_FP32,
                                    [&](const TimbreLayerRef& t, int j, float* y, uint16_t* yimg) {
      return film(2 * (int)(&t - f.timbre.data()) + j, y, yimg);
    });
    if (rc != AB_OK) return rc;
    if ((rc = film(8, w.H, nullptr)) != AB_OK) return rc;   // last_ln
  }
  // facodec.py:746-756: out = x_t, + the content rows, + the residual rows, one add at a time
  return L.done(embed(w.H, nq[0], rows - nq[0], nullptr, dev_out));
}

// ---------------------------------------------------------------------------
// FACodec encoder
// ---------------------------------------------------------------------------
// ---------------------------------------------------------------------------
// The codec's ResidualVQ (AB_GEN_RVQ)
// ---------------------------------------------------------------------------
static int rvq_check(const ab_generator* g, int64_t B, int64_t T, int32_t n, const char* what) {
  if (!g) return fail(AB_ERR_ARG, "%s: null handle", what);
  if (g->cfg.kind != AB_GEN_RVQ) return fail(AB_ERR_ARG, "%s: not a residual VQ handle", what);
  if (!g->finalized) return fail(AB_ERR_STATE, "%s: finalize() the handle first", what);
  if (B <= 0 || T <= 0 || B > 65535 || T > (1ll << 30))
    return fail(AB_ERR_ARG, "%s: batch %lld / frames %lld out of range", what, (long long)B, (long long)T);
  if (n < 1 || n > g->cfg.vq_num_q[0])
    return fail(AB_ERR_ARG, "%s: n_quantizers %d outside 1..%d", what, n, g->cfg.vq_num_q[0]);
  return AB_OK;
}

int ab_rvq_quantize(ab_generator* g, const float* dev_x, const int64_t x_strides[3], int64_t B, int64_t T,
                    int32_t n_quantizers, float* dev_quantized_out, int64_t* dev_codes_out, float* dev_layers_out,
                    void* stream) {
  int rc = rvq_check(g, B, T, n_quantizers, "rvq_quantize");
  if (rc != AB_OK) return rc;
  if (!dev_x || !x_strides || !dev_quantized_out || !dev_codes_out)
    return fail(AB_ERR_ARG, "rvq_quantize: null argument");
  const int C = g->cfg.n_mel, D = g->cfg.vq_codebook_dim;
  FacRvqParams p;
  memset(&p, 0, sizeof(p));
  p.x = dev_x; p.xsb = x_strides[0]; p.xsc = x_strides[1]; p.xst = x_strides[2];
  p.nused[0] = n_quantizers;
  for (int q = 0; q < n_quantizers; ++q) {
    const FacodecLayerRef& l = g->fac.layers[q];
    p.w_in[q] = g->fptr(l.in_proj.w); p.b_in[q] = g->fptr(l.in_proj.b);
    p.w_out[q] = g->fptr(l.out_proj.w); p.b_out[q] = g->fptr(l.out_proj.b);
    p.cb[q] = g->fptr(l.cb);
    p.cbn[q] = reinterpret_cast<const float*>(g->arena + l.cbn_offset);
    p.cbn2[q] = reinterpret_cast<const float*>(g->arena + l.cbn_offset +
                                               align_up((size_t)l.rows * FAC_MAX_CODEBOOK_DIM * sizeof(float), 256));
    p.rows[q] = l.rows;
  }
  p.ngroups = 1;
  p.B = (int)B; p.C = C; p.T = (int)T; p.D = D;
  p.codes = dev_codes_out; p.quantized = dev_quantized_out;
  Launch L{g, static_cast<cudaStream_t>(stream)};
  const double el = (double)B * T, n = n_quantizers, rows = (double)g->cfg.vq_codebook_size;
  rc = L.timed(12, 4.0 * el * n * C * D + 2.0 * el * n * rows * D,
               4.0 * el * C * (2 + (dev_layers_out ? n : 0)) + 8.0 * el * n + 4.0 * n * rows * (FAC_MAX_CODEBOOK_DIM + 1) +
                   8.0 * n * C * D,
               [&] { return launch_facodec_rvq(p, L.st, nullptr, dev_layers_out, true); });
  return L.done(rc);
}

int ab_rvq_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_quantizers,
                  int64_t B, int64_t T, float* dev_out, void* stream) {
  int rc = rvq_check(g, B, T, n_quantizers, "rvq_vq2emb");
  if (rc != AB_OK) return rc;
  if (!dev_codes || !codes_strides || !dev_out) return fail(AB_ERR_ARG, "rvq_vq2emb: null argument");
  FacVqParams p;
  memset(&p, 0, sizeof(p));
  p.codes = dev_codes; p.cs0 = codes_strides[0]; p.cs1 = codes_strides[1]; p.cs2 = codes_strides[2];
  p.nq = n_quantizers;
  for (int q = 0; q < p.nq; ++q) {
    const FacodecLayerRef& l = g->fac.layers[q];
    p.cb[q] = g->fptr(l.cb); p.w[q] = g->fptr(l.out_proj.w); p.bias[q] = g->fptr(l.out_proj.b); p.rows[q] = l.rows;
  }
  p.group_end[0] = p.nq;
  p.ngroups = 1;
  p.B = (int)B; p.C = g->cfg.n_mel; p.T = (int)T; p.D = g->cfg.vq_codebook_dim; p.out = dev_out;
  Launch L{g, static_cast<cudaStream_t>(stream)};
  const double el = (double)B * T;
  rc = L.timed(11, 2.0 * el * p.nq * p.C * p.D, 8.0 * el * p.nq + 4.0 * el * p.C + 4.0 * p.nq * (double)p.C * (p.D + 1),
               [&] { return launch_facodec_vq2emb(p, L.st); });
  return L.done(rc);
}

int64_t ab_facodec_encoder_frames(const ab_generator* g, int64_t samples) {
  if (!g || g->cfg.kind != AB_GEN_FACODEC_ENCODER || samples <= 0) return 0;
  int64_t t = samples;
  for (auto& st : g->stages) t = encoder_stage_length(t, st.down);
  return t;
}

int ab_facodec_encode(ab_generator* g, const float* dev_wav, int64_t B, int64_t N, const int64_t wav_strides[3],
                      float* dev_out, void* dev_workspace, size_t workspace_bytes, void* stream) {
  if (!g) return fail(AB_ERR_ARG, "facodec_encode: null handle");
  if (g->cfg.kind != AB_GEN_FACODEC_ENCODER) return fail(AB_ERR_ARG, "facodec_encode: not a FACodec encoder handle");
  if (!dev_wav || !wav_strides || !dev_out) return fail(AB_ERR_ARG, "facodec_encode: null argument");
  if (B <= 0 || N <= 0) return fail(AB_ERR_ARG, "facodec_encode: batch %lld / samples %lld out of range", (long long)B, (long long)N);
  if (ab_facodec_encoder_frames(g, N) <= 0)
    return fail(AB_ERR_ARG, "facodec_encode: %lld samples leave a stage with no output (a strided conv's padded input is "
                "shorter than its kernel)", (long long)N);
  Launch L{g, static_cast<cudaStream_t>(stream)};
  return L.done(forward_generator(L, dev_wav, B, N, wav_strides, nullptr, 0, dev_out, dev_workspace, workspace_bytes));
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

int ab_activation1d_packed_forward(const float* dev_x, float* dev_y, uint16_t* dev_yimg, int64_t B, int64_t C,
                                   int64_t T, const float* dev_alpha, const float* dev_beta, int32_t logscale,
                                   const float* f_up, const float* f_down, int32_t precision, void* stream) {
  if (!dev_x || !dev_alpha || !dev_beta || !f_up || !f_down) return fail(AB_ERR_ARG, "activation1d_packed: null argument");
  if (!dev_y && !dev_yimg) return fail(AB_ERR_ARG, "activation1d_packed: no output requested");
  if (precision != AB_PREC_FP32 && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "activation1d_packed: unknown precision %d", precision);
  if (dev_yimg && precision == AB_PREC_FP32)
    return fail(AB_ERR_ARG, "activation1d_packed: the operand image needs a tensor-core precision");
  if (B < 1 || C < 1 || T < 1) return fail(AB_ERR_ARG, "activation1d_packed: bad shape");
  if (B > 65535 || C > 65535 * 8) return fail(AB_ERR_UNSUPPORTED, "activation1d_packed: B or C too large");
  if (T > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "activation1d_packed: sequence too long");
  SnakeCoef kc;
  pack_snake_coef(f_up, f_down, &kc);
  const SnakeParams p = generator_snake_params(&kc, precision, dev_x, dev_y, dev_yimg, dev_alpha, dev_beta, nullptr,
                                               nullptr, logscale, (int)B, (int)C, (int)T);
  return launch_activation1d(p, static_cast<cudaStream_t>(stream));
}

int ab_snake1d_forward(const float* dev_x, float* dev_y, uint16_t* dev_yimg, int64_t B, int64_t C, int64_t T,
                       const float* dev_alpha, int32_t precision, void* stream) {
  if (!dev_x || !dev_alpha) return fail(AB_ERR_ARG, "snake1d: null argument");
  if (!dev_y && !dev_yimg) return fail(AB_ERR_ARG, "snake1d: no output requested");
  if (precision != AB_PREC_FP32 && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "snake1d: unknown precision %d", precision);
  if (dev_yimg && precision == AB_PREC_FP32) return fail(AB_ERR_ARG, "snake1d: the operand image needs a tensor-core precision");
  if (B < 1 || C < 1 || T < 1) return fail(AB_ERR_ARG, "snake1d: bad shape");
  if (B > 65535 || C > 65536 || T > (1ll << 30)) return fail(AB_ERR_UNSUPPORTED, "snake1d: shape too large");
  return launch_snake1d(dev_x, dev_y, dev_yimg, precision == AB_PREC_TC_BF16, dev_alpha, (int)B, (int)C, (int)T,
                        static_cast<cudaStream_t>(stream));
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
  if (k < u || ((k - u) & 1))   // padding (k - u) / 2, hifigan.py:176-186
    return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: kernel %d / stride %d: need k >= stride and (k - stride) even", k, u);
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
  p.pad = (k - u) / 2;
  return launch_conv_transpose1d_fp32(p, st);
}

size_t ab_tc_conv_workspace_bytes(int32_t mode, int64_t cin, int64_t cout, int32_t k, int32_t d_or_u) {
  return align_up((size_t)cin * cout * k * sizeof(float), 256) +
         align_up(tc_weight_image_bytes(mode, (int)cin, (int)cout, k, d_or_u), 256);
}

int ab_tc_conv_forward(int32_t mode, const float* dev_x, const int64_t x_strides[3], float pre_slope,
                       const uint16_t* dev_ximg, const float* dev_w, const float* dev_bias, const float* dev_residual,
                       const float* dev_acc_prev, float out_div, int32_t reflect, float* dev_y, uint16_t* dev_yimg,
                       float img_slope, int64_t B, int64_t cin, int64_t cout, int64_t T, int32_t k, int32_t d_or_u,
                       int32_t pad, int32_t precision, void* ws, size_t ws_bytes, void* stream) {
  if (!dev_w || !ws || (dev_x && !dev_ximg && !x_strides)) return fail(AB_ERR_ARG, "tc conv: null argument");
  if (ws_bytes < ab_tc_conv_workspace_bytes(mode, cin, cout, k, d_or_u)) return fail(AB_ERR_WORKSPACE, "tc conv: workspace too small");
  if (B > INT32_MAX || cin > INT32_MAX || cout > INT32_MAX || T * (mode == 1 ? d_or_u : 1) > (1ll << 30))
    return fail(AB_ERR_UNSUPPORTED, "tc conv: shape too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* w_t = static_cast<float*>(ws);
  void* img = static_cast<char*>(ws) + align_up((size_t)cin * cout * k * sizeof(float), 256);
  int rc = mode == 1 ? launch_repack_weight(dev_w, nullptr, w_t, (int)cin, (int)cout, k, 1, st)
                     : launch_repack_weight(dev_w, nullptr, w_t, (int)cout, (int)cin, k, 0, st);
  if (rc != AB_OK) return rc;
  rc = launch_tc_pack_weight(w_t, img, mode, (int)cin, (int)cout, k, d_or_u, precision, st);
  if (rc != AB_OK) return rc;
  TcConvParams p;
  p.mode = mode;
  p.x = dev_x; p.ximg = dev_ximg; p.pre_slope = pre_slope;
  if (dev_x && !dev_ximg) { p.xsb = x_strides[0]; p.xsc = x_strides[1]; p.xst = x_strides[2]; }
  p.w = img; p.bias = dev_bias; p.residual = dev_residual; p.acc_prev = dev_acc_prev; p.out_div = out_div;
  p.reflect = reflect; p.pad = pad;
  p.y = dev_y; p.yimg = dev_yimg; p.img_slope = img_slope;
  p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)T; p.k = k; p.d_or_u = d_or_u; p.precision = precision;
  return launch_tc_conv(p, st);
}

int ab_vocos_norm_forward(const float* dev_x, const float* dev_dw_w, const float* dev_dw_b, const float* dev_ln_w,
                          const float* dev_ln_b, float eps, float* dev_y, uint16_t* dev_yimg, int32_t precision, int64_t B,
                          int64_t C, int64_t T, void* stream) {
  if (!dev_x || !dev_ln_w || !dev_ln_b) return fail(AB_ERR_ARG, "vocos_norm: null argument");
  if ((!dev_y) == (!dev_yimg)) return fail(AB_ERR_ARG, "vocos_norm: give exactly one of y and yimg");
  if ((!dev_dw_w) != (!dev_dw_b)) return fail(AB_ERR_ARG, "vocos_norm: give both or neither of dw_w and dw_b");
  if (dev_yimg && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "vocos_norm: the operand image needs a tensor-core precision (got %d)", precision);
  if (B < 1 || C < 1 || T < 1 || B > INT32_MAX || C > INT32_MAX || T > (1ll << 30))
    return fail(AB_ERR_ARG, "vocos_norm: batch %lld, %lld channels, length %lld", (long long)B, (long long)C, (long long)T);
  NormParams p;
  p.x = dev_x; p.dw_w = dev_dw_w; p.dw_b = dev_dw_b; p.ln_w = dev_ln_w; p.ln_b = dev_ln_b;
  p.y = dev_y; p.yimg = dev_yimg; p.bf16 = precision == AB_PREC_TC_BF16;
  p.B = (int)B; p.C = (int)C; p.T = (int)T; p.eps = eps;
  return launch_vocos_norm(p, static_cast<cudaStream_t>(stream));
}

static_assert(AB_VOCOS_PW_GELU == AB_PW_GELU && AB_VOCOS_PW_GAMMA == AB_PW_GAMMA_RESIDUAL &&
                  AB_VOCOS_PW_SPECTRUM == AB_PW_SPECTRUM && AB_VOCOS_PW_LINEAR == AB_PW_LINEAR,
              "the public pointwise epilogues name launch_tc_pointwise's");

size_t ab_vocos_pointwise_workspace_bytes(int32_t epilogue, int64_t B, int64_t cin, int64_t cout, int64_t T,
                                          int32_t precision) {
  if (B < 1 || cin < 1 || cout < 1 || T < 1 || cin > INT32_MAX || cout > INT32_MAX) return 0;
  const size_t w = align_up((size_t)cin * cout * sizeof(float), 256);
  if (precision != AB_PREC_FP32) {
    const size_t img = tc_weight_image_bytes(0, (int)cin, (int)cout, 1, 1);
    return img == 0 ? 0 : w + align_up(img, 256);
  }
  // SPECTRUM: the Linear's output [B, C_out, T] before the spectral head
  return w + (epilogue == AB_VOCOS_PW_SPECTRUM ? align_up((size_t)B * cout * T * sizeof(float), 256) : 0);
}

int ab_vocos_pointwise_forward(int32_t epilogue, const float* dev_x, const uint16_t* dev_ximg, const float* dev_w,
                               const float* dev_bias, const float* dev_gamma, float* dev_y, uint16_t* dev_yimg,
                               float* dev_spec, int64_t B, int64_t cin, int64_t cout, int64_t T, int32_t precision,
                               void* ws, size_t ws_bytes, void* stream) {
  if (epilogue < AB_VOCOS_PW_GELU || epilogue > AB_VOCOS_PW_LINEAR)
    return fail(AB_ERR_ARG, "vocos_pointwise: unknown epilogue %d", epilogue);
  if (precision != AB_PREC_FP32 && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "vocos_pointwise: unknown precision %d", precision);
  const bool tc = precision != AB_PREC_FP32;
  if (!dev_w || !dev_bias) return fail(AB_ERR_ARG, "vocos_pointwise: null weight or bias");
  if (tc ? (!dev_ximg || dev_x) : (!dev_x || dev_ximg))
    return fail(AB_ERR_ARG, "vocos_pointwise: precision %d takes its input as %s", precision, tc ? "ximg" : "x");
  const bool out_ok = epilogue == AB_VOCOS_PW_GELU ? (tc ? dev_yimg != nullptr : dev_y != nullptr)
                      : epilogue == AB_VOCOS_PW_GAMMA ? dev_y && dev_gamma
                      : epilogue == AB_VOCOS_PW_LINEAR ? dev_y != nullptr
                                                       : dev_spec != nullptr;
  if (!out_ok) return fail(AB_ERR_ARG, "vocos_pointwise: epilogue %d: missing output or gamma", epilogue);
  if (epilogue == AB_VOCOS_PW_LINEAR && (dev_gamma || dev_yimg || dev_spec))
    return fail(AB_ERR_ARG, "vocos_pointwise: epilogue %d (Linear) writes y alone: gamma, yimg and spec must be NULL",
                epilogue);
  if (epilogue == AB_VOCOS_PW_SPECTRUM && (cout & 1))
    return fail(AB_ERR_ARG, "vocos_pointwise: the spectrum needs an even C_out (magnitude and phase halves), got %lld",
                (long long)cout);
  if (B < 1 || cin < 1 || cout < 1 || T < 1 || B > 65535 || cin > INT32_MAX || cout > INT32_MAX || T > (1ll << 30))
    return fail(AB_ERR_ARG, "vocos_pointwise: batch %lld, C_in %lld, C_out %lld, length %lld", (long long)B,
                (long long)cin, (long long)cout, (long long)T);
  const size_t need = ab_vocos_pointwise_workspace_bytes(epilogue, B, cin, cout, T, precision);
  if (need == 0) return fail(AB_ERR_UNSUPPORTED, "vocos_pointwise: %s", ab_last_error());
  int rc = check_workspace("vocos_pointwise", ws, ws_bytes, need);
  if (rc != AB_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* w_t = static_cast<float*>(ws);
  char* rest = static_cast<char*>(ws) + align_up((size_t)cin * cout * sizeof(float), 256);
  rc = launch_repack_weight(dev_w, nullptr, w_t, (int)cout, (int)cin, 1, 0, st);
  if (rc != AB_OK) return rc;
  if (tc) {
    rc = epilogue == AB_VOCOS_PW_SPECTRUM ? launch_tc_pack_head_weight(w_t, rest, (int)cin, (int)cout, precision, st)
                                          : launch_tc_pack_weight(w_t, rest, 0, (int)cin, (int)cout, 1, 1, precision, st);
    if (rc != AB_OK) return rc;
    TcPwParams p;
    p.epilogue = epilogue; p.ximg = dev_ximg; p.w = rest; p.bias = dev_bias; p.gamma = dev_gamma;
    p.yimg = dev_yimg; p.y = dev_y; p.spec = dev_spec;
    p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)T; p.precision = precision;
    return launch_tc_pointwise(p, st);
  }
  float* head = reinterpret_cast<float*>(rest);
  ConvParams p;
  p.x = dev_x; p.xsb = cin * T; p.xsc = T; p.xst = 1; p.w_t = w_t; p.bias = dev_bias;
  p.residual = epilogue == AB_VOCOS_PW_GAMMA ? dev_y : nullptr; p.acc_prev = nullptr;
  p.y = epilogue == AB_VOCOS_PW_SPECTRUM ? head : dev_y;
  p.B = (int)B; p.Cin = (int)cin; p.Cout = (int)cout; p.T = (int)T; p.k = 1; p.d = 1;
  p.pre_slope = 1.0f; p.out_div = 1.0f; p.post_tanh = 0;
  p.epi = epilogue == AB_VOCOS_PW_GELU ? CONV_EPI_GELU : epilogue == AB_VOCOS_PW_GAMMA ? CONV_EPI_GAMMA_RESIDUAL
          : epilogue == AB_VOCOS_PW_LINEAR ? CONV_EPI_LINEAR : CONV_EPI_NONE;
  p.gamma = dev_gamma;
  rc = launch_conv1d_fp32(p, st);
  // [B, 2 bins, T]: the magnitude and phase halves of one utterance are bins * T apart (forward_vocos)
  const int64_t bins = cout / 2;
  for (int64_t b = 0; rc == AB_OK && epilogue == AB_VOCOS_PW_SPECTRUM && b < B; ++b) {
    const float* hb = head + b * cout * T;
    rc = ab_spectral_head_forward(hb, hb + bins * T, nullptr, 1, bins, T, 1e2f, nullptr, nullptr, nullptr,
                                  dev_spec + b * T * bins * 2, st);
  }
  return rc;
}

size_t ab_diffwave_layer_workspace_bytes(int32_t n_mel) {
  return n_mel < 1 ? 0 : dw_layer_packed_floats(n_mel) * sizeof(float);
}

int ab_diffwave_layer_forward(const float* dev_x_in, const float* dev_d, int64_t d_batch_stride, const float* dev_cond,
                              const float* dev_wdil, const float* dev_bdil, const float* dev_wcond, const float* dev_bcond,
                              const float* dev_wout, const float* dev_bout, float* dev_x_out, float* dev_skip, int64_t B,
                              int64_t L, int32_t n_mel, int32_t dilation, int32_t first, int32_t precision, void* ws,
                              size_t ws_bytes, void* stream) {
  if (!dev_x_in || !dev_d || !dev_cond || !dev_wdil || !dev_bdil || !dev_wcond || !dev_bcond || !dev_wout || !dev_bout ||
      !dev_x_out || !dev_skip || !ws)
    return fail(AB_ERR_ARG, "diffwave_layer: null argument");
  if (dev_x_out == dev_x_in) return fail(AB_ERR_ARG, "diffwave_layer: x_out must not be x_in (tiles read x_in's halo)");
  if (precision != AB_PREC_FP32 && precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16)
    return fail(AB_ERR_ARG, "diffwave_layer: unknown precision %d", precision);
  if (B < 1 || B > 65535 || L < 1 || L > (1ll << 30) || n_mel < 1 || dilation < 1 || d_batch_stride < 0)
    return fail(AB_ERR_ARG, "diffwave_layer: batch %lld, length %lld, %d mels, dilation %d, d stride %lld", (long long)B,
                (long long)L, n_mel, dilation, (long long)d_batch_stride);
  if (dw_layer_smem_bytes(n_mel, precision) > 227 * 1024)
    return fail(AB_ERR_UNSUPPORTED, "diffwave_layer: %d mels do not fit the layer tile", n_mel);
  if (ws_bytes < ab_diffwave_layer_workspace_bytes(n_mel) || reinterpret_cast<uintptr_t>(ws) % 256)
    return fail(AB_ERR_WORKSPACE, "diffwave_layer: workspace %zu B (256-byte aligned) < required %zu B", ws_bytes,
                ab_diffwave_layer_workspace_bytes(n_mel));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const DwLayerPack lp = dw_layer_pack(static_cast<char*>(ws), n_mel, 0);
  DwPackParams pk;
  pk.wdil = dev_wdil; pk.bdil = dev_bdil; pk.wcond = dev_wcond; pk.bcond = dev_bcond; pk.wout = dev_wout; pk.bout = dev_bout;
  pk.w1p = lp.w1; pk.b1p = lp.b1; pk.w2p = lp.w2; pk.b2p = lp.b2;
  pk.w1h = precision != AB_PREC_FP32 ? lp.w1h : nullptr; pk.w2h = lp.w2h;
  pk.bf16 = precision == AB_PREC_TC_BF16;
  pk.n_mel = n_mel;
  int rc = launch_dw_pack(pk, st);
  if (rc != AB_OK) return rc;
  DwLayerParams p;
  p.x_in = dev_x_in; p.x_out = dev_x_out; p.skip = dev_skip; p.cond = dev_cond; p.d = dev_d; p.d_bstride = d_batch_stride;
  p.w1 = lp.w1; p.b1 = lp.b1; p.w2 = lp.w2; p.b2 = lp.b2; p.w1h = lp.w1h; p.w2h = lp.w2h; p.precision = precision;
  p.B = (int)B; p.n_mel = n_mel; p.dil = dilation; p.first = first != 0; p.L = L;
  return launch_dw_layer(p, st);
}

int ab_diffwave_tail_forward(const float* dev_skip, const float* dev_wsk, const float* dev_bsk, const float* dev_wo,
                             const float* dev_bo, float skip_div, int64_t B, int64_t L, float* dev_eps, float* dev_audio,
                             const float* dev_noise, float c1, float c2, float sigma, void* stream) {
  if (!dev_skip || !dev_wsk || !dev_bsk || !dev_wo || !dev_bo || (!dev_eps && !dev_audio))
    return fail(AB_ERR_ARG, "diffwave_tail: null argument");
  if (B < 1 || L < 1 || B > INT32_MAX || B * L > (1ll << 40))
    return fail(AB_ERR_ARG, "diffwave_tail: batch %lld, length %lld", (long long)B, (long long)L);
  DwTailParams t;
  t.skip = dev_skip; t.wsk = dev_wsk; t.bsk = dev_bsk; t.wo = dev_wo; t.bo = dev_bo; t.skip_div = skip_div;
  t.B = (int)B; t.L = L; t.eps = dev_eps; t.audio = dev_audio; t.noise = dev_noise;
  t.c1 = c1; t.c2 = c2; t.sigma = sigma;
  return launch_dw_tail(t, static_cast<cudaStream_t>(stream));
}

int ab_diffwave_upsample_forward(const float* dev_mel, const int64_t mel_strides[3], const float* dev_w1, const float* dev_b1,
                                 const float* dev_w2, const float* dev_b2, int32_t f1, int32_t f2, int64_t B, int32_t n_mel,
                                 int64_t frames, float* dev_out, void* stream) {
  if (!dev_mel || !mel_strides || !dev_w1 || !dev_b1 || !dev_w2 || !dev_b2 || !dev_out)
    return fail(AB_ERR_ARG, "diffwave_upsample: null argument");
  if (f1 < 2 || f2 < 2 || (f1 & 1) || (f2 & 1))
    return fail(AB_ERR_UNSUPPORTED, "diffwave_upsample: factors %d, %d (need even factors >= 2)", f1, f2);
  if (B < 1 || n_mel < 1 || frames < 1 || B > INT32_MAX || frames * f1 * f2 > (1ll << 30))
    return fail(AB_ERR_ARG, "diffwave_upsample: batch %lld, %d mels, %lld frames", (long long)B, n_mel, (long long)frames);
  DwUpsampleParams up;
  up.mel = dev_mel; up.msb = mel_strides[0]; up.msc = mel_strides[1]; up.mst = mel_strides[2];
  up.w1 = dev_w1; up.b1 = dev_b1; up.w2 = dev_w2; up.b2 = dev_b2; up.out = dev_out;
  up.B = (int)B; up.n_mel = n_mel; up.F = (int)frames; up.f1 = f1; up.f2 = f2;
  return launch_dw_upsample(up, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
