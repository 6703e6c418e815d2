/*
 * amphion_b200 — C ABI of the H100-native vocoder-inference hot path.
 *
 * The reference (open-mmlab/Amphion) is pure Python: it has no FFI.  Its
 * "operator API" for this path is the duck-typed Python surface listed in
 * SURVEY.md §8(b).  Each entry point below names the reference interface it
 * sits under (paths relative to the reference root); the Python mirror of that
 * interface lives in amphion_b200/ and is the only caller.  INTEGRATION.md
 * shows the ctypes stub a reference maintainer would add.
 *
 * Conventions
 *   - plain C types only; every pointer named dev_* is a CUDA device pointer
 *     owned by the caller (allocated by PyTorch) and outlives the call.  The
 *     library never allocates or frees device memory and never synchronises:
 *     all work is enqueued on the `stream` argument (a cudaStream_t passed as
 *     void*, 0 = legacy default stream).
 *   - every function returns AB_OK (0) or a negative AB_ERR_* code;
 *     ab_last_error() returns a thread-local, human readable message.
 *   - a handle may be used by one host thread at a time.
 */
#ifndef AMPHION_B200_H_
#define AMPHION_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AB_OK 0
#define AB_ERR_ARG (-1)         /* null pointer, bad shape, unknown tensor name */
#define AB_ERR_UNSUPPORTED (-2) /* valid request this build cannot serve */
#define AB_ERR_CUDA (-3)        /* a CUDA runtime / cuFFT call failed */
#define AB_ERR_STATE (-4)       /* call order violated (e.g. forward before finalize) */
#define AB_ERR_WORKSPACE (-5)   /* workspace / arena too small */

#define AB_MAX_STAGES 8
#define AB_MAX_KERNELS 8
#define AB_MAX_DILATIONS 8

/* AB_GEN_NSFHIFIGAN: NSFHiFiGAN.forward (models/vocoders/gan/generator/nsfhifigan.py:262-283).  As written in the
 * reference the harmonic source never reaches the output: `x_source = x[:, :, :length]` (:269) overwrites the
 * noise-conv result, so every stage computes x = ups(x) + ups(x).  The native path reproduces exactly that: the
 * HiFi-GAN pipeline with the transposed-conv weights and biases doubled at load time (exact, power of two); the
 * tensor list is HiFi-GAN's (m_source.* / noise_convs.* do not influence the samples).  Configurations whose
 * noise conv would come out shorter than the stage (odd product of the later upsample rates, :264-266) are refused.
 * AB_GEN_TRUNK: the frame-rate ResNet trunk of the iSTFT-head generators — APNet's amplitude / phase streams
 * (models/vocoders/gan/generator/apnet.py:283-375): x = conv_pre(mel) [k = trunk_in_kernel]; xs = sum_j ResBlock1_j(x)
 * / num_kernels; y = conv_post(leaky_relu(xs, 0.01)) [C -> trunk_out_channels, k = trunk_out_kernel], no tanh.
 * num_upsamples = 0, upsample_initial_channel = the trunk width; tensors "conv_pre", "resblocks.j.convs{1,2}.p",
 * "conv_post" (the caller maps ASP_input_conv / ASP_ResNet.j / ASP_output_conv ... onto them).
 * AB_GEN_MELGAN: MelGAN.forward (models/vocoders/gan/generator/melgan.py:50-101): reflection-padded conv_pre (k = 7),
 * then per ratio r: leaky_relu(0.2), ConvTranspose1d(k = 2r, stride r, padding r//2 + r%2, output_padding r%2) and
 * n_residual_layers ResnetBlocks x = shortcut(x) + conv1x1(lrelu(conv3(lrelu(x, 0.2), reflect-padded, dilation 3^j), 0.2));
 * then leaky_relu(0.2), reflection-padded conv_post (k = 7), tanh.  Config fields: upsample_rates = ratios,
 * upsample_kernel_sizes = 2 * ratios, upsample_initial_channel = ngf * 2^len(ratios), num_kernels = 1,
 * resblock_kernel_sizes[0] = 3, num_dilations[0] = n_residual_layers, resblock_dilation_sizes[0][j] = 3^j; anything else
 * is refused.  Tensors keep the reference's nn.Sequential names: "model.1" (conv_pre), "model.{2+i(2+R)+1}" (ConvTranspose
 * of stage i), "model.{2+i(2+R)+2+j}.block.2" / ".block.4" / ".shortcut" (block j), "model.{2+n(2+R)+2}" (conv_post),
 * R = n_residual_layers, n = len(ratios).  A forward whose mel has fewer than 4 frames, or whose stage is not longer
 * than one of its dilations, fails with AB_ERR_ARG before any launch (the reference's ReflectionPad1d raises).
 * AB_GEN_VOCOS: Vocos.forward (models/codec/amphion_codec/vocos.py:824-881, non-conditional backbone, "same" padding):
 * x = LayerNorm(embed(mel)) [Conv1d k = 7]; num_layers ConvNeXt blocks x = x + gamma * pwconv2(gelu(pwconv1(LayerNorm(
 * dwconv(x))))) [depthwise k = 7, LayerNorm eps 1e-6, Linear layers over channels] (:469-527); final LayerNorm; ISTFTHead:
 * Linear(dim, n_fft + 2), S = min(exp(mag), 1e2) (cos p + i sin p), ISTFT "same" with the loaded window (:84-167,
 * :314-361).  Config fields: n_mel = input_channels, upsample_initial_channel = dim, ffn_channels = intermediate_dim,
 * num_layers, istft_n_fft (even), istft_hop (<= n_fft, n_fft - hop even); every other field 0.  Tensors keep the
 * reference's state-dict names ("backbone.embed.weight", "backbone.convnext.3.pwconv1.weight" [out, in], ".gamma",
 * "backbone.final_layer_norm.bias", "head.out.weight", "head.istft.window", ...).  Output: wav [B, 1, T * istft_hop];
 * with tail events the iSTFT runs in the batch chunks.
 * AB_GEN_VOCOS_LINEAR: nn.Sequential(VocosBackbone, nn.Linear(dim, out)), RepCodec's encoder and decoder
 * (models/codec/kmeans/repcodec_model.py:108-127, vocos.py:719-783): AB_GEN_VOCOS's backbone, then y = Linear(x)
 * (fp32 accumulation, then the bias) in place of the ISTFTHead.  Config fields: n_mel = input_channels,
 * upsample_initial_channel = dim, ffn_channels = intermediate_dim, num_layers, trunk_out_channels = out_features;
 * every other field 0.  Tensors keep the Sequential's names: "0.embed.weight", "0.norm.*", "0.convnext.{i}.{dwconv,
 * norm,pwconv1,pwconv2}.*", "0.convnext.{i}.gamma", "0.final_layer_norm.*", "1.weight" [out, dim], "1.bias".  Input
 * [B, input_channels, T] with any strides (ab_generator_forward); output y [B, T, out] fp32 contiguous, the layout
 * nn.Linear returns.  The embed conv runs on the tensor cores iff input_channels <= 512 (AB_GEN_VOCOS's routing), the
 * Linear on the pointwise GEMM's AB_VOCOS_PW_LINEAR epilogue at 16 bits; with tail events the Linear runs in the batch
 * chunks.
 * AB_GEN_DIFFWAVE: DiffWave.forward (models/vocoders/diffusion/diffwave/diffwave.py:130-183): x = relu(input_projection(
 * audio)); per residual layer i (dilation 2^(i % dilation_cycle)): y = dilated_conv(x + diffusion_projection(emb)) +
 * conditioner_projection(up(mel)), z = sigmoid(y[:C]) tanh(y[C:]), (r, s) = output_projection(z), x = (x + r) / sqrt(2),
 * skip += s; eps = output_projection(relu(skip_projection(skip / sqrt(layers)))).  emb = silu(projection2(silu(
 * projection1(lerp of the embedding table at the step))))); up = two ConvTranspose2d(1, 1, [3, 2f], stride [1, f],
 * padding [1, f/2]) each followed by leaky_relu(0.4).  Config fields: n_mel, upsample_initial_channel = residual_channels
 * (64), num_layers = residual_layers, num_upsamples = 2, upsample_rates = upsample_factors (even), dilation_cycle,
 * embedding_rows = len(noise_schedule); every other field 0.  Tensors keep the reference's names, including the
 * non-persistent "diffusion_embedding.embedding" [embedding_rows, 128].  At AB_PREC_TC_F16 / TC_BF16 the residual
 * layers' convolutions take 16-bit operands (x + d, the upsampled mel, the gate, the weights) with fp32 accumulation;
 * the x and skip streams, the upsampler, the step embeddings and the tail stay fp32 at every precision.  It runs
 * through the ab_diffwave_* entry points below, not ab_generator_forward.
 * AB_GEN_FACODEC: the waveform path of NaturalSpeech 3's FACodecDecoder (models/codec/ns3_codec/facodec.py:220-240,
 * :556-576): vq2emb (codebook rows through each layer's weight-normed out_proj, summed per ResidualVQ) and inference:
 * x = LayerNorm(x over channels, no affine, eps 1e-5) * gamma + beta, (gamma, beta) = timbre_linear(speaker embedding);
 * conv_pre (k = 7); per stage i: Activation1d(SnakeBeta), ConvTranspose1d(k = 2u, stride u, padding u//2 + u%2,
 * output_padding u%2) and three ResidualUnits x = x + conv_k1(act(conv_k7(act(x), dilation d))); final act, conv_post
 * (C -> 1, k = 7), tanh.  Config fields: n_mel = in_channels (= vq_dim), upsample_initial_channel, num_upsamples and
 * upsample_rates = up_ratios, upsample_kernel_sizes = 2 u, resblock = 1, num_kernels = 1, resblock_kernel_sizes[0] = 7,
 * num_dilations[0] = 3 with dilations (1, 3, 9), activation = AB_ACT_SNAKEBETA, snake_logscale = 1, and the vq_* fields;
 * every other field 0.  Tensors keep the reference's names: "model.0" (conv_pre), "model.{1+i}.block.0" (the stage's
 * activation), "model.{1+i}.block.1" (ConvTranspose), "model.{1+i}.block.{2,3,4}.block.{0,1,2,3}" (a ResidualUnit's
 * act, k = 7 conv, act, k = 1 conv), "model.{1+n}" (final act), "model.{2+n}" (conv_post), "timbre_linear.{weight,bias}",
 * "quantizer.{q}.layers.{j}._codebook.weight" and ".out_proj.weight" (weight-normed nn.Linear: load_weight_norm with
 * weight_g [out, 1]) / ".out_proj.bias".  Runs through the ab_facodec_* entry points, not ab_generator_forward.
 * AB_GEN_FACODEC_ENCODER: NaturalSpeech 3's FACodecEncoder.forward / .inference (models/codec/ns3_codec/facodec.py:121-194):
 * wav [B, 1, N] -> conv_pre (1 -> ngf, k = 7, padding 3); per stride s (C = ngf 2^i): three ResidualUnits
 * x = x + conv_k1(act(conv_k7(act(x), dilation d))) with d = 1, 3, 9, then Activation1d(SnakeBeta) and Conv1d(C, 2C,
 * k = 2s, stride s, padding s//2 + s%2); final act, conv_post (k = 3, padding 1) -> [B, out_channels, F], no tanh.  Each
 * strided conv leaves (t + 2 (s//2 + s%2) - 2s) / s + 1 of its t samples (ab_facodec_encoder_frames).  Config fields, in
 * the decoder's conventions: n_mel = 1 (the waveform channel), upsample_initial_channel = ngf, num_upsamples and
 * upsample_rates = up_ratios in encoder order (first stride first, each 1..8), upsample_kernel_sizes = 2 s, resblock = 1,
 * num_kernels = 1, resblock_kernel_sizes[0] = 7, num_dilations[0] = 3 with dilations (1, 3, 9), activation =
 * AB_ACT_SNAKEBETA, snake_logscale = 1, trunk_out_channels = out_channels; every other field 0.  Tensors keep the
 * reference's nn.Sequential names: "block.0" (conv_pre), "block.{1+i}.block.{0,1,2}.block.{0,1,2,3}" (a ResidualUnit's
 * act, k = 7 conv, act, k = 1 conv), "block.{1+i}.block.3" (the stage's activation), "block.{1+i}.block.4" (the strided
 * conv), "block.{1+n}" (final act), "block.{2+n}" (conv_post).  conv_pre (one input channel) runs on the fp32 CUDA cores
 * at every precision.  Runs through ab_facodec_encode, not ab_generator_forward.
 * The same kind with activation = AB_ACT_SNAKE1D and snake_logscale = 0 serves the codec encoder of MaskGCT, Metis and
 * DebaTTS, CodecEncoder.forward (models/codec/amphion_codec/codec.py:60-143, use_tanh = False): d_model is ngf, and every
 * activation is a plain Snake1d, y = x + (alpha + 1e-9)^-1 sin(alpha x)^2 per channel (no anti-aliasing, no logscale; see
 * ab_snake1d_forward for its rounding).  Its tensors are then "<module>.alpha" [1, C, 1] in place of each Activation1d's
 * alpha, beta and filters; the convolutions, their routing and the workspace are the FACodec encoder's.
 * AB_GEN_RVQ: the codec's ResidualVQ of FactorizedVectorQuantize layers (models/codec/amphion_codec/quantize/residual_vq.py,
 * factorized_vector_quantize.py, quantizer_type "fvq", use_l2_normlize = True), alone.  Config fields: n_mel = input_dim,
 * vq_num_q[0] = num_quantizers (1..AB_FACODEC_MAX_Q), vq_codebook_size (any size >= 1), vq_codebook_dim (1..16, !=
 * input_dim); every other field 0.  input_dim above AB_RVQ_MAX_INPUT_DIM (1447) fails with AB_ERR_UNSUPPORTED at
 * ab_generator_create.  Tensors keep the reference's names: "quantizers.{i}.in_project.weight" [codebook_dim,
 * input_dim, 1] (weight norm over every dim but 0) / ".bias", "quantizers.{i}.out_project.weight" [input_dim, codebook_dim,
 * 1] / ".bias", "quantizers.{i}.codebook.weight" [codebook_size, codebook_dim].  Runs through ab_rvq_*.
 * AB_GEN_FACODEC_REDECODER: NaturalSpeech 3's FACodecRedecoder (models/codec/ns3_codec/facodec.py:602-769), the README's
 * zero-shot voice conversion: vq2emb (ab_facodec_redecoder_vq2emb) and inference (ab_facodec_inference, the decoder's
 * FiLM and generator).  Config fields: the generator fields as for AB_GEN_FACODEC, n_mel = in_channels = vq_dim = 256
 * (the prosody transformer's width), vq_num_q = (prosody >= 1, content >= 1, residual >= 0) tables and
 * vq_codebook_bits (1..24) their sizes; vq_codebook_dim = 0, facodec_quantize = 0; every other field 0.  Tensors keep the
 * reference's names (the 265 entries of ns3_facodec_redecoder.bin at the default constructor):
 * "{prosody,content,residual}_embs.{j}.weight" [2^bits, 256], the decoder's "model.*" and "timbre_linear.{weight,bias}",
 * "timbre_cond_prosody_enc.position_emb.pe" [5000, 1, 256], per layer l "timbre_cond_prosody_enc.layers.{l}.{ln_1,ln_2}.
 * style.{weight [512, 256], bias [512]}", ".self_attn.in_proj_{weight,bias}", ".self_attn.out_proj.{weight,bias}",
 * ".ffn.ffn_1.{weight,bias}" (k = 5), ".ffn.ffn_2.{weight,bias}", and "timbre_cond_prosody_enc.last_ln.style.{weight,bias}".
 * The reference's forward (:691-732) transposes the [B, T, d] sum before timbre_norm and is not served. */
enum ab_generator_kind {
  AB_GEN_HIFIGAN = 0, AB_GEN_BIGVGAN = 1, AB_GEN_NSFHIFIGAN = 2, AB_GEN_TRUNK = 3, AB_GEN_MELGAN = 4, AB_GEN_VOCOS = 5,
  AB_GEN_DIFFWAVE = 6, AB_GEN_FACODEC = 7, AB_GEN_FACODEC_ENCODER = 8, AB_GEN_FACODEC_REDECODER = 9, AB_GEN_RVQ = 10,
  AB_GEN_VOCOS_LINEAR = 11
};
#define AB_FACODEC_MAX_Q 32   /* most codebook layers over the three ResidualVQs */
#define AB_RVQ_MAX_INPUT_DIM 1447   /* widest AB_GEN_RVQ input_dim (the quantize kernel's two shared-memory planes) */
enum ab_activation { AB_ACT_LRELU = 0, AB_ACT_SNAKE = 1, AB_ACT_SNAKEBETA = 2, AB_ACT_SNAKE1D = 3 };
/* arithmetic of the k-tap channel-mixing convolutions */
enum ab_precision {
  AB_PREC_FP32 = 0,   /* CUDA-core FFMA, fp32 operands and accumulation */
  AB_PREC_TC_F16 = 1, /* wgmma, fp16 operands (saturating cvt), fp32 accumulation */
  AB_PREC_TC_BF16 = 2 /* wgmma, bf16 operands, fp32 accumulation */
};

const char* ab_last_error(void);
int ab_version(void);
/* 1 if the current device is compute capability 9.x (wgmma path usable) */
int ab_device_is_sm90(void);

/* ------------------------------------------------------------------------
 * Generator: HiFiGAN.forward     (models/vocoders/gan/generator/hifigan.py:203-219)
 *            BigVGAN.forward     (models/vocoders/gan/generator/bigvgan.py:313-331)
 *            NSFHiFiGAN.forward  (models/vocoders/gan/generator/nsfhifigan.py:262-283)
 *            MelGAN.forward      (models/vocoders/gan/generator/melgan.py:100-101)
 *            Vocos.forward       (models/codec/amphion_codec/vocos.py:877-881)
 *            DiffWave.forward    (models/vocoders/diffusion/diffwave/diffwave.py:164-183), see ab_diffwave_*
 * The config mirrors cfg.model.{hifigan,bigvgan}.* + cfg.preprocess.n_mel
 * (hifigan.py:151-201, bigvgan.py:232-311).
 * ---------------------------------------------------------------------- */
typedef struct ab_generator ab_generator;

typedef struct ab_generator_config {
  int32_t kind;                                 /* ab_generator_kind */
  int32_t n_mel;                                /* cfg.preprocess.n_mel */
  int32_t upsample_initial_channel;
  int32_t num_upsamples;
  int32_t upsample_rates[AB_MAX_STAGES];
  int32_t upsample_kernel_sizes[AB_MAX_STAGES];
  int32_t resblock;                             /* 1 = ResBlock1/AMPBlock1, 2 = ResBlock2/AMPBlock2 */
  int32_t num_kernels;
  int32_t resblock_kernel_sizes[AB_MAX_KERNELS];
  int32_t num_dilations[AB_MAX_KERNELS];
  int32_t resblock_dilation_sizes[AB_MAX_KERNELS][AB_MAX_DILATIONS];
  int32_t activation;                           /* ab_activation; LRELU for HiFi-GAN */
  int32_t snake_logscale;                       /* cfg.model.bigvgan.snake_logscale */
  /* HiFiGAN_vits (hifigan.py:376-449, the decoder inside VITS): kind AB_GEN_HIFIGAN plus */
  int32_t gin_channels;                         /* > 0: tensors "cond.weight" [C0, gin, 1], "cond.bias" [C0] (:424-425) */
  int32_t conv_post_no_bias;                    /* 1: conv_post = Conv1d(ch, 1, 7, bias=False) (:421), no "conv_post.bias" */
  /* AB_GEN_TRUNK only (0 elsewhere), and trunk_out_channels for AB_GEN_FACODEC_ENCODER (its out_channels) */
  int32_t trunk_out_channels;                   /* conv_post output channels (n_fft/2+1, or 2*(n_fft/2+1) for R|I) */
  int32_t trunk_in_kernel;                      /* conv_pre kernel size (odd) */
  int32_t trunk_out_kernel;                     /* conv_post kernel size (odd) */
  /* AB_GEN_VOCOS only (0 elsewhere) */
  int32_t ffn_channels;                         /* ConvNeXt intermediate_dim */
  int32_t num_layers;                           /* ConvNeXt blocks */
  int32_t istft_n_fft;
  int32_t istft_hop;
  /* AB_GEN_DIFFWAVE only (0 elsewhere) */
  int32_t dilation_cycle;                       /* dilation_cycle_length */
  int32_t embedding_rows;                       /* rows of the diffusion-step table, len(noise_schedule) */
  /* AB_GEN_FACODEC: the prosody, content and residual ResidualVQs (facodec.py:286-334); AB_GEN_FACODEC_REDECODER: its
   * embedding tables (vq_num_q, vq_codebook_bits; vq_codebook_dim 0); 0 elsewhere */
  int32_t vq_num_q[3];                          /* vq_num_q_p, vq_num_q_c, vq_num_q_r (the residual group may be 0) */
  int32_t vq_codebook_bits[3];                  /* codebook_size_{prosody,content,residual}: 2^bits rows */
  int32_t vq_codebook_dim;                      /* codebook_dim */
  /* AB_GEN_FACODEC only (0 elsewhere): 1 = the handle also serves FACodecDecoder.forward(vq=True) (ab_facodec_quantize)
   * and lists the quantizers' in_proj and the timbre encoder's tensors; needs n_mel == 256 */
  int32_t facodec_quantize;
  /* AB_GEN_FACODEC with facodec_quantize = 1 only (0 elsewhere): 1 = FACodecDecoderV2 (facodec.py:848-1094): the handle
   * also lists "melspec_linear.{weight,bias}" ([256, 20], [256]) and the prosody transformer "melspec_encoder.*" (named
   * as "timbre_encoder.*"), and its forward(vq=True) is ab_facodec_quantize_prosody (ab_facodec_quantize refuses it) */
  int32_t facodec_prosody_encoder;
  /* AB_GEN_RVQ only (0 elsewhere): rows of every codebook, any size >= 1 */
  int32_t vq_codebook_size;
} ab_generator_config;

int ab_generator_create(const ab_generator_config* cfg, ab_generator** out);
void ab_generator_destroy(ab_generator* g);

/* Parameter arena: the caller allocates ab_generator_param_bytes() of device
 * memory (256-byte aligned) and binds it; load_* calls repack into it. */
size_t ab_generator_param_bytes(const ab_generator* g);
int ab_generator_bind_params(ab_generator* g, void* dev_arena, size_t bytes);

/* Number / names of the tensors the generator expects, in reference
 * state-dict naming with weight norm folded away: "conv_pre.weight",
 * "conv_pre.bias", "ups.0.weight" ("ups.0.0.weight" for BigVGAN),
 * "resblocks.3.convs1.2.weight", "resblocks.3.activations.4.act.alpha",
 * "resblocks.3.activations.4.upsample.filter", ... (SURVEY.md §10). */
int ab_generator_num_tensors(const ab_generator* g);
const char* ab_generator_tensor_name(const ab_generator* g, int index);

/* Load one fp32 tensor (contiguous, device) by name.  shape must match the
 * reference state-dict shape. */
int ab_generator_load_tensor(ab_generator* g, const char* name, const float* dev_src,
                             const int64_t* shape, int32_t ndim, void* stream);
/* Load "<name>" from its weight-norm decomposition (old-style
 * torch.nn.utils.weight_norm, dim=0: hifigan.py:157-199): w = g*v/||v||,
 * norm over all dims but 0.  shape is the shape of v. */
int ab_generator_load_weight_norm(ab_generator* g, const char* name, const float* dev_g,
                                  const float* dev_v, const int64_t* shape, int32_t ndim, void* stream);
/* After all tensors are loaded: pick the conv arithmetic and build the packed
 * operand images it needs.  Fails with AB_ERR_STATE if a tensor is missing. */
int ab_generator_finalize(ab_generator* g, int32_t precision, void* stream);

/* 0 for AB_GEN_DIFFWAVE (see ab_diffwave_workspace_bytes) */
size_t ab_generator_workspace_bytes(const ab_generator* g, int64_t batch, int64_t frames);
/* mel [B, n_mel, T] fp32 with arbitrary element strides (the reference feeds
 * transposed views: models/vocoders/vocoder_inference.py:349,505)
 * -> wav [B, 1, T*prod(upsample_rates)] fp32 contiguous ([B, trunk_out_channels, T] for AB_GEN_TRUNK). */
int ab_generator_forward(ab_generator* g, const float* dev_mel, int64_t batch, int64_t frames,
                         const int64_t mel_strides[3], float* dev_wav, void* dev_workspace,
                         size_t workspace_bytes, void* stream);
/* HiFiGAN_vits.forward(x, g) (hifigan.py:427-445): as above with x = conv_pre(x) + cond(g) when dev_g is given.
 * dev_g [B, gin_channels] fp32 with row stride g_batch_stride (the reference's g is [B, gin, 1]); NULL = no
 * conditioning (`if g is not None`, :429).  Needs a generator created with gin_channels > 0. */
int ab_generator_forward_cond(ab_generator* g, const float* dev_x, int64_t batch, int64_t frames,
                              const int64_t x_strides[3], const float* dev_g, int64_t g_batch_stride,
                              float* dev_wav, void* dev_workspace, size_t workspace_bytes, void* stream);
/* number of kernels the last forward enqueued (bench.py's gpu_launches) */
int ab_generator_last_launches(const ab_generator* g);

/* Per-kernel-class device timing for the roofline report: when enabled, every
 * launch inside ab_generator_forward is bracketed by CUDA events on `stream`.
 * ab_generator_get_profile synchronises on the recorded events, accumulates
 * (launches, milliseconds, algorithmic FLOPs, algorithmic HBM bytes) per class
 * since the last call, and resets.  Classes: "tc_conv", "conv1d_fp32",
 * "conv_transpose1d_fp32", "activation1d", "tc_gemmconv" (max_entries >= 5), then, when max_entries >= 7,
 * "tc_pointwise" (Vocos' pointwise GEMMs and head) and "vocos_norm" (its depthwise conv + LayerNorm kernels); a DiffWave
 * handle lists, when max_entries >= 11, also "diffwave_cond" (spectrogram upsampler and step embeddings, once per
 * call), "diffwave_input" (input projection), "diffwave_layer" (residual layers) and "diffwave_tail" (skip/output
 * projections and the sampler update).  A FACodec handle lists the first five and "facodec_prologue" (timbre_linear, the
 * LayerNorm and the FiLM, and vq2emb) when max_entries >= 12, the six unused classes with zero launches; a handle created
 * with facodec_quantize also lists "facodec_quantize" (the RVQ with the positional add, and the time mean) and
 * "timbre_attention" (max_entries >= 14).  ab_facodec_quantize counts its GEMMs in "tc_conv" (tensor-core precision)
 * or "conv1d_fp32", and its LayerNorms in "vocos_norm".  A FACodec redecoder handle lists the same 14 classes:
 * ab_facodec_redecoder_vq2emb counts its style Linears, style LayerNorms and embedding gathers in "facodec_prologue",
 * its attention in "timbre_attention" and its GEMMs in "tc_conv" or "conv1d_fp32"; "facodec_quantize" stays empty. */
typedef struct ab_profile_entry {
  char name[32];
  int32_t launches;
  float ms;
  double flops;   /* 2*MACs of the convolutions as the reference defines them */
  double bytes;   /* compulsory fp32 tensor reads+writes of the launch + its weights once */
} ab_profile_entry;
int ab_generator_set_profiling(ab_generator* g, int32_t enable);
/* Execution-plan options (no reference counterpart; tuning / test knobs, results stay within the stated tolerance):
 *   "resblock_fusion": 0, 1 = one launch per (c1, c2) pair (the intermediate stays in shared memory); 2 (default) = a
 *   whole ResBlock per launch (residual stream in registers, halo recomputed in the tile) where served (C <= 128) and
 *   the recompute is small, else per pair; 3, 4 = a whole ResBlock per launch wherever served.  All plans run the same
 *   arithmetic in the same order: their outputs are bit-equal.
 *   "nsf_source_frames" (NSF-HiFiGAN, one-shot, consumed by the next forward): frames of the f0 track when it does
 *   not cover the mel; every stage is then truncated to the harmonic source's length as the reference does
 *   (nsfhifigan.py:264-268) and the output holds ab_generator_output_samples() samples per utterance.
 *   Returns AB_ERR_ARG for an unknown key / value. */
int ab_generator_set_option(ab_generator* g, const char* key, int32_t value);
/* samples per utterance of the forward of `frames` mel frames (frames * hop, or less for NSF-HiFiGAN when the f0 track
 * of `source_frames` frames is shorter than the mel or a source stride is odd; source_frames = 0: covers the mel) */
int64_t ab_generator_output_samples(const ab_generator* g, int64_t frames, int64_t source_frames);
/* Final-gather hook for the batch-sharded multi-GPU path (SURVEY 8e; no reference counterpart): the NEXT
 * ab_generator_forward[_cond] runs conv_post (hifigan.py:216-217) in n contiguous batch chunks
 * [B*i/n, B*(i+1)/n) and records events[i] (cudaEvent_t, caller-owned) on `stream` after chunk i, so the caller
 * can start sending chunk i while chunk i+1 is computed.  One-shot: cleared by that forward.  n = 0 clears. */
int ab_generator_set_tail_events(ab_generator* g, void* const* events, int32_t n);
int ab_generator_get_profile(ab_generator* g, ab_profile_entry* out, int32_t max_entries, int32_t* n_out);

/* ------------------------------------------------------------------------
 * DiffWave (AB_GEN_DIFFWAVE): DiffWave.forward and the denoising step of vocoder_inference
 * (models/vocoders/diffusion/diffusion_vocoder_inference.py:13-73).  The conditioning (upsampled mel and the diffusion
 * projections of every step the call will use) is computed once into the workspace by ab_diffwave_condition; each
 * ab_diffwave_step is one network pass over the audio that reads it.  The audio of `frames` mel frames has
 * frames * prod(upsample_rates) samples.  Workspace: ab_diffwave_workspace_bytes(g, batch, frames, n_steps), 256-byte
 * aligned; the same workspace and shapes for the condition call and the steps that follow it.
 * ---------------------------------------------------------------------- */
size_t ab_diffwave_workspace_bytes(const ab_generator* g, int64_t batch, int64_t frames, int32_t n_steps);
/* mel [B, n_mel, frames] fp32, any element strides; host_steps [n_steps] diffusion steps (an integer step as its float
 * value, which the lerp reproduces exactly), each with 0 <= floor and ceil < embedding_rows. */
int ab_diffwave_condition(ab_generator* g, const float* dev_mel, int64_t batch, int64_t frames, const int64_t mel_strides[3],
                          const float* host_steps, int32_t n_steps, void* dev_workspace, size_t workspace_bytes,
                          void* stream);
/* One network pass over dev_audio [B, frames * hop] (contiguous) with the step of conditioning row step_row for every
 * utterance, or row b for utterance b when step_row = -1 (n_steps == B).  dev_eps != NULL: eps [B, 1, frames * hop]
 * is written and the audio is left alone.  dev_eps == NULL: the sampler update in place, audio = clamp(c1 (audio -
 * c2 eps) + sigma noise, -1, 1), the noise term only when dev_noise [B, frames * hop] is given. */
int ab_diffwave_step(ab_generator* g, float* dev_audio, int64_t batch, int64_t frames, int32_t step_row, float c1,
                     float c2, float sigma, const float* dev_noise, float* dev_eps, void* dev_workspace,
                     size_t workspace_bytes, void* stream);
/* DiffWave.forward(audio, diffusion_step, spectrogram): ab_diffwave_condition with n_steps = 1 (one step for the batch)
 * or B (one per utterance), then ab_diffwave_step writing eps. */
int ab_diffwave_forward(ab_generator* g, const float* dev_audio, int64_t batch, int64_t frames, const float* dev_mel,
                        const int64_t mel_strides[3], const float* host_steps, int32_t n_steps, float* dev_eps,
                        void* dev_workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * FACodec decoder (AB_GEN_FACODEC): FACodecDecoder.vq2emb and .inference (models/codec/ns3_codec/facodec.py:556-576).
 * ---------------------------------------------------------------------- */
/* codes int64 [n_q, B, T] with element strides codes_strides (prosody layers, then content, then residual) ->
 * out [B, in_channels, T] fp32 contiguous.  Each ResidualVQ sums its layers in layer order (quantize/rvq.py:75-81), then
 * out = prosody + content [+ residual].  n_q is the total number of layers, or the prosody + content layers when
 * use_residual == 0.  A code outside [0, 2^bits) is never read: its time step of `out` is written as NaN. */
int ab_facodec_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_q, int64_t batch,
                      int64_t frames, int32_t use_residual, float* dev_out, void* stream);
/* x [B, in_channels, T] fp32 with any element strides, spk [B, in_channels] fp32 with row stride spk_row_stride ->
 * wav [B, 1, T * prod(up_ratios)].  Also serves a redecoder handle (FACodecRedecoder.inference, facodec.py:761-769).  Workspace: ab_generator_workspace_bytes.  Tail events (ab_generator_set_tail_events)
 * split conv_post into batch chunks as for the other generators.  set_option's "resblock_fusion" is accepted and
 * changes nothing: every FACodec conv runs as a single conv. */
int ab_facodec_inference(ab_generator* g, const float* dev_x, int64_t batch, int64_t frames, const int64_t x_strides[3],
                         const float* dev_spk, int64_t spk_row_stride, float* dev_wav, void* dev_workspace,
                         size_t workspace_bytes, void* stream);
/* FACodecDecoder.forward(x, vq=True) in eval (facodec.py:408-471, quantize/rvq.py, quantize/fvq.py, transformer.py), on a
 * handle created with facodec_quantize = 1 (else AB_ERR_STATE).  Extra tensors: "quantizer.{q}.layers.{j}.in_proj.weight"
 * (weight norm) / ".in_proj.bias", "timbre_encoder.position_emb.pe" [5000, 1, 256], per layer l
 * "timbre_encoder.layers.{l}.{ln_1,ln_2}.{weight,bias}", ".self_attn.in_proj_weight" [768, 256], ".self_attn.in_proj_bias",
 * ".self_attn.out_proj.{weight,bias}", ".ffn.ffn_1.{weight,bias}" (k = 5), ".ffn.ffn_2.{weight,bias}", and
 * "timbre_encoder.last_ln.{weight,bias}".
 * x [B, 256, T] fp32 with any element strides.  Each ResidualVQ runs its first min(n_quantizers, layers) layers; per
 * layer z_e = in_proj(residual), code = argmin over the L2-normalised codebook of the squared distance to the
 * normalised z_e (ties: the lowest code), z_q = z_e + (codebook[code] - z_e) in fp32, q = out_proj(z_q), residual -= q,
 * and the group's sum += q; the residual group reads x - (prosody + content).  All of it in fp32 on CUDA cores at every
 * precision.  Outputs (contiguous): emb_out [B, 256, T] = prosody + content [+ residual], codes_out int64
 * [n_used, B, T] (each group's rows in order), quantized_out [G, B, 256, T] (each group's sum; G = 2 + (residual group
 * present)), spk_out [B, 256] = the time mean of the timbre encoder's output, which adds row b of "pe" to every time
 * step of utterance b (the reference's batch-first PositionalEncoding), then 4 pre-LN layers (MHA with 4 heads, no mask;
 * a k = 5 conv FFN with ReLU) and last_ln.  Refused before any launch: n_quantizers < 1, B > 5000 (the rows of pe).
 * Workspace: ab_facodec_quantize_workspace_bytes, 256-byte aligned. */
size_t ab_facodec_quantize_workspace_bytes(const ab_generator* g, int64_t batch, int64_t frames);
int ab_facodec_quantize(ab_generator* g, const float* dev_x, const int64_t x_strides[3], int64_t batch, int64_t frames,
                        int32_t n_quantizers, float* dev_emb_out, int64_t* dev_codes_out, float* dev_quantized_out,
                        float* dev_spk_out, void* dev_workspace, size_t workspace_bytes, void* stream);
/* FACodecDecoderV2.forward(x, prosody_feature, vq=True) in eval (facodec.py:1027-1094), on a handle created with
 * facodec_prosody_encoder = 1 (else AB_ERR_STATE; ab_facodec_quantize refuses such a handle with AB_ERR_STATE, as the V2
 * forward has no form without the prosody feature).  prosody [B, 20, T] fp32 with any element strides, T the frames of
 * x.  The prosody group quantizes melspec_encoder(melspec_linear(prosody^T))^T instead of x: per frame the input
 * projection (an fp32 FMA chain over the 20 rows from 0, then the bias) plus row b of "melspec_encoder.position_emb.pe",
 * then 4 pre-LN layers and last_ln, all fp32 on CUDA cores at every precision (its output is quantized).  The content
 * group reads x, the residual group x - (prosody + content); everything else, the outputs and their layout are as in
 * ab_facodec_quantize.  Launches: 1 input projection, 4 x 7 layer launches, last_ln, then ab_facodec_quantize's 31.
 * Workspace: ab_facodec_quantize_workspace_bytes (on such a handle it sizes this call), 256-byte aligned. */
int ab_facodec_quantize_prosody(ab_generator* g, const float* dev_x, const int64_t x_strides[3], const float* dev_prosody,
                                const int64_t prosody_strides[3], int64_t batch, int64_t frames, int32_t n_quantizers,
                                float* dev_emb_out, int64_t* dev_codes_out, float* dev_quantized_out, float* dev_spk_out,
                                void* dev_workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * FACodec redecoder (AB_GEN_FACODEC_REDECODER): FACodecRedecoder.vq2emb (models/codec/ns3_codec/facodec.py:734-759);
 * its inference is ab_facodec_inference above.
 * ---------------------------------------------------------------------- */
/* codes int64 [n_q, B, T] with element strides codes_strides, read by position (prosody rows, content rows, then
 * residual rows; rows past those read are ignored), spk [B, 256] fp32 with row stride spk_row_stride -> out [B, 256, T]
 * fp32 contiguous.  Per prosody table i: x_t = Transformer(x_t + prosody_embs[i](codes[i])) (x_t starts at 0), where the
 * transformer adds row b of "pe" to every time step of utterance b (the batch-first PositionalEncoding) and runs 4 pre-LN
 * layers (MHA with 4 heads, no mask; a k = 5 conv FFN with ReLU) and last_ln, every LayerNorm style-adaptive:
 * gamma * LayerNorm(x) + beta (eps 1e-5, no affine) with (gamma, beta) = style(speaker embedding).  (The reference feeds
 * style the time mean of the embedding expanded over T, the embedding itself up to fp32 rounding of the sum.)  Then
 * out = ((x_t + content_0) + content_1 ...) [+ residual_0 ...] with use_residual, one fp32 add per term.  The gathers,
 * sums, style Linears and LayerNorm statistics are fp32 at every precision; the GEMMs take 16-bit operands at
 * AB_PREC_TC_*.  A code outside its table is never read: its time step is written as NaN (a bad prosody code spreads
 * through the attention to its whole utterance).  Refused before any launch: n_q below the rows read, B > 5000 (the rows
 * of pe), a short or unaligned workspace.  Launches: 9 style Linears, per prosody table 30 (the gather, 4 x 7 layer
 * launches, last_ln), and the tail gather.  Workspace: ab_facodec_redecoder_vq2emb_workspace_bytes, 256-byte aligned. */
size_t ab_facodec_redecoder_vq2emb_workspace_bytes(const ab_generator* g, int64_t batch, int64_t frames);
int ab_facodec_redecoder_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_q,
                                int64_t batch, int64_t frames, const float* dev_spk, int64_t spk_row_stride,
                                int32_t use_residual, float* dev_out, void* dev_workspace, size_t workspace_bytes,
                                void* stream);

/* ------------------------------------------------------------------------
 * The codec's ResidualVQ (AB_GEN_RVQ): ResidualVQ.forward in eval and ResidualVQ.vq2emb
 * (models/codec/amphion_codec/quantize/residual_vq.py:69-144).  The first n_quantizers layers run (1..num_quantizers).
 * Per layer, in fp32 on CUDA cores: z_e = in_project(residual) (an FMA chain over the input channels from 0, then the
 * bias); code = argmin over the L2-normalised codebook of the squared distance to the normalised z_e (ties: the lowest
 * code); z_q = z_e + (codebook[code] - z_e); q = out_project(z_q) (an FMA chain from 0, then the bias); residual -= q.
 * quantized_out = ((0 + q_0) + q_1) + ..., the reference's order.  No workspace.
 * ---------------------------------------------------------------------- */
/* x [B, input_dim, T] fp32 with any element strides -> quantized_out [B, input_dim, T], codes_out int64 [n, B, T] and
 * layers_out [n, B, input_dim, T] (each layer's q, the reference's all_quantized), all contiguous.  layers_out may be
 * NULL: nothing is written in its place.  One launch. */
int ab_rvq_quantize(ab_generator* g, const float* dev_x, const int64_t x_strides[3], int64_t batch, int64_t frames,
                    int32_t n_quantizers, float* dev_quantized_out, int64_t* dev_codes_out, float* dev_layers_out,
                    void* stream);
/* codes int64 [>= n, B, T] with element strides codes_strides -> out [B, input_dim, T] fp32 contiguous, the sum of
 * out_project(codebook[code]) over the first n layers in layer order, from 0.  A code outside [0, codebook_size) is never
 * read: its time step of `out` is written as NaN.  One launch. */
int ab_rvq_vq2emb(ab_generator* g, const int64_t* dev_codes, const int64_t codes_strides[3], int32_t n_quantizers,
                  int64_t batch, int64_t frames, float* dev_out, void* stream);

/* ------------------------------------------------------------------------
 * FACodec encoder (AB_GEN_FACODEC_ENCODER): FACodecEncoder.forward / .inference (models/codec/ns3_codec/facodec.py:157-194).
 * ---------------------------------------------------------------------- */
/* frames F of the encoder's output for `samples` input samples; 0 when a stage would be empty (or g is not an encoder) */
int64_t ab_facodec_encoder_frames(const ab_generator* g, int64_t samples);
/* wav [B, 1, N] fp32 with any element strides -> out [B, out_channels, F] fp32 contiguous, F = ab_facodec_encoder_frames.
 * Workspace: ab_generator_workspace_bytes(g, B, N), 256-byte aligned.  AB_ERR_ARG before any launch when F == 0. */
int ab_facodec_encode(ab_generator* g, const float* dev_wav, int64_t batch, int64_t samples, const int64_t wav_strides[3],
                      float* dev_out, void* dev_workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Activation1d(Snake|SnakeBeta).forward  (modules/anti_aliasing/act.py:31-36,
 * resample.py:36-45,62-65, filter.py:92-99, activation_functions/snake.py:51-61,110-122)
 * standalone: x [B,C,T] -> y [B,C,T], both contiguous fp32.  beta may alias alpha (Snake).
 * ---------------------------------------------------------------------- */
int ab_activation1d_forward(const float* dev_x, float* dev_y, int64_t batch, int64_t channels,
                            int64_t length, const float* dev_alpha, const float* dev_beta,
                            int32_t logscale, const float* dev_filter_up12,
                            const float* dev_filter_down12, void* stream);
/* The same Activation1d as one launch of what a generator handle runs (no reference counterpart; exposed for the
 * bit-exact tests): the 12 + 12 taps are HOST arrays, packed as ab_generator_finalize packs them and passed by value.
 * y (fp32 [B, C, T]) and yimg (operand image [B][ceil16(C)/8][T][8] of y, padding channels zero, rounded to
 * `precision` = AB_PREC_TC_F16 | AB_PREC_TC_BF16) may each be NULL, not both.  At a tensor-core precision a launch
 * with yimg and no y evaluates sin(u a) without the explicit range reduction, as the tensor-core generators do
 * (DESIGN 4.3); every launch with y keeps it.  AB_ERR_ARG before any launch for a NULL input, no output, yimg at
 * AB_PREC_FP32 or an unknown precision. */
int ab_activation1d_packed_forward(const float* dev_x, float* dev_y, uint16_t* dev_yimg, int64_t batch,
                                   int64_t channels, int64_t length, const float* dev_alpha, const float* dev_beta,
                                   int32_t logscale, const float* filter_up12, const float* filter_down12,
                                   int32_t precision, void* stream);

/* Snake1d (models/codec/amphion_codec/codec.py:32-48) as one launch of what the codec encoder runs (no reference
 * counterpart; exposed for the bit-exact tests).  x [B, C, T] fp32 contiguous, alpha [C] -> y (fp32 [B, C, T]) and / or
 * yimg (the operand image [B][ceil16(C)/8][T][8] of y, padding channels zero, rounded to nearest with saturation to
 * `precision` = AB_PREC_TC_F16 | AB_PREC_TC_BF16); either may be NULL, not both.  Per element, in fp32 with no
 * contraction: s = sinf(alpha x) (CUDA's sinf), y = x + (1 / (alpha + 1e-9)) * (s * s), the reciprocal correctly
 * rounded; the same at every precision.  AB_ERR_ARG before any launch for a NULL input, no output, yimg at AB_PREC_FP32
 * or an unknown precision. */
int ab_snake1d_forward(const float* dev_x, float* dev_y, uint16_t* dev_yimg, int64_t batch, int64_t channels,
                       int64_t length, const float* dev_alpha, int32_t precision, void* stream);

/* ------------------------------------------------------------------------
 * Building blocks exposed for parity tests (each is one launch of the kernel
 * the generator itself uses).
 * conv1d:  y = post( (bias + W * pre(x)) [+ residual] ), "same" zero padding,
 *          F.conv1d semantics of hifigan.py:96-99.  w is [Cout, Cin, k].
 * conv_transpose1d: nn.ConvTranspose1d(stride=u, padding=(k-u)/2) of
 *          hifigan.py:176-186.  w is [Cin, Cout, k].
 * pre_slope: 1.0 = no activation, otherwise leaky_relu negative slope.
 * ---------------------------------------------------------------------- */
int ab_conv1d_forward(const float* dev_x, const float* dev_w, const float* dev_bias,
                      const float* dev_residual, float* dev_y, int64_t batch, int64_t cin,
                      int64_t cout, int64_t length, int32_t ksize, int32_t dilation,
                      float pre_slope, int32_t post_tanh, int32_t precision,
                      void* dev_workspace, size_t workspace_bytes, void* stream);
size_t ab_conv1d_workspace_bytes(int64_t cin, int64_t cout, int32_t ksize, int32_t precision);
size_t ab_conv_transpose1d_workspace_bytes(int64_t cin, int64_t cout, int32_t ksize, int32_t stride,
                                          int32_t precision);
int ab_conv_transpose1d_forward(const float* dev_x, const float* dev_w, const float* dev_bias,
                                float* dev_y, int64_t batch, int64_t cin, int64_t cout,
                                int64_t length_in, int32_t ksize, int32_t stride, float pre_slope,
                                int32_t precision, void* dev_workspace, size_t workspace_bytes,
                                void* stream);
/* tc_conv: one launch of the tensor-core convolution that the generators' wgmma layers run on (hconv_kernel from fp32
 * input; a ConvTranspose1d from an operand image on hitem_kernel).  act(x) = rnd(lrelu(x, pre_slope)) of x [B, Cin, T]
 * with element strides x_strides, or, when dev_ximg is given, the 16-bit operand image [B][ceil16(Cin)/8][T][8] of the
 * already activated input (mode 1: Cin % 16 == 0); rnd = round to nearest, saturating, to `precision`
 * (AB_PREC_TC_F16 | AB_PREC_TC_BF16).  The weight is repacked and packed into the workspace as ab_conv1d_forward does.
 *   mode 0, Conv1d "same", dilation d_or_u, odd k, w [Cout, Cin, k]:
 *     y = (((conv(act(x)) + bias) + residual) + acc_prev) * (1.0f / out_div); reflect = 1: ReflectionPad1d((k-1)d/2)
 *     in place of the zero padding (AB_ERR_ARG, nothing launched, when the reflection needs more than T samples)
 *   mode 1, ConvTranspose1d stride u = d_or_u, padding pad (-1: (k-u)/2), T*u outputs, w [Cin, Cout, k]:
 *     y = conv_transpose(act(x)) + bias; residual, acc_prev and out_div != 1 are refused
 *   mode 2, strided Conv1d, stride s = d_or_u (1..8), any k >= s, zero padding 0 <= pad < k, w [Cout, Cin, k]:
 *     y[t] = bias + sum_j W_j act(x)[s t + j - pad], T_out = (T + 2 pad - k) / s + 1 (AB_ERR_ARG when T + 2 pad < k);
 *     residual, acc_prev, out_div != 1, reflect and yimg are refused
 *   y fp32 [B, Cout, T_out]; dev_yimg (nullable): the operand image [B][ceil16(Cout)/8][T_out][8] of
 *   rnd(lrelu(y, img_slope)), padding channels zero (mode 1: Cout % 16 == 0).  bias, residual, acc_prev nullable. */
size_t ab_tc_conv_workspace_bytes(int32_t mode, int64_t cin, int64_t cout, int32_t ksize, int32_t d_or_u);
int ab_tc_conv_forward(int32_t mode, const float* dev_x, const int64_t x_strides[3], float pre_slope,
                       const uint16_t* dev_ximg, const float* dev_w, const float* dev_bias, const float* dev_residual,
                       const float* dev_acc_prev, float out_div, int32_t reflect, float* dev_y, uint16_t* dev_yimg,
                       float img_slope, int64_t batch, int64_t cin, int64_t cout, int64_t length, int32_t ksize,
                       int32_t d_or_u, int32_t pad, int32_t precision, void* dev_workspace, size_t workspace_bytes,
                       void* stream);
/* DiffWave building blocks: one launch each of the kernels ab_diffwave_step / ab_diffwave_condition run (no reference
 * counterpart; exposed for the bit-exact tests).  Every tensor fp32, contiguous unless strides are given; C = 64.
 * diffwave_layer: one ResidualBlock (diffwave.py:96-124) from the state-dict layouts dilated_conv [2C, C, 3] + [2C],
 *   conditioner_projection [2C, n_mel(, 1)] + [2C], output_projection [2C, C(, 1)] + [2C]; the weights are packed into
 *   the workspace (ab_diffwave_layer_workspace_bytes(n_mel), 256-byte aligned) as ab_generator_finalize packs them,
 *   then the layer kernel of `precision` runs once.  x_in [B, C, L]; d: utterance b's diffusion projection [C] at
 *   d + b d_batch_stride (0: one for the batch); cond: the upsampled mel [B, n_mel, L]; any L >= 1, dilation >= 1.
 *   y = dilated_conv(x + d) + conditioner_projection(cond) (the two biases summed first), z = sigmoid(gate) tanh(filter),
 *   (res, s) = output_projection(z); x_out = (x_in + res) / sqrt(2) (x_out != x_in), skip = s (first != 0) or skip + s.
 * diffwave_tail: skip [B, C, L] -> s = skip / skip_div, h = relu(skip_projection(s)), e = output_projection(h); dev_eps
 *   != NULL: eps [B, L] = e; otherwise audio [B, L] = clamp(c1 (audio - c2 e) + sigma noise, -1, 1) in place, the noise
 *   term only when dev_noise [B, L] is given.  wsk [C, C(, 1)], bsk [C], wo [1, C(, 1)], bo [1].
 * diffwave_upsample: SpectrogramUpsampler (diffwave.py:68-93) of mel [B, n_mel, frames] with element strides mel_strides:
 *   two ConvTranspose2d(1, 1, [3, 2f], stride [1, f], padding [1, f / 2]) (weights [3, 2f], biases [1]), each followed by
 *   leaky_relu(0.4), even f1, f2 -> out [B, n_mel, frames f1 f2]. */
/* FACodecDecoderV2's prosody input projection: the first launch of ab_facodec_quantize_prosody, alone (no reference
 * counterpart; exposed for the bit-exact tests).  x [B, 20, T] fp32 with any element
 *   strides, w [256, 20] (nn.Linear layout), bias [256], pe [>= B][256] (row b for utterance b) -> y [B, 256, T] fp32
 *   contiguous, y[b, c, t] = ((fma chain over i = 0..19 of w[c][i] x[b, i, t], from 0) + bias[c]) + pe[b][c]. */
int ab_facodec_prosody_input_forward(const float* dev_x, const int64_t x_strides[3], const float* dev_w,
                                     const float* dev_bias, const float* dev_pe, int64_t batch, int64_t frames,
                                     float* dev_y, void* stream);
/* Vocos building blocks: one launch each of the kernels forward_vocos runs for a ConvNeXt block and the head (no
 * reference counterpart; exposed for the bit-exact tests).  Every fp32 tensor contiguous.
 * vocos_norm: LayerNorm over channels (two-pass mean and biased variance, then (x - mean) * rstd * ln_w + ln_b) of x
 *   [B, C, T], optionally after the k = 7 zero-padded depthwise conv (dw_w [C, 1, 7] and dw_b [C], both or neither).
 *   Exactly one of y (fp32 [B, C, T]) and yimg (operand image [B][ceil16(C)/8][T][8], padding channels zero, rounded
 *   to `precision` = AB_PREC_TC_F16 | AB_PREC_TC_BF16; ignored for y) is given.  AB_ERR_UNSUPPORTED, nothing launched,
 *   when a time tile of C channels does not fit shared memory.
 * vocos_pointwise: Linear over channels, w [C_out, C_in] (nn.Linear) and bias [C_out], packed into the workspace
 *   (ab_vocos_pointwise_workspace_bytes, 256-byte aligned) as ab_generator_finalize packs it, then
 *     AB_VOCOS_PW_GELU:     tc: ximg in -> yimg = the image of gelu(W x + b) (padding channels zero);
 *                           fp32: x [B, C_in, T] in -> y = gelu(W x + b)
 *     AB_VOCOS_PW_GAMMA:    y = y + gamma * (W x + b) in place, fp32 [B, C_out, T] (tc: from ximg; fp32: from x)
 *     AB_VOCOS_PW_SPECTRUM: spec [B*T][C_out/2] complex (interleaved re, im) = min(exp(m), 1e2) (cos p + i sin p), m and
 *                           p the first and second halves of W x + b (Vocos' ISTFTHead; even C_out)
 *     AB_VOCOS_PW_LINEAR:   y = W x + b written time-major, fp32 [B, T, C_out] (nn.Linear's layout; tc: from ximg;
 *                           fp32: from x, acc = fma(w[co][ci], x[ci], acc) for ci ascending from 0, then + b[co]);
 *                           gamma, yimg and spec must be NULL
 *   At AB_PREC_TC_F16 / TC_BF16 the input is the operand image ximg [B][ceil16(C_in)/8][T][8] and one pointwise wgmma
 *   GEMM launch runs; at AB_PREC_FP32 the input is x and the CUDA-core conv kernel runs with k = 1 (SPECTRUM: into the
 *   workspace, then ab_spectral_head_forward per utterance).  The other input and the outputs an epilogue does not
 *   write may be NULL.  AB_ERR_ARG before any launch for an input that does not match the precision, a missing
 *   output or gamma, or an odd C_out with SPECTRUM. */
#define AB_VOCOS_PW_GELU 0
#define AB_VOCOS_PW_GAMMA 1
#define AB_VOCOS_PW_SPECTRUM 2
#define AB_VOCOS_PW_LINEAR 3
int ab_vocos_norm_forward(const float* dev_x, const float* dev_dw_w, const float* dev_dw_b, const float* dev_ln_w,
                          const float* dev_ln_b, float eps, float* dev_y, uint16_t* dev_yimg, int32_t precision,
                          int64_t batch, int64_t channels, int64_t length, void* stream);
size_t ab_vocos_pointwise_workspace_bytes(int32_t epilogue, int64_t batch, int64_t cin, int64_t cout, int64_t length,
                                          int32_t precision);
int ab_vocos_pointwise_forward(int32_t epilogue, const float* dev_x, const uint16_t* dev_ximg, const float* dev_w,
                               const float* dev_bias, const float* dev_gamma, float* dev_y, uint16_t* dev_yimg,
                               float* dev_spec, int64_t batch, int64_t cin, int64_t cout, int64_t length,
                               int32_t precision, void* dev_workspace, size_t workspace_bytes, void* stream);
size_t ab_diffwave_layer_workspace_bytes(int32_t n_mel);
int ab_diffwave_layer_forward(const float* dev_x_in, const float* dev_d, int64_t d_batch_stride, const float* dev_cond,
                              const float* dev_wdil, const float* dev_bdil, const float* dev_wcond, const float* dev_bcond,
                              const float* dev_wout, const float* dev_bout, float* dev_x_out, float* dev_skip, int64_t batch,
                              int64_t length, int32_t n_mel, int32_t dilation, int32_t first, int32_t precision,
                              void* dev_workspace, size_t workspace_bytes, void* stream);
int ab_diffwave_tail_forward(const float* dev_skip, const float* dev_wsk, const float* dev_bsk, const float* dev_wo,
                             const float* dev_bo, float skip_div, int64_t batch, int64_t length, float* dev_eps,
                             float* dev_audio, const float* dev_noise, float c1, float c2, float sigma, void* stream);
int ab_diffwave_upsample_forward(const float* dev_mel, const int64_t mel_strides[3], const float* dev_w1, const float* dev_b1,
                                 const float* dev_w2, const float* dev_b2, int32_t f1, int32_t f2, int64_t batch,
                                 int32_t n_mel, int64_t frames, float* dev_out, void* stream);

/* ------------------------------------------------------------------------
 * Mel front end:
 *   extract_mel_features / mel_spectrogram_torch / extract_linear_features
 *     (utils/mel.py:20-170): pad = (n_fft-hop)/2, eps = 1e-9 / 1e-6
 *   TacotronSTFT.mel_spectrogram (utils/stft.py:259-278 over STFT.transform
 *     :152-181): pad = n_fft/2, eps = 0, with_energy
 * Pipeline: reflect-pad + frame + window kernel -> cuFFT R2C (the libcufft.so.11
 * already loaded in the process, i.e. the one torch.stft uses) -> fused
 * |.|, mel filterbank, log(clamp) kernel.
 * ---------------------------------------------------------------------- */
typedef struct ab_mel ab_mel;

typedef struct ab_mel_config {
  int32_t n_fft;
  int32_t hop;
  int32_t win;      /* window length; the window is centred in n_fft (torch.stft / pad_center) */
  int32_t n_mel;    /* 0 = magnitude only (extract_linear_features) */
  int32_t pad;      /* reflect padding per side */
  float eps;        /* added under the sqrt */
  float clamp;      /* log(clamp(x, min=clamp)); 1e-5 in the reference */
} ab_mel_config;

int ab_mel_create(const ab_mel_config* cfg, ab_mel** out);
void ab_mel_destroy(ab_mel* m);
int64_t ab_mel_num_frames(const ab_mel* m, int64_t samples);
size_t ab_mel_workspace_bytes(const ab_mel* m, int64_t batch, int64_t samples);
/* wav [B,T] contiguous; window [win]; mel_basis [n_mel, n_fft/2+1];
 * outputs (each may be NULL): magnitude [B, n_fft/2+1, F], mel [B, n_mel, F],
 * energy [B, F] (l2 norm of the magnitude over bins, utils/stft.py:276). */
int ab_mel_forward(ab_mel* m, const float* dev_wav, int64_t batch, int64_t samples,
                   const float* dev_window, const float* dev_mel_basis, float* dev_magnitude,
                   float* dev_mel, float* dev_energy, void* dev_workspace, size_t workspace_bytes,
                   void* stream);
/* Gradient of ab_mel_forward's log-mel output with respect to the waveform (the mel loss of the vocoder trainers,
 * models/vocoders/gan/gan_vocoder_trainer.py:368-396): grad_mel [B, n_mel, F] in, grad_wav [B, T] out (overwritten).
 * The spectrum is recomputed from wav, turned into its cotangent in place, taken back with cuFFT C2R and
 * overlap-added through the window and the reflect padding.  The clamp passes the gradient where the mel value
 * is >= clamp, as torch.clamp does.  Workspace: ab_mel_backward_workspace_bytes, 256-byte aligned. */
size_t ab_mel_backward_workspace_bytes(const ab_mel* m, int64_t batch, int64_t samples);
int ab_mel_backward(ab_mel* m, const float* dev_wav, int64_t batch, int64_t samples,
                    const float* dev_window, const float* dev_mel_basis, const float* dev_grad_mel,
                    float* dev_grad_wav, void* dev_workspace, size_t workspace_bytes, void* stream);
/* amplitude_phase_spectrum (utils/mel.py:244-280; APNet's training features, cfg.preprocess.extract_amplitude_phase):
 * the framing + cuFFT of ab_mel_forward, then log(|X| + 1e-5), atan2(im, re), re, im, each [B, n_fft/2+1, F] (any may
 * be NULL).  re / im are bit-identical to torch.stft on the same device.  Workspace: ab_mel_workspace_bytes. */
int ab_amplitude_phase_forward(ab_mel* m, const float* dev_wav, int64_t batch, int64_t samples, const float* dev_window,
                               float* dev_logamp, float* dev_pha, float* dev_rea, float* dev_imag,
                               void* dev_workspace, size_t workspace_bytes, void* stream);
/* iSTFT head of the amplitude/phase generators (APNet.forward, models/vocoders/gan/generator/apnet.py:378-399):
 * logamp, R, I [B, bins, F] -> pha = atan2(I, R), rea = exp(logamp) cos(pha), imag = exp(logamp) sin(pha)
 * (each output [B, bins, F], may be NULL) and the complex spectrum [B*F][bins] (interleaved re, im; may be NULL)
 * laid out for ab_istft_forward.  dev_i == NULL: dev_r already is the phase, and amp_max > 0 clips exp(logamp) —
 * Vocos' ISTFTHead (models/codec/kmeans/vocos.py:333-361: S = clip(exp(mag), max=1e2) (cos p + i sin p)). */
int ab_spectral_head_forward(const float* dev_logamp, const float* dev_r, const float* dev_i, int64_t batch, int64_t bins,
                             int64_t frames, float amp_max, float* dev_pha, float* dev_rea, float* dev_imag, float* dev_spec,
                             void* stream);
/* ISTFT.forward with padding="same" (apnet.py:46-104): irfft (norm "backward") of every frame, times the window,
 * overlap-add, divided by the overlap-added squared window, trimmed by (win - hop)/2 per side.
 * spec [B*F][n_fft/2+1] complex interleaved (overwritten), window [win], wav [B, F*hop].  The handle supplies
 * n_fft / hop / win (win == n_fft, as the reference's broadcast requires); 256-byte aligned workspace. */
size_t ab_istft_workspace_bytes(const ab_mel* m, int64_t batch, int64_t frames);
int ab_istft_forward(ab_mel* m, float* dev_spec, int64_t batch, int64_t frames, const float* dev_window, float* dev_wav,
                     void* dev_workspace, size_t workspace_bytes, void* stream);
/* Same mel / energy outputs from ONE kernel for n_fft = 1024 (the 22.05 / 24 kHz configs): frame, window, an in-kernel
 * 512-point complex FFT of the even/odd-packed frame, real-FFT post-processing, |.|, mel filterbank, log — the wav is
 * the only HBM read and mel / energy the only writes (utils/stft.py:259-278, utils/mel.py:145-169).  fp32 with an own
 * FFT: agrees with ab_mel_forward to ~1e-6 in the log-mel, NOT bit for bit (use ab_mel_forward where the spectrum
 * must equal torch.stft's).  AB_ERR_UNSUPPORTED for other n_fft / n_mel > 128.  Workspace: >= 1 KB, 256-byte aligned. */
int ab_mel_forward_fused(ab_mel* m, const float* dev_wav, int64_t batch, int64_t samples,
                         const float* dev_window, const float* dev_mel_basis, float* dev_mel, float* dev_energy,
                         void* dev_workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Waveform -> 16-bit PCM: the arithmetic of save_audio (utils/io.py:49-76) on the device, applied to a
 * batch of generator outputs before the D2H copy (SURVEY 8f rank 1).
 *   dev_wav [batch, samples] fp32 with row stride `row_stride`; dev_lengths [batch] int64 valid samples per
 *   row (NULL = all `samples`); turn_up: scale each row by volume_peak / max|w| over its valid samples
 *   (io.py:59-62); silence: zero samples put before and after each row (fs // 20 for add_silence, io.py:64-68);
 *   dev_out [batch, out_stride] int16, out_stride even and >= samples + 2*silence; the tail of every row
 *   beyond silence + length + silence is zero.  Quantiser: clamp(floor(w * 32768 + 0.5), -32768, 32767)
 *   (torchaudio 2.0.2 sox_io, PCM_S 16 — io.py:76).  Workspace: ab_pcm16_workspace_bytes(batch) when turn_up. */
size_t ab_pcm16_workspace_bytes(int64_t batch);
int ab_pcm16_forward(const float* dev_wav, int64_t batch, int64_t samples, int64_t row_stride,
                     const int64_t* dev_lengths, int32_t turn_up, float volume_peak, int64_t silence,
                     int16_t* dev_out, int64_t out_stride, void* dev_workspace, size_t workspace_bytes,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AMPHION_B200_H_ */
