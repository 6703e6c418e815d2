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
 * "conv_post" (the caller maps ASP_input_conv / ASP_ResNet.j / ASP_output_conv ... onto them). */
enum ab_generator_kind { AB_GEN_HIFIGAN = 0, AB_GEN_BIGVGAN = 1, AB_GEN_NSFHIFIGAN = 2, AB_GEN_TRUNK = 3 };
enum ab_activation { AB_ACT_LRELU = 0, AB_ACT_SNAKE = 1, AB_ACT_SNAKEBETA = 2 };
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
  /* AB_GEN_TRUNK only (0 elsewhere) */
  int32_t trunk_out_channels;                   /* conv_post output channels (n_fft/2+1, or 2*(n_fft/2+1) for R|I) */
  int32_t trunk_in_kernel;                      /* conv_pre kernel size (odd) */
  int32_t trunk_out_kernel;                     /* conv_post kernel size (odd) */
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
 * "conv_transpose1d_fp32", "activation1d", "tc_gemmconv" (max_entries >= 5). */
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
 *   whole ResBlock per launch (residual stream in registers, halo recomputed in the tile) where served (C <= 64) and
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
 * Activation1d(Snake|SnakeBeta).forward  (modules/anti_aliasing/act.py:31-36,
 * resample.py:36-45,62-65, filter.py:92-99, activation_functions/snake.py:51-61,110-122)
 * standalone: x [B,C,T] -> y [B,C,T], both contiguous fp32.  beta may alias alpha (Snake).
 * ---------------------------------------------------------------------- */
int ab_activation1d_forward(const float* dev_x, float* dev_y, int64_t batch, int64_t channels,
                            int64_t length, const float* dev_alpha, const float* dev_beta,
                            int32_t logscale, const float* dev_filter_up12,
                            const float* dev_filter_down12, void* stream);

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
