// Shared host/device helpers for libamphion_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/amphion_b200.h"

namespace ab {

// ---- error plumbing (thread-local message, integer codes across the C ABI) ----
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

#define AB_CUDA_TRY(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess)                                                             \
      return ::ab::fail(AB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                           \
  } while (0)

#define AB_LAUNCH_CHECK(what)                                                          \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess)                                                             \
      return ::ab::fail(AB_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(_e)); \
  } while (0)

// cudaFuncSetAttribute is per device: `flags` (one static array per call site) remembers which devices were set up
struct DeviceOnce {
  bool done[64] = {};
  bool need() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
  }
};

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- fp32 (CUDA-core) convolution parameters --------------------------------
// y = post( ((bias + W * lrelu(x, pre_slope)) + residual + acc_prev) / out_div )
struct ConvParams {
  const float* x;       // [B, Cin, T] with element strides xsb/xsc/xst
  int64_t xsb, xsc, xst;
  const float* w_t;     // repacked [Cin][k][Cout]
  const float* bias;    // [Cout] or nullptr
  const float* residual;  // contiguous [B, Cout, T] or nullptr
  const float* acc_prev;  // contiguous [B, Cout, T] or nullptr (branch accumulation)
  float* y;             // contiguous [B, Cout, T]
  int B, Cin, Cout, T;
  int k, d;
  float pre_slope;      // 1.0f = no activation
  float out_div;        // 1.0f = none (IEEE division, as the reference's xs / num_kernels)
  int post_tanh;
  int reflect = 0;      // 1: ReflectionPad1d((k-1)*d/2) in place of zero padding (MelGAN, melgan.py:39-40,59-66,90-95)
  // Vocos' pointwise layers (vocos.py:509-527), replacing residual / acc_prev / out_div / tanh:
  //   CONV_EPI_GELU: y = gelu(bias + W x) (exact erf);  CONV_EPI_GAMMA_RESIDUAL: y = residual + gamma * (bias + W x)
  //   CONV_EPI_LINEAR (k = 1 only): y = W x + bias written time-major, y[b, t, co] of a contiguous [B, T, Cout]
  int epi = 0;
  const float* gamma = nullptr;   // [Cout]
};
enum { CONV_EPI_NONE = 0, CONV_EPI_GELU = 1, CONV_EPI_GAMMA_RESIDUAL = 2, CONV_EPI_LINEAR = 3 };

struct ConvTParams {
  const float* x;       // contiguous [B, Cin, Tin]
  const float* w_t;     // repacked [Cin][k][Cout]
  const float* bias;
  float* y;             // contiguous [B, Cout, Tin*u]
  int B, Cin, Cout, Tin;
  int k, u;
  int pad;              // ConvTranspose1d padding: (k-u)/2 for HiFi-GAN, r//2 + r%2 for MelGAN (melgan.py:73-80)
  float pre_slope;
};

#ifdef __CUDACC__
// ReflectionPad1d: the row of a length-T sequence that time t of the padded sequence reads (t in (-T, 2T - 1)); callers
// zero-fill when the result lies outside [0, T), which only happens for rows no valid output reads.
__device__ __forceinline__ int reflect_time(int t, int T) { return t < 0 ? -t : (t >= T ? 2 * (T - 1) - t : t); }

// fp32 pairs in an aligned 64-bit register, so that 8- and 16-byte shared-memory loads deliver pairs without any
// move.  Hopper has no packed fp32 arithmetic: each op is two scalar IEEE round-to-nearest ops (the explicit
// intrinsics keep the compiler from contracting a mul and an add into one FMA).
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk2(float lo, float hi) {
  f32x2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ float hsum2(f32x2 v) {
  float lo, hi;
  upk2(v, lo, hi);
  return __fadd_rn(lo, hi);
}

__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1); upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}

#endif

// Filter taps of one Activation1d as the packed pairs the kernel multiplies with (host-side copy, passed by value so
// they sit in the constant bank / uniform registers): see snake_segment in ab_kernels_fp32.cu.
struct SnakeCoef {
  float2 ce_a[3], co_a[3], ce_b[4], co_b[4], fd2[6];
};
void pack_snake_coef(const float* f_up, const float* f_down, SnakeCoef* out);   // host pointers, 12 taps each

struct SnakeParams {
  SnakeCoef kc;         // valid when have_kc (the generator path); otherwise the kernel reads f_up / f_down
  int have_kc = 0;
  int fast_snake = 0;   // image-only launches may use the snake without explicit range reduction (tensor-core generators)
  const float* x;       // contiguous [B, C, T]
  float* y;
  const float* alpha;   // [C]
  const float* beta;    // [C] (== alpha for Snake)
  const float* f_up;    // [12]
  const float* f_down;  // [12]
  int B, C, T;
  int logscale;
  uint16_t* yimg;       // optional 16-bit operand image [B][ceil16(C)/8][T][8] of y (y itself may then be null)
  int bf16;
};

// Vocos LayerNorm over the channels of every time step (eps, two-pass mean and biased variance, affine; vocos.py:
// 493-527, :758-783), optionally after the k = 7 zero-padded depthwise conv with bias (ConvNeXtBlock.dwconv).
struct NormParams {
  const float* x = nullptr;       // contiguous [B, C, T] fp32
  const float* dw_w = nullptr;    // nullable: depthwise weight [C][7]; dw_b its bias [C]
  const float* dw_b = nullptr;
  const float* ln_w = nullptr;    // [C]
  const float* ln_b = nullptr;    // [C]
  float* y = nullptr;             // fp32 [B, C, T] output, or
  uint16_t* yimg = nullptr;       // 16-bit operand image [B][ceil16(C)/8][T][8] (padding channels zero)
  int bf16 = 0;
  int B = 0, C = 0, T = 0;
  float eps = 1e-6f;
};

// ---- DiffWave (ab_diffwave.cu) -------------------------------------------
constexpr int DW_CHANNELS = 64;   // residual_channels the DiffWave kernels are compiled for

struct DwUpsampleParams {   // SpectrogramUpsampler: mel [B, n_mel, F] (element strides) -> out [B, n_mel, F f1 f2]
  const float* mel;
  int64_t msb, msc, mst;
  const float *w1, *b1, *w2, *b2;   // ConvTranspose2d weights [3][2 f] and biases [1]
  float* out;
  int B, n_mel, F, f1, f2;
};
struct DwEmbedParams {      // d [steps][layers][C] from the step values (host-checked to index the table)
  const float* steps;
  const float* table;               // [rows][128]
  const float *w1, *b1, *w2, *b2;   // projection1 [512][128], projection2 [512][512]
  const float *wd, *bd;             // every layer's diffusion_projection, [layers][C][512] and [layers][C]
  float* d;
  int layers;
};
struct DwLayerParams {      // one ResidualBlock
  const float* x_in;      // [B, C, L]
  float* x_out;           // [B, C, L], not x_in (neighbouring tiles read x_in's halo)
  float* skip;            // [B, C, L] running skip sum
  const float* cond;      // upsampled mel [B, n_mel, L]
  const float* d;         // this layer's diffusion projection [C] of utterance 0
  int64_t d_bstride;      // 0: one step for the batch
  const float *w1, *b1, *w2, *b2;   // packed by launch_dw_pack (b1 / b2 serve both paths)
  const uint16_t *w1h, *w2h;        // 16-bit images for the tensor-core layer kernel (precision != AB_PREC_FP32)
  int precision;
  int B, n_mel, dil, first;
  int64_t L;
};
struct DwTailParams {
  const float* skip;
  const float *wsk, *bsk, *wo, *bo;   // skip_projection [C][C], output_projection [C]
  float skip_div;                      // sqrt(residual_layers)
  int B;
  int64_t L;
  float* eps;                          // [B, L], or nullptr: sampler update of audio
  float* audio;
  const float* noise;                  // nullable
  float c1, c2, sigma;
};
struct DwPackParams {
  const float *wdil, *bdil, *wcond, *bcond, *wout, *bout;   // state-dict layouts
  float *w1p, *b1p, *w2p, *b2p;   // [3C + n_mel][2C], [2C], [C][2C], [2C]
  uint16_t *w1h, *w2h;            // nullptr, or the 16-bit images [2C][dw_k1p(n_mel)] and [2C][C] (column-major in K)
  int bf16;
  int n_mel;
};
// K of the tensor-core conv1: three dilated taps of C channels, then n_mel rounded up to 16
inline int dw_k1p(int n_mel) { return 3 * DW_CHANNELS + (n_mel + 15) / 16 * 16; }
size_t dw_layer_smem_bytes(int n_mel, int precision);
int launch_dw_upsample(const DwUpsampleParams& p, cudaStream_t s);
int launch_dw_embed(const DwEmbedParams& p, int steps, cudaStream_t s);
int launch_dw_input(const float* audio, const float* w, const float* bias, float* x, int B, int64_t L, cudaStream_t s);
int launch_dw_layer(const DwLayerParams& p, cudaStream_t s);
int launch_dw_tail(const DwTailParams& p, cudaStream_t s);
int launch_dw_pack(const DwPackParams& p, cudaStream_t s);

// ---- FACodec decoder prologue (ab_facodec.cu) ----------------------------
constexpr int FAC_MAX_CODEBOOK_DIM = 16;
struct FacFilmParams {      // y = LayerNorm(x over channels, eps 1e-5, no affine) * gamma + beta
  const float* x;           // [B, C, T] with element strides xsb / xsc / xst
  int64_t xsb, xsc, xst;
  const float* style;       // [B][2C]: gamma then beta (timbre_linear's output)
  float* y;                 // fp32 [B, C, T], or
  uint16_t* yimg;           // 16-bit operand image [B][ceil16(C)/8][T][8] (padding channels zero)
  int bf16;
  int B, C, T;
};
struct FacVqParams {        // out [B, C, T] = sum over the groups of (sum over the group's layers of out_proj(codebook[code]))
  const int64_t* codes;     // [nq, B, T] with element strides cs0 / cs1 / cs2
  int64_t cs0, cs1, cs2;
  const float* cb[AB_FACODEC_MAX_Q];     // codebook [rows][D]
  const float* w[AB_FACODEC_MAX_Q];      // out_proj, repacked [D][C] (weight norm folded)
  const float* bias[AB_FACODEC_MAX_Q];   // [C]
  int64_t rows[AB_FACODEC_MAX_Q];
  int group_end[3];         // layer q belongs to the first group g with q < group_end[g]
  int ngroups, nq;
  int B, C, T, D;
  float* out;
};
int launch_facodec_style(const float* spk, int64_t spk_stride, const float* w, const float* bias, float* style, int B,
                         int C, cudaStream_t s);
int launch_facodec_film(const FacFilmParams& p, cudaStream_t s);
int launch_facodec_vq2emb(const FacVqParams& p, cudaStream_t s);

// ---- FACodecDecoder.forward(vq=True): the RVQ and the timbre encoder's own kernels (ab_facodec.cu) ----
constexpr int FAC_TIMBRE_C = 256;         // encoder_hidden of the timbre encoder (transformer.py:154-217)
constexpr int FAC_TIMBRE_HEADS = 4;
constexpr int FAC_PE_ROWS = 5000;         // PositionalEncoding's max_len: the rows of "pe"
struct FacRvqParams {       // quantize (facodec.py:408-445) for one tile of frames per CTA, and the positional add
  const float* x;           // [B, C, T] with element strides xsb / xsc / xst
  int64_t xsb, xsc, xst;
  const float* w_in[AB_FACODEC_MAX_Q];     // in_proj, repacked [C][D] (weight norm folded)
  const float* b_in[AB_FACODEC_MAX_Q];     // [D]
  const float* w_out[AB_FACODEC_MAX_Q];    // out_proj, repacked [D][C]
  const float* b_out[AB_FACODEC_MAX_Q];    // [C]
  const float* cb[AB_FACODEC_MAX_Q];       // codebook [rows][D] (the unnormalised rows z_q reads)
  const float* cbn[AB_FACODEC_MAX_Q];      // normalised codebook, rows padded to 16 floats [rows][16]
  const float* cbn2[AB_FACODEC_MAX_Q];     // squared norms of the normalised rows [rows]
  int64_t rows[AB_FACODEC_MAX_Q];
  int layer0[3], nused[3];  // per group: first layer index, layers run (0: group absent)
  int code_row0[3];         // per group: first row of codes_out
  int ngroups;              // 2 or 3: the planes of quantized_out
  int B, C, T, D;
  float* emb;               // [B, C, T]
  int64_t* codes;           // [n_used, B, T]
  float* quantized;         // [ngroups, B, C, T]
  const float* pe;          // nullable: [rows][C]; stream[b, c, t] = x[b, c, t] + pe[b][c]
  float* stream;            // [B, C, T]
};
// normalised codebook rows (F.normalize, eps 1e-12) padded to 16 floats, and their squared norms
int launch_facodec_cbnorm(const float* cb, float* cbn, float* cbn2, int64_t rows, int D, cudaStream_t s);
// prosody == nullptr: FACodecDecoder's RVQ (every group reads x); else FACodecDecoderV2's (facodec.py:1027-1094): the
// prosody group reads prosody [B, C, T] (contiguous), the content group x, the residual group x - (prosody + content).
// one_group: the codec's ResidualVQ, one group (ngroups 1, emb unused, C <= AB_RVQ_MAX_INPUT_DIM): quantized [B, C, T]
// is its sum and layers, when given, [n_used, B, C, T] each layer's term
int launch_facodec_rvq(const FacRvqParams& p, cudaStream_t s, const float* prosody = nullptr, float* layers = nullptr,
                       bool one_group = false);
// softmax(q k^T / 8) v per (utterance, head) from qkv [B, 3 * 256, T] (q, k, v rows; time fastest) -> y fp32 [B, 256, T]
// or the operand image yimg [B][32][T][8]
int launch_facodec_attention(const float* qkv, float* y, uint16_t* yimg, int bf16, int B, int T, cudaStream_t s);
// spk[b][c] = sum_t y[b, c, t] / T (fixed order)
int launch_facodec_time_mean(const float* y, float* spk, int B, int C, int T, cudaStream_t s);

// ---- FACodecDecoderV2.forward(vq=True): the prosody transformer's input (ab_facodec.cu) ----
constexpr int FAC_PROSODY_BINS = 20;      // melspec_linear's in_features: the first 20 mel rows
struct FacProsodyInParams { // y[b, c, t] = ((sum_i w[c][i] x[b, i, t]) + bias[c]) + pe[b][c]
  const float* x;           // [B, 20, T] with element strides xsb / xsi / xst
  int64_t xsb, xsi, xst;
  const float* w;           // melspec_linear.weight [256][20] (nn.Linear layout)
  const float* bias;        // [256]
  const float* pe;          // [>= B][256]
  float* y;                 // fp32 [B, 256, T]
  int B, T;
};
int launch_facodec_prosody_input(const FacProsodyInParams& p, cudaStream_t s);

// ---- FACodecRedecoder.vq2emb: the embedding gathers and sums (ab_facodec.cu) ----
struct FacEmbedParams {     // out[b, c, t] = ((prev[b, c, t] + tab[0][code_0][c]) + tab[1][code_1][c] ...) + pe[b][c],
                            // one fp32 add per term in that order; without prev the first table's row is the first term
  const int64_t* codes;     // [n_q, B, T] with element strides cs0 / cs1 / cs2; table j reads code row row0 + j
  int64_t cs0, cs1, cs2;
  int row0, ntab;
  const float* tab[AB_FACODEC_MAX_Q];   // nn.Embedding weights [rows][C]
  int64_t rows[AB_FACODEC_MAX_Q];
  const float* prev;        // nullable: fp32 [B, C, T]
  const float* pe;          // nullable: [>= B][C]; row b is added last
  float* out;               // fp32 [B, C, T]; a time step with a code outside its table holds NaN in every channel
  int B, C, T;
};
int launch_facodec_embed(const FacEmbedParams& p, cudaStream_t s);

// launchers (ab_kernels_fp32.cu)
int launch_vocos_norm(const NormParams& p, cudaStream_t s);
int launch_conv1d_fp32(const ConvParams& p, cudaStream_t s);
// strided conv1d (zero padding pad, (T + 2 pad - k) / stride + 1 outputs; p.d = 1, no epilogue terms): p.T is the input
// length and p.y holds [B, Cout, T_out]
int launch_conv1d_strided_fp32(const ConvParams& p, int stride, int pad, cudaStream_t s);
int launch_conv_transpose1d_fp32(const ConvTParams& p, cudaStream_t s);
int launch_activation1d(const SnakeParams& p, cudaStream_t s);
// Snake1d (codec.py:32-48) of contiguous x [B, C, T]: fp32 y and / or the operand image yimg [B][ceil16(C)/8][T][8]
int launch_snake1d(const float* x, float* y, uint16_t* yimg, int bf16, const float* alpha, int B, int C, int T,
                   cudaStream_t s);
// Repack a conv weight into [Cin][k][Cout] fp32, folding weight norm if g != nullptr.
// transposed == 0: src is [Cout][Cin][k] (Conv1d); 1: src is [Cin][Cout][k] (ConvTranspose1d).
int launch_repack_weight(const float* v, const float* g, float* dst, int d0, int d1, int k,
                         int transposed, cudaStream_t s);

int launch_scale_inplace(float* p, size_t n, float gain, cudaStream_t s);
// x[b, c, :] += bias[c] + sum_i w[c, i] * g[b, i]   (1x1 conditioning conv on a per-utterance vector, hifigan.py:429-430)
int launch_cond_add(float* x, const float* g, int64_t g_batch_stride, const float* w, const float* bias, int B, int C,
                    int gin, int T, cudaStream_t s);

}  // namespace ab
