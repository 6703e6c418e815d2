// Tensor-core (wgmma / bulk-TMA) convolution path — interface.  One kernel (ab_kernels_tc.cu) serves the three
// parameter sets below; the weight image of a layer depends only on (mode, C_in, C_out, k, dilation | stride).
#pragma once
#include "ab_common.cuh"

namespace ab {

// One launch = nconv (1 or 2) k-tap "same" convolutions over C channels:
//   nconv == 2:  y = ((conv2(lrelu(conv1(lrelu(x,pre),d1)+b1, mid), 1)+b2) + residual + acc_prev) / out_div
//   nconv == 1:  y = ((conv1(lrelu(x,pre),d1)+b1) + residual + acc_prev) / out_div
// i.e. one (c1, c2) step of ResBlock1.forward (hifigan.py:93-100) or one step
// of ResBlock2.forward (:139-144), plus the branch mix of hifigan.py:208-214.
struct TcConvParams {
  const float* x;         // contiguous [B, C, T] fp32
  float* y;               // contiguous [B, C, T] fp32
  const float* residual;  // nullable
  const float* acc_prev;  // nullable
  const void* w1;         // operand image built by launch_tc_pack_weight
  const float* b1;
  const void* w2;         // nullable when nconv == 1
  const float* b2;
  int B, C, T;
  int k, d1, nconv;
  float pre_slope, mid_slope, out_div;
  int precision;          // AB_PREC_TC_F16 | AB_PREC_TC_BF16
  // fp16/bf16 operand images [B][Np/8][T][8] (Np = C rounded up to 16): when ximg is given the prologue is
  // a cp.async burst of already activated operands (pre_slope is ignored); when yimg is given the epilogue
  // also stores cvt(lrelu(y, img_slope)) for the next kernel
  const uint16_t* ximg;
  uint16_t* yimg;
  float img_slope;
};

// Non-square Conv1d (mode 0) and polyphase ConvTranspose1d (mode 1), N-blocked over C_out
struct GcParams {
  const float* x;         // [B, Cin, Tin] fp32 with element strides xsb / xsc / xst
  int64_t xsb, xsc, xst;
  const uint16_t* ximg;   // optional: already activated operand image [B][ceil16(Cin)/8][Tin][8] (then x is unused)
  float* y;               // conv: [B, Cout, Tin]; conv-transpose: [B, Cout, Tin*u]
  const void* w;          // operand image built by launch_gc_pack_weight
  const float* bias;      // nullable
  const float* residual;  // conv only, nullable
  int B, Cin, Cout, Tin;
  int mode;               // 0 conv, 1 conv-transpose
  int k, d, u;
  float pre_slope;
  int post_tanh;          // conv only
  int precision;
  uint16_t* yimg;         // conv-transpose only, nullable: operand image of lrelu(y, img_slope)
  float img_slope;
};
bool gc_can_emit_image(int cout, int k, int u);

// Wide layers (C > 256, several N blocks): like GcParams with a contiguous input, the branch sum and out_div.
//   y = ((conv(act(x), d) + bias) + residual + acc_prev) / out_div
struct GsParams {
  const uint16_t* ximg;   // [B][ceil16(Cin)/8][T][8] already activated operands, or nullptr ->
  const float* x;         //   fp32 [B, Cin, T] contiguous, activated with lrelu(., pre_slope) in the loader
  float pre_slope;
  int mode;               // 0 conv ("same", dilation d); 1 conv-transpose (stride u, padding (k-u)/2)
  int u;
  uint16_t* yimg;         // conv-transpose only, nullable
  float img_slope;
  float* y;               // conv: [B, Cout, T]; conv-transpose: [B, Cout, T*u]
  const void* w;          // image built by launch_gs_pack_weight
  const float* bias;
  const float* residual;  // nullable
  const float* acc_prev;  // nullable
  int B, Cin, Cout, T;
  int k, d;
  float out_div;
  int precision;
};
size_t gs_weight_image_bytes(int mode, int cin, int cout, int k, int d_or_u);
int launch_gs_pack_weight(const float* w_t, void* image, int mode, int cin, int cout, int k, int d_or_u,
                          int precision, cudaStream_t s);
bool gs_can_emit_image(int cout, int k, int u);
int launch_gemmconv_stream(const GsParams& p, cudaStream_t s);
size_t gc_weight_image_bytes(int mode, int cin, int cout, int k, int d_or_u);
int launch_gc_pack_weight(const float* w_t, void* image, int mode, int cin, int cout, int k, int d_or_u,
                          int precision, cudaStream_t s);
int launch_gemmconv(const GcParams& p, cudaStream_t s);


// One whole ResBlock per launch ("block mode", C <= 64): npairs x nconv k-tap convs with the residual stream x_p in
// registers and the halo recomputed inside the time tile, so the block reads its input once and writes its output once.
//   for q < npairs:  x <- x + conv[q][1](lrelu(conv[q][0](lrelu(x, slope), dil[q]) + b, slope), 1) + b   (nconv == 2)
//                    x <- x + conv[q][0](lrelu(x, slope), dil[q]) + b                                      (nconv == 1)
//   y = (x + acc_prev) / out_div ; yimg = cvt(lrelu(y, img_slope))
// Same arithmetic in the same order as npairs launches of launch_tc_conv: the results are bit-equal.
constexpr int AB_TC_CHAIN_MAX_PAIRS = 3;
constexpr int AB_TC_CHAIN_MAX_C = 64;
struct TcChainParams {
  const float* x;          // contiguous [B, C, T] fp32 (block input = first residual)
  const uint16_t* ximg;    // nullable: operand image of lrelu(x, slope), [B][ceil16(C)/8][T][8]
  float* y;                // contiguous [B, C, T] fp32
  const float* acc_prev;   // nullable (may alias y)
  uint16_t* yimg;          // nullable
  const void* w[2 * AB_TC_CHAIN_MAX_PAIRS];      // tc weight images, step = pair * nconv + conv
  const float* bias[2 * AB_TC_CHAIN_MAX_PAIRS];  // nullable entries
  int dil[AB_TC_CHAIN_MAX_PAIRS];
  int npairs, nconv;
  int B, C, T, k;
  float slope, img_slope, out_div;
  int precision;
};
// rows computed per valid output row (>= 1) of the block-mode tile, 0 when the block is not served
double tc_chain_recompute(int C, int k, const int* dil, int npairs, int nconv);
int launch_tc_chain(const TcChainParams& p, cudaStream_t s);

int tc_max_channels();
bool tc_conv_supported(int C, int k);
size_t tc_weight_image_bytes(int cin, int cout, int k);
size_t tc_act_image_bytes(int64_t B, int C, int64_t T);
// w_t: fp32 [Cin][k][Cout] (the repacked fp32 image) -> 16-bit operand image
int launch_tc_pack_weight(const float* w_t, void* image, int cin, int cout, int k, int precision,
                          cudaStream_t s);
int launch_tc_conv(const TcConvParams& p, cudaStream_t s);

}  // namespace ab
