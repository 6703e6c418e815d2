// Tensor-core (wgmma / bulk-TMA) convolution path — interface.  hconv_kernel (ab_kernels_tc.cu) runs every
// tensor-core Conv1d and ConvTranspose1d through launch_tc_conv; block mode (launch_tc_chain) has a kernel of its own.
// The weight image of a layer depends only on (mode, C_in, C_out, k, dilation | stride).
#pragma once
#include "ab_common.cuh"

namespace ab {

// One launch of hconv_kernel, act(x) = lrelu(x, pre_slope) or the operand image ximg:
//   conv (mode 0, "same", dilation d_or_u):  y = ((conv(act(x), d) + bias) + residual + acc_prev) / out_div  [tanh]
//   pair (mode 0 with w2):  y = ((conv2(lrelu(conv(act(x), d) + bias, mid_slope), 1) + b2) + residual + acc_prev) / out_div
//     i.e. one (c1, c2) step of ResBlock1.forward (hifigan.py:93-100); a single conv is one step of ResBlock2
//     (:139-144); residual, acc_prev and out_div are the branch mix of hifigan.py:208-214
//   conv-transpose (mode 1, stride u = d_or_u, padding (k-u)/2):  y = conv_transpose(act(x), u) + bias
struct TcConvParams {
  int mode = 0;                      // 0 conv, 1 conv-transpose
  const float* x = nullptr;          // fp32 [B, Cin, T] with element strides xsb / xsc / xst (unused when ximg is given)
  int64_t xsb = 0, xsc = 0, xst = 0;
  const uint16_t* ximg = nullptr;    // nullable: operand image [B][ceil16(Cin)/8][T][8] of the activated input
  float pre_slope = 1.0f;
  const void* w = nullptr;           // weight image built by launch_tc_pack_weight
  const float* bias = nullptr;       // nullable
  const void* w2 = nullptr;          // pair mode (conv, C_in == C_out, tc_conv_supported): conv2's image and bias
  const float* b2 = nullptr;
  float mid_slope = 1.0f;
  const float* residual = nullptr;   // conv only, nullable
  const float* acc_prev = nullptr;   // conv only, nullable (may alias y)
  float out_div = 1.0f;              // conv only
  int post_tanh = 0;                 // conv only
  float* y = nullptr;                // conv: [B, Cout, T]; conv-transpose: [B, Cout, T*u]
  uint16_t* yimg = nullptr;          // nullable (tc_can_emit_image): operand image of lrelu(y, img_slope) for the next kernel
  float img_slope = 1.0f;
  int B = 0, Cin = 0, Cout = 0, T = 0, k = 0, d_or_u = 1;
  int precision = AB_PREC_FP32;      // set to AB_PREC_TC_F16 | AB_PREC_TC_BF16 (fp32 is rejected)
};
// 16-bit weight image of a layer, 0 when hconv_kernel cannot run it
size_t tc_weight_image_bytes(int mode, int cin, int cout, int k, int d_or_u);
// w_t: fp32 [Cin][k][Cout] (the repacked fp32 image) -> the layer's weight image
int launch_tc_pack_weight(const float* w_t, void* image, int mode, int cin, int cout, int k, int d_or_u, int precision,
                          cudaStream_t s);
// whether a launch of this layer can write yimg (the image's padding channels come out zero)
bool tc_can_emit_image(int mode, int cin, int cout, int k, int d_or_u);
int launch_tc_conv(const TcConvParams& p, cudaStream_t s);


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

// square convs that pair mode and block mode serve (C <= 256, odd k <= 31)
bool tc_conv_supported(int C, int k);
size_t tc_act_image_bytes(int64_t B, int C, int64_t T);

}  // namespace ab
