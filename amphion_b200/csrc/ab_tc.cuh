// Tensor-core (wgmma / bulk-TMA) convolution path — interface.  launch_tc_conv runs every tensor-core Conv1d and
// ConvTranspose1d (ab_kernels_tc.cu: hconv_kernel, or the persistent hpair_kernel for a conv pair and hitem_kernel for
// a ConvTranspose1d from an operand image); block mode (launch_tc_chain) runs on hchain_kernel and Vocos' pointwise
// layers (launch_tc_pointwise) on hitem_kernel.  The weight image of a layer depends only on (mode, C_in, C_out, k,
// dilation | stride).
#pragma once
#include "ab_common.cuh"

namespace ab {

// One launch of launch_tc_conv, act(x) = lrelu(x, pre_slope) or the operand image ximg:
//   conv (mode 0, "same", dilation d_or_u):  y = ((conv(act(x), d) + bias) + residual + acc_prev) / out_div  [tanh]
//   pair (mode 0 with w2):  y = ((conv2(lrelu(conv(act(x), d) + bias, mid_slope), 1) + b2) + residual + acc_prev) / out_div
//     i.e. one (c1, c2) step of ResBlock1.forward (hifigan.py:93-100); a single conv is one step of ResBlock2
//     (:139-144); residual, acc_prev and out_div are the branch mix of hifigan.py:208-214
//   conv-transpose (mode 1, stride u = d_or_u, padding `pad`, T*u outputs):  y = conv_transpose(act(x), u) + bias
struct TcConvParams {
  int mode = 0;                      // 0 conv, 1 conv-transpose, 2 strided conv (stride d_or_u, padding pad)
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
  float* y = nullptr;                // conv: [B, Cout, T]; conv-transpose: [B, Cout, T*u]; strided: [B, Cout, (T+2pad-k)/s+1]
  uint16_t* yimg = nullptr;          // nullable (tc_can_emit_image): operand image of lrelu(y, img_slope) for the next kernel
  float img_slope = 1.0f;
  int B = 0, Cin = 0, Cout = 0, T = 0, k = 0, d_or_u = 1;
  int precision = AB_PREC_FP32;      // set to AB_PREC_TC_F16 | AB_PREC_TC_BF16 (fp32 is rejected)
  int reflect = 0;                   // conv only, no w2: ReflectionPad1d((k-1)*d/2) in place of zero padding (MelGAN)
  int pad = -1;                      // conv-transpose padding, 0 <= pad < k; -1 = (k-u)/2 (HiFi-GAN; MelGAN: u//2 + u%2);
                                     // strided conv: zero padding on both sides, 0 <= pad < k
};
// 16-bit weight image of a layer, 0 when launch_tc_conv cannot run it
size_t tc_weight_image_bytes(int mode, int cin, int cout, int k, int d_or_u);
// w_t: fp32 [Cin][k][Cout] (the repacked fp32 image) -> the layer's weight image
int launch_tc_pack_weight(const float* w_t, void* image, int mode, int cin, int cout, int k, int d_or_u, int precision,
                          cudaStream_t s);
// whether a launch of this layer can write yimg (the image's padding channels come out zero)
bool tc_can_emit_image(int mode, int cin, int cout, int k, int d_or_u);
int launch_tc_conv(const TcConvParams& p, cudaStream_t s);


// One whole ResBlock per launch ("block mode", C <= 128): npairs x nconv k-tap convs with the residual stream x_p in
// registers and the halo recomputed inside the time tile, so the block reads its input once and writes its output once.
// The residual stream takes as many registers per thread as the accumulators (64 up to N = 128, one m64 tile per
// consumer warpgroup at 128); at N = 256 the two would need 128 + 128.
//   for q < npairs:  x <- x + conv[q][1](lrelu(conv[q][0](lrelu(x, slope), dil[q]) + b, slope), 1) + b   (nconv == 2)
//                    x <- x + conv[q][0](lrelu(x, slope), dil[q]) + b                                      (nconv == 1)
//   y = (x + acc_prev) / out_div ; yimg = cvt(lrelu(y, img_slope))
// Same arithmetic in the same order as npairs launches of launch_tc_conv: the results are bit-equal.
constexpr int AB_TC_CHAIN_MAX_PAIRS = 3;
constexpr int AB_TC_CHAIN_MAX_C = 128;
// largest stride of launch_tc_conv's strided conv (mode 2)
constexpr int AB_TC_MAX_STRIDE = 8;
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

// Pointwise (1x1, nn.Linear over channels) GEMM of Vocos (hitem_kernel): input the operand image of x, any C_in / C_out.
//   AB_PW_GELU:            yimg = image of gelu(W x + b)                    (ConvNeXtBlock pwconv1 + nn.GELU())
//   AB_PW_GAMMA_RESIDUAL:  y = y + gamma * (W x + b), fp32 [B, C_out, T]    (pwconv2, layer scale, residual)
//   AB_PW_SPECTRUM:        spec [B*T][C_out/2] complex = min(exp(m), 1e2) (cos p + i sin p), m / p the two halves of
//                          W x + b (ISTFTHead); w from launch_tc_pack_head_weight
//   AB_PW_LINEAR:          y = W x + b, fp32 time-major [B, T, C_out]       (nn.Linear's output layout)
enum { AB_PW_GELU = 0, AB_PW_GAMMA_RESIDUAL = 1, AB_PW_SPECTRUM = 2, AB_PW_LINEAR = 3 };
struct TcPwParams {
  int epilogue = AB_PW_GELU;
  const uint16_t* ximg = nullptr;   // [B][ceil16(Cin)/8][T][8], padding channels zero
  const void* w = nullptr;          // launch_tc_pack_weight(mode 0, k 1) image, or launch_tc_pack_head_weight
  const float* bias = nullptr;      // [Cout]
  const float* gamma = nullptr;     // AB_PW_GAMMA_RESIDUAL
  uint16_t* yimg = nullptr;         // AB_PW_GELU: [B][ceil16(Cout)/8][T][8] (padding channels written as zero)
  float* y = nullptr;               // AB_PW_GAMMA_RESIDUAL [B, C_out, T]; AB_PW_LINEAR [B, T, C_out]
  float* spec = nullptr;            // AB_PW_SPECTRUM: interleaved (re, im)
  int B = 0, Cin = 0, Cout = 0, T = 0;
  int precision = AB_PREC_TC_F16;
};
int launch_tc_pack_head_weight(const float* w_t, void* image, int cin, int cout, int precision, cudaStream_t s);
int launch_tc_pointwise(const TcPwParams& p, cudaStream_t s);

// square convs that pair mode and block mode serve (C <= 256, odd k <= 31)
bool tc_conv_supported(int C, int k);
size_t tc_act_image_bytes(int64_t B, int C, int64_t T);

}  // namespace ab
