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
};

struct ConvTParams {
  const float* x;       // contiguous [B, Cin, Tin]
  const float* w_t;     // repacked [Cin][k][Cout]
  const float* bias;
  float* y;             // contiguous [B, Cout, Tin*u]
  int B, Cin, Cout, Tin;
  int k, u;
  float pre_slope;
};

#ifdef __CUDACC__
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
  return lo + hi;
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

// launchers (ab_kernels_fp32.cu)
int launch_conv1d_fp32(const ConvParams& p, cudaStream_t s);
int launch_conv_transpose1d_fp32(const ConvTParams& p, cudaStream_t s);
int launch_activation1d(const SnakeParams& p, cudaStream_t s);
// Repack a conv weight into [Cin][k][Cout] fp32, folding weight norm if g != nullptr.
// transposed == 0: src is [Cout][Cin][k] (Conv1d); 1: src is [Cin][Cout][k] (ConvTranspose1d).
int launch_repack_weight(const float* v, const float* g, float* dst, int d0, int d1, int k,
                         int transposed, cudaStream_t s);

int launch_scale_inplace(float* p, size_t n, float gain, cudaStream_t s);
// x[b, c, :] += bias[c] + sum_i w[c, i] * g[b, i]   (1x1 conditioning conv on a per-utterance vector, hifigan.py:429-430)
int launch_cond_add(float* x, const float* g, int64_t g_batch_stride, const float* w, const float* bias, int B, int C,
                    int gin, int T, cudaStream_t s);

}  // namespace ab
