// CUDA-core fp32 kernels: the exact-arithmetic path (AB_PREC_FP32) and the
// pieces that are not channel-mixing contractions (anti-aliased Snake, weight
// repacking).  Reference semantics are cited per kernel (paths relative to the
// Amphion reference root).
#include <stdlib.h>

#include <algorithm>

#include "ab_common.cuh"

namespace ab {

// ===========================================================================
// conv1d: F.conv1d with "same" zero padding and dilation, fused with the
// leaky_relu in front of it, bias, residual add, branch accumulation, /nk and
// tanh  (hifigan.py:93-100 ResBlock1.forward, :139-144 ResBlock2.forward,
// :208-217 branch mix + conv_post + tanh).
// Tile: 64 output channels x 128 time steps per CTA, 4x8 outputs per thread.
// ===========================================================================
namespace {
constexpr int CO_T = 64;
constexpr int TT = 128;
constexpr int CI_T = 8;
constexpr int NT = 256;

// REFLECT: ReflectionPad1d(halo / 2) in place of the zero padding (MelGAN's ResnetBlock conv, melgan.py:39-40)
// EPI: ConvParams::epi (Vocos' pointwise layers); 0 = the generic epilogue below
template <int REFLECT, int EPI = CONV_EPI_NONE>
__global__ void __launch_bounds__(NT) conv1d_fp32_kernel(ConvParams p) {
  extern __shared__ float smem[];
  const int halo = (p.k - 1) * p.d;
  const int XW = TT + halo;
  float* xs = smem;               // [CI_T][XW]
  float* ws = smem + CI_T * XW;   // [CI_T][k][CO_T]
  const int t0 = blockIdx.x * TT, co0 = blockIdx.y * CO_T, b = blockIdx.z;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int pad = halo >> 1;
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.xsb;

  float acc[4][8];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += CI_T) {
    for (int idx = threadIdx.x; idx < CI_T * XW; idx += NT) {
      const int ci = idx / XW, n = idx - ci * XW;
      const int t = REFLECT ? reflect_time(t0 - pad + n, p.T) : t0 - pad + n, c = ci0 + ci;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.T) {
        v = __ldg(xb + (int64_t)c * p.xsc + (int64_t)t * p.xst);
        v = v >= 0.f ? v : v * slope;
      }
      xs[idx] = v;
    }
    const int wn = CI_T * p.k * CO_T;
    for (int idx = threadIdx.x; idx < wn; idx += NT) {
      const int co = idx & (CO_T - 1);
      const int r = idx / CO_T;  // ci * k + j
      const int ci = r / p.k;
      float v = 0.f;
      if (ci0 + ci < p.Cin && co0 + co < p.Cout)
        v = __ldg(p.w_t + ((int64_t)ci0 * p.k + r) * p.Cout + co0 + co);
      ws[idx] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < CI_T; ++ci) {
      const float* xr = xs + ci * XW + tx;
      const float* wr = ws + ci * p.k * CO_T + ty * 4;
      for (int j = 0; j < p.k; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(wr + j * CO_T);
        const float* xj = xr + j * p.d;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xv = xj[16 * i];
          acc[0][i] = fmaf(w.x, xv, acc[0][i]);
          acc[1][i] = fmaf(w.y, xv, acc[1][i]);
          acc[2][i] = fmaf(w.z, xv, acc[2][i]);
          acc[3][i] = fmaf(w.w, xv, acc[3][i]);
        }
      }
    }
    __syncthreads();
  }

  if constexpr (EPI == CONV_EPI_LINEAR) {
    // y[b, t, co] = acc + bias: the thread's 4 channels of a time step are one 16-byte store when C_out % 4 == 0
    // and y is 16-byte aligned
    const int cb = co0 + ty * 4;
    const bool vec = !(p.Cout & 3) && !(reinterpret_cast<uintptr_t>(p.y) & 15);
    float bv[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) bv[c] = cb + c < p.Cout ? __ldg(p.bias + cb + c) : 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + tx + 16 * i;
      if (t >= p.T) continue;
      float* y = p.y + ((int64_t)b * p.T + t) * p.Cout + cb;
      const float v[4] = {acc[0][i] + bv[0], acc[1][i] + bv[1], acc[2][i] + bv[2], acc[3][i] + bv[3]};
      if (vec && cb < p.Cout) {
        *reinterpret_cast<float4*>(y) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (cb + c < p.Cout) y[c] = v[c];
      }
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int co = co0 + ty * 4 + c;
    if (co >= p.Cout) continue;
    const float bv = p.bias ? __ldg(p.bias + co) : 0.f;
    const int64_t row = ((int64_t)b * p.Cout + co) * p.T;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + tx + 16 * i;
      if (t >= p.T) continue;
      float v = acc[c][i] + bv;
      if constexpr (EPI == CONV_EPI_GELU) {   // (0.5 v) (1 + erff(v / sqrt 2)), every step rounded
        v = __fmul_rn(__fmul_rn(0.5f, v), __fadd_rn(1.0f, erff(__fmul_rn(v, 0.70710678118654752440f))));
      } else if constexpr (EPI == CONV_EPI_GAMMA_RESIDUAL) {
        v = __fadd_rn(__ldg(p.residual + row + t), __fmul_rn(__ldg(p.gamma + co), v));
      } else {
        if (p.residual) v += __ldg(p.residual + row + t);
        if (p.acc_prev) v += __ldg(p.acc_prev + row + t);
        if (p.out_div != 1.0f) v = v / p.out_div;
        if (p.post_tanh) v = tanhf(v);
      }
      p.y[row + t] = v;
    }
  }
}

// Few output channels (conv_post: C -> 1, hifigan.py:199,216): one CTA per
// (batch, 1024-sample tile), all Cout (<= 4) per thread; HBM-bound.
constexpr int PT = 1024;
constexpr int PCI = 8;
template <int REFLECT>
__global__ void __launch_bounds__(NT) conv1d_fewout_fp32_kernel(ConvParams p) {
  extern __shared__ float smem[];
  const int halo = (p.k - 1) * p.d;
  const int XW = PT + halo;
  float* xs = smem;              // [PCI][XW]
  float* ws = smem + PCI * XW;   // [Cin][k][Cout] (whole filter)
  const int t0 = blockIdx.x * PT, b = blockIdx.z;
  const int pad = halo >> 1;
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.xsb;
  for (int idx = threadIdx.x; idx < p.Cin * p.k * p.Cout; idx += NT) ws[idx] = __ldg(p.w_t + idx);

  float acc[4][4];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[c][r] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += PCI) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < PCI * XW; idx += NT) {
      const int ci = idx / XW, n = idx - ci * XW;
      const int t = REFLECT ? reflect_time(t0 - pad + n, p.T) : t0 - pad + n, c = ci0 + ci;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.T) {
        v = __ldg(xb + (int64_t)c * p.xsc + (int64_t)t * p.xst);
        v = v >= 0.f ? v : v * slope;
      }
      xs[idx] = v;
    }
    __syncthreads();
    const int nci = min(PCI, p.Cin - ci0);
    for (int ci = 0; ci < nci; ++ci) {
      for (int j = 0; j < p.k; ++j) {
        const float* wv = ws + ((ci0 + ci) * p.k + j) * p.Cout;
        const float* xr = xs + ci * XW + j * p.d + threadIdx.x;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float xv = xr[NT * r];
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < p.Cout) acc[c][r] = fmaf(wv[c], xv, acc[c][r]);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c >= p.Cout) continue;
    const float bv = p.bias ? __ldg(p.bias + c) : 0.f;
    const int64_t row = ((int64_t)b * p.Cout + c) * p.T;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int t = t0 + threadIdx.x + NT * r;
      if (t >= p.T) continue;
      float v = acc[c][r] + bv;
      if (p.residual) v += __ldg(p.residual + row + t);
      if (p.acc_prev) v += __ldg(p.acc_prev + row + t);
      if (p.out_div != 1.0f) v = v / p.out_div;
      if (p.post_tanh) v = tanhf(v);
      p.y[row + t] = v;
    }
  }
}
// conv_post specialisation: one output channel, k = K taps, dilation 1 (hifigan.py:199,215-217).  Four
// consecutive outputs per thread from a (4 + K - 1)-sample register window (3 x LDS.128 per input channel),
// weights of the current 8-channel chunk in registers.  HBM-bound: reads C x T fp32 once.
template <int K, int REFLECT = 0>
__global__ void __launch_bounds__(NT) conv_post_fp32_kernel(ConvParams p) {
  constexpr int XWP = PT + 8;                   // padded row: 1024 outputs + K - 1 (<= 8) halo, 16-byte rows
  __shared__ __align__(16) float xs[PCI][XWP];
  __shared__ float ws[PCI * K];
  const int t0 = blockIdx.x * PT, b = blockIdx.z;
  constexpr int pad = (K - 1) / 2;
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.xsb;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int tl = 4 * threadIdx.x;
  for (int ci0 = 0; ci0 < p.Cin; ci0 += PCI) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < PCI * XWP; idx += NT) {
      const int ci = idx / XWP, n = idx - ci * XWP;
      const int t = REFLECT ? reflect_time(t0 - pad + n, p.T) : t0 - pad + n, c = ci0 + ci;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.T && n < PT + K - 1) {
        v = __ldg(xb + (int64_t)c * p.xsc + (int64_t)t * p.xst);
        v = v >= 0.f ? v : v * slope;
      }
      xs[ci][n] = v;
    }
    if (threadIdx.x < PCI * K) {
      const int ci = threadIdx.x / K, j = threadIdx.x - ci * K;
      ws[threadIdx.x] = (ci0 + ci < p.Cin) ? __ldg(p.w_t + (int64_t)(ci0 + ci) * K + j) : 0.f;   // [Cin][K][1]
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < PCI; ++ci) {
      float w[12];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(&xs[ci][tl + 4 * q]);
        w[4 * q] = t4.x; w[4 * q + 1] = t4.y; w[4 * q + 2] = t4.z; w[4 * q + 3] = t4.w;
      }
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const float wj = ws[ci * K + j];
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = fmaf(wj, w[r + j], acc[r]);
      }
    }
  }
  const float bv = p.bias ? __ldg(p.bias) : 0.f;
  float* yr = p.y + (int64_t)b * p.T + t0 + tl;
  float o[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float v = acc[r] + bv;
    if (p.post_tanh) v = tanhf(v);
    o[r] = v;
  }
  if (t0 + tl + 3 < p.T && (p.T & 3) == 0) {
    *reinterpret_cast<float4*>(yr) = make_float4(o[0], o[1], o[2], o[3]);
  } else {
#pragma unroll
    for (int r = 0; r < 4; ++r)
      if (t0 + tl + r < p.T) yr[r] = o[r];
  }
}
// The same arithmetic (same accumulation order: bit-identical results) for the layout the generators produce —
// contiguous rows, T % 4 == 0, 16-byte aligned: rows are staged with 16-byte loads/stores (the tile's aligned
// superset [t0 - 4, t0 + PT + 4) consists of float4 groups that lie entirely inside or outside the row), the weights
// are read as two broadcast LDS.128 per channel.  The generic kernel above spent ~25 instructions per staged
// element (index division, 64-bit address math, scalar LDG/STS): 1575 instructions per output against ~370 here.
// REFLECT (MelGAN's ReflectionPad1d(3) before conv_post, melgan.py:90-95): the staged tile is completed at the
// sequence ends from its own rows, which lie inside it (T % 4 == 0, T >= 4).
template <int K, int REFLECT = 0>
__global__ void __launch_bounds__(NT) conv_post_vec_kernel(ConvParams p) {
  static_assert(K <= 8, "weights are padded to 8 per channel");
  constexpr int XG = PT / 4 + 2;                // float4 groups per staged row
  __shared__ __align__(16) float xs[PCI][XG * 4];
  __shared__ __align__(16) float ws[PCI * 8];
  const int t0 = blockIdx.x * PT, b = blockIdx.z;
  constexpr int pad = (K - 1) / 2;
  static_assert(pad <= 3, "window offset");
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.xsb;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int tl = 4 * threadIdx.x;
  // All of a chunk's 16-byte groups are in flight at once: a thread owns groups tid, tid + 256, ... of the flattened
  // [PCI][XG] tile (loading row by row exposed one DRAM latency per row), and the NEXT chunk's groups are requested
  // before the current chunk is multiplied, so the latency hides under the FMAs.
  constexpr int NG = (PCI * XG + NT - 1) / NT;
  float4 v[NG];
  auto request = [&](int ci0) {
#pragma unroll
    for (int i = 0; i < NG; ++i) {
      const int idx = threadIdx.x + NT * i;
      const int ci = idx / XG, q = idx - ci * XG;
      const int t = t0 - 4 + 4 * q;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < PCI * XG && ci0 + ci < p.Cin && t >= 0 && t < p.T)
        v[i] = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)(ci0 + ci) * p.xsc + (t0 - 4)) + q);
    }
  };
  request(0);
  for (int ci0 = 0; ci0 < p.Cin; ci0 += PCI) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NG; ++i) {
      const int idx = threadIdx.x + NT * i;
      const int ci = idx / XG, q = idx - ci * XG;
      float4 w = v[i];
      w.x = w.x >= 0.f ? w.x : w.x * slope;
      w.y = w.y >= 0.f ? w.y : w.y * slope;
      w.z = w.z >= 0.f ? w.z : w.z * slope;
      w.w = w.w >= 0.f ? w.w : w.w * slope;
      if (idx < PCI * XG) *reinterpret_cast<float4*>(&xs[ci][4 * q]) = w;
    }
    if (REFLECT) {   // staged index n holds time t0 - 4 + n: x[-r] = x[r], x[T - 1 + r] = x[T - 1 - r], r = 1..pad
      __syncthreads();
      if (threadIdx.x < PCI * pad) {
        const int ci = threadIdx.x / pad, r = threadIdx.x - ci * pad + 1;
        if (t0 == 0) xs[ci][4 - r] = xs[ci][4 + r];
        const int n = p.T - 1 + r - t0 + 4;
        if (n >= 0 && n < XG * 4) xs[ci][n] = xs[ci][n - 2 * r];
      }
    }
    if (ci0 + PCI < p.Cin) request(ci0 + PCI);
    if (threadIdx.x < PCI * 8) {
      const int ci = threadIdx.x >> 3, j = threadIdx.x & 7;
      ws[threadIdx.x] = (ci0 + ci < p.Cin && j < K) ? __ldg(p.w_t + (int64_t)(ci0 + ci) * K + j) : 0.f;   // [Cin][K][1]
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < PCI; ++ci) {
      // staged index n holds time t0 - 4 + n: this thread's window starts at t0 + tl - pad = n0 + (4 - pad), n0 = tl
      float w[12];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(&xs[ci][tl + 4 * q]);
        w[4 * q] = t4.x; w[4 * q + 1] = t4.y; w[4 * q + 2] = t4.z; w[4 * q + 3] = t4.w;
      }
      float wj[8];
      {
        const float4 a4 = *reinterpret_cast<const float4*>(&ws[ci * 8]);
        const float4 b4 = *reinterpret_cast<const float4*>(&ws[ci * 8 + 4]);
        wj[0] = a4.x; wj[1] = a4.y; wj[2] = a4.z; wj[3] = a4.w; wj[4] = b4.x; wj[5] = b4.y; wj[6] = b4.z; wj[7] = b4.w;
      }
#pragma unroll
      for (int j = 0; j < K; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = fmaf(wj[j], w[r + j + (4 - pad)], acc[r]);
    }
  }
  const float bv = p.bias ? __ldg(p.bias) : 0.f;
  if (t0 + tl < p.T) {
    float o[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float v = acc[r] + bv;
      if (p.post_tanh) v = tanhf(v);
      o[r] = v;
    }
    *reinterpret_cast<float4*>(p.y + (int64_t)b * p.T + t0 + tl) = make_float4(o[0], o[1], o[2], o[3]);
  }
}
}  // namespace

int launch_conv1d_fp32(const ConvParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.Cin <= 0 || p.Cout <= 0 || p.T <= 0 || p.k <= 0 || p.d <= 0)
    return fail(AB_ERR_ARG, "conv1d: bad shape B=%d Cin=%d Cout=%d T=%d k=%d d=%d", p.B, p.Cin,
                p.Cout, p.T, p.k, p.d);
  if (((p.k - 1) * p.d) & 1)
    return fail(AB_ERR_UNSUPPORTED, "conv1d: (k-1)*dilation must be even for 'same' padding (k=%d d=%d)",
                p.k, p.d);
  if (p.B > 65535) return fail(AB_ERR_UNSUPPORTED, "conv1d: batch %d > 65535", p.B);
  const int halo = (p.k - 1) * p.d;
  if (p.reflect && halo / 2 >= p.T)
    return fail(AB_ERR_ARG, "conv1d: reflection padding %d needs more than %d samples", halo / 2, p.T);
  if (p.epi != CONV_EPI_NONE) {
    if (p.reflect || (p.epi == CONV_EPI_GAMMA_RESIDUAL && (!p.residual || !p.gamma)) || p.epi > CONV_EPI_LINEAR ||
        (p.epi == CONV_EPI_LINEAR && (p.k != 1 || !p.bias)))
      return fail(AB_ERR_ARG, "conv1d: epilogue %d needs zero padding (residual + gamma for the layer scale; k = 1 and "
                              "a bias for the Linear)", p.epi);
  } else if (p.Cout == 1 && p.k == 7 && p.d == 1 && !p.residual && !p.acc_prev && p.out_div == 1.0f) {
    dim3 grid((unsigned)ceil_div(p.T, PT), 1, (unsigned)p.B);
    const bool vec = p.xst == 1 && (p.T & 3) == 0 && (p.xsc & 3) == 0 && (p.xsb & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.y) & 15) == 0;
    if (p.reflect) {
      if (vec) conv_post_vec_kernel<7, 1><<<grid, NT, 0, s>>>(p);
      else conv_post_fp32_kernel<7, 1><<<grid, NT, 0, s>>>(p);
    } else {
      if (vec) conv_post_vec_kernel<7><<<grid, NT, 0, s>>>(p);
      else conv_post_fp32_kernel<7><<<grid, NT, 0, s>>>(p);
    }
    AB_LAUNCH_CHECK("conv_post_fp32_kernel");
    return AB_OK;
  }
  if (p.Cout <= 4 && p.epi == CONV_EPI_NONE) {
    const size_t smem = sizeof(float) * ((size_t)PCI * (PT + halo) + (size_t)p.Cin * p.k * p.Cout);
    if (smem > 200 * 1024) return fail(AB_ERR_UNSUPPORTED, "conv1d(few-out): filter too large for smem");
    static DeviceOnce configured[2];
    auto kern = p.reflect ? conv1d_fewout_fp32_kernel<1> : conv1d_fewout_fp32_kernel<0>;
    if (smem > 48 * 1024 && configured[p.reflect ? 1 : 0].need())
      AB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    dim3 grid((unsigned)ceil_div(p.T, PT), 1, (unsigned)p.B);
    kern<<<grid, NT, smem, s>>>(p);
    AB_LAUNCH_CHECK("conv1d_fewout_fp32_kernel");
    return AB_OK;
  }
  const size_t smem = sizeof(float) * ((size_t)CI_T * (TT + halo) + (size_t)CI_T * p.k * CO_T);
  if (smem > 200 * 1024)
    return fail(AB_ERR_UNSUPPORTED, "conv1d: k=%d dilation=%d needs %zu B of shared memory", p.k, p.d, smem);
  static DeviceOnce configured[5];
  auto kern = p.epi == CONV_EPI_GELU ? conv1d_fp32_kernel<0, CONV_EPI_GELU>
              : p.epi == CONV_EPI_GAMMA_RESIDUAL ? conv1d_fp32_kernel<0, CONV_EPI_GAMMA_RESIDUAL>
              : p.epi == CONV_EPI_LINEAR ? conv1d_fp32_kernel<0, CONV_EPI_LINEAR>
              : p.reflect ? conv1d_fp32_kernel<1> : conv1d_fp32_kernel<0>;
  if (smem > 48 * 1024 && configured[p.epi ? 1 + p.epi : (p.reflect ? 1 : 0)].need()) {
    AB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  if (ceil_div(p.Cout, CO_T) > 65535) return fail(AB_ERR_UNSUPPORTED, "conv1d: too many channels");
  dim3 grid((unsigned)ceil_div(p.T, TT), (unsigned)ceil_div(p.Cout, CO_T), (unsigned)p.B);
  kern<<<grid, NT, smem, s>>>(p);
  AB_LAUNCH_CHECK("conv1d_fp32_kernel");
  return AB_OK;
}

// ===========================================================================
// Strided conv1d, y[co, t] = bias[co] + sum_ci sum_j W[co, ci, j] act(x)[ci, s t + j - pad] with zero padding,
// (T + 2 pad - k) / s + 1 outputs (the downsampling conv of FACodec's EncoderBlock, facodec.py:136-154: k = 2s,
// pad = s//2 + s%2).  The conv1d_fp32_kernel tile: 64 output channels x 128 outputs per CTA, 4 x 8 per thread; the
// staged input row of a tile spans s (TT - 1) + k samples, stored by phase (sample n at [n % s][n / s], L per phase) so
// that output t's tap j = s q + r reads [r][t + q]: consecutive lanes read consecutive words, free of bank conflicts.
// ===========================================================================
namespace {
__global__ void __launch_bounds__(NT) conv1d_strided_fp32_kernel(ConvParams p, int stride, int pad, int Tout) {
  extern __shared__ float smem[];
  const int XW = stride * (TT - 1) + p.k, L = TT - 1 + (p.k + stride - 1) / stride;
  float* xs = smem;                        // [CI_T][stride][L]
  float* ws = smem + CI_T * stride * L;    // [CI_T][k][CO_T]
  const int t0 = blockIdx.x * TT, co0 = blockIdx.y * CO_T, b = blockIdx.z;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.xsb;
  const int64_t tin0 = (int64_t)t0 * stride - pad;

  float acc[4][8];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += CI_T) {
    for (int idx = threadIdx.x; idx < CI_T * XW; idx += NT) {
      const int ci = idx / XW, n = idx - ci * XW, c = ci0 + ci, q = n / stride;
      const int64_t t = tin0 + n;
      float v = 0.f;
      if (c < p.Cin && t >= 0 && t < p.T) {
        v = __ldg(xb + (int64_t)c * p.xsc + t * p.xst);
        v = v >= 0.f ? v : v * slope;
      }
      xs[(ci * stride + (n - q * stride)) * L + q] = v;
    }
    const int wn = CI_T * p.k * CO_T;
    for (int idx = threadIdx.x; idx < wn; idx += NT) {
      const int co = idx & (CO_T - 1);
      const int r = idx / CO_T;  // ci * k + j
      const int ci = r / p.k;
      float v = 0.f;
      if (ci0 + ci < p.Cin && co0 + co < p.Cout)
        v = __ldg(p.w_t + ((int64_t)ci0 * p.k + r) * p.Cout + co0 + co);
      ws[idx] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < CI_T; ++ci) {
      const float* xr = xs + ci * stride * L + tx;
      const float* wr = ws + ci * p.k * CO_T + ty * 4;
      for (int j = 0; j < p.k; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(wr + j * CO_T);
        const int q = j / stride;
        const float* xj = xr + (j - q * stride) * L + q;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xv = xj[16 * i];
          acc[0][i] = fmaf(w.x, xv, acc[0][i]);
          acc[1][i] = fmaf(w.y, xv, acc[1][i]);
          acc[2][i] = fmaf(w.z, xv, acc[2][i]);
          acc[3][i] = fmaf(w.w, xv, acc[3][i]);
        }
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int co = co0 + ty * 4 + c;
    if (co >= p.Cout) continue;
    const float bv = p.bias ? __ldg(p.bias + co) : 0.f;
    const int64_t row = ((int64_t)b * p.Cout + co) * Tout;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + tx + 16 * i;
      if (t < Tout) p.y[row + t] = acc[c][i] + bv;
    }
  }
}
}  // namespace

int launch_conv1d_strided_fp32(const ConvParams& p, int stride, int pad, cudaStream_t s) {
  if (p.B <= 0 || p.Cin <= 0 || p.Cout <= 0 || p.T <= 0 || p.k <= 0 || stride <= 0 || stride > 64 || pad < 0 || pad >= p.k)
    return fail(AB_ERR_ARG, "conv1d strided: bad shape B=%d Cin=%d Cout=%d T=%d k=%d stride=%d pad=%d", p.B, p.Cin, p.Cout,
                p.T, p.k, stride, pad);
  if (p.residual || p.acc_prev || p.out_div != 1.0f || p.post_tanh || p.reflect || p.epi != CONV_EPI_NONE || p.d != 1)
    return fail(AB_ERR_ARG, "conv1d strided: no dilation, residual, acc_prev, out_div, tanh, reflection or epilogue");
  if ((int64_t)p.T + 2 * pad < p.k) return fail(AB_ERR_ARG, "conv1d strided: %d samples are shorter than the kernel %d", p.T, p.k);
  if (p.B > 65535) return fail(AB_ERR_UNSUPPORTED, "conv1d strided: batch %d > 65535", p.B);
  const int Tout = (p.T + 2 * pad - p.k) / stride + 1;
  const size_t smem = sizeof(float) * ((size_t)CI_T * stride * (TT - 1 + (p.k + stride - 1) / stride) +
                                      (size_t)CI_T * p.k * CO_T);
  if (smem > 200 * 1024) return fail(AB_ERR_UNSUPPORTED, "conv1d strided: k=%d stride=%d needs %zu B of shared memory", p.k, stride, smem);
  static DeviceOnce configured;
  if (smem > 48 * 1024 && configured.need())
    AB_CUDA_TRY(cudaFuncSetAttribute(conv1d_strided_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  if (ceil_div(p.Cout, CO_T) > 65535) return fail(AB_ERR_UNSUPPORTED, "conv1d strided: too many channels");
  dim3 grid((unsigned)ceil_div(Tout, TT), (unsigned)ceil_div(p.Cout, CO_T), (unsigned)p.B);
  conv1d_strided_fp32_kernel<<<grid, NT, smem, s>>>(p, stride, pad, Tout);
  AB_LAUNCH_CHECK("conv1d_strided_fp32_kernel");
  return AB_OK;
}

// ===========================================================================
// ConvTranspose1d(stride=u, padding=p) fused with the leaky_relu in front of it (hifigan.py:206-207, p = (k-u)/2;
// bigvgan.py:316-318 has no activation; melgan.py:73-80, p = u//2 + u%2 with output_padding u%2), Tin*u outputs:
//   y[co,t] = b[co] + sum_ci sum_{j = (t+p) mod u, +u, ... < k} x[ci,(t+p-j)/u] * W[ci,co,j]
// ===========================================================================
namespace {
__global__ void __launch_bounds__(NT) convT_fp32_kernel(ConvTParams p, int XW, int M) {
  extern __shared__ float smem[];
  float* xs = smem;               // [CI_T][XW]
  float* ws = smem + CI_T * XW;   // [CI_T][k][CO_T]
  const int Tout = p.Tin * p.u;
  const int t0 = blockIdx.x * TT, co0 = blockIdx.y * CO_T, b = blockIdx.z;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int pd = p.pad;
  const int s_min = (t0 + pd) / p.u - (M - 1);
  const float slope = p.pre_slope;
  const float* xb = p.x + (int64_t)b * p.Cin * p.Tin;

  int phi[8], sl[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int q = t0 + tx + 16 * i + pd;
    phi[i] = q % p.u;
    sl[i] = q / p.u - s_min;
  }
  float acc[4][8];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[c][i] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += CI_T) {
    for (int idx = threadIdx.x; idx < CI_T * XW; idx += NT) {
      const int ci = idx / XW, n = idx - ci * XW;
      const int sidx = s_min + n, c = ci0 + ci;
      float v = 0.f;
      if (c < p.Cin && sidx >= 0 && sidx < p.Tin) {
        v = __ldg(xb + (int64_t)c * p.Tin + sidx);
        v = v >= 0.f ? v : v * slope;
      }
      xs[idx] = v;
    }
    const int wn = CI_T * p.k * CO_T;
    for (int idx = threadIdx.x; idx < wn; idx += NT) {
      const int co = idx & (CO_T - 1);
      const int r = idx / CO_T;
      const int ci = r / p.k;
      float v = 0.f;
      if (ci0 + ci < p.Cin && co0 + co < p.Cout)
        v = __ldg(p.w_t + ((int64_t)ci0 * p.k + r) * p.Cout + co0 + co);
      ws[idx] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < CI_T; ++ci) {
      const float* xr = xs + ci * XW;
      const float* wr = ws + ci * p.k * CO_T + ty * 4;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        for (int m = 0; m < M; ++m) {
          const int j = phi[i] + m * p.u;
          if (j < p.k) {
            const float4 w = *reinterpret_cast<const float4*>(wr + j * CO_T);
            const float xv = xr[sl[i] - m];
            acc[0][i] = fmaf(w.x, xv, acc[0][i]);
            acc[1][i] = fmaf(w.y, xv, acc[1][i]);
            acc[2][i] = fmaf(w.z, xv, acc[2][i]);
            acc[3][i] = fmaf(w.w, xv, acc[3][i]);
          }
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int co = co0 + ty * 4 + c;
    if (co >= p.Cout) continue;
    const float bv = p.bias ? __ldg(p.bias + co) : 0.f;
    const int64_t row = ((int64_t)b * p.Cout + co) * Tout;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + tx + 16 * i;
      if (t < Tout) p.y[row + t] = acc[c][i] + bv;
    }
  }
}
}  // namespace

int launch_conv_transpose1d_fp32(const ConvTParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.Cin <= 0 || p.Cout <= 0 || p.Tin <= 0 || p.k <= 0 || p.u <= 0)
    return fail(AB_ERR_ARG, "conv_transpose1d: bad shape");
  if (p.k < p.u || p.pad < 0 || p.pad > p.k)
    return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: kernel %d / stride %d / padding %d: need k >= stride, 0 <= padding <= k",
                p.k, p.u, p.pad);
  if (p.B > 65535) return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: batch %d > 65535", p.B);
  const int M = (p.k + p.u - 1) / p.u;
  const int XW = TT / p.u + 2 + M;
  const size_t smem = sizeof(float) * ((size_t)CI_T * XW + (size_t)CI_T * p.k * CO_T);
  if (smem > 200 * 1024) return fail(AB_ERR_UNSUPPORTED, "conv_transpose1d: kernel %d too large", p.k);
  static DeviceOnce configured;
  if (smem > 48 * 1024 && configured.need()) {
    AB_CUDA_TRY(cudaFuncSetAttribute(convT_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     200 * 1024));
  }
  const int64_t Tout = (int64_t)p.Tin * p.u;
  dim3 grid((unsigned)ceil_div(Tout, TT), (unsigned)ceil_div(p.Cout, CO_T), (unsigned)p.B);
  convT_fp32_kernel<<<grid, NT, smem, s>>>(p, XW, M);
  AB_LAUNCH_CHECK("convT_fp32_kernel");
  return AB_OK;
}

// ===========================================================================
// Activation1d(Snake|SnakeBeta): up-FIR x2 -> snake -> down-FIR /2, replicate
// edges, never materialising the 2x-rate tensor in HBM.
//   up   (resample.py:36-45):  u[2q]   = 2 sum_m f[11-2m] xh[q-3+m]
//                              u[2q+1] = 2 sum_m f[10-2m] xh[q-2+m],  xh = replicate(x)
//   act  (snake.py:51-61,110-122): v = u + 1/(b+1e-9) * sin(u*a)^2
//   down (filter.py:92-99):    y[t] = sum_j f[j] v[clamp(2t+j-5, 0, 2T-1)]
// One CTA = (batch, group of 8 channels, 960-sample tile); every warp owns 120 consecutive outputs for all
// 8 channels and works on private shared-memory windows, so there are no block-level barriers in the loop.
// The kernel is instruction-issue bound (ncu: ~80 % of issue slots), so the design minimises instructions per
// sample: 16-byte window fetches, taps pre-scaled by the x2 gain (exact: power of two), per-channel
// exp / reciprocal computed once per CTA, and a lane-private transposition buffer for the operand image.
// ===========================================================================
namespace {
#ifndef AB_SNAKE_BLOCKS
#define AB_SNAKE_BLOCKS 4      // CTAs per SM the activation kernel is compiled for (64 registers: measured best of 2..5)
#endif
constexpr int SN_WS = 120;                 // outputs per warp segment (30 lanes x 4)
constexpr int SN_XS = 136;                 // xs[m] = xh[t0 - 8 + m]            (34 float4)
#ifndef AB_SNAKE_AHEAD
#define AB_SNAKE_AHEAD 2       // channels whose windows are in flight ahead of the one being computed
#endif
constexpr int SN_AHEAD = AB_SNAKE_AHEAD;
constexpr int SN_XR = SN_AHEAD + 1;        // x windows per warp (cp.async ring)
constexpr int SN_VS = 256;                 // vs[n] = vh[2*t0 - 7 + n]          (64 groups of 4 = 2 full rounds)
constexpr int SN_TR = 8 * 32 * 2;          // image transposition: [8 ch][32 lanes] x 8 B, lane-private
constexpr int WT = 8 * SN_WS;              // outputs per CTA tile (8 warps)

__device__ __forceinline__ float snake_eval(float u, float a, float invb) {
  // sin(u*a)^2 with explicit range reduction to [-pi, pi] before the MUFU (Cody-Waite: 2 pi as a high and a low part);
  // every rounding is an explicit intrinsic, restated step by step in tests/activation1d_exact_oracle.py
  const float arg = __fmul_rn(u, a);
  const float kf = rintf(__fmul_rn(arg, 0.15915494309189535f));
  float r = __fmaf_rn(-kf, 6.2831854820251465f, arg);
  r = __fmaf_rn(-kf, -1.7484555314695172e-07f, r);
  const float sv = __sinf(r);
  return __fmaf_rn(invb, __fmul_rn(sv, sv), u);
}

// Two snake evaluations at once, without explicit range reduction: sin.approx multiplies by 1/2pi and the MUFU
// reduces in turns, so the phase error is ~1.2e-7 * |u a| rad.  Used on the 16-bit operand path only (the operand
// rounding is 5e-4 relative); the fp32 outputs keep the Cody-Waite reduction of snake_eval.
__device__ __forceinline__ f32x2 snake_eval2_fast(f32x2 u, f32x2 a2, f32x2 invb2) {
  float r0, r1;
  upk2(mul2(u, a2), r0, r1);
  const f32x2 sv = pk2(__sinf(r0), __sinf(r1));
  return fma2(mul2(sv, sv), invb2, u);
}

template <int BF16>
__device__ __forceinline__ uint32_t cvt_pair(float lo, float hi) {
  uint32_t r;
  if (BF16) asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// All 8 channels of one warp segment.  FAST: the whole window [t0-8, t0+128) lies inside the row and rows are
// 16-byte aligned, so the fetch is one float4 per lane and no index is clamped; otherwise (sequence edges,
// odd T) every index is replicate-clamped exactly as the reference's padding does.
// MODE 0: taps from global memory, outputs chosen at run time (the standalone operator).
// MODE 1: taps pre-packed in the kernel parameters (uniform registers), outputs chosen at run time.
// MODE 2: as 1, operand image only and the short snake (tensor-core generators).
template <bool FAST, int BF16, int MODE>
__device__ __forceinline__ void snake_segment(const SnakeParams& p, const float* __restrict__ xb, int c8, int b, int t0,
                                              const float (*prm)[2], float* xs, float* vs, uint2* tr, int lane) {
  constexpr bool KP = MODE != 0;
  const int T = p.T, C = p.C;
  const bool want_y = MODE != 2 && p.y != nullptr;
  const bool want_img = MODE == 2 || p.yimg != nullptr;
  float fu2[12], fd[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) {            // scalar taps: the sequence-edge path (and the pairs below when !KP)
    fu2[j] = KP ? ((10 - j) % 4 == 0 ? p.kc.ce_a[(10 - j) / 4].x : (10 - j) % 4 == 2 ? p.kc.ce_a[(8 - j) / 4].y
                   : (11 - j) % 4 == 0 ? p.kc.co_a[(11 - j) / 4].x : p.kc.co_a[(9 - j) / 4].y)
                : 2.0f * __ldg(p.f_up + j);
    fd[j] = KP ? (j % 2 == 0 ? p.kc.fd2[j / 2].x : p.kc.fd2[j / 2].y) : __ldg(p.f_down + j);
  }
  // coefficient pairs: even-phase taps ce[m] = fu2[10-2m], odd-phase co[m] = fu2[11-2m].  Outputs at input position
  // q use xs pairs (w[2p], w[2p+1]) with (c[2p], c[2p+1]); those at q+1 use the same pairs with (c[2p-1], c[2p]).
  f32x2 ce_a[3], co_a[3], ce_b[4], co_b[4], fd2[6];
  if (KP) {                                  // pre-packed on the host: constant-bank / uniform-register operands
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      ce_a[q] = *reinterpret_cast<const f32x2*>(&p.kc.ce_a[q]);
      co_a[q] = *reinterpret_cast<const f32x2*>(&p.kc.co_a[q]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      ce_b[q] = *reinterpret_cast<const f32x2*>(&p.kc.ce_b[q]);
      co_b[q] = *reinterpret_cast<const f32x2*>(&p.kc.co_b[q]);
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) fd2[q] = *reinterpret_cast<const f32x2*>(&p.kc.fd2[q]);
  } else {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      ce_a[q] = pk2(fu2[10 - 4 * q], fu2[8 - 4 * q]);
      co_a[q] = pk2(fu2[11 - 4 * q], fu2[9 - 4 * q]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      ce_b[q] = pk2(q > 0 ? fu2[12 - 4 * q] : 0.f, q < 3 ? fu2[10 - 4 * q] : 0.f);
      co_b[q] = pk2(q > 0 ? fu2[13 - 4 * q] : 0.f, q < 3 ? fu2[11 - 4 * q] : 0.f);
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) fd2[q] = pk2(fd[2 * q], fd[2 * q + 1]);
  }
  const int i0 = 2 * t0 - 7, imax = 2 * T - 1;
  const int tl = 4 * lane;
  float ne[5] = {0.f, 0.f, 0.f, 0.f, 0.f};                     // edge path: prefetch registers
  // FAST: 16-byte cp.async straight into a ring of SN_XR windows, issued SN_AHEAD channels ahead (DRAM latency under
  // load exceeds one channel's compute); one commit group per channel, empty groups keep the count uniform.
  // Source pointer and ring offsets advance by increments (no per-channel multiplies or modulo).
  const int c_first = c8 * 8;
  const float* src = xb + (int64_t)c_first * T + (t0 - 8) + 4 * lane;      // FAST: this lane's 16 bytes of channel c
  const uint32_t ring0 = (uint32_t)__cvta_generic_to_shared(xs) + 16u * lane;
  constexpr uint32_t SLOT_B = SN_XS * 4;
  auto fetch_fast = [&](const float* sp, uint32_t slot_off) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ring0 + slot_off), "l"(sp) : "memory");
    if (lane < 2)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ring0 + slot_off + 512u), "l"(sp + 128) : "memory");
  };
  auto fetch_edge = [&](int c) {
    const float* xr = xb + (int64_t)c * T;
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const int m = lane + 32 * q;
      const int t = min(max(t0 - 8 + m, 0), T - 1);
      ne[q] = (m < SN_XS) ? __ldg(xr + t) : 0.f;
    }
  };
  if (FAST) {
#pragma unroll
    for (int pre = 0; pre < SN_AHEAD; ++pre) {
      if (c_first + pre < C) fetch_fast(src + (int64_t)pre * T, pre * SLOT_B);
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  } else if (c_first < C) {
    fetch_edge(c_first);
  }
  const float* src_nxt = src + SN_AHEAD * (int64_t)T;          // channel c + SN_AHEAD
  uint32_t slot_cur = 0, slot_nxt = SN_AHEAD * SLOT_B;         // byte offsets of the windows of channels c and c + SN_AHEAD
  float* yr = want_y ? p.y + ((int64_t)b * C + c_first) * T + t0 + tl : nullptr;
  float* const xs_ring = xs;
  // The 2x-rate window vs is stored by 16-byte units u = n / 4 at position u ^ ((u >> 3) & 1): phase 2 reads units
  // 2 lane + q, a 32-byte lane stride that would otherwise put lanes l and l + 4 of a quarter warp on the same banks.
  // Units 2m and 2m + 1 share their group of 8, so a pair keeps its 32 bytes and only swaps halves when the bit is set.
  const int sw_l = (lane >> 2) & 1;
  float* const vs_wA = vs + 8 * lane + 4 * sw_l;           // group 2 lane
  float* const vs_wB = vs + 8 * lane + 4 * (1 - sw_l);     // group 2 lane + 1
  const float* vs_r[3][2];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int m = lane + q, sm = (m >> 2) & 1;
    vs_r[q][0] = vs + 8 * m + 4 * sm;
    vs_r[q][1] = vs + 8 * m + 4 * (1 - sm);
  }
#pragma unroll 1
  for (int cg = 0; cg < 8; ++cg) {
    const int c = c_first + cg;
    if (c >= C) {
      if (want_img) tr[cg * 32 + lane] = make_uint2(0u, 0u);   // padding channels of the image
      continue;
    }
    const float a = prm[cg][0], invb = prm[cg][1];
    if (FAST) {
      asm volatile("cp.async.wait_group %0;" ::"n"(SN_AHEAD - 1) : "memory");   // this channel's window has landed
      __syncwarp();                                          // ... for every lane; also: phase 2 of cg-1 is done with vs
      xs = reinterpret_cast<float*>(reinterpret_cast<char*>(xs_ring) + slot_cur);
      // the slot of channel c + SN_AHEAD was read in iteration cg - 1, which every lane has left
      if (c + SN_AHEAD < C && cg + SN_AHEAD < 8) fetch_fast(src_nxt, slot_nxt);
      asm volatile("cp.async.commit_group;" ::: "memory");
      src_nxt += T;
      slot_cur = slot_cur == SN_AHEAD * SLOT_B ? 0u : slot_cur + SLOT_B;
      slot_nxt = slot_nxt == SN_AHEAD * SLOT_B ? 0u : slot_nxt + SLOT_B;
    } else {
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const int m = lane + 32 * q;
        if (m < SN_XS) xs[m] = ne[q];
      }
      __syncwarp();
      if (c + 1 < C && cg + 1 < 8) fetch_edge(c + 1);
    }
    const f32x2 a2 = pk2(a, a), invb2 = pk2(invb, invb);
    // phase 1: 256 samples of the 2x-rate signal = 64 groups of 4; lane l computes the adjacent groups 2l and 2l+1.
    // Group j holds v[i0 + 4j .. +3] = (u[2q+1], u[2q+2], u[2q+3], u[2q+4]), q = t0 - 4 + 2j, from
    // xh[q-2 .. q+4] = xs[2j+2 .. 2j+8]: both groups read xs[4l+2 .. 4l+11] (one 8-byte and two 16-byte loads).
    {
      f32x2 wp[5];
      wp[0] = *reinterpret_cast<const f32x2*>(xs + 4 * lane + 2);
      {
        const ulonglong2 t4 = *reinterpret_cast<const ulonglong2*>(xs + 4 * lane + 4);
        wp[1] = t4.x; wp[2] = t4.y;
        const ulonglong2 t5 = *reinterpret_cast<const ulonglong2*>(xs + 4 * lane + 8);
        wp[3] = t5.x; wp[4] = t5.y;
      }
#pragma unroll
      for (int gq = 0; gq < 2; ++gq) {
        const int j = 2 * lane + gq;
        const int n0 = 4 * j;
        float v0, v1, v2, v3;
        if (FAST || (i0 + n0 >= 0 && i0 + n0 + 3 <= imax)) {
          const f32x2* w2 = wp + gq;
          f32x2 s0 = mul2(ce_a[0], w2[0]), s1 = mul2(co_a[0], w2[0]);
          f32x2 s2 = mul2(ce_b[0], w2[0]), s3 = mul2(co_b[0], w2[0]);
#pragma unroll
          for (int q = 1; q < 3; ++q) {
            s0 = fma2(ce_a[q], w2[q], s0);
            s1 = fma2(co_a[q], w2[q], s1);
          }
#pragma unroll
          for (int q = 1; q < 4; ++q) {
            s2 = fma2(ce_b[q], w2[q], s2);
            s3 = fma2(co_b[q], w2[q], s3);
          }
          const float u0 = hsum2(s0), u1 = hsum2(s1), u2 = hsum2(s2), u3 = hsum2(s3);
          if (MODE == 2) {
            upk2(snake_eval2_fast(pk2(u0, u1), a2, invb2), v0, v1);
            upk2(snake_eval2_fast(pk2(u2, u3), a2, invb2), v2, v3);
          } else {
            v0 = snake_eval(u0, a, invb);
            v1 = snake_eval(u1, a, invb);
            v2 = snake_eval(u2, a, invb);
            v3 = snake_eval(u3, a, invb);
          }
        } else {
          float vv[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {      // sequence edges: replicate-clamped 2x-rate index, generic taps
            const int ic = min(max(i0 + n0 + k, 0), imax);
            const int q = ic >> 1, odd = ic & 1;
            const int xi = min(max(q - 3 + odd - (t0 - 8), 0), SN_XS - 6);
            const float* xp = xs + xi;
            float u = 0.f;
#pragma unroll
            for (int m = 0; m < 6; ++m) u = fmaf(odd ? fu2[10 - 2 * m] : fu2[11 - 2 * m], xp[m], u);
            vv[k] = snake_eval(u, a, invb);
          }
          v0 = vv[0]; v1 = vv[1]; v2 = vv[2]; v3 = vv[3];
        }
        *reinterpret_cast<float4*>(gq ? vs_wB : vs_wA) = make_float4(v0, v1, v2, v3);
      }
    }
    __syncwarp();
    // phase 2: y[t0 + tl + k] = sum_j fd[j] v[2*(tl + k) + j + 2], v = the logical (unswizzled) 2x-rate window
    if (lane < SN_WS / 4) {
      // v[2 tl .. 2 tl + 23] as twelve aligned pairs (three 32-byte unit pairs); y[k] = sum_q fd2[q] . pair[k + 1 + q]
      f32x2 w2[12];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const ulonglong2 ta = *reinterpret_cast<const ulonglong2*>(vs_r[q][0]);
        const ulonglong2 tb = *reinterpret_cast<const ulonglong2*>(vs_r[q][1]);
        w2[4 * q] = ta.x; w2[4 * q + 1] = ta.y;
        w2[4 * q + 2] = tb.x; w2[4 * q + 3] = tb.y;
      }
      float y[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        f32x2 acc = mul2(fd2[0], w2[k + 1]);
#pragma unroll
        for (int q = 1; q < 6; ++q) acc = fma2(fd2[q], w2[k + 1 + q], acc);
        y[k] = hsum2(acc);
      }
      if (want_y) {
        if (FAST || (t0 + tl + 3 < T && (T & 3) == 0)) {
          *reinterpret_cast<float4*>(yr) = make_float4(y[0], y[1], y[2], y[3]);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (t0 + tl + k < T) yr[k] = y[k];
        }
      }
      if (want_img) tr[cg * 32 + lane] = make_uint2(cvt_pair<BF16>(y[0], y[1]), cvt_pair<BF16>(y[2], y[3]));
    }
    if (want_y) yr += T;
  }
  // operand image: 8 channels = 16 B per time step; every lane re-reads its own 4 rows x 8 channels
  if (want_img && lane < SN_WS / 4) {
    uint2 h[8];
#pragma unroll
    for (int cg = 0; cg < 8; ++cg) h[cg] = tr[cg * 32 + lane];
    uint16_t* yi = p.yimg + (((size_t)b * gridDim.y + c8) * (size_t)T + t0 + tl) * 8;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint4 q;
      const uint32_t sel = (k & 1) ? 0x7632u : 0x5410u;
      if (k < 2) {
        q.x = __byte_perm(h[0].x, h[1].x, sel); q.y = __byte_perm(h[2].x, h[3].x, sel);
        q.z = __byte_perm(h[4].x, h[5].x, sel); q.w = __byte_perm(h[6].x, h[7].x, sel);
      } else {
        q.x = __byte_perm(h[0].y, h[1].y, sel); q.y = __byte_perm(h[2].y, h[3].y, sel);
        q.z = __byte_perm(h[4].y, h[5].y, sel); q.w = __byte_perm(h[6].y, h[7].y, sel);
      }
      if (FAST || t0 + tl + k < T) *reinterpret_cast<uint4*>(yi + (size_t)k * 8) = q;
    }
  }
}

template <int BF16, int MODE>
__global__ void __launch_bounds__(NT, AB_SNAKE_BLOCKS) activation1d_warp_kernel(const __grid_constant__ SnakeParams p) {
  __shared__ __align__(16) float win_all[8][SN_XR * SN_XS + SN_VS + SN_TR];
  __shared__ float prm[8][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t0 = blockIdx.x * WT + warp * SN_WS, c8 = blockIdx.y, b = blockIdx.z;
  const int T = p.T;
  if (threadIdx.x < 8) {
    const int c = c8 * 8 + threadIdx.x;
    float a = 0.f, bb = 1.f;
    if (c < p.C) {
      a = __ldg(p.alpha + c);
      bb = __ldg(p.beta + c);
      if (p.logscale) {
        a = expf(a);
        bb = expf(bb);
      }
    }
    prm[threadIdx.x][0] = a;
    prm[threadIdx.x][1] = __frcp_rn(__fadd_rn(bb, 1e-9f));
  }
  __syncthreads();
  if (t0 >= T) return;                           // warp-uniform; no block barriers below
  float* xs = win_all[warp];
  float* vs = xs + SN_XR * SN_XS;
  uint2* tr = reinterpret_cast<uint2*>(vs + SN_VS);
  const float* xb = p.x + (int64_t)b * p.C * T;
  const bool fast = t0 >= 8 && t0 + 128 <= T && (T & 3) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 &&
                    (p.y == nullptr || (reinterpret_cast<uintptr_t>(p.y) & 15) == 0);
  if (fast) snake_segment<true, BF16, MODE>(p, xb, c8, b, t0, prm, xs, vs, tr, lane);
  else snake_segment<false, BF16, MODE>(p, xb, c8, b, t0, prm, xs, vs, tr, lane);
}
}  // namespace

void pack_snake_coef(const float* f_up, const float* f_down, SnakeCoef* out) {
  float fu2[12];
  for (int j = 0; j < 12; ++j) fu2[j] = 2.0f * f_up[j];       // the x2 gain of UpSample1d (resample.py:43), exact
  for (int q = 0; q < 3; ++q) {
    out->ce_a[q] = make_float2(fu2[10 - 4 * q], fu2[8 - 4 * q]);
    out->co_a[q] = make_float2(fu2[11 - 4 * q], fu2[9 - 4 * q]);
  }
  for (int q = 0; q < 4; ++q) {
    out->ce_b[q] = make_float2(q > 0 ? fu2[12 - 4 * q] : 0.f, q < 3 ? fu2[10 - 4 * q] : 0.f);
    out->co_b[q] = make_float2(q > 0 ? fu2[13 - 4 * q] : 0.f, q < 3 ? fu2[11 - 4 * q] : 0.f);
  }
  for (int q = 0; q < 6; ++q) out->fd2[q] = make_float2(f_down[2 * q], f_down[2 * q + 1]);
}

int launch_activation1d(const SnakeParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.C <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "activation1d: bad shape");
  if (p.C > 65535 * 8 || p.B > 65535) return fail(AB_ERR_UNSUPPORTED, "activation1d: B or C too large");
  if (p.y == nullptr && p.yimg == nullptr) return fail(AB_ERR_ARG, "activation1d: no output requested");
  // channel groups: the operand image covers ceil16(C) channels (padding groups are written as zeros)
  const int c8n = p.yimg ? (int)(ceil_div(p.C, 16) * 2) : (int)ceil_div(p.C, 8);
  dim3 grid((unsigned)ceil_div(p.T, WT), (unsigned)c8n, (unsigned)p.B);
  const int mode = !p.have_kc ? 0 : (p.fast_snake && p.y == nullptr && p.yimg != nullptr) ? 2 : 1;
  if (mode == 2) {
    if (p.bf16) activation1d_warp_kernel<1, 2><<<grid, NT, 0, s>>>(p);
    else activation1d_warp_kernel<0, 2><<<grid, NT, 0, s>>>(p);
  } else if (mode == 1) {
    if (p.bf16) activation1d_warp_kernel<1, 1><<<grid, NT, 0, s>>>(p);
    else activation1d_warp_kernel<0, 1><<<grid, NT, 0, s>>>(p);
  } else {
    if (p.bf16) activation1d_warp_kernel<1, 0><<<grid, NT, 0, s>>>(p);
    else activation1d_warp_kernel<0, 0><<<grid, NT, 0, s>>>(p);
  }
  AB_LAUNCH_CHECK("activation1d_warp_kernel");
  return AB_OK;
}

// ===========================================================================
// Weight repack (+ weight-norm fold, old-style torch.nn.utils.weight_norm with
// dim=0: w = g * v / ||v||_{dims != 0}; hifigan.py:157-199, SURVEY Q6):
// src row r = dim 0.  Conv1d: src [Cout][Cin][k]; ConvTranspose1d: [Cin][Cout][k].
// dst is always [Cin][k][Cout] so the conv kernels read it coalesced.
// ===========================================================================
namespace {
__global__ void __launch_bounds__(256) repack_weight_kernel(const float* __restrict__ v,
                                                            const float* __restrict__ g,
                                                            float* __restrict__ dst, int d0, int d1,
                                                            int k, int transposed) {
  __shared__ float red[8];
  __shared__ float scale_s;
  const int r = blockIdx.x;
  const int n = d1 * k;
  const float* row = v + (int64_t)r * n;
  float scale = 1.0f;
  if (g != nullptr) {
    float ss = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) {
      const float x = row[i];
      ss = fmaf(x, x, ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < 8; ++w) tot += red[w];
      scale_s = g[r] / sqrtf(tot);
    }
    __syncthreads();
    scale = scale_s;
  }
  const int Cout = transposed ? d1 : d0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const int inner = i / k, j = i - inner * k;
    const int ci = transposed ? r : inner;
    const int co = transposed ? inner : r;
    dst[((int64_t)ci * k + j) * Cout + co] = row[i] * scale;
  }
}
}  // namespace

int launch_repack_weight(const float* v, const float* g, float* dst, int d0, int d1, int k,
                         int transposed, cudaStream_t s) {
  if (d0 <= 0 || d1 <= 0 || k <= 0) return fail(AB_ERR_ARG, "repack_weight: bad shape");
  repack_weight_kernel<<<d0, 256, 0, s>>>(v, g, dst, d0, d1, k, transposed);
  AB_LAUNCH_CHECK("repack_weight_kernel");
  return AB_OK;
}

namespace {
__global__ void scale_inplace_kernel(float* p, size_t n, float gain) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] *= gain;
}
}  // namespace

namespace {
// one CTA per (channel, batch): warp-reduced dot product, then the row update
__global__ void __launch_bounds__(128) cond_add_kernel(float* __restrict__ x, const float* __restrict__ g, int64_t gsb,
                                                       const float* __restrict__ w, const float* __restrict__ bias,
                                                       int C, int gin, int T) {
  const int c = blockIdx.x, b = blockIdx.y;
  const float* gr = g + (int64_t)b * gsb;
  const float* wr = w + (int64_t)c * gin;
  float acc = 0.f;
  for (int i = threadIdx.x; i < gin; i += 128) acc = fmaf(__ldg(wr + i), __ldg(gr + i), acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float part[4];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  const float v = ((part[0] + part[1]) + (part[2] + part[3])) + (bias ? __ldg(bias + c) : 0.f);
  float* xr = x + ((int64_t)b * C + c) * T;
  for (int t = threadIdx.x; t < T; t += 128) xr[t] += v;
}
}  // namespace

int launch_cond_add(float* x, const float* g, int64_t g_batch_stride, const float* w, const float* bias, int B, int C,
                    int gin, int T, cudaStream_t s) {
  if (B <= 0 || C <= 0 || gin <= 0 || T <= 0 || B > 65535) return fail(AB_ERR_ARG, "cond_add: bad shape");
  cond_add_kernel<<<dim3((unsigned)C, (unsigned)B), 128, 0, s>>>(x, g, g_batch_stride, w, bias, C, gin, T);
  AB_LAUNCH_CHECK("cond_add_kernel");
  return AB_OK;
}

// ===========================================================================
// Vocos LayerNorm, optionally after the depthwise conv (vocos.py:493-527, :758-783).  One CTA per (utterance, tile of
// TT time steps): the values of all C channels of the tile go to shared memory [C][TT] once, then the mean, the
// biased variance (a second pass over the centred values, as torch.layer_norm) and the affine output per time step.
// DW: the k = 7 zero-padded depthwise conv with bias first.  OUT: 0 fp32 [B, C, T]; 1 / 2 the fp16 / bf16 operand image.
// The divisions, the square root and the output (v - mean) * rstd * w + b (a multiply, then an FMA) are explicit
// __f*_rn intrinsics, so that no build can contract or reorder them differently: tests/vocos_exact_oracle.py restates
// every rounding step.
// ===========================================================================
namespace {
constexpr int LN_THREADS = 256;

template <int DW, int OUT>
__global__ void __launch_bounds__(LN_THREADS) vocos_norm_kernel(NormParams p, int TT, int tiles) {
  extern __shared__ float lsm[];   // [C][TT] values, [LN_THREADS] partial sums, [TT] mean, [TT] 1/std
  float* part = lsm + (size_t)p.C * TT;
  float* mean_s = part + LN_THREADS;
  float* rstd_s = mean_s + TT;
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * TT;
  const int tid = threadIdx.x, tt = tid % TT, grp = tid / TT, ngrp = LN_THREADS / TT;
  const float* xb = p.x + (int64_t)b * p.C * p.T;
  const int n = p.C * TT;
  for (int i = tid; i < n; i += LN_THREADS) {
    const int c = i / TT, t = t0 + (i - c * TT);
    float v = 0.f;
    if (t < p.T) {
      const float* xr = xb + (int64_t)c * p.T;
      if (DW) {
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < 7; ++j) {
          const int s = t + j - 3;
          if (s >= 0 && s < p.T) a = fmaf(__ldg(p.dw_w + c * 7 + j), __ldg(xr + s), a);
        }
        v = a + __ldg(p.dw_b + c);
      } else {
        v = __ldg(xr + t);
      }
    }
    lsm[i] = v;
  }
  __syncthreads();
  float a = 0.f;
  for (int c = grp; c < p.C; c += ngrp) a += lsm[c * TT + tt];
  part[tid] = a;
  __syncthreads();
  if (tid < TT) {
    float s = 0.f;
    for (int q = 0; q < ngrp; ++q) s += part[q * TT + tid];
    mean_s[tid] = __fdiv_rn(s, (float)p.C);
  }
  __syncthreads();
  const float mu = mean_s[tt];
  a = 0.f;
  for (int c = grp; c < p.C; c += ngrp) {
    const float d = __fsub_rn(lsm[c * TT + tt], mu);
    a = fmaf(d, d, a);
  }
  part[tid] = a;
  __syncthreads();
  if (tid < TT) {
    float s = 0.f;
    for (int q = 0; q < ngrp; ++q) s += part[q * TT + tid];
    rstd_s[tid] = __frcp_rn(__fsqrt_rn(__fadd_rn(__fdiv_rn(s, (float)p.C), p.eps)));
  }
  __syncthreads();
  auto norm = [&](int c, int u) {
    return __fmaf_rn(__fmul_rn(__fsub_rn(lsm[c * TT + u], mean_s[u]), rstd_s[u]), __ldg(p.ln_w + c), __ldg(p.ln_b + c));
  };
  if (OUT == 0) {
    for (int i = tid; i < n; i += LN_THREADS) {
      const int c = i / TT, u = i - c * TT, t = t0 + u;
      if (t < p.T) p.y[((int64_t)b * p.C + c) * p.T + t] = norm(c, u);
    }
  } else {
    const int c8n = (p.C + 15) / 16 * 2;
    for (int i = tid; i < c8n * TT; i += LN_THREADS) {
      const int c8 = i / TT, u = i - c8 * TT, t = t0 + u;
      if (t >= p.T) continue;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = c8 * 8 + e < p.C ? norm(c8 * 8 + e, u) : 0.f;
      *reinterpret_cast<uint4*>(p.yimg + (((size_t)b * c8n + c8) * p.T + t) * 8) =
          make_uint4(cvt_pair<OUT - 1>(v[0], v[1]), cvt_pair<OUT - 1>(v[2], v[3]), cvt_pair<OUT - 1>(v[4], v[5]),
                     cvt_pair<OUT - 1>(v[6], v[7]));
    }
  }
}
}  // namespace

int launch_vocos_norm(const NormParams& p, cudaStream_t s) {
  if (!p.x || !p.ln_w || !p.ln_b || (!p.y) == (!p.yimg) || (!p.dw_w) != (!p.dw_b))
    return fail(AB_ERR_ARG, "vocos norm: null argument");
  if (p.B <= 0 || p.C <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "vocos norm: bad shape");
  // time tile: up to 16 steps, fewer for wide C so that a few CTAs share an SM
  int TT = 16;
  auto smem_of = [&](int tt) { return sizeof(float) * ((size_t)p.C * tt + LN_THREADS + 2 * tt); };
  while (TT > 1 && smem_of(TT) > 64 * 1024) TT >>= 1;
  const size_t smem = smem_of(TT);
  if (smem > 200 * 1024) return fail(AB_ERR_UNSUPPORTED, "vocos norm: %d channels do not fit shared memory", p.C);
  const int64_t tiles = ceil_div(p.T, TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "vocos norm: grid too large");
  const int out = p.y ? 0 : (p.bf16 ? 2 : 1);
  void (*kerns[2][3])(NormParams, int, int) = {{vocos_norm_kernel<0, 0>, vocos_norm_kernel<0, 1>, vocos_norm_kernel<0, 2>},
                                                {vocos_norm_kernel<1, 0>, vocos_norm_kernel<1, 1>, vocos_norm_kernel<1, 2>}};
  const int dw = p.dw_w ? 1 : 0;
  static DeviceOnce configured[2][3];
  if (smem > 48 * 1024 && configured[dw][out].need())
    AB_CUDA_TRY(cudaFuncSetAttribute(kerns[dw][out], cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  kerns[dw][out]<<<(unsigned)grid, LN_THREADS, smem, s>>>(p, TT, (int)tiles);
  AB_LAUNCH_CHECK("vocos_norm_kernel");
  return AB_OK;
}

// ===========================================================================
// Snake1d (models/codec/amphion_codec/codec.py:32-48): y = x + (alpha[c] + 1e-9)^-1 * sin(alpha[c] x)^2 with every step
// rounded as the reference's TorchScript snake rounds it: u = alpha x, s = sinf(u) (the accurate sinf torch.sin calls),
// r = 1 / (alpha + 1e-9) (correctly rounded), y = x + r (s s); nothing contracted into an FMA.  The same arithmetic at
// every precision.  One thread per (utterance, 8-channel group, time step): consecutive threads take consecutive time
// steps, so the 8 fp32 loads and stores and the 16-byte image store of a warp are each coalesced.  IMG: 0 no image,
// 1 / 2 the fp16 / bf16 operand image [B][ceil16(C)/8][T][8] (saturating round to nearest, padding channels zero).
// ===========================================================================
namespace {
template <int IMG>
__global__ void __launch_bounds__(256) snake1d_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                      uint16_t* __restrict__ yimg, const float* __restrict__ alpha,
                                                      int C, int c8n, int T, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int t = (int)(i % T);
  const int64_t bc = i / T;
  const int c8 = (int)(bc % c8n), b = (int)(bc / c8n);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = c8 * 8 + e;
    v[e] = 0.f;
    if (c < C) {
      const int64_t at = ((int64_t)b * C + c) * T + t;
      const float xv = __ldg(x + at), a = __ldg(alpha + c);
      const float s = sinf(__fmul_rn(a, xv));
      v[e] = __fadd_rn(xv, __fmul_rn(__frcp_rn(__fadd_rn(a, 1e-9f)), __fmul_rn(s, s)));
      if (y) y[at] = v[e];
    }
  }
  if (IMG)
    *reinterpret_cast<uint4*>(yimg + (((size_t)b * c8n + c8) * T + t) * 8) =
        make_uint4(cvt_pair<IMG - 1>(v[0], v[1]), cvt_pair<IMG - 1>(v[2], v[3]), cvt_pair<IMG - 1>(v[4], v[5]),
                   cvt_pair<IMG - 1>(v[6], v[7]));
}
}  // namespace

int launch_snake1d(const float* x, float* y, uint16_t* yimg, int bf16, const float* alpha, int B, int C, int T,
                   cudaStream_t s) {
  if (!x || !alpha || (!y && !yimg)) return fail(AB_ERR_ARG, "snake1d: null argument");
  if (B <= 0 || C <= 0 || T <= 0) return fail(AB_ERR_ARG, "snake1d: bad shape");
  const int c8n = (C + 15) / 16 * 2;
  const int64_t total = (int64_t)B * c8n * T, grid = ceil_div(total, 256);
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "snake1d: grid too large");
  void (*kerns[3])(const float*, float*, uint16_t*, const float*, int, int, int, int64_t) = {
      snake1d_kernel<0>, snake1d_kernel<1>, snake1d_kernel<2>};
  kerns[yimg ? (bf16 ? 2 : 1) : 0]<<<(unsigned)grid, 256, 0, s>>>(x, y, yimg, alpha, C, c8n, T, total);
  AB_LAUNCH_CHECK("snake1d_kernel");
  return AB_OK;
}

int launch_scale_inplace(float* p, size_t n, float gain, cudaStream_t s) {
  if (n == 0) return AB_OK;
  const int blocks = (int)std::min<size_t>((n + 255) / 256, 148 * 8);
  scale_inplace_kernel<<<blocks, 256, 0, s>>>(p, n, gain);
  AB_LAUNCH_CHECK("scale_inplace_kernel");
  return AB_OK;
}

}  // namespace ab
