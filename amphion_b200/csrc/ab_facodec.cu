// FACodec decoder prologue kernels (models/codec/ns3_codec/facodec.py:556-576): the codebook decode (vq2emb), the
// timbre projection and the LayerNorm + FiLM in front of conv_pre.  The generator itself runs on the BigVGAN path of
// ab_capi.cu's forward_impl.
#include <algorithm>

#include "ab_common.cuh"

namespace ab {
namespace {

// saturating round-to-nearest pair conversion, as the other operand-image writers do
template <int BF16>
__device__ __forceinline__ uint32_t fac_cvt_pair(float lo, float hi) {
  uint32_t r;
  if (BF16) asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// style[b][o] = bias[o] + sum_i w[o][i] spk[b][i]: one warp per output row, lane-strided partial sums, butterfly
// reduction (facodec.py:569, timbre_linear(speaker_embedding))
__global__ void __launch_bounds__(256) facodec_style_kernel(const float* __restrict__ spk, int64_t spk_stride,
                                                            const float* __restrict__ w, const float* __restrict__ bias,
                                                            float* __restrict__ style, int C) {
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = blockIdx.x * 8 + warp;
  if (o >= 2 * C) return;
  const float* s = spk + b * spk_stride;
  const float* wr = w + (int64_t)o * C;
  float a = 0.f;
  for (int i = lane; i < C; i += 32) a = fmaf(__ldg(wr + i), __ldg(s + i), a);
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
  if (lane == 0) style[(int64_t)b * 2 * C + o] = a + __ldg(bias + o);
}

// y = LayerNorm(x)[c] * gamma[c] + beta[c] per (utterance, time step), the LayerNorm over channels without affine
// (eps 1e-5): two-pass fp32 mean and biased variance.  One CTA per (utterance, tile of TT time steps); the tile's
// C x TT values sit in shared memory.  OUT: 0 fp32 [B, C, T]; 1 / 2 the fp16 / bf16 operand image.
constexpr int FILM_THREADS = 256;

template <int OUT>
__global__ void __launch_bounds__(FILM_THREADS) facodec_film_kernel(FacFilmParams p, int TT, int tiles) {
  extern __shared__ float fsm[];   // [C][TT] values, [FILM_THREADS] partial sums, [TT] mean, [TT] 1/std
  float* part = fsm + (size_t)p.C * TT;
  float* mean_s = part + FILM_THREADS;
  float* rstd_s = mean_s + TT;
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * TT;
  const int tid = threadIdx.x, tt = tid % TT, grp = tid / TT, ngrp = FILM_THREADS / TT;
  const float* xb = p.x + (int64_t)b * p.xsb;
  const int n = p.C * TT;
  for (int i = tid; i < n; i += FILM_THREADS) {
    const int c = i / TT, t = t0 + (i - c * TT);
    fsm[i] = t < p.T ? __ldg(xb + c * p.xsc + (int64_t)t * p.xst) : 0.f;
  }
  __syncthreads();
  float a = 0.f;
  for (int c = grp; c < p.C; c += ngrp) a = __fadd_rn(a, fsm[c * TT + tt]);
  part[tid] = a;
  __syncthreads();
  if (tid < TT) {
    float s = 0.f;
    for (int q = 0; q < ngrp; ++q) s = __fadd_rn(s, part[q * TT + tid]);
    mean_s[tid] = __fdiv_rn(s, (float)p.C);
  }
  __syncthreads();
  const float mu = mean_s[tt];
  a = 0.f;
  for (int c = grp; c < p.C; c += ngrp) {
    const float d = __fsub_rn(fsm[c * TT + tt], mu);
    a = __fmaf_rn(d, d, a);
  }
  part[tid] = a;
  __syncthreads();
  if (tid < TT) {
    float s = 0.f;
    for (int q = 0; q < ngrp; ++q) s = __fadd_rn(s, part[q * TT + tid]);
    rstd_s[tid] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(s, (float)p.C), 1e-5f)));
  }
  __syncthreads();
  const float* gamma = p.style + (int64_t)b * 2 * p.C;
  const float* beta = gamma + p.C;
  // x_norm * gamma + beta with both roundings (facodec.py:574), never contracted into an FMA
  auto film = [&](int c, int u) {
    const float xn = __fmul_rn(__fsub_rn(fsm[c * TT + u], mean_s[u]), rstd_s[u]);
    return __fadd_rn(__fmul_rn(xn, __ldg(gamma + c)), __ldg(beta + c));
  };
  if (OUT == 0) {
    for (int i = tid; i < n; i += FILM_THREADS) {
      const int c = i / TT, u = i - c * TT, t = t0 + u;
      if (t < p.T) p.y[((int64_t)b * p.C + c) * p.T + t] = film(c, u);
    }
  } else {
    const int c8n = (p.C + 15) / 16 * 2;
    for (int i = tid; i < c8n * TT; i += FILM_THREADS) {
      const int c8 = i / TT, u = i - c8 * TT, t = t0 + u;
      if (t >= p.T) continue;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = c8 * 8 + e < p.C ? film(c8 * 8 + e, u) : 0.f;
      *reinterpret_cast<uint4*>(p.yimg + (((size_t)b * c8n + c8) * p.T + t) * 8) =
          make_uint4(fac_cvt_pair<OUT - 1>(v[0], v[1]), fac_cvt_pair<OUT - 1>(v[2], v[3]),
                     fac_cvt_pair<OUT - 1>(v[4], v[5]), fac_cvt_pair<OUT - 1>(v[6], v[7]));
    }
  }
}

// vq2emb: one CTA per (utterance, tile of VQ_TT time steps).  The tile's codebook rows go to shared memory once
// (a code outside its codebook is not read and marks its time step); every output (c, t) then applies each layer's
// out_proj (a D-term dot product from 0, then the bias) and sums the layers of a ResidualVQ in layer order, then the
// groups in order (rvq.py:75-81, facodec.py:556-566).
constexpr int VQ_TT = 16;
constexpr int VQ_THREADS = 256;

__global__ void __launch_bounds__(VQ_THREADS) facodec_vq2emb_kernel(FacVqParams p, int tiles) {
  extern __shared__ float vsm[];   // [nq][VQ_TT][D] codebook rows
  __shared__ int bad[VQ_TT];
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * VQ_TT;
  const int D = p.D;
  if (threadIdx.x < VQ_TT) bad[threadIdx.x] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < p.nq * VQ_TT; i += VQ_THREADS) {
    const int q = i / VQ_TT, u = i - q * VQ_TT, t = t0 + u;
    float* e = vsm + (size_t)i * D;
    if (t >= p.T) continue;
    const int64_t code = p.codes[q * p.cs0 + b * p.cs1 + t * p.cs2];
    if (code < 0 || code >= p.rows[q]) {
      bad[u] = 1;
      for (int j = 0; j < D; ++j) e[j] = 0.f;
    } else {
      const float* row = p.cb[q] + code * D;
      for (int j = 0; j < D; ++j) e[j] = __ldg(row + j);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < p.C * VQ_TT; i += VQ_THREADS) {
    const int c = i / VQ_TT, u = i - c * VQ_TT, t = t0 + u;
    if (t >= p.T) continue;
    float out = 0.f;
    for (int gi = 0, q = 0; gi < p.ngroups; ++gi) {
      float gsum = 0.f;
      for (const int qe = p.group_end[gi]; q < qe; ++q) {
        const float* e = vsm + ((size_t)q * VQ_TT + u) * D;
        const float* w = p.w[q];   // repacked out_proj [D][C]
        float a = 0.f;
        for (int j = 0; j < D; ++j) a = __fmaf_rn(e[j], __ldg(w + (size_t)j * p.C + c), a);
        a = __fadd_rn(a, __ldg(p.bias[q] + c));
        gsum = __fadd_rn(gsum, a);
      }
      out = __fadd_rn(out, gsum);
    }
    p.out[((int64_t)b * p.C + c) * p.T + t] = bad[u] ? __int_as_float(0x7fc00000) : out;
  }
}

}  // namespace

int launch_facodec_style(const float* spk, int64_t spk_stride, const float* w, const float* bias, float* style, int B,
                         int C, cudaStream_t s) {
  if (!spk || !w || !bias || !style) return fail(AB_ERR_ARG, "facodec style: null argument");
  if (B <= 0 || B > 65535 || C <= 0) return fail(AB_ERR_ARG, "facodec style: bad shape");
  facodec_style_kernel<<<dim3((unsigned)ceil_div(2 * C, 8), (unsigned)B), 256, 0, s>>>(spk, spk_stride, w, bias, style, C);
  AB_LAUNCH_CHECK("facodec_style_kernel");
  return AB_OK;
}

int launch_facodec_film(const FacFilmParams& p, cudaStream_t s) {
  if (!p.x || !p.style || (!p.y) == (!p.yimg)) return fail(AB_ERR_ARG, "facodec film: null argument");
  if (p.B <= 0 || p.C <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "facodec film: bad shape");
  // time tile: up to 16 steps, fewer for wide C so that a few CTAs share an SM
  int TT = 16;
  auto smem_of = [&](int tt) { return sizeof(float) * ((size_t)p.C * tt + FILM_THREADS + 2 * tt); };
  while (TT > 1 && smem_of(TT) > 64 * 1024) TT >>= 1;
  const size_t smem = smem_of(TT);
  if (smem > 200 * 1024) return fail(AB_ERR_UNSUPPORTED, "facodec film: %d channels do not fit shared memory", p.C);
  const int64_t tiles = ceil_div(p.T, TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "facodec film: grid too large");
  const int out = p.y ? 0 : (p.bf16 ? 2 : 1);
  void (*kerns[3])(FacFilmParams, int, int) = {facodec_film_kernel<0>, facodec_film_kernel<1>, facodec_film_kernel<2>};
  static DeviceOnce configured[3];
  if (smem > 48 * 1024 && configured[out].need())
    AB_CUDA_TRY(cudaFuncSetAttribute(kerns[out], cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  kerns[out]<<<(unsigned)grid, FILM_THREADS, smem, s>>>(p, TT, (int)tiles);
  AB_LAUNCH_CHECK("facodec_film_kernel");
  return AB_OK;
}

int launch_facodec_vq2emb(const FacVqParams& p, cudaStream_t s) {
  if (!p.codes || !p.out) return fail(AB_ERR_ARG, "facodec vq2emb: null argument");
  if (p.B <= 0 || p.C <= 0 || p.T <= 0 || p.D <= 0 || p.D > FAC_MAX_CODEBOOK_DIM || p.nq <= 0 ||
      p.nq > AB_FACODEC_MAX_Q || p.ngroups <= 0 || p.ngroups > 3 || p.group_end[p.ngroups - 1] != p.nq)
    return fail(AB_ERR_ARG, "facodec vq2emb: bad shape");
  const size_t smem = sizeof(float) * (size_t)p.nq * VQ_TT * p.D;
  const int64_t tiles = ceil_div(p.T, VQ_TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "facodec vq2emb: grid too large");
  static DeviceOnce configured;
  if (smem > 48 * 1024 && configured.need())
    AB_CUDA_TRY(cudaFuncSetAttribute(facodec_vq2emb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  facodec_vq2emb_kernel<<<(unsigned)grid, VQ_THREADS, smem, s>>>(p, (int)tiles);
  AB_LAUNCH_CHECK("facodec_vq2emb_kernel");
  return AB_OK;
}

}  // namespace ab
