// FACodec decoder prologue kernels (models/codec/ns3_codec/facodec.py:556-576): the codebook decode (vq2emb), the
// timbre projection and the LayerNorm + FiLM in front of conv_pre.  The generator itself runs on the BigVGAN path of
// ab_capi.cu's forward_impl.  Then the kernels of FACodecDecoder.forward(vq=True) (facodec.py:408-471): the residual
// vector quantizer, the timbre encoder's attention and the time mean; its GEMMs and LayerNorms run on the shared
// convolution and LayerNorm kernels; FACodecDecoderV2 adds the prosody transformer's input and an RVQ whose prosody
// group reads that transformer's output.  Last the embedding gathers of FACodecRedecoder.vq2emb (facodec.py:734-759); its
// prosody transformer reuses the style, FiLM and attention kernels above.
#include <algorithm>
#include <type_traits>

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


// ---- FACodecDecoder.forward(vq=True) ------------------------------------------------------------------------------

// F.normalize(codebook) (eps 1e-12) into rows of 16 floats (zero padded) and the squared norms of the normalised rows,
// as fvq.py:103-111 computes them.  One thread per row.
__global__ void __launch_bounds__(256) facodec_cbnorm_kernel(const float* __restrict__ cb, float* __restrict__ cbn,
                                                             float* __restrict__ cbn2, int64_t rows, int D) {
  const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (r >= rows) return;
  float v[FAC_MAX_CODEBOOK_DIM];
  float n2 = 0.f;
#pragma unroll
  for (int d = 0; d < FAC_MAX_CODEBOOK_DIM; ++d) {
    v[d] = d < D ? __ldg(cb + r * D + d) : 0.f;
    n2 = __fmaf_rn(v[d], v[d], n2);
  }
  const float den = fmaxf(__fsqrt_rn(n2), 1e-12f);
  float c2 = 0.f;
#pragma unroll
  for (int d = 0; d < FAC_MAX_CODEBOOK_DIM; ++d) {
    const float c = d < D ? __fdiv_rn(v[d], den) : 0.f;
    cbn[r * FAC_MAX_CODEBOOK_DIM + d] = c;
    c2 = __fmaf_rn(c, c, c2);
  }
  cbn2[r] = c2;
}

// The residual vector quantizer, all groups in one launch.  One CTA per (utterance, tile of RVQ_TT frames): the tile's
// x, the running residual, the current group's sum and prosody + content sit in shared memory [C][RVQ_TT]; each layer
// streams its normalised codebook through shared memory in chunks of RVQ_CH rows, so any codebook size is served.
// Per layer and frame (fvq.py:52-91):
//   z_e = b_in + sum_c W_in[d][c] r[c]  (an fp32 FMA chain over c ascending, then the bias)
//   e = z_e / max(|z_e|, 1e-12);  dist_i = (|e|^2 - 2 e.c_i) + |c_i|^2;  code = the lowest i of the least dist
//   z_q = z_e + (codebook[code] - z_e)  (the straight-through step, two fp32 roundings)
//   q = sum_d W_out[c][d] z_q[d] (an FMA chain from 0) + b_out[c];  r -= q;  group sum += q
// The groups' sums are written as they complete; emb = (prosody + content) + residual.  Three instantiations, so that
// V1's code holds neither of the others' sources: RVQ_FACODEC; RVQ_PROSODY (FACodecDecoderV2, facodec.py:1027-1094): the
// prosody group's residual starts from the prosody transformer's output instead of x, the content and residual groups
// and the positional add are V1's; RVQ_LAYERS (the codec's ResidualVQ, amphion_codec/quantize/residual_vq.py:69-134):
// one group, whose sum ((0 + q_0) + q_1) + ... is quantized_out, and each layer's q also written to its plane of `layers`
// when that is given.  With one group x is needed only once, so RVQ_LAYERS loads it straight into the residual and keeps
// two [C][TT] planes (residual, sum) where the FACodec modes keep four: 128 C + 19,584 bytes, which fits C <= 1447
// (RepCodec's 1024-wide features) in the 200 KB the launch allows.  Its arithmetic is the other modes'.
constexpr int RVQ_TT = 16;
constexpr int RVQ_THREADS = 256;
constexpr int RVQ_CH = 256;
constexpr int RVQ_LANES = RVQ_THREADS / RVQ_TT;   // threads scanning one frame's codebook
constexpr int RVQ_SMEM_MAX = 200 * 1024;

enum RvqMode { RVQ_FACODEC = 0, RVQ_PROSODY = 1, RVQ_LAYERS = 2 };

constexpr size_t rvq_smem_bytes(int C, bool layers) {
  return sizeof(float) * ((size_t)(layers ? 2 : 4) * C * RVQ_TT + RVQ_CH * (FAC_MAX_CODEBOOK_DIM + 1) +
                          RVQ_TT * (2 * FAC_MAX_CODEBOOK_DIM + 1)) + sizeof(int) * RVQ_TT;
}
static_assert(rvq_smem_bytes(AB_RVQ_MAX_INPUT_DIM, true) <= RVQ_SMEM_MAX &&
                  rvq_smem_bytes(AB_RVQ_MAX_INPUT_DIM + 1, true) > RVQ_SMEM_MAX,
              "AB_RVQ_MAX_INPUT_DIM is the widest input RVQ_LAYERS' shared memory holds");
struct FacRvqProsodyParams : FacRvqParams {
  const float* prosody;     // [B, C, T], the prosody transformer's output
};
struct FacRvqLayersParams : FacRvqParams {
  float* layers;            // [n_used, B, C, T]: layer q's out_proj(z_q) in plane q
};
template <int MODE>
using RvqArgs = typename std::conditional<MODE == RVQ_PROSODY, FacRvqProsodyParams,
                                          typename std::conditional<MODE == RVQ_LAYERS, FacRvqLayersParams,
                                                                    FacRvqParams>::type>::type;

template <int MODE>
__global__ void __launch_bounds__(RVQ_THREADS, 1) facodec_rvq_kernel(RvqArgs<MODE> p, int tiles) {
  extern __shared__ __align__(16) float qsm[];
  const int C = p.C, D = p.D, tid = threadIdx.x;
  constexpr bool ONE = MODE == RVQ_LAYERS;   // one group: x is the first residual, no x or s01 plane
  float* xs = qsm;                          // [C][TT] x
  float* rs = ONE ? qsm : xs + C * RVQ_TT;  // [C][TT] residual
  float* gs = rs + C * RVQ_TT;              // [C][TT] current group's sum
  float* s01 = gs + C * RVQ_TT;             // [C][TT] prosody, then prosody + content
  float* cbs = ONE ? s01 : s01 + C * RVQ_TT;   // [RVQ_CH][16] normalised codebook chunk
  float* cb2s = cbs + RVQ_CH * FAC_MAX_CODEBOOK_DIM;    // [RVQ_CH]
  float* zes = cb2s + RVQ_CH;               // [TT][16] z_e, then z_q
  float* es = zes + RVQ_TT * FAC_MAX_CODEBOOK_DIM;      // [TT][16] normalised z_e
  float* e2s = es + RVQ_TT * FAC_MAX_CODEBOOK_DIM;      // [TT] |e|^2
  int* codes = reinterpret_cast<int*>(e2s + RVQ_TT);    // [TT]
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * RVQ_TT;
  const int n = C * RVQ_TT;
  const float* xb = p.x + (int64_t)b * p.xsb;
  if constexpr (ONE) {
    // residual = x, sum = 0.  The walk follows x's smaller stride, so that both [B, C, T] and the [B, T, C] view
    // RepCodec's encoder hands over are read in runs along memory
    const bool cfast = p.xsc < p.xst;
    for (int i = tid; i < n; i += RVQ_THREADS) {
      const int q = cfast ? i / C : i / RVQ_TT, r = cfast ? i - q * C : i - q * RVQ_TT;
      const int c = cfast ? r : q, u = cfast ? q : r, t = t0 + u;
      rs[c * RVQ_TT + u] = t < p.T ? __ldg(xb + c * p.xsc + (int64_t)t * p.xst) : 0.f;
      gs[c * RVQ_TT + u] = 0.f;
    }
  } else {
    for (int i = tid; i < n; i += RVQ_THREADS) {
      const int c = i / RVQ_TT, t = t0 + (i - c * RVQ_TT);
      float v = 0.f;
      if (t < p.T) {
        v = __ldg(xb + c * p.xsc + (int64_t)t * p.xst);
        // transformer.py:43-45 on the batch-first stream: utterance b adds row b of pe at every time step
        if (p.stream) p.stream[((int64_t)b * C + c) * p.T + t] = __fadd_rn(v, __ldg(p.pe + (int64_t)b * C + c));
      }
      xs[i] = v;
    }
  }
  const int fu = tid / RVQ_LANES, lane = tid % RVQ_LANES;   // search: frame fu, rows lane, lane + RVQ_LANES, ...
  for (int g = 0; g < (ONE ? 1 : 3); ++g) {
    if (p.nused[g] == 0) continue;
    __syncthreads();
    if constexpr (!ONE) {
      for (int i = tid; i < n; i += RVQ_THREADS) {
        rs[i] = g < 2 ? xs[i] : __fsub_rn(xs[i], s01[i]);   // facodec.py:436: x - (prosody + content)
        gs[i] = 0.f;
      }
    }
    if constexpr (MODE == RVQ_PROSODY) {
      if (g == 0) {   // facodec.py:1038-1042: the prosody group quantizes melspec_encoder's output
        for (int i = tid; i < n; i += RVQ_THREADS) {
          const int c = i / RVQ_TT, t = t0 + (i - c * RVQ_TT);
          rs[i] = t < p.T ? __ldg(p.prosody + ((int64_t)b * C + c) * p.T + t) : 0.f;
        }
      }
    }
    for (int j = 0; j < p.nused[g]; ++j) {
      const int q = p.layer0[g] + j;
      __syncthreads();
      // z_e: thread (d, u)
      {
        const int d = tid / RVQ_TT, u = tid % RVQ_TT;
        if (d < D) {
          const float* w = p.w_in[q] + d;
          float a = 0.f;
          for (int c = 0; c < C; ++c) a = __fmaf_rn(__ldg(w + (size_t)c * D), rs[c * RVQ_TT + u], a);
          zes[u * FAC_MAX_CODEBOOK_DIM + d] = __fadd_rn(a, __ldg(p.b_in[q] + d));
        }
      }
      __syncthreads();
      if (tid < RVQ_TT) {   // F.normalize(z_e) and |e|^2
        const float* z = zes + tid * FAC_MAX_CODEBOOK_DIM;
        float n2 = 0.f;
        for (int d = 0; d < D; ++d) n2 = __fmaf_rn(z[d], z[d], n2);
        const float den = fmaxf(__fsqrt_rn(n2), 1e-12f);
        float e2 = 0.f;
        for (int d = 0; d < FAC_MAX_CODEBOOK_DIM; ++d) {
          const float e = d < D ? __fdiv_rn(z[d], den) : 0.f;
          es[tid * FAC_MAX_CODEBOOK_DIM + d] = e;
          e2 = __fmaf_rn(e, e, e2);
        }
        e2s[tid] = e2;
      }
      __syncthreads();
      float e[FAC_MAX_CODEBOOK_DIM];
#pragma unroll
      for (int d = 0; d < FAC_MAX_CODEBOOK_DIM; ++d) e[d] = es[fu * FAC_MAX_CODEBOOK_DIM + d];
      const float e2 = e2s[fu];
      float best = __int_as_float(0x7f800000);
      int best_i = 0x7fffffff;
      const int64_t rows = p.rows[q];
      for (int64_t r0 = 0; r0 < rows; r0 += RVQ_CH) {
        const int nr = rows - r0 < RVQ_CH ? (int)(rows - r0) : RVQ_CH;
        __syncthreads();
        const float4* src = reinterpret_cast<const float4*>(p.cbn[q] + r0 * FAC_MAX_CODEBOOK_DIM);
        for (int i = tid; i < nr * (FAC_MAX_CODEBOOK_DIM / 4); i += RVQ_THREADS)
          reinterpret_cast<float4*>(cbs)[i] = __ldg(src + i);
        for (int i = tid; i < nr; i += RVQ_THREADS) cb2s[i] = __ldg(p.cbn2[q] + r0 + i);
        __syncthreads();
        for (int i = lane; i < nr; i += RVQ_LANES) {
          const float4* c4 = reinterpret_cast<const float4*>(cbs + i * FAC_MAX_CODEBOOK_DIM);
          float dot = 0.f;
#pragma unroll
          for (int k = 0; k < FAC_MAX_CODEBOOK_DIM / 4; ++k) {
            const float4 c = c4[k];
            dot = __fmaf_rn(e[4 * k], c.x, dot);
            dot = __fmaf_rn(e[4 * k + 1], c.y, dot);
            dot = __fmaf_rn(e[4 * k + 2], c.z, dot);
            dot = __fmaf_rn(e[4 * k + 3], c.w, dot);
          }
          const float dist = __fadd_rn(__fsub_rn(e2, __fmul_rn(2.0f, dot)), cb2s[i]);
          if (dist < best) { best = dist; best_i = (int)(r0 + i); }   // rows ascend: the first of equals stays
        }
      }
      // the least dist over the frame's lanes, the lowest code among equals
#pragma unroll
      for (int m = RVQ_LANES / 2; m > 0; m >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, m);
        const int oi = __shfl_xor_sync(0xffffffffu, best_i, m);
        if (ob < best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
      }
      if (lane == 0) {
        // no finite distance (a NaN input): code 0, as argmax over NaNs is not defined either way
        codes[fu] = best_i == 0x7fffffff ? 0 : best_i;
      }
      __syncthreads();
      if (tid < RVQ_TT * FAC_MAX_CODEBOOK_DIM) {   // z_q = z_e + (codebook[code] - z_e)
        const int u = tid / FAC_MAX_CODEBOOK_DIM, d = tid % FAC_MAX_CODEBOOK_DIM;
        if (d < D) {
          const float z = zes[tid];
          zes[tid] = __fadd_rn(z, __fsub_rn(__ldg(p.cb[q] + (int64_t)codes[u] * D + d), z));
        }
        if (d == 0 && t0 + u < p.T)
          p.codes[((int64_t)(p.code_row0[g] + j) * p.B + b) * p.T + t0 + u] = codes[u];
      }
      __syncthreads();
      const float* wo = p.w_out[q];
      for (int i = tid; i < n; i += RVQ_THREADS) {
        const int c = i / RVQ_TT, u = i - c * RVQ_TT;
        const float* z = zes + u * FAC_MAX_CODEBOOK_DIM;
        float a = 0.f;
        for (int d = 0; d < D; ++d) a = __fmaf_rn(z[d], __ldg(wo + (size_t)d * C + c), a);
        a = __fadd_rn(a, __ldg(p.b_out[q] + c));
        rs[i] = __fsub_rn(rs[i], a);
        gs[i] = __fadd_rn(gs[i], a);
        if constexpr (ONE) {
          const int t = t0 + u;
          if (p.layers && t < p.T) p.layers[(((int64_t)q * p.B + b) * C + c) * p.T + t] = a;
        }
      }
    }
    __syncthreads();
    for (int i = tid; i < n; i += RVQ_THREADS) {
      const int c = i / RVQ_TT, t = t0 + (i - c * RVQ_TT);
      const float v = gs[i];
      if (t < p.T) p.quantized[(((int64_t)g * p.B + b) * C + c) * p.T + t] = v;
      if (ONE) continue;
      if (g == 0) s01[i] = v;
      else if (g == 1) s01[i] = __fadd_rn(s01[i], v);
      else if (t < p.T) p.emb[((int64_t)b * C + c) * p.T + t] = __fadd_rn(s01[i], v);
    }
    if (!ONE && g == 1 && p.nused[2] == 0) {
      for (int i = tid; i < n; i += RVQ_THREADS) {
        const int c = i / RVQ_TT, t = t0 + (i - c * RVQ_TT);
        if (t < p.T) p.emb[((int64_t)b * C + c) * p.T + t] = s01[i];
      }
    }
  }
}

// FACodecDecoderV2's prosody input (facodec.py:1036-1038 and transformer.py:43-45): melspec_linear over the 20 mel rows
// of each frame, then the batch-first PositionalEncoding's row b.  One CTA per (utterance, tile of PIN_TT frames),
// thread c = output channel: the input tile [20][PIN_TT] is read along time into shared memory (every thread then reads
// the same element: a broadcast), thread c holds row c of the weight, and the output tile [256][PIN_TT + 1] is written
// back along time.  Per output, in this order:
//   a = 0;  a = fma(w[c][i], x[i], a) for i = 0 .. 19;  a = a + bias[c];  a = a + pe[b][c]
constexpr int PIN_TT = 16;
constexpr int PIN_THREADS = FAC_TIMBRE_C;

__global__ void __launch_bounds__(PIN_THREADS) facodec_prosody_input_kernel(FacProsodyInParams p, int tiles) {
  __shared__ float xs[FAC_PROSODY_BINS][PIN_TT];
  __shared__ float ys[FAC_TIMBRE_C][PIN_TT + 1];
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * PIN_TT;
  const int tid = threadIdx.x;
  const float* xb = p.x + (int64_t)b * p.xsb;
  for (int i = tid; i < FAC_PROSODY_BINS * PIN_TT; i += PIN_THREADS) {
    const int j = i / PIN_TT, u = i - j * PIN_TT, t = t0 + u;
    xs[j][u] = t < p.T ? __ldg(xb + j * p.xsi + (int64_t)t * p.xst) : 0.f;
  }
  float w[FAC_PROSODY_BINS];
#pragma unroll
  for (int j = 0; j < FAC_PROSODY_BINS; ++j) w[j] = __ldg(p.w + tid * FAC_PROSODY_BINS + j);
  const float bias = __ldg(p.bias + tid), pe = __ldg(p.pe + (int64_t)b * FAC_TIMBRE_C + tid);
  __syncthreads();
#pragma unroll 4
  for (int u = 0; u < PIN_TT; ++u) {
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < FAC_PROSODY_BINS; ++j) a = __fmaf_rn(w[j], xs[j][u], a);
    ys[tid][u] = __fadd_rn(__fadd_rn(a, bias), pe);
  }
  __syncthreads();
  float* yb = p.y + (int64_t)b * FAC_TIMBRE_C * p.T;
  for (int i = tid; i < FAC_TIMBRE_C * PIN_TT; i += PIN_THREADS) {
    const int c = i / PIN_TT, u = i - c * PIN_TT, t = t0 + u;
    if (t < p.T) yb[(int64_t)c * p.T + t] = ys[c][u];
  }
}

// Multi-head self-attention core of nn.MultiheadAttention(256, 4, batch_first=True) without a mask
// (transformer.py:113-138): per head, softmax(q k^T / 8) v, flash style on the CUDA cores in fp32.  One CTA per
// (64-query tile, head, utterance) loops over 64-key tiles with an online max and sum (precise expf); T x T is never
// stored.  Thread (query i = tid / 4, quarter part = tid % 4) scores keys part*16 .. +15 of a tile and accumulates
// output dims part*16 .. +15.  OUT: 0 fp32 [B, 256, T]; 1 / 2 the fp16 / bf16 operand image [B][32][T][8].
constexpr int ATT_TILE = 64;
constexpr int ATT_HD = FAC_TIMBRE_C / FAC_TIMBRE_HEADS;   // 64
constexpr int ATT_THREADS = 256;
constexpr size_t ATT_SMEM = sizeof(float) * (2 * ATT_HD * ATT_TILE + ATT_TILE * (ATT_TILE + 4));

template <int OUT>
__global__ void __launch_bounds__(ATT_THREADS, 1) facodec_attention_kernel(const float* __restrict__ qkv, float* y,
                                                                       uint16_t* yimg, int T) {
  extern __shared__ __align__(16) float asm_[];
  float* ks = asm_;                          // [d][key] of the tile
  float* vs = ks + ATT_HD * ATT_TILE;        // [d][key]
  float* ps = vs + ATT_HD * ATT_TILE;        // [query][key] probabilities, rows padded to 68
  constexpr int PSTR = ATT_TILE + 4;
  const int h = blockIdx.y, b = blockIdx.z, q0 = blockIdx.x * ATT_TILE;
  const int tid = threadIdx.x, qi = tid >> 2, part = tid & 3;
  const int64_t base = (int64_t)b * 3 * FAC_TIMBRE_C * T;
  const float* qrow = qkv + base + (int64_t)(h * ATT_HD) * T;
  const float* krow = qkv + base + (int64_t)(FAC_TIMBRE_C + h * ATT_HD) * T;
  const float* vrow = qkv + base + (int64_t)(2 * FAC_TIMBRE_C + h * ATT_HD) * T;
  const int tq = q0 + qi;
  float q[ATT_HD];
#pragma unroll
  for (int d = 0; d < ATT_HD; ++d) q[d] = tq < T ? __ldg(qrow + (int64_t)d * T + tq) : 0.f;
  float o[16], l = 0.f, m = __int_as_float(0xff800000);
#pragma unroll
  for (int k = 0; k < 16; ++k) o[k] = 0.f;
  for (int k0 = 0; k0 < T; k0 += ATT_TILE) {
    __syncthreads();
    for (int i = tid; i < ATT_HD * ATT_TILE; i += ATT_THREADS) {
      const int d = i / ATT_TILE, j = i - d * ATT_TILE, t = k0 + j;
      ks[i] = t < T ? __ldg(krow + (int64_t)d * T + t) : 0.f;
      vs[i] = t < T ? __ldg(vrow + (int64_t)d * T + t) : 0.f;
    }
    __syncthreads();
    float s[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) s[k] = 0.f;
#pragma unroll
    for (int d = 0; d < ATT_HD; ++d) {
      const float4* kr = reinterpret_cast<const float4*>(ks + d * ATT_TILE + part * 16);
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const float4 kv = kr[k4];
        s[4 * k4] = __fmaf_rn(q[d], kv.x, s[4 * k4]);
        s[4 * k4 + 1] = __fmaf_rn(q[d], kv.y, s[4 * k4 + 1]);
        s[4 * k4 + 2] = __fmaf_rn(q[d], kv.z, s[4 * k4 + 2]);
        s[4 * k4 + 3] = __fmaf_rn(q[d], kv.w, s[4 * k4 + 3]);
      }
    }
    float mt = __int_as_float(0xff800000);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      s[k] = k0 + part * 16 + k < T ? __fmul_rn(s[k], 0.125f) : __int_as_float(0xff800000);
      mt = fmaxf(mt, s[k]);
    }
    mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
    mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
    const float mn = fmaxf(m, mt);               // every tile holds a key: finite
    const float alpha = expf(__fsub_rn(m, mn));  // 0 on the first tile (m = -inf)
    m = mn;
    float ls = 0.f;
    float4* pr = reinterpret_cast<float4*>(ps + qi * PSTR + part * 16);
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      float pv[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        pv[e] = expf(__fsub_rn(s[4 * k4 + e], mn));   // exp(-inf) = 0 for the keys past T
        ls = __fadd_rn(ls, pv[e]);
      }
      pr[k4] = make_float4(pv[0], pv[1], pv[2], pv[3]);
    }
    l = __fadd_rn(__fmul_rn(l, alpha), ls);
#pragma unroll
    for (int k = 0; k < 16; ++k) o[k] = __fmul_rn(o[k], alpha);
    __syncthreads();
    const int nk = min(ATT_TILE, T - k0);
    const float* prow = ps + qi * PSTR;
    const float* vcol = vs + part * 16 * ATT_TILE;
    for (int j = 0; j < nk; j += 4) {   // rows past nk hold zeros in v and p: 4-key steps stay exact
      const float4 p4 = *reinterpret_cast<const float4*>(prow + j);
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float4 v4 = *reinterpret_cast<const float4*>(vcol + k * ATT_TILE + j);
        o[k] = __fmaf_rn(p4.x, v4.x, o[k]);
        o[k] = __fmaf_rn(p4.y, v4.y, o[k]);
        o[k] = __fmaf_rn(p4.z, v4.z, o[k]);
        o[k] = __fmaf_rn(p4.w, v4.w, o[k]);
      }
    }
  }
  // the row sum over the four quarters, in a fixed order
  l = __fadd_rn(l, __shfl_xor_sync(0xffffffffu, l, 1));
  l = __fadd_rn(l, __shfl_xor_sync(0xffffffffu, l, 2));
  if (tq >= T) return;
  float r[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) r[k] = __fdiv_rn(o[k], l);
  const int c0 = h * ATT_HD + part * 16;
  if (OUT == 0) {
#pragma unroll
    for (int k = 0; k < 16; ++k) y[((int64_t)b * FAC_TIMBRE_C + c0 + k) * T + tq] = r[k];
  } else {
    constexpr int c8n = FAC_TIMBRE_C / 8;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
      *reinterpret_cast<uint4*>(yimg + (((size_t)b * c8n + c0 / 8 + hf) * T + tq) * 8) =
          make_uint4(fac_cvt_pair<OUT - 1>(r[8 * hf], r[8 * hf + 1]), fac_cvt_pair<OUT - 1>(r[8 * hf + 2], r[8 * hf + 3]),
                     fac_cvt_pair<OUT - 1>(r[8 * hf + 4], r[8 * hf + 5]), fac_cvt_pair<OUT - 1>(r[8 * hf + 6], r[8 * hf + 7]));
  }
}

// spk[b][c] = (sum over t of y[b, c, t]) / T: one warp per row, lane-strided partial sums in time order, a butterfly
// reduction (facodec.py:469, torch.mean(x_timbre, dim=2))
__global__ void __launch_bounds__(256) facodec_time_mean_kernel(const float* __restrict__ y, float* __restrict__ spk,
                                                               int rows, int T) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* yr = y + (int64_t)row * T;
  float a = 0.f;
  for (int t = lane; t < T; t += 32) a = __fadd_rn(a, __ldg(yr + t));
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) a = __fadd_rn(a, __shfl_xor_sync(0xffffffffu, a, m));
  if (lane == 0) spk[row] = __fdiv_rn(a, (float)T);
}


// ---- FACodecRedecoder.vq2emb ---------------------------------------------------------------------------------------

// The embedding sums of FACodecRedecoder.vq2emb (facodec.py:734-759).  One CTA per (utterance, tile of EMB_TT time
// steps).  The tile sits in shared memory [C][EMB_TT + 1]: prev is read into it along time, the table rows are then
// read along channels and summed into it in the reference's order, and the tile is written along time.  The padded
// row length keeps both access orders free of bank conflicts.  A code outside its table is not read and marks its
// time step, which is written as NaN.  Two uses: the prosody stream fed to the transformer (prev = the previous run's
// output or none, one prosody table, pe), and the tail (prev = last_ln's output, the content then residual tables).
constexpr int EMB_TT = 16;
constexpr int EMB_THREADS = 256;

__global__ void __launch_bounds__(EMB_THREADS) facodec_embed_kernel(FacEmbedParams p, int tiles) {
  extern __shared__ float esm[];   // [C][EMB_TT + 1]
  __shared__ int code_s[AB_FACODEC_MAX_Q][EMB_TT];
  __shared__ int bad[EMB_TT];
  constexpr int LD = EMB_TT + 1;
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * EMB_TT;
  const int C = p.C, tid = threadIdx.x, n = C * EMB_TT;
  if (tid < EMB_TT) bad[tid] = 0;
  __syncthreads();
  for (int i = tid; i < p.ntab * EMB_TT; i += EMB_THREADS) {
    const int j = i / EMB_TT, u = i - j * EMB_TT, t = t0 + u;
    int code = 0;
    if (t < p.T) {
      const int64_t v = p.codes[(p.row0 + j) * p.cs0 + b * p.cs1 + t * p.cs2];
      if (v < 0 || v >= p.rows[j]) bad[u] = 1;
      else code = (int)v;
    }
    code_s[j][u] = code;
  }
  if (p.prev) {
    const float* pb = p.prev + (int64_t)b * C * p.T;
    for (int i = tid; i < n; i += EMB_THREADS) {
      const int c = i / EMB_TT, u = i - c * EMB_TT, t = t0 + u;
      esm[c * LD + u] = t < p.T ? __ldg(pb + (int64_t)c * p.T + t) : 0.f;
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += EMB_THREADS) {
    const int u = i / C, c = i - u * C;
    if (t0 + u >= p.T || bad[u]) continue;
    int j = 0;
    float a = p.prev ? esm[c * LD + u] : __ldg(p.tab[j++] + (int64_t)code_s[0][u] * C + c);
    for (; j < p.ntab; ++j) a = __fadd_rn(a, __ldg(p.tab[j] + (int64_t)code_s[j][u] * C + c));
    if (p.pe) a = __fadd_rn(a, __ldg(p.pe + (int64_t)b * C + c));
    esm[c * LD + u] = a;
  }
  __syncthreads();
  float* ob = p.out + (int64_t)b * C * p.T;
  for (int i = tid; i < n; i += EMB_THREADS) {
    const int c = i / EMB_TT, u = i - c * EMB_TT, t = t0 + u;
    if (t < p.T) ob[(int64_t)c * p.T + t] = bad[u] ? __int_as_float(0x7fc00000) : esm[c * LD + u];
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

int launch_facodec_cbnorm(const float* cb, float* cbn, float* cbn2, int64_t rows, int D, cudaStream_t s) {
  if (!cb || !cbn || !cbn2 || rows <= 0 || D <= 0 || D > FAC_MAX_CODEBOOK_DIM)
    return fail(AB_ERR_ARG, "facodec cbnorm: bad argument");
  facodec_cbnorm_kernel<<<(unsigned)ceil_div(rows, 256), 256, 0, s>>>(cb, cbn, cbn2, rows, D);
  AB_LAUNCH_CHECK("facodec_cbnorm_kernel");
  return AB_OK;
}

int launch_facodec_rvq(const FacRvqParams& p, cudaStream_t s, const float* prosody, float* layers, bool one_group) {
  // one_group: the codec's single group, which writes quantized_out through `quantized`, no emb and no stream
  if (!p.x || (!one_group && !p.emb) || !p.codes || !p.quantized || (!p.pe) != (!p.stream) ||
      (one_group && (prosody || p.stream)) || (layers && !one_group))
    return fail(AB_ERR_ARG, "facodec rvq: null argument");
  const bool groups_ok = one_group ? p.ngroups == 1 && p.nused[1] == 0 && p.nused[2] == 0
                                   : p.nused[1] > 0 && p.ngroups >= 2 && p.ngroups <= 3;
  if (p.B <= 0 || p.C <= 0 || p.T <= 0 || p.D <= 0 || p.D > FAC_MAX_CODEBOOK_DIM || p.nused[0] <= 0 || !groups_ok)
    return fail(AB_ERR_ARG, "facodec rvq: bad shape");
  const size_t smem = rvq_smem_bytes(p.C, one_group);
  if (smem > RVQ_SMEM_MAX) return fail(AB_ERR_UNSUPPORTED, "facodec rvq: %d channels do not fit shared memory", p.C);
  const int64_t tiles = ceil_div(p.T, RVQ_TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "facodec rvq: grid too large");
  if (prosody) {
    static DeviceOnce configured;
    if (smem > 48 * 1024 && configured.need())
      AB_CUDA_TRY(cudaFuncSetAttribute(facodec_rvq_kernel<RVQ_PROSODY>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FacRvqProsodyParams q;
    static_cast<FacRvqParams&>(q) = p;
    q.prosody = prosody;
    facodec_rvq_kernel<RVQ_PROSODY><<<(unsigned)grid, RVQ_THREADS, smem, s>>>(q, (int)tiles);
    AB_LAUNCH_CHECK("facodec_rvq_kernel<RVQ_PROSODY>");
    return AB_OK;
  }
  if (one_group) {
    static DeviceOnce configured;
    if (smem > 48 * 1024 && configured.need())
      AB_CUDA_TRY(cudaFuncSetAttribute(facodec_rvq_kernel<RVQ_LAYERS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FacRvqLayersParams q;
    static_cast<FacRvqParams&>(q) = p;
    q.layers = layers;
    facodec_rvq_kernel<RVQ_LAYERS><<<(unsigned)grid, RVQ_THREADS, smem, s>>>(q, (int)tiles);
    AB_LAUNCH_CHECK("facodec_rvq_kernel<RVQ_LAYERS>");
    return AB_OK;
  }
  static DeviceOnce configured;
  if (smem > 48 * 1024 && configured.need())
    AB_CUDA_TRY(cudaFuncSetAttribute(facodec_rvq_kernel<RVQ_FACODEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  facodec_rvq_kernel<RVQ_FACODEC><<<(unsigned)grid, RVQ_THREADS, smem, s>>>(p, (int)tiles);
  AB_LAUNCH_CHECK("facodec_rvq_kernel");
  return AB_OK;
}

int launch_facodec_prosody_input(const FacProsodyInParams& p, cudaStream_t s) {
  if (!p.x || !p.w || !p.bias || !p.pe || !p.y) return fail(AB_ERR_ARG, "facodec prosody input: null argument");
  if (p.B <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "facodec prosody input: bad shape");
  const int64_t tiles = ceil_div(p.T, PIN_TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "facodec prosody input: grid too large");
  facodec_prosody_input_kernel<<<(unsigned)grid, PIN_THREADS, 0, s>>>(p, (int)tiles);
  AB_LAUNCH_CHECK("facodec_prosody_input_kernel");
  return AB_OK;
}

int launch_facodec_attention(const float* qkv, float* y, uint16_t* yimg, int bf16, int B, int T, cudaStream_t s) {
  if (!qkv || (!y) == (!yimg)) return fail(AB_ERR_ARG, "facodec attention: null argument");
  if (B <= 0 || B > 65535 || T <= 0) return fail(AB_ERR_ARG, "facodec attention: bad shape");
  const int out = y ? 0 : (bf16 ? 2 : 1);
  void (*kerns[3])(const float*, float*, uint16_t*, int) = {facodec_attention_kernel<0>, facodec_attention_kernel<1>,
                                                            facodec_attention_kernel<2>};
  static DeviceOnce configured[3];
  if (configured[out].need())
    AB_CUDA_TRY(cudaFuncSetAttribute(kerns[out], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ATT_SMEM));
  kerns[out]<<<dim3((unsigned)ceil_div(T, ATT_TILE), FAC_TIMBRE_HEADS, (unsigned)B), ATT_THREADS, ATT_SMEM, s>>>(qkv, y, yimg, T);
  AB_LAUNCH_CHECK("facodec_attention_kernel");
  return AB_OK;
}

int launch_facodec_time_mean(const float* y, float* spk, int B, int C, int T, cudaStream_t s) {
  if (!y || !spk || B <= 0 || C <= 0 || T <= 0) return fail(AB_ERR_ARG, "facodec time mean: bad argument");
  const int rows = B * C;
  facodec_time_mean_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, s>>>(y, spk, rows, T);
  AB_LAUNCH_CHECK("facodec_time_mean_kernel");
  return AB_OK;
}

int launch_facodec_embed(const FacEmbedParams& p, cudaStream_t s) {
  if (!p.codes || !p.out) return fail(AB_ERR_ARG, "facodec embed: null argument");
  if (p.B <= 0 || p.C <= 0 || p.T <= 0 || p.ntab <= 0 || p.ntab > AB_FACODEC_MAX_Q || p.row0 < 0)
    return fail(AB_ERR_ARG, "facodec embed: bad shape");
  for (int j = 0; j < p.ntab; ++j)
    if (!p.tab[j] || p.rows[j] <= 0 || p.rows[j] > (1 << 24)) return fail(AB_ERR_ARG, "facodec embed: bad table %d", j);
  const size_t smem = sizeof(float) * (size_t)p.C * (EMB_TT + 1);
  if (smem > 48 * 1024) return fail(AB_ERR_UNSUPPORTED, "facodec embed: %d channels do not fit shared memory", p.C);
  const int64_t tiles = ceil_div(p.T, EMB_TT), grid = (int64_t)p.B * tiles;
  if (grid > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "facodec embed: grid too large");
  facodec_embed_kernel<<<(unsigned)grid, EMB_THREADS, smem, s>>>(p, (int)tiles);
  AB_LAUNCH_CHECK("facodec_embed_kernel");
  return AB_OK;
}

}  // namespace ab
