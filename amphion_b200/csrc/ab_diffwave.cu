// DiffWave (AB_GEN_DIFFWAVE) kernels, fp32 CUDA-core arithmetic.  The network of
// models/vocoders/diffusion/diffwave/diffwave.py runs as:
//   once per call    dw_upsample_kernel  SpectrogramUpsampler (two 1-channel ConvTranspose2d + leaky_relu(0.4))
//                    dw_embed_kernel     DiffusionEmbedding (table lerp, Linear, SiLU, Linear, SiLU) and every
//                                        layer's diffusion_projection, for every diffusion step of the call
//   per network pass dw_input_kernel     relu(input_projection(audio))
//                    dw_layer_kernel     one ResidualBlock per launch: dilated conv + conditioner, gate, output
//                                        projection, residual update and skip sum (fp32 FMAs)
//                    dw_layer_tc_kernel  the same layer on the tensor cores (mma.sync m16n8k16, fp16 / bf16 operands,
//                                        fp32 accumulation, fp32 x and skip streams)
//                    dw_tail_kernel      skip / sqrt(L), skip_projection, relu, output_projection; writes eps or
//                                        applies one sampler update to the audio in place
// Sums run in a fixed order and the reference's divisions stay IEEE divisions, so repeated runs are bit-equal.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "ab_common.cuh"
#include "ab_tc_ptx.cuh"

namespace ab {

namespace {

constexpr int DW_C = DW_CHANNELS;   // residual channels (the kernels are compiled for this width)
constexpr int DW_TT = 64;           // time samples per layer tile (two per lane)
constexpr int DW_LAYER_THREADS = 4 * DW_C;   // warp w owns channels 8w .. 8w + 7 of both halves

__device__ __forceinline__ float lrelu04(float x) { return x > 0.f ? x : __fmul_rn(x, 0.4f); }
__device__ __forceinline__ float sigmoidf_(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// One ConvTranspose2d(1, 1, [3, 2f], stride [1, f], padding [1, f/2]) output at (h, w) of an [H, W] input with element
// strides (sh, sw), followed by leaky_relu(0.4).  Row h reads input rows h + 1 - kh; column w reads the two input
// columns j0 and j0 - 1 with kernel columns r and r + f, where w + f/2 = j0 f + r.
template <typename Src>
__device__ __forceinline__ float convt2d_lrelu(Src src, const float* w, float bias, int H, int64_t W, int f, int h,
                                               int64_t col) {
  const int64_t q = col + f / 2;
  const int64_t j0 = q / f;
  const int r = (int)(q - j0 * f);
  float acc = 0.f;
  for (int kh = 0; kh < 3; ++kh) {
    const int hh = h + 1 - kh;
    if (hh < 0 || hh >= H) continue;
    for (int e = 0; e < 2; ++e) {
      const int64_t j = j0 - e;
      if (j < 0 || j >= W) continue;
      acc = __fmaf_rn(src(hh, j), w[kh * 2 * f + r + e * f], acc);
    }
  }
  return lrelu04(__fadd_rn(acc, bias));
}

__global__ void dw_upsample_kernel(const DwUpsampleParams p) {
  const int64_t L1 = (int64_t)p.F * p.f1, L = L1 * p.f2;
  const int64_t n = (int64_t)p.B * p.n_mel * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i % L;
    const int h = (int)((i / L) % p.n_mel);
    const int b = (int)(i / (L * p.n_mel));
    const float* mel = p.mel + b * p.msb;
    auto mel_at = [&](int hh, int64_t j) { return mel[hh * p.msc + j * p.mst]; };
    auto up1_at = [&](int hh, int64_t j) { return convt2d_lrelu(mel_at, p.w1, p.b1[0], p.n_mel, p.F, p.f1, hh, j); };
    p.out[i] = convt2d_lrelu(up1_at, p.w2, p.b2[0], p.n_mel, L1, p.f2, h, t);
  }
}

__device__ __forceinline__ float siluf_(float x) { return __fmul_rn(x, sigmoidf_(x)); }

// grid = steps, block = 512: e = lerp(table[floor t], table[ceil t], t - floor t); h = silu(W2 silu(W1 e + b1) + b2);
// d[s][l][c] = bd[l][c] + Wd[l][c] . h
__global__ void __launch_bounds__(512) dw_embed_kernel(const DwEmbedParams p) {
  __shared__ float e[128], h1[512], h2[512];
  const int s = blockIdx.x, tid = threadIdx.x;
  const float t = p.steps[s];
  const float lo = floorf(t);
  const float* low = p.table + (int64_t)lo * 128;
  const float* high = p.table + (int64_t)ceilf(t) * 128;
  if (tid < 128) e[tid] = __fadd_rn(low[tid], __fmul_rn(__fsub_rn(high[tid], low[tid]), __fsub_rn(t, lo)));
  __syncthreads();
  float a = 0.f;
  for (int i = 0; i < 128; ++i) a = __fmaf_rn(p.w1[tid * 128 + i], e[i], a);
  h1[tid] = siluf_(__fadd_rn(a, p.b1[tid]));
  __syncthreads();
  a = 0.f;
  for (int i = 0; i < 512; ++i) a = __fmaf_rn(p.w2[tid * 512 + i], h1[i], a);
  h2[tid] = siluf_(__fadd_rn(a, p.b2[tid]));
  __syncthreads();
  const int n = p.layers * DW_C;
  for (int o = tid; o < n; o += blockDim.x) {
    const float* w = p.wd + (int64_t)o * 512;
    a = 0.f;
    for (int i = 0; i < 512; ++i) a = __fmaf_rn(w[i], h2[i], a);
    p.d[(int64_t)s * n + o] = __fadd_rn(a, p.bd[o]);
  }
}

__global__ void dw_input_kernel(const float* __restrict__ audio, const float* __restrict__ w, const float* __restrict__ bias,
                                float* __restrict__ x, int B, int64_t L) {
  const int64_t n = (int64_t)B * DW_C * L;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i % L;
    const int c = (int)((i / L) % DW_C);
    const int64_t b = i / (L * DW_C);
    x[i] = fmaxf(__fadd_rn(__fmul_rn(w[c], audio[b * L + t]), bias[c]), 0.f);
  }
}

// grid (ceil(L / 64), B), 4 C threads.  Shared: S [3C + n_mel][64] = the three dilated taps of y = x + d (zero outside
// the utterance, as the conv's zero padding sees them), each its own 64-row window however large the dilation, then the
// upsampled mel; Z [C][64] = sigmoid(gate) tanh(filter).  Packed weights put gate channel c and filter channel c (and
// residual c / skip c) in the same warp's 16-column group: columns 16w .. 16w + 7 are channels 8w .. 8w + 7 of the first
// half, 16w + 8 .. 16w + 15 the same channels of the second half.
__global__ void __launch_bounds__(DW_LAYER_THREADS) dw_layer_kernel(const DwLayerParams p) {
  extern __shared__ float sm[];
  constexpr int C = DW_C, C2 = 2 * DW_C;
  const int K1 = 3 * C + p.n_mel;
  float* S = sm;
  float* Z = sm + K1 * DW_TT;
  const int b = blockIdx.y;
  const int64_t L = p.L, t0 = (int64_t)blockIdx.x * DW_TT;
  const float* xb = p.x_in + (int64_t)b * C * L;
  const float* db = p.d + b * p.d_bstride;
  for (int i = threadIdx.x; i < 3 * C * DW_TT; i += blockDim.x) {
    const int t = i % DW_TT, c = (i / DW_TT) % C, tap = i / (DW_TT * C);
    const int64_t tt = t0 + t + (int64_t)(tap - 1) * p.dil;
    S[i] = (tt >= 0 && tt < L) ? __fadd_rn(xb[c * L + tt], db[c]) : 0.f;
  }
  const float* mb = p.cond + (int64_t)b * p.n_mel * L;
  for (int i = threadIdx.x; i < p.n_mel * DW_TT; i += blockDim.x) {
    const int t = i % DW_TT, m = i / DW_TT;
    S[3 * C * DW_TT + i] = t0 + t < L ? mb[m * L + t0 + t] : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float a[16][2];
#pragma unroll
  for (int j = 0; j < 16; ++j) a[j][0] = a[j][1] = 0.f;
  const float* w1 = p.w1 + warp * 16;
#pragma unroll 2
  for (int k = 0; k < K1; ++k) {
    const float s0 = S[k * DW_TT + lane], s1 = S[k * DW_TT + lane + 32];
    const float4* w = reinterpret_cast<const float4*>(w1 + (int64_t)k * C2);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = __ldg(w + q);
      a[4 * q + 0][0] = __fmaf_rn(v.x, s0, a[4 * q + 0][0]); a[4 * q + 0][1] = __fmaf_rn(v.x, s1, a[4 * q + 0][1]);
      a[4 * q + 1][0] = __fmaf_rn(v.y, s0, a[4 * q + 1][0]); a[4 * q + 1][1] = __fmaf_rn(v.y, s1, a[4 * q + 1][1]);
      a[4 * q + 2][0] = __fmaf_rn(v.z, s0, a[4 * q + 2][0]); a[4 * q + 2][1] = __fmaf_rn(v.z, s1, a[4 * q + 2][1]);
      a[4 * q + 3][0] = __fmaf_rn(v.w, s0, a[4 * q + 3][0]); a[4 * q + 3][1] = __fmaf_rn(v.w, s1, a[4 * q + 3][1]);
    }
  }
  // gate, filter = chunk(y, 2): sigmoid(gate) * tanh(filter); the two biases of y are folded into b1
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float bg = p.b1[warp * 16 + i], bf = p.b1[warp * 16 + 8 + i];
#pragma unroll
    for (int e = 0; e < 2; ++e)
      Z[(warp * 8 + i) * DW_TT + lane + 32 * e] =
          __fmul_rn(sigmoidf_(__fadd_rn(a[i][e], bg)), tanhf(__fadd_rn(a[8 + i][e], bf)));
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 16; ++j) a[j][0] = a[j][1] = 0.f;
  const float* w2 = p.w2 + warp * 16;
#pragma unroll 4
  for (int k = 0; k < C; ++k) {
    const float s0 = Z[k * DW_TT + lane], s1 = Z[k * DW_TT + lane + 32];
    const float4* w = reinterpret_cast<const float4*>(w2 + (int64_t)k * C2);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = __ldg(w + q);
      a[4 * q + 0][0] = __fmaf_rn(v.x, s0, a[4 * q + 0][0]); a[4 * q + 0][1] = __fmaf_rn(v.x, s1, a[4 * q + 0][1]);
      a[4 * q + 1][0] = __fmaf_rn(v.y, s0, a[4 * q + 1][0]); a[4 * q + 1][1] = __fmaf_rn(v.y, s1, a[4 * q + 1][1]);
      a[4 * q + 2][0] = __fmaf_rn(v.z, s0, a[4 * q + 2][0]); a[4 * q + 2][1] = __fmaf_rn(v.z, s1, a[4 * q + 2][1]);
      a[4 * q + 3][0] = __fmaf_rn(v.w, s0, a[4 * q + 3][0]); a[4 * q + 3][1] = __fmaf_rn(v.w, s1, a[4 * q + 3][1]);
    }
  }
  // residual, skip = chunk(y, 2): x' = (x + residual) / sqrt(2); skip sum += skip (the first layer stores it)
  float* xo = p.x_out + (int64_t)b * C * L;
  float* sk = p.skip + (int64_t)b * C * L;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = warp * 8 + i;
    const float br = p.b2[warp * 16 + i], bs = p.b2[warp * 16 + 8 + i];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int64_t t = t0 + lane + 32 * e;
      if (t >= L) continue;
      const int64_t o = c * L + t;
      xo[o] = __fdiv_rn(__fadd_rn(xb[o], __fadd_rn(a[i][e], br)), 1.41421356237309515f);
      const float s = __fadd_rn(a[8 + i][e], bs);
      sk[o] = p.first ? s : __fadd_rn(s, sk[o]);
    }
  }
}

// One thread per (utterance, sample): h = relu(Wsk (skip / sqrt(L)) + bsk); eps = wo . h + bo.  eps != nullptr: store
// eps; otherwise audio = clamp(c1 (audio - c2 eps) [+ sigma noise], -1, 1) in place (one step of vocoder_inference).
__global__ void __launch_bounds__(128) dw_tail_kernel(const DwTailParams p) {
  __shared__ float W[DW_C * DW_C], bsk[DW_C], wo[DW_C];
  for (int i = threadIdx.x; i < DW_C * DW_C; i += blockDim.x) W[i] = p.wsk[i];
  if (threadIdx.x < DW_C) {
    bsk[threadIdx.x] = p.bsk[threadIdx.x];
    wo[threadIdx.x] = p.wo[threadIdx.x];
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)p.B * p.L) return;
  const int64_t b = i / p.L, t = i % p.L;
  const float* sk = p.skip + b * DW_C * p.L + t;
  float s[DW_C];
#pragma unroll
  for (int c = 0; c < DW_C; ++c) s[c] = __fdiv_rn(sk[c * p.L], p.skip_div);
  float e = 0.f;
#pragma unroll 4
  for (int o = 0; o < DW_C; ++o) {
    float h = 0.f;
#pragma unroll
    for (int c = 0; c < DW_C; ++c) h = __fmaf_rn(W[o * DW_C + c], s[c], h);
    e = __fmaf_rn(wo[o], fmaxf(__fadd_rn(h, bsk[o]), 0.f), e);
  }
  e = __fadd_rn(e, p.bo[0]);
  if (p.eps) {
    p.eps[i] = e;
    return;
  }
  float v = __fmul_rn(p.c1, __fsub_rn(p.audio[i], __fmul_rn(p.c2, e)));
  if (p.noise) v = __fadd_rn(v, __fmul_rn(p.sigma, p.noise[i]));
  p.audio[i] = fminf(fmaxf(v, -1.f), 1.f);
}

// Finalize: one layer's weights into the column groups dw_layer_kernel reads (see there).
__global__ void dw_pack_kernel(const DwPackParams p) {
  constexpr int C = DW_C, C2 = 2 * DW_C;
  const int K1 = 3 * C + p.n_mel;
  auto src = [](int j) { const int g = j / 16, r = j % 16; return r < 8 ? g * 8 + r : C + g * 8 + r - 8; };
  const int n1 = K1 * C2, n2 = C * C2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2 + C2; i += gridDim.x * blockDim.x) {
    if (i < n1) {
      const int k = i / C2, o = src(i % C2);
      p.w1p[i] = k < 3 * C ? p.wdil[(o * C + k % C) * 3 + k / C] : p.wcond[o * p.n_mel + k - 3 * C];
    } else if (i < n1 + n2) {
      const int k = (i - n1) / C2, o = src((i - n1) % C2);
      p.w2p[i - n1] = p.wout[o * C + k];
    } else {
      const int o = src(i - n1 - n2);
      p.b1p[i - n1 - n2] = __fadd_rn(p.bdil[o], p.bcond[o]);
      p.b2p[i - n1 - n2] = p.bout[o];
    }
  }
}


// ---- tensor-core layer ------------------------------------------------------------------------------------------
// fp32 -> 16-bit operand, round to nearest and saturating (cvt.rn.satfinite): an operand never becomes inf, whose
// products with the zero weights of its k16 block would be NaN (DESIGN.md §5)
template <bool BF16>
__device__ __forceinline__ uint16_t to16(float v) {
  return (uint16_t)(tcx::pack2t<BF16>(v, 0.f) & 0xffffu);
}

template <bool BF16>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[j] += A[16 rows from a_row][K] x W[n0 + 8 j + .. ][K] over K in steps of 16.  A is time-major in shared memory
// (row stride lda halves), W is [column][K] (stride ldw halves) in global memory, read through L1.
template <bool BF16>
__device__ __forceinline__ void mma_rows(float (&acc)[8][4], const uint16_t* A, int lda, const uint16_t* W, int ldw,
                                         int K, int lane) {
  const int g = lane >> 2, q = lane & 3;
  const uint16_t* a0p = A + g * lda + 2 * q;
  const uint16_t* wp = W + g * ldw + 2 * q;
#pragma unroll 2
  for (int k = 0; k < K; k += 16) {
    uint32_t a[4];
    a[0] = *reinterpret_cast<const uint32_t*>(a0p + k);
    a[1] = *reinterpret_cast<const uint32_t*>(a0p + 8 * lda + k);
    a[2] = *reinterpret_cast<const uint32_t*>(a0p + k + 8);
    a[3] = *reinterpret_cast<const uint32_t*>(a0p + 8 * lda + k + 8);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint16_t* w = wp + (size_t)8 * j * ldw + k;
      mma16816<BF16>(acc[j], a, __ldg(reinterpret_cast<const unsigned int*>(w)), __ldg(reinterpret_cast<const unsigned int*>(w + 8)));
    }
  }
}

// grid (ceil(L / 64), B), 256 threads.  Shared: A1 [64 t][K1p (+8)] = the three dilated taps of x + d (each its own
// 64-row window, zero outside the utterance) and the upsampled mel, as 16-bit operands; Z [64 t][C (+8)] = the gate.
// Warp w computes rows 16 (w & 3) .. + 15 and packed columns 64 (w >> 2) .. + 63; in that column block n-tile j < 4
// holds gate channels 32 (w >> 2) + 8 j .. + 7 and n-tile j + 4 the filter (conv1), resp. residual and skip (conv2),
// of the same channels, so every thread finishes its channels without an exchange.
template <bool BF16>
__global__ void __launch_bounds__(256) dw_layer_tc_kernel(const DwLayerParams p) {
  extern __shared__ __align__(16) uint16_t smh[];
  constexpr int C = DW_C;
  const int K1p = 3 * C + (p.n_mel + 15) / 16 * 16, lda = K1p + 8, ldz = C + 8;
  uint16_t* A1 = smh;
  uint16_t* Z = smh + DW_TT * lda;
  const int b = blockIdx.y;
  const int64_t L = p.L, t0 = (int64_t)blockIdx.x * DW_TT;
  const float* xb = p.x_in + (int64_t)b * C * L;
  const float* db = p.d + b * p.d_bstride;
  const float* mb = p.cond + (int64_t)b * p.n_mel * L;
  for (int i = threadIdx.x; i < K1p * DW_TT; i += blockDim.x) {
    const int t = i % DW_TT, k = i / DW_TT;
    float v = 0.f;
    if (k < 3 * C) {
      const int c = k % C, tap = k / C;
      const int64_t tt = t0 + t + (int64_t)(tap - 1) * p.dil;
      if (tt >= 0 && tt < L) v = __fadd_rn(xb[c * L + tt], db[c]);
    } else if (k - 3 * C < p.n_mel && t0 + t < L) {
      v = mb[(k - 3 * C) * L + t0 + t];
    }
    A1[t * lda + k] = to16<BF16>(v);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int r0 = 16 * (warp & 3), nb = 64 * (warp >> 2), ch0 = 32 * (warp >> 2);
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  mma_rows<BF16>(acc, A1 + r0 * lda, lda, p.w1h + (size_t)nb * K1p, K1p, K1p, lane);
  // gate: z = sigmoid(gate + b) tanh(filter + b); accumulator element e is row r0 + g + 8 (e >> 1), column 2 q + (e & 1)
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = 8 * j + 2 * q + (e & 1), c = ch0 + col, bc = (c >> 3) * 16 + (c & 7);   // b1 in dw_pack order
      const float z = __fmul_rn(sigmoidf_(__fadd_rn(acc[j][e], p.b1[bc])), tanhf(__fadd_rn(acc[j + 4][e], p.b1[bc + 8])));
      Z[(r0 + g + 8 * (e >> 1)) * ldz + c] = to16<BF16>(z);
    }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  mma_rows<BF16>(acc, Z + r0 * ldz, ldz, p.w2h + (size_t)nb * C, C, C, lane);
  float* xo = p.x_out + (int64_t)b * C * L;
  float* sk = p.skip + (int64_t)b * C * L;
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = 8 * j + 2 * q + (e & 1), c = ch0 + col, bc = (c >> 3) * 16 + (c & 7);
      const int64_t t = t0 + r0 + g + 8 * (e >> 1);
      if (t >= L) continue;
      const int64_t o = c * L + t;
      xo[o] = __fdiv_rn(__fadd_rn(xb[o], __fadd_rn(acc[j][e], p.b2[bc])), 1.41421356237309515f);
      const float s = __fadd_rn(acc[j + 4][e], p.b2[bc + 8]);
      sk[o] = p.first ? s : __fadd_rn(s, sk[o]);
    }
}

// Finalize, tensor-core images: column n of the packed order (see dw_layer_tc_kernel) as a K-contiguous row.
__global__ void dw_pack_tc_kernel(const DwPackParams p) {
  constexpr int C = DW_C, C2 = 2 * DW_C;
  const int K1p = 3 * C + (p.n_mel + 15) / 16 * 16;
  // n = 64 h + 8 j + r: j < 4 -> first-half channel 32 h + 8 j + r, j >= 4 -> second-half channel of 32 h + 8 (j - 4) + r
  auto src = [](int n) { const int h = n / 64, j = (n % 64) / 8, r = n % 8; return j < 4 ? 32 * h + 8 * j + r : C + 32 * h + 8 * (j - 4) + r; };
  const int n1 = C2 * K1p, n2 = C2 * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += gridDim.x * blockDim.x) {
    float v;
    if (i < n1) {
      const int n = i / K1p, k = i % K1p, o = src(n);
      v = k < 3 * C ? p.wdil[(o * C + k % C) * 3 + k / C] : (k - 3 * C < p.n_mel ? p.wcond[o * p.n_mel + k - 3 * C] : 0.f);
    } else {
      const int n = (i - n1) / C, k = (i - n1) % C;
      v = p.wout[src(n) * C + k];
    }
    const uint16_t h = p.bf16 ? to16<true>(v) : to16<false>(v);
    (i < n1 ? p.w1h[i] : p.w2h[i - n1]) = h;
  }
}

int grid_for(int64_t n, int threads) { return (int)std::min<int64_t>(ceil_div(n, threads), 148 * 32); }

}  // namespace

size_t dw_layer_smem_bytes(int n_mel, int precision) {
  if (precision != AB_PREC_FP32) return (size_t)DW_TT * (dw_k1p(n_mel) + 8 + DW_C + 8) * sizeof(uint16_t);
  return (size_t)(4 * DW_C + n_mel) * DW_TT * sizeof(float);
}

int launch_dw_upsample(const DwUpsampleParams& p, cudaStream_t s) {
  dw_upsample_kernel<<<grid_for((int64_t)p.B * p.n_mel * p.F * p.f1 * p.f2, 256), 256, 0, s>>>(p);
  AB_LAUNCH_CHECK("dw_upsample_kernel");
  return AB_OK;
}

int launch_dw_embed(const DwEmbedParams& p, int steps, cudaStream_t s) {
  dw_embed_kernel<<<steps, 512, 0, s>>>(p);
  AB_LAUNCH_CHECK("dw_embed_kernel");
  return AB_OK;
}

int launch_dw_input(const float* audio, const float* w, const float* bias, float* x, int B, int64_t L, cudaStream_t s) {
  dw_input_kernel<<<grid_for((int64_t)B * DW_C * L, 256), 256, 0, s>>>(audio, w, bias, x, B, L);
  AB_LAUNCH_CHECK("dw_input_kernel");
  return AB_OK;
}

int launch_dw_layer(const DwLayerParams& p, cudaStream_t s) {
  static DeviceOnce once;
  if (once.need()) {
    AB_CUDA_TRY(cudaFuncSetAttribute(dw_layer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    AB_CUDA_TRY(cudaFuncSetAttribute(dw_layer_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    AB_CUDA_TRY(cudaFuncSetAttribute(dw_layer_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  const dim3 grid((unsigned)ceil_div(p.L, DW_TT), p.B);
  const size_t smem = dw_layer_smem_bytes(p.n_mel, p.precision);
  if (p.precision == AB_PREC_TC_BF16)
    dw_layer_tc_kernel<true><<<grid, 256, smem, s>>>(p);
  else if (p.precision == AB_PREC_TC_F16)
    dw_layer_tc_kernel<false><<<grid, 256, smem, s>>>(p);
  else
    dw_layer_kernel<<<grid, DW_LAYER_THREADS, smem, s>>>(p);
  AB_LAUNCH_CHECK("dw_layer_kernel");
  return AB_OK;
}

int launch_dw_tail(const DwTailParams& p, cudaStream_t s) {
  dw_tail_kernel<<<(unsigned)ceil_div((int64_t)p.B * p.L, 128), 128, 0, s>>>(p);
  AB_LAUNCH_CHECK("dw_tail_kernel");
  return AB_OK;
}

int launch_dw_pack(const DwPackParams& p, cudaStream_t s) {
  dw_pack_kernel<<<128, 256, 0, s>>>(p);
  AB_LAUNCH_CHECK("dw_pack_kernel");
  if (p.w1h) {
    dw_pack_tc_kernel<<<128, 256, 0, s>>>(p);
    AB_LAUNCH_CHECK("dw_pack_tc_kernel");
  }
  return AB_OK;
}

}  // namespace ab
