// wgmma implicit-GEMM convolutions (sm_90a): the ResBlock / AMPBlock convs, ConvTranspose1d, the non-square / wide
// Conv1d layers and Vocos' pointwise layers.
//
// Mapping (DESIGN.md §4):  D[row, n] += sum_{tap} A[row + shift(tap), ci] * W[tap][n, ci]
//   M = time rows, N = output channels (<= 256 per N block), K = C_in per tap.
//   Conv1d ("same", dilation d): row = output time, n = c_out, tap j reads row + j*d.
//   ConvTranspose1d (stride u, padding (k-u)/2, polyphase):
//     y[co, s*u - p + phi] = b[co] + sum_m sum_ci act(x)[ci, s - m] * W[ci, co, phi + u*m]
//     -> row = input time s, virtual channel n = co_local*u + phi, taps m = 0..ceil(k/u)-1; every MAC is useful.
//   Conv pair (one ResBlock1 step, hifigan.py:93-100): conv1 -> +b1, lrelu -> a shared-memory operand tile ->
//     conv2 -> +b2 + residual (+ branch sum, / num_kernels) in one launch; the intermediate never leaves the SM.
//
// Operands (ab_tc_ptx.cuh): fp16/bf16, K-major 8x16-byte core matrices without swizzle, so a tap is a row shift of
// the descriptor start and one activation tile serves all taps.
//   A: streamed in 32-channel chunks [4][rowsA][16 B]: lrelu + cvt of fp32 input in the loader, or a cp.async copy
//      of the 16-bit operand image the producing kernel left in HBM.
//   W: pre-packed in global memory in exactly the shared-memory image of one (N block, K chunk, tap) stage and
//      streamed with cp.async.bulk (TMA 1-D) through an mbarrier ring; thread 0 refills a stage once every warp
//      has released it.
//   D: fp32 in the registers of two consumer warpgroups (MT m64 tiles each); the epilogues run on the fragments.
// Kernels: hconv_kernel (one CTA per tile: conv and conv-transpose from fp32 input), and three persistent,
// warp-specialised kernels on one pipeline (Rings, Batches): hpair_kernel (conv pair), hchain_kernel (block mode) and
// hitem_kernel ((utterance, tile, N block) work items: conv-transpose from an operand image, Vocos' pointwise GEMM).
// They share the operand loader, the wgmma batch, the intermediate-tile and output epilogues and the shared-memory
// layout below; they differ in how they schedule them.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "ab_tc.cuh"
#include "ab_tc_ptx.cuh"
#include "ab_wgmma.cuh"

namespace ab {

using namespace tcx;

namespace {

constexpr int HC_WG = 2;                      // consumer warpgroups per CTA
constexpr int HC_THREADS = HC_WG * 128;
constexpr int HC_STAGES_MAX = 6;
constexpr int TC_MAX_C = 256;
constexpr uint32_t HC_SMEM_1CTA = 227 * 1024;  // N = 256: 128 accumulator registers per thread, one CTA per SM
constexpr uint32_t HC_SMEM_2CTA = 113 * 1024;  // N <= 128: two CTAs per SM overlap one's loads with the other's MMAs

// m64 tiles per warpgroup: at most 64 accumulator registers per thread below N = 256
__host__ __device__ constexpr int mt_of(int nw) { return nw >= 128 ? 1 : (nw == 64 ? 2 : 4); }

struct HcArgs {
  const float* x;          // fp32 input with element strides (used when ximg is null)
  int64_t xsb, xsc, xst;
  const uint16_t* ximg;    // operand image [B][c8n_in][Tin][8] of the already activated input, or null
  float pre_slope;
  int B, Cin, Cout;
  // conv s of the launch (a single conv: 0; pair: 0, 1; block mode: pair * nconv + conv): its weight image, stages in
  // (N block, K chunk, tap) order, and its bias (nullable)
  const void* ws[2 * AB_TC_CHAIN_MAX_PAIRS];
  const float* bs[2 * AB_TC_CHAIN_MAX_PAIRS];
  float* y;                // [B, Cout, Tout]
  const float* residual;   // nullable, [B, Cout, Tout]
  const float* acc_prev;   // nullable, may alias y
  int post_tanh;
  uint16_t* yimg;          // nullable: operand image of lrelu(y, img_slope), [B][c8n_out][Tout][8]
  float img_slope;
};

struct HcGeom {
  int mode;                // 0 conv, 1 conv-transpose (hconv_kernel; hitem_kernel from an operand image), 2 conv pair (hpair_kernel)
  int NB, cc;              // N blocks; output channels per block
  int R, V, tiles;         // rows per CTA tile, valid output rows per tile, tiles per sequence
  int ntaps, d;            // taps of every conv; the row step between the (first) conv's taps
  int a0, rowsA, nkc;      // time of A row 0 = tile origin - a0; rows of the A chunk; 32-channel chunks of C_in
  int h2, rowsI;           // pair mode: intermediate row 0 = origin - h2; its rows
  int c8n_in, c8n_out;
  int nstages;
  uint32_t stage_bytes, off_i, off_w, off_bias, off_bar, smem_bytes;
  int Tin, Tout, u, pad;
  float out_scale, mid_slope;
  int nsteps;              // convs of the launch: 1 single conv, 2 pair, npairs * nconv block mode
  // block mode: output row r is time origin - H + r, the operand tiles keep G guard rows on both sides so that every
  // tap shift is a non-negative row offset
  int nconv, H, G, rowsX;
  int dil[AB_TC_CHAIN_MAX_PAIRS];
  int nabuf;               // pair mode: A chunk buffers
};

// ------------------------------------------------------------------------------------------------ shared device code

// Accumulator fragment (m64nNk16, fp32) of consumer warpgroup cw: element [c*4 + 2h + e] of m64 tile mt is tile row
// row(mt, h) = 64 (cw MT + mt) + 16 wq + lane/4 + 8h and N-block column 8c + col + e, col = 2 (lane % 4).
template <int MT>
struct Frag {
  int row0, col;
  __device__ __forceinline__ explicit Frag(int cw)
      : row0(cw * MT * 64 + ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2)), col(2 * (threadIdx.x & 3)) {}
  __device__ __forceinline__ int row(int mt, int h) const { return row0 + mt * 64 + 8 * h; }
};

// Stage i of conv st's weight image; a launch streams its convs' images one after another.
__device__ __forceinline__ const uint8_t* weight_stage(const HcArgs& p, const HcGeom& g, int st, int i) {
  return static_cast<const uint8_t*>(p.ws[st]) + (size_t)i * g.stage_bytes;
}

// Biases of the launch's convs into shared memory, per_step per conv, zero beyond C_out.
__device__ __forceinline__ void stage_biases(float* bias_s, const HcArgs& p, int nsteps, int per_step, int tid,
                                             int nthreads) {
  for (int i = tid; i < nsteps * per_step; i += nthreads) {
    const int st = i / per_step, c = i - st * per_step;
    bias_s[i] = (p.bs[st] && c < p.Cout) ? __ldg(p.bs[st] + c) : 0.f;
  }
}

// Operand tile at `tile`: c8 planes [c8_0, c8_0 + nplanes) x rows [0, rows), row at time t0 + row, from the operand
// image or from lrelu(x, pre_slope); zero outside [0, Tin) and C_in.  Thread lt of nthreads cooperating threads.
// REFLECT: time t outside [0, Tin) reads row -t or 2 (Tin - 1) - t instead (ReflectionPad1d, MelGAN), zero where that
// row does not exist either (rows no valid output reads).
// STRIDED: the polyphase operand of a stride-s conv (make_geom mode 3): K chunk kc = c8_0 / 4 holds phase
// r = kc / ceil(C_in / 32) of the input channels [32 (kc mod ceil(C_in / 32)), + 32), and row tau is input time
// s tau + r - pad (s = g.u, pad = g.pad), so each row is gathered from its own input time.
template <int BF16, int REFLECT = 0, int STRIDED = 0>
__device__ __forceinline__ void load_tile(const HcArgs& p, const HcGeom& g, int b, uint8_t* tile, int c8_0, int nplanes,
                                          int rows, int t0, int lt, int nthreads) {
  const int items = nplanes * rows;
  int tmul = 1, toff = 0;
  if constexpr (STRIDED) {
    const int nkc_in = (p.Cin + 31) >> 5, r = (c8_0 >> 2) / nkc_in;
    c8_0 -= 4 * r * nkc_in;
    tmul = g.u;
    toff = r - g.pad;
  }
  auto time_of = [&](int row) {
    if constexpr (REFLECT) return reflect_time(t0 + row, g.Tin);
    else if constexpr (STRIDED) return tmul * (t0 + row) + toff;
    else return t0 + row;
  };
  if (p.ximg != nullptr) {
    const uint16_t* xb = p.ximg + (size_t)b * g.c8n_in * g.Tin * 8;
    for (int idx = lt; idx < items; idx += nthreads) {
      const int c = idx / rows, row = idx - c * rows;
      const int c8 = c8_0 + c, t = time_of(row);
      const bool ok = c8 < g.c8n_in && t >= 0 && t < g.Tin;
      cp_async16(smem_u32(tile) + unit_offset(rows, c, row),
                 ok ? (const void*)(xb + ((size_t)c8 * g.Tin + t) * 8) : (const void*)xb, ok ? 16u : 0u);
    }
    cp_async_wait_all();
  } else {
    const float* xb = p.x + (int64_t)b * p.xsb;
    for (int idx = lt; idx < items; idx += nthreads) {
      const int c = idx / rows, row = idx - c * rows;
      const int t = time_of(row);
      const bool ok = t >= 0 && t < g.Tin;
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int ci = (c8_0 + c) * 8 + e;
        v[e] = (ok && ci < p.Cin) ? lrelu(__ldg(xb + (int64_t)ci * p.xsc + (int64_t)t * p.xst), p.pre_slope) : 0.f;
      }
      uint4 q;
      q.x = pack2t<BF16>(v[0], v[1]);
      q.y = pack2t<BF16>(v[2], v[3]);
      q.z = pack2t<BF16>(v[4], v[5]);
      q.w = pack2t<BF16>(v[6], v[7]);
      *reinterpret_cast<uint4*>(tile + unit_offset(rows, c, row)) = q;
    }
  }
}

// One tap's wgmma batch over a 32-channel K chunk: acc[mt] (+)= A x W for both k16 halves, A rows starting at
// row0 + 64 mt of the operand at aBase (aRows rows per c8 plane), W the stage at wS.
template <int NW, int BF16, int MT>
__device__ __forceinline__ void mma_batch(float (&acc)[MT][NW / 2], uint32_t aBase, int aRows, int row0, uint32_t wS,
                                          bool first) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const uint32_t a = aBase + (uint32_t)(2 * ks * aRows + row0 + mt * 64) * 16u;
      const uint32_t w = wS + (uint32_t)(2 * ks * NW) * 16u;
      Wgmma<NW, BF16>::mma(acc[mt], make_desc(a, (uint32_t)aRows), make_desc(w, (uint32_t)NW), (first && ks == 0) ? 0 : 1);
    }
  }
}

// Intermediate tile: lrelu(v [+ bias], slope) of the fragment -> the 16-bit operand tile at `tile` (rows per c8
// plane), fragment row r to tile row r + roff; zero where time t0 + r is outside [0, T).  Planes >= nplanes are not
// written.
template <int NW, int BF16, int MT>
__device__ __forceinline__ void store_frag_tile(uint8_t* tile, const float (&v)[MT][NW / 2], const float* bias,
                                                const Frag<MT>& f, int rows, int roff, int t0, int T, int nplanes,
                                                float slope) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = f.row(mt, h), t = t0 + row;
      const bool ok = t >= 0 && t < T;
#pragma unroll
      for (int c = 0; c < NW / 8; ++c) {
        if (c >= nplanes) continue;
        const int col = c * 8 + f.col;
        float a0 = v[mt][c * 4 + 2 * h], a1 = v[mt][c * 4 + 2 * h + 1];
        if (bias) {
          a0 += bias[col];
          a1 += bias[col + 1];
        }
        const uint32_t q = ok ? pack2t<BF16>(lrelu(a0, slope), lrelu(a1, slope)) : 0u;
        *reinterpret_cast<uint32_t*>(tile + unit_offset(rows, c, row + roff) + 2 * f.col) = q;
      }
    }
}

// What epilogue_out reads from HBM and applies; a term that is not compiled in is either never set by the kernel's
// launches (block mode: residual, tanh) or already part of val (the residual and branch sum that hpair_kernel and
// hchain_kernel fold in with add_terms).
enum : int { EP_RESIDUAL = 1, EP_ACC_PREV = 2, EP_TANH = 4, EP_ALL = 7 };

// Output epilogue on fragment rows [r0, r1) at times t0 + row < Tout, output channels co0 + column < C_out:
//   y = ((val + residual) + acc_prev) * out_scale [tanh] ; yimg = cvt(lrelu(y, img_slope))
// where val(mt, c, h, e) is the value of accumulator element [mt][c*4 + 2h + e] before the epilogue.  EP selects the
// terms that are compiled in.
template <int NW, int BF16, int EP, int MT, class Val>
__device__ __forceinline__ void epilogue_out(const HcArgs& p, const HcGeom& g, const Frag<MT>& f, int b, int t0, int r0,
                                             int r1, int co0, Val val) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = f.row(mt, h), t = t0 + row;
      if (row < r0 || row >= r1 || t >= g.Tout) continue;
#pragma unroll
      for (int c = 0; c < NW / 8; ++c) {
        const int co = co0 + c * 8 + f.col;
        float ve[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          ve[e] = 0.f;
          if (co + e < p.Cout) {
            const int64_t idx = ((int64_t)b * p.Cout + co + e) * g.Tout + t;
            float v = val(mt, c, h, e);
            if ((EP & EP_RESIDUAL) && p.residual) v += __ldg(p.residual + idx);
            if ((EP & EP_ACC_PREV) && p.acc_prev) v += p.acc_prev[idx];
            v *= g.out_scale;
            if ((EP & EP_TANH) && p.post_tanh) v = tanhf(v);
            p.y[idx] = v;
            ve[e] = v;
          }
        }
        if (p.yimg != nullptr && (co >> 3) < g.c8n_out)
          *reinterpret_cast<uint32_t*>(p.yimg + (((size_t)b * g.c8n_out + (co >> 3)) * g.Tout + t) * 8 + (co & 7)) =
              pack2t<BF16>(lrelu(ve[0], p.img_slope), lrelu(ve[1], p.img_slope));
      }
    }
  }
}

// The additive terms of epilogue_out folded into the accumulators first, in its association:
//   acc = ((acc [+ bias]) [+ residual]) [+ acc_prev]     (each term when its pointer is non-null)
// on the valid fragment rows [r0, r1) at time t0 + row (pair mode: [0, V) at O + row; block mode: [H, H + V) at
// O - H + row) and output channels co0 + column.  The loads of both terms go out G fragment columns at a time, so that
// a group waits for one HBM round trip: read inside epilogue_out, between its fp32 stores (which may alias acc_prev),
// every element would wait for its own.  epilogue_out then runs without EP_RESIDUAL / EP_ACC_PREV on the accumulators.
template <int NW, int MT>
__device__ __forceinline__ void add_terms(float (&acc)[MT][NW / 2], const Frag<MT>& f, const float* bias,
                                          const float* residual, const float* acc_prev, const HcArgs& p,
                                          const HcGeom& g, int b, int t0, int r0, int r1, int co0) {
  static_assert(MT * NW / 2 <= 64, "add_terms: 64 accumulators per thread at most");
  constexpr int G = NW / 8 < 8 ? NW / 8 : 8;   // columns per group
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = f.row(mt, h), t = t0 + row;
      const bool ok = (unsigned)(row - r0) < (unsigned)(r1 - r0) && t < g.Tout;
      const int64_t base = ((int64_t)b * p.Cout + co0 + f.col) * g.Tout + t;   // element of column f.col
#pragma unroll
      for (int c0 = 0; c0 < NW / 8; c0 += G) {
        float r[G][2], a[G][2];
#pragma unroll
        for (int c = 0; c < G; ++c)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = co0 + (c0 + c) * 8 + f.col + e;
            const bool in = ok && co < p.Cout;
            const int64_t idx = base + (int64_t)((c0 + c) * 8 + e) * g.Tout;
            r[c][e] = in && residual ? __ldg(residual + idx) : 0.f;
            a[c][e] = in && acc_prev ? acc_prev[idx] : 0.f;
          }
#pragma unroll
        for (int c = 0; c < G; ++c)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = acc[mt][(c0 + c) * 4 + 2 * h + e];
            if (bias) v += bias[(c0 + c) * 8 + f.col + e];
            if (residual) v += r[c][e];
            if (acc_prev) v += a[c][e];
          }
      }
    }
}

// ------------------------------------------------------------------------------------------------ kernels

// modes 0 (conv) and 1 (conv-transpose from fp32 input); launch_hconv runs conv-transpose from an operand image on
// hitem_kernel, pair mode (2) on hpair_kernel, and block mode runs on hchain_kernel.  The mode-2 branch below is no longer launched but stays: without it ptxas (nvcc 12.9, build.py's
// flags) reports spill stores / loads of 956 / 1220 bytes at N = 256 and 784 / 1020 at N = 128, against 4 / 4 and
// 16 / 20 with it, which made HiFi-GAN V1's ConvTranspose layers about 5 ms per step slower (H100 80GB HBM3, 400 W
// power limit).  Re-check those numbers before deleting it.
// REFLECT (mode 0 only): ReflectionPad1d in place of the zero "same" padding (MelGAN's conv_pre and ResnetBlock conv).
// STRIDED (mode 0 only): the stride-s conv as a stride-1 conv over the polyphase operand (load_tile, make_geom mode 3).
template <int NW, int BF16, int REFLECT = 0, int STRIDED = 0>
__global__ void __launch_bounds__(HC_THREADS, NW >= 256 ? 1 : 2) hconv_kernel(HcArgs p, HcGeom g) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const int b = blockIdx.x / g.tiles, tile = blockIdx.x - b * g.tiles;
  const int O = tile * g.V;   // output time (conv) / input time (conv-transpose) of row 0
  const uint32_t sA = smem_u32(smem), sI = sA + g.off_i, sW = sA + g.off_w;
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const uint32_t bar0 = smem_u32(smem + g.off_bar);
  auto bar_full = [&](int s) { return bar0 + 8u * s; };
  auto bar_empty = [&](int s) { return bar0 + 8u * (HC_STAGES_MAX + s); };

  const int per_step = g.NB * g.nkc * g.ntaps;
  const int total = g.nsteps * per_step;
  // stage j of the launch's stream: at most two convs (pair mode), so the conv is one comparison on the per-tap path
  auto stage_src = [&](int j) {
    const int st = j >= per_step;
    return weight_stage(p, g, st, j - st * per_step);
  };

  if (tid == 0) {
    for (int s = 0; s < g.nstages; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), HC_THREADS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  stage_biases(bias_s, p, g.nsteps, g.NB * NW, tid, HC_THREADS);
  if (g.mode == 2) {   // channels of the intermediate beyond the accumulator width stay zero
    const int n16 = g.nkc * 4 * g.rowsI;
    for (int i = tid; i < n16; i += HC_THREADS) *reinterpret_cast<uint4*>(smem + g.off_i + (size_t)i * 16) = make_uint4(0, 0, 0, 0);
  }
  __syncthreads();
  if (tid == 0) {
    for (int s = 0; s < g.nstages && s < total; ++s) {
      mbar_arrive_expect_tx(bar_full(s), g.stage_bytes);
      bulk_g2s(sW + (uint32_t)s * g.stage_bytes, stage_src(s), g.stage_bytes, bar_full(s));
    }
  }

  float acc[MT][NACC];
  int it = 0;

  // the taps of one 32-channel K chunk over the A operand at aBase (aRows rows per c8 plane)
  auto mma_chunk = [&](uint32_t aBase, int aRows, int ntaps, int tapstep, bool reversed, bool& first) {
    for (int j = 0; j < ntaps; ++j, ++it) {
      const int s = it % g.nstages;
      const uint32_t ph = (uint32_t)(it / g.nstages) & 1u;
      mbar_wait(bar_full(s), ph);
      const int shift = reversed ? (ntaps - 1 - j) : j * tapstep;
      const uint32_t wS = sW + (uint32_t)s * g.stage_bytes;
      wg_fence();
      mma_batch<NW, BF16>(acc, aBase, aRows, wg * MT * 64 + shift, wS, first);
      wg_commit();
      wg_wait<0>();
      first = false;
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty(s));
      if (tid == 0 && it + g.nstages < total) {
        mbar_wait(bar_empty(s), ph);
        mbar_arrive_expect_tx(bar_full(s), g.stage_bytes);
        bulk_g2s(wS, stage_src(it + g.nstages), g.stage_bytes, bar_full(s));
      }
    }
  };

  // A chunk kc: rows [0, rowsA) at times O - a0 + row, channels [32 kc, 32 kc + 32)
  auto load_chunk = [&](int kc) {
    __syncthreads();   // every warp has finished the MMAs that read the previous chunk
    load_tile<BF16, REFLECT, STRIDED>(p, g, b, smem, 4 * kc, 4, g.rowsA, O - g.a0, tid, HC_THREADS);
    fence_proxy_async();
    __syncthreads();
  };

  // y = ((acc + bias) + residual + acc_prev) * out_scale [tanh] on the valid rows [0, V).  The fragment coordinates
  // are built where they are used: kept live across the MMA loops, they make ptxas spill more.
  auto epilogue_conv = [&](int nb, const float* bias_blk) {
    const Frag<MT> f(wg);
    epilogue_out<NW, BF16, EP_ALL>(p, g, f, b, O, 0, g.V, nb * NW, [&](int mt, int c, int h, int e) {
      return acc[mt][c * 4 + 2 * h + e] + bias_blk[c * 8 + f.col + e];
    });
  };

  if (g.mode != 2) {
    for (int nb = 0; nb < g.NB; ++nb) {
      bool first = true;
      for (int kc = 0; kc < g.nkc; ++kc) {
        load_chunk(kc);
        mma_chunk(sA, g.rowsA, g.ntaps, g.d, g.mode == 1, first);
      }
      if (g.mode == 0) {
        epilogue_conv(nb, bias_s + nb * NW);
      } else {
        // conv-transpose: column n = cl*u + phi of input time s is y[nb*cc + cl, s*u - pad + phi]
        const Frag<MT> f(wg);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int s = O + f.row(mt, h);
#pragma unroll
            for (int c = 0; c < NW / 8; ++c) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int n = c * 8 + f.col + e;
                const int cl = n / g.u, phi = n - cl * g.u, co = nb * g.cc + cl;
                const int t = s * g.u - g.pad + phi;
                if (cl >= g.cc || co >= p.Cout || t < 0 || t >= g.Tout) continue;
                const float v = acc[mt][c * 4 + 2 * h + e] + bias_s[co];
                p.y[((int64_t)b * p.Cout + co) * g.Tout + t] = v;
                if (p.yimg != nullptr)
                  p.yimg[(((size_t)b * g.c8n_out + (co >> 3)) * g.Tout + t) * 8 + (co & 7)] =
                      (uint16_t)(pack2t<BF16>(lrelu(v, p.img_slope), 0.f) & 0xffffu);
              }
            }
          }
        }
      }
    }
  } else {
    bool first = true;
    for (int kc = 0; kc < g.nkc; ++kc) {
      load_chunk(kc);
      mma_chunk(sA, g.rowsA, g.ntaps, g.d, false, first);
    }
    // intermediate = lrelu(conv1 + b1, mid_slope) -> shared-memory operand tile, zero outside [0, T)
    store_frag_tile<NW, BF16>(smem + g.off_i, acc, bias_s, Frag<MT>(wg), g.rowsI, 0, O - g.h2, g.Tin, 4 * g.nkc, g.mid_slope);
    fence_proxy_async();
    __syncthreads();
    first = true;
    for (int kc = 0; kc < g.nkc; ++kc)
      mma_chunk(sI + (uint32_t)(kc * 4 * g.rowsI) * 16u, g.rowsI, g.ntaps, 1, false, first);
    epilogue_conv(0, bias_s + NW);
  }
}

// ------------------------------------------------------------------------------------------------ persistent pipeline
// hchain_kernel, hpair_kernel and hitem_kernel are warp-specialised and persistent: one CTA of three warpgroups per SM
// walks the work items with a static stride, and all three run the pipeline below.
//   warpgroup 0 (producer, setmaxnreg 40): thread 0 streams each item's weight stages through the W ring, running ahead
//     across items (Rings::stream_weights); warps 1-3 load each item's A operand through the A ring as soon as the
//     consumers release a buffer (Rings::load_item), so the next item's loads run under this item's epilogue.
//   warpgroups 1-2 (consumers, setmaxnreg 232): one wgmma batch per tap with up to D batches left in flight; a W slot,
//     and an A buffer after the last tap that reads it, is released once the batch that read it has completed
//     (Batches).  Consumer-only synchronisation is a named barrier.
constexpr int HB_THREADS = 3 * 128;
constexpr int HB_LOADERS = 96;
constexpr int HB_PRODUCER_REGS = 40;
constexpr int HB_CONSUMER_REGS = 232;
static_assert(128 * HB_PRODUCER_REGS + 256 * HB_CONSUMER_REGS <= 65536, "setmaxnreg split of the register file");
// A chunk buffers of hpair_kernel and hitem_kernel: as many as fit (one for very wide tap reach)
constexpr int HP_ABUF_MAX = 3;

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Splits the register file between the roles: true in the producer warpgroup, false in the two consumer warpgroups.
__device__ __forceinline__ bool producer_warpgroup(int wg) {
  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HB_PRODUCER_REGS));
    return true;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HB_CONSUMER_REGS));
  return false;
}

// Position in a ring of n mbarrier slots: the slot, the parity of its current round, and whether the ring has wrapped
// (the producer waits for a slot's release from the second round on).  Counters instead of a division per tap.
struct RingPos {
  int s = 0;
  uint32_t ph = 0;
  bool wrapped = false;
  __device__ __forceinline__ void next(int n) {
    if (++s == n) {
      s = 0;
      ph ^= 1u;
      wrapped = true;
    }
  }
};

// The W ring (g.nstages weight stages at sW) and the A ring (nabuf <= AMAX operand buffers from shared-memory offset
// 0) and their mbarriers at bar0: W full / empty (HC_STAGES_MAX each), then A full / empty (AMAX each).  A full slot
// takes thread 0's expect_tx (W) or every loader thread's arrival (A); an empty slot one arrival per consumer warp (8:
// both consumer warpgroups read every slot).
template <int AMAX>
struct Rings {
  static constexpr uint32_t BAR_BYTES = 8u * (2 * HC_STAGES_MAX + 2 * AMAX);
  uint32_t bar0, sW;
  __device__ __forceinline__ uint32_t w_full(int s) const { return bar0 + 8u * s; }
  __device__ __forceinline__ uint32_t w_empty(int s) const { return bar0 + 8u * (HC_STAGES_MAX + s); }
  __device__ __forceinline__ uint32_t a_full(int s) const { return bar0 + 8u * (2 * HC_STAGES_MAX + s); }
  __device__ __forceinline__ uint32_t a_empty(int s) const { return bar0 + 8u * (2 * HC_STAGES_MAX + AMAX + s); }

  // thread 0, before the __syncthreads that precedes every use
  __device__ __forceinline__ void init(int nstages, int nabuf) const {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), 8);
    }
    for (int s = 0; s < nabuf; ++s) {
      mbar_init(a_full(s), HB_LOADERS);
      mbar_init(a_empty(s), 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  // thread 0: stages [i0, i0 + n) of conv st's weight image into the next W slots
  __device__ __forceinline__ void stream_weights(const HcArgs& p, const HcGeom& g, RingPos& r, int st, int i0,
                                                 int n) const {
    for (int i = 0; i < n; ++i, r.next(g.nstages)) {
      if (r.wrapped) mbar_wait(w_empty(r.s), r.ph ^ 1u);
      mbar_arrive_expect_tx(w_full(r.s), g.stage_bytes);
      bulk_g2s(sW + (uint32_t)r.s * g.stage_bytes, weight_stage(p, g, st, i0 + i), g.stage_bytes, w_full(r.s));
    }
  }

  // thread 0: columns [HW n, HW n + HW) of stages [0, nst) of conv st's weight image (HW = half its width) into the
  // next W slots, one copy per c8 plane, so that a half stage is the [4 c8][HW rows][8] stage of an N = HW wgmma.  Two
  // consecutive half stages share a slot (the last one alone when nst is odd), so the ring holds as many bytes and as
  // much MMA work ahead of the consumers as with whole stages.
  template <int HW>
  __device__ __forceinline__ void stream_weight_half(const HcArgs& p, const HcGeom& g, RingPos& r, int st, int n,
                                                     int nst) const {
    const uint32_t plane = g.stage_bytes / 4u, hbytes = HW * 16u;   // a c8 plane of the image's stage; HW of its rows
    for (int i = 0; i < nst; i += 2, r.next(g.nstages)) {
      const int m = min(2, nst - i);
      if (r.wrapped) mbar_wait(w_empty(r.s), r.ph ^ 1u);
      mbar_arrive_expect_tx(w_full(r.s), (uint32_t)m * 4u * hbytes);
      for (int j = 0; j < m; ++j) {
        const uint8_t* src = weight_stage(p, g, st, i + j) + n * hbytes;
        const uint32_t dst = sW + (uint32_t)r.s * g.stage_bytes + (uint32_t)j * 4u * hbytes;
#pragma unroll
        for (int c = 0; c < 4; ++c) bulk_g2s(dst + c * hbytes, src + c * plane, hbytes, w_full(r.s));
      }
    }
  }

  // loader warps (producer threads 32-127): one work item's A operand into the next nchunks A buffers, chunk kc holding
  // c8 planes [planes kc, planes (kc + 1)) x `rows` rows at times t0 + row of utterance b
  template <int BF16>
  __device__ __forceinline__ void load_item(const HcArgs& p, const HcGeom& g, RingPos& r, uint8_t* smem, int nabuf,
                                            int b, int t0, int nchunks, int planes, int rows) const {
    const uint32_t abytes = (uint32_t)(planes * rows) * 16u;
    for (int kc = 0; kc < nchunks; ++kc, r.next(nabuf)) {
      if (r.wrapped) mbar_wait(a_empty(r.s), r.ph ^ 1u);
      load_tile<BF16>(p, g, b, smem + r.s * abytes, planes * kc, planes, rows, t0, threadIdx.x - 32, HB_LOADERS);
      fence_proxy_async();
      mbar_arrive(a_full(r.s));
    }
  }
};

// keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
template <int MT, int NACC>
__device__ __forceinline__ void fence_acc(float (&acc)[MT][NACC]) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < NACC; ++i) asm volatile("" : "+f"(acc[mt][i])::"memory");
}

template <int MT, int NACC>
__device__ __forceinline__ void zero_acc(float (&acc)[MT][NACC]) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[mt][i] = 0.f;
}

// Consumer side of the rings: one wgmma batch per weight stage, in stream order.  After each batch is issued, at most D
// batches stay in flight, D - 1 when !deep (rings too small to leave a slot to fill next to the ones D batches hold).
// w[] / a[]: the W slot and the A buffer (-1: none) that the batches in flight read, oldest first; a batch holds its A
// buffer when it ran the last tap of the buffer's chunk.
template <int D, int AMAX>
struct Batches {
  static_assert(D == 1 || D == 2, "one or two wgmma batches in flight");
  const Rings<AMAX>& R;
  const HcGeom& g;
  const bool deep;
  RingPos wr;   // W slot of the next weight stage
  int w[D], a[D];

  __device__ __forceinline__ Batches(const Rings<AMAX>& rings, const HcGeom& geom, bool deep_)
      : R(rings), g(geom), deep(deep_) {
#pragma unroll
    for (int i = 0; i < D; ++i) w[i] = a[i] = -1;
  }

  __device__ __forceinline__ void release(int ws, int as) const {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
      if (ws >= 0) mbar_arrive(R.w_empty(ws));
      if (as >= 0) mbar_arrive(R.a_empty(as));
    }
  }

  // acc (+)= the next weight stage x the operand at aBase (aRows rows per c8 plane) from row row0; the batch holds A
  // buffer abuf (-1: none).  A slot may hold several stages (Rings::stream_weight_half): the stage at byte wofs of the
  // current slot, whose full barrier the batch at wofs = 0 waits for; the batch with slot_end moves to the next slot
  // and holds this one, so that it is released when the slot's last batch has completed.
  template <int NW, int BF16, int MT>
  __device__ __forceinline__ void mma(float (&acc)[MT][NW / 2], uint32_t aBase, int aRows, int row0, int abuf,
                                      bool& first, uint32_t wofs = 0, bool slot_end = true) {
    const int s = wr.s;
    if (wofs == 0) mbar_wait(R.w_full(s), wr.ph);
    if (slot_end) wr.next(g.nstages);
    fence_acc(acc);
    wg_fence();
    mma_batch<NW, BF16>(acc, aBase, aRows, row0, R.sW + (uint32_t)s * g.stage_bytes + wofs, first);
    wg_commit();
    if constexpr (D == 2) {
      if (deep) {
        wg_wait<2>();   // the batch before the previous one has completed: its W slot (and A buffer) can be refilled
        fence_acc(acc);
        release(w[0], a[0]);
        w[0] = w[1];
        a[0] = a[1];
      } else {
        wg_wait<1>();
        fence_acc(acc);
        release(w[1], a[1]);
      }
      w[1] = slot_end ? s : -1;
      a[1] = abuf;
    } else if (deep) {
      wg_wait<1>();   // the previous batch has completed
      fence_acc(acc);
      release(w[0], a[0]);
      w[0] = slot_end ? s : -1;
      a[0] = abuf;
    } else {
      wg_wait<0>();
      fence_acc(acc);
      release(slot_end ? s : -1, abuf);
    }
    first = false;
  }

  // the ntaps taps of one 32-channel K chunk, tap j from row row0 + j tapstep; the last one holds A buffer abuf
  template <int NW, int BF16, int MT>
  __device__ __forceinline__ void chunk(float (&acc)[MT][NW / 2], uint32_t aBase, int aRows, int row0, int ntaps,
                                        int tapstep, int abuf, bool& first) {
    for (int j = 0; j < ntaps; ++j)
      mma<NW, BF16>(acc, aBase, aRows, row0 + j * tapstep, j == ntaps - 1 ? abuf : -1, first);
  }

  // every batch has completed and released its slots
  template <int MT, int NACC>
  __device__ __forceinline__ void drain(float (&acc)[MT][NACC]) {
    wg_wait<0>();
    fence_acc(acc);
#pragma unroll
    for (int i = 0; i < D; ++i) {
      release(w[i], a[i]);
      w[i] = a[i] = -1;
    }
  }
};

// Block mode (launch_tc_chain): the work items are (utterance, time tile).  The A ring is a single buffer, the operand
// tile X of all channels, which the loaders refill for the next tile once the consumers have finished their last MMA
// on it.  Two wgmma batches in flight where the W ring leaves a slot to fill next to the two they hold.  The residual
// stream x_p of the whole ResBlock stays in registers in the accumulator fragment layout.
// The accumulation order of every output element is that of hconv_kernel's per-pair mode (K chunk -> tap -> k16).
template <int NW, int BF16>
__global__ void __launch_bounds__(HB_THREADS, 1) hchain_kernel(HcArgs p, HcGeom g) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t sX = smem_u32(smem), sI = sX + g.off_i;
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const Rings<1> R{smem_u32(smem + g.off_bar), sX + g.off_w};
  const int nwork = p.B * g.tiles;
  const int per_step = g.nkc * g.ntaps;

  if (tid == 0) R.init(g.nstages, 1);
  stage_biases(bias_s, p, g.nsteps, NW, tid, HB_THREADS);
  // rows and channels of the intermediate that no step writes stay zero for every tile
  for (int i = tid; i < g.nkc * 4 * g.rowsX; i += HB_THREADS)
    *reinterpret_cast<uint4*>(smem + g.off_i + (size_t)i * 16) = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  // ------------------------------------------------------------------------------------------------ producer
  if (producer_warpgroup(wg)) {
    RingPos r;
    if (tid == 0) {
      for (int w = blockIdx.x; w < nwork; w += gridDim.x)
        for (int st = 0; st < g.nsteps; ++st) R.stream_weights(p, g, r, st, 0, per_step);
    } else if (tid >= 32) {
      // X <- lrelu(x, pre_slope) over all channels, rows [0, rowsX) at times O - H - G + row
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        const int b = w / g.tiles;
        R.load_item<BF16>(p, g, r, smem, 1, b, (w - b * g.tiles) * g.V - g.H - g.G, 1, 4 * g.nkc, g.rowsX);
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  const int cw = wg - 1;
  const Frag<MT> f(cw);
  float acc[MT][NACC];
  Batches<2, 1> batches(R, g, g.nstages >= 3);

  int n = 0;
  for (int w = blockIdx.x; w < nwork; w += gridDim.x, ++n) {
    const int b = w / g.tiles, O = (w - b * g.tiles) * g.V;
    // residual stream in the fragment layout: xr = x at (row, column) of this thread's accumulators
    float xr[MT][NACC];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = O - g.H + f.row(mt, h);
#pragma unroll
        for (int c = 0; c < NW / 8; ++c)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = c * 8 + f.col + e;
            xr[mt][c * 4 + 2 * h + e] = (t >= 0 && t < g.Tin && co < p.Cout) ? __ldg(p.x + ((int64_t)b * p.Cout + co) * g.Tin + t) : 0.f;
          }
      }
    mbar_wait(R.a_full(0), (uint32_t)n & 1u);
    // lrelu(v [+ bb], mid_slope) of the fragment -> operand tile at off (rows offset by G)
    auto store_tile = [&](uint32_t off, const float (&v)[MT][NACC], const float* bb) {
      consumer_sync();   // both warpgroups have finished the MMAs that read the tile (ResBlock2 overwrites X)
      store_frag_tile<NW, BF16>(smem + off, v, bb, f, g.rowsX, g.G, O - g.H, g.Tin, 4 * g.nkc, g.mid_slope);
      fence_proxy_async();
      consumer_sync();
    };
    for (int st = 0; st < g.nsteps; ++st) {
      const int pr = st / g.nconv, cv = st - pr * g.nconv;
      const int d = cv == 0 ? g.dil[pr] : 1, hh = (g.ntaps - 1) * d / 2;
      const uint32_t aT = cv == 0 ? sX : sI;
      bool first = true;
      for (int kc = 0; kc < g.nkc; ++kc)
        batches.chunk<NW, BF16>(acc, aT + (uint32_t)(kc * 4 * g.rowsX + g.G - hh) * 16u, g.rowsX, cw * MT * 64,
                                g.ntaps, d, -1, first);
      batches.drain(acc);
      const float* bb = bias_s + st * NW;
      if (g.nconv == 2 && cv == 0) {
        store_tile(g.off_i, acc, bb);
      } else {
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int c = 0; c < NW / 8; ++c)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              float a = acc[mt][c * 4 + i] + bb[c * 8 + f.col + (i & 1)];
              a += xr[mt][c * 4 + i];
              xr[mt][c * 4 + i] = a;
            }
        if (st + 1 < g.nsteps) store_tile(0, xr, nullptr);
      }
    }
    // every MMA of this tile has completed: the producer may load the next X
    batches.release(-1, 0);
    // y = (x_L + acc_prev) * out_scale on the valid rows [H, H + V); acc_prev (which may alias y) is read in batches
    add_terms<NW>(xr, f, nullptr, nullptr, p.acc_prev, p, g, b, O - g.H, g.H, g.H + g.V, 0);
    epilogue_out<NW, BF16, 0>(p, g, f, b, O - g.H, g.H, g.H + g.V, 0,
                              [&](int mt, int c, int h, int e) { return xr[mt][c * 4 + 2 * h + e]; });
  }
}

// Pair mode (launch_tc_conv with a second conv; one ResBlock1 step): the work items are (utterance, time tile), with
// the per-pair tile geometry of make_geom (output row r at time O + r, V = R - (k - 1)).  The loaders stream the A
// operand in 32-channel K chunks through g.nabuf buffers; conv2 reads only the intermediate tile, so the next tile's
// chunks load under this tile's conv2 and output epilogue.
// conv2 runs in NH column halves of HW columns, one after the other: one half below N = 256, two of 128 at N = 256
// (C in (128, 256], so both hold output channels).  Each half holds at most 64 accumulators per thread, which leaves
// room for the residual of its fragment: each consumer loads it into registers before the half's MMAs (below N = 256
// at the start of the tile), so that HBM read runs under them.  The branch sum would need another 64 registers (ptxas
// spills) and is read after the MMAs by add_terms.  At N = 256 conv1 keeps its 128 accumulators, which are dead once
// the intermediate tile is stored, and a half's wgmmas are m64n128k16 on weight stages of the half's columns only
// (Rings::stream_weight_half).  Two of those 8 KB stages share a 16 KB slot of the W ring, so the ring, its layout and
// the bytes and MMA work it holds ahead of the consumers stay those of conv1 and of the other kernels.
// Accumulation order (K chunk -> tap -> k16, conv1 then conv2) and epilogue association are those of the per-pair
// arithmetic, so neither the tile shape nor the column halves enter any output element.
// Both consumer warpgroups work on every tile, warpgroup cw on its mt_of(N) m64 row tiles from row 64 mt_of(N) cw, and
// they meet at a named barrier on either side of the intermediate tile's store.
template <int NW, int BF16>
__global__ void __launch_bounds__(HB_THREADS, 1) hpair_kernel(HcArgs p, HcGeom g) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  constexpr int NH = NW > 128 ? 2 : 1, HW = NW / NH;   // conv2's column halves and their width
  static_assert(MT * HW / 2 <= 64, "a conv2 half leaves room for its prefetched residual");
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t sA = smem_u32(smem), sI = sA + g.off_i;
  const uint32_t abytes = (uint32_t)g.rowsA * 64u;   // one A chunk: 4 c8 planes x rowsA rows
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const Rings<HP_ABUF_MAX> R{smem_u32(smem + g.off_bar), sA + g.off_w};
  const int nwork = p.B * g.tiles;
  const int per_step = g.nkc * g.ntaps;

  if (tid == 0) R.init(g.nstages, g.nabuf);
  stage_biases(bias_s, p, 2, NW, tid, HB_THREADS);
  // rows and channels of the intermediate that store_frag_tile does not write stay zero for every tile
  for (int i = tid; i < g.nkc * 4 * g.rowsI; i += HB_THREADS)
    *reinterpret_cast<uint4*>(smem + g.off_i + (size_t)i * 16) = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  // ------------------------------------------------------------------------------------------------ producer
  if (producer_warpgroup(wg)) {
    RingPos r;
    if (tid == 0) {
      for (int w = blockIdx.x; w < nwork; w += gridDim.x)
        for (int st = 0; st < 2; ++st) {
          if (NH == 1 || st == 0) R.stream_weights(p, g, r, st, 0, per_step);
          else
            for (int n = 0; n < NH; ++n) R.stream_weight_half<HW>(p, g, r, st, n, per_step);
        }
    } else if (tid >= 32) {
      // A chunk kc of a tile: rows [0, rowsA) at times O - a0 + row, channels [32 kc, 32 kc + 32)
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        const int b = w / g.tiles;
        R.load_item<BF16>(p, g, r, smem, g.nabuf, b, (w - b * g.tiles) * g.V - g.a0, g.nkc, 4, g.rowsA);
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  const int cw = wg - 1;
  RingPos ar;   // A buffer of the next chunk
  // Two batches stay in flight when the rings allow it: every W slot held by an in-flight batch must leave one to fill
  // (nstages >= 3), and the loaders must not need the buffer of the last tap of the chunk before the previous one
  // (ntaps >= 2, or three buffers; one buffer is drained after every chunk).
  Batches<2, HP_ABUF_MAX> batches(R, g, g.nstages >= 3 && (g.ntaps >= 2 || g.nabuf != 2));

  for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int b = w / g.tiles, O = (w - b * g.tiles) * g.V;
    // conv1's and each conv2 half's accumulators start at zero, although their first batch does not read them: the
    // wgmma operands are read-write, so without a value here ptxas keeps the registers live from the kernel's entry,
    // next to the other array
    float acc[MT][NACC];
    zero_acc(acc);
    // residual of this thread's output elements in conv2's half n, in flight under the MMAs that follow
    float xres[MT][HW / 2];
    auto prefetch_residual = [&](int n) {
      const Frag<MT> f(cw);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = f.row(mt, h), t = O + row;
          const bool ok = row < g.V && t < g.Tout;
#pragma unroll
          for (int c = 0; c < HW / 8; ++c)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int co = n * HW + c * 8 + f.col + e;
              const bool in = ok && co < p.Cout && p.residual;
              xres[mt][c * 4 + 2 * h + e] = in ? __ldg(p.residual + ((int64_t)b * p.Cout + co) * g.Tout + t) : 0.f;
            }
        }
    };
    if constexpr (NH == 1) prefetch_residual(0);
    // conv1 over the A chunks
    bool first = true;
    for (int kc = 0; kc < g.nkc; ++kc) {
      const int abuf = ar.s;
      mbar_wait(R.a_full(abuf), ar.ph);
      ar.next(g.nabuf);
      batches.chunk<NW, BF16>(acc, sA + (uint32_t)abuf * abytes, g.rowsA, cw * MT * 64, g.ntaps, g.d, abuf, first);
      if (g.nabuf == 1) batches.drain(acc);   // the loaders refill the only buffer with the next chunk
    }
    batches.drain(acc);
    // intermediate = lrelu(conv1 + b1, mid_slope) -> operand tile, row 0 at time O - h2, zero outside [0, T)
    consumer_sync();   // both warpgroups have finished the previous tile's conv2, which read the intermediate
    store_frag_tile<NW, BF16>(smem + g.off_i, acc, bias_s, Frag<MT>(cw), g.rowsI, 0, O - g.h2, g.Tin, 4 * g.nkc,
                              g.mid_slope);
    fence_proxy_async();
    consumer_sync();
    // conv2, columns [HW n, HW n + HW) at a time
    for (int n = 0; n < NH; ++n) {
      if constexpr (NH > 1) prefetch_residual(n);
      float acc2[MT][HW / 2];
      zero_acc(acc2);
      first = true;
      // stage i = kc ntaps + tap; two half stages per W slot (Rings::stream_weight_half)
      for (int kc = 0; kc < g.nkc; ++kc)
        for (int j = 0; j < g.ntaps; ++j) {
          const int i = kc * g.ntaps + j, sub = NH > 1 ? i & 1 : 0;
          batches.mma<HW, BF16>(acc2, sI + (uint32_t)(kc * 4 * g.rowsI) * 16u, g.rowsI, cw * MT * 64 + j, -1, first,
                                (uint32_t)sub * HW * 64u, NH == 1 || sub == 1 || i == per_step - 1);
        }
      batches.drain(acc2);
      // y = ((acc2 + b2) + residual) + acc_prev) * out_scale [tanh] on the valid rows [0, V)
      const Frag<MT> f(cw);
      const float* b2 = bias_s + NW + n * HW;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int i = 0; i < HW / 2; ++i) {
          acc2[mt][i] += b2[(i >> 2) * 8 + f.col + (i & 1)];
          if (p.residual) acc2[mt][i] += xres[mt][i];
        }
      add_terms<HW>(acc2, f, nullptr, nullptr, p.acc_prev, p, g, b, O, 0, g.V, n * HW);
      epilogue_out<HW, BF16, EP_TANH>(p, g, f, b, O, 0, g.V, n * HW,
                                      [&](int mt, int c, int h, int e) { return acc2[mt][c * 4 + 2 * h + e]; });
    }
  }
}

// 16-bit halves: lo of a and lo of b (SEL_LO), hi of a and hi of b (SEL_HI)
constexpr uint32_t SEL_LO = 0x5410u, SEL_HI = 0x7632u;
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}

// Conv-transpose epilogue of one work item: column n = cl*u + phi of input time s = s0 + row is
//   y[co = co0 + cl, t = s*u - pad + phi] = acc + b[co] ;  yimg = cvt(lrelu(y, img_slope))
// for cl < cc, co < C_out, 0 <= t < T_out.  bias is indexed by co.  With n = 8c + col + e (Frag), U = u = 8, 4, 2 fixes
// cl and phi per fragment column at compile time:
//   U = 8: cl = c, phi = col + e.  The thread holds channels 8m..8m+7 at its two phases: image units need no exchange.
//   U = 4: cl = 2c + q/2 (q = lane % 4), phi = 2 (q % 2) + e.  Lanes q and q^2 hold the even and odd channels of the
//          same phases; one exchange of 4 values leaves each with all 8 channels of one phase.
//   U = 2: cl = 4c + q, phi = e.  The quad holds channels 16p..16p+15 at phases 0 and 1 for c = 4p..4p+3: a 4 x 4
//          transpose of packed channel pairs gives lane q the 8 channels of unit 2p + q/2 at phase q % 2.
// fp32 outputs go out as pairs of adjacent samples, 8-byte aligned: two phases of one row, or at u = 2 with odd pad the
// second phase of row s and the first of row s + 1 (a shuffle from the lane holding row s + 1).  U = 0 (other strides,
// or odd pad at u = 4 and 8) stores element by element; cl comes from a float reciprocal, exact for n < 256.
template <int NW, int BF16, int U, int MT>
__device__ __forceinline__ void epilogue_convt(const HcArgs& p, const HcGeom& g, const Frag<MT>& f,
                                               const float (&acc)[MT][NW / 2], const float* bias, int b, int s0,
                                               int co0) {
  const int lane = threadIdx.x & 31, q = lane & 3;
  const int Tout = g.Tout, u = U ? U : g.u;
  const int ccv = min(g.cc, p.Cout - co0);   // valid channels of this N block
  float* yb = p.y + (int64_t)b * p.Cout * Tout;
  uint16_t* ib = p.yimg ? p.yimg + (size_t)b * g.c8n_out * Tout * 8 : nullptr;
  const float sl = p.img_slope;
  auto val = [&](int mt, int c, int h, int e, int cl) { return acc[mt][c * 4 + 2 * h + e] + bias[co0 + cl]; };
  auto put_pair = [&](int cl, int t, float v0, float v1) {   // t even, T_out even
    if (t >= 0 && t < Tout) *reinterpret_cast<float2*>(yb + (int64_t)(co0 + cl) * Tout + t) = make_float2(v0, v1);
  };
  auto put_one = [&](int cl, int t, float v) {
    if (t >= 0 && t < Tout) yb[(int64_t)(co0 + cl) * Tout + t] = v;
  };
  auto put_unit = [&](int cl8, int t, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {   // channels cl8..cl8+7
    if (t >= 0 && t < Tout)
      *reinterpret_cast<uint4*>(ib + ((size_t)((co0 + cl8) >> 3) * Tout + t) * 8) = make_uint4(w0, w1, w2, w3);
  };
  auto img2 = [&](float a, float c) { return pack2t<BF16>(lrelu(a, sl), lrelu(c, sl)); };

  if constexpr (U == 0) {
    const float inv_u = 1.0f / (float)u;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int s = s0 + f.row(mt, h);
#pragma unroll
        for (int c = 0; c < NW / 8; ++c) {
          // opaque per column: the mapping is computed where it is used rather than kept live (ptxas spills)
          float iu = inv_u;
          asm volatile("" : "+f"(iu)::"memory");
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = c * 8 + f.col + e;
            const int cl = (int)(((float)n + 0.5f) * iu), t = s * u - g.pad + (n - cl * u);
            if (cl >= ccv || t < 0 || t >= Tout) continue;
            const float v = val(mt, c, h, e, cl);
            yb[(int64_t)(co0 + cl) * Tout + t] = v;
            if (ib) {
              const int co = co0 + cl;
              ib[((size_t)(co >> 3) * Tout + t) * 8 + (co & 7)] = (uint16_t)(img2(v, 0.f) & 0xffffu);
            }
          }
        }
      }
  } else if constexpr (U == 8) {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int tq = (s0 + f.row(mt, h)) * 8 - g.pad + 2 * q;   // t of phase 2q
#pragma unroll
        for (int c = 0; c < NW / 8; ++c)
          if (c < ccv) put_pair(c, tq, val(mt, c, h, 0, c), val(mt, c, h, 1, c));
        if (ib) {
#pragma unroll
          for (int m = 0; m < NW / 64; ++m) {
            if (8 * m >= ccv) continue;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              uint32_t w[4];
#pragma unroll
              for (int i = 0; i < 4; ++i)
                w[i] = img2(val(mt, 8 * m + 2 * i, h, e, 8 * m + 2 * i), val(mt, 8 * m + 2 * i + 1, h, e, 8 * m + 2 * i + 1));
              put_unit(8 * m, tq + e, w[0], w[1], w[2], w[3]);
            }
          }
        }
      }
  } else if constexpr (U == 4) {
    const int hq = q >> 1, ek = hq;   // channel parity; the phase of (q % 2) pair this lane keeps for the image
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int tq = (s0 + f.row(mt, h)) * 4 - g.pad + 2 * (q & 1);
#pragma unroll
        for (int c = 0; c < NW / 8; ++c) {
          const int cl = 2 * c + hq;
          if (cl < ccv) put_pair(cl, tq, val(mt, c, h, 0, cl), val(mt, c, h, 1, cl));
        }
        if (ib) {
#pragma unroll
          for (int m = 0; m < NW / 32; ++m) {
            if (8 * m >= ccv) continue;   // C_out % 16 == 0 with an image: all 8 channels or none
            float vk[4], vs[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int c = 4 * m + i, cl = 2 * c + hq;
              const float v0 = val(mt, c, h, 0, cl), v1 = val(mt, c, h, 1, cl);
              vk[i] = ek ? v1 : v0;
              vs[i] = ek ? v0 : v1;
            }
            const uint32_t k0 = img2(vk[0], vk[1]), k1 = img2(vk[2], vk[3]);
            const uint32_t r0 = __shfl_xor_sync(0xffffffffu, img2(vs[0], vs[1]), 2);
            const uint32_t r1 = __shfl_xor_sync(0xffffffffu, img2(vs[2], vs[3]), 2);
            const uint32_t e0 = hq ? r0 : k0, o0 = hq ? k0 : r0, e1 = hq ? r1 : k1, o1 = hq ? k1 : r1;
            put_unit(8 * m, tq + ek, prmt(e0, o0, SEL_LO), prmt(e0, o0, SEL_HI), prmt(e1, o1, SEL_LO), prmt(e1, o1, SEL_HI));
          }
        }
      }
  } else {
    static_assert(U == 2, "vector conv-transpose epilogue: u = 2, 4 or 8");
    const bool odd = g.pad & 1;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const int sA = s0 + f.row(mt, 0);   // row of h = 0; h = 1 is 8 rows later
#pragma unroll
      for (int c = 0; c < NW / 8; ++c) {
        const int cl = 4 * c + q;
        const float a00 = val(mt, c, 0, 0, cl), a01 = val(mt, c, 0, 1, cl);
        const float a10 = val(mt, c, 1, 0, cl), a11 = val(mt, c, 1, 1, cl);
        if (!odd) {
          if (cl < ccv) {
            put_pair(cl, sA * 2 - g.pad, a00, a01);
            put_pair(cl, (sA + 8) * 2 - g.pad, a10, a11);
          }
        } else {
          // phase 0 of the next row: row + 1 is lane + 4 at the same h, except row 7 -> row 8 (lane - 28, h = 1);
          // the warp's rows 0 (phase 0) and 15 (phase 1) have no partner in it
          int src = (lane + 4) & 31;
          asm volatile("" : "+r"(src)::"memory");   // one column at a time: scheduled all at once, they spill at N = 256
          const float x0 = __shfl_sync(0xffffffffu, a00, src), x1 = __shfl_sync(0xffffffffu, a10, src);
          if (cl < ccv) {
            const int t0 = sA * 2 - g.pad + 1, t1 = t0 + 16;
            put_pair(cl, t0, a01, lane < 28 ? x0 : x1);
            if (lane < 28) put_pair(cl, t1, a11, x1);
            else put_one(cl, t1, a11);
            if (lane < 4) put_one(cl, t0 - 1, a00);
          }
        }
      }
      if (ib) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int s = sA + 8 * h;
#pragma unroll
          for (int pp = 0; pp < NW / 32; ++pp) {
            if (16 * pp >= ccv) continue;   // C_out % 16 == 0 with an image: all 16 channels or none
            int cb = co0;   // one unit pair at a time, as above
            asm volatile("" : "+r"(cb)::"memory");
            // a[j]: channels (8m + q, 8m + 4 + q) of unit m = 2pp + j/2 at phase j % 2, for lane j of the quad
            uint32_t a[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int c = 4 * pp + 2 * (j >> 1);
              a[j] = img2(acc[mt][c * 4 + 2 * h + (j & 1)] + bias[cb + 4 * c + q],
                          acc[mt][c * 4 + 4 + 2 * h + (j & 1)] + bias[cb + 4 * c + 4 + q]);
            }
            // transpose over the quad: lane q ends with x[r] = a[q] of lane r
            const bool b1 = q & 2, b0 = q & 1;
            const uint32_t k0 = b1 ? a[2] : a[0], k1 = b1 ? a[3] : a[1];
            const uint32_t t0 = __shfl_xor_sync(0xffffffffu, b1 ? a[0] : a[2], 2);
            const uint32_t t1 = __shfl_xor_sync(0xffffffffu, b1 ? a[1] : a[3], 2);
            // k0 / t0: from lanes q and q^2 for lane (q & 2); k1 / t1: the same for lane (q & 2) | 1
            const uint32_t u0 = __shfl_xor_sync(0xffffffffu, b0 ? k0 : k1, 1);
            const uint32_t u1 = __shfl_xor_sync(0xffffffffu, b0 ? t0 : t1, 1);
            // y[i]: from lane q ^ i
            const uint32_t y0 = b0 ? k1 : k0, y1 = u0, y2 = b0 ? t1 : t0, y3 = u1;
            const uint32_t p0 = b1 ? y2 : y0, p1 = b1 ? y3 : y1, r0 = b1 ? y0 : y2, r1 = b1 ? y1 : y3;
            const uint32_t x0 = b0 ? p1 : p0, x1 = b0 ? p0 : p1, x2 = b0 ? r1 : r0, x3 = b0 ? r0 : r1;
            put_unit(16 * pp + 8 * (q >> 1), s * 2 - g.pad + (q & 1), prmt(x0, x1, SEL_LO), prmt(x2, x3, SEL_LO),
                     prmt(x0, x1, SEL_HI), prmt(x2, x3, SEL_HI));
          }
        }
      }
    }
  }
}

// Epilogues of Vocos' pointwise (1x1) GEMM D[t, n] = sum_ci A[t, ci] W[n, ci] (launch_tc_pointwise) on hitem_kernel,
// output channels co0 + column at time O + row:
//   PW_GELU:     yimg = cvt(gelu(acc + b))                           (pwconv1 + nn.GELU(), exact erf; (0.5 v) (1 + erff),
//                                                                     every step an explicit __f*_rn)
//   PW_GAMMA:    y = y + gamma * (acc + b), fp32 in place            (pwconv2, layer scale and residual, vocos.py:509-527)
//   PW_SPECTRUM: columns 2j, 2j + 1 hold bin j's log-magnitude and phase (launch_tc_pack_head_weight):
//                spec[b T + t][j] = min(exp(m), 1e2) (cos p, sin p)  (ISTFTHead, vocos.py:343-361)
//   PW_LINEAR:   y[b, t, co] = acc + b, fp32 time-major [B, T, C_out]  (nn.Linear after a VocosBackbone, RepCodec's
//                encoder and decoder): a thread's two adjacent columns are one 8-byte store, so a quad of threads
//                writes 32 contiguous bytes of a row; an odd C_out (or a y that is not 8-byte aligned) takes scalar
//                stores
// ITEM_CONVT selects hitem_kernel's ConvTranspose epilogue, epilogue_convt.
enum ItemEpi : int {
  PW_GELU = AB_PW_GELU, PW_GAMMA = AB_PW_GAMMA_RESIDUAL, PW_SPECTRUM = AB_PW_SPECTRUM, PW_LINEAR = AB_PW_LINEAR, ITEM_CONVT
};
struct PwArgs {
  const float* gamma;   // PW_GAMMA: [C_out]
  float2* spec;         // PW_SPECTRUM: [B*T][C_out / 2]
};

template <int NW, int BF16, int EPI, int MT>
__device__ __forceinline__ void epilogue_pw(const HcArgs& p, const HcGeom& g, const PwArgs& e, const Frag<MT>& f,
                                            const float (&acc)[MT][NW / 2], const float* bias_s, int b, int O, int co0) {
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = O + f.row(mt, h);
      if (t >= g.Tout) continue;
#pragma unroll
      for (int c = 0; c < NW / 8; ++c) {
        const int co = co0 + c * 8 + f.col;
        const float a0 = acc[mt][c * 4 + 2 * h], a1 = acc[mt][c * 4 + 2 * h + 1];
        if constexpr (EPI == PW_GELU) {
          if ((co >> 3) >= g.c8n_out) continue;
          float v[2] = {a0 + bias_s[co], a1 + bias_s[co + 1]};
#pragma unroll
          for (int q = 0; q < 2; ++q)
            v[q] = co + q < p.Cout
                       ? __fmul_rn(__fmul_rn(0.5f, v[q]), __fadd_rn(1.0f, erff(__fmul_rn(v[q], 0.70710678118654752440f))))
                       : 0.f;
          *reinterpret_cast<uint32_t*>(p.yimg + (((size_t)b * g.c8n_out + (co >> 3)) * g.Tout + t) * 8 + (co & 7)) =
              pack2t<BF16>(v[0], v[1]);
        } else if constexpr (EPI == PW_GAMMA) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            if (co + q >= p.Cout) continue;
            const float v = (q ? a1 : a0) + bias_s[co + q];
            float* y = p.y + ((int64_t)b * p.Cout + co + q) * g.Tout + t;
            *y = __fadd_rn(*y, __fmul_rn(__ldg(e.gamma + co + q), v));
          }
        } else if constexpr (EPI == PW_LINEAR) {
          if (co >= p.Cout) continue;
          float* y = p.y + ((int64_t)b * g.Tout + t) * p.Cout + co;
          const float v0 = a0 + bias_s[co], v1 = a1 + bias_s[co + 1];   // bias_s is zero beyond C_out
          if (!(p.Cout & 1) && !(reinterpret_cast<uintptr_t>(p.y) & 7)) {
            *reinterpret_cast<float2*>(y) = make_float2(v0, v1);
          } else {
            y[0] = v0;
            if (co + 1 < p.Cout) y[1] = v1;
          }
        } else {
          static_assert(EPI == PW_SPECTRUM, "pointwise epilogue");
          const int bins = p.Cout >> 1, j = co >> 1;
          if (j >= bins) continue;
          float amp = expf(a0 + bias_s[j]);
          amp = fminf(amp, 1e2f);
          float sn, cs;
          sincosf(a1 + bias_s[bins + j], &sn, &cs);
          e.spec[((int64_t)b * g.Tout + t) * bins + j] = make_float2(amp * cs, amp * sn);
        }
      }
    }
}

// The (utterance, time tile, N block) walk over an operand image: ConvTranspose1d from an image (launch_tc_conv mode 1
// with ximg, EPI = ITEM_CONVT) and Vocos' pointwise GEMM (EPI = PW_*; one tap, K = C_in and N = C_out unbounded).  The
// N block is fastest, so the NB items of a tile run at once on different SMs and read their A chunks from L2.  An item
// streams its A chunks through g.nabuf buffers and its N block's (K chunk, tap) weight stages.  The ConvTranspose
// keeps two wgmma batches in flight where the rings allow it (hpair_kernel's condition); the GEMM keeps one where both
// rings leave a slot to fill next to it, none otherwise.
// Accumulation order: K chunk -> tap m in the reversed row shift ntaps - 1 - m -> k16, then the bias.
template <int NW, int BF16, int EPI>
__global__ void __launch_bounds__(HB_THREADS, 1) hitem_kernel(HcArgs p, HcGeom g, PwArgs e) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  constexpr bool CONVT = EPI == ITEM_CONVT;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t sA = smem_u32(smem);
  const uint32_t abytes = (uint32_t)g.rowsA * 64u;   // one A chunk: 4 c8 planes x rowsA rows
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const Rings<HP_ABUF_MAX> R{smem_u32(smem + g.off_bar), sA + g.off_w};
  const int nwork = p.B * g.tiles * g.NB;
  const int ntaps = CONVT ? g.ntaps : 1;   // compile time for the GEMM: no tap loop in its chunk loop
  const int per_nb = g.nkc * ntaps;

  if (tid == 0) R.init(g.nstages, g.nabuf);
  stage_biases(bias_s, p, 1, g.NB * g.cc, tid, HB_THREADS);
  __syncthreads();

  // ------------------------------------------------------------------------------------------------ producer
  if (producer_warpgroup(wg)) {
    RingPos r;
    if (tid == 0) {
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) R.stream_weights(p, g, r, 0, (w % g.NB) * per_nb, per_nb);
    } else if (tid >= 32) {
      // A chunk kc of an item: rows [0, rowsA) at times O - a0 + row, channels [32 kc, 32 kc + 32)
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        const int bt = w / g.NB, b = bt / g.tiles;
        R.load_item<BF16>(p, g, r, smem, g.nabuf, b, (bt - b * g.tiles) * g.V - g.a0, g.nkc, 4, g.rowsA);
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  const int cw = wg - 1;
  float acc[MT][NACC];
  RingPos ar;   // A buffer of the next chunk
  Batches<CONVT ? 2 : 1, HP_ABUF_MAX> batches(
      R, g, CONVT ? g.nstages >= 3 && (g.ntaps >= 2 || g.nabuf != 2) : g.nstages >= 3 && g.nabuf >= 3);

  for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int bt = w / g.NB, nb = w - bt * g.NB, b = bt / g.tiles, O = (bt - b * g.tiles) * g.V;
    bool first = true;
    for (int kc = 0; kc < g.nkc; ++kc) {
      const int abuf = ar.s;
      mbar_wait(R.a_full(abuf), ar.ph);
      ar.next(g.nabuf);
      batches.chunk<NW, BF16>(acc, sA + (uint32_t)abuf * abytes, g.rowsA, cw * MT * 64 + ntaps - 1, ntaps, -1, abuf,
                              first);
      // the loaders refill the only buffer with the next chunk; the GEMM, never deep with one buffer, has released it
      if (CONVT && g.nabuf == 1) batches.drain(acc);
    }
    batches.drain(acc);
    const Frag<MT> f(cw);
    const int co0 = nb * g.cc;
    if constexpr (CONVT) {
      switch (g.pad & 1 ? (g.u == 2 ? 2 : 0) : g.u) {
        case 8: epilogue_convt<NW, BF16, 8>(p, g, f, acc, bias_s, b, O, co0); break;
        case 4: epilogue_convt<NW, BF16, 4>(p, g, f, acc, bias_s, b, O, co0); break;
        case 2: epilogue_convt<NW, BF16, 2>(p, g, f, acc, bias_s, b, O, co0); break;
        default: epilogue_convt<NW, BF16, 0>(p, g, f, acc, bias_s, b, O, co0); break;
      }
    } else {
      epilogue_pw<NW, BF16, EPI>(p, g, e, f, acc, bias_s, b, O, co0);
    }
  }
}

// ---------------------------------------------------------------------------
// weight images: stage (nb, kc, tap) = [4 c8][NW rows][8] — the A/B operand layout of ab_tc_ptx.cuh
// ---------------------------------------------------------------------------
struct HcLayer {
  int mode, NW, NB, cc, ntaps, nkc, u;
};

int rup(int x, int a) { return (x + a - 1) / a * a; }
int pow2_at_least(int x) {
  int n = 16;
  while (n < x) n <<= 1;
  return n;
}

// mode 0 conv (d_or_u = dilation), 1 conv-transpose (d_or_u = stride), 2 strided conv (d_or_u = stride s): a stride-1
// conv over s phases of the input, K chunk r * ceil(C_in / 32) + kc holding phase r, tap m holding kernel tap s m + r
int layer_geom(int mode, int cin, int cout, int k, int d_or_u, HcLayer& L) {
  if (cin <= 0 || cout <= 0 || k <= 0 || d_or_u <= 0) return fail(AB_ERR_ARG, "tc conv: bad layer shape");
  L.mode = mode;
  L.nkc = (cin + 31) / 32;
  if (mode == 2) {
    const int s = d_or_u;
    if (s > AB_TC_MAX_STRIDE) return fail(AB_ERR_UNSUPPORTED, "tc conv: stride %d > %d", s, AB_TC_MAX_STRIDE);
    if (k < s) return fail(AB_ERR_UNSUPPORTED, "tc conv: strided conv needs k >= stride (k %d, stride %d)", k, s);
    L.NW = std::min(256, pow2_at_least(rup(cout, 16)));
    L.NB = (cout + L.NW - 1) / L.NW;
    L.cc = L.NW;
    L.ntaps = (k + s - 1) / s;
    L.nkc *= s;
    L.u = s;
  } else if (mode == 0) {
    if (!(k & 1)) return fail(AB_ERR_UNSUPPORTED, "tc conv: conv kernel size must be odd");
    L.NW = std::min(256, pow2_at_least(rup(cout, 16)));
    L.NB = (cout + L.NW - 1) / L.NW;
    L.cc = L.NW;
    L.ntaps = k;
    L.u = 1;
  } else {
    const int u = d_or_u;
    if (k < u) return fail(AB_ERR_UNSUPPORTED, "tc conv: conv-transpose needs k >= stride");
    if (u > 64) return fail(AB_ERR_UNSUPPORTED, "tc conv: stride %d too large", u);
    L.cc = std::min(256 / u, cout);
    L.NW = pow2_at_least(L.cc * u);
    L.NB = (cout + L.cc - 1) / L.cc;
    L.ntaps = (k + u - 1) / u;
    L.u = u;
  }
  return AB_OK;
}

size_t layer_image_bytes(const HcLayer& L) { return (size_t)L.NB * L.nkc * L.ntaps * 64u * L.NW; }

__global__ void hc_pack_weight_kernel(const float* __restrict__ w_t, uint16_t* __restrict__ img, HcLayer L, int cin,
                                      int cout, int k, int bf16) {
  const int64_t total = (int64_t)L.NB * L.nkc * L.ntaps * 32 * L.NW;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(idx & 7);
    int64_t r = idx >> 3;
    const int n = (int)(r % L.NW);
    r /= L.NW;
    const int c8l = (int)(r & 3);
    r >>= 2;
    const int tap = (int)(r % L.ntaps);
    r /= L.ntaps;
    const int kc = (int)(r % L.nkc);
    const int nb = (int)(r / L.nkc);
    const int ci = kc * 32 + c8l * 8 + e;
    float v = 0.f;
    if (L.mode == 0) {
      const int co = nb * L.NW + n;
      if (ci < cin && co < cout) v = w_t[((int64_t)ci * k + tap) * cout + co];
    } else if (L.mode == 1) {
      const int cl = n / L.u, phi = n - cl * L.u, co = nb * L.cc + cl, j = phi + L.u * tap;
      if (ci < cin && cl < L.cc && co < cout && j < k) v = w_t[((int64_t)ci * k + j) * cout + co];
    } else {
      const int nkc_in = L.nkc / L.u, r = kc / nkc_in, cr = ci - 32 * r * nkc_in, co = nb * L.NW + n, j = L.u * tap + r;
      if (cr < cin && co < cout && j < k) v = w_t[((int64_t)cr * k + j) * cout + co];
    }
    img[idx] = (uint16_t)(pack2(v, 0.f, bf16) & 0xffffu);
  }
}

// Weight image of Vocos' iSTFT head for the PW_SPECTRUM epilogue (k = 1, conv layout): image column 2j holds output
// row j (log-magnitude of bin j), column 2j + 1 row bins + j (its phase), so one thread's accumulator pair is one bin.
__global__ void hc_pack_head_weight_kernel(const float* __restrict__ w_t, uint16_t* __restrict__ img, HcLayer L, int cin,
                                           int cout, int bf16) {
  const int64_t total = (int64_t)L.NB * L.nkc * 32 * L.NW;
  const int bins = cout >> 1;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(idx & 7);
    int64_t r = idx >> 3;
    const int n = (int)(r % L.NW);
    r /= L.NW;
    const int c8l = (int)(r & 3);
    r >>= 2;
    const int kc = (int)(r % L.nkc);
    const int nb = (int)(r / L.nkc);
    const int ci = kc * 32 + c8l * 8 + e, col = nb * L.NW + n, j = col >> 1;
    const int co = (col & 1) ? bins + j : j;
    const float v = (ci < cin && j < bins) ? w_t[(int64_t)ci * cout + co] : 0.f;
    img[idx] = (uint16_t)(pack2(v, 0.f, bf16) & 0xffffu);
  }
}

// Shared-memory layout of both kernels: the operand tile (abytes) at 0, the intermediate tile (ibytes) at off_i, then
// the W ring of as many stages as fit (at most HC_STAGES_MAX), nbias fp32 biases and bar_bytes of mbarriers.  Needs
// g.stage_bytes; false when two W stages do not fit in limit.
bool layout_smem(HcGeom& g, uint32_t abytes, uint32_t ibytes, uint32_t nbias, uint32_t bar_bytes, uint32_t limit) {
  g.off_i = (abytes + 127u) & ~127u;
  g.off_w = (g.off_i + ibytes + 127u) & ~127u;
  const uint32_t fixed = g.off_w + nbias * 4u + 16u + bar_bytes;
  if (fixed + 2u * g.stage_bytes > limit) return false;
  g.nstages = (int)std::min<uint32_t>((limit - fixed) / g.stage_bytes, HC_STAGES_MAX);
  g.off_bias = g.off_w + (uint32_t)g.nstages * g.stage_bytes;
  g.off_bar = (g.off_bias + nbias * 4u + 15u) & ~15u;
  g.smem_bytes = g.off_bar + bar_bytes;
  return true;
}

// Launch geometry.  mode 2 (pair): C_in = C_out = C <= 256, conv1 dilation d_or_u, conv2 dilation 1.  mode 1: padding
// pad (-1: (k - u) / 2), Tin * u outputs.  mode 3 (strided conv, stride d_or_u, padding pad): runs as mode 0 over the
// polyphase operand, output row t reading operand rows t .. t + ceil(k / s) - 1, (Tin + 2 pad - k) / s + 1 outputs.  persistent: for hpair_kernel or hitem_kernel (one CTA per SM, as many A
// chunk buffers as fit next to two W stages) rather than hconv_kernel.
int make_geom(int mode, int cin, int cout, int k, int d_or_u, int Tin, bool persistent, HcGeom& g, int pad = -1) {
  HcLayer L;
  int rc = layer_geom(mode == 2 ? 0 : mode == 3 ? 2 : mode, cin, cout, k, d_or_u, L);
  if (rc != AB_OK) return rc;
  if (mode == 2 && (cin != cout || L.NB != 1)) return fail(AB_ERR_UNSUPPORTED, "tc conv pair: C=%d not in [1,%d]", cin, TC_MAX_C);
  g.mode = mode == 3 ? 0 : mode;
  g.nsteps = mode == 2 ? 2 : 1;
  g.NB = L.NB;
  g.cc = L.cc;
  g.ntaps = L.ntaps;
  g.nkc = L.nkc;
  g.u = L.u;
  g.R = HC_WG * mt_of(L.NW) * 64;
  g.Tin = Tin;
  g.c8n_in = rup(cin, 16) / 8;
  g.c8n_out = rup(cout, 16) / 8;
  g.h2 = 0;
  g.rowsI = 0;
  int maxshift, rows_total;
  if (mode == 1) {
    g.d = 1;
    g.pad = pad < 0 ? (k - L.u) / 2 : pad;
    g.Tout = Tin * L.u;
    maxshift = g.ntaps - 1;
    g.a0 = maxshift;
    g.V = g.R;
    rows_total = (g.Tout - 1 + g.pad) / L.u + 1;
  } else if (mode == 3) {
    g.d = 1;
    g.pad = pad;
    g.Tout = (Tin + 2 * pad - k) / L.u + 1;
    maxshift = g.ntaps - 1;
    g.a0 = 0;
    g.V = g.R;
    rows_total = g.Tout;
  } else {
    g.d = d_or_u;
    g.pad = 0;
    g.Tout = Tin;
    maxshift = (k - 1) * d_or_u;
    g.a0 = maxshift / 2;
    g.V = g.R;
    rows_total = Tin;
    if (mode == 2) {
      g.h2 = (k - 1) / 2;
      g.a0 += g.h2;
      g.V = g.R - (k - 1);
      g.rowsI = rup(g.R + k - 1, 8);
    }
  }
  if (g.V < 8) return fail(AB_ERR_UNSUPPORTED, "tc conv: kernel size %d too large for a tile", k);
  g.rowsA = rup(g.R + maxshift, 8);
  if (g.rowsA > 16383 || g.rowsI > 16383) return fail(AB_ERR_UNSUPPORTED, "tc conv: tap reach %d too large", maxshift);
  g.tiles = (rows_total + g.V - 1) / g.V;
  g.stage_bytes = 64u * (uint32_t)L.NW;
  const uint32_t abytes = (uint32_t)g.rowsA * 64u, nbias = (uint32_t)(g.nsteps * g.NB * L.NW);
  bool fits;
  if (persistent) {
    const uint32_t ibytes = (uint32_t)g.nkc * 64u * (uint32_t)g.rowsI;
    g.nabuf = HP_ABUF_MAX;
    while (!(fits = layout_smem(g, (uint32_t)g.nabuf * abytes, ibytes, nbias, Rings<HP_ABUF_MAX>::BAR_BYTES,
                                HC_SMEM_1CTA)) && g.nabuf > 1)
      --g.nabuf;
  } else {
    g.nabuf = 1;
    fits = layout_smem(g, abytes, 0, nbias, 16u * HC_STAGES_MAX, L.NW >= 256 ? HC_SMEM_1CTA : HC_SMEM_2CTA);
  }
  if (!fits) return fail(AB_ERR_UNSUPPORTED, "tc conv: C=%d k=%d reach %d does not fit shared memory", cin, k, maxshift);
  g.out_scale = 1.0f;
  g.mid_slope = 1.0f;
  return AB_OK;
}

// Launches K<<<grid, threads, smem, s>>>(args...) after raising its dynamic shared-memory limit to `limit`, once per
// device and instantiation.
template <auto K, class... Args>
int launch_kernel(const char* name, unsigned grid, int threads, uint32_t limit, uint32_t smem, cudaStream_t s,
                  const Args&... args) {
  static DeviceOnce configured;
  if (configured.need()) AB_CUDA_TRY(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
  K<<<grid, threads, smem, s>>>(args...);
  AB_LAUNCH_CHECK(name);
  return AB_OK;
}

template <int V>
using IntC = std::integral_constant<int, V>;

// f(IntC<NW>(), IntC<BF16>()) for the N width of g and a tensor-core precision: the kernels' template arguments
template <class F>
int with_nw(const HcGeom& g, int precision, F f) {
  auto with_prec = [&](auto nw) { return precision == AB_PREC_TC_BF16 ? f(nw, IntC<1>()) : f(nw, IntC<0>()); };
  switch ((int)(g.stage_bytes / 64u)) {
    case 16: return with_prec(IntC<16>());
    case 32: return with_prec(IntC<32>());
    case 64: return with_prec(IntC<64>());
    case 128: return with_prec(IntC<128>());
    case 256: return with_prec(IntC<256>());
  }
  return fail(AB_ERR_UNSUPPORTED, "tc conv: N block %u", g.stage_bytes / 64u);
}

// Block-mode geometry: npairs x nconv convs of one ResBlock (C <= 128) with the halo recomputed inside the tile.
int make_chain_geom(int C, int k, const int* dil, int npairs, int nconv, int T, HcGeom& g) {
  if (npairs < 1 || npairs > AB_TC_CHAIN_MAX_PAIRS || (nconv != 1 && nconv != 2) || !tc_conv_supported(C, k))
    return fail(AB_ERR_UNSUPPORTED, "tc block: unsupported block");
  HcLayer L;
  int rc = layer_geom(0, C, C, k, 1, L);
  if (rc != AB_OK) return rc;
  if (L.NW > AB_TC_CHAIN_MAX_C) return fail(AB_ERR_UNSUPPORTED, "tc block: C=%d > %d", C, AB_TC_CHAIN_MAX_C);
  memset(&g, 0, sizeof(g));
  g.NB = 1; g.ntaps = k; g.nkc = L.nkc;
  g.nconv = nconv; g.nsteps = npairs * nconv;
  g.H = 0; g.G = 0;
  for (int q = 0; q < npairs; ++q) {
    if (dil[q] <= 0) return fail(AB_ERR_ARG, "tc block: dilation must be positive");
    g.dil[q] = dil[q];
    g.H += (k - 1) * dil[q] / 2 + (nconv == 2 ? (k - 1) / 2 : 0);
    g.G = std::max(g.G, (k - 1) * dil[q] / 2);
  }
  g.R = HC_WG * mt_of(L.NW) * 64;
  g.V = g.R - 2 * g.H;
  if (g.V < 8) return fail(AB_ERR_UNSUPPORTED, "tc block: halo %d too wide for %d rows", g.H, g.R);
  g.rowsX = rup(g.R + 2 * g.G, 8);
  if (g.rowsX > 16383) return fail(AB_ERR_UNSUPPORTED, "tc block: halo too wide");
  g.Tin = g.Tout = T;
  g.tiles = (T + g.V - 1) / g.V;
  g.c8n_in = g.c8n_out = rup(C, 16) / 8;
  g.stage_bytes = 64u * (uint32_t)L.NW;
  const uint32_t xbytes = (uint32_t)g.nkc * 64u * (uint32_t)g.rowsX;   // X and the intermediate tile
  // X is the A ring's only buffer
  if (!layout_smem(g, xbytes, xbytes, (uint32_t)(g.nsteps * L.NW), Rings<1>::BAR_BYTES, HC_SMEM_1CTA))
    return fail(AB_ERR_UNSUPPORTED, "tc block: does not fit shared memory");
  g.out_scale = 1.0f;
  g.mid_slope = 1.0f;
  return AB_OK;
}

// Grid of a persistent kernel: min(work items, SMs), the CTAs striding over the items.
int persistent_grid(int64_t work, const char* what, unsigned& grid) {
  if (work > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "%s: too many tiles", what);
  int dev = 0, sms = 0;
  AB_CUDA_TRY(cudaGetDevice(&dev));
  AB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  grid = (unsigned)std::min<int64_t>(work, sms);
  return AB_OK;
}

// One CTA of HB_THREADS per SM over `work` items: kernel(IntC<NW>(), IntC<BF16>()) names the instantiation for g's N
// width and the precision.
template <class Kernel, class... Args>
int launch_persistent(const char* name, const char* what, int64_t work, const HcGeom& g, int precision, cudaStream_t s,
                      Kernel kernel, const Args&... args) {
  unsigned grid = 0;
  const int rc = persistent_grid(work, what, grid);
  if (rc != AB_OK) return rc;
  return with_nw(g, precision, [&](auto nw, auto bf16) {
    constexpr auto K = kernel(nw, bf16);
    return launch_kernel<K>(name, grid, HB_THREADS, HC_SMEM_1CTA, g.smem_bytes, s, args...);
  });
}

// conv and conv-transpose from fp32 input on hconv_kernel (one CTA per tile); conv-transpose from an operand image
// on the persistent hitem_kernel, pair mode on the persistent hpair_kernel.  From fp32 input, hitem_kernel's 96 loader
// threads (8 scattered loads in flight each) cannot keep up with the MMAs and it is slower than hconv_kernel, whose
// 256 threads all load.
int launch_hconv(const HcArgs& a, const HcGeom& g, int precision, cudaStream_t s, bool reflect = false,
                 bool strided = false) {
  if (precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16) return fail(AB_ERR_ARG, "tc conv: bad precision");
  const int64_t work = (int64_t)a.B * g.tiles;
  if (g.mode == 1 && a.ximg)
    return launch_persistent("hitem_kernel", "tc conv-transpose", work * g.NB, g, precision, s, [](auto nw, auto bf16) {
      return hitem_kernel<decltype(nw)::value, decltype(bf16)::value, ITEM_CONVT>;
    }, a, g, PwArgs{});
  if (g.mode == 2)
    return launch_persistent("hpair_kernel", "tc conv pair", work, g, precision, s, [](auto nw, auto bf16) {
      return hpair_kernel<decltype(nw)::value, decltype(bf16)::value>;
    }, a, g);
  if (work > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "tc conv: grid too large");
  return with_nw(g, precision, [&](auto nw, auto bf16) {
    constexpr int NW = decltype(nw)::value;
    constexpr uint32_t limit = NW >= 256 ? HC_SMEM_1CTA : HC_SMEM_2CTA;
    if (reflect)
      return launch_kernel<hconv_kernel<NW, decltype(bf16)::value, 1>>("hconv_kernel", (unsigned)work, HC_THREADS, limit,
                                                                        g.smem_bytes, s, a, g);
    if (strided)
      return launch_kernel<hconv_kernel<NW, decltype(bf16)::value, 0, 1>>("hconv_kernel", (unsigned)work, HC_THREADS,
                                                                           limit, g.smem_bytes, s, a, g);
    return launch_kernel<hconv_kernel<NW, decltype(bf16)::value>>("hconv_kernel", (unsigned)work, HC_THREADS, limit,
                                                                   g.smem_bytes, s, a, g);
  });
}

HcArgs base_args(const float* x, int64_t xsb, int64_t xsc, int64_t xst, const uint16_t* ximg, float pre_slope, int B,
                 int cin, int cout) {
  HcArgs a;
  memset(&a, 0, sizeof(a));
  a.x = x; a.xsb = xsb; a.xsc = xsc; a.xst = xst; a.ximg = ximg; a.pre_slope = pre_slope;
  a.B = B; a.Cin = cin; a.Cout = cout; a.img_slope = 1.0f;
  return a;
}

}  // namespace

double tc_chain_recompute(int C, int k, const int* dil, int npairs, int nconv) {
  HcGeom g;
  if (make_chain_geom(C, k, dil, npairs, nconv, 1 << 20, g) != AB_OK) return 0.0;
  return (double)g.R / g.V;
}

int launch_tc_chain(const TcChainParams& p, cudaStream_t s) {
  if (!p.x || !p.y) return fail(AB_ERR_ARG, "tc block: null argument");
  if (p.B <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "tc block: bad shape");
  if (p.precision != AB_PREC_TC_F16 && p.precision != AB_PREC_TC_BF16) return fail(AB_ERR_ARG, "tc block: bad precision");
  HcGeom g;
  int rc = make_chain_geom(p.C, p.k, p.dil, p.npairs, p.nconv, p.T, g);
  if (rc != AB_OK) return rc;
  g.out_scale = 1.0f / p.out_div;
  g.mid_slope = p.slope;
  HcArgs a = base_args(p.x, (int64_t)p.C * p.T, p.T, 1, p.ximg, p.slope, p.B, p.C, p.C);
  for (int i = 0; i < g.nsteps; ++i) {
    if (!p.w[i]) return fail(AB_ERR_ARG, "tc block: null weight image");
    a.ws[i] = p.w[i];
    a.bs[i] = p.bias[i];
  }
  a.y = p.y; a.acc_prev = p.acc_prev; a.yimg = p.yimg; a.img_slope = p.img_slope;
  // make_chain_geom rejects N blocks wider than AB_TC_CHAIN_MAX_C: the clamp only keeps them from being compiled
  return launch_persistent("hchain_kernel", "tc block", (int64_t)a.B * g.tiles, g, p.precision, s, [](auto nw, auto bf16) {
    return hchain_kernel<std::min(decltype(nw)::value, AB_TC_CHAIN_MAX_C), decltype(bf16)::value>;
  }, a, g);
}

bool tc_conv_supported(int C, int k) { return C > 0 && C <= TC_MAX_C && (k & 1) && k <= 31; }

size_t tc_act_image_bytes(int64_t B, int C, int64_t T) { return (size_t)B * rup(C, 16) * (size_t)T * 2; }

size_t tc_weight_image_bytes(int mode, int cin, int cout, int k, int d_or_u) {
  HcLayer L;
  if (layer_geom(mode, cin, cout, k, d_or_u, L) != AB_OK) return 0;
  return layer_image_bytes(L);
}

int launch_tc_pack_weight(const float* w_t, void* image, int mode, int cin, int cout, int k, int d_or_u, int precision,
                          cudaStream_t s) {
  HcLayer L;
  int rc = layer_geom(mode, cin, cout, k, d_or_u, L);
  if (rc != AB_OK) return rc;
  const int64_t total = (int64_t)layer_image_bytes(L) / 2;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 132 * 8);
  hc_pack_weight_kernel<<<blocks, 256, 0, s>>>(w_t, static_cast<uint16_t*>(image), L, cin, cout, k,
                                               precision == AB_PREC_TC_BF16 ? 1 : 0);
  AB_LAUNCH_CHECK("hc_pack_weight_kernel");
  return AB_OK;
}

// The conv epilogue (epilogue_out) writes every time and every channel of the image's c8n_out planes, the padding
// channels as zero; the conv-transpose epilogue writes only c_out < C_out.
bool tc_can_emit_image(int mode, int cin, int cout, int k, int d_or_u) {
  HcLayer L;
  return layer_geom(mode, cin, cout, k, d_or_u, L) == AB_OK && (mode == 0 || (mode == 1 && (cout % 16) == 0));
}

int launch_tc_conv(const TcConvParams& p, cudaStream_t s) {
  const bool pair = p.w2 != nullptr;
  if ((!p.x && !p.ximg) || !p.y || !p.w) return fail(AB_ERR_ARG, "tc conv: null argument");
  if (p.B <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "tc conv: bad shape");
  if (p.mode < 0 || p.mode > 2) return fail(AB_ERR_ARG, "tc conv: mode must be 0 (conv), 1 (conv-transpose) or 2 (strided conv)");
  if (p.mode != 0 && (p.residual || p.acc_prev || p.out_div != 1.0f || p.post_tanh))
    return fail(AB_ERR_ARG, "tc conv: residual, acc_prev, out_div and tanh belong to mode 0");
  if (p.mode == 2) {
    if (pair || p.reflect || p.yimg) return fail(AB_ERR_ARG, "tc strided conv: no second conv, reflection or output image");
    if (p.d_or_u < 1 || p.d_or_u > AB_TC_MAX_STRIDE || p.k < p.d_or_u)
      return fail(AB_ERR_UNSUPPORTED, "tc strided conv: stride %d needs 1 <= stride <= %d and k = %d >= stride", p.d_or_u,
                  AB_TC_MAX_STRIDE, p.k);
    if (p.pad < 0 || p.pad >= p.k) return fail(AB_ERR_ARG, "tc strided conv: padding %d outside [0, k = %d)", p.pad, p.k);
    if ((int64_t)p.T + 2 * p.pad < p.k)
      return fail(AB_ERR_ARG, "tc strided conv: %d samples with padding %d are shorter than the kernel %d", p.T, p.pad, p.k);
  }
  if (pair && !(p.mode == 0 && p.Cin == p.Cout && tc_conv_supported(p.Cin, p.k)))
    return fail(AB_ERR_UNSUPPORTED, "tc conv pair: C_in=%d C_out=%d k=%d", p.Cin, p.Cout, p.k);
  if (p.mode == 1 && p.ximg && (p.Cin % 16) != 0)
    return fail(AB_ERR_UNSUPPORTED, "tc conv-transpose: operand-image input needs C_in %% 16 == 0");
  if (p.yimg && !tc_can_emit_image(p.mode, p.Cin, p.Cout, p.k, p.d_or_u))
    return fail(AB_ERR_UNSUPPORTED, "tc conv: cannot emit an operand image for this layer");
  if (p.mode == 1 && (p.pad < -1 || p.pad >= p.k))
    return fail(AB_ERR_ARG, "tc conv-transpose: padding %d outside [0, k = %d)", p.pad, p.k);
  if (p.reflect && (p.mode != 0 || pair))
    return fail(AB_ERR_UNSUPPORTED, "tc conv: reflection padding belongs to a single conv (mode 0)");
  HcGeom g;
  // pairs and ConvTranspose layers from an operand image run on the persistent kernels (launch_hconv)
  const bool persistent = pair || (p.mode == 1 && p.ximg);
  int rc = make_geom(pair ? 2 : p.mode == 2 ? 3 : p.mode, p.Cin, p.Cout, p.k, p.d_or_u, p.T, persistent, g, p.pad);
  if (rc != AB_OK) return rc;
  if (p.reflect && g.a0 >= p.T)
    return fail(AB_ERR_ARG, "tc conv: reflection padding %d needs more than %d samples", g.a0, p.T);
  g.out_scale = 1.0f / p.out_div;
  g.mid_slope = p.mid_slope;
  HcArgs a = base_args(p.x, p.xsb, p.xsc, p.xst, p.ximg, p.pre_slope, p.B, p.Cin, p.Cout);
  a.ws[0] = p.w; a.bs[0] = p.bias;
  a.ws[1] = p.w2; a.bs[1] = p.b2;
  a.y = p.y; a.residual = p.residual; a.acc_prev = p.acc_prev; a.post_tanh = p.post_tanh;
  a.yimg = p.yimg; a.img_slope = p.img_slope;
  return launch_hconv(a, g, p.precision, s, p.reflect != 0, p.mode == 2);
}


int launch_tc_pack_head_weight(const float* w_t, void* image, int cin, int cout, int precision, cudaStream_t s) {
  HcLayer L;
  int rc = layer_geom(0, cin, cout, 1, 1, L);
  if (rc != AB_OK) return rc;
  if (cout & 1) return fail(AB_ERR_ARG, "tc head weight: C_out %d must be even (magnitude and phase halves)", cout);
  const int64_t total = (int64_t)layer_image_bytes(L) / 2;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, 132 * 8);
  hc_pack_head_weight_kernel<<<blocks, 256, 0, s>>>(w_t, static_cast<uint16_t*>(image), L, cin, cout,
                                                    precision == AB_PREC_TC_BF16 ? 1 : 0);
  AB_LAUNCH_CHECK("hc_pack_head_weight_kernel");
  return AB_OK;
}

int launch_tc_pointwise(const TcPwParams& p, cudaStream_t s) {
  if (!p.ximg || !p.w || !p.bias) return fail(AB_ERR_ARG, "tc pointwise: null argument");
  if (p.B <= 0 || p.T <= 0 || p.Cin <= 0 || p.Cout <= 0) return fail(AB_ERR_ARG, "tc pointwise: bad shape");
  if (p.precision != AB_PREC_TC_F16 && p.precision != AB_PREC_TC_BF16) return fail(AB_ERR_ARG, "tc pointwise: bad precision");
  if ((p.epilogue == AB_PW_GELU && !p.yimg) || (p.epilogue == AB_PW_GAMMA_RESIDUAL && (!p.y || !p.gamma)) ||
      (p.epilogue == AB_PW_SPECTRUM && (!p.spec || (p.Cout & 1))) || (p.epilogue == AB_PW_LINEAR && !p.y))
    return fail(AB_ERR_ARG, "tc pointwise: epilogue %d: missing output or odd C_out", p.epilogue);
  HcGeom g;
  int rc = make_geom(0, p.Cin, p.Cout, 1, 1, p.T, true, g);   // k = 1 conv tiles
  if (rc != AB_OK) return rc;
  HcArgs a = base_args(nullptr, 0, 0, 0, p.ximg, 1.0f, p.B, p.Cin, p.Cout);
  a.ws[0] = p.w; a.bs[0] = p.bias;
  a.y = p.y; a.yimg = p.yimg;
  PwArgs e;
  e.gamma = p.gamma;
  e.spec = reinterpret_cast<float2*>(p.spec);
  auto run = [&](auto epi) {
    return launch_persistent("hitem_kernel", "tc pointwise", (int64_t)p.B * g.tiles * g.NB, g, p.precision, s,
                             [](auto nw, auto bf16) {
                               return hitem_kernel<decltype(nw)::value, decltype(bf16)::value, decltype(epi)::value>;
                             }, a, g, e);
  };
  switch (p.epilogue) {
    case AB_PW_GELU: return run(IntC<PW_GELU>());
    case AB_PW_GAMMA_RESIDUAL: return run(IntC<PW_GAMMA>());
    case AB_PW_SPECTRUM: return run(IntC<PW_SPECTRUM>());
    case AB_PW_LINEAR: return run(IntC<PW_LINEAR>());
  }
  return fail(AB_ERR_ARG, "tc pointwise: unknown epilogue %d", p.epilogue);
}

}  // namespace ab
