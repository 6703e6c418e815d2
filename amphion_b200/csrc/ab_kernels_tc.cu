// wgmma implicit-GEMM convolutions (sm_90a): the ResBlock / AMPBlock convs, ConvTranspose1d and the
// non-square / wide Conv1d layers.
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
// hconv_kernel (conv, conv-transpose), hpair_kernel (conv pair) and hchain_kernel (block mode) share the operand
// loader, the wgmma batch, the intermediate-tile and output epilogues and the shared-memory layout below; they differ in
// how they schedule them.
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
  int mode;                // 0 conv, 1 conv-transpose (hconv_kernel), 2 conv pair (hpair_kernel)
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
template <int BF16>
__device__ __forceinline__ void load_tile(const HcArgs& p, const HcGeom& g, int b, uint8_t* tile, int c8_0, int nplanes,
                                          int rows, int t0, int lt, int nthreads) {
  const int items = nplanes * rows;
  if (p.ximg != nullptr) {
    const uint16_t* xb = p.ximg + (size_t)b * g.c8n_in * g.Tin * 8;
    for (int idx = lt; idx < items; idx += nthreads) {
      const int c = idx / rows, row = idx - c * rows;
      const int c8 = c8_0 + c, t = t0 + row;
      const bool ok = c8 < g.c8n_in && t >= 0 && t < g.Tin;
      cp_async16(smem_u32(tile) + unit_offset(rows, c, row),
                 ok ? (const void*)(xb + ((size_t)c8 * g.Tin + t) * 8) : (const void*)xb, ok ? 16u : 0u);
    }
    cp_async_wait_all();
  } else {
    const float* xb = p.x + (int64_t)b * p.xsb;
    for (int idx = lt; idx < items; idx += nthreads) {
      const int c = idx / rows, row = idx - c * rows;
      const int t = t0 + row;
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
// launches (block mode: residual, tanh) or already part of val (hpair_kernel's prefetched residual and branch sum).
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

// ------------------------------------------------------------------------------------------------ kernels

// modes 0 (conv) and 1 (conv-transpose); launch_hconv runs pair mode (2) on hpair_kernel, and block mode runs on
// hchain_kernel.  The mode-2 branch below is no longer launched but stays: without it ptxas (nvcc 12.9, build.py's
// flags) reports spill stores / loads of 956 / 1220 bytes at N = 256 and 784 / 1020 at N = 128, against 4 / 4 and
// 16 / 20 with it, which made HiFi-GAN V1's ConvTranspose layers about 5 ms per step slower (H100 80GB HBM3, 400 W
// power limit).  Re-check those numbers before deleting it.
template <int NW, int BF16>
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
    load_tile<BF16>(p, g, b, smem, 4 * kc, 4, g.rowsA, O - g.a0, tid, HC_THREADS);
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

// Block mode (launch_tc_chain): warp-specialised and persistent.  One CTA of three warpgroups per SM walks the
// (utterance, time tile) work items with a static stride.
//   warpgroup 0 (producer, setmaxnreg 40): thread 0 streams the weight stages of every tile through the W ring;
//     warps 1-3 load the operand tile X of the next work item as soon as the consumers release it, so that load
//     overlaps the current tile's output epilogue.
//   warpgroups 1-2 (consumers, setmaxnreg 232): one wgmma batch per tap with the two previous batches still in flight; a
//     W slot is released once the batch that read it has completed.  Consumer-only synchronisation is a named
//     barrier.  The residual stream x_p of the whole ResBlock stays in registers in the accumulator fragment layout.
// The accumulation order of every output element is that of hconv_kernel's per-pair mode (K chunk -> tap -> k16).
constexpr int HB_THREADS = 3 * 128;
constexpr int HB_LOADERS = 96;
constexpr int HB_PRODUCER_REGS = 40;
constexpr int HB_CONSUMER_REGS = 232;
static_assert(128 * HB_PRODUCER_REGS + 256 * HB_CONSUMER_REGS <= 65536, "setmaxnreg split of the register file");
constexpr int HP_ABUF_MAX = 3;   // hpair_kernel: A chunk buffers, as many as fit (one for very wide tap reach)

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

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

template <int NW, int BF16>
__global__ void __launch_bounds__(HB_THREADS, 1) hchain_kernel(HcArgs p, HcGeom g) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const uint32_t sX = smem_u32(smem), sI = sX + g.off_i, sW = sX + g.off_w;
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const uint32_t bar0 = smem_u32(smem + g.off_bar);
  auto w_full = [&](int s) { return bar0 + 8u * s; };
  auto w_empty = [&](int s) { return bar0 + 8u * (HC_STAGES_MAX + s); };
  const uint32_t x_full = bar0 + 16u * HC_STAGES_MAX, x_empty = x_full + 8u;
  const int nwork = p.B * g.tiles;
  const int per_step = g.nkc * g.ntaps;

  if (tid == 0) {
    for (int s = 0; s < g.nstages; ++s) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), 8);
    }
    mbar_init(x_full, HB_LOADERS);
    mbar_init(x_empty, 8);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  stage_biases(bias_s, p, g.nsteps, NW, tid, HB_THREADS);
  // rows and channels of the intermediate that no step writes stay zero for every tile
  for (int i = tid; i < g.nkc * 4 * g.rowsX; i += HB_THREADS)
    *reinterpret_cast<uint4*>(smem + g.off_i + (size_t)i * 16) = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  // ------------------------------------------------------------------------------------------------ producer
  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HB_PRODUCER_REGS));
    if (tid == 0) {
      RingPos r;
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        for (int st = 0; st < g.nsteps; ++st)
          for (int i = 0; i < per_step; ++i, r.next(g.nstages)) {
            if (r.wrapped) mbar_wait(w_empty(r.s), r.ph ^ 1u);
            mbar_arrive_expect_tx(w_full(r.s), g.stage_bytes);
            bulk_g2s(sW + (uint32_t)r.s * g.stage_bytes, weight_stage(p, g, st, i), g.stage_bytes, w_full(r.s));
          }
      }
    } else if (tid >= 32) {
      // X <- lrelu(x, pre_slope) over all channels, rows [0, rowsX) at times O - H - G + row
      int n = 0;
      for (int w = blockIdx.x; w < nwork; w += gridDim.x, ++n) {
        const int b = w / g.tiles, t0 = (w - b * g.tiles) * g.V - g.H - g.G;
        if (n > 0) mbar_wait(x_empty, (uint32_t)(n - 1) & 1u);
        load_tile<BF16>(p, g, b, smem, 0, 4 * g.nkc, g.rowsX, t0, tid - 32, HB_LOADERS);
        fence_proxy_async();
        mbar_arrive(x_full);
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HB_CONSUMER_REGS));
  const int cw = wg - 1;
  const Frag<MT> f(cw);
  float acc[MT][NACC];
  RingPos wr;        // W slot of the next weight stage
  // W slots read by the batches in flight, oldest first (-1: none).  Two batches stay in flight when the ring leaves a
  // slot to fill next to the two they hold.
  const bool deep = g.nstages >= 3;
  int pw0 = -1, pw1 = -1;

  // keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
  auto fence_acc = [&]() {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < NACC; ++i) asm volatile("" : "+f"(acc[mt][i])::"memory");
  };
  auto release_w = [&](int pw) {
    __syncwarp();
    if (lane == 0 && pw >= 0) mbar_arrive(w_empty(pw));
  };
  // the taps of one 32-channel K chunk over the operand at aBase
  auto mma_chunk = [&](uint32_t aBase, int ntaps, int tapstep, bool& first) {
    for (int j = 0; j < ntaps; ++j) {
      const int s = wr.s;
      mbar_wait(w_full(s), wr.ph);
      wr.next(g.nstages);
      const uint32_t wS = sW + (uint32_t)s * g.stage_bytes;
      fence_acc();
      wg_fence();
      mma_batch<NW, BF16>(acc, aBase, g.rowsX, cw * MT * 64 + j * tapstep, wS, first);
      wg_commit();
      if (deep) {
        wg_wait<2>();    // the batch before the previous one has completed: its W slot can be refilled
        fence_acc();
        release_w(pw0);
        pw0 = pw1;
      } else {
        wg_wait<1>();
        fence_acc();
        release_w(pw1);
      }
      pw1 = s;
      first = false;
    }
  };
  auto drain = [&]() {
    wg_wait<0>();
    fence_acc();
    release_w(pw0);
    release_w(pw1);
    pw0 = pw1 = -1;
  };

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
    mbar_wait(x_full, (uint32_t)n & 1u);
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
      for (int kc = 0; kc < g.nkc; ++kc) mma_chunk(aT + (uint32_t)(kc * 4 * g.rowsX + g.G - hh) * 16u, g.ntaps, d, first);
      drain();
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
    __syncwarp();
    if (lane == 0) mbar_arrive(x_empty);
    // y = (x_L + acc_prev) * out_scale on the valid rows [H, H + V)
    epilogue_out<NW, BF16, EP_ACC_PREV>(p, g, f, b, O - g.H, g.H, g.H + g.V, 0,
                                        [&](int mt, int c, int h, int e) { return xr[mt][c * 4 + 2 * h + e]; });
  }
}

// Pair mode (launch_tc_conv with a second conv; one ResBlock1 step): warp-specialised and persistent like
// hchain_kernel, with the per-pair tile geometry of make_geom (output row r at time O + r, V = R - (k - 1)).
//   warpgroup 0 (producer, setmaxnreg 40): thread 0 streams both convs' weight stages of every tile through the W
//     ring; warps 1-3 stream the A operand in 32-channel K chunks through a ring of g.nabuf chunk buffers.  Conv2 reads
//     only the intermediate tile, so the next tile's chunks load under this tile's conv2 and output epilogue.
//   warpgroups 1-2 (consumers, setmaxnreg 232): two wgmma batches in flight (one where the rings are too small); a
//     W slot, and an A buffer after its last tap, is released once the batch that read it has completed.  Below N = 256 each consumer loads the residual
//     of its fragment into registers at the start of the tile, so that HBM read runs under the MMAs; the branch sum
//     would need another 64 registers at N = 128 (ptxas spills) and is read in the epilogue.
// Accumulation order (K chunk -> tap -> k16, conv1 then conv2) and epilogue association are those of the per-pair
// arithmetic, so the tile shape does not enter any output element.
template <int NW, int BF16>
__global__ void __launch_bounds__(HB_THREADS, 1) hpair_kernel(HcArgs p, HcGeom g) {
  constexpr int MT = mt_of(NW);
  constexpr int NACC = NW / 2;
  constexpr bool PREFETCH = MT * NACC <= 64;   // 64 accumulators leave room for 64 prefetched residuals
  constexpr int PM = PREFETCH ? MT : 1, PN = PREFETCH ? NACC : 1;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const uint32_t sA = smem_u32(smem), sI = sA + g.off_i, sW = sA + g.off_w;
  const uint32_t abytes = (uint32_t)g.rowsA * 64u;   // one A chunk: 4 c8 planes x rowsA rows
  float* bias_s = reinterpret_cast<float*>(smem + g.off_bias);
  const uint32_t bar0 = smem_u32(smem + g.off_bar);
  auto w_full = [&](int s) { return bar0 + 8u * s; };
  auto w_empty = [&](int s) { return bar0 + 8u * (HC_STAGES_MAX + s); };
  auto a_full = [&](int s) { return bar0 + 8u * (2 * HC_STAGES_MAX + s); };
  auto a_empty = [&](int s) { return bar0 + 8u * (2 * HC_STAGES_MAX + HP_ABUF_MAX + s); };
  const int nwork = p.B * g.tiles;
  const int per_step = g.nkc * g.ntaps;

  if (tid == 0) {
    for (int s = 0; s < g.nstages; ++s) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), 8);
    }
    for (int s = 0; s < g.nabuf; ++s) {
      mbar_init(a_full(s), HB_LOADERS);
      mbar_init(a_empty(s), 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  stage_biases(bias_s, p, 2, NW, tid, HB_THREADS);
  // rows and channels of the intermediate that store_frag_tile does not write stay zero for every tile
  for (int i = tid; i < g.nkc * 4 * g.rowsI; i += HB_THREADS)
    *reinterpret_cast<uint4*>(smem + g.off_i + (size_t)i * 16) = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  // ------------------------------------------------------------------------------------------------ producer
  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HB_PRODUCER_REGS));
    if (tid == 0) {
      RingPos r;
      for (int w = blockIdx.x; w < nwork; w += gridDim.x)
        for (int st = 0; st < 2; ++st)
          for (int i = 0; i < per_step; ++i, r.next(g.nstages)) {
            if (r.wrapped) mbar_wait(w_empty(r.s), r.ph ^ 1u);
            mbar_arrive_expect_tx(w_full(r.s), g.stage_bytes);
            bulk_g2s(sW + (uint32_t)r.s * g.stage_bytes, weight_stage(p, g, st, i), g.stage_bytes, w_full(r.s));
          }
    } else if (tid >= 32) {
      // A chunk kc of a tile: rows [0, rowsA) at times O - a0 + row, channels [32 kc, 32 kc + 32)
      int q = 0;
      for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
        const int b = w / g.tiles, t0 = (w - b * g.tiles) * g.V - g.a0;
        for (int kc = 0; kc < g.nkc; ++kc, ++q) {
          const int s = q % g.nabuf;
          if (q >= g.nabuf) mbar_wait(a_empty(s), (uint32_t)(q / g.nabuf - 1) & 1u);
          load_tile<BF16>(p, g, b, smem + s * abytes, 4 * kc, 4, g.rowsA, t0, tid - 32, HB_LOADERS);
          fence_proxy_async();
          mbar_arrive(a_full(s));
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------------------------------------ consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HB_CONSUMER_REGS));
  const int cw = wg - 1;
  float acc[MT][NACC];
  RingPos wr;             // W slot of the next weight stage
  int q = 0;              // A chunks consumed so far
  // Batches in flight, oldest first: the W slot each read, and the A buffer whose last tap it was (-1: none).  Two
  // stay in flight when the rings allow it: every W slot held by an in-flight batch must leave one to fill
  // (nstages >= 3), and the loaders must not need the buffer of the last tap of the chunk before the previous one
  // (ntaps >= 2, or three buffers; one buffer is drained after every chunk).
  const bool deep = g.nstages >= 3 && (g.ntaps >= 2 || g.nabuf != 2);
  int pw0 = -1, pw1 = -1, pa0 = -1, pa1 = -1;

  auto fence_acc = [&]() {
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < NACC; ++i) asm volatile("" : "+f"(acc[mt][i])::"memory");
  };
  auto release = [&](int w, int a) {
    __syncwarp();
    if (lane == 0) {
      if (w >= 0) mbar_arrive(w_empty(w));
      if (a >= 0) mbar_arrive(a_empty(a));
    }
  };
  // the taps of one 32-channel K chunk over the operand at aBase (aRows rows per c8 plane); abuf: the A buffer it
  // reads, or -1 for the intermediate tile
  auto mma_chunk = [&](uint32_t aBase, int aRows, int tapstep, int abuf, bool& first) {
    for (int j = 0; j < g.ntaps; ++j) {
      const int s = wr.s;
      mbar_wait(w_full(s), wr.ph);
      wr.next(g.nstages);
      const uint32_t wS = sW + (uint32_t)s * g.stage_bytes;
      fence_acc();
      wg_fence();
      mma_batch<NW, BF16>(acc, aBase, aRows, cw * MT * 64 + j * tapstep, wS, first);
      wg_commit();
      const int a = j == g.ntaps - 1 ? abuf : -1;
      if (deep) {
        wg_wait<2>();    // the batch before the previous one has completed: its W slot (and A buffer) can be refilled
        fence_acc();
        release(pw0, pa0);
        pw0 = pw1;
        pa0 = pa1;
      } else {
        wg_wait<1>();
        fence_acc();
        release(pw1, pa1);
      }
      pw1 = s;
      pa1 = a;
      first = false;
    }
  };
  auto drain = [&]() {
    wg_wait<0>();
    fence_acc();
    release(pw0, pa0);
    release(pw1, pa1);
    pw0 = pw1 = pa0 = pa1 = -1;
  };

  for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int b = w / g.tiles, O = (w - b * g.tiles) * g.V;
    // residual of this thread's output elements, in flight under the MMAs
    float xres[PM][PN];
    if constexpr (PREFETCH) {
      const Frag<MT> f(cw);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = f.row(mt, h), t = O + row;
          const bool ok = row < g.V && t < g.Tout;
#pragma unroll
          for (int c = 0; c < NW / 8; ++c)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int co = c * 8 + f.col + e;
              const bool in = ok && co < p.Cout && p.residual;
              xres[mt][c * 4 + 2 * h + e] = in ? __ldg(p.residual + ((int64_t)b * p.Cout + co) * g.Tout + t) : 0.f;
            }
        }
    }
    // conv1 over the A chunks
    bool first = true;
    for (int kc = 0; kc < g.nkc; ++kc, ++q) {
      const int s = q % g.nabuf;
      mbar_wait(a_full(s), (uint32_t)(q / g.nabuf) & 1u);
      mma_chunk(sA + (uint32_t)s * abytes, g.rowsA, g.d, s, first);
      if (g.nabuf == 1) drain();   // the loaders refill the only buffer with the next chunk
    }
    drain();
    // intermediate = lrelu(conv1 + b1, mid_slope) -> operand tile, row 0 at time O - h2, zero outside [0, T)
    consumer_sync();   // both warpgroups have finished the previous tile's conv2, which read the intermediate
    store_frag_tile<NW, BF16>(smem + g.off_i, acc, bias_s, Frag<MT>(cw), g.rowsI, 0, O - g.h2, g.Tin, 4 * g.nkc,
                              g.mid_slope);
    fence_proxy_async();
    consumer_sync();
    first = true;
    for (int kc = 0; kc < g.nkc; ++kc) mma_chunk(sI + (uint32_t)(kc * 4 * g.rowsI) * 16u, g.rowsI, 1, -1, first);
    drain();
    // y = ((acc + b2) + residual) + acc_prev) * out_scale [tanh] on the valid rows [0, V)
    const Frag<MT> f(cw);
    const float* b2 = bias_s + NW;
    if constexpr (PREFETCH) {
      epilogue_out<NW, BF16, EP_ACC_PREV | EP_TANH>(p, g, f, b, O, 0, g.V, 0, [&](int mt, int c, int h, int e) {
        const int i = c * 4 + 2 * h + e;
        const float v = acc[mt][i] + b2[c * 8 + f.col + e];
        return p.residual ? v + xres[mt][i] : v;
      });
    } else {
      epilogue_out<NW, BF16, EP_ALL>(p, g, f, b, O, 0, g.V, 0, [&](int mt, int c, int h, int e) {
        return acc[mt][c * 4 + 2 * h + e] + b2[c * 8 + f.col + e];
      });
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

// mode 0 conv (d_or_u = dilation), 1 conv-transpose (d_or_u = stride)
int layer_geom(int mode, int cin, int cout, int k, int d_or_u, HcLayer& L) {
  if (cin <= 0 || cout <= 0 || k <= 0 || d_or_u <= 0) return fail(AB_ERR_ARG, "tc conv: bad layer shape");
  L.mode = mode;
  L.nkc = (cin + 31) / 32;
  if (mode == 0) {
    if (!(k & 1)) return fail(AB_ERR_UNSUPPORTED, "tc conv: conv kernel size must be odd");
    L.NW = std::min(256, pow2_at_least(rup(cout, 16)));
    L.NB = (cout + L.NW - 1) / L.NW;
    L.cc = L.NW;
    L.ntaps = k;
    L.u = 1;
  } else {
    const int u = d_or_u;
    if (k < u || ((k - u) & 1)) return fail(AB_ERR_UNSUPPORTED, "tc conv: conv-transpose needs k >= stride, k-stride even");
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
    } else {
      const int cl = n / L.u, phi = n - cl * L.u, co = nb * L.cc + cl, j = phi + L.u * tap;
      if (ci < cin && cl < L.cc && co < cout && j < k) v = w_t[((int64_t)ci * k + j) * cout + co];
    }
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

// Launch geometry.  mode 2 (pair): C_in = C_out = C <= 256, conv1 dilation d_or_u, conv2 dilation 1.
int make_geom(int mode, int cin, int cout, int k, int d_or_u, int Tin, HcGeom& g) {
  HcLayer L;
  int rc = layer_geom(mode == 2 ? 0 : mode, cin, cout, k, d_or_u, L);
  if (rc != AB_OK) return rc;
  if (mode == 2 && (cin != cout || L.NB != 1)) return fail(AB_ERR_UNSUPPORTED, "tc conv pair: C=%d not in [1,%d]", cin, TC_MAX_C);
  g.mode = mode;
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
    g.pad = (k - L.u) / 2;
    g.Tout = Tin * L.u;
    maxshift = g.ntaps - 1;
    g.a0 = maxshift;
    g.V = g.R;
    rows_total = (g.Tout - 1 + g.pad) / L.u + 1;
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
  if (mode == 2) {   // hpair_kernel: one CTA per SM, as many A chunk buffers as fit next to two W stages
    const uint32_t ibytes = (uint32_t)g.nkc * 64u * (uint32_t)g.rowsI;
    g.nabuf = HP_ABUF_MAX;
    while (!(fits = layout_smem(g, (uint32_t)g.nabuf * abytes, ibytes, nbias,
                                16u * (HC_STAGES_MAX + HP_ABUF_MAX), HC_SMEM_1CTA)) && g.nabuf > 1)
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

// Launches K after raising its dynamic shared-memory limit to `limit`, once per device.
template <void (*K)(HcArgs, HcGeom)>
int launch_kernel(const char* name, unsigned grid, int threads, uint32_t limit, const HcArgs& a, const HcGeom& g,
                  cudaStream_t s) {
  static DeviceOnce configured;
  if (configured.need()) AB_CUDA_TRY(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit));
  K<<<grid, threads, g.smem_bytes, s>>>(a, g);
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

// Block-mode geometry: npairs x nconv convs of one ResBlock (C <= 64) with the halo recomputed inside the tile.
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
  // mbarriers: W ring full / empty, X full / empty
  if (!layout_smem(g, xbytes, xbytes, (uint32_t)(g.nsteps * L.NW), 16u * HC_STAGES_MAX + 16u, HC_SMEM_1CTA))
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

// modes 0 and 1 on hconv_kernel (one CTA per tile), pair mode on the persistent hpair_kernel
int launch_hconv(const HcArgs& a, const HcGeom& g, int precision, cudaStream_t s) {
  if (precision != AB_PREC_TC_F16 && precision != AB_PREC_TC_BF16) return fail(AB_ERR_ARG, "tc conv: bad precision");
  const int64_t work = (int64_t)a.B * g.tiles;
  if (g.mode == 2) {
    unsigned grid = 0;
    const int rc = persistent_grid(work, "tc conv pair", grid);
    if (rc != AB_OK) return rc;
    return with_nw(g, precision, [&](auto nw, auto bf16) {
      return launch_kernel<hpair_kernel<decltype(nw)::value, decltype(bf16)::value>>("hpair_kernel", grid, HB_THREADS,
                                                                                     HC_SMEM_1CTA, a, g, s);
    });
  }
  if (work > 0x7fffffffll) return fail(AB_ERR_UNSUPPORTED, "tc conv: grid too large");
  return with_nw(g, precision, [&](auto nw, auto bf16) {
    constexpr int NW = decltype(nw)::value;
    return launch_kernel<hconv_kernel<NW, decltype(bf16)::value>>("hconv_kernel", (unsigned)work, HC_THREADS,
                                                                   NW >= 256 ? HC_SMEM_1CTA : HC_SMEM_2CTA, a, g, s);
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
  unsigned grid = 0;
  rc = persistent_grid((int64_t)a.B * g.tiles, "tc block", grid);
  if (rc != AB_OK) return rc;
  return with_nw(g, p.precision, [&](auto nw, auto bf16) {
    constexpr int NW = decltype(nw)::value;
    if constexpr (NW > AB_TC_CHAIN_MAX_C)   // make_chain_geom rejects wider blocks
      return fail(AB_ERR_UNSUPPORTED, "tc block: N block %d", NW);
    else
      return launch_kernel<hchain_kernel<NW, decltype(bf16)::value>>("hchain_kernel", grid, HB_THREADS, HC_SMEM_1CTA, a,
                                                                      g, s);
  });
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

// The conv epilogue zero-fills the image's padding channels; the conv-transpose epilogue writes only c_out < C_out.
bool tc_can_emit_image(int mode, int cin, int cout, int k, int d_or_u) {
  if (mode == 0) return cin == cout && tc_conv_supported(cin, k);
  HcLayer L;
  return layer_geom(1, cin, cout, k, d_or_u, L) == AB_OK && (cout % 16) == 0;
}

int launch_tc_conv(const TcConvParams& p, cudaStream_t s) {
  const bool pair = p.w2 != nullptr;
  if ((!p.x && !p.ximg) || !p.y || !p.w) return fail(AB_ERR_ARG, "tc conv: null argument");
  if (p.B <= 0 || p.T <= 0) return fail(AB_ERR_ARG, "tc conv: bad shape");
  if (p.mode != 0 && p.mode != 1) return fail(AB_ERR_ARG, "tc conv: mode must be 0 (conv) or 1 (conv-transpose)");
  if (p.mode == 1 && (p.residual || p.acc_prev || p.out_div != 1.0f || p.post_tanh))
    return fail(AB_ERR_ARG, "tc conv-transpose: residual, acc_prev, out_div and tanh belong to conv");
  if (pair && !(p.mode == 0 && p.Cin == p.Cout && tc_conv_supported(p.Cin, p.k)))
    return fail(AB_ERR_UNSUPPORTED, "tc conv pair: C_in=%d C_out=%d k=%d", p.Cin, p.Cout, p.k);
  if (p.mode == 1 && p.ximg && (p.Cin % 16) != 0)
    return fail(AB_ERR_UNSUPPORTED, "tc conv-transpose: operand-image input needs C_in %% 16 == 0");
  if (p.yimg && !tc_can_emit_image(p.mode, p.Cin, p.Cout, p.k, p.d_or_u))
    return fail(AB_ERR_UNSUPPORTED, "tc conv: cannot emit an operand image for this layer");
  HcGeom g;
  int rc = make_geom(pair ? 2 : p.mode, p.Cin, p.Cout, p.k, p.d_or_u, p.T, g);
  if (rc != AB_OK) return rc;
  g.out_scale = 1.0f / p.out_div;
  g.mid_slope = p.mid_slope;
  HcArgs a = base_args(p.x, p.xsb, p.xsc, p.xst, p.ximg, p.pre_slope, p.B, p.Cin, p.Cout);
  a.ws[0] = p.w; a.bs[0] = p.bias;
  a.ws[1] = p.w2; a.bs[1] = p.b2;
  a.y = p.y; a.residual = p.residual; a.acc_prev = p.acc_prev; a.post_tanh = p.post_tanh;
  a.yimg = p.yimg; a.img_slope = p.img_slope;
  return launch_hconv(a, g, p.precision, s);
}

}  // namespace ab
