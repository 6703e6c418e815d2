"""Kernel-order restatement of DiffWave's CUDA kernels (amphion_b200/csrc/ab_diffwave.cu), the checker of them at the
bit level.  numpy only: it imports nothing of the product.

Every kernel operation is an explicit `__fmaf_rn` / `__fadd_rn` / `__fmul_rn` / `__fdiv_rn`, so the compiler never
contracts or reorders them, and each is restated here with the same operands in the same order:
  fadd / fmul / fdiv   numpy float32 arithmetic (IEEE, round to nearest even);
  fma                  fp32 fused multiply-add emulated exactly: a*b is exact in float64, the sum with c is carried as
                       a TwoSum pair, and a float64 sum that lands exactly on an fp32 midpoint is settled by the sign of
                       the TwoSum error.
What cannot be restated is the gate's `expf` / `tanhf`: the layer functions take the gate z as an input (the tests read
it back from the kernel), and `gate64` is the float64 gate of fp32 pre-activations for the ulp-band checks.

The layer (`dw_layer_kernel` at fp32, `dw_layer_tc_kernel` at tc_f16 / tc_bf16), C = 64 channels:
  S      = [tap 0 | tap 1 | tap 2 | mel] (K order: tap-major, then channel; then the n_mel mel rows), where tap j of
           channel c at time t is x[c, t + (j - 1) dil] + d[c], zero outside [0, L) (the padding of x + d)
  pre    = acc1 + (bdil + bcond)          fp32: acc1 = the FMA chain over K in that order; tensor cores: one MMA sum
  z      = sigmoid(pre_gate) tanh(pre_filter)   (rounded to the 16-bit type before conv2 on the tensor cores)
  res, s = acc2 + bout                    fp32: acc2 = the FMA chain over the 64 channels of z in order
  x_out  = (x + (acc2_res + bres)) / 1.41421356237309515f,   skip = s (first) or s + skip
Tensor-core operands are rounded with `resblock_oracle.rnd` (cvt.rn.satfinite)."""
from __future__ import annotations

import numpy as np

from resblock_oracle import rnd

C = 64
SQRT2 = np.float32(1.41421356237309515)


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def _f32(v):
    return np.asarray(v, np.float32)


def fma(a, b, c):
    """fp32 fma(a, b, c) = round_fp32(a b + c), exact, elementwise with broadcasting."""
    a, b, c = _f32(a), _f32(b), _f32(c)
    p = a.astype(np.float64) * b.astype(np.float64)          # exact: 24 + 24 significand bits
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                           # TwoSum: s + e == p + c exactly
    r = s.astype(np.float32)
    # s on an fp32 midpoint with e != 0: round_fp32(s) may have gone the wrong way; the exact sum lies on e's side
    with np.errstate(over="ignore", invalid="ignore"):
        toward = np.where(s > r.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
        other = np.nextafter(r, toward)
        mid = (r.astype(np.float64) + other.astype(np.float64)) * 0.5
        tie = (s == mid) & (e != 0) & np.isfinite(s)
        if np.any(tie):
            up = e > 0
            lo = np.where(r.astype(np.float64) < s, r, other)
            hi = np.where(r.astype(np.float64) < s, other, r)
            r = np.where(tie, np.where(up, hi, lo), r)
    return r.astype(np.float32)


def lrelu04(v):
    """x > 0 ? x : x * 0.4f"""
    v = _f32(v)
    return np.where(v > 0, v, v * np.float32(0.4)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ upsampler
def _convt2d_lrelu(src, w, bias, f):
    """One ConvTranspose2d(1, 1, [3, 2f], stride [1, f], padding [1, f/2]) + leaky_relu(0.4) of src [B, H, W] in the
    kernel's order: kh = 0..2 (input row h + 1 - kh), then e = 0..1 (input column j0 - e, kernel column r + e f)."""
    B, H, W = src.shape
    w = _f32(w).reshape(3, 2 * f)
    col = np.arange(W * f)
    q = col + f // 2
    j0, r = q // f, q % f
    acc = np.zeros((B, H, W * f), np.float32)
    for kh in range(3):
        hh = np.arange(H) + 1 - kh
        okh = (hh >= 0) & (hh < H)
        for e in range(2):
            j = j0 - e
            okj = (j >= 0) & (j < W)
            v = src[:, np.clip(hh, 0, H - 1)][:, :, np.clip(j, 0, W - 1)]
            ok = okh[None, :, None] & okj[None, None, :]
            acc = np.where(ok, fma(v, w[kh, r + e * f][None, None, :], acc), acc)
    return lrelu04(acc + _f32(bias).reshape(-1)[0])


def upsample(mel, w1, b1, w2, b2, f1, f2):
    """dw_upsample_kernel: mel [B, n_mel, F] -> [B, n_mel, F f1 f2]."""
    return _convt2d_lrelu(_convt2d_lrelu(_f32(mel), w1, b1, f1), w2, b2, f2)


def input_projection(audio, w, b):
    """dw_input_kernel: relu(w[c] audio + b[c]) (a multiply and an add, not an FMA) -> [B, C, L]."""
    a = _f32(audio)[:, None, :]
    return np.maximum(a * _f32(w).reshape(-1)[None, :, None] + _f32(b)[None, :, None], np.float32(0)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the layer
def conv1_operands(x, d, cond, dil):
    """S [B, 3C + n_mel, L]: the three dilated taps of x + d (x [B, C, L], d [B, C]), zero outside [0, L), then the
    mel rows cond [B, n_mel, L]."""
    x, d, cond = _f32(x), _f32(d), _f32(cond)
    B, _, L = x.shape
    y = x + d[:, :, None]
    taps = []
    for j in range(3):
        t = np.arange(L) + (j - 1) * dil
        ok = (t >= 0) & (t < L)
        taps.append(np.where(ok[None, None, :], y[:, :, np.clip(t, 0, L - 1)], np.float32(0)))
    return np.concatenate(taps + [cond], axis=1).astype(np.float32)


def conv1_weight(wdil, wcond):
    """[2C, 3C + n_mel] in S's K order from dilated_conv [2C, C, 3] and conditioner_projection [2C, n_mel(, 1)]."""
    wdil, wcond = _f32(wdil), _f32(wcond)
    return np.concatenate([wdil[:, :, 0], wdil[:, :, 1], wdil[:, :, 2], wcond.reshape(wcond.shape[0], -1)], axis=1)


def fma_chain(w, a):
    """out[b, o, t] = the FMA chain acc = fma(w[o, k], a[b, k, t], acc) over k = 0, 1, ... from acc = 0."""
    w, a = _f32(w), _f32(a)
    acc = np.zeros((a.shape[0], w.shape[0], a.shape[2]), np.float32)
    for k in range(w.shape[1]):
        acc = fma(w[None, :, k, None], a[:, k:k + 1, :], acc)
    return acc


def exact_sum(w, a):
    """sum_k w[o, k] a[b, k, t] in float64 (exact for the one-hot and small dense sums the tests use, up to the last
    float64 bit) -> float64."""
    return np.einsum("ok,bkt->bot", _f32(w).astype(np.float64), _f32(a).astype(np.float64))


def conv1_pre(S, w1, bdil, bcond, prec=None, chain=False):
    """Pre-activations [B, 2C, L] (gate, then filter): acc1 + (bdil + bcond).  chain (fp32 only): acc1 is
    dw_layer_kernel's FMA chain over K; otherwise the operands and weights, rounded to prec ("f16" / "bf16" / None),
    summed exactly and rounded once, which is what either kernel computes when one weight per output is non-zero."""
    b1 = _f32(bdil) + _f32(bcond)
    acc = fma_chain(w1, S) if chain else exact_sum(rnd(w1, prec), rnd(S, prec)).astype(np.float32)
    return (acc + b1[None, :, None]).astype(np.float32)


def gate64(pre):
    """sigmoid(gate) tanh(filter) in float64 of fp32 pre-activations [B, 2C, L] -> float64 [B, C, L]."""
    p = np.asarray(pre, np.float64)
    return 1.0 / (1.0 + np.exp(-p[:, :C])) * np.tanh(p[:, C:])


def layer_out(x, z, wout, bout, skip_prev=None, prec=None):
    """(x_out, skip) of the layer from its gate z [B, C, L] (as the kernel holds it: fp32, or already 16-bit
    rounded).  prec None: conv2 is dw_layer_kernel's FMA chain; "f16" / "bf16": the exact sum over rnd(z) rnd(wout)
    rounded once (valid when the MMA sum is exact).  skip_prev None: the first layer."""
    x, wout, bout = _f32(x), _f32(wout).reshape(2 * C, C), _f32(bout)
    acc = fma_chain(wout, z) if prec is None else exact_sum(rnd(wout, prec), rnd(z, prec)).astype(np.float32)
    return epilogue(x, acc, bout, skip_prev)


def epilogue(x, acc, bout, skip_prev=None):
    """x_out = (x + (acc_res + bres)) / sqrt2_f, s = acc_skip + bskip, skip = s or s + skip_prev."""
    x, acc, bout = _f32(x), _f32(acc), _f32(bout)
    x_out = ((x + (acc[:, :C] + bout[None, :C, None])) / SQRT2).astype(np.float32)
    s = (acc[:, C:] + bout[None, C:, None]).astype(np.float32)
    return x_out, (s if skip_prev is None else (s + _f32(skip_prev)).astype(np.float32))


def layer(x, d, cond, wdil, bdil, wcond, bcond, wout, bout, dil, skip_prev=None):
    """A whole fp32 layer in kernel order, the gate from `gate64` rounded once (the kernel's expf / tanhf differ from
    it by a few ulp): the oracle's own check against the float64 network."""
    pre = conv1_pre(conv1_operands(x, d, cond, dil), conv1_weight(wdil, wcond), bdil, bcond, chain=True)
    z = (1.0 / (1.0 + np.exp(-pre[:, :C].astype(np.float64)))).astype(np.float32) * np.tanh(
        pre[:, C:].astype(np.float64)).astype(np.float32)
    return layer_out(x, z, wout, bout, skip_prev)


# ------------------------------------------------------------------------------------------------ the tail
def tail(skip, wsk, bsk, wo, bo, skip_div, audio=None, c1=1.0, c2=0.0, sigma=0.0, noise=None):
    """dw_tail_kernel: s = skip / skip_div; h_o = FMA chain over c of wsk[o, c] s_c; e = FMA chain over o of
    wo[o] max(h_o + bsk[o], 0); e += bo.  audio None: eps [B, L]; otherwise the sampler update
    clamp(c1 (audio - c2 e) [+ sigma noise], -1, 1) [B, L]."""
    s = (_f32(skip) / np.float32(skip_div)).astype(np.float32)
    wsk, bsk, wo = _f32(wsk).reshape(C, C), _f32(bsk), _f32(wo).reshape(C)
    h = fma_chain(wsk, s)                                                # [B, C, L]
    e = np.zeros((s.shape[0], s.shape[2]), np.float32)
    for o in range(C):
        e = fma(wo[o], np.maximum(h[:, o] + bsk[o], np.float32(0)), e)
    e = (e + _f32(bo).reshape(-1)[0]).astype(np.float32)
    if audio is None:
        return e
    v = np.float32(c1) * (_f32(audio) - np.float32(c2) * e)
    if noise is not None:
        v = v + np.float32(sigma) * _f32(noise)
    return np.minimum(np.maximum(v, np.float32(-1)), np.float32(1)).astype(np.float32)
