"""Kernel-order restatement of Vocos' CUDA kernels, the checker of them at the bit level: `vocos_norm_kernel`
(amphion_b200/csrc/ab_kernels_fp32.cu), the pointwise GEMM epilogues of `hitem_kernel` (ab_kernels_tc.cu,
`epilogue_pw`) and of `conv1d_fp32_kernel`, and the head's column pairing (`hc_pack_head_weight_kernel`).  numpy and
scipy only: it imports nothing of the product.

LayerNorm (`layer_norm_kernel_order`), every operation an explicit `__f*_rn` intrinsic in the kernel:
  tile    TT = 16, halved while 4 (C TT + 256 + 2 TT) > 64 KiB; ngrp = 256 / TT thread groups per time step
  dw      optional depthwise conv: the FMA chain over taps 0..6 (taps outside [0, T) skipped), then + dw_b
  mean    group g sums channels g, g + ngrp, ... in order from 0; the ngrp partials are summed q = 0.. in order; / C
  var     the same partition over fma(d, d, a), d = v - mean; rstd = 1 / sqrt(var_sum / C + eps) (each step rounded)
  out     fma((v - mean) * rstd, ln_w, ln_b)
The transcendental epilogues (erff, expf, sinf / cosf) cannot be restated bit for bit.  `gelu_interval` and
`spectrum_interval` give the interval of the kernel's fp32 result from CUDA's documented bound of 2 ulp on each of
those functions, with the rest of each expression evaluated at the ends (it is monotone in the function's value)."""
from __future__ import annotations

import numpy as np
from scipy.special import erf

from diffwave_exact_oracle import fma
from resblock_oracle import OneHot

LN_THREADS = 256
ULPS = 2                     # CUDA's maximum ulp error of erff, expf, sinf and cosf
INV_SQRT2 = np.float32(0.70710678118654752440)
AMP_MAX = np.float32(1e2)


def _f32(v):
    return np.asarray(v, np.float32)


# ------------------------------------------------------------------------------------------------ LayerNorm
def norm_tile(C):
    """(TT, ngrp) of launch_vocos_norm for C channels."""
    TT = 16
    while TT > 1 and 4 * (C * TT + LN_THREADS + 2 * TT) > 64 * 1024:
        TT //= 2
    return TT, LN_THREADS // TT


def norm_fits(C):
    """launch_vocos_norm's rule: the tile at its TT must fit 200 KB of shared memory."""
    TT, _ = norm_tile(C)
    return 4 * (C * TT + LN_THREADS + 2 * TT) <= 200 * 1024


def dwconv_kernel_order(x, dw_w, dw_b):
    """The k = 7 zero-padded depthwise conv of x [B, C, T]: fma chain over taps j = 0..6 (input t + j - 3), + dw_b."""
    x = _f32(x)
    w = _f32(dw_w).reshape(x.shape[1], 7)
    T = x.shape[2]
    a = np.zeros_like(x)
    for j in range(7):
        t = np.arange(T) + j - 3
        ok = (t >= 0) & (t < T)
        a = np.where(ok[None, None, :], fma(w[None, :, j, None], x[:, :, np.clip(t, 0, T - 1)], a), a)
    return (a + _f32(dw_b)[None, :, None]).astype(np.float32)


def layer_norm_kernel_order(x, dw, ln_w, ln_b, eps):
    """vocos_norm_kernel's fp32 output for x [B, C, T]; dw None or (dw_w [C, 1, 7], dw_b [C])."""
    x = _f32(x)
    if dw is not None:
        x = dwconv_kernel_order(x, *dw)
    B, C, T = x.shape
    _, ngrp = norm_tile(C)
    steps = -(-C // ngrp)
    eps, Cf = np.float32(eps), np.float32(C)
    # group g, step i holds channel g + i ngrp
    part = np.zeros((B, ngrp, T), np.float32)
    for i in range(steps):
        c = np.arange(ngrp) + i * ngrp
        ok = (c < C)[None, :, None]
        part = np.where(ok, part + x[:, np.minimum(c, C - 1)], part).astype(np.float32)
    s = np.zeros((B, T), np.float32)
    for q in range(ngrp):
        s = (s + part[:, q]).astype(np.float32)
    mean = (s / Cf).astype(np.float32)
    part = np.zeros((B, ngrp, T), np.float32)
    for i in range(steps):
        c = np.arange(ngrp) + i * ngrp
        ok = (c < C)[None, :, None]
        d = (x[:, np.minimum(c, C - 1)] - mean[:, None, :]).astype(np.float32)
        part = np.where(ok, fma(d, d, part), part)
    s = np.zeros((B, T), np.float32)
    for q in range(ngrp):
        s = (s + part[:, q]).astype(np.float32)
    rstd = (np.float32(1) / np.sqrt(((s / Cf).astype(np.float32) + eps).astype(np.float32))).astype(np.float32)
    t = ((x - mean[:, None, :]).astype(np.float32) * rstd[:, None, :]).astype(np.float32)
    return fma(t, _f32(ln_w)[None, :, None], _f32(ln_b)[None, :, None])


# ------------------------------------------------------------------------------------------------ intervals
def _ulp_ball(e64):
    """float32 bounds (lo, hi) of every float within ULPS ulp of the float64 values e64 (the ulp of float32 at
    |e64|, rounded outward)."""
    e64 = np.asarray(e64, np.float64)
    u = np.spacing(np.abs(e64).astype(np.float32)).astype(np.float64)
    lo, hi = (e64 - ULPS * u).astype(np.float32), (e64 + ULPS * u).astype(np.float32)
    lo = np.where(lo.astype(np.float64) > e64 - ULPS * u, np.nextafter(lo, np.float32(-np.inf)), lo)
    hi = np.where(hi.astype(np.float64) < e64 + ULPS * u, np.nextafter(hi, np.float32(np.inf)), hi)
    return lo.astype(np.float32), hi.astype(np.float32)


def _gelu32(v, e):
    """The kernels' fp32 GELU of v given erff's result e: (0.5 v) (1 + e), each step rounded."""
    return ((np.float32(0.5) * v).astype(np.float32) * (np.float32(1) + e).astype(np.float32)).astype(np.float32)


def gelu_interval(v):
    """(lo, hi), float32: the interval of 0.5f * v * (1 + erff(v * 0.70710677f)) for fp32 v.  erff(t) lies within
    2 ulp of erf(t) and within [-1, 1] (CUDA computes it as copysign(1 - 2^(.), t) above |t| = 0.93); where 1 - |erf(t)|
    is below 2^-26, a quarter of the float32 gap below 1, 1 - 2^(.) rounds to 1 and erff is +-1 exactly.  The
    interval then collapses to one value: v for large v, -0 for large negative v."""
    v = _f32(v)
    t = (v * INV_SQRT2).astype(np.float32)
    t64 = t.astype(np.float64)
    e64 = erf(t64)
    lo, hi = _ulp_ball(e64)
    lo, hi = np.maximum(lo, np.float32(-1)), np.minimum(hi, np.float32(1))
    one = (1.0 - np.abs(e64)) < 2.0 ** -26
    sgn = np.where(t64 < 0, np.float32(-1), np.float32(1))
    lo, hi = np.where(one, sgn, lo), np.where(one, sgn, hi)
    a, b = _gelu32(v, lo), _gelu32(v, hi)
    return np.minimum(a, b), np.maximum(a, b)


def spectrum_interval(m, p):
    """((re_lo, re_hi), (im_lo, im_hi)), float32: the interval of amp (cos p, sin p), amp = fminf(expf(m), 1e2), for
    fp32 m, p, with expf, sinf and cosf each within 2 ulp (sin and cos within [-1, 1]).  Exact: m >= 5 gives amp = 100
    (e^5 = 148); p = +-0 gives (amp, +-0)."""
    m, p = _f32(m), _f32(p)
    a_lo, a_hi = _ulp_ball(np.exp(m.astype(np.float64)))
    a_lo, a_hi = np.minimum(a_lo, AMP_MAX), np.minimum(a_hi, AMP_MAX)
    big = m >= 5
    a_lo, a_hi = np.where(big, AMP_MAX, a_lo), np.where(big, AMP_MAX, a_hi)
    p64 = p.astype(np.float64)
    c_lo, c_hi = _ulp_ball(np.cos(p64))
    s_lo, s_hi = _ulp_ball(np.sin(p64))
    c_lo, c_hi = np.maximum(c_lo, np.float32(-1)), np.minimum(c_hi, np.float32(1))
    s_lo, s_hi = np.maximum(s_lo, np.float32(-1)), np.minimum(s_hi, np.float32(1))
    zero = p == 0
    c_lo, c_hi = np.where(zero, np.float32(1), c_lo), np.where(zero, np.float32(1), c_hi)
    s_lo, s_hi = np.where(zero, p, s_lo), np.where(zero, p, s_hi)

    def corners(x_lo, x_hi):
        c = [(a * x).astype(np.float32) for a in (a_lo, a_hi) for x in (x_lo, x_hi)]
        return np.minimum.reduce(c), np.maximum.reduce(c)

    return corners(c_lo, c_hi), corners(s_lo, s_hi)


def in_interval(got, lo, hi):
    """Elementwise lo <= got <= hi, and where lo and hi are the same float (sign of zero included) got is that float."""
    got, lo, hi = _f32(got), _f32(lo), _f32(hi)
    same = lo.view(np.uint32) == hi.view(np.uint32)
    return np.where(same, got.view(np.uint32) == lo.view(np.uint32), (got >= lo) & (got <= hi))


# ------------------------------------------------------------------------------------------------ the GEMM
def pointwise_geometry(cout):
    """(NW, NB): the N block width and count launch_tc_pointwise tiles C_out into (k = 1 conv tiles)."""
    c16 = -(-cout // 16) * 16
    nw = 16
    while nw < c16:
        nw *= 2
    nw = min(nw, 256)
    return nw, -(-cout // nw)


def head_columns(cout):
    """hc_pack_head_weight_kernel's column map: image column col holds Linear row j (log-magnitude of bin j) when
    col = 2j, row bins + j (its phase) when col = 2j + 1, and nothing (-1) for j >= bins, over all NB NW columns."""
    nw, nb = pointwise_geometry(cout)
    bins = cout // 2
    col = np.arange(nb * nw)
    j = col // 2
    return np.where(j < bins, np.where(col % 2 == 0, j, bins + j), -1)


def one_hot_linear(rng, cin, cout, exps, avoid=()):
    """A Linear weight [C_out, C_in] as resblock_oracle.OneHot (k = 1): one +-2^e per output channel, every 32-channel
    K chunk of C_in (the last, partial one and channel C_in - 1 included) hit by at least one output channel outside
    `avoid` (rows the caller zeroes)."""
    perm = rng.integers(0, cin, cout)
    nkc = -(-cin // 32)
    free = np.setdiff1d(np.arange(cout), np.asarray(avoid, np.int64))
    if len(free) >= nkc + 1:
        rows = rng.permutation(free)[:nkc + 1]
        for kc, r in enumerate(rows[:nkc]):
            perm[r] = min(32 * kc + int(rng.integers(0, 32)), cin - 1)
        perm[rows[nkc]] = cin - 1
    scale = rng.choice([-1.0, 1.0], cout) * np.exp2(rng.choice(np.asarray(exps, np.float64), cout))
    return OneHot(perm, np.zeros(cout, np.int64), scale, cin, 1)
