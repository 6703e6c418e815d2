"""Kernel-order restatement of `activation1d_warp_kernel` (amphion_b200/csrc/ab_kernels_fp32.cu), the anti-aliased
Snake / SnakeBeta, the checker of it at the bit level.  numpy only: it imports nothing of the product.

Every rounding step of the kernel is an explicit intrinsic (`__fmul_rn`, `__fadd_rn`, `__fmaf_rn`, `__frcp_rn`,
`rintf`), restated here with the same operands in the same order (`fma` of diffwave_exact_oracle is the exact fp32
FMA).  What cannot be restated, `__sinf`, `sin.approx` and `expf`, is given as an interval.

Up-FIR (2x rate, replicate edges; fu2 = 2 f_up, exact).  The kernel computes the 2x-rate window of a 120-output
segment at t0 in groups of 4 starting at i0 = 2 t0 - 7 + 4 j; t0 is a multiple of 120, so every group starts at
i = 1 (mod 4), whichever segment computes it.  A group [g, g + 3] lying wholly inside [0, 2T - 1] takes the PAIR form
(Q = (g - 1) / 2, xh = replicate(x)):
  u[g + k] = lo + hi,  lo / hi = FMA chains that start with a multiply, over the packed tap pairs P_k[q] of
  `pack` with the window pairs (xh[Q - 2 + 2q], xh[Q - 1 + 2q]):  k = 0 ce_a, 1 co_a (q < 3), 2 ce_b, 3 co_b (q < 4).
ce_b / co_b carry zero taps at q = 0 (lo) and q = 3 (hi): their products with xh[Q - 2] and xh[Q + 5] are exact
zeros for finite x, and NaN for a non-finite one.  Any other group takes the edge path's SCALAR chain for all 4 of its
samples, at the clamped index ic = clamp(i, 0, 2T - 1), q = ic >> 1, o = ic & 1:
  u = FMA chain from 0 over m = 0..5 of (o ? fu2[10 - 2m] : fu2[11 - 2m]) xh[q - 3 + o + m].
So u[i] depends on (i, T) only.  The group holding index 0 ([-3, 0]) and the one holding 2T - 1 (odd, never a group's
last) are always scalar, so the window value at any i outside [0, 2T - 1] is the value at clamp(i).
Snake (MODE 0 and 1, and the edge groups of MODE 2):  arg = fmul(u, a), kf = rint(fmul(arg, 1/2pi_f)),
  r = fma(-kf, 2pi_hi, arg), r = fma(-kf, 2pi_lo, r) (Cody-Waite), s = __sinf(r), v = fma(invb, fmul(s, s), u)
with |__sinf(r) - sin r| <= 2^-21.41 for |r| <= pi (CUDA Programming Guide, intrinsic functions).  MODE 2's pair
groups: s = __sinf(fmul(u, a)) with no reduction, v = fma(fmul(s, s), invb, u).  `__sinf` is FMUL.RZ by the fp32
1/2pi, then MUFU.SIN in turns, so its phase error is below (2^-23 + |1 - 2 pi c|) |u a| = 1.6e-7 |u a| rad (c the
fp32 constant; both errors shrink |u a|): PHASE.
Per channel: a = alpha (or expf(alpha), within 2 ulp of exp), invb = frcp(fadd(b, 1e-9)), b = beta (or expf(beta)).
Down-FIR:  y[t] = fadd(lo, hi), lo = the chain mul(fd[0], v[2t - 5]), fma(fd[2q], v[2t - 5 + 2q], .) q = 1..5, hi the
same over the odd taps, v's index clamped to [0, 2T - 1].
Image (16-bit operand): rnd(y) at [B][ceil16(C)/8][T][8], padding channels zero."""
from __future__ import annotations

import numpy as np

from diffwave_exact_oracle import fma
from resblock_oracle import rnd

SEG = 120                                   # outputs per warp segment
INV_2PI = np.float32(0.15915494309189535)
TWO_PI_HI = np.float32(6.2831854820251465)
TWO_PI_LO = np.float32(-1.7484555314695172e-07)
SINF_ERR = 2.0 ** -21.41                    # |__sinf(r) - sin r|, |r| <= pi
MUFU_TURNS = np.float32(0.15915493667125701904)   # the constant of __sinf's FMUL.RZ (cuobjdump -sass)
PHASE = 2.0 ** -23 + abs(1.0 - 2.0 * np.pi * float(MUFU_TURNS))   # sin.approx's phase error per unit |u a|


def _f32(v):
    return np.asarray(v, np.float32)


# ------------------------------------------------------------------------------------------------ taps
def pack(f_up, f_down):
    """pack_snake_coef: dict of [n, 2] fp32 pairs ce_a, co_a (3), ce_b, co_b (4), fd2 (6)."""
    fu2 = _f32(f_up).reshape(12) * np.float32(2)
    fd = _f32(f_down).reshape(12)
    z = np.float32(0)
    kc = {"ce_a": [(fu2[10 - 4 * q], fu2[8 - 4 * q]) for q in range(3)],
          "co_a": [(fu2[11 - 4 * q], fu2[9 - 4 * q]) for q in range(3)],
          "ce_b": [(fu2[12 - 4 * q] if q > 0 else z, fu2[10 - 4 * q] if q < 3 else z) for q in range(4)],
          "co_b": [(fu2[13 - 4 * q] if q > 0 else z, fu2[11 - 4 * q] if q < 3 else z) for q in range(4)],
          "fd2": [(fd[2 * q], fd[2 * q + 1]) for q in range(6)]}
    return {k: np.array(v, np.float32) for k, v in kc.items()}


PAIR_KEYS = ("ce_a", "co_a", "ce_b", "co_b")   # group offset k -> its tap pairs


# ------------------------------------------------------------------------------------------------ up-FIR
def xh(x, n):
    """replicate(x)[..., n] for any integer array n: x[..., clamp(n, 0, T - 1)]."""
    x = _f32(x)
    return x[..., np.clip(n, 0, x.shape[-1] - 1)]


def pair_group(i, T):
    """True where 2x-rate index i belongs to a group of 4 (starting at 1 mod 4) wholly inside [0, 2T - 1]."""
    i = np.asarray(i)
    g = i - (i - 1) % 4
    return (g >= 0) & (g + 3 <= 2 * T - 1)


def up_pair(x, i, kc):
    """u at indices i (all in pair groups) by the pair form."""
    i = np.asarray(i)
    k = (i - 1) % 4
    Q = (i - k - 1) // 2
    out = np.empty(x.shape[:-1] + i.shape, np.float32)
    for kk, key in enumerate(PAIR_KEYS):
        sel = k == kk
        if not sel.any():
            continue
        P, q0 = kc[key], Q[sel]
        lo = _f32(P[0, 0] * xh(x, q0 - 2))
        hi = _f32(P[0, 1] * xh(x, q0 - 1))
        for q in range(1, len(P)):
            lo = fma(P[q, 0], xh(x, q0 - 2 + 2 * q), lo)
            hi = fma(P[q, 1], xh(x, q0 - 1 + 2 * q), hi)
        out[..., sel] = lo + hi
    return out


def up_scalar(x, i, f_up):
    """u at indices i by the edge path's scalar chain at clamp(i, 0, 2T - 1)."""
    fu2 = _f32(f_up).reshape(12) * np.float32(2)
    ic = np.clip(np.asarray(i), 0, 2 * x.shape[-1] - 1)
    q, o = ic >> 1, ic & 1
    u = np.zeros(x.shape[:-1] + ic.shape, np.float32)
    for m in range(6):
        u = fma(np.where(o == 1, fu2[10 - 2 * m], fu2[11 - 2 * m]), xh(x, q - 3 + o + m), u)
    return u


def up(x, f_up, i=None):
    """The kernel's u [..., len(i)] at 2x-rate indices i (default all of [0, 2T)), each by the form its group takes."""
    x = _f32(x)
    T = x.shape[-1]
    i = np.arange(2 * T) if i is None else np.asarray(i)
    kc = pack(f_up, np.zeros(12, np.float32))
    pg = pair_group(i, T)
    u = np.empty(x.shape[:-1] + i.shape, np.float32)
    if pg.any():
        u[..., pg] = up_pair(x, i[pg], kc)
    if (~pg).any():
        u[..., ~pg] = up_scalar(x, i[~pg], f_up)
    return u


def up_by_segments(x, f_up):
    """The up-FIR exactly as the kernel's segments compute it: for every segment t0 = 0, 120, ..., its 64 groups at
    i0 = 2 t0 - 7 + 4 j, pair form when the group is inside [0, 2T - 1] (FAST segments: always), scalar otherwise;
    -> {(t0, n): u of window slot n} for the slots inside [0, 2T).  The check of `up`'s (i, T) rule."""
    x = _f32(x)
    T = x.shape[-1]
    kc = pack(f_up, np.zeros(12, np.float32))
    out = {}
    for t0 in range(0, T, SEG):
        fast = t0 >= 8 and t0 + 128 <= T and T % 4 == 0        # the aligned run's FAST test
        i = 2 * t0 - 7 + np.arange(256)
        n0 = i - (i - 1) % 4
        inside = fast | ((n0 >= 0) & (n0 + 3 <= 2 * T - 1))
        u = np.where(inside, up_pair(x, np.where(inside, i, 1), kc), up_scalar(x, i, f_up))
        for n in np.flatnonzero((i >= 0) & (i < 2 * T)):
            out[(t0, int(i[n]))] = u[..., n]
    return out


# ------------------------------------------------------------------------------------------------ snake
def channel_params(alpha, beta, logscale):
    """Per channel: the candidate sets of a and invb the kernel may hold ([C, n] each; n = 1 without logscale, else
    the 5 fp32 values within 2 ulp of exp)."""
    def cands(v):
        v = _f32(v)
        if not logscale:
            return v[:, None]
        e = np.exp(v.astype(np.float64)).astype(np.float32)
        lo1 = np.nextafter(e, np.float32(-np.inf)); hi1 = np.nextafter(e, np.float32(np.inf))
        return np.stack([np.nextafter(lo1, np.float32(-np.inf)), lo1, e, hi1,
                         np.nextafter(hi1, np.float32(np.inf))], 1)
    a, b = cands(alpha), cands(beta)
    invb = (np.float32(1) / (b + np.float32(1e-9))).astype(np.float32)
    return a, invb


def reduce(u, a):
    """The Cody-Waite r of snake_eval (fp32, exact)."""
    arg = _f32(u) * _f32(a)
    kf = np.rint(arg * INV_2PI).astype(np.float32)
    r = fma(-kf, TWO_PI_HI, arg)
    return fma(-kf, TWO_PI_LO, r)


def _ss_interval(s64, err):
    """fmul(s, s) over every fp32 s within err of s64 -> (lo, hi) fp32."""
    with np.errstate(over="ignore"):
        slo = np.maximum(s64 - err, -1.0).astype(np.float32)
        shi = np.minimum(s64 + err, 1.0).astype(np.float32)
    slo = np.where(slo.astype(np.float64) < s64 - err, np.nextafter(slo, np.float32(1)), slo)
    shi = np.where(shi.astype(np.float64) > s64 + err, np.nextafter(shi, np.float32(-1)), shi)
    m_hi = np.maximum(np.abs(slo), np.abs(shi))
    m_lo = np.where((slo <= 0) & (shi >= 0), np.float32(0), np.minimum(np.abs(slo), np.abs(shi)))
    return m_lo * m_lo, m_hi * m_hi


def snake_interval(u, a, invb, fast=False):
    """[lo, hi] of the kernel's v for u [..., C, n] and one candidate a, invb per channel ([C] each).  fast: MODE 2's
    pair form (no reduction, the phase error PHASE |u a| on top of the MUFU error)."""
    u = _f32(u)
    a, invb = _f32(a)[:, None], _f32(invb)[:, None]
    if fast:
        r = u * a
        err = SINF_ERR + PHASE * np.abs(r.astype(np.float64))
    else:
        r = reduce(u, a)
        err = SINF_ERR
    ss_lo, ss_hi = _ss_interval(np.sin(r.astype(np.float64)), err)
    v1, v2 = fma(invb, ss_lo, u), fma(invb, ss_hi, u)
    return np.minimum(v1, v2), np.maximum(v1, v2)


def snake_mid(u, a, invb):
    """v with __sinf replaced by sin in float64 (the reduction and the other roundings as the kernel's): the CPU
    checks' value."""
    u = _f32(u)
    a, invb = _f32(a)[:, None], _f32(invb)[:, None]
    s = np.sin(reduce(u, a).astype(np.float64)).astype(np.float32)
    return fma(invb, s * s, u)


# ------------------------------------------------------------------------------------------------ down-FIR
def down(v, f_down):
    """y [..., T] from the kernel's 2x-rate signal v [..., 2T]: two FMA chains over the fd2 pairs, then lo + hi."""
    v = _f32(v)
    T = v.shape[-1] // 2
    fd2 = pack(np.zeros(12, np.float32), f_down)["fd2"]
    base = 2 * np.arange(T) - 5
    at = lambda j: v[..., np.clip(base + j, 0, 2 * T - 1)]   # noqa: E731
    lo, hi = _f32(fd2[0, 0] * at(0)), _f32(fd2[0, 1] * at(1))
    for q in range(1, 6):
        lo = fma(fd2[q, 0], at(2 * q), lo)
        hi = fma(fd2[q, 1], at(2 * q + 1), hi)
    return lo + hi


def activation1d(x, alpha, beta, logscale, f_up, f_down):
    """The whole kernel at fp32 with snake_mid for the snake: the CPU checks' value."""
    a, invb = channel_params(alpha, beta, logscale)
    return down(snake_mid(up(x, f_up), a[:, a.shape[1] // 2], invb[:, invb.shape[1] // 2]), f_down)


def image(y, prec):
    """The operand image [B][ceil16(C)/8][T][8] (uint16) of rnd(y, prec), padding channels zero."""
    r = rnd(y, prec)
    bits = r.astype(np.float16).view(np.uint16) if prec == "f16" else (r.view(np.uint32) >> 16).astype(np.uint16)
    B, C, T = bits.shape
    c16 = (C + 15) // 16 * 16
    img = np.zeros((B, c16, T), np.uint16)
    img[:, :C] = bits
    return np.ascontiguousarray(img.reshape(B, c16 // 8, 8, T).transpose(0, 1, 3, 2))
