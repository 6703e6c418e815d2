"""Operand-rounded restatement of the tensor-core ResBlock path (`hpair_kernel`, `hchain_kernel`, `hconv_kernel` in
amphion_b200/csrc/ab_kernels_tc.cu, sequenced by `forward_impl` in ab_capi.cu), the checker of the fused kernels at
the bit level.  numpy only: it imports nothing of the product.

One ResBlock1 step (dilation pair p of block j), every value fp32 unless stated:
    a       = rnd(lrelu(x_p, 0.1))                 the operand loader
    h       = f32(conv1(a, rnd(W1), d)) + b1       conv1's accumulator, then the intermediate-tile store
    m       = rnd(lrelu(h, 0.1)), zero outside [0, T)
    x_{p+1} = (f32(conv2(m, rnd(W2))) + b2) + x_p  add_terms / the block-mode residual update
then on the last pair `+ acc_prev` (the branch sum, blocks j > 0) and on the last block `* (1.0f / nk)`
(epilogue_out).  ResBlock2 drops conv2: x_{p+1} = (f32(conv1(a, rnd(W1), d)) + b1) + x_p.  No multiply feeds an add in
these epilogues, so there is no fused multiply-add to mirror.

`rnd` is `cvt.rn.satfinite`: clamp to the largest finite value of the 16-bit type, then round to nearest even.
`f32(conv)` is the accumulation, in the kernels' order (32-channel K chunk -> tap -> 16-channel half):
  "f64"  sums in float64 (exact enough) and rounds once;
  "f32"  sums in IEEE float32, the 16-term partial sums left to BLAS: one more valid fp32 order;
  "mma"  adds each 16-term partial sum exactly and truncates the accumulator to fp32 (round toward zero), a model of
         the H100's wgmma accumulation: on a single dense conv it matches the measured error to 1.1-1.3x, with the
         same 84 % of errors toward zero, where IEEE float32 sits 3-15x closer to the exact sum (DESIGN.md §5).
With one-hot weights (`OneHot`) every output is one exact product, so every order gives the same bits and the
convolution is a gather.  `conv_transpose` and `OneHotT` are the same for the ConvTranspose layers (`hconv_kernel`
from fp32 input, `hitem_kernel` from an operand image), and `image_bits` / `to_image` give the operand images."""
from __future__ import annotations

import numpy as np

F16_MAX = np.float32(65504.0)
BF16_MAX = np.uint32(0x7F7F0000).view(np.float32)
SLOPE = 0.1


def rnd(v, prec):
    """fp32 -> the 16-bit operand type ("f16", "bf16") and back, saturating; None: unchanged."""
    v = np.asarray(v, np.float32)
    if prec is None:
        return v
    if prec == "f16":
        return np.clip(v, -F16_MAX, F16_MAX).astype(np.float16).astype(np.float32)
    assert prec == "bf16", prec
    u = np.clip(v, -BF16_MAX, BF16_MAX).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def lrelu(v, slope):
    """fmaxf(v, v * slope) in fp32, as the loaders and epilogues compute it."""
    v = np.asarray(v, np.float32)
    return np.maximum(v, v * np.float32(slope))


class OneHot:
    """A conv weight [C_out, C_in, k] with one non-zero per output channel: W[co, perm[co], tap[co]] = scale[co]."""

    def __init__(self, perm, tap, scale, cin, k):
        self.perm, self.tap = np.asarray(perm, np.int64), np.asarray(tap, np.int64)
        self.scale, self.cin, self.k = np.asarray(scale, np.float32), int(cin), int(k)

    @property
    def shape(self):
        return (len(self.perm), self.cin, self.k)

    def dense(self):
        w = np.zeros(self.shape, np.float32)
        w[np.arange(len(self.perm)), self.perm, self.tap] = self.scale
        return w

    def rounded(self, prec):
        return OneHot(self.perm, self.tap, rnd(self.scale, prec), self.cin, self.k)


def random_one_hot(rng, cout, cin, k, exps):
    """perm: a random permutation (cout == cin) or random channels; tap: random; scale: +-2^e, e drawn from exps."""
    perm = rng.permutation(cin)[:cout] if cout <= cin else rng.integers(0, cin, cout)
    scale = rng.choice([-1.0, 1.0], cout) * np.exp2(rng.choice(np.asarray(exps, np.float64), cout))
    return OneHot(perm, rng.integers(0, k, cout), scale, cin, k)


def _round_w(w, prec):
    return w.rounded(prec) if isinstance(w, OneHot) else rnd(w, prec)


def conv(a, w, d, acc="f64", reflect=False):
    """'same' Conv1d without bias of the operand a [B, C_in, T] (any strides) with w (dense [C_out, C_in, k] or
    OneHot), dilation d, summed as `acc` says and rounded to fp32 once: [B, C_out, T] float32.  reflect: ReflectionPad1d
    ((k-1) d / 2) in place of the zero padding, zero where the reflected time is outside [0, T) too."""
    a = np.asarray(a, np.float32)
    B, cin, T = a.shape
    k = w.shape[2]
    h = (k - 1) * d // 2
    ap = np.zeros((B, cin, T + 2 * h), np.float32)
    if reflect:
        t = np.arange(-h, T + h)
        t = np.where(t < 0, -t, np.where(t >= T, 2 * (T - 1) - t, t))
        ok = (t >= 0) & (t < T)
        ap[:, :, ok] = a[:, :, t[ok]]
    else:
        ap[:, :, h:h + T] = a
    if isinstance(w, OneHot):
        idx = w.tap[:, None] * d + np.arange(T)[None, :]                 # [C_out, T]
        return (ap[:, w.perm[:, None], idx].astype(np.float64) * w.scale[None, :, None]).astype(np.float32)
    w = np.asarray(w, np.float32)
    if acc == "f64":
        w64, ap64 = w.astype(np.float64), ap.astype(np.float64)
        y = sum(np.matmul(w64[:, :, j], ap64[:, :, j * d:j * d + T]) for j in range(k))
        return y.astype(np.float32)
    assert acc in ("f32", "mma"), acc
    y = np.zeros((B, w.shape[0], T), np.float32)
    w64, ap64 = (w.astype(np.float64), ap.astype(np.float64)) if acc == "mma" else (None, None)
    for c0 in range(0, cin, 32):                                         # K chunk
        for j in range(k):                                               # tap
            for c1 in range(c0, min(c0 + 32, cin), 16):                  # k16 half
                if acc == "f32":
                    y += np.matmul(w[:, c1:c1 + 16, j], ap[:, c1:c1 + 16, j * d:j * d + T])
                else:
                    y = _to_f32_rz(y + np.matmul(w64[:, c1:c1 + 16, j], ap64[:, c1:c1 + 16, j * d:j * d + T]))
    return y


def _to_f32_rz(v):
    """float64 -> float32 rounded toward zero."""
    r = v.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(v)
    r[over] = np.nextafter(r[over], np.float32(0))
    return r


class OneHotT:
    """A ConvTranspose weight [C_in, C_out, k] of stride u with one non-zero per (output channel co, phase phi):
    W[ci[co, phi], co, phi + u m[co, phi]] = scale[co, phi].  Output t = s u - pad + phi is then one product,
    act(x)[ci, s - m] * scale (zero where s - m is outside [0, T))."""

    def __init__(self, ci, m, scale, cin, u, k):
        self.ci, self.m = np.asarray(ci, np.int64), np.asarray(m, np.int64)
        self.scale, self.cin, self.u, self.k = np.asarray(scale, np.float32), int(cin), int(u), int(k)

    @property
    def shape(self):
        return (self.cin, self.ci.shape[0], self.k)

    def dense(self):
        w = np.zeros(self.shape, np.float32)
        co, phi = np.meshgrid(np.arange(self.ci.shape[0]), np.arange(self.u), indexing="ij")
        w[self.ci, co, phi + self.u * self.m] = self.scale
        return w

    def rounded(self, prec):
        return OneHotT(self.ci, self.m, rnd(self.scale, prec), self.cin, self.u, self.k)


def random_one_hot_t(rng, cin, cout, k, u, exps):
    """ci: random channels; m: a random tap of the phase (phi + u m < k); scale: +-2^e, e drawn from exps."""
    taps = (k - np.arange(u) + u - 1) // u                             # taps m of phase phi
    m = np.minimum((rng.random((cout, u)) * taps[None, :]).astype(np.int64), taps[None, :] - 1)
    scale = rng.choice([-1.0, 1.0], (cout, u)) * np.exp2(rng.choice(np.asarray(exps, np.float64), (cout, u)))
    return OneHotT(rng.integers(0, cin, (cout, u)), m, scale, cin, u, k)


def conv_transpose(a, w, u, pad, acc="f64"):
    """ConvTranspose1d without bias of a [B, C_in, T] with w (dense [C_in, C_out, k] or OneHotT), stride u, padding pad
    in [0, k), T_out = T * u: torch's conv_transpose1d with output_padding u + 2 pad - k where that is in [0, u).
    Output t = s u - pad + phi sums the taps m of phase phi (k index phi + u m) over input time s - m; "mma" and "f32"
    in the kernels' order, 32-channel K chunk -> tap m -> 16-channel half."""
    a = np.asarray(a, np.float32)
    B, cin, T = a.shape
    k, Tout = w.shape[2], T * u
    if isinstance(w, OneHotT):
        q = np.arange(Tout) + pad
        s, phi = q // u, q % u
        src = s[None, :] - w.m[:, phi]                                   # [C_out, T_out]
        ok = (src >= 0) & (src < T)
        g = a[:, w.ci[:, phi], np.clip(src, 0, T - 1)].astype(np.float64) * w.scale[None, :, phi]
        return np.where(ok[None], g, 0.0).astype(np.float32)
    w = np.asarray(w, np.float32)
    cout = w.shape[1]
    full_len = max((T - 1) * u + k, pad + Tout)     # position s u + j of input time s and k index j
    if acc == "f64":
        w64, a64 = w.astype(np.float64), a.astype(np.float64)
        full = np.zeros((B, cout, full_len))
        for j in range(k):
            full[:, :, j:j + (T - 1) * u + 1:u] += np.matmul(w64[:, :, j].T, a64)
        return full[:, :, pad:pad + Tout].astype(np.float32)
    assert acc in ("f32", "mma"), acc
    dt = np.float32 if acc == "f32" else np.float64
    full = np.zeros((B, cout, full_len), np.float32)
    for c0 in range(0, cin, 32):                                         # K chunk
        for m in range((k + u - 1) // u):                                # tap
            for c1 in range(c0, min(c0 + 32, cin), 16):                  # k16 half
                for phi in range(u):                                     # disjoint outputs
                    j = phi + u * m
                    if j >= k:
                        continue
                    s = slice(j, j + (T - 1) * u + 1, u)
                    part = np.matmul(np.asarray(w[c1:c1 + 16, :, j], dt).T, np.asarray(a[:, c1:c1 + 16], dt))
                    full[:, :, s] = (full[:, :, s] + part if acc == "f32"
                                     else _to_f32_rz(full[:, :, s].astype(np.float64) + part))
    return full[:, :, pad:pad + Tout]


def image_bits(v, slope, prec):
    """The 16-bit patterns (uint16) of rnd(lrelu(v, slope), prec): the values an operand image holds."""
    r = rnd(lrelu(v, slope), prec)
    if prec == "f16":
        return r.astype(np.float16).view(np.uint16)
    assert prec == "bf16", prec
    return (r.view(np.uint32) >> 16).astype(np.uint16)


def to_image(bits):
    """[B, C, T] uint16 -> the operand-image layout [B][ceil16(C)/8][T][8], padding channels zero."""
    B, C, T = bits.shape
    c16 = (C + 15) // 16 * 16
    img = np.zeros((B, c16, T), np.uint16)
    img[:, :C] = bits
    return np.ascontiguousarray(img.reshape(B, c16 // 8, 8, T).transpose(0, 1, 3, 2))


def from_image(img, C):
    """The inverse of to_image: [B][c8][T][8] -> [B, C, T] (and the padding channels as [B, c16 - C, T])."""
    B, c8n, T, _ = img.shape
    full = np.asarray(img).transpose(0, 1, 3, 2).reshape(B, c8n * 8, T)
    return full[:, :C], full[:, C:]


def block(k, dils, c1, c2=None):
    """One ResBlock: kernel size k, dilations, conv1 (W, b) per dilation and conv2 (W, b) per dilation (ResBlock1)
    or None (ResBlock2)."""
    return dict(k=k, dils=list(dils), c1=list(c1), c2=None if c2 is None else list(c2))


def stage(x, blocks, prec, acc="f64"):
    """One stage's ResBlocks on the stage input x [B, C, T]: (sum_j block_j(x)) * (1 / nk) in the tensor path's order."""
    x = np.asarray(x, np.float32)
    nk = len(blocks)
    out = None
    for j, blk in enumerate(blocks):
        cur = x
        for p, d in enumerate(blk["dils"]):
            w1, b1 = blk["c1"][p]
            a = rnd(lrelu(cur, SLOPE), prec)
            h = conv(a, _round_w(w1, prec), d, acc) + np.asarray(b1, np.float32)[None, :, None]
            if blk["c2"] is not None:
                w2, b2 = blk["c2"][p]
                m = rnd(lrelu(h, SLOPE), prec)
                h = conv(m, _round_w(w2, prec), 1, acc) + np.asarray(b2, np.float32)[None, :, None]
            cur = h + cur
        if j > 0:
            cur = cur + out
        if j == nk - 1:
            cur = cur * (np.float32(1.0) / np.float32(nk))
        out = cur
    return out


def hifigan_blocks(params, prefix, k, dils, resblock):
    """block() of the state-dict entries `<prefix>.convs1.p` / `.convs2.p` (ResBlock1) or `.convs.p` (ResBlock2),
    plain (weight-norm removed) weights."""
    g = lambda n: (np.asarray(params[n + ".weight"], np.float32), np.asarray(params[n + ".bias"], np.float32))  # noqa: E731
    if str(resblock) == "1":
        return block(k, dils, [g(f"{prefix}.convs1.{p}") for p in range(len(dils))],
                     [g(f"{prefix}.convs2.{p}") for p in range(len(dils))])
    return block(k, dils, [g(f"{prefix}.convs.{p}") for p in range(len(dils))])


def hifigan(params, hp, mel, prec, acc="f64"):
    """HiFi-GAN generator on the tensor path (DESIGN.md §4.1): conv_pre on the tensor cores from the unactivated mel;
    each ConvTranspose from rnd(lrelu(x, 0.1)) (the operand image its producer emits holds exactly that); the stages
    as stage(); conv_post (C -> 1) exact in fp32 on lrelu(x, 0.01), then tanh.  params: plain weights.  -> [B, 1, L]."""
    f = lambda n: np.asarray(params[n], np.float32)  # noqa: E731
    x = conv(rnd(mel, prec), rnd(f("conv_pre.weight"), prec), 1, acc) + f("conv_pre.bias")[None, :, None]
    nk = len(hp["resblock_kernel_sizes"])
    for i, (u, ku) in enumerate(zip(hp["upsample_rates"], hp["upsample_kernel_sizes"])):
        a = rnd(lrelu(x, SLOPE), prec)
        x = conv_transpose(a, rnd(f(f"ups.{i}.weight"), prec), u, (ku - u) // 2, acc) + f(f"ups.{i}.bias")[None, :, None]
        blocks = [hifigan_blocks(params, f"resblocks.{i * nk + j}", k, d, hp["resblock"])
                  for j, (k, d) in enumerate(zip(hp["resblock_kernel_sizes"], hp["resblock_dilation_sizes"]))]
        x = stage(x, blocks, prec, acc)
    y = conv(lrelu(x, 0.01), f("conv_post.weight"), 1, "f64" if acc == "f64" else "f32") + f("conv_post.bias")[None, :, None]
    return np.tanh(y.astype(np.float64)).astype(np.float32)


def floor_stats(got, o64, o32):
    """(mean, max) of |got - o64| and of the floor |o32 - o64| (o32: a float32-accumulation order)."""
    e, fl = np.abs(np.asarray(got, np.float64) - o64), np.abs(np.asarray(o32, np.float64) - o64)
    return float(e.mean()), float(e.max()), float(fl.mean()), float(fl.max())
