"""DiffWave's kernels (amphion_b200/csrc/ab_diffwave.cu) against the kernel-order oracle (tests/diffwave_exact_oracle.py),
bit for bit, through the single-launch entry points ab_diffwave_layer_forward / _tail_forward / _upsample_forward.

The gate z = sigmoid(gate) tanh(filter) is not a kernel output, and expf / tanhf cannot be restated bit for bit, so the
layer tests read z back: with first = 1, an output_projection whose skip half maps z channel c to skip channel c with
weight 1 and a zero skip bias, the skip output is z exactly at every precision (one exact product, the other terms
zeros).  A second launch with the same conv1 weights and inputs (so the same z) and the output_projection under test
is then checked against the oracle fed that z.
* One-hot conv1 (+-2^e on one (tap, channel) or mel row per gate / filter channel): the pre-activations are exact; z
  is within Z_ULPS of the float64 gate of them (fp32), and at tc_f16 / tc_bf16 the 16-bit z equals the float64 gate
  rounded once, except where the gate lies within that band of a 16-bit rounding boundary (counted, bounded).
* Residual and skip bit-equal: fp32 with a dense conv2 (the 64-term FMA chain), tensor cores with a one-hot conv2.
* A saturated gate (gate bias +30: sigmoid is exactly 1) and filter pre-activations below 2^-12 (tanh rounds to its
  argument) make z the conv1 operand itself: the padded taps (zero, not d), per-utterance and shared d, f16 subnormal
  operands, the bias fold bdil + bcond.
* f16 operands past 65504 saturate (cvt.rn.satfinite): no inf operand, no 0 * inf = NaN.
* A dense conv2 on mma.sync within the floor rule of test_resblock_exact.py of the float64 sum over the read-back z.
* The tail (eps; update with and without noise, clamped) and the upsampler (transposed mel view), dense weights.
Outputs are pre-filled with NaN, and inputs are followed by NaN so that a read past them shows."""
import ctypes as C
import fractions
import math

import numpy as np
import pytest
import torch

import diffwave_exact_oracle as dx
import resblock_oracle as ro

DEV = "cuda:0"
CH = dx.C
PRECS = {"fp32": None, "tc_f16": "f16", "tc_bf16": "bf16"}
# |z - gate64(pre)| in fp32 ulps of the gate: expf and tanhf are 2 ulp each, and the sigmoid's add, divide and the
# product round three more times; measured at most 4.5 ulp on an H100
Z_ULPS = 6
# tensor cores: share of z allowed within Z_ULPS of a 16-bit rounding boundary (about 2 Z_ULPS 2^-13 at f16: 0.15 %)
Z_EXEMPT_FRACTION = 4e-3
FLOOR_MEAN, FLOOR_MAX = 2.0, 3.0   # test_resblock_exact.py's floor rule
MMA_SYNC_MODEL = "mma"    # resblock_oracle's accumulation model that mma.sync's fp32 accumulation follows (DESIGN §5)


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def _round_fraction_f32(q):
    """A Fraction rounded to fp32, nearest, ties to even, by exact comparison with the neighbours."""
    r = np.float32(float(q))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    dist = [abs(fractions.Fraction(float(c)) - q) for c in cands]
    best = min(dist)
    ties = [c for c, dd in zip(cands, dist) if dd == best]
    return ties[0] if len(ties) == 1 else [c for c in ties if not (np.float32(c).view(np.uint32) & 1)][0]


def _fma_triples(rng):
    a = rng.normal(0, 1, 400) * np.exp2(rng.integers(-20, 20, 400))
    b = rng.normal(0, 1, 400) * np.exp2(rng.integers(-20, 20, 400))
    c = rng.normal(0, 1, 400) * np.exp2(rng.integers(-30, 30, 400))
    # adversarial: a b = +-half an ulp of c times (1 - 2^-46), so a b + c lies just off an fp32 midpoint and the
    # float64 sum rounds onto it
    c2 = (rng.normal(0, 1, 400) * np.exp2(rng.integers(-10, 10, 400))).astype(np.float32)
    half_ulp = np.spacing(np.abs(c2)).astype(np.float64) / 2
    a2 = rng.choice([-1.0, 1.0], 400) * half_ulp * (1 + 2.0 ** -23)
    b2 = np.full(400, 1 - 2.0 ** -23)
    a = np.concatenate([a, a2, [2.0 ** -24 * (1 + 2.0 ** -23)]])
    b = np.concatenate([b, b2, [1 - 2.0 ** -23]])
    c = np.concatenate([c, c2, [1 + 2.0 ** -23]])
    return a.astype(np.float32), b.astype(np.float32), c.astype(np.float32)


def test_fma_is_exactly_rounded():
    a, b, c = _fma_triples(np.random.default_rng(0))
    got = dx.fma(a, b, c)
    want = np.array([_round_fraction_f32(fractions.Fraction(float(x)) * fractions.Fraction(float(y)) +
                                         fractions.Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    naive = (a.astype(np.float64) * b + c).astype(np.float32)   # double rounding: wrong on the adversarial triples
    assert (naive != want).sum() >= 100


@pytest.mark.parametrize("f1,f2", [(4, 4), (16, 16), (2, 8)])
def test_upsample_oracle_matches_torch(f1, f2):
    rng = np.random.default_rng(f1 * f2)
    mel = rng.normal(0, 1, (2, 7, 5)).astype(np.float32)
    ws = [(rng.normal(0, 0.3, (3, 2 * f)).astype(np.float32), rng.normal(0, 0.3, 1).astype(np.float32)) for f in (f1, f2)]
    got = dx.upsample(mel, ws[0][0], ws[0][1], ws[1][0], ws[1][1], f1, f2)
    x = torch.from_numpy(mel).double()[:, None]
    for (w, b), f in zip(ws, (f1, f2)):
        x = torch.nn.functional.conv_transpose2d(x, torch.from_numpy(w).double()[None, None], torch.from_numpy(b).double(),
                                                 stride=(1, f), padding=(1, f // 2))
        x = torch.nn.functional.leaky_relu(x, 0.4)
    want = x[:, 0].numpy()
    assert got.shape == want.shape == (2, 7, 5 * f1 * f2)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


def test_layer_and_tail_oracle_match_float64_network():
    """One residual layer and the tail in kernel order against tests/diffwave_oracle.py at residual_layers = 1."""
    from diffwave_oracle import diffwave_forward
    rng = np.random.default_rng(3)
    nm, B, L, dil = 10, 2, 96, 4
    hp = dict(residual_channels=CH, residual_layers=1, dilation_cycle_length=1, upsample_factors=[4, 4])
    n = lambda *s, std=None: rng.normal(0, std if std else 1 / np.sqrt(np.prod(s[1:])), s).astype(np.float32)  # noqa: E731
    sd = {"input_projection.weight": n(CH, 1, 1), "input_projection.bias": n(CH, std=0.1),
          "diffusion_embedding.projection1.weight": n(512, 128), "diffusion_embedding.projection1.bias": n(512, std=0.1),
          "diffusion_embedding.projection2.weight": n(512, 512), "diffusion_embedding.projection2.bias": n(512, std=0.1),
          "residual_layers.0.dilated_conv.weight": n(2 * CH, CH, 3), "residual_layers.0.dilated_conv.bias": n(2 * CH, std=0.1),
          "residual_layers.0.diffusion_projection.weight": n(CH, 512),
          "residual_layers.0.diffusion_projection.bias": n(CH, std=0.1),
          "residual_layers.0.conditioner_projection.weight": n(2 * CH, nm, 1),
          "residual_layers.0.conditioner_projection.bias": n(2 * CH, std=0.1),
          "residual_layers.0.output_projection.weight": n(2 * CH, CH, 1),
          "residual_layers.0.output_projection.bias": n(2 * CH, std=0.1),
          "skip_projection.weight": n(CH, CH, 1), "skip_projection.bias": n(CH, std=0.1),
          "output_projection.weight": n(1, CH, 1), "output_projection.bias": n(1, std=0.1)}
    table = n(50, 128, std=1.0)
    audio = n(B, L, std=0.5)
    cond = n(B, nm, L, std=1.0)
    # the network's layer 0 has dilation 1; the dilated conv at `dil` is checked on its own below
    eps64, outs = diffwave_forward(sd, hp, table, audio, [3.0], None, layers_out=True, cond=cond.astype(np.float64))
    from diffwave_oracle import step_embedding
    emb = step_embedding(sd, table, [3.0])
    d = (emb @ sd["residual_layers.0.diffusion_projection.weight"].T.astype(np.float64)
         + sd["residual_layers.0.diffusion_projection.bias"]).astype(np.float32)
    x = dx.input_projection(audio, sd["input_projection.weight"], sd["input_projection.bias"])
    g = lambda k: sd["residual_layers.0." + k]  # noqa: E731
    x1, s1 = dx.layer(x, np.repeat(d, B, 0), cond, g("dilated_conv.weight"), g("dilated_conv.bias"),
                      g("conditioner_projection.weight"), g("conditioner_projection.bias"), g("output_projection.weight"),
                      g("output_projection.bias"), 1)
    x64, s64 = outs[0]
    assert np.abs(x1 - x64).max() <= 2e-6 * np.abs(x64).max()
    assert np.abs(s1 - s64).max() <= 2e-6 * np.abs(s64).max()
    eps = dx.tail(s1, sd["skip_projection.weight"], sd["skip_projection.bias"], sd["output_projection.weight"],
                  sd["output_projection.bias"], 1.0)
    assert np.abs(eps - eps64[:, 0]).max() <= 2e-6 * np.abs(eps64).max()
    # a larger dilation against a float64 restatement of the dilated conv (zero padding of x + d)
    y = x.astype(np.float64) + d.astype(np.float64)[:, :, None]
    yp = np.pad(y, ((0, 0), (0, 0), (dil, dil)))
    w = g("dilated_conv.weight").astype(np.float64)
    pre64 = sum(np.einsum("oc,bct->bot", w[:, :, j], yp[:, :, j * dil:j * dil + L]) for j in range(3))
    pre64 += np.einsum("om,bmt->bot", g("conditioner_projection.weight")[:, :, 0].astype(np.float64), cond)
    pre64 += (g("dilated_conv.bias").astype(np.float64) + g("conditioner_projection.bias"))[None, :, None]
    pre = dx.conv1_pre(dx.conv1_operands(x, np.repeat(d, B, 0), cond, dil),
                       dx.conv1_weight(g("dilated_conv.weight"), g("conditioner_projection.weight")),
                       g("dilated_conv.bias"), g("conditioner_projection.bias"), chain=True)
    assert np.abs(pre - pre64).max() <= 2e-6 * np.abs(pre64).max()


def test_tail_update_oracle():
    rng = np.random.default_rng(4)
    skip = rng.normal(0, 3, (2, CH, 50)).astype(np.float32)
    wsk, bsk = rng.normal(0, 0.125, (CH, CH)).astype(np.float32), rng.normal(0, 0.1, CH).astype(np.float32)
    wo, bo = rng.normal(0, 0.125, CH).astype(np.float32), np.float32([0.05])
    audio = rng.normal(0, 0.7, (2, 50)).astype(np.float32)
    noise = rng.normal(0, 1, (2, 50)).astype(np.float32)
    e = dx.tail(skip, wsk, bsk, wo, bo, 2.0).astype(np.float64)
    s = skip.astype(np.float64) / 2.0
    h = np.maximum(np.einsum("oc,bct->bot", wsk.astype(np.float64), s) + bsk[None, :, None], 0)
    e64 = np.einsum("o,bot->bt", wo.astype(np.float64), h) + bo[0]
    assert np.abs(e - e64).max() <= 1e-6 * np.abs(e64).max()
    got = dx.tail(skip, wsk, bsk, wo, bo, 2.0, audio=audio, c1=1.3, c2=0.4, sigma=0.3, noise=noise)
    want = np.clip(1.3 * (audio - 0.4 * e) + 0.3 * noise, -1, 1)
    assert np.abs(got - want).max() <= 1e-6 and (np.abs(got) == 1).any()


# ------------------------------------------------------------------------------------------------ the harness
def _dev(a, tail=0):
    """a (numpy) on the device, contiguous, followed by `tail` NaN floats: a read past it shows as NaN."""
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.full((a.size + tail,), float("nan"), device=DEV)
    buf[:a.size] = torch.from_numpy(a.reshape(-1)).to(DEV)
    return buf


def _ws(need):
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    return ws, C.c_void_p((ws.data_ptr() + 255) // 256 * 256)


def _run_layer(prec, x, d, cond, wdil, bdil, wcond, bcond, wout, bout, dil, first, skip_prev=None, shared_d=False):
    """One ab_diffwave_layer_forward.  d [B, C] (per utterance, batch stride C) or, shared_d, [C] (stride 0).
    -> (x_out, skip); asserts rc == 0 and that x_in is unchanged."""
    from amphion_b200 import _capi
    lib = _capi.lib
    B, _, L = x.shape
    nm = cond.shape[1]
    xd, dd, cd = _dev(x, L + 64), _dev(d, 2 * CH), _dev(cond, L + 64)
    w = [_dev(a, 64) for a in (wdil, bdil, wcond, bcond, wout, bout)]
    xo = torch.full((B, CH, L), float("nan"), device=DEV)
    sk = (torch.full((B, CH, L), float("nan"), device=DEV) if skip_prev is None
          else torch.from_numpy(np.ascontiguousarray(skip_prev, np.float32)).to(DEV))
    need = lib.ab_diffwave_layer_workspace_bytes(nm)
    ws, wsp = _ws(need)
    rc = lib.ab_diffwave_layer_forward(_capi.ptr(xd), _capi.ptr(dd), 0 if shared_d else CH, _capi.ptr(cd),
                                       *[_capi.ptr(t) for t in w], _capi.ptr(xo), _capi.ptr(sk), B, L, nm, dil, first,
                                       _capi.PRECISIONS[prec], wsp, need, _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, _capi.last_error()
    assert np.array_equal(xd[:x.size].cpu().numpy(), x.reshape(-1)), "x_in changed"
    return xo.cpu().numpy(), sk.cpu().numpy()


def _assert_equal(what, got, want):
    assert np.isfinite(want).all(), what
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


def _one_hot_conv1(rng, nm, exps, kmax=None):
    """wdil [2C, C, 3], wcond [2C, nm]: one +-2^e per output channel at a random K index of S (taps, then mel)."""
    K1 = 3 * CH + nm
    k = rng.integers(0, K1 if kmax is None else kmax, 2 * CH)
    scale = (rng.choice([-1.0, 1.0], 2 * CH) * np.exp2(rng.choice(np.asarray(exps, np.float64), 2 * CH))).astype(np.float32)
    w1 = np.zeros((2 * CH, K1), np.float32)
    w1[np.arange(2 * CH), k] = scale
    wdil = np.ascontiguousarray(np.stack([w1[:, j * CH:(j + 1) * CH] for j in range(3)], axis=2))
    return wdil, np.ascontiguousarray(w1[:, 3 * CH:]), w1


def _z_reader():
    """output_projection that copies z into the skip half: W[C + c, c] = 1, zero bias."""
    w = np.zeros((2 * CH, CH), np.float32)
    w[CH + np.arange(CH), np.arange(CH)] = 1
    return w, np.zeros(2 * CH, np.float32)


def _read_z(prec, x, dfull, cond, wdil, bdil, wcond, bcond, dil, shared_d):
    wr, br = _z_reader()
    d_in = dfull[0] if shared_d else dfull
    xo, z = _run_layer(prec, x, d_in, cond, wdil, bdil, wcond, bcond, wr, br, dil, 1, shared_d=shared_d)
    _assert_equal("x_out of the z-reading launch", xo, dx.epilogue(x, np.zeros((x.shape[0], 2 * CH, x.shape[2]),
                                                                              np.float32), br)[0])
    assert np.isfinite(z).all()
    return z


def _ulps(got, want64):
    """|got - want64| in fp32 ulps of want64 rounded to fp32."""
    w32 = np.abs(want64.astype(np.float32))
    return np.abs(got.astype(np.float64) - want64) / np.spacing(np.maximum(w32, np.float32(np.finfo(np.float32).tiny)))


def _check_z(prec, z, pre):
    """fp32: z within Z_ULPS of gate64(pre).  16-bit: z == rnd(gate64) except within Z_ULPS of a rounding boundary.
    -> (max ulps or exemptions, elements)"""
    z64 = dx.gate64(pre)
    op = PRECS[prec]
    if op is None:
        u = _ulps(z, z64)
        assert u.max() <= Z_ULPS, f"z is {u.max():.1f} ulp from the float64 gate (band {Z_ULPS})"
        return float(u.max()), z.size
    z32 = z64.astype(np.float32)
    step = np.spacing(np.abs(z32)) * Z_ULPS
    lo, hi = ro.rnd(z32 - step, op), ro.rnd(z32 + step, op)
    exempt = lo != hi
    want = ro.rnd(z32, op)
    bad = (z != want) & ~exempt
    assert not bad.any(), f"{int(bad.sum())} z differ from the rounded float64 gate, first {z[bad][0]!r} vs {want[bad][0]!r}"
    assert exempt.sum() <= Z_EXEMPT_FRACTION * z.size, (int(exempt.sum()), z.size)
    return int(exempt.sum()), z.size


# ------------------------------------------------------------------------------------------------ GPU: the layer
# (id, B, L, n_mel, dilation, shared d, first)
GEOMS = [
    ("B3-L200-m80-d1", 3, 200, 80, 1, False, 1),
    ("B3-L63-m10-d64-shared", 3, 63, 10, 64, True, 0),
    ("B2-L64-m16-d128", 2, 64, 16, 128, False, 0),
    ("B2-L65-m100-d512-shared", 2, 65, 100, 512, True, 1),
    ("B1-L1-m1-d1", 1, 1, 1, 1, False, 0),
    ("B2-L333-m100-d2", 2, 333, 100, 2, False, 0),
    ("B3-L150-m80-d512", 3, 150, 80, 512, False, 1),
]


def _inputs(rng, B, L, nm, xs=2.0, ds=0.5, ms=1.0):
    return (rng.normal(0, xs, (B, CH, L)).astype(np.float32), rng.normal(0, ds, (B, CH)).astype(np.float32),
            rng.normal(0, ms, (B, nm, L)).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_layer_one_hot_conv1(geom, prec):
    """z within the gate's band; then residual and skip bit-equal to the oracle fed the read-back z (fp32: a dense
    conv2 in the kernel's FMA order; tensor cores: a one-hot conv2, the epilogue's association, / sqrt2, bias order)."""
    name, B, L, nm, dil, shared, first = geom
    op = PRECS[prec]
    rng = np.random.default_rng(B * 1000 + L + nm + dil)
    x, d, cond = _inputs(rng, B, L, nm)
    if shared:
        d[:] = d[0]
    wdil, wcond, w1 = _one_hot_conv1(rng, nm, (-2, -1, 0, 1))
    bdil, bcond = rng.normal(0, 0.5, 2 * CH).astype(np.float32), rng.normal(0, 0.5, 2 * CH).astype(np.float32)
    z = _read_z(prec, x, d, cond, wdil, bdil, wcond, bcond, dil, shared)
    S = dx.conv1_operands(x, d, cond, dil)
    pre = dx.conv1_pre(S, w1, bdil, bcond, op)
    band, n = _check_z(prec, z, pre)
    print(f"{name} {prec}: z {'max ulps' if op is None else 'exemptions'} {band} of {n}")
    if op is None:
        wout = rng.normal(0, 1 / 8, (2 * CH, CH)).astype(np.float32)
    else:
        oh = ro.random_one_hot(rng, 2 * CH, CH, 1, (-1, 0, 1, 2))
        wout = oh.dense()[:, :, 0]
    bout = rng.normal(0, 0.3, 2 * CH).astype(np.float32)
    skip_prev = None if first else rng.normal(0, 2, (B, CH, L)).astype(np.float32)
    xo, sk = _run_layer(prec, x, d[0] if shared else d, cond, wdil, bdil, wcond, bcond, wout, bout, dil, first,
                        skip_prev=skip_prev, shared_d=shared)
    want_x, want_s = dx.layer_out(x, z, wout, bout, skip_prev, op)
    _assert_equal(f"{name} {prec} x_out", xo, want_x)
    _assert_equal(f"{name} {prec} skip", sk, want_s)


# (id, B, L, n_mel, dilation, shared d, K indices the filter channels read: taps / mel)
SATURATED = [
    ("taps-d3-L40", 2, 40, 10, 3, False),
    ("taps-d64-L63-shared", 3, 63, 16, 64, True),
    ("taps-d128-L100", 2, 100, 80, 128, False),
    ("taps-d512-L65", 2, 65, 1, 512, False),
    ("taps-d1-L130-shared", 3, 130, 100, 1, True),
]


def _saturated_layer(rng, B, L, nm, opscale, bscale, subnormal=False):
    x = (rng.normal(0, opscale, (B, CH, L))).astype(np.float32)
    d = (rng.normal(0, opscale, (B, CH))).astype(np.float32)
    cond = (rng.normal(0, opscale, (B, nm, L))).astype(np.float32)
    wdil, wcond, w1 = _one_hot_conv1(rng, nm, (0,))
    bdil = np.concatenate([np.full(CH, 30.0), rng.normal(0, bscale, CH)]).astype(np.float32)
    bcond = np.concatenate([np.zeros(CH), rng.normal(0, bscale, CH)]).astype(np.float32)
    return x, d, cond, wdil, wcond, w1, bdil, bcond


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", SATURATED, ids=[c[0] for c in SATURATED])
def test_layer_saturated_gate_reads_exact_operands(case, prec):
    """Gate bias +30 and |filter| < 2^-12: z is the filter pre-activation itself, rnd(S[k]) * +-1 + (bdil + bcond),
    exactly: every tap (zero where it pads, not d), every mel row, d per utterance or shared, the bias fold."""
    name, B, L, nm, dil, shared = case
    op = PRECS[prec]
    rng = np.random.default_rng(L * 7 + dil)
    x, d, cond, wdil, wcond, w1, bdil, bcond = _saturated_layer(rng, B, L, nm, 2e-5, 1e-5)
    if shared:
        d[:] = d[0]
    z = _read_z(prec, x, d, cond, wdil, bdil, wcond, bcond, dil, shared)
    pre = dx.conv1_pre(dx.conv1_operands(x, d, cond, dil), w1, bdil, bcond, op)
    assert np.abs(pre[:, CH:]).max() < 2.0 ** -12
    _assert_equal(f"{name} {prec} z", z, ro.rnd(pre[:, CH:], op))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_layer_subnormal_f16_operands(prec):
    """Operands of ~1e-6 (f16 subnormals below 2^-14) and no filter bias: z = rnd(S[k]) * 2^e through both mma.sync
    products, conv1's A operand and conv2's z; mma.sync keeps f16 subnormals (does not flush them)."""
    rng = np.random.default_rng(11)
    B, L, nm, dil = 2, 130, 16, 2
    x, d, cond, wdil, wcond, w1, bdil, bcond = _saturated_layer(rng, B, L, nm, 1e-6, 0.0)
    z = _read_z(prec, x, d, cond, wdil, bdil, wcond, bcond, dil, False)
    S = dx.conv1_operands(x, d, cond, dil)
    want = ro.rnd(dx.conv1_pre(S, w1, bdil, bcond, PRECS[prec])[:, CH:], PRECS[prec])
    if prec == "tc_f16":
        sub = (want != 0) & (np.abs(want) < 2.0 ** -14)
        assert sub.mean() > 0.5, "the case must put most operands in the f16 subnormal range"
    _assert_equal(f"subnormal {prec} z", z, want)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_layer_saturating_operands(prec):
    """|x + d| and mel values past 65504: the f16 operands saturate to +-65504 (cvt.rn.satfinite), so no inf meets the
    zero weights of its k16 block (0 * inf = NaN in every output column of the row).  bf16 covers the same values."""
    name, B, L, nm, dil = "saturation", 2, 200, 10, 3
    op = PRECS[prec]
    rng = np.random.default_rng(13)
    x, d, cond = _inputs(rng, B, L, nm, xs=1e5, ds=3e4, ms=1e5)
    wdil, wcond, w1 = _one_hot_conv1(rng, nm, (-18, -17, -16))
    bdil, bcond = rng.normal(0, 0.5, 2 * CH).astype(np.float32), rng.normal(0, 0.5, 2 * CH).astype(np.float32)
    S = dx.conv1_operands(x, d, cond, dil)
    assert (np.abs(S) > 65504).mean() > 0.3
    z = _read_z(prec, x, d, cond, wdil, bdil, wcond, bcond, dil, False)
    _check_z(prec, z, dx.conv1_pre(S, w1, bdil, bcond, op))
    oh = ro.random_one_hot(rng, 2 * CH, CH, 1, (-1, 0, 1))
    bout = rng.normal(0, 0.3, 2 * CH).astype(np.float32)
    xo, sk = _run_layer(prec, x, d, cond, wdil, bdil, wcond, bcond, oh.dense()[:, :, 0], bout, dil, 1)
    want_x, want_s = dx.layer_out(x, z, oh.dense()[:, :, 0], bout, None, op)
    _assert_equal(f"{name} {prec} x_out", xo, want_x)
    _assert_equal(f"{name} {prec} skip", sk, want_s)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_layer_dense_conv2_floor(prec):
    """mma.sync's fp32 accumulation of a dense conv2 over the read-back z: the skip half (zero skip bias) within the
    floor rule of the float64 sum, the floor being MMA_SYNC_MODEL's accumulation (k16 steps in K order)."""
    op = PRECS[prec]
    rng = np.random.default_rng(17)
    B, L, nm, dil = 3, 300, 80, 4
    x, d, cond = _inputs(rng, B, L, nm)
    wdil, wcond, _ = _one_hot_conv1(rng, nm, (-1, 0, 1))
    bdil, bcond = rng.normal(0, 0.5, 2 * CH).astype(np.float32), rng.normal(0, 0.5, 2 * CH).astype(np.float32)
    z = _read_z(prec, x, d, cond, wdil, bdil, wcond, bcond, dil, False)
    wout = rng.normal(0, 1 / 8, (2 * CH, CH)).astype(np.float32)
    bout = np.concatenate([rng.normal(0, 0.3, CH), np.zeros(CH)]).astype(np.float32)
    xo, sk = _run_layer(prec, x, d, cond, wdil, bdil, wcond, bcond, wout, bout, dil, 1)
    w16 = ro.rnd(wout, op)[:, :, None]
    o64 = {acc: ro.conv(z, w16, 1, acc)[:, CH:] for acc in ("f64", "f32", "mma")}
    ratios = {}
    for acc in ("f32", "mma"):
        e_mean, e_max, f_mean, f_max = ro.floor_stats(sk, o64["f64"].astype(np.float64), o64[acc])
        ratios[acc] = (e_mean / f_mean, e_max / f_max)
        print(f"dense conv2 {prec} against the {acc} floor: mean {e_mean:.3e} = {e_mean / f_mean:.2f} x floor, "
              f"max {e_max:.3e} = {e_max / f_max:.2f} x floor")
    assert np.isfinite(xo).all()
    m_mean, m_max = ratios[MMA_SYNC_MODEL]
    assert m_mean <= FLOOR_MEAN and m_max <= FLOOR_MAX, ratios


# ------------------------------------------------------------------------------------------------ GPU: tail, upsampler
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["eps", "update", "update-noise"])
def test_tail_is_exact(mode):
    from amphion_b200 import _capi
    rng = np.random.default_rng(len(mode))
    B, L, skip_div = 3, 517, float(np.float32(math.sqrt(30)))
    skip = rng.normal(0, 4, (B, CH, L)).astype(np.float32)
    wsk, bsk = rng.normal(0, 0.125, (CH, CH)).astype(np.float32), rng.normal(0, 0.1, CH).astype(np.float32)
    wo, bo = rng.normal(0, 0.25, CH).astype(np.float32), rng.normal(0, 0.1, 1).astype(np.float32)
    audio = rng.normal(0, 0.8, (B, L)).astype(np.float32)
    noise = rng.normal(0, 1, (B, L)).astype(np.float32) if mode == "update-noise" else None
    c1, c2, sigma = 1.02, 0.35, 0.4
    sd, ws_ = _dev(skip, 64), [_dev(a, 64) for a in (wsk, bsk, wo, bo)]
    a_dev = torch.from_numpy(audio).to(DEV)
    eps = torch.full((B, L), float("nan"), device=DEV) if mode == "eps" else None
    nd = None if noise is None else torch.from_numpy(noise).to(DEV)
    rc = _capi.lib.ab_diffwave_tail_forward(_capi.ptr(sd), *[_capi.ptr(t) for t in ws_], skip_div, B, L, _capi.ptr(eps),
                                            _capi.ptr(a_dev), _capi.ptr(nd), c1, c2, sigma, _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, _capi.last_error()
    if mode == "eps":
        _assert_equal("eps", eps.cpu().numpy(), dx.tail(skip, wsk, bsk, wo, bo, skip_div))
        assert np.array_equal(a_dev.cpu().numpy(), audio)
        return
    want = dx.tail(skip, wsk, bsk, wo, bo, skip_div, audio=audio, c1=c1, c2=c2, sigma=sigma, noise=noise)
    assert (np.abs(want) == 1).mean() > 0.01, "the case must clamp"
    _assert_equal(mode, a_dev.cpu().numpy(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("f1,f2", [(16, 16), (4, 4), (2, 6)])
def test_upsample_is_exact(f1, f2):
    from amphion_b200 import _capi
    rng = np.random.default_rng(f1 + f2)
    B, nm, F = 2, 100, 9
    mel_t = rng.normal(0, 1, (B, F, nm)).astype(np.float32)
    mel = torch.from_numpy(mel_t).to(DEV).transpose(1, 2)               # [B, n_mel, F] view, strides (F nm, 1, nm)
    ws = [rng.normal(0, 0.3, s).astype(np.float32) for s in ((3, 2 * f1), (1,), (3, 2 * f2), (1,))]
    wd = [_dev(a, 16) for a in ws]
    out = torch.full((B, nm, F * f1 * f2), float("nan"), device=DEV)
    rc = _capi.lib.ab_diffwave_upsample_forward(_capi.ptr(mel), _capi.shape_array(mel.stride()), *[_capi.ptr(t) for t in wd],
                                                f1, f2, B, nm, F, _capi.ptr(out), _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, _capi.last_error()
    _assert_equal(f"upsample {f1}x{f2}", out.cpu().numpy(), dx.upsample(mel_t.transpose(0, 2, 1), *ws[:2], *ws[2:], f1, f2))
