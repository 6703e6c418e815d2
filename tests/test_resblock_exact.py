"""The fused ResBlock kernels against the operand-rounded oracle (tests/resblock_oracle.py).

GPU harness: an `AB_GEN_TRUNK` handle (`_Stage`) with n_mel = C = trunk_out_channels and 1-tap conv_pre / conv_post.
Those two have C_in == C_out and so run on the exact fp32 CUDA-core kernel; loaded as identity matrices with zero
bias, the stage sees the test's fp32 input exactly and the handle returns lrelu(stage output, 0.01) exactly.  The
ResBlock convs are plain tensors (no weight-norm fold), so the only rounding is the tensor path's own.

* One-hot weights (output channel co reads input channel perm(co) at tap tap(co), scale +-2^e): every accumulator
  holds one exact product, so the whole stage is deterministic and every route — pairs (`resblock_fusion` 1), block
  mode (2, 3) and the single-conv route (C = 320, k = 33) — must equal the oracle bit for bit.  That pins tap shifts
  and dilations, halos, ragged tiles, K-chunk / N-block mapping, padded channels, zeroing outside [0, T), bias
  placement, epilogue association, RN rounding and saturation.
* Dense weights: the kernels' distance from the float64-accumulation oracle against the floor, the distance from it
  of the oracle with the H100 MMA's truncating fp32 accumulation ("mma" in resblock_oracle.py; IEEE float32 sits
  3-15x closer to the exact sum than the tensor cores do, so it would understate the floor).  This covers
  accumulation over all K chunks and taps.
* Whole HiFi-GAN generators (ResBlock1 and ResBlock2) under the same floor rule.

Not covered: a change of the fp32 accumulation order alone.  One-hot weights make every order give the same bits, and
with dense weights such a change moves the output by about the floor, which the floor rule admits.  (For the
ConvTranspose layers, test_tc_conv_exact.py compares `hitem_kernel` with `hconv_kernel` bit for bit on dense weights,
which catches such a change in either kernel.)"""
import numpy as np
import pytest
import torch

import resblock_oracle as ro

DEV = "cuda:0"
PRECS = {"tc_f16": "f16", "tc_bf16": "bf16"}
ROUTES = (1, 2, 3)   # resblock_fusion
# floor rule: the kernel's distance from the float64 oracle within these multiples of the floor's mean and maximum
FLOOR_MEAN, FLOOR_MAX = 2.0, 3.0


# ------------------------------------------------------------------------------------------------ routing restated
def _nw(C):
    n = 16
    while n < (C + 15) // 16 * 16:
        n *= 2
    return min(n, 256)


def _chain_recompute(C, k, dils, nconv):
    """tc_chain_recompute (ab_kernels_tc.cu): tile rows per output row of block mode, 0 where it cannot serve."""
    nw = _nw(C)
    if len(dils) > 3 or nw > 128:
        return 0.0
    R = 2 * (1 if nw >= 128 else 2 if nw == 64 else 4) * 64
    H = sum((k - 1) * d // 2 + ((k - 1) // 2 if nconv == 2 else 0) for d in dils)
    G = max((k - 1) * d // 2 for d in dils)
    V = R - 2 * H
    rows = (R + 2 * G + 7) // 8 * 8
    xbytes = (C + 31) // 32 * 64 * rows
    off_w = ((xbytes + 127) // 128 * 128 + xbytes + 127) // 128 * 128
    fixed = off_w + len(dils) * nconv * nw * 4 + 16 + 112
    if V < 8 or rows > 16383 or fixed + 2 * 64 * nw > 227 * 1024:
        return 0.0
    return R / V


def _launches(C, shape, fusion, nconv=2):
    """Launches of the trunk forward: conv_pre, each block's (one per block in block mode, one per pair, or one per
    conv on the single-conv route), conv_post."""
    n = 2
    for k, dils in shape:
        if not (C <= 256 and k <= 31):
            n += nconv * len(dils)
            continue
        rec = _chain_recompute(C, k, dils, nconv) if fusion >= 2 else 0.0
        n += 1 if rec > 0 and (fusion >= 3 or rec <= 1.5) else len(dils)
    return n


# ------------------------------------------------------------------------------------------------ the harness
def _stage_class():
    from amphion_b200 import _capi
    from amphion_b200.vocoders.generator import NativeGenerator

    class _Stage(NativeGenerator):
        """One ResBlock1 stage between identity conv_pre / conv_post on a trunk handle; tensors: name -> CPU tensor."""
        kind = "trunk"

        def __init__(self, C, shape, tensors):
            super().__init__()
            self._C, self._shape, self._tensors = C, shape, tensors

        def _c_config(self):
            c = _capi.GeneratorConfig()
            c.kind, c.n_mel, c.upsample_initial_channel, c.num_upsamples, c.resblock = _capi.GEN_TRUNK, self._C, self._C, 0, 1
            c.num_kernels = len(self._shape)
            for j, (k, ds) in enumerate(self._shape):
                c.resblock_kernel_sizes[j], c.num_dilations[j] = k, len(ds)
                for p, d in enumerate(ds):
                    c.resblock_dilation_sizes[j][p] = d
            c.activation = _capi.ACT_LRELU
            c.trunk_out_channels, c.trunk_in_kernel, c.trunk_out_kernel = self._C, 1, 1
            return c

        def named_parameters(self, *a, **k):
            return iter(self._tensors.items())

        def parameters(self, *a, **k):
            return iter(self._tensors.values())

        def named_buffers(self, *a, **k):
            return iter(())

        def buffers(self, *a, **k):
            return iter(())

        def run(self, x, prec, fusion):
            """x [B, C, T] -> (lrelu(stage(x), 0.01) [B, C, T] on the host, launches)"""
            import ctypes as C
            self.precision = prec
            self.set_option("resblock_fusion", fusion)
            x = torch.from_numpy(x).to(DEV)
            B, _, T = x.shape
            with torch.cuda.device(x.device):
                self._sync_params(x.device)
                lib, h = _capi.lib, self._handle
                need = lib.ab_generator_workspace_bytes(h, B, T)
                ws = torch.empty(need + 256, dtype=torch.uint8, device=x.device)
                out = torch.empty(B, self._C, T, dtype=torch.float32, device=x.device)
                _capi.check(lib.ab_generator_forward(h, _capi.ptr(x), B, T, _capi.shape_array(x.stride()), _capi.ptr(out),
                                                     C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need,
                                                     _capi.stream_ptr()), "ab_generator_forward")
                launches = lib.ab_generator_last_launches(h)
            return out.cpu().numpy(), launches

    return _Stage


def _make_stage(C, blocks):
    eye = torch.eye(C, dtype=torch.float32)[:, :, None]
    t = {"conv_pre.weight": eye, "conv_pre.bias": torch.zeros(C), "conv_post.weight": eye.clone(),
         "conv_post.bias": torch.zeros(C)}
    for j, blk in enumerate(blocks):
        for p in range(len(blk["dils"])):
            for name, (w, b) in (("convs1", blk["c1"][p]), ("convs2", blk["c2"][p])):
                w = w.dense() if isinstance(w, ro.OneHot) else w
                t[f"resblocks.{j}.{name}.{p}.weight"] = torch.from_numpy(np.ascontiguousarray(w, np.float32))
                t[f"resblocks.{j}.{name}.{p}.bias"] = torch.from_numpy(np.asarray(b, np.float32))
    return _stage_class()(C, [(blk["k"], tuple(blk["dils"])) for blk in blocks], t)


def _blocks(rng, C, shape, weights, exps=(-2, -1, 0, 1), bias_std=0.5):
    def conv(k):
        if weights == "one-hot":
            return ro.random_one_hot(rng, C, C, k, exps), rng.normal(0, bias_std, C).astype(np.float32)
        w = rng.normal(0, 1 / np.sqrt(C * k), (C, C, k)).astype(np.float32)
        return w, rng.normal(0, bias_std, C).astype(np.float32)
    return [ro.block(k, d, [conv(k) for _ in d], [conv(k) for _ in d]) for k, d in shape]


def _post(v):
    return ro.lrelu(v, 0.01)


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def test_rnd_is_saturating_round_to_nearest_even():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.normal(0, 1, 4000), rng.normal(0, 1e-5, 2000), rng.normal(0, 3e4, 2000),
                        # exact ties of f16 (1 + 2^-11) and bf16 (1 + 2^-8, 1 + 3 * 2^-8)
                        [1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8)]]).astype(np.float32)
    t = torch.from_numpy(v)
    ok = np.abs(v) <= 65504
    assert np.array_equal(ro.rnd(v, "f16")[ok], t.half().float().numpy()[ok])
    assert np.array_equal(ro.rnd(v, "bf16"), t.bfloat16().float().numpy())
    assert np.array_equal(ro.rnd(np.float32([1e5, -7e4, 65519, 65520]), "f16"), np.float32([65504, -65504, 65504, 65504]))
    fmax = np.finfo(np.float32).max
    assert np.array_equal(ro.rnd(np.float32([fmax, -fmax]), "bf16"), np.float32([ro.BF16_MAX, -ro.BF16_MAX]))
    assert ro.rnd(np.float32([2 ** -24, 3 * 2 ** -26]), "f16").tolist() == [2 ** -24, 2 ** -24]   # f16 subnormals


@pytest.mark.parametrize("C,k,d", [(40, 7, 3), (16, 1, 1), (130, 11, 5)])
def test_one_hot_gather_equals_dense_conv(C, k, d):
    rng = np.random.default_rng(C)
    a = ro.rnd(rng.normal(0, 1, (2, C, 57)), "f16")
    w = ro.random_one_hot(rng, C, C, k, (-3, 0, 2))
    want = ro.conv(a, w, d)
    for acc in ("f64", "f32", "mma"):
        assert np.array_equal(ro.conv(a, w.dense(), d, acc), want), acc


def test_f32_twin_is_ieee_fp32():
    """One 128-channel, k = 11 conv: the float32-accumulation twin sits about 1e-7 (relative) from float64."""
    rng = np.random.default_rng(1)
    a = ro.rnd(rng.normal(0, 1, (2, 128, 300)), "f16")
    w = ro.rnd(rng.normal(0, 1 / np.sqrt(128 * 11), (128, 128, 11)), "f16")
    c64, c32 = ro.conv(a, w, 3, "f64"), ro.conv(a, w, 3, "f32")
    rel = float(np.abs(c32.astype(np.float64) - c64).mean() / np.abs(c64).mean())
    assert 1e-8 < rel < 1e-6, rel


@pytest.mark.parametrize("resblock", ["1", "2"])
def test_unrounded_oracle_matches_the_generator_oracle(resblock):
    """Rounding off, float64 accumulation: the stage and the whole generator equal oracle/generator.py (CPU torch
    fp32) to within fp32 noise."""
    from helpers import build_model, sd_numpy
    from oracle import generator as og

    hp = dict(resblock=resblock, upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4], upsample_initial_channel=64,
              resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3], [1, 5]])
    model = build_model("hifigan", hp, 12, seed=3)
    model.remove_weight_norm()
    sd = sd_numpy(model)
    mel = np.random.default_rng(2).normal(0, 1, (2, 12, 40)).astype(np.float32)
    x = np.random.default_rng(4).normal(0, 1, (2, 32, 80)).astype(np.float32)
    blocks = [ro.hifigan_blocks(sd, f"resblocks.{j}", k, d, resblock)
              for j, (k, d) in enumerate(zip(hp["resblock_kernel_sizes"], hp["resblock_dilation_sizes"]))]
    rb = og.resblock1 if resblock == "1" else og.resblock2
    with torch.no_grad():
        want = sum(rb(sd, f"resblocks.{j}", torch.from_numpy(x), k, d).numpy()
                   for j, (k, d) in enumerate(zip(hp["resblock_kernel_sizes"], hp["resblock_dilation_sizes"]))) / 2
    got = ro.stage(x, blocks, None)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    want = og.hifigan_forward(sd, hp, mel)
    got = ro.hifigan(sd, hp, mel, None)
    assert np.abs(got - want).max() <= 1e-5 * max(np.abs(want).max(), 1e-3)


def test_plan_options():
    """set_option takes `resblock_fusion` 0..4 and no pair-schedule key."""
    from amphion_b200 import _capi
    from helpers import build_model
    hp = dict(resblock="1", upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4], upsample_initial_channel=64,
              resblock_kernel_sizes=[3], resblock_dilation_sizes=[[1]])
    h = build_model("hifigan", hp, 20, seed=1)._ensure_handle()
    assert _capi.lib.ab_generator_set_option(h, b"pair_schedule", 0) == -1
    assert "pair_schedule" in _capi.last_error()
    for v in range(5):
        assert _capi.lib.ab_generator_set_option(h, b"resblock_fusion", v) == 0
    for v in (-1, 5):
        assert _capi.lib.ab_generator_set_option(h, b"resblock_fusion", v) == -1
        assert "resblock_fusion" in _capi.last_error()


# ------------------------------------------------------------------------------------------------ GPU: one-hot, exact
# (id, C, [(k, dilations)], B, T, values)
ONE_HOT = [
    ("c16-T1", 16, [(3, (1, 3, 5))], 2, 1, "ordinary"),
    ("c48-padded-below-halo", 48, [(7, (1, 3, 5)), (3, (1, 3, 5))], 2, 30, "ordinary"),
    ("c64-ragged", 64, [(3, (1, 3, 5)), (7, (1, 3, 5)), (11, (1, 3, 5))], 2, 700, "ordinary"),
    # more than 2 x 132 items with a partial last stride: the persistent walks of the pair and block-mode kernels
    ("c64-walk", 64, [(3, (1, 3, 5)), (11, (1, 3, 5))], 6, 6000, "ordinary"),
    ("c96-k13-k1", 96, [(13, (1, 3, 5)), (1, (1, 3, 5))], 2, 300, "ordinary"),
    ("c128-walk", 128, [(3, (1, 3, 5)), (7, (1, 3, 5)), (11, (1, 3, 5))], 7, 5000, "ordinary"),
    # k = 31 at dilation 70, tap reach 2100: one A chunk buffer and two W stages next to the intermediate tile
    ("c128-k31-d70", 128, [(31, (70, 1)), (3, (1, 3))], 20, 800, "ordinary"),
    ("c200-partial-chunk", 200, [(7, (1, 4)), (31, (5, 1))], 2, 333, "ordinary"),
    ("c256", 256, [(3, (1, 3, 5)), (11, (1, 3, 5))], 3, 600, "ordinary"),
    ("c256-k31-d26", 256, [(31, (26, 1))], 2, 240, "ordinary"),   # tap reach 780: one A chunk buffer
    ("c320-single-conv", 320, [(3, (1, 3))], 2, 300, "ordinary"),
    ("c64-k33-single-conv", 64, [(33, (1, 2)), (3, (1, 3))], 2, 200, "ordinary"),
    ("c64-saturation", 64, [(3, (1, 3)), (7, (1, 2))], 2, 300, "saturation"),
    ("c128-subnormal", 128, [(3, (1, 3, 5)), (5, (1, 2))], 2, 300, "subnormal"),
    ("c32-subnormal", 32, [(7, (1, 3, 5))], 2, 500, "subnormal"),
]
VALUES = {   # input scale, weight exponents, bias std
    "ordinary": (2.0, (-2, -1, 0, 1), 0.5),
    "saturation": (3e4, (0, 1, 2), 1.0),      # f16: |x| and |h| past 65504
    "subnormal": (1e-5, (-3, -2, -1, 0), 1e-6),  # f16: operands and products below 2^-14
}


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", ONE_HOT, ids=[c[0] for c in ONE_HOT])
def test_one_hot_stage_is_exact_on_every_route(case, prec):
    _, C, shape, B, T, values = case
    scale, exps, bias_std = VALUES[values]
    rng = np.random.default_rng(C * 1000 + T)
    blocks = _blocks(rng, C, shape, "one-hot", exps, bias_std)
    x = (rng.normal(0, 1, (B, C, T)) * scale).astype(np.float32)
    want = _post(ro.stage(x, blocks, PRECS[prec]))
    assert np.isfinite(want).all()
    stage = _make_stage(C, blocks)
    for fusion in ROUTES:
        got, launches = stage.run(x, prec, fusion)
        assert launches == _launches(C, shape, fusion), (fusion, launches)
        bad = got != want
        assert not bad.any(), (f"fusion {fusion}: {int(bad.sum())} of {bad.size} differ, first at "
                               f"{np.argwhere(bad)[0].tolist()}: {got[bad][0]!r} vs {want[bad][0]!r}")


# ------------------------------------------------------------------------------------------------ GPU: dense, floor
DENSE = [
    ("c64", 64, [(3, (1, 3, 5)), (7, (1, 3, 5)), (11, (1, 3, 5))], 2, 700),
    ("c128", 128, [(3, (1, 3, 5)), (7, (1, 3, 5)), (11, (1, 3, 5))], 2, 400),
    ("c200", 200, [(7, (1, 4)), (3, (5, 1))], 2, 300),
    ("c256", 256, [(3, (1, 3, 5)), (11, (1, 3, 5))], 2, 300),
    ("c320-single-conv", 320, [(3, (1, 3))], 2, 200),
]


def _floor_check(what, got, o64, o32):
    e_mean, e_max, f_mean, f_max = ro.floor_stats(got, o64, o32)
    print(f"{what}: mean {e_mean:.3e} = {e_mean / f_mean:.2f} x floor {f_mean:.3e}; "
          f"max {e_max:.3e} = {e_max / f_max:.2f} x floor {f_max:.3e}")
    assert e_mean <= FLOOR_MEAN * f_mean and e_max <= FLOOR_MAX * f_max, what


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_stage_within_the_floor_on_every_route(case, prec):
    _, C, shape, B, T = case
    rng = np.random.default_rng(C + T)
    blocks = _blocks(rng, C, shape, "dense", bias_std=0.1)
    x = rng.normal(0, 1, (B, C, T)).astype(np.float32)
    o64, o32 = (_post(ro.stage(x, blocks, PRECS[prec], acc)) for acc in ("f64", "mma"))
    stage = _make_stage(C, blocks)
    for fusion in ROUTES:
        got, launches = stage.run(x, prec, fusion)
        assert launches == _launches(C, shape, fusion)
        _floor_check(f"{case[0]} {prec} fusion {fusion}", got, o64, o32)


# ------------------------------------------------------------------------------------------------ GPU: generators
GENERATORS = {
    # stage 0 (128 channels): k = 3 in block mode, k = 7 / 11 as pairs at fusion 2; stage 1 (64): k = 3 / 7 blocks
    "resblock1": (dict(resblock="1", upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4], upsample_initial_channel=256,
                       resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3), 150),
    # ResBlock2: block mode with one conv per step
    "resblock2": (dict(resblock="2", upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4], upsample_initial_channel=128,
                       resblock_kernel_sizes=[3, 5, 7], resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]), 120),
}


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(GENERATORS))
def test_generator_within_the_floor(name, prec):
    from helpers import build_model, sd_numpy
    hp, T = GENERATORS[name]
    model = build_model("hifigan", hp, 20, seed=5)
    model.remove_weight_norm()
    g = torch.Generator().manual_seed(6)
    with torch.no_grad():   # dense weights at unit gain, so the branches matter as much as the residual
        for n, p in model.named_parameters():
            if n.endswith(".weight"):
                # fan-in of an output sample; a ConvTranspose [C_in, C_out, k] of stride u sums C_in * k / u terms
                up = n.startswith("ups.")
                fan = p.shape[0] * p.shape[2] / hp["upsample_rates"][int(n.split(".")[1])] if up else p.shape[1] * p.shape[2]
                p.copy_(torch.randn(p.shape, generator=g) / float(np.sqrt(fan)))
    model = model.to(DEV)
    sd = sd_numpy(model)
    mel = torch.randn(2, 20, T, generator=torch.Generator().manual_seed(7))
    o64, o32 = (ro.hifigan(sd, hp, mel.numpy(), PRECS[prec], acc) for acc in ("f64", "mma"))
    model.precision = prec
    for fusion in (1, 2, 3):
        model.set_option("resblock_fusion", fusion)
        with torch.no_grad():
            got = model(mel.to(DEV)).cpu().numpy()
        _floor_check(f"{name} {prec} fusion {fusion}", got, o64, o32)
    model.set_option("resblock_fusion", 2)
