"""FACodec encoder (models/codec/ns3_codec/facodec.py:121-194) on the native pipeline, and the strided convolution it
runs on (`ab_tc_conv_forward` mode 2).

* CPU: the float64 oracle (tests/facodec_encode_oracle.py) against the reference fixture (tests/golden/fac_encoder*.npz,
  written by tests/golden/gen_facodec_encode.py), strict loading of the README geometry's state dict, the frame count
  for any N, and the refusals before launch.
* GPU: mode 2 bit for bit against the operand-rounded oracle with one-hot weights; the encoder at every precision
  against the fixture and the oracle; repeat runs, batch slices and transposed views bit-equal; the README geometry
  into the decoder; the profile.  Bars are fractions of the output's peak, as in test_facodec.py."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import facodec_encode_oracle as feo
import resblock_oracle as ro
from conftest import GOLDEN

BARS = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}   # test_facodec.py's bars, fractions of the output's peak
# The 16-bit precisions are held to the oracle with their operands rounded, and their bar is the larger of BARS and
# FLOOR x the distance between that oracle in fp32 and in float64 arithmetic (the floor of any fp32-accumulating
# implementation: fp32 round-off that crosses a rounding boundary moves an operand by a whole 16-bit ulp).  Without
# the kernels involved, operand rounding alone moves fixture a's output by 9.5e-4 (f16) / 7.5e-3 (bf16) of its peak,
# and the fp32 oracle sits 6.0e-4 / 4.3e-3 from the float64 one: above BARS["tc_bf16"].
FLOOR = 2.0
OPERANDS = {"fp32": None, "tc_f16": "f16", "tc_bf16": "bf16"}
PRECS = {"tc_f16": "f16", "tc_bf16": "bf16"}
DEV = "cuda:0"
# ab_facodec_encoder_frames at the README geometry, as the reference computes them
README_FRAMES = {16000: 80, 16001: 80, 16199: 81, 200: 1, 400: 2, 1000: 5}


def load_fixture():
    d = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "fac_encoder*.npz"))):
        z = np.load(p)
        d.update({k: z[k] for k in z.files})
    return d


def variant(d, tag):
    io = {k[len(tag) + 1:]: v for k, v in d.items() if k.startswith(tag + ":") and ":sd:" not in k}
    sd = {k[len(tag) + 4:]: v for k, v in d.items() if k.startswith(tag + ":sd:")}
    return io, sd


def build(hp, sd=None, seed=0):
    from amphion_b200.vocoders import FACodecEncoder
    torch.manual_seed(seed)
    m = FACodecEncoder(**hp)
    if sd is not None:
        m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()}, strict=True)
    return m.eval()


def perturb(model, seed):
    """Every parameter at the fixture generator's scales (tests/golden/gen_facodec_encode.py)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("weight_g"):
                scale = 0.25 if re.fullmatch(r"block\.\d+\.block\.[012]\.block\.3\.weight_g", name) else 1.0
                p.copy_((torch.rand(p.shape, generator=g) * 0.6 + 0.6) * scale)
            elif name.endswith("weight_v"):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith((".alpha", ".beta")):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    model.invalidate()


def _bar(prec, sd, up_ratios, wav, want, peak):
    """BARS[prec] x peak, or FLOOR x the fp32 oracle's distance from `want` where that is larger (16-bit precisions)."""
    if OPERANDS[prec] is None:
        return BARS[prec] * peak
    o32 = feo.encoder(sd, up_ratios, wav, operands=OPERANDS[prec], dtype=torch.float32).numpy()
    floor = _err(o32, want)
    print(f"  {prec}: fp32-arithmetic oracle floor / peak = {floor / peak:.2e}")
    return max(BARS[prec] * peak, FLOOR * floor)


def _err(got, want):
    return float(np.abs(np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64)).max())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_fixture(tag):
    io, sd = variant(load_fixture(), tag)
    hp, B, N = feo.GOLDEN_FACODEC_ENCODE[tag]
    enc, stages = feo.encoder(sd, hp["up_ratios"], io["wav"], return_stages=True)
    assert io["wav"].shape == (B, 1, N) and enc.shape == io["enc"].shape
    assert enc.shape[2] == feo.frames(hp["up_ratios"], N)
    for i, st in enumerate(stages):
        assert _err(st, io[f"stage{i}"]) <= 1e-5 * np.abs(io[f"stage{i}"]).max(), i
    assert _err(enc, io["enc"]) <= 1e-5 * np.abs(io["enc"]).max()


def test_strided_conv_oracle_matches_torch():
    """The one-hot oracle of the GPU tests below: y[t] = sum_j W_j a[s t + j - pad] as F.conv1d computes it."""
    rng = np.random.default_rng(3)
    for s, k, pad in ((2, 4, 1), (3, 6, 2), (5, 10, 3), (8, 16, 4), (4, 5, 0)):
        a = rng.normal(0, 1, (2, 12, 37))
        w = ro.random_one_hot(rng, 20, 12, k, (-1, 0, 1))
        want = F.conv1d(torch.from_numpy(a), torch.from_numpy(w.dense()).double(), stride=s, padding=pad).numpy()
        assert np.array_equal(_strided(a, w, s, pad), want), (s, k, pad)


def test_readme_state_dict_loads_strictly():
    d = load_fixture()
    m = build(feo.README_FACODEC_ENCODER)
    want = {k: tuple(int(s) for s in shp if s >= 0) for k, shp in zip(d["readme_keys"].tolist(), d["readme_shapes"])}
    assert len(want) == 206
    have = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert have == want
    m.load_state_dict({k: torch.zeros(s) for k, s in want.items()}, strict=True)


def test_fixture_state_dicts_load_strictly():
    d = load_fixture()
    for tag in ("a", "b"):
        _, sd = variant(d, tag)
        m = build(feo.GOLDEN_FACODEC_ENCODE[tag][0], sd)
        for k, v in sd.items():
            assert np.array_equal(m.state_dict()[k].numpy(), v), k


def test_frames_follow_the_reference():
    from amphion_b200 import _capi
    m = build(feo.README_FACODEC_ENCODER)
    h = m._ensure_handle()
    for n, f in README_FRAMES.items():
        assert feo.frames(m.up_ratios, n) == f, n
        assert m.frames(n) == f, n
        assert _capi.lib.ab_facodec_encoder_frames(h, n) == f, n
    for n in range(1, 260):   # every length, including those a stage empties
        want = feo.frames(m.up_ratios, n)
        assert m.frames(n) == want == _capi.lib.ab_facodec_encoder_frames(h, n), n
    assert _capi.lib.ab_facodec_encoder_frames(h, 0) == 0
    # a stride-1 stage (k = 2, padding 1) after an emptied one: the reference raises, so the count stays 0
    m1 = build(dict(ngf=8, up_ratios=[4, 1], out_channels=16))
    for n in (1, 2, 3, 4):
        want = feo.frames(m1.up_ratios, n)
        assert m1.frames(n) == want == _capi.lib.ab_facodec_encoder_frames(m1._ensure_handle(), n), n
    assert m1.frames(1) == 0 and m1.frames(4) == 2


def test_refusals_before_launch():
    from amphion_b200 import _capi
    m = build(feo.GOLDEN_FACODEC_ENCODE["a"][0])
    with pytest.raises(ValueError, match=r"\[B, 1, N\]"):
        m(torch.zeros(1, 2, 100))
    with pytest.raises(ValueError, match=r"\[B, 1, N\]"):
        m(torch.zeros(1, 100))
    with pytest.raises(ValueError, match="too short"):
        m(torch.zeros(1, 1, 3))
    with pytest.raises(ValueError, match="empty"):
        m(torch.zeros(0, 1, 100))
    lib = _capi.lib
    h = m._ensure_handle()
    # the C entry refuses a length a stage would empty, and a non-encoder handle, before any launch
    st = _capi.shape_array((3, 3, 1))
    assert lib.ab_facodec_encode(h, C.c_void_p(16), 1, 3, st, C.c_void_p(16), C.c_void_p(256), 1 << 20, None) == -1
    assert "no output" in _capi.last_error()
    assert lib.ab_generator_forward(h, C.c_void_p(16), 1, 100, st, C.c_void_p(16), C.c_void_p(256), 1 << 20, None) == -1
    assert "ab_facodec_encode" in _capi.last_error()
    from amphion_b200.vocoders import FACodecDecoder
    dec = FACodecDecoder(in_channels=16, upsample_initial_channel=64, up_ratios=[3, 2], vq_dim=16)
    assert lib.ab_facodec_encode(dec._ensure_handle(), C.c_void_p(16), 1, 100, st, C.c_void_p(16), C.c_void_p(256),
                                 1 << 20, None) == -1
    assert "not a FACodec encoder" in _capi.last_error()


def test_c_abi_config_checks():
    from amphion_b200 import _capi
    m = build(feo.GOLDEN_FACODEC_ENCODE["a"][0])
    lib = _capi.lib

    def create(edit):
        c = m._c_config()
        edit(c)
        h = C.c_void_p()
        rc = lib.ab_generator_create(C.byref(c), C.byref(h))
        if rc == 0:
            lib.ab_generator_destroy(h)
        return rc

    assert create(lambda c: None) == 0
    assert create(lambda c: setattr(c, "n_mel", 2)) != 0
    assert create(lambda c: setattr(c, "snake_logscale", 0)) != 0
    assert create(lambda c: setattr(c, "trunk_out_channels", 0)) != 0
    assert create(lambda c: c.upsample_kernel_sizes.__setitem__(0, 5)) != 0
    # strides the tensor-core strided conv serves (1..8), not a silent fp32 fallback or a failure mid-forward
    assert create(lambda c: (c.upsample_rates.__setitem__(0, 8), c.upsample_kernel_sizes.__setitem__(0, 16))) == 0
    assert create(lambda c: (c.upsample_rates.__setitem__(0, 9), c.upsample_kernel_sizes.__setitem__(0, 18))) != 0
    assert "stride 9" in _capi.last_error()
    assert create(lambda c: c.resblock_dilation_sizes[0].__setitem__(1, 2)) != 0
    assert create(lambda c: c.vq_num_q.__setitem__(0, 1)) != 0          # vq_* belong to the decoder kind
    assert create(lambda c: setattr(c, "gin_channels", 4)) != 0
    assert create(lambda c: setattr(c, "num_layers", 2)) != 0


# ------------------------------------------------------------------------------------------------ GPU: mode 2
def _strided(a, w, s, pad):
    """y[b, co, t] = sum_{ci, j} W[co, ci, j] a[b, ci, s t + j - pad], zero padding (float64; one term per output for
    one-hot weights, so exact)."""
    w = w.dense() if isinstance(w, ro.OneHot) else w
    B, cin, T = a.shape
    cout, _, k = w.shape
    Tout = (T + 2 * pad - k) // s + 1
    ap = np.zeros((B, cin, T + 2 * pad + s * Tout + k))
    ap[:, :, pad:pad + T] = a
    y = np.zeros((B, cout, Tout))
    for j in range(k):
        y += np.einsum("oc,bct->bot", w[:, :, j].astype(np.float64), ap[:, :, j:j + s * Tout:s])
    return y


def _run_strided(prec, w, bias, B, cin, cout, T, k, s, pad, x=None, ximg=None, pre_slope=1.0):
    from amphion_b200 import _capi
    lib = _capi.lib
    Tout = (T + 2 * pad - k) // s + 1
    wd = torch.from_numpy(np.ascontiguousarray(w, np.float32)).to(DEV)
    bd = torch.from_numpy(bias).to(DEV)
    xi = None if ximg is None else torch.from_numpy(np.ascontiguousarray(ximg).view(np.int16)).to(DEV)
    y = torch.full((B, cout, Tout), float("nan"), device=DEV)
    need = lib.ab_tc_conv_workspace_bytes(2, cin, cout, k, s)
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    rc = lib.ab_tc_conv_forward(2, _capi.ptr(x), None if x is None else _capi.shape_array(x.stride()), pre_slope,
                                _capi.ptr(xi), _capi.ptr(wd), _capi.ptr(bd), None, None, 1.0, 0, _capi.ptr(y), None, 1.0,
                                B, cin, cout, T, k, s, pad, _capi.PRECISIONS[prec],
                                C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, _capi.stream_ptr())
    torch.cuda.synchronize()
    return rc, y.cpu().numpy()


# (id, C_in, C_out, k, s, pad, B, T)
STRIDED = [
    ("s2-encoder", 32, 64, 4, 2, 1, 2, 1001),       # FACodec's first EncoderBlock conv; ragged tiles
    ("s3", 16, 32, 6, 3, 2, 2, 700),
    ("s4-encoder", 64, 128, 8, 4, 2, 2, 900),
    ("s5-encoder", 128, 256, 10, 5, 3, 2, 1300),    # N = 256: one m64 tile per warpgroup
    ("s5-512", 256, 512, 10, 5, 3, 1, 600),         # two N blocks
    ("s8", 32, 64, 16, 8, 4, 2, 2100),
    ("s2-partial-n", 48, 80, 4, 2, 1, 2, 333),      # a partial K chunk and N blocks of 128 with 80 channels used
    ("s3-odd-k", 32, 24, 7, 3, 0, 3, 50),           # odd k, no padding, C_out % 16 != 0
    ("s4-cin8", 8, 16, 8, 4, 2, 2, 99),             # one partial K chunk per phase
    ("s2-T-short", 32, 64, 4, 2, 1, 2, 3),          # one output tile, most rows outside the sequence
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", STRIDED, ids=[c[0] for c in STRIDED])
def test_one_hot_strided_conv_is_exact(case, prec):
    """Every output is one exact product plus the bias: fp32 input (lrelu and rounding in the loader, from a strided
    view) and, at C_in % 16 == 0, the operand image must both equal the oracle bit for bit."""
    name, cin, cout, k, s, pad, B, T = case
    rng = np.random.default_rng(cin * 3 + cout + k * s + T)
    w = ro.random_one_hot(rng, cout, cin, k, (-2, -1, 0, 1))
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    slope = 0.1
    x = (rng.normal(0, 2.0, (B, T, cin))).astype(np.float32)          # stored [B, T, C], seen as [B, C, T]
    xc = np.ascontiguousarray(x.transpose(0, 2, 1))
    act = ro.rnd(ro.lrelu(xc, slope), PRECS[prec])
    want = (_strided(act, w.rounded(PRECS[prec]), s, pad).astype(np.float32) + bias[None, :, None]).astype(np.float32)
    runs = [("fp32 in", dict(x=torch.from_numpy(x).to(DEV).transpose(1, 2), pre_slope=slope))]
    if cin % 16 == 0:
        runs.append(("image in", dict(ximg=ro.to_image(ro.image_bits(xc, slope, PRECS[prec])))))
    for what, src in runs:
        rc, y = _run_strided(prec, w.dense(), bias, B, cin, cout, T, k, s, pad, **src)
        assert rc == 0, (name, what, rc)
        assert np.isfinite(want).all()
        bad = y != want
        assert not bad.any(), (f"{name} {what}: {int(bad.sum())} of {bad.size} differ, first at "
                               f"{np.argwhere(bad)[0].tolist()}")


@pytest.mark.gpu
def test_strided_conv_refusals():
    from amphion_b200 import _capi
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.normal(0, 1, (1, 16, 20)).astype(np.float32)).to(DEV)
    bias = np.zeros(16, np.float32)
    for k, s, pad, T, msg in ((4, 9, 1, 20, "stride"), (2, 4, 0, 20, "stride"), (4, 2, 4, 20, "padding"),
                              (10, 2, 1, 5, "shorter")):
        w = rng.normal(0, 1, (16, 16, k)).astype(np.float32)
        rc, y = _run_strided("tc_f16", w, bias, 1, 16, 16, T, k, s, pad, x=x[:, :, :T]) if T + 2 * pad >= k else \
            (None, None)
        if rc is None:   # T_out would be empty: the output buffer cannot even be shaped, call directly
            need = _capi.lib.ab_tc_conv_workspace_bytes(2, 16, 16, k, s)
            ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
            wd = torch.from_numpy(w).to(DEV)
            out = torch.empty(16, device=DEV)
            rc = _capi.lib.ab_tc_conv_forward(2, _capi.ptr(x), _capi.shape_array(x.stride()), 1.0, None, _capi.ptr(wd),
                                              None, None, None, 1.0, 0, _capi.ptr(out), None, 1.0, 1, 16, 16, T, k, s,
                                              pad, 1, C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need,
                                              _capi.stream_ptr())
        else:
            assert np.isnan(y).all()
        assert rc != 0 and msg in _capi.last_error(), (k, s, pad, T, _capi.last_error())


# ------------------------------------------------------------------------------------------------ GPU: the encoder
@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    io, sd = variant(load_fixture(), tag)
    hp, B, N = feo.GOLDEN_FACODEC_ENCODE[tag]
    m = build(hp, sd).to(DEV)
    wav = torch.from_numpy(io["wav"]).to(DEV)
    peak = float(np.abs(io["enc"]).max())
    for prec in ("fp32", "tc_f16", "tc_bf16"):
        m.precision = prec
        enc = m(wav).cpu().numpy()
        assert enc.shape == io["enc"].shape
        # conv_pre; per stage 3 x (2 activations + 2 convs), the activation and the strided conv; final act, conv_post
        assert m.last_launches == 1 + 14 * len(hp["up_ratios"]) + 2
        want = feo.encoder(sd, hp["up_ratios"], io["wav"], operands=OPERANDS[prec]).numpy()
        err_fix, err_or = _err(enc, io["enc"]), _err(enc, want)
        print(f"facodec encoder {tag} {prec}: |native - fixture| / peak = {err_fix / peak:.2e}, "
              f"|native - oracle| / peak = {err_or / peak:.2e}")
        if prec == "fp32":
            assert err_fix <= BARS[prec] * peak
        else:
            assert err_or <= _bar(prec, sd, hp["up_ratios"], io["wav"], want, peak)
        assert np.array_equal(m.inference(wav).cpu().numpy(), enc)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "tc_f16", "tc_bf16"])
def test_bit_equal_runs(prec):
    io, sd = variant(load_fixture(), "a")
    m = build(feo.GOLDEN_FACODEC_ENCODE["a"][0], sd).to(DEV)
    m.precision = prec
    wav = torch.from_numpy(io["wav"]).to(DEV)
    ref = m(wav)
    assert torch.equal(m(wav), ref)                                                   # repeat run
    for b in range(wav.shape[0]):                                                     # batch independence
        assert torch.equal(m(wav[b:b + 1]), ref[b:b + 1])
    wt = wav[:, 0, :].t().contiguous().t().unsqueeze(1)                               # a [B, 1, N] view with stride B
    assert wt.stride(2) == wav.shape[0]
    assert torch.equal(m(wt), ref)
    out = torch.full_like(ref, float("nan"))
    assert m(wav, out=out) is out and torch.equal(out, ref)
    with pytest.raises(ValueError):
        m(wav, out=torch.empty(1, 2, 3, device=DEV))


@pytest.mark.gpu
def test_readme_geometry_into_the_decoder():
    """The README flow's encoder at 16 kHz: 16001 samples -> 80 frames of 256 channels at every precision against the
    oracle, then FACodecDecoder.inference of them gives 80 * 200 samples."""
    import facodec_oracle as fo
    from amphion_b200.vocoders import FACodecDecoder
    hp = feo.README_FACODEC_ENCODER
    m = build(hp)
    perturb(m, 5)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    g = torch.Generator().manual_seed(11)
    wav = torch.randn(2, 1, 16001, generator=g) * 0.3
    for prec in ("fp32", "tc_f16", "tc_bf16"):
        m.precision = prec
        enc = m(wav.to(DEV))
        assert enc.shape == (2, 256, 80) and enc.dtype == torch.float32
        want = feo.encoder(sd, hp["up_ratios"], wav.numpy(), operands=OPERANDS[prec]).numpy()
        peak = float(np.abs(want).max())
        err = _err(enc.cpu(), want)
        print(f"facodec encoder readme {prec}: |native - oracle| / peak = {err / peak:.2e}")
        assert err <= _bar(prec, sd, hp["up_ratios"], wav.numpy(), want, peak)
    torch.manual_seed(0)
    dec = FACodecDecoder(**fo.README_FACODEC).eval().to(DEV)
    out = dec.inference(enc, torch.randn(2, 256, device=DEV))
    assert out.shape == (2, 1, 80 * 200) and torch.isfinite(out).all()


@pytest.mark.gpu
def test_profile_and_generator_forward_refused():
    io, sd = variant(load_fixture(), "b")
    m = build(feo.GOLDEN_FACODEC_ENCODE["b"][0], sd).to(DEV)
    wav = torch.from_numpy(io["wav"]).to(DEV)
    for prec, strided_cls in (("fp32", "conv1d_fp32"), ("tc_f16", "tc_gemmconv")):
        m.precision = prec
        m(wav)
        m.set_profiling(True)
        m(wav)
        prof = m.get_profile()
        m.set_profiling(False)
        assert sum(v["launches"] for v in prof.values()) == m.last_launches
        assert prof["activation1d"]["launches"] == 7 * 2 + 1
        assert prof[strided_cls]["launches"] >= 2
    with pytest.raises(RuntimeError, match="ab_facodec_encode"):
        m._forward_native(wav)
