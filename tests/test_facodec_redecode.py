"""FACodecRedecoder (models/codec/ns3_codec/facodec.py:602-769) on the native kernels: vq2emb's embedding gathers and
speaker-conditioned prosody transformer, and inference on the decoder's generator.

* CPU: the float64 oracle (tests/facodec_redecode_oracle.py) against the reference fixture (tests/golden/fac_redecoder*.npz,
  written by tests/golden/gen_facodec_redecode.py) with the redrawn weights' digests, strict loading of the released
  state dict, the config and C-entry refusals, and the bound on the condition mean the native path skips.
* GPU, at every precision: fixture parity for vq2emb and the waveform, the released geometry, ragged T and strided code
  views, extra code rows, the positional quirk, batch independence, repeat runs, out= / tail_events, the tail's
  operation order bit for bit (NaN for a bad code), the README voice-conversion flow, and the profile."""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

import facodec_encode_oracle as feo
import facodec_oracle as fo
import facodec_quantize_oracle as fqo
import facodec_redecode_oracle as fro
from conftest import GOLDEN

BARS = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}          # fractions of the peak
OPERANDS = {"fp32": None, "tc_f16": None, "tc_bf16": "bf16"}    # tc_f16 against the fp32 oracle, bf16 operand-rounded
FLOOR = 2.0
PRECS = ("fp32", "tc_f16", "tc_bf16")
DEV = "cuda:0"
SEEDS = {"a": 111, "b": 113}
N_RELEASED = 265          # state-dict entries of ns3_facodec_redecoder.bin
N_RELEASED_ELEMS = 37609690


def load_fixture():
    d = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "fac_redecoder*.npz"))):
        z = np.load(p)
        d.update({k: z[k] for k in z.files})
    return d


def variant(d, tag):
    return {k[len(tag) + 1:]: v for k, v in d.items() if k.startswith(tag + ":")}


def build(hp, seed):
    """The fixture's module: every parameter redrawn from the seed, pe computed."""
    from amphion_b200.vocoders import FACodecRedecoder
    m = FACodecRedecoder(**hp).eval()
    fro.perturb(m.named_parameters(), seed + 100, len(hp["up_ratios"]))
    with torch.no_grad():
        m.timbre_cond_prosody_enc.position_emb.pe.copy_(fro.positional_encoding())
    m.invalidate()
    return m


def state(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _err(got, want):
    return float(np.abs(_np(got).astype(np.float64) - _np(want).astype(np.float64)).max())


def _emb_bar(prec, sd, codes, spk, n, use_residual, want, peak):
    """BARS of the peak; at tc_bf16 at least FLOOR x the bf16-operand oracle's fp32-vs-float64 distance."""
    bar = BARS[prec] * peak
    if prec == "tc_bf16":
        f32 = fro.vq2emb(sd, codes, spk, n, use_residual, operands="bf16", dtype=torch.float32)
        bar = max(bar, FLOOR * _err(f32, want))
    return bar


def _wav_bar(prec, sd, up_ratios, emb, spk, want, peak):
    """BARS of the peak; at tc_bf16 at least FLOOR x the bf16-operand oracle's fp32-vs-float64 distance."""
    bar = BARS[prec] * peak
    if prec == "tc_bf16":
        f32 = fro.inference(sd, up_ratios, emb, spk, operands="bf16", dtype=torch.float32)
        bar = max(bar, FLOOR * _err(f32, want))
    return bar


def _codes(hp, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    p, c, r = fro.n_tables(hp)
    rows = []
    for k, n in zip(("prosody", "content", "residual"), (p, c, r)):
        rows += [torch.randint(0, 2 ** hp[f"codebook_size_{k}"], (1, B, T), generator=g) for _ in range(n)]
    return torch.cat(rows), torch.randn(B, 256, generator=g)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_fixture(tag):
    io = variant(load_fixture(), tag)
    hp, B, T = fro.GOLDEN_FACODEC_REDECODE[tag]
    m = build(hp, SEEDS[tag])
    sd = state(m)
    assert dict(zip(io["digest_names"].tolist(), io["digests"].tolist())) == fro.digests(sd)
    n = fro.n_tables(hp)
    assert io["codes"].shape == (sum(n), B, T)
    for key, use_residual in (("emb", False), ("emb_res", True)):
        got, runs = fro.vq2emb(sd, io["codes"], io["spk"], n, use_residual, return_layers=True)
        assert _err(got, io[key]) <= 1e-6 * np.abs(io[key]).max(), key
    assert len(runs) == n[0]
    for r, layers in enumerate(runs):
        for i, h in enumerate(layers):
            want = io["layers"][r, i]
            assert _err(h, want) <= 1e-6 * np.abs(want).max(), (r, i)
    wav = fro.inference(sd, hp["up_ratios"], io["emb"], io["spk"])
    assert _err(wav, io["wav"]) <= 1e-6 * np.abs(io["wav"]).max()


def test_condition_mean_bound():
    """The reference feeds the style Linears mean(spk expanded over T); the native path the embedding itself.  In fp32
    the two differ by far less than the fp32 bar at the fixture sizes."""
    for tag in ("a", "b"):
        io = variant(load_fixture(), tag)
        hp, _, _ = fro.GOLDEN_FACODEC_REDECODE[tag]
        sd = state(build(hp, SEEDS[tag]))
        n = fro.n_tables(hp)
        lit = fro.vq2emb(sd, io["codes"], io["spk"], n, True, dtype=torch.float32)
        vec = fro.vq2emb(sd, io["codes"], io["spk"], n, True, dtype=torch.float32, literal_mean=False)
        peak = np.abs(io["emb_res"]).max()
        d = _err(lit, vec)
        print(f"facodec redecode {tag}: |mean - vector| / peak = {d / peak:.2e}")
        assert d <= 0.1 * BARS["fp32"] * peak


def test_released_state_dict_loads_strictly():
    """The default constructor's state dict is the released checkpoint's (265 entries, 37,609,690 elements, names and
    shapes as the reference lists them), and the handle lists exactly those names."""
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecRedecoder
    d = load_fixture()
    m = FACodecRedecoder().eval()
    sd = m.state_dict()
    assert len(sd) == N_RELEASED and sum(v.numel() for v in sd.values()) == N_RELEASED_ELEMS
    assert list(sd.keys()) == d["released_keys"].tolist()
    for k, shp in zip(d["released_keys"].tolist(), d["released_shapes"]):
        assert tuple(sd[k].shape) == tuple(int(s) for s in shp if s >= 0), k
    h = m._ensure_handle()
    lib = _capi.lib
    names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(lib.ab_generator_num_tensors(h))]
    covered = set()
    for name in names:
        if name in sd:
            covered.add(name)
        else:
            assert name + "_v" in sd and name + "_g" in sd, name
            covered |= {name + "_v", name + "_g"}
    assert covered == set(sd.keys())
    assert len(names) == len(set(names))
    m.load_state_dict({k: torch.zeros_like(v) for k, v in sd.items()}, strict=True)


def test_config_refusals():
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecRedecoder
    with pytest.raises(ValueError, match="256"):
        FACodecRedecoder(in_channels=128, vq_dim=128)
    with pytest.raises(ValueError, match="256"):
        FACodecRedecoder(vq_dim=128)
    m = FACodecRedecoder(**fro.GOLDEN_FACODEC_REDECODE["a"][0])
    lib = _capi.lib

    def bits(i, v):
        return lambda c: c.vq_codebook_bits.__setitem__(i, v)

    def nq(i, v):
        return lambda c: c.vq_num_q.__setitem__(i, v)

    for edit, ok in ((lambda c: None, True), (nq(2, 0), True), (nq(0, 2), True),
                     (lambda c: setattr(c, "n_mel", 128), False), (lambda c: setattr(c, "vq_codebook_dim", 8), False),
                     (lambda c: setattr(c, "facodec_quantize", 1), False), (nq(0, 0), False), (nq(1, 0), False),
                     (nq(2, -1), False), (nq(2, 30), False), (bits(0, 0), False), (bits(2, 25), False),
                     (lambda c: setattr(c, "snake_logscale", 0), False),
                     (lambda c: setattr(c, "kind", 10), False)):
        c = m._c_config()
        edit(c)
        h = C.c_void_p()
        rc = lib.ab_generator_create(C.byref(c), C.byref(h))
        if rc == 0:
            lib.ab_generator_destroy(h)
        assert (rc == 0) == ok, _capi.last_error()
    assert m._c_config().kind == _capi.GEN_FACODEC_REDECODER == 9


def test_refusals_before_launch():
    """The Python refusals that need no device, and the C entry's refusals of a handle that cannot run yet."""
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecDecoder
    hp = fro.GOLDEN_FACODEC_REDECODE["a"][0]
    m = build(hp, 0)
    codes, spk = _codes(hp, 2, 5, 0)
    with pytest.raises(NotImplementedError, match="reference"):
        m(codes, spk)
    with pytest.raises(ValueError, match="integer"):
        m.vq2emb(codes.float(), spk)
    with pytest.raises(ValueError, match="code rows"):
        m.vq2emb(codes[:5], spk)
    # without use_residual the residual rows are not needed: refused only for the device
    with pytest.raises(RuntimeError, match="CPU fallback"):
        m.vq2emb(codes[:3], spk, use_residual=False)
    with pytest.raises(ValueError, match="speaker embedding"):
        m.vq2emb(codes, spk[:1])
    with pytest.raises(ValueError, match="speaker embedding"):
        m.vq2emb(codes, spk[:, :128])
    with pytest.raises(RuntimeError, match="CPU fallback"):
        m.vq2emb(codes, spk)
    with pytest.raises(ValueError, match="expects x"):
        m.inference(torch.zeros(2, 128, 5), spk)
    lib = _capi.lib
    st = _capi.shape_array((10, 5, 1))
    p = C.c_void_p(16)

    def call(h, n_q=6, B=2):
        return lib.ab_facodec_redecoder_vq2emb(h, p, st, n_q, B, 5, p, 256, 1, p, C.c_void_p(256), 1 << 40, None)

    assert call(None) != 0 and "null handle" in _capi.last_error()
    assert call(m._ensure_handle(), B=5001) != 0 and "positional" in _capi.last_error()
    assert call(m._ensure_handle()) == -4 and "finalize" in _capi.last_error()   # AB_ERR_STATE
    dec = FACodecDecoder(**fqo.GOLDEN_FACODEC_QUANTIZE["a"][0])
    assert call(dec._ensure_handle()) != 0 and "not a FACodec redecoder" in _capi.last_error()
    assert lib.ab_facodec_redecoder_vq2emb_workspace_bytes(dec._ensure_handle(), 2, 5) == 0
    # the decoder's own vq2emb and quantize entries refuse a redecoder handle
    h = m._ensure_handle()
    assert lib.ab_facodec_vq2emb(h, p, st, 6, 2, 5, 1, p, None) != 0 and "not a FACodec handle" in _capi.last_error()
    # the generator entry refuses it
    assert lib.ab_generator_forward(h, p, 2, 5, st, p, C.c_void_p(256), 1 << 40, None) != 0
    assert "ab_facodec_inference" in _capi.last_error()


# ------------------------------------------------------------------------------------------------ GPU
def _emb(m, codes, spk, prec, use_residual=True):
    m.precision = prec
    r = m.vq2emb(codes, spk, use_residual=use_residual)
    torch.cuda.synchronize()
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    io = variant(load_fixture(), tag)
    hp, B, T = fro.GOLDEN_FACODEC_REDECODE[tag]
    m = build(hp, SEEDS[tag]).to(DEV)
    sd = state(m)
    n = fro.n_tables(hp)
    codes, spk = torch.from_numpy(io["codes"]).to(DEV), torch.from_numpy(io["spk"]).to(DEV)
    for prec in PRECS:
        for key, use_residual in (("emb", False), ("emb_res", True)):
            got = _emb(m, codes, spk, prec, use_residual)
            assert got.shape == (B, 256, T) and got.dtype == torch.float32 and got.is_contiguous()
            assert m.last_launches == 9 + 30 * n[0] + 1
            want = fro.vq2emb(sd, io["codes"], io["spk"], n, use_residual, operands=OPERANDS[prec])
            peak = float(np.abs(io[key]).max())
            err = _err(got, want)
            print(f"facodec redecode {tag} {prec} {key}: |native - oracle| / peak = {err / peak:.2e} "
                  f"(|native - fixture| / peak = {_err(got, io[key]) / peak:.2e})")
            assert err <= _emb_bar(prec, sd, io["codes"], io["spk"], n, use_residual, want, peak), (prec, key)
        emb = _emb(m, codes, spk, prec, False)
        wav = m.inference(emb, spk)
        torch.cuda.synchronize()
        assert wav.shape == io["wav"].shape
        want = fo.inference(sd, hp["up_ratios"], _np(emb), io["spk"], OPERANDS[prec]).numpy()
        peak = float(np.abs(io["wav"]).max())
        err = _err(wav, want)
        print(f"facodec redecode {tag} {prec} wav: |native - oracle| / peak = {err / peak:.2e} "
              f"(|native - fixture| / peak = {_err(wav, io['wav']) / peak:.2e})")
        assert err <= _wav_bar(prec, sd, hp["up_ratios"], _np(emb), io["spk"], want, peak), prec
        if prec == "fp32":   # end to end against the reference's waveform
            assert _err(wav, io["wav"]) <= 1e-4 * peak


@pytest.mark.gpu
def test_released_geometry():
    """The default constructor (1280 channels, up_ratios (5, 5, 4, 2)): conv_pre 256 -> 1280 and a u = 5
    ConvTranspose 1280 -> 640, with seeded weights against the oracle at B = 2, T = 8."""
    hp = fro.RELEASED
    m = build(hp, 7)
    sd = state(m)
    m = m.to(DEV)
    n = fro.n_tables(hp)
    codes, spk = _codes(hp, 2, 8, 3)
    cd, sp = codes.to(DEV), spk.to(DEV)
    for prec in PRECS:
        emb = _emb(m, cd, sp, prec, False)
        want = fro.vq2emb(sd, codes, spk, n, False, operands=OPERANDS[prec])
        peak = float(want.abs().max())
        err = _err(emb, want)
        print(f"facodec redecode released {prec}: |emb - oracle| / peak = {err / peak:.2e}")
        assert err <= _emb_bar(prec, sd, codes, spk, n, False, want, peak)
        wav = m.inference(emb, sp)
        torch.cuda.synchronize()
        assert wav.shape == (2, 1, 8 * 200)
        want = fo.inference(sd, hp["up_ratios"], _np(emb), spk.numpy(), OPERANDS[prec]).numpy()
        peak = float(np.abs(want).max())
        err = _err(wav, want)
        bar = _wav_bar(prec, sd, hp["up_ratios"], _np(emb), spk.numpy(), want, peak)
        print(f"facodec redecode released {prec}: |wav - oracle| / peak = {err / peak:.2e} (bar {bar / peak:.2e})")
        assert err <= bar


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 63, 64, 65, 333])
def test_shapes_and_code_views(T):
    hp = fro.GOLDEN_FACODEC_REDECODE["a"][0]
    m = build(hp, SEEDS["a"])
    sd = state(m)
    m = m.to(DEV)
    n = fro.n_tables(hp)
    codes, spk = _codes(hp, 2, T, T)
    cd, sp = codes.to(DEV), spk.to(DEV)
    views = {
        "transposed": codes.permute(2, 1, 0).contiguous().permute(2, 1, 0).to(DEV),   # time stride n_q * B
        "strided": torch.stack([codes, -codes - 1], 1).reshape(2 * codes.shape[0], 2, T).to(DEV)[::2],
        "int32": codes.int().to(DEV),
    }
    assert views["strided"].stride(0) == 2 * 2 * T
    for prec in ("fp32", "tc_bf16"):
        ref = _emb(m, cd, sp, prec)
        for name, v in views.items():
            assert torch.equal(_emb(m, v, sp, prec), ref), (prec, name)
        want = fro.vq2emb(sd, codes, spk, n, True, operands=OPERANDS[prec])
        peak = float(want.abs().max())
        err = _err(ref, want)
        print(f"facodec redecode T={T} {prec}: |emb - oracle| / peak = {err / peak:.2e}")
        assert err <= _emb_bar(prec, sd, codes, spk, n, True, want, peak)


@pytest.mark.gpu
def test_extra_rows_quirk_batch_and_repeats():
    """Code rows past those read are ignored (the README passes the decoder's six rows with use_residual=False);
    utterance b adds row b of pe, so swapping utterances changes their output as the oracle says; an utterance's output
    does not depend on the others in its batch; repeat runs, out= and tail_events are bit-equal."""
    hp = fro.GOLDEN_FACODEC_REDECODE["a"][0]
    m = build(hp, SEEDS["a"])
    sd = state(m)
    m = m.to(DEV)
    n = fro.n_tables(hp)
    codes, spk = _codes(hp, 3, 40, 5)
    cd, sp = codes.to(DEV), spk.to(DEV)
    junk = torch.full((2, 3, 40), -7, dtype=torch.long, device=DEV)   # never read: not range-checked either
    swap = [1, 0, 2]
    for prec in PRECS:
        full = _emb(m, cd, sp, prec)
        assert torch.equal(_emb(m, torch.cat([cd, junk]), sp, prec), full), prec
        nores = _emb(m, cd, sp, prec, False)
        assert torch.equal(_emb(m, cd[:3], sp, prec, False), nores), prec
        assert torch.equal(_emb(m, torch.cat([cd[:3], junk]), sp, prec, False), nores), prec
        assert torch.equal(_emb(m, cd, sp, prec), full), prec                          # repeat run
        assert torch.equal(_emb(m, cd[:, :1], sp[:1], prec), full[:1]), prec           # batch independence
        assert torch.equal(_emb(m, cd[:, :2], sp[:2], prec), full[:2]), prec
        swapped = _emb(m, cd[:, swap], sp[swap], prec)
        assert torch.equal(swapped[2], full[2]), prec
        wav = m.inference(nores, sp)
        out = torch.full_like(wav, float("nan"))
        evs = [torch.cuda.Event() for _ in range(2)]
        m.inference(nores, sp, out=out, tail_events=evs)
        for e in evs:
            e.synchronize()
        assert torch.equal(out, wav) and torch.equal(m.inference(nores, sp), wav), prec
    want = fro.vq2emb(sd, codes, spk, n, True)
    want_s = fro.vq2emb(sd, codes[:, swap], spk[swap], n, True)
    assert float((want_s[0] - want[1]).abs().max()) > 1e-3        # the position changes the output
    got_s = _emb(m, cd[:, swap], sp[swap], "fp32")
    peak = float(want.abs().max())
    assert _err(got_s, want_s) <= BARS["fp32"] * peak
    assert _err(_emb(m, cd, sp, "fp32"), want) <= BARS["fp32"] * peak


@pytest.mark.gpu
def test_tail_order_is_exact_and_bad_codes():
    """With last_ln's style weight and gamma bias zero, the transformer's output is beta exactly, so vq2emb must equal
    numpy float32 ((beta + c0) + c1) + r0 ... bit for bit at every precision.  Through the C entry a content code
    outside its table is not read and its time step is NaN; the Python method refuses it before the launch."""
    from amphion_b200 import _capi
    hp = fro.GOLDEN_FACODEC_REDECODE["a"][0]
    m = build(hp, SEEDS["a"])
    with torch.no_grad():
        m.timbre_cond_prosody_enc.last_ln.style.weight.zero_()
        m.timbre_cond_prosody_enc.last_ln.style.bias[:256].zero_()
    m.invalidate()
    sd = state(m)
    beta = sd["timbre_cond_prosody_enc.last_ln.style.bias"][256:]
    m = m.to(DEV)
    n = fro.n_tables(hp)
    B, T = 2, 21
    codes, spk = _codes(hp, B, T, 9)
    cd, sp = codes.to(DEV), spk.to(DEV)
    for prec in PRECS:
        for use_residual in (False, True):
            want = fro.tail_kernel_order(sd, codes.numpy(), np.broadcast_to(beta, (B, 256)), n, use_residual)
            assert np.array_equal(_np(_emb(m, cd, sp, prec, use_residual)), want), (prec, use_residual)
    bad = cd.clone()
    bad[1, 1, 3] = 1 << 10          # the first content table has 2^10 rows
    bad[4, 0, 20] = -1              # a residual row
    with pytest.raises(ValueError, match="outside"):
        m.vq2emb(bad, sp)
    lib = _capi.lib
    h = m._handle
    m.precision = "fp32"
    m.vq2emb(cd, sp)
    need = lib.ab_facodec_redecoder_vq2emb_workspace_bytes(h, B, T)
    ws = torch.empty(need + 512, dtype=torch.uint8, device=DEV)
    wb = (ws.data_ptr() + 255) // 256 * 256
    out = torch.empty(B, 256, T, device=DEV)
    rc = lib.ab_facodec_redecoder_vq2emb(h, _capi.ptr(bad), _capi.shape_array(bad.stride()), 6, B, T, _capi.ptr(sp), 256,
                                         1, _capi.ptr(out), C.c_void_p(wb), need, _capi.stream_ptr())
    assert rc == 0, _capi.last_error()
    torch.cuda.synchronize()
    want = fro.tail_kernel_order(sd, codes.numpy(), np.broadcast_to(beta, (B, 256)), n, True)
    got = _np(out)
    assert np.isnan(got[1, :, 3]).all() and np.isnan(got[0, :, 20]).all()
    mask = np.ones((B, T), bool)
    mask[1, 3] = mask[0, 20] = False
    assert np.array_equal(got.transpose(0, 2, 1)[mask], want.transpose(0, 2, 1)[mask])
    # refusals before any launch leave the output untouched
    out.fill_(float("nan"))
    st = _capi.shape_array(cd.stride())
    for args, msg in (((5, B, wb, need), "code rows"), ((6, 5001, wb, need), "positional"),
                      ((6, B, wb, need - 256), "workspace"), ((6, B, wb + 16, need), "aligned")):
        n_q, b, base, size = args
        assert lib.ab_facodec_redecoder_vq2emb(h, _capi.ptr(cd), st, n_q, b, T, _capi.ptr(sp), 256, 1, _capi.ptr(out),
                                               C.c_void_p(base), size, _capi.stream_ptr()) != 0, msg
        assert msg in _capi.last_error(), (msg, _capi.last_error())
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
    m.timbre_cond_prosody_enc.layers[0].train()
    with pytest.raises(NotImplementedError, match="training mode"):
        m.vq2emb(cd, sp)
    m.eval()
    with pytest.raises(ValueError, match="different devices"):
        m.vq2emb(cd, spk)


@pytest.mark.gpu
def test_readme_voice_conversion():
    """The README's conversion at a small geometry: FACodecEncoder on two utterances, FACodecDecoder.forward(vq=True)
    on each, then vq2emb(vq_id_a, spk_b, use_residual=False) and inference(., spk_b), each step against its oracle on
    the previous step's native output."""
    from amphion_b200.vocoders import FACodecDecoder, FACodecEncoder
    torch.manual_seed(0)
    ehp = dict(ngf=8, up_ratios=[2, 3, 5], out_channels=256)
    enc = FACodecEncoder(**ehp).eval()
    esd = state(enc)
    qhp = fqo.GOLDEN_FACODEC_QUANTIZE["a"][0]
    torch.manual_seed(1)
    dec = FACodecDecoder(**qhp).eval()
    fqo.perturb(dec.named_parameters(), 191)
    with torch.no_grad():
        dec.timbre_encoder.position_emb.pe.copy_(fqo.positional_encoding())
    dec.invalidate()
    dsd = state(dec)
    rhp = fro.GOLDEN_FACODEC_REDECODE["a"][0]
    red = build(rhp, 5)
    rsd = state(red)
    enc, dec, red = enc.to(DEV), dec.to(DEV), red.to(DEV)
    g = torch.Generator().manual_seed(13)
    wav_a, wav_b = (torch.randn(1, 1, 30 * 20, generator=g) * 0.3 for _ in range(2))
    nq = (1, 2, 3)
    for prec in ("fp32", "tc_f16"):
        enc.precision = dec.precision = red.precision = prec
        enc_a, enc_b = enc(wav_a.to(DEV)), enc(wav_b.to(DEV))
        if prec == "fp32":
            for w, e in ((wav_a, enc_a), (wav_b, enc_b)):
                want = feo.encoder(esd, ehp["up_ratios"], w.numpy()).numpy()
                assert _err(e, want) <= BARS[prec] * np.abs(want).max()
        _, vq_id_a, _, _, _ = dec(enc_a, eval_vq=False, vq=True)
        _, _, _, _, spk_b = dec(enc_b, eval_vq=False, vq=True)
        torch.cuda.synchronize()
        assert vq_id_a.shape == (6, 1, 20)
        _, q_free, _, gaps = fqo.quantize(dsd, _np(enc_a), nq)
        clear = gaps.numpy() > fqo.TAU
        assert np.array_equal(_np(vq_id_a)[clear], q_free.numpy()[clear])
        want = fqo.timbre(dsd, _np(enc_b), operands=OPERANDS[prec]).numpy()
        assert _err(spk_b, want) <= BARS[prec] * np.abs(want).max()
        emb = red.vq2emb(vq_id_a, spk_b, use_residual=False)
        out = red.inference(emb, spk_b)
        torch.cuda.synchronize()
        assert out.shape == (1, 1, 20 * 20) and torch.isfinite(out).all()
        want = fro.vq2emb(rsd, _np(vq_id_a), _np(spk_b), nq, False, operands=OPERANDS[prec])
        peak = float(want.abs().max())
        assert _err(emb, want) <= _emb_bar(prec, rsd, _np(vq_id_a), _np(spk_b), nq, False, want, peak)
        want = fro.inference(rsd, rhp["up_ratios"], _np(emb), _np(spk_b), OPERANDS[prec]).numpy()
        err = _err(out, want)
        print(f"facodec voice conversion {prec}: |wav - oracle| / peak = {err / np.abs(want).max():.2e}")
        assert err <= BARS[prec] * np.abs(want).max()


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_profile(tag):
    hp, B, T = fro.GOLDEN_FACODEC_REDECODE[tag]
    m = build(hp, SEEDS[tag]).to(DEV)
    p = fro.n_tables(hp)[0]
    codes, spk = _codes(hp, 2, 50, 1)
    cd, sp = codes.to(DEV), spk.to(DEV)
    for prec, gemm in (("fp32", "conv1d_fp32"), ("tc_f16", "tc_conv")):
        _emb(m, cd, sp, prec)
        m.set_profiling(True)
        _emb(m, cd, sp, prec)
        prof = m.get_profile()
        m.set_profiling(False)
        assert len(prof) == 14
        # 9 style Linears; per prosody table the gather, 4 x (2 style LayerNorms, 4 GEMMs, the attention), last_ln;
        # the tail gather
        assert m.last_launches == 9 + 30 * p + 1
        assert sum(v["launches"] for v in prof.values()) == m.last_launches
        assert prof["facodec_prologue"]["launches"] == 9 + 10 * p + 1
        assert prof["timbre_attention"]["launches"] == 4 * p and prof[gemm]["launches"] == 16 * p
        assert prof["facodec_quantize"]["launches"] == 0 and prof["vocos_norm"]["launches"] == 0
        emb = _emb(m, cd, sp, prec)
        m.set_profiling(True)
        m.inference(emb, sp)
        prof = m.get_profile()
        m.set_profiling(False)
        assert prof["facodec_prologue"]["launches"] == 2      # timbre_linear and the FiLM, then the generator
