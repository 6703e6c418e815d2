"""FACodecEncoderV2.get_prosody_feature and FACodecDecoderV2.forward(x, prosody_feature, vq=True)
(models/codec/ns3_codec/facodec.py:772-1199) on the native kernels.

* CPU: the float64 oracle (tests/facodec_v2_oracle.py) against the reference fixture (tests/golden/fac_v2*.npz, written
  by tests/golden/gen_facodec_v2.py), the redrawn weights' digests, the reference key sets and strict loading, the
  refusals before launch, and V1's handles left exactly as they were.
* GPU: the prosody feature against the native 80-row mel, torch.stft and the fixture; codes outside the near-tie margin,
  outs and the groups' sums bit-equal across precisions, spk_embs at every precision; shapes and views; the input
  kernel and the prosody RVQ bit for bit; the README V2 conversion; the launch count and profile."""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

import facodec_oracle as fo
import facodec_quantize_oracle as fqo
import facodec_v2_oracle as fvo
from conftest import GOLDEN

BARS = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}   # spk_embs and audio, fractions of the peak
OPERANDS = {"fp32": None, "tc_f16": None, "tc_bf16": "bf16"}
FLOOR = 2.0
PRECS = ("fp32", "tc_f16", "tc_bf16")
DEV = "cuda:0"
SEEDS = {"a": 191, "b": 193}
LAUNCHES = 1 + 4 * 7 + 1 + 31
# V1's handles of the parent commit: (tensors, arena bytes) decode-only and quantizing, README and fixture "a" geometry
V1_HANDLES = {"readme": ((196, 104697088), 196 + 6 * 2 + 1 + 4 * 12 + 2), "a": ((70, 1194752), 70 + 6 * 2 + 1 + 4 * 12 + 2)}


def load_fixture():
    d = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "fac_v2*.npz"))):
        z = np.load(p)
        d.update({k: z[k] for k in z.files})
    return d


def variant(d, tag):
    return {k[len(tag) + 1:]: v for k, v in d.items() if k.startswith(tag + ":")}


def build(tag, seed=None):
    """The fixture's modules: the seeds, then the quantizers, transformers and melspec_linear redrawn, pe computed."""
    from amphion_b200.vocoders import FACodecDecoderV2, FACodecEncoderV2
    enc_hp, dec_hp, _, _, _ = fvo.GOLDEN_FACODEC_V2[tag]
    seed = SEEDS[tag] if seed is None else seed
    torch.manual_seed(seed)
    enc = FACodecEncoderV2(**enc_hp).eval()
    dec = FACodecDecoderV2(**dec_hp).eval()
    fvo.perturb(dec.named_parameters(), seed + 100)
    with torch.no_grad():
        for t in (dec.timbre_encoder, dec.melspec_encoder):
            t.position_emb.pe.copy_(fqo.positional_encoding())
    dec.invalidate()
    return enc, dec


def state(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _err(got, want):
    return float(np.abs(_np(got).astype(np.float64) - _np(want).astype(np.float64)).max())


def _nq(hp):
    return (hp["vq_num_q_p"], hp["vq_num_q_c"], hp["vq_num_q_r"])


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_fixture(tag):
    io = variant(load_fixture(), tag)
    enc_hp, dec_hp, B, N, nq = fvo.GOLDEN_FACODEC_V2[tag]
    enc, dec = build(tag)
    sd = state(dec)
    dg = fvo.digests(sd)
    stored = dict(zip(io["digest_names"].tolist(), io["digests"].tolist()))
    assert all(stored[k] == v for k, v in dg.items())
    n = _nq(dec_hp)
    P, layers = fvo.prosody_stream(sd, io["pf"], return_layers=True)
    for i, h in enumerate(layers):
        assert _err(h, io[f"player{i}"]) <= 1e-6 * np.abs(io[f"player{i}"]).max(), i
    outs, qs, bufs, gaps = fvo.quantize(sd, io["enc"], P, n, nq)
    clear = gaps.numpy() > fqo.TAU
    assert clear.mean() > 0.9
    assert np.array_equal(qs.numpy()[clear], io["qs"][clear])
    outs, _, bufs, _ = fvo.quantize(sd, io["enc"], P, n, nq, forced=io["qs"])
    assert _err(outs, io["outs"]) <= 1e-6 * np.abs(io["outs"]).max()
    for i, b in enumerate(bufs):
        assert _err(b, io[f"buf{i}"]) <= 1e-6 * np.abs(io[f"buf{i}"]).max(), i
    spk = fqo.timbre(sd, io["enc"])
    assert _err(spk, io["spk_embs"]) <= 1e-6 * np.abs(io["spk_embs"]).max()


def test_key_sets_and_strict_load():
    """The modules' state dicts have the reference's keys and shapes; a V2 handle lists only state-dict names."""
    from amphion_b200 import _capi
    io = variant(load_fixture(), "a")
    enc, dec = build("a")
    for name, m in (("enc", enc), ("dec", dec)):
        got = {k: ",".join(map(str, v.shape)) for k, v in m.state_dict().items()}
        assert got == dict(zip(io[f"{name}_keys"].tolist(), io[f"{name}_shapes"].tolist())), name
        m.load_state_dict({k: torch.zeros_like(v) for k, v in m.state_dict().items()}, strict=True)
    enc, dec = build("a")
    assert np.allclose(_np(enc.mel_transform.mel_basis), io["mel_basis"], rtol=1e-5, atol=1e-8)
    dec._quantize_handle = True
    h = dec._ensure_handle()
    lib = _capi.lib
    names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(lib.ab_generator_num_tensors(h))]
    sd = dec.state_dict()
    assert len(names) == V1_HANDLES["a"][1] + 2 + 1 + 4 * 12 + 2
    for n in names:
        assert n in sd or (n + "_v" in sd and n + "_g" in sd), n
    for k in sd:
        if k.startswith(("melspec_encoder.", "melspec_linear.", "timbre_encoder.")):
            assert k in names, k


def test_v1_handles_unchanged():
    from amphion_b200 import _capi
    lib = _capi.lib
    for key, hp in (("readme", fo.README_FACODEC), ("a", fqo.GOLDEN_FACODEC_QUANTIZE["a"][0])):
        from amphion_b200.vocoders import FACodecDecoder
        torch.manual_seed(0)
        m = FACodecDecoder(**hp).eval()
        h = m._ensure_handle()
        assert (lib.ab_generator_num_tensors(h), lib.ab_generator_param_bytes(h)) == V1_HANDLES[key][0]
        m._quantize_handle = True
        m._handle = None
        h = m._ensure_handle()
        names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(lib.ab_generator_num_tensors(h))]
        assert len(names) == V1_HANDLES[key][1]
        assert not any(s.startswith("melspec_") for s in names)
        assert m._c_config().facodec_prosody_encoder == 0


def test_refusals_before_launch():
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecDecoderV2
    enc, dec = build("b")
    x, pf = torch.zeros(1, 256, 4), torch.zeros(1, 20, 4)
    with pytest.raises(NotImplementedError, match="get_vq"):
        dec(x, pf, get_vq=True)
    with pytest.raises(NotImplementedError, match="training branch"):
        dec(x, pf, vq=False)
    with pytest.raises(ValueError, match=r"prosody feature of shape \[1, 20, T\]"):
        dec(x, torch.zeros(1, 80, 4))
    with pytest.raises(ValueError, match=r"prosody feature of shape"):
        dec(x, None)
    # N = 16199 at hop 200: the encoder gives 81 frames, the mel 80
    enc_r = type(enc)(ngf=2, up_ratios=(2, 4, 5, 5), out_channels=256)
    assert enc_r.frames(16199) == 81 and enc_r.prosody_frames(16199) == 80
    with pytest.raises(ValueError, match="81 frames and the prosody feature 80"):
        dec(torch.zeros(1, 256, 81), torch.zeros(1, 20, 80))
    with pytest.raises(NotImplementedError, match="CUDA"):
        dec(x, pf)
    small = FACodecDecoderV2(in_channels=16, upsample_initial_channel=64, up_ratios=[3, 2], vq_dim=16).eval()
    with pytest.raises(ValueError, match="256"):
        small(torch.zeros(1, 16, 4), pf)
    # get_prosody_feature: N <= 412 (the reflect pad), a bad shape, a CPU tensor
    with pytest.raises(ValueError, match="412"):
        enc.get_prosody_feature(torch.zeros(1, 1, 412))
    with pytest.raises(ValueError, match=r"\[B, 1, N\]"):
        enc.get_prosody_feature(torch.zeros(1, 413))
    with pytest.raises(RuntimeError, match="CUDA"):
        enc.get_prosody_feature(torch.zeros(1, 1, 413))
    # config: the field needs facodec_quantize, is 0 / 1, belongs to AB_GEN_FACODEC
    lib = _capi.lib
    for edit, ok in ((lambda c: None, True), (lambda c: setattr(c, "facodec_quantize", 0), False),
                     (lambda c: setattr(c, "facodec_prosody_encoder", 2), False),
                     (lambda c: setattr(c, "kind", _capi.GEN_FACODEC_REDECODER), False)):
        c = dec._c_config_decode()
        c.facodec_quantize, c.facodec_prosody_encoder = 1, 1
        edit(c)
        h = C.c_void_p()
        rc = lib.ab_generator_create(C.byref(c), C.byref(h))
        if rc == 0:
            lib.ab_generator_destroy(h)
        assert (rc == 0) == ok
    # the C entries on handles that are not finalized: AB_ERR_STATE before any launch
    dec._quantize_handle = True
    h = dec._ensure_handle()
    st = _capi.shape_array((256 * 4, 4, 1))
    p = C.c_void_p(16)
    assert lib.ab_facodec_quantize_prosody(h, p, st, p, st, 1, 4, 1, p, p, p, p, C.c_void_p(256), 1 << 40, None) == -4
    assert lib.ab_facodec_quantize(h, p, st, 1, 4, 1, p, p, p, p, C.c_void_p(256), 1 << 40, None) == -4


# ------------------------------------------------------------------------------------------------ GPU
def _run(m, x, pf, prec, n_quantizers=None):
    m.precision = prec
    r = m(x, pf, vq=True, n_quantizers=n_quantizers)
    torch.cuda.synchronize()
    return r


@pytest.mark.gpu
def test_c_entry_state_refusals():
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecDecoder
    lib = _capi.lib
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["b"][0]
    v1 = FACodecDecoder(**hp).eval().to(DEV)
    _, v2 = build("b")
    v2 = v2.to(DEV)
    x, pf = torch.zeros(1, 256, 4, device=DEV), torch.zeros(1, 20, 4, device=DEV)
    v1(x, vq=True)
    _run(v2, x, pf, "fp32")
    out = torch.full((4096,), float("nan"), device=DEV)
    ws = torch.empty(1 << 22, dtype=torch.uint8, device=DEV)
    wb = C.c_void_p((ws.data_ptr() + 255) // 256 * 256)
    p, st = C.c_void_p(out.data_ptr()), _capi.shape_array(x.stride())
    pst = _capi.shape_array(pf.stride())
    assert lib.ab_facodec_quantize_prosody(v1._handle, _capi.ptr(x), st, _capi.ptr(pf), pst, 1, 4, 1, p, p, p, p, wb,
                                           1 << 21, None) == -4
    assert "facodec_prosody_encoder" in _capi.last_error()
    assert lib.ab_facodec_quantize(v2._handle, _capi.ptr(x), st, 1, 4, 1, p, p, p, p, wb, 1 << 21, None) == -4
    assert "prosody feature" in _capi.last_error()
    assert lib.ab_facodec_quantize_workspace_bytes(v2._handle, 2, 50) > lib.ab_facodec_quantize_workspace_bytes(
        v1._handle, 2, 50)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
    v2.melspec_encoder.train()
    with pytest.raises(NotImplementedError, match="melspec_encoder in training mode"):
        v2(x, pf, vq=True)
    v2.eval()
    with pytest.raises(ValueError, match="n_quantizers"):
        v2(x, pf, vq=True, n_quantizers=0)


@pytest.mark.gpu
def test_prosody_feature():
    """Bit-equal to rows 0..19 of the native 80-row mel, within 1e-5 of torch.stft + matmul on the same GPU, within
    2e-4 of the fixture; strided input and N = 413."""
    from amphion_b200.mel import native_stft_mel
    io = variant(load_fixture(), "a")
    enc, _ = build("a")
    with torch.no_grad():
        enc.mel_transform.mel_basis.copy_(torch.from_numpy(io["mel_basis"]))
    enc = enc.to(DEV)
    mt = enc.mel_transform
    g = torch.Generator().manual_seed(3)
    for wav in (torch.from_numpy(io["wav"]), torch.randn(3, 1, 413, generator=g) * 0.3,
                torch.randn(2, 1, 16199, generator=g) * 0.3):
        wd = wav.to(DEV)
        pf = enc.get_prosody_feature(wd)
        B, _, N = wav.shape
        assert pf.shape == (B, 20, enc.prosody_frames(N)) and pf.dtype == torch.float32
        _, mel80, _ = native_stft_mel(wd[:, 0], 1024, 200, 800, mt.hann_window, mt.mel_basis, 412, 1e-9)
        assert torch.equal(pf, mel80[:, :20])
        y = torch.nn.functional.pad(wd, (412, 412), mode="reflect").squeeze(1)
        spec = torch.view_as_real(torch.stft(y, 1024, 200, 800, window=mt.hann_window, center=False,
                                             return_complex=True))
        spec = torch.sqrt(spec.pow(2).sum(-1) + 1e-9)
        want = torch.log(torch.clamp(torch.matmul(mt.mel_basis[:20], spec), min=1e-5))
        e = float((pf - want).abs().max())
        print(f"prosody feature N={N}: |native - torch.stft| = {e:.2e}")
        assert e <= 1e-5
        strided = torch.zeros(B, 3, N * 2, device=DEV)[:, 1:2, ::2]
        strided.copy_(wd)
        assert torch.equal(enc.get_prosody_feature(strided), pf)
    pf = enc.get_prosody_feature(torch.from_numpy(io["wav"]).to(DEV))
    e = _err(pf, io["pf"])
    print(f"prosody feature: |native - fixture| = {e:.2e}")
    assert e <= 2e-4


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    io = variant(load_fixture(), tag)
    enc_hp, dec_hp, B, N, nq = fvo.GOLDEN_FACODEC_V2[tag]
    _, dec = build(tag)
    dec = dec.to(DEV)
    sd = state(dec)
    n = _nq(dec_hp)
    P = fvo.prosody_stream(sd, io["pf"])
    p_err = _err(fvo.prosody_stream(sd, io["pf"], dtype=torch.float32), P)
    # the code margin: 8 x the relative error of the prosody group's input when the oracle runs in fp32 arithmetic (a
    # relative input error e moves a distance between unit vectors by at most about 4e); the content and residual
    # inputs are x and one fp32 subtraction, far below that
    margin = max(fqo.TAU, 8.0 * p_err / float(P.abs().max()))
    _, q64, _, gaps = fvo.quantize(sd, io["enc"], P, n, nq)
    x, pf = torch.from_numpy(io["enc"]).to(DEV), torch.from_numpy(io["pf"]).to(DEV)
    res = {}
    for prec in PRECS:
        outs, qs, commit, bufs, spk = _run(dec, x, pf, prec, nq)
        assert qs.dtype == torch.int64 and tuple(qs.shape) == io["qs"].shape
        assert commit.shape == (qs.shape[0],) and not commit.any()
        assert len(bufs) == (3 if n[2] else 2) and not spk.requires_grad
        assert dec.last_launches == LAUNCHES
        res[prec] = [_np(outs), _np(qs)] + [_np(b) for b in bufs] + [_np(spk)]
    qs = res["fp32"][1]
    clear = gaps.numpy() > margin
    print(f"facodec v2 {tag}: margin {margin:.1e}, {int((~clear).sum())} of {clear.size} codes inside it, "
          f"{int((qs != io['qs']).sum())} differ from the fixture")
    assert np.array_equal(qs[clear], io["qs"][clear])
    outs_o, _, bufs_o, _ = fvo.quantize(sd, io["enc"], P, n, nq, forced=qs)
    peak = np.abs(io["outs"]).max()
    e = _err(res["fp32"][0], outs_o)
    print(f"facodec v2 {tag}: |outs - oracle| / peak = {e / peak:.2e}")
    assert e <= 2e-6 * peak
    for i, b in enumerate(bufs_o):
        assert _err(res["fp32"][2 + i], b) <= 2e-6 * np.abs(io[f"buf{i}"]).max(), i
    for prec in ("tc_f16", "tc_bf16"):   # the prosody transformer and the RVQ are fp32 at every precision
        for a, b in zip(res[prec][:-1], res["fp32"][:-1]):
            assert np.array_equal(a, b), prec
    speak = np.abs(io["spk_embs"]).max()
    for prec in PRECS:
        want = fqo.timbre(sd, io["enc"], operands=OPERANDS[prec]).numpy()
        ref = want if prec != "tc_f16" else res["fp32"][-1]
        err = _err(res[prec][-1], ref)
        bar = BARS[prec] * speak
        if prec == "tc_bf16":
            bar = max(bar, FLOOR * _err(fqo.timbre(sd, io["enc"], operands="bf16", dtype=torch.float32).numpy(), want))
        print(f"facodec v2 {tag} {prec}: |spk - oracle| / peak = {err / speak:.2e}")
        assert err <= bar, prec


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 63, 64, 65, 333])
def test_shapes_and_views(T):
    _, dec = build("a")
    dec = dec.to(DEV)
    sd = state(dec)
    n = (1, 2, 3)
    g = torch.Generator().manual_seed(T)
    x = torch.randn(2, 256, T, generator=g)
    pf = torch.randn(2, 20, T, generator=g) * 2 - 6
    xt = x.transpose(1, 2).contiguous().transpose(1, 2)
    pft = torch.zeros(2, 40, 2 * T)[:, ::2, ::2]
    pft.copy_(pf)
    P = fvo.prosody_stream(sd, pf.numpy())
    for prec in ("fp32", "tc_bf16"):
        for k in (None, 1, 2):
            outs, qs, _, bufs, spk = _run(dec, xt.to(DEV), pft.to(DEV), prec, k)
            ref = _run(dec, x.to(DEV), pf.to(DEV), prec, k)
            assert torch.equal(outs, ref[0]) and torch.equal(qs, ref[1]) and torch.equal(spk, ref[4])
            assert qs.shape[0] == sum(min(k or 3, c) for c in n)
            _, q_free, _, gaps = fvo.quantize(sd, x.numpy(), P, n, k)
            clear = gaps.numpy() > 1e-4
            assert np.array_equal(_np(qs)[clear], q_free.numpy()[clear])
            o, _, _, _ = fvo.quantize(sd, x.numpy(), P, n, k, forced=_np(qs))
            assert _err(outs, o) <= 2e-6 * float(o.abs().max())


@pytest.mark.gpu
def test_swapped_utterances_and_repeat_runs():
    _, dec = build("a")
    dec = dec.to(DEV)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(3, 256, 40, generator=g).to(DEV)
    pf = (torch.randn(3, 20, 40, generator=g) * 2 - 6).to(DEV)
    perm = [1, 0, 2]
    a = _run(dec, x, pf, "fp32")
    b = _run(dec, x[perm], pf[perm], "fp32")
    # pe[b] enters both transformers, so swapping utterances changes the prosody stream; the native run of the swapped
    # batch must still match the oracle of the swapped batch
    sd = state(dec)
    P = fvo.prosody_stream(sd, _np(pf[perm]))
    o, _, _, _ = fvo.quantize(sd, _np(x[perm]), P, (1, 2, 3), forced=_np(b[1]))
    assert _err(b[0], o) <= 2e-6 * float(o.abs().max())
    for prec in PRECS:
        r1, r2 = _run(dec, x, pf, prec), _run(dec, x, pf, prec)
        for u, v in zip(r1, r2):
            if isinstance(u, list):
                assert all(torch.equal(p, q) for p, q in zip(u, v))
            else:
                assert torch.equal(u, v), prec


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_prosody_input_exact(dense):
    from amphion_b200 import _capi
    rng = np.random.default_rng(11 + dense)
    B, T = 3, 37
    if dense:
        w = rng.normal(0, 1, (256, 20)).astype(np.float32)
    else:
        w = np.zeros((256, 20), np.float32)
        w[np.arange(256), rng.integers(0, 20, 256)] = 1.0
    bias = rng.normal(0, 0.1, 256).astype(np.float32)
    pe = fqo.positional_encoding().numpy()
    pf = (rng.normal(0, 2, (B, 20, T)) - 6).astype(np.float32)
    want = fvo.prosody_input_exact(w, bias, pe, pf)
    pft = torch.zeros(B, 20, 3 * T)[:, :, ::3]
    pft.copy_(torch.from_numpy(pf))
    pft = pft.to(DEV)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in dict(w=w, bias=bias, pe=pe).items()}
    y = torch.full((B, 256, T), float("nan"), device=DEV)
    _capi.check(_capi.lib.ab_facodec_prosody_input_forward(_capi.ptr(pft), _capi.shape_array(pft.stride()),
                                                           _capi.ptr(t["w"]), _capi.ptr(t["bias"]), _capi.ptr(t["pe"]),
                                                           B, T, _capi.ptr(y), _capi.stream_ptr()), "prosody input")
    torch.cuda.synchronize()
    assert np.array_equal(_np(y), want)


@pytest.mark.gpu
def test_prosody_rvq_exact():
    """last_ln.weight = 0: the prosody stream is last_ln.bias exactly; one-hot projections and a tied codebook pair:
    codes, outs and the sums bit-equal to the kernel-order oracle, the tie going to the lowest code."""
    _, dec = build("a")
    rng = np.random.default_rng(0)
    with torch.no_grad():
        for name, p in dec.named_parameters():
            if name.startswith("quantizer."):
                if name.endswith("weight_g"):
                    p.fill_(1.0)
                elif name.endswith("in_proj.weight_v"):
                    p.zero_()
                    p[torch.arange(p.shape[0]), torch.from_numpy(rng.choice(256, p.shape[0], replace=False))] = 1.0
                elif name.endswith("out_proj.weight_v"):
                    p.zero_()
                    p[torch.arange(p.shape[0]), torch.from_numpy(rng.integers(0, p.shape[1], p.shape[0]))] = 1.0
                elif name.endswith("_codebook.weight"):
                    cb = torch.from_numpy(rng.normal(0, 1, tuple(p.shape)).astype(np.float32))
                    cb[5] = 2.0 * cb[3]
                    p.copy_(cb)
                elif name.endswith("in_proj.bias"):
                    p.zero_()
        dec.melspec_encoder.last_ln.weight.zero_()
        beta = torch.from_numpy(rng.normal(0, 1, 256).astype(np.float32))
        # the prosody layer's z_e points along codebook row 3 (= row 5, the same direction): a tie at every frame
        w_in = fqo._weight({k: v.numpy() for k, v in dec.state_dict().items()}, "quantizer.0.layers.0.in_proj").numpy()
        beta[torch.from_numpy(w_in.argmax(1))] = dec.quantizer[0].layers[0]._codebook.weight[3] * 1.5
        dec.melspec_encoder.last_ln.bias.copy_(beta)
    dec.invalidate()
    dec = dec.to(DEV)
    sd = state(dec)
    B, T = 2, 37
    x = rng.normal(0, 1, (B, 256, T)).astype(np.float32)
    pf = (rng.normal(0, 2, (B, 20, T)) - 6).astype(np.float32)
    P = np.broadcast_to(beta.numpy()[None, :, None], (B, 256, T)).astype(np.float32)
    want_outs, want_qs, want_bufs = fvo.quantize_kernel_order(sd, x, P, (1, 2, 3))
    assert (want_qs[0] == 3).all()
    for prec in PRECS:
        outs, qs, _, bufs, _ = _run(dec, torch.from_numpy(x).to(DEV), torch.from_numpy(pf).to(DEV), prec)
        assert np.array_equal(_np(qs), want_qs), prec
        assert np.array_equal(_np(outs), want_outs), prec
        for b, w in zip(bufs, want_bufs):
            assert np.array_equal(_np(b), w), prec


@pytest.mark.gpu
def test_readme_v2_conversion():
    """README V2 flow on the fixture: encoder and get_prosody_feature on A and B, forward(vq=True) x 2,
    vq2emb(codes of A, use_residual=False), inference(., spk of B), at each precision."""
    io = variant(load_fixture(), "a")
    enc, dec = build("a")
    with torch.no_grad():
        enc.mel_transform.mel_basis.copy_(torch.from_numpy(io["mel_basis"]))
    enc, dec = enc.to(DEV), dec.to(DEV)
    sd = state(dec)
    wa, wb = torch.from_numpy(io["wav"]).to(DEV), torch.from_numpy(io["wav_b"]).to(DEV)
    peak = np.abs(io["vc"]).max()
    for prec in PRECS:
        enc.precision = dec.precision = prec
        ha, hb = enc(wa), enc(wb)
        pa, pb = enc.get_prosody_feature(wa), enc.get_prosody_feature(wb)
        _, qa, _, _, _ = dec(ha, pa, vq=True)
        _, qb, _, _, spk_b = dec(hb, pb, vq=True)
        emb = dec.vq2emb(qa, use_residual=False)
        wav = dec.inference(emb, spk_b)
        torch.cuda.synchronize()
        assert wav.shape == io["vc"].shape
        if prec == "fp32":
            assert np.array_equal(_np(qa), io["qs"]) and np.array_equal(_np(qb), io["qs_b"])
            e = _err(emb, io["emb_nores"])
            assert e <= 1e-5 * np.abs(io["emb_nores"]).max()
        e = _err(wav, io["vc"])
        print(f"facodec v2 README conversion {prec}: |wav - fixture| / peak = {e / peak:.2e}")
        # the fp32 fixture is the reference at every precision here: no bf16-operand restatement of the encoder and
        # the generator is run, so tc_bf16 gets the end-to-end bar of 3e-2 (measured 1.1e-2 on an H100 80GB HBM3)
        assert e <= (3e-2 if prec == "tc_bf16" else BARS[prec]) * peak, prec


@pytest.mark.gpu
def test_profile():
    _, dec = build("a")
    dec = dec.to(DEV)
    x, pf = torch.randn(2, 256, 50).to(DEV), torch.randn(2, 20, 50).to(DEV)
    for prec, gemm in (("fp32", "conv1d_fp32"), ("tc_f16", "tc_conv")):
        dec.precision = prec
        dec(x, pf, vq=True)
        dec.set_profiling(True)
        dec(x, pf, vq=True)
        prof = dec.get_profile()
        dec.set_profiling(False)
        assert len(prof) == 14 and dec.last_launches == LAUNCHES
        assert sum(v["launches"] for v in prof.values()) == LAUNCHES
        assert prof["facodec_prologue"]["launches"] == 1 and prof["facodec_quantize"]["launches"] == 2
        assert prof["timbre_attention"]["launches"] == 8 and prof["vocos_norm"]["launches"] == 18
        assert prof["conv1d_fp32"]["launches"] == 16 + (16 if prec == "fp32" else 0)
        assert prof[gemm]["launches"] >= 16
