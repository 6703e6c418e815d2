"""FACodecDecoder.forward(vq=True) (models/codec/ns3_codec/facodec.py:408-471) on the native kernels: the residual
vector quantizers, the timbre encoder and the speaker embedding.

* CPU: the float64 oracle (tests/facodec_quantize_oracle.py) against the reference fixture (tests/golden/fac_quantize*.npz,
  written by tests/golden/gen_facodec_quantize.py), the redrawn weights' digests, strict loading of the README state
  dict, the refusals before launch, and the decode-only handle left exactly as it was.
* GPU: codes against the fixture outside the near-tie band, outs and the groups' sums bit-equal across precisions,
  one-hot projections bit for bit against the kernel-order oracle (ties included), spk_embs at every precision, ragged
  shapes, the positional quirk, repeat runs, the README round trip and the profile."""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

import facodec_oracle as fo
import facodec_quantize_oracle as fqo
from conftest import GOLDEN

BARS = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}   # spk_embs, fractions of its peak (test_facodec.py's bars)
OPERANDS = {"fp32": None, "tc_f16": None, "tc_bf16": "bf16"}   # tc_f16 against the fp32 oracle, bf16 operand-rounded
FLOOR = 2.0
PRECS = ("fp32", "tc_f16", "tc_bf16")
DEV = "cuda:0"
# the decode-only handles of the parent commit: (tensors, arena bytes, workspace bytes at B = 2, T = 50)
DECODE_ONLY = {"readme": (196, 104697088, 46186496), "a": (70, 1194752, 221696)}
SEEDS = {"a": 91, "b": 93}


def load_fixture():
    d = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "fac_quantize*.npz"))):
        z = np.load(p)
        d.update({k: z[k] for k in z.files})
    return d


def variant(d, tag):
    return {k[len(tag) + 1:]: v for k, v in d.items() if k.startswith(tag + ":")}


def build(hp, seed):
    """The fixture's module: the generator's seed, then the quantizers and the timbre encoder redrawn, pe computed."""
    from amphion_b200.vocoders import FACodecDecoder
    torch.manual_seed(seed)
    m = FACodecDecoder(**hp).eval()
    fqo.perturb(m.named_parameters(), seed + 100)
    with torch.no_grad():
        m.timbre_encoder.position_emb.pe.copy_(fqo.positional_encoding())
    m.invalidate()
    return m


def state(m):
    return {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _err(got, want):
    return float(np.abs(_np(got).astype(np.float64) - _np(want).astype(np.float64)).max())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_fixture(tag):
    io = variant(load_fixture(), tag)
    hp, B, T, nq = fqo.GOLDEN_FACODEC_QUANTIZE[tag]
    m = build(hp, SEEDS[tag])
    sd = state(m)
    dg = fqo.digests(sd)
    assert dict(zip(io["digest_names"].tolist(), io["digests"].tolist())) == dg
    n = (hp["vq_num_q_p"], hp["vq_num_q_c"], hp["vq_num_q_r"])
    outs, qs, bufs, gaps = fqo.quantize(sd, io["x"], n, nq)
    clear = gaps.numpy() > fqo.TAU
    assert clear.mean() > 0.9
    assert np.array_equal(qs.numpy()[clear], io["qs"][clear])
    outs, qs, bufs, _ = fqo.quantize(sd, io["x"], n, nq, forced=io["qs"])
    peak = np.abs(io["outs"]).max()
    assert _err(outs, io["outs"]) <= 1e-6 * peak
    for i, b in enumerate(bufs):
        assert _err(b, io[f"buf{i}"]) <= 1e-6 * np.abs(io[f"buf{i}"]).max(), i
    spk, layers = fqo.timbre(sd, io["x"], return_layers=True)
    for i, h in enumerate(layers):
        assert _err(h, io[f"layer{i}"]) <= 1e-6 * np.abs(io[f"layer{i}"]).max(), i
    assert _err(spk, io["spk_embs"]) <= 1e-6 * np.abs(io["spk_embs"]).max()


def test_readme_state_dict_loads_strictly():
    """The handle with quantization lists only the reference's names, each with the state dict's shape."""
    from amphion_b200 import _capi
    m = build(fo.README_FACODEC, 0)
    m._quantize_handle = True
    h = m._ensure_handle()
    lib = _capi.lib
    names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(lib.ab_generator_num_tensors(h))]
    sd = m.state_dict()
    assert len(names) == 196 + 6 * 2 + 1 + 4 * 12 + 2
    for n in names:
        assert n in sd or (n + "_v" in sd and n + "_g" in sd), n
    for k in sd:
        if k.startswith("timbre_encoder."):
            assert k in names, k
    m.load_state_dict({k: torch.zeros_like(v) for k, v in sd.items()}, strict=True)


def test_decode_only_handle_unchanged():
    from amphion_b200 import _capi
    lib = _capi.lib
    for key, hp in (("readme", fo.README_FACODEC), ("a", fqo.GOLDEN_FACODEC_QUANTIZE["a"][0])):
        m = build(hp, 0)
        h = m._ensure_handle()
        n = lib.ab_generator_num_tensors(h)
        assert (n, lib.ab_generator_param_bytes(h), lib.ab_generator_workspace_bytes(h, 2, 50)) == DECODE_ONLY[key]
        names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(n)]
        assert not any(s.startswith("timbre_encoder.") or ".in_proj." in s for s in names)
        assert lib.ab_facodec_quantize_workspace_bytes(h, 2, 50) == 0
        assert m._c_config().facodec_quantize == 0


def test_refusals_before_launch():
    from amphion_b200 import _capi
    from amphion_b200.vocoders import FACodecDecoder
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["b"][0]
    m = build(hp, 0)
    # the CPU tensor first, with the served list
    with pytest.raises(NotImplementedError, match="vq2emb"):
        m(torch.zeros(1, 256, 4))
    with pytest.raises(NotImplementedError, match="training branch"):
        m(torch.zeros(1, 256, 4), vq=False)
    with pytest.raises(NotImplementedError, match="get_vq"):
        m(torch.zeros(1, 256, 4), get_vq=True)
    # a 16-channel decoder: the device check, then in_channels
    small = FACodecDecoder(in_channels=16, upsample_initial_channel=64, up_ratios=[3, 2], vq_dim=16).eval()
    with pytest.raises(NotImplementedError, match="vq2emb"):
        small(torch.zeros(1, 16, 4))
    if torch.cuda.is_available():
        with pytest.raises(ValueError, match="256"):
            small(torch.zeros(1, 16, 4, device=DEV))
    lib = _capi.lib
    # config: the field belongs to FACodec, and needs n_mel == 256
    for edit, ok in ((lambda c: None, True), (lambda c: setattr(c, "n_mel", 128), False),
                     (lambda c: setattr(c, "facodec_quantize", 2), False),
                     (lambda c: setattr(c, "kind", _capi.GEN_FACODEC_ENCODER), False)):
        c = m._c_config_decode()
        c.facodec_quantize = 1
        edit(c)
        h = C.c_void_p()
        rc = lib.ab_generator_create(C.byref(c), C.byref(h))
        if rc == 0:
            lib.ab_generator_destroy(h)
        assert (rc == 0) == ok
    # the C entry: a decode-only handle (AB_ERR_STATE), n_quantizers < 1, B > the rows of pe; all before any launch
    st = _capi.shape_array((256 * 4, 4, 1))
    args = lambda h, B, k: (h, C.c_void_p(16), st, B, 4, k, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16),
                            C.c_void_p(256), 1 << 40, None)
    h0 = m._ensure_handle()
    lib.ab_generator_bind_params(h0, C.c_void_p(256), lib.ab_generator_param_bytes(h0))
    assert lib.ab_facodec_quantize(*args(h0, 1, 1)) != 0   # not finalized, or not a quantize handle
    m2 = build(hp, 0)
    m2._quantize_handle = True
    h2 = m2._ensure_handle()
    assert lib.ab_facodec_quantize(*args(h2, 1, 1)) == -4 and "finalize" in _capi.last_error()   # AB_ERR_STATE


# ------------------------------------------------------------------------------------------------ GPU
def _run(m, x, prec, n_quantizers=None):
    m.precision = prec
    r = m(x, vq=True, n_quantizers=n_quantizers)
    torch.cuda.synchronize()
    return r


@pytest.mark.gpu
def test_c_entry_refusals():
    from amphion_b200 import _capi
    lib = _capi.lib
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["b"][0]
    m = build(hp, 0).to(DEV)
    x = torch.zeros(1, 256, 4, device=DEV)
    m.vq2emb(torch.zeros(3, 1, 4, dtype=torch.long, device=DEV))   # a decode-only handle
    h = m._handle
    st = _capi.shape_array(x.stride())
    out = torch.full((4096,), float("nan"), device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    wb = C.c_void_p((ws.data_ptr() + 255) // 256 * 256)
    p = C.c_void_p(out.data_ptr())
    assert lib.ab_facodec_quantize(h, _capi.ptr(x), st, 1, 4, 1, p, p, p, p, wb, 1 << 19, None) == -4   # AB_ERR_STATE
    assert "without facodec_quantize" in _capi.last_error()
    _run(m, x, "fp32")
    h = m._handle
    for B, k, msg in ((1, 0, "n_quantizers"), (5001, 1, "positional")):
        assert lib.ab_facodec_quantize(h, _capi.ptr(x), st, B, 4, k, p, p, p, p, wb, 1 << 19, None) != 0
        assert msg in _capi.last_error()
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
    with pytest.raises(ValueError, match="n_quantizers"):
        m(x, vq=True, n_quantizers=0)
    m.timbre_encoder.train()
    with pytest.raises(NotImplementedError, match="training mode"):
        m(x, vq=True)
    m.eval()
    m.quantizer.train()
    m(x, vq=True)                       # eval_vq=True puts the quantizer in eval, as the reference does
    m.quantizer.train()
    with pytest.raises(NotImplementedError, match="training mode"):
        m(x, vq=True, eval_vq=False)


def _check_codes(qs, io_qs, gaps, tag):
    clear = gaps > fqo.TAU
    assert np.array_equal(qs[clear], io_qs[clear]), tag
    n_band = int((~clear).sum())
    print(f"facodec quantize {tag}: {n_band} of {clear.size} codes inside the near-tie band, "
          f"{int((qs != io_qs).sum())} differ from the fixture")


def _near(qs, sd, x, n, nq):
    """Inside the band, the native code must be one of the near-tied codes of the float64 oracle (teacher-forced)."""
    _, _, _, gaps = fqo.quantize(sd, x, n, nq, forced=qs)
    return gaps


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    io = variant(load_fixture(), tag)
    hp, B, T, nq = fqo.GOLDEN_FACODEC_QUANTIZE[tag]
    m = build(hp, SEEDS[tag]).to(DEV)
    sd = state(m)
    n = (hp["vq_num_q_p"], hp["vq_num_q_c"], hp["vq_num_q_r"])
    x = torch.from_numpy(io["x"]).to(DEV)
    _, _, _, gaps = fqo.quantize(sd, io["x"], n, nq)
    res = {}
    for prec in PRECS:
        outs, qs, commit, bufs, spk = _run(m, x, prec, nq)
        assert qs.dtype == torch.int64 and tuple(qs.shape) == io["qs"].shape
        assert commit.shape == (qs.shape[0],) and not commit.any()
        assert len(bufs) == (3 if n[2] else 2) and all(b.shape == (B, 256, T) for b in bufs)
        assert not outs.requires_grad and not spk.requires_grad and spk.shape == (B, 256)
        # 1 RVQ launch, per layer 2 LayerNorms, 4 GEMMs and the attention, last_ln, the time mean
        assert m.last_launches == 1 + 4 * 7 + 2
        res[prec] = [_np(outs), _np(qs)] + [_np(b) for b in bufs] + [_np(spk)]
    qs = res["fp32"][1]
    _check_codes(qs, io["qs"], gaps.numpy(), tag)
    # teacher-forced: the oracle continues with the native codes
    outs_o, _, bufs_o, _ = fqo.quantize(sd, io["x"], n, nq, forced=qs)
    peak = np.abs(io["outs"]).max()
    e = _err(res["fp32"][0], outs_o)
    print(f"facodec quantize {tag}: |outs - oracle| / peak = {e / peak:.2e}")
    assert e <= 2e-6 * peak
    if np.array_equal(qs, io["qs"]):
        assert _err(res["fp32"][0], io["outs"]) <= 2e-6 * peak
    for i, b in enumerate(bufs_o):
        assert _err(res["fp32"][2 + i], b) <= 2e-6 * np.abs(io[f"buf{i}"]).max(), i
    for prec in ("tc_f16", "tc_bf16"):   # the RVQ is fp32 at every precision: bit-equal
        for a, b in zip(res[prec][:-1], res["fp32"][:-1]):
            assert np.array_equal(a, b), prec
    speak = np.abs(io["spk_embs"]).max()
    for prec in PRECS:
        spk = res[prec][-1]
        want = fqo.timbre(sd, io["x"], operands=OPERANDS[prec]).numpy()
        err = _err(spk, want)
        bar = BARS[prec] * speak
        if prec != "fp32":
            floor = _err(fqo.timbre(sd, io["x"], operands=OPERANDS[prec], dtype=torch.float32).numpy(), want)
            bar = max(bar, FLOOR * floor)
            print(f"  {prec}: fp32-arithmetic oracle floor / peak = {floor / speak:.2e}")
        print(f"facodec quantize {tag} {prec}: |spk - oracle| / peak = {err / speak:.2e} "
              f"(|spk - fixture| / peak = {_err(spk, io['spk_embs']) / speak:.2e})")
        assert err <= bar, prec


def _one_hot_module(n_rows_bits=4, seed=0):
    """A small decoder whose in_proj / out_proj fold to one-hot weights (g = 1, one-hot v) and whose codebooks have a
    tied pair: row 5 = 2 x row 3 (the same direction, so the same normalised row), other rows apart."""
    hp = dict(fqo.GOLDEN_FACODEC_QUANTIZE["a"][0], codebook_size_prosody=n_rows_bits, codebook_size_content=n_rows_bits,
              codebook_size_residual=n_rows_bits)
    m = build(hp, seed)
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if not name.startswith("quantizer."):
                continue
            if name.endswith("weight_g"):
                p.fill_(1.0)
            elif name.endswith("in_proj.weight_v"):    # [D, C]: z_e[d] = x[cols[d]] + b[d]
                p.zero_()
                cols = rng.choice(256, p.shape[0], replace=False)
                p[torch.arange(p.shape[0]), torch.from_numpy(cols)] = 1.0
            elif name.endswith("out_proj.weight_v"):   # [C, D]: q[c] = z_q[d(c)] + b[c]
                p.zero_()
                p[torch.arange(p.shape[0]), torch.from_numpy(rng.integers(0, p.shape[1], p.shape[0]))] = 1.0
            elif name.endswith("_codebook.weight"):
                cb = torch.from_numpy(rng.normal(0, 1, tuple(p.shape)).astype(np.float32))
                cb[5] = 2.0 * cb[3]
                p.copy_(cb)
            elif name.endswith("in_proj.bias"):
                p.zero_()
            else:
                p.copy_(torch.from_numpy(rng.normal(0, 0.1, tuple(p.shape)).astype(np.float32)))
    m.invalidate()
    return m


@pytest.mark.gpu
def test_one_hot_projections_are_exact():
    m = _one_hot_module()
    sd = state(m)
    rng = np.random.default_rng(1)
    B, T = 2, 37
    x = rng.normal(0, 1, (B, 256, T)).astype(np.float32)
    # frames 0..5 of utterance 0 point the prosody layer's z_e along codebook row 3 (= row 5): a tie, lowest code 3
    w_in = fqo._weight(sd, "quantizer.0.layers.0.in_proj").numpy()
    cols = w_in.argmax(1)
    cb = sd["quantizer.0.layers.0._codebook.weight"]
    for t in range(6):
        x[0, cols, t] = cb[3] * (1.5 + 0.25 * t)
    m = m.to(DEV)
    n = (1, 2, 3)
    want_outs, want_qs, want_bufs = fqo.quantize_kernel_order(sd, x, n)
    _, _, _, gaps = fqo.quantize(sd, x, n)
    ties = gaps.numpy() == 0
    assert ties[0, 0, :6].all()
    assert (gaps.numpy()[~ties] > 1e-4).all()
    assert (want_qs[0, 0, :6] == 3).all()
    for prec in PRECS:
        outs, qs, _, bufs, _ = _run(m, torch.from_numpy(x).to(DEV), prec)
        assert np.array_equal(_np(qs), want_qs), prec
        assert np.array_equal(_np(outs), want_outs), prec
        for b, w in zip(bufs, want_bufs):
            assert np.array_equal(_np(b), w), prec


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 63, 64, 65, 333])
def test_shapes(T):
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["a"][0]
    m = build(hp, SEEDS["a"]).to(DEV)
    sd = state(m)
    n = (1, 2, 3)
    g = torch.Generator().manual_seed(T)
    x = torch.randn(2, 256, T, generator=g)
    xt = x.transpose(1, 2).contiguous().transpose(1, 2)     # a [B, C, T] view with time stride 256
    for prec in ("fp32", "tc_bf16"):
        for k in (None, 1, 2):
            outs, qs, _, bufs, spk = _run(m, xt.to(DEV), prec, k)
            ref = _run(m, x.to(DEV), prec, k)
            assert torch.equal(outs, ref[0]) and torch.equal(qs, ref[1]) and torch.equal(spk, ref[4])
            assert qs.shape[0] == sum(min(k or 3, c) for c in n)
            _, _, _, gaps = fqo.quantize(sd, x.numpy(), n, k)
            o, q, b, _ = fqo.quantize(sd, x.numpy(), n, k, forced=_np(qs))
            clear = gaps.numpy() > fqo.TAU
            _, q_free, _, _ = fqo.quantize(sd, x.numpy(), n, k)
            assert np.array_equal(_np(qs)[clear], q_free.numpy()[clear])
            assert _err(outs, o) <= 2e-6 * float(o.abs().max())
        want = fqo.timbre(sd, x.numpy(), operands=OPERANDS[prec]).numpy()
        peak = np.abs(want).max()
        bar = BARS[prec] * peak
        if prec != "fp32":
            bar = max(bar, FLOOR * _err(fqo.timbre(sd, x.numpy(), operands=OPERANDS[prec], dtype=torch.float32).numpy(),
                                        want))
        err = _err(spk, want)
        print(f"facodec quantize T={T} {prec}: |spk - oracle| / peak = {err / peak:.2e}")
        assert err <= bar


@pytest.mark.gpu
def test_position_quirk_and_repeat_runs():
    """Utterance b adds row b of pe: swapping two utterances changes their spk_embs as the oracle says, and not their
    codes.  Two runs are bit-equal."""
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["a"][0]
    m = build(hp, SEEDS["a"]).to(DEV)
    sd = state(m)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(3, 256, 40, generator=g)
    xs = x[[1, 0, 2]]
    a = _run(m, x.to(DEV), "fp32")
    b = _run(m, xs.to(DEV), "fp32")
    assert torch.equal(a[1][:, [1, 0, 2]], b[1])
    assert torch.equal(a[0][[1, 0, 2]], b[0])
    want_a = fqo.timbre(sd, x.numpy()).numpy()
    want_b = fqo.timbre(sd, xs.numpy()).numpy()
    moved = np.abs(want_b[0] - want_a[1]).max()
    assert moved > 1e-3                                  # the position changes the embedding
    peak = np.abs(want_a).max()
    assert _err(b[4].cpu(), want_b) <= BARS["fp32"] * peak
    assert _err(a[4].cpu(), want_a) <= BARS["fp32"] * peak
    for prec in PRECS:
        r1, r2 = _run(m, x.to(DEV), prec), _run(m, x.to(DEV), prec)
        for u, v in zip(r1, r2):
            if isinstance(u, list):
                assert all(torch.equal(p, q) for p, q in zip(u, v))
            else:
                assert torch.equal(u, v), prec


@pytest.mark.gpu
def test_readme_round_trip():
    """README flow at its geometry: encoder -> forward(vq=True) -> vq2emb(qs) -> inference.  vq2emb reproduces outs;
    inference is bit-equal before and after the handle gained the quantizer and the timbre encoder."""
    import facodec_encode_oracle as feo
    from amphion_b200.vocoders import FACodecEncoder
    torch.manual_seed(0)
    enc = FACodecEncoder(**feo.README_FACODEC_ENCODER).eval().to(DEV)
    dec = build(fo.README_FACODEC, 3).to(DEV)
    g = torch.Generator().manual_seed(5)
    wav = (torch.randn(2, 1, 16000, generator=g) * 0.3).to(DEV)
    for prec in ("fp32", "tc_f16"):
        enc.precision = dec.precision = prec
        h = enc(wav)
        spk_in = torch.randn(2, 256, generator=g).to(DEV)
        if prec == "fp32":
            z = torch.randn(2, 256, 80, generator=g).to(DEV)
            before = dec.inference(z, spk_in)
        outs, qs, _, bufs, spk = dec(h, vq=True)
        assert qs.shape == (6, 2, 80) and spk.shape == (2, 256)
        emb = dec.vq2emb(qs)
        peak = float(outs.abs().max())
        e = float((emb - outs).abs().max())
        print(f"facodec readme {prec}: |vq2emb(qs) - outs| / peak = {e / peak:.2e}")
        assert e <= 1e-6 * peak
        wav_out = dec.inference(emb, spk)
        assert wav_out.shape == (2, 1, 80 * 200) and torch.isfinite(wav_out).all()
        if prec == "fp32":
            assert torch.equal(dec.inference(z, spk_in), before)


@pytest.mark.gpu
def test_profile():
    hp = fqo.GOLDEN_FACODEC_QUANTIZE["a"][0]
    m = build(hp, SEEDS["a"]).to(DEV)
    x = torch.randn(2, 256, 50).to(DEV)
    m.vq2emb(torch.zeros(6, 1, 4, dtype=torch.long, device=DEV))
    m.set_profiling(True)
    m.vq2emb(torch.zeros(6, 1, 4, dtype=torch.long, device=DEV))
    assert len(m.get_profile()) == 12                     # a decode-only handle reports its classes
    for prec, gemm in (("fp32", "conv1d_fp32"), ("tc_f16", "tc_conv")):
        m.precision = prec
        m.set_profiling(False)
        m(x, vq=True)
        m.set_profiling(True)
        m(x, vq=True)
        prof = m.get_profile()
        m.set_profiling(False)
        assert len(prof) == 14
        assert m.last_launches == 31
        assert sum(v["launches"] for v in prof.values()) == m.last_launches
        assert prof["facodec_quantize"]["launches"] == 2 and prof["timbre_attention"]["launches"] == 4
        assert prof[gemm]["launches"] == 16 and prof["vocos_norm"]["launches"] == 9
