"""The acoustic codec of MaskGCT, Metis and DebaTTS (amphion_b200.vocoders.CodecEncoder / CodecDecoder) against the
reference's own outputs (tests/golden/amphion_codec*.npz, tests/golden/gen_amphion_codec.py) and the float64 oracle
(tests/amphion_codec_oracle.py).  Bars (DESIGN §3, the FACodec rows): encoder and waveform fp32 2e-5 of the peak,
tc_f16 1e-3 of the peak against fp32, tc_bf16 4e-3 against the bf16-operand oracle; codes equal to the reference's
wherever the float64 gap between the best and the runner-up distance exceeds TAU; quantized_out and all_quantized 2e-6
of the peak against the oracle teacher-forced with the native codes, and bit-equal across precisions."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import amphion_codec_oracle as aco
from conftest import load_golden

DEV = "cuda:0"
PRECS = ["fp32", "tc_f16", "tc_bf16"]
OPERANDS = {"fp32": None, "tc_f16": "f16", "tc_bf16": "bf16"}


def _golden():
    return load_golden("amphion_codec")[0]


def _build(tag, precision="fp32"):
    """The native encoder and decoder of fixture `tag`: seeded construction, the fixture's perturbation, and its
    digests checked (so the draw order is the reference's)."""
    from amphion_b200.vocoders import CodecDecoder, CodecEncoder
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC[tag]
    torch.manual_seed(aco.SEEDS[tag])
    enc, dec = CodecEncoder(**enc_hp).eval(), CodecDecoder(**dec_hp).eval()
    aco.perturb(enc.named_parameters(), aco.SEEDS[tag] + 100)
    aco.perturb(dec.named_parameters(), aco.SEEDS[tag] + 200)
    g = _golden()
    for who, m in (("enc", enc), ("dec", dec)):
        dg = aco.digests({k: v.detach().numpy() for k, v in m.state_dict().items()})
        assert list(dg.keys()) == list(g[f"{tag}:{who}_digest_names"])
        assert list(dg.values()) == list(g[f"{tag}:{who}_digests"]), f"{who}: the seeded draw differs from the reference's"
    for m in (enc, dec.quantizer, dec.model):
        m.precision = precision
    return enc, dec


def _sd(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _codes_ok(codes, want, gaps):
    sure = gaps > aco.TAU
    return bool((np.asarray(codes)[sure] == np.asarray(want)[sure]).all())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_on_the_reference_fixture(tag):
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC[tag]
    g = _golden()
    enc, dec = _build(tag)
    esd, dsd = _sd(enc), {"quantizer." + k: v for k, v in _sd(dec.quantizer).items()}
    dsd.update({"model." + k: v for k, v in _sd(dec.model).items()})
    z, stages = aco.encoder(esd, enc_hp["up_ratios"], g[f"{tag}:wav"], return_stages=True)
    for i, s in enumerate(stages):
        assert _rel(s, g[f"{tag}:stage{i}"]) < 1e-6
    assert _rel(z, g[f"{tag}:enc"]) < 1e-6
    qo, codes, layers, gaps = aco.quantize(dsd, g[f"{tag}:enc"], nq)
    assert _codes_ok(codes, g[f"{tag}:codes"], gaps.numpy())
    qo, _, layers, _ = aco.quantize(dsd, g[f"{tag}:enc"], nq, forced=g[f"{tag}:codes"])
    assert _rel(qo, g[f"{tag}:quantized_out"]) < 1e-6 and _rel(layers, g[f"{tag}:all_quantized"]) < 1e-6
    emb = aco.vq2emb(dsd, g[f"{tag}:codes"], nq)
    assert _rel(emb, g[f"{tag}:vq2emb"]) < 1e-6
    # the reference's fp32 waveform (fp32 iSTFT on the CPU) sits 2.8e-6 of the peak off its float64 restatement
    assert _rel(aco.decode(dsd, dec_hp, g[f"{tag}:vq2emb"]), g[f"{tag}:out"]) < 5e-6
    assert tuple(g[f"{tag}:enc"].shape[2:]) == (enc.frames(N),)


def test_maskgct_parameter_trees_match_the_reference():
    from amphion_b200.vocoders import CodecDecoder, CodecEncoder
    g = _golden()
    dec_cfg = dict(aco.MASKGCT_DECODER, in_channel=256, upsample_initial_channel=1536, up_ratios=[8, 5, 4, 3],
                   codebook_type="euclidean", kmeans_init=False, kmeans_iters=10, decay=0.8, eps=0.5,
                   threshold_ema_dead_code=2, weight_init=False, padding="same")
    dec_cfg.pop("in_channels")   # the config's own spelling, "in_channel", leaves the default 256
    for who, m in (("enc", CodecEncoder(cfg=types.SimpleNamespace(**aco.MASKGCT_ENCODER))),
                   ("dec", CodecDecoder(cfg=types.SimpleNamespace(**dec_cfg)))):
        names, ndim, flat = g[f"maskgct:{who}_names"], g[f"maskgct:{who}_ndim"], g[f"maskgct:{who}_shapes"]
        shapes, o = [], 0
        for n in ndim:
            shapes.append(tuple(int(v) for v in flat[o:o + n]))
            o += n
        sd = m.state_dict()
        assert list(sd.keys()) == list(names)
        assert [tuple(v.shape) for v in sd.values()] == shapes
        m.load_state_dict({k: torch.randn(s) for k, s in zip(names, shapes)}, strict=True)


def test_refusals_at_construction():
    from amphion_b200.vocoders import CodecDecoder, CodecEncoder
    base = dict(in_channels=24, num_quantizers=2, codebook_size=10, codebook_dim=8, quantizer_type="fvq",
                use_l2_normlize=True, use_vocos=True, vocos_dim=16, vocos_intermediate_dim=32, vocos_num_layers=1,
                n_fft=24, hop_size=6)
    for change, what in ((dict(use_vocos=False), "use_vocos=False"), (dict(quantizer_type="vq"), "'vq'"),
                         (dict(quantizer_type="lfq"), "'lfq'"), (dict(use_l2_normlize=False), "use_l2_normlize=False")):
        with pytest.raises(NotImplementedError, match=what):
            CodecDecoder(**dict(base, **change))
    with pytest.raises(ValueError, match="Unknown quantizer type"):
        CodecDecoder(**dict(base, quantizer_type="rvq"))
    with pytest.raises(NotImplementedError, match="use_tanh=True"):
        CodecEncoder(8, [2], 16, use_tanh=True)
    dec = CodecDecoder(**base)
    z = torch.zeros(1, 24, 3)
    with pytest.raises(NotImplementedError, match="training mode"):
        dec.quantizer.train()(z)
    with pytest.raises(NotImplementedError, match="training mode"):
        dec(z, vq=True, eval_vq=False)
    dec.eval()
    with pytest.raises(ValueError, match="n_quantizers 3 outside 1..2"):
        dec(z, vq=True, n_quantizers=3)
    with pytest.raises(ValueError, match="n_quantizers 3 outside 1..2"):
        dec.vq2emb(torch.zeros(3, 1, 3, dtype=torch.long), n_quantizers=3)
    with pytest.raises(NotImplementedError, match="latent2dist"):
        dec.latent2dist(z)


def test_c_abi_refuses_snake1d_outside_the_encoder_and_a_malformed_rvq():
    from amphion_b200 import _capi
    from amphion_b200.vocoders import CodecEncoder, FACodecDecoder
    h = C.c_void_p()
    c = FACodecDecoder(in_channels=256, vq_dim=256, upsample_initial_channel=32, up_ratios=[2])._c_config()
    c.activation = _capi.ACT_SNAKE1D
    assert _capi.lib.ab_generator_create(C.byref(c), C.byref(h)) != 0 and "SnakeBeta" in _capi.last_error()
    c = CodecEncoder(8, [2], 16)._c_config()
    c.snake_logscale = 1
    assert _capi.lib.ab_generator_create(C.byref(c), C.byref(h)) != 0
    c = _capi.GeneratorConfig()
    c.kind, c.n_mel, c.vq_num_q[0], c.vq_codebook_dim, c.vq_codebook_size = _capi.GEN_RVQ, 24, 2, 8, 100
    assert _capi.lib.ab_generator_create(C.byref(c), C.byref(h)) == 0
    _capi.lib.ab_generator_destroy(h)
    for field, v in (("num_upsamples", 1), ("vq_codebook_size", 0), ("vq_codebook_dim", 24), ("activation", 3)):
        bad = _capi.GeneratorConfig.from_buffer_copy(c)
        setattr(bad, field, v)
        assert _capi.lib.ab_generator_create(C.byref(bad), C.byref(h)) != 0, field


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC[tag]
    g = _golden()
    wav = torch.from_numpy(g[f"{tag}:wav"]).to(DEV)
    res = {}
    for prec in PRECS:
        enc, dec = _build(tag, prec)
        with torch.no_grad():
            z = enc.to(DEV)(wav)
            dec = dec.to(DEV)
            qo, codes, cl, cbl, layers = dec(torch.from_numpy(g[f"{tag}:enc"]).to(DEV), vq=True, eval_vq=True,
                                             n_quantizers=nq)
            emb = dec.vq2emb(codes, n_quantizers=nq)
            y = dec(emb)
        res[prec] = [t.cpu().numpy() for t in (z, qo, codes, layers, emb, y)]
        assert tuple(cl.shape) == (nq,) and not cl.any() and not cbl.any()
    esd = _sd(_build(tag)[0])
    dsd_dec = _build(tag)[1]
    dsd = {"quantizer." + k: v for k, v in _sd(dsd_dec.quantizer).items()}
    dsd.update({"model." + k: v for k, v in _sd(dsd_dec.model).items()})
    z32, qo, codes, layers, emb, y32 = res["fp32"]
    assert _rel(z32, g[f"{tag}:enc"]) < 2e-5
    assert _rel(res["tc_f16"][0], z32) < 1e-3
    assert _rel(res["tc_bf16"][0], aco.encoder(esd, enc_hp["up_ratios"], g[f"{tag}:wav"], operands="bf16")) < 4e-3
    _, _, _, gaps = aco.quantize(dsd, g[f"{tag}:enc"], nq)
    assert _codes_ok(codes, g[f"{tag}:codes"], gaps.numpy())
    f_qo, _, f_layers, _ = aco.quantize(dsd, g[f"{tag}:enc"], nq, forced=codes)
    assert _rel(qo, f_qo) < 2e-6 and _rel(layers, f_layers) < 2e-6
    assert _rel(emb, aco.vq2emb(dsd, codes, nq)) < 2e-6 and _rel(emb, qo) < 1e-5
    for prec in ("tc_f16", "tc_bf16"):   # the quantizer runs in fp32 at every precision
        for a, b in zip(res[prec][1:5], (qo, codes, layers, emb)):
            assert np.array_equal(a, b)
    if np.array_equal(codes, g[f"{tag}:codes"]):
        assert _rel(y32, g[f"{tag}:out"]) < 2e-5
        assert _rel(res["tc_f16"][5], g[f"{tag}:out"]) < 1e-3
    assert _rel(res["tc_bf16"][5], aco.decode(dsd, dec_hp, emb, operands="bf16")) < 4e-3


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 63, 64, 65, 333])
def test_quantizer_shapes_views_and_code_types(T):
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC["a"]
    _, dec = _build("a")
    dec = dec.to(DEV)
    dsd = {"quantizer." + k: v for k, v in _sd(dec.quantizer).items()}
    gen = torch.Generator().manual_seed(T)
    x = torch.randn(3, T, 64, generator=gen).to(DEV).transpose(1, 2)     # a transposed view
    for n in (1, 12):
        qo, codes, _, _, layers = dec(x, vq=True, eval_vq=True, n_quantizers=n)
        qc, cc, _, _, lc = dec(x.contiguous(), vq=True, n_quantizers=n)
        assert torch.equal(qo, qc) and torch.equal(codes, cc) and torch.equal(layers, lc)
        f_qo, _, f_layers, _ = aco.quantize(dsd, x.cpu().numpy(), n, forced=codes.cpu().numpy())
        assert _rel(qo.cpu(), f_qo) < 2e-6 and _rel(layers.cpu(), f_layers) < 2e-6
        wide = torch.zeros(2 * n + 1, 3, 2 * T, dtype=torch.int64, device=DEV)
        wide[::2][:n, :, ::2] = codes
        e1 = dec.vq2emb(codes, n_quantizers=n)
        assert torch.equal(dec.vq2emb(wide[::2, :, ::2], n_quantizers=n), e1)     # strided codes
        assert torch.equal(dec.vq2emb(codes.int(), n_quantizers=n), e1)           # int32 codes
        assert _rel(e1.cpu(), aco.vq2emb(dsd, codes.cpu().numpy(), n)) < 2e-6
    strided = torch.randn(3, 64, 2 * T, generator=gen).to(DEV)[:, :, ::2]
    assert torch.equal(dec.quantize(strided)[1], dec.quantize(strided.contiguous())[1])


@pytest.mark.gpu
def test_batch_independence_repeat_and_out():
    _, _, B, N, nq = aco.GOLDEN_CODEC["a"]
    for prec in PRECS:
        enc, dec = _build("a", prec)
        enc, dec = enc.to(DEV), dec.to(DEV)
        wav = torch.randn(3, 1, 4000, generator=torch.Generator().manual_seed(5)).to(DEV) * 0.3
        z = enc(wav)
        assert torch.equal(enc(wav), z)
        out = torch.empty_like(z)
        assert enc(wav, out=out) is out and torch.equal(out, z)
        qo, codes, _, _, layers = dec(z, vq=True, eval_vq=True)
        emb = dec.vq2emb(codes)
        y = dec(emb)
        for b in range(3):
            assert torch.equal(enc(wav[b:b + 1]), z[b:b + 1])
            q1, c1, _, _, l1 = dec(z[b:b + 1], vq=True)
            assert torch.equal(q1, qo[b:b + 1]) and torch.equal(c1, codes[:, b:b + 1]) and torch.equal(l1, layers[:, b:b + 1])
            assert torch.equal(dec.vq2emb(codes[:, b:b + 1]), emb[b:b + 1])
        assert torch.equal(dec(z, vq=True)[0], qo) and torch.equal(dec.decode(emb), y)


@pytest.mark.gpu
def test_out_of_range_codes():
    from amphion_b200 import _capi
    _, dec = _build("b")
    dec = dec.to(DEV)
    codes = torch.zeros(3, 1, 5, dtype=torch.int64, device=DEV)
    codes[0, 0, 2] = 100
    with pytest.raises(ValueError, match=r"outside the codebook \[0, 100\)"):
        dec.vq2emb(codes, n_quantizers=1)
    codes[0, 0, 2] = -1
    with pytest.raises(ValueError, match="outside the codebook"):
        dec.vq2emb(codes, n_quantizers=1)
    # a C-ABI caller that skips the check gets NaN in that time step and nowhere else
    q = dec.quantizer
    out = torch.empty(1, 24, 5, device=DEV)
    with q._launch(codes.device) as h:
        _capi.check(_capi.lib.ab_rvq_vq2emb(h, _capi.ptr(codes), _capi.shape_array(codes.stride()), 1, 1, 5,
                                            _capi.ptr(out), _capi.stream_ptr()), "ab_rvq_vq2emb")
    assert torch.isnan(out[:, :, 2]).all() and torch.isfinite(out[:, :, [0, 1, 3, 4]]).all()


@pytest.mark.gpu
def test_maskgct_geometry_round_trip():
    """MaskGCT's codec at full size, seeded, B = 2, one second: wav -> codes -> wav against the oracle."""
    from amphion_b200.vocoders import CodecDecoder, CodecEncoder
    torch.manual_seed(3)
    enc = CodecEncoder(**aco.MASKGCT_ENCODER).eval()
    dec = CodecDecoder(**aco.MASKGCT_DECODER).eval()
    aco.perturb(enc.named_parameters(), 4)
    aco.perturb(dec.named_parameters(), 5)
    for m in (enc, dec.quantizer, dec.model):
        m.precision = "fp32"
    esd = _sd(enc)
    dsd = {"quantizer." + k: v for k, v in _sd(dec.quantizer).items()}
    dsd.update({"model." + k: v for k, v in _sd(dec.model).items()})
    enc, dec = enc.to(DEV), dec.to(DEV)
    wav = torch.randn(2, 1, 24000, generator=torch.Generator().manual_seed(6)) * 0.3
    z = enc(wav.to(DEV))
    assert tuple(z.shape) == (2, 256, 50)
    assert _rel(z.cpu(), aco.encoder(esd, aco.MASKGCT_ENCODER["up_ratios"], wav.numpy())) < 2e-5
    qo, codes = dec.quantize(z, n_quantizers=12)
    f_qo, _, _, _ = aco.quantize(dsd, z.cpu().numpy(), 12, forced=codes.cpu().numpy())
    assert _rel(qo.cpu(), f_qo) < 2e-6
    y = dec(dec.vq2emb(codes, n_quantizers=12))
    assert tuple(y.shape) == (2, 1, 24000)
    assert _rel(y.cpu(), aco.decode(dsd, aco.MASKGCT_DECODER, dec.vq2emb(codes, n_quantizers=12).cpu().numpy())) < 2e-5
    for prec in ("tc_f16", "tc_bf16"):
        for m in (enc, dec.quantizer, dec.model):
            m.precision = prec
        z16 = enc(wav.to(DEV))
        assert _rel(z16.cpu(), z.cpu()) < (1e-3 if prec == "tc_f16" else 4e-2)
        assert torch.isfinite(dec(dec.vq2emb(dec.quantize(z16)[1]))).all()


@pytest.mark.gpu
def test_one_hot_projections_are_exact():
    """With one-hot projections every term is exact, so quantized_out, all_quantized and vq2emb are bit-equal to the
    numpy float32 restatement in the reference's order ((0 + q_0) + q_1) + ...; any other summation order shows."""
    _, dec = _build("a")
    rvq = dec.quantizer
    sd = dict(rvq.named_parameters())
    aco.one_hot_projections(sd, 17)
    dsd = {"quantizer." + k: v.detach().clone() for k, v in sd.items()}
    x = torch.randn(2, 64, 65, generator=torch.Generator().manual_seed(20)) * 2.0
    _, _, _, gaps = aco.quantize(dsd, x.numpy(), 12)
    assert (gaps > aco.TAU).all()
    want_q, want_codes, want_layers = aco.quantize_kernel_order(dsd, x.numpy(), 12)
    rvq.invalidate()
    qo, codes, _, _, layers = rvq.to(DEV)(x.to(DEV), n_quantizers=12)
    assert np.array_equal(codes.cpu().numpy(), want_codes)
    assert np.array_equal(qo.cpu().numpy(), want_q) and np.array_equal(layers.cpu().numpy(), want_layers)
