"""RepCodec, the semantic codec of MaskGCT, Metis and Vevo (amphion_b200.vocoders.RepCodec), against the reference's own
outputs (tests/golden/repcodec*.npz, tests/golden/gen_repcodec.py) and the float64 oracle (tests/repcodec_oracle.py),
and its two new kernel paths bit for bit:

* the pointwise GEMM's Linear epilogue (`hitem_kernel` PW_LINEAR, through ab_vocos_pointwise_forward): one-hot weights
  hitting every K chunk give exact accumulators, dense weights equal `hconv_kernel`'s k = 1 conv, written time-major;
  the fp32 route (`conv1d_fp32_kernel` at k = 1) against its FMA chain.  Outputs are pre-filled with NaN and followed by
  NaN guards, so an unwritten element or a store out of bounds shows;
* the RVQ's one-group layout (`facodec_rvq_kernel<RVQ_LAYERS>`) at RepCodec's 1024 channels, against the kernel-order
  restatement (amphion_codec_oracle.quantize_kernel_order), ragged codebooks and tied codes included.

Bars (DESIGN §3): encoder output and x_rec fp32 2e-5 of the peak, tc_f16 1e-3 against fp32, tc_bf16 4e-3 against the
bf16-operand oracle; codes equal wherever the float64 gap between the best and the runner-up distance exceeds TAU
(at 16 bits against the oracle RVQ fed the native encoder output); quantized 2e-6 of the peak against the oracle
teacher-forced with the native codes, and bit-equal across precisions given the same encoder output."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import amphion_codec_oracle as aco
import repcodec_oracle as rco
import resblock_oracle as ro
from conftest import load_golden
from diffwave_exact_oracle import fma_chain

DEV = "cuda:0"
PRECS = ["fp32", "tc_f16", "tc_bf16"]
OPERANDS = {"fp32": None, "tc_f16": "f16", "tc_bf16": "bf16"}
LINEAR = 3          # AB_VOCOS_PW_LINEAR
GUARD = 4096        # NaN elements after every output


def _capi():
    from amphion_b200 import _capi
    return _capi


def _golden():
    return load_golden("repcodec")[0]


def _build(tag, precision="fp32"):
    """The native codec of fixture `tag`: seeded construction, the fixture's perturbation, its digests checked."""
    from amphion_b200.vocoders import RepCodec
    hp, B, T = rco.GOLDEN_REPCODEC[tag]
    torch.manual_seed(rco.SEEDS[tag])
    m = RepCodec(**hp).eval()
    rco.perturb(m.named_parameters(), rco.SEEDS[tag] + 100)
    g = _golden()
    dg = rco.digests({k: v.detach().numpy() for k, v in m.state_dict().items()})
    assert list(dg.keys()) == list(g[f"{tag}:digest_names"])
    assert list(dg.values()) == list(g[f"{tag}:digests"]), "the seeded draw differs from the reference's"
    m.precision = precision
    return m


def _sd(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _codes_ok(codes, want, gaps):
    sure = np.asarray(gaps) > rco.TAU
    return bool((np.asarray(codes).reshape(sure.shape)[sure] == np.asarray(want).reshape(sure.shape)[sure]).all())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_on_the_reference_fixture(tag):
    hp, B, T = rco.GOLDEN_REPCODEC[tag]
    g = _golden()
    sd = _sd(_build(tag))
    n = hp["num_quantizers"]
    enc = rco.encoder(sd, g[f"{tag}:x"])
    assert _rel(enc, g[f"{tag}:enc"]) < 1e-6
    codes = g[f"{tag}:codes"].reshape(n, B, T)
    _, _, _, gaps = rco.rvq(sd, g[f"{tag}:enc"], n)
    assert _codes_ok(codes, rco.rvq(sd, g[f"{tag}:enc"], n)[1].numpy(), gaps.numpy())
    qo, _, _, _ = rco.rvq(sd, g[f"{tag}:enc"], n, forced=codes)
    assert _rel(qo.numpy().transpose(0, 2, 1), g[f"{tag}:quantized"]) < 1e-6
    assert _rel(rco.decoder(sd, g[f"{tag}:quantized"].transpose(0, 2, 1)), g[f"{tag}:x_rec"]) < 1e-6


def test_maskgct_key_list_loads_strictly_and_the_cfg_quirk():
    from amphion_b200.vocoders import RepCodec
    g = _golden()
    m = RepCodec(cfg=types.SimpleNamespace(**rco.MASKGCT_SEMANTIC))
    names, ndim, flat = g["maskgct:names"], g["maskgct:ndim"], g["maskgct:shapes"]
    shapes, o = [], 0
    for nd in ndim:
        shapes.append(tuple(int(v) for v in flat[o:o + nd]))
        o += nd
    sd = m.state_dict()
    assert len(names) == 239 and list(sd.keys()) == list(names)
    assert [tuple(v.shape) for v in sd.values()] == shapes
    m.load_state_dict({k: torch.randn(s) for k, s in zip(names, shapes)}, strict=True)
    # repcodec_model.py:67-76: vocos_intermediate_dim and vocos_num_layers come from cfg only when it has vocos_dim
    small = dict(codebook_size=10, hidden_size=24, codebook_dim=4)
    m = RepCodec(vocos_dim=16, vocos_intermediate_dim=32, vocos_num_layers=1,
                 cfg=types.SimpleNamespace(**small, vocos_intermediate_dim=40, vocos_num_layers=2))
    assert (m.vocos_dim, m.vocos_intermediate_dim, m.vocos_num_layers) == (16, 32, 1)
    m = RepCodec(cfg=types.SimpleNamespace(**small, vocos_dim=8, vocos_intermediate_dim=40, vocos_num_layers=2))
    assert (m.vocos_dim, m.vocos_intermediate_dim, m.vocos_num_layers) == (8, 40, 2)
    assert m.encoder[1].weight.shape == (24, 8) and len(m.encoder[0].convnext) == 2
    assert not hasattr(m, "down")
    with pytest.raises(AttributeError, match="vocos_intermediate_dim"):   # as the reference's cfg rule raises
        RepCodec(cfg=types.SimpleNamespace(**small, vocos_dim=8))
    m = RepCodec(cfg=types.SimpleNamespace(**small, vocos_dim=8, vocos_intermediate_dim=40, vocos_num_layers=1,
                                           downsample_scale=2, num_quantizers=3))
    assert "down.weight" in m.state_dict() and "up.bias" in m.state_dict() and len(m.quantizer.quantizers) == 3


def test_refusals():
    from amphion_b200.vocoders import RepCodec
    m = RepCodec(codebook_size=10, hidden_size=24, codebook_dim=4, vocos_dim=16, vocos_intermediate_dim=32,
                 vocos_num_layers=1)
    x = torch.zeros(1, 5, 24)
    with pytest.raises(NotImplementedError, match="training mode"):
        m.train().quantize(x)
    with pytest.raises(NotImplementedError, match="training mode"):
        m(x)
    m.eval()
    m.quantizer.train()
    with pytest.raises(NotImplementedError, match="training mode"):
        m.quantize(x)
    m.eval()
    with pytest.raises(ValueError, match=r"\[B, T, 24\]"):
        m.quantize(torch.zeros(1, 24, 5))
    with pytest.raises(ValueError, match=r"\[B, T, 24\]"):
        m(torch.zeros(5, 24))
    with pytest.raises(ValueError, match="empty"):
        m.quantize(torch.zeros(0, 5, 24))
    with pytest.raises(ValueError, match="floating-point"):
        m.quantize(torch.zeros(1, 5, 24, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"\[B, 24, T\]"):
        m.encoder(torch.zeros(1, 5, 24))
    with pytest.raises(RuntimeError, match="needs a CUDA tensor"):
        m.quantize(x)
    with pytest.raises(RuntimeError, match="needs a CUDA tensor"):
        m.decoder(x.transpose(1, 2))


def test_c_abi_config_of_the_linear_kind_and_a_too_wide_rvq():
    from amphion_b200.vocoders import RepCodec
    capi = _capi()
    lib, h = capi.lib, C.c_void_p()
    m = RepCodec(codebook_size=10, hidden_size=24, codebook_dim=4, vocos_dim=16, vocos_intermediate_dim=32,
                 vocos_num_layers=2)
    c = m.encoder._c_config()
    assert c.kind == capi.GEN_VOCOS_LINEAR
    assert lib.ab_generator_create(C.byref(c), C.byref(h)) == 0, capi.last_error()
    names = [lib.ab_generator_tensor_name(h, i).decode() for i in range(lib.ab_generator_num_tensors(h))]
    lib.ab_generator_destroy(h)
    assert sorted(names) == sorted(m.encoder.state_dict().keys()) and len(names) == len(set(names))
    assert names[-2:] == ["1.weight", "1.bias"] and names[0] == "0.embed.weight"
    for field, v in (("istft_n_fft", 24), ("istft_hop", 6), ("trunk_out_channels", 0), ("num_layers", 0),
                     ("activation", 3), ("vq_codebook_size", 10), ("upsample_initial_channel", 0)):
        bad = capi.GeneratorConfig.from_buffer_copy(c)
        setattr(bad, field, v)
        assert lib.ab_generator_create(C.byref(bad), C.byref(h)) != 0, field
    # the Linear epilogue of the pointwise entry point writes y alone (the pointers are never dereferenced)
    a, f16 = C.c_void_p(256), capi.PRECISIONS["tc_f16"]
    need = lib.ab_vocos_pointwise_workspace_bytes(LINEAR, 2, 48, 66, 10, f16)
    assert need > 0
    for gamma, y, yimg, spec in ((a, a, None, None), (None, a, a, None), (None, a, None, a), (None, None, None, None)):
        assert lib.ab_vocos_pointwise_forward(LINEAR, None, a, a, a, gamma, y, yimg, spec, 2, 48, 66, 10, f16, a, need,
                                              None) == -1 and "epilogue 3" in capi.last_error()
    assert lib.ab_vocos_pointwise_forward(4, None, a, a, a, None, a, None, None, 2, 48, 66, 10, f16, a, need, None) == -1
    c = capi.GeneratorConfig()
    c.kind, c.vq_num_q[0], c.vq_codebook_dim, c.vq_codebook_size = capi.GEN_RVQ, 1, 8, 8192
    for width, rc in ((1024, 0), (1447, 0), (1448, -2), (4096, -2)):
        c.n_mel = width
        assert lib.ab_generator_create(C.byref(c), C.byref(h)) == rc, width
        if rc == 0:
            lib.ab_generator_destroy(h)
        else:
            assert "at most 1447" in capi.last_error()


# ------------------------------------------------------------------------------------------------ GPU: PW_LINEAR
def _dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _linear(prec, w, bias, B, cin, cout, T, *, x=None, ximg=None):
    """One ab_vocos_pointwise_forward with AB_VOCOS_PW_LINEAR into a NaN buffer with a NaN guard -> y [B, T, C_out]."""
    capi = _capi()
    xd = None if x is None else _dev(x)
    xi = None if ximg is None else _dev(np.ascontiguousarray(ximg).view(np.int16), torch.int16)
    wd, bd = _dev(w), _dev(bias)
    buf = torch.full((B * T * cout + GUARD,), float("nan"), device=DEV)
    need = capi.lib.ab_vocos_pointwise_workspace_bytes(LINEAR, B, cin, cout, T, capi.PRECISIONS[prec])
    assert need > 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    rc = capi.lib.ab_vocos_pointwise_forward(LINEAR, capi.ptr(xd), capi.ptr(xi), capi.ptr(wd), capi.ptr(bd), None,
                                             capi.ptr(buf), None, None, B, cin, cout, T, capi.PRECISIONS[prec],
                                             C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, capi.last_error()
    out = buf.cpu().numpy()
    assert np.isnan(out[B * T * cout:]).all(), "a store past the end of y"
    return out[:B * T * cout].reshape(B, T, cout)


def _assert_bits(what, got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


# (id, C_in, C_out, B, T): RepCodec's Linear (two N blocks of 256 + 512 ... C_out 1024 in 4 blocks), a partial N block,
# odd widths (scalar stores), 128-row tiles cut at 127 / 128 / 129
LIN = [
    ("rep-T1", 384, 1024, 2, 1),
    ("rep-T127", 384, 1024, 1, 127),
    ("rep-T333", 384, 1024, 2, 333),
    ("c1000-T128", 384, 1000, 2, 128),
    ("odd333-T129", 40, 333, 3, 129),
    ("odd47-T333", 48, 47, 1, 333),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("case", LIN, ids=[c[0] for c in LIN])
def test_linear_epilogue_one_hot_is_exact(case, prec):
    import vocos_exact_oracle as vx
    name, cin, cout, B, T = case
    op = OPERANDS[prec]
    rng = np.random.default_rng(cin * 7 + cout + T)
    x = rng.normal(0, 2, (B, cin, T)).astype(np.float32)
    oh = vx.one_hot_linear(rng, cin, cout, (-2, -1, 0, 1))
    w = oh.dense()[:, :, 0]
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    acc = ro.conv(ro.rnd(x, op), oh.rounded(op), 1)                  # the one product of each output
    want = (acc + bias[None, :, None]).astype(np.float32).transpose(0, 2, 1)
    y = _linear(prec, w, bias, B, cin, cout, T, ximg=ro.to_image(ro.image_bits(x, 1.0, op)))
    _assert_bits(f"{name} LINEAR", y, want)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("case", [LIN[1], LIN[3], LIN[4]], ids=["rep-T127", "c1000-T128", "odd333-T129"])
def test_linear_epilogue_dense_equals_hconv(case, prec):
    """The Linear epilogue's y[b, t, co] is hconv_kernel's k = 1 conv y[b, co, t] from the same image, bit for bit."""
    from test_vocos_exact import _hconv_k1
    name, cin, cout, B, T = case
    rng = np.random.default_rng(cin + cout + T)
    x = rng.normal(0, 1, (B, cin, T)).astype(np.float32)
    w = rng.normal(0, 1 / np.sqrt(cin), (cout, cin)).astype(np.float32)
    bias = rng.normal(0, 0.1, cout).astype(np.float32)
    ximg = ro.to_image(ro.image_bits(x, 1.0, OPERANDS[prec]))
    v = _hconv_k1(prec, ximg, w, bias, B, cin, cout, T)
    assert np.isfinite(v).all()
    _assert_bits(f"{name} LINEAR", _linear(prec, w, bias, B, cin, cout, T, ximg=ximg), v.transpose(0, 2, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,B,T", [(384, 1024, 2, 129), (40, 333, 1, 17), (48, 47, 2, 5), (384, 1000, 1, 1)])
def test_linear_fp32_route_is_its_fma_chain(cin, cout, B, T):
    rng = np.random.default_rng(cin * cout + T)
    x = rng.normal(0, 2, (B, cin, T)).astype(np.float32)
    w = rng.normal(0, 2 / np.sqrt(cin), (cout, cin)).astype(np.float32)
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    want = (fma_chain(w, x) + bias[None, :, None]).astype(np.float32).transpose(0, 2, 1)
    _assert_bits("fp32 LINEAR", _linear("fp32", w, bias, B, cin, cout, T, x=x), want)


# ------------------------------------------------------------------------------------------------ GPU: the wide RVQ
def _wide_rvq(rows, seed):
    """A native ResidualVQ at RepCodec's width (1024 -> 8) with one-hot projections, and its state dict under the
    oracle's names."""
    from amphion_b200.vocoders.amphion_codec import ResidualVQ
    torch.manual_seed(seed)
    rvq = ResidualVQ(input_dim=1024, num_quantizers=1, codebook_size=rows, codebook_dim=8, quantizer_type="fvq",
                     quantizer_dropout=0.0, commitment=0.15, use_l2_normlize=True).eval()
    sd = dict(rvq.named_parameters())
    aco.one_hot_projections(sd, seed + 1)
    with torch.no_grad():
        v = sd["quantizers.0.in_project.weight_v"]   # z_e[0] reads the last channel: the x load's last chunk counts
        v[0].zero_()
        v[0, 1023, 0] = 1.0
        for k, v in sd.items():
            if k.endswith("bias"):
                v.copy_(torch.randn(v.shape) * 0.1)
    return rvq, {"quantizer." + k: v.detach().clone() for k, v in sd.items()}


def _views(x, B, T, kind):
    """x [B, 1024, T] as a contiguous tensor, the encoder's transposed view of [B, T, 1024], or a strided view."""
    if kind == "contiguous":
        return x.contiguous()
    if kind == "transposed":
        return x.transpose(1, 2).contiguous().transpose(1, 2)
    wide = torch.full((B, 1024, 2 * T), float("nan"), device=x.device)
    wide[:, :, ::2] = x
    return wide[:, :, ::2]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [8192, 8191, 8193])
def test_wide_rvq_is_the_kernel_order_with_ties_and_views(rows):
    """C = 1024 on the one-group layout: codes (ties go to the lowest code), quantized_out and all_quantized bit-equal
    to the kernel-order restatement, for every view of x; with a null all_quantized nothing else changes."""
    rvq, dsd = _wide_rvq(rows, rows)
    rvq = rvq.to(DEV)
    for T in (1, 15, 16, 17, 333):
        B = 2
        x = torch.randn(B, 1024, T, generator=torch.Generator().manual_seed(T + rows + 100000)) * 2.0
        # tie: rows c0 + 1 and rows - 1 (in the ragged last chunk when rows % 256 != 0) repeat row c0, a code frames pick
        c0 = int(aco.quantize(dsd, x.numpy(), 1)[1][0, 0, 0])
        cb = dsd["quantizer.quantizers.0.codebook.weight"]
        dups = sorted({min(c0 + 1, rows - 1), rows - 1} - {c0})
        for r in dups:
            cb[r] = cb[c0]
        with torch.no_grad():
            rvq.quantizers[0].codebook.weight.copy_(cb)
        _, _, _, gaps = aco.quantize(dsd, x.numpy(), 1)
        gaps = gaps.numpy()
        assert ((gaps > aco.TAU) | (gaps == 0)).all(), f"T {T}: a near tie in the test data"
        want_q, want_codes, want_layers = aco.quantize_kernel_order(dsd, x.numpy(), 1)
        # the copies of row c0 give equal distances in the kernel (BLAS may part them in the last bit): the lowest wins
        want_codes[np.isin(want_codes, dups)] = c0
        assert (want_codes == c0).any()
        for kind in ("contiguous", "transposed", "strided"):
            xv = _views(x.to(DEV), B, T, kind)
            qo, codes, _, _, layers = rvq(xv)
            assert np.array_equal(codes.cpu().numpy(), want_codes), f"T {T} {kind}: codes"
            _assert_bits(f"T {T} {kind} quantized_out", qo.cpu().numpy(), want_q)
            _assert_bits(f"T {T} {kind} all_quantized", layers.cpu().numpy(), want_layers)
        # a null all_quantized: quantized_out and codes unchanged, nothing written past them
        capi = _capi()
        out = torch.full((B * 1024 * T + GUARD,), float("nan"), device=DEV)
        cds = torch.full((B * T + GUARD,), -7, dtype=torch.int64, device=DEV)
        xv = _views(x.to(DEV), B, T, "transposed")
        with rvq._launch(xv.device) as h:
            capi.check(capi.lib.ab_rvq_quantize(h, capi.ptr(xv), capi.shape_array(xv.stride()), B, T, 1, capi.ptr(out),
                                                capi.ptr(cds), None, capi.stream_ptr()), "ab_rvq_quantize")
        _assert_bits(f"T {T} null layers", out[:B * 1024 * T].cpu().numpy().reshape(B, 1024, T), want_q)
        assert np.array_equal(cds[:B * T].cpu().numpy().reshape(1, B, T), want_codes)
        assert torch.isnan(out[B * 1024 * T:]).all() and (cds[B * T:] == -7).all()


@pytest.mark.gpu
def test_too_wide_rvq_is_refused_before_any_launch():
    from amphion_b200.vocoders.amphion_codec import ResidualVQ
    rvq = ResidualVQ(input_dim=1448, num_quantizers=1, codebook_size=16, codebook_dim=8, quantizer_type="fvq").eval()
    x = torch.zeros(1, 1448, 3, device=DEV)
    with pytest.raises(RuntimeError, match="at most 1447"):
        rvq.to(DEV)(x)
    assert rvq._handle is None


# ------------------------------------------------------------------------------------------------ GPU: the codec
def _run(m, x):
    with torch.no_grad():
        enc = m.encoder(x.transpose(1, 2))
        codes, quantized = m.quantize(x)
        x_rec, loss, all_indices = m(x)
    return enc, codes, quantized, x_rec, loss, all_indices


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    hp, B, T = rco.GOLDEN_REPCODEC[tag]
    n = hp["num_quantizers"]
    g = _golden()
    x = torch.from_numpy(g[f"{tag}:x"]).to(DEV)
    sd = _sd(_build(tag))
    res = {}
    for prec in PRECS:
        m = _build(tag, prec).to(DEV)
        enc, codes, quantized, x_rec, loss, all_indices = _run(m, x)
        assert loss.dim() == 0 and float(loss) == 0.0 and loss.device == x.device
        assert tuple(codes.shape) == ((B, T) if n == 1 else (n, B, T)) and codes.dtype == torch.int64
        assert tuple(all_indices.shape) == (n, B, T) and torch.equal(all_indices.reshape(codes.shape), codes)
        assert tuple(quantized.shape) == (B, T, hp["hidden_size"]) and quantized.stride() == (hp["hidden_size"] * T, 1, T)
        assert x_rec.is_contiguous() and tuple(x_rec.shape) == (B, T, hp["hidden_size"])
        res[prec] = [t.cpu().numpy() for t in (enc, codes, quantized, x_rec)]
        # codes and quantized against the oracle RVQ fed this precision's encoder output
        e = res[prec][0]
        _, _, _, gaps = rco.rvq(sd, e, n)
        want = rco.rvq(sd, e, n)[1].numpy()
        assert _codes_ok(res[prec][1], want, gaps.numpy()), prec
        f_qo = rco.rvq(sd, e, n, forced=res[prec][1].reshape(n, B, T))[0].numpy().transpose(0, 2, 1)
        assert _rel(res[prec][2], f_qo) < 2e-6, prec
        # given this precision's encoder output, the RVQ is fp32 at every precision: equal to an fp32 quantizer's
        q32 = _build(tag, "fp32").to(DEV).quantizer
        qo32, c32, _, _, _ = q32(torch.from_numpy(e).to(DEV).transpose(1, 2))
        assert np.array_equal(res[prec][2], qo32.transpose(1, 2).cpu().numpy())
        assert np.array_equal(res[prec][1].reshape(n, B, T), c32.cpu().numpy())
    e32, c32, q32, r32 = res["fp32"]
    print(f"{tag}: enc fp32 {_rel(e32, g[f'{tag}:enc']):.2e}, f16 {_rel(res['tc_f16'][0], e32):.2e}, bf16 "
          f"{_rel(res['tc_bf16'][0], rco.encoder(sd, g[f'{tag}:x'], 'bf16')):.2e}; x_rec fp32 "
          f"{_rel(r32, g[f'{tag}:x_rec']):.2e}; codes equal {np.array_equal(c32, g[f'{tag}:codes'])}")
    assert _rel(e32, g[f"{tag}:enc"]) < 2e-5
    _, _, _, gaps = rco.rvq(sd, g[f"{tag}:enc"], n)
    assert _codes_ok(c32, g[f"{tag}:codes"], gaps.numpy())
    if np.array_equal(c32, g[f"{tag}:codes"]):
        assert _rel(r32, g[f"{tag}:x_rec"]) < 2e-5
    assert _rel(r32, rco.decoder(sd, q32.transpose(0, 2, 1))) < 2e-5
    assert _rel(res["tc_f16"][0], e32) < 1e-3
    assert _rel(res["tc_bf16"][0], rco.encoder(sd, g[f"{tag}:x"], "bf16")) < 4e-3
    for prec in ("tc_f16", "tc_bf16"):
        r = res[prec][3]
        q = res[prec][2].transpose(0, 2, 1)
        want = rco.decoder(sd, q, OPERANDS[prec] if prec == "tc_bf16" else None)
        print(f"{tag} {prec}: x_rec {_rel(r, want):.2e}, quantized vs forced oracle "
              f"{_rel(res[prec][2], rco.rvq(sd, res[prec][0], n, forced=res[prec][1].reshape(n, B, T))[0].numpy().transpose(0, 2, 1)):.2e}")
        assert _rel(r, want) < (4e-3 if prec == "tc_bf16" else 1e-3), prec


@pytest.mark.gpu
def test_released_geometry_one_second():
    """MaskGCT's semantic codec at full size, seeded, B = 2, 50 frames, against the oracle at every precision."""
    from amphion_b200.vocoders import RepCodec
    torch.manual_seed(7)
    m = RepCodec(cfg=types.SimpleNamespace(**rco.MASKGCT_SEMANTIC)).eval()
    rco.perturb(m.named_parameters(), 8)
    sd = _sd(m)
    m = m.to(DEV)
    x = torch.randn(2, 50, 1024, generator=torch.Generator().manual_seed(9))
    want_enc = rco.encoder(sd, x.numpy())
    for prec in PRECS:
        m.precision = prec
        enc, codes, quantized, x_rec, _, _ = _run(m, x.to(DEV))
        assert tuple(codes.shape) == (2, 50) and m.last_launches == 41 + 40
        e = enc.cpu().numpy()
        bar, ref = {"fp32": (2e-5, want_enc), "tc_f16": (1e-3, want_enc),
                    "tc_bf16": (4e-3, rco.encoder(sd, x.numpy(), "bf16"))}[prec]
        assert _rel(e, ref) < bar, prec
        _, _, _, gaps = rco.rvq(sd, e, 1)
        assert _codes_ok(codes.cpu().numpy(), rco.rvq(sd, e, 1)[1].numpy(), gaps.numpy()), prec
        f_qo = rco.rvq(sd, e, 1, forced=codes.cpu().numpy()[None])[0].numpy()
        assert _rel(quantized.cpu().numpy(), f_qo.transpose(0, 2, 1)) < 2e-6
        want_rec = rco.decoder(sd, quantized.cpu().numpy().transpose(0, 2, 1), "bf16" if prec == "tc_bf16" else None)
        print(f"released {prec}: enc {_rel(e, ref):.2e}, x_rec {_rel(x_rec.cpu().numpy(), want_rec):.2e}, quantized "
              f"{_rel(quantized.cpu().numpy(), f_qo.transpose(0, 2, 1)):.2e}")
        assert _rel(x_rec.cpu().numpy(), want_rec) < bar, prec


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS)
def test_views_batch_independence_repeats_and_launches(prec):
    m = _build("a", prec).to(DEV)
    x = torch.randn(3, 40, 1024, generator=torch.Generator().manual_seed(11)).to(DEV)
    codes, q = m.quantize(x)
    assert m.last_launches == 41
    # the embed conv at C_in 1024 from the [B, T, 1024] transposed view equals the conv on a contiguous copy
    enc = m.encoder(x.transpose(1, 2))
    assert m.encoder.last_launches == 40
    assert torch.equal(m.encoder(x.transpose(1, 2).contiguous()), enc)
    assert torch.equal(m.encoder(x.half().transpose(1, 2)), m.encoder(x.half().float().transpose(1, 2)))
    c2, q2 = m.quantize(x)
    assert torch.equal(c2, codes) and torch.equal(q2, q)
    x_rec = m(x)[0]
    assert m.last_launches == 41 + 40      # forward: the encoder and the RVQ, then the decoder's 40
    for b in range(3):
        cb, qb = m.quantize(x[b:b + 1])
        assert torch.equal(cb, codes[b:b + 1]) and torch.equal(qb, q[b:b + 1])
        assert torch.equal(m(x[b:b + 1])[0], x_rec[b:b + 1])


@pytest.mark.gpu
def test_parent_load_state_dict_reaches_the_native_handles():
    from amphion_b200.vocoders import RepCodec
    hp, B, T = rco.GOLDEN_REPCODEC["b"]
    m = _build("b").to(DEV)
    x = torch.randn(2, 9, hp["hidden_size"], generator=torch.Generator().manual_seed(12)).to(DEV)
    before = m(x)[0]
    torch.manual_seed(99)
    other = RepCodec(**hp).eval()
    rco.perturb(other.named_parameters(), 98)
    m.load_state_dict(other.state_dict(), strict=True)
    after = m(x)[0]
    assert not torch.equal(before, after)
    sd = _sd(other)
    _, codes = m._encode(x, "forward")
    qo = rco.rvq(sd, m.encoder(x.transpose(1, 2)).cpu().numpy(), 2, forced=codes.cpu().numpy())[0].numpy()
    assert _rel(after.cpu().numpy(), rco.decoder(sd, qo)) < 2e-5
