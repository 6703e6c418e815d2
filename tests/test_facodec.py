"""FACodec decoder (models/codec/ns3_codec/facodec.py:556-576) on the native pipeline: the float64 oracle and the host
module against the reference fixture (tests/golden/facodec*.npz, written by tests/golden/gen_facodec.py), strict loading
of the README geometry's state dict, the refusal paths, and on the GPU vq2emb and inference at every precision against
the fixture and the oracle.  Bars are fractions of the audio peak."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest
import torch

import facodec_oracle as fo
from conftest import GOLDEN

BARS = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}
OPERANDS = {"fp32": None, "tc_f16": None, "tc_bf16": "bf16"}   # the oracle each precision is held to


def load_fixture():
    d = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "facodec*.npz"))):
        z = np.load(p)
        d.update({k: z[k] for k in z.files})
    return d


def variant(d, tag):
    io = {k[len(tag) + 1:]: v for k, v in d.items() if k.startswith(tag + ":") and ":sd:" not in k}
    sd = {k[len(tag) + 4:]: v for k, v in d.items() if k.startswith(tag + ":sd:")}
    return io, sd


def build(hp, sd=None, seed=0):
    from amphion_b200.vocoders import FACodecDecoder
    torch.manual_seed(seed)
    m = FACodecDecoder(**hp)
    if sd is not None:
        full = m.state_dict()
        full.update({k: torch.as_tensor(v) for k, v in sd.items()})
        m.load_state_dict(full, strict=True)
    return m.eval()


def perturb(model, seed):
    """Decode-path parameters at the fixture generator's scales (tests/golden/gen_facodec.py)."""
    g = torch.Generator().manual_seed(seed)
    n = len(model.up_ratios)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if not (name.startswith(("model.", "timbre_linear.")) or ".out_proj." in name or "._codebook." in name):
                continue
            if name.endswith("weight_g"):
                scale = 0.1 if name.startswith(f"model.{n + 2}.") else \
                    0.25 if re.fullmatch(r"model\.\d+\.block\.[234]\.block\.3\.weight_g", name) else 1.0
                p.copy_((torch.rand(p.shape, generator=g) * 0.6 + 0.6) * scale)
            elif name.endswith("weight_v") or name.endswith("_codebook.weight"):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith((".alpha", ".beta")):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            elif name == "timbre_linear.weight":
                p.copy_(torch.randn(p.shape, generator=g) * (0.3 / p.shape[1] ** 0.5))
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
                if name == "timbre_linear.bias":
                    p[:p.shape[0] // 2] += 1.0
    model.invalidate()


def sd_numpy(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_fixture(tag):
    io, sd = variant(load_fixture(), tag)
    hp, _, _ = fo.GOLDEN_FACODEC[tag]
    if tag == "a":
        emb = fo.vq2emb(sd, io["codes"]).numpy()
        assert np.abs(emb - io["emb"]).max() <= 1e-6 * np.abs(io["emb"]).max()
        nores = fo.vq2emb(sd, io["codes"], use_residual=False).numpy()
        assert np.abs(nores - io["emb_nores"]).max() <= 1e-6 * np.abs(io["emb_nores"]).max()
        x = io["emb"]
    else:
        x = io["x"]
    film = fo.film(sd, x, io["spk"])
    assert np.abs(film.numpy() - io["film"]).max() <= 1e-6 * np.abs(io["film"]).max()
    wav, stages = fo.generator(sd, hp["up_ratios"], film, return_stages=True)
    for i, s in enumerate(stages):
        assert np.abs(s.numpy() - io[f"stage{i}"]).max() <= 1e-5 * np.abs(io[f"stage{i}"]).max(), i
    peak = np.abs(io["wav"]).max()
    assert wav.shape == io["wav"].shape
    assert np.abs(wav.numpy() - io["wav"]).max() <= 1e-6 * peak


def test_readme_state_dict_loads_strictly():
    d = load_fixture()
    m = build(fo.README_FACODEC)
    want = {k: tuple(int(s) for s in shp if s >= 0) for k, shp in zip(d["readme_keys"].tolist(), d["readme_shapes"])}
    have = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert have == want
    sd = {k: torch.zeros(s) for k, s in want.items()}
    m.load_state_dict(sd, strict=True)


def test_fixture_state_dicts_load_strictly():
    d = load_fixture()
    for tag in ("a", "b"):
        _, sd = variant(d, tag)
        m = build(fo.GOLDEN_FACODEC[tag][0], sd)
        for k, v in sd.items():
            assert np.array_equal(m.state_dict()[k].numpy(), v), k


def test_refusals_before_launch():
    from amphion_b200.vocoders import FACodecDecoder
    with pytest.raises(ValueError, match="vq_dim"):
        FACodecDecoder(in_channels=32, upsample_initial_channel=64, up_ratios=[2], vq_dim=64)
    m = build(fo.GOLDEN_FACODEC["b"][0])
    C = m.in_channels
    with pytest.raises(NotImplementedError, match="vq2emb"):
        m(torch.zeros(1, C, 4))
    with pytest.raises(NotImplementedError, match="inference"):
        m(torch.zeros(1, C, 4), vq=False, quantized=[torch.zeros(1, C, 4)] * 3, speaker_embedding=torch.zeros(1, C))
    with pytest.raises(ValueError, match="code rows"):
        m.vq2emb(torch.zeros(5, 1, 4, dtype=torch.long))
    with pytest.raises(ValueError, match="code rows"):
        m.vq2emb(torch.zeros(4, 1, 4, dtype=torch.long), use_residual_code=True)
    with pytest.raises(ValueError, match="integer"):
        m.vq2emb(torch.zeros(6, 1, 4))
    with pytest.raises(ValueError, match="speaker embedding"):
        m.inference(torch.zeros(2, C, 4), torch.zeros(1, C))
    with pytest.raises(ValueError, match="speaker embedding"):
        m.inference(torch.zeros(1, C, 4), torch.zeros(1, C + 1))
    with pytest.raises(ValueError, match="expects x"):
        m.inference(torch.zeros(1, C + 1, 4), torch.zeros(1, C))


def test_c_abi_config_checks():
    from amphion_b200 import _capi
    m = build(fo.GOLDEN_FACODEC["b"][0])
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
    assert create(lambda c: setattr(c, "snake_logscale", 0)) != 0
    assert create(lambda c: c.resblock_dilation_sizes[0].__setitem__(2, 5)) != 0
    assert create(lambda c: c.upsample_kernel_sizes.__setitem__(0, 5)) != 0
    assert create(lambda c: c.vq_num_q.__setitem__(0, 0)) != 0
    assert create(lambda c: setattr(c, "vq_codebook_dim", 17)) != 0
    # the vq_* fields belong to the FACodec kind
    c = m._c_config()
    c.kind = _capi.GEN_BIGVGAN
    h = C.c_void_p()
    assert lib.ab_generator_create(C.byref(c), C.byref(h)) != 0


# ------------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"


def _err(got, want):
    return float(np.abs(np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["a", "b"])
def test_fixture_parity(tag):
    io, sd = variant(load_fixture(), tag)
    hp, _, _ = fo.GOLDEN_FACODEC[tag]
    m = build(hp, sd).to(DEV)
    spk = torch.from_numpy(io["spk"]).to(DEV)
    peak = float(np.abs(io["wav"]).max())
    if tag == "a":
        emb = m.vq2emb(torch.from_numpy(io["codes"]).to(DEV))
        assert m.last_launches == 1
        assert _err(emb.cpu(), io["emb"]) <= 1e-6 * np.abs(io["emb"]).max()
        x = emb
    else:
        x = torch.from_numpy(io["x"]).to(DEV)
    for prec in ("fp32", "tc_f16", "tc_bf16"):
        m.precision = prec
        wav = m.inference(x, spk).cpu().numpy()
        assert m.last_launches == 5 + 14 * len(hp["up_ratios"])
        err_fix = _err(wav, io["wav"])
        want = fo.inference(sd, hp["up_ratios"], x.cpu(), io["spk"], operands=OPERANDS[prec]).numpy()
        err_or = _err(wav, want)
        print(f"facodec {tag} {prec}: |native - fixture| / peak = {err_fix / peak:.2e}, "
              f"|native - oracle| / peak = {err_or / peak:.2e}")
        if prec == "tc_bf16":
            assert err_or <= BARS[prec] * peak
        else:
            assert err_fix <= BARS[prec] * peak


@pytest.mark.gpu
@pytest.mark.parametrize("use_residual", [True, False])
def test_vq2emb_matches_oracle(use_residual):
    io, sd = variant(load_fixture(), "a")
    m = build(fo.GOLDEN_FACODEC["a"][0], sd).to(DEV)
    codes = torch.from_numpy(io["codes"])
    got = m.vq2emb(codes.to(DEV), use_residual_code=use_residual).cpu().numpy()
    want = fo.vq2emb(sd, io["codes"], use_residual=use_residual).numpy()
    assert _err(got, want) <= 1e-6 * np.abs(want).max()
    # the prosody + content rows alone, and codes with permuted strides
    if not use_residual:
        assert np.array_equal(m.vq2emb(codes[:3].to(DEV), use_residual_code=False).cpu().numpy(), got)
    strided = codes.permute(2, 0, 1).contiguous().permute(1, 2, 0).to(DEV)
    assert np.array_equal(m.vq2emb(strided, use_residual_code=use_residual).cpu().numpy(), got)


@pytest.mark.gpu
def test_vq2emb_reports_bad_codes():
    from amphion_b200 import _capi
    io, sd = variant(load_fixture(), "a")
    m = build(fo.GOLDEN_FACODEC["a"][0], sd).to(DEV)
    codes = torch.from_numpy(io["codes"]).to(DEV)
    good = m.vq2emb(codes)
    bad = codes.clone()
    bad[4, 1, 3] = 1024
    with pytest.raises(ValueError, match="outside the codebook"):
        m.vq2emb(bad)
    # a C-ABI caller that skips the check: the kernel reads nothing out of range and marks the time step
    out = torch.empty_like(good)
    _capi.check(_capi.lib.ab_facodec_vq2emb(m._handle, _capi.ptr(bad), _capi.shape_array(bad.stride()), 6, 2, 12, 1,
                                            _capi.ptr(out), _capi.stream_ptr()), "vq2emb")
    o = out.cpu()
    assert torch.isnan(o[1, :, 3]).all()
    o[1, :, 3] = good[1, :, 3].cpu()
    assert torch.equal(o, good.cpu())


@pytest.mark.gpu
def test_readme_geometry_matches_oracle():
    hp = fo.README_FACODEC
    m = build(hp)
    perturb(m, 5)
    sd = sd_numpy(m)
    m = m.to(DEV)
    g = torch.Generator().manual_seed(9)
    codes = torch.randint(0, 1024, (6, 2, 8), generator=g)
    spk = torch.randn(2, hp["in_channels"], generator=g)
    emb = m.vq2emb(codes.to(DEV))
    want_emb = fo.vq2emb(sd, codes)
    assert _err(emb.cpu(), want_emb) <= 1e-6 * float(want_emb.abs().max())
    for prec in ("fp32", "tc_f16", "tc_bf16"):
        m.precision = prec
        wav = m.inference(emb, spk.to(DEV)).cpu().numpy()
        assert wav.shape == (2, 1, 8 * 200)
        want = fo.inference(sd, hp["up_ratios"], emb.cpu(), spk, operands=OPERANDS[prec]).numpy()
        peak = float(np.abs(want).max())
        err = _err(wav, want)
        print(f"facodec readme {prec}: |native - oracle| / peak = {err / peak:.2e}")
        assert err <= BARS[prec] * peak


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "tc_f16"])
def test_bit_equal_runs(prec):
    io, sd = variant(load_fixture(), "a")
    m = build(fo.GOLDEN_FACODEC["a"][0], sd).to(DEV)
    m.precision = prec
    x = torch.from_numpy(io["emb"]).to(DEV)
    spk = torch.from_numpy(io["spk"]).to(DEV)
    ref = m.inference(x, spk)
    assert torch.equal(m.inference(x, spk), ref)                                      # repeat run
    for b in range(2):                                                                # batch independence
        assert torch.equal(m.inference(x[b:b + 1], spk[b:b + 1]), ref[b:b + 1])
    xt = x.transpose(1, 2).contiguous().transpose(1, 2)                               # transposed latent
    assert torch.equal(m.inference(xt, spk), ref)
    one = m.inference(x[:, :, :1], spk)                                               # T = 1
    assert one.shape == (2, 1, m.hop_length)
    assert torch.equal(m.inference(x[:, :, :1], spk), one)
    hp = fo.GOLDEN_FACODEC["a"][0]
    want = fo.inference(sd, hp["up_ratios"], io["emb"][:, :, :1], io["spk"]).numpy()
    assert _err(one.cpu(), want) <= BARS[prec] * float(np.abs(want).max())


@pytest.mark.gpu
def test_out_and_tail_events():
    io, sd = variant(load_fixture(), "a")
    m = build(fo.GOLDEN_FACODEC["a"][0], sd).to(DEV)
    x = torch.from_numpy(io["emb"]).to(DEV)
    spk = torch.from_numpy(io["spk"]).to(DEV)
    ref = m.inference(x, spk)
    out = torch.full_like(ref, float("nan"))
    assert m.inference(x, spk, out=out) is out
    assert torch.equal(out, ref)
    events = [torch.cuda.Event() for _ in range(2)]
    wav = m.inference(x, spk, tail_events=events)
    assert m.last_launches == 5 + 14 * 3 + 1                                          # conv_post in two chunks
    for ev in events:
        ev.synchronize()
    assert torch.equal(wav, ref)
    with pytest.raises(ValueError):
        m.inference(x, spk, out=torch.empty(2, 1, 7, device=DEV))


@pytest.mark.gpu
def test_profile_and_generator_forward_refused():
    io, sd = variant(load_fixture(), "b")
    m = build(fo.GOLDEN_FACODEC["b"][0], sd).to(DEV)
    x = torch.from_numpy(io["x"]).to(DEV)
    spk = torch.from_numpy(io["spk"]).to(DEV)
    m.inference(x, spk)
    m.set_profiling(True)
    m.inference(x, spk)
    prof = m.get_profile()
    m.set_profiling(False)
    assert prof["facodec_prologue"]["launches"] == 2
    assert sum(v["launches"] for v in prof.values()) == m.last_launches
    m.set_option("resblock_fusion", 0)   # accepted; every FACodec conv runs as a single conv
    assert torch.equal(m.inference(x, spk), m.inference(x, spk))
    with pytest.raises(RuntimeError, match="ab_facodec_inference"):
        m._forward_native(x)
