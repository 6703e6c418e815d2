"""Vocos (models/codec/amphion_codec/vocos.py) on the native pipeline: the CPU oracle and the host module against the
reference fixture (tests/golden/vocos.npz, written by tests/golden/gen_vocos.py), the C ABI's config checks, and on
the GPU every precision against the fixture and the oracle."""
import ctypes as C
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from vocos_oracle import GOLDEN_VOCOS, HP_VOCOS_RECIPE, vocos_forward


def load_vocos(tag):
    z = np.load(os.path.join(GOLDEN, "vocos.npz"))
    d = {k[len(tag) + 1:]: z[k] for k in z.files if k.startswith(tag + ":")}
    sd = {k[3:]: v for k, v in d.items() if k.startswith("sd:")}
    init = {k[5:]: v for k, v in d.items() if k.startswith("init:")}
    return {k: v for k, v in d.items() if not k.startswith(("sd:", "init:"))}, sd, init


def build_vocos(hp, state_dict=None, seed=None):
    from amphion_b200.vocoders import Vocos
    if seed is not None:
        torch.manual_seed(seed)
    m = Vocos(**hp)
    if state_dict is not None:
        m.load_state_dict({k: torch.as_tensor(v) for k, v in state_dict.items()}, strict=True)
    return m.eval()


def sd_numpy(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


# ------------------------------------------------------------------------------------------------ CPU


@pytest.mark.parametrize("tag", sorted(GOLDEN_VOCOS))
def test_oracle_matches_reference_fixture(tag):
    hp, _, _ = GOLDEN_VOCOS[tag]
    g, sd, _ = load_vocos(tag)
    wav, blocks, feat = vocos_forward(sd, hp, g["mel"], stages=True)
    assert wav.shape == g["wav"].shape
    assert float(np.abs(wav - g["wav"]).max()) <= 1e-5
    # stages: within 1e-6 of each stage's peak (the reference runs in fp32, the oracle in fp64)
    for i, b in enumerate(blocks):
        if f"block{i}" in g:
            assert float(np.abs(b - g[f"block{i}"]).max()) <= 1e-6 * float(np.abs(g[f"block{i}"]).max())
    if "backbone" in g:
        assert float(np.abs(feat - g["backbone"]).max()) <= 1e-6 * float(np.abs(g["backbone"]).max())


def test_seeded_module_reproduces_reference_initial_state_dict():
    hp, _, _ = GOLDEN_VOCOS["a"]
    g, _, init = load_vocos("a")
    msd = sd_numpy(build_vocos(hp, seed=int(g["seed"])))
    assert list(msd) == list(init)
    for k in init:
        assert msd[k].shape == init[k].shape, k
        assert np.array_equal(msd[k], init[k]), k


@pytest.mark.parametrize("tag", sorted(GOLDEN_VOCOS))
def test_strict_load_and_attributes(tag):
    hp, _, _ = GOLDEN_VOCOS[tag]
    _, sd, _ = load_vocos(tag)
    model = build_vocos(hp, sd)
    assert model.hop_length == hp["hop_size"]
    for k, v in sd_numpy(model).items():
        assert np.array_equal(v, sd[k]), k


def test_cfg_overrides_keyword_defaults():
    from amphion_b200.vocoders import Vocos
    cfg = NS(input_channels=12, dim=40, intermediate_dim=120, num_layers=2, n_fft=48, hop_size=12)
    m = Vocos(input_channels=99, dim=64, cfg=cfg)
    assert (m.input_channels, m.dim, m.intermediate_dim, m.num_layers, m.n_fft, m.hop_length) == (12, 40, 120, 2, 48, 12)
    assert tuple(m.head.out.weight.shape) == (50, 40)
    assert Vocos().hop_length == 200   # the reference's keyword defaults


def test_not_in_registry_but_exported():
    import amphion_b200.vocoders as v
    assert "Vocos" in v.__all__
    assert all(cls is not v.Vocos for cls in v._vocoders.values())


@pytest.mark.parametrize("tag", sorted(GOLDEN_VOCOS))
def test_tensor_table_without_gpu(tag):
    from amphion_b200 import _capi
    hp, _, _ = GOLDEN_VOCOS[tag]
    model = build_vocos(hp)
    h = model._ensure_handle()
    names = [_capi.lib.ab_generator_tensor_name(h, i).decode() for i in range(_capi.lib.ab_generator_num_tensors(h))]
    sd = model.state_dict()
    assert sorted(names) == sorted(sd)   # every tensor of the state dict, the window included, and nothing else
    assert "head.istft.window" in names and "backbone.convnext.1.gamma" in names
    rc = _capi.lib.ab_generator_forward(h, C.c_void_p(8), 1, 4, _capi.shape_array((1, 1, 1)), C.c_void_p(8),
                                        C.c_void_p(256), 1 << 30, None)
    assert rc == -4 and "finalize" in _capi.last_error()
    assert _capi.lib.ab_generator_output_samples(h, 5, 0) == 5 * hp["hop_size"]
    for key in ("resblock_fusion", "nsf_source_frames"):
        assert _capi.lib.ab_generator_set_option(h, key.encode(), 0) == -1


def _create(cfg):
    from amphion_b200 import _capi
    h = C.c_void_p()
    rc = _capi.lib.ab_generator_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        _capi.lib.ab_generator_destroy(h)
    return rc, _capi.last_error()


@pytest.mark.parametrize("what,code", [("odd_n_fft", -2), ("hop_above_n_fft", -2), ("odd_overlap", -2), ("layers", -1),
                                       ("dim", -1), ("ffn", -1), ("foreign_field", -1), ("vocos_field_elsewhere", -1)])
def test_create_refuses_malformed_configs(what, code):
    from amphion_b200 import _capi
    hp, _, _ = GOLDEN_VOCOS["b"]
    cfg = build_vocos(hp)._c_config()
    assert _create(cfg)[0] == 0
    if what == "odd_n_fft":
        cfg.istft_n_fft = 47
    elif what == "hop_above_n_fft":
        cfg.istft_hop = 50
    elif what == "odd_overlap":
        cfg.istft_hop = 11
    elif what == "layers":
        cfg.num_layers = 0
    elif what == "dim":
        cfg.upsample_initial_channel = -4
    elif what == "ffn":
        cfg.ffn_channels = 0
    elif what == "foreign_field":
        cfg.num_upsamples = 1
    else:
        cfg.kind = _capi.GEN_MELGAN
    rc, msg = _create(cfg)
    assert rc == code and ("Vocos" in msg or "VOCOS" in msg), (rc, msg)


def test_constructor_refusals():
    from amphion_b200.vocoders import Vocos
    with pytest.raises(ValueError, match="adanorm"):
        Vocos(input_channels=8, dim=16, intermediate_dim=32, num_layers=1, n_fft=16, hop_size=4, adanorm_num_embeddings=4)
    with pytest.raises(NotImplementedError, match="same"):
        Vocos(input_channels=8, dim=16, intermediate_dim=32, num_layers=1, n_fft=16, hop_size=4, padding="center")


def test_inner_modules_and_cpu_tensors_raise():
    hp, _, _ = GOLDEN_VOCOS["a"]
    model = build_vocos(hp)
    x = torch.zeros(1, hp["input_channels"], 8)
    for mod, arg in ((model.backbone, x), (model.backbone.convnext[0], torch.zeros(1, hp["dim"], 8)),
                     (model.head, torch.zeros(1, 8, hp["dim"])), (model.head.istft, torch.zeros(1, 33, 8))):
        with pytest.raises(RuntimeError, match="pipeline"):
            mod(arg)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        model(x)


def test_hop_of_falls_back_to_hop_length():
    from amphion_b200.dist import _hop_of
    hp, _, _ = GOLDEN_VOCOS["b"]
    assert _hop_of(build_vocos(hp)) == hp["hop_size"]
    assert _hop_of(NS(cfg=NS(preprocess=NS(hop_size=256)), hop_length=7)) == 256
    assert _hop_of(NS(cfg=None)) is None


# ------------------------------------------------------------------------------------------------ GPU

TOL = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}   # fractions of the audio's peak
# bf16 operands alone move fixture a's audio by 5.1e-3 of its peak (the operand-rounded oracle against the fp32 one), more
# than TOL: at tc_bf16 the bar holds against the operand-rounded oracle, and the fixture gets the bar on top of that floor


def _run(model, mel, prec, **kw):
    model.precision = prec
    with torch.no_grad():
        return model(mel, **kw)


def _trained_like(model, seed):
    """Trained-like parameter scales (as the fixture generator sets them)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("gamma"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.8 + 0.2)
            elif "norm" in name and name.endswith("weight"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + 1.0)
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif "dwconv" in name:
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            elif name.startswith("head.out"):
                p.copy_(torch.randn(p.shape, generator=g) * (0.5 / p.shape[1] ** 0.5))
            else:
                p.copy_(torch.randn(p.shape, generator=g) / p[0].numel() ** 0.5)
    return model


def _logmel(B, n, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, n, L, generator=g) * 13.5 - 11.5


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(TOL))
@pytest.mark.parametrize("tag", sorted(GOLDEN_VOCOS))
def test_fixture_parity(tag, prec):
    hp, _, _ = GOLDEN_VOCOS[tag]
    g, sd, _ = load_vocos(tag)
    model = build_vocos(hp, sd).cuda()
    want = vocos_forward(sd, hp, g["mel"])
    got = _run(model, torch.from_numpy(g["mel"]).cuda(), prec).cpu().numpy()
    assert got.shape == g["wav"].shape
    peak = float(np.abs(g["wav"]).max())
    floor = 0.0
    if prec == "tc_bf16":
        rounded = vocos_forward(sd, hp, g["mel"], operands="bf16")
        floor = float(np.abs(rounded - g["wav"]).max())
        assert float(np.abs(got - rounded).max()) <= TOL[prec] * peak
    err, ref_err = float(np.abs(got - want).max()), float(np.abs(got - g["wav"]).max())
    print(f"{tag} {prec}: {ref_err / peak:.2e} of the peak from the fixture (operand floor {floor / peak:.2e})")
    assert err <= TOL[prec] * peak + floor and ref_err <= TOL[prec] * peak + floor, (err, ref_err, peak, floor)


@pytest.mark.gpu
def test_f16_against_operand_rounded_oracle():
    # dim 256, intermediate 1024: 4 N blocks on pwconv1 and 32 K chunks on pwconv2; L = 200 is not a multiple of the
    # 128-row time tile.  Measured on an H100: 2.4e-4 of the peak.  The bar cannot go below the rounding-boundary noise
    # of the 16-bit operands: values that reach the fp16 rounding from fp32 instead of fp64 arithmetic land on the other
    # side of a boundary now and then, and a 1e-7 relative perturbation before the rounding moves this oracle's own
    # output by 3.1e-4 of the peak.
    hp = dict(input_channels=24, dim=256, intermediate_dim=1024, num_layers=2, n_fft=64, hop_size=16)
    model = _trained_like(build_vocos(hp, seed=21), 22).cuda()
    sd = sd_numpy(model)
    mel = _logmel(3, 24, 200, 23)
    want = vocos_forward(sd, hp, mel.numpy(), operands="f16")
    got = _run(model, mel.cuda(), "tc_f16").cpu().numpy()
    peak = float(np.abs(want).max())
    err = float(np.abs(got - want).max())
    print(f"tc_f16 vs operand-rounded oracle: {err / peak:.2e} of the peak")
    assert err <= 5e-4 * peak, (err, peak)


@pytest.mark.gpu
def test_recipe_geometry_against_oracle():
    model = _trained_like(build_vocos(HP_VOCOS_RECIPE, seed=31), 32).cuda()
    sd = sd_numpy(model)
    mel = _logmel(2, 128, 64, 33)
    want = vocos_forward(sd, HP_VOCOS_RECIPE, mel.numpy())
    peak = float(np.abs(want).max())
    for prec, tol in (("tc_f16", 2e-3), ("fp32", 1e-4)):
        got = _run(model, mel.cuda(), prec).cpu().numpy()
        assert got.shape == (2, 1, 64 * 480)
        err = float(np.abs(got - want).max())
        print(f"recipe {prec}: {err / peak:.2e} of the peak")
        assert err <= tol * peak, (prec, err, peak)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "fp32"])
def test_batch_independence_bit_equal(prec):
    hp, _, _ = GOLDEN_VOCOS["a"]
    _, sd, _ = load_vocos("a")
    model = build_vocos(hp, sd).cuda()
    mel = _logmel(5, hp["input_channels"], 150, 41).cuda()
    full = _run(model, mel, prec)
    for b in range(5):
        assert torch.equal(full[b:b + 1], _run(model, mel[b:b + 1].contiguous(), prec)), b


@pytest.mark.gpu
@pytest.mark.parametrize("tag", sorted(GOLDEN_VOCOS))
def test_transposed_view_tail_events_and_out(tag):
    hp, _, _ = GOLDEN_VOCOS[tag]
    g, sd, _ = load_vocos(tag)
    model = build_vocos(hp, sd).cuda()
    mel = torch.from_numpy(g["mel"]).cuda()
    for prec in ("tc_f16", "tc_bf16", "fp32"):
        base = _run(model, mel, prec)
        # Vevo calls vocoder_model(mel.transpose(1, 2)) on a [B, L, n_mels] tensor
        view = mel.transpose(1, 2).contiguous().transpose(1, 2)
        assert not view.is_contiguous()
        assert torch.equal(_run(model, view, prec), base)
        events = [torch.cuda.Event() for _ in range(3)]
        assert torch.equal(_run(model, mel, prec, tail_events=events), base)
        out = torch.full_like(base, float("nan"))
        assert _run(model, mel, prec, out=out) is out
        assert torch.equal(out, base)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(TOL))
def test_single_frame(prec):
    hp, _, _ = GOLDEN_VOCOS["b"]
    g, sd, _ = load_vocos("b")
    model = build_vocos(hp, sd).cuda()
    mel = g["mel"][:, :, :1]
    want = vocos_forward(sd, hp, mel)
    got = _run(model, torch.from_numpy(mel).cuda(), prec).cpu().numpy()
    assert got.shape == (1, 1, hp["hop_size"])
    assert float(np.abs(got - want).max()) <= TOL[prec] * max(float(np.abs(want).max()), 1e-3)


@pytest.mark.gpu
def test_profile_classes():
    hp, _, _ = GOLDEN_VOCOS["a"]
    _, sd, _ = load_vocos("a")
    model = build_vocos(hp, sd).cuda()
    mel = _logmel(2, hp["input_channels"], 40, 51).cuda()
    _run(model, mel, "tc_f16")
    model.set_profiling(True)
    _run(model, mel, "tc_f16")
    prof = model.get_profile()
    model.set_profiling(False)
    L = hp["num_layers"]
    assert prof["tc_pointwise"]["launches"] == 2 * L + 1
    assert prof["vocos_norm"]["launches"] == L + 2
    assert prof["conv1d_fp32"]["launches"] == 0
    assert prof["tc_pointwise"]["flops"] == pytest.approx(2 * 2 * 40 * hp["dim"] * (2 * L * hp["intermediate_dim"] + hp["n_fft"] + 2))
