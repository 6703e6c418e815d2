"""MelGAN (models/vocoders/gan/generator/melgan.py) on the native pipeline: the CPU oracle and the host module against
the reference fixture (tests/golden/melgan.npz, written by tests/golden/gen_melgan.py), the C ABI's config checks,
and on the GPU every precision against the oracle."""
import ctypes as C
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from melgan_oracle import GOLDEN_MELGAN, HP_MELGAN_RECIPE, melgan_forward


def load_melgan(tag):
    z = np.load(os.path.join(GOLDEN, "melgan.npz"))
    d = {k[len(tag) + 1:]: z[k] for k in z.files if k.startswith(tag + ":")}
    sd = {k[3:]: v for k, v in d.items() if k.startswith("sd:")}
    return {k: v for k, v in d.items() if not k.startswith("sd:")}, sd


def melgan_cfg(hp, n_mel):
    hop = int(np.prod(hp["ratios"]))
    pre = NS(n_mel=n_mel, hop_size=hop, sample_rate=24000, extract_amplitude_phase=False)
    return NS(preprocess=pre, model=NS(generator="melgan", melgan=NS(**hp)))


def build_melgan(hp, n_mel, state_dict=None, seed=None):
    from amphion_b200.vocoders import _vocoders
    if seed is not None:
        torch.manual_seed(seed)
    m = _vocoders["melgan"](melgan_cfg(hp, n_mel))
    if state_dict is not None:
        m.load_state_dict({k: torch.as_tensor(v) for k, v in state_dict.items()}, strict=True)
    return m.eval()


def sd_numpy(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


# ------------------------------------------------------------------------------------------------ CPU


@pytest.mark.parametrize("tag", sorted(GOLDEN_MELGAN))
def test_oracle_matches_reference_fixture(tag):
    hp, _, _, _ = GOLDEN_MELGAN[tag]
    g, sd = load_melgan(tag)
    wav, stages = melgan_forward(sd, hp, g["mel"], stages=True)
    assert wav.shape == g["wav"].shape
    assert float(np.abs(wav - g["wav"]).max()) <= 1e-6
    for i, s in enumerate(stages):
        if f"stage{i}" in g:
            assert float(np.abs(s - g[f"stage{i}"]).max()) <= 1e-6


@pytest.mark.parametrize("tag", sorted(GOLDEN_MELGAN))
def test_seeded_module_reproduces_reference_state_dict(tag):
    hp, n_mel, _, _ = GOLDEN_MELGAN[tag]
    g, sd = load_melgan(tag)
    model = build_melgan(hp, n_mel, seed=int(g["seed"]))
    msd = sd_numpy(model)
    assert list(msd) == list(sd)
    for k in sd:
        assert msd[k].shape == sd[k].shape, k
        assert np.array_equal(msd[k], sd[k]), k
    assert model.hop_length == int(np.prod(hp["ratios"]))


def test_registry_entries():
    from amphion_b200.vocoders import MelGAN, _vocoder_forward_funcs, _vocoder_infer_funcs, _vocoders
    from amphion_b200.vocoders.gan_vocoder_inference import synthesis_audios, vocoder_inference
    assert _vocoders["melgan"] is MelGAN
    assert _vocoder_forward_funcs["melgan"] is vocoder_inference
    assert _vocoder_infer_funcs["melgan"] is synthesis_audios


def test_inner_modules_do_not_run_on_their_own():
    hp, n_mel, _, _ = GOLDEN_MELGAN["a"]
    model = build_melgan(hp, n_mel)
    with pytest.raises(RuntimeError, match="pipeline"):
        model.model(torch.zeros(1, n_mel, 8))
    with pytest.raises(RuntimeError, match="pipeline"):
        model.model[4](torch.zeros(1, 32, 8))


@pytest.mark.parametrize("tag", sorted(GOLDEN_MELGAN))
def test_tensor_table_without_gpu(tag):
    from amphion_b200 import _capi
    hp, n_mel, _, _ = GOLDEN_MELGAN[tag]
    model = build_melgan(hp, n_mel)
    h = model._ensure_handle()
    names = [_capi.lib.ab_generator_tensor_name(h, i).decode() for i in range(_capi.lib.ab_generator_num_tensors(h))]
    sd = model.state_dict()
    for n in names:
        assert n in sd or (n + "_v" in sd and n + "_g" in sd), n
    # every weight and bias of the module is consumed
    wanted = {n + s for n in names for s in ("", "_v", "_g")}
    assert set(sd) <= wanted, set(sd) - wanted
    assert "model.1.weight" in names and "model.4.block.2.weight" in names and "model.4.shortcut.bias" in names
    assert _capi.lib.ab_generator_workspace_bytes(h, 2, 21) > 0
    rc = _capi.lib.ab_generator_forward(h, C.c_void_p(8), 1, 4, _capi.shape_array((1, 1, 1)), C.c_void_p(8),
                                        C.c_void_p(256), 1 << 30, None)
    assert rc == -4 and "finalize" in _capi.last_error()


def _create(cfg):
    from amphion_b200 import _capi
    h = C.c_void_p()
    rc = _capi.lib.ab_generator_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        _capi.lib.ab_generator_destroy(h)
    return rc, _capi.last_error()


@pytest.mark.parametrize("what", ["kernel", "dilation", "upsample_kernel", "num_kernels", "channels"])
def test_create_refuses_malformed_configs(what):
    hp, n_mel, _, _ = GOLDEN_MELGAN["b"]
    cfg = build_melgan(hp, n_mel)._c_config()
    assert _create(cfg)[0] == 0
    if what == "kernel":
        cfg.resblock_kernel_sizes[0] = 5
    elif what == "dilation":
        cfg.resblock_dilation_sizes[0][1] = 2
    elif what == "upsample_kernel":
        cfg.upsample_kernel_sizes[1] = 9
    elif what == "num_kernels":
        cfg.num_kernels = 2
        cfg.resblock_kernel_sizes[1] = 3
        cfg.num_dilations[1] = 1
        cfg.resblock_dilation_sizes[1][0] = 1
    else:
        cfg.upsample_initial_channel += 1
    rc, msg = _create(cfg)
    assert rc == -1 and "MelGAN" in msg, (rc, msg)


# ------------------------------------------------------------------------------------------------ GPU

TOL = {"fp32": 2e-5, "tc_f16": 1e-3, "tc_bf16": 4e-3}


def _run(model, mel, prec, **kw):
    model.precision = prec
    with torch.no_grad():
        return model(mel, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", sorted(TOL))
@pytest.mark.parametrize("tag", sorted(GOLDEN_MELGAN))
def test_fixture_parity(tag, prec):
    hp, n_mel, _, _ = GOLDEN_MELGAN[tag]
    g, sd = load_melgan(tag)
    model = build_melgan(hp, n_mel, sd).cuda()
    want = melgan_forward(sd, hp, g["mel"])
    got = _run(model, torch.from_numpy(g["mel"]).cuda(), prec).cpu().numpy()
    assert got.shape == g["wav"].shape
    err, ref_err = float(np.abs(got - want).max()), float(np.abs(got - g["wav"]).max())
    assert err <= TOL[prec] and ref_err <= TOL[prec], (err, ref_err)


def _recipe(ngf, seed):
    hp = dict(HP_MELGAN_RECIPE, ngf=ngf)
    model = build_melgan(hp, 100, seed=seed).cuda()
    return hp, model, sd_numpy(model)


def _logmel(B, T, seed, n_mel=100):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, n_mel, T, generator=g) * 13.5 - 11.5


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_odd_ratio_conv_transpose_on_tensor_cores(prec):
    hp, n_mel, _, _ = GOLDEN_MELGAN["b"]   # ratios [3, 5]: padding r//2 + 1, output_padding 1
    g, sd = load_melgan("b")
    model = build_melgan(hp, n_mel, sd).cuda()
    model.precision = prec
    model.set_profiling(True)
    got = _run(model, torch.from_numpy(g["mel"]).cuda(), prec).cpu().numpy()
    prof = model.get_profile()
    model.set_profiling(False)
    assert prof["conv_transpose1d_fp32"]["launches"] == 0
    assert prof["tc_gemmconv"]["launches"] >= 2   # conv_pre and both ConvTranspose layers
    assert float(np.abs(got - melgan_forward(sd, hp, g["mel"])).max()) <= TOL[prec]
    # longer input, several time tiles per stage, against the oracle
    mel = _logmel(2, 300, 5, n_mel)
    got = _run(model, mel.cuda(), prec).cpu().numpy()
    assert float(np.abs(got - melgan_forward(sd, hp, mel.numpy())).max()) <= TOL[prec]


@pytest.mark.gpu
def test_recipe_geometry_against_oracle():
    hp, model, sd = _recipe(32, 7)
    mel = _logmel(2, 64, 8)
    want = melgan_forward(sd, hp, mel.numpy())
    for prec, tol in (("tc_f16", 1e-3), ("fp32", 5e-5)):
        got = _run(model, mel.cuda(), prec).cpu().numpy()
        assert got.shape == (2, 1, 64 * 256)
        err = float(np.abs(got - want).max())
        assert err <= tol, (prec, err)


@pytest.mark.gpu
def test_wide_blocks_against_oracle():
    hp, model, sd = _recipe(64, 9)   # stage 0 has 512 channels
    mel = _logmel(1, 16, 10)
    want = melgan_forward(sd, hp, mel.numpy())
    for prec, tol in (("tc_f16", 1e-3), ("fp32", 5e-5)):
        err = float(np.abs(_run(model, mel.cuda(), prec).cpu().numpy() - want).max())
        assert err <= tol, (prec, err)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "fp32"])
def test_batch_independence_bit_equal(prec):
    hp, model, _ = _recipe(32, 11)
    mel = _logmel(9, 12, 12).cuda()
    full = _run(model, mel, prec)
    for b in range(9):
        assert torch.equal(full[b:b + 1], _run(model, mel[b:b + 1].contiguous(), prec)), b


@pytest.mark.gpu
@pytest.mark.parametrize("tag", sorted(GOLDEN_MELGAN))
def test_transposed_view_tail_events_and_out(tag):
    hp, n_mel, _, _ = GOLDEN_MELGAN[tag]
    g, sd = load_melgan(tag)
    model = build_melgan(hp, n_mel, sd).cuda()
    mel = torch.from_numpy(g["mel"]).cuda()
    for prec in ("tc_f16", "fp32"):
        base = _run(model, mel, prec)
        view = mel.transpose(1, 2).contiguous().transpose(1, 2)
        assert not view.is_contiguous()
        assert torch.equal(_run(model, view, prec), base)
        events = [torch.cuda.Event() for _ in range(3)]
        assert torch.equal(_run(model, mel, prec, tail_events=events), base)
        out = torch.full_like(base, float("nan"))
        assert _run(model, mel, prec, out=out) is out
        assert torch.equal(out, base)


@pytest.mark.gpu
def test_reflection_length_limits():
    hp, n_mel, _, _ = GOLDEN_MELGAN["a"]
    g, sd = load_melgan("a")
    model = build_melgan(hp, n_mel, sd).cuda()
    mel = torch.from_numpy(g["mel"][:, :, :4]).cuda()
    for prec in ("tc_f16", "fp32"):
        got = _run(model, mel, prec).cpu().numpy()
        assert float(np.abs(got - melgan_forward(sd, hp, mel.cpu().numpy())).max()) <= TOL[prec]
        with pytest.raises(RuntimeError, match="ReflectionPad1d"):
            _run(model, mel[:, :, :3], prec)


@pytest.mark.gpu
def test_synthesis_through_registry(tmp_path):
    from scipy.io import wavfile

    from amphion_b200.vocoders import _vocoder_infer_funcs, _vocoders, synthesize_to_files
    hp, n_mel, _, _ = GOLDEN_MELGAN["a"]
    _, sd = load_melgan("a")
    cfg = melgan_cfg(hp, n_mel)
    model = _vocoders["melgan"](cfg)
    model.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()}, strict=True)
    model = model.cuda().eval()
    model.precision = "fp32"
    gen = torch.Generator().manual_seed(3)
    mels = [torch.randn(n_mel, t, generator=gen) for t in (9, 14, 5, 11)]
    Tmax, hop = max(m.shape[-1] for m in mels), int(np.prod(hp["ratios"]))
    want = []
    for m in mels:   # the reference: every utterance alone on the zero-padded mel, trimmed
        padded = torch.zeros(1, n_mel, Tmax)
        padded[0, :, :m.shape[-1]] = m
        want.append(melgan_forward(sd, hp, padded.numpy())[0, 0, :m.shape[-1] * hop])
    plain = _vocoder_infer_funcs["melgan"](cfg, model, mels, batch_size=None)
    for a, w in zip(plain, want):
        assert a.shape == w.shape
        assert float(np.abs(a.numpy() - w).max()) <= 2e-5
    # one batch: bucketing only reorders the utterances, the padding stays -> bit-equal
    for a, b in zip(_vocoder_infer_funcs["melgan"](cfg, model, mels, batch_size=None, bucket=True), plain):
        assert torch.equal(a, b)
    # batches of 2 by length, (5, 9) and (11, 14): each utterance is padded to its bucket's longest mel (the reflection
    # at the padded end reaches back about ten frames, so the samples differ from the plain run's), and equals the
    # oracle's B = 1 run on that padding
    order = sorted(range(len(mels)), key=lambda i: mels[i].shape[-1])
    bucketed = _vocoder_infer_funcs["melgan"](cfg, model, mels, batch_size=2, bucket=True)
    for q in range(0, len(order), 2):
        group = order[q:q + 2]
        Tb = max(mels[i].shape[-1] for i in group)
        for i in group:
            m = mels[i]
            padded = torch.zeros(1, n_mel, Tb)
            padded[0, :, :m.shape[-1]] = m
            wb = melgan_forward(sd, hp, padded.numpy())[0, 0, :m.shape[-1] * hop]
            assert bucketed[i].shape == wb.shape
            assert float(np.abs(bucketed[i].numpy() - wb).max()) <= 2e-5
    paths = [str(tmp_path / f"{i}.wav") for i in range(len(mels))]
    synthesize_to_files(cfg, model, mels, paths, fs=24000)
    for p, w in zip(paths, want):
        fs, pcm = wavfile.read(p)
        assert fs == 24000 and pcm.shape == w.shape
        q = np.clip(np.floor(w * 32768 + 0.5), -32768, 32767)
        assert np.abs(pcm.astype(np.int64) - q).max() <= 1
