"""DiffWave (models/vocoders/diffusion/diffwave/diffwave.py) and its sampler on the native pipeline: the float64 oracle and
the host module against the reference fixture (tests/golden/diffwave*.npz, written by tests/golden/gen_diffwave.py), the
C ABI's config checks and refusals, and on the GPU the forward and the sampler against the oracle and the fixture."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from conftest import load_golden
from diffwave_oracle import (GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, HP_DIFFWAVE_RECIPE, diffwave_cfg, diffwave_forward,
                             sample, schedule)

FP32_TOL = 1e-4   # forward eps, fraction of the peak
SAMPLER_TOL = 1e-4   # 6-step sampler, absolute
# forward eps at each precision: (operand rounding of the oracle it is compared with, bar as a fraction of the peak)
PREC_TOL = {"fp32": (None, FP32_TOL), "tc_f16": (None, 2e-3), "tc_bf16": ("bf16", 4e-3)}
PRECISIONS = sorted(PREC_TOL)


def load_dw():
    g, sd = load_golden("diffwave")
    init = {k[5:]: str(v) for k, v in g.items() if k.startswith("init:")}
    return {k: v for k, v in g.items() if not k.startswith("init:")}, sd, init


def build(hp, n_mel, state_dict=None, seed=None, hop=None, precision="fp32"):
    from amphion_b200.vocoders import _vocoders
    if seed is not None:
        torch.manual_seed(seed)
    m = _vocoders["diffwave"](diffwave_cfg(hp, n_mel, hop))
    if state_dict is not None:
        m.load_state_dict({k: torch.as_tensor(v) for k, v in state_dict.items()}, strict=True)
    m.precision = precision
    return m.eval()


def trained_like(model, seed):
    """Trained-like scales as tests/golden/gen_diffwave.py draws them (non-zero output projection)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif name.startswith("spectrogram_upsampler"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            else:
                p.copy_(torch.randn(p.shape, generator=g) / p[0].numel() ** 0.5)
    return model


def sd_numpy(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


def digest(a):
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + np.ascontiguousarray(a).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------ CPU


def test_oracle_matches_reference_fixture():
    g, sd, _ = load_dw()
    hp = GOLDEN_DIFFWAVE
    eps, outs = diffwave_forward(sd, hp, g["table"], g["audio"], [2.37], g["mel"], layers_out=True)
    assert float(np.abs(eps - g["eps_float"]).max()) <= 1e-6 * float(np.abs(g["eps_float"]).max())
    for i, (x, s) in enumerate(outs):
        assert float(np.abs(x[:1] - g[f"x{i}"]).max()) <= 1e-6 * float(np.abs(g[f"x{i}"]).max()), i
        assert float(np.abs(s[:1] - g[f"skip{i}"]).max()) <= 1e-6 * float(np.abs(g[f"skip{i}"]).max()), i
    eps = diffwave_forward(sd, hp, g["table"], g["audio"], g["steps_int"], g["mel"])
    assert float(np.abs(eps - g["eps_int"]).max()) <= 1e-6 * float(np.abs(g["eps_int"]).max())
    noises = {n: g[f"sampler_noise{n}"] for n in range(1, len(hp["inference_noise_schedule"]))}
    audio = sample(sd, hp, g["table"], g["sampler_mel"], g["sampler_noise0"], noises)
    assert float(np.abs(audio - g["sampler_audio"]).max()) <= 1e-6


def test_seeded_module_reproduces_reference_initial_state_dict_and_table():
    g, _, init = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, seed=int(g["seed"]))
    msd = sd_numpy(m)
    assert list(msd) == list(init)
    for k, v in msd.items():
        assert digest(v) == init[k], k
    assert np.array_equal(m.diffusion_embedding.embedding.numpy(), g["table"])
    assert "diffusion_embedding.embedding" not in msd   # non-persistent, as in the reference
    assert not np.any(msd["output_projection.weight"])


def test_strict_load():
    _, sd, _ = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd)
    for k, v in sd_numpy(m).items():
        assert np.array_equal(v, sd[k]), k


def test_constructor_writes_noise_schedule_into_cfg():
    from amphion_b200.vocoders import DiffWave
    cfg = diffwave_cfg(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL)
    assert not hasattr(cfg.model.diffwave, "noise_schedule")
    DiffWave(cfg)
    assert cfg.model.diffwave.noise_schedule == np.linspace(1e-4, 0.05, 50).tolist()


@pytest.mark.parametrize("fast", [True, False])
def test_step_schedule(fast):
    from amphion_b200.vocoders import DiffWave
    from amphion_b200.vocoders.diffusion_vocoder_inference import noise_schedule
    cfg = diffwave_cfg(HP_DIFFWAVE_RECIPE, 100)
    DiffWave(cfg)
    T, alpha, beta, alpha_cum = noise_schedule(cfg, fast)
    T_o, alpha_o, beta_o, alpha_cum_o = schedule(HP_DIFFWAVE_RECIPE, fast)
    assert T.dtype == np.float32 and np.array_equal(T, T_o)
    assert np.array_equal(alpha, alpha_o) and np.array_equal(beta, beta_o) and np.array_equal(alpha_cum, alpha_cum_o)
    assert len(T) == len(alpha) == (6 if fast else 50)
    assert np.all(np.diff(T) > 0) and T[0] >= 0 and np.ceil(T[-1]) < 50


def test_registry_entries():
    import amphion_b200.vocoders as v
    from amphion_b200.vocoders import diffusion_vocoder_inference as dvi
    from amphion_b200.vocoders.gan_vocoder_inference import synthesis_audios, vocoder_inference
    assert v._vocoders["diffwave"] is v.DiffWave
    assert v._vocoder_forward_funcs["diffwave"] is dvi.vocoder_inference
    assert v._vocoder_infer_funcs["diffwave"] is dvi.synthesis_audios
    for k in ("hifigan", "bigvgan", "nsfhifigan", "melgan", "apnet"):
        assert v._vocoder_forward_funcs[k] is vocoder_inference and v._vocoder_infer_funcs[k] is synthesis_audios


def test_tensor_table_and_options_without_gpu():
    from amphion_b200 import _capi
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL)
    h = m._ensure_handle()
    names = [_capi.lib.ab_generator_tensor_name(h, i).decode() for i in range(_capi.lib.ab_generator_num_tensors(h))]
    assert sorted(names) == sorted(list(m.state_dict()) + ["diffusion_embedding.embedding"])
    assert _capi.lib.ab_generator_output_samples(h, 5, 0) == 5 * 16
    assert _capi.lib.ab_generator_workspace_bytes(h, 1, 5) == 0
    assert _capi.lib.ab_diffwave_workspace_bytes(h, 1, 5, 1) > 0
    for key in ("resblock_fusion", "pair_schedule"):
        assert _capi.lib.ab_generator_set_option(h, key.encode(), 0) == -1
    rc = _capi.lib.ab_diffwave_step(h, C.c_void_p(256), 1, 5, 0, 1.0, 0.0, 0.0, None, C.c_void_p(256), C.c_void_p(256),
                                    1 << 30, None)
    assert rc == -4   # no conditioning yet


def _config(**kw):
    from amphion_b200 import _capi
    c = _capi.GeneratorConfig()
    c.kind, c.n_mel, c.upsample_initial_channel, c.num_layers, c.num_upsamples = _capi.GEN_DIFFWAVE, 10, 64, 6, 2
    c.upsample_rates[0] = c.upsample_rates[1] = 4
    c.dilation_cycle, c.embedding_rows = 3, 50
    for k, v in kw.items():
        if k == "rate":
            c.upsample_rates[1] = v
        else:
            setattr(c, k, v)
    return c


@pytest.mark.parametrize("what,kw,code", [("ok", {}, 0), ("odd_factor", dict(rate=3), -2), ("channels", dict(upsample_initial_channel=32), -2),
                                          ("three_factors", dict(num_upsamples=3), -1), ("cycle", dict(dilation_cycle=0), -1),
                                          ("foreign_field", dict(ffn_channels=8), -1),
                                          ("field_elsewhere", dict(kind=0, dilation_cycle=3), -1)])
def test_create_refuses_malformed_configs(what, kw, code):
    from amphion_b200 import _capi
    h = C.c_void_p()
    rc = _capi.lib.ab_generator_create(C.byref(_config(**kw)), C.byref(h))
    if rc == 0:
        _capi.lib.ab_generator_destroy(h)
    assert rc == code, (what, _capi.last_error())


def test_refusals():
    from amphion_b200.vocoders.diffusion_vocoder_inference import vocoder_inference
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL)
    mel = torch.zeros(1, GOLDEN_DIFFWAVE_MEL, 5)
    with pytest.raises(ValueError, match="hop_size"):
        vocoder_inference(diffwave_cfg(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, hop=12), m, mel)
    with pytest.raises(ValueError, match="audio must be"):
        m(torch.zeros(1, 5 * 16 + 1), torch.tensor([1]), mel)
    hp = dict(GOLDEN_DIFFWAVE, upsample_factors=[4, 3])
    with pytest.raises(ValueError, match="even"):
        build(hp, GOLDEN_DIFFWAVE_MEL)(torch.zeros(1, 60), torch.tensor([1]), mel)


# ------------------------------------------------------------------------------------------------ GPU


def _eps(model, audio, steps, mel):
    return model(torch.as_tensor(audio).cuda(), steps, mel).cpu().numpy()


def _strided(mel):
    """the same values as a transposed (non-contiguous) view, as synthesis() feeds mels"""
    return torch.from_numpy(np.ascontiguousarray(np.swapaxes(mel, 1, 2))).cuda().transpose(1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_matches_fixture_and_oracle(precision):
    g, sd, _ = load_dw()
    operands, tol = PREC_TOL[precision]
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd, precision=precision).cuda()
    mel = _strided(g["mel"])
    for steps, want in ((torch.tensor([2.37]), g["eps_float"]), (torch.tensor(g["steps_int"]), g["eps_int"])):
        got = _eps(m, g["audio"], steps, mel)
        oracle = diffwave_forward(sd, GOLDEN_DIFFWAVE, g["table"], g["audio"], steps.numpy(), g["mel"], operands=operands)
        peak = float(np.abs(want).max())
        assert got.shape == want.shape
        assert float(np.abs(got - oracle).max()) <= tol * peak
        if operands is None:
            assert float(np.abs(got - want).max()) <= tol * peak


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("steps", ["int1", "float1", "intB", "floatB"])
def test_forward_recipe_geometry(steps, precision):
    n_mel, B, F = 100, 2, 8
    operands, tol = PREC_TOL[precision]
    m = trained_like(build(HP_DIFFWAVE_RECIPE, n_mel, seed=5, precision=precision), 6).cuda()
    sd, table = sd_numpy(m), m.diffusion_embedding.embedding.cpu().numpy()
    gen = torch.Generator().manual_seed(7)
    mel = torch.randn(B, n_mel, F, generator=gen).numpy()
    audio = (torch.randn(B, F * 256, generator=gen) * 0.5).numpy()
    step = {"int1": torch.tensor([17]), "float1": torch.tensor([3.61]), "intB": torch.tensor([0, 49]),
            "floatB": torch.tensor([0.25, 48.5])}[steps]
    got = _eps(m, audio, step.cuda(), _strided(mel))
    want = diffwave_forward(sd, HP_DIFFWAVE_RECIPE, table, audio, step.numpy(), mel, operands=operands)
    assert float(np.abs(got - want).max()) <= tol * float(np.abs(want).max())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cycle,F", [(8, 7), (8, 3), (10, 2)])
def test_large_dilations_ragged_tiles_and_short_utterances(cycle, F, precision):
    """dilations up to 128 / 512 >= the 64-sample tile; 112 samples (ragged last tile), 48 and 32 samples (shorter than
    the largest dilation); 12 mels (the tensor-core K padding)"""
    hp = dict(GOLDEN_DIFFWAVE, residual_layers=cycle, dilation_cycle_length=cycle)
    operands, tol = PREC_TOL[precision]
    m = trained_like(build(hp, 12, seed=9, precision=precision), 10).cuda()
    sd, table = sd_numpy(m), m.diffusion_embedding.embedding.cpu().numpy()
    gen = torch.Generator().manual_seed(11)
    mel = torch.randn(2, 12, F, generator=gen).numpy()
    audio = (torch.randn(2, F * 16, generator=gen) * 0.5).numpy()
    got = _eps(m, audio, torch.tensor([1.5]), _strided(mel))
    want = diffwave_forward(sd, hp, table, audio, [1.5], mel, operands=operands)
    assert float(np.abs(got - want).max()) <= tol * float(np.abs(want).max())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_batch_independence_and_repeat_runs_bit_equal(precision):
    g, sd, _ = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd, precision=precision).cuda()
    mel = torch.from_numpy(g["mel"]).cuda()
    audio = torch.from_numpy(g["audio"]).cuda()
    both = m(audio, torch.tensor([2.37]), mel).cpu()
    assert torch.equal(both, m(audio, torch.tensor([2.37]), mel).cpu())
    for b in range(2):
        assert torch.equal(both[b:b + 1], m(audio[b:b + 1], torch.tensor([2.37]), mel[b:b + 1]).cpu())


@pytest.mark.gpu
@pytest.mark.parametrize("precision,tol", [("fp32", SAMPLER_TOL), ("tc_f16", 5e-3)])
def test_sampler_with_injected_noise_matches_fixture(monkeypatch, precision, tol):
    from amphion_b200.vocoders import diffusion_vocoder_inference as dvi
    g, sd, _ = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd, precision=precision).cuda()
    n_steps = len(GOLDEN_DIFFWAVE["inference_noise_schedule"])
    queue = [g["sampler_noise0"]] + [g[f"sampler_noise{n}"] for n in range(n_steps - 1, 0, -1)]

    def draw(*shape, **kw):
        return torch.from_numpy(queue.pop(0)).cuda()

    monkeypatch.setattr(dvi.torch, "randn", draw)
    monkeypatch.setattr(dvi.torch, "randn_like", lambda t: draw())
    cfg = diffwave_cfg(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL)
    cfg.model.diffwave.noise_schedule = m.cfg.model.diffwave.noise_schedule
    got = dvi.vocoder_inference(cfg, m, torch.from_numpy(g["sampler_mel"]), device="cuda", fast_inference=True)
    assert not queue and got.device.type == "cpu"
    assert float(np.abs(got.numpy() - g["sampler_audio"]).max()) <= tol


@pytest.mark.gpu
@pytest.mark.parametrize("fast", [True, False])
def test_seeded_sampler_draws_the_reference_noise(fast):
    """Native sampler from seed s == the oracle fed with torch.randn / randn_like drawn from seed s in the reference's
    order (initial audio, then one draw per step n > 0)."""
    from amphion_b200.vocoders.diffusion_vocoder_inference import vocoder_inference
    _, sd, _ = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd).cuda()
    cfg = m.cfg
    mel = torch.randn(1, GOLDEN_DIFFWAVE_MEL, 4, generator=torch.Generator().manual_seed(3))
    torch.manual_seed(1234)
    got = vocoder_inference(cfg, m, mel, device=torch.device("cuda"), fast_inference=fast).numpy()
    torch.manual_seed(1234)
    audio0 = torch.randn(1, 64, device="cuda")
    T = schedule(GOLDEN_DIFFWAVE, fast)[0]
    noises = {n: torch.randn_like(audio0).cpu().numpy() for n in range(len(T) - 1, 0, -1)}
    want = sample(sd, GOLDEN_DIFFWAVE, m.diffusion_embedding.embedding.cpu().numpy(), mel.numpy(), audio0.cpu().numpy(), noises,
                  fast_inference=fast)
    assert float(np.abs(got - want).max()) <= (SAMPLER_TOL if fast else 1e-3)


@pytest.mark.gpu
def test_synthesis_runs_the_recipe_generator(tmp_path):
    """synthesis() with cfg.model.generator == "diffwave": registry construction, checkpoint load, per-utterance sampler,
    trimmed lengths"""
    from amphion_b200.vocoders import synthesis
    _, sd, _ = load_dw()
    path = tmp_path / "ckpt.pt"
    torch.save({"generator_state_dict": {k: torch.as_tensor(v) for k, v in sd.items()}}, path)
    cfg = diffwave_cfg(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL)
    mels = [np.random.default_rng(i).standard_normal((f, GOLDEN_DIFFWAVE_MEL)).astype(np.float32) for i, f in enumerate((5, 3, 7))]
    out = synthesis(cfg, str(path), None, mels, fast_inference=True)
    assert [len(a) for a in out] == [5 * 16, 3 * 16, 7 * 16]
    assert all(a.device.type == "cpu" and float(a.abs().max()) <= 1.0 for a in out)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_profile_classes(precision):
    """a DiffWave handle reports 11 classes; one forward is 2 conditioning, 1 input, one per layer and 1 tail launch"""
    g, sd, _ = load_dw()
    m = build(GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL, sd, precision=precision).cuda()
    m.set_profiling(True)
    m(torch.from_numpy(g["audio"]).cuda(), torch.tensor([2.37]), torch.from_numpy(g["mel"]).cuda())
    prof = m.get_profile()
    assert len(prof) == 11
    want = {"diffwave_cond": 2, "diffwave_input": 1, "diffwave_layer": GOLDEN_DIFFWAVE["residual_layers"], "diffwave_tail": 1}
    assert {k: v["launches"] for k, v in prof.items() if v["launches"]} == want
    assert all(prof[k]["ms"] > 0 and prof[k]["flops"] > 0 and prof[k]["bytes"] > 0 for k in want)
    assert m.last_launches == sum(want.values())
