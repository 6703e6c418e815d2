"""Float64 numpy restatement of DiffWave (models/vocoders/diffusion/diffwave/diffwave.py) and of its sampler
(models/vocoders/diffusion/diffusion_vocoder_inference.py:13-73), the checker of the native path.  The step-embedding
table is an input: the reference builds it in fp32 from angles up to 10^4 times the step, where fp32 rounding of the
angle alone moves sin / cos by up to ~1e-2, so the oracle uses the fp32 table the model holds."""
from types import SimpleNamespace as NS

import numpy as np

# reduced geometry of tests/golden/diffwave*.npz (tests/golden/gen_diffwave.py)
GOLDEN_DIFFWAVE = dict(residual_channels=64, residual_layers=6, dilation_cycle_length=3, upsample_factors=[4, 4],
                       noise_schedule_factors=[1.0e-4, 0.05, 50],
                       inference_noise_schedule=[0.0001, 0.001, 0.01, 0.05, 0.2, 0.5])
GOLDEN_DIFFWAVE_MEL = 10    # n_mel of the fixture
GOLDEN_DIFFWAVE_BF = (2, 6)  # batch, frames

# egs/vocoder/diffusion/diffwave/exp_config.json over config/vocoder.json
HP_DIFFWAVE_RECIPE = dict(residual_channels=64, residual_layers=30, dilation_cycle_length=10, upsample_factors=[16, 16],
                          noise_schedule_factors=[1.0e-4, 0.05, 50],
                          inference_noise_schedule=[0.0001, 0.001, 0.01, 0.05, 0.2, 0.5])


def diffwave_cfg(hp, n_mel, hop=None):
    f = hp["upsample_factors"]
    return NS(preprocess=NS(n_mel=n_mel, hop_size=hop if hop is not None else f[0] * f[1]),
              model=NS(generator="diffwave", diffwave=NS(**{k: list(v) if isinstance(v, list) else v for k, v in hp.items()})))


def _convt2d_lrelu(x, w, b, f):
    """ConvTranspose2d(1, 1, [3, 2f], stride [1, f], padding [1, f // 2]) on [B, H, W], then leaky_relu(0.4)."""
    B, H, W = x.shape
    full = np.zeros((B, H + 2, (W - 1) * f + 2 * f))
    for kh in range(3):
        for kw in range(2 * f):
            full[:, kh:kh + H, kw:kw + (W - 1) * f + 1:f] += x * w[kh, kw]
    wout = (W - 1) * f - 2 * (f // 2) + 2 * f
    y = full[:, 1:1 + H, f // 2:f // 2 + wout] + b
    return np.where(y > 0, y, 0.4 * y)


def upsample(sd, hp, mel):
    x = np.asarray(mel, np.float64)
    for i, f in enumerate(hp["upsample_factors"]):
        pre = f"spectrogram_upsampler.conv{i + 1}"
        x = _convt2d_lrelu(x, np.asarray(sd[pre + ".weight"], np.float64).reshape(3, 2 * f), float(sd[pre + ".bias"][0]), f)
    return x


def _silu(x):
    return x / (1.0 + np.exp(-x))


def step_embedding(sd, table, steps):
    """[n, 512] for float steps (an integer step is its own float value)."""
    t = np.asarray(steps, np.float64).reshape(-1)
    tab = np.asarray(table, np.float64)
    lo, hi = np.floor(t).astype(np.int64), np.ceil(t).astype(np.int64)
    e = tab[lo] + (tab[hi] - tab[lo]) * (t - lo)[:, None]
    g = lambda k: np.asarray(sd[k], np.float64)  # noqa: E731
    h = _silu(e @ g("diffusion_embedding.projection1.weight").T + g("diffusion_embedding.projection1.bias"))
    return _silu(h @ g("diffusion_embedding.projection2.weight").T + g("diffusion_embedding.projection2.bias"))


def round_operand(a, operands):
    """a rounded to the 16-bit type the tensor-core layer kernel feeds its MMAs ("f16" / "bf16"), or as is (None)."""
    if operands is None:
        return a
    import torch
    t = torch.from_numpy(np.asarray(a, np.float32)).to(torch.float16 if operands == "f16" else torch.bfloat16)
    return t.to(torch.float64).numpy()


def diffwave_forward(sd, hp, table, audio, steps, mel, layers_out=False, cond=None, operands=None):
    """audio [B, L], steps (1 or B values), mel [B, n_mel, F] -> eps [B, 1, L] (and per-layer (x, skip) if asked).
    operands = "f16" / "bf16": the residual layers' conv operands (x + d, the upsampled mel, the gate and the three
    weights) rounded to that type, as the tensor-core path computes them."""
    g = lambda k: np.asarray(sd[k], np.float64)  # noqa: E731
    r = lambda a: round_operand(a, operands)  # noqa: E731
    nl, cyc = hp["residual_layers"], hp["dilation_cycle_length"]
    a = np.asarray(audio, np.float64)
    B, L = a.shape
    x = np.maximum(g("input_projection.weight")[None, :, 0, :] * a[:, None, :] + g("input_projection.bias")[None, :, None], 0)
    C = x.shape[1]
    c = upsample(sd, hp, mel) if cond is None else cond
    emb = step_embedding(sd, table, steps)
    skip, outs = None, []
    for i in range(nl):
        pre, d = f"residual_layers.{i}", 2 ** (i % cyc)
        dp = emb @ g(pre + ".diffusion_projection.weight").T + g(pre + ".diffusion_projection.bias")
        y = x + dp[:, :, None]
        yp = np.pad(r(y), ((0, 0), (0, 0), (d, d)))
        w = r(g(pre + ".dilated_conv.weight"))
        z = sum(np.einsum("oc,bct->bot", w[:, :, k], yp[:, :, k * d:k * d + L]) for k in range(3))
        z = z + g(pre + ".dilated_conv.bias")[None, :, None]
        z = z + np.einsum("om,bmt->bot", r(g(pre + ".conditioner_projection.weight")[:, :, 0]), r(c))
        z = z + g(pre + ".conditioner_projection.bias")[None, :, None]
        gated = 1.0 / (1.0 + np.exp(-z[:, :C])) * np.tanh(z[:, C:])
        o = np.einsum("oc,bct->bot", r(g(pre + ".output_projection.weight")[:, :, 0]), r(gated))
        o = o + g(pre + ".output_projection.bias")[None, :, None]
        x = (x + o[:, :C]) / np.sqrt(2.0)
        skip = o[:, C:] if skip is None else o[:, C:] + skip
        outs.append((x, skip))
    s = skip / np.sqrt(nl)
    h = np.maximum(np.einsum("oc,bct->bot", g("skip_projection.weight")[:, :, 0], s) + g("skip_projection.bias")[None, :, None], 0)
    eps = np.einsum("oc,bct->bot", g("output_projection.weight")[:, :, 0], h) + g("output_projection.bias")[None, :, None]
    return (eps, outs) if layers_out else eps


def schedule(hp, fast_inference=True):
    """(T, alpha, beta, alpha_cum) of vocoder_inference (:22-46), T in float32 as the reference stores it."""
    f = hp["noise_schedule_factors"]
    train = np.linspace(f[0], f[1], f[2])
    beta = np.array(hp["inference_noise_schedule"]) if fast_inference else train
    talpha_cum = np.cumprod(1 - train)
    alpha = 1 - beta
    alpha_cum = np.cumprod(alpha)
    T = []
    for s in range(len(beta)):
        for t in range(len(train) - 1):
            if talpha_cum[t + 1] <= alpha_cum[s] <= talpha_cum[t]:
                T.append(t + (talpha_cum[t] ** 0.5 - alpha_cum[s] ** 0.5) / (talpha_cum[t] ** 0.5 - talpha_cum[t + 1] ** 0.5))
                break
    return np.array(T, dtype=np.float32), alpha, beta, alpha_cum


def sample(sd, hp, table, mel, audio0, noises, fast_inference=True, operands=None):
    """The sampler loop with the given initial audio and noises[n] (n > 0) -> audio [B, L]."""
    T, alpha, beta, alpha_cum = schedule(hp, fast_inference)
    cond = upsample(sd, hp, mel)
    audio = np.asarray(audio0, np.float64)
    for n in range(len(alpha) - 1, -1, -1):
        c1 = 1 / alpha[n] ** 0.5
        c2 = beta[n] / (1 - alpha_cum[n]) ** 0.5
        eps = diffwave_forward(sd, hp, table, audio, [float(T[n])], mel, cond=cond, operands=operands)[:, 0]
        audio = c1 * (audio - c2 * eps)
        if n > 0:
            sigma = ((1.0 - alpha_cum[n - 1]) / (1.0 - alpha_cum[n]) * beta[n]) ** 0.5
            audio = audio + sigma * np.asarray(noises[n], np.float64)
        audio = np.clip(audio, -1.0, 1.0)
    return audio
