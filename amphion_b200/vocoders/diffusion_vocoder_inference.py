"""The DiffWave sampler with the reference's signatures and semantics
(models/vocoders/diffusion/diffusion_vocoder_inference.py:13-131).  The loop stays on the host, step for step as the
reference runs it, and draws its noise from the torch CUDA generator in the same order: the initial ``torch.randn``,
then one ``torch.randn_like`` per step with n > 0.  The network draws nothing, so drawing step n's noise just before its
launches hands every step the reference's noise values.  What changes is that the conditioning (upsampled mel, step
embeddings), which does not depend on the step, is computed once per call, and each step is one native network pass
whose last kernel also applies the update and the clamp."""
from __future__ import annotations

import numpy as np
import torch

from ..util import pad_mels_to_tensors


def noise_schedule(cfg, fast_inference=False):
    """(T, alpha, beta, alpha_cum) as vocoder_inference computes them: T[s] is the fractional training step whose
    cumulative alpha matches the inference schedule's, in float32."""
    training_noise_schedule = np.array(cfg.model.diffwave.noise_schedule)
    inference_noise_schedule = (np.array(cfg.model.diffwave.inference_noise_schedule) if fast_inference
                                else np.array(cfg.model.diffwave.noise_schedule))
    talpha = 1 - training_noise_schedule
    talpha_cum = np.cumprod(talpha)
    beta = inference_noise_schedule
    alpha = 1 - beta
    alpha_cum = np.cumprod(alpha)
    T = []
    for s in range(len(inference_noise_schedule)):
        for t in range(len(training_noise_schedule) - 1):
            if talpha_cum[t + 1] <= alpha_cum[s] <= talpha_cum[t]:
                twiddle = (talpha_cum[t] ** 0.5 - alpha_cum[s] ** 0.5) / (talpha_cum[t] ** 0.5 - talpha_cum[t + 1] ** 0.5)
                T.append(t + twiddle)
                break
    return np.array(T, dtype=np.float32), alpha, beta, alpha_cum


def vocoder_inference(cfg, model, mels, f0s=None, device=None, fast_inference=False):
    """mels [B, n_mel, F] -> audio [B, hop_size * F] on the CPU (fp32)."""
    model.eval()
    hop = int(cfg.preprocess.hop_size)
    if hop != model._hop():
        raise ValueError(f"amphion_b200: cfg.preprocess.hop_size {hop} must equal the product of the DiffWave upsample "
                         f"factors {model.upsample_factors}")
    if device is None:
        device = next(model.parameters()).device
    with torch.no_grad():
        T, alpha, beta, alpha_cum = noise_schedule(cfg, fast_inference)
        if len(T) != len(alpha):
            raise ValueError("amphion_b200: an inference noise level lies outside the training schedule's range")
        mels = mels.to(device)
        audio = torch.randn(mels.shape[0], hop * mels.shape[-1], device=device)
        mels = model._check_mel(mels)
        with torch.cuda.device(mels.device):
            ws, need = model._condition(mels, T)
            for n in range(len(alpha) - 1, -1, -1):
                c1 = 1 / alpha[n] ** 0.5
                c2 = beta[n] / (1 - alpha_cum[n]) ** 0.5
                noise, sigma = None, 0.0
                if n > 0:
                    noise = torch.randn_like(audio)
                    sigma = ((1.0 - alpha_cum[n - 1]) / (1.0 - alpha_cum[n]) * beta[n]) ** 0.5
                model._step(audio, n, c1, c2, sigma, noise, ws, need)
    return audio.detach().cpu()


def synthesis_audios(cfg, model, mels, f0s=None, batch_size=None, fast_inference=False):
    """mels: list of [n_mel, F] tensors -> list of 1-D CPU audios, one sampler call per utterance on its zero-padded
    batch row (as the reference does), trimmed to frames * hop_size."""
    device = next(model.parameters()).device
    audios = []
    mel_batches, mel_frames = pad_mels_to_tensors(mels, batch_size)
    for mel_batch, mel_frame in zip(mel_batches, mel_frames):
        for i in range(mel_batch.shape[0]):
            audio = vocoder_inference(cfg, model, mel_batch[i].unsqueeze(0), device=device,
                                      fast_inference=fast_inference).squeeze(0)
            audios.append(audio[:mel_frame[i] * cfg.preprocess.hop_size])
    return audios
