"""Oracle: mel-spectrogram front end (utils/mel.py, utils/stft.py), restated.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Third-party arithmetic not present of the reference (open-mmlab/Amphion) is restated here from
its published algorithm (the reference pins ``librosa==0.9.1`` in env.sh:13):
  * ``librosa.filters.mel`` (Slaney scale, ``norm="slaney"``)  -> ``slaney_mel_filterbank``
  * ``librosa.util.pad_center``                                  -> ``pad_center``
All citations are to files of the reference (open-mmlab/Amphion).
"""
from __future__ import annotations

import numpy as np


# --------------------------------------------------------------------------
# librosa 0.9.1 restatements
# --------------------------------------------------------------------------
def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    if f.ndim:
        m = f >= min_log_hz
        mels[m] = min_log_mel + np.log(f[m] / min_log_hz) / logstep
    elif f >= min_log_hz:
        mels = min_log_mel + np.log(f / min_log_hz) / logstep
    return mels


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    log_t = m >= min_log_mel
    freqs[log_t] = min_log_hz * np.exp(logstep * (m[log_t] - min_log_mel))
    return freqs


def slaney_mel_filterbank(sr, n_fft, n_mels, fmin, fmax) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) with htk=False,
    norm='slaney', dtype float32, as called at utils/mel.py:66-72,133-139 and
    utils/stft.py:245-247.  Returns [n_mels, n_fft//2+1] float32."""
    if fmax is None:
        fmax = float(sr) / 2
    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, float(sr) / 2, n_bins, endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, n_bins), dtype=np.float32)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


def pad_center(data, size):
    n = data.shape[-1]
    lpad = int((size - n) // 2)
    return np.pad(data, (lpad, int(size - n - lpad)), mode="constant")


def hann_periodic(n) -> np.ndarray:
    """torch.hann_window(n) (periodic) == scipy.signal.get_window('hann', n,
    fftbins=True) (utils/mel.py:26,142; utils/stft.py:141)."""
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n))


# --------------------------------------------------------------------------
# utils/mel.py family
# --------------------------------------------------------------------------
def _reflect_pad(y, p):
    return np.pad(y, ((0, 0), (p, p)), mode="reflect") if p > 0 else y


def stft_magnitude(y, n_fft, hop, win, eps, pad):
    """reflect-pad ``pad`` each side, frame (center=False), periodic hann of
    length ``win`` centred in n_fft, one-sided DFT, sqrt(re^2+im^2+eps).
    y [B, T] float32 -> [B, n_fft//2+1, F] float32 (utils/mel.py:145-166)."""
    y = np.asarray(y, np.float32)
    yp = _reflect_pad(y, pad)
    nfr = 1 + (yp.shape[1] - n_fft) // hop
    w = pad_center(hann_periodic(win).astype(np.float32), n_fft).astype(np.float32)
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]
    frames = yp[:, idx] * w[None, None, :]                    # fp32 multiply, as torch.stft does
    spec = np.fft.rfft(frames.astype(np.float32), axis=-1)    # [B, F, bins]
    re = spec.real.astype(np.float32)
    im = spec.imag.astype(np.float32)
    mag = np.sqrt(re * re + im * im + np.float32(eps), dtype=np.float32)
    return np.ascontiguousarray(mag.transpose(0, 2, 1))


def log_compress(x, clip=1e-5):
    # utils/mel.py:10-12, utils/stft.py:97-103
    return np.log(np.maximum(x, np.float32(clip))).astype(np.float32)


def extract_linear_features(y, n_fft, hop, win):
    """utils/mel.py:20-52 (eps 1e-9)."""
    return stft_magnitude(y, n_fft, hop, win, 1e-9, (n_fft - hop) // 2)


def extract_mel_features(y, mel_basis, n_fft, hop, win, eps=1e-9):
    """utils/mel.py:111-170 (eps 1e-9); mel_spectrogram_torch :55-104 uses eps 1e-6.
    y [B,T] -> [B, n_mel, F] (the caller applies the reference's squeeze(0))."""
    mag = stft_magnitude(y, n_fft, hop, win, eps, (n_fft - hop) // 2)
    mel = np.einsum("mk,bkf->bmf", np.asarray(mel_basis, np.float32), mag, dtype=np.float32)
    return log_compress(mel)


def amplitude_phase_spectrum(y, n_fft, hop, win):
    """utils/mel.py:244-280: log(|X| + 1e-5), atan2(im, re), re, im of the reflect-padded, hann-windowed STFT
    (center=False).  y [B, T] -> four arrays [B, n_fft//2+1, F] float32."""
    y = np.asarray(y, np.float32)
    yp = _reflect_pad(y, (n_fft - hop) // 2)
    nfr = 1 + (yp.shape[1] - n_fft) // hop
    w = pad_center(hann_periodic(win).astype(np.float32), n_fft).astype(np.float32)
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]
    spec = np.fft.rfft((yp[:, idx] * w[None, None, :]).astype(np.float32), axis=-1).transpose(0, 2, 1)
    re, im = spec.real.astype(np.float32), spec.imag.astype(np.float32)
    logamp = np.log(np.sqrt(re * re + im * im) + np.float32(1e-5)).astype(np.float32)
    return logamp, np.arctan2(im, re).astype(np.float32), re, im


def extract_mel_features_vjp(y, mel_basis, grad_mel, n_fft, hop, win, eps=1e-9, clip=1e-5):
    """Cotangent of the waveform for a cotangent ``grad_mel`` [B, n_mel, F] of ``extract_mel_features`` — what
    autograd computes through utils/mel.py:145-169 when the trainers differentiate the mel loss
    (models/vocoders/gan/gan_vocoder_trainer.py:368-396).  Written from the definitions in float64: explicit
    cos/sin DFT matrices, ``d sqrt``, ``torch.clamp`` semantics (gradient passes where the value is >= clip),
    scatter-add through the frame and reflect-pad index maps.  Pinned against the reference's own autograd result
    in tests/golden/mel_grad.npz (tests/test_oracle.py).  y [B, T] -> [B, T] float64."""
    y = np.asarray(y, np.float64)
    B, T = y.shape
    pad = (n_fft - hop) // 2
    ridx = np.pad(np.arange(T), (pad, pad), mode="reflect")              # padded position -> sample index
    nfr = 1 + (T + 2 * pad - n_fft) // hop
    w = pad_center(hann_periodic(win).astype(np.float32), n_fft).astype(np.float64)
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]       # [F, n_fft] padded positions
    frames = y[:, ridx[idx]] * w[None, None, :]                           # [B, F, n_fft]
    k = np.arange(n_fft // 2 + 1)[:, None] * np.arange(n_fft)[None, :]
    cosm, sinm = np.cos(2 * np.pi * k / n_fft), np.sin(2 * np.pi * k / n_fft)
    re = frames @ cosm.T                                                  # [B, F, bins]
    im = -(frames @ sinm.T)
    mag = np.sqrt(re * re + im * im + eps)
    basis = np.asarray(mel_basis, np.float64)
    acc = np.einsum("mk,bfk->bmf", basis, mag)
    g_acc = np.where(acc >= clip, np.asarray(grad_mel, np.float64) / np.maximum(acc, 1e-300), 0.0)
    g_mag = np.einsum("mk,bmf->bfk", basis, g_acc)
    g_re, g_im = g_mag * re / mag, g_mag * im / mag
    g_frames = (g_re @ cosm - g_im @ sinm) * w[None, None, :]            # [B, F, n_fft]
    gy = np.zeros((B, T))
    tgt = ridx[idx]                                                       # [F, n_fft] sample index of every frame tap
    for b in range(B):
        np.add.at(gy[b], tgt.reshape(-1), g_frames[b].reshape(-1))
    return gy


# --------------------------------------------------------------------------
# utils/stft.py TacotronSTFT
# --------------------------------------------------------------------------
def tacotron_forward_basis(n_fft, win) -> np.ndarray:
    """utils/stft.py:126-147: rows = [Re; Im] of fft(eye(n_fft))[:n_fft/2+1],
    times the centred periodic hann, cast to float32. [n_fft+2, n_fft]."""
    fb = np.fft.fft(np.eye(n_fft))
    cutoff = n_fft // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff]), np.imag(fb[:cutoff])]).astype(np.float32)
    w = pad_center(hann_periodic(win), n_fft).astype(np.float32)
    return (fb * w[None, :]).astype(np.float32)


def tacotron_mel(y, mel_basis, n_fft, hop, win):
    """TacotronSTFT.mel_spectrogram (utils/stft.py:259-278) over STFT.transform
    (:152-181): reflect-pad n_fft/2, conv with the windowed DFT basis at stride
    hop, magnitude WITHOUT eps, mel, log-clamp; energy = l2 norm over bins.
    Returns (mel [B,n_mel,F], energy [B,F])."""
    y = np.asarray(y, np.float32)
    assert y.min() >= -1 and y.max() <= 1          # utils/stft.py:269-270
    yp = _reflect_pad(y, n_fft // 2)
    nfr = 1 + (yp.shape[1] - n_fft) // hop
    basis = tacotron_forward_basis(n_fft, win)      # [n_fft+2, n_fft]
    idx = np.arange(n_fft)[None, :] + hop * np.arange(nfr)[:, None]
    frames = yp[:, idx]                             # [B, F, n_fft]
    ft = np.einsum("kn,bfn->bkf", basis, frames, dtype=np.float32)
    cutoff = n_fft // 2 + 1
    re, im = ft[:, :cutoff], ft[:, cutoff:]
    mag = np.sqrt(re * re + im * im, dtype=np.float32)
    mel = np.einsum("mk,bkf->bmf", np.asarray(mel_basis, np.float32), mag, dtype=np.float32)
    energy = np.sqrt((mag * mag).sum(axis=1, dtype=np.float32), dtype=np.float32)
    return log_compress(mel), energy
