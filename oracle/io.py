"""Oracle: the arithmetic of save_audio (utils/io.py of the reference:49-76) in numpy.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

``save_audio_float`` follows :59-75 (turn_up, add_silence, mono) and is pinned by tests/golden/save_audio.npz,
which was produced by RUNNING the reference's save_audio with ``torchaudio.save`` intercepted (the tensor it
receives is the fixture).  ``pcm16`` restates the last step, ``torchaudio.save(..., encoding="PCM_S",
bits_per_sample=16)`` (:76), from the published algorithm of the reference's pinned torchaudio 2.0.2 (sox_io
backend): float32 * 2^31 -> int32, then SOX_SAMPLE_TO_SIGNED_16BIT = (s + 0x8000) >> 16 with clipping, i.e.
clamp(floor(x * 32768 + 0.5), -32768, 32767).  PARITY UNPINNED for ``pcm16``: torchaudio.save cannot run in
the build container (needs torchcodec / sox), so there is no reference output to pin it to.
"""
from __future__ import annotations

import numpy as np


def save_audio_float(waveform, fs, add_silence=False, turn_up=False, volume_peak=0.9):
    """-> float32 [1, T'] exactly as handed to torchaudio.save (:70-76)."""
    waveform = np.asarray(waveform, np.float32)
    if turn_up:  # :59-62 (numpy 2 scalar promotion: the ratio is float32)
        peak = max(waveform.max(), abs(waveform.min()))
        # an all-zero waveform makes the reference divide by zero (NaN samples); the product keeps it silent
        ratio = np.float32(volume_peak) / peak if peak > 0 else np.float32(1.0)
        waveform = waveform * ratio
    if add_silence:  # :64-68
        silence = np.zeros((fs // 20,), dtype=waveform.dtype)
        waveform = np.concatenate([silence, waveform, silence])
    if waveform.ndim == 1:
        waveform = waveform[None, :]
    elif waveform.shape[0] != 1:
        waveform = waveform.mean(axis=0, keepdims=True, dtype=np.float32)
    return waveform.astype(np.float32)


def pcm16(x):
    q = np.floor(np.asarray(x, np.float32) * np.float32(32768.0) + np.float32(0.5))
    return np.clip(q, -32768, 32767).astype(np.int16)
