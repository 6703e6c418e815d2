"""Function boundary of the GAN vocoders, signatures as in the reference's
``models/vocoders/gan/gan_vocoder_inference.py`` (vocoder_inference :11,
synthesis_audios :41)."""
from __future__ import annotations

import torch

from ..util import pad_f0_to_tensors, pad_mels_to_tensors


def vocoder_inference(cfg, model, mels, f0s=None, device=None, fast_inference=False):
    """mels [B, n_mel, T] (any device / strides) -> audios [B, T*hop] on the CPU,
    detached fp32 — the reference's output contract (:38).  ``fast_inference``
    is accepted and ignored, as in the reference."""
    model.eval()
    with torch.no_grad():
        if device is None:
            device = next(model.parameters()).device
        mels = mels.to(device, non_blocking=True)
        if f0s is None and getattr(cfg.preprocess, "extract_amplitude_phase", False):
            _, _, _, _, output = model.forward(mels)     # amplitude/phase generators (APNet), :27-34
        elif f0s is None:
            host = _forward_chunked_to_host(model, mels)
            if host is not None:
                return host
            output = model.forward(mels)
        else:  # f0-conditioned generators (NSF-HiFiGAN), :36
            output = model.forward(mels, f0s.to(device, non_blocking=True))
        output = output.squeeze(1).detach()
        # the reference's `.cpu()` (:38) lands in pageable memory; a pinned buffer is
        # still a CPU tensor and lets the D2H copy run at full PCIe rate
        host = torch.empty(output.shape, dtype=output.dtype, pin_memory=True)
        host.copy_(output, non_blocking=True)
        torch.cuda.current_stream(output.device).synchronize()
        return host


_D2H_CHUNKS = 4
_copy_streams = {}


def _forward_chunked_to_host(model, mels):
    """Native generators run their last layer in batch chunks with an event after each
    (``forward(..., tail_events=...)``): the D2H copy of chunk i then runs on a side stream under the last layer of
    chunk i + 1 instead of after the whole forward.  Returns the pinned CPU tensor [B, T*hop], or None when the
    model has no such hook (the caller then copies after the forward, as the reference's ``.cpu()`` does)."""
    import inspect
    try:
        hooked = "tail_events" in inspect.signature(model.forward).parameters
    except (TypeError, ValueError):
        hooked = False
    B = mels.shape[0]
    if not (hooked and mels.is_cuda and B >= 2):
        return None
    n = min(_D2H_CHUNKS, B)
    dev = mels.device
    events = [torch.cuda.Event() for _ in range(n)]
    output = model.forward(mels, tail_events=events)          # [B, 1, L] on the current stream
    main = torch.cuda.current_stream(dev)
    side = _copy_streams.setdefault(str(dev), torch.cuda.Stream(device=dev))
    host = torch.empty((B, output.shape[-1]), dtype=output.dtype, pin_memory=True)
    flat = output.detach().squeeze(1)
    with torch.cuda.stream(side):
        for i in range(n):
            b0, b1 = B * i // n, B * (i + 1) // n                # the chunk bounds of NativeGenerator._arm_tail_events
            side.wait_event(events[i])
            host[b0:b1].copy_(flat[b0:b1], non_blocking=True)
    output.record_stream(side)
    side.synchronize()
    main.synchronize()
    return host


def _batches(cfg, model, mels, f0s, batch_size, bucket):
    """Yield (indices, padded mel batch, frames, padded f0 batch).  ``bucket``: utterances are grouped by length
    (stable sort by frame count) so a batch pads to the longest of SIMILAR lengths — less padded compute.  The
    reference batches in input order (:52-56), and an utterance's last receptive field of samples depends on how
    much zero mel follows it (Q12), so bucketing is opt-in: with it, those tail samples equal the reference run
    on the same grouping, not on the input-order grouping."""
    device = next(model.parameters()).device
    order = list(range(len(mels)))
    if bucket:
        order.sort(key=lambda i: int(mels[i].shape[-1]))
    step = len(order) if batch_size is None else int(batch_size)
    for start in range(0, len(order), max(step, 1)):
        idx = order[start:start + step]
        mb, mf = pad_mels_to_tensors([mels[i].to(device) for i in idx], None)
        fb = pad_f0_to_tensors([f0s[i].to(device) for i in idx], None)[0] if f0s is not None else None
        yield idx, mb[0], mf[0], fb


def synthesis_audios(cfg, model, mels, f0s=None, batch_size=None, fast_inference=False, bucket=False):
    """List of ``[n_mel, T_i]`` mels -> list of 1-D CPU audios trimmed to
    ``T_i * hop``.  The reference pads to the batch maximum and then runs every
    utterance alone (B=1) on its zero-padded mel (:59-75); the generator has no
    cross-batch op, so running the padded batch in ONE forward gives the same
    samples with one launch sequence and one D2H copy per batch.
    ``bucket=True`` (beyond the reference signature) groups utterances of similar length, see ``_batches``."""
    device = next(model.parameters()).device
    hop = model.cfg.preprocess.hop_size
    audios = [None] * len(mels)
    for idx, mel_batch, mel_frame, f0_batch in _batches(cfg, model, mels, f0s, batch_size, bucket):
        out = vocoder_inference(cfg, model, mel_batch, f0s=f0_batch, device=device, fast_inference=fast_inference)
        for j, i in enumerate(idx):
            audios[i] = out[j, : int(mel_frame[j]) * hop].clone()
    return audios


def synthesize_to_files(cfg, model, mels, paths, fs=None, f0s=None, batch_size=None, bucket=False,
                        add_silence=False, turn_up=False, volume_peak=0.9):
    """Generate and save: the body of ``VocoderInference.inference`` (models/vocoders/vocoder_inference.py:336-371 —
    forward, trim to ``target_len * hop``, ``save_audio`` per utterance) as one device pipeline per batch: generator
    forward, trim + peak-normalise + 16-bit PCM quantisation on the GPU (``ab_pcm16_forward``, utils/io.py:49-76),
    ONE int16 D2H copy (half the bytes of the reference's fp32 ``.cpu()``), then the RIFF files.  Returns ``paths``."""
    from ..io import waveform_to_pcm16, write_wav_pcm16
    if len(paths) != len(mels):
        raise ValueError(f"{len(paths)} paths for {len(mels)} mels")
    device = next(model.parameters()).device
    hop = model.cfg.preprocess.hop_size
    fs = int(fs if fs is not None else cfg.preprocess.sample_rate)
    silence = fs // 20 if add_silence else 0
    model.eval()
    with torch.no_grad():
        for idx, mel_batch, mel_frame, f0_batch in _batches(cfg, model, mels, f0s, batch_size, bucket):
            wav = model.forward(mel_batch) if f0_batch is None else model.forward(mel_batch, f0_batch)
            lens = [int(f) * hop for f in mel_frame]
            pcm = waveform_to_pcm16(wav.squeeze(1), lens, silence, turn_up, volume_peak)
            host = torch.empty(pcm.shape, dtype=torch.int16, pin_memory=True)
            host.copy_(pcm, non_blocking=True)
            torch.cuda.current_stream(device).synchronize()
            arr = host.numpy()
            for j, i in enumerate(idx):
                write_wav_pcm16(paths[i], arr[j, : lens[j] + 2 * silence], fs)
    return list(paths)
