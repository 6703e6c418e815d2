"""Config 4: TacotronSTFT(1024,256,1024,80,22050,0,8000).mel_spectrogram on 64 x 10 s @ 22.05 kHz (device-resident)."""
import os, sys, json, time, warnings
warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from amphion_b200 import mel as M
from amphion_b200.stft import TacotronSTFT
g = torch.Generator().manual_seed(0)
y = ((torch.rand(64, 220500, generator=g) * 2 - 1) * 0.9).cuda()
taco = TacotronSTFT(1024, 256, 1024, 80, 22050, 0, 8000)
win, basis = taco.stft_fn.fft_window, taco.mel_basis.cuda()
def step():
    return M.native_stft_mel(y, 1024, 256, 1024, win, basis, 512, 0.0, want_energy=True)
for _ in range(5): step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
ts = []
for _ in range(10):
    flush.zero_()                      # flush L2 between timed iterations
    e0.record(); out = step(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
ms = sorted(ts)[len(ts) // 2]
F = out[1].shape[-1]
algo_bytes = y.numel() * 4 + out[1].numel() * 4 + out[2].numel() * 4
print(json.dumps(dict(workload="TacotronSTFT mel 64x10s@22.05kHz", frames=int(64 * F), ms=ms, best_ms=min(ts),
                      frames_per_s=64 * F / ms * 1e3, audio_samples_per_s=y.numel() / ms * 1e3,
                      algorithmic_GBs=algo_bytes / ms / 1e6, hbm_frac=algo_bytes / ms / 1e6 / 3350.0)))   # H100 SXM data-sheet HBM3 GB/s
# torch eager (the reference's ops on the same GPU, TF32 off) for context
torch.backends.cuda.matmul.allow_tf32 = False
def ref():
    yp = torch.nn.functional.pad(y.unsqueeze(1), (512, 512), mode="reflect").squeeze(1)
    s = torch.stft(yp, 1024, hop_length=256, win_length=1024, window=win.cuda(), center=False, return_complex=True)
    mag = s.abs()
    return torch.log(torch.clamp(torch.matmul(basis, mag), min=1e-5)), torch.norm(mag, dim=1)
for _ in range(3): ref()
torch.cuda.synchronize(); e0.record()
for _ in range(10): ref()
e1.record(); torch.cuda.synchronize()
print(json.dumps(dict(torch_eager_fft_ms=e0.elapsed_time(e1) / 10)))
