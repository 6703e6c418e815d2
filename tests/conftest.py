import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


# The CPU oracle (oneDNN convs on small channel counts) gets slower, not faster, beyond ~16 threads: on the
# 128-thread GPU box the wide-model oracle took minutes.  Cap the threads the test process uses.
try:
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))
except Exception:  # pragma: no cover
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def load_golden(name):
    # a fixture may be split over name.npz and name.part<N>.npz (every stored file stays under 1 MB)
    d = {}
    for f in [name + ".npz"] + sorted(glob.glob(os.path.join(GOLDEN, glob.escape(name) + ".part*.npz"))):
        z = np.load(os.path.join(GOLDEN, f))
        d.update({k: z[k] for k in z.files})
    sd = {k[3:]: v for k, v in d.items() if k.startswith("sd:")}
    rest = {k: v for k, v in d.items() if not k.startswith("sd:")}
    return rest, sd


# hyper-parameters of the golden fixtures (must match tests/golden/gen_golden.py)
GOLDEN_MODELS = {
    "hifigan_rb1": ("hifigan", dict(resblock="1", upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4],
                                    upsample_initial_channel=64, resblock_kernel_sizes=[3, 7, 11],
                                    resblock_dilation_sizes=[[1, 3, 5]] * 3), 16),
    "hifigan_rb2": ("hifigan", dict(resblock="2", upsample_rates=[4, 4], upsample_kernel_sizes=[8, 8],
                                    upsample_initial_channel=32, resblock_kernel_sizes=[3, 5, 7],
                                    resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]), 20),
    "bigvgan_rb1": ("bigvgan", dict(resblock="1", upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4],
                                    upsample_initial_channel=64, resblock_kernel_sizes=[3, 7, 11],
                                    resblock_dilation_sizes=[[1, 3, 5]] * 3, activation="snakebeta",
                                    snake_logscale=True), 20),
    "bigvgan_rb2": ("bigvgan", dict(resblock="2", upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4],
                                    upsample_initial_channel=32, resblock_kernel_sizes=[3, 5],
                                    resblock_dilation_sizes=[[1, 2], [2, 6]], activation="snake",
                                    snake_logscale=False), 12),
}


# NSF-HiFiGAN fixture (needs f0 and cfg.preprocess.sample_rate; no per-stage hooks) — tests/golden/gen_golden.py:gen_nsfhifigan
GOLDEN_NSF = ("nsfhifigan", dict(resblock="1", harmonic_num=8, upsample_rates=[4, 2, 2], upsample_kernel_sizes=[8, 4, 4],
                                 upsample_initial_channel=64, resblock_kernel_sizes=[3, 7, 11],
                                 resblock_dilation_sizes=[[1, 3, 5]] * 3), 20)


# APNet fixture (tests/golden/gen_golden.py:gen_apnet): cfg.model.apnet and cfg.preprocess
GOLDEN_APNET = (dict(ASP_channel=32, ASP_resblock_kernel_sizes=[3, 7, 11], ASP_resblock_dilation_sizes=[[1, 3, 5]] * 3,
                     ASP_input_conv_kernel_size=7, ASP_output_conv_kernel_size=7,
                     PSP_channel=48, PSP_resblock_kernel_sizes=[3, 7], PSP_resblock_dilation_sizes=[[1, 3, 5], [1, 2, 4]],
                     PSP_input_conv_kernel_size=5, PSP_output_R_conv_kernel_size=7, PSP_output_I_conv_kernel_size=7),
                dict(n_mel=12, n_fft=64, hop_size=16, win_size=64, extract_amplitude_phase=True, sample_rate=16000))


# HiFiGAN_vits fixtures (positional constructor; tests/golden/gen_golden.py:gen_hifigan_vits)
GOLDEN_VITS = {
    "a": dict(initial_channel=24, resblock="1", resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3,
              upsample_rates=[4, 2], upsample_initial_channel=64, upsample_kernel_sizes=[8, 4], gin_channels=10),
    "b": dict(initial_channel=12, resblock="2", resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 2], [2, 6]],
              upsample_rates=[2, 2], upsample_initial_channel=32, upsample_kernel_sizes=[4, 4], gin_channels=0),
}


def load_golden_vits(tag):
    z = np.load(os.path.join(GOLDEN, "hifigan_vits.npz"))
    d = {k[len(tag) + 1:]: z[k] for k in z.files if k.startswith(tag + ":")}
    sd = {k[3:]: v for k, v in d.items() if k.startswith("sd:")}
    return {k: v for k, v in d.items() if not k.startswith("sd:")}, sd


@pytest.fixture(scope="session")
def golden_models():
    return GOLDEN_MODELS
