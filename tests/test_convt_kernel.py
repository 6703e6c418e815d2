"""ConvTranspose1d launches.  From an operand image they run on `hitem_kernel`: persistent CTAs over (utterance, time
tile, N block) work items and the polyphase epilogue with 16-byte operand-image stores.  The single-layer cases go
through `ab_conv_transpose1d_forward`, whose fp32 input runs on `hconv_kernel`; the generators exercise conv_pre's
operand image and the image-in, image-out ConvTranspose layers of HiFi-GAN at strides 8 and 2.  test_tc_conv_exact.py
launches both kernels directly and checks every epilogue specialisation and the operand images bit for bit."""
import numpy as np
import pytest
import torch

from helpers import build_model, sd_numpy
from oracle import generator as og
from test_gpu_parity import oracle_conv_transpose1d, run_conv_transpose1d

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"tc_f16": 1e-3, "tc_bf16": 4e-3}


@pytest.mark.parametrize("case", [
    (1, 1536, 768, 40, 8, 4),    # BigVGAN-large stage 0: 12 N blocks, 48 K chunks
    (40, 512, 256, 70, 16, 8),   # 40 x 1 x 8 = 320 work items: more than twice the SMs, a partial last stride
])
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_convt_matches_operand_rounded_oracle(case, prec):
    got = run_conv_transpose1d(case, 0.1, prec)[0]
    assert np.isfinite(got).all()          # every output element written exactly once (buffer pre-filled with NaN)
    dt = torch.float16 if prec == "tc_f16" else torch.bfloat16
    np.testing.assert_allclose(got, oracle_conv_transpose1d(case, 0.1, dt), atol=3e-5, rtol=1e-5)


def _hp(rates, c0):
    return dict(resblock="1", upsample_rates=list(rates), upsample_kernel_sizes=[2 * u for u in rates],
                upsample_initial_channel=c0, resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3], [1, 3]])


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_convt_walk_does_not_depend_on_the_batch(prec):
    """300 utterances through a generator whose stage 0 is a 256 -> 128, u = 8 ConvTranspose from conv_pre's operand
    image: 300 x 1 tile x 4 N blocks = 1,200 work items.  Each utterance must come out bit-equal to the same utterance
    in a batch of 7, which gives a different grid and walk."""
    hp = _hp((8, 2), 256)
    model = build_model("hifigan", hp, 20, seed=5).to(DEV)
    model.precision = prec
    mel = torch.randn(300, 20, 64, generator=torch.Generator().manual_seed(11)).to(DEV)
    with torch.no_grad():
        full = model(mel)
        assert torch.isfinite(full).all()
        for i in range(0, 300, 7):
            assert torch.equal(model(mel[i:i + 7]), full[i:i + 7]), i


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("rates", [(8, 2), (2, 8)])
def test_hifigan_convt_stages_match_the_oracle(prec, rates):
    """128 -> 64 -> 32 channels: conv_pre emits the operand image of lrelu(x, 0.1) that stage 0's ConvTranspose reads,
    and each ConvTranspose emits the image its ResBlocks read, at u = 8 (no exchange) and u = 2 (quad transpose,
    odd padding)."""
    hp = _hp(rates, 128)
    model = build_model("hifigan", hp, 20, seed=17).to(DEV)
    mel = torch.randn(2, 20, 90, generator=torch.Generator().manual_seed(3))
    model.precision = prec
    with torch.no_grad():
        got = model(mel.to(DEV)).cpu().numpy()
    want = og.generator_forward("hifigan", sd_numpy(model), hp, mel.numpy())
    err = float(np.abs(got - want).max())
    assert err <= TOL[prec], err
