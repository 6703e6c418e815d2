"""ResBlock pair launches (`hpair_kernel`, one launch per dilation pair: `resblock_fusion` 1) on small HiFi-GAN
generators.  Each case is checked against whole-block launches (`resblock_fusion` 3) bit for bit where block mode
serves the stage (C <= 64), and against the CPU oracle where it does not.  The bars here are whole-generator ones;
the bit-level check of every route at every width (N = 128 and 256 included) is test_resblock_exact.py, which
compares single stages with one-hot weights against the operand-rounded oracle exactly.  A change of the fp32
accumulation order alone passes both.  Every generator has at least two stages
and two ResBlock kernel sizes, so the branch sum (`acc_prev` aliasing `y`) and the operand image a stage emits for
the next one are exercised."""
import numpy as np
import pytest
import torch

from helpers import build_model, sd_numpy
from oracle import generator as og

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"tc_f16": 1e-3, "tc_bf16": 4e-3}


def _hp(c0, ks, dils, rates=(2, 2)):
    return dict(resblock="1", upsample_rates=list(rates), upsample_kernel_sizes=[2 * u for u in rates],
                upsample_initial_channel=c0, resblock_kernel_sizes=list(ks), resblock_dilation_sizes=[list(d) for d in dils])


def _run(model, mel, prec, fusion):
    model.precision = prec
    model.set_option("resblock_fusion", fusion)
    with torch.no_grad():
        out = model(mel.to(DEV))
    model.set_option("resblock_fusion", 2)
    return out


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("B,T", [(6, 6000), (2, 45), (1, 20)])
def test_pair_launches_are_bit_equal_to_block_mode(prec, B, T):
    """Stages of 64 and 32 channels, k = 3 / 7 / 11 with dilations 1, 3, 5.  B=6, T=6000: the 64-channel k=3 pairs
    have 6 x 48 = 288 work items, more than twice the SMs of an H100 and not a multiple of the grid, with a ragged last
    tile; T=45 and T=20 are shorter than one tile."""
    hp = _hp(128, (3, 7, 11), [(1, 3, 5)] * 3)
    model = build_model("hifigan", hp, 80, seed=101).to(DEV)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(T))
    pairs, blocks = _run(model, mel, prec, 1), _run(model, mel, prec, 3)
    assert torch.isfinite(pairs).all()
    assert torch.equal(pairs, blocks)


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("c0,ks,dils,T", [
    (512, (3, 11), [(1, 3, 5), (1, 3, 5)], 150),   # C = 256 and 128, several tiles per utterance
    (512, (31, 3), [(1, 5), (2, 3)], 40),           # k = 31 at dilation 5: V = 98 rows at N = 256
    (192, (3, 11), [(1, 3, 5), (1, 5)], 70),        # C = 96 and 48: N block 128 and 64, padded
    (400, (7, 31), [(1, 4), (5, 1)], 33),           # C = 200 and 100: padded N, a partial last K chunk
    (512, (31, 3), [(26, 1), (1, 3)], 60),          # tap reach 780 at N = 256: one A chunk buffer fits
])
def test_pair_launches_match_the_oracle(prec, c0, ks, dils, T):
    hp = _hp(c0, ks, dils)
    model = build_model("hifigan", hp, 20, seed=7).to(DEV)
    mel = torch.randn(2, 20, T, generator=torch.Generator().manual_seed(c0 + T))
    want = og.generator_forward("hifigan", sd_numpy(model), hp, mel.numpy())
    got = _run(model, mel, prec, 1).cpu().numpy()
    err = float(np.abs(got - want).max())
    assert err <= TOL[prec], err


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
def test_pair_launch_walk_does_not_depend_on_the_batch(prec):
    """C = 256 and 128 at 300 utterances: the 256-channel pairs have 600 work items, so every CTA of the persistent
    grid walks several and the last stride is partial.  Each utterance must come out bit-equal to the same utterance
    run in a batch of 7 (a different grid and walk), and two of them must match the oracle."""
    hp = _hp(512, (3, 11), [(1, 3), (1, 5)])
    model = build_model("hifigan", hp, 20, seed=3).to(DEV)
    mel = torch.randn(300, 20, 64, generator=torch.Generator().manual_seed(5))
    full = _run(model, mel, prec, 1)
    for i in range(0, 300, 7):
        part = _run(model, mel[i:i + 7], prec, 1)
        assert torch.equal(part, full[i:i + 7]), i
    want = og.generator_forward("hifigan", sd_numpy(model), hp, mel[[0, 299]].numpy())
    err = float(np.abs(full[[0, 299]].cpu().numpy() - want).max())
    assert err <= TOL[prec], err
