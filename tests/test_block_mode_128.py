"""Block mode (`hchain_kernel`, one launch per ResBlock: `resblock_fusion` 3) at 128 channels against the per-pair
launches (`hpair_kernel`, `resblock_fusion` 1).  Both run the same arithmetic in the same order, so the outputs must
be bit-equal, as the 64- and 32-channel ones are in test_pair_kernel.py.  Agreement of the two routes does not show
that either is right: test_resblock_exact.py checks each of them against the operand-rounded oracle bit for bit."""
import pytest
import torch

from helpers import build_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(model, mel, prec, fusion):
    model.precision = prec
    model.set_option("resblock_fusion", fusion)
    with torch.no_grad():
        out = model(mel.to(DEV))
    model.set_option("resblock_fusion", 2)
    return out


@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("B,T", [(2, 7000), (1, 37)])
def test_128_channel_pairs_are_bit_equal_to_block_mode(prec, B, T):
    """Stages of 128 and 64 channels, k = 3 / 7 / 11 with dilations 1, 3, 5: at 128 channels block mode's tile has
    V = 104 valid rows for k = 3 and V = 8 for k = 11.  B=2, T=7000: 14000 samples per utterance at the 128-channel
    stage, 2 x 135 = 270 k = 3 work items (more than twice the SMs of an H100, not a multiple of the grid) with a
    ragged last tile; T=37 is one ragged tile."""
    hp = dict(resblock="1", upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4], upsample_initial_channel=256,
              resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3)
    model = build_model("hifigan", hp, 80, seed=202).to(DEV)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(T))
    pairs, blocks = _run(model, mel, prec, 1), _run(model, mel, prec, 3)
    assert torch.isfinite(pairs).all()
    assert torch.equal(pairs, blocks)
