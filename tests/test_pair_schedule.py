"""`pair_schedule` of the ResBlock pair launches (`resblock_fusion` 1): the ping-pong schedule (1) of `hpair_kernel` at
128 and 64 channels gives each consumer warpgroup its own time tile with the tile geometry of the cooperative schedule
(0, the default), in which both warpgroups share one tile.  Both accumulate every output element in the same
order with the same epilogue association, so the outputs must be bit-equal.  Ping-pong runs only where a launch has
more tiles than the GPU has SMs, so every GPU case below has more than 132 (one H100) per pair launch it covers."""
import pytest
import torch

from helpers import build_model

DEV = "cuda:0"


def _hp(c0, ks, dils, rates=(2, 2)):
    return dict(resblock="1", upsample_rates=list(rates), upsample_kernel_sizes=[2 * u for u in rates],
                upsample_initial_channel=c0, resblock_kernel_sizes=list(ks), resblock_dilation_sizes=[list(d) for d in dils])


def _run(model, mel, prec, schedule):
    model.precision = prec
    model.set_option("resblock_fusion", 1)
    model.set_option("pair_schedule", schedule)
    with torch.no_grad():
        out = model(mel.to(DEV))
    model.set_option("pair_schedule", 0)
    model.set_option("resblock_fusion", 2)
    return out


def test_pair_schedule_values():
    from amphion_b200 import _capi
    model = build_model("hifigan", _hp(64, (3,), [(1,)]), 20, seed=1)
    h = model._ensure_handle()
    for v in (0, 1):
        assert _capi.lib.ab_generator_set_option(h, b"pair_schedule", v) == 0
    for v in (-1, 2):
        assert _capi.lib.ab_generator_set_option(h, b"pair_schedule", v) == -1
        assert "pair_schedule" in _capi.last_error()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["tc_f16", "tc_bf16"])
@pytest.mark.parametrize("c0,ks,dils,B,T", [
    # C = 128 and 64, k = 3 / 7 / 11 at dilations 1, 3, 5: 570-612 tiles per launch, the last tile of each utterance
    # ragged
    (256, (3, 7, 11), [(1, 3, 5)] * 3, 6, 6000),
    # 300 utterances shorter than one tile: 300 items, so 36 CTAs of 132 walk an odd number and warpgroup 1 has
    # nothing in their last round
    (256, (3, 11), [(1, 3), (5, 1)], 300, 20),
    # C = 128, k = 31 at dilation 70: two intermediate tiles do not fit next to the A chunk, so this launch falls back
    # to the cooperative schedule (180 tiles); C = 64, k = 3 still ping-pongs
    (256, (31, 3), [(70, 1), (1, 3)], 20, 400),
])
def test_ping_pong_is_bit_equal_to_cooperative(prec, c0, ks, dils, B, T):
    model = build_model("hifigan", _hp(c0, ks, dils), 80, seed=11).to(DEV)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(B + T))
    coop, ping = _run(model, mel, prec, 0), _run(model, mel, prec, 1)
    assert torch.isfinite(ping).all()
    assert torch.equal(ping, coop)
