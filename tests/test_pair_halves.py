"""The 256-wide pair kernel (`hpair_kernel` at N = 256) on channel counts whose second column half is mostly empty.

At N = 256 the pair's second conv runs in two halves of 128 output columns, each streaming only its own weight columns
and prefetching its own residual.  C = 136 leaves one 8-column group of the second half valid, C = 200 nine; both
halves must come out bit for bit as the operand-rounded oracle (tests/resblock_oracle.py) with one-hot weights, and
within the floor with dense ones.  Channels above C are padding in every operand and must not leak into the output.
Harness and rules: test_resblock_exact.py."""
import numpy as np
import pytest

import resblock_oracle as ro
from test_resblock_exact import PRECS, VALUES, _blocks, _floor_check, _launches, _make_stage, _post

pytestmark = pytest.mark.gpu
PAIRS = 1   # resblock_fusion: one launch per pair; block mode does not serve C > 128, so every route runs pairs

# (id, C, [(k, dilations)], B, T)
ONE_HOT = [
    ("c136", 136, [(3, (1, 3, 5)), (11, (1, 3, 5))], 3, 700),
    # 4 x 49 = 196 work items at k = 3: more than the SMs of an H100 and a partial last stride
    ("c200-walk", 200, [(3, (1, 3)), (7, (1,))], 4, 6000),
    ("c136-k31-d26", 136, [(31, (26, 1))], 2, 240),   # tap reach 780: one A chunk buffer
    ("c200-T5", 200, [(5, (1, 2))], 2, 5),            # shorter than a tile
]
DENSE = [
    ("c136", 136, [(3, (1, 3, 5)), (11, (1, 3, 5))], 2, 300),
    ("c200", 200, [(3, (1, 3)), (11, (1, 5))], 2, 300),
]


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", ONE_HOT, ids=[c[0] for c in ONE_HOT])
def test_one_hot_pairs_are_exact(case, prec):
    _, C, shape, B, T = case
    scale, exps, bias_std = VALUES["ordinary"]
    rng = np.random.default_rng(C * 7 + T)
    blocks = _blocks(rng, C, shape, "one-hot", exps, bias_std)
    x = (rng.normal(0, 1, (B, C, T)) * scale).astype(np.float32)
    want = _post(ro.stage(x, blocks, PRECS[prec]))
    got, launches = _make_stage(C, blocks).run(x, prec, PAIRS)
    assert launches == _launches(C, shape, PAIRS), launches
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_pairs_within_the_floor(case, prec):
    _, C, shape, B, T = case
    rng = np.random.default_rng(C * 11 + T)
    blocks = _blocks(rng, C, shape, "dense", bias_std=0.1)
    x = rng.normal(0, 1, (B, C, T)).astype(np.float32)
    o64, o32 = (_post(ro.stage(x, blocks, PRECS[prec], acc)) for acc in ("f64", "mma"))
    got, launches = _make_stage(C, blocks).run(x, prec, PAIRS)
    assert launches == _launches(C, shape, PAIRS)
    _floor_check(f"{case[0]} {prec}", got, o64, o32)
