"""The codec's Snake1d kernel (`snake1d_kernel`, models/codec/amphion_codec/codec.py:32-48) one launch at a time through
ab_snake1d_forward, against a restatement of its rounding order in numpy float32:

    u = fl(alpha x);  s = sinf(u);  r = fl(1 / fl(alpha + 1e-9));  y = fl(x + fl(r fl(s s)))

sinf is taken as an interval: CUDA's sinf is within 2 ulp of sin, so s is one of the five float32 values within two
steps of the correctly rounded sin(u), and y must equal the restatement at one of them, bit for bit (the same for
every element of an fp32 output and of its 16-bit operand image).  The image is the saturating round to nearest of y:
past 65504 an f16 element holds 65504, and inf (alpha = -1e-9 makes alpha + 1e-9 exactly 0) the largest finite value.
Cases: C = 12 (padding channels in the image), 96 and 1536; T = 1, 17 and 333; alphas of both signs, small alphas
where the 1e-9 matters, alpha = 0 and alpha = -1e-9 (whose inf / NaN the reference formula gives on the CPU too); inputs
with alpha x = 0 exactly.  Outputs are pre-filled with NaN / 0xFFFF, so an unwritten element shows."""
import numpy as np
import pytest
import torch

DEV = "cuda:0"
F16, BF16 = 1, 2


def _capi():
    from amphion_b200 import _capi
    return _capi


def _case(C, T, B=2, seed=0):
    rng = np.random.default_rng(seed + 7 * C + T)
    alpha = (rng.uniform(0.2, 2.0, C) * np.where(rng.random(C) < 0.35, -1.0, 1.0)).astype(np.float32)
    special = np.array([0.0, -1e-9, 1e-9, 1e-3, -1e-4, 0.0123, 3e-2, 7.5], np.float32)
    alpha[:min(C, special.size)] = special[:min(C, special.size)]
    x = (rng.standard_normal((B, C, T)) * 3.0).astype(np.float32)
    x[:, :, ::5] = 0.0                                   # alpha x = 0 exactly
    x[0, :, -1] = 1e5                                    # past f16's largest finite value
    x[-1, :, 0] = -7e4
    return x, alpha


def _reference(x, alpha):
    """codec.py's formula in numpy float32 (no FMA): the inf / NaN it gives at alpha = -1e-9 included."""
    a = alpha.reshape(1, -1, 1)
    with np.errstate(all="ignore"):
        r = np.float32(1.0) / (a + np.float32(1e-9))
        s = np.sin(a * x)
        return x + r * (s * s)


def _candidates(x, alpha):
    """The restated y at each of the five sinf candidates, [5, B, C, T] float32."""
    a = alpha.reshape(1, -1, 1)
    with np.errstate(all="ignore"):
        u = (a * x).astype(np.float32)
        s0 = np.sin(u.astype(np.float64)).astype(np.float32)
        r = (np.float32(1.0) / (a + np.float32(1e-9))).astype(np.float32)
        outs = []
        for k in (-2, -1, 0, 1, 2):
            s = s0
            for _ in range(abs(k)):
                s = np.nextafter(s, np.float32(np.sign(k) * np.inf)).astype(np.float32)
            outs.append((x + (r * (s * s)).astype(np.float32)).astype(np.float32))
    return np.stack(outs)


def _same(a, b):
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


def _image_of(y, bf16):
    """Saturating round to nearest of y to f16 / bf16, as uint16 [B, C, T]; NaN stays NaN."""
    t = torch.from_numpy(np.ascontiguousarray(y))
    mx = torch.finfo(torch.bfloat16 if bf16 else torch.float16).max
    t = torch.where(torch.isnan(t), t, t.clamp(-mx, mx))
    return t.to(torch.bfloat16 if bf16 else torch.float16).view(torch.int16).numpy().view(np.uint16)


def _launch(x, alpha, want_y, prec):
    cap = _capi()
    B, C, T = x.shape
    xd = torch.from_numpy(x).to(DEV)
    ad = torch.from_numpy(alpha).to(DEV)
    y = torch.full((B, C, T), float("nan"), device=DEV) if want_y else None
    img = torch.full((B, (C + 15) // 16 * 2, T, 8), -1, dtype=torch.int16, device=DEV) if prec else None
    cap.check(cap.lib.ab_snake1d_forward(cap.ptr(xd), cap.ptr(y), cap.ptr(img), B, C, T, cap.ptr(ad), prec,
                                         cap.stream_ptr()), "ab_snake1d_forward")
    torch.cuda.synchronize()
    return (None if y is None else y.cpu().numpy()), (None if img is None else img.cpu().numpy().view(np.uint16))


def _unpack(img, C):
    """[B, C8, T, 8] -> [B, C8 * 8, T]"""
    B, c8n, T, _ = img.shape
    return img.transpose(0, 1, 3, 2).reshape(B, c8n * 8, T)


def test_reference_formula_gives_inf_and_nan_at_alpha_minus_1e9():
    x, alpha = _case(12, 17)
    y = _reference(x, alpha)
    assert np.isinf(y[:, 1, 1:4]).all()           # alpha + 1e-9 == 0: 1 / 0 times sin^2 > 0
    assert np.isnan(y[0, 1, 5])                   # and times sin(0)^2 = 0
    cand = _candidates(x, alpha)
    # numpy's float32 sin is not CUDA's: the restatement holds the formula's value for nearly every element, and
    # its inf / NaN at alpha = -1e-9 for every one
    assert _same(cand, y[None]).any(0).mean() > 0.999
    assert _same(cand, y[None]).any(0)[:, 1].all()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [12, 96, 1536])
@pytest.mark.parametrize("T", [1, 17, 333])
def test_snake1d_is_exact(C, T):
    x, alpha = _case(C, T)
    cand = _candidates(x, alpha)
    y32, _ = _launch(x, alpha, True, 0)
    hit = _same(cand, y32[None])
    assert hit.any(0).all(), f"{int((~hit.any(0)).sum())} fp32 outputs outside the sinf interval"
    ref = _reference(x, alpha)
    assert (np.isinf(y32) == np.isinf(ref)).all() and (np.isnan(y32) == np.isnan(ref)).all()
    for prec, bf16 in ((F16, False), (BF16, True)):
        for want_y in (False, True):
            y, img = _launch(x, alpha, want_y, prec)
            if want_y:
                assert _same(y, y32).all(), "y differs between launch modes"
            full = _unpack(img, C)
            assert (full[:, C:] == 0).all(), "padding channels not zero"
            got = full[:, :C]
            exp = _image_of(y32, bf16)
            nan = np.isnan(y32)
            assert (got[~nan] == exp[~nan]).all(), f"{int((got[~nan] != exp[~nan]).sum())} image elements differ"
            assert np.isnan(torch.from_numpy(got[nan].view(np.int16)).view(
                torch.bfloat16 if bf16 else torch.float16).float().numpy()).all()
    if C >= 12:   # f16 saturation: x = 1e5 / -7e4 hold +-65504, inf the largest finite value
        _, img = _launch(x, alpha, False, F16)
        got = _unpack(img, C)[:, :C]
        assert (got[0, 8:, -1] == 0x7BFF).all() and (got[-1, 8:, 0] == 0xFBFF).all()
        assert (got[:, 1, 1:][np.isposinf(y32[:, 1, 1:])] == 0x7BFF).all()


def test_entry_point_refuses_malformed_requests():
    cap = _capi()
    p = cap.ptr
    dummy = torch.zeros(4)
    assert cap.lib.ab_snake1d_forward(p(None), p(dummy), p(None), 1, 1, 1, p(dummy), 0, None) != 0
    assert cap.lib.ab_snake1d_forward(p(dummy), p(None), p(None), 1, 1, 1, p(dummy), 0, None) != 0
    assert cap.lib.ab_snake1d_forward(p(dummy), p(None), p(dummy), 1, 1, 1, p(dummy), 0, None) != 0   # image at fp32
    assert cap.lib.ab_snake1d_forward(p(dummy), p(dummy), p(None), 1, 1, 1, p(dummy), 7, None) != 0
    assert cap.lib.ab_snake1d_forward(p(dummy), p(dummy), p(None), 0, 1, 1, p(dummy), 0, None) != 0
