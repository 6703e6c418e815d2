"""`activation1d_warp_kernel` (the anti-aliased Snake / SnakeBeta) against the kernel-order oracle
(tests/activation1d_exact_oracle.py), one launch at a time: MODE 0 through ab_activation1d_forward (taps read from
global memory), MODE 1 and MODE 2 through ab_activation1d_packed_forward (taps packed on the host, the generator's
launch; MODE 2 is the image-only launch at 16 bits, with the short snake).

The 2x-rate signal is read out through one-hot taps: f_down = e_5 (then e_6) makes y[t] = v[2t] (v[2t + 1]) exactly,
so every v[i], i in [0, 2T), is visible.
* alpha = 0 makes v = u: the up-FIR bit for bit (MODE 0 / 1; MODE 2 through the image), with Kaiser taps and with
  one-hot f_up taps, one launch per tap, which pins each tap's place in the packed pairs and the replicate window.
* alpha != 0: v lies in the oracle's snake interval (CUDA's __sinf bound; expf's 2 ulp under logscale), with |u a| up
  to ~1e3 at fp32, where a dropped Cody-Waite low constant shows, and up to ~1e4 for MODE 2's image under the
  sin.approx phase bound.
* The down-FIR on the Kaiser taps: y equals the oracle's kernel-order down-FIR of the v read out with the same x,
  alpha and beta (v does not depend on f_down), bit for bit.
* MODE 0 and MODE 1 give the same bits; x offset by one float (every segment on the edge path) gives the aligned
  run's bits; at 16 bits MODE 1's y with the image equals its y alone, and the image is rnd(y).
Shapes hit every seam: T around the 120-output segments and the 960-output CTAs (248 is the first T whose segment 1
is FAST; every T mod 4), C around the 8- and 16-channel groups, B = 3.  Outputs start as NaN (images 0xFFFF), every
input is followed by NaN, so an unwritten element or a read past an input shows."""
import ctypes as C

import numpy as np
import pytest
import torch

import activation1d_exact_oracle as ao
from conftest import load_golden

DEV = "cuda:0"
GUARD = 1024
TS = [1, 2, 3, 5, 7, 8, 9, 121, 247, 248, 249, 959, 960, 961, 1088, 2884]
CS = [1, 7, 8, 9, 16, 17, 24, 33]
VARIANTS = [("snakebeta", True), ("snake", False), ("snakebeta", False), ("snake", True)]
CASES = [(T, CS[n % len(CS)], *VARIANTS[n % len(VARIANTS)]) for n, T in enumerate(TS)]
GAMMA7 = 7 * 2.0 ** -24 / (1 - 7 * 2.0 ** -24)      # the FMA-chain / pair-sum error bound of up to 7 roundings


def _lib():
    from amphion_b200 import _capi
    return _capi


def _kaiser():
    from amphion_b200.vocoders.activations import DownSample1d, UpSample1d
    return (UpSample1d(12, 2).filter.reshape(-1).numpy().astype(np.float32),
            DownSample1d(2, 12).lowpass.filter.reshape(-1).numpy().astype(np.float32))


def _one_hot(j, value=1.0):
    f = np.zeros(12, np.float32)
    f[j] = value
    return f


# ------------------------------------------------------------------------------------------------ CPU: the oracle
def _up64(x, f_up):
    """UpSample1d in float64 (resample.py:36-45): replicate pad 5, conv_transpose1d stride 2 of 2 f, crop 15."""
    xt = torch.from_numpy(np.asarray(x, np.float64))
    B, Cn, T = xt.shape
    xp = torch.nn.functional.pad(xt, (5, 5), mode="replicate")
    w = (2.0 * torch.from_numpy(np.asarray(f_up, np.float64))).view(1, 1, 12).expand(Cn, 1, 12)
    return torch.nn.functional.conv_transpose1d(xp, w, stride=2, groups=Cn)[..., 15:15 + 2 * T].numpy()


def _down64(v, f_down):
    """DownSample1d in float64 (filter.py:92-99): replicate pad 5 / 6, conv1d stride 2."""
    vt = torch.from_numpy(np.asarray(v, np.float64))
    Cn = vt.shape[1]
    w = torch.from_numpy(np.asarray(f_down, np.float64)).view(1, 1, 12).expand(Cn, 1, 12)
    return torch.nn.functional.conv1d(torch.nn.functional.pad(vt, (5, 6), mode="replicate"), w, stride=2,
                                      groups=Cn).numpy()


def _abs_up(x, f_up):
    return _up64(np.abs(x), np.abs(f_up))


@pytest.mark.parametrize("T", [1, 2, 3, 8, 9, 247, 249, 961])
def test_up_and_down_fir_within_reassociation_bound(T):
    rng = np.random.default_rng(T)
    f_up, f_down = _kaiser()
    x = rng.standard_normal((2, 3, T)).astype(np.float32)
    u = ao.up(x, f_up)
    u64 = _up64(x, f_up)
    assert (np.abs(u - u64) <= GAMMA7 * _abs_up(x, f_up) + 1e-300).all()
    y, y64 = ao.down(u, f_down), _down64(u.astype(np.float64), f_down)
    assert (np.abs(y - y64) <= GAMMA7 * _down64(np.abs(u).astype(np.float64), np.abs(f_down)) + 1e-300).all()


@pytest.mark.parametrize("T", [1, 5, 8, 121, 247, 248, 249, 960, 961, 1088])
def test_up_fir_depends_on_index_and_length_only(T):
    """Every segment the kernel runs computes the same u[i]: the (i, T) rule of `up` restated segment by segment."""
    rng = np.random.default_rng(100 + T)
    f_up, _ = _kaiser()
    x = rng.standard_normal((1, 2, T)).astype(np.float32)
    u = ao.up(x, f_up)
    seen = ao.up_by_segments(x, f_up)
    assert {i for _, i in seen} == set(range(2 * T))
    for (t0, i), val in seen.items():
        assert (val.view(np.uint32) == u[..., i].view(np.uint32)).all(), (t0, i)


def test_packed_pairs_place_every_tap():
    """pack_snake_coef's documented order: with f_up = e_k, the pair form of each group offset gives the float64
    UpSample1d exactly (one product per output), and the zero-padded ce_b / co_b taps contribute nothing."""
    rng = np.random.default_rng(7)
    T = 64
    x = rng.standard_normal((1, 1, T)).astype(np.float32)
    i = np.arange(2 * T)
    i = i[ao.pair_group(i, T)]
    kc = ao.pack(np.arange(12, dtype=np.float32), np.arange(12, dtype=np.float32))
    assert kc["ce_b"][0, 0] == 0 and kc["co_b"][0, 0] == 0 and kc["ce_b"][3, 1] == 0 and kc["co_b"][3, 1] == 0
    assert kc["fd2"].reshape(-1).tolist() == list(range(12))
    for k in range(12):
        f = _one_hot(k, 0.25)
        got = ao.up_pair(x, i, ao.pack(f, f))
        assert (got == _up64(x, f)[..., i]).all(), k
        assert (ao.up_scalar(x, i, f) == got).all(), k


def test_oracle_on_the_reference_fixture():
    """The oracle on tests/golden/activation1d.npz's input, within the first-order error bound of the fixture's y."""
    g, _ = load_golden("activation1d")
    x, f_up, f_down = g["x"], g["f_up"].reshape(-1), g["f_down"].reshape(-1)
    y = ao.activation1d(x, g["alpha"], g["beta"], True, f_up, f_down)
    a = np.exp(g["alpha"].astype(np.float64))[None, :, None]
    ib = 1.0 / (np.exp(g["beta"].astype(np.float64)) + 1e-9)[None, :, None]
    u64 = _up64(x, f_up)
    v64 = u64 + ib * np.sin(u64 * a) ** 2
    e = 16 * 2.0 ** -24
    bu = e * _abs_up(x, f_up)                                          # both sides' up-FIR roundings
    bv = (1 + ib * a) * bu + e * (np.abs(v64) + ib) + ib * 2 * np.abs(u64 * a) * e + ib * ao.SINF_ERR * 2
    by = _down64(bv, np.abs(f_down)) + e * _down64(np.abs(v64), np.abs(f_down))
    assert (np.abs(y - g["y"]) <= 2 * by).all()
    assert (np.abs(y - _down64(v64, f_down)) <= by).all()


def test_snake_interval_contains_the_float64_snake():
    rng = np.random.default_rng(3)
    u = (rng.standard_normal((2, 4, 500)) * 4).astype(np.float32)
    a, invb = ao.channel_params(np.log([0.5, 3.0, 200.0, 900.0]), np.log([0.3, 1.0, 2.0, 5.0]), True)
    for c in range(a.shape[1]):
        lo, hi = ao.snake_interval(u, a[:, c], invb[:, c])
        v64 = u + invb[None, :, c, None].astype(np.float64) * np.sin(u.astype(np.float64) * a[None, :, c, None]) ** 2
        assert ((lo <= v64 + 1e-5 * np.abs(u)) & (v64 - 1e-5 * np.abs(u) <= hi)).all()
        mid = ao.snake_mid(u, a[:, c], invb[:, c])
        assert ((lo <= mid) & (mid <= hi)).all()
        assert (hi - lo).max() < 5e-6 * (1 + np.abs(u).max())


def test_entry_point_refuses_malformed_requests():
    """AB_ERR_ARG / AB_ERR_UNSUPPORTED before any launch (the pointers are never dereferenced)."""
    capi = _lib()
    P = C.c_void_p
    a = P(256)
    taps = (C.c_float * 12)()
    f16, fp32 = capi.PRECISIONS["tc_f16"], capi.PRECISIONS["fp32"]

    def call(x=a, y=a, img=None, B=2, C_=8, T=16, prec=fp32, fu=taps, fd=taps):
        return capi.lib.ab_activation1d_packed_forward(x, y, img, B, C_, T, a, a, 1, fu, fd, prec, None)

    assert call(x=None) == -1 and "null" in capi.last_error()
    assert call(fu=None) == -1
    assert call(y=None) == -1 and "output" in capi.last_error()
    assert call(img=a, prec=fp32) == -1 and "image" in capi.last_error()
    assert call(y=None, img=a, prec=fp32) == -1
    assert call(prec=7) == -1 and "precision" in capi.last_error()
    assert call(B=0) == -1 and call(C_=0) == -1 and call(T=0) == -1
    assert call(C_=65535 * 8 + 1, prec=f16) == -2
    assert call(T=(1 << 30) + 1) == -2


# ------------------------------------------------------------------------------------------------ the harness
def _guarded(a, offset=0):
    """fp32 numpy -> (buffer, pointer): offset NaNs, a, then GUARD NaNs."""
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.full((offset + a.size + GUARD,), float("nan"), device=DEV)
    buf[offset:offset + a.size] = torch.from_numpy(a.reshape(-1)).to(DEV)
    return buf, C.c_void_p(buf.data_ptr() + 4 * offset)


def _run(x, alpha, beta, logscale, f_up, f_down, *, api="packed", prec="fp32", y=True, img=False, offset=0):
    """One launch -> (rc, y or None, image bits or None).  api "forward": ab_activation1d_forward (MODE 0);
    "packed": ab_activation1d_packed_forward (MODE 1, MODE 2 when img without y at 16 bits).  beta None: Snake (beta
    is alpha's buffer)."""
    capi = _lib()
    B, Cn, T = x.shape
    xb, xp = _guarded(x, offset)
    ab, ap = _guarded(alpha)
    bb, bp = (ab, ap) if beta is None else _guarded(beta)
    yd = torch.full((B, Cn, T), float("nan"), device=DEV) if y else None
    im = torch.full((B, (Cn + 15) // 16 * 2, T, 8), -1, dtype=torch.int16, device=DEV) if img else None
    if api == "forward":
        fu, fdn = _guarded(f_up)[0], _guarded(f_down)[0]
        rc = capi.lib.ab_activation1d_forward(xp, capi.ptr(yd), B, Cn, T, ap, bp, int(logscale), capi.ptr(fu),
                                              capi.ptr(fdn), capi.stream_ptr())
    else:
        fu = (C.c_float * 12)(*np.asarray(f_up, np.float32).tolist())
        fdn = (C.c_float * 12)(*np.asarray(f_down, np.float32).tolist())
        rc = capi.lib.ab_activation1d_packed_forward(xp, capi.ptr(yd), capi.ptr(im), B, Cn, T, ap, bp, int(logscale),
                                                     fu, fdn, capi.PRECISIONS[prec], capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, capi.last_error()
    for buf, n in ((xb, x.size), (ab, alpha.size)):
        assert torch.isnan(buf[offset + n if buf is xb else n:]).all(), "an input was written"
    return (yd.cpu().numpy() if y else None), (im.cpu().numpy().view(np.uint16) if img else None)


def _readout(x, alpha, beta, logscale, f_up, **kw):
    """v [B, C, 2T] through f_down = e_5, then e_6 (y or the image, as kw asks) -> (v, vimg bits or None)."""
    outs = [_run(x, alpha, beta, logscale, f_up, _one_hot(j), **kw) for j in (5, 6)]
    B, Cn, T = x.shape
    v = vimg = None
    if outs[0][0] is not None:
        v = np.empty((B, Cn, 2 * T), np.float32)
        v[..., 0::2], v[..., 1::2] = outs[0][0], outs[1][0]
    if outs[0][1] is not None:
        vimg = np.empty(outs[0][1].shape[:2] + (2 * T, 8), np.uint16)
        vimg[:, :, 0::2], vimg[:, :, 1::2] = outs[0][1], outs[1][1]
    return v, vimg


def _no_snake(u):
    """v at a = 0: fma(invb, +0, u) = u, except that -0 becomes +0."""
    return (u + np.float32(0)).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _assert_equal(what, got, want):
    bad = _bits(got) != _bits(want)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


def _assert_img(what, got, want):
    bad = np.asarray(got) != np.asarray(want)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{hex(got[bad][0])} vs {hex(want[bad][0])}")


def _img_values(bits, prec, C):
    """image bits [B][c8][T][8] -> fp32 [B, C, T]"""
    B, c8n, T, _ = bits.shape
    full = bits.transpose(0, 1, 3, 2).reshape(B, c8n * 8, T)[:, :C]
    if prec == "f16":
        return full.view(np.float16).astype(np.float32)
    return (full.astype(np.uint32) << 16).view(np.float32)


def _params(rng, Cn, kind, logscale, amax):
    """alpha, beta (None for Snake) with |a| spread up to amax and, for SnakeBeta, b in [0.3, 3]."""
    mag = np.exp(rng.uniform(np.log(0.5), np.log(amax), Cn))
    if logscale:
        alpha = np.log(mag).astype(np.float32)
        beta = np.log(rng.uniform(0.3, 3.0, Cn)).astype(np.float32)
    else:
        alpha = (mag * rng.choice([-1, 1], Cn)).astype(np.float32)
        beta = rng.uniform(0.3, 3.0, Cn).astype(np.float32)
    return alpha, (beta if kind == "snakebeta" else None)


def _assert_snake(what, v, u, alpha, beta, logscale, img_prec=None):
    """Every channel's v lies in the oracle's interval for one of the kernel's candidate (a, invb).  img_prec: v is
    MODE 2's image ("f16" / "bf16"), the pair groups take the short snake's interval, all of it rounded."""
    fast = ao.pair_group(np.arange(u.shape[-1]), u.shape[-1] // 2) if img_prec else None
    a_c, ib_c = ao.channel_params(alpha, alpha if beta is None else beta, logscale)
    for c in range(v.shape[1]):
        ok = False
        for a in a_c[c]:
            for ib in ib_c[c]:
                lo, hi = ao.snake_interval(u[:, c:c + 1], a[None], ib[None])
                if fast is not None:
                    flo, fhi = ao.snake_interval(u[:, c:c + 1], a[None], ib[None], fast=True)
                    lo, hi = np.where(fast, flo, lo), np.where(fast, fhi, hi)
                    lo, hi = ao.rnd(lo, img_prec), ao.rnd(hi, img_prec)
                if ((lo <= v[:, c:c + 1]) & (v[:, c:c + 1] <= hi)).all():
                    ok = True
                    break
            if ok:
                break
        if not ok:
            lo, hi = ao.snake_interval(u[:, c:c + 1], a_c[c, a_c.shape[1] // 2][None], ib_c[c, ib_c.shape[1] // 2][None])
            bad = ~((lo <= v[:, c:c + 1]) & (v[:, c:c + 1] <= hi))
            n = np.argwhere(bad)[0]
            pytest.fail(f"{what}: channel {c}: {int(bad.sum())} of {bad.size} outside, first at {n.tolist()}: "
                        f"{v[:, c:c + 1][tuple(n)]!r} not in [{lo[tuple(n)]!r}, {hi[tuple(n)]!r}] "
                        f"(u = {u[:, c:c + 1][tuple(n)]!r}, a = {a_c[c].tolist()}, invb = {ib_c[c].tolist()})")



# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("T,Cn,kind,logscale", CASES)
def test_activation1d_is_exact(T, Cn, kind, logscale):
    rng = np.random.default_rng(T * 64 + Cn)
    B = 3
    f_up, f_down = _kaiser()
    prec = "f16" if T % 2 else "bf16"
    tc = "tc_" + prec
    x = rng.standard_normal((B, Cn, T)).astype(np.float32)
    zero = np.full(Cn, -np.inf if logscale else 0.0, np.float32)       # a = 0
    beta0 = None if kind == "snake" else rng.uniform(0.3, 3.0, Cn).astype(np.float32)
    u = ao.up(x, f_up)
    v0 = _no_snake(u)
    ys_want = ao.down(v0, f_down)

    # the up-FIR, bit for bit (alpha = 0: v = u), MODE 0, 1 and 2
    for api in ("forward", "packed"):
        v, _ = _readout(x, zero, beta0, logscale, f_up, api=api)
        _assert_equal(f"up-FIR {api}", v, _interleave(ao.down(v0, _one_hot(5)), ao.down(v0, _one_hot(6))))
    _, vimg = _readout(x, zero, beta0, logscale, f_up, prec=tc, y=False, img=True)
    _assert_img(f"up-FIR MODE 2 {prec}", vimg,
                _interleave_img(ao.image(ao.down(v0, _one_hot(5)), prec), ao.image(ao.down(v0, _one_hot(6)), prec)))

    # the down-FIR on real taps at alpha = 0: MODE 0 / 1 y and MODE 2's image
    y0 = _run(x, zero, beta0, logscale, f_up, f_down, api="forward")[0]
    _assert_equal("down-FIR MODE 0, alpha = 0", y0, ys_want)
    _assert_img(f"MODE 2 image {prec}, alpha = 0",
                _run(x, zero, beta0, logscale, f_up, f_down, prec=tc, y=False, img=True)[1], ao.image(ys_want, prec))

    # the snake: |u a| up to ~1e3 (fp32)
    alpha, beta = _params(rng, Cn, kind, logscale, 300.0)
    v, _ = _readout(x, alpha, beta, logscale, f_up)
    _assert_snake("snake MODE 1", v, u, alpha, beta, logscale)
    v0, _ = _readout(x, alpha, beta, logscale, f_up, api="forward")
    _assert_equal("v: MODE 0 vs MODE 1", v0, v)

    # the down-FIR on real taps: y is the kernel-order down-FIR of the v read out above
    y1 = _run(x, alpha, beta, logscale, f_up, f_down)[0]
    _assert_equal("down-FIR MODE 1", y1, ao.down(v, f_down))
    _assert_equal("MODE 0 vs MODE 1", _run(x, alpha, beta, logscale, f_up, f_down, api="forward")[0], y1)
    _assert_equal("x offset by one float (edge path everywhere)",
                  _run(x, alpha, beta, logscale, f_up, f_down, offset=1)[0], y1)
    yb, ib = _run(x, alpha, beta, logscale, f_up, f_down, prec=tc, y=True, img=True)
    _assert_equal(f"MODE 1 y with the {prec} image", yb, y1)
    _assert_img(f"MODE 1 {prec} image", ib, ao.image(y1, prec))

    # MODE 2: the short snake on the pair groups, |u a| up to ~1e4, through the image
    alpha, beta = _params(rng, Cn, kind, logscale, 3000.0)
    _, vimg = _readout(x, alpha, beta, logscale, f_up, prec=tc, y=False, img=True)
    _assert_snake(f"snake MODE 2 {prec}", _img_values(vimg, prec, Cn), u, alpha, beta, logscale, img_prec=prec)
    pad = vimg.transpose(0, 1, 3, 2).reshape(B, -1, 2 * T)[:, Cn:]
    assert (pad == 0).all(), "padding channels of the image"


def _interleave(even, odd):
    v = np.empty(even.shape[:-1] + (2 * even.shape[-1],), np.float32)
    v[..., 0::2], v[..., 1::2] = even, odd
    return v


def _interleave_img(even, odd):
    v = np.empty(even.shape[:2] + (2 * even.shape[2], 8), np.uint16)
    v[:, :, 0::2], v[:, :, 1::2] = even, odd
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("T,Cn", [(9, 3), (247, 9), (961, 17), (1088, 8)])
def test_one_hot_up_taps(T, Cn):
    """f_up = e_k, k = 0..11, read out through f_down = e_5 / e_6: each tap's place in the packed pairs (MODE 1) and in
    the taps MODE 0 reads, and the replicate window, bit for bit."""
    rng = np.random.default_rng(T)
    x = rng.standard_normal((3, Cn, T)).astype(np.float32)
    zero = np.zeros(Cn, np.float32)
    for k in range(12):
        f = _one_hot(k, 0.75)
        v0 = _no_snake(ao.up(x, f))
        want = _interleave(ao.down(v0, _one_hot(5)), ao.down(v0, _one_hot(6)))
        for api in ("forward", "packed"):
            _assert_equal(f"tap {k} {api}", _readout(x, zero, zero, False, f, api=api)[0], want)
        _, vimg = _readout(x, zero, zero, False, f, prec="tc_f16", y=False, img=True)
        _assert_img(f"tap {k} MODE 2", vimg, ao.image(want, "f16").reshape(vimg.shape))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_sin_errors(mode, capsys):
    """__sinf (MODE 1) and sin.approx (MODE 2) measured on u ~ 2^-20 (u = x, v ~ s^2: the snake alone), and checked
    against the oracle's intervals.  Prints the largest errors observed."""
    rng = np.random.default_rng(11)
    B, Cn, T = 1, 16, 4096
    f = _one_hot(5, 0.5)                                     # fu2[5] = 1: u[2q + 1] = x[q]
    x = (rng.uniform(-1, 1, (B, Cn, T)) * 2.0 ** -20).astype(np.float32)
    amax = 1e3 if mode == "fp32" else 1e4
    alpha = (2.0 ** 20 * np.linspace(1.0, amax, Cn)).astype(np.float32)
    beta = np.ones(Cn, np.float32)                           # invb = frcp(1 + 1e-9) = 1
    u = ao.up(x, f)
    arg = (u * alpha[None, :, None]).astype(np.float64)     # fl(u a): the reference rounds the product too
    if mode == "fp32":
        v, _ = _readout(x, alpha, beta, False, f)
        _assert_snake("snake MODE 1", v, u, alpha, beta, False)
        r = ao.reduce(u, alpha[:, None]).astype(np.float64)
        s = np.sqrt(np.maximum(v.astype(np.float64) - u, 0))
        sel = np.abs(np.sin(r)) > 0.5
        err = np.abs(s - np.abs(np.sin(r)))[sel].max()
        with capsys.disabled():
            print(f"\n__sinf: largest |s - sin r| observed {err:.3e} (bound {ao.SINF_ERR:.3e}; resolution ~6e-8), "
                  f"|u a| <= {np.abs(arg).max():.0f}, device {torch.cuda.get_device_name()}")
    else:
        _, vimg = _readout(x, alpha, beta, False, f, prec="tc_f16", y=False, img=True)
        vv = _img_values(vimg, "f16", Cn)
        _assert_snake("snake MODE 2", vv, u, alpha, beta, False, img_prec="f16")
        # where |sin(u a)| is small, f16 resolves s = sqrt(v - u) to ~2^-12 relative, so the phase error
        # | |s| - |sin(u a)| | / |cos(u a)| shows down to ~1e-10 |u a| at |u a| > 2000
        fast = ao.pair_group(np.arange(2 * T), T)[None, None, :]
        s = np.sqrt(np.maximum(vv.astype(np.float64) - u, 0))
        sel = fast & (np.abs(arg) > 2000) & (np.abs(np.sin(arg)) > 0.01) & (np.abs(np.sin(arg)) < 0.2)
        coef = (np.abs(s[sel] - np.abs(np.sin(arg[sel]))) / np.abs(np.cos(arg[sel])) / np.abs(arg[sel])).max()
        with capsys.disabled():
            print(f"\nsin.approx: largest phase error observed {coef:.3e} |u a| rad (bound {ao.PHASE:.3e}; "
                  f"{int(sel.sum())} samples), "
                  f"|u a| <= {np.abs(arg).max():.0f}, device {torch.cuda.get_device_name()}")


@pytest.mark.gpu
@pytest.mark.parametrize("T,where", [(1088, [500, 501, 3, 1085]), (249, [0, 130, 131, 248])])
def test_non_finite_input_span(T, where):
    """A NaN or inf at x[p] gives NaN exactly where the oracle's literal pair form puts it: the reference's y span
    [p - 5, p + 5], and one more output on one side where a pair group's zero tap multiplies x[p] (p + 6 for even p,
    p - 6 for odd p)."""
    f_up, f_down = _kaiser()
    rng = np.random.default_rng(5)
    Cn = len(where)
    x = rng.standard_normal((1, Cn, T)).astype(np.float32)
    for c, p in enumerate(where):
        x[0, c, p] = np.nan if c % 2 else np.inf
    zero = np.zeros(Cn, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        u = ao.up(x, f_up)
        vnan = ~np.isfinite(u)
        want = ao.down(np.where(vnan, np.float32(np.nan), np.float32(0)), f_down)
        ref = _down64(np.where(np.isfinite(_up64(x, f_up)), 0.0, np.nan), f_down)
    for api in ("forward", "packed"):
        y = _run(x, zero, None, False, f_up, f_down, api=api)[0]
        assert (np.isnan(y) == np.isnan(want)).all(), api
    for c, p in enumerate(where):
        got = np.flatnonzero(np.isnan(y[0, c]))
        span = np.flatnonzero(np.isnan(ref[0, c]))
        assert span.tolist() == list(range(max(p - 5, 0), min(p + 6, T)))
        extra = sorted(set(got) - set(span))
        assert set(span) <= set(got) and len(extra) <= 1, (p, extra)
        if extra:
            assert extra == [p + 6 if p % 2 == 0 else p - 6], (p, extra)
