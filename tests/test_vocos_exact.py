"""Vocos' kernels against the kernel-order oracle (tests/vocos_exact_oracle.py), one launch at a time through
ab_vocos_norm_forward / ab_vocos_pointwise_forward, and the generator's forward against the chain of those launches.

* `vocos_norm_kernel` (LayerNorm over channels, with and without the depthwise conv; fp32 out and both operand
  images) bit for bit, at channel counts that reach every time tile (16, 8, 4 and 2 steps), sequences shorter than the
  conv's halo, ragged tiles, a constant channel vector (variance exactly 0: the output is ln_b), an offset of 1e4 over
  unit noise (the two-pass variance) and an ln_w that saturates the f16 image.
* The pointwise wgmma GEMM (`hitem_kernel`, `launch_tc_pointwise`) with one-hot weights (+-2^e at one input channel
  per output, every K chunk hit): every accumulator is one exact product, so GAMMA is bit for bit, GELU's image lies
  in the interval of CUDA's erff bound, and every spectrum bin in that of expf / sinf / cosf; bins driven to m >= 5
  and p = 0 read exactly (100, +0), which pins the head's column pairing.  Dense weights: the GEMM's accumulator
  equals `hconv_kernel`'s from the same operand image (the same K chunk -> k16 order), which sits within the floor
  rule of test_resblock_exact.py of the float64 GEMM, and the epilogues are checked on that accumulator.
* The fp32 route (`conv1d_fp32_kernel` at k = 1, a sequential FMA chain over C_in; the head through
  ab_spectral_head_forward) against the same oracle.
* A Vocos generator's forward equals the chain of single launches bit for bit at every precision.

Outputs are filled with NaN (images with 0xFFFF, a NaN in f16 and bf16) before each launch, and every input is
followed by NaN (0xFFFF after an image), so an unwritten element or a read past an input shows."""
import ctypes as C

import numpy as np
import pytest
import torch

import resblock_oracle as ro
import vocos_exact_oracle as vx
from diffwave_exact_oracle import fma_chain

DEV = "cuda:0"
PRECS = {"tc_f16": "f16", "tc_bf16": "bf16"}
GELU, GAMMA, SPECTRUM = 0, 1, 2
GUARD = 4096          # NaN elements after every input
FLOOR_MEAN, FLOOR_MAX = 2.0, 3.0   # test_resblock_exact.py's floor rule


def _lib():
    from amphion_b200 import _capi
    return _capi


# ------------------------------------------------------------------------------------------------ the harness
def _guarded(a):
    """fp32 numpy -> a device buffer holding a, then GUARD NaNs (the tensor, a view of the front)."""
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.full((a.size + GUARD,), float("nan"), device=DEV)
    buf[:a.size] = torch.from_numpy(a.reshape(-1)).to(DEV)
    return buf


def _guarded_img(img):
    """uint16 operand image -> a device buffer holding it, then GUARD 0xFFFF."""
    img = np.ascontiguousarray(img).view(np.int16)
    buf = torch.full((img.size + GUARD,), -1, dtype=torch.int16, device=DEV)
    buf[:img.size] = torch.from_numpy(img.reshape(-1)).to(DEV)
    return buf


def _img_out(B, C, T):
    return torch.full((B, (C + 15) // 16 * 2, T, 8), -1, dtype=torch.int16, device=DEV)


def _host_img(t):
    return t.cpu().numpy().view(np.uint16)


def _bits_to_f32(bits, prec):
    bits = np.asarray(bits, np.uint16)
    if prec == "f16":
        return bits.view(np.float16).astype(np.float32)
    return (bits.astype(np.uint32) << 16).view(np.float32)


def _assert_equal(what, got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


def _assert_in(what, got, lo, hi):
    ok = vx.in_interval(got, lo, hi)
    assert ok.all(), (f"{what}: {int((~ok).sum())} of {ok.size} outside, first at {np.argwhere(~ok)[0].tolist()}: "
                      f"{got[~ok][0]!r} not in [{lo[~ok][0]!r}, {hi[~ok][0]!r}]")


def _norm(x, dw, ln_w, ln_b, eps, prec):
    """One ab_vocos_norm_forward -> (rc, y fp32 or image bits [B, c8n, T, 8])."""
    capi = _lib()
    B, Cn, T = x.shape
    xd = _guarded(x)
    dww, dwb = (None, None) if dw is None else (_guarded(dw[0]), _guarded(dw[1]))
    lw, lb = _guarded(ln_w), _guarded(ln_b)
    y = torch.full((B, Cn, T), float("nan"), device=DEV) if prec == "fp32" else None
    img = _img_out(B, Cn, T) if prec != "fp32" else None
    rc = capi.lib.ab_vocos_norm_forward(capi.ptr(xd), capi.ptr(dww), capi.ptr(dwb), capi.ptr(lw), capi.ptr(lb), eps,
                                        capi.ptr(y), capi.ptr(img), capi.PRECISIONS[prec], B, Cn, T, capi.stream_ptr())
    torch.cuda.synchronize()
    return rc, (y.cpu().numpy() if y is not None else _host_img(img))


def _pointwise(epi, prec, w, bias, B, cin, cout, T, *, x=None, ximg=None, gamma=None, y0=None):
    """One ab_vocos_pointwise_forward.  x fp32 [B, C_in, T] (fp32) or ximg image bits (tc).  -> (rc, out): GELU the
    image bits (tc) or y; GAMMA y; SPECTRUM spec [B, T, bins, 2]."""
    capi = _lib()
    xd = None if x is None else _guarded(x)
    xi = None if ximg is None else _guarded_img(ximg)
    wd, bd = _guarded(w), _guarded(bias)
    gd = None if gamma is None else _guarded(gamma)
    y = yimg = spec = None
    if epi == GAMMA:
        y = torch.from_numpy(np.ascontiguousarray(y0, np.float32)).to(DEV)
    elif epi == GELU and prec == "fp32":
        y = torch.full((B, cout, T), float("nan"), device=DEV)
    elif epi == GELU:
        yimg = _img_out(B, cout, T)
    else:
        spec = torch.full((B, T, cout // 2, 2), float("nan"), device=DEV)
    need = capi.lib.ab_vocos_pointwise_workspace_bytes(epi, B, cin, cout, T, capi.PRECISIONS[prec])
    assert need > 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    rc = capi.lib.ab_vocos_pointwise_forward(epi, capi.ptr(xd), capi.ptr(xi), capi.ptr(wd), capi.ptr(bd), capi.ptr(gd),
                                             capi.ptr(y), capi.ptr(yimg), capi.ptr(spec), B, cin, cout, T,
                                             capi.PRECISIONS[prec], C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need,
                                             capi.stream_ptr())
    torch.cuda.synchronize()
    out = yimg if yimg is not None else spec if spec is not None else y
    return rc, (_host_img(out) if yimg is not None else out.cpu().numpy())


def _hconv_k1(prec, ximg, w, bias, B, cin, cout, T):
    """ab_tc_conv_forward mode 0, k = 1 (hconv_kernel) from the operand image: y = acc + bias."""
    capi = _lib()
    xi, wd, bd = _guarded_img(ximg), _guarded(w[:, :, None]), _guarded(bias)
    y = torch.full((B, cout, T), float("nan"), device=DEV)
    need = capi.lib.ab_tc_conv_workspace_bytes(0, cin, cout, 1, 1)
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    rc = capi.lib.ab_tc_conv_forward(0, None, None, 1.0, capi.ptr(xi), capi.ptr(wd), capi.ptr(bd), None, None, 1.0, 0,
                                     capi.ptr(y), None, 1.0, B, cin, cout, T, 1, 1, 0, capi.PRECISIONS[prec],
                                     C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, capi.last_error()
    return y.cpu().numpy()


# ------------------------------------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("C,T", [(12, 9), (48, 17), (256, 5), (1024, 3), (2500, 2), (4096, 1)])
@pytest.mark.parametrize("dw", [False, True], ids=["ln", "dw-ln"])
def test_kernel_order_layer_norm_matches_torch(C, T, dw):
    rng = np.random.default_rng(C + T + dw)
    x = (rng.normal(0, 2, (2, C, T)) + rng.normal(0, 3, (2, 1, T))).astype(np.float32)
    ln_w, ln_b = rng.normal(1, 0.2, C).astype(np.float32), rng.normal(0, 0.1, C).astype(np.float32)
    d = (rng.normal(0, 0.3, (C, 1, 7)).astype(np.float32), rng.normal(0, 0.1, C).astype(np.float32)) if dw else None
    got = vx.layer_norm_kernel_order(x, d, ln_w, ln_b, 1e-6)
    h = torch.from_numpy(x).double()
    if dw:
        h = torch.nn.functional.conv1d(h, torch.from_numpy(d[0]).double(), torch.from_numpy(d[1]).double(), padding=3,
                                       groups=C)
    want = torch.layer_norm(h.transpose(1, 2), (C,), torch.from_numpy(ln_w).double(), torch.from_numpy(ln_b).double(),
                            1e-6).transpose(1, 2).numpy()
    err = float(np.abs(got - want).max())
    assert err <= 1e-6 * float(np.abs(want).max()), err


def test_norm_tiles():
    assert [vx.norm_tile(c)[0] for c in (12, 256, 1000, 1024, 2500, 4096, 16000)] == [16, 16, 16, 8, 4, 2, 1]
    assert vx.norm_fits(50000) and not vx.norm_fits(51200)


def test_gelu_interval_contains_float64_and_collapses():
    from scipy.special import erf
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.normal(0, 3, 20000), rng.uniform(-4.5, -3.5, 5000), np.linspace(-12, 12, 4001),
                        [0.0, -0.0, 1e-30, -1e-30, 6.0, -6.0, 100.0, -100.0, 3e38, -3e38]]).astype(np.float32)
    lo, hi = vx.gelu_interval(v)
    v64 = v.astype(np.float64)
    g64 = 0.5 * v64 * (1 + erf(v64 / np.sqrt(2)))
    # the float64 GELU of v: within the interval, up to the rounding of the steps (4 ulp) and of v * 0.70710677f,
    # whose relative error of 1e-7 the tail of the GELU magnifies by about v^2
    slack = (4 * np.spacing(np.maximum(np.abs(lo), np.abs(hi))).astype(np.float64)
             + 2e-7 * (1 + v64 ** 2) * np.abs(g64))
    col = lo.view(np.uint32) == hi.view(np.uint32)
    assert ((lo - slack <= g64) & (g64 <= hi + slack))[~col].all()
    # where it collapsed, erff is +-1 exactly and the float64 GELU is within 2^-26 |v| of v or of 0
    assert (np.abs(g64 - lo)[col] <= 2.0 ** -26 * np.abs(v64[col]) + slack[col]).all()
    assert (lo <= hi).all()
    big, neg = v >= 6, v <= -6
    assert (lo[big] == v[big]).all() and (hi[big] == v[big]).all()
    assert (lo[neg].view(np.uint32) == np.float32(-0.0).view(np.uint32)).all()
    assert (hi[neg].view(np.uint32) == np.float32(-0.0).view(np.uint32)).all()
    # in between: the interval spans a few ulp, never more than 2^-18 of 0.5 |v| (+ a subnormal floor)
    mid = ~big & ~neg
    assert ((hi - lo)[mid] <= 2.0 ** -18 * np.abs(v[mid]) + 1e-37).all()
    # the cancellation in 1 + erf near v = -4 is inside the interval, not a relative error on the result
    near = (v > -4.5) & (v < -3.5)
    assert ((hi - lo)[near] > 0).all()


def test_spectrum_interval_contains_float64_and_collapses():
    rng = np.random.default_rng(1)
    m = np.concatenate([rng.normal(0, 3, 20000), [5.0, 6.0, 90.0, 4.0, -100.0]]).astype(np.float32)
    p = np.concatenate([rng.normal(0, 4, 20000), [0.0, -0.0, 1.0, 0.0, 3.0]]).astype(np.float32)
    (re_lo, re_hi), (im_lo, im_hi) = vx.spectrum_interval(m, p)
    amp = np.minimum(np.exp(m.astype(np.float64)), 100.0)
    re, im = amp * np.cos(p.astype(np.float64)), amp * np.sin(p.astype(np.float64))
    assert ((re_lo <= re) & (re <= re_hi) & (im_lo <= im) & (im <= im_hi)).all()
    # m = 5 and 6 with p = +0 and -0: exactly (100, +0) and (100, -0)
    for i, zero in ((-5, 0x00000000), (-4, 0x80000000)):
        assert re_lo[i] == re_hi[i] == 100
        assert im_lo[i].view(np.uint32) == im_hi[i].view(np.uint32) == zero
    assert re_lo[-2] < re_hi[-2] and im_lo[-2] == im_hi[-2] == 0                # m = 4: e^4 < 100, amp is not pinned
    ordinary = np.abs(m) < 10
    assert ((re_hi - re_lo)[ordinary] <= 2.0 ** -19 * amp[ordinary] + 1e-30).all()


@pytest.mark.parametrize("cout", [66, 50, 300, 1922])
def test_head_columns_pair_each_bin(cout):
    rng = np.random.default_rng(cout)
    cin, bins = 24, cout // 2
    w = rng.integers(-8, 9, (cout, cin)).astype(np.float64)    # integer sums: exact in any order
    x = rng.integers(-8, 9, (2, cin, 5)).astype(np.float64)
    cols = vx.head_columns(cout)
    nw, nb = vx.pointwise_geometry(cout)
    assert cols.shape == (nb * nw,) and (cols[2 * bins:] == -1).all()
    dense = np.einsum("oc,bct->bot", w, x)
    packed = np.einsum("oc,bct->bot", np.where(cols[:, None] >= 0, w[np.maximum(cols, 0)], 0.0), x)
    assert np.array_equal(packed[:, 0:2 * bins:2], dense[:, :bins])       # column 2j: bin j's log-magnitude
    assert np.array_equal(packed[:, 1:2 * bins:2], dense[:, bins:])       # column 2j + 1: its phase
    assert not packed[:, 2 * bins:].any()


@pytest.mark.parametrize("cin,cout", [(48, 144), (40, 120), (4096, 1024), (1024, 1922), (33, 7)])
def test_one_hot_linear_hits_every_k_chunk(cin, cout):
    w = vx.one_hot_linear(np.random.default_rng(cin), cin, cout, (0, 1))
    hit = set((w.perm // 32).tolist())
    if cout > -(-cin // 32):
        assert hit == set(range(-(-cin // 32))) and cin - 1 in w.perm.tolist()
    assert (np.count_nonzero(w.dense(), axis=(1, 2)) == 1).all()


def test_entry_points_refuse_malformed_requests():
    """AB_ERR_ARG / AB_ERR_UNSUPPORTED before any launch (the pointers are never dereferenced)."""
    capi = _lib()
    lib, P = capi.lib, C.c_void_p
    f16, fp32 = capi.PRECISIONS["tc_f16"], capi.PRECISIONS["fp32"]
    a = P(256)

    def norm(y, img, prec=f16, dw=(None, None), C_=48):
        return lib.ab_vocos_norm_forward(a, dw[0], dw[1], a, a, 1e-6, y, img, prec, 2, C_, 10, None)

    assert norm(a, a) == -1 and "exactly one" in capi.last_error()
    assert norm(None, None) == -1
    assert norm(a, None, dw=(a, None)) == -1 and "dw" in capi.last_error()
    assert norm(None, a, prec=fp32) == -1 and "precision" in capi.last_error()
    assert norm(a, None, C_=51200) == -2 and "shared memory" in capi.last_error()
    assert norm(a, None, C_=0) == -1

    need = lib.ab_vocos_pointwise_workspace_bytes(SPECTRUM, 2, 48, 66, 10, f16)
    assert need > 0 and lib.ab_vocos_pointwise_workspace_bytes(SPECTRUM, 2, 48, 66, 10, fp32) > \
        lib.ab_vocos_pointwise_workspace_bytes(GAMMA, 2, 48, 66, 10, fp32)

    def pw(epi, x, ximg, prec=f16, gamma=a, y=a, yimg=a, spec=a, cout=66, ws=need):
        return lib.ab_vocos_pointwise_forward(epi, x, ximg, a, a, gamma, y, yimg, spec, 2, 48, cout, 10, prec, a, ws, None)

    assert pw(SPECTRUM, None, a, cout=65) == -1 and "even" in capi.last_error()
    assert pw(GELU, a, None) == -1 and "ximg" in capi.last_error()          # tensor cores take the image
    assert pw(GELU, a, a) == -1
    assert pw(GELU, None, a, prec=fp32) == -1 and "x" in capi.last_error()  # fp32 takes x
    assert pw(GAMMA, None, a, gamma=None) == -1 and "gamma" in capi.last_error()
    assert pw(GAMMA, None, a, y=None) == -1
    assert pw(GELU, None, a, yimg=None) == -1
    assert pw(GELU, a, None, prec=fp32, y=None) == -1
    assert pw(SPECTRUM, None, a, spec=None) == -1
    assert pw(3, None, a) == -1 and "epilogue" in capi.last_error()
    assert pw(GELU, None, a, ws=need - 1) == -5


# ------------------------------------------------------------------------------------------------ GPU: LayerNorm
def _norm_inputs(rng, values, B, C, T, dw):
    dw_w = rng.normal(0, 0.3, (C, 1, 7)).astype(np.float32)
    dw_b = rng.normal(0, 0.1, C).astype(np.float32)
    ln_w, ln_b = rng.normal(1, 0.2, C).astype(np.float32), rng.normal(0, 0.1, C).astype(np.float32)
    if values == "ordinary":
        x = rng.normal(0, 2, (B, C, T)).astype(np.float32)
    elif values == "constant":   # the same dyadic value in every channel: the sums are exact, the variance 0
        x = np.repeat(rng.integers(-16, 17, (B, 1, T)) * 0.25, C, axis=1).astype(np.float32)
        dw_w = np.repeat(rng.choice([-0.5, -0.25, 0.25, 0.5, 1.0], (1, 1, 7)), C, axis=0).astype(np.float32)
        dw_b = np.full(C, rng.choice([-0.75, 0.5]), np.float32)
    elif values == "offset":     # 1e4 over unit noise: a one-pass variance loses it
        x = (1e4 + rng.normal(0, 1, (B, C, T))).astype(np.float32)
        dw_w = np.repeat(rng.normal(0, 0.3, (1, 1, 7)), C, axis=0).astype(np.float32)
    else:
        assert values == "saturation"   # |y| far past 65504: the f16 image holds +-65504
        x = rng.normal(0, 2, (B, C, T)).astype(np.float32)
        ln_w = (rng.choice([-1.0, 1.0], C) * rng.uniform(3e4, 1e5, C)).astype(np.float32)
    return x, ((dw_w, dw_b) if dw else None), ln_w, ln_b


# (C, T, B, value sets): every time tile (C 1024: 8 steps, 2500: 4, 4096: 2), T shorter than the conv's halo, one
# tile, one step past it, ragged
NORM_SHAPES = [
    (12, 1, 3, ("ordinary", "constant")), (12, 17, 1, ("ordinary", "offset", "saturation")),
    (40, 3, 3, ("ordinary",)), (40, 333, 1, ("ordinary", "constant")),
    (48, 15, 3, ("ordinary", "offset")), (48, 16, 1, ("ordinary", "saturation")),
    (256, 17, 3, ("ordinary", "constant", "offset", "saturation")), (256, 333, 1, ("ordinary",)),
    (1024, 3, 3, ("ordinary", "offset")), (1024, 333, 1, ("ordinary", "saturation")),
    (2500, 16, 3, ("ordinary", "constant")), (2500, 1, 1, ("ordinary",)),
    (4096, 15, 1, ("ordinary", "offset", "saturation")), (4096, 17, 3, ("ordinary", "constant")),
]


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("out", ["fp32", "tc_f16", "tc_bf16"])
@pytest.mark.parametrize("dw", [False, True], ids=["ln", "dw-ln"])
def test_layer_norm_is_exact(dw, out, eps):
    for C_, T, B, sets in NORM_SHAPES:
        for values in sets:
            what = f"C {C_} T {T} B {B} {values}"
            rng = np.random.default_rng(C_ * 1000 + T * 10 + B + len(values) + dw)
            x, d, ln_w, ln_b = _norm_inputs(rng, values, B, C_, T, dw)
            want = vx.layer_norm_kernel_order(x, d, ln_w, ln_b, eps)
            assert np.isfinite(want).all(), what
            if values == "constant":
                assert np.array_equal(want, np.broadcast_to(ln_b[None, :, None], want.shape)), what
            rc, got = _norm(x, d, ln_w, ln_b, eps, out)
            assert rc == 0, (what, _lib().last_error())
            if out == "fp32":
                _assert_equal(what, got, want)
                continue
            bits, padding = ro.from_image(got, C_)
            assert np.array_equal(bits, ro.image_bits(want, 1.0, PRECS[out])), what
            assert not padding.any(), f"{what}: padding channels of the image are not zero"
            if values == "saturation" and out == "tc_f16":
                assert (np.abs(_bits_to_f32(bits, "f16")) == 65504).any(), what


@pytest.mark.gpu
def test_layer_norm_too_wide_writes_nothing():
    rng = np.random.default_rng(2)
    C_ = 51200                                   # one time step of 51200 channels is past 200 KB of shared memory
    x = rng.normal(0, 1, (1, C_, 2)).astype(np.float32)
    ln = np.ones(C_, np.float32)
    for out in ("fp32", "tc_f16"):
        rc, got = _norm(x, None, ln, ln, 1e-6, out)
        assert rc == -2 and "shared memory" in _lib().last_error()
        assert np.isnan(got).all() if out == "fp32" else (got == 0xFFFF).all()


# ------------------------------------------------------------------------------------------------ GPU: pointwise GEMM
def _ximg(x, prec):
    return ro.to_image(ro.image_bits(x, 1.0, PRECS[prec]))


def _check_gamma(what, prec, w, bias, B, cin, cout, T, ximg, v, rng):
    """GAMMA of accumulator-plus-bias v [B, C_out, T]: y = y0 + gamma * v, each step rounded."""
    y0 = rng.normal(0, 1, (B, cout, T)).astype(np.float32)
    gamma = rng.uniform(0.2, 1.0, cout).astype(np.float32)
    rc, y = _pointwise(GAMMA, prec, w, bias, B, cin, cout, T, ximg=ximg, gamma=gamma, y0=y0)
    assert rc == 0, _lib().last_error()
    _assert_equal(f"{what} GAMMA", y, y0 + (gamma[None, :, None] * v).astype(np.float32))


def _check_gelu(what, prec, w, bias, B, cin, cout, T, ximg, v):
    rc, img = _pointwise(GELU, prec, w, bias, B, cin, cout, T, ximg=ximg)
    assert rc == 0, _lib().last_error()
    bits, padding = ro.from_image(img, cout)
    assert not padding.any(), f"{what} GELU: padding channels of the image are not zero"
    lo, hi = vx.gelu_interval(v)
    _assert_in(f"{what} GELU", _bits_to_f32(bits, PRECS[prec]), ro.rnd(lo, PRECS[prec]), ro.rnd(hi, PRECS[prec]))


def _check_spectrum(what, spec, m, p):
    """spec [B, T, bins, 2] against the intervals of m, p [B, bins, T]."""
    with np.errstate(over="ignore"):
        (re_lo, re_hi), (im_lo, im_hi) = (tuple(a.transpose(0, 2, 1) for a in iv) for iv in vx.spectrum_interval(m, p))
    _assert_in(f"{what} SPECTRUM re", spec[..., 0], re_lo, re_hi)
    _assert_in(f"{what} SPECTRUM im", spec[..., 1], im_lo, im_hi)


# (id, C_in, C_out, B, T, epilogues): the fixtures' layers and heads, NW 64 / 128 / 256, C_out 300 (N blocks of 256 and
# 44), the recipe (16 N blocks, 32 K chunks; 128 K chunks; the head's partial 130-column block), 128-row tiles cut at
# 127 / 128 / 129, a 1000-step walk of B 8 x 8 tiles x 16 N blocks = 1024 items
PW = [
    ("a-pw1", 48, 144, 2, 129, (GELU, GAMMA)),
    ("a-pw2", 144, 48, 2, 127, (GELU, GAMMA)),
    ("b-pw1", 40, 120, 1, 128, (GELU, GAMMA)),
    ("b-pw2", 120, 40, 3, 1, (GELU, GAMMA)),
    ("a-head", 48, 66, 2, 129, (SPECTRUM,)),
    ("b-head", 40, 50, 1, 1000, (SPECTRUM,)),
    ("cout300", 64, 300, 2, 1000, (GELU, GAMMA, SPECTRUM)),
    ("recipe-pw1", 1024, 4096, 1, 129, (GELU, GAMMA)),
    ("recipe-pw2", 4096, 1024, 2, 128, (GELU, GAMMA)),
    ("recipe-head", 1024, 1922, 2, 127, (SPECTRUM,)),
    ("recipe-walk", 1024, 4096, 8, 1000, (GAMMA,)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", PW, ids=[c[0] for c in PW])
def test_one_hot_pointwise_is_exact(case, prec):
    name, cin, cout, B, T, epis = case
    rng = np.random.default_rng(cin * 3 + cout + T)
    x = rng.normal(0, 2, (B, cin, T)).astype(np.float32)
    ximg = _ximg(x, prec)
    a = ro.rnd(x, PRECS[prec])
    bins = cout // 2
    driven = np.array([], np.int64)
    if SPECTRUM in epis:
        # bins read exactly (100, +0): magnitude row zero with bias 6 (e^6 > 1e2), phase row zero with bias +0
        nw, nb = vx.pointwise_geometry(cout)
        driven = np.unique(np.concatenate([np.arange(0, bins, 7), [bins - 1, bins - 2],
                                           np.arange((nb - 1) * nw // 2, bins)[::3]]))
    oh = vx.one_hot_linear(rng, cin, cout, (-2, -1, 0, 1), avoid=np.concatenate([driven, bins + driven]))
    w = oh.dense()[:, :, 0]
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    w[driven] = 0
    w[bins + driven] = 0
    bias[driven], bias[bins + driven] = 6.0, 0.0
    acc = ro.conv(a, oh.rounded(PRECS[prec]), 1)                     # the one product of each output
    acc[:, driven], acc[:, bins + driven] = 0, 0
    v = (acc + bias[None, :, None]).astype(np.float32)
    for epi in epis:
        if epi == GAMMA:
            _check_gamma(name, prec, w, bias, B, cin, cout, T, ximg, v, rng)
        elif epi == GELU:
            _check_gelu(name, prec, w, bias, B, cin, cout, T, ximg, v)
        else:
            rc, spec = _pointwise(SPECTRUM, prec, w, bias, B, cin, cout, T, ximg=ximg)
            assert rc == 0, _lib().last_error()
            _check_spectrum(name, spec, v[:, :bins], v[:, bins:])
            exact = spec[:, :, driven]
            assert (exact[..., 0] == 100).all(), f"{name}: a driven bin's magnitude is not 100"
            assert (exact[..., 1].view(np.uint32) == 0).all(), f"{name}: a driven bin's phase term is not +0"


# (id, C_in, C_out, B, T)
DENSE = [
    ("a-pw1", 48, 144, 2, 129),
    ("a-head", 48, 66, 2, 127),
    ("cout300", 64, 300, 2, 200),
    ("recipe-pw1", 1024, 4096, 1, 129),
    ("recipe-pw2", 4096, 1024, 1, 128),
    ("recipe-head", 1024, 1922, 2, 129),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_pointwise_equals_hconv(case, prec):
    """The GEMM's acc + b equals hconv_kernel's k = 1 conv from the same image, bit for bit; the epilogues on it."""
    name, cin, cout, B, T = case
    rng = np.random.default_rng(cin + cout + T)
    x = rng.normal(0, 1, (B, cin, T)).astype(np.float32)
    w = rng.normal(0, 1 / np.sqrt(cin), (cout, cin)).astype(np.float32)
    bias = rng.normal(0, 0.1, cout).astype(np.float32)
    ximg = _ximg(x, prec)
    v = _hconv_k1(prec, ximg, w, bias, B, cin, cout, T)
    assert np.isfinite(v).all()
    a = ro.rnd(x, PRECS[prec])
    o64, o32 = (ro.conv(a, ro.rnd(w, PRECS[prec])[:, :, None], 1, acc) + bias[None, :, None] for acc in ("f64", "mma"))
    e_mean, e_max, f_mean, f_max = ro.floor_stats(v, o64, o32)
    print(f"{name} {prec}: mean {e_mean / f_mean:.2f} x floor, max {e_max / f_max:.2f} x floor")
    assert e_mean <= FLOOR_MEAN * f_mean and e_max <= FLOOR_MAX * f_max
    rc, y = _pointwise(GAMMA, prec, w, bias, B, cin, cout, T, ximg=ximg, gamma=np.ones(cout, np.float32),
                       y0=np.zeros((B, cout, T), np.float32))
    assert rc == 0
    assert np.array_equal(y, v), f"{name}: hitem_kernel's acc + b differs from hconv_kernel's"
    _check_gamma(name, prec, w, bias, B, cin, cout, T, ximg, v, rng)
    _check_gelu(name, prec, w, bias, B, cin, cout, T, ximg, v)
    if cout % 2 == 0:
        rc, spec = _pointwise(SPECTRUM, prec, w, bias, B, cin, cout, T, ximg=ximg)
        assert rc == 0
        _check_spectrum(name, spec, v[:, :cout // 2], v[:, cout // 2:])


# ------------------------------------------------------------------------------------------------ GPU: fp32 route
@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,B,T", [(48, 144, 2, 129), (144, 48, 1, 300), (48, 66, 2, 17), (256, 258, 1, 130)])
def test_fp32_pointwise_is_exact(cin, cout, B, T):
    rng = np.random.default_rng(cin * cout + T)
    x = rng.normal(0, 2, (B, cin, T)).astype(np.float32)
    w = rng.normal(0, 2 / np.sqrt(cin), (cout, cin)).astype(np.float32)
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    v = (fma_chain(w, x) + bias[None, :, None]).astype(np.float32)   # conv1d_fp32_kernel at k = 1, then + bias
    y0 = rng.normal(0, 1, (B, cout, T)).astype(np.float32)
    gamma = rng.uniform(0.2, 1.0, cout).astype(np.float32)
    rc, y = _pointwise(GAMMA, "fp32", w, bias, B, cin, cout, T, x=x, gamma=gamma, y0=y0)
    assert rc == 0, _lib().last_error()
    _assert_equal("fp32 GAMMA", y, y0 + (gamma[None, :, None] * v).astype(np.float32))
    rc, y = _pointwise(GELU, "fp32", w, bias, B, cin, cout, T, x=x)
    assert rc == 0
    lo, hi = vx.gelu_interval(v)
    _assert_in("fp32 GELU", y, lo, hi)
    rc, spec = _pointwise(SPECTRUM, "fp32", w, bias, B, cin, cout, T, x=x)
    assert rc == 0
    _check_spectrum("fp32", spec, v[:, :cout // 2], v[:, cout // 2:])


# ------------------------------------------------------------------------------------------------ GPU: composition
def _embed(model, mel, prec, on_tc):
    """conv_pre (k = 7) as the generator runs it: the wgmma conv from the mel view, or the fp32 conv."""
    capi = _lib()
    w = model.backbone.embed.weight.detach().float().contiguous()
    b = model.backbone.embed.bias.detach().float().contiguous()
    B, cin, T = mel.shape
    D = w.shape[0]
    y = torch.full((B, D, T), float("nan"), device=DEV)
    if on_tc:
        need = capi.lib.ab_tc_conv_workspace_bytes(0, cin, D, 7, 1)
        ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
        rc = capi.lib.ab_tc_conv_forward(0, capi.ptr(mel), capi.shape_array(mel.stride()), 1.0, None, capi.ptr(w),
                                         capi.ptr(b), None, None, 1.0, 0, capi.ptr(y), None, 0.1, B, cin, D, T, 7, 1, 0,
                                         capi.PRECISIONS[prec], C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need,
                                         capi.stream_ptr())
    else:
        x = mel.contiguous()
        need = capi.lib.ab_conv1d_workspace_bytes(cin, D, 7, 0)
        ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
        rc = capi.lib.ab_conv1d_forward(capi.ptr(x), capi.ptr(w), capi.ptr(b), None, capi.ptr(y), B, cin, D, T, 7, 1, 1.0,
                                        0, 0, C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, capi.stream_ptr())
    assert rc == 0, capi.last_error()
    return y


def _chain(model, mel, prec, on_tc):
    """Vocos.forward as single launches: embed, norm, the ConvNeXt blocks, final norm, head, iSTFT."""
    capi = _lib()
    lib, P = capi.lib, capi.ptr
    sd = {k: v.detach().float().contiguous() for k, v in model.state_dict().items()}
    B, _, T = mel.shape
    D, F, n_fft, hop = model.dim, model.intermediate_dim, model.n_fft, model.hop_length
    pr = capi.PRECISIONS[prec]
    tc = prec != "fp32"
    st = capi.stream_ptr()

    def norm(x, pre, dw, y=None, img=None):
        dww, dwb = (sd[pre + "dwconv.weight"], sd[pre + "dwconv.bias"]) if dw else (None, None)
        rc = lib.ab_vocos_norm_forward(P(x), P(dww), P(dwb), P(sd[pre + "norm.weight"] if dw else sd[pre + "weight"]),
                                       P(sd[pre + "norm.bias"] if dw else sd[pre + "bias"]), 1e-6, P(y), P(img), pr, B, D,
                                       T, st)
        assert rc == 0, capi.last_error()

    def pointwise(epi, name, cin, cout, x=None, ximg=None, y=None, yimg=None, gamma=None, spec=None):
        need = lib.ab_vocos_pointwise_workspace_bytes(epi, B, cin, cout, T, pr)
        ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
        rc = lib.ab_vocos_pointwise_forward(epi, P(x), P(ximg), P(sd[name + ".weight"]), P(sd[name + ".bias"]), P(gamma),
                                            P(y), P(yimg), P(spec), B, cin, cout, T, pr,
                                            C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, st)
        assert rc == 0, capi.last_error()

    X = torch.full((B, D, T), float("nan"), device=DEV)
    norm(_embed(model, mel, prec, on_tc), "backbone.norm.", False, y=X)
    for i in range(model.num_layers):
        pre = f"backbone.convnext.{i}."
        if tc:
            H, I = _img_out(B, D, T), _img_out(B, F, T)
            norm(X, pre, True, img=H)
            pointwise(GELU, pre + "pwconv1", D, F, ximg=H, yimg=I)
            pointwise(GAMMA, pre + "pwconv2", F, D, ximg=I, y=X, gamma=sd[pre + "gamma"])
        else:
            H, I = (torch.full((B, c, T), float("nan"), device=DEV) for c in (D, F))
            norm(X, pre, True, y=H)
            pointwise(GELU, pre + "pwconv1", D, F, x=H, y=I)
            pointwise(GAMMA, pre + "pwconv2", F, D, x=I, y=X, gamma=sd[pre + "gamma"])
    bins = n_fft // 2 + 1
    S = torch.full((B, T, bins, 2), float("nan"), device=DEV)
    if tc:
        H = _img_out(B, D, T)
        norm(X, "backbone.final_layer_norm.", False, img=H)
        pointwise(SPECTRUM, "head.out", D, 2 * bins, ximg=H, spec=S)
    else:
        Y = torch.full((B, D, T), float("nan"), device=DEV)
        norm(X, "backbone.final_layer_norm.", False, y=Y)
        pointwise(SPECTRUM, "head.out", D, 2 * bins, x=Y, spec=S)
    m = C.c_void_p()
    assert lib.ab_mel_create(C.byref(capi.MelConfig(n_fft, hop, n_fft, 0, 0, 0.0, 0.0)), C.byref(m)) == 0
    try:
        need = lib.ab_istft_workspace_bytes(m, B, T)
        ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
        wav = torch.full((B, 1, T * hop), float("nan"), device=DEV)
        rc = lib.ab_istft_forward(m, P(S), B, T, P(sd["head.istft.window"]), P(wav),
                                  C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need, st)
        assert rc == 0, capi.last_error()
        torch.cuda.synchronize()
    finally:
        lib.ab_mel_destroy(m)
    return wav


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "tc_f16", "tc_bf16"])
@pytest.mark.parametrize("model_id", ["fixture-a", "256-1024"])
def test_forward_is_the_chain_of_single_launches(model_id, prec):
    from test_vocos import _trained_like, build_vocos, load_vocos
    from vocos_oracle import GOLDEN_VOCOS
    if model_id == "fixture-a":
        hp = GOLDEN_VOCOS["a"][0]
        model = build_vocos(hp, load_vocos("a")[1]).cuda()
        B, T = 2, 24
    else:
        hp = dict(input_channels=100, dim=256, intermediate_dim=1024, num_layers=2, n_fft=256, hop_size=64)
        model = _trained_like(build_vocos(hp, seed=61), 62).cuda()
        B, T = 2, 150
    g = torch.Generator().manual_seed(63)
    mel_t = (torch.rand(B, T, hp["input_channels"], generator=g) * 13.5 - 11.5).cuda()
    mel = mel_t.transpose(1, 2)                   # Vevo's vocoder_model(mel.transpose(1, 2))
    assert not mel.is_contiguous()
    model.precision = prec
    with torch.no_grad():
        model(mel)
        model.set_profiling(True)
        want = model(mel)
        prof = model.get_profile()
        model.set_profiling(False)
    on_tc = prof["tc_gemmconv"]["launches"] + prof["tc_conv"]["launches"] == 1
    L = hp["num_layers"]
    assert prof["conv1d_fp32"]["launches"] == (0 if on_tc else 1) + (2 * L + 1 if prec == "fp32" else 0)
    assert on_tc == (prec != "fp32")
    got = _chain(model, mel, prec, on_tc)
    assert torch.isfinite(want).all()
    assert torch.equal(got, want), float((got - want).abs().max())
