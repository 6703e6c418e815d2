"""Single launches of the tensor-core convolution (`launch_tc_conv` through `ab_tc_conv_forward`) against the
operand-rounded oracle (tests/resblock_oracle.py), bit for bit, fp32 output and operand image both.

* ConvTranspose1d on `hitem_kernel` (operand image in) and on `hconv_kernel` (fp32 input, lrelu and rounding in the
  loader), one-hot weights: every output is one exact product plus the bias, so both kernels must equal the oracle
  exactly.  The cases reach each specialisation of the polyphase epilogue (`epilogue_convt`): u = 8 (no exchange),
  u = 4 (a shfl.xor 2 exchange and prmt packing), u = 2 (the quad transpose; with odd padding the fp32 pairs across
  rows, including the warp's rows 7 -> 8 and its unpaired rows 0 and 15) and the generic path (u = 3, 5, 6, 10, odd
  padding at u = 4), with several N blocks, partial N blocks and K chunks, short and ragged sequences and a walk of
  more than two items per SM.
* Conv1d (mode 0) on `hconv_kernel`: conv_pre from a transposed mel view emitting the image (padding channels zero),
  ReflectionPad1d (MelGAN), image input, and the epilogue's (((conv + bias) + residual) + acc_prev) * (1 / out_div).
* Dense weights: a ConvTranspose on `hitem_kernel` from an image equals the same layer on `hconv_kernel` from the fp32
  input that rounds to the same operands, bit for bit (both accumulate K chunk -> tap -> k16 half, DESIGN.md §4.1),
  and both sit within the floor rule of test_resblock_exact.py of the float64 oracle.

Output buffers are filled with NaN / 0xFFFF before each launch, so an element that is not written fails."""
import ctypes as C

import numpy as np
import pytest
import torch

import resblock_oracle as ro

DEV = "cuda:0"
PRECS = {"tc_f16": "f16", "tc_bf16": "bf16"}
IMG_SLOPE = 0.1
FLOOR_MEAN, FLOOR_MAX = 2.0, 3.0   # test_resblock_exact.py's floor rule
VALUES = {   # input scale, weight exponents, bias std
    "ordinary": (2.0, (-2, -1, 0, 1), 0.5),
    "saturation": (3e4, (0, 1, 2), 1.0),         # f16: |x| and |y| past 65504, the image holds +-65504
    "subnormal": (1e-5, (-3, -2, -1, 0), 1e-6),  # f16: operands and products below 2^-14
}


# ------------------------------------------------------------------------------------------------ the harness
def _run(mode, prec, w, bias, B, cin, cout, T, k, d_or_u, *, x=None, pre_slope=1.0, ximg=None, pad=-1, residual=None,
         acc_prev=None, out_div=1.0, reflect=0, emit_image=False):
    """One ab_tc_conv_forward.  x: fp32 tensor on the device (any strides) or None; ximg: operand image (numpy uint16)
    or None; w, bias, residual, acc_prev: numpy.  -> (rc, y, yimg or None), y and yimg on the host."""
    from amphion_b200 import _capi
    lib = _capi.lib
    Tout = T * d_or_u if mode == 1 else T
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)  # noqa: E731
    wd, bd, rd, ad = dev(w), dev(bias), dev(residual), dev(acc_prev)
    xi = None if ximg is None else torch.from_numpy(np.ascontiguousarray(ximg).view(np.int16)).to(DEV)
    y = torch.full((B, cout, Tout), float("nan"), device=DEV)
    yimg = (torch.full((B, (cout + 15) // 16 * 2, Tout, 8), -1, dtype=torch.int16, device=DEV) if emit_image else None)
    need = lib.ab_tc_conv_workspace_bytes(mode, cin, cout, k, d_or_u)
    ws = torch.empty(need + 256, dtype=torch.uint8, device=DEV)
    rc = lib.ab_tc_conv_forward(mode, _capi.ptr(x), None if x is None else _capi.shape_array(x.stride()), pre_slope,
                                _capi.ptr(xi), _capi.ptr(wd), _capi.ptr(bd), _capi.ptr(rd), _capi.ptr(ad), out_div, reflect,
                                _capi.ptr(y), _capi.ptr(yimg), IMG_SLOPE, B, cin, cout, T, k, d_or_u, pad,
                                _capi.PRECISIONS[prec], C.c_void_p((ws.data_ptr() + 255) // 256 * 256), need,
                                _capi.stream_ptr())
    torch.cuda.synchronize()
    return rc, y.cpu().numpy(), None if yimg is None else yimg.cpu().numpy().view(np.uint16)


def _assert_equal(what, got, want):
    bad = got != want
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}: "
                           f"{got[bad][0]!r} vs {want[bad][0]!r}")


def _check(what, prec, y, yimg, want, cout):
    """y bit-equal to want; the image holds the bits of rnd(lrelu(want, IMG_SLOPE)) and zero padding channels."""
    assert np.isfinite(want).all(), what
    _assert_equal(f"{what} y", y, want)
    if yimg is not None:
        bits, padding = ro.from_image(yimg, cout)
        _assert_equal(f"{what} image", bits, ro.image_bits(want, IMG_SLOPE, PRECS[prec]))
        assert not padding.any(), f"{what}: padding channels of the image are not zero"


def _input(rng, B, C, T, scale):
    return (rng.normal(0, 1, (B, C, T)) * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------------ CPU: the oracle
@pytest.mark.parametrize("cin,cout,k,u,pad", [(40, 24, 16, 8, 4), (48, 16, 10, 5, 3), (16, 8, 6, 3, 2), (20, 12, 4, 2, 1),
                                              (32, 16, 10, 4, 3), (16, 16, 2, 2, 0), (33, 7, 20, 10, 0)])
def test_one_hot_convt_gather_equals_dense(cin, cout, k, u, pad):
    rng = np.random.default_rng(cin * k)
    a = ro.rnd(rng.normal(0, 1, (2, cin, 9)), "bf16")
    w = ro.random_one_hot_t(rng, cin, cout, k, u, (-3, 0, 2))
    assert (np.count_nonzero(w.dense(), axis=(0,)) <= 1).all() and np.count_nonzero(w.dense()) == cout * u
    want = ro.conv_transpose(a, w, u, pad)
    for acc in ("f64", "f32", "mma"):
        assert np.array_equal(ro.conv_transpose(a, w.dense(), u, pad, acc), want), acc


@pytest.mark.parametrize("k,u,pad", [(16, 8, 4), (8, 4, 2), (4, 2, 1), (6, 2, 2), (10, 5, 3), (6, 3, 2), (12, 6, 3),
                                     (20, 10, 5), (10, 4, 3), (7, 3, 2)])
def test_convt_matches_torch_with_output_padding(k, u, pad):
    """T_out = T u: torch's ConvTranspose1d with padding pad and output_padding u + 2 pad - k."""
    rng = np.random.default_rng(k * u + pad)
    a = rng.normal(0, 1, (2, 20, 11)).astype(np.float32)
    w = rng.normal(0, 1, (20, 12, k)).astype(np.float32)
    want = torch.nn.functional.conv_transpose1d(torch.from_numpy(a).double(), torch.from_numpy(w).double(), stride=u,
                                                padding=pad, output_padding=u + 2 * pad - k).numpy()
    assert want.shape[2] == 11 * u
    for acc in ("f64", "f32", "mma"):
        got = ro.conv_transpose(a, w, u, pad, acc)
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), acc


@pytest.mark.parametrize("k,d,T", [(7, 1, 4), (3, 9, 10), (7, 1, 40), (3, 3, 7)])
def test_reflect_conv_matches_torch(k, d, T):
    rng = np.random.default_rng(k * d + T)
    a = rng.normal(0, 1, (2, 6, 20))[:, :, :T].astype(np.float32)      # a strided view
    w = rng.normal(0, 1, (5, 6, k)).astype(np.float32)
    h = (k - 1) * d // 2
    want = torch.nn.functional.conv1d(torch.nn.ReflectionPad1d(h)(torch.from_numpy(a).double()),
                                      torch.from_numpy(w).double(), dilation=d).numpy()
    for acc in ("f64", "f32", "mma"):
        got = ro.conv(a, w, d, acc, reflect=True)
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), acc
    oh = ro.random_one_hot(rng, 5, 6, k, (0, 1))
    assert np.array_equal(ro.conv(a, oh, d, reflect=True), ro.conv(a, oh.dense(), d, "mma", reflect=True))


def test_image_bits_are_torch_casts():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.normal(0, 1, 4000), rng.normal(0, 1e-5, 2000), rng.normal(0, 3e4, 2000), [0.0, -0.0],
                        [1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -8, -(1 + 3 * 2 ** -8)]]).astype(np.float32)
    act = torch.from_numpy(ro.lrelu(v, 0.1))
    ok = np.abs(act.numpy()) <= 65504
    assert np.array_equal(ro.image_bits(v, 0.1, "f16")[ok], act.half().view(torch.int16).numpy().view(np.uint16)[ok])
    assert np.array_equal(ro.image_bits(v, 0.1, "bf16"), act.bfloat16().view(torch.int16).numpy().view(np.uint16))
    assert ro.image_bits(np.float32([1e6, -1e6]), 1.0, "f16").tolist() == [0x7BFF, 0xFBFF]   # +-65504, not inf
    bits = ro.image_bits(rng.normal(0, 1, (2, 24, 5)), 0.1, "f16")
    img = ro.to_image(bits)
    assert img.shape == (2, 4, 5, 8)
    back, padding = ro.from_image(img, 24)
    assert np.array_equal(back, bits) and padding.shape == (2, 8, 5) and not padding.any()


# ------------------------------------------------------------------------------------------------ GPU: ConvTranspose
# (id, C_in, C_out, k, u, pad, B, T, values)
CONVT = [
    ("u8-512-256", 512, 256, 16, 8, 4, 2, 150, "ordinary"),    # 8 N blocks, 16 K chunks
    ("u8-256-128", 256, 128, 16, 8, 4, 2, 200, "ordinary"),
    ("u4", 128, 64, 8, 4, 2, 2, 300, "ordinary"),
    ("u4-partial-nblock", 32, 80, 8, 4, 2, 2, 150, "ordinary"),   # N blocks of 64 and 16 channels
    ("u2-odd", 64, 32, 4, 2, 1, 2, 700, "ordinary"),             # tiles of 256 rows, ragged
    ("u2-odd-256", 256, 128, 4, 2, 1, 2, 300, "ordinary"),       # N = 256: one m64 tile per warpgroup
    ("u2-k2-p0", 32, 16, 2, 2, 0, 2, 100, "ordinary"),
    ("u2-k6-p2", 64, 32, 6, 2, 2, 2, 333, "ordinary"),
    ("u4-odd-pad", 64, 32, 10, 4, 3, 2, 150, "ordinary"),        # the generic path with an image out
    ("u5-facodec", 64, 32, 10, 5, 3, 2, 120, "ordinary"),
    ("u3-melgan", 32, 16, 6, 3, 2, 2, 100, "ordinary"),          # output_padding 1
    ("u6", 32, 16, 12, 6, 3, 2, 60, "ordinary"),
    ("u10", 32, 16, 20, 10, 5, 2, 40, "ordinary"),
    ("u8-cout40", 32, 40, 16, 8, 4, 2, 50, "ordinary"),          # C_out % 16 != 0, a partial last N block: fp32 only
    ("u2-odd-cout24", 64, 24, 4, 2, 1, 2, 90, "ordinary"),
    ("u8-cin16", 16, 32, 16, 8, 4, 2, 70, "ordinary"),           # one partial K chunk
    ("u4-cin48", 48, 32, 8, 4, 2, 2, 70, "ordinary"),            # a full and a partial K chunk
    ("u8-T1", 32, 16, 16, 8, 4, 3, 1, "ordinary"),
    ("u2-short", 32, 16, 4, 2, 1, 2, 5, "ordinary"),             # T_out shorter than one tile
    ("u8-walk", 512, 256, 16, 8, 4, 12, 300, "ordinary"),        # 12 x 3 tiles x 8 N blocks = 288 items
    ("u8-saturation", 64, 32, 16, 8, 4, 2, 80, "saturation"),
    ("u4-saturation", 64, 32, 8, 4, 2, 2, 80, "saturation"),
    ("u2-odd-saturation", 64, 32, 4, 2, 1, 2, 80, "saturation"),
    ("u8-subnormal", 64, 32, 16, 8, 4, 2, 80, "subnormal"),
    ("u2-odd-subnormal", 64, 32, 4, 2, 1, 2, 80, "subnormal"),
    ("u5-subnormal", 64, 32, 10, 5, 3, 2, 80, "subnormal"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", CONVT, ids=[c[0] for c in CONVT])
def test_one_hot_convt_is_exact(case, prec):
    name, cin, cout, k, u, pad, B, T, values = case
    scale, exps, bias_std = VALUES[values]
    rng = np.random.default_rng(cin * 7 + cout * 13 + k * u + T)
    w = ro.random_one_hot_t(rng, cin, cout, k, u, exps)
    bias = rng.normal(0, bias_std, cout).astype(np.float32)
    x = _input(rng, B, cin, T, scale)
    act = ro.rnd(ro.lrelu(x, IMG_SLOPE), PRECS[prec])
    want = ro.conv_transpose(act, w.rounded(PRECS[prec]), u, pad) + bias[None, :, None]
    emit = cout % 16 == 0
    runs = [("hconv_kernel", dict(x=torch.from_numpy(x).to(DEV), pre_slope=IMG_SLOPE))]
    if cin % 16 == 0:
        runs.append(("hitem_kernel", dict(ximg=ro.to_image(ro.image_bits(x, IMG_SLOPE, PRECS[prec])))))
    for kernel, src in runs:
        rc, y, yimg = _run(1, prec, w.dense(), bias, B, cin, cout, T, k, u, pad=pad, emit_image=emit, **src)
        assert rc == 0, (kernel, rc)
        _check(f"{name} {kernel}", prec, y, yimg, want, cout)


# ------------------------------------------------------------------------------------------------ GPU: Conv1d
@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("n_mel,cout", [(80, 512), (100, 24)])
def test_one_hot_conv_pre_from_a_transposed_mel(n_mel, cout, prec):
    """conv_pre (k = 7) of a [B, T, n_mel] tensor seen as [B, n_mel, T], emitting the image of lrelu(y, 0.1); at
    C_out = 24 the image has padding channels 24..31."""
    rng = np.random.default_rng(n_mel + cout)
    w = ro.random_one_hot(rng, cout, n_mel, 7, (-2, -1, 0, 1))
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    B, T = 2, 333
    mel_t = _input(rng, B, T, n_mel, 2.0)
    x = torch.from_numpy(mel_t).to(DEV).transpose(1, 2)
    want = ro.conv(ro.rnd(mel_t.transpose(0, 2, 1), PRECS[prec]), w.rounded(PRECS[prec]), 1) + bias[None, :, None]
    rc, y, yimg = _run(0, prec, w.dense(), bias, B, n_mel, cout, T, 7, 1, x=x, emit_image=True)
    assert rc == 0
    _check(f"conv_pre {n_mel} -> {cout}", prec, y, yimg, want, cout)


# (id, C_in, C_out, k, d, B, T, image input)
REFLECT = [
    ("k7-T4", 16, 32, 7, 1, 2, 4, False),
    ("k3-d9-T10", 32, 32, 3, 9, 2, 10, False),
    ("k7-ragged", 48, 40, 7, 1, 2, 1100, False),      # tiles of 256 rows
    ("k3-d3-image", 32, 32, 3, 3, 2, 600, True),
    ("k7-T4-image", 24, 16, 7, 1, 2, 4, True),        # padding channels in the input image
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", REFLECT, ids=[c[0] for c in REFLECT])
def test_one_hot_reflect_conv_is_exact(case, prec):
    name, cin, cout, k, d, B, T, image = case
    rng = np.random.default_rng(cin + k * d + T)
    w = ro.random_one_hot(rng, cout, cin, k, (-2, -1, 0, 1))
    bias = rng.normal(0, 0.5, cout).astype(np.float32)
    x = _input(rng, B, cin, T, 2.0)
    slope = 0.2                                       # MelGAN's leaky_relu
    want = ro.conv(ro.rnd(ro.lrelu(x, slope), PRECS[prec]), w.rounded(PRECS[prec]), d, reflect=True) + bias[None, :, None]
    src = (dict(ximg=ro.to_image(ro.image_bits(x, slope, PRECS[prec]))) if image
           else dict(x=torch.from_numpy(x).to(DEV), pre_slope=slope))
    rc, y, yimg = _run(0, prec, w.dense(), bias, B, cin, cout, T, k, d, reflect=1, emit_image=True, **src)
    assert rc == 0
    _check(f"reflect {name}", prec, y, yimg, want, cout)


@pytest.mark.gpu
def test_reflection_longer_than_the_sequence_is_refused():
    """ReflectionPad1d(3) of 3 samples: AB_ERR_ARG and nothing written."""
    from amphion_b200 import _capi
    rng = np.random.default_rng(1)
    w = rng.normal(0, 0.1, (16, 16, 7)).astype(np.float32)
    x = torch.from_numpy(_input(rng, 2, 16, 3, 1.0)).to(DEV)
    rc, y, yimg = _run(0, "tc_f16", w, None, 2, 16, 16, 3, 7, 1, x=x, reflect=1, emit_image=True)
    assert rc == -1 and "reflection" in _capi.last_error(), (rc, _capi.last_error())
    assert np.isnan(y).all() and (yimg == 0xFFFF).all()
    rc, y, _ = _run(0, "tc_f16", w, None, 2, 16, 16, 4, 7, 1, x=torch.from_numpy(_input(rng, 2, 16, 4, 1.0)).to(DEV),
                    reflect=1)
    assert rc == 0 and np.isfinite(y).all()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("image", [False, True], ids=["fp32-in", "image-in"])
def test_one_hot_conv_epilogue_association(image, prec):
    """y = (((conv + bias) + residual) + acc_prev) * (1 / out_div), the terms of different magnitudes so that another
    association moves the last bits."""
    rng = np.random.default_rng(5 + image)
    B, C, T, k, d = 2, 64, 500, 5, 2
    w = ro.random_one_hot(rng, C, C, k, (-2, -1, 0, 1))
    bias = rng.normal(0, 0.5, C).astype(np.float32)
    x = _input(rng, B, C, T, 2.0)
    res = _input(rng, B, C, T, 3e2)
    prev = _input(rng, B, C, T, 1e-2)
    want = ro.conv(ro.rnd(ro.lrelu(x, IMG_SLOPE), PRECS[prec]), w.rounded(PRECS[prec]), d) + bias[None, :, None]
    want = ((want + res) + prev) * (np.float32(1.0) / np.float32(3.0))
    src = (dict(ximg=ro.to_image(ro.image_bits(x, IMG_SLOPE, PRECS[prec]))) if image
           else dict(x=torch.from_numpy(x).to(DEV), pre_slope=IMG_SLOPE))
    rc, y, yimg = _run(0, prec, w.dense(), bias, B, C, C, T, k, d, residual=res, acc_prev=prev, out_div=3.0,
                       emit_image=True, **src)
    assert rc == 0
    _check("residual + acc_prev + out_div", prec, y, yimg, want, C)


# ------------------------------------------------------------------------------------------------ GPU: dense
# (id, C_in, C_out, k, u, pad, B, T)
DENSE = [
    ("u8", 256, 128, 16, 8, 4, 2, 200),
    ("u4", 128, 64, 8, 4, 2, 2, 300),
    ("u2-odd", 64, 32, 4, 2, 1, 2, 700),
    ("u5", 64, 32, 10, 5, 3, 2, 200),
]


def _floor_check(what, got, o64, o32):
    e_mean, e_max, f_mean, f_max = ro.floor_stats(got, o64, o32)
    print(f"{what}: mean {e_mean:.3e} = {e_mean / f_mean:.2f} x floor {f_mean:.3e}; "
          f"max {e_max:.3e} = {e_max / f_max:.2f} x floor {f_max:.3e}")
    assert e_mean <= FLOOR_MEAN * f_mean and e_max <= FLOOR_MAX * f_max, what


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("case", DENSE, ids=[c[0] for c in DENSE])
def test_dense_convt_hitem_equals_hconv(case, prec):
    name, cin, cout, k, u, pad, B, T = case
    rng = np.random.default_rng(cin + k + T)
    w = rng.normal(0, 1 / np.sqrt(cin * k / u), (cin, cout, k)).astype(np.float32)
    bias = rng.normal(0, 0.1, cout).astype(np.float32)
    x = _input(rng, B, cin, T, 1.0)
    rc, y_conv, img_conv = _run(1, prec, w, bias, B, cin, cout, T, k, u, pad=pad, x=torch.from_numpy(x).to(DEV),
                                pre_slope=IMG_SLOPE, emit_image=True)
    assert rc == 0
    rc, y_item, img_item = _run(1, prec, w, bias, B, cin, cout, T, k, u, pad=pad, emit_image=True,
                                ximg=ro.to_image(ro.image_bits(x, IMG_SLOPE, PRECS[prec])))
    assert rc == 0
    _assert_equal(f"{name}: hitem_kernel y against hconv_kernel", y_item, y_conv)
    _assert_equal(f"{name}: hitem_kernel image against hconv_kernel", img_item, img_conv)
    act = ro.rnd(ro.lrelu(x, IMG_SLOPE), PRECS[prec])
    o64, o32 = (ro.conv_transpose(act, ro.rnd(w, PRECS[prec]), u, pad, acc) + bias[None, :, None] for acc in ("f64", "mma"))
    assert np.isfinite(y_conv).all()
    _floor_check(f"{name} {prec}", y_conv, o64, o32)
