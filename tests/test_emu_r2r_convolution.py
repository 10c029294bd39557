"""CPU: convolution plans with DCT / DST (performConvolution + performDCT / performDST) on the kernel-body emulation.

VkFFTAppend(app, -1) runs the forward type-k transform on every axis, multiplies every point by the real `kernel` (the
buffer's layout, one plane per coordinate feature, shared by every batch), and runs the inverse transform on every axis in
reverse order (II <-> III, I and IV self-inverse), each inverse axis carrying the R2R plans' normalisation.  The launches are
the R2R plans' own forward passes, one real product launch and their inverse passes; for type 2 on a packed layout with one
kernel set and no matrix the last axis runs DCT-II (DST-II), product and DCT-III (DST-III) as one launch, and that route
agrees with the chain (B200FFT_NO_FUSED_CONV=1) to rounding.  Every caller buffer lies between guard
bands (tests/layout_util.py); each case checks the float64 oracle, the launch count, that the source and the kernel are
unchanged bit for bit, and that nothing outside the logical array is written."""
import os

import numpy as np
import pytest

import emu
import layout_util as lu
import vkfft_oracle as orc

TOL = {0: 1e-6, 1: 1e-12}       # relative l2 against the float64 oracle


def rdt(prec):
    return np.float32 if prec == 0 else np.float64


def oracle(x, K, mode, kind, nd, normalize, M=0, sym=0, NK=1):
    """x: [B, C, ...] float64, K: [planes, ...] float64 -> forward, product, inverse"""
    f = orc.dct if mode == "dct" else orc.dst
    X = f(x, kind, nd)
    C = x.shape[1]
    if M:
        idx = lambda r, c: (min(r, c) * M - min(r, c) * (min(r, c) - 1) // 2 + abs(r - c)) if sym else r * M + c
        kp = M * (M + 1) // 2 if sym else M * M
        Y = np.stack([np.stack([sum(K[k * kp + idx(r, c)] * X[0, c] for c in range(M)) for r in range(M)]) for k in range(NK)])
    elif NK > 1:
        Y = np.stack([X[0] * K[k * C:(k + 1) * C] for k in range(NK)])
    else:
        Y = X * K[None]
    return f(Y, kind, nd, inverse=True, normalize=bool(normalize))


def plan_launches(shape, batch, prec, mode, kind, inv, **kw):
    rc, txt = emu.describe(emu.make_desc(shape, batch, prec, **{"perform_" + mode: kind}, **kw), inv)
    assert rc == 0, rc
    return txt.strip().split("\n")


def conv_case(mode, kind, shape, batch, prec, C=1, M=0, sym=0, NK=1, normalize=1, formatted=False, pad=(0, 0)):
    """one convolution on guarded layouts; pad = (row pad, batch pad) of buffer / inputBuffer / kernel pitches"""
    dt = rdt(prec)
    nd = len(shape)
    strides = lu.packed_strides(shape, shape[0] + pad[0])
    strides[-1] += pad[1]
    # features are batches of the layout: [B * C] lines of planes, the kernel [planes] with the same pitches
    planes = (M * (M + 1) // 2 if sym else M * M) if M else C
    nbuf = max(batch, NK) * C
    x = orc.random_input((batch, C) + tuple(reversed(shape)), dt, seed=sum(shape) + 7 * kind + batch + C)
    k = orc.random_input((planes * NK,) + tuple(reversed(shape)), dt, seed=kind + 3 * C + NK)
    buf = lu.make_layout(shape, nbuf, strides, dt)
    ker = lu.make_layout(shape, planes * NK, strides, dt)
    ker.scatter(k)
    kw = dict(coordinate_features=C, perform_convolution=1, normalize=normalize, buffer_stride=strides)
    if M:
        kw.update(matrix_convolution=M, symmetric_kernel=sym)
    if NK > 1:
        kw["number_kernels"] = NK
    if formatted:
        src = lu.make_layout(shape, batch * C, strides, dt)
        src.scatter(x.reshape((batch * C,) + x.shape[2:]))
        kw.update(is_input_formatted=1, input_stride=strides)
    else:
        buf.view[:batch * C] = x.reshape((batch * C,) + x.shape[2:])
        src = None
    before = {"buffer": buf.flat.copy(), "kernel": ker.flat.copy()}
    if src is not None:
        before["input"] = src.flat.copy()
    d = emu.make_desc(shape, batch, prec, **{"perform_" + mode: kind}, **kw)
    rc, npass = emu.exec_plan(d, -1, buf.data, inp=src.data if src is not None else None, kernel=ker.data)
    assert rc == 0, rc
    lu.assert_bit_identical(ker.flat, before["kernel"], "kernel")
    if src is not None:
        lu.assert_bit_identical(src.flat, before["input"], "inputBuffer (the source)")
    lu.assert_untouched(buf.flat, before["buffer"], buf.mask, buf, "buffer")
    got = buf.gather().reshape((max(batch, NK), C) + x.shape[2:])
    ref = oracle(x.astype(np.float64), k.astype(np.float64), mode, kind, nd, normalize, M, sym, NK)
    if NK > 1:
        ref = ref.reshape(got.shape)
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < TOL[prec], e
    plan_text = listing = emu.describe(d, -1)[1]
    if "fused r2r convolution" in listing:
        # the last axis runs forward, product and inverse in one launch: 2 nd - 1 launches; the chain gives the same numbers
        assert npass == 2 * sum(n > 1 for n in shape) - 1, (npass, listing)
        os.environ["B200FFT_NO_FUSED_CONV"] = "1"
        try:
            chain = buf.flat.copy()
            chain[buf.guard:][...] = before["buffer"][buf.guard:]
            rc, npass = emu.exec_plan(d, -1, chain[buf.guard:], inp=src.data if src is not None else None, kernel=ker.data)
            listing = emu.describe(d, -1)[1]
        finally:
            os.environ.pop("B200FFT_NO_FUSED_CONV")
        assert rc == 0 and "fused r2r convolution" not in listing
        e = orc.error_metrics(got, lu.Layout(chain, shape, nbuf, strides, buf.guard).gather().reshape(got.shape))["l2_rel"]
        assert e < TOL[prec], e
    # the chain: the R2R plan's forward launches, one product launch, its inverse launches (on every output batch)
    lay = dict(coordinate_features=C, buffer_stride=strides)
    fwd = plan_launches(shape, batch, prec, mode, kind, -1, **lay, **(dict(is_input_formatted=1, input_stride=strides) if formatted else {}))
    back = plan_launches(shape, max(batch, NK), prec, mode, kind, 1, normalize=normalize, **lay)
    assert npass == len(fwd) + 1 + len(back), (npass, len(fwd), len(back))
    assert sum("real spectrum x kernel" in t for t in listing.split("\n")) == 1, listing
    return plan_text


TYPES = [("dct", 1), ("dct", 2), ("dct", 3), ("dct", 4), ("dst", 1), ("dst", 2), ("dst", 3), ("dst", 4)]
SHAPES = [((64,), 3), ((32, 24), 2), ((16, 8, 12), 1)]


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("shape,batch", SHAPES, ids=lambda s: "x".join(map(str, s)) if isinstance(s, tuple) else str(s))
@pytest.mark.parametrize("mode,kind", TYPES, ids=lambda t: str(t))
def test_every_type(mode, kind, shape, batch, prec):
    conv_case(mode, kind, shape, batch, prec)


@pytest.mark.parametrize("mode,kind,shape,batch", [
    ("dct", 2, (45, 16), 1),            # odd nx: no complex view of column pairs
    ("dst", 2, (45, 16), 1),
    ("dct", 2, (262, 8), 1),            # 262 = 2 * 131: the composed route on the lower axis
    ("dct", 3, (16, 262), 1),           # ... and on the last axis
    ("dct", 2, (1000,), 3),             # a non-power-of-two length
    ("dct", 2, (16, 4096), 1),          # long strided last axis (three-launch Four-Step)
    ("dct", 4, (45,), 5),
])
def test_routes(mode, kind, shape, batch):
    conv_case(mode, kind, shape, batch, 0)


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("mode,kind", [("dct", 2), ("dst", 2), ("dct", 1), ("dst", 4)])
def test_padded_pitches(mode, kind, prec):
    conv_case(mode, kind, (24, 10), 3, prec, pad=(4, 6))
    conv_case(mode, kind, (12, 6, 5), 2, prec, C=2, pad=(2, 10))


@pytest.mark.parametrize("normalize", [0, 1])
@pytest.mark.parametrize("prec", [0, 1])
def test_features_and_normalize(prec, normalize):
    conv_case("dct", 2, (32, 16), 3, prec, C=2, normalize=normalize)
    conv_case("dst", 1, (40,), 2, prec, C=3, normalize=normalize)


@pytest.mark.parametrize("M,sym", [(2, 0), (2, 1), (3, 0), (3, 1)])
@pytest.mark.parametrize("mode,kind", [("dct", 2), ("dst", 3)])
def test_matrix_kernel(mode, kind, M, sym):
    conv_case(mode, kind, (32, 12), 1, 0, C=M, M=M, sym=sym)


@pytest.mark.parametrize("M,sym", [(0, 0), (2, 1)])
def test_number_kernels(M, sym):
    conv_case("dct", 2, (24, 8), 1, 0, C=M or 1, M=M, sym=sym, NK=2)


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("mode,kind", [("dct", 2), ("dct", 4), ("dst", 1)])
def test_input_formatted(mode, kind, prec):
    conv_case(mode, kind, (32, 20), 3, prec, C=1, formatted=True)
    conv_case(mode, kind, (20, 6, 8), 1, prec, C=2, formatted=True, pad=(2, 4))
    conv_case(mode, kind, (16, 64), 3, prec, C=1, formatted=True)          # type 2: the fused last axis after a formatted first axis


def test_ones_kernel_returns_the_source():
    """normalize = 1: the inverse undoes the forward, so a kernel of ones is the identity (to rounding)"""
    x = orc.random_input((2, 48, 64), np.float64, seed=3)
    for mode, kind in TYPES:
        buf = x.copy()
        d = emu.make_desc((64, 48), 2, 1, **{"perform_" + mode: kind}, perform_convolution=1, normalize=1)
        assert emu.exec_plan(d, -1, buf, kernel=np.ones((48, 64)))[0] == 0
        assert orc.error_metrics(buf, x)["l2_rel"] < 1e-13, (mode, kind)


def test_kernel_application_is_an_ordinary_forward_plan():
    """kernelConvolution = 1 with performDCT / performDST: the forward transform of the kernel array, nothing else"""
    x = orc.random_input((2, 24, 32), np.float32, seed=4)
    for mode, kind in (("dct", 2), ("dst", 4)):
        a, b = x.copy(), x.copy()
        assert emu.exec_plan(emu.make_desc((32, 24), 2, 0, **{"perform_" + mode: kind}, kernel_convolution=1), -1, a)[0] == 0
        assert emu.exec_plan(emu.make_desc((32, 24), 2, 0, **{"perform_" + mode: kind}), -1, b)[0] == 0
        assert np.array_equal(lu.bits(a), lu.bits(b))


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("mode", ["dct", "dst"])
@pytest.mark.parametrize("shape,batch", [((64,), 3), ((256,), 5), ((512,), 1), ((64, 64), 2), ((16, 256), 1), ((12, 10, 64), 1),
                                         ((8, 4, 256), 2)])
def test_fused_last_axis(mode, shape, batch, prec):
    """type 2, packed, one kernel set: the last axis runs DCT-II (DST-II), product and DCT-III (DST-III) in one launch.
    An odd number of real lines leaves the last complex line with one real line."""
    listing = conv_case(mode, 2, shape, batch, prec, C=1 if batch % 2 else 2)
    assert prec == 1 or "fused r2r convolution" in listing, listing


def test_refusals():
    buf = np.zeros((2, 64, 64), np.float32)
    base = dict(perform_dct=2, perform_convolution=1)
    for kw in (dict(conjugate_convolution=1), dict(conjugate_convolution=2), dict(cross_power_spectrum_normalization=1),
               dict(is_output_formatted=1), dict(omit_dimension=[1, 0]), dict(omit_dimension=[0, 1])):
        d = emu.make_desc((64, 64), 2, 0, **base, **kw)
        assert emu.exec_plan(d, -1, buf, inp=buf.copy(), out=buf.copy(), kernel=buf[0].copy())[0] == 3002, kw
    assert emu.describe(emu.make_desc((64, 64), 1, 2, **base))[0] == 3002                                      # half storage
    assert emu.describe(emu.make_desc((64, 64), 1, 0, **base, dist_world=2, user_temp_buffer=1))[0] == 3002    # distributed
    assert emu.describe(emu.make_desc((64, 64), 1, 0, perform_dst=2, perform_convolution=1, dist_world=2, user_temp_buffer=1))[0] == 3002
