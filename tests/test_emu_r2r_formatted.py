"""CPU: out-of-place DCT / DST (formatted inputBuffer / outputBuffer) on the kernel-body emulation, against the oracle.

The data flow is the engine's C2C one: forward, the first axis reads inputBuffer (isInputFormatted) and the last axis writes
outputBuffer (isOutputFormatted); inverse, the first axis reads outputBuffer and the last one writes inputBuffer when
inverseReturnToInputBuffer is set; everything in between lives in `buffer`.  Every case covers one route of the planner
(fused contiguous DCT-II/III, fused strided complex view, long strided Four-Step, composed around a C2C plan, runtime-scheduled
kernel) with every caller buffer between guard bands (tests/layout_util.py).  Each checks: the result against the oracle, the
source bit for bit, every gap and guard, and -- where the launches are those of the in-place plan -- bit identity with the
in-place result.  The scratch is checked against its reported size on the device (tests/test_gpu_r2r_formatted.py)."""
import ctypes

import numpy as np
import pytest

import emu
import layout_util as lu
import vkfft_oracle as orc

T32, T64 = 2e-6, 3e-15          # relative l2 (FP32: the composed real transforms' split / merge step, as in the layout tests)
C_POINT = 6.0


def rdt(prec):
    return np.float32 if prec == 0 else np.float64


def check(got, ref, prec, n_total):
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < (T32 if prec == 0 else T64), e
    eps = np.finfo(rdt(prec)).eps
    r = lu.max_line_error(got, ref)
    assert r <= lu.point_bound(n_total, eps, C_POINT), r / lu.point_bound(n_total, eps, 1.0)


def kernels(desc, inverse):
    """the launches of a plan without their buffer roles"""
    rc, txt = emu.describe(desc, inverse)
    assert rc == 0, rc
    return [line.rsplit("  ", 1)[0] for line in txt.strip().split("\n")]


def strides_of(shape, pad, batch_pad):
    s = lu.packed_strides(shape, shape[0] + pad)
    s[-1] += batch_pad
    return s


# pitches of inputBuffer / buffer / outputBuffer: (row pad, batch pad) -- all even, so that no route is lost to an odd pitch
PITCH = {"input": (2, 6), "buffer": (4, 0), "output": (6, 10)}


def run_plan(shape, batch, prec, inv, roles, x, src_role, **kw):
    """plan with the layouts `roles` ({role: strides}), x in `src_role`; -> ({role: Layout}, desc)"""
    dt = rdt(prec)
    L = {r: lu.make_layout(shape, batch, s, dt) for r, s in roles.items()}
    L[src_role].scatter(x)
    before = {r: l.flat.copy() for r, l in L.items()}
    args = dict(buffer_stride=roles["buffer"])
    if "input" in roles:
        args["input_stride"] = roles["input"]
    if "output" in roles:
        args["output_stride"] = roles["output"]
    args.update(kw)
    d = emu.make_desc(shape, batch, prec, **args)
    data = {r: L[r].data if r in L else None for r in ("buffer", "input", "output")}
    rc, npass = emu.exec_plan(d, inv, data["buffer"], inp=data["input"], out=data["output"])
    assert rc == 0 and npass >= 1, rc
    for r, l in L.items():
        if r == src_role and r != "buffer":
            lu.assert_bit_identical(l.flat, before[r], f"{r} (the source)")
        else:
            lu.assert_untouched(l.flat, before[r], l.mask, l, r)
    return L, d


# combination -> (flags, buffers given, source role, destination role) per direction
def flow(combo, inv):
    if combo == "in":
        return dict(is_input_formatted=1), ("input", "buffer"), ("buffer" if inv == 1 else "input"), "buffer"
    if combo == "out":
        return dict(is_output_formatted=1), ("buffer", "output"), ("output" if inv == 1 else "buffer"), ("buffer" if inv == 1 else "output")
    if combo == "both":
        return (dict(is_input_formatted=1, is_output_formatted=1), ("input", "buffer", "output"),
                ("output" if inv == 1 else "input"), ("buffer" if inv == 1 else "output"))
    assert combo == "back"
    return (dict(is_input_formatted=1, inverse_return_to_input=1), ("input", "buffer"), ("buffer" if inv == 1 else "input"),
            ("input" if inv == 1 else "buffer"))


def r2r_case(mode, kind, shape, batch, prec, combo, inv, normalize=0, omit=None, expect=None):
    flags, given, src, dst = flow(combo, inv)
    kw = {"perform_" + mode: kind, "normalize": normalize, **flags}
    if omit is not None:
        kw["omit_dimension"] = list(omit)
    roles = {r: strides_of(shape, *PITCH[r]) for r in given}
    x = orc.random_input((batch,) + tuple(reversed(shape)), rdt(prec), seed=sum(shape) + kind + batch)
    L, d = run_plan(shape, batch, prec, inv, roles, x, src, **kw)
    keep = [a for a in range(len(shape)) if omit is None or not omit[a]]
    axes = tuple(len(shape) - a for a in keep)
    f = orc.dct if mode == "dct" else orc.dst
    # the oracle over the transformed axes only: move them last
    xm = np.moveaxis(x, axes, tuple(range(x.ndim - len(axes), x.ndim)))
    ref = f(xm, kind, len(axes), inverse=(inv == 1), normalize=bool(normalize))
    ref = np.moveaxis(ref, tuple(range(x.ndim - len(axes), x.ndim)), axes)
    got = L[dst].gather()
    check(got, ref, prec, int(np.prod([shape[a] for a in keep])))
    txt = kernels(d, inv)
    # the in-place plan on the packed layout: the same route, and the same launches give the same bits
    dref = emu.make_desc(shape, batch, prec, **{"perform_" + mode: kind, "normalize": normalize},
                         **({"omit_dimension": list(omit)} if omit is not None else {}))
    tref = kernels(dref, inv)
    if expect is not None:
        assert sum(expect in t for t in txt) == sum(expect in t for t in tref), (expect, txt, tref)
        assert prec == 1 or any(expect in t for t in txt), (expect, txt)      # every route has its FP32 kernels here
    if tref == txt:
        buf = np.ascontiguousarray(x)
        assert emu.exec_plan(dref, inv, buf)[0] == 0
        assert np.array_equal(lu.bits(got), lu.bits(buf)), "out of place differs from in place with the same launches"
        return True
    return False


ROUTES = [
    # (mode, kind, shape, batch, the launch that shows the route)
    ("dct", 2, (64,), 3, "dct axis (fused)"), ("dct", 3, (64,), 3, "dct axis (fused)"),
    ("dct", 2, (1000,), 2, "dct axis (fused)"), ("dct", 3, (4096,), 2, "dct axis (fused)"),
    ("dct", 2, (64, 64), 2, "DCT_COLS"), ("dct", 3, (64, 64), 2, "DCT_COLS"),
    ("dct", 2, (16, 4096), 1, "long dct-i"), ("dct", 3, (16, 4096), 1, "long dct-i"),
    ("dct", 2, (4391,), 2, "r2r (composed)"), ("dst", 3, (4391,), 1, "r2r (composed)"),
    ("dct", 1, (33,), 3, "dct axis"), ("dct", 4, (64,), 3, "dct axis"), ("dct", 4, (45,), 3, "dct axis"),
    ("dst", 1, (100,), 2, "dct axis"), ("dst", 2, (100,), 2, "dct axis"), ("dst", 3, (100,), 2, "dct axis"), ("dst", 4, (100,), 2, "dct axis"),
]


def _rid(r):
    return f"{r[0]}{r[1]}-{'x'.join(map(str, r[2]))}"


@pytest.mark.parametrize("combo", ["in", "out", "both", "back"])
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("route", ROUTES, ids=_rid)
def test_routes_out_of_place(route, prec, combo):
    mode, kind, shape, batch, expect = route
    for inv in (-1, 1):
        if combo == "in" and inv == 1:
            continue                        # isInputFormatted alone: the inverse runs in `buffer`, in place
        r2r_case(mode, kind, shape, batch, prec, combo, inv, normalize=int(inv == 1), expect=expect)


@pytest.mark.parametrize("inv", [-1, 1])
@pytest.mark.parametrize("kind", [2, 3])
def test_720x480_strided_axis(kind, inv):
    r2r_case("dct", kind, (720, 480), 1, 0, "both", inv, expect="DCT_COLS")


@pytest.mark.parametrize("omit", [(0, 1), (1, 0)])
@pytest.mark.parametrize("combo", ["in", "both", "back"])
def test_omit_dimension(omit, combo):
    for inv in (-1, 1):
        if combo == "in" and inv == 1:
            continue
        r2r_case("dct", 2, (64, 32), 2, 0, combo, inv, normalize=1, omit=omit)


def test_same_pitches_same_launches_same_bits():
    """packed formatted buffers: the out-of-place plan lists the in-place plan's launches and computes the same bits"""
    for mode, kind, shape, batch, _ in ROUTES:
        x = orc.random_input((batch,) + tuple(reversed(shape)), np.float32, seed=kind)
        for inv, flags in ((-1, dict(is_input_formatted=1)), (1, dict(is_output_formatted=1))):
            d = emu.make_desc(shape, batch, 0, **{"perform_" + mode: kind}, **flags)
            dref = emu.make_desc(shape, batch, 0, **{"perform_" + mode: kind})
            assert kernels(d, inv) == kernels(dref, inv), (mode, kind, shape)
            src, out, ref = x.copy(), np.zeros_like(x), x.copy()
            args = dict(inp=src) if inv == -1 else dict(out=src)
            assert emu.exec_plan(d, inv, out, **args)[0] == 0
            assert emu.exec_plan(dref, inv, ref)[0] == 0
            assert np.array_equal(src, x) and np.array_equal(lu.bits(out), lu.bits(ref)), (mode, kind, shape, inv)


def test_odd_pitch_leaves_the_complex_view():
    """an odd inputBuffer pitch cannot be read as complex pairs: the strided axis falls to the runtime-scheduled kernel"""
    shape, batch = (64, 32), 2
    kw = dict(perform_dct=2, is_input_formatted=1, input_stride=strides_of(shape, 1, 0))
    txt = kernels(emu.make_desc(shape, batch, 0, **kw), -1)
    assert not any("DCT_COLS" in t for t in txt) and any("generic" in t for t in txt), txt
    roles = {"input": strides_of(shape, 1, 0), "buffer": strides_of(shape, 4, 0)}
    x = orc.random_input((batch,) + tuple(reversed(shape)), np.float32, seed=5)
    L, _ = run_plan(shape, batch, 0, -1, roles, x, "input", perform_dct=2, is_input_formatted=1)
    check(L["buffer"].gather(), orc.dct(x, 2, 2), 0, 64 * 32)


def test_refusals_that_stay():
    buf = np.zeros((2, 64), np.float32)
    # zero padding of a formatted source, half precision, distributed plans
    d = emu.make_desc((64,), 2, 0, perform_dct=2, is_input_formatted=1, perform_zeropadding=[1, 0, 0, 0],
                      zeropad_left=[32, 0, 0, 0], zeropad_right=[64, 0, 0, 0])
    assert emu.exec_plan(d, -1, buf, inp=buf.copy())[0] == 3002
    assert emu.describe(emu.make_desc((64,), 2, 2, perform_dct=2, is_input_formatted=1))[0] == 3002
    assert emu.describe(emu.make_desc((64, 64), 1, 0, perform_dct=2, is_input_formatted=1, dist_world=2, user_temp_buffer=1))[0] == 3002


# ---------------------------------------------------------------- the product planner ----------------------------------------------------------------
def _product_text(L, shape, batch, prec, inverse, **kw):
    d = emu.make_desc(shape, batch, prec, **kw)
    buf = ctypes.create_string_buffer(1 << 15)
    rc = L.b200fft_debug_plan_text(ctypes.byref(d), int(inverse), buf, len(buf))
    return rc, [line.rsplit("  ", 1)[0] for line in buf.value.decode().strip().split("\n")]


@pytest.mark.parametrize("shape,batch,kind", [((8192, 8192), 2, 2), ((720, 480), 1, 2), ((1280, 720), 1, 2), ((300, 300, 300), 1, 2),
                                              ((720, 480), 1, 3), ((1280, 720), 1, 3)])
def test_product_planner_out_of_place_keeps_the_in_place_kernels(shape, batch, kind):
    """with packed formatted buffers the product library (plan-time kernels included) plans the launches of the in-place plan"""
    from vkfft_b200 import _lib
    L = _lib.load()
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here: no plan-time kernels to plan with")
    for inv, flags in ((-1, dict(is_input_formatted=1)), (1, dict(is_output_formatted=1)),
                       (-1, dict(is_input_formatted=1, is_output_formatted=1))):
        rc0, ref = _product_text(L, shape, batch, 0, inv, perform_dct=kind)
        rc1, got = _product_text(L, shape, batch, 0, inv, perform_dct=kind, **flags)
        assert rc0 == 0 and rc1 == 0, (rc0, rc1)
        assert got == ref, (flags, got, ref)
