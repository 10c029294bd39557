"""CPU: padded and user-strided buffer layouts (bufferStride, inputBufferStride, outputBufferStride, omitDimension) on the
kernel-body emulation, against the oracle.

Every buffer is allocated with guard bands, and the guards and every gap between rows, planes and batches hold a NaN
sentinel (tests/layout_util.py): a transform that reads a gap poisons its result, a transform that stores outside its
footprint changes a bit pattern.  The scratch users also run launch by launch on a guarded scratch buffer of exactly the size
the plan asks for.
Addressing must not change arithmetic: where the plan's launches are the same, the padded run equals the packed run bit
for bit."""
import numpy as np
import pytest

import emu
import layout_util as lu
import vkfft_oracle as orc

T32, T64 = 8e-7, 3e-15          # relative l2, as in tests/test_emu_transforms.py
# per point: max|got - ref| <= C_POINT * eps * sqrt(log2 N) * max|ref| of the line.  The largest value seen over this file is
# 1.55 x eps x sqrt(log2 N) (printed with -s); a wrong point is off by ~1/eps times that.
C_POINT = 6.0
R_R2C, R_OMIT = 3003, 3005
observed = {"worst": 0.0}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print(f"\nlargest per-point error seen: {observed['worst']:.2f} x eps x sqrt(log2 N)")


def cdt(prec):
    return np.complex64 if prec == 0 else np.complex128


def rdt(prec):
    return np.float32 if prec == 0 else np.float64


def check(got, ref, prec, n_total, l2=None):
    tol = (T32 if prec == 0 else T64) if l2 is None else l2
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < tol, e
    eps = np.finfo(rdt(prec)).eps
    r = lu.max_line_error(got, ref)
    observed["worst"] = max(observed["worst"], r / lu.point_bound(n_total, eps, 1.0))
    assert r <= lu.point_bound(n_total, eps, C_POINT), r / lu.point_bound(n_total, eps, 1.0)


def launches(desc, inverse):
    rc, txt = emu.describe(desc, inverse)
    assert rc == 0, rc
    return txt


def kernels_of(txt):
    """the launches of a plan listing: kernel, tile shape, grid and threads of each"""
    return txt.strip().split("\n")


def run_inplace(shape, batch, prec, inv, strides, x=None, dtype=None, **kw):
    """scatter x into a guarded layout with `strides` (None: packed), transform in place, check the gaps and guards;
    -> (x, result as a dense array, number of launches, desc)"""
    dt = cdt(prec) if dtype is None else dtype
    if x is None:
        x = orc.random_input((batch,) + tuple(reversed(shape)), dt, seed=sum(shape) + batch)
    st = lu.packed_strides(shape) if strides is None else list(strides)
    L = lu.make_layout(shape, batch, st, dt)
    L.scatter(x)
    before = L.flat.copy()
    d = emu.make_desc(shape, batch, prec, **(dict(buffer_stride=st) if strides is not None else {}), **kw)
    rc, npass = emu.exec_plan(d, inv, L.data)
    assert rc == 0, rc
    lu.assert_untouched(L.flat, before, L.mask, L)
    return x, L.gather(), npass, d


def c2c_case(shape, batch, prec, inv, strides, same_bits_as_packed=False, **kw):
    x, got, npass, d = run_inplace(shape, batch, prec, inv, strides, **kw)
    check(got, orc.c2c(x, len(shape), inv == 1), prec, int(np.prod(shape)))
    if same_bits_as_packed:
        _, packed, npass_p, dp = run_inplace(shape, batch, prec, inv, None, x=x, **kw)
        if kernels_of(launches(d, inv)) == kernels_of(launches(dp, inv)):
            assert np.array_equal(lu.bits(got.reshape(-1)), lu.bits(packed.reshape(-1))), "the pitch changed the arithmetic"
        else:
            assert orc.error_metrics(got, packed)["l2_rel"] < (T32 if prec == 0 else T64)
    return npass, d


# ---------------------------------------------------------------- 1-D C2C ----------------------------------------------------------------
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("inv", [-1, 1])
@pytest.mark.parametrize("pad", ["+1", "+3", "x2"])
@pytest.mark.parametrize("n", [8, 16, 32])
def test_short_lines_ragged_batch(n, pad, inv, prec):
    """the staged short-line kernels gather 128 lines per tile: 130 lines leave a ragged second tile, a pitch != N takes the
    per-line gather instead of the dense copy"""
    pitch = {"+1": n + 1, "+3": n + 3, "x2": 2 * n}[pad]
    c2c_case((n,), 130, prec, inv, [pitch], same_bits_as_packed=(pad == "+1"))


@pytest.mark.parametrize("prec,pad", [(0, 1), (0, 2), (0, 16), (1, 1), (1, 16)])
@pytest.mark.parametrize("inv", [-1, 1])
@pytest.mark.parametrize("n", [64, 1000, 4096])
def test_single_pass_rows(n, inv, prec, pad):
    """pitch N+1: lines only 8-byte aligned (FP32); N+2: 16-byte; N+16: 128-byte"""
    c2c_case((n,), 5, prec, inv, [n + pad], same_bits_as_packed=(pad == 1 and inv == -1))


@pytest.mark.parametrize("pad", [2, 1])
def test_16384_points_pipelined_kernel(pad):
    """pitch N+2: aligned lines, one bulk copy per line; N+1: the unaligned stand-in kernel"""
    c2c_case((16384,), 3, 0, -1, [16384 + pad], same_bits_as_packed=True)


@pytest.mark.parametrize("pad", [2, 1])
@pytest.mark.parametrize("split", ["8,2048", "2048,8"])
def test_four_step_with_a_2048_point_pass(split, pad, monkeypatch):
    monkeypatch.setenv("B200FFT_MAX_SINGLE_PASS", "4096")
    monkeypatch.setenv("B200FFT_FOUR_STEP_SPLIT", split)
    n = 16384
    npass, d = c2c_case((n,), 2, 0, -1, [n + pad])
    assert npass == 2


@pytest.mark.parametrize("n,split,batch", [(1 << 15, None, 2), (10 ** 4, "100,100", 3)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_four_step_padded_batch_pitch_keeps_two_launches(n, split, batch, inv, monkeypatch):
    """the fused and the cluster Four-Step launches assume sequences back to back: with a padded batch pitch the plan is the
    two stand-alone launches"""
    if split:
        monkeypatch.setenv("B200FFT_MAX_SINGLE_PASS", "1024")
        monkeypatch.setenv("B200FFT_FOUR_STEP_SPLIT", split)
    monkeypatch.setenv("B200FFT_FUSED4", "1")
    npass, d = c2c_case((n,), batch, 0, inv, [n + 8], same_bits_as_packed=(split is not None and inv == -1))
    txt = launches(d, inv)
    assert npass == 2 and "fused" not in txt and "cluster" not in txt, txt


def planned_scratch_bytes(shape, batch, prec, **kw):
    """the scratch a plan needs: the smallest tempBufferSize its creation accepts with userTempBuffer = 1 (0: none)"""
    def accepted(nbytes):
        return emu.describe(emu.make_desc(shape, batch, prec, user_temp_buffer=1, temp_buffer_size=nbytes, **kw))[0] == 0
    lo, hi = 0, 1 << 40                    # every size in (lo, hi] ... accepted(hi); 1 byte stands for "no scratch at all"
    assert accepted(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (lo, mid) if accepted(mid) else (mid, hi)
    return 0 if hi == 1 else hi


@pytest.mark.parametrize("n,batch,pad,env", [(1 << 15, 2, 8, {}), (10 ** 4, 3, 8, {"B200FFT_MAX_SINGLE_PASS": "1024", "B200FFT_FOUR_STEP_SPLIT": "100,100"}),
                                             (16384, 2, 2, {"B200FFT_MAX_SINGLE_PASS": "4096", "B200FFT_FOUR_STEP_SPLIT": "8,2048"}),
                                             (16384, 2, 1, {"B200FFT_MAX_SINGLE_PASS": "4096", "B200FFT_FOUR_STEP_SPLIT": "2048,8"}),
                                             (509, 3, 5, {"B200FFT_NO_FUSED_BLUESTEIN": "1"}), (4093, 3, 1, {}), (4391, 2, 5, {})])
@pytest.mark.parametrize("inv", [-1, 1])
def test_scratch_users_stay_inside_the_scratch_they_ask_for(n, batch, pad, env, inv, monkeypatch):
    """Four-Step and Bluestein plans size their scratch from the caller's pitches: launch by launch on a scratch buffer of
    exactly that size between two guard bands, nothing may land outside it"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kw = dict(buffer_stride=[n + pad])
    nbytes = planned_scratch_bytes((n,), batch, 0, **kw)
    assert nbytes > 0 and nbytes % 8 == 0, nbytes
    x = orc.random_input((batch, n), np.complex64, seed=n + pad)
    L = lu.make_layout((n,), batch, [n + pad], np.complex64)
    L.scatter(x)
    before = L.flat.copy()
    temp, tmask = lu.make_flat(nbytes // 8, np.complex64)
    tbefore = temp.copy()
    d = emu.make_desc((n,), batch, 0, **kw)
    rc, npass, _ = emu.exec_plan_pass(d, inv, L.data, temp[lu.GUARD:], -1)
    assert rc == 0 and npass >= 2
    for i in range(npass):
        assert emu.exec_plan_pass(d, inv, L.data, temp[lu.GUARD:], i)[0] == 0
        lu.assert_untouched(temp, tbefore, tmask, what=f"tempBuffer after launch {i}")
    lu.assert_untouched(L.flat, before, L.mask, L)
    check(L.gather(), orc.c2c(x, 1, inv == 1), 0, n)


@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("pad", [1, 5])
@pytest.mark.parametrize("n", [77, 2 * 127, 509, 4093, 4391])
def test_runtime_scheduled_rader_and_bluestein(n, pad, prec):
    """77: runtime-scheduled kernel; 254: prime 127; 509: Bluestein in one launch; 4093: two launches; 4391: long"""
    if prec == 1 and n > 509:
        pytest.skip("the long Bluestein plans are covered in FP32 (emulation time)")
    for inv in (-1, 1):
        c2c_case((n,), 3, prec, inv, [n + pad], same_bits_as_packed=(pad == 1 and inv == -1 and n <= 509))


def test_bluestein_two_launches_and_rader_stage_padded(monkeypatch):
    monkeypatch.setenv("B200FFT_NO_FUSED_BLUESTEIN", "1")
    npass, _ = c2c_case((509,), 3, 0, -1, [509 + 5])
    assert npass == 2
    monkeypatch.delenv("B200FFT_NO_FUSED_BLUESTEIN")
    monkeypatch.setenv("B200FFT_RADER_MAX_PRIME", "127")
    c2c_case((2032,), 2, 0, -1, [2032 + 3])


# ---------------------------------------------------------------- N-D C2C ----------------------------------------------------------------
def nd_layouts(shape):
    """name -> strides: padded row pitch only; padded plane pitch only; both; batch pitch larger than the volume"""
    nd = len(shape)

    def build(p0, plane_pad, batch_pad):
        s = [p0]
        for a in range(1, nd):
            s.append(s[-1] * shape[a])
            if a == 1 and nd > 2:
                s[-1] += plane_pad * s[0]
        s[-1] += batch_pad
        return s
    out = {"row": build(shape[0] + 3, 0, 0), "batch": build(shape[0], 0, 5 * shape[0] + 1)}
    if nd > 2:
        out["plane"] = build(shape[0], 3, 0)
        out["both"] = build(shape[0] + 1, 3, 7)
    else:
        out["both"] = build(shape[0] + 1, 0, 7)
    return out


@pytest.mark.parametrize("which", ["row", "plane", "both", "batch"])
@pytest.mark.parametrize("shape,prec", [((64, 32), 0), ((48, 20), 0), ((32, 16, 8), 0), ((32, 16, 8), 1), ((105, 30), 0)])
def test_2d_3d_padded_pitches(shape, prec, which):
    lay = nd_layouts(shape)
    if which not in lay:
        pytest.skip("a 2-D shape has no plane pitch")
    for inv in (-1, 1):
        c2c_case(shape, 2, prec, inv, lay[which], same_bits_as_packed=(which == "both" and inv == -1))


@pytest.mark.parametrize("prec", [0, 1])
def test_sub_volume_of_a_bigger_array(prec):
    """logical (32,16,8) in the corner of an allocation of (40,20,8): everything else of the big array must survive"""
    shape, strides = (32, 16, 8), [40, 800, 6400]
    for inv in (-1, 1):
        c2c_case(shape, 1, prec, inv, strides, same_bits_as_packed=(inv == -1))
    # two such volumes: the batch pitch is the big array
    c2c_case(shape, 2, prec, -1, strides)


def test_4d_with_no_mergeable_dimensions():
    """every pitch padded: no two dimensions fold into one, every pass carries the most outer dimensions a launch can"""
    shape, batch = (16, 8, 4, 2), 3
    strides = [17, 17 * 8 + 5, (17 * 8 + 5) * 4 + 3, ((17 * 8 + 5) * 4 + 3) * 2 + 11]
    x, got, npass, d = run_inplace(shape, batch, 0, -1, strides)
    check(got, orc.c2c(x, 4, False), 0, int(np.prod(shape)))
    _, packed, npass_packed, _ = run_inplace(shape, batch, 0, -1, None, x=x)
    assert npass == npass_packed == 4, (npass, npass_packed)      # x + three outer dimensions still fit one launch per axis
    assert orc.error_metrics(got, packed)["l2_rel"] < T32
    x, got, _, _ = run_inplace(shape, batch, 0, 1, strides, normalize=1)
    check(got, orc.c2c(x, 4, True) / np.prod(shape), 0, int(np.prod(shape)))


# ---------------------------------------------------------------- out of place ----------------------------------------------------------------
@pytest.mark.parametrize("shape,batch", [((1024,), 6), ((64, 16), 3)])
@pytest.mark.parametrize("prec", [0, 1])
def test_out_of_place_three_different_pitches(shape, batch, prec):
    """input -> buffer -> output with a pitch of its own each; the input keeps every bit, gaps included"""
    dt, nd = cdt(prec), len(shape)
    x = orc.random_input((batch,) + tuple(reversed(shape)), dt, seed=7)
    s_in, s_buf, s_out = (lu.packed_strides(shape, shape[0] + p) for p in (1, 4, 7))
    s_in[-1] += 3; s_out[-1] += 9
    Li, Lb, Lo = (lu.make_layout(shape, batch, s, dt) for s in (s_in, s_buf, s_out))
    kw = dict(buffer_stride=s_buf, input_stride=s_in, output_stride=s_out, is_input_formatted=1, is_output_formatted=1)
    Li.scatter(x)
    bi, bb, bo = Li.flat.copy(), Lb.flat.copy(), Lo.flat.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, batch, prec, **kw), -1, Lb.data, inp=Li.data, out=Lo.data)
    assert rc == 0
    lu.assert_bit_identical(Li.flat, bi, "inputBuffer")
    lu.assert_untouched(Lb.flat, bb, Lb.mask, Lb, "buffer")
    lu.assert_untouched(Lo.flat, bo, Lo.mask, Lo, "outputBuffer")
    spec = Lo.gather()
    check(spec, orc.c2c(x, nd, False), prec, int(np.prod(shape)))
    # inverse: outputBuffer -> buffer, or -> inputBuffer with inverseReturnToInputBuffer
    for back in (0, 1):
        Li2, Lb2 = lu.make_layout(shape, batch, s_in, dt), lu.make_layout(shape, batch, s_buf, dt)
        bi2, bb2, bo2 = Li2.flat.copy(), Lb2.flat.copy(), Lo.flat.copy()
        d = emu.make_desc(shape, batch, prec, inverse_return_to_input=back, **kw)
        rc, _ = emu.exec_plan(d, 1, Lb2.data, inp=Li2.data, out=Lo.data)
        assert rc == 0
        lu.assert_bit_identical(Lo.flat, bo2, "outputBuffer (source of the inverse)")
        lu.assert_untouched(Lb2.flat, bb2, Lb2.mask, Lb2, "buffer")
        if back:
            lu.assert_untouched(Li2.flat, bi2, Li2.mask, Li2, "inputBuffer")
            if nd == 1:
                lu.assert_bit_identical(Lb2.flat, bb2, "buffer (a one-launch plan goes straight to inputBuffer)")
        else:
            lu.assert_bit_identical(Li2.flat, bi2, "inputBuffer")
        res = (Li2 if back else Lb2).gather()
        check(res, orc.c2c(spec.astype(np.complex128), nd, True), prec, int(np.prod(shape)))


# ---------------------------------------------------------------- R2C / C2R ----------------------------------------------------------------
def r2c_inplace(shape, batch, prec, pad):
    """in place: complex rows H + pad apart, the real rows live in the same rows, 2 * (H + pad) reals apart"""
    nd, nx = len(shape), shape[0]
    H = nx // 2 + 1
    cshape = (H,) + tuple(shape[1:])
    cs = lu.packed_strides(cshape, H + pad)
    cs[-1] += 2 * pad
    x = orc.random_input((batch,) + tuple(reversed(shape)), rdt(prec), seed=sum(shape) + pad)
    L = lu.make_layout(cshape, batch, cs, cdt(prec))
    real = lu.view_of(L.flat, shape, batch, [2 * s for s in cs], rdt(prec), L.guard)
    real[...] = x
    before = L.flat.copy()
    d = emu.make_desc(shape, batch, prec, perform_r2c=1, buffer_stride=cs)
    rc, _ = emu.exec_plan(d, -1, L.data)
    assert rc == 0, rc
    lu.assert_untouched(L.flat, before, L.mask, L)
    check(L.gather(), orc.r2c(x, nd), prec, int(np.prod(shape)))
    before = L.flat.copy()
    rc, _ = emu.exec_plan(d, 1, L.data)
    assert rc == 0, rc
    lu.assert_untouched(L.flat, before, L.mask, L)
    check(np.array(real), x.astype(np.float64) * np.prod(shape), prec, int(np.prod(shape)))


@pytest.mark.parametrize("pad", [1, 3])
@pytest.mark.parametrize("shape,batch,prec", [((64,), 4, 0), ((1000,), 2, 0), ((4096,), 2, 0), ((15,), 3, 0), ((131,), 3, 0),
                                              ((64, 32), 2, 0), ((1000, 6), 2, 0), ((64,), 4, 1), ((15,), 3, 1), ((64, 32), 2, 1)])
def test_r2c_c2r_in_place_padded_spectrum_pitch(shape, batch, prec, pad):
    r2c_inplace(shape, batch, prec, pad)


@pytest.mark.parametrize("shape,batch", [((64,), 4), ((1000,), 2), ((64, 32), 2), ((15,), 3)])
@pytest.mark.parametrize("rpad", [0, 6, 1])
def test_r2c_out_of_place_real_pitch(shape, batch, rpad):
    """isInputFormatted: the reals come from inputBuffer, inputBufferStride in REAL elements.  An odd pitch cannot be read as
    complex pairs by the even-length kernels: the plan is refused (VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C), not run wrongly"""
    nd, nx = len(shape), shape[0]
    H = nx // 2 + 1
    cshape = (H,) + tuple(shape[1:])
    cs = lu.packed_strides(cshape, H + 2)
    rs = lu.packed_strides(shape, nx + rpad)
    x = orc.random_input((batch,) + tuple(reversed(shape)), np.float32, seed=nx + rpad)
    Li, Lb = lu.make_layout(shape, batch, rs, np.float32), lu.make_layout(cshape, batch, cs, np.complex64)
    Li.scatter(x)
    bi, bb = Li.flat.copy(), Lb.flat.copy()
    kw = dict(perform_r2c=1, is_input_formatted=1, buffer_stride=cs, input_stride=rs)
    rc, _ = emu.exec_plan(emu.make_desc(shape, batch, 0, **kw), -1, Lb.data, inp=Li.data)
    if nx % 2 == 0 and any(s % 2 for s in rs[:nd]):
        assert rc == R_R2C
        lu.assert_bit_identical(Lb.flat, bb, "buffer of a refused plan")
        return
    assert rc == 0, rc
    lu.assert_bit_identical(Li.flat, bi, "inputBuffer")
    lu.assert_untouched(Lb.flat, bb, Lb.mask, Lb)
    check(Lb.gather(), orc.r2c(x, nd), 0, int(np.prod(shape)))
    # C2R back into a fresh inputBuffer
    Li2 = lu.make_layout(shape, batch, rs, np.float32)
    bi2, bb = Li2.flat.copy(), Lb.flat.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, batch, 0, inverse_return_to_input=1, normalize=1, **kw), 1, Lb.data, inp=Li2.data)
    assert rc == 0, rc
    lu.assert_untouched(Li2.flat, bi2, Li2.mask, Li2, "inputBuffer")
    lu.assert_untouched(Lb.flat, bb, Lb.mask, Lb)
    check(Li2.gather(), x, 0, int(np.prod(shape)))


# ---------------------------------------------------------------- DCT / DST ----------------------------------------------------------------
@pytest.mark.parametrize("mode", ["dct", "dst"])
@pytest.mark.parametrize("kind", [1, 2, 3, 4])
@pytest.mark.parametrize("shape,batch,prec", [((64,), 3, 0), ((33,), 2, 1), ((100,), 2, 1), ((32, 16), 3, 0)])
@pytest.mark.parametrize("pad", [1, 2])
def test_dct_dst_padded_pitch(mode, kind, shape, batch, prec, pad):
    """an odd pitch: two neighbouring real lines are not one complex line, the paired-line kernels must not be chosen"""
    strides = lu.packed_strides(shape, shape[0] + pad)
    strides[-1] += pad
    f = orc.dct if mode == "dct" else orc.dst
    for inv in (-1, 1):
        x, got, _, _ = run_inplace(shape, batch, prec, inv, strides, dtype=rdt(prec), **{"perform_" + mode: kind})
        check(got, f(x, kind, len(shape), inverse=(inv == 1)), prec, int(np.prod(shape)))


# ---------------------------------------------------------------- omitDimension ----------------------------------------------------------------
@pytest.mark.parametrize("omit", [(0, 1, 0), (0, 0, 1), (0, 1, 1), (1, 0, 0), (1, 0, 1)])
@pytest.mark.parametrize("padded", [False, True])
def test_omit_dimension_c2c(omit, padded):
    """only the axes that are not omitted are transformed; normalize = 1 divides by the product of THEIR sizes"""
    shape, batch = (32, 16, 8), 2
    strides = [33, 33 * 16 + 2, (33 * 16 + 2) * 8 + 5] if padded else None
    axes = tuple(3 - a for a in range(3) if not omit[a])          # numpy axis of dimension a in [batch, z, y, x]
    n = int(np.prod([shape[a] for a in range(3) if not omit[a]]))
    x, got, _, _ = run_inplace(shape, batch, 0, -1, strides, omit_dimension=list(omit))
    check(got, np.fft.fftn(x.astype(np.complex128), axes=axes), 0, n)
    x, got, _, _ = run_inplace(shape, batch, 0, 1, strides, omit_dimension=list(omit), normalize=1)
    check(got, np.fft.ifftn(x.astype(np.complex128), axes=axes), 0, n)


def test_omit_dimension_dct_and_refusals():
    shape, batch = (64, 32), 2
    x, got, _, _ = run_inplace(shape, batch, 0, -1, [66, 66 * 32 + 4], dtype=np.float32, perform_dct=2, omit_dimension=[0, 1])
    check(got, orc.dct(x, 2, 1), 0, 64)
    x, got, _, _ = run_inplace(shape, batch, 0, -1, [66, 66 * 32 + 4], dtype=np.float32, perform_dct=2, omit_dimension=[1, 0])
    check(np.swapaxes(got, 1, 2), orc.dct(np.ascontiguousarray(np.swapaxes(x, 1, 2)), 2, 1), 0, 32)
    buf = np.zeros((2, 32, 34), np.complex64)
    assert emu.exec_plan(emu.make_desc(shape, 2, 0, perform_r2c=1, omit_dimension=[1, 0]), -1, buf)[0] == R_OMIT
    assert emu.exec_plan(emu.make_desc(shape, 2, 0, perform_convolution=1, omit_dimension=[0, 1]), -1, buf, kernel=buf)[0] == R_OMIT


# ---------------------------------------------------------------- convolution ----------------------------------------------------------------
@pytest.mark.parametrize("shape", [(256,), (64, 32)])
def test_convolution_padded_layout_takes_the_three_step_path(shape):
    """the fused last axis assumes the packed layout: with padded pitches the plan is forward, product, inverse; the kernel
    spectrum is made by a kernelConvolution plan with the same strides"""
    C, B, nd = 2, 2, len(shape)
    axes = tuple(range(-nd, 0))
    strides = lu.packed_strides(shape, shape[0] + 2)
    strides[-1] += 6
    k = orc.random_input((C,) + tuple(reversed(shape)), np.complex64, seed=1)
    x = orc.random_input((B * C,) + tuple(reversed(shape)), np.complex64, seed=2)
    LK = lu.make_layout(shape, C, strides, np.complex64)
    LK.flat[~LK.mask] = 0.5 + 1j        # finite gaps here: a product of two NaN gaps is the same NaN again and would hide a store
    LK.scatter(k)
    bk = LK.flat.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, 1, 0, coordinate_features=C, kernel_convolution=1, buffer_stride=strides), -1, LK.data)
    assert rc == 0
    lu.assert_untouched(LK.flat, bk, LK.mask, LK, "kernel")
    L = lu.make_layout(shape, B * C, strides, np.complex64)
    L.flat[~L.mask] = 3 - 2j
    L.scatter(x)
    before, bk = L.flat.copy(), LK.flat.copy()
    d = emu.make_desc(shape, B, 0, coordinate_features=C, perform_convolution=1, normalize=1, buffer_stride=strides)
    assert "fused convolution" not in launches(d, -1)
    assert "fused convolution" in launches(emu.make_desc(shape, B, 0, coordinate_features=C, perform_convolution=1, normalize=1), -1)
    rc, _ = emu.exec_plan(d, -1, L.data, kernel=LK.data)
    assert rc == 0
    lu.assert_bit_identical(LK.flat, bk, "kernel")
    lu.assert_untouched(L.flat, before, L.mask, L)
    X = np.fft.fftn(x.astype(np.complex128), axes=axes).reshape((B, C) + x.shape[1:])
    K = np.fft.fftn(k.astype(np.complex128), axes=axes)
    ref = np.fft.ifftn(X * K[None], axes=axes).reshape(x.shape)
    check(L.gather(), ref, 0, int(np.prod(shape)), l2=2e-6)       # two transforms and a product (tests/test_emu_convolution.py)


# ---------------------------------------------------------------- half storage, zero padding ----------------------------------------------------------------
@pytest.mark.parametrize("shape,batch", [((1024,), 3), ((64, 64), 2)])
def test_half_storage_padded_pitch(shape, batch):
    """complex32 buffers, FP32 arithmetic: the error is the rounding of the stored result to half"""
    strides = lu.packed_strides(shape, shape[0] + 2)
    strides[-1] += 2
    x = orc.random_input((batch,) + tuple(reversed(shape)), np.complex64, seed=3)
    xh = np.ascontiguousarray(np.stack([x.real, x.imag], axis=-1).astype(np.float16))
    L = lu.make_layout(shape, batch, strides, np.uint32)           # one complex32 element = 32 bits; the sentinel's imaginary half is NaN
    L.scatter(xh.view(np.uint32)[..., 0])
    before = L.flat.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, batch, 2, buffer_stride=strides), -1, L.data)
    assert rc == 0
    lu.assert_untouched(L.flat, before, L.mask, L)
    gh = L.gather()[..., None].view(np.float16).astype(np.float64)
    got = gh[..., 0] + 1j * gh[..., 1]
    ref = orc.c2c(xh[..., 0].astype(np.float64) + 1j * xh[..., 1].astype(np.float64), len(shape))
    assert orc.error_metrics(got, ref)["l2_rel"] < 6e-4          # half: eps = 9.8e-4, rounding once on the way out


def test_zero_padding_skipped_lines_leave_their_gaps_alone():
    """(64,64) with the upper half of y zero-padded: the x pass skips those rows; with a padded row pitch their gaps, and the
    gaps of the rows it does transform, keep their contents"""
    shape, batch, strides = (64, 64), 2, [67, 67 * 64 + 5]
    x = orc.random_input((batch, 64, 64), np.complex64, seed=4)
    clean = x.copy(); clean[:, 32:, :] = 0
    kw = dict(perform_zeropadding=[0, 1], zeropad_left=[0, 32], zeropad_right=[0, 64])
    xx, got, npass, d = run_inplace(shape, batch, 0, -1, strides, x=x, **kw)
    check(got, orc.c2c(clean, 2, False), 0, 64 * 64)
    _, packed, _, _ = run_inplace(shape, batch, 0, -1, None, x=x, **kw)
    assert np.array_equal(lu.bits(got.reshape(-1)), lu.bits(packed.reshape(-1)))
