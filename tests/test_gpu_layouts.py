"""GPU (-m gpu): padded and user-strided buffer layouts on the device, with guard bands around every buffer.

The flat allocations of tests/layout_util.py are uploaded guards and all; after the transform the whole allocation comes back
and every element outside the logical array -- guards, gaps between rows, planes and batches -- must hold the bit pattern
it was given.  Plans run with userTempBuffer = 1 on a scratch buffer of exactly the size the plan reports, between two guard
bands of its own, so a launch that stores past the scratch is seen as well.  Values are compared with the oracle on the dense
double-precision array.  Nothing here provokes a fault: every stray access these tests look for lands in memory they own."""
import contextlib
import os

import numpy as np
import pytest

import layout_util as lu
import vkfft_oracle as orc

pytestmark = pytest.mark.gpu

TOL32, TOL64 = 1e-6, 1e-12      # relative l2 against the exact transform
TOL_REAL32 = 2e-6               # composed real transforms in FP32: the conditioning of the split / merge step puts the reference's
                                # own error at up to 1.4e-6 (tests/gpu_util.py); no stored reference error exists for padded layouts
# per point: max|got - ref| <= C_POINT * eps * sqrt(log2 N) * max|ref| of the line.  The largest value seen over this file on
# an H100 is 2.1 x eps x sqrt(log2 N) (printed with -s); a wrong point is off by ~1/eps times that
C_POINT = 8.0
TEMP_GUARD = 512                # bytes before and after the scratch buffer
observed = {"worst": 0.0}


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    import vkfft_b200  # noqa: F401  (fails loudly if libb200fft.so is missing)
    yield torch
    print(f"\nlargest per-point error seen: {observed['worst']:.2f} x eps x sqrt(log2 N); "
          f"peak device memory held by the tests: {torch.cuda.max_memory_allocated() / 2 ** 20:.0f} MiB")


@contextlib.contextmanager
def environ(**kv):
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def check(got, ref, double, n_total, l2=None):
    tol = (TOL64 if double else TOL32) if l2 is None else l2
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < tol, e
    eps = np.finfo(np.float64 if double else np.float32).eps
    r = lu.max_line_error(got, ref)
    observed["worst"] = max(observed["worst"], r / lu.point_bound(n_total, eps, 1.0))
    assert r <= lu.point_bound(n_total, eps, C_POINT), r / lu.point_bound(n_total, eps, 1.0)


class Dev:
    """a guarded host allocation and its copy on the device"""

    def __init__(self, torch, flat, mask, layout=None, what="buffer"):
        self.torch, self.flat, self.mask, self.layout, self.what = torch, flat, mask, layout, what
        self.before = flat.copy()
        host = flat.view(np.float16) if flat.dtype == np.uint32 else flat          # complex32 travels as pairs of halves
        self.t = torch.from_numpy(host).cuda()
        guard = layout.guard if layout is not None else lu.GUARD
        self.ptr = int(self.t.data_ptr()) + guard * flat.dtype.itemsize

    def fetch(self):
        """copy back and check everything outside the footprint"""
        back = self.t.cpu().numpy()
        self.flat[...] = back.view(self.flat.dtype) if back.dtype != self.flat.dtype else back
        lu.assert_untouched(self.flat, self.before, self.mask, self.layout, self.what)
        return self

    def fetch_unmodified(self):
        back = self.t.cpu().numpy()
        lu.assert_bit_identical(back.view(self.flat.dtype), self.before, self.what)


def dev_layout(torch, shape, batch, strides, dtype, x=None, what="buffer", guard=lu.GUARD):
    L = lu.make_layout(shape, batch, strides, dtype, guard)
    if x is not None:
        L.scatter(x)
    return L, Dev(torch, L.flat, L.mask, L, what)


class Plan:
    """a plan with caller-owned scratch of exactly the reported size between two guard bands"""

    def __init__(self, torch, shape, batch, env=None, **cfgkw):
        import vkfft_b200 as vk
        self.vk, self.torch = vk, torch
        self.app = vk.VkFFTApplication()
        with environ(**(env or {})):
            rc = vk.initializeVkFFT(self.app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0,
                                                                    userTempBuffer=1, **cfgkw))
        self.rc = rc
        if rc != 0:
            return
        self.info = vk.planInfo(self.app)
        self.temp_bytes = int(self.info["temp_bytes"])
        self.temp = torch.full((TEMP_GUARD + self.temp_bytes + TEMP_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")

    def text(self, inverse=-1):
        return self.info["inverse" if inverse == 1 else "forward"]

    def run(self, inverse, buffer, inp=None, out=None, kernel=None, **lpkw):
        vk = self.vk
        lp = vk.VkFFTLaunchParams(buffer=buffer, inputBuffer=inp, outputBuffer=out, kernel=kernel,
                                  tempBuffer=int(self.temp.data_ptr()) + TEMP_GUARD, **lpkw)
        rc = vk.VkFFTAppend(self.app, inverse, lp)
        assert rc == 0, vk.getVkFFTErrorString(rc)
        self.torch.cuda.synchronize()
        g = self.temp.cpu().numpy()
        ok = (g[:TEMP_GUARD] == 0xA5).all() and (g[TEMP_GUARD + self.temp_bytes:] == 0xA5).all()
        assert ok, (f"a launch stored outside tempBuffer ({self.temp_bytes} bytes as reported by the plan): "
                    f"{int((g[:TEMP_GUARD] != 0xA5).sum())} bytes before, {int((g[TEMP_GUARD + self.temp_bytes:] != 0xA5).sum())} bytes after")

    def close(self):
        if self.rc == 0:
            self.vk.deleteVkFFT(self.app)


def cdt(double):
    return np.complex128 if double else np.complex64


def rdt(double):
    return np.float64 if double else np.float32


def run_inplace(torch, shape, batch, inverse, strides, x=None, double=False, dtype=None, env=None, expect=None, **cfgkw):
    """-> (x, result as a dense array, plan listing, reported scratch bytes); strides None = the packed default layout"""
    dt = cdt(double) if dtype is None else dtype
    if x is None:
        x = orc.random_input((batch,) + tuple(reversed(shape)), dt, seed=sum(shape) + batch)
    st = lu.packed_strides(shape) if strides is None else list(strides)
    L, D = dev_layout(torch, shape, batch, st, dt, x)
    if strides is not None:
        cfgkw["bufferStride"] = st
    p = Plan(torch, shape, batch, env=env, doublePrecision=int(double), **cfgkw)
    assert p.rc == 0, p.rc
    try:
        if expect:
            expect(p.text(inverse))
        p.run(inverse, D.ptr)
        D.fetch()
        return x, L.gather(), p.text(inverse), p.temp_bytes
    finally:
        p.close()


def same_bits(a, b):
    return np.array_equal(lu.bits(np.ascontiguousarray(a).reshape(-1)), lu.bits(np.ascontiguousarray(b).reshape(-1)))


# ---------------------------------------------------------------- 1-D C2C ----------------------------------------------------------------
@pytest.mark.parametrize("batch", [37, 130, 1])
@pytest.mark.parametrize("n", [8, 16, 32, 4096, 16384, 1 << 16])
def test_packed_layout_ragged_batches_stay_inside_the_buffer(gpu, n, batch):
    """the default layout, batches that do not fill the last tile of lines: nothing may land one past the end"""
    for inverse in (-1, 1):
        x, got, _, _ = run_inplace(gpu, (n,), batch, inverse, None)
        check(got, orc.c2c(x, 1, inverse == 1), False, n)


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("pad", ["+1", "+3", "x2"])
@pytest.mark.parametrize("n", [8, 16, 32])
def test_short_lines_padded_pitch(gpu, n, pad, double):
    pitch = {"+1": n + 1, "+3": n + 3, "x2": 2 * n}[pad]
    for batch in (130, 4099):
        for inverse in (-1, 1):
            x, got, _, _ = run_inplace(gpu, (n,), batch, inverse, [pitch], double=double)
            check(got, orc.c2c(x, 1, inverse == 1), double, n)
    _, packed, _, _ = run_inplace(gpu, (n,), batch, inverse, None, x=x, double=double)
    assert same_bits(got, packed), "the pitch changed the arithmetic"


@pytest.mark.parametrize("double,pad", [(False, 1), (False, 2), (False, 16), (True, 1), (True, 16)])
@pytest.mark.parametrize("n", [64, 1000, 4096, 1100, 2002, 77, 254, 509, 4093, 4391, 20011])
def test_one_axis_padded_pitch(gpu, n, double, pad):
    """ahead-of-time, plan-time (1100, 2002), runtime-scheduled (77) kernels, Rader (254) and Bluestein in one launch (509),
    two launches (4093) and long (4391, 20011): the Bluestein plans' scratch is guarded"""
    for inverse in (-1, 1):
        x, got, _, _ = run_inplace(gpu, (n,), 5, inverse, [n + pad], double=double)
        check(got, orc.c2c(x, 1, inverse == 1), double, n)
    _, packed, txt_p, _ = run_inplace(gpu, (n,), 5, inverse, None, x=x, double=double)
    assert orc.error_metrics(got, packed)["l2_rel"] < (TOL64 if double else TOL32)


@pytest.mark.parametrize("pad", [2, 1])
@pytest.mark.parametrize("logn", [13, 14, 15, 16, 17, 20, 22])
def test_long_power_of_two_padded_batch_pitch(gpu, logn, pad):
    """2^13, 2^14: one pipelined launch (pitch N+2: one bulk copy per line; N+1: the unaligned kernel); 2^15, 2^16: the cluster
    launch takes one sequence per cluster wherever it starts, so it serves a padded batch pitch too and must equal the two
    launches and the packed plan bit for bit; 2^17, 2^20: two launches; 2^22: three.  The scratch of the Four-Step plans is
    guarded (the cluster launch leaves it alone)."""
    n, batch = 1 << logn, 3
    for inverse in (-1, 1):
        x, got, txt, temp_bytes = run_inplace(gpu, (n,), batch, inverse, [n + pad])
        check(got, orc.c2c(x, 1, inverse == 1), False, n)
        assert "fused" not in txt and ("one cluster launch" in txt) == (logn in (15, 16)), txt
        if logn >= 15:
            assert temp_bytes > 0 and len(txt.strip().split("\n")) == (3 if logn == 22 else 2), txt
        if logn in (15, 16):
            for strides in ([n + pad], None):
                _, two, txt_2, _ = run_inplace(gpu, (n,), batch, inverse, strides, x=x, env={"B200FFT_NO_CLUSTER4": "1"})
                assert "cluster" not in txt_2, txt_2
                assert same_bits(got, two), "the cluster launch on a padded batch pitch differs from the two launches"


def test_fused_four_step_falls_back_with_a_padded_batch_pitch(gpu):
    n, batch = 1 << 16, 3
    x, got, txt, _ = run_inplace(gpu, (n,), batch, -1, [n + 2], env={"B200FFT_FUSED4": "1", "B200FFT_NO_CLUSTER4": "1"})
    assert "fused" not in txt and len(txt.strip().split("\n")) == 2, txt
    _, packed, txt_p, _ = run_inplace(gpu, (n,), batch, -1, None, x=x, env={"B200FFT_FUSED4": "1", "B200FFT_NO_CLUSTER4": "1"})
    assert "fused" in txt_p, txt_p
    assert same_bits(got, packed)
    check(got, orc.c2c(x, 1), False, n)


# ---------------------------------------------------------------- N-D C2C ----------------------------------------------------------------
@pytest.mark.parametrize("shape,double,strides", [
    ((64, 32), False, [67, 67 * 32]), ((64, 32), False, [64, 64 * 32 + 321]), ((48, 20), False, [49, 49 * 20 + 7]),
    ((105, 30), False, [106, 106 * 30 + 7]), ((32, 16, 8), False, [32, 32 * 16 + 96, (32 * 16 + 96) * 8]),
    ((32, 16, 8), True, [33, 33 * 16 + 99, (33 * 16 + 99) * 8 + 7]), ((32, 16, 8), False, [40, 800, 6400]),
    ((1100, 154), False, [1101, 1101 * 154 + 3]), ((8192, 8), False, [8192, 8192 * 8 + 2]), ((8, 8192), False, [9, 9 * 8192 + 5]),
    ((128, 64, 32), True, [160, 160 * 64, 160 * 64 * 32]), ((16, 8, 4, 2), False, [17, 141, 567, 1145])])
def test_nd_padded_pitches(gpu, shape, double, strides):
    """padded row, plane and batch pitches; a sub-volume of a bigger array (FP32 (32,16,8) in (40,20,8), FP64 (128,64,32) in
    (160,64,32)); plan-time kernels (1100,154); a Four-Step axis along contiguous lines and along a stride (scratch guarded);
    4-D with no two dimensions mergeable"""
    nd = len(shape)
    for inverse in (-1, 1):
        x, got, _, _ = run_inplace(gpu, shape, 2, inverse, strides, double=double)
        check(got, orc.c2c(x, nd, inverse == 1), double, int(np.prod(shape)))
    _, packed, _, _ = run_inplace(gpu, shape, 2, inverse, None, x=x, double=double)
    assert orc.error_metrics(got, packed)["l2_rel"] < (TOL64 if double else TOL32)


@pytest.mark.parametrize("omit", [(0, 1, 0), (0, 0, 1), (0, 1, 1), (1, 0, 0)])
def test_omit_dimension(gpu, omit):
    shape, batch, strides = (32, 16, 8), 3, [33, 33 * 16 + 2, (33 * 16 + 2) * 8 + 5]
    axes = tuple(3 - a for a in range(3) if not omit[a])
    n = int(np.prod([shape[a] for a in range(3) if not omit[a]]))
    x, got, _, _ = run_inplace(gpu, shape, batch, -1, strides, omitDimension=list(omit))
    check(got, np.fft.fftn(x.astype(np.complex128), axes=axes), False, n)
    x, got, _, _ = run_inplace(gpu, shape, batch, 1, strides, omitDimension=list(omit), normalize=1)
    check(got, np.fft.ifftn(x.astype(np.complex128), axes=axes), False, n)


# ---------------------------------------------------------------- out of place, offsets ----------------------------------------------------------------
@pytest.mark.parametrize("shape,batch,double", [((1024,), 6, False), ((64, 16), 3, False), ((1 << 15,), 2, False), ((4096,), 3, True)])
def test_out_of_place_three_different_pitches(gpu, shape, batch, double):
    torch, dt, nd = gpu, cdt(double), len(shape)
    x = orc.random_input((batch,) + tuple(reversed(shape)), dt, seed=7)
    s_in, s_buf, s_out = (lu.packed_strides(shape, shape[0] + p) for p in (1, 4, 7))
    s_in[-1] += 3; s_out[-1] += 9
    cfg = dict(bufferStride=s_buf, inputBufferStride=s_in, outputBufferStride=s_out, isInputFormatted=1, isOutputFormatted=1,
               doublePrecision=int(double))
    (Li, Di), (Lb, Db), (Lo, Do) = (dev_layout(torch, shape, batch, s, dt, xx, w) for s, xx, w in
                                    ((s_in, x, "inputBuffer"), (s_buf, None, "buffer"), (s_out, None, "outputBuffer")))
    p = Plan(torch, shape, batch, **cfg)
    assert p.rc == 0
    p.run(-1, Db.ptr, inp=Di.ptr, out=Do.ptr)
    p.close()
    Di.fetch_unmodified(); Db.fetch(); Do.fetch()
    spec = Lo.gather()
    check(spec, orc.c2c(x, nd), double, int(np.prod(shape)))
    for back in (0, 1):
        (Li2, Di2), (Lb2, Db2) = (dev_layout(torch, shape, batch, s, dt, None, w) for s, w in ((s_in, "inputBuffer"), (s_buf, "buffer")))
        Do.before = Do.flat.copy()
        p = Plan(torch, shape, batch, inverseReturnToInputBuffer=back, **cfg)
        assert p.rc == 0
        p.run(1, Db2.ptr, inp=Di2.ptr, out=Do.ptr)
        p.close()
        Do.fetch_unmodified(); Db2.fetch()
        if back:
            Di2.fetch()
        else:
            Di2.fetch_unmodified()
        check((Li2 if back else Lb2).gather(), orc.c2c(spec.astype(np.complex128), nd, True), double, int(np.prod(shape)))


@pytest.mark.parametrize("at_launch", [0, 1])
@pytest.mark.parametrize("off", [8, 24])
@pytest.mark.parametrize("n,pad", [(4096, 2), (16384, 2), (1 << 16, 0), (1 << 16, 2), (509, 1)])
def test_buffer_offsets_with_padded_pitches(gpu, n, pad, off, at_launch):
    """buffer / input / output / temp offsets of 8 and 24 bytes, given at plan time or at launch: the buffers are then only
    8-byte aligned, which the bulk-copy kernels cannot take"""
    torch, batch = gpu, 3
    import vkfft_b200 as vk
    x = orc.random_input((batch, n), np.complex64, seed=n + off)
    k = off // 8
    s_in, s_buf, s_out = [n + pad + 1], [n + pad], [n + pad + 3]
    (Li, Di), (Lb, Db), (Lo, Do) = (dev_layout(torch, (n,), batch, s, np.complex64, xx, w, guard=lu.GUARD + k) for s, xx, w in
                                    ((s_in, x, "inputBuffer"), (s_buf, None, "buffer"), (s_out, None, "outputBuffer")))
    offs = dict(bufferOffset=Lb.guard * 8, inputBufferOffset=Li.guard * 8, outputBufferOffset=Lo.guard * 8, tempBufferOffset=TEMP_GUARD + off)
    cfg = dict(bufferStride=s_buf, inputBufferStride=s_in, outputBufferStride=s_out, isInputFormatted=1, isOutputFormatted=1,
               specifyOffsetsAtLaunch=at_launch, **({} if at_launch else offs))
    p = Plan(torch, (n,), batch, **cfg)
    assert p.rc == 0
    # the scratch starts `off` bytes into its slot: keep the rear guard in place
    p.temp = torch.full((TEMP_GUARD + off + p.temp_bytes + TEMP_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
    lp = vk.VkFFTLaunchParams(buffer=Db.t, inputBuffer=Di.t, outputBuffer=Do.t, tempBuffer=p.temp, **(offs if at_launch else {}))
    assert vk.VkFFTAppend(p.app, -1, lp) == 0
    torch.cuda.synchronize()
    g = p.temp.cpu().numpy()
    assert (g[:TEMP_GUARD + off] == 0xA5).all() and (g[TEMP_GUARD + off + p.temp_bytes:] == 0xA5).all(), "stores outside tempBuffer"
    p.close()
    Di.fetch_unmodified(); Db.fetch(); Do.fetch()
    check(Lo.gather(), orc.c2c(x, 1), False, n)


# ---------------------------------------------------------------- real transforms ----------------------------------------------------------------
@pytest.mark.parametrize("shape,batch,double,pad", [((64,), 40, False, 1), ((1000,), 3, False, 3), ((4096,), 3, False, 1), ((15,), 7, False, 1),
                                                    ((131,), 3, False, 3), ((64, 32), 2, False, 1), ((1000, 6), 2, True, 3),
                                                    ((1 << 17,), 2, False, 1), ((2 * 4391,), 2, False, 3), ((4096, 4096), 1, False, 7)])
def test_r2c_c2r_in_place_padded_spectrum_pitch(gpu, shape, batch, double, pad):
    """complex rows H + pad apart, real rows in the same rows; long (2^17), non-smooth (2*4391) and odd (131) lengths use
    scratch; 4096^2 with bufferStride[0] = 2049 + 7"""
    torch, nd, nx = gpu, len(shape), shape[0]
    H = nx // 2 + 1
    cshape = (H,) + tuple(shape[1:])
    cs = lu.packed_strides(cshape, H + pad)
    cs[-1] += 2 * pad
    x = orc.random_input((batch,) + tuple(reversed(shape)), rdt(double), seed=sum(shape) + pad)
    L = lu.make_layout(cshape, batch, cs, cdt(double))
    real = lu.view_of(L.flat, shape, batch, [2 * s for s in cs], rdt(double), L.guard)
    real[...] = x
    D = Dev(torch, L.flat, L.mask, L)
    p = Plan(torch, shape, batch, performR2C=1, bufferStride=cs, doublePrecision=int(double))
    assert p.rc == 0
    try:
        p.run(-1, D.ptr)
        D.fetch()
        check(L.gather(), orc.r2c(x, nd), double, int(np.prod(shape)), l2=None if double else TOL_REAL32)
        D.before = L.flat.copy()
        p.run(1, D.ptr)
        D.fetch()
        check(np.array(real), x.astype(np.float64) * np.prod(shape), double, int(np.prod(shape)), l2=None if double else TOL_REAL32)
    finally:
        p.close()


@pytest.mark.parametrize("shape,batch,rpad", [((64,), 40, 6), ((1000,), 3, 0), ((64, 32), 2, 6), ((15,), 7, 1), ((4096,), 3, 2), ((64,), 4, 1)])
def test_r2c_out_of_place_real_pitch(gpu, shape, batch, rpad):
    """inputBufferStride in REAL elements; an odd pitch of an even length is refused at plan creation"""
    torch, nd, nx = gpu, len(shape), shape[0]
    import vkfft_b200 as vk
    H = nx // 2 + 1
    cshape = (H,) + tuple(shape[1:])
    cs, rs = lu.packed_strides(cshape, H + 2), lu.packed_strides(shape, nx + rpad)
    x = orc.random_input((batch,) + tuple(reversed(shape)), np.float32, seed=nx + rpad)
    cfg = dict(performR2C=1, isInputFormatted=1, bufferStride=cs, inputBufferStride=rs)
    p = Plan(torch, shape, batch, **cfg)
    if nx % 2 == 0 and rs[0] % 2:
        assert p.rc == vk.VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C
        return
    assert p.rc == 0
    (Li, Di), (Lb, Db) = dev_layout(torch, shape, batch, rs, np.float32, x, "inputBuffer"), dev_layout(torch, cshape, batch, cs, np.complex64)
    p.run(-1, Db.ptr, inp=Di.ptr)
    p.close()
    Di.fetch_unmodified(); Db.fetch()
    check(Lb.gather(), orc.r2c(x, nd), False, int(np.prod(shape)), l2=TOL_REAL32)
    Li2, Di2 = dev_layout(torch, shape, batch, rs, np.float32, None, "inputBuffer")
    Db.before = Lb.flat.copy()
    p = Plan(torch, shape, batch, inverseReturnToInputBuffer=1, normalize=1, **cfg)
    assert p.rc == 0
    p.run(1, Db.ptr, inp=Di2.ptr)
    p.close()
    Di2.fetch(); Db.fetch()
    check(Li2.gather(), x, False, int(np.prod(shape)), l2=TOL_REAL32)


@pytest.mark.parametrize("mode,kind,shape,batch,double,pad", [
    ("dct", 2, (64,), 33, False, 1), ("dct", 3, (64,), 33, False, 2), ("dct", 1, (33,), 5, True, 1), ("dct", 4, (100,), 5, True, 2),
    ("dst", 1, (64,), 33, False, 1), ("dst", 2, (100,), 5, False, 2), ("dst", 3, (32, 16), 3, False, 1), ("dst", 4, (33,), 5, True, 1),
    ("dct", 2, (32, 16), 3, False, 1), ("dct", 2, (1024, 512), 1, False, 2), ("dct", 3, (1024, 512), 1, False, 2),
    ("dct", 2, (8, 4096), 1, False, 2), ("dct", 3, (8, 4096), 1, False, 1), ("dct", 2, (20000,), 2, False, 1), ("dct", 4, (131,), 3, False, 1)])
def test_dct_dst_padded_pitch(gpu, mode, kind, shape, batch, double, pad):
    """odd pitches refuse the paired-line kernels; (1024,512) with pitch 1026; a long strided axis (8,4096) and the lengths
    composed with a C2C plan (20000, 131) use scratch"""
    strides = lu.packed_strides(shape, shape[0] + pad)
    strides[-1] += pad
    f = orc.dct if mode == "dct" else orc.dst
    for inverse in (-1, 1):
        x, got, _, _ = run_inplace(gpu, shape, batch, inverse, strides, double=double, dtype=rdt(double),
                                   **{"performDCT" if mode == "dct" else "performDST": kind})
        check(got, f(x, kind, len(shape), inverse=(inverse == 1)), double, int(np.prod(shape)), l2=None if double else TOL_REAL32)


# ---------------------------------------------------------------- convolution, half storage ----------------------------------------------------------------
@pytest.mark.parametrize("shape", [(256,), (64, 32), (4096,)])
def test_convolution_padded_layout(gpu, shape):
    torch = gpu
    C, B, nd = 2, 2, len(shape)
    axes = tuple(range(-nd, 0))
    strides = lu.packed_strides(shape, shape[0] + 2)
    strides[-1] += 6
    k = orc.random_input((C,) + tuple(reversed(shape)), np.complex64, seed=1)
    x = orc.random_input((B * C,) + tuple(reversed(shape)), np.complex64, seed=2)
    LK, DK = dev_layout(torch, shape, C, strides, np.complex64, k, "kernel")
    p = Plan(torch, shape, 1, coordinateFeatures=C, kernelConvolution=1, bufferStride=strides)
    assert p.rc == 0
    p.run(-1, DK.ptr)
    p.close()
    DK.fetch()
    DK.before = LK.flat.copy()
    L, D = dev_layout(torch, shape, B * C, strides, np.complex64, x)
    p = Plan(torch, shape, B, coordinateFeatures=C, performConvolution=1, normalize=1, bufferStride=strides)
    assert p.rc == 0 and "fused convolution" not in p.text(), p.text()
    p.run(-1, D.ptr, kernel=DK.ptr)
    p.close()
    DK.fetch_unmodified(); D.fetch()
    X = np.fft.fftn(x.astype(np.complex128), axes=axes).reshape((B, C) + x.shape[1:])
    K = np.fft.fftn(k.astype(np.complex128), axes=axes)
    check(L.gather(), np.fft.ifftn(X * K[None], axes=axes).reshape(x.shape), False, int(np.prod(shape)), l2=2e-6)


@pytest.mark.parametrize("shape,batch", [((1024,), 9), ((64, 64), 2), ((1 << 14,), 2), ((1 << 16,), 2)])
def test_half_storage_padded_pitch(gpu, shape, batch):
    strides = lu.packed_strides(shape, shape[0] + 2)
    strides[-1] += 2
    x = orc.random_input((batch,) + tuple(reversed(shape)), np.complex64, seed=3) / np.sqrt(np.prod(shape))      # keep the spectrum in half's range
    xh = np.ascontiguousarray(np.stack([x.real, x.imag], axis=-1).astype(np.float16))
    _, got, _, _ = run_inplace(gpu, shape, batch, -1, strides, x=xh.view(np.uint32)[..., 0], dtype=np.uint32, halfPrecision=1)
    gh = np.ascontiguousarray(got)[..., None].view(np.float16).astype(np.float64)
    ref = orc.c2c(xh[..., 0].astype(np.float64) + 1j * xh[..., 1].astype(np.float64), len(shape))
    assert orc.error_metrics(gh[..., 0] + 1j * gh[..., 1], ref)["l2_rel"] < 1e-3         # half: eps = 9.8e-4


# ---------------------------------------------------------------- the torch front-end ----------------------------------------------------------------
def test_fft_module_refuses_non_contiguous_views_and_leaves_their_storage_alone(gpu):
    """vkfft_b200.fft takes contiguous tensors only (it raises before any launch); on a contiguous copy of a view the result is
    right and the wider tensor the view was cut from keeps every bit"""
    torch = gpu
    from vkfft_b200 import fft as vkfft
    wide = orc.random_input((6, 40, 80), np.complex64, seed=9)
    t = torch.from_numpy(wide).cuda()
    for view in (t[..., :64], t.transpose(1, 2), t[:, ::2, :]):
        with pytest.raises(ValueError):
            vkfft.fftn(view, ndim=2)
        with pytest.raises(ValueError):
            vkfft.ifftn(view, view, ndim=1)
    y = vkfft.fftn(t[..., :64].contiguous(), ndim=2, norm=0)
    torch.cuda.synchronize()
    assert same_bits(t.cpu().numpy(), wide)
    check(y.cpu().numpy(), orc.c2c(wide[..., :64], 2), False, 40 * 64)
    r = torch.from_numpy(wide.real.copy()).cuda()
    with pytest.raises(ValueError):
        vkfft.rfftn(r[..., :64], ndim=1)
    with pytest.raises(ValueError):
        vkfft.dctn(r.transpose(0, 1), ndim=1)
    h = vkfft.rfftn(r[..., :64].contiguous(), ndim=1, norm=0)
    torch.cuda.synchronize()
    assert same_bits(r.cpu().numpy(), wide.real)
    check(h.cpu().numpy(), orc.r2c(wide.real[..., :64], 1), False, 64, l2=TOL_REAL32)
    vkfft.clear_cache()
