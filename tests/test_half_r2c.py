"""halfPrecision with performR2C: even-length R2C / C2R with half-precision storage on both sides (real rows of float16, the
spectrum in complex32), FP32 arithmetic.  An even-length R2C addresses its real samples in pairs, and a pair of half reals is
one 32-bit element -- the element the half C2C kernels already convert -- so the fused R2C / C2R kernels (stockham.cuh RMODE 1 /
2) and the Hermitian launch of the long lengths (ew.cuh) get half variants that convert at the HBM boundary only.

Tolerance as in test_half_storage.py: the oracle runs in float64 on the SAME half inputs, the result is rounded to half once,
so the relative l2 error is a few 1e-4; 1e-3 is asserted (2e-3 for a round trip, which rounds twice)."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import vkfft_oracle as orc

TOL = 1e-3
HALF, HALF_IO = 2, 3                    # b200fft_desc.precision: halfPrecision, halfPrecisionMemoryOnly
R2C_UNSUPPORTED = 3003                  # VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C
OP_REAL_EVEN, OP_HALF_IN, OP_HALF_OUT = 16, 2048, 4096


def _real_half(shape, seed, scale=1.0):
    """half-representable reals as float16 and as float64"""
    rng = np.random.default_rng(seed)
    h = (rng.uniform(-1, 1, shape) * scale).astype(np.float16)
    return h, h.astype(np.float64)


def _spectrum_half(batch_shape, n, seed, scale):
    """a half-representable Hermitian half spectrum (the spectrum of a real signal, times `scale`), packed [..., n//2+1, 2]"""
    _, x = _real_half(tuple(batch_shape) + (n,), seed)
    y = orc.r2c(x, 1) * scale
    y[..., 0] = y[..., 0].real
    y[..., -1] = y[..., -1].real                  # n even: DC and Nyquist are real
    packed = np.empty(y.shape + (2,), np.float16)
    packed[..., 0], packed[..., 1] = y.real, y.imag
    return packed


def _unpack(packed):
    return packed[..., 0].astype(np.float64) + 1j * packed[..., 1].astype(np.float64)


def _half_c2c_length(n):
    """the support rule of the half C2C plans up to 4096 points (test_planner_product.py): 31-smooth, not a bare prime 17...31.
    Longer lengths run as Four-Step, whose factors are 2...16-smooth"""
    m = n
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31):
        while m % p == 0:
            m //= p
    return n >= 2 and m == 1 and n not in (17, 19, 23, 29, 31)


# ------------------------------------------------------------ CPU emulation ------------------------------------------------------------
@pytest.mark.parametrize("N,b", [(128, 37), (200, 5), (2048, 3)])
def test_emulated_fused_r2c_c2r_in_place(N, b):
    """one launch per direction; rows of N + 2 halves (the spectrum's n/2+1 complex32 elements)"""
    import emu
    H = N // 2 + 1
    buf = np.zeros((b, N + 2), np.float16)
    buf[:, :N], x = _real_half((b, N), N + b)
    d = emu.make_desc((N,), b, HALF, perform_r2c=1)
    rc, npass = emu.exec_plan(d, -1, buf)
    assert rc == 0 and npass == 1, rc
    assert orc.error_metrics(_unpack(buf.reshape(b, H, 2)), orc.r2c(x, 1))["l2_rel"] < TOL
    spec = _spectrum_half((b,), N, N + 1, 1.0 / N)
    buf = spec.reshape(b, N + 2).copy()
    rc, npass = emu.exec_plan(d, 1, buf)
    assert rc == 0 and npass == 1, rc
    assert orc.error_metrics(buf[:, :N].astype(np.float64), orc.c2r(_unpack(spec), 1, N))["l2_rel"] < TOL


@pytest.mark.parametrize("N,b", [(128, 9), (2048, 2)])
def test_emulated_out_of_place_and_normalised_round_trip(N, b):
    """isInputFormatted + inverseReturnToInputBuffer: the real rows stay in inputBuffer, the forward leaves them bit for bit"""
    import emu
    H = N // 2 + 1
    src, x = _real_half((b, N), 3 * N)
    keep = src.copy()
    spec = np.zeros((b, H, 2), np.float16)
    d = emu.make_desc((N,), b, HALF, perform_r2c=1, is_input_formatted=1, inverse_return_to_input=1, normalize=1)
    rc, npass = emu.exec_plan(d, -1, spec, inp=src)
    assert rc == 0 and npass == 1 and np.array_equal(src.view(np.uint16), keep.view(np.uint16))
    assert orc.error_metrics(_unpack(spec), orc.r2c(x, 1))["l2_rel"] < TOL
    src[:] = 0
    rc, npass = emu.exec_plan(d, 1, spec, inp=src)
    assert rc == 0 and npass == 1
    assert orc.error_metrics(src.astype(np.float64), x)["l2_rel"] < 2 * TOL


def test_emulated_four_step_and_half_hermitian_launch(monkeypatch):
    """N = 8192: no one-launch kernel for n = 4096 -> Four-Step 64 x 64 on the real pairs (scratch in half) + the half Hermitian
    launch; forward, inverse and the normalised round trip"""
    import emu
    monkeypatch.setenv("B200FFT_MAX_SINGLE_PASS", "64")
    N, b = 8192, 3
    buf = np.zeros((b, N + 2), np.float16)
    buf[:, :N], x = _real_half((b, N), 5)
    d = emu.make_desc((N,), b, HALF, perform_r2c=1)
    rc, text = emu.describe(d, -1)
    assert rc == 0 and "hermitian" in text and "half in+out" in text, text
    rc, npass = emu.exec_plan(d, -1, buf)
    assert rc == 0 and npass == 3, (rc, npass)
    assert orc.error_metrics(_unpack(buf.reshape(b, N // 2 + 1, 2)), orc.r2c(x, 1))["l2_rel"] < TOL
    spec = _spectrum_half((b,), N, 6, 1.0 / N)
    buf = spec.reshape(b, N + 2).copy()
    rc, npass = emu.exec_plan(d, 1, buf)
    assert rc == 0 and npass == 3
    assert orc.error_metrics(buf[:, :N].astype(np.float64), orc.c2r(_unpack(spec), 1, N))["l2_rel"] < TOL
    buf = np.zeros((b, N + 2), np.float16)
    buf[:, :N], x = _real_half((b, N), 7)
    d = emu.make_desc((N,), b, HALF, perform_r2c=1, normalize=1)
    assert emu.exec_plan(d, -1, buf)[0] == 0 and emu.exec_plan(d, 1, buf)[0] == 0
    assert orc.error_metrics(buf[:, :N].astype(np.float64), x)["l2_rel"] < 2 * TOL


def test_emulated_lengths_without_a_half_plan_are_refused():
    import emu
    for N in (63, 2, 34, 2 * 37):          # odd, N = 2, N/2 a bare prime 17 (Bluestein), N/2 = 37 (not 31-smooth)
        buf = np.zeros((2, N + 2), np.float16)
        assert emu.exec_plan(emu.make_desc((N,), 2, HALF, perform_r2c=1), -1, buf)[0] == R2C_UNSUPPORTED, N


# ------------------------------------------------------------ product planner, no device ------------------------------------------------------------
def _text(L, shape, batch=2, prec=HALF, inverse=-1, **kw):
    import emu                                   # only for the ctypes mirror of b200fft_desc
    d = emu.make_desc(shape, batch, prec, **kw)
    buf = ctypes.create_string_buffer(1 << 15)
    rc = L.b200fft_debug_plan_text(ctypes.byref(d), int(inverse), buf, len(buf))
    return rc, buf.value.decode()


@pytest.fixture(scope="module")
def lib():
    from vkfft_b200 import _lib
    L = _lib.load()
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here: no plan-time kernels to plan with")
    L.b2_jit_selftest.restype = ctypes.c_long
    return L


def _all_half(txt):
    lines = txt.strip().split("\n")
    return lines and all("half in+out" in l for l in lines)


def test_every_even_length_with_a_half_c2c_plan_plans_in_half(lib):
    """N even up to 20000: planned entirely from half kernels exactly where a half C2C plan of N/2 exists, else 3003"""
    planned = fused = 0
    for N in range(2, 20001, 2):
        rc_c2c, _ = _text(lib, (N // 2,))
        if N <= 8192:
            assert N == 2 or (rc_c2c == 0) == _half_c2c_length(N // 2), N      # (a 1-point C2C is the identity)
        for inverse in ((-1, 1) if N <= 4200 or N % 64 == 0 else (-1,)):
            rc, txt = _text(lib, (N,), 3, inverse=inverse, perform_r2c=1)
            if N == 2 or rc_c2c != 0:
                assert rc == R2C_UNSUPPORTED, (N, rc)
                continue
            assert rc == 0, (N, inverse, rc)
            assert _all_half(txt), (N, txt)
            planned += 1
            fused += "fused" in txt
    assert planned > 1500 and fused > 1000, (planned, fused)
    for N in (3, 15, 1001, 4097):
        assert _text(lib, (N,), 3, perform_r2c=1)[0] == R2C_UNSUPPORTED, N


def test_multidimensional_half_r2c_plans_in_half(lib):
    for shape in ((4096, 4096), (1000, 300), (128, 64, 32)):
        for inverse in (-1, 1):
            rc, txt = _text(lib, shape, 2, inverse=inverse, perform_r2c=1)
            assert rc == 0 and _all_half(txt), (shape, rc, txt)
            assert txt.count("\n") + 1 >= len(shape)


def test_refused_half_real_combinations(lib, monkeypatch):
    # halfPrecisionMemoryOnly has no real-data variant
    assert _text(lib, (4096,), 2, HALF_IO, is_input_formatted=1, perform_r2c=1)[0] == 3002
    # cosine transforms and convolution stay refused in half
    assert _text(lib, (64,), 2, HALF, perform_dct=2)[0] == 3002
    assert _text(lib, (64,), 2, HALF, perform_convolution=1)[0] == 3002
    # half kernels exist only as plan-time instantiations
    monkeypatch.setenv("B200FFT_NO_JIT", "1")
    assert _text(lib, (4096,), 2, HALF, perform_r2c=1)[0] != 0


def test_half_real_kernels_compile_without_a_gpu(lib):
    for n in (2048, 500, 550, 8192):
        size = lib.b2_jit_selftest(0, 0, n, OP_REAL_EVEN | OP_HALF_IN | OP_HALF_OUT)
        assert size > 5000, (n, size, lib.b2_jit_last_log().decode() if size < 0 else "")
    # mixed storage and non-contiguous real kernels do not exist
    assert lib.b2_jit_selftest(0, 0, 64, OP_REAL_EVEN | OP_HALF_IN) == 0
    assert lib.b2_jit_selftest(0, 0, 64, OP_REAL_EVEN | OP_HALF_OUT) == 0
    assert lib.b2_jit_selftest(2, 0, 64, OP_REAL_EVEN | OP_HALF_IN | OP_HALF_OUT) == 0


# ---------------------------------------------------------------- GPU ----------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    import vkfft_b200  # noqa: F401
    from vkfft_b200 import _lib
    if not _lib.load().b2_jit_available():
        pytest.skip("half-storage kernels are instantiated at plan time: libnvrtc is not loadable here")
    return torch


class _App:
    def __init__(self, shape, batch, **kw):
        import vkfft_b200 as vk
        self.vk = vk
        self.app = vk.VkFFTApplication()
        rc = vk.initializeVkFFT(self.app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0,
                                                                performR2C=1, **kw))
        assert rc == 0, vk.getVkFFTErrorString(rc)
        self.info = vk.planInfo(self.app)

    def run(self, torch, inverse, **lp):
        assert self.vk.VkFFTAppend(self.app, inverse, self.vk.VkFFTLaunchParams(**lp)) == 0
        torch.cuda.synchronize()

    def close(self):
        self.vk.deleteVkFFT(self.app)


def _input_scale(shape):
    # keep the spectrum inside half's range: |X| ~ sqrt(n) * s stays far below 65504
    return 1.0 if int(np.prod(shape)) <= (1 << 16) else 2.0 ** -6


GPU_CASES = [((8,), 1001), ((64,), 333), ((1000,), 17), ((1100,), 5), ((4096,), 9), ((16384,), 3), ((1 << 15,), 3),
             ((1 << 20,), 2), ((10 ** 6,), 1), ((4096, 4096), 2), ((1000, 300), 3), ((128, 64, 32), 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,batch", GPU_CASES)
@pytest.mark.parametrize("inplace", [True, False])
def test_half_r2c_c2r_vs_oracle(gpu, shape, batch, inplace):
    torch, nd, N = gpu, len(shape), shape[0]
    H = N // 2 + 1
    rshape = (batch,) + tuple(reversed(shape))
    cshape = rshape[:-1] + (H,)
    xh, x = _real_half(rshape, sum(shape) + batch, _input_scale(shape))
    # inverse input: the spectrum of real data scaled by 1/prod(shape), so that the unnormalised C2R stays inside half's range
    if nd == 1:
        spec = _spectrum_half(rshape[:-1], N, sum(shape) + 1, 1.0 / N)
    else:            # Hermitian along every axis: half rounding keeps conjugate pairs conjugate
        spec_c = orc.r2c(_real_half(rshape, sum(shape) + 2)[1], nd) / int(np.prod(shape))
        spec = np.stack([spec_c.real, spec_c.imag], -1).astype(np.float16)
    ref_inv = orc.c2r(_unpack(spec), nd, N)
    if inplace:
        app = _App(shape, batch, halfPrecision=1)
        try:
            assert _all_half(app.info["forward"]) and _all_half(app.info["inverse"]), app.info
            buf = np.zeros(rshape[:-1] + (N + 2,), np.float16)
            buf[..., :N] = xh
            t = torch.from_numpy(buf).cuda()
            app.run(torch, -1, buffer=t)
            got = t.cpu().numpy().reshape(cshape + (2,))
            assert orc.error_metrics(_unpack(got), orc.r2c(x, nd))["l2_rel"] < TOL
            t = torch.from_numpy(spec.reshape(rshape[:-1] + (N + 2,)).copy()).cuda()
            app.run(torch, 1, buffer=t)
            assert orc.error_metrics(t.cpu().numpy()[..., :N].astype(np.float64), ref_inv)["l2_rel"] < TOL
        finally:
            app.close()
    else:
        app = _App(shape, batch, halfPrecision=1, isInputFormatted=1, inverseReturnToInputBuffer=1)
        try:
            src = torch.from_numpy(xh.copy()).cuda()
            dst = torch.zeros(cshape + (2,), dtype=torch.float16, device="cuda")
            app.run(torch, -1, buffer=dst, inputBuffer=src)
            assert np.array_equal(src.cpu().numpy().view(np.uint16), xh.view(np.uint16)), "the source of the forward was modified"
            assert orc.error_metrics(_unpack(dst.cpu().numpy()), orc.r2c(x, nd))["l2_rel"] < TOL
            dst = torch.from_numpy(spec.copy()).cuda()
            src.zero_()
            app.run(torch, 1, buffer=dst, inputBuffer=src)
            assert orc.error_metrics(src.cpu().numpy().astype(np.float64), ref_inv)["l2_rel"] < TOL
        finally:
            app.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4096, 1000])
def test_half_forward_equals_rounded_fp32_storage(gpu, N):
    """single-launch R2C: the same FP32 schedule on the same (half-representable) input, rounded to half once at the store --
    the half result is float16(FP32-storage result) bit for bit"""
    torch, b = gpu, 7
    xh, _ = _real_half((b, N), N)
    outs = {}
    for half in (0, 1):
        app = _App((N,), b, halfPrecision=half)
        try:
            assert "fused" in app.info["forward"] and app.info["forward"].strip().count("\n") == 0, app.info["forward"]
            buf = np.zeros((b, N + 2), np.float16 if half else np.float32)
            buf[:, :N] = xh
            t = torch.from_numpy(buf).cuda()
            app.run(torch, -1, buffer=t)
            outs[half] = t.cpu().numpy()
        finally:
            app.close()
    want = outs[0].astype(np.float16)
    assert np.array_equal(outs[1].view(np.uint16), want.view(np.uint16)), \
        f"{int((outs[1].view(np.uint16) != want.view(np.uint16)).sum())} of {want.size} halves differ"


@pytest.mark.gpu
def test_half_r2c_guard_bands(gpu):
    """padded pitch in place (spectrum rows H + 3 complex32 apart, real rows in the same rows) and out of place with a padded real
    pitch; caller-owned scratch of exactly temp_bytes between guards.  Nothing outside the footprints may change"""
    import layout_util as lu
    from test_gpu_layouts import Dev, Plan, dev_layout
    torch = gpu
    for shape, batch in (((4096,), 3), ((1 << 15,), 2)):
        N = shape[0]
        H = N // 2 + 1
        cs = lu.packed_strides((H,), H + 3)
        cs[-1] += 6
        xh, x = _real_half((batch, N), N + 11, _input_scale(shape))
        L = lu.make_layout((H,), batch, cs, np.uint32)
        lu.view_of(L.flat, shape, batch, [2 * s for s in cs], np.float16, L.guard)[...] = xh
        D = Dev(torch, L.flat, L.mask, L)
        p = Plan(torch, shape, batch, performR2C=1, bufferStride=cs, halfPrecision=1)
        assert p.rc == 0
        try:
            assert _all_half(p.text(-1)) and _all_half(p.text(1))
            p.run(-1, D.ptr)
            D.fetch()
            got = L.gather().view(np.float16).reshape(batch, H, 2)
            assert orc.error_metrics(_unpack(got), orc.r2c(x, 1))["l2_rel"] < TOL
            D.before = L.flat.copy()
            p.run(1, D.ptr)
            D.fetch()
            real = np.array(lu.view_of(L.flat, shape, batch, [2 * s for s in cs], np.float16, L.guard)).astype(np.float64)
            assert orc.error_metrics(real, orc.c2r(_unpack(got), 1, N))["l2_rel"] < TOL
        finally:
            p.close()
        # out of place: real rows N + 6 halves apart in inputBuffer, packed spectrum rows with a gap
        rs = lu.packed_strides(shape, N + 6)
        cs = lu.packed_strides((H,), H + 2)
        cfg = dict(performR2C=1, isInputFormatted=1, bufferStride=cs, inputBufferStride=rs, halfPrecision=1)
        p = Plan(torch, shape, batch, **cfg)
        assert p.rc == 0
        (Li, Di), (Lb, Db) = dev_layout(torch, shape, batch, rs, np.float16, xh, "inputBuffer"), dev_layout(torch, (H,), batch, cs, np.uint32)
        try:
            p.run(-1, Db.ptr, inp=Di.ptr)
        finally:
            p.close()
        Di.fetch_unmodified(); Db.fetch()
        got = Lb.gather().view(np.float16).reshape(batch, H, 2)
        assert orc.error_metrics(_unpack(got), orc.r2c(x, 1))["l2_rel"] < TOL


# torch's half FFT rounds between its stages; against it, a looser bound than against the float64 oracle
TORCH_TOL = 1e-2


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [0, 1, "ortho"])
@pytest.mark.parametrize("shape,ndim", [((6, 1024), 1), ((64, 128), 2), ((3, 16384), 1)])
def test_fft_module_half_dtypes(gpu, norm, shape, ndim):
    """rfftn / irfftn on float16 / complex32 and fftn / ifftn on complex32 against torch.fft on the same tensors and the oracle"""
    torch = gpu
    from vkfft_b200 import fft as vf
    tnorm = {0: None, 1: "backward", "ortho": "ortho"}[norm]
    axes = tuple(range(len(shape) - ndim, len(shape)))
    n = int(np.prod(shape[len(shape) - ndim:]))
    xh, x = _real_half(shape, n + ndim)
    r = torch.from_numpy(xh).cuda()
    h = vf.rfftn(r, ndim=ndim, norm=norm)
    assert h.dtype == torch.complex32 and tuple(h.shape) == shape[:-1] + (shape[-1] // 2 + 1,)
    want = orc.r2c(x, ndim) / (np.sqrt(n) if norm == "ortho" else 1.0)
    got = _unpack(torch.view_as_real(h).cpu().numpy())
    assert orc.error_metrics(got, want)["l2_rel"] < TOL
    if tnorm is not None:
        th = torch.fft.rfftn(r, dim=axes, norm=tnorm)
        assert orc.error_metrics(got, _unpack(torch.view_as_real(th).cpu().numpy()))["l2_rel"] < TORCH_TOL
    hin = got
    back = vf.irfftn(h, ndim=ndim, norm=norm, n_last=shape[-1])
    assert back.dtype == torch.float16
    want = orc.c2r(hin, ndim, shape[-1]) / (np.sqrt(n) if norm == "ortho" else (n if norm == 1 else 1.0))
    assert orc.error_metrics(back.cpu().numpy().astype(np.float64), want)["l2_rel"] < TOL
    if norm != 0:
        assert orc.error_metrics(back.cpu().numpy().astype(np.float64), x)["l2_rel"] < 2 * TOL
    # complex32 C2C, out of place and in place
    c = torch.view_as_complex(torch.stack([r, r.flip(-1)], -1).contiguous())
    cx = _unpack(torch.view_as_real(c).cpu().numpy())
    y = vf.fftn(c, ndim=ndim, norm=norm)
    assert y.dtype == torch.complex32
    got = _unpack(torch.view_as_real(y).cpu().numpy())
    assert orc.error_metrics(got, orc.c2c(cx, ndim) / (np.sqrt(n) if norm == "ortho" else 1.0))["l2_rel"] < TOL
    if tnorm is not None:
        ty = torch.fft.fftn(c, dim=axes, norm=tnorm)
        assert orc.error_metrics(got, _unpack(torch.view_as_real(ty).cpu().numpy()))["l2_rel"] < TORCH_TOL
    yin = _unpack(torch.view_as_real(y).cpu().numpy())
    vf.ifftn(y, y, ndim=ndim, norm=norm)
    want = orc.c2c(yin, ndim, inverse=True) / (np.sqrt(n) if norm == "ortho" else (n if norm == 1 else 1.0))
    assert orc.error_metrics(_unpack(torch.view_as_real(y).cpu().numpy()), want)["l2_rel"] < TOL


@pytest.mark.gpu
def test_fft_module_refuses_dtypes_without_a_variant(gpu):
    torch = gpu
    from vkfft_b200 import fft as vf
    before = dict(vf._CACHE)
    r16 = torch.zeros((4, 64), dtype=torch.float16, device="cuda")
    bf = torch.zeros((4, 64), dtype=torch.bfloat16, device="cuda")
    for call in (lambda: vf.dctn(r16), lambda: vf.dstn(r16), lambda: vf.idctn(r16), lambda: vf.rfftn(bf), lambda: vf.dctn(bf),
                 lambda: vf.fftn(bf), lambda: vf.irfftn(bf), lambda: vf.rfftn(torch.zeros((4, 64), dtype=torch.int32, device="cuda"))):
        with pytest.raises(TypeError):
            call()
    assert vf._CACHE == before, "a refused dtype created a plan"
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_half_r2c_timing_is_reported(gpu):
    """N = 4096 x 2^15 R2C + C2R in place: the half pair moves half the bytes; the test records both times and only guards
    against a pathological kernel (halving the bytes need not halve a single-pass kernel's time)"""
    import vkfft_b200 as vk
    torch = gpu
    N, batch = 4096, 1 << 15
    times = {}
    for half in (0, 1):
        t = torch.zeros(batch * (N + 2), dtype=torch.float16 if half else torch.float32, device="cuda").uniform_(-1, 1)
        app = _App((N,), batch, halfPrecision=half, normalize=1)
        lp = vk.VkFFTLaunchParams(buffer=t)
        for _ in range(3):
            vk.VkFFTAppend(app.app, -1, lp); vk.VkFFTAppend(app.app, 1, lp)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            vk.VkFFTAppend(app.app, -1, lp); vk.VkFFTAppend(app.app, 1, lp)
        b.record(); torch.cuda.synchronize()
        times[half] = a.elapsed_time(b) / 10
        app.close()
        del t
    print(f"R2C+C2R N=4096 x 2^15: FP32 storage {times[0]:.3f} ms, half storage {times[1]:.3f} ms per pair")
    assert times[1] < 2.0 * times[0], times
