"""halfPrecision (vkFFT_Structs.h:210): every buffer holds half-precision complex elements (32 bits: half re, half im), the
arithmetic is FP32; the conversion is fused into the first-stage load / last-stage store of the specialised kernels
(stockham.cuh KCfg::ST).  The product instantiates these kernels at plan time (jit.cpp); the CPU emulation registers a few
ahead of time so that the conversion code runs in the CPU suite.  Tolerance: the result is rounded to half once (relative
2^-11 per element), the input is exactly representable, so the L2 error against the oracle on the SAME half inputs is a few
1e-4; 1e-3 is asserted (the reference's own half-precision test, sample_13, only prints its errors)."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import vkfft_oracle as orc

TOL = 1e-3


def _half_input(shape, seed):
    """complex values exactly representable in half, as the uint32-per-element buffer and as complex128"""
    rng = np.random.default_rng(seed)
    re = rng.uniform(-1, 1, shape).astype(np.float16)
    im = rng.uniform(-1, 1, shape).astype(np.float16)
    packed = np.empty(shape + (2,), np.float16)
    packed[..., 0], packed[..., 1] = re, im
    return packed, re.astype(np.float64) + 1j * im.astype(np.float64)


def _unpack(packed):
    return packed[..., 0].astype(np.float64) + 1j * packed[..., 1].astype(np.float64)


# ------------------------------------------------------------ CPU emulation ------------------------------------------------------------
def test_host_half_conversions_match_ieee_round_to_nearest_even():
    """the conversions behind the emulated kernels: every half value survives half -> float -> half, and float -> half agrees
    with numpy (ties to even, subnormals, overflow to infinity) on random values, on every midpoint and next to it"""
    import emu
    L = emu.lib()
    L.emu_half_bits_to_float.restype = ctypes.c_float
    L.emu_half_bits_to_float.argtypes = [ctypes.c_ushort]
    L.emu_float_to_half_bits.restype = ctypes.c_ushort
    L.emu_float_to_half_bits.argtypes = [ctypes.c_float]
    allh = np.arange(65536, dtype=np.uint16)
    vals = allh.view(np.float16).astype(np.float32)
    for h, v in zip(allh[::7].tolist(), vals[::7].tolist()):
        if np.isnan(v):
            continue
        assert L.emu_half_bits_to_float(h) == v or (v == 0 and L.emu_half_bits_to_float(h) == 0), h
        assert L.emu_float_to_half_bits(v) == h, h
    rng = np.random.default_rng(0)
    finite = vals[np.isfinite(vals)]
    mids = ((finite[:-1].astype(np.float64) + np.roll(finite, -1)[:-1].astype(np.float64)) / 2).astype(np.float32)[::13]
    cases = np.concatenate([rng.uniform(-70000, 70000, 3000).astype(np.float32), rng.uniform(-1e-4, 1e-4, 3000).astype(np.float32),
                            mids, np.nextafter(mids, np.float32(np.inf)), np.nextafter(mids, np.float32(-np.inf))])
    with np.errstate(over="ignore"):
        want = cases.astype(np.float16).view(np.uint16)
    for c, w in zip(cases.tolist(), want.tolist()):
        assert L.emu_float_to_half_bits(c) == w, (c, w)



@pytest.mark.parametrize("n,b", [(64, 37), (100, 5), (1024, 3), (8, 200)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_emulated_single_pass(n, b, inv):
    import emu
    buf, x = _half_input((b, n), n + b)
    rc, npass = emu.exec_plan(emu.make_desc((n,), b, 2), inv, buf)
    assert rc == 0 and npass == 1
    ref = orc.c2c(x, 1, inv == 1)
    assert orc.error_metrics(_unpack(buf), ref)["l2_rel"] < TOL


def test_emulated_four_step_and_strided_axis(monkeypatch):
    """4096 = 64 x 64 (strided + phase launch, then contiguous launch with transposed store; scratch in half as well), and a
    2-D transform whose second axis runs on the strided kernel"""
    import emu
    monkeypatch.setenv("B200FFT_MAX_SINGLE_PASS", "64")
    buf, x = _half_input((3, 4096), 7)
    rc, npass = emu.exec_plan(emu.make_desc((4096,), 3, 2), -1, buf)
    assert rc == 0 and npass == 2
    assert orc.error_metrics(_unpack(buf) / 64, orc.c2c(x, 1) / 64)["l2_rel"] < TOL
    buf, x = _half_input((2, 64, 64), 8)
    rc, npass = emu.exec_plan(emu.make_desc((64, 64), 2, 2), -1, buf)
    assert rc == 0 and npass == 2
    assert orc.error_metrics(_unpack(buf), orc.c2c(x, 2))["l2_rel"] < TOL


def test_emulated_normalised_round_trip_and_out_of_place():
    import emu
    buf, x = _half_input((9, 64), 3)
    d = emu.make_desc((64,), 9, 2, normalize=1)
    assert emu.exec_plan(d, -1, buf)[0] == 0
    assert emu.exec_plan(d, 1, buf)[0] == 0
    assert orc.error_metrics(_unpack(buf), x)["l2_rel"] < 2 * TOL      # two roundings to half
    src, x = _half_input((4, 100), 5)
    dst = np.zeros_like(src)
    keep = src.copy()
    d = emu.make_desc((100,), 4, 2, is_input_formatted=1)
    rc, _ = emu.exec_plan(d, -1, dst, inp=src)
    assert rc == 0 and np.array_equal(src, keep)
    assert orc.error_metrics(_unpack(dst), orc.c2c(x, 1))["l2_rel"] < TOL


def test_emulated_memory_only_half_input_buffer():
    """halfPrecisionMemoryOnly (precision 3): inputBuffer in half, buffer in FP32; forward inputBuffer -> buffer, inverse with
    inverseReturnToInputBuffer buffer -> inputBuffer (the reference converts in exactly these two places,
    vkFFT_InitAPIParameters.h:153-172)"""
    import emu
    src, x = _half_input((5, 64), 11)
    keep = src.copy()
    buf = np.zeros((5, 64), np.complex64)
    d = emu.make_desc((64,), 5, 3, is_input_formatted=1, inverse_return_to_input=1, normalize=1)
    rc, npass = emu.exec_plan(d, -1, buf, inp=src)
    assert rc == 0 and npass == 1 and np.array_equal(src, keep)
    assert orc.error_metrics(buf, orc.c2c(x, 1))["l2_rel"] < 1e-6           # half -> FP32 is exact, the spectrum is FP32
    src[:] = 0
    rc, npass = emu.exec_plan(d, 1, buf, inp=src)
    assert rc == 0 and npass == 1
    assert orc.error_metrics(_unpack(src), x)["l2_rel"] < TOL
    # Four-Step: the first launch converts on load, the scratch and the second launch are FP32
    import os
    os.environ["B200FFT_MAX_SINGLE_PASS"] = "64"
    try:
        src, x = _half_input((2, 4096), 12)
        buf = np.zeros((2, 4096), np.complex64)
        d = emu.make_desc((4096,), 2, 3, is_input_formatted=1, inverse_return_to_input=1)
        rc, npass = emu.exec_plan(d, -1, buf, inp=src)
        assert rc == 0 and npass == 2
        assert orc.error_metrics(buf, orc.c2c(x, 1))["l2_rel"] < 1e-6
    finally:
        del os.environ["B200FFT_MAX_SINGLE_PASS"]
    # without a formatted input buffer there is nothing to be half
    assert emu.exec_plan(emu.make_desc((64,), 5, 3), -1, buf)[0] == 3002


@pytest.mark.parametrize("kw", [dict(perform_r2c=1), dict(perform_dct=2), dict(perform_convolution=1)])
def test_operators_without_a_half_variant_are_refused(kw):
    import emu
    buf = np.zeros((2, 64, 2), np.float16)
    rc, _ = emu.exec_plan(emu.make_desc((64,), 2, 2, **kw), -1, buf)
    assert rc in (3002, 3003, 3004)


def test_half_kernels_compile_at_plan_time_without_a_gpu():
    from vkfft_b200 import _lib
    L = _lib.load()
    L.b2_jit_selftest.restype = ctypes.c_long
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here")
    for kind, n, ops in ((0, 4096, 2048 | 4096), (0, 8, 2048 | 4096), (2, 512, 1 | 2048 | 4096), (1, 1024, 2048 | 4096), (0, 1000, 2048)):
        assert L.b2_jit_selftest(kind, 0, n, ops) > 5000, (kind, n, ops)
    assert L.b2_jit_selftest(0, 1, 64, 2048 | 4096) == 0          # FP64 arithmetic with half storage does not exist
    assert L.b2_jit_selftest(0, 0, 64, 16 | 2048) == 0             # nor the fused real transforms


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


def _run_gpu(torch, shape, batch, inverse, buf, **kw):
    import vkfft_b200 as vk
    t = torch.from_numpy(buf.view(np.int16).copy()).cuda()       # torch has no complex32 buffer type to lean on: raw bits
    app = vk.VkFFTApplication()
    rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0, halfPrecision=1, **kw))
    assert rc == 0, vk.getVkFFTErrorString(rc)
    try:
        info = vk.planInfo(app)
        assert "half in+out" in info["forward"], info["forward"]
        assert vk.VkFFTAppend(app, inverse, vk.VkFFTLaunchParams(buffer=t)) == 0
        torch.cuda.synchronize()
        return t.cpu().numpy().view(np.float16).reshape(buf.shape), info
    finally:
        vk.deleteVkFFT(app)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,batch", [((8,), 1000), ((64,), 333), ((1000,), 17), ((4096,), 9), ((1 << 16,), 3), ((1 << 20,), 2),
                                         ((1 << 23,), 1), ((256, 256), 3), ((128, 64, 32), 2), ((1100,), 5), ((4096, 2048), 1)])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_c2c_half_storage_vs_oracle(gpu, shape, batch, inverse):
    buf, x = _half_input((batch,) + tuple(reversed(shape)), sum(shape))
    n = int(np.prod(shape))
    # keep the spectrum inside half's range: scale the input so that |X| ~ sqrt(n) * s stays far below 65504
    s = 1.0 if n <= (1 << 16) else 2.0 ** -6
    buf = (buf.astype(np.float32) * s).astype(np.float16)
    x = _unpack(buf)
    got, info = _run_gpu(gpu, shape, batch, inverse, buf)
    ref = orc.c2c(x, len(shape), inverse == 1)
    assert orc.error_metrics(_unpack(got), ref)["l2_rel"] < TOL


@pytest.mark.gpu
def test_half_storage_timing_is_reported(gpu):
    """2^27 points, N = 4096.  The half variant issues the same number of (32-bit instead of 64-bit) accesses plus the
    conversions, so halving the bytes need not halve the time of a single-pass kernel.  The test records the two numbers
    and only guards against a pathological kernel."""
    import torch
    import vkfft_b200 as vk
    n, batch = 4096, 1 << 15
    times = {}
    for half in (0, 1):
        t = torch.zeros(n * batch * 2, dtype=torch.float32, device="cuda").uniform_(-1, 1) if not half else \
            torch.zeros(n * batch, dtype=torch.int32, device="cuda")
        app = vk.VkFFTApplication()
        assert vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=1, size=[n], numberBatches=batch, device=0, halfPrecision=half)) == 0
        lp = vk.VkFFTLaunchParams(buffer=t)
        for _ in range(3):
            vk.VkFFTAppend(app, -1, lp)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            vk.VkFFTAppend(app, -1, lp)
        b.record(); torch.cuda.synchronize()
        times[half] = a.elapsed_time(b) / 10
        vk.deleteVkFFT(app)
        del t
    print(f"N=4096 x 2^15: FP32 storage {times[0]:.3f} ms, half storage {times[1]:.3f} ms")
    assert times[1] < 2.0 * times[0], times


@pytest.mark.gpu
@pytest.mark.parametrize("n,batch", [(4096, 7), (1 << 16, 2), (1000, 9)])
def test_memory_only_half_input_buffer(gpu, n, batch):
    """halfPrecisionMemoryOnly: half inputBuffer, FP32 buffer; forward inputBuffer -> buffer, inverse back into inputBuffer"""
    import torch
    import vkfft_b200 as vk
    src, x = _half_input((batch, n), n)
    tin = torch.from_numpy(src.view(np.int16).copy()).cuda()
    tbuf = torch.zeros((batch, n), dtype=torch.complex64, device="cuda")
    app = vk.VkFFTApplication()
    rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=1, size=[n], numberBatches=batch, device=0, halfPrecision=1, halfPrecisionMemoryOnly=1,
                                                       isInputFormatted=1, inverseReturnToInputBuffer=1, normalize=1))
    assert rc == 0, vk.getVkFFTErrorString(rc)
    try:
        lp = vk.VkFFTLaunchParams(buffer=tbuf, inputBuffer=tin)
        assert vk.VkFFTAppend(app, -1, lp) == 0
        torch.cuda.synchronize()
        assert orc.error_metrics(tbuf.cpu().numpy(), orc.c2c(x, 1))["l2_rel"] < 1e-6
        tin.zero_()
        assert vk.VkFFTAppend(app, 1, lp) == 0
        torch.cuda.synchronize()
        back = tin.cpu().numpy().view(np.float16).reshape(src.shape)
        assert orc.error_metrics(_unpack(back), x)["l2_rel"] < TOL
    finally:
        vk.deleteVkFFT(app)
