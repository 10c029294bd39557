"""CPU: the runtime-scheduled kernel (generic.cuh) with its fused operators -- non power-of-two radices, Bluestein,
R2C/C2R, DCT-I..IV -- executed as whole plans on the kernel-body emulation and compared with the oracle."""
import numpy as np
import pytest

import emu
import vkfft_oracle as orc

T32, T64 = 8e-7, 3e-15


@pytest.mark.parametrize("shape,b,prec", [((1000,), 3, 0), ((2187,), 2, 0), ((77,), 5, 1), ((30030,), 1, 0), ((105, 30), 2, 0),
                                          ((7, 11, 13), 2, 1), ((48, 20), 1, 0), ((13 * 13,), 3, 0), ((11 * 11 * 11,), 1, 1)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_smooth_non_pow2_c2c(shape, b, prec, inv):
    dt = np.complex64 if prec == 0 else np.complex128
    x = orc.random_input((b,) + tuple(reversed(shape)), dt, seed=sum(shape))
    buf = x.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec), inv, buf)
    assert rc == 0
    assert orc.error_metrics(buf, orc.c2c(x, len(shape), inv == 1))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("shape,b,prec", [((131,), 4, 0), ((509,), 2, 0), ((1019,), 1, 1), ((262,), 3, 0), ((149, 8), 2, 0),
                                          ((8, 139), 2, 1), ((4093,), 1, 0), ((4391,), 2, 0), ((5003,), 1, 1),
                                          ((20011,), 1, 0), ((6, 4391), 1, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_bluestein_c2c(shape, b, prec, inv):
    dt = np.complex64 if prec == 0 else np.complex128
    x = orc.random_input((b,) + tuple(reversed(shape)), dt, seed=sum(shape) + 1)
    buf = x.copy()
    rc, npass = emu.exec_plan(emu.make_desc(shape, b, prec), inv, buf)
    assert rc == 0
    assert orc.error_metrics(buf, orc.c2c(x, len(shape), inv == 1))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("shape,b,prec", [((77,), 5, 0), ((1430,), 2, 0), ((2 * 3 * 5 * 7 * 11,), 1, 1), ((66, 26), 2, 0), ((13,), 9, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_runtime_scheduled_kernel_first_and_last_stage_from_registers(shape, b, prec, inv, monkeypatch):
    """generic.cuh::stage_io (opt-in, B200FFT_GENERIC_FUSED_IO=1: measured slower than the separate copy phases, kept
    for the record): the first butterflies read the lines from global memory, the last ones write them, operators in registers"""
    monkeypatch.setenv("B200FFT_GENERIC_FUSED_IO", "1")
    dt = np.complex64 if prec == 0 else np.complex128
    x = orc.random_input((b,) + tuple(reversed(shape)), dt, seed=sum(shape) + 17)
    buf = x.copy()
    d = emu.make_desc(shape, b, prec)
    d.normalize = 1
    rc, npass = emu.exec_plan(d, inv, buf)
    assert rc == 0
    ref = orc.c2c(x, len(shape), inv == 1)
    if inv == 1:
        ref = ref / np.prod(shape)
    assert orc.error_metrics(buf, ref)["l2_rel"] < (T32 if prec == 0 else T64)


def _one_launch_lengths():
    """every padded length of kernel_list_blue1.def, reached from the largest N it serves and from the smallest one"""
    ms = {0: sorted(k["n"] for k in emu.kernels() if k["ops"] == 1024 and k["prec"] == 0),
          1: sorted(k["n"] for k in emu.kernels() if k["ops"] == 1024 and k["prec"] == 1)}
    cases = []
    for prec, lst in ms.items():
        prev = 0
        for m in lst:
            hi, lo = (m + 1) // 2, prev // 2 + 1           # 2N-1 <= m  and  2N-1 > previous padded length
            for n in sorted({hi, max(lo, 2)}):
                cases.append((n, m, prec))
            prev = m
    return cases


@pytest.mark.parametrize("n,m,prec", _one_launch_lengths())
def test_bluestein_in_one_launch_every_padded_length(n, m, prec, monkeypatch):
    """stockham.cuh RMODE 11 (chirp, FFT_M, filter in registers, IFFT_M, chirp in ONE launch, no scratch): every registered
    padded length M in both precisions, forward and inverse with normalisation, ragged batch, against the oracle; the
    generic route is forced (no curated kernel, no Rader stage) so that smooth N take the Bluestein path as well"""
    monkeypatch.setenv("B200FFT_FORCE_BLUESTEIN", "1")
    dt = np.complex64 if prec == 0 else np.complex128
    b = 37 if m <= 256 else (5 if m <= 2048 else 2)
    x = orc.random_input((b, n), dt, seed=n + m)
    buf = x.copy()
    rc, npass = emu.exec_plan(emu.make_desc((n,), b, prec), -1, buf)
    assert rc == 0 and npass == 1
    tol = T32 if prec == 0 else T64
    assert orc.error_metrics(buf, orc.c2c(x, 1))["l2_rel"] < tol
    d = emu.make_desc((n,), b, prec)
    d.normalize = 1
    rc, npass = emu.exec_plan(d, 1, buf)
    assert rc == 0 and npass == 1
    assert orc.error_metrics(buf, x)["l2_rel"] < 2 * tol


def test_bluestein_one_launch_equals_two_launches(monkeypatch):
    """same tables, same stage code: the one-launch kernel and the two-launch plan agree to rounding"""
    x = orc.random_input((6, 509), np.complex64, seed=5)
    a, b2 = x.copy(), x.copy()
    rc, n1 = emu.exec_plan(emu.make_desc((509,), 6, 0), -1, a)
    monkeypatch.setenv("B200FFT_NO_FUSED_BLUESTEIN", "1")
    rc2, n2 = emu.exec_plan(emu.make_desc((509,), 6, 0), -1, b2)
    assert rc == 0 and rc2 == 0 and n1 == 1 and n2 == 2
    assert orc.error_metrics(a, b2)["l2_rel"] < 3e-7


@pytest.mark.parametrize("shape,b,prec", [((17,), 5, 0), ((127,), 3, 1), ((1088,), 2, 0), ((2032,), 2, 0), ((94,), 3, 0), ((529,), 2, 0),
                                          ((323,), 2, 1), ((12167,), 1, 0), ((64, 17), 2, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_rader_prime_radix_stages(shape, b, prec, inv, monkeypatch):
    """prime factors 17..127 as Rader stages inside one shared-memory pass (reference probe: 1088 = 17.16.4,
    2032 = 8.127.2, 12167 = 23^3 in two passes; SURVEY.md appendix C).  Since the GPU timings of round 2 the planner only
    takes this path above 2048 points (below, Bluestein is faster); the switch keeps
    the Rader code under test at every length."""
    monkeypatch.setenv("B200FFT_RADER_MAX_PRIME", "127")
    dt = np.complex64 if prec == 0 else np.complex128
    x = orc.random_input((b,) + tuple(reversed(shape)), dt, seed=sum(shape) + 3)
    buf = x.copy()
    rc, npass = emu.exec_plan(emu.make_desc(shape, b, prec), inv, buf)
    assert rc == 0 and npass == (2 if shape in ((12167,), (64, 17)) else 1)
    assert orc.error_metrics(buf, orc.c2c(x, len(shape), inv == 1))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("n,launches", [(127, 1), (2032, 2), (94, 1), (323, 1), (1088, 1), (136, 1), (12167, 2)])
def test_lengths_with_prime_factors_17_to_127_default_routing(n, launches):
    """up to 2048 points: a curated kernel with a direct prime butterfly (1088 = 17.64, 136 = 17.8) or the one-launch Bluestein
    kernel; longer ones keep the Rader stages (12167 = 23^3 in two passes)"""
    x = orc.random_input((3, n), np.complex64, seed=n)
    buf = x.copy()
    rc, npass = emu.exec_plan(emu.make_desc((n,), 3, 0), -1, buf)
    assert rc == 0 and npass == launches
    assert orc.error_metrics(buf, orc.c2c(x, 1))["l2_rel"] < T32


@pytest.mark.parametrize("shape,b,prec", [((64,), 4, 0), ((4096,), 2, 0), ((64, 32), 2, 0), ((30,), 3, 1), ((15,), 3, 0),
                                          ((128, 8, 4), 1, 1), ((9, 6), 2, 0), ((1000,), 2, 0)])
def test_r2c_c2r_in_place_padded(shape, b, prec):
    rdt = np.float32 if prec == 0 else np.float64
    cdt = np.complex64 if prec == 0 else np.complex128
    tol = T32 if prec == 0 else T64
    nx = shape[0]
    H = nx // 2 + 1
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=sum(shape))
    buf = np.zeros(x.shape[:-1] + (2 * H,), rdt)      # rows padded to 2*(nx/2+1) reals (vkFFT_InitializeApp.h:1000-1005)
    buf[..., :nx] = x
    d = emu.make_desc(shape, b, prec, perform_r2c=1)
    rc, _ = emu.exec_plan(d, -1, buf)
    assert rc == 0
    assert orc.error_metrics(buf.view(cdt), orc.r2c(x, len(shape)))["l2_rel"] < tol
    rc, _ = emu.exec_plan(d, 1, buf)
    assert rc == 0
    assert orc.error_metrics(buf[..., :nx], x.astype(np.float64) * np.prod(shape))["l2_rel"] < tol


def test_r2c_out_of_place_and_return_to_input():
    shape, b = (64, 16), 2
    x = orc.random_input((b, 16, 64), np.float32, 5)
    out = np.zeros((b, 16, 33), np.complex64)
    rc, _ = emu.exec_plan(emu.make_desc(shape, b, 0, perform_r2c=1, is_input_formatted=1), -1, out, inp=x.copy())
    assert rc == 0 and orc.error_metrics(out, orc.r2c(x, 2))["l2_rel"] < T32
    back = np.zeros_like(x)
    d = emu.make_desc(shape, b, 0, perform_r2c=1, is_input_formatted=1, inverse_return_to_input=1, normalize=1)
    rc, _ = emu.exec_plan(d, 1, out.copy(), inp=back)
    assert rc == 0 and orc.error_metrics(back, x)["l2_rel"] < T32


@pytest.mark.parametrize("kind", [1, 2, 3, 4])
@pytest.mark.parametrize("shape,b,prec", [((64,), 3, 0), ((33,), 2, 1), ((32, 16), 3, 0), ((100,), 2, 1), ((8, 6, 4), 2, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_dct(kind, shape, b, prec, inv):
    rdt = np.float32 if prec == 0 else np.float64
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=kind + sum(shape))
    buf = x.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec, perform_dct=kind), inv, buf)
    assert rc == 0
    assert orc.error_metrics(buf, orc.dct(x, kind, len(shape), inverse=(inv == 1)))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("shape,b,prec", [((64, 256), 2, 0), ((256, 64), 1, 0), ((63, 64), 2, 0), ((512, 256), 1, 1), ((128, 64, 4), 1, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_dct23_fused_into_specialised_kernels(kind, shape, b, prec, inv):
    """axis 0: pairs of contiguous real lines; other axes: pairs of neighbouring real columns as one complex column;
    odd size[0] falls back to the runtime-scheduled kernel"""
    rdt = np.float32 if prec == 0 else np.float64
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=kind + sum(shape))
    buf = x.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec, perform_dct=kind), inv, buf)
    assert rc == 0
    assert orc.error_metrics(buf, orc.dct(x, kind, len(shape), inverse=(inv == 1)))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("kind,shape,b,prec,inv", [(k, sh, b, p, i) for k in (2, 3) for sh, b, p in (((8, 4096), 1, 0), ((6, 8192), 1, 0), ((4, 8192), 1, 1))
                                                   for i in (-1, 1) if sh[1] == 4096 or (k == 2) == (i == -1)])     # 8192: DCT-II forward, DCT-III inverse
def test_long_strided_dct23(kind, shape, b, prec, inv):
    """strided axis of 4096 / 8192 points: Four-Step along the stride, Makhoul permutation folded into the first gather
    (DCT-II) or the last scatter (DCT-III), split/merge as an elementwise launch"""
    rdt = np.float32 if prec == 0 else np.float64
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=kind + sum(shape))
    buf = x.copy()
    rc, npass = emu.exec_plan(emu.make_desc(shape, b, prec, perform_dct=kind), inv, buf)
    assert rc == 0 and npass == 4
    assert orc.error_metrics(buf, orc.dct(x, kind, len(shape), inverse=(inv == 1)))["l2_rel"] < (T32 if prec == 0 else T64)


def test_dct_normalized_round_trip():
    x = orc.random_input((2, 16, 32), np.float32, 9)
    for kind in (1, 2, 3, 4):
        buf = x.copy()
        d = emu.make_desc((32, 16), 2, 0, perform_dct=kind, normalize=1)
        assert emu.exec_plan(d, -1, buf)[0] == 0
        assert emu.exec_plan(d, 1, buf)[0] == 0
        assert orc.error_metrics(buf, x)["l2_rel"] < T32


@pytest.mark.parametrize("kind", [1, 2, 3, 4])
@pytest.mark.parametrize("shape,b,prec", [((64,), 3, 0), ((33,), 2, 1), ((32, 16), 3, 0), ((8, 6, 4), 2, 0)])
@pytest.mark.parametrize("inv", [-1, 1])
def test_dst(kind, shape, b, prec, inv):
    rdt = np.float32 if prec == 0 else np.float64
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=kind + sum(shape))
    buf = x.copy()
    rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec, perform_dst=kind), inv, buf)
    assert rc == 0
    assert orc.error_metrics(buf, orc.dst(x, kind, len(shape), inverse=(inv == 1)))["l2_rel"] < (T32 if prec == 0 else T64)


@pytest.mark.parametrize("shape,b,prec", [((65536,), 2, 0), ((2 * 4391,), 1, 0), ((34,), 3, 0), ((32768, 4), 1, 1), ((2 * 509, 6), 2, 0)])
def test_long_and_non_smooth_even_r2c(shape, b, prec):
    """half-length C2C (Four-Step / Bluestein) + separate Hermitian pass"""
    rdt = np.float32 if prec == 0 else np.float64
    cdt = np.complex64 if prec == 0 else np.complex128
    tol = T32 if prec == 0 else T64
    nx, H = shape[0], shape[0] // 2 + 1
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=sum(shape))
    buf = np.zeros(x.shape[:-1] + (2 * H,), rdt)
    buf[..., :nx] = x
    d = emu.make_desc(shape, b, prec, perform_r2c=1)
    assert emu.exec_plan(d, -1, buf)[0] == 0
    assert orc.error_metrics(buf.view(cdt), orc.r2c(x, len(shape)))["l2_rel"] < tol
    assert emu.exec_plan(d, 1, buf)[0] == 0
    assert orc.error_metrics(buf[..., :nx], x.astype(np.float64) * np.prod(shape))["l2_rel"] < tol


def test_r2r_composed_with_a_c2c_plan_for_lengths_the_single_launch_kernel_cannot_take():
    """transform lengths with a prime factor above 127 (DST-I 130 -> 262 = 2*131, DCT-IV 131 -> 262) or too long for one
    shared-memory pass: operator load side, C2C plan on scratch, operator store side"""
    import scipy.fft as sfft
    rng = np.random.default_rng(3)
    for mode, kind, n in (("dst", 1, 130), ("dct", 4, 131), ("dct", 2, 131), ("dct", 3, 262), ("dct", 1, 132), ("dst", 4, 139), ("dct", 2, 20000)):
        x = rng.uniform(-1, 1, (2, n)).astype(np.float32)
        buf = x.copy()
        rc, npass = emu.exec_plan(emu.make_desc((n,), 2, 0, **{"perform_" + mode: kind}), -1, buf)
        assert rc == 0 and npass >= 3, (mode, kind, n, rc, npass)
        f = sfft.dst if mode == "dst" else sfft.dct
        assert orc.error_metrics(buf, f(x.astype(np.float64), type=kind, axis=-1))["l2_rel"] < T32, (mode, kind, n)


@pytest.mark.parametrize("shape,b,prec", [((131,), 3, 0), ((263,), 2, 1), ((4391,), 2, 0), ((19683,), 1, 0), ((131, 6), 2, 0), ((139, 4, 3), 1, 1)])
def test_odd_r2c_composed_with_a_c2c_plan(shape, b, prec):
    """odd lengths the single-launch kernel cannot take (prime factor > 127, or too long): real -> complex scratch, C2C plan
    (Bluestein / Four-Step), first n/2+1 points; inverse: Hermitian expansion, C2C, real part"""
    rdt = np.float32 if prec == 0 else np.float64
    cdt = np.complex64 if prec == 0 else np.complex128
    tol = T32 if prec == 0 else T64
    nx, H = shape[0], shape[0] // 2 + 1
    x = orc.random_input((b,) + tuple(reversed(shape)), rdt, seed=sum(shape))
    buf = np.zeros(x.shape[:-1] + (2 * H,), rdt)
    buf[..., :nx] = x
    d = emu.make_desc(shape, b, prec, perform_r2c=1, normalize=1)
    assert emu.exec_plan(d, -1, buf)[0] == 0
    assert orc.error_metrics(buf.view(cdt), orc.r2c(x, len(shape)))["l2_rel"] < tol
    assert emu.exec_plan(d, 1, buf)[0] == 0
    assert orc.error_metrics(buf[..., :nx], x)["l2_rel"] < tol


@pytest.mark.parametrize("case", ["c2c3d", "r2c2d", "dct1d", "freq"])
def test_zero_padding_clears_the_flagged_ranges_before_the_first_read(case):
    """performZeropadding (API guide :1786-1807, sample_4 / sample_51): the padded ranges may hold anything, the transform
    must behave as if they were zero"""
    rng = np.random.default_rng(5)
    if case == "c2c3d":
        shape = (16, 12, 8)
        x = (rng.uniform(-1, 1, (2, 8, 12, 16)) + 1j * rng.uniform(-1, 1, (2, 8, 12, 16))).astype(np.complex64)
        left, right = [8, 6, 4], [16, 12, 8]
        clean = x.copy(); clean[..., 8:] = 0; clean[:, :, 6:, :] = 0; clean[:, 4:, :, :] = 0
        buf = x.copy()
        d = emu.make_desc(shape, 2, 0, perform_zeropadding=[1, 1, 1], zeropad_left=left, zeropad_right=right)
        assert emu.exec_plan(d, -1, buf)[0] == 0
        assert orc.error_metrics(buf, np.fft.fftn(clean.astype(np.complex128), axes=(1, 2, 3)))["l2_rel"] < T32
    elif case == "r2c2d":
        nx, ny = 32, 10
        x = rng.uniform(-1, 1, (3, ny, nx)).astype(np.float32)
        clean = x.copy(); clean[..., 20:] = 0; clean[:, 5:8, :] = 0
        buf = np.full((3, ny, nx + 2), 7.0, np.float32); buf[..., :nx] = x
        d = emu.make_desc((nx, ny), 3, 0, perform_r2c=1, perform_zeropadding=[1, 1], zeropad_left=[20, 5], zeropad_right=[32, 8])
        assert emu.exec_plan(d, -1, buf)[0] == 0
        assert orc.error_metrics(buf.view(np.complex64), np.fft.rfft2(clean.astype(np.float64)))["l2_rel"] < T32
    elif case == "dct1d":
        n = 64
        x = rng.uniform(-1, 1, (4, n)).astype(np.float32)
        clean = x.copy(); clean[:, 40:] = 0
        buf = x.copy()
        d = emu.make_desc((n,), 4, 0, perform_dct=2, perform_zeropadding=[1], zeropad_left=[40], zeropad_right=[64])
        assert emu.exec_plan(d, -1, buf)[0] == 0
        assert orc.error_metrics(buf, orc.dct(clean, 2, 1))["l2_rel"] < T32
    else:
        n = 256
        x = (rng.uniform(-1, 1, (2, n)) + 1j * rng.uniform(-1, 1, (2, n))).astype(np.complex64)
        clean = x.copy(); clean[:, 64:192] = 0
        d = emu.make_desc((n,), 2, 0, perform_zeropadding=[1], zeropad_left=[64], zeropad_right=[192], frequency_zeropadding=1)
        buf = x.copy()
        assert emu.exec_plan(d, -1, buf)[0] == 0                    # forward: untouched by frequency-domain padding
        assert orc.error_metrics(buf, np.fft.fft(x.astype(np.complex128), axis=-1))["l2_rel"] < T32
        buf = x.copy()
        assert emu.exec_plan(d, 1, buf)[0] == 0
        assert orc.error_metrics(buf, np.fft.ifft(clean.astype(np.complex128), axis=-1) * n)["l2_rel"] < T32
