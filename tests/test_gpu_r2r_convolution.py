"""GPU (-m gpu): convolution plans with DCT / DST on the device, and the spectral Poisson solves they exist for.

A plan with performConvolution and performDCT / performDST runs the forward transform, the product with a real kernel in the
buffer's layout and the inverse transform behind one VkFFTAppend(app, -1).  The cases compare with the float64 oracle
(forward, product, inverse), solve Poisson's equation with Neumann (DCT-II) and Dirichlet (DST-I) walls against a float64
solve that checks itself with the 5-point Laplacian, run on caller-owned scratch of exactly the reported size, and run the
torch front-end `fft.convolve_r2r`."""
import numpy as np
import pytest

import vkfft_oracle as orc

pytestmark = pytest.mark.gpu

TOL = {False: 1e-6, True: 1e-12}
TEMP_GUARD = 512


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    import vkfft_b200  # noqa: F401
    return torch


def reference(x, k, mode, kind, nd, normalize=True):
    f = orc.dct if mode == "dct" else orc.dst
    return f(f(x, kind, nd) * k, kind, nd, inverse=True, normalize=normalize)


CASES = [   # (shape x-first, batch, double, types)
    ((8192,), 16, False, [("dct", 2), ("dst", 2), ("dct", 1), ("dst", 3)]),
    ((2048, 2048), 2, False, [("dct", 2), ("dst", 2), ("dct", 3), ("dst", 4)]),
    ((720, 480), 1, False, [("dct", 2), ("dst", 2), ("dct", 4), ("dst", 1)]),
    ((4096, 4096), 1, False, [("dct", 2), ("dst", 2)]),
    ((256, 256, 256), 1, False, [("dct", 2), ("dst", 2)]),
    ((256, 256, 128), 1, True, [("dct", 2), ("dst", 2), ("dct", 1), ("dst", 4)]),
]


@pytest.mark.parametrize("shape,batch,double,types", CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else None)
def test_against_the_oracle(gpu, shape, batch, double, types):
    from vkfft_b200 import fft
    torch = gpu
    dt = np.float64 if double else np.float32
    nps = tuple(reversed(shape))
    x = orc.random_input((batch,) + nps, dt, seed=sum(shape))
    k = orc.random_input(nps, dt, seed=len(shape))
    xs, ks = torch.from_numpy(x).cuda(), torch.from_numpy(k).cuda()
    for mode, kind in types:
        y = fft.convolve_r2r(xs, ks, ndim=len(shape), kind=kind, dst=(mode == "dst"))
        torch.cuda.synchronize()
        e = orc.error_metrics(y.cpu().numpy(), reference(x, k.astype(np.float64), mode, kind, len(shape)))["l2_rel"]
        assert e < TOL[double], (mode, kind, e)
    assert np.array_equal(xs.cpu().numpy(), x) and np.array_equal(ks.cpu().numpy(), k)
    fft.clear_cache()


@pytest.mark.parametrize("shape,batch", [((8192,), 16), ((2048, 2048), 2), ((1024, 1024), 2), ((64, 64, 256), 2)])
@pytest.mark.parametrize("dst", [False, True])
def test_fused_last_axis_matches_the_chain(gpu, shape, batch, dst):
    """type 2, packed: the last axis runs as ONE launch (2 nd - 1 launches); the chain (B200FFT_NO_FUSED_CONV=1) agrees.
    2-D / 3-D out of place (the first axis reads inputBuffer); 1-D in place, as for C2C (the fused launch reads `buffer`)"""
    import os
    import vkfft_b200 as vk
    torch = gpu
    nps = tuple(reversed(shape))
    x = orc.random_input((batch,) + nps, np.float32, seed=21)
    k = orc.random_input(nps, np.float32, seed=22)
    src, ker = torch.from_numpy(x).cuda(), torch.from_numpy(k).cuda()
    out = {}
    for chain in (False, True):
        if chain:
            os.environ["B200FFT_NO_FUSED_CONV"] = "1"
        try:
            app = vk.VkFFTApplication()
            rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0,
                                                               normalize=1, performConvolution=1, isInputFormatted=int(len(shape) > 1),
                                                               **{"performDST" if dst else "performDCT": 2}))
        finally:
            os.environ.pop("B200FFT_NO_FUSED_CONV", None)
        assert rc == 0, vk.getVkFFTErrorString(rc)
        try:
            txt = vk.planInfo(app)["forward"].strip().split("\n")
            assert (len(txt) == 2 * len(shape) - 1 and sum("fused r2r convolution" in t for t in txt) == 1) != chain, txt
            buf = torch.empty_like(src) if len(shape) > 1 else src.clone()
            assert vk.VkFFTAppend(app, -1, vk.VkFFTLaunchParams(buffer=buf, inputBuffer=src if len(shape) > 1 else None, kernel=ker)) == 0
            torch.cuda.synchronize()
            out[chain] = buf.cpu().numpy()
        finally:
            vk.deleteVkFFT(app)
    ref = reference(x, k.astype(np.float64), "dst" if dst else "dct", 2, len(shape))
    assert orc.error_metrics(out[False], ref)["l2_rel"] < TOL[False]
    assert orc.error_metrics(out[False], out[True].astype(np.float64))["l2_rel"] < TOL[False]
    assert np.array_equal(src.cpu().numpy(), x) and np.array_equal(ker.cpu().numpy(), k)


def laplacian(u, bc):
    """5-point Laplacian (unit spacing) with reflective (Neumann, half-sample symmetric ghosts) or zero (Dirichlet) walls"""
    p = np.pad(u, 1, mode="symmetric" if bc == "neumann" else "constant")
    return p[:-2, 1:-1] + p[2:, 1:-1] + p[1:-1, :-2] + p[1:-1, 2:] - 4 * u


def poisson_kernel(n, bc):
    """multiplier of the transformed right-hand side: 1 / (eigenvalue of the 5-point Laplacian), 0 for the Neumann mean"""
    if bc == "neumann":
        lam1 = 2 - 2 * np.cos(np.pi * np.arange(n) / n)                 # DCT-II modes
    else:
        lam1 = 2 - 2 * np.cos(np.pi * (np.arange(n) + 1) / (n + 1))     # DST-I modes
    lam = lam1[:, None] + lam1[None, :]
    with np.errstate(divide="ignore"):
        k = np.where(lam > 0, -1.0 / lam, 0.0)
    return k


@pytest.mark.parametrize("bc,mode,kind", [("neumann", "dct", 2), ("dirichlet", "dst", 1)])
def test_poisson_solve(gpu, bc, mode, kind):
    from vkfft_b200 import fft
    torch = gpu
    n = 512
    rng = np.random.default_rng(11)
    f = rng.standard_normal((n, n))
    if bc == "neumann":
        f -= f.mean()                                                   # solvable: zero-mean right-hand side
    k = poisson_kernel(n, bc)
    u64 = reference(f, k, mode, kind, 2)                                # the float64 solve ...
    if bc == "neumann":
        u64 -= u64.mean()
    r = laplacian(u64, bc) - f
    assert np.linalg.norm(r) / np.linalg.norm(f) < 1e-10                # ... checked against the discrete operator
    u = fft.convolve_r2r(torch.from_numpy(f.astype(np.float32)).cuda(), torch.from_numpy(k.astype(np.float32)).cuda(),
                         kind=kind, dst=(mode == "dst")).cpu().numpy().astype(np.float64)
    if bc == "neumann":
        u -= u.mean()
    # Δ amplifies FP32 rounding by about n^2: the FP32 result is compared with the float64 solution, not through the residual
    assert orc.error_metrics(u, u64)["l2_rel"] < 1e-5
    fft.clear_cache()


@pytest.mark.parametrize("shape,mode,kind", [((4096, 4096), "dct", 2), ((262, 64), "dct", 2), ((128, 64), "dst", 4)])
def test_caller_owned_scratch(gpu, shape, mode, kind):
    """userTempBuffer = 1 on exactly temp_bytes between guard bands; isInputFormatted: the source is read, never written"""
    import vkfft_b200 as vk
    torch = gpu
    nps = tuple(reversed(shape))
    x = orc.random_input((2,) + nps, np.float32, seed=5)
    k = orc.random_input(nps, np.float32, seed=6)
    src, ker = torch.from_numpy(x).cuda(), torch.from_numpy(k).cuda()
    buf = torch.empty_like(src)
    app = vk.VkFFTApplication()
    rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=2, device=0, normalize=1,
                                                       performConvolution=1, isInputFormatted=1, userTempBuffer=1,
                                                       **{"perform" + mode.upper(): kind}))
    assert rc == 0, vk.getVkFFTErrorString(rc)
    try:
        temp_bytes = int(vk.planInfo(app)["temp_bytes"])
        temp = torch.full((TEMP_GUARD + temp_bytes + TEMP_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        lp = vk.VkFFTLaunchParams(buffer=buf, inputBuffer=src, kernel=ker, tempBuffer=int(temp.data_ptr()) + TEMP_GUARD)
        assert vk.VkFFTAppend(app, -1, lp) == 0
        torch.cuda.synchronize()
        g = temp.cpu().numpy()
        assert (g[:TEMP_GUARD] == 0xA5).all() and (g[TEMP_GUARD + temp_bytes:] == 0xA5).all(), "stores outside tempBuffer"
    finally:
        vk.deleteVkFFT(app)
    assert np.array_equal(src.cpu().numpy(), x) and np.array_equal(ker.cpu().numpy(), k)
    e = orc.error_metrics(buf.cpu().numpy(), reference(x, k.astype(np.float64), mode, kind, len(shape)))["l2_rel"]
    assert e < TOL[False], e


def test_convolve_r2r_front_end(gpu):
    from vkfft_b200 import fft
    torch = gpu
    x = orc.random_input((3, 40, 64), np.float64, seed=8)
    k = orc.random_input((40, 64), np.float64, seed=9)
    xs, ks = torch.from_numpy(x).cuda(), torch.from_numpy(k).cuda()
    for ndim, kk in ((2, k), (1, k[0])):
        kt = torch.from_numpy(np.ascontiguousarray(kk)).cuda()
        for norm in (0, 1):
            y = fft.convolve_r2r(xs, kt, ndim=ndim, kind=3, norm=norm)
            ref = reference(x, kk, "dct", 3, ndim, normalize=bool(norm))
            assert orc.error_metrics(y.cpu().numpy(), ref)["l2_rel"] < TOL[True]
    assert np.array_equal(xs.cpu().numpy(), x)
    # in place: dest is src
    y = xs.clone()
    assert fft.convolve_r2r(y, ks, dest=y, ndim=2, dst=True) is y
    assert orc.error_metrics(y.cpu().numpy(), reference(x, k, "dst", 2, 2))["l2_rel"] < TOL[True]
    # a kernel of ones returns the source
    one = fft.convolve_r2r(xs, torch.ones_like(ks), ndim=2, kind=4)
    assert orc.error_metrics(one.cpu().numpy(), x)["l2_rel"] < 1e-13
    for dt in (torch.float16, torch.bfloat16, torch.int32, torch.complex64):
        t = torch.zeros((4, 8), dtype=dt, device="cuda")
        with pytest.raises(TypeError):
            fft.convolve_r2r(t, t)
    for bad in (ks.float(), ks[0], xs):
        with pytest.raises(ValueError):
            fft.convolve_r2r(xs, bad, ndim=2)
    fft.clear_cache()
