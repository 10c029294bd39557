"""GPU (-m gpu): out-of-place DCT / DST with formatted inputBuffer / outputBuffer on the device.

Every buffer is a guarded allocation of tests/layout_util.py with a pitch of its own; plans run with userTempBuffer = 1 on a
scratch of exactly the reported size between two guard bands.  Each case checks the result against the oracle, the source bit
for bit, every gap and guard, and -- where the plan lists the in-place plan's launches -- bit identity with the in-place
result.  The torch front-end (dctn / idctn / dstn / idstn) must leave its source alone and give the bits of the in-place call."""
import numpy as np
import pytest

import layout_util as lu
import vkfft_oracle as orc

pytestmark = pytest.mark.gpu

TOL32, TOL64 = 2e-6, 1e-12
C_POINT = 8.0
TEMP_GUARD = 512
PITCH = {"input": (2, 6), "buffer": (4, 0), "output": (6, 10)}


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    import vkfft_b200  # noqa: F401
    return torch


def rdt(double):
    return np.float64 if double else np.float32


def check(got, ref, double, n_total):
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < (TOL64 if double else TOL32), e
    eps = np.finfo(rdt(double)).eps
    r = lu.max_line_error(got, ref)
    assert r <= lu.point_bound(n_total, eps, C_POINT), r / lu.point_bound(n_total, eps, 1.0)


def strides_of(shape, pad, batch_pad):
    s = lu.packed_strides(shape, shape[0] + pad)
    s[-1] += batch_pad
    return s


def launches(vk, app, inverse):
    txt = vk.planInfo(app)["inverse" if inverse == 1 else "forward"]
    return [line.split(": ", 1)[1].rsplit("  ", 1)[0] for line in txt.strip().split("\n")]


def flow(combo, inv):
    """-> (flags, buffers given, source role, destination role) of one direction"""
    if combo == "in":
        return dict(isInputFormatted=1), ("input", "buffer"), ("buffer" if inv == 1 else "input"), "buffer"
    if combo == "out":
        return dict(isOutputFormatted=1), ("buffer", "output"), ("output" if inv == 1 else "buffer"), ("buffer" if inv == 1 else "output")
    if combo == "both":
        return (dict(isInputFormatted=1, isOutputFormatted=1), ("input", "buffer", "output"), ("output" if inv == 1 else "input"),
                ("buffer" if inv == 1 else "output"))
    return (dict(isInputFormatted=1, inverseReturnToInputBuffer=1), ("input", "buffer"), ("buffer" if inv == 1 else "input"),
            ("input" if inv == 1 else "buffer"))


def run_case(torch, mode, kind, shape, batch, double, combo, inv, offset=0, at_launch=0, expect=None):
    """offset: byte offset of every buffer (given at plan time, or at launch with at_launch = 1)"""
    import vkfft_b200 as vk
    flags, given, src, dst = flow(combo, inv)
    dt = rdt(double)
    esz = np.dtype(dt).itemsize
    k = offset // esz
    L = {r: lu.make_layout(shape, batch, strides_of(shape, *PITCH[r]), dt, guard=lu.GUARD + k) for r in given}
    x = orc.random_input((batch,) + tuple(reversed(shape)), dt, seed=sum(shape) + kind)
    L[src].scatter(x)
    before = {r: l.flat.copy() for r, l in L.items()}
    dev = {r: torch.from_numpy(l.flat).cuda() for r, l in L.items()}
    # a buffer's data starts guard elements in: the first `offset` bytes of that reach come from the offset
    ptr = {r: int(t.data_ptr()) + (L[r].guard - k) * esz for r, t in dev.items()}
    offs = {"buffer": "bufferOffset", "input": "inputBufferOffset", "output": "outputBufferOffset"}
    cfg = dict(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0, userTempBuffer=1, doublePrecision=int(double),
               normalize=int(inv == 1), bufferStride=strides_of(shape, *PITCH["buffer"]), **{"perform" + mode.upper(): kind}, **flags)
    for r in given:
        if r != "buffer":
            cfg[r + "BufferStride"] = strides_of(shape, *PITCH[r])
    off_kw = {offs[r]: offset for r in given} if offset else {}
    if at_launch:
        cfg["specifyOffsetsAtLaunch"] = 1
    else:
        cfg.update(off_kw)
    app = vk.VkFFTApplication()
    rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(**cfg))
    assert rc == 0, vk.getVkFFTErrorString(rc)
    try:
        temp_bytes = int(vk.planInfo(app)["temp_bytes"])
        temp = torch.full((TEMP_GUARD + temp_bytes + TEMP_GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        lp = vk.VkFFTLaunchParams(buffer=ptr["buffer"], inputBuffer=ptr.get("input"), outputBuffer=ptr.get("output"),
                                  tempBuffer=int(temp.data_ptr()) + TEMP_GUARD, **(off_kw if at_launch else {}))
        assert vk.VkFFTAppend(app, inv, lp) == 0
        torch.cuda.synchronize()
        g = temp.cpu().numpy()
        assert (g[:TEMP_GUARD] == 0xA5).all() and (g[TEMP_GUARD + temp_bytes:] == 0xA5).all(), "stores outside tempBuffer"
        txt = launches(vk, app, inv)
    finally:
        vk.deleteVkFFT(app)
    for r, l in L.items():
        l.flat[...] = dev[r].cpu().numpy()
        if r == src and r != "buffer":
            lu.assert_bit_identical(l.flat, before[r], f"{r} (the source)")
        else:
            lu.assert_untouched(l.flat, before[r], l.mask, l, r)
    f = orc.dct if mode == "dct" else orc.dst
    got = L[dst].gather()
    check(got, f(x, kind, len(shape), inverse=(inv == 1), normalize=(inv == 1)), double, int(np.prod(shape)))
    # the in-place plan on a packed copy: the same launches give the same bits
    app = vk.VkFFTApplication()
    assert vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0,
                                                         doublePrecision=int(double), normalize=int(inv == 1),
                                                         **{"perform" + mode.upper(): kind})) == 0
    try:
        tref = launches(vk, app, inv)
        if expect is not None:      # the route of the in-place plan, which FP32 takes on every shape here
            assert sum(expect in t for t in txt) == sum(expect in t for t in tref), (expect, txt, tref)
            assert double or any(expect in t for t in txt), (expect, txt)
        if tref == txt:
            t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
            assert vk.VkFFTAppend(app, inv, vk.VkFFTLaunchParams(buffer=t)) == 0
            torch.cuda.synchronize()
            assert np.array_equal(lu.bits(got), lu.bits(t.cpu().numpy())), "out of place differs from in place with the same launches"
    finally:
        vk.deleteVkFFT(app)


ROUTES = [
    ("dct", 2, (64,), 33, "dct axis (fused)"), ("dct", 3, (1000,), 5, "dct axis (fused)"), ("dct", 2, (4096,), 3, "dct axis (fused)"),
    ("dct", 2, (64, 32), 2, "(fused)"), ("dct", 3, (720, 480), 1, "(fused)"), ("dct", 2, (720, 480), 2, "(fused)"),
    ("dct", 2, (16, 4096), 1, "long dct-i"), ("dct", 3, (16, 4096), 1, "long dct-i"),
    ("dct", 2, (4391,), 2, "r2r (composed)"), ("dst", 3, (4391,), 2, "r2r (composed)"),
    ("dct", 1, (33,), 5, None), ("dct", 4, (64,), 5, None), ("dct", 4, (45,), 5, None),
    ("dst", 1, (100,), 3, None), ("dst", 2, (100,), 3, None), ("dst", 3, (100,), 3, None), ("dst", 4, (100,), 3, None),
]


def _rid(r):
    return f"{r[0]}{r[1]}-{'x'.join(map(str, r[2]))}"


@pytest.mark.parametrize("combo", ["in", "out", "both", "back"])
@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("route", ROUTES, ids=_rid)
def test_routes_out_of_place(gpu, route, double, combo):
    mode, kind, shape, batch, expect = route
    for inv in (-1, 1):
        if combo == "in" and inv == 1:
            continue
        run_case(gpu, mode, kind, shape, batch, double, combo, inv, expect=expect)


# byte offsets: multiples of the complex element (8 bytes in FP32, 16 in FP64) -- the complex view of a strided axis reads pairs
@pytest.mark.parametrize("at_launch", [0, 1])
@pytest.mark.parametrize("route,double,offset", [(ROUTES[0], False, 8), (ROUTES[3], False, 24), (ROUTES[6], False, 8),
                                                 (ROUTES[8], True, 16), (ROUTES[13], True, 48)], ids=lambda v: str(v) if not isinstance(v, tuple) else _rid(v))
def test_byte_offsets(gpu, route, double, offset, at_launch):
    mode, kind, shape, batch, expect = route
    for inv in (-1, 1):
        run_case(gpu, mode, kind, shape, batch, double, "both", inv, offset=offset, at_launch=at_launch, expect=expect)


# ---------------------------------------------------------------- torch front-end ----------------------------------------------------------------
@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("ndim,shape", [(1, (6, 100)), (1, (3, 64)), (2, (2, 48, 64)), (3, (12, 10, 16))])
@pytest.mark.parametrize("kind", [1, 2, 3, 4])
@pytest.mark.parametrize("fn", ["dctn", "idctn", "dstn", "idstn"])
def test_front_end_out_of_place_equals_in_place(gpu, fn, kind, ndim, shape, double):
    torch = gpu
    from vkfft_b200 import fft as vkfft
    f = getattr(vkfft, fn)
    key = "dst_type" if "dst" in fn else "dct_type"
    g = torch.Generator(device="cpu").manual_seed(kind + ndim)
    x = torch.rand(shape, generator=g, dtype=torch.float64 if double else torch.float32).cuda() - 0.5
    src = x.clone()
    y = f(x, ndim=ndim, **{key: kind})
    torch.cuda.synchronize()
    assert torch.equal(x.view(torch.int64 if double else torch.int32), src.view(torch.int64 if double else torch.int32)), "src changed"
    z = src.clone()
    f(z, dest=z, ndim=ndim, **{key: kind})
    dest = torch.full_like(x, float("nan"))
    f(x, dest=dest, ndim=ndim, **{key: kind})
    torch.cuda.synchronize()
    iv = torch.int64 if double else torch.int32
    assert torch.equal(y.view(iv), z.view(iv)) and torch.equal(dest.view(iv), z.view(iv))
    ref = (orc.dst if "dst" in fn else orc.dct)(src.cpu().numpy(), kind, ndim, inverse=fn.startswith("i"))
    n = 1
    for s in shape[len(shape) - ndim:]:
        n *= 2 * (s - 1) if (kind == 1 and "dct" in fn) else (2 * (s + 1) if kind == 1 else 2 * s)
    if fn.startswith("i"):
        ref = ref / n                     # norm=1: the backward transform carries 1/N
    assert orc.error_metrics(y.cpu().numpy(), ref)["l2_rel"] < (1e-12 if double else 2e-6)


def test_front_end_identity_and_dest_checks(gpu):
    torch = gpu
    from vkfft_b200 import fft as vkfft
    x = torch.rand((4, 1), device="cuda")
    y = vkfft.dctn(x, ndim=1, dct_type=2)
    torch.cuda.synchronize()
    assert y.data_ptr() != x.data_ptr() and torch.equal(y, x)
    with pytest.raises(ValueError):
        vkfft.dctn(torch.rand((4, 8), device="cuda"), dest=torch.empty((4, 9), device="cuda"))
