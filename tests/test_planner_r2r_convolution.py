"""Planning DCT / DST convolution plans in the PRODUCT library without a device (b200fft_debug_plan_text): unlike the
emulation's planner it sees the plan-time kernels.  A convolution plan is the R2R plan's forward launches, one real product
launch and the R2R plan's inverse launches (normalised), whatever route each axis takes -- except that for type 2 with a fused
DCT / DST convolution kernel for the last axis, that axis's forward launch, the product and its inverse launch are one."""
import ctypes
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))


def _launches(L, shape, batch, inverse, **kw):
    import emu                                   # only for the ctypes mirror of b200fft_desc
    d = emu.make_desc(shape, batch, 0, **kw)
    buf = ctypes.create_string_buffer(1 << 16)
    rc = L.b200fft_debug_plan_text(ctypes.byref(d), int(inverse), buf, len(buf))
    assert rc == 0, (shape, kw, rc)
    return [line.split(": ", 1)[-1] for line in buf.value.decode().strip().split("\n")]


@pytest.fixture(scope="module")
def lib():
    from vkfft_b200 import _lib
    L = _lib.load()
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here: no plan-time kernels to plan with")
    return L


@pytest.mark.parametrize("mode", ["dct", "dst"])
@pytest.mark.parametrize("shape,batch,count", [((1024, 1024), 1, 3), ((256, 256, 256), 1, 5), ((4096,), 64, 1), ((720, 480), 1, 3),
                                               ((4096, 4096), 1, None)])
def test_fused_last_axis_or_chain(lib, shape, batch, count, mode):
    kw = {"perform_" + mode: 2}
    got = _launches(lib, shape, batch, -1, perform_convolution=1, normalize=1, **kw)
    fwd = _launches(lib, shape, batch, -1, **kw)
    inv = _launches(lib, shape, batch, 1, normalize=1, **kw)
    fused = [t for t in got if "fused r2r convolution" in t]
    if fused:
        # the other axes: the R2R plan's launches of those axes, around the one fused launch
        nd = len(shape)
        assert len(fused) == 1 and got.index(fused[0]) == nd - 1 and len(got) == 2 * nd - 1, got
        assert got[:nd - 1] == fwd[:nd - 1] and got[nd:] == inv[1:], got
    else:
        assert got == fwd + [got[len(fwd)]] + inv, got
        assert "real spectrum x kernel" in got[len(fwd)]
    if count is not None:
        assert len(got) == count, got
    if shape == (4096, 4096) and mode == "dct":
        # a strided last axis longer than 2048 has no fused kernel: the long strided route runs on both sides of the product
        assert not fused and sum("long dct-ii " in t for t in got) == 3 and sum("long dct-iii" in t for t in got) == 3, got
