"""Planning distributed R2C slab plans in the PRODUCT library without a device (b200fft_debug_plan_text): unlike the
emulation's planner it sees the plan-time kernels.  A rank's plan of a 512 x 512 x 256 real field runs the kernels of the
single-GPU plan of the same array -- specialised ones only -- with as many launches."""
import ctypes
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))


def _text(L, shape, inverse, **kw):
    import emu                                   # only for the ctypes mirror of b200fft_desc
    d = emu.make_desc(shape, 1, 0, perform_r2c=1, **kw)
    buf = ctypes.create_string_buffer(1 << 15)
    rc = L.b200fft_debug_plan_text(ctypes.byref(d), int(inverse), buf, len(buf))
    return rc, buf.value.decode()


@pytest.fixture(scope="module")
def lib():
    from vkfft_b200 import _lib
    L = _lib.load()
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here: no plan-time kernels to plan with")
    return L


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_distributed_r2c_plan_uses_only_specialised_kernels(lib, world, inverse):
    shape = (512, 512, 256)
    rc, single = _text(lib, shape, inverse)
    assert rc == 0
    for rank in (0, world - 1):
        rc, txt = _text(lib, shape, inverse, user_temp_buffer=1, dist_world=world, dist_rank=rank)
        assert rc == 0, rc
        lines = txt.strip().split("\n")
        assert len(lines) == len(single.strip().split("\n")), txt
        assert "generic" not in txt, txt
        assert sum("r2c axis0 (fused)" in l or "c2r axis0 (fused)" in l for l in lines) == 1, txt
