"""Planning distributed DCT / DST slab plans in the PRODUCT library without a device (b200fft_debug_plan_text): unlike the
emulation's planner it sees the plan-time kernels.

- A rank's plan of BASELINE config 4 (DCT-II 8192 x 8192, FP32) and of a 512 x 512 x 256 DCT-II / DST-II runs the kernels of the
  single-GPU plan of the same array, with as many launches.
- The distributed C2C and R2C plans keep their plan texts: tests/golden/dist_plan_texts_c2c_r2c.json holds the texts the
  planner gave before distributed DCT / DST existed, written by this file's `_record` in a fresh process (kernel lookups may
  depend on the plan-time kernels a process has instantiated before), and this test records them the same way."""
import ctypes
import json
import os
import re
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "dist_plan_texts_c2c_r2c.json")
sys.path.insert(0, os.path.join(HERE, "emu"))

# distributed C2C and R2C plans whose texts must not change: (shape, R2C, world)
KEPT = [
    ((1 << 16,), 0, 2), ((256, 128), 0, 2), ((64, 32, 16), 0, 4), ((512, 512, 256), 0, 8), ((8192, 8192), 0, 4),
    ((2048, 1024), 1, 2), ((128, 64), 1, 4), ((64, 8192), 1, 2), ((256, 128, 64), 1, 2), ((512, 512, 256), 1, 4),
    ((512, 512, 256), 1, 8),
]


def _text(L, shape, inverse, **kw):
    import emu                                   # only for the ctypes mirror of b200fft_desc
    d = emu.make_desc(shape, 1, 0, **kw)
    buf = ctypes.create_string_buffer(1 << 16)
    rc = L.b200fft_debug_plan_text(ctypes.byref(d), int(inverse), buf, len(buf))
    return rc, buf.value.decode()


def _kernels(text):
    """the kernel of every launch, in order (pass numbers, grid sizes, item counts and barrier marks left out)"""
    return [re.sub(r" (grid|items)=\d+", "", re.split(r"  (buffer|temp) ->", line.split(": ", 1)[-1])[0]).split(" n=", 1)[-1]
            for line in text.strip().split("\n")]


def _record(L):
    out = {}
    for shape, r2c, world in KEPT:
        for rank in sorted({0, world - 1}):
            for inv in (-1, 1):
                rc, txt = _text(L, shape, inv, perform_r2c=r2c, user_temp_buffer=1, dist_world=world, dist_rank=rank)
                key = f"{'r2c' if r2c else 'c2c'} {'x'.join(map(str, shape))} R={world} rank={rank} {'inverse' if inv == 1 else 'forward'}"
                out[key] = [rc, txt]
    return out


@pytest.fixture(scope="module")
def lib():
    from vkfft_b200 import _lib
    L = _lib.load()
    if not L.b2_jit_available():
        pytest.skip("libnvrtc not loadable here: no plan-time kernels to plan with")
    return L


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("inverse", [-1, 1])
@pytest.mark.parametrize("shape,mode", [((8192, 8192), "dct"), ((512, 512, 256), "dct"), ((512, 512, 256), "dst")])
def test_distributed_r2r_plan_runs_the_single_gpu_kernels(lib, shape, mode, world, inverse):
    kw = {"perform_" + mode: 2}
    rc, single = _text(lib, shape, inverse, **kw)
    assert rc == 0
    for rank in (0, world - 1):
        rc, txt = _text(lib, shape, inverse, user_temp_buffer=1, dist_world=world, dist_rank=rank, **kw)
        assert rc == 0, rc
        assert _kernels(txt) == _kernels(single), (txt, single)
    if shape == (8192, 8192) and mode == "dct":
        assert sum("long dct-ii" in line for line in single.strip().split("\n")) == 3, single


def test_distributed_c2c_and_r2c_plan_texts_unchanged(lib):
    out = subprocess.run([sys.executable, os.path.abspath(__file__)], capture_output=True, text=True, check=True,
                         cwd=os.path.dirname(HERE)).stdout
    got = json.loads(out)
    with open(GOLDEN) as fh:
        want = json.load(fh)
    assert sorted(got) == sorted(want)
    for key in want:
        assert got[key] == want[key], (key, got[key], want[key])


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    from vkfft_b200 import _lib
    print(json.dumps(_record(_lib.load()), indent=1, sort_keys=True))
