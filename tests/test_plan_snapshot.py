"""CPU: the planner's choices for the headline workload are the measured-best ones (the pass costs in
planner.cpp::split_four_step: every registered kernel timed alone on a 2 GiB pass by tools/ktune.py).  A change here is a
performance change: re-measure with tools/ktune.py / bench.py before updating."""
import os
import re
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402

SWEEP = {
    7: [("128", "ROWS")], 8: [("256", "ROWS")], 9: [("512", "ROWS")], 10: [("1024", "ROWS")], 11: [("2048", "ROWS")],
    12: [("4096", "ROWS")], 13: [("8192", "ROWS")], 14: [("16384", "PIPE1_ROWS")],
    15: [("128", "COLS"), ("256", "ROWS_TOUT")], 16: [("128", "COLS"), ("512", "ROWS_TOUT")],
    17: [("128", "COLS"), ("1024", "ROWS_TOUT")], 18: [("512", "COLS"), ("512", "ROWS_TOUT")],
    19: [("512", "COLS"), ("1024", "ROWS_TOUT")], 20: [("2048", "COLS"), ("512", "ROWS_TOUT")],
    21: [("2048", "COLS"), ("1024", "ROWS_TOUT")], 22: [("128", "COLS"), ("128", "COLS"), ("256", "ROWS_TOUT")],
}


def _launches(desc, inverse=-1):
    rc, txt = emu.describe(desc, inverse)
    assert rc == 0
    return [l for l in txt.strip().split("\n") if l]


@pytest.mark.parametrize("log2n", sorted(SWEEP))
def test_sweep_plan(log2n):
    for inv in (-1, 1):
        got = [re.search(r"n=(\d+) (\S+?)<", l).groups() for l in _launches(emu.make_desc((1 << log2n,), (1 << 28) >> log2n, 0), inv)]
        assert got == SWEEP[log2n]


@pytest.mark.parametrize("desc_kw,launches", [
    (dict(shape=(256, 256, 256), b=8, prec=1), 3),                              # 3-D FP64: one launch per axis
    (dict(shape=(512, 512, 512), b=1, prec=1), 3),
    (dict(shape=(4096, 4096), b=16, prec=0, perform_r2c=1), 3),                 # fused R2C axis 0 + Four-Step along the stride
    (dict(shape=(8192, 8192), b=2, prec=0, perform_dct=2), 4),                  # fused DCT rows + long strided DCT (3 launches)
    (dict(shape=(1 << 26,), b=4, prec=0), 3),                                   # three-launch Four-Step
    (dict(shape=(1088,), b=1 << 17, prec=0), 1),                                # prime-radix specialised kernel
    (dict(shape=(509,), b=1 << 18, prec=0), 1),                                 # the whole Bluestein transform in one launch
    (dict(shape=(4093,), b=1 << 14, prec=0), 2),                                # Bluestein, two launches on the specialised kernels
    (dict(shape=(4096,), b=1 << 16, prec=0, perform_convolution=1), 1),         # fused convolution
])
def test_launch_counts_of_the_other_baseline_configurations(desc_kw, launches):
    kw = dict(desc_kw)
    shape, b, prec = kw.pop("shape"), kw.pop("b"), kw.pop("prec")
    assert len(_launches(emu.make_desc(shape, b, prec, **kw))) == launches
