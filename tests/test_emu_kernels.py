"""CPU: the kernel *bodies* (the same templates nvcc compiles for sm_90a) run on the thread-per-CUDA-thread
emulation in tests/emu and are compared with the oracle; whole plans (planner + kernels) too.  This is how
index maps, twiddle tables, the autosort scatter and the Four-Step plumbing are verified without a GPU."""
import os

import numpy as np
import pytest

import emu
import vkfft_oracle as orc


def _kernels():
    return [k for k in emu.kernels() if k["ops"] == 0 and k["kind"] <= emu.KIND_COLS]


def _ids(k):
    return f"kind{k['kind']}-p{k['prec']}-n{k['n']}-inv{k['inv']}-v{k['variant']}"


@pytest.mark.parametrize("k", [k for k in _kernels() if k["n"] <= 2048], ids=_ids)
def test_every_kernel_matches_oracle(k):
    n, q = k["n"], k["q"]
    dt = np.complex64 if k["prec"] == 0 else np.complex128
    G = q + 3 if n * q <= 16384 else q          # ragged group where cheap
    x = orc.random_input((G, n), dt, seed=n + k["kind"])
    ref = orc.c2c(x, 1, bool(k["inv"]))
    if k["kind"] == emu.KIND_ROWS:
        y = np.zeros_like(x)
        rep = emu.run_pass(k["kind"], k["prec"], n, k["inv"], 0, x, y, G, in_gs=n, out_gs=n, log=True, variant=k['variant'])
        got = y
    elif k["kind"] == emu.KIND_ROWS_TOUT:
        y = np.zeros((n, G), dtype=dt)
        rep = emu.run_pass(k["kind"], k["prec"], n, k["inv"], 0, x, y, G, in_gs=n, out_gs=1, out_es=G, log=True, variant=k['variant'])
        got = y.T
    else:
        xt = np.ascontiguousarray(x.T)
        y = np.zeros((n, G), dtype=dt)
        rep = emu.run_pass(k["kind"], k["prec"], n, k["inv"], 0, xt, y, G, in_gs=1, out_gs=1, in_es=G, out_es=G, log=True, variant=k['variant'])
        got = y.T
    assert orc.error_metrics(got, ref)["l2_rel"] < (3e-7 if k["prec"] == 0 else 1e-15)
    # shared-memory traffic: never worse than 2-way conflicts on average 1.5 wavefronts per ideal one
    if k["variant"] == 0 and (n & (n - 1)) == 0:
        assert rep["mean"] <= 2.0 and rep["worst"] <= 4.0
    else:           # tuning variants and odd radices: only guard against pathological layouts
        assert rep["mean"] <= 6.0


def _plan_case(shape_xyz, batches, prec, env=None, inverse=-1, normalize=0):
    for key in ("B200FFT_FOUR_STEP_SPLIT", "B200FFT_MAX_SINGLE_PASS"):
        os.environ.pop(key, None)
    if env:
        os.environ.update(env)
    try:
        dt = np.complex64 if prec == 0 else np.complex128
        x = orc.random_input((batches,) + tuple(reversed(shape_xyz)), dt, seed=sum(shape_xyz))
        buf = x.copy()
        rc, npass = emu.exec_plan(emu.make_desc(shape_xyz, batches, prec, normalize=normalize), inverse, buf)
        assert rc == 0
        ref = orc.c2c(x, len(shape_xyz), inverse == 1, bool(normalize))
        return orc.error_metrics(buf, ref)["l2_rel"], npass
    finally:
        for key in ("B200FFT_FOUR_STEP_SPLIT", "B200FFT_MAX_SINGLE_PASS"):
            os.environ.pop(key, None)


@pytest.mark.parametrize("case", [
    dict(shape_xyz=(4096,), batches=3, prec=0, passes=1),
    dict(shape_xyz=(4096,), batches=3, prec=0, inverse=1, normalize=1, passes=1),
    dict(shape_xyz=(32768,), batches=2, prec=0, passes=2),
    dict(shape_xyz=(32768,), batches=2, prec=0, inverse=1, passes=2),
    dict(shape_xyz=(65536,), batches=1, prec=1, passes=2),
    dict(shape_xyz=(4096,), batches=3, prec=0, env={"B200FFT_MAX_SINGLE_PASS": "1024"}, passes=2),
    dict(shape_xyz=(4096,), batches=3, prec=0, env={"B200FFT_MAX_SINGLE_PASS": "1024", "B200FFT_FOUR_STEP_SPLIT": "16,16,16"}, passes=3),
    dict(shape_xyz=(32768,), batches=2, prec=0, inverse=1, env={"B200FFT_FOUR_STEP_SPLIT": "32,16,64"}, passes=3),
    dict(shape_xyz=(32768,), batches=2, prec=0, env={"B200FFT_FOUR_STEP_SPLIT": "16,2048"}, passes=2),   # TMA-fed last pass
    dict(shape_xyz=(16384,), batches=3, prec=0, passes=1),                                                # TMA-fed single pass
    dict(shape_xyz=(16, 8192), batches=1, prec=0, passes=3),                                              # strided Four-Step
    dict(shape_xyz=(24, 256), batches=2, prec=0, inverse=1, env={"B200FFT_MAX_SINGLE_PASS": "64"}, passes=3),
    dict(shape_xyz=(8, 4, 128), batches=2, prec=1, env={"B200FFT_MAX_SINGLE_PASS": "32"}, passes=4),
    dict(shape_xyz=(64, 32), batches=2, prec=0, passes=2),
    dict(shape_xyz=(32, 16, 8), batches=2, prec=1, passes=3),
    dict(shape_xyz=(32, 16, 8), batches=2, prec=1, inverse=1, normalize=1, passes=3),
    dict(shape_xyz=(8, 4, 4, 2), batches=3, prec=0, passes=4),
], ids=lambda c: "-".join(str(v) for v in c.values()))
def test_whole_plans_on_emulation(case):
    passes = case.pop("passes")
    err, npass = _plan_case(**case)
    assert npass == passes
    assert err < (5e-7 if case["prec"] == 0 else 1e-15)


def test_planner_rejects_what_it_cannot_do():
    d = emu.make_desc((130,), 1, 0, perform_dst=1, perform_dct=2)     # two real-to-real kinds at once
    rc, _ = emu.exec_plan(d, -1, np.zeros(130, np.float32))
    assert rc == 3004
    d = emu.make_desc((8,), 1, 0)
    d.fft_dim = 0
    assert emu.exec_plan(d, -1, np.zeros(8, np.complex64))[0] == 2001
    d = emu.make_desc((8,), 1, 0)
    d.fft_dim = 5
    assert emu.exec_plan(d, -1, np.zeros(8, np.complex64))[0] == 7


def test_emulation_checkers_catch_races_and_out_of_bounds_accesses():
    """the emulation's racecheck / bounds check must fire on deliberately broken kernels (and stay quiet on a correct one),
    otherwise "0 hazards" in the kernel tests above would mean nothing"""
    L = emu.lib()
    assert L.emu_selftest_checkers(0) == 0          # write own slot, barrier, read the neighbour's
    assert L.emu_selftest_checkers(1) > 0           # same without the barrier: read-after-write hazard
    assert L.emu_selftest_checkers(2) > 0           # two threads write the same word
    assert L.emu_selftest_checkers(3) == 1          # store one element past the allocation
