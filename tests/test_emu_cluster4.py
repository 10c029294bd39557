"""CPU: the cluster Four-Step launch (csrc/cluster4.cuh) on the kernel-body emulation with thread-block clusters
(tests/emu/cuda_emu_cluster.h, tests/emu/emu_cluster.py).

The emulated planner sees a cluster-capable device only when emu.set_cluster_capable(True) is called; by default it plans
for a device without clusters, as the product library does on a machine without a GPU.  The emulation runs the CTAs of one
cluster concurrently with a cluster-wide barrier, maps peer shared memory for the distributed-shared-memory stores, and checks
every such access for bounds and for races between cluster barriers.  Both passes run the stage code of the two stand-alone
kernels, so the result must equal the two-launch plan bit for bit."""
import os
import re

import numpy as np
import pytest

import emu_cluster as emu
import vkfft_oracle as orc


class env:
    def __init__(self, **kw):
        self.kw = {k: str(v) for k, v in kw.items()}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kw}
        os.environ.update(self.kw)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class clusters:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        emu.set_cluster_capable(self.on)

    def __exit__(self, *a):
        emu.set_cluster_capable(False)


def run(desc, inv, x, capable=True, **kw):
    with env(**kw), clusters(capable):
        rc, txt = emu.describe(desc, inv)
        buf = x.copy()
        rc2, npass = emu.exec_plan(desc, inv, buf)
    assert rc == 0 and rc2 == 0, (rc, rc2)
    return buf, txt


def pinned(txt):
    return [re.search(r"n=(\d+) (\S+?)<", l).groups() for l in txt.strip().split("\n") if l]


@pytest.mark.parametrize("logn", [15, 16])
@pytest.mark.parametrize("inv", [-1, 1])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("normalize", [0, 1])
def test_cluster_matches_two_launch_plan_and_oracle(logn, inv, batch, normalize):
    n = 1 << logn
    x = orc.random_input((batch, n), np.complex64, seed=logn * 10 + batch)
    d = emu.make_desc((n,), batch, normalize=normalize)
    got, txt = run(d, inv, x)
    assert "one cluster launch with the next pass: CLUSTER4<" in txt and "[runs inside the previous launch]" in txt, txt
    plain, txt2 = run(d, inv, x, capable=False)
    assert "cluster" not in txt2
    assert np.array_equal(got.view(np.float32), plain.view(np.float32))
    ref = orc.c2c(x, 1, inv == 1)
    if normalize and inv == 1:
        ref = ref / n
    assert orc.error_metrics(got, ref)["l2_rel"] < 8e-7


@pytest.mark.parametrize("logn", [15, 16])
def test_plan_text_keeps_the_pinned_lines(logn):
    d = emu.make_desc((1 << logn,), (1 << 28) >> logn, 0)
    for inv in (-1, 1):
        with clusters():
            rc, txt = emu.describe(d, inv)
        rc2, txt2 = emu.describe(d, inv)
        assert rc == 0 and rc2 == 0
        assert pinned(txt) == pinned(txt2) and len(pinned(txt)) == 2
        lines = txt.strip().split("\n")
        assert "one cluster launch with the next pass" in lines[0] and "runs inside the previous launch" in lines[1]
        assert "fused" not in txt


def test_long_axis_of_a_2d_shape():
    nx, ny, batch = 1 << 15, 3, 2
    x = orc.random_input((batch, ny, nx), np.complex64, seed=11)
    d = emu.make_desc((nx, ny), batch)
    got, txt = run(d, -1, x)
    assert "one cluster launch" in txt, txt
    plain, _ = run(d, -1, x, capable=False)
    assert np.array_equal(got.view(np.float32), plain.view(np.float32))
    assert orc.error_metrics(got, orc.c2c(x, 2, False))["l2_rel"] < 8e-7


def test_out_of_place_and_user_temp_buffer():
    n, batch = 1 << 16, 2
    x = orc.random_input((batch, n), np.complex64, seed=5)
    for kw in (dict(user_temp_buffer=1), dict(is_input_formatted=1)):
        d = emu.make_desc((n,), batch, **kw)
        with clusters():
            rc, txt = emu.describe(d, -1)
            assert rc == 0 and "one cluster launch" in txt, txt
            buf = np.zeros_like(x) if kw.get("is_input_formatted") else x.copy()
            inp = x.copy() if kw.get("is_input_formatted") else None
            if inp is None:
                assert emu.exec_plan(d, -1, buf)[0] == 0
            else:
                assert emu.exec_plan(d, -1, buf, inp=inp)[0] == 0
                assert np.array_equal(inp, x)                 # the input is only read
        assert orc.error_metrics(buf, orc.c2c(x, 1))["l2_rel"] < 8e-7


def test_plans_without_cluster_launch():
    n = 1 << 16
    with clusters():
        with env(B200FFT_NO_CLUSTER4=1):
            assert "cluster" not in emu.describe(emu.make_desc((n,), 2), -1)[1]
        assert "cluster" not in emu.describe(emu.make_desc((n,), 2, prec=1), -1)[1]          # FP64
        assert "cluster" not in emu.describe(emu.make_desc((n,), 2, prec=2), -1)[1]          # half-precision storage
        rc, txt = emu.describe(emu.make_desc((n,), 1, 0, user_temp_buffer=1, dist_world=2, dist_rank=0), -1)
        assert rc == 0 and "cluster" not in txt                                            # distributed
        with env(B200FFT_FUSED4=1):                                                        # the opt-in L2 fusion keeps priority
            txt = emu.describe(emu.make_desc((n,), 2), -1)[1]
            assert "fused with the next launch" in txt and "cluster" not in txt
        for logn in (17, 18):                                                              # no cluster kernel registered
            assert "cluster" not in emu.describe(emu.make_desc((1 << logn,), 2), -1)[1]
    assert "cluster" not in emu.describe(emu.make_desc((n,), 2), -1)[1]                     # no cluster-capable device


def test_cluster_checkers():
    assert emu.selftest_checkers(0) == 0      # barrier between the local and the remote store
    assert emu.selftest_checkers(1) > 0       # no barrier: another CTA's store races with the owner's
    assert emu.selftest_checkers(2) == 1      # beyond the peer's allocation
    assert emu.selftest_checkers(3) == 1      # a CTA rank outside the cluster
