"""CPU: distributed 2-D / 3-D R2C / C2R slab plans (desc.dist_world > 1, perform_r2c) on the kernel-body emulation.

Two guarded host arrays stand for the two peer windows (`buffer` and scratch).  The array lies in the in-place R2C layout
(H = nx/2+1 complex per row, row pitch p0 >= H, in 3-D plane pitch p1 >= ny*p0); rank g's slab is the last-dimension indices
[g*n/R, (g+1)*n/R), i.e. the (n/R)*pitch complex elements from g*(n/R)*pitch on, in both windows.  Every rank's plan is built
and its launches are played in the orders the plan's barriers allow (all ranks up, all ranks down), as test_emu_dist.py does
for the C2C slab plans.  Checked: the result against numpy rfftn / irfftn in float64, two barrier-separated segments per
direction, padding gaps and guard bands bit for bit, that a rank's local segment writes only its own slabs, bit identity
with the single-device plan of the same array where both plans name the same kernels, and the refusals.
"""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import layout_util as lu  # noqa: E402


class _env:
    def __init__(self, env):
        self.env = env or {}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _kernels(text):
    """the kernel of every launch of a plan text, in order (grid sizes and barrier marks left out)"""
    return [re.sub(r" grid=\d+", "", re.split(r"  (buffer|temp) ->", line)[0]).split(" n=", 1)[-1] for line in text.strip().split("\n")]


def _pitches(shape, pad):
    nx, ny = shape[0], shape[1]
    h = nx // 2 + 1
    p0 = h + (3 if pad else 0)
    if len(shape) == 2:
        return [p0, shape[1] * p0]
    p1 = ny * p0 + (5 if pad else 0)
    return [p0, p1, shape[2] * p1]


def _play(shape, world, inverse, order, prec=0, normalize=0, pad=False, env=None):
    """plays every rank's launches of one direction; returns (relative l2 error, launches, segments, bit-identical to the
    single-device plan or None where the two plans name different kernels)"""
    rdt, cdt = (np.float32, np.complex64) if prec == 0 else (np.float64, np.complex128)
    nd = len(shape)
    nx, n_last = shape[0], shape[-1]
    h = nx // 2 + 1
    strides = _pitches(shape, pad)
    ext = strides[nd - 1]
    slab = ext // world
    csize = (h,) + tuple(shape[1:])
    rng = np.random.default_rng(int(np.prod(shape)) + world + 7 * prec)
    x = rng.uniform(-1, 1, tuple(reversed(shape)))
    lay = lu.make_layout(csize, 1, strides, cdt)
    real = lu.view_of(lay.flat, shape, 1, [2 * s for s in strides], rdt, lay.guard)
    if inverse == 1:
        lay.scatter(np.fft.rfftn(x)[None].astype(cdt))
    else:
        real[...] = x[None].astype(rdt)
    tflat, tmask = lu.make_flat(ext, cdt)
    start = lay.flat.copy()
    with _env(env):
        kw = dict(perform_r2c=1, buffer_stride=strides, normalize=normalize)
        descs = [emu.make_desc(shape, 1, prec, user_temp_buffer=1, dist_world=world, dist_rank=r, **kw) for r in range(world)]
        rc, npass, sync = emu.exec_plan_pass(descs[0], inverse, lay.data, tflat[lu.GUARD:], -1)
        assert rc == 0, rc
        segs, cur = [], []
        for p in range(npass):
            if sync[p] and cur:
                segs.append(cur)
                cur = []
            cur.append(p)
        segs.append(cur)
        # the segment that stays inside the slabs: forward the first one, inverse the last one
        local = 0 if inverse == -1 else len(segs) - 1
        for si, seg in enumerate(segs):
            for r in (range(world) if order == "up" else range(world - 1, -1, -1)):
                if si == local:
                    b0, t0 = lu.bits(lay.flat), lu.bits(tflat)
                for p in seg:
                    rc, _, _ = emu.exec_plan_pass(descs[r], inverse, lay.data, tflat[lu.GUARD:], p)
                    assert rc == 0, rc
                if si == local:
                    for now, before, what in ((lay.flat, b0, "buffer"), (tflat, t0, "temp")):
                        changed = np.flatnonzero((lu.bits(now) != before).any(axis=1)) - lu.GUARD
                        assert changed.size == 0 or (changed.min() >= r * slab and changed.max() < (r + 1) * slab), \
                            f"rank {r}'s local launches wrote outside its {what} slab: {changed.min()}..{changed.max()}"
        texts = [emu.describe(dd, inverse) for dd in descs]
        assert all(t[0] == 0 for t in texts)
        single = emu.make_desc(shape, 1, prec, **kw)
        rc, stext = emu.describe(single, inverse)
        assert rc == 0
        same = all(_kernels(t[1]) == _kernels(stext) for t in texts)
        ref_flat = start.copy()
        rc, _ = emu.exec_plan(single, inverse, ref_flat[lay.guard:])
        assert rc == 0
    lu.assert_untouched(lay.flat, start, lay.mask, lay, "buffer")
    lu.assert_untouched(tflat, _sentinel_like(tflat), tmask, None, "temp")
    if inverse == 1:
        got = np.array(real[0], dtype=np.float64)
        ref = x * (1.0 if normalize else float(np.prod(shape)))
        identical = np.array_equal(lu.bits(np.ascontiguousarray(real)), lu.bits(np.ascontiguousarray(
            lu.view_of(ref_flat, shape, 1, [2 * s for s in strides], rdt, lay.guard))))
    else:
        got = lay.gather()[0].astype(np.complex128)
        ref = np.fft.rfftn(x)
        identical = np.array_equal(lu.bits(lay.flat)[lay.mask], lu.bits(ref_flat)[lay.mask])
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    return err, npass, len(segs), (identical if same else None)


def _sentinel_like(flat):
    s = np.empty_like(flat)
    lu.fill_sentinel(s)
    return s


SHAPES = [
    # shape, world, env
    ((64, 32), 2, None),
    ((128, 64), 4, None),          # H = 65 columns over 4 ranks: 16 + 16 + 16 + 17
    ((32, 16, 8), 2, None),
    ((64, 32, 16), 4, None),
    ((48, 40, 12), 2, None),
]


@pytest.mark.parametrize("shape,world,env", SHAPES)
@pytest.mark.parametrize("pad", [False, True])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_distributed_r2c_slab_plans(shape, world, env, pad, inverse):
    for order in ("up", "down"):
        err, npass, nseg, same = _play(shape, world, inverse, order, pad=pad, env=env)
        assert npass == len(shape) and nseg == 2, (npass, nseg)
        assert err < 2e-6, err
        assert same, "differs from the single-device plan of the same array, or names other kernels"


@pytest.mark.parametrize("pad", [False, True])
def test_distributed_r2c_long_last_axis_runs_as_strided_four_step(pad):
    for inverse in (-1, 1):
        err, npass, nseg, same = _play((32, 4096), 2, inverse, "up", pad=pad, env={"B200FFT_MAX_SINGLE_PASS": "1024"})
        assert npass == 3 and nseg == 2, (npass, nseg)
        assert err < 2e-6, err
        assert same


@pytest.mark.parametrize("pad", [False, True])
def test_distributed_r2c_composed_x_axis(pad):
    """nx = 40000 has no one-launch R2C kernel: half-length C2C Four-Step on the rank's slab (scratch: its temp slab) + the
    Hermitian launch"""
    rc, text = emu.describe(emu.make_desc((40000, 4), 1, 0, perform_r2c=1, user_temp_buffer=1, dist_world=2, dist_rank=1), -1)
    assert rc == 0 and "hermitian" in text and "four-step" in text, text
    for inverse in (-1, 1):
        for order in ("up", "down"):
            err, npass, nseg, same = _play((40000, 4), 2, inverse, order, pad=pad)
            assert npass == 4 and nseg == 2, (npass, nseg)
            assert err < 2e-6, err
            assert same


@pytest.mark.parametrize("shape", [(64, 32, 16), (128, 64)])
def test_distributed_r2c_double_and_normalize(shape):
    err, _, nseg, same = _play(shape, 2, -1, "down", prec=1, pad=True)
    assert err < 1e-13 and nseg == 2 and same, err
    err, _, nseg, same = _play(shape, 2, 1, "up", prec=1, normalize=1, pad=True)
    assert err < 1e-13 and nseg == 2 and same, err


def _rc(shape, world=2, rank=0, batches=1, prec=0, **kw):
    d = emu.make_desc(shape, batches, prec, perform_r2c=1, dist_world=world, dist_rank=rank, **kw)
    z = np.zeros(1 << 16, np.complex64)
    return emu.exec_plan_pass(d, -1, z, z.copy(), -1)[0]


def test_distributed_r2c_refusals():
    assert _rc((4096,), user_temp_buffer=1) == 3002                     # 1-D: the Nyquist point and k / N-k cross the slabs
    assert _rc((63, 32), user_temp_buffer=1) == 3002                    # odd nx: its scratch does not fit into a slab
    assert _rc((64, 32), batches=2, user_temp_buffer=1) == 3002         # batches are sharded whole, not distributed
    assert _rc((64, 30), world=4, user_temp_buffer=1) == 3002           # 4 ranks cannot split 30 rows
    assert _rc((64, 32), user_temp_buffer=1, is_input_formatted=1) == 3002
    assert _rc((64, 32), user_temp_buffer=1, is_output_formatted=1) == 3002
    assert _rc((64, 32), prec=2, user_temp_buffer=1) == 3002            # half storage
    assert _rc((64, 32), rank=2, user_temp_buffer=1) == 1002
    assert _rc((64, 32)) == 2006                                        # windows must be supplied (temp included)
    assert _rc((64, 32), user_temp_buffer=1, buffer_stride=[32, 32 * 32]) == 3002   # a row pitch below H = 33
