"""CPU: distributed 2-D / 3-D DCT / DST slab plans (desc.dist_world > 1, perform_dct / perform_dst) on the kernel-body emulation.

Two guarded host arrays stand for the two peer windows (`buffer` and scratch), both `ext` real elements long.  The real array lies
with row pitch p0 >= nx (and in 3-D plane pitch p1 >= ny*p0), real elements; rank g's slab is the last-dimension indices
[g*n/R, (g+1)*n/R), i.e. the (n/R)*pitch real elements from g*(n/R)*pitch on, in both windows (the scratch counts complex
elements: the same bytes).  Every rank's plan is built and its launches are played in the orders the plan's barriers allow (all
ranks up, all ranks down), as test_emu_dist_r2c.py does for the R2C slab plans.  Checked: the result against the oracle in
float64, two barrier-separated segments per direction, padding gaps and guard bands bit for bit, that a rank's local segment
writes only its own slabs, bit identity with the single-device plan of the same array where both plans name the same kernels,
and the refusals.
"""
import os
import re

import numpy as np
import pytest

import emu
import layout_util as lu
import vkfft_oracle as orc

T32, T64 = 2e-6, 3e-15          # the bounds of the single-GPU DCT / DST tests (test_emu_r2r_formatted.py)
C_POINT = 6.0


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
    """the kernel of every launch of a plan text, in order (grid sizes, item counts and barrier marks left out)"""
    return [re.sub(r" (grid|items)=\d+", "", re.split(r"  (buffer|temp) ->", line)[0]).split(" n=", 1)[-1]
            for line in text.strip().split("\n")]


def _pitches(shape, pad):
    """real-element pitches; the padded ones stay even so that no route is lost to an odd pitch"""
    p0 = shape[0] + (4 if pad else 0)
    if len(shape) == 2:
        return [p0, shape[1] * p0]
    p1 = shape[1] * p0 + (6 if pad else 0)
    return [p0, p1, shape[2] * p1]


def _check(got, ref, prec, n_total):
    e = orc.error_metrics(got, ref)["l2_rel"]
    assert e < (T32 if prec == 0 else T64), e
    eps = np.finfo(np.float32 if prec == 0 else np.float64).eps
    r = lu.max_line_error(got, ref)
    assert r <= lu.point_bound(n_total, eps, C_POINT), r / lu.point_bound(n_total, eps, 1.0)


def _play(mode, kind, shape, world, inverse, order, prec=0, normalize=0, pad=False, env=None):
    """plays every rank's launches of one direction and checks the result; returns (plan text of rank 0, single-device plan
    text, launches, segments, bit-identical to the single-device plan or None where the two plans name different kernels)"""
    dt = np.float32 if prec == 0 else np.float64
    nd = len(shape)
    strides = _pitches(shape, pad)
    ext = strides[nd - 1]
    slab = ext // world
    x = orc.random_input(tuple(reversed(shape)), dt, seed=int(np.prod(shape)) + world + kind + 7 * prec)
    lay = lu.make_layout(shape, 1, strides, dt)
    lay.scatter(x[None])
    tflat, tmask = lu.make_flat(ext + ext % 2, dt)       # the scratch window: complex elements, the data window's bytes
    start = lay.flat.copy()
    kw = {"perform_" + mode: kind, "buffer_stride": strides, "normalize": normalize}
    with _env(env):
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
    sentinel = np.empty_like(tflat)
    lu.fill_sentinel(sentinel)
    lu.assert_untouched(tflat, sentinel, tmask, None, "temp")
    f = orc.dct if mode == "dct" else orc.dst
    _check(lay.gather()[0], f(x, kind, nd, inverse=(inverse == 1), normalize=bool(normalize)), prec, int(np.prod(shape)))
    identical = np.array_equal(lu.bits(lay.flat)[lay.mask], lu.bits(ref_flat)[lay.mask])
    return texts[0][1], stext, npass, len(segs), (identical if same else None)


def _run(mode, kind, shape, world, pad, inverse, **kw):
    """both rank orders; every launch list has two barrier segments and, where it names the single-device plan's kernels,
    its bits"""
    for order in ("up", "down"):
        text, stext, npass, nseg, same = _play(mode, kind, shape, world, inverse, order, pad=pad, **kw)
        assert nseg == 2, (nseg, text)
        assert same is not False, ("differs from the single-device plan that runs the same kernels", text)
    return text, stext


# every type on 2-D and 3-D shapes; 3-D at R = 4 splits the y rows of the cross-slab axis (12 % 4 == 0)
TYPES = [(m, k) for m in ("dct", "dst") for k in (1, 2, 3, 4)]
SHAPES = [((64, 32), 2), ((40, 24), 4), ((32, 16, 8), 2), ((16, 12, 16), 4)]


@pytest.mark.parametrize("shape,world", SHAPES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else f"R{v}")
@pytest.mark.parametrize("mode,kind", TYPES, ids=lambda v: str(v))
@pytest.mark.parametrize("pad", [False, True])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_distributed_r2r_slab_plans(mode, kind, shape, world, pad, inverse):
    _run(mode, kind, shape, world, pad, inverse)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("pad", [False, True])
def test_fused_strided_cross_slab_axis(kind, world, pad):
    """64 columns of 64 points: the complex view of neighbouring column pairs on the fused DCT-II/III strided kernel"""
    for inverse in (-1, 1):
        text, _ = _run("dct", kind, (64, 64), world, pad, inverse)
        assert "DCT_COLS" in text.strip().split("\n")[-1 if inverse == -1 else 0], text


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("pad", [False, True])
def test_long_strided_cross_slab_axis(kind, world, pad):
    """a 4096-point last axis has no well-shaped strided launch here: the single-GPU plan takes the three-launch long strided
    route, and so does every rank, on its share of the columns, with no barrier between the three launches"""
    for inverse in (-1, 1):
        text, stext = _run("dct", kind, (16, 4096), world, pad, inverse)
        for t in (text, stext):
            assert sum("long dct-i" in line for line in t.strip().split("\n")) == 3, t
        marks = ["[barrier before]" in line for line in text.strip().split("\n") if "long dct-i" in line]
        assert marks == [True, False, False], text


@pytest.mark.parametrize("mode,kind", [("dst", 2), ("dct", 4), ("dct", 1)])
@pytest.mark.parametrize("pad", [False, True])
def test_runtime_scheduled_cross_slab_axis(mode, kind, pad):
    for inverse in (-1, 1):
        text, _ = _run(mode, kind, (64, 32), 2, pad, inverse)
        assert "generic" in text.strip().split("\n")[-1 if inverse == -1 else 0], text


@pytest.mark.parametrize("mode,kind,world", [("dct", 2, 2), ("dst", 2, 4), ("dct", 4, 4)])
@pytest.mark.parametrize("pad", [False, True])
def test_ragged_split_of_the_columns(mode, kind, world, pad):
    """82 columns = 41 pairs, which no R divides: ranges of 8 pairs (16 columns), the last rank taking the remainder"""
    for inverse in (-1, 1):
        _run(mode, kind, (82, 64), world, pad, inverse)


@pytest.mark.parametrize("mode,kind,world", [("dct", 2, 2), ("dct", 2, 4), ("dst", 3, 2), ("dct", 4, 2), ("dst", 1, 4)])
@pytest.mark.parametrize("pad", [False, True])
def test_odd_nx_on_the_runtime_scheduled_kernel(mode, kind, world, pad):
    """45 columns: no complex view, the runtime-scheduled kernel pairs real columns and runs the last one unpaired"""
    for inverse in (-1, 1):
        text, _ = _run(mode, kind, (45, 32), world, pad, inverse)
        assert "generic" in text.strip().split("\n")[-1 if inverse == -1 else 0], text


@pytest.mark.parametrize("mode,kind,shape", [("dct", 2, (64, 32)), ("dst", 3, (32, 16, 8)), ("dct", 4, (64, 64)),
                                             ("dct", 3, (16, 4096))])
def test_double_and_normalize(mode, kind, shape):
    for inverse, order in ((-1, "down"), (1, "up")):
        _, _, _, nseg, same = _play(mode, kind, shape, 2, inverse, order, prec=1, normalize=int(inverse == 1), pad=True)
        assert nseg == 2 and same is not False


def _rc(shape, world=2, rank=0, batches=1, prec=0, mode="dct", kind=2, **kw):
    d = emu.make_desc(shape, batches, prec, **{"perform_" + mode: kind}, dist_world=world, dist_rank=rank, **kw)
    return emu.describe(d, -1)[0]


def test_distributed_r2r_refusals():
    assert _rc((64, 32), user_temp_buffer=1) == 0
    assert _rc((4096,), user_temp_buffer=1) == 3002                     # 1-D: the Makhoul permutation crosses the slabs
    assert _rc((64, 32), batches=2, user_temp_buffer=1) == 3002         # batches are sharded whole, not distributed
    assert _rc((64, 30), world=4, user_temp_buffer=1) == 3002           # 4 ranks cannot split 30 rows
    assert _rc((64, 33), kind=1, user_temp_buffer=1) == 3002            # a DCT-I grid of 2^k+1 points on the last axis
    assert _rc((64, 32), prec=2, user_temp_buffer=1) == 3002            # half storage
    assert _rc((4391, 4), user_temp_buffer=1) == 3002                   # composed route on a local axis: scratch > temp slab
    assert _rc((64, 262), user_temp_buffer=1) == 3002                   # composed route across the slabs (2 * 131)
    assert _rc((64, 262), mode="dst", kind=4, user_temp_buffer=1) == 3002
    assert _rc((64, 32), user_temp_buffer=1, is_input_formatted=1) == 3002
    assert _rc((64, 32), user_temp_buffer=1, perform_zeropadding=[1, 0, 0, 0], zeropad_left=[32, 0, 0, 0],
               zeropad_right=[64, 0, 0, 0]) == 3002
    assert _rc((64, 32), user_temp_buffer=1, omit_dimension=[0, 1, 0, 0]) == 3002
    assert _rc((64, 32), user_temp_buffer=1, buffer_stride=[60, 60 * 32]) == 3002   # a row pitch below nx
    assert _rc((64, 32), rank=2, user_temp_buffer=1) == 1002
    assert _rc((64, 32)) == 2006                                        # windows must be supplied (temp included)
