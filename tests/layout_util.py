"""Padded / user-strided buffer layouts for the layout tests (plain numpy, no CUDA).

A layout is one flat allocation `guard + extent + guard` elements long, extent = batch * strides[fft_dim - 1], in which the
logical array [batch, ..., y, x] lives with the caller's pitches (strides[0] = distance between rows, strides[1] between
planes, ..., strides[fft_dim - 1] between batches, in elements -- the meaning of bufferStride).  Everything that is not a
logical element -- both guard bands and the gaps between rows, planes and batches -- holds a NaN with a fixed payload: a
transform that reads it poisons its result, and a transform that stores to it changes a bit pattern that
`assert_untouched` compares exactly.  A stray store therefore lands in memory the test owns and is reported by comparison."""
import numpy as np
from numpy.lib.stride_tricks import as_strided

GUARD = 96                      # elements before and after every buffer
SENT32 = np.uint32(0x7FC0BEEF)            # quiet NaNs with a recognisable payload
SENT64 = np.uint64(0x7FF8DEADBEEFCAFE)
SENT16 = np.uint16(0x7EAD)


def _word(dtype):
    """unsigned integer type of one real component of dtype"""
    dtype = np.dtype(dtype)
    comp = dtype.itemsize // (2 if dtype.kind == "c" else 1)
    return {2: np.uint16, 4: np.uint32, 8: np.uint64}[comp]


def bits(a):
    """bit patterns of a flat array, one row per element (a float comparison would call every NaN sentinel changed)"""
    a = np.ascontiguousarray(a)
    w = _word(a.dtype)
    return a.view(w).reshape(a.size, -1)


def fill_sentinel(flat):
    w = _word(flat.dtype)
    flat.view(w)[...] = {np.uint16: SENT16, np.uint32: SENT32, np.uint64: SENT64}[w]


def packed_strides(size_xyz, pitch0=None):
    s = [size_xyz[0] if pitch0 is None else pitch0]
    for n in size_xyz[1:]:
        s.append(s[-1] * n)
    return s


class Layout:
    """flat: the whole allocation; data: flat[guard:] (what the transform is given); view: the logical array
    [batch, ..., y, x] inside flat; mask: True for the elements of flat that belong to the logical array"""

    def __init__(self, flat, size_xyz, batch, strides, guard):
        self.flat, self.size, self.batch, self.strides, self.guard = flat, tuple(size_xyz), batch, list(strides), guard
        self.view = view_of(flat, size_xyz, batch, strides, flat.dtype, guard)
        m = np.zeros(flat.size, bool)
        view_of(m, size_xyz, batch, strides, bool, guard)[...] = True
        self.mask = m

    @property
    def data(self):
        return self.flat[self.guard:]

    def scatter(self, dense):
        assert dense.shape == self.view.shape, (dense.shape, self.view.shape)
        self.view[...] = dense

    def gather(self):
        return np.array(self.view)

    def where(self, i):
        """flat index -> text: which guard, or (batch, ..., y, x) with the coordinate that lies in a gap"""
        j = int(i) - self.guard
        extent = self.flat.size - 2 * self.guard
        if j < 0:
            return f"front guard, {-j} elements before the buffer"
        if j >= extent:
            return f"rear guard, {j - extent} elements past the end of the buffer"
        nd = len(self.size)
        names = ["batch"] + ["w", "z", "y"][4 - nd:]
        coords, sizes = [], [self.batch] + list(reversed(self.size[1:]))
        for name, pitch, n in zip(names, reversed(self.strides[:nd]), sizes):
            c, j = divmod(j, pitch)
            coords.append(f"{name}={c}" + (" (gap)" if c >= n else ""))
        coords.append(f"x={j}" + (" (gap)" if j >= self.size[0] else ""))
        return ", ".join(coords)


def view_of(flat, size_xyz, batch, strides, dtype, guard):
    """as_strided logical view [batch, ..., y, x] of dtype on the memory of the 1-D array `flat`, starting `guard` elements of
    flat's own type in; strides in elements of dtype"""
    dtype = np.dtype(dtype)
    raw = flat[guard:].view(dtype)
    nd = len(size_xyz)
    assert len(strides) >= nd
    shape = (batch,) + tuple(reversed(size_xyz))
    st = [strides[nd - 1]] + [strides[a - 1] for a in range(nd - 1, 0, -1)] + [1]
    last = sum((n - 1) * s for n, s in zip(shape, st))
    assert last < raw.size - guard * flat.dtype.itemsize // dtype.itemsize, "the logical array does not fit into the extent"
    return as_strided(raw, shape=shape, strides=[s * dtype.itemsize for s in st])


def make_layout(size_xyz, batch, strides, elem_dtype, guard=GUARD, extent=None):
    """-> Layout with every element (guards and gaps included) set to the sentinel"""
    nd = len(size_xyz)
    extent = batch * strides[nd - 1] if extent is None else extent
    flat = np.empty(guard + extent + guard, np.dtype(elem_dtype))
    fill_sentinel(flat)
    return Layout(flat, size_xyz, batch, strides, guard)


def make_flat(n, elem_dtype, guard=GUARD):
    """a guarded allocation without a logical array (scratch): n elements between two guard bands, all sentinel"""
    flat = np.empty(guard + n + guard, np.dtype(elem_dtype))
    fill_sentinel(flat)
    mask = np.zeros(flat.size, bool)
    mask[guard:guard + n] = True
    return flat, mask


def assert_untouched(after, before, mask, layout=None, what="buffer"):
    """every element outside `mask` has the bit pattern it had before the transform"""
    a, b = bits(after), bits(before)
    assert a.shape == b.shape
    changed = (a != b).any(axis=1) & ~mask
    if changed.any():
        i = int(np.flatnonzero(changed)[0])
        where = layout.where(i) if layout is not None else f"flat index {i} of {after.size}"
        raise AssertionError(f"{what}: {int(changed.sum())} elements outside the transform's footprint were overwritten; "
                             f"the first one at {where}, now {after[i]!r}")


def assert_bit_identical(after, before, what="input"):
    assert np.array_equal(bits(after), bits(before)), f"{what} was modified"


def max_line_error(got, ref):
    """largest max|got - ref| / max|ref| over the lines (last axis) of the result: l2 over a batch hides one wrong point"""
    got = np.asarray(got).astype(np.complex128 if np.iscomplexobj(got) else np.float64)
    ref = np.asarray(ref)
    err = np.abs(got - ref).reshape(-1, ref.shape[-1]).max(axis=1)
    scale = np.abs(ref).reshape(-1, ref.shape[-1]).max(axis=1)
    assert np.isfinite(err).all(), "the result holds NaN / Inf: the transform read a gap or a guard"
    return float((err / np.maximum(scale, np.finfo(np.float64).tiny)).max())


def point_bound(n_total, eps, c):
    """per-point bound c * eps * sqrt(log2 N) relative to the largest point of the line"""
    return c * eps * np.sqrt(max(np.log2(max(n_total, 2)), 1.0))
