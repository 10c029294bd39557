"""TEST INFRASTRUCTURE (oracle) -- imported only by tests/, __graft_entry__.smoke() and bench.py's CPU baseline.
The product (vkfft_b200/, include/) never imports, links or executes anything in this directory.

CPU restatement, in double precision, of what the reference's hot path computes, with the reference's
conventions (documentation/VkFFT_API_guide.tex:263-352):
  * forward exponent -1, inverse +1 and UNNORMALISED unless normalize=1 (:302-304);
  * WHDCN layout: size[0] is the fastest dimension, numpy arrays here are indexed [batch, ..., z, y, x];
  * R2C keeps x/2+1 complex per row (Hermitian half, :305-329); DCT/DST I-IV follow FFTW's
    REDFT00/10/01/11 and RODFT00/10/01/11 definitions, unnormalised (:330-348).
The reference's own oracle is FFTW in double precision (sample_11_precision_VkFFT_single.cpp:116-132,
sample_16_...dct.cpp:138-198).  FFTW is not installed in this image, so the same mathematical definitions are
evaluated with pocketfft (scipy.fft); `dft_definition` below is the literal O(N^2) sum used to pin pocketfft,
and oracle/stockham_ref.c restates the reference's Stockham/Four-Step algorithm itself.
Pinning: tests/test_oracle.py checks all of these against each other and against tests/golden/*.npz, which
hold outputs of the reference's CUDA backend (generated on a GPU by tests/golden/make_golden.py).
"""
import ctypes
import os

import numpy as np
import scipy.fft as sfft

_HERE = os.path.dirname(os.path.abspath(__file__))


# ----------------------------------------------------------------------------------------------------------------
# definitions
def dft_definition(x, inverse=False):
    """Literal O(N^2) DFT along the last axis in extended precision (API guide :263-304)."""
    x = np.asarray(x)
    n = x.shape[-1]
    sign = 1.0 if inverse else -1.0
    # reduce the angle exactly (integer k*n mod N) before evaluating sin/cos
    kk = (np.outer(np.arange(n), np.arange(n)) % n).astype(np.longdouble)
    ang = sign * 2 * np.longdouble(np.pi) * kk / np.longdouble(n)
    wr, wi = np.cos(ang), np.sin(ang)
    xr, xi = x.real.astype(np.longdouble), x.imag.astype(np.longdouble)
    yr = xr @ wr.T - xi @ wi.T
    yi = xr @ wi.T + xi @ wr.T
    return (yr + 1j * yi).astype(np.complex128)


def c2c(x, ndim, inverse=False, normalize=False, workers=None):
    """C2C over the last `ndim` axes of x (numpy order [..., z, y, x]); complex128 result."""
    x = np.asarray(x, dtype=np.complex128)
    axes = tuple(range(x.ndim - ndim, x.ndim))
    if inverse:
        y = sfft.ifftn(x, axes=axes, norm="forward", workers=workers)  # norm="forward": unscaled inverse
        if normalize:
            y = y / np.prod([x.shape[a] for a in axes])
        return y
    return sfft.fftn(x, axes=axes, workers=workers)


def r2c(x, ndim, workers=None):
    """Forward R2C: real [..., y, x] -> complex [..., y, x//2+1] (API guide :305-329)."""
    x = np.asarray(x, dtype=np.float64)
    axes = tuple(range(x.ndim - ndim, x.ndim))
    return sfft.rfftn(x, axes=axes, workers=workers)


def c2r(y, ndim, nx, normalize=False, workers=None):
    """Inverse C2R of the Hermitian half-spectrum y [..., y, nx//2+1] -> real [..., y, nx], unnormalised."""
    y = np.asarray(y, dtype=np.complex128)
    axes = tuple(range(y.ndim - ndim, y.ndim))
    shape = [y.shape[a] for a in axes]
    shape[-1] = nx
    x = sfft.irfftn(y, s=shape, axes=axes, norm="forward", workers=workers)
    if normalize:
        x = x / np.prod(shape)
    return x


def dct(x, kind, ndim, inverse=False, normalize=False, workers=None):
    """DCT-I..IV over the last ndim axes == FFTW REDFT00/10/01/11, unnormalised (API guide :330-339).
    The reference's "inverse" DCT-II is DCT-III and vice versa (I and IV are their own inverses)."""
    x = np.asarray(x, dtype=np.float64)
    axes = tuple(range(x.ndim - ndim, x.ndim))
    t = kind
    if inverse and kind in (2, 3):
        t = 5 - kind
    y = sfft.dctn(x, type=t, axes=axes, norm=None, workers=workers)
    if inverse and normalize:
        for a in axes:
            n = x.shape[a]
            y = y / (2 * (n - 1) if kind == 1 else 2 * n)
    return y


def dst(x, kind, ndim, inverse=False, normalize=False, workers=None):
    """DST-I..IV == FFTW RODFT00/10/01/11 (API guide :340-348)."""
    x = np.asarray(x, dtype=np.float64)
    axes = tuple(range(x.ndim - ndim, x.ndim))
    t = kind
    if inverse and kind in (2, 3):
        t = 5 - kind
    y = sfft.dstn(x, type=t, axes=axes, norm=None, workers=workers)
    if inverse and normalize:
        for a in axes:
            n = x.shape[a]
            y = y / (2 * (n + 1) if kind == 1 else 2 * n)
    return y


# ----------------------------------------------------------------------------------------------------------------
# the reference's error report (sample_11_precision_VkFFT_single.cpp:289-331) plus a norm-wise figure
def error_metrics(got, ref):
    got = np.asarray(got).astype(np.complex128).ravel()
    ref = np.asarray(ref).astype(np.complex128).ravel()
    diff = np.abs(got - ref)
    mag = np.abs(ref)
    nz = mag > 0
    rel = np.zeros_like(diff)
    rel[nz] = diff[nz] / mag[nz]
    return {
        "avg_difference": float(diff.mean()), "max_difference": float(diff.max()),
        "avg_eps": float(rel.mean()), "max_eps": float(rel.max()),
        "l2_rel": float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-300)),
    }


def random_input(shape, dtype, seed):
    """uniform[-1,1) re/im like the reference's samples (sample_11...cpp:105-114), but seeded."""
    rng = np.random.default_rng(seed)
    if np.issubdtype(np.dtype(dtype), np.complexfloating):
        real_dt = np.float32 if np.dtype(dtype) == np.complex64 else np.float64
        return (rng.uniform(-1, 1, shape).astype(real_dt) + 1j * rng.uniform(-1, 1, shape).astype(real_dt)).astype(dtype)
    return rng.uniform(-1, 1, shape).astype(dtype)


# ----------------------------------------------------------------------------------------------------------------
# C restatement of the reference's Stockham / Four-Step algorithm (oracle/stockham_ref.c)
_stock = None


def _stockham_lib():
    global _stock
    if _stock is None:
        so = os.path.join(_HERE, "_build", "liboracle_stockham.so")
        src = os.path.join(_HERE, "stockham_ref.c")
        if not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
            import subprocess
            subprocess.check_call(["make", "-C", _HERE, "_build/liboracle_stockham.so"], stdout=subprocess.DEVNULL)
        _stock = ctypes.CDLL(so)
    return _stock


def stockham_c2c(x, inverse=False):
    """batched 1-D C2C of x [batch, n] through the C restatement (n must be 13-smooth)."""
    a = np.ascontiguousarray(np.asarray(x, dtype=np.complex128)).copy()
    b, n = a.shape
    rc = _stockham_lib().oracle_stockham_c2c(a.ctypes.data_as(ctypes.c_void_p), ctypes.c_long(n), ctypes.c_long(b),
                                             int(bool(inverse)))
    if rc != 0:
        raise ValueError("length is not 13-smooth")
    return a


def four_step_c2c(x, n1, n2, inverse=False):
    a = np.ascontiguousarray(np.asarray(x, dtype=np.complex128)).copy()
    b, n = a.shape
    assert n == n1 * n2
    rc = _stockham_lib().oracle_four_step_c2c(a.ctypes.data_as(ctypes.c_void_p), ctypes.c_long(n1), ctypes.c_long(n2),
                                              ctypes.c_long(b), int(bool(inverse)))
    if rc != 0:
        raise ValueError("factor is not 13-smooth")
    return a


# ----------------------------------------------------------------------------------------------------------------
# the reference itself (CUDA backend), when oracle/_ref/libvkfft_ref.so was built and a GPU is present
REF_LIB_PATH = os.path.join(_HERE, "_ref", "libvkfft_ref.so")


class RefDesc(ctypes.Structure):
    """same layout as b200fft_desc (include/b200fft.h) -- the wrapper reuses that plain-C struct"""
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("fft_dim", ctypes.c_uint32),
        ("size", ctypes.c_uint64 * 4), ("number_batches", ctypes.c_uint64), ("coordinate_features", ctypes.c_uint64),
        ("precision", ctypes.c_uint32), ("perform_r2c", ctypes.c_uint32), ("perform_dct", ctypes.c_uint32),
        ("perform_dst", ctypes.c_uint32), ("normalize", ctypes.c_uint32), ("disable_reorder_four_step", ctypes.c_uint32),
        ("make_forward_plan_only", ctypes.c_uint32), ("make_inverse_plan_only", ctypes.c_uint32),
        ("is_input_formatted", ctypes.c_uint32), ("is_output_formatted", ctypes.c_uint32),
        ("inverse_return_to_input", ctypes.c_uint32), ("user_temp_buffer", ctypes.c_uint32),
        ("buffer_stride", ctypes.c_uint64 * 4), ("input_stride", ctypes.c_uint64 * 4), ("output_stride", ctypes.c_uint64 * 4),
        ("omit_dimension", ctypes.c_uint32 * 4), ("buffer_size", ctypes.c_uint64), ("temp_buffer_size", ctypes.c_uint64),
        ("device", ctypes.c_int32), ("reserved0", ctypes.c_uint32), ("stream", ctypes.c_void_p),
        ("reserved", ctypes.c_uint64 * 8),
    ]


def ref_available():
    return os.path.exists(REF_LIB_PATH)


_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        L = ctypes.CDLL(REF_LIB_PATH)
        vp = ctypes.c_void_p
        L.vkref_open.argtypes = [ctypes.POINTER(RefDesc), ctypes.POINTER(vp)]
        L.vkref_append.argtypes = [vp, ctypes.c_int, vp, vp, vp]
        L.vkref_close.argtypes = [vp]
        L.vkref_close.restype = None
        L.vkref_run.argtypes = [ctypes.POINTER(RefDesc), ctypes.c_int, vp, vp, vp]
        L.vkref_axis0_uploads.argtypes = [vp]
        L.vkref_bench_pairs.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double),
                                        ctypes.POINTER(ctypes.c_double)]
        _ref = L
    return _ref


def ref_desc(size_xyz, batches=1, double=False, device=0, use_lut=0, **kw):
    d = RefDesc()
    d.struct_size = ctypes.sizeof(RefDesc)
    d.fft_dim = len(size_xyz)
    for i, s in enumerate(size_xyz):
        d.size[i] = int(s)
    d.number_batches = batches
    d.precision = 1 if double else 0
    d.device = device
    d.reserved[0] = use_lut
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def ref_run(desc, inverse, buffer_ptr, input_ptr=None, output_ptr=None):
    """Run the reference's CUDA backend once on device pointers (synchronous). Returns VkFFTResult."""
    return ref_lib().vkref_run(ctypes.byref(desc), int(inverse), buffer_ptr, input_ptr, output_ptr)
