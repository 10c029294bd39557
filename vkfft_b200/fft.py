"""pyvkfft-style convenience functions on torch CUDA tensors (SURVEY.md section 8f, row 1).

The reference's most common real caller is a Python wrapper that hides the application object behind `fftn(src, dest)`
calls and caches one application per (shape, dtype, flags) -- pyvkfft's `pyvkfft.fft` module (reference README.md:90).
This module gives the same surface over the C ABI:

    from vkfft_b200 import fft as vkfft
    y = vkfft.fftn(x)                 # complex -> complex, all dims, out of place
    vkfft.ifftn(y, y)                 # in place
    h = vkfft.rfftn(r, ndim=2)        # real -> half-Hermitian complex (last axis n//2+1)
    r2 = vkfft.irfftn(h, ndim=2, n_last=r.shape[-1])
    c = vkfft.dctn(r, dct_type=2)     # FFTW REDFT10 convention, idctn / dstn / idstn likewise (out of place: r is not written)
    u = vkfft.convolve_r2r(r, k, ndim=2)   # idctn(dctn(r) * k) in one convolution plan (dst=True: DST)

`ndim` = number of trailing dimensions to transform (the fast axes; leading dimensions are batches), as in pyvkfft.
`norm`: 0 = nothing (the library's own convention: unnormalised inverse), 1 = backward transform scaled by 1/N (numpy's
default), "ortho" = both directions scaled by 1/sqrt(N).  Plans are cached per configuration; tensors must be contiguous.
PyTorch is used for device memory only.

Precision follows the dtype: complex64 / float32 (FP32), complex128 / float64 (FP64), and complex32 / float16 for
fftn / ifftn / rfftn / irfftn (halfPrecision: half storage, FP32 arithmetic).  The cosine / sine transforms take float32
and float64 only; any other dtype (bfloat16, integers, half DCT / DST) raises TypeError before anything is planned.
A half inverse with norm=1 is scaled in FP32 inside the transform (the plan's `normalize`): scaled afterwards, the
unnormalised result would leave half's range at modest sizes.
"""
import math
from typing import Dict, Optional, Tuple

from . import api

_CACHE: Dict[Tuple, api.VkFFTApplication] = {}


def clear_cache():
    for app in _CACHE.values():
        api.deleteVkFFT(app)
    _CACHE.clear()


def _plan(key, **cfg):
    app = _CACHE.get(key)
    if app is None:
        app = api.VkFFTApplication()
        rc = api.initializeVkFFT(app, api.VkFFTConfiguration(**cfg))
        if rc != 0:
            raise RuntimeError("initializeVkFFT: " + api.getVkFFTErrorString(rc))
        _CACHE[key] = app
    return app


def _split(shape, ndim):
    ndim = len(shape) if ndim is None else ndim
    if not 1 <= ndim <= min(len(shape), 3):
        raise ValueError("ndim must be between 1 and min(tensor.ndim, 3)")
    sizes = list(reversed(shape[len(shape) - ndim:]))      # x (fastest) first, as VkFFT counts
    batch = 1
    for s in shape[:len(shape) - ndim]:
        batch *= s
    return ndim, sizes, batch


def _check(t, name):
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous CUDA tensor")


def _stream(torch, cuda_stream):
    return cuda_stream if cuda_stream is not None else torch.cuda.current_stream().cuda_stream


# VkFFTConfiguration precision of each dtype: 0 FP32, 1 FP64, 2 half storage
_COMPLEX_PREC = {"complex64": 0, "complex128": 1, "complex32": 2}
_REAL_PREC = {"float32": 0, "float64": 1, "float16": 2}


def _prec(t, table, what):
    p = table.get(str(t.dtype).replace("torch.", ""))
    if p is None:
        raise TypeError(f"{what}: unsupported dtype {t.dtype} (supported: {', '.join(table)})")
    return p


def _prec_cfg(prec, norm):
    """configuration keys of a precision; half plans apply norm=1 themselves (normalize = 1 on the inverse)"""
    return {"doublePrecision": int(prec == 1), "halfPrecision": int(prec == 2), "normalize": int(prec == 2 and norm == 1)}


def _scale_after(t, n, norm, inverse, prec=0):
    import torch
    if norm == "ortho":
        # complex32 has no multiply: scale its float16 view
        (torch.view_as_real(t) if prec == 2 and t.is_complex() else t).mul_(1.0 / math.sqrt(n))
    elif norm == 1 and inverse:
        if prec != 2:                          # half: already scaled by the plan
            t.mul_(1.0 / n)
    elif norm not in (0, 1, "ortho"):
        raise ValueError("norm must be 0, 1 or 'ortho'")


def _check_norm(norm):
    if norm not in (0, 1, "ortho"):
        raise ValueError("norm must be 0, 1 or 'ortho'")


def _c2c(src, dest, ndim, norm, cuda_stream, inverse):
    import torch
    _check_norm(norm)                      # before any launch
    _check(src, "src")
    if not src.is_complex():
        raise TypeError("complex tensor expected; use rfftn for real input")
    prec = _prec(src, _COMPLEX_PREC, "fftn / ifftn")
    inplace = dest is not None and dest.data_ptr() == src.data_ptr()
    if dest is None:
        dest = torch.empty_like(src)
    _check(dest, "dest")
    if dest.shape != src.shape or dest.dtype != src.dtype:
        raise ValueError("dest must match src")
    nd, sizes, batch = _split(src.shape, ndim)
    dev = src.device.index
    if all(s == 1 for s in sizes):
        # every transformed axis has one point: the plan has no launch (plan_direction_c2c skips such axes), so an
        # out-of-place call would hand back uninitialised memory -- the transform is the identity
        if not inplace:
            with torch.cuda.stream(torch.cuda.ExternalStream(_stream(torch, cuda_stream))):
                dest.copy_(src)
        return dest
    # out of place (API guide :365-376): the forward transform reads inputBuffer, the inverse reads outputBuffer; both
    # leave the result in `buffer`
    fmt = {} if inplace else ({"isOutputFormatted": 1, "makeInversePlanOnly": 1} if inverse else
                              {"isInputFormatted": 1, "makeForwardPlanOnly": 1})
    pc = _prec_cfg(prec, norm)
    app = _plan(("c2c", tuple(sizes), batch, prec, pc["normalize"], dev, inplace, inverse and not inplace), FFTdim=nd, size=sizes,
                numberBatches=batch, device=dev, **pc, **fmt)
    lp = api.VkFFTLaunchParams(buffer=dest, stream=_stream(torch, cuda_stream))
    if not inplace:
        if inverse:
            lp.outputBuffer = src
        else:
            lp.inputBuffer = src
    rc = api.VkFFTAppend(app, 1 if inverse else -1, lp)
    if rc != 0:
        raise RuntimeError("VkFFTAppend: " + api.getVkFFTErrorString(rc))
    n = 1
    for s in sizes:
        n *= s
    _scale_after(dest, n, norm, inverse, prec)
    return dest


def fftn(src, dest=None, ndim=None, norm=1, cuda_stream=None):
    """forward complex transform over the last `ndim` dimensions; dest=src for in place"""
    return _c2c(src, dest, ndim, norm, cuda_stream, False)


def ifftn(src, dest=None, ndim=None, norm=1, cuda_stream=None):
    return _c2c(src, dest, ndim, norm, cuda_stream, True)


def rfftn(src, dest=None, ndim=None, norm=1, cuda_stream=None):
    """real -> complex; the last axis of the result has n//2+1 points (even n only on the fast path, like the reference)"""
    import torch
    _check_norm(norm)
    _check(src, "src")
    if src.is_complex():
        raise TypeError("real tensor expected")
    prec = _prec(src, _REAL_PREC, "rfftn")
    nd, sizes, batch = _split(src.shape, ndim)
    cdt = (torch.complex64, torch.complex128, torch.complex32)[prec]
    oshape = tuple(src.shape[:-1]) + (src.shape[-1] // 2 + 1,)
    if dest is None:
        dest = torch.empty(oshape, dtype=cdt, device=src.device)
    _check(dest, "dest")
    if tuple(dest.shape) != oshape or dest.dtype != cdt:
        raise ValueError(f"dest must be {oshape} {cdt}")
    dev = src.device.index
    pc = _prec_cfg(prec, norm)
    app = _plan(("r2c", tuple(sizes), batch, prec, pc["normalize"], dev), FFTdim=nd, size=sizes, numberBatches=batch, device=dev,
                performR2C=1, isInputFormatted=1, inverseReturnToInputBuffer=1, **pc)
    rc = api.VkFFTAppend(app, -1, api.VkFFTLaunchParams(buffer=dest, inputBuffer=src, stream=_stream(torch, cuda_stream)))
    if rc != 0:
        raise RuntimeError("VkFFTAppend: " + api.getVkFFTErrorString(rc))
    n = 1
    for s in sizes:
        n *= s
    _scale_after(dest, n, norm, False, prec)
    return dest


def irfftn(src, dest=None, ndim=None, norm=1, cuda_stream=None, n_last=None):
    """half-Hermitian complex -> real; n_last = length of the real fast axis (default 2*(src.shape[-1]-1)).
    Like the reference's C2R, the transform may overwrite `src`."""
    import torch
    _check_norm(norm)
    _check(src, "src")
    if not src.is_complex():
        raise TypeError("complex tensor expected")
    prec = _prec(src, _COMPLEX_PREC, "irfftn")
    n_last = 2 * (src.shape[-1] - 1) if n_last is None else n_last
    if n_last // 2 + 1 != src.shape[-1]:
        raise ValueError("n_last does not match the Hermitian axis")
    rshape = tuple(src.shape[:-1]) + (n_last,)
    rdt = (torch.float32, torch.float64, torch.float16)[prec]
    if dest is None:
        dest = torch.empty(rshape, dtype=rdt, device=src.device)
    _check(dest, "dest")
    if tuple(dest.shape) != rshape or dest.dtype != rdt:
        raise ValueError(f"dest must be {rshape} {rdt}")
    nd, sizes, batch = _split(rshape, ndim)
    dev = src.device.index
    pc = _prec_cfg(prec, norm)
    app = _plan(("r2c", tuple(sizes), batch, prec, pc["normalize"], dev), FFTdim=nd, size=sizes, numberBatches=batch, device=dev,
                performR2C=1, isInputFormatted=1, inverseReturnToInputBuffer=1, **pc)
    rc = api.VkFFTAppend(app, 1, api.VkFFTLaunchParams(buffer=src, inputBuffer=dest, stream=_stream(torch, cuda_stream)))
    if rc != 0:
        raise RuntimeError("VkFFTAppend: " + api.getVkFFTErrorString(rc))
    n = 1
    for s in sizes:
        n *= s
    _scale_after(dest, n, norm, True, prec)
    return dest


def _r2r(src, dest, ndim, norm, cuda_stream, inverse, kind, dst):
    import torch
    _check_norm(norm)
    _check(src, "src")
    if src.is_complex():
        raise TypeError("real tensor expected")
    prec = _prec(src, {k: v for k, v in _REAL_PREC.items() if v != 2}, "dctn / dstn")    # no half cosine / sine transforms
    inplace = dest is not None and dest.data_ptr() == src.data_ptr()
    if dest is None:
        dest = torch.empty_like(src)
    _check(dest, "dest")
    if dest.shape != src.shape or dest.dtype != src.dtype:
        raise ValueError("dest must match src")
    nd, sizes, batch = _split(src.shape, ndim)
    dev = src.device.index
    if all(s == 1 for s in sizes):
        # no axis has a launch: the transform is the identity (as in _c2c)
        if not inplace:
            with torch.cuda.stream(torch.cuda.ExternalStream(_stream(torch, cuda_stream))):
                dest.copy_(src)
        return dest
    # out of place as in _c2c: the forward transform reads inputBuffer, the inverse reads outputBuffer, the result is in
    # `buffer`; the source is not written
    fmt = {} if inplace else ({"isOutputFormatted": 1, "makeInversePlanOnly": 1} if inverse else
                              {"isInputFormatted": 1, "makeForwardPlanOnly": 1})
    name = "performDST" if dst else "performDCT"
    app = _plan((name, kind, tuple(sizes), batch, prec, dev, inplace, inverse and not inplace), FFTdim=nd, size=sizes,
                numberBatches=batch, device=dev, doublePrecision=int(prec == 1), **{name: kind}, **fmt)
    lp = api.VkFFTLaunchParams(buffer=dest, stream=_stream(torch, cuda_stream))
    if not inplace:
        if inverse:
            lp.outputBuffer = src
        else:
            lp.inputBuffer = src
    rc = api.VkFFTAppend(app, 1 if inverse else -1, lp)
    if rc != 0:
        raise RuntimeError("VkFFTAppend: " + api.getVkFFTErrorString(rc))
    n = 1
    for s in sizes:   # logical size of the underlying periodic sequence (FFTW manual, "1d Real-even DFTs")
        n *= (2 * (s - 1) if (kind == 1 and not dst) else (2 * (s + 1) if kind == 1 else 2 * s))
    _scale_after(dest, n, norm, inverse)
    return dest


def dctn(src, dest=None, ndim=None, norm=1, dct_type=2, cuda_stream=None):
    return _r2r(src, dest, ndim, norm, cuda_stream, False, dct_type, False)


def idctn(src, dest=None, ndim=None, norm=1, dct_type=2, cuda_stream=None):
    """inverse of dctn(dct_type): runs DCT-III for type 2 and vice versa (types 1 and 4 are their own inverses)"""
    return _r2r(src, dest, ndim, norm, cuda_stream, True, dct_type, False)


def dstn(src, dest=None, ndim=None, norm=1, dst_type=2, cuda_stream=None):
    return _r2r(src, dest, ndim, norm, cuda_stream, False, dst_type, True)


def idstn(src, dest=None, ndim=None, norm=1, dst_type=2, cuda_stream=None):
    return _r2r(src, dest, ndim, norm, cuda_stream, True, dst_type, True)


def convolve_r2r(src, kernel, dest=None, ndim=None, kind=2, dst=False, norm=1, cuda_stream=None):
    """forward DCT (DST with dst=True) of type `kind` over the last `ndim` dimensions, product with the real multiplier
    array `kernel` (the shape of those dimensions, applied to every leading batch), inverse transform -- one plan, one
    VkFFTAppend.  The spectral step of a Poisson / Helmholtz solver with Neumann (DCT) or Dirichlet (DST) walls.
    norm=1: the inverse carries the plan's normalisation, so a kernel of ones returns src; norm=0: unnormalised.
    Out of place unless dest is src; src is not written then."""
    import torch
    if norm not in (0, 1):
        raise ValueError("norm must be 0 or 1")
    if kind not in (1, 2, 3, 4):
        raise ValueError("kind must be 1, 2, 3 or 4")
    _check(src, "src")
    if src.is_complex():
        raise TypeError("real tensor expected")
    prec = _prec(src, {k: v for k, v in _REAL_PREC.items() if v != 2}, "convolve_r2r")
    nd, sizes, batch = _split(src.shape, ndim)
    _check(kernel, "kernel")
    if kernel.dtype != src.dtype or tuple(kernel.shape) != tuple(src.shape[len(src.shape) - nd:]):
        raise ValueError(f"kernel must be {tuple(src.shape[len(src.shape) - nd:])} {src.dtype}")
    inplace = dest is not None and dest.data_ptr() == src.data_ptr()
    if dest is None:
        dest = torch.empty_like(src)
    _check(dest, "dest")
    if dest.shape != src.shape or dest.dtype != src.dtype:
        raise ValueError("dest must match src")
    if kernel.device != src.device or dest.device != src.device:
        raise ValueError("src, kernel and dest must be on the same device")
    dev = src.device.index
    name = "performDST" if dst else "performDCT"
    fmt = {} if inplace else {"isInputFormatted": 1}
    app = _plan(("conv_r2r", name, kind, tuple(sizes), batch, prec, norm, dev, inplace), FFTdim=nd, size=sizes,
                numberBatches=batch, device=dev, doublePrecision=int(prec == 1), normalize=norm, performConvolution=1,
                **{name: kind}, **fmt)
    lp = api.VkFFTLaunchParams(buffer=dest, kernel=kernel, stream=_stream(torch, cuda_stream))
    if not inplace:
        lp.inputBuffer = src
    rc = api.VkFFTAppend(app, -1, lp)
    if rc != 0:
        raise RuntimeError("VkFFTAppend: " + api.getVkFFTErrorString(rc))
    return dest
