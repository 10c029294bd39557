"""Helpers for the -m gpu tests: run a plan through the C ABI (ctypes) on torch-owned device memory, and the unmodified
reference's results they compare with.

Those results are stored in tests/golden/reference/outputs.npz, one entry per comparison, keyed by the test's node id and
the comparison's ordinal within the test: a fixed, seeded sample of the reference's output points (`sampled` picks the same
points of this engine's output) and the reference's l2 error against the exact transform over its whole output
(assert_f32_parity keeps only that error, and only where this engine's own error exceeds the tolerance).  They were
recorded on an H100 from the reference's CUDA backend (DTolm/VkFFT 1.3.4, built into oracle/_ref/ by oracle/Makefile):

    B200FFT_RECORD_REFERENCE=/tmp/outputs.npz python -m pytest -m gpu tests    # then copy it to tests/golden/reference/
"""
import atexit
import os
import re
import zlib

import numpy as np

import vkfft_b200 as vk

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "outputs.npz")
RECORD = os.environ.get("B200FFT_RECORD_REFERENCE")
POINTS = 128                     # output points stored per comparison
_calls = {}
_stored = None
_recorded = {}


def torch_mod():
    import torch
    return torch


def run_c2c(x_np, size_xyz, batches=1, inverse=-1, double=False, **cfgkw):
    """x_np: numpy complex array [batch, ..., y, x] (contiguous).  Returns the transformed numpy array."""
    torch = torch_mod()
    t = torch.from_numpy(np.ascontiguousarray(x_np)).cuda()
    cfg = vk.VkFFTConfiguration(FFTdim=len(size_xyz), size=list(size_xyz), numberBatches=batches, device=0,
                                doublePrecision=int(double), **cfgkw)
    app = vk.VkFFTApplication()
    rc = vk.initializeVkFFT(app, cfg)
    assert rc == vk.VKFFT_SUCCESS, vk.getVkFFTErrorString(rc)
    try:
        rc = vk.VkFFTAppend(app, inverse, vk.VkFFTLaunchParams(buffer=t))
        assert rc == vk.VKFFT_SUCCESS, vk.getVkFFTErrorString(rc)
        torch.cuda.synchronize()
        out = t.cpu().numpy()
    finally:
        vk.deleteVkFFT(app)
    return out


def next_key():
    """key of the current test's next comparison with the reference"""
    node = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    _calls[node] = _calls.get(node, 0) + 1
    return re.sub(r"[^A-Za-z0-9_.:\[\]=-]", "_", f"{node}#{_calls[node]}")


def sampled(arr, key):
    """the stored points of comparison `key` taken from an output of the same shape"""
    flat = np.asarray(arr).reshape(-1)
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    return flat[np.sort(rng.choice(flat.size, min(POINTS, flat.size), replace=False))]


def _record(key, theirs, exact, points):
    import vkfft_oracle as orc
    if not _recorded:
        atexit.register(lambda: np.savez_compressed(RECORD, **_recorded))
    _recorded[key + ".out"] = sampled(theirs, key) if points else np.zeros(0, np.float32)
    _recorded[key + ".err"] = np.float64(orc.error_metrics(theirs, exact)["l2_rel"] if exact is not None else np.nan)


def _lookup(key):
    global _stored
    if RECORD:
        store, names = _recorded, _recorded
    else:
        if _stored is None:
            _stored = np.load(GOLDEN)
        store, names = _stored, _stored.files
    assert key + ".err" in names, f"no stored reference result for {key}"
    return store[key + ".out"], float(store[key + ".err"])


def reference_result(theirs_fn, exact=None, points=True):
    """(key, the reference's output at the stored points, the reference's l2 error against `exact`) for the current test's
    next comparison.  theirs_fn runs the reference; it is only called when recording."""
    key = next_key()
    if RECORD:
        _record(key, theirs_fn(), exact, points)
    return (key,) + _lookup(key)


def assert_f32_parity(mine, exact, theirs_fn, tol=1e-6):
    """north_star tolerance for FP32: 1e-6 relative (l2) against the exact result.  Where a transform's own conditioning puts
    BOTH engines beyond that (the composed real transforms: the reference's FP32 error reaches ~1.4e-6, README.md:76-80),
    the criterion of the C2C reference test applies instead: this engine is at least as close to the exact result as the
    unmodified reference's CUDA backend on the same input (|mine - exact| <= 1.05 |reference - exact|), with the reference's
    error as stored in tests/golden/reference/outputs.npz."""
    import vkfft_oracle as orc
    e_m = orc.error_metrics(mine, exact)["l2_rel"]
    key = next_key()
    if e_m < tol:
        return e_m
    if RECORD:
        _record(key, theirs_fn(), exact, points=False)
    _, e_t = _lookup(key)
    assert e_m <= 1.05 * e_t + 1e-8, f"l2_rel {e_m:.3e} vs reference {e_t:.3e} (north-star 1e-6)"
    return e_m


def ref_inplace(arr, size_xyz, batch, inverse, double=False, use_lut=1, **kw):
    """the unmodified reference's CUDA backend (oracle/_ref) on a copy of `arr`: run only when recording"""
    import vkfft_oracle as orc
    assert orc.ref_available(), "recording the reference's results needs oracle/_ref/libvkfft_ref.so"
    torch = torch_mod()
    t = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
    rc = orc.ref_run(orc.ref_desc(size_xyz, batch, double, use_lut=use_lut, **kw), inverse, t.data_ptr())
    assert rc == 0, rc
    return t.cpu().numpy()
