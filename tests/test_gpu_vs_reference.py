"""GPU (-m gpu): same inputs through the engine and through the UNMODIFIED reference (DTolm/VkFFT 1.3.4, CUDA backend).
North-star tolerance: 1e-6 rel FP32 / 1e-12 rel FP64.  The reference's results are stored in
tests/golden/reference/outputs.npz (see gpu_util): per comparison a fixed, seeded sample of its output points, compared
with the same points of this engine's output, and its l2 error against the exact result over the whole output.
The reference's default FP32 path evaluates twiddles with __sincosf (its own error vs FFTW is up to ~1.4e-6,
README.md:76-80), so the comparison is norm-wise, and also run against the reference with useLUT=1."""
import numpy as np
import pytest

import vkfft_oracle as orc
from gpu_util import ref_inplace, reference_result, run_c2c, sampled

pytestmark = pytest.mark.gpu


def _l2(a, b):
    return orc.error_metrics(a, b)["l2_rel"]


@pytest.mark.parametrize("n", [8, 128, 1024, 4096, 8192, 1 << 15, 1 << 18, 1 << 20, 1 << 23])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_c2c_f32_matches_reference(n, inverse):
    batch = max(1, (1 << 23) // n)
    x = orc.random_input((batch, n), np.complex64, seed=n % 9973)
    mine = run_c2c(x, (n,), batch, inverse)
    key, theirs, _ = reference_result(lambda: ref_inplace(x, (n,), batch, inverse, use_lut=1))
    assert _l2(sampled(mine, key), theirs) < 1e-6
    # reference default (on-chip sincos) carries its own ~1e-6 error for large N; both must sit within 1e-6 of
    # the exact result's neighbourhood: |mine - theirs| <= |mine - exact| + |theirs - exact|
    exact = orc.c2c(x, 1, inverse == 1)
    key, theirs, e_t = reference_result(lambda: ref_inplace(x, (n,), batch, inverse, use_lut=0), exact)
    e_m = _l2(mine, exact)
    assert e_m < 1e-6 and e_m <= e_t * 1.05 + 1e-8
    m_s, x_s = sampled(mine, key), sampled(exact, key)
    assert _l2(m_s, theirs) < _l2(m_s, x_s) + _l2(theirs, x_s) + 1e-9


@pytest.mark.parametrize("size_xyz", [(4096,), (1 << 16,), (256, 256, 256)])
def test_c2c_f64_matches_reference(size_xyz):
    x = orc.random_input((1,) + tuple(reversed(size_xyz)), np.complex128, seed=int(np.prod(size_xyz)) % 9973)
    mine = run_c2c(x, size_xyz, 1, -1, double=True)
    key, theirs, _ = reference_result(lambda: ref_inplace(x, size_xyz, 1, -1, double=True, use_lut=0))
    assert _l2(sampled(mine, key), theirs) < 1e-12


@pytest.mark.parametrize("size_xyz,batch", [((1000,), 8), ((2187,), 3), ((30030,), 2), ((17,), 64), ((509,), 8), ((105, 30), 2)])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_non_pow2_matches_reference(size_xyz, batch, inverse):
    x = orc.random_input((batch,) + tuple(reversed(size_xyz)), np.complex64, seed=sum(size_xyz))
    mine = run_c2c(x, size_xyz, batch, inverse)
    key, theirs, _ = reference_result(lambda: ref_inplace(x, size_xyz, batch, inverse))
    assert _l2(sampled(mine, key), theirs) < 1e-6


@pytest.mark.parametrize("size_xyz,batch", [((64,), 8), ((4096,), 4), ((4096, 4096), 1), ((30, 4), 3)])
def test_r2c_c2r_matches_reference(size_xyz, batch):
    nx, H = size_xyz[0], size_xyz[0] // 2 + 1
    x = orc.random_input((batch,) + tuple(reversed(size_xyz)), np.float32, seed=sum(size_xyz))
    buf = np.zeros(x.shape[:-1] + (2 * H,), np.float32)
    buf[..., :nx] = x

    def theirs_forward():
        return ref_inplace(buf, size_xyz, batch, -1, perform_r2c=1)
    mine = run_c2c(buf, size_xyz, batch, -1, performR2C=1)
    key, theirs, _ = reference_result(lambda: theirs_forward().view(np.complex64))
    assert _l2(sampled(mine.view(np.complex64), key), theirs) < 1e-6
    # the inverse of each engine's own spectrum (the two spectra agree to 1e-6, and C2R is well conditioned)
    mine2 = run_c2c(mine, size_xyz, batch, 1, performR2C=1)
    key, theirs2, _ = reference_result(lambda: ref_inplace(theirs_forward(), size_xyz, batch, 1, perform_r2c=1)[..., :nx])
    assert _l2(sampled(mine2[..., :nx], key), theirs2) < 1e-6


@pytest.mark.parametrize("kind", [1, 2, 3, 4])
@pytest.mark.parametrize("size_xyz,batch", [((64,), 6), ((100,), 4), ((32, 16), 3), ((2048, 256), 1)])
@pytest.mark.parametrize("inverse", [-1, 1])
def test_dct_matches_reference(kind, size_xyz, batch, inverse):
    x = orc.random_input((batch,) + tuple(reversed(size_xyz)), np.float32, seed=kind + sum(size_xyz))
    mine = run_c2c(x, size_xyz, batch, inverse, performDCT=kind)
    exact = orc.dct(x, kind, len(size_xyz), inverse=(inverse == 1))
    key, theirs, e_t = reference_result(lambda: ref_inplace(x, size_xyz, batch, inverse, perform_dct=kind), exact)
    # north-star 1e-6 between the two engines; where the transform's conditioning puts the reference itself further than
    # that from the exact result, this engine must be at least as close to it as the reference is
    m_s = sampled(mine, key)
    d = _l2(m_s, theirs)
    if d >= 1e-6:
        e_m = _l2(mine, exact)
        x_s = sampled(exact, key)
        assert e_m <= 1.05 * e_t + 1e-8 and d < _l2(m_s, x_s) + _l2(theirs, x_s) + 1e-9, (d, e_m, e_t)
