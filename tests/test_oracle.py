"""CPU: pin the oracle.  definition == pocketfft == C restatement of the reference's Stockham/Four-Step
algorithm, known-answer vectors, and the committed golden outputs of the reference's CUDA backend."""
import glob
import os

import numpy as np
import pytest

import vkfft_oracle as orc

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 8, 11, 13, 16, 30, 64, 105, 128])
@pytest.mark.parametrize("inverse", [False, True])
def test_pocketfft_matches_definition(n, inverse):
    x = orc.random_input((3, n), np.complex128, seed=n)
    ref = orc.dft_definition(x, inverse)
    got = orc.c2c(x, 1, inverse)
    assert orc.error_metrics(got, ref)["l2_rel"] < 1e-14


@pytest.mark.parametrize("n", [2, 8, 13, 64, 77, 343, 1000, 4096, 2 * 3 * 5 * 7 * 11 * 13])
@pytest.mark.parametrize("inverse", [False, True])
def test_stockham_restatement_matches_pocketfft(n, inverse):
    x = orc.random_input((2, n), np.complex128, seed=n + 1)
    got = orc.stockham_c2c(x, inverse)
    assert orc.error_metrics(got, orc.c2c(x, 1, inverse))["l2_rel"] < 1e-13


@pytest.mark.parametrize("n1,n2", [(8, 8), (16, 64), (128, 256), (15, 77)])
@pytest.mark.parametrize("inverse", [False, True])
def test_four_step_restatement(n1, n2, inverse):
    x = orc.random_input((2, n1 * n2), np.complex128, seed=n1)
    got = orc.four_step_c2c(x, n1, n2, inverse)
    assert orc.error_metrics(got, orc.c2c(x, 1, inverse))["l2_rel"] < 1e-13


def test_known_answers():
    # impulse -> all ones ; shifted impulse -> pure phase ramp ; constant -> N*delta
    n = 64
    e = np.zeros((1, n), np.complex128); e[0, 0] = 1
    assert np.allclose(orc.c2c(e, 1), 1.0)
    e = np.zeros((1, n), np.complex128); e[0, 3] = 1
    k = np.arange(n)
    assert np.allclose(orc.c2c(e, 1)[0], np.exp(-2j * np.pi * 3 * k / n))
    assert np.allclose(orc.c2c(e, 1, inverse=True)[0], np.exp(+2j * np.pi * 3 * k / n))   # unnormalised inverse
    c = np.ones((1, n), np.complex128)
    y = orc.c2c(c, 1)
    assert np.isclose(y[0, 0], n) and np.allclose(y[0, 1:], 0)
    # inverse(forward(x)) = N x without normalize, x with normalize
    x = orc.random_input((2, n), np.complex128, 5)
    assert np.allclose(orc.c2c(orc.c2c(x, 1), 1, inverse=True), n * x)
    assert np.allclose(orc.c2c(orc.c2c(x, 1), 1, inverse=True, normalize=True), x)


def test_real_transform_definitions():
    n = 16
    x = orc.random_input((2, n), np.float64, 7)
    full = orc.c2c(x.astype(np.complex128), 1)
    assert np.allclose(orc.r2c(x, 1), full[:, : n // 2 + 1])
    assert np.allclose(orc.c2r(orc.r2c(x, 1), 1, n), n * x)
    # DCT-II (REDFT10): X_k = 2 sum x_n cos(pi (n+1/2) k / N)
    nn = np.arange(n)
    X = np.array([[2 * np.sum(row * np.cos(np.pi * (nn + 0.5) * k / n)) for k in range(n)] for row in x])
    assert np.allclose(orc.dct(x, 2, 1), X)
    # DCT-I (REDFT00), DCT-IV (REDFT11)
    X1 = np.array([[row[0] + (-1) ** k * row[-1] + 2 * np.sum(row[1:-1] * np.cos(np.pi * nn[1:-1] * k / (n - 1)))
                    for k in range(n)] for row in x])
    assert np.allclose(orc.dct(x, 1, 1), X1)
    X4 = np.array([[2 * np.sum(row * np.cos(np.pi * (nn + 0.5) * (k + 0.5) / n)) for k in range(n)] for row in x])
    assert np.allclose(orc.dct(x, 4, 1), X4)
    # reference inverse pairs: DCT-III(DCT-II(x)) = 2N x
    assert np.allclose(orc.dct(orc.dct(x, 2, 1), 2, 1, inverse=True), 2 * n * x)


def test_golden_vectors_from_reference_cuda_backend():
    """tests/golden/*.npz were produced by the reference itself (CUDA backend); the oracle must agree
    with them to the reference's own single/double precision accuracy."""
    files = sorted(glob.glob(os.path.join(GOLD, "*.npz")))
    if not files:
        pytest.skip("no golden vectors committed yet (generated on the GPU box by tests/golden/make_golden.py)")
    for f in files:
        z = np.load(f)
        kind = str(z["kind"])
        x, y = z["input"], z["output"]
        ndim = int(z["ndim"])
        inverse = bool(z["inverse"])
        if kind == "c2c":
            ref = orc.c2c(x, ndim, inverse)
        elif kind == "r2c":
            ref = orc.r2c(x, ndim)
        elif kind.startswith("dct"):
            ref = orc.dct(x, int(kind[3]), ndim, inverse)
        else:
            continue
        tol = 2e-6 if y.dtype in (np.complex64, np.float32) else 1e-12
        assert orc.error_metrics(y, ref)["l2_rel"] < tol, f
