"""CPU: thinned versions of the exhaustive emulation sweeps of tools/emu_sweep_*.py (the reference's precision samples
11-18 walk size ranges the same way: sample_11/14/15/16_precision_VkFFT_*.cpp)."""
import os
import sys

import numpy as np
import pytest
import scipy.fft as sfft

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.mark.parametrize("part", range(4))
def test_every_length_up_to_256_and_a_comb_above(part):
    rng = np.random.default_rng(part)
    sizes = list(range(2, 257)) + list(range(257, 4300, 29))
    for n in sizes[part::4]:
        x = (rng.uniform(-1, 1, (2, n)) + 1j * rng.uniform(-1, 1, (2, n))).astype(np.complex64)
        inv = -1 if n % 3 else 1
        buf = x.copy()
        rc, _ = emu.exec_plan(emu.make_desc((n,), 2, 0), inv, buf)
        assert rc == 0, (n, rc)
        ref = np.fft.fft(x.astype(np.complex128), axis=-1) if inv == -1 else np.fft.ifft(x.astype(np.complex128), axis=-1) * n
        assert _rel(buf, ref) < 2e-6, (n, inv)


@pytest.mark.parametrize("mode", ["r2c", "dct", "dst"])
def test_real_transforms_every_length_up_to_130(mode):
    rng = np.random.default_rng(7)
    for n in range(2, 131):
        x = rng.uniform(-1, 1, (3, n)).astype(np.float32)
        if mode == "r2c":
            H = n // 2 + 1
            buf = np.zeros((3, 2 * H), np.float32)
            buf[:, :n] = x
            d = emu.make_desc((n,), 3, 0, perform_r2c=1)
            assert emu.exec_plan(d, -1, buf)[0] == 0, n
            assert _rel(buf.view(np.complex64), np.fft.rfft(x.astype(np.float64), axis=-1)) < 2e-6, n
            assert emu.exec_plan(d, 1, buf)[0] == 0, n
            assert _rel(buf[:, :n], x.astype(np.float64) * n) < 2e-6, n
        else:
            kind = 1 + n % 4
            f = sfft.dst if mode == "dst" else sfft.dct
            buf = x.copy()
            rc, _ = emu.exec_plan(emu.make_desc((n,), 3, 0, **{"perform_" + mode: kind}), -1, buf)
            if rc == 3004:      # transform length with a prime factor above 127 (DCT-I: 2n-2, DST-I: 2n+2)
                continue
            assert rc == 0, (n, kind, rc)
            assert _rel(buf, f(x.astype(np.float64), type=kind, axis=-1)) < 3e-6, (n, kind)
