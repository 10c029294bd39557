#!/usr/bin/env python3
"""Generates tests/golden/*.npz ON A GPU BOX by running the UNMODIFIED reference (DTolm/VkFFT, CUDA backend,
built by oracle/Makefile into oracle/_ref/libvkfft_ref.so) on seeded inputs.  The reference ships no golden
vectors of its own (SURVEY.md section 4), so these files are what pins the CPU oracle to the reference:
tests/test_oracle.py::test_golden_vectors_from_reference_cuda_backend compares the oracle with them.

    python tests/golden/make_golden.py /tmp/golden      # on a GPU machine with oracle/_ref built; then copy the .npz files here
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import torch  # noqa: E402
import vkfft_oracle as orc  # noqa: E402

CASES = [
    # (kind, size_xyz, batch, double, inverse, use_lut)
    ("c2c", (8,), 3, False, False, 1), ("c2c", (64,), 2, False, True, 1), ("c2c", (1000,), 2, False, False, 1),
    ("c2c", (4096,), 2, False, False, 1), ("c2c", (4096,), 2, False, False, 0), ("c2c", (4096,), 1, True, False, 0),
    ("c2c", (32768,), 1, False, False, 1), ("c2c", (65536,), 1, True, True, 0), ("c2c", (17,), 4, False, False, 1),
    ("c2c", (509,), 2, False, False, 1), ("c2c", (2187,), 1, False, False, 1), ("c2c", (30030,), 1, False, False, 1),
    ("c2c", (64, 32), 2, False, False, 1), ("c2c", (32, 16, 8), 1, True, False, 0), ("c2c", (48, 20), 1, False, True, 1),
    ("r2c", (64,), 4, False, False, 1), ("r2c", (64, 32), 2, False, False, 1), ("r2c", (4096,), 2, False, False, 1),
    ("dct1", (33,), 2, False, False, 1), ("dct2", (64,), 2, False, False, 1), ("dct3", (64,), 2, False, False, 1),
    ("dct4", (64,), 2, False, False, 1), ("dct2", (32, 16), 2, False, False, 1), ("dct2", (100,), 2, True, False, 0),
]


def main(outdir):
    os.makedirs(outdir, exist_ok=True)
    assert orc.ref_available(), "build oracle/_ref first (make -C oracle ref)"
    for i, (kind, size, batch, dbl, inverse, lut) in enumerate(CASES):
        shape = (batch,) + tuple(reversed(size))
        cdt = np.complex128 if dbl else np.complex64
        rdt = np.float64 if dbl else np.float32
        kw = {}
        if kind == "c2c":
            x = orc.random_input(shape, cdt, seed=100 + i)
            dev = torch.from_numpy(x.copy()).cuda()
        elif kind == "r2c":
            # in-place padded layout: rows of (nx/2+1) complex == nx+2 reals (vkFFT_InitializeApp.h:1000-1005)
            x = orc.random_input(shape, rdt, seed=100 + i)
            nx = size[0]
            pad = np.zeros(shape[:-1] + (nx + 2,), rdt)
            pad[..., :nx] = x
            dev = torch.from_numpy(pad).cuda()
            kw["perform_r2c"] = 1
        else:
            x = orc.random_input(shape, rdt, seed=100 + i)
            dev = torch.from_numpy(x.copy()).cuda()
            kw["perform_dct"] = int(kind[3])
        d = orc.ref_desc(size, batch, dbl, use_lut=lut, **kw)
        rc = orc.ref_run(d, 1 if inverse else -1, dev.data_ptr())
        if rc != 0:
            print("case", i, kind, size, "reference returned", rc)
            continue
        out = dev.cpu().numpy()
        if kind == "r2c":
            out = out.view(cdt)                      # [..., nx/2+1] complex
        name = f"{i:02d}_{kind}_{'x'.join(map(str, size))}_b{batch}_{'f64' if dbl else 'f32'}_{'inv' if inverse else 'fwd'}_lut{lut}.npz"
        np.savez_compressed(os.path.join(outdir, name), kind=kind, input=x, output=out, ndim=len(size), inverse=inverse,
                            size=np.array(size), use_lut=lut)
        print("wrote", name)


if __name__ == "__main__":
    main(sys.argv[1])
