"""Bug hunt on the CPU emulation of the kernels (no GPU)."""
import os, sys, time, json
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'emu'))
import numpy as np, emu
lo, hi, step, prec = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
bad = []
t0 = time.time()
cdt = np.complex64 if prec == 0 else np.complex128
tol = 2e-6 if prec == 0 else 1e-12
rng = np.random.default_rng(1)
for n in range(lo, hi, step):
    x = (rng.uniform(-1, 1, (2, n)) + 1j * rng.uniform(-1, 1, (2, n))).astype(cdt)
    for inv in (-1, 1):
        buf = x.copy()
        rc, npass = emu.exec_plan(emu.make_desc((n,), 2, prec), inv, buf)
        if rc != 0:
            bad.append((n, inv, 'rc', rc)); continue
        ref = np.fft.fft(x.astype(np.complex128), axis=-1) if inv == -1 else np.fft.ifft(x.astype(np.complex128), axis=-1) * n
        err = np.linalg.norm(buf - ref) / np.linalg.norm(ref)
        if not err < tol:
            bad.append((n, inv, 'err', float(err), npass))
print(json.dumps({"range": [lo, hi, step], "prec": prec, "bad": bad, "sec": round(time.time() - t0, 1)}))
