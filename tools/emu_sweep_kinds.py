"""Bug hunt on the CPU emulation of the kernels (no GPU)."""
import os, sys, time, json
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'emu')); 
import numpy as np, emu, scipy.fft as sfft
mode, lo, hi, step = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
bad = []; t0 = time.time(); rng = np.random.default_rng(2)
def rel(a, b): return float(np.linalg.norm(a - b) / np.linalg.norm(b))
for n in range(lo, hi, step):
    try:
        if mode == "c2c64":
            x = (rng.uniform(-1, 1, (2, n)) + 1j * rng.uniform(-1, 1, (2, n)))
            for inv in (-1, 1):
                buf = x.copy(); rc, _ = emu.exec_plan(emu.make_desc((n,), 2, 1), inv, buf)
                ref = np.fft.fft(x, axis=-1) if inv == -1 else np.fft.ifft(x, axis=-1) * n
                if rc or not rel(buf, ref) < 1e-12: bad.append((n, inv, rc, rel(buf, ref) if not rc else None))
        elif mode == "r2c":
            x = rng.uniform(-1, 1, (3, n)).astype(np.float32); H = n // 2 + 1
            buf = np.zeros((3, 2 * H), np.float32); buf[:, :n] = x
            d = emu.make_desc((n,), 3, 0, perform_r2c=1)
            rc, _ = emu.exec_plan(d, -1, buf)
            if rc: bad.append((n, -1, rc)); continue
            e = rel(buf.view(np.complex64), np.fft.rfft(x.astype(np.float64), axis=-1))
            rc2, _ = emu.exec_plan(d, 1, buf)
            e2 = rel(buf[:, :n], x.astype(np.float64) * n) if not rc2 else None
            if rc2 or not e < 2e-6 or not e2 < 2e-6: bad.append((n, rc2, e, e2))
        elif mode.startswith("dct") or mode.startswith("dst"):
            kind = int(mode[3]); isdst = mode.startswith("dst")
            x = rng.uniform(-1, 1, (3, n)).astype(np.float32)
            for inv in (-1, 1):
                buf = x.copy()
                kw = {"perform_dst" if isdst else "perform_dct": kind}
                rc, _ = emu.exec_plan(emu.make_desc((n,), 3, 0, **kw), inv, buf)
                if rc:
                    bad.append((n, inv, 'rc', rc)); continue
                t = kind if inv == -1 else {1: 1, 2: 3, 3: 2, 4: 4}[kind]
                f = sfft.dst if isdst else sfft.dct
                ref = f(x.astype(np.float64), type=t, axis=-1)
                if not rel(buf, ref) < 3e-6: bad.append((n, inv, 'err', rel(buf, ref)))
        elif mode == "big":
            x = (rng.uniform(-1, 1, (1, n)) + 1j * rng.uniform(-1, 1, (1, n))).astype(np.complex64)
            buf = x.copy(); rc, _ = emu.exec_plan(emu.make_desc((n,), 1, 0), -1, buf)
            ref = np.fft.fft(x.astype(np.complex128), axis=-1)
            if rc or not rel(buf, ref) < 2e-6: bad.append((n, rc, rel(buf, ref) if not rc else None))
    except Exception as e:
        bad.append((n, 'exc', repr(e)))
hard=[b for b in bad if not ("rc" in b and (3003 in b or 3004 in b)) and not (len(b)==3 and b[2] in (3003,3004))]
print(json.dumps({"mode": mode, "range": [lo, hi, step], "hard": hard[:40], "nhard": len(hard), "nbad": len(bad), "sec": round(time.time() - t0, 1)}))
