"""Bug hunt on the CPU emulation of the kernels (no GPU)."""
import os, sys, time, json
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'emu')); 
import numpy as np, emu, scipy.fft as sfft
seed, count = int(sys.argv[1]), int(sys.argv[2])
rng = np.random.default_rng(seed)
bad = []; t0 = time.time(); done = 0
def rel(a, b):
    nb = np.linalg.norm(b)
    return float(np.linalg.norm(a - b) / (nb if nb else 1))
SIZES = [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 21, 22, 24, 25, 26, 27, 28, 30, 32, 33, 34, 35, 36, 39, 40, 42, 44, 45, 48, 49, 50, 51, 52, 54, 55, 56, 60, 63, 64, 65, 66, 68, 70, 72, 75, 77, 80, 81, 84, 85, 88, 90, 91, 96, 98, 99, 100, 102, 104, 105, 108, 110, 112, 119, 120, 121, 125, 126, 128, 130, 132, 135, 136, 140, 143, 144, 150, 153, 154, 160, 162, 165, 168, 169, 170, 175, 176, 180, 187, 189, 192, 195, 196, 198, 200, 204, 208, 210, 216, 220, 221, 224, 225, 231, 234, 238, 240, 242, 243, 245, 250, 252, 255, 256, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61, 67, 71, 73, 79, 83, 89, 97, 101, 103, 107, 109, 113, 127, 131, 137, 139, 211, 251]
for it in range(count):
    nd = int(rng.integers(1, 4))
    shape = tuple(int(rng.choice(SIZES)) for _ in range(nd))
    while np.prod(shape) > 60000:
        shape = tuple(max(2, s // 2) for s in shape)
    b = int(rng.integers(1, 4)); prec = int(rng.integers(0, 2)); inv = int(rng.choice([-1, 1])); norm = int(rng.integers(0, 2))
    mode = str(rng.choice(["c2c", "r2c", "dct", "dst"]))
    kind = int(rng.integers(1, 5))
    rdt, cdt = (np.float32, np.complex64) if prec == 0 else (np.float64, np.complex128)
    tol = 3e-6 if prec == 0 else 1e-12
    npshape = (b,) + tuple(reversed(shape)); axes = tuple(range(1, nd + 1))
    tag = (mode, kind if mode in ("dct", "dst") else 0, shape, b, prec, inv, norm)
    try:
        if mode == "c2c":
            x = (rng.uniform(-1, 1, npshape) + 1j * rng.uniform(-1, 1, npshape)).astype(cdt)
            buf = x.copy(); rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec, normalize=norm), inv, buf)
            ref = np.fft.fftn(x.astype(np.complex128), axes=axes) if inv == -1 else np.fft.ifftn(x.astype(np.complex128), axes=axes) * (1 if norm else np.prod(shape))
            if rc or not rel(buf, ref) < tol: bad.append((tag, rc, rel(buf, ref) if not rc else None))
        elif mode == "r2c":
            nx = shape[0]; H = nx // 2 + 1
            x = rng.uniform(-1, 1, npshape).astype(rdt)
            buf = np.zeros(npshape[:-1] + (2 * H,), rdt); buf[..., :nx] = x
            d = emu.make_desc(shape, b, prec, perform_r2c=1, normalize=norm)
            rc, _ = emu.exec_plan(d, -1, buf)
            if rc:
                if rc != 3003: bad.append((tag, rc))
                continue
            e1 = rel(buf.view(cdt), np.fft.rfftn(x.astype(np.float64), axes=axes))
            rc2, _ = emu.exec_plan(d, 1, buf)
            e2 = rel(buf[..., :nx], x.astype(np.float64) * (1 if norm else np.prod(shape)))
            if rc2 or not e1 < tol or not e2 < tol: bad.append((tag, rc2, e1, e2))
        else:
            x = rng.uniform(-1, 1, npshape).astype(rdt)
            buf = x.copy()
            kw = {"perform_dst" if mode == "dst" else "perform_dct": kind}
            rc, _ = emu.exec_plan(emu.make_desc(shape, b, prec, normalize=norm, **kw), inv, buf)
            if rc:
                if rc != 3004: bad.append((tag, rc))
                continue
            t = kind if inv == -1 else {1: 1, 2: 3, 3: 2, 4: 4}[kind]
            f = sfft.dstn if mode == "dst" else sfft.dctn
            ref = f(x.astype(np.float64), type=t, axes=axes)
            if inv == 1 and norm:
                sc = 1.0
                for s in shape:
                    sc *= (2 * (s - 1) if (kind == 1 and mode == "dct") else (2 * (s + 1) if kind == 1 else 2 * s))
                ref = ref / sc
            if not rel(buf, ref) < tol * 2: bad.append((tag, 'err', rel(buf, ref)))
        done += 1
    except Exception as e:
        bad.append((tag, 'exc', repr(e)))
print(json.dumps({"seed": seed, "done": done, "bad": [str(b) for b in bad[:30]], "nbad": len(bad), "sec": round(time.time() - t0, 1)}))
