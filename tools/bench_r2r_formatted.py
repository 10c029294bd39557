"""Out-of-place DCT-II: what running the cosine transform out of place saves, and what the kernel change costs in place.

  1. torch front-end: dctn(x) as it ran before out-of-place plans existed (clone of x, then the in-place plan on the clone)
     against dctn(x) now (one out-of-place plan: inputBuffer = x, buffer = the result);
  2. C ABI: the in-place plan against the out-of-place plan (isInputFormatted) of the same shape -- the same launches;
  3. --parent-lib PATH: the in-place plans of another build of libb200fft.so (e.g. the previous commit's) against this one.

Variants alternate, each timed over windows of at least --window seconds with CUDA events; the median per call is printed in
ms with the card's name and power limit.  One JSON line per comparison.

    python tools/bench_r2r_formatted.py [--parent-lib build_parent/libb200fft.so] [--rounds 5] [--window 0.5]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [("4096x4096 x4", (4096, 4096), 4), ("4096 x4096 (1-D batched)", (4096,), 4096), ("8192x8192", (8192, 8192), 1),
          ("720x480", (720, 480), 1)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().split("\n")[0]
        return q
    except Exception as e:                      # noqa: BLE001 -- the figures are printed either way, with the reason
        return f"unknown ({e})"


def timed(torch, fn, window):
    """ms per call over a window of at least `window` seconds"""
    fn()
    torch.cuda.synchronize()
    reps = 1
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= window * 1e3:
            return ms / reps
        reps = max(reps * 2, int(reps * window * 1e3 / max(ms, 1e-3)) + 1)


def compare(torch, variants, rounds, window):
    res = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            res[k].append(timed(torch, fn, window))
    return {k: round(statistics.median(v), 4) for k, v in res.items()}


class CPlan:
    """an FP32 DCT-II plan straight through the C ABI of one libb200fft.so"""

    def __init__(self, L, shape, batch, stream, out_of_place):
        from vkfft_b200 import _lib
        self.L, self._lib = L, _lib
        d = _lib.b200fft_desc()
        d.struct_size = ctypes.sizeof(d)
        d.fft_dim = len(shape)
        for i, s in enumerate(shape):
            d.size[i] = s
        d.number_batches = batch
        d.perform_dct = 2
        d.make_forward_plan_only = 1
        d.is_input_formatted = int(out_of_place)
        self.p = ctypes.c_void_p()
        L.b200fft_plan_create.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.b200fft_exec.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.b200fft_plan_destroy.argtypes = [ctypes.c_void_p]
        rc = L.b200fft_plan_create(ctypes.byref(d), ctypes.byref(self.p))
        if rc != 0:
            raise RuntimeError(f"b200fft_plan_create: {rc}")
        self.stream = stream

    def run(self, buf, src=None):
        b = self._lib.b200fft_buffers()
        b.buffer = buf.data_ptr()
        if src is not None:
            b.input_buffer = src.data_ptr()
        b.stream = self.stream
        rc = self.L.b200fft_exec(self.p, -1, ctypes.byref(b))
        if rc != 0:
            raise RuntimeError(f"b200fft_exec: {rc}")

    def close(self):
        self.L.b200fft_plan_destroy(self.p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    import torch
    from vkfft_b200 import _lib
    from vkfft_b200 import fft as vkfft
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    gpu = card()
    stream = torch.cuda.current_stream().cuda_stream
    L = _lib.load()
    P = ctypes.CDLL(os.path.abspath(a.parent_lib)) if a.parent_lib else None
    for name, shape, batch in SHAPES:
        x = torch.rand((batch,) + tuple(reversed(shape)), device="cuda", dtype=torch.float32)
        n_bytes = x.numel() * 4
        out = {"shape": name, "gpu": gpu, "bytes_per_array": n_bytes}
        if name != "720x480":
            def before():
                y = x.clone()
                return vkfft.dctn(y, dest=y, ndim=len(shape))
            out["torch_dctn_ms"] = compare(torch, {"clone_then_in_place": before,
                                                   "out_of_place": lambda: vkfft.dctn(x, ndim=len(shape))}, a.rounds, a.window)
            # the two results agree bit for bit
            assert torch.equal(before().view(torch.int32), vkfft.dctn(x, ndim=len(shape)).view(torch.int32))
            buf = torch.empty_like(x)
            ip, oop = CPlan(L, shape, batch, stream, False), CPlan(L, shape, batch, stream, True)
            out["c_api_ms"] = compare(torch, {"in_place": lambda: ip.run(buf), "out_of_place": lambda: oop.run(buf, x)}, a.rounds, a.window)
            ip.close(); oop.close()
            del buf
        if P is not None and name in ("8192x8192", "720x480"):
            buf = x.clone()
            mine, theirs = CPlan(L, shape, batch, stream, False), CPlan(P, shape, batch, stream, False)
            out["in_place_library_ms"] = compare(torch, {"parent": lambda: theirs.run(buf), "this": lambda: mine.run(buf)}, a.rounds, a.window)
            mine.close(); theirs.close()
        print(json.dumps(out), flush=True)
        del x
        vkfft.clear_cache()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
