"""DCT / DST convolution: the fused plan, the chain plan and the same work as three calls.

  plan:      fft.convolve_r2r(x, k): one convolution plan as the planner picks it -- the last axis's DCT-II, kernel product and
             DCT-III in one launch where a fused kernel exists (2 nd - 1 launches), otherwise the chain;
  chain:     the same plan made with B200FFT_NO_FUSED_CONV=1: forward R2R passes, one real product launch, inverse R2R passes;
  separate:  fft.dctn(x) -> mul_(k) -> fft.idctn (dstn / idstn for DST).

FP32, DCT-II and DST-II, norm=1.  The variants alternate, each timed over windows of at least --window seconds with CUDA events;
the median per call is printed in ms with the card's name and power limit, read in the same run, and the share of 3.35 TB/s
(H100 SXM HBM3) that each variant's algorithmic bytes reach: one FP32 read and write per point for every axis pass in each
direction plus three for the product (x, k, result), i.e. (16 nd + 12) bytes per point for the chain and (16 nd - 4) for the
fused plan.  One JSON line per shape and type.

    python tools/bench_r2r_conv.py [--rounds 5] [--window 0.5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BPS = 3.35e12
SHAPES = [("4096 x65536 (1-D batched)", (4096,), 1 << 16), ("2048x2048 x16", (2048, 2048), 16), ("1024x1024 x64", (1024, 1024), 64),
          ("256^3 x4", (256, 256, 256), 4), ("512x512x256", (512, 512, 256), 1), ("4096x4096 x4", (4096, 4096), 4)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().split("\n")[0]
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


def conv_app(vk, shape, batch, dst, chain):
    """a convolution plan through the C ABI; chain=True: made with B200FFT_NO_FUSED_CONV=1"""
    if chain:
        os.environ["B200FFT_NO_FUSED_CONV"] = "1"
    try:
        app = vk.VkFFTApplication()
        rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0, normalize=1,
                                                           performConvolution=1, isInputFormatted=1, **{"performDST" if dst else "performDCT": 2}))
    finally:
        os.environ.pop("B200FFT_NO_FUSED_CONV", None)
    assert rc == 0, vk.getVkFFTErrorString(rc)
    return app


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    a = ap.parse_args()
    import torch
    import vkfft_b200 as vk
    from vkfft_b200 import fft
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    gpu = card()
    for name, shape, batch in SHAPES:
        nps = tuple(reversed(shape))
        x = torch.rand((batch,) + nps, device="cuda", dtype=torch.float32)
        k = torch.rand(nps, device="cuda", dtype=torch.float32)
        y = torch.empty_like(x)
        points = x.numel()
        for dst in (False, True):
            fwd, inv = (fft.dstn, fft.idstn) if dst else (fft.dctn, fft.idctn)
            chain_app = conv_app(vk, shape, batch, dst, True)
            probe = conv_app(vk, shape, batch, dst, False)
            launches = len(vk.planInfo(probe)["forward"].strip().split("\n"))
            vk.deleteVkFFT(probe)
            fused = launches == 2 * len(shape) - 1
            stream = torch.cuda.current_stream().cuda_stream

            def plan():
                fft.convolve_r2r(x, k, dest=y, ndim=len(shape), dst=dst)

            def chain():
                assert vk.VkFFTAppend(chain_app, -1, vk.VkFFTLaunchParams(buffer=y, inputBuffer=x, kernel=k, stream=stream)) == 0

            def separate():
                t = fwd(x, ndim=len(shape))
                t.mul_(k)
                inv(t, dest=y, ndim=len(shape))

            variants = {"plan": plan, "chain": chain, "separate": separate}
            plan()
            ref = y.clone()
            err = {}
            for v in ("chain", "separate"):
                variants[v]()
                err[v] = float((y - ref).norm() / ref.norm())
            res = {v: [] for v in variants}
            for _ in range(a.rounds):
                for v, fn in variants.items():
                    res[v].append(timed(torch, fn, a.window))
            ms = {v: round(statistics.median(t), 4) for v, t in res.items()}
            nbytes = {v: (16 * len(shape) + (-4 if (v == "plan" and fused) else 12)) * points for v in variants}
            share = {v: round(nbytes[v] / (m * 1e-3) / PEAK_BPS, 3) for v, m in ms.items()}
            print(json.dumps({"shape": name, "type": "DST-II" if dst else "DCT-II", "gpu": gpu, "plan_launches": launches, "fused": fused,
                              "ms": ms, "share_of_3.35TBps": share, "algorithmic_bytes": nbytes, "rel_l2_vs_plan": err}), flush=True)
            vk.deleteVkFFT(chain_app)
        del x, k, y
        fft.clear_cache()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
