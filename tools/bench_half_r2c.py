#!/usr/bin/env python3
"""R2C + C2R in place with FP32 storage vs half-precision storage (halfPrecision = 1), alternating the two in one process.

Workloads: the 4096 x 4096 x 16 R2C of BASELINE config 4, 4096-point rows x 2^15 (one fused launch per direction) and
2^20-point rows x 64 (Four-Step + the Hermitian launch).  Every plan is warmed up first; each timed window runs at least
half a second of forward+inverse pairs between CUDA events, the two storages alternate window by window, and the median
window is reported.  Bytes are the plan's algorithmic bytes (one read + one write of the data per transformed axis and
direction), the fraction is of the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line, with the GPU's name and power
limit read in the same run.
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import vkfft_b200 as vk

PEAK_TBS = 3.35
WORKLOADS = [("4096x4096x16", (4096, 4096), 16), ("4096x2^15", (4096,), 1 << 15), ("2^20x64", (1 << 20,), 64)]
WINDOW_S, ROUNDS = 0.5, 5


def gpu_facts():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().split("\n")[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


class Case:
    def __init__(self, shape, batch, half):
        nx = shape[0]
        rows = batch
        for s in shape[1:]:
            rows *= s
        dt = torch.float16 if half else torch.float32
        self.buf = torch.empty(rows * (nx + 2), dtype=dt, device="cuda").uniform_(-1, 1)
        self.app = vk.VkFFTApplication()
        rc = vk.initializeVkFFT(self.app, vk.VkFFTConfiguration(FFTdim=len(shape), size=list(shape), numberBatches=batch, device=0,
                                                                performR2C=1, normalize=1, halfPrecision=int(half)))
        assert rc == 0, vk.getVkFFTErrorString(rc)
        info = vk.planInfo(self.app)
        self.pair_bytes = 2 * info["algorithmic_bytes"]
        self.launches = info["forward"].strip().count("\n") + 1
        self.lp = vk.VkFFTLaunchParams(buffer=self.buf)

    def pairs(self, k):
        for _ in range(k):
            assert vk.VkFFTAppend(self.app, -1, self.lp) == 0
            assert vk.VkFFTAppend(self.app, 1, self.lp) == 0

    def window(self, k):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self.pairs(k)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / k

    def close(self):
        vk.deleteVkFFT(self.app)
        del self.buf


def main():
    name, power = gpu_facts()
    result = {"gpu": name, "power_limit": power, "peak_tb_s": PEAK_TBS, "workloads": {}}
    for label, shape, batch in WORKLOADS:
        cases = {h: Case(shape, batch, h) for h in (0, 1)}
        reps = {}
        for h, c in cases.items():                 # warm-up, then size the window to >= WINDOW_S
            c.pairs(3)
            torch.cuda.synchronize()
            ms = c.window(3)
            reps[h] = max(3, int(WINDOW_S * 1e3 / ms) + 1)
        times = {0: [], 1: []}
        for _ in range(ROUNDS):
            for h in (0, 1):
                times[h].append(cases[h].window(reps[h]))
        row = {}
        for h, key in ((0, "fp32"), (1, "half")):
            t = sorted(times[h])
            med = t[len(t) // 2]
            c = cases[h]
            row[key] = {"ms_per_pair": round(med, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
                        "launches_per_direction": c.launches, "algorithmic_bytes_per_pair": c.pair_bytes,
                        "fraction_of_peak": round(c.pair_bytes / (med * 1e-3) / (PEAK_TBS * 1e12), 3)}
        row["half_over_fp32_time"] = round(row["half"]["ms_per_pair"] / row["fp32"]["ms_per_pair"], 3)
        result["workloads"][label] = row
        for c in cases.values():
            c.close()
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
