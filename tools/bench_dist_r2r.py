#!/usr/bin/env python3
"""Distributed 2-D / 3-D DCT / DST (FusedDistributedR2RND) against one single-GPU plan of the same array.

Spawns R ranks (default 2), one process each, on GPU rank % device_count -- on a one-GPU box every rank shares cuda:0, so the
distributed figures show the barriers and the launch overhead of the slab plan, NOT multi-GPU scaling (the output says which).
Per shape it reports:
  - ms per forward + inverse pair (DCT-II + DCT-III by default) of the distributed plan (CUDA events on every rank around the
    same number of pairs, max over ranks);
  - ms per pair of one single-GPU plan of the whole array with the same pitches (rank 0, while the others wait);
  - the `timed()` breakdown of one forward and one inverse execution (launches and device-side barriers, rank 0);
  - the GPU's name and power limit, read in the same run.
Prints a markdown table and one JSON line; `--out FILE` also writes the JSON there.
"""
import argparse
import json
import os
import socket
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(8192, 8192), (4096, 4096), (256, 256, 256), (512, 512, 256)]     # 8192 x 8192: BASELINE config 4


def gpu_facts():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().split("\n")[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def _pairs_ms(torch, fwd, inv, steps, warmup):
    for _ in range(warmup):
        fwd()
        inv()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fwd()
        inv()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _worker(rank, world, port, shape, kind, dst, double, steps, warmup, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vkfft_b200 import api
        from vkfft_b200.dist import FusedDistributedR2RND, max_over_ranks
        dev = rank % torch.cuda.device_count()
        torch.cuda.set_device(dev)
        f = FusedDistributedR2RND(shape, dist, dev, kind=kind, dst=dst, double=double, normalize=True)
        f.local.uniform_(-1, 1)
        torch.cuda.synchronize()
        dist.barrier()
        f()
        f(inverse=True)
        torch.cuda.synchronize()
        dist.barrier()
        ms = max_over_ranks(_pairs_ms(torch, lambda: f(), lambda: f(inverse=True), steps, warmup), dist)
        f.check()
        dist.barrier()
        brk = (f.timed(False), f.timed(True))
        f.check()
        single = None
        if rank == 0:
            nd = len(shape)
            p = f.pitches
            buf = torch.empty(shape[-1] * p[nd - 2], dtype=torch.float64 if double else torch.float32, device=dev).uniform_(-1, 1)
            app = api.VkFFTApplication()
            cfg = api.VkFFTConfiguration(FFTdim=nd, size=list(shape), performDCT=0 if dst else kind, performDST=kind if dst else 0,
                                         bufferStride=list(p), device=dev, doublePrecision=int(double), normalize=1)
            assert api.initializeVkFFT(app, cfg) == 0
            lp = api.VkFFTLaunchParams(buffer=buf, stream=torch.cuda.current_stream().cuda_stream)
            single = _pairs_ms(torch, lambda: api.VkFFTAppend(app, -1, lp), lambda: api.VkFFTAppend(app, 1, lp), steps, warmup)
            api.deleteVkFFT(app)
            del buf
        dist.barrier()
        f.close()
        q.put((rank, ms, single, brk, f.pitches, None))
    except Exception as e:  # noqa: BLE001
        q.put((rank, None, None, None, None, repr(e)))
    finally:
        dist.destroy_process_group()


def run(shape, world, kind, dst, double, steps, warmup):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, shape, kind, dst, double, steps, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=900) for _ in procs)
    for p in procs:
        p.join(timeout=120)
    for r in res:
        if r[5] is not None:
            raise RuntimeError(f"rank {r[0]}: {r[5]}")
    return res[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kind", type=int, default=2)
    ap.add_argument("--dst", action="store_true")
    ap.add_argument("--double", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu == 0:
        raise SystemExit("no GPU: nothing to measure")
    name, power = gpu_facts()
    shared = ngpu < a.world
    note = (f"{a.world} ranks share {ngpu} GPU(s): the distributed figures show barrier and launch overhead, not multi-GPU scaling"
            if shared else f"{a.world} ranks on {a.world} GPUs")
    rows = []
    for shape in SHAPES:
        _, ms, single, brk, pitches, _ = run(shape, a.world, a.kind, a.dst, a.double, a.steps, a.warmup)
        rows.append(dict(shape=list(shape), pitches=pitches, dist_ms=round(ms, 4), single_ms=round(single, 4),
                         forward=brk[0], inverse=brk[1]))
    prec = "FP64" if a.double else "FP32"
    tf = f"{'DST' if a.dst else 'DCT'}-{'I' * a.kind if a.kind < 4 else 'IV'}"
    print(f"{name}, power limit {power}; {prec} {tf}, in place, normalised, ms per forward + inverse pair; {note}")
    print("| shape (x, y[, z]) | distributed, R = %d | single-GPU plan, same pitches | forward launches / barriers (ms) | inverse (ms) |" % a.world)
    print("|---|---|---|---|---|")
    for r in rows:
        fmt = lambda b: " ".join(f"{'K' if k == 'kernel' else 'B'}{v:.3f}" for k, v in b)
        print(f"| {' x '.join(map(str, r['shape']))} | {r['dist_ms']:.3f} | {r['single_ms']:.3f} | {fmt(r['forward'])} | {fmt(r['inverse'])} |")
    print("K = a launch, B = a device-side barrier (the last B of a direction is the trailing one)")
    res = dict(gpu=name, power_limit=power, world=a.world, gpus=ngpu, shared_gpu=shared, precision=prec, transform=tf, rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
