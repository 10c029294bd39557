"""GPU: distributed 2-D / 3-D R2C / C2R (FusedDistributedRFFTND: slabs of the in-place R2C layout in peer windows, device-side
barriers) with two processes.

Uses two GPUs when the box has them; on a one-GPU box both ranks map their slabs on cuda:0, as test_gpu_dist_fused.py does.
Checked per rank: the forward spectrum against torch.fft.rfftn in float64, the normalised round trip, no barrier time-out, and
bit identity with the single-GPU R2C plan of the same array with the same pitches where both plans run the same kernels."""
import ctypes
import os
import re
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _kernels(text):
    return [re.sub(r" grid=\d+", "", re.split(r"  (buffer|temp) ->", line.split(": ", 1)[-1])[0]).split(" n=", 1)[-1]
            for line in text.strip().split("\n")]


def _describe(app, inverse):
    from vkfft_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 15)
    _lib.load().b200fft_plan_describe(app._plan, inverse, buf, len(buf))
    return buf.value.decode()


def _single_gpu_spectrum(torch, api, shape_xyz, pitches, double, full, dev):
    """forward R2C of the whole field by one single-GPU plan with the same pitches: (spectrum [n_last, ..., H], kernels)"""
    nd = len(shape_xyz)
    cdt, rdt = (torch.complex128, torch.float64) if double else (torch.complex64, torch.float32)
    h = shape_xyz[0] // 2 + 1
    inner = tuple(reversed(shape_xyz[1:-1]))
    inner_pitch = tuple(pitches[:nd - 2][::-1])
    flat = torch.zeros(shape_xyz[-1] * pitches[nd - 2], dtype=cdt, device=dev)
    real = torch.view_as_real(flat).view(-1).as_strided((shape_xyz[-1],) + inner + (shape_xyz[0],),
                                                        tuple(2 * p for p in (pitches[nd - 2],) + inner_pitch) + (1,))
    real.copy_(full.to(rdt))
    app = api.VkFFTApplication()
    cfg = api.VkFFTConfiguration(FFTdim=nd, size=list(shape_xyz), performR2C=1, bufferStride=list(pitches), device=dev,
                                 doublePrecision=int(double))
    assert api.initializeVkFFT(app, cfg) == 0
    assert api.VkFFTAppend(app, -1, api.VkFFTLaunchParams(buffer=flat)) == 0
    torch.cuda.synchronize()
    kernels = _kernels(_describe(app, -1))
    api.deleteVkFFT(app)
    spec = flat.as_strided((shape_xyz[-1],) + inner + (h,), (pitches[nd - 2],) + inner_pitch + (1,))
    return spec.cpu(), kernels


def _worker(rank, world, port, shape_xyz, double, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vkfft_b200 import api
        from vkfft_b200.dist import FusedDistributedRFFTND
        dev = rank % torch.cuda.device_count()
        torch.cuda.set_device(dev)
        g = torch.Generator(device="cpu").manual_seed(17)
        np_shape = tuple(reversed(shape_xyz))
        full = torch.empty(np_shape, dtype=torch.float64).uniform_(-1, 1, generator=g)
        if not double:
            full = full.to(torch.float32)
        sl = np_shape[0] // world
        mine = full[rank * sl:(rank + 1) * sl]
        f = FusedDistributedRFFTND(shape_xyz, dist, dev, double=double, normalize=True)
        f.real.copy_(mine)
        torch.cuda.synchronize()
        dist.barrier()
        f()
        f.check()
        got = f.local.cpu()
        ref = torch.fft.rfftn(full.to(torch.float64))[rank * sl:(rank + 1) * sl]
        err = ((got.to(torch.complex128) - ref).abs().norm() / ref.abs().norm()).item()
        single, kernels = _single_gpu_spectrum(torch, api, shape_xyz, f.pitches, double, full, dev)
        same = _kernels(_describe(f.app, -1)) == kernels
        identical = torch.equal(torch.view_as_real(got), torch.view_as_real(single[rank * sl:(rank + 1) * sl])) if same else None
        f(inverse=True)
        f.check()
        back = ((f.real.cpu().to(torch.float64) - mine.to(torch.float64)).norm() / mine.to(torch.float64).norm()).item()
        f.close()
        q.put((rank, err, back, identical, None))
    except Exception as e:  # noqa: BLE001
        q.put((rank, None, None, None, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("shape_xyz,double", [((2048, 1024), False), ((256, 128, 64), False),
                                              ((64, 8192), False),           # the last axis as a Four-Step across the slabs
                                              ((128, 64, 32), True)])
def test_distributed_rfft_two_ranks(shape_xyz, double):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, shape_xyz, double, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    tol = 1e-12 if double else 1e-6
    for rank, err, back, identical, exc in res:
        assert exc is None, exc
        assert err < tol, (rank, err)
        assert back < tol, (rank, back)
        assert identical is not False, (rank, "differs from the single-GPU plan that runs the same kernels")
