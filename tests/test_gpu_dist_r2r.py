"""GPU: distributed 2-D / 3-D DCT / DST (FusedDistributedR2RND: slabs of the real array in peer windows, device-side barriers)
with two processes.

Uses two GPUs when the box has them; on a one-GPU box both ranks map their slabs on cuda:0, as test_gpu_dist_rfft.py does.
Checked per rank: the forward transform against scipy.fft.dctn / dstn in float64, the normalised round trip, no barrier
time-out, and bit identity with the single-GPU plan of the same array with the same pitches where both plans run the same
kernels."""
import ctypes
import os
import re
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _kernels(text):
    return [re.sub(r" (grid|items)=\d+", "", re.split(r"  (buffer|temp) ->", line.split(": ", 1)[-1])[0]).split(" n=", 1)[-1]
            for line in text.strip().split("\n")]


def _describe(app, inverse):
    from vkfft_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 15)
    _lib.load().b200fft_plan_describe(app._plan, inverse, buf, len(buf))
    return buf.value.decode()


def _single_gpu(torch, api, shape_xyz, pitches, kind, dst, double, full, dev):
    """forward transform of the whole field by one single-GPU plan with the same pitches: (result [n_last, ..., nx], kernels)"""
    nd = len(shape_xyz)
    rdt = torch.float64 if double else torch.float32
    view_shape = (shape_xyz[-1],) + tuple(reversed(shape_xyz[1:-1])) + (shape_xyz[0],)
    view_strides = (pitches[nd - 2],) + tuple(pitches[:nd - 2][::-1]) + (1,)
    flat = torch.zeros(shape_xyz[-1] * pitches[nd - 2], dtype=rdt, device=dev)
    flat.as_strided(view_shape, view_strides).copy_(full.to(rdt))
    app = api.VkFFTApplication()
    cfg = api.VkFFTConfiguration(FFTdim=nd, size=list(shape_xyz), performDCT=0 if dst else kind, performDST=kind if dst else 0,
                                 bufferStride=list(pitches), device=dev, doublePrecision=int(double))
    assert api.initializeVkFFT(app, cfg) == 0
    assert api.VkFFTAppend(app, -1, api.VkFFTLaunchParams(buffer=flat)) == 0
    torch.cuda.synchronize()
    kernels = _kernels(_describe(app, -1))
    api.deleteVkFFT(app)
    return flat.as_strided(view_shape, view_strides).cpu(), kernels


def _worker(rank, world, port, shape_xyz, kind, dst, double, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    import numpy as np
    import scipy.fft as sfft
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from vkfft_b200 import api
        from vkfft_b200.dist import FusedDistributedR2RND
        dev = rank % torch.cuda.device_count()
        torch.cuda.set_device(dev)
        g = torch.Generator(device="cpu").manual_seed(23)
        np_shape = tuple(reversed(shape_xyz))
        full = torch.empty(np_shape, dtype=torch.float64).uniform_(-1, 1, generator=g)
        if not double:
            full = full.to(torch.float32)
        sl = np_shape[0] // world
        mine = full[rank * sl:(rank + 1) * sl]
        f = FusedDistributedR2RND(shape_xyz, dist, dev, kind=kind, dst=dst, double=double, normalize=True)
        f.local.copy_(mine)
        torch.cuda.synchronize()
        dist.barrier()
        f()
        f.check()
        got = f.local.cpu().to(torch.float64).numpy()
        ref = (sfft.dstn if dst else sfft.dctn)(full.to(torch.float64).numpy(), type=kind)[rank * sl:(rank + 1) * sl]
        err = float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
        text = _describe(f.app, -1)
        single, kernels = _single_gpu(torch, api, shape_xyz, f.pitches, kind, dst, double, full, dev)
        same = _kernels(text) == kernels
        identical = torch.equal(f.local.cpu(), single[rank * sl:(rank + 1) * sl]) if same else None
        f(inverse=True)
        f.check()
        back = ((f.local.cpu().to(torch.float64) - mine.to(torch.float64)).norm() / mine.to(torch.float64).norm()).item()
        f.close()
        q.put((rank, err, back, identical, text, None))
    except Exception as e:  # noqa: BLE001
        q.put((rank, None, None, None, None, repr(e)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("shape_xyz,kind,dst,double", [((2048, 1024), 2, False, False), ((256, 128, 64), 2, True, False),
                                                       ((64, 8192), 2, False, False),    # the long strided route across the slabs
                                                       ((128, 64, 32), 4, False, True)])
def test_distributed_r2r_two_ranks(shape_xyz, kind, dst, double):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, shape_xyz, kind, dst, double, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    tol = 1e-12 if double else 2e-6
    for rank, err, back, identical, text, exc in res:
        assert exc is None, exc
        assert err < tol, (rank, err)
        assert back < tol, (rank, back)
        assert identical is not False, (rank, "differs from the single-GPU plan that runs the same kernels")
        if shape_xyz == (64, 8192):
            assert sum("long dct-ii" in line for line in text.strip().split("\n")) == 3, text
