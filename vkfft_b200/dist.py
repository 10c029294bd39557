"""Batch sharding of one VkFFT configuration over the GPUs of a box (one process per GPU).

Batched transforms are independent units along the outermost (batch) stride (API guide :285-289), so a job splits
into contiguous slabs of `numberBatches` with NO data-path collective; torch.distributed is used only for the
barrier and the max-over-ranks time (NCCL on GPUs, gloo in the CPU tests).  The reference has no multi-GPU mode
(README.md:26-28 lists it as future work)."""
from dataclasses import replace
from typing import Tuple


def shard_batches(number_batches: int, world: int, rank: int) -> Tuple[int, int]:
    """contiguous slab [start, start+count) of the batch dimension owned by `rank`; slabs differ by at most 1"""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad world/rank")
    base, extra = divmod(max(number_batches, 1), world)
    count = base + (1 if rank < extra else 0)
    start = rank * base + min(rank, extra)
    return start, count


def shard_configuration(cfg, world: int, rank: int):
    """per-rank copy of a VkFFTConfiguration: numberBatches cut to the rank's slab, device = local rank.
    Returns (cfg_rank, first_batch, byte_offset_of_slab) -- byte offset in the global (unsharded) buffer layout."""
    nb = cfg.numberBatches or 1
    start, count = shard_batches(nb, world, rank)
    per_batch = 1
    for s in cfg.size[: cfg.FFTdim]:
        per_batch *= s
    if cfg.performR2C:
        per_batch = per_batch // cfg.size[0] * (cfg.size[0] // 2 + 1)
    esz = (16 if cfg.doublePrecision else 8) if not cfg.performDCT else (8 if cfg.doublePrecision else 4)
    per_batch *= (cfg.coordinateFeatures or 1)
    out = replace(cfg, numberBatches=count, device=rank)
    return out, start, start * per_batch * esz


def max_over_ranks(value: float, dist=None) -> float:
    """max of a per-rank scalar (timings) over the job; identity when not distributed"""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return value
    import torch
    backend = dist.get_backend()
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    t = torch.tensor([value], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


class DistributedFFT1D:
    """One very long 1-D C2C transform spread over the GPUs of a box: the outer Four-Step axis is sharded
    (BASELINE.json config 5; SURVEY.md section 8e).  N = N1*N2, world R divides N1 and N2.

    Every rank holds a contiguous slab of N/R input points in natural order and receives the matching slab of the
    spectrum in natural order.  Data flow (x viewed as [N1][N2], n = n1*N2 + n2, k = k1 + N1*k2):

        rows n1-slab  --all-to-all-->  columns n2-slab : strided length-N1 transforms + phase W_N^(n2*k1)   (engine plan)
                      --all-to-all-->  rows k1-slab    : contiguous length-N2 transforms                     (engine plan)
                      --all-to-all-->  natural-order slab of X (skipped with transposed_output=True)

    The exchanges are torch.distributed all_to_all_single calls (NCCL over NVLink on GPUs, gloo in the CPU tests);
    packing is plain tensor permutes.  The two local transforms go through the engine's C ABI unless `local_cols` /
    `local_rows` callables are injected (the CPU tests inject numpy so the index algebra is verified without a GPU).
    """

    def __init__(self, n1, n2, dist, inverse=False, transposed_output=False, local_cols=None, local_rows=None, device=None):
        import torch
        self.torch = torch
        self.dist = dist
        self.R = dist.get_world_size()
        self.r = dist.get_rank()
        self.n1, self.n2, self.n = n1, n2, n1 * n2
        if n1 % self.R or n2 % self.R:
            raise ValueError("world size must divide both Four-Step factors")
        self.inverse = inverse
        self.transposed_output = transposed_output
        self.device = device
        self._apps = []
        self.local_cols = local_cols or self._engine_cols
        self.local_rows = local_rows or self._engine_rows
        # phase table of this rank's columns: W_N^(+-(n2*k1)), n2 = r*N2/R + j   (float64 -> complex64)
        c = n2 // self.R
        k1 = torch.arange(n1, dtype=torch.float64).unsqueeze(1)
        j = (self.r * c + torch.arange(c, dtype=torch.float64)).unsqueeze(0)
        sign = 1.0 if inverse else -1.0
        e = torch.remainder(k1 * j, float(self.n))                  # exact in float64 for N <= 2^26
        ang = sign * 2.0 * 3.141592653589793238 * e / float(self.n)
        self.phase = torch.complex(torch.cos(ang), torch.sin(ang)).to(torch.complex64)
        if device is not None:
            self.phase = self.phase.to(device)

    # ---- local transforms through the engine --------------------------------------------------------------------------
    def _plan(self, key, cfg):
        from . import api
        for k, app in self._apps:
            if k == key:
                return app
        app = api.VkFFTApplication()
        rc = api.initializeVkFFT(app, cfg)
        if rc != 0:
            raise RuntimeError(api.getVkFFTErrorString(rc))
        self._apps.append((key, app))
        return app

    def _engine_cols(self, b):          # b: [N1][C] complex64 on the GPU, transform along dim 0 in place
        from . import api
        c = b.shape[1]
        cfg = api.VkFFTConfiguration(FFTdim=2, size=[c, self.n1], omitDimension=[1, 0], device=b.device.index)
        app = self._plan(("cols", c), cfg)
        lp = api.VkFFTLaunchParams(buffer=b, stream=self.torch.cuda.current_stream().cuda_stream)
        rc = api.VkFFTAppend(app, 1 if self.inverse else -1, lp)
        if rc != 0:
            raise RuntimeError(api.getVkFFTErrorString(rc))
        return b

    def _engine_rows(self, b):          # b: [B][N2], transform along dim 1 in place
        from . import api
        cfg = api.VkFFTConfiguration(FFTdim=1, size=[self.n2], numberBatches=b.shape[0], device=b.device.index)
        app = self._plan(("rows", b.shape[0]), cfg)
        lp = api.VkFFTLaunchParams(buffer=b, stream=self.torch.cuda.current_stream().cuda_stream)
        rc = api.VkFFTAppend(app, 1 if self.inverse else -1, lp)
        if rc != 0:
            raise RuntimeError(api.getVkFFTErrorString(rc))
        return b

    def close(self):
        from . import api
        for _, app in self._apps:
            api.deleteVkFFT(app)
        self._apps = []

    # ---- the distributed transform ------------------------------------------------------------------------------------
    def __call__(self, x):
        """x: this rank's slab, 1-D complex tensor of N/R points (natural order). Returns this rank's slab of X."""
        torch, dist, R = self.torch, self.dist, self.R
        n1, n2 = self.n1, self.n2
        r1, c = n1 // R, n2 // R
        a = x.view(r1, R, c).permute(1, 0, 2).contiguous()          # [dest][n1_local][n2_local]
        b = torch.empty_like(a)
        dist.all_to_all_single(b, a)                                # b: [src][n1_local][n2_local] == [N1][C]
        b = self.local_cols(b.view(n1, c))                          # FFT over n1
        b = b * self.phase if b.dtype == self.phase.dtype else b * self.phase.to(b.dtype)
        a2 = torch.empty_like(b)
        dist.all_to_all_single(a2, b.contiguous())                  # send row-chunks; receive [src][k1_local][n2_local]
        rows = a2.view(R, r1, c).permute(1, 0, 2).contiguous().view(r1, n2)   # [k1_local][n2]
        rows = self.local_rows(rows)                                # FFT over n2 -> [k1_local][k2] = X[k1 + N1 k2]
        if self.transposed_output:
            return rows
        s = rows.view(r1, R, c).permute(1, 0, 2).contiguous()       # [dest t][k1_local][k2_local]
        t = torch.empty_like(s)
        dist.all_to_all_single(t, s)                                # [src e][k1_local][k2_local]
        return t.view(R, r1, c).permute(2, 0, 1).contiguous().view(-1)   # [k2_local][k1] -> natural order slab


class FusedDistributedFFT1D:
    """One long 1-D C2C sequence over the GPUs of a box with the exchange fused into the FFT launches
    (SURVEY.md section 8e, second row; BASELINE.json config 5).

    Memory: two peer windows (window.PeerWindow) -- the sequence itself and a scratch of the same size; rank g's slab
    is elements [g*N/R, (g+1)*N/R) of both, and every rank sees both as flat arrays of N points.  Execution: every rank
    runs its slice of the ordinary Four-Step launches (planner.cpp plan_c2c, `dist` branches):

        launch 1  columns [g*C, (g+1)*C): strided loads gather the column from all slabs (NVLink reads), phase
                  multiply, stores scatter it to the scratch slabs of its owners (NVLink writes)
        (launch 2 of a 3-launch split: local)
        last      rows of the rank's own scratch slab, transposed store into every slab of the sequence window

    so the all-to-all exchanges of DistributedFFT1D (3 NCCL collectives + pack/unpack passes + a phase pass) become
    the loads and stores of 2-3 kernels, separated by device-side barriers on a signal pad.  Input and output are both
    in natural order, in place in `self.local` (this rank's slab)."""

    def __init__(self, n, dist, device, double=False, normalize=False):
        import torch
        from . import api
        self.torch, self.dist, self.api = torch, dist, api
        self.R, self.r = dist.get_world_size(), dist.get_rank()
        if n % self.R:
            raise ValueError("world size must divide N")
        esz = 16 if double else 8
        self.n = n
        cfg = api.VkFFTConfiguration(FFTdim=1, size=[n], device=device, doublePrecision=int(double), normalize=int(normalize),
                                     userTempBuffer=1, distWorld=self.R, distRank=self.r)
        self._open(n // self.R * esz, cfg, device)
        self.local = self.seq.tensor(torch, torch.complex128 if double else torch.complex64)

    def _open(self, slab_bytes, cfg, device):
        """the two peer windows (data and scratch, `slab_bytes` per rank) and this rank's plan, bound to the data window"""
        from . import _lib
        from .window import PeerWindow
        self.seq = PeerWindow(slab_bytes, self.dist, device)
        self.tmp = PeerWindow(slab_bytes, self.dist, device)
        self.app = self.api.VkFFTApplication()
        rc = self.api.initializeVkFFT(self.app, cfg)
        if rc != 0:
            self.close()
            raise RuntimeError(self.api.getVkFFTErrorString(rc))
        _lib.load().b200fft_plan_attach_window(self.app._plan, self.seq.handle)

    def __call__(self, inverse=False):
        """transform the sequence held in the windows in place; asynchronous on the current stream"""
        lp = self.api.VkFFTLaunchParams(buffer=self.seq.base, tempBuffer=self.tmp.base,
                                        stream=self.torch.cuda.current_stream().cuda_stream)
        rc = self.api.VkFFTAppend(self.app, 1 if inverse else -1, lp)
        if rc != 0:
            raise RuntimeError(self.api.getVkFFTErrorString(rc))
        return self.local

    def timed(self, inverse=False):
        """one execution with an event after every launch: [('barrier'|'kernel', ms), ...] (tuning aid; synchronises)"""
        import ctypes
        from . import _lib
        L = _lib.load()
        b = _lib.b200fft_buffers()
        b.buffer, b.temp_buffer = self.seq.base, self.tmp.base
        b.stream = self.torch.cuda.current_stream().cuda_stream
        ms, kind, n = (ctypes.c_float * 16)(), (ctypes.c_int * 16)(), ctypes.c_int(0)
        L.b200fft_debug_exec_timed.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_int, ctypes.c_void_p]
        rc = L.b200fft_debug_exec_timed(self.app._plan, 1 if inverse else -1, ctypes.byref(b), ms, kind, 16, ctypes.byref(n))
        if rc != 0:
            raise RuntimeError(self.api.getVkFFTErrorString(rc))
        return [("kernel" if kind[i] else "barrier", round(ms[i], 4)) for i in range(min(n.value, 16))]

    def check(self):
        """synchronise and raise if a device-side barrier timed out (a rank died or never launched)"""
        if self.seq.status() != 0:
            raise RuntimeError("distributed FFT: a device-side barrier timed out")

    def close(self):
        if getattr(self, "app", None) is not None and self.app._plan is not None:
            self.torch.cuda.synchronize()
            self.api.deleteVkFFT(self.app)
        for w in ("seq", "tmp"):
            if getattr(self, w, None) is not None:
                getattr(self, w).close()
                setattr(self, w, None)


class FusedDistributedFFTND(FusedDistributedFFT1D):
    """A 2-D or 3-D C2C transform whose array is spread over the GPUs of a box in SLABS along its last (slowest) dimension
    (SURVEY.md section 8 f4).

    `shape_xyz` = (nx, ny[, nz]) with x fastest, as VkFFT counts; rank g holds the planes [g*n_last/R, (g+1)*n_last/R) of the
    array, contiguous, in `self.local` (shape (n_last/R, ..., nx)).  The lower axes are transformed inside every rank's own slab;
    the last axis runs as strided launches over the peer window whose lines are shared out over the ranks -- their loads gather
    a line from all slabs and their stores scatter it back, which IS the exchange of the textbook slab algorithm (no transposes,
    no collective; planner.cpp plan_direction_c2c).  One device-side barrier separates the two parts.  In place, natural order."""

    def __init__(self, shape_xyz, dist, device, double=False, normalize=False):
        import torch
        from . import api
        self.torch, self.dist, self.api = torch, dist, api
        self.R, self.r = dist.get_world_size(), dist.get_rank()
        shape_xyz = tuple(int(v) for v in shape_xyz)
        if not 2 <= len(shape_xyz) <= 3:
            raise ValueError("2-D or 3-D shapes; one long sequence is FusedDistributedFFT1D")
        if shape_xyz[-1] % self.R:
            raise ValueError("world size must divide the last dimension")
        total = 1
        for v in shape_xyz:
            total *= v
        esz = 16 if double else 8
        self.n = total
        self.shape_xyz = shape_xyz
        cfg = api.VkFFTConfiguration(FFTdim=len(shape_xyz), size=list(shape_xyz), device=device, doublePrecision=int(double),
                                     normalize=int(normalize), userTempBuffer=1, distWorld=self.R, distRank=self.r)
        self._open(total // self.R * esz, cfg, device)
        dt = torch.complex128 if double else torch.complex64
        local_shape = (shape_xyz[-1] // self.R,) + tuple(reversed(shape_xyz[:-1]))
        self.local = self.seq.tensor(torch, dt).reshape(local_shape)


def r2c_slab_pitches(shape_xyz, world, esz, granularity):
    """complex-element pitches (bufferStride) of the in-place R2C layout whose slabs -- n_last/world outermost indices each --
    fill whole mapping granules: H = nx/2+1 complex per row, and only the outermost pitch of a slab (the row pitch in 2-D, the
    plane pitch in 3-D) padded, to the smallest value that makes a slab a multiple of `granularity` bytes.  Whenever n_last/world
    is a power of two that adds less than one granule per slab."""
    import math
    nx, rows = shape_xyz[0], shape_xyz[-1] // world
    h = nx // 2 + 1
    inner = h if len(shape_xyz) == 2 else h * shape_xyz[1]
    step = granularity // math.gcd(granularity, rows * esz)       # pitch multiple that makes rows * pitch * esz whole granules
    outer = -(-inner // step) * step
    return [outer, outer * shape_xyz[1]] if len(shape_xyz) == 2 else [h, outer, outer * shape_xyz[2]]


class FusedDistributedRFFTND(FusedDistributedFFT1D):
    """A 2-D or 3-D real-to-complex transform (and its complex-to-real inverse) whose array is spread over the GPUs of a box in
    slabs along its last dimension, like FusedDistributedFFTND, in the in-place R2C layout.

    `shape_xyz` = (nx, ny[, nz]) with x fastest, nx even.  Every row holds H = nx/2+1 complex points (the spectrum) or, before the
    forward transform and after the inverse one, nx reals in the same memory.  Rank g holds the last-dimension indices
    [g*n/R, (g+1)*n/R).  Its slab is padded on its outermost pitch only (`pitches`, complex elements: r2c_slab_pitches) so that it
    maps onto whole granules of the peer window.  Two views of the same memory:

        local   complex spectrum of shape (n/R, [ny,] H)
        real    the real field, shape (n/R, [ny,] nx), row pitch 2*pitches[0] reals

    `self()` runs the R2C forward, `self(inverse=True)` the C2R inverse (scaled by 1/(nx*ny[*nz]) with `normalize`), in place and
    asynchronously on the current stream.  Forward: x (and y) inside the slab, a device-side barrier, the last axis across the
    slabs on this rank's share of the spectrum columns; the inverse the other way round."""

    def __init__(self, shape_xyz, dist, device, double=False, normalize=False):
        import torch
        from . import api, _lib
        self.torch, self.dist, self.api = torch, dist, api
        self.R, self.r = dist.get_world_size(), dist.get_rank()
        shape_xyz = tuple(int(v) for v in shape_xyz)
        if not 2 <= len(shape_xyz) <= 3:
            raise ValueError("2-D or 3-D shapes")
        if shape_xyz[0] % 2 or shape_xyz[0] <= 2:
            raise ValueError("nx must be even and larger than 2")
        if shape_xyz[-1] % self.R:
            raise ValueError("world size must divide the last dimension")
        esz = 16 if double else 8
        gran = int(_lib.load().b200fft_window_granularity(int(device)))
        if gran == 0:
            raise RuntimeError("CUDA virtual memory management is not available on this device")
        self.shape_xyz = shape_xyz
        self.pitches = r2c_slab_pitches(shape_xyz, self.R, esz, gran)
        rows = shape_xyz[-1] // self.R
        nd = len(shape_xyz)
        self.n = 1
        for v in shape_xyz:
            self.n *= v
        cfg = api.VkFFTConfiguration(FFTdim=nd, size=list(shape_xyz), performR2C=1, bufferStride=list(self.pitches), device=device,
                                     doublePrecision=int(double), normalize=int(normalize), userTempBuffer=1,
                                     distWorld=self.R, distRank=self.r)
        self._open(rows * self.pitches[nd - 2] * esz, cfg, device)
        h = shape_xyz[0] // 2 + 1
        inner = tuple(reversed(shape_xyz[1:-1]))                          # (ny,) in 3-D
        inner_pitch = tuple(self.pitches[:nd - 2][::-1])                  # (H,) in 3-D
        cdt, rdt = (torch.complex128, torch.float64) if double else (torch.complex64, torch.float32)
        self.local = self.seq.tensor(torch, cdt).as_strided((rows,) + inner + (h,), (self.pitches[nd - 2],) + inner_pitch + (1,))
        self.real = self.seq.tensor(torch, rdt).as_strided((rows,) + inner + (shape_xyz[0],),
                                                           tuple(2 * p for p in (self.pitches[nd - 2],) + inner_pitch) + (1,))

