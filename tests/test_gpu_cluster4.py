"""GPU (-m gpu): the cluster Four-Step launch (csrc/cluster4.cuh) against the two-launch plan and the oracle.

For 2^15 and 2^16 points the default FP32 plan runs both Four-Step passes as one launch of thread-block clusters, one cluster
per sequence, the intermediate in distributed shared memory.  Both passes run the stage code of the two stand-alone kernels,
so every case must equal the same plan under B200FFT_NO_CLUSTER4=1 (two launches) bit for bit -- a missed barrier, a wrong
row owner or a stale tile shows up as a difference."""
import os

import numpy as np
import pytest

import vkfft_oracle as orc

pytestmark = pytest.mark.gpu

SIZES = [15, 16]


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    return torch


def make_app(size, batch, cluster, **cfgkw):
    import vkfft_b200 as vk
    old = os.environ.get("B200FFT_NO_CLUSTER4")
    if cluster:
        os.environ.pop("B200FFT_NO_CLUSTER4", None)
    else:
        os.environ["B200FFT_NO_CLUSTER4"] = "1"
    try:
        app = vk.VkFFTApplication()
        rc = vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=len(size), size=list(size), numberBatches=batch, device=0, **cfgkw))
    finally:
        if old is None:
            os.environ.pop("B200FFT_NO_CLUSTER4", None)
        else:
            os.environ["B200FFT_NO_CLUSTER4"] = old
    assert rc == 0, vk.getVkFFTErrorString(rc)
    txt = vk.planInfo(app)["forward"] + vk.planInfo(app)["inverse"]
    assert ("one cluster launch with the next pass" in txt) == cluster, txt
    return app


def run(torch, x, size, batch, inverse, cluster, **cfgkw):
    """in place on `buffer`, no tempBuffer"""
    import vkfft_b200 as vk
    app = make_app(size, batch, cluster, **cfgkw)
    t = torch.from_numpy(x).cuda()
    try:
        assert vk.VkFFTAppend(app, inverse, vk.VkFFTLaunchParams(buffer=t)) == 0
        torch.cuda.synchronize()
        return t.cpu().numpy()
    finally:
        vk.deleteVkFFT(app)


def same_bits(a, b):
    return np.array_equal(a.view(np.float32), b.view(np.float32))


@pytest.mark.parametrize("logn", SIZES)
@pytest.mark.parametrize("inverse", [-1, 1])
def test_batches_match_two_launches_and_oracle(gpu, logn, inverse):
    n = 1 << logn
    for batch in (1, 7, (1 << 25) // n + 1):          # one sequence, an odd batch, ~256 MiB
        x = orc.random_input((batch, n), np.complex64, seed=logn * 100 + batch)
        got = run(gpu, x, (n,), batch, inverse, True)
        assert same_bits(got, run(gpu, x, (n,), batch, inverse, False))
        rows = sorted({0, batch // 2, batch - 1})
        assert orc.error_metrics(got[rows], orc.c2c(x[rows], 1, inverse == 1))["l2_rel"] < 1e-6


@pytest.mark.parametrize("logn", SIZES)
def test_user_temp_buffer_and_out_of_place(gpu, logn):
    import vkfft_b200 as vk
    torch = gpu
    n, batch = 1 << logn, 5
    x = orc.random_input((batch, n), np.complex64, seed=logn)
    want = run(torch, x, (n,), batch, -1, False)
    # in place with the caller's tempBuffer (the cluster launch does not touch it)
    app = make_app((n,), batch, True, userTempBuffer=1, tempBufferSize=batch * n * 8)
    t = torch.from_numpy(x).cuda()
    tmp = torch.zeros(batch * n, dtype=torch.complex64, device="cuda")
    assert vk.VkFFTAppend(app, -1, vk.VkFFTLaunchParams(buffer=t, tempBuffer=tmp)) == 0
    torch.cuda.synchronize()
    vk.deleteVkFFT(app)
    assert same_bits(t.cpu().numpy(), want)
    # out of place: inputBuffer -> buffer; the input is only read
    app = make_app((n,), batch, True, isInputFormatted=1)
    tin = torch.from_numpy(x).cuda()
    tout = torch.zeros_like(tin)
    assert vk.VkFFTAppend(app, -1, vk.VkFFTLaunchParams(buffer=tout, inputBuffer=tin)) == 0
    torch.cuda.synchronize()
    vk.deleteVkFFT(app)
    assert same_bits(tout.cpu().numpy(), want)
    assert same_bits(tin.cpu().numpy(), x)


@pytest.mark.parametrize("logn", SIZES)
def test_normalised_round_trips(gpu, logn):
    """the same plan executed back to back, forward and inverse"""
    import vkfft_b200 as vk
    torch = gpu
    n, batch = 1 << logn, 9
    x = orc.random_input((batch, n), np.complex64, seed=3)
    outs = []
    for cluster in (True, False):
        app = make_app((n,), batch, cluster, normalize=1)
        t = torch.from_numpy(x).cuda()
        lp = vk.VkFFTLaunchParams(buffer=t)
        for _ in range(4):
            assert vk.VkFFTAppend(app, -1, lp) == 0
            assert vk.VkFFTAppend(app, 1, lp) == 0
        torch.cuda.synchronize()
        vk.deleteVkFFT(app)
        outs.append(t.cpu().numpy())
    assert same_bits(outs[0], outs[1])
    assert orc.error_metrics(outs[0], x)["l2_rel"] < 3e-6           # eight transforms


@pytest.mark.parametrize("logn", SIZES)
def test_8_byte_buffer_offset(gpu, logn):
    """a buffer that is only 8-byte aligned: the cluster launch uses plain loads and runs as usual"""
    import vkfft_b200 as vk
    torch = gpu
    n, batch = 1 << logn, 3
    x = orc.random_input((batch, n), np.complex64, seed=5)
    outs = []
    for cluster in (True, False):
        raw = torch.zeros(batch * n + 1, dtype=torch.complex64, device="cuda")
        raw[1:] = torch.from_numpy(x.reshape(-1)).cuda()
        app = make_app((n,), batch, cluster, specifyOffsetsAtLaunch=1)
        assert vk.VkFFTAppend(app, -1, vk.VkFFTLaunchParams(buffer=raw, bufferOffset=8)) == 0
        torch.cuda.synchronize()
        vk.deleteVkFFT(app)
        outs.append(raw[1:].cpu().numpy().reshape(batch, n))
    assert same_bits(outs[0], outs[1])
    assert orc.error_metrics(outs[0], orc.c2c(x, 1))["l2_rel"] < 1e-6


@pytest.mark.parametrize("logn", SIZES)
def test_long_axis_of_a_2d_shape(gpu, logn):
    nx, ny, batch = 1 << logn, 6, 1
    x = orc.random_input((batch, ny, nx), np.complex64, seed=11)
    got = run(gpu, x, (nx, ny), batch, -1, True)
    assert same_bits(got, run(gpu, x, (nx, ny), batch, -1, False))
    assert orc.error_metrics(got, orc.c2c(x, 2, False))["l2_rel"] < 1e-6


def test_2p17_keeps_two_launches(gpu):
    """no cluster shape beat the two launches at 2^17 on the H100: none is registered"""
    import vkfft_b200 as vk
    assert "B200FFT_NO_CLUSTER4" not in os.environ
    app = vk.VkFFTApplication()
    assert vk.initializeVkFFT(app, vk.VkFFTConfiguration(FFTdim=1, size=[1 << 17], numberBatches=3, device=0)) == 0
    txt = vk.planInfo(app)["forward"]
    vk.deleteVkFFT(app)
    assert "cluster" not in txt and len(txt.strip().split("\n")) == 2, txt
