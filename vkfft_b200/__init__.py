"""vkfft_b200 -- H100-native FFT engine behind the VkFFT application API (CUDA backend only).

The product is csrc/ (hand-written sm_90a kernels + planner + C ABI, built into lib/libb200fft.so) and
include/vkFFT.h (the header-only C/C++ drop-in).  This Python package is the thin host-side mirror of the
same API used by the tests and the benchmark.
"""
from .api import *  # noqa: F401,F403
from .api import (VkFFTApplication, VkFFTConfiguration, VkFFTLaunchParams, VkFFTAppend, deleteVkFFT, execHost,
                  getVkFFTErrorString, initializeVkFFT, planInfo, VkFFTGetVersion)
