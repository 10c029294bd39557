"""Host-side mirror of the reference's application API for its hot path, on top of the C ABI.

Same names, argument meaning and error behaviour as the reference (vkFFT_InitializeApp.h:1468,
vkFFT_RunApp.h:79, vkFFT_DeleteApp.h:28; structs vkFFT_Structs.h:93-379):

    cfg = VkFFTConfiguration(FFTdim=1, size=[4096], numberBatches=64, device=0)
    app = VkFFTApplication()
    assert initializeVkFFT(app, cfg) == VKFFT_SUCCESS
    lp = VkFFTLaunchParams(buffer=tensor)          # torch CUDA tensor or raw device pointer (int)
    VkFFTAppend(app, -1, lp)                       # -1 forward, +1 inverse; asynchronous
    deleteVkFFT(app)

Functions return VkFFTResult integers and never raise for engine errors (as the C API does).
PyTorch is only used by callers for device memory; nothing here imports it.
"""
import ctypes
from dataclasses import dataclass, field
from typing import Any, List, Optional

from . import _lib

VKFFT_SUCCESS = 0
VKFFT_ERROR_PLAN_NOT_INITIALIZED = 4
VKFFT_ERROR_FFTdim_GT_MAX_FFT_DIMENSIONS = 7
VKFFT_ERROR_NONZERO_APP_INITIALIZATION = 8
VKFFT_ERROR_INVALID_DEVICE = 1002
VKFFT_ERROR_ONLY_FORWARD_FFT_INITIALIZED = 1006
VKFFT_ERROR_ONLY_INVERSE_FFT_INITIALIZED = 1007
VKFFT_ERROR_EMPTY_FFTdim = 2001
VKFFT_ERROR_EMPTY_size = 2002
VKFFT_ERROR_EMPTY_buffer = 2004
VKFFT_ERROR_EMPTY_tempBuffer = 2006
VKFFT_ERROR_EMPTY_inputBuffer = 2008
VKFFT_ERROR_EMPTY_outputBuffer = 2010
VKFFT_ERROR_EMPTY_kernel = 2012
VKFFT_ERROR_EMPTY_app = 2015
VKFFT_ERROR_UNSUPPORTED_RADIX = 3001
VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH = 3002
VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C = 3003
VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2R = 3004
VKFFT_ERROR_UNSUPPORTED_FFT_OMIT = 3005
VKFFT_ERROR_FAILED_TO_ALLOCATE = 4001
VKFFT_ERROR_FAILED_TO_LAUNCH_KERNEL = 4039


def getVkFFTErrorString(result: int) -> str:
    return _lib.load().b200fft_error_string(int(result)).decode()


def VkFFTGetVersion() -> int:
    return 10304


def _ptr(x) -> Optional[int]:
    """device pointer of a torch tensor / anything with data_ptr(), or an int, or None"""
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return int(x.data_ptr())
    return int(x)


@dataclass
class VkFFTConfiguration:
    """The members of the reference's VkFFTConfiguration that the hot path consumes (zero/None = default)."""
    FFTdim: int = 0
    size: List[int] = field(default_factory=list)
    device: Optional[int] = None           # CUDA device ordinal (the reference takes CUdevice*)
    stream: Optional[int] = None           # cudaStream_t as int
    numberBatches: int = 0
    coordinateFeatures: int = 0
    doublePrecision: int = 0
    halfPrecision: int = 0            # half-precision storage (complex32 / float16 buffers), FP32 arithmetic; C2C, even-length R2C
    halfPrecisionMemoryOnly: int = 0  # only inputBuffer (isInputFormatted = 1) is half; buffer / tempBuffer / outputBuffer FP32
    performR2C: int = 0
    performDCT: int = 0
    performDST: int = 0
    normalize: int = 0
    disableReorderFourStep: int = 0
    makeForwardPlanOnly: int = 0
    makeInversePlanOnly: int = 0
    isInputFormatted: int = 0
    isOutputFormatted: int = 0
    inverseReturnToInputBuffer: int = 0
    userTempBuffer: int = 0
    bufferStride: List[int] = field(default_factory=list)
    inputBufferStride: List[int] = field(default_factory=list)
    outputBufferStride: List[int] = field(default_factory=list)
    omitDimension: List[int] = field(default_factory=list)
    buffer: Any = None
    tempBuffer: Any = None
    inputBuffer: Any = None
    outputBuffer: Any = None
    bufferOffset: int = 0
    tempBufferOffset: int = 0
    inputBufferOffset: int = 0
    outputBufferOffset: int = 0
    specifyOffsetsAtLaunch: int = 0
    bufferSize: int = 0
    tempBufferSize: int = 0
    # convolution / cross-correlation (API guide "Convolution parameters"): VkFFTAppend(app, -1) = FFT -> x kernel -> iFFT
    performConvolution: int = 0
    kernelConvolution: int = 0
    matrixConvolution: int = 0
    symmetricKernel: int = 0
    numberKernels: int = 0
    conjugateConvolution: int = 0
    crossPowerSpectrumNormalization: int = 0
    kernel: Any = None
    kernelOffset: int = 0
    # reference features outside the engine's scope: accepted here so that setting them fails like the C shim
    performZeropadding: List[int] = field(default_factory=list)
    fft_zeropad_left: List[int] = field(default_factory=list)
    fft_zeropad_right: List[int] = field(default_factory=list)
    frequencyZeroPadding: int = 0
    # engine extension (no reference counterpart, the reference is single-device): one sequence over peer windows,
    # see b200fft_desc.dist_world in include/b200fft.h and vkfft_b200/dist.py FusedDistributedFFT1D
    distWorld: int = 0
    distRank: int = 0


@dataclass
class VkFFTLaunchParams:
    buffer: Any = None
    tempBuffer: Any = None
    inputBuffer: Any = None
    outputBuffer: Any = None
    bufferOffset: int = 0
    tempBufferOffset: int = 0
    inputBufferOffset: int = 0
    outputBufferOffset: int = 0
    stream: Optional[int] = None
    kernel: Any = None
    kernelOffset: int = 0


class VkFFTApplication:
    """Zero-initialised application handle; initializeVkFFT fills it, deleteVkFFT zeroes it again."""

    def __init__(self):
        self.configuration = None
        self._plan = None

    def _is_zero(self):
        return self.configuration is None and self._plan is None


def _to_desc(cfg: VkFFTConfiguration) -> "_lib.b200fft_desc":
    d = _lib.b200fft_desc()
    d.struct_size = ctypes.sizeof(_lib.b200fft_desc)
    d.fft_dim = cfg.FFTdim
    for i, s in enumerate(cfg.size[:4]):
        d.size[i] = int(s)
    for name, dst in (("bufferStride", d.buffer_stride), ("inputBufferStride", d.input_stride),
                      ("outputBufferStride", d.output_stride), ("omitDimension", d.omit_dimension)):
        for i, s in enumerate(getattr(cfg, name)[:4]):
            dst[i] = int(s)
    d.number_batches = cfg.numberBatches
    d.coordinate_features = cfg.coordinateFeatures
    d.precision = 1 if cfg.doublePrecision else (3 if cfg.halfPrecisionMemoryOnly else (2 if cfg.halfPrecision else 0))
    d.perform_r2c = cfg.performR2C
    d.perform_dct = cfg.performDCT
    d.perform_dst = cfg.performDST
    d.normalize = cfg.normalize
    d.disable_reorder_four_step = cfg.disableReorderFourStep
    d.make_forward_plan_only = cfg.makeForwardPlanOnly
    d.make_inverse_plan_only = cfg.makeInversePlanOnly
    d.is_input_formatted = cfg.isInputFormatted
    d.is_output_formatted = cfg.isOutputFormatted
    d.inverse_return_to_input = cfg.inverseReturnToInputBuffer
    d.user_temp_buffer = cfg.userTempBuffer
    d.buffer_size = cfg.bufferSize
    d.temp_buffer_size = cfg.tempBufferSize
    d.device = int(cfg.device)
    d.stream = cfg.stream
    d.dist_world = cfg.distWorld
    d.dist_rank = cfg.distRank
    for i, v in enumerate(cfg.performZeropadding[:4]):
        d.perform_zeropadding[i] = int(v)
    for i, v in enumerate(cfg.fft_zeropad_left[:4]):
        d.zeropad_left[i] = int(v)
    for i, v in enumerate(cfg.fft_zeropad_right[:4]):
        d.zeropad_right[i] = int(v)
    d.frequency_zeropadding = cfg.frequencyZeroPadding
    d.perform_convolution = cfg.performConvolution
    d.kernel_convolution = cfg.kernelConvolution
    d.matrix_convolution = cfg.matrixConvolution
    d.symmetric_kernel = cfg.symmetricKernel
    d.number_kernels = cfg.numberKernels
    d.conjugate_convolution = cfg.conjugateConvolution
    d.cross_power_spectrum_normalization = cfg.crossPowerSpectrumNormalization
    return d


def initializeVkFFT(app: VkFFTApplication, inputLaunchConfiguration: VkFFTConfiguration) -> int:
    if app is None:
        return VKFFT_ERROR_EMPTY_app
    if not app._is_zero():
        return VKFFT_ERROR_NONZERO_APP_INITIALIZATION
    cfg = inputLaunchConfiguration
    if cfg.device is None:
        return VKFFT_ERROR_INVALID_DEVICE
    if cfg.FFTdim == 0:
        return VKFFT_ERROR_EMPTY_FFTdim
    if cfg.FFTdim > _lib.MAX_DIMS:
        return VKFFT_ERROR_FFTdim_GT_MAX_FFT_DIMENSIONS
    if not cfg.size or cfg.size[0] == 0:
        return VKFFT_ERROR_EMPTY_size
    if (cfg.halfPrecision or cfg.halfPrecisionMemoryOnly) and cfg.doublePrecision:
        return VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH
    L = _lib.load()
    d = _to_desc(cfg)
    plan = ctypes.c_void_p()
    rc = L.b200fft_plan_create(ctypes.byref(d), ctypes.byref(plan))
    if rc != VKFFT_SUCCESS:
        return rc
    app.configuration = cfg
    app._plan = plan
    return VKFFT_SUCCESS


def VkFFTAppend(app: VkFFTApplication, inverse: int, launchParams: Optional[VkFFTLaunchParams] = None) -> int:
    if app is None:
        return VKFFT_ERROR_EMPTY_app
    if app._plan is None:
        return VKFFT_ERROR_PLAN_NOT_INITIALIZED
    c = app.configuration
    lp = launchParams or VkFFTLaunchParams()
    b = _lib.b200fft_buffers()
    b.buffer = _ptr(lp.buffer if lp.buffer is not None else c.buffer)
    b.temp_buffer = _ptr(lp.tempBuffer if lp.tempBuffer is not None else c.tempBuffer)
    b.input_buffer = _ptr(lp.inputBuffer if lp.inputBuffer is not None else c.inputBuffer)
    b.output_buffer = _ptr(lp.outputBuffer if lp.outputBuffer is not None else c.outputBuffer)
    src = lp if c.specifyOffsetsAtLaunch else c
    b.buffer_offset = src.bufferOffset
    b.temp_buffer_offset = src.tempBufferOffset
    b.input_buffer_offset = src.inputBufferOffset
    b.output_buffer_offset = src.outputBufferOffset
    b.stream = lp.stream
    b.kernel = _ptr(lp.kernel if lp.kernel is not None else c.kernel)
    b.kernel_offset = src.kernelOffset
    return _lib.load().b200fft_exec(app._plan, int(inverse), ctypes.byref(b))


def deleteVkFFT(app: VkFFTApplication) -> None:
    if app is None:
        return
    if app._plan is not None:
        _lib.load().b200fft_plan_destroy(app._plan)
    app.configuration = None
    app._plan = None


def planInfo(app: VkFFTApplication) -> dict:
    """Engine-side facts about a plan (passes, scratch, algorithmic bytes/flops) -- used by bench.py."""
    info = _lib.b200fft_plan_info()
    rc = _lib.load().b200fft_plan_get_info(app._plan, ctypes.byref(info))
    if rc != 0:
        raise RuntimeError(getVkFFTErrorString(rc))
    out = {k: getattr(info, k) for k, _ in info._fields_}
    buf = ctypes.create_string_buffer(8192)
    _lib.load().b200fft_plan_describe(app._plan, -1, buf, len(buf))
    out["forward"] = buf.value.decode()
    _lib.load().b200fft_plan_describe(app._plan, 1, buf, len(buf))
    out["inverse"] = buf.value.decode()
    return out


def execHost(app: VkFFTApplication, inverse: int, host_in_ptr: int, host_out_ptr: int, nbytes_in: int,
             nbytes_out: int) -> int:
    """b200fft_exec_host: host buffer -> HBM -> transform -> host buffer (synchronous)."""
    return _lib.load().b200fft_exec_host(app._plan, int(inverse), host_in_ptr, host_out_ptr, nbytes_in, nbytes_out)
