/* vkFFT.h -- header-only drop-in for the CUDA backend (VKFFT_BACKEND==1) of DTolm/VkFFT, backed by the
 * H100-native engine in libb200fft.so.
 *
 * User code written against the reference keeps compiling unchanged:
 *
 *     VkFFTConfiguration cfg = {};  VkFFTApplication app = {};
 *     cfg.FFTdim = 1; cfg.size[0] = N; cfg.numberBatches = B; cfg.device = &cuDevice; cfg.buffer = &d_ptr;
 *     initializeVkFFT(&app, cfg);          // reference: vkFFT_InitializeApp.h:1468
 *     VkFFTAppend(&app, -1, &launchParams); // reference: vkFFT_RunApp.h:79   (-1 forward, +1 inverse)
 *     deleteVkFFT(&app);                   // reference: vkFFT_DeleteApp.h:28
 *
 * What changes underneath: no kernel text is generated; the three calls forward to the C ABI in b200fft.h (plain
 * pointers and sizes), which launches hand-written sm_90a kernels -- compiled ahead of time for the powers of two and the
 * curated lengths, instantiated from the same templates at plan time for other smooth lengths (csrc/jit.cpp).
 * VkFFTConfiguration / VkFFTLaunchParams keep the reference's member names, order and types for
 * VKFFT_BACKEND==1 (vkFFT_Structs.h:93-379) so that sizeof/offsetof agree with the reference build
 * (1168 and 80 bytes on x86-64; checked in tests/test_abi.py).  Members that configure the reference's
 * code generator are accepted and ignored; features outside the engine's scope return the reference's
 * VKFFT_ERROR_UNSUPPORTED_* codes instead of silently doing something else.
 *
 * Link with -lb200fft (and the CUDA driver/runtime the application already uses).
 */
#ifndef VKFFT_H
#define VKFFT_H

#include <inttypes.h>
#include <stdlib.h>
#include <string.h>

#ifndef VKFFT_BACKEND
#define VKFFT_BACKEND 1
#endif
#if (VKFFT_BACKEND != 1)
#error "this vkFFT.h only provides the CUDA backend (VKFFT_BACKEND==1)"
#endif

#include <cuda.h>
#include <cuda_runtime_api.h>

#include "b200fft.h"

#ifdef __cplusplus
#define VKFFT_ZERO_INIT {}
#else
#define VKFFT_ZERO_INIT {0}
#endif

#ifndef VKFFT_MAX_FFT_DIMENSIONS
#define VKFFT_MAX_FFT_DIMENSIONS 4
#endif
#if (VKFFT_MAX_FFT_DIMENSIONS != 4)
#error "the engine is built for VKFFT_MAX_FFT_DIMENSIONS == 4"
#endif

#define pfLD long double
#define pfUINT uint64_t
#define pfINT int64_t

/* ---- plan-time parameters (member list == reference, CUDA backend) ------------------------------------ */
typedef struct {
    pfUINT FFTdim;
    pfUINT size[VKFFT_MAX_FFT_DIMENSIONS];
    CUdevice* device;
    cudaStream_t* stream;
    pfUINT num_streams;

    pfUINT userTempBuffer;
    pfUINT bufferNum, tempBufferNum, inputBufferNum, outputBufferNum, kernelNum;
    pfUINT *bufferSize, *tempBufferSize, *inputBufferSize, *outputBufferSize, *kernelSize;
    void **buffer, **tempBuffer, **inputBuffer, **outputBuffer, **kernel;
    pfUINT bufferOffset, tempBufferOffset, inputBufferOffset, outputBufferOffset, kernelOffset;
    pfUINT specifyOffsetsAtLaunch;

    pfUINT coalescedMemory, aimThreads, numSharedBanks;      /* code-generator hints: ignored */
    pfUINT inverseReturnToInputBuffer;
    pfUINT numberBatches;
    pfUINT useUint64;
    pfUINT omitDimension[VKFFT_MAX_FFT_DIMENSIONS];
    int performBandwidthBoost;
    pfUINT groupedBatch[VKFFT_MAX_FFT_DIMENSIONS];

    pfUINT doublePrecision;
    pfUINT quadDoubleDoublePrecision, quadDoubleDoublePrecisionDoubleMemory;   /* unsupported */
    pfUINT halfPrecision;                                       /* half storage, FP32 arithmetic: C2C and even-length R2C */
    pfUINT halfPrecisionMemoryOnly;                             /* half inputBuffer (isInputFormatted), FP32 everywhere else */
    pfUINT doublePrecisionFloatMemory;                          /* unsupported */

    pfUINT performR2C, performDCT, performDST;
    pfUINT disableMergeSequencesR2C, forceCallbackVersionRealTransforms;

    pfUINT normalize;
    pfUINT disableReorderFourStep;
    pfINT useLUT, useLUT_4step;                               /* the engine always uses exact tables */
    pfUINT makeForwardPlanOnly, makeInversePlanOnly;

    pfUINT bufferStride[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT isInputFormatted, isOutputFormatted;
    pfUINT inputBufferStride[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT outputBufferStride[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT swapTo2Stage4Step, swapTo3Stage4Step;

    pfUINT considerAllAxesStrided, keepShaderCode, printMemoryLayout;
    pfUINT saveApplicationToString, loadApplicationFromString;
    void* loadApplicationString;
    pfUINT disableSetLocale;

    pfUINT fixMaxRadixBluestein, forceBluesteinSequenceSize, useCustomBluesteinPaddingPattern;
    pfUINT *primeSizes, *paddedSizes;
    pfUINT fixMinRaderPrimeMult, fixMaxRaderPrimeMult, fixMinRaderPrimeFFT, fixMaxRaderPrimeFFT;

    pfUINT performZeropadding[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT fft_zeropad_left[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT fft_zeropad_right[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT frequencyZeroPadding;

    pfUINT performConvolution, conjugateConvolution, crossPowerSpectrumNormalization;
    pfUINT coordinateFeatures, matrixConvolution, symmetricKernel, numberKernels, kernelConvolution;

    pfUINT registerBoost, registerBoostNonPow2, registerBoost4Step;
    pfUINT devicePageSize, localPageSize;

    /* filled in by initializeVkFFT in the reference; reported here for the GPU the plan was made on */
    pfUINT computeCapabilityMajor, computeCapabilityMinor;
    pfUINT maxComputeWorkGroupCount[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT maxComputeWorkGroupSize[VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT maxThreadsNum, sharedMemorySizeStatic, sharedMemorySize, sharedMemorySizePow2, warpSize, halfThreads;
    pfUINT allocateTempBuffer;
    pfUINT reorderFourStep;
    pfINT maxCodeLength, maxTempLength;
    pfUINT autoCustomBluesteinPaddingPattern, useRaderUintLUT, vendorID;
    cudaEvent_t* stream_event;
    pfUINT streamCounter, streamID;
} VkFFTConfiguration;

/* ---- launch-time parameters ------------------------------------------------------------------------------ */
typedef struct {
    void **buffer, **tempBuffer, **inputBuffer, **outputBuffer, **kernel;
    pfUINT bufferOffset, tempBufferOffset, inputBufferOffset, outputBufferOffset, kernelOffset;
} VkFFTLaunchParams;

/* ---- result codes: same numeric values as the reference (vkFFT_Structs.h:380-477) ------------------------ */
typedef enum VkFFTResult {
    VKFFT_SUCCESS = 0,
    VKFFT_ERROR_MALLOC_FAILED = 1,
    VKFFT_ERROR_INSUFFICIENT_CODE_BUFFER = 2,
    VKFFT_ERROR_INSUFFICIENT_TEMP_BUFFER = 3,
    VKFFT_ERROR_PLAN_NOT_INITIALIZED = 4,
    VKFFT_ERROR_NULL_TEMP_PASSED = 5,
    VKFFT_ERROR_MATH_FAILED = 6,
    VKFFT_ERROR_FFTdim_GT_MAX_FFT_DIMENSIONS = 7,
    VKFFT_ERROR_NONZERO_APP_INITIALIZATION = 8,
    VKFFT_ERROR_INVALID_PHYSICAL_DEVICE = 1001,
    VKFFT_ERROR_INVALID_DEVICE = 1002,
    VKFFT_ERROR_INVALID_QUEUE = 1003,
    VKFFT_ERROR_INVALID_COMMAND_POOL = 1004,
    VKFFT_ERROR_INVALID_FENCE = 1005,
    VKFFT_ERROR_ONLY_FORWARD_FFT_INITIALIZED = 1006,
    VKFFT_ERROR_ONLY_INVERSE_FFT_INITIALIZED = 1007,
    VKFFT_ERROR_INVALID_CONTEXT = 1008,
    VKFFT_ERROR_INVALID_PLATFORM = 1009,
    VKFFT_ERROR_ENABLED_saveApplicationToString = 1010,
    VKFFT_ERROR_EMPTY_FILE = 1011,
    VKFFT_ERROR_EMPTY_FFTdim = 2001,
    VKFFT_ERROR_EMPTY_size = 2002,
    VKFFT_ERROR_EMPTY_bufferSize = 2003,
    VKFFT_ERROR_EMPTY_buffer = 2004,
    VKFFT_ERROR_EMPTY_tempBufferSize = 2005,
    VKFFT_ERROR_EMPTY_tempBuffer = 2006,
    VKFFT_ERROR_EMPTY_inputBufferSize = 2007,
    VKFFT_ERROR_EMPTY_inputBuffer = 2008,
    VKFFT_ERROR_EMPTY_outputBufferSize = 2009,
    VKFFT_ERROR_EMPTY_outputBuffer = 2010,
    VKFFT_ERROR_EMPTY_kernelSize = 2011,
    VKFFT_ERROR_EMPTY_kernel = 2012,
    VKFFT_ERROR_EMPTY_applicationString = 2013,
    VKFFT_ERROR_EMPTY_useCustomBluesteinPaddingPattern_arrays = 2014,
    VKFFT_ERROR_EMPTY_app = 2015,
    VKFFT_ERROR_INVALID_user_tempBuffer_too_small = 2016,
    VKFFT_ERROR_UNSUPPORTED_RADIX = 3001,
    VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH = 3002,
    VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2C = 3003,
    VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH_R2R = 3004,
    VKFFT_ERROR_UNSUPPORTED_FFT_OMIT = 3005,
    VKFFT_ERROR_FAILED_TO_ALLOCATE = 4001,
    /* 4002-4027, 4030-4034: codes of the other backends; never returned here, present so that code switching on them compiles */
    VKFFT_ERROR_FAILED_TO_MAP_MEMORY = 4002, VKFFT_ERROR_FAILED_TO_ALLOCATE_COMMAND_BUFFERS = 4003,
    VKFFT_ERROR_FAILED_TO_BEGIN_COMMAND_BUFFER = 4004, VKFFT_ERROR_FAILED_TO_END_COMMAND_BUFFER = 4005,
    VKFFT_ERROR_FAILED_TO_SUBMIT_QUEUE = 4006, VKFFT_ERROR_FAILED_TO_WAIT_FOR_FENCES = 4007,
    VKFFT_ERROR_FAILED_TO_RESET_FENCES = 4008, VKFFT_ERROR_FAILED_TO_CREATE_DESCRIPTOR_POOL = 4009,
    VKFFT_ERROR_FAILED_TO_CREATE_DESCRIPTOR_SET_LAYOUT = 4010, VKFFT_ERROR_FAILED_TO_ALLOCATE_DESCRIPTOR_SETS = 4011,
    VKFFT_ERROR_FAILED_TO_CREATE_PIPELINE_LAYOUT = 4012, VKFFT_ERROR_FAILED_SHADER_PREPROCESS = 4013,
    VKFFT_ERROR_FAILED_SHADER_PARSE = 4014, VKFFT_ERROR_FAILED_SHADER_LINK = 4015, VKFFT_ERROR_FAILED_SPIRV_GENERATE = 4016,
    VKFFT_ERROR_FAILED_TO_CREATE_SHADER_MODULE = 4017, VKFFT_ERROR_FAILED_TO_CREATE_INSTANCE = 4018,
    VKFFT_ERROR_FAILED_TO_SETUP_DEBUG_MESSENGER = 4019, VKFFT_ERROR_FAILED_TO_FIND_PHYSICAL_DEVICE = 4020,
    VKFFT_ERROR_FAILED_TO_CREATE_DEVICE = 4021, VKFFT_ERROR_FAILED_TO_CREATE_FENCE = 4022,
    VKFFT_ERROR_FAILED_TO_CREATE_COMMAND_POOL = 4023, VKFFT_ERROR_FAILED_TO_CREATE_BUFFER = 4024,
    VKFFT_ERROR_FAILED_TO_ALLOCATE_MEMORY = 4025, VKFFT_ERROR_FAILED_TO_BIND_BUFFER_MEMORY = 4026,
    VKFFT_ERROR_FAILED_TO_FIND_MEMORY = 4027,
    VKFFT_ERROR_FAILED_TO_SYNCHRONIZE = 4028,
    VKFFT_ERROR_FAILED_TO_COPY = 4029,
    VKFFT_ERROR_FAILED_TO_CREATE_PROGRAM = 4030, VKFFT_ERROR_FAILED_TO_COMPILE_PROGRAM = 4031,
    VKFFT_ERROR_FAILED_TO_GET_CODE_SIZE = 4032, VKFFT_ERROR_FAILED_TO_GET_CODE = 4033, VKFFT_ERROR_FAILED_TO_DESTROY_PROGRAM = 4034,
    VKFFT_ERROR_FAILED_TO_LOAD_MODULE = 4035,
    VKFFT_ERROR_FAILED_TO_GET_FUNCTION = 4036,
    VKFFT_ERROR_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY = 4037,
    VKFFT_ERROR_FAILED_TO_MODULE_GET_GLOBAL = 4038,
    VKFFT_ERROR_FAILED_TO_LAUNCH_KERNEL = 4039,
    VKFFT_ERROR_FAILED_TO_EVENT_RECORD = 4040,
    VKFFT_ERROR_FAILED_TO_ADD_NAME_EXPRESSION = 4041, VKFFT_ERROR_FAILED_TO_INITIALIZE = 4042,
    VKFFT_ERROR_FAILED_TO_SET_DEVICE_ID = 4043, VKFFT_ERROR_FAILED_TO_GET_DEVICE = 4044,
    VKFFT_ERROR_FAILED_TO_CREATE_CONTEXT = 4045, VKFFT_ERROR_FAILED_TO_CREATE_PIPELINE = 4046,
    VKFFT_ERROR_FAILED_TO_SET_KERNEL_ARG = 4047, VKFFT_ERROR_FAILED_TO_CREATE_COMMAND_QUEUE = 4048,
    VKFFT_ERROR_FAILED_TO_RELEASE_COMMAND_QUEUE = 4049, VKFFT_ERROR_FAILED_TO_ENUMERATE_DEVICES = 4050,
    VKFFT_ERROR_FAILED_TO_GET_ATTRIBUTE = 4051,
    VKFFT_ERROR_FAILED_TO_CREATE_EVENT = 4052,
    VKFFT_ERROR_FAILED_TO_CREATE_COMMAND_LIST = 4053, VKFFT_ERROR_FAILED_TO_DESTROY_COMMAND_LIST = 4054,
    VKFFT_ERROR_FAILED_TO_SUBMIT_BARRIER = 4055
} VkFFTResult;

static inline const char* getVkFFTErrorString(VkFFTResult result) { return b200fft_error_string((int)result); }

/* ---- application handle ---------------------------------------------------------------------------------- */
/* What callers read from the reference's VkFFTPlan (vkFFT_Structs.h:1118-1130): how many launches each axis takes.  The
 * reference's own benchmark samples use it to turn time into "bandwidth" (sample_0_benchmark_VkFFT_single.cpp:234-237). */
typedef struct {
    pfUINT actualFFTSizePerAxis[VKFFT_MAX_FFT_DIMENSIONS][VKFFT_MAX_FFT_DIMENSIONS];
    pfUINT numAxisUploads[VKFFT_MAX_FFT_DIMENSIONS];
} VkFFTPlan;

typedef struct {
    VkFFTConfiguration configuration;   /* normalised copy of what the caller passed (as in the reference) */
    VkFFTPlan* localFFTPlan;            /* forward / inverse launch counts (allocated by initializeVkFFT) */
    VkFFTPlan* localFFTPlan_inverse;
    b200fft_plan* b200fftPlan;          /* the engine's plan: owns tables, scratch, kernel selection */
    pfUINT actualNumBatches;
    pfUINT applicationStringSize;       /* saveApplicationToString: opaque blob, nothing to cache (no JIT) */
    void* saveApplicationString;
} VkFFTApplication;

static inline int VkFFTGetVersion(void) { return 10304; /* API level of the reference this header mirrors */ }

static inline void deleteVkFFT(VkFFTApplication* app) {
    if (!app) return;
    if (app->b200fftPlan) b200fft_plan_destroy(app->b200fftPlan);
    if (app->configuration.stream_event) {       /* num_streams > 1: the events that order the streams (below) */
        for (pfUINT s_ = 0; s_ < app->configuration.num_streams; s_++)
            if (app->configuration.stream_event[s_]) cudaEventDestroy(app->configuration.stream_event[s_]);
        free(app->configuration.stream_event);
    }
    if (app->saveApplicationString) free(app->saveApplicationString);
    if (app->localFFTPlan) free(app->localFFTPlan);
    if (app->localFFTPlan_inverse) free(app->localFFTPlan_inverse);
    memset(app, 0, sizeof(VkFFTApplication));
}

static inline VkFFTResult initializeVkFFT(VkFFTApplication* app, VkFFTConfiguration inputLaunchConfiguration) {
    if (app == 0) return VKFFT_ERROR_EMPTY_app;
    {   /* the reference insists on a zero-initialised application (vkFFT_InitializeApp.h:1471-1477) */
        static const VkFFTApplication zeroApp = VKFFT_ZERO_INIT;
        if (memcmp(app, &zeroApp, sizeof(VkFFTApplication)) != 0) return VKFFT_ERROR_NONZERO_APP_INITIALIZATION;
    }
    const VkFFTConfiguration* c = &inputLaunchConfiguration;
    if (c->device == 0) return VKFFT_ERROR_INVALID_DEVICE;
    if (c->FFTdim == 0) return VKFFT_ERROR_EMPTY_FFTdim;
    if (c->FFTdim > VKFFT_MAX_FFT_DIMENSIONS) return VKFFT_ERROR_FFTdim_GT_MAX_FFT_DIMENSIONS;
    if (c->size[0] == 0) return VKFFT_ERROR_EMPTY_size;
    /* features of the reference outside this engine's hot path */
    if (c->quadDoubleDoublePrecision || c->quadDoubleDoublePrecisionDoubleMemory || c->doublePrecisionFloatMemory ||
        ((c->halfPrecision || c->halfPrecisionMemoryOnly) && c->doublePrecision))
        return VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH;
    if (c->bufferNum > 1 || c->tempBufferNum > 1 || c->inputBufferNum > 1 || c->outputBufferNum > 1)
        return VKFFT_ERROR_UNSUPPORTED_FFT_LENGTH;
    if (c->loadApplicationFromString && c->saveApplicationToString) return VKFFT_ERROR_ENABLED_saveApplicationToString;
    if (c->loadApplicationFromString && c->loadApplicationString == 0) return VKFFT_ERROR_EMPTY_applicationString;

    b200fft_desc d;
    memset(&d, 0, sizeof d);
    d.struct_size = (uint32_t)sizeof d;
    d.fft_dim = (uint32_t)c->FFTdim;
    for (int i = 0; i < VKFFT_MAX_FFT_DIMENSIONS; i++) {
        d.size[i] = c->size[i];
        d.buffer_stride[i] = c->bufferStride[i];
        d.input_stride[i] = c->inputBufferStride[i];
        d.output_stride[i] = c->outputBufferStride[i];
        d.omit_dimension[i] = (uint32_t)c->omitDimension[i];
        d.perform_zeropadding[i] = (uint32_t)c->performZeropadding[i];
        d.zeropad_left[i] = c->fft_zeropad_left[i];
        d.zeropad_right[i] = c->fft_zeropad_right[i];
    }
    d.frequency_zeropadding = (uint32_t)c->frequencyZeroPadding;
    d.number_batches = c->numberBatches;
    d.coordinate_features = c->coordinateFeatures;
    /* halfPrecision (vkFFT_Structs.h:210): every buffer holds half-precision complex elements, arithmetic in FP32 -- B200FFT_F16 */
    /* halfPrecisionMemoryOnly (:211): half only in the caller's formatted inputBuffer (forward reads it, the inverse returns to it) */
    d.precision = c->doublePrecision ? B200FFT_F64 : (c->halfPrecisionMemoryOnly ? B200FFT_F16_IO : (c->halfPrecision ? B200FFT_F16 : B200FFT_F32));
    d.perform_r2c = (uint32_t)c->performR2C;
    d.perform_dct = (uint32_t)c->performDCT;
    d.perform_dst = (uint32_t)c->performDST;
    d.normalize = (uint32_t)c->normalize;
    d.disable_reorder_four_step = (uint32_t)c->disableReorderFourStep;
    d.make_forward_plan_only = (uint32_t)c->makeForwardPlanOnly;
    d.make_inverse_plan_only = (uint32_t)c->makeInversePlanOnly;
    d.is_input_formatted = (uint32_t)c->isInputFormatted;
    d.is_output_formatted = (uint32_t)c->isOutputFormatted;
    d.inverse_return_to_input = (uint32_t)c->inverseReturnToInputBuffer;
    d.user_temp_buffer = (uint32_t)c->userTempBuffer;
    d.perform_convolution = (uint32_t)c->performConvolution;
    d.kernel_convolution = (uint32_t)c->kernelConvolution;
    d.matrix_convolution = (uint32_t)c->matrixConvolution;
    d.symmetric_kernel = (uint32_t)c->symmetricKernel;
    d.number_kernels = (uint32_t)c->numberKernels;
    d.conjugate_convolution = (uint32_t)c->conjugateConvolution;
    d.cross_power_spectrum_normalization = (uint32_t)c->crossPowerSpectrumNormalization;
    if (c->bufferSize) d.buffer_size = c->bufferSize[0];
    if (c->userTempBuffer && c->tempBufferSize) d.temp_buffer_size = c->tempBufferSize[0];
    {   /* CUdevice handle -> runtime ordinal */
        int ndev = 0, found = -1;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess) return VKFFT_ERROR_INVALID_DEVICE;
        for (int i = 0; i < ndev && found < 0; i++) {
            CUdevice h;
            if (cuDeviceGet(&h, i) == CUDA_SUCCESS && h == *c->device) found = i;
        }
        if (found < 0) return VKFFT_ERROR_INVALID_DEVICE;
        d.device = found;
    }
    d.stream = (c->stream && c->num_streams > 0) ? (void*)c->stream[0] : 0;

    b200fft_plan* plan = 0;
    int rc = b200fft_plan_create(&d, &plan);
    if (rc != 0) { memset(app, 0, sizeof(VkFFTApplication)); return (VkFFTResult)rc; }
    app->configuration = inputLaunchConfiguration;
    if (app->configuration.numberBatches == 0) app->configuration.numberBatches = 1;
    if (app->configuration.coordinateFeatures == 0) app->configuration.coordinateFeatures = 1;
    app->configuration.reorderFourStep = c->disableReorderFourStep ? 0 : 1;
    app->configuration.warpSize = 32;
    app->configuration.vendorID = 0x10DE;
    app->actualNumBatches = app->configuration.numberBatches;
    app->b200fftPlan = plan;
    app->configuration.stream_event = 0;
    if (c->stream && c->num_streams > 1) {
        /* Several streams (vkFFT_DispatchPlan.h:218-225: the reference deals split dispatches round-robin over them and
           records one event per stream).  The launches of one transform depend on each other, so they all go to stream[0];
           the events make that equivalent for the caller: stream[0] first waits for everything already enqueued on the
           other streams, and afterwards every other stream waits for the transform. */
        app->configuration.stream_event = (cudaEvent_t*)calloc(c->num_streams, sizeof(cudaEvent_t));
        if (!app->configuration.stream_event) { deleteVkFFT(app); return VKFFT_ERROR_MALLOC_FAILED; }
        for (pfUINT s_ = 0; s_ < c->num_streams; s_++)
            if (cudaEventCreateWithFlags(&app->configuration.stream_event[s_], cudaEventDisableTiming) != cudaSuccess) {
                deleteVkFFT(app);
                return VKFFT_ERROR_FAILED_TO_CREATE_EVENT;
            }
    }
    for (int dir = 0; dir < 2; dir++) {
        VkFFTPlan* pl = (VkFFTPlan*)calloc(1, sizeof(VkFFTPlan));
        if (!pl) { deleteVkFFT(app); return VKFFT_ERROR_MALLOC_FAILED; }
        uint32_t up[B200FFT_MAX_DIMS] = {0, 0, 0, 0};
        b200fft_plan_axis_uploads(plan, dir ? 1 : -1, up);
        for (int a = 0; a < VKFFT_MAX_FFT_DIMENSIONS; a++) {
            pl->numAxisUploads[a] = up[a];
            for (int b = 0; b < VKFFT_MAX_FFT_DIMENSIONS; b++) pl->actualFFTSizePerAxis[a][b] = c->size[b] ? c->size[b] : 1;
        }
        if (dir) app->localFFTPlan_inverse = pl; else app->localFFTPlan = pl;
    }
    if (c->saveApplicationToString) {   /* the plan holds no generated binary worth saving, so the "binary" is a tag */
        static const char tag[] = "b200fft:aot:sm_90a";
        app->saveApplicationString = malloc(sizeof tag);
        if (!app->saveApplicationString) { deleteVkFFT(app); return VKFFT_ERROR_MALLOC_FAILED; }
        memcpy(app->saveApplicationString, tag, sizeof tag);
        app->applicationStringSize = sizeof tag;
    }
    return VKFFT_SUCCESS;
}

/* inverse: -1 forward, +1 inverse.  Asynchronous: only enqueues work on the plan's stream. */
static inline VkFFTResult VkFFTAppend(VkFFTApplication* app, int inverse, VkFFTLaunchParams* launchParams) {
    if (app == 0) return VKFFT_ERROR_EMPTY_app;
    if (app->b200fftPlan == 0) return VKFFT_ERROR_PLAN_NOT_INITIALIZED;
    const VkFFTConfiguration* c = &app->configuration;
    b200fft_buffers b;
    memset(&b, 0, sizeof b);
    /* launch-time buffers override plan-time ones (vkFFT_UpdateBuffers.h:628-775) */
    void** buf = (launchParams && launchParams->buffer) ? launchParams->buffer : c->buffer;
    void** tmp = (launchParams && launchParams->tempBuffer) ? launchParams->tempBuffer : c->tempBuffer;
    void** inb = (launchParams && launchParams->inputBuffer) ? launchParams->inputBuffer : c->inputBuffer;
    void** oub = (launchParams && launchParams->outputBuffer) ? launchParams->outputBuffer : c->outputBuffer;
    void** ker = (launchParams && launchParams->kernel) ? launchParams->kernel : c->kernel;
    b.kernel = ker ? *ker : 0;
    b.buffer = buf ? *buf : 0;
    b.temp_buffer = tmp ? *tmp : 0;
    b.input_buffer = inb ? *inb : 0;
    b.output_buffer = oub ? *oub : 0;
    if (c->specifyOffsetsAtLaunch && launchParams) {
        b.buffer_offset = launchParams->bufferOffset; b.temp_buffer_offset = launchParams->tempBufferOffset;
        b.input_buffer_offset = launchParams->inputBufferOffset; b.output_buffer_offset = launchParams->outputBufferOffset;
        b.kernel_offset = launchParams->kernelOffset;
    } else {
        b.kernel_offset = c->kernelOffset;
        b.buffer_offset = c->bufferOffset; b.temp_buffer_offset = c->tempBufferOffset;
        b.input_buffer_offset = c->inputBufferOffset; b.output_buffer_offset = c->outputBufferOffset;
    }
    if (c->stream_event && c->stream) {
        for (pfUINT s_ = 1; s_ < c->num_streams; s_++) {
            if (cudaEventRecord(c->stream_event[s_], c->stream[s_]) != cudaSuccess) return VKFFT_ERROR_FAILED_TO_EVENT_RECORD;
            if (cudaStreamWaitEvent(c->stream[0], c->stream_event[s_], 0) != cudaSuccess) return VKFFT_ERROR_FAILED_TO_SYNCHRONIZE;
        }
    }
    VkFFTResult res_ = (VkFFTResult)b200fft_exec(app->b200fftPlan, inverse, &b);
    if (res_ == VKFFT_SUCCESS && c->stream_event && c->stream) {
        if (cudaEventRecord(c->stream_event[0], c->stream[0]) != cudaSuccess) return VKFFT_ERROR_FAILED_TO_EVENT_RECORD;
        for (pfUINT s_ = 1; s_ < c->num_streams; s_++)
            if (cudaStreamWaitEvent(c->stream[s_], c->stream_event[0], 0) != cudaSuccess) return VKFFT_ERROR_FAILED_TO_SYNCHRONIZE;
        app->configuration.streamCounter++;
    }
    return res_;
}

#endif /* VKFFT_H */
