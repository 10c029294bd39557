/* b200fft -- C ABI of the H100-native FFT engine (libb200fft.so).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference exposes the path as three
 * `static inline` functions in a header (everything else is reached through them):
 *     initializeVkFFT   vkFFT/vkFFT/vkFFT_AppManagement/vkFFT_InitializeApp.h:1468
 *     VkFFTAppend       vkFFT/vkFFT/vkFFT_AppManagement/vkFFT_RunApp.h:79
 *     deleteVkFFT       vkFFT/vkFFT/vkFFT_AppManagement/vkFFT_DeleteApp.h:28
 * include/vkFFT.h keeps those three names/structs (header-only, C or C++) and forwards to the entry points
 * below; foreign-language bindings (ctypes, cgo, JNI ...) bind the entry points below directly.
 *
 * Conventions kept from the reference (documentation/VkFFT_API_guide.tex:263-352):
 *   - forward transform uses exp(-2*pi*i*nk/N), inverse is unnormalised unless `normalize` is set;
 *   - data layout is WHDCN: size[0] is the fastest (contiguous) dimension, then size[1]..., then batches;
 *   - complex numbers are interleaved (re,im); R2C packs N/2+1 complex per row;
 *   - all functions return a VkFFTResult-compatible code (0 = VKFFT_SUCCESS), never throw, never abort.
 * Only plain C types cross this boundary: no CUDA, torch or C++ types in any signature.  Device pointers
 * and streams travel as void*.
 */
#ifndef B200FFT_H
#define B200FFT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200FFT_MAX_DIMS 4
#define B200FFT_VERSION 10000 /* engine version; VkFFTGetVersion() of the shim still reports 10304 */

/* B200FFT_F16: half-precision STORAGE -- every buffer holds 32-bit complex elements (half re, half im), arithmetic and tables are
   FP32 (the reference's halfPrecision, vkFFT_Structs.h:210; C2C transforms and even-length R2C / C2R, whose real rows hold half
   values, kernels instantiated at plan time) */
/* B200FFT_F16_IO: halfPrecisionMemoryOnly -- only the caller's inputBuffer (is_input_formatted = 1) is half: the forward transform
   reads it, the inverse transform (inverse_return_to_input = 1) writes it; buffer / tempBuffer / outputBuffer are FP32 */
typedef enum b200fft_precision { B200FFT_F32 = 0, B200FFT_F64 = 1, B200FFT_F16 = 2, B200FFT_F16_IO = 3 } b200fft_precision;

/* Plan description: the subset of VkFFTConfiguration (vkFFT_Structs.h:93-324) the hot path consumes.
 * Zero means "default" for every field, exactly like the reference's zero-initialised configuration. */
typedef struct b200fft_desc {
    uint32_t struct_size;                 /* = sizeof(b200fft_desc); lets the ABI grow */
    uint32_t fft_dim;                     /* FFTdim: 1..4 */
    uint64_t size[B200FFT_MAX_DIMS];      /* size[]: logical transform lengths, x first */
    uint64_t number_batches;              /* numberBatches (0 -> 1) */
    uint64_t coordinate_features;         /* coordinateFeatures (0 -> 1); treated as one more batch level */
    uint32_t precision;                   /* doublePrecision -> B200FFT_F64, halfPrecision -> B200FFT_F16 */
    uint32_t perform_r2c;                 /* performR2C */
    uint32_t perform_dct;                 /* performDCT: 1..4 */
    uint32_t perform_dst;                 /* performDST: 1..4 */
    uint32_t normalize;                   /* normalize */
    uint32_t disable_reorder_four_step;   /* disableReorderFourStep */
    uint32_t make_forward_plan_only;      /* makeForwardPlanOnly */
    uint32_t make_inverse_plan_only;      /* makeInversePlanOnly */
    uint32_t is_input_formatted;          /* isInputFormatted: read from `input` with input_stride */
    uint32_t is_output_formatted;         /* isOutputFormatted: write to `output` with output_stride */
    uint32_t inverse_return_to_input;     /* inverseReturnToInputBuffer */
    uint32_t user_temp_buffer;            /* userTempBuffer: caller supplies the temp buffer */
    uint64_t buffer_stride[B200FFT_MAX_DIMS];  /* bufferStride[] in elements (0 -> packed default) */
    uint64_t input_stride[B200FFT_MAX_DIMS];
    uint64_t output_stride[B200FFT_MAX_DIMS];
    uint32_t omit_dimension[B200FFT_MAX_DIMS]; /* omitDimension[] */
    uint64_t buffer_size;                 /* bytes; 0 = unknown (only used for validation) */
    uint64_t temp_buffer_size;            /* bytes of the user temp buffer when user_temp_buffer=1 */
    int32_t device;                       /* CUDA device ordinal (what *cfg.device holds for the runtime API) */
    uint32_t reserved0;
    void* stream;                         /* cudaStream_t or NULL for the default stream */
    /* One long 1-D C2C sequence spread over the GPUs of a box (no counterpart in the reference, which is single
     * device: README.md:26-28).  dist_world > 1: `buffer` and `temp_buffer` are the bases of two peer windows
     * (b200fft_window_*, below) holding the whole sequence, slab g on GPU g; this plan runs rank dist_rank's share
     * of every Four-Step launch and exchanges data through loads/stores to peer memory inside those launches. */
    uint32_t dist_world;
    uint32_t dist_rank;
    /* Convolution / cross-correlation (API guide "Convolution parameters", :1809-1852): one VkFFTAppend(app, -1) runs
     * forward transform -> product with the pre-transformed kernel -> inverse transform, result in `buffer`.
     * The kernel holds the natural-order spectrum a plan created with kernel_convolution=1 produces. */
    uint32_t perform_convolution;         /* performConvolution */
    uint32_t kernel_convolution;          /* kernelConvolution: this plan only transforms the kernel (plain forward plan) */
    uint32_t matrix_convolution;          /* matrixConvolution: 0/1 = per-feature product, 2 / 3 = matrix-vector product */
    uint32_t symmetric_kernel;            /* symmetricKernel: upper triangle stored (xx,xy,yy / xx,xy,xz,yy,yz,zz) */
    uint32_t number_kernels;              /* numberKernels: one input, this many outputs (0 -> 1) */
    uint32_t conjugate_convolution;       /* conjugateConvolution: 1 conjugates the sequence spectrum, 2 the kernel */
    uint32_t cross_power_spectrum_normalization; /* crossPowerSpectrumNormalization */
    uint32_t reserved1;
    uint64_t reserved[3];
    /* ---- fields added after the first release of the struct: only read when struct_size covers them ---- */
    /* Zero padding (API guide "Zero padding parameters", :1786-1807): elements [zeropad_left, zeropad_right) of every line along
     * a flagged axis count as zero on the first read of the forward transform (of the inverse one with frequency_zeropadding).
     * The engine clears those ranges in `buffer` with a streaming launch before the transform and then runs the ordinary
     * plan: same results as the reference, without its saving from skipped lines. */
    uint32_t perform_zeropadding[B200FFT_MAX_DIMS];   /* performZeropadding[] */
    uint64_t zeropad_left[B200FFT_MAX_DIMS];          /* fft_zeropad_left[] */
    uint64_t zeropad_right[B200FFT_MAX_DIMS];         /* fft_zeropad_right[] */
    uint32_t frequency_zeropadding;                   /* frequencyZeroPadding */
    uint32_t reserved2[3];
} b200fft_desc;

/* Buffers for one execution == VkFFTLaunchParams (vkFFT_Structs.h:326-379) with plain pointers.
 * All pointers are DEVICE pointers; offsets are in bytes like the reference's *BufferOffset fields. */
typedef struct b200fft_buffers {
    void* buffer;
    void* temp_buffer;     /* only when user_temp_buffer=1 */
    void* input_buffer;    /* only when is_input_formatted=1 */
    void* output_buffer;   /* only when is_output_formatted=1 */
    uint64_t buffer_offset, temp_buffer_offset, input_buffer_offset, output_buffer_offset;
    void* stream;          /* overrides desc.stream when non-NULL */
    void* kernel;          /* only when perform_convolution=1 */
    uint64_t kernel_offset;
} b200fft_buffers;

typedef struct b200fft_plan b200fft_plan; /* opaque */

/* Facts about a plan, for diagnostics / benchmarks (mirrors what printMemoryLayout prints, vkFFT_RunApp.h:58-78). */
typedef struct b200fft_plan_info {
    uint32_t num_passes_forward;    /* kernel launches per forward execution */
    uint32_t num_passes_inverse;
    uint64_t temp_bytes;            /* scratch this plan needs (engine-owned, or the minimum size of the caller's tempBuffer
                                       when user_temp_buffer = 1).  NOTE: it can exceed the size of `buffer` (Bluestein pads
                                       to M >= 2N-1 points per line, odd-length R2C and composed DCT/DST plans widen their
                                       lines): a caller-owned tempBuffer must be at least this large */
    uint64_t lut_bytes;             /* twiddle tables resident in HBM */
    uint64_t algorithmic_bytes;     /* 2 * sizeof(elem) * points * transformed axes, per direction */
    double flops;                   /* 5 N log2 N convention, per direction */
} b200fft_plan_info;

/* == initializeVkFFT.  Returns 0 or a VkFFTResult error code; *plan is NULL on failure. */
int b200fft_plan_create(const b200fft_desc* desc, b200fft_plan** plan);
/* == VkFFTAppend: enqueue the transform (inverse: -1 forward, +1 inverse) on the plan's stream. Asynchronous. */
int b200fft_exec(b200fft_plan* plan, int inverse, const b200fft_buffers* buffers);
/* == deleteVkFFT */
void b200fft_plan_destroy(b200fft_plan* plan);
int b200fft_plan_get_info(const b200fft_plan* plan, b200fft_plan_info* info);
/* kernel launches per axis of one direction == VkFFTPlan.numAxisUploads (vkFFT_Structs.h:1118-1130), which the reference's
 * benchmark samples read to convert time into "bandwidth" (sample_0_benchmark_VkFFT_single.cpp:234-237) */
int b200fft_plan_axis_uploads(const b200fft_plan* plan, int inverse, uint32_t uploads[B200FFT_MAX_DIMS]);
/* human-readable list of the plan's passes; returns bytes written (excluding NUL) */
size_t b200fft_plan_describe(const b200fft_plan* plan, int inverse, char* dst, size_t cap);

/* End-to-end convenience used by the benchmark's e2e leg and by language bindings without device memory
 * management: host buffer -> (pinned staging) -> HBM -> transform -> host buffer, synchronous.
 * `host_in`/`host_out` may alias. Byte counts must match the plan's buffer layout. */
int b200fft_exec_host(b200fft_plan* plan, int inverse, const void* host_in, void* host_out, uint64_t bytes_in,
                      uint64_t bytes_out);

/* page-locked host memory for b200fft_exec_host (NULL on failure) */
void* b200fft_host_alloc(uint64_t bytes);
void b200fft_host_free(void* p);

/* ---- peer windows: one flat virtual address range over every GPU's slab (multi-process, one process per GPU) --------
 * Each rank creates the window (allocates its own slab with the CUDA virtual memory API and reserves world*slab_bytes
 * of address space), exports two POSIX file descriptors (slab, signal pad), passes them to every peer (the host side
 * does that, e.g. over a unix socket with SCM_RIGHTS: vkfft_b200/window.py) and imports the peers' descriptors; after
 * that  base + g*slab_bytes  addresses GPU g's slab from every rank, over NVLink for g != rank.
 * slab_bytes must be a multiple of b200fft_window_granularity(device). */
typedef struct b200fft_window b200fft_window;
uint64_t b200fft_window_granularity(int device);
int b200fft_window_create(int device, uint32_t world, uint32_t rank, uint64_t slab_bytes, b200fft_window** window);
int b200fft_window_export(b200fft_window* window, int fds[2]);
int b200fft_window_import(b200fft_window* window, uint32_t peer, const int fds[2]);
void* b200fft_window_base(b200fft_window* window);      /* flat base: slab g at base + g*slab_bytes */
void* b200fft_window_local(b200fft_window* window);     /* == base + rank*slab_bytes */
/* device-side barrier over all ranks of the window, enqueued on `stream` (every rank must call it the same number
 * of times); a rank that waits longer than ~4 s gives up and b200fft_window_status() returns non-zero afterwards */
int b200fft_window_barrier(b200fft_window* window, void* stream);
int b200fft_window_status(b200fft_window* window);      /* synchronises the device; 0 = no barrier timed out */
void b200fft_window_destroy(b200fft_window* window);
/* a plan created with dist_world > 1 needs the window of its `buffer` for the barriers between its launches */
int b200fft_plan_attach_window(b200fft_plan* plan, b200fft_window* window);

const char* b200fft_error_string(int code);
int b200fft_version(void);
/* number of ahead-of-time compiled kernel instantiations in the library (0 would mean a broken build) */
int b200fft_kernel_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200FFT_H */
