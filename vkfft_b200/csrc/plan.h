// Host-side plan graph: what initializeVkFFT builds in the reference through VkFFTScheduler
// (vkFFT_Scheduler.h:2223) + VkFFTPlanAxis (vkFFT_Plan_FFT.h:33), minus all code generation:
// here a plan is an ordered list of launches of ahead-of-time compiled kernels plus the twiddle
// tables they need.  Pure host C++ (no CUDA calls) so the CPU tests can execute a plan on the
// kernel-body emulation.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/b200fft.h"
#include "kernel_registry.h"
#include "pass_params.h"

namespace b200fft {

// VkFFTResult values used by the engine (vkFFT_Structs.h:380-477)
enum {
    R_SUCCESS = 0,
    R_MALLOC_FAILED = 1,
    R_PLAN_NOT_INITIALIZED = 4,
    R_NULL_TEMP_PASSED = 5,
    R_FFTDIM_GT_MAX = 7,
    R_INVALID_DEVICE = 1002,
    R_ONLY_FORWARD = 1006,
    R_ONLY_INVERSE = 1007,
    R_EMPTY_FFTDIM = 2001,
    R_EMPTY_SIZE = 2002,
    R_EMPTY_BUFFER = 2004,
    R_EMPTY_TEMPBUFFER = 2006,
    R_EMPTY_INPUTBUFFER = 2008,
    R_EMPTY_OUTPUTBUFFER = 2010,
    R_EMPTY_KERNEL = 2012,
    R_EMPTY_APP = 2015,
    R_USER_TEMP_TOO_SMALL = 2016,
    R_UNSUPPORTED_RADIX = 3001,
    R_UNSUPPORTED_FFT_LENGTH = 3002,
    R_UNSUPPORTED_FFT_LENGTH_R2C = 3003,
    R_UNSUPPORTED_FFT_LENGTH_R2R = 3004,
    R_UNSUPPORTED_FFT_OMIT = 3005,
    R_FAILED_TO_ALLOCATE = 4001,
    R_FAILED_TO_SYNCHRONIZE = 4028,
    R_FAILED_TO_COPY = 4029,
    R_FAILED_TO_SET_DYNAMIC_SHARED_MEMORY = 4037,
    R_FAILED_TO_LAUNCH_KERNEL = 4039,
};

enum BufRole { ROLE_BUFFER = 0, ROLE_TEMP = 1, ROLE_INPUT = 2, ROLE_OUTPUT = 3, ROLE_KERNEL = 4, ROLE_COUNT = 5 };

struct LutSpec {       // stage twiddles of one kernel schedule
    int prec;
    std::vector<int> radices;
};
struct TwSpec {        // two-level four-step table for modulus M
    int prec;
    uint64_t M;
};

struct AuxSpec {       // operator tables (lut.h make_aux)
    int prec, kind;
    uint64_t a, b;
};

struct PassPlan {
    const b2_kernel_info* k = nullptr;
    const b2_kernel_info* k_unaligned = nullptr;   // used instead of a pipelined kernel when the input is not 16-byte aligned
    b2_pass_params P{};          // pointer members are filled in by the runtime at launch
    unsigned grid = 0;
    int in_role = ROLE_BUFFER, out_role = ROLE_BUFFER;
    int64_t in_off = 0, out_off = 0;   // complex-element offsets added to the role's base pointer
    int lut_id = -1;
    int lut_id_unaligned = -1;   // stage twiddles of k_unaligned (its radix schedule may differ)
    int tw_id = -1;
    int aux0_id = -1, aux1_id = -1;
    int aux0_role = -1;          // >= 0: aux0 is a caller buffer (the convolution kernel), not a plan-owned table
    bool sync_before = false;    // distributed plans: barrier over all ranks of the window before this launch
    bool in_scalar = false, out_scalar = false;   // offsets (and strides) of that side count scalars, not complex elements
    // fused Four-Step (fused4.cuh): this launch and the NEXT one of the list run as one persistent kernel; the two
    // PassPlans stay in the list (the second is skipped at run time) so that un-fusing is a matter of clearing the pointer
    const b2_fused_info* fused = nullptr;
    uint32_t fz_nseq = 0, fz_U = 0, fz_NU = 0, fz_R = 0, fz_TA = 0, fz_TB = 0, fz_L = 1;
    int lut_id_plain = -1;       // stage tables of the stand-alone kernel `k` when lut_id belongs to the fused pair
    // cluster Four-Step (cluster4.cuh): this launch and the NEXT one run as one launch of thread-block clusters, one per
    // sequence (same stage tables as the two stand-alone kernels; both PassPlans stay in the list as for `fused`)
    const b2_cluster_info* cluster = nullptr;
    uint32_t cl_nseq = 0;
    std::string note;            // human readable (plan_describe)
};

struct PlanGraph {
    b200fft_desc desc{};         // normalised copy (defaults filled in)
    int prec = 0;
    uint64_t stride[B200FFT_MAX_DIMS] = {0, 0, 0, 0};      // buffer strides in elements
    uint64_t batches = 1;        // numberBatches * coordinateFeatures
    uint64_t batch_stride = 0;
    uint64_t total_elems = 0;    // logical complex points of one execution
    uint64_t temp_elems = 0;     // scratch the engine needs (complex elements)
    bool has_fwd = false, has_inv = false;
    std::vector<PassPlan> fwd, inv;
    std::vector<LutSpec> luts;
    std::vector<TwSpec> tws;
    std::vector<AuxSpec> auxs;
    uint64_t temp_elems_real = 0;   // (unused placeholder for real-sized scratch accounting)
    double flops = 0;
    uint64_t algorithmic_bytes = 0;
    uint32_t axis_uploads[2][B200FFT_MAX_DIMS] = {{0, 0, 0, 0}, {0, 0, 0, 0}};   // launches per axis, [0] forward / [1] inverse (the reference's numAxisUploads)
    int skip_axis = -1;          // convolution plans: this axis is transformed by the fused kernel, the direction planners leave it out
    int conv_axis = -1;          // DCT / DST convolution: plan_direction_dct plans only this axis, as the fused convolution launch
    uint64_t ctl_words = 0;      // control block of the fused Four-Step launches (largest one of the plan)
    // half-precision storage (desc.precision = B200FFT_F16: the reference's halfPrecision, vkFFT_Structs.h:210): arithmetic, tables
    // and g.prec are FP32, the elements of the flagged buffer roles are 32-bit (half re, half im); strides / offsets count elements
    bool role_half[ROLE_COUNT] = {false, false, false, false, false};
    bool distributed = false;    // desc.dist_world > 1: one more barrier follows the last launch of a direction
};

// Build the plan graph for `d`.  Returns a VkFFTResult-compatible code.
int build_plan(const b200fft_desc& d, PlanGraph& g);

}  // namespace b200fft
