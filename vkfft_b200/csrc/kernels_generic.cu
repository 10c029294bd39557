// The runtime-scheduled kernel (generic.cuh), one instantiation per precision.
#define B2_SHARD 1000
#include "kernel_inst.cuh"

static ::b200fft::GenericRegistrar<float, 8> b2_generic_f32_8("generic<float,r<=8>");
static ::b200fft::GenericRegistrar<float, 11> b2_generic_f32_11("generic<float,r<=11>");
static ::b200fft::GenericRegistrar<float, 16> b2_generic_f32_16("generic<float,r<=16>");
static ::b200fft::GenericRegistrar<double, 8> b2_generic_f64_8("generic<double,r<=8>");
static ::b200fft::GenericRegistrar<double, 11> b2_generic_f64_11("generic<double,r<=11>");
static ::b200fft::GenericRegistrar<double, 16> b2_generic_f64_16("generic<double,r<=16>");
static ::b200fft::ElementwiseRegistrar<float> b2_ew_f32("elementwise<float>");
static ::b200fft::ElementwiseRegistrar<double> b2_ew_f64("elementwise<double>");
static ::b200fft::ElementwiseRegistrar<float, true> b2_ew_f32_half("elementwise<float,half in+out>");
