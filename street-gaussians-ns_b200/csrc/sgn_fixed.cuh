// Deterministic-mode helpers shared by the blend backward (blend.cu) and the sky backward (sky.cu): the largest finite
// |cotangent| and the power-of-two fixed-point grid derived from it.  Static: each file that includes this header
// instantiates its own copy, compiled with that file's flags.
#pragma once
#include "sgn_common.cuh"

// ---- scale = 2^32 / max |cotangent| (gradients are linear in the cotangents: the fixed-point grid adapts to their
// magnitude; 2^31 of headroom above it, and the conic components of large Gaussians give up more places, fixed_shift in
// blend.cu), then fixed point -> float
static __global__ void __launch_bounds__(256)
cot_max_kernel(const float* __restrict__ a, long long n, unsigned* __restrict__ out_bits) {
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fabsf(a[i]);
        m = (v == v && v < 3.0e38f) ? fmaxf(m, v) : m;
    }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16)); m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4)); m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out_bits, __float_as_uint(m));  // non-negative floats order like their bits
}
static __global__ void fixed_scale_kernel(float* scale) {
    const float m = scale[0];  // the bits cot_max_kernel left are the float itself
    scale[0] = m > 0.f ? exp2f(32.f - ceilf(log2f(m))) : 4294967296.f;  // a power of two: scaling is exact
}
