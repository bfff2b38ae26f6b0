// Fused multi-tensor Adam over the flat gradient arena (SURVEY.md 8f rank 1).
//
// The reference optimises the six Gaussian parameter groups of every sub-model with nine torch Adam
// optimizers (street_gaussians_ns/sgn_config.py:71-108: lr per group, eps 1e-15, betas (0.9, 0.999), no weight
// decay), i.e. ~200 parameter tensors per step.  Here ONE launch walks all of them: gradients and both
// moments live in flat arenas with the layout of the project backward's gradient arena, parameters stay
// where the model keeps them (a pointer table).  Semantics: torch.optim.Adam (dense: moments decay for
// Gaussians that were not visible, as in the reference).  HBM-bound: 28 B per element.  sgn_adam_step_visible is the
// selective form (gsplat's visible_adam): only the rows the frame's camera saw are read and written.
#include "sgn_common.cuh"

#define ADAM_THREADS 256
#define ADAM_CHUNK 4096  // elements per block

__global__ void __launch_bounds__(ADAM_THREADS)
adam_kernel(const sgn_adam_tensor* __restrict__ table, int ntensors, const float* __restrict__ grads,
            float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq) {
    extern __shared__ int s_chunk0[];
    for (int i = threadIdx.x; i < ntensors; i += blockDim.x) s_chunk0[i] = table[i].chunk0;
    __syncthreads();
    int lo = 0, hi = ntensors - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_chunk0[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const sgn_adam_tensor t = table[lo];
    const long long e0 = (long long)(blockIdx.x - t.chunk0) * ADAM_CHUNK;
    const long long n = t.numel;
    float* __restrict__ p = t.param;
    const float* __restrict__ g = grads + t.grad_offset;
    float* __restrict__ m = exp_avg + t.arena_offset;
    float* __restrict__ v = exp_avg_sq + t.arena_offset;
    const float b1 = t.beta1, b2 = t.beta2, step_size = t.step_size, sqrt_bc2 = t.sqrt_bc2, eps = t.eps;
    const float w1 = t.one_minus_beta1, w2 = t.one_minus_beta2;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) && ((t.arena_offset & 3) == 0) && ((t.grad_offset & 3) == 0);
#pragma unroll
    for (int it = 0; it < ADAM_CHUNK / (ADAM_THREADS * 4); ++it) {
        const long long e = e0 + ((long long)it * ADAM_THREADS + threadIdx.x) * 4;
        if (e >= n) break;
        if (vec && e + 4 <= n) {
            const float4 gg = *reinterpret_cast<const float4*>(g + e);
            float4 mm = *reinterpret_cast<const float4*>(m + e);
            float4 vv = *reinterpret_cast<const float4*>(v + e);
            float4 pp = *reinterpret_cast<const float4*>(p + e);
            float* ga = (float*)&gg; float* ma = (float*)&mm; float* va = (float*)&vv; float* pa = (float*)&pp;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                ma[k] = ma[k] + w1 * (ga[k] - ma[k]);        // exp_avg.lerp_(grad, 1 - beta1)
                va[k] = va[k] * b2 + w2 * ga[k] * ga[k];     // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                const float denom = sqrtf(va[k]) / sqrt_bc2 + eps;
                pa[k] = pa[k] - step_size * (ma[k] / denom);
            }
            *reinterpret_cast<float4*>(m + e) = mm;
            *reinterpret_cast<float4*>(v + e) = vv;
            *reinterpret_cast<float4*>(p + e) = pp;
        } else {
            for (int k = 0; k < 4 && e + k < n; ++k) {
                const float gk = g[e + k];
                const float mk = m[e + k] + w1 * (gk - m[e + k]);
                const float vk = v[e + k] * b2 + w2 * gk * gk;
                m[e + k] = mk; v[e + k] = vk;
                p[e + k] = p[e + k] - step_size * (mk / (sqrtf(vk) / sqrt_bc2 + eps));
            }
        }
    }
}

// Selective Adam (gsplat's visible_adam, Taming 3DGS): the same update, restricted to the rows whose visibility byte is set.
// Element e of a tensor with flag_row0 >= 0 belongs to row e / row_width and is stepped when visible[flag_row0 + row] != 0;
// the parameter and both moments of every other element keep their bits.  flag_row0 = -1: the tensor is stepped densely (the
// extra tensors).  A stepped element gets exactly adam_kernel's update: the same expressions in the same order (the float4 and
// scalar paths round alike).
//
// Each thread first reads the flags of its four float4s (independent loads: one latency, not four), then steps them.  A float4
// whose rows were all unseen is skipped without loading anything.  On the float4 path a float4 that straddles a seen and an
// unseen row is loaded whole and stored whole, its unseen elements with the bits just loaded: a full 16-byte store instead of
// partial ones, which HBM would have to merge into its sectors.  Misaligned tensors take the scalar path for the set bits.
#define ADAM_ITERS (ADAM_CHUNK / (ADAM_THREADS * 4))
__global__ void __launch_bounds__(ADAM_THREADS)
adam_visible_kernel(const sgn_adam_tensor* __restrict__ table, const sgn_adam_rows* __restrict__ rows, int ntensors,
                    const float* __restrict__ grads, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                    const uint8_t* __restrict__ visible) {
    extern __shared__ int s_chunk0[];
    for (int i = threadIdx.x; i < ntensors; i += blockDim.x) s_chunk0[i] = table[i].chunk0;
    __syncthreads();
    int lo = 0, hi = ntensors - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_chunk0[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const sgn_adam_tensor t = table[lo];
    const sgn_adam_rows rw = rows[lo];
    // tensor-local indices fit in 32 bits (every tensor holds fewer than 2^31 elements)
    const unsigned e0 = (unsigned)(blockIdx.x - t.chunk0) * ADAM_CHUNK;
    const unsigned n = (unsigned)min(t.numel, (int64_t)0x7FFFFFFF);
    const bool dense = rw.flag_row0 < 0;
    const unsigned w = dense ? 1u : (unsigned)rw.row_width;
    const uint8_t* __restrict__ vis = visible + (dense ? 0 : rw.flag_row0);
    // bit k of mask[it]: element e + k of the thread's it-th float4 is stepped.  One 32-bit division per float4; the rows of
    // e+1 .. e+3 by increments
    unsigned mask[ADAM_ITERS];
#pragma unroll
    for (int it = 0; it < ADAM_ITERS; ++it) {
        const unsigned e = e0 + ((unsigned)it * ADAM_THREADS + threadIdx.x) * 4;
        const unsigned cnt = e < n ? min(4u, n - e) : 0u;
        mask[it] = (1u << cnt) - 1u;
        if (!dense && cnt) {
            unsigned r = e / w, rem = e - r * w;
            unsigned f = vis[r] != 0 ? 1u : 0u, mk = f;
            for (unsigned k = 1; k < cnt; ++k) {
                if (++rem == w) { rem = 0; ++r; f = vis[r] != 0 ? 1u : 0u; }
                mk |= f << k;
            }
            mask[it] = mk;
        }
    }
    float* __restrict__ p = t.param;
    const float* __restrict__ g = grads + t.grad_offset;
    float* __restrict__ m = exp_avg + t.arena_offset;
    float* __restrict__ v = exp_avg_sq + t.arena_offset;
    const float b2 = t.beta2, step_size = t.step_size, sqrt_bc2 = t.sqrt_bc2, eps = t.eps;
    const float w1 = t.one_minus_beta1, w2 = t.one_minus_beta2;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) & 15u) == 0) && ((t.arena_offset & 3) == 0) && ((t.grad_offset & 3) == 0);
#pragma unroll
    for (int it = 0; it < ADAM_ITERS; ++it) {
        const unsigned mk = mask[it];
        if (mk == 0) continue;  // no row of this float4 was seen (or it lies behind the tensor): nothing is loaded or stored
        const unsigned e = e0 + ((unsigned)it * ADAM_THREADS + threadIdx.x) * 4;
        if (vec && e + 4 <= n) {
            const float4 gg = *reinterpret_cast<const float4*>(g + e);
            float4 mm = *reinterpret_cast<const float4*>(m + e);
            float4 vv = *reinterpret_cast<const float4*>(v + e);
            float4 pp = *reinterpret_cast<const float4*>(p + e);
            float* ga = (float*)&gg; float* ma = (float*)&mm; float* va = (float*)&vv; float* pa = (float*)&pp;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float mn = ma[k] + w1 * (ga[k] - ma[k]);        // exp_avg.lerp_(grad, 1 - beta1)
                const float vn = va[k] * b2 + w2 * ga[k] * ga[k];     // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                const float denom = sqrtf(vn) / sqrt_bc2 + eps;
                const float pn = pa[k] - step_size * (mn / denom);
                if ((mk >> k) & 1u) { ma[k] = mn; va[k] = vn; pa[k] = pn; }  // an unseen element is stored with its own bits
            }
            *reinterpret_cast<float4*>(m + e) = mm;
            *reinterpret_cast<float4*>(v + e) = vv;
            *reinterpret_cast<float4*>(p + e) = pp;
        } else {
            for (unsigned k = 0; k < 4; ++k) {
                if (!((mk >> k) & 1u)) continue;
                const float gk = g[e + k];
                const float mn = m[e + k] + w1 * (gk - m[e + k]);
                const float vn = v[e + k] * b2 + w2 * gk * gk;
                m[e + k] = mn; v[e + k] = vn;
                p[e + k] = p[e + k] - step_size * (mn / (sqrtf(vn) / sqrt_bc2 + eps));
            }
        }
    }
}

// seen[dst_row0[s] + j] |= flags[src_row0[s] + j] for the rows j < rows[s] of every segment s: the frame's visibility bytes
// folded into a mask kept across frames (the rows a gradient-accumulation cycle has seen).  Segments lie back to back in
// the frame (src_row0 non-decreasing, each starting where the previous one ends), so one launch covers them all.
__global__ void __launch_bounds__(256)
visible_or_kernel(const int64_t* __restrict__ segs, int nseg, int64_t n, const uint8_t* __restrict__ flags, uint8_t* __restrict__ seen) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (segs[3 * mid] <= i) lo = mid; else hi = mid - 1;
    }
    const int64_t j = i - segs[3 * lo];
    if (j < segs[3 * lo + 2]) seen[segs[3 * lo + 1] + j] = 1;
}

extern "C" size_t sgn_sizeof_adam_tensor(void) { return sizeof(sgn_adam_tensor); }
extern "C" size_t sgn_sizeof_adam_rows(void) { return sizeof(sgn_adam_rows); }
extern "C" int sgn_adam_chunk_elems(void) { return ADAM_CHUNK; }

extern "C" int sgn_adam_step(const sgn_adam_tensor* table_dev, int ntensors, int num_chunks, const float* grad_arena,
                             float* exp_avg, float* exp_avg_sq, void* stream) {
    SGN_RANGE("sgn_adam_step");
    SGN_REQUIRE(table_dev && grad_arena && exp_avg && exp_avg_sq, "sgn_adam_step: null pointer");
    SGN_REQUIRE(ntensors >= 1 && ntensors <= 8192, "sgn_adam_step: ntensors=%d out of range [1,8192]", ntensors);
    SGN_REQUIRE(sgn_aligned16(grad_arena) && sgn_aligned16(exp_avg) && sgn_aligned16(exp_avg_sq), "arenas must be 16-byte aligned");
    if (num_chunks <= 0) return SGN_OK;
    adam_kernel<<<num_chunks, ADAM_THREADS, ntensors * sizeof(int), (cudaStream_t)stream>>>(table_dev, ntensors, grad_arena,
                                                                                          exp_avg, exp_avg_sq);
    SGN_CHECK_LAUNCH("adam_kernel");
    return SGN_OK;
}

extern "C" int sgn_adam_step_visible(const sgn_adam_tensor* table_dev, const sgn_adam_rows* rows_dev, int ntensors, int num_chunks,
                                     const float* grad_arena, float* exp_avg, float* exp_avg_sq, const uint8_t* visible, void* stream) {
    SGN_RANGE("sgn_adam_step_visible");
    SGN_REQUIRE(table_dev && rows_dev && grad_arena && exp_avg && exp_avg_sq && visible, "sgn_adam_step_visible: null pointer");
    SGN_REQUIRE(ntensors >= 1 && ntensors <= 8192, "sgn_adam_step_visible: ntensors=%d out of range [1,8192]", ntensors);
    SGN_REQUIRE(sgn_aligned16(grad_arena) && sgn_aligned16(exp_avg) && sgn_aligned16(exp_avg_sq), "arenas must be 16-byte aligned");
    SGN_REQUIRE((reinterpret_cast<uintptr_t>(rows_dev) & 7u) == 0, "sgn_adam_step_visible: rows table must be 8-byte aligned");
    if (num_chunks <= 0) return SGN_OK;
    adam_visible_kernel<<<num_chunks, ADAM_THREADS, ntensors * sizeof(int), (cudaStream_t)stream>>>(
        table_dev, rows_dev, ntensors, grad_arena, exp_avg, exp_avg_sq, visible);
    SGN_CHECK_LAUNCH("adam_visible_kernel");
    return SGN_OK;
}

extern "C" int sgn_visible_or(const int64_t* segs_dev, int nseg, int64_t n, const uint8_t* flags, uint8_t* seen, void* stream) {
    SGN_RANGE("sgn_visible_or");
    SGN_REQUIRE(segs_dev && flags && seen && nseg >= 1 && n >= 0, "sgn_visible_or: bad argument");
    SGN_REQUIRE((reinterpret_cast<uintptr_t>(segs_dev) & 7u) == 0, "sgn_visible_or: segment table must be 8-byte aligned");
    if (n == 0) return SGN_OK;
    visible_or_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(segs_dev, nseg, n, flags, seen);
    SGN_CHECK_LAUNCH("visible_or_kernel");
    return SGN_OK;
}
