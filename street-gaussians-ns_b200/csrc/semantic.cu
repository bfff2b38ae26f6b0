// Per-Gaussian semantic logits: the cross-entropy term of the rendered semantic map against a 2D segmentation, its cotangent,
// the confusion matrix of eval, and the carry of the logits (and their Adam moments) through a refinement.  Street Gaussians
// gives every Gaussian a vector of class logits, alpha-blends them into a semantic map (sgn_blend_extra_fwd) and supervises it
// with cross-entropy; the reference's loader carries the segmentation as batch["semantic"] (data/sgn_dataset.py:125).
//
// Loss: per valid pixel (0 <= label < C and mask != 0) CE = logsumexp(S) - S[label], in fp32 with the max subtracted; per-block
// partials summed in fp64 (the pixel counts as int64), then added in a fixed order by a one-block finish kernel, as depth.cu:
// the same bits every run.  The valid-pixel count stays on the device.
//
// Metrics: one pass that counts (label, argmax) pairs in a per-block shared histogram, flushed with integer atomics (the
// counts do not depend on the order of the adds).
//
// Carry: the rebuild sgn_refine_apply does for features_dc, through the same per-element rule (sgn_refine_apply_elem) with
// the one tensor in features_dc's slot: a carried row is the same bits as the features_dc rows of the same plan.
#include <math.h>

#include <algorithm>

#include "sgn_common.cuh"
#include "sgn_refine_rules.cuh"

#define SEM_THREADS 256
#define SEM_BLOCKS 1056  // 132 SMs (H100 SXM) x 8 resident blocks of 256 threads
#define SEM_MAX_C 64

struct SemParams {
    long long P;
    int C;
    const float* logits;      // [P, C]
    const long long* labels;  // [P]
    const float* mask;        // [P] or null
};

__device__ __forceinline__ int sem_label(const SemParams& p, long long i) {
    const long long l = p.labels[i];
    if (l < 0 || l >= p.C) return -1;
    if (p.mask && p.mask[i] == 0.f) return -1;
    return (int)l;
}

// max and sum of exp(S - max) over the pixel's C logits
__device__ __forceinline__ void sem_softmax_stats(const float* s, int C, float& m, float& z) {
    m = s[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, s[c]);
    z = 0.f;
    for (int c = 0; c < C; ++c) z += expf(s[c] - m);
}

template <typename T>
__device__ __forceinline__ T sem_block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < SEM_THREADS / 32) t = smem[threadIdx.x];
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// partial: double[gridDim.x] = sum CE over the valid pixels, then int64[gridDim.x] = their count
__global__ void __launch_bounds__(SEM_THREADS) semantic_loss_fwd_kernel(const SemParams p, double* __restrict__ partial) {
    __shared__ double s_red[SEM_THREADS / 32];
    __shared__ long long s_red_i[SEM_THREADS / 32];
    double s = 0.0;
    long long n = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        const int l = sem_label(p, i);
        if (l < 0) continue;
        const float* x = p.logits + i * p.C;
        float m, z;
        sem_softmax_stats(x, p.C, m, z);
        const float lse = m + logf(z);
        s += (double)(lse - x[l]);
        ++n;
    }
    const double a = sem_block_sum(s, s_red);
    const long long b = sem_block_sum(n, s_red_i);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = a;
        reinterpret_cast<long long*>(partial + gridDim.x)[blockIdx.x] = b;
    }
}

// loss = w * sum / n_valid (exactly 0 when n_valid = 0)
__global__ void __launch_bounds__(SEM_THREADS) semantic_loss_finish_kernel(const double* __restrict__ partial, int nblocks, float w,
                                                                           float* __restrict__ loss, int* __restrict__ n_valid) {
    __shared__ double s_red[SEM_THREADS / 32];
    __shared__ long long s_red_i[SEM_THREADS / 32];
    double s = 0.0;
    long long n = 0;
    const long long* pn = reinterpret_cast<const long long*>(partial + nblocks);
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { s += partial[i]; n += pn[i]; }
    s = sem_block_sum(s, s_red);
    n = sem_block_sum(n, s_red_i);
    if (threadIdx.x == 0) {
        *loss = n > 0 ? (float)((double)w * (s / (double)n)) : 0.f;
        *n_valid = (int)n;
    }
}

// v_logits = g * w / n_valid * (softmax(S) - onehot(label)) on the valid pixels, 0 elsewhere
__global__ void __launch_bounds__(SEM_THREADS) semantic_loss_bwd_kernel(const SemParams p, float w, const int* __restrict__ n_valid,
                                                                        const float* __restrict__ g, float* __restrict__ v_logits) {
    const int n = *n_valid;
    const float k = n > 0 ? (g ? *g : 1.f) * w / (float)n : 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        float* v = v_logits + i * p.C;
        const int l = n > 0 ? sem_label(p, i) : -1;
        if (l < 0) {
            for (int c = 0; c < p.C; ++c) v[c] = 0.f;
            continue;
        }
        const float* x = p.logits + i * p.C;
        float m, z;
        sem_softmax_stats(x, p.C, m, z);
        for (int c = 0; c < p.C; ++c) v[c] = k * (expf(x[c] - m) / z - (c == l ? 1.f : 0.f));
    }
}

// confusion[label * C + argmax] += 1 over the valid pixels; ties go to the lowest class index
__global__ void __launch_bounds__(SEM_THREADS) semantic_confusion_kernel(const SemParams p, unsigned long long* __restrict__ confusion) {
    __shared__ unsigned s_hist[SEM_MAX_C * SEM_MAX_C];
    const int CC = p.C * p.C;
    for (int j = threadIdx.x; j < CC; j += blockDim.x) s_hist[j] = 0u;
    __syncthreads();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        const int l = sem_label(p, i);
        if (l < 0) continue;
        const float* x = p.logits + i * p.C;
        int a = 0;
        float best = x[0];
        for (int c = 1; c < p.C; ++c)
            if (x[c] > best) { best = x[c]; a = c; }
        atomicAdd(s_hist + l * p.C + a, 1u);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < CC; j += blockDim.x)
        if (s_hist[j]) atomicAdd(confusion + j, (unsigned long long)s_hist[j]);
}

static int sem_fill(SemParams& p, int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, const char* who) {
    SGN_REQUIRE(H > 0 && W > 0, "%s: empty image %dx%d", who, H, W);
    SGN_REQUIRE(C >= 1 && C <= SEM_MAX_C, "%s: C=%d out of range [1,%d]", who, C, SEM_MAX_C);
    SGN_REQUIRE(logits && labels, "%s: null logits or labels", who);
    p.P = (long long)H * W;
    p.C = C;
    p.logits = logits;
    p.labels = reinterpret_cast<const long long*>(labels);
    p.mask = mask;
    return SGN_OK;
}

extern "C" size_t sgn_semantic_scratch_bytes(void) { return (sizeof(double) + sizeof(long long)) * SEM_BLOCKS; }

extern "C" int sgn_semantic_loss_fwd(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, float weight,
                                     float* loss, int32_t* n_valid, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_semantic_loss_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SemParams p;
    if (int rc = sem_fill(p, H, W, C, logits, labels, mask, "sgn_semantic_loss_fwd")) return rc;
    SGN_REQUIRE(loss && n_valid && scratch, "sgn_semantic_loss_fwd: null output or scratch");
    if (scratch_bytes < sgn_semantic_scratch_bytes()) {
        sgn_set_error("sgn_semantic_loss_fwd: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_semantic_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    semantic_loss_fwd_kernel<<<SEM_BLOCKS, SEM_THREADS, 0, stream>>>(p, (double*)scratch);
    SGN_CHECK_LAUNCH("semantic_loss_fwd_kernel");
    semantic_loss_finish_kernel<<<1, SEM_THREADS, 0, stream>>>((const double*)scratch, SEM_BLOCKS, weight, loss, n_valid);
    SGN_CHECK_LAUNCH("semantic_loss_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_semantic_loss_bwd(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, float weight,
                                     const int32_t* n_valid, const float* grad_loss, float* v_logits, void* stream_) {
    SGN_RANGE("sgn_semantic_loss_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SemParams p;
    if (int rc = sem_fill(p, H, W, C, logits, labels, mask, "sgn_semantic_loss_bwd")) return rc;
    SGN_REQUIRE(n_valid && v_logits, "sgn_semantic_loss_bwd: null n_valid or output");
    semantic_loss_bwd_kernel<<<SEM_BLOCKS, SEM_THREADS, 0, stream>>>(p, weight, n_valid, grad_loss, v_logits);
    SGN_CHECK_LAUNCH("semantic_loss_bwd_kernel");
    return SGN_OK;
}

extern "C" int sgn_semantic_metrics(int H, int W, int C, const float* logits, const int64_t* labels, const float* mask, int64_t* confusion,
                                    void* stream_) {
    SGN_RANGE("sgn_semantic_metrics");
    cudaStream_t stream = (cudaStream_t)stream_;
    SemParams p;
    if (int rc = sem_fill(p, H, W, C, logits, labels, mask, "sgn_semantic_metrics")) return rc;
    SGN_REQUIRE(confusion, "sgn_semantic_metrics: null confusion matrix");
    SGN_CHECK_CUDA(cudaMemsetAsync(confusion, 0, sizeof(int64_t) * C * C, stream));
    const int blocks = (int)std::min<long long>((p.P + SEM_THREADS - 1) / SEM_THREADS, SEM_BLOCKS);
    semantic_confusion_kernel<<<blocks, SEM_THREADS, 0, stream>>>(p, reinterpret_cast<unsigned long long*>(confusion));
    SGN_CHECK_LAUNCH("semantic_confusion_kernel");
    return SGN_OK;
}

// ---- carry through a refinement ------------------------------------------------------------------------------------------

struct carry_totals {
    int32_t v[4];
};

__global__ void __launch_bounds__(SEM_THREADS)
refine_carry_kernel(int n, int width, const sgn_refine_config cfg, const sgn_refine_tensors t, const uint8_t* __restrict__ flags,
                    const int32_t* __restrict__ scan, const carry_totals totals) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)n * width) return;
    const long long i = e / width;
    const int c = (int)(e - i * width);
    // width[SGN_RT_DC] is the only non-zero width: column c lands in features_dc's slot and takes its path (no split offset,
    // no rescale, so no samples are read)
    sgn_refine_apply_elem(i, c, n, cfg, t, flags, scan, totals.v, nullptr);
}

extern "C" int sgn_refine_carry(int n, const sgn_refine_config* cfg, const uint8_t* flags, const int32_t* scan, const int32_t* totals,
                                const float* src, float* dst, int width, const float* src_m, const float* src_v, float* dst_m,
                                float* dst_v, void* stream) {
    SGN_RANGE("sgn_refine_carry");
    SGN_REQUIRE(n >= 0, "sgn_refine_carry: n=%d", n);
    SGN_REQUIRE(cfg != nullptr && totals != nullptr, "sgn_refine_carry: null config / totals");
    SGN_REQUIRE(cfg->n_split_samples >= 1 && cfg->n_split_samples <= 16, "sgn_refine_carry: n_split_samples=%d out of range [1,16]",
                cfg->n_split_samples);
    SGN_REQUIRE(width >= 1 && width <= SEM_MAX_C, "sgn_refine_carry: width=%d out of range [1,%d]", width, SEM_MAX_C);
    if (n == 0) return SGN_OK;
    SGN_REQUIRE(flags && scan && src, "sgn_refine_carry: null flags / scan / src");
    SGN_REQUIRE(totals[0] >= 0 && totals[1] >= 0 && totals[2] >= 0 && totals[3] >= totals[1] && totals[0] <= n && totals[3] <= n &&
                    totals[2] <= n,
                "sgn_refine_carry: inconsistent totals {%d,%d,%d,%d} for n=%d", totals[0], totals[1], totals[2], totals[3], n);
    const long long out_rows = (long long)totals[0] + (long long)cfg->n_split_samples * totals[1] + totals[2];
    SGN_REQUIRE(out_rows < (1ll << 31), "sgn_refine_carry: %lld output rows exceed the int32 row space", out_rows);
    SGN_REQUIRE(out_rows == 0 || dst, "sgn_refine_carry: null dst");
    const bool m = src_m && src_v && (out_rows == 0 || (dst_m && dst_v));
    SGN_REQUIRE(m || (!src_m && !src_v), "sgn_refine_carry: partial optimizer state");
    if (out_rows == 0) return SGN_OK;
    sgn_refine_tensors t = {};
    t.src[SGN_RT_DC] = src;
    t.dst[SGN_RT_DC] = dst;
    if (m) {
        t.src_m[SGN_RT_DC] = src_m; t.src_v[SGN_RT_DC] = src_v;
        t.dst_m[SGN_RT_DC] = dst_m; t.dst_v[SGN_RT_DC] = dst_v;
    }
    t.width[SGN_RT_DC] = width;
    carry_totals tt;
    for (int k = 0; k < 4; ++k) tt.v[k] = totals[k];
    const long long blocks = ((long long)n * width + SEM_THREADS - 1) / SEM_THREADS;
    SGN_REQUIRE(blocks < (1ll << 31), "sgn_refine_carry: grid too large");
    refine_carry_kernel<<<(unsigned)blocks, SEM_THREADS, 0, (cudaStream_t)stream>>>(n, width, *cfg, t, flags, scan, tt);
    SGN_CHECK_LAUNCH("refine_carry_kernel");
    return SGN_OK;
}
