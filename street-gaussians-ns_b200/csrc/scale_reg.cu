// PhysGaussian's scale regularisation, the term nerfstudio's SplatfactoModel.get_loss_dict adds every tenth step when
// use_scale_regularization is set (the reference's config sets it, sgn_splatfacto.py:206-211, its loss override drops it):
//
//   s = exp(scales) [N,3];  r = amax(s) / amin(s);  scale_reg = 0.1 * mean(max(r, max_ratio) - max_ratio)
//
// over the N rows of the frame (the visible sub-models, read in place through the device segment table in the 128-row chunks
// project.cu and metrics.cu use).
//
// Forward: one thread per row, expf / IEEE division / max in fp32 as torch computes them; the per-row terms are summed in fp64
// per thread, then per block, and a one-block finish kernel adds the per-block partials in a fixed order: the same bits every
// run.  The mean is rounded once to fp32 and multiplied by 0.1f in fp32, as torch's `0.1 * reg.mean()`.
//
// Backward: elementwise, so deterministic as it stands.  Each row's gradient follows torch autograd's chain step by step
// (explicit _rn intrinsics, nothing contracted): g = (v * 0.1f) * (1.0f / N) (torch's mean backward multiplies by the
// reciprocal of a scalar divisor), halved at r == max_ratio (torch.maximum's tie), then g / amin for the max and
// -g * (r / amin) for the min, each split evenly between tied elements (amax / amin's backward), times exp(x).  A row with
// r < max_ratio has no gradient and is not written.
#include "sgn_common.cuh"

#define SR_CHUNK 128      // rows per chunk of the segment table (sgn_segment.chunk0); one thread per row
#define SR_BLOCKS 1056    // forward: 132 SMs (H100 SXM) x 8 resident blocks
#define SR_THREADS SR_CHUNK

// the last segment whose first chunk is <= c (a zero-row segment shares its chunk0 with the next one)
__device__ __forceinline__ int sr_segment_of(const sgn_segment* __restrict__ segs, int nseg, int c) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (segs[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

template <typename T>
__device__ __forceinline__ T sr_block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < SR_THREADS / 32 ? smem[threadIdx.x] : T(0);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

__global__ void __launch_bounds__(SR_THREADS) scale_reg_fwd_kernel(const sgn_segment* __restrict__ segs, int nseg, int num_chunks,
                                                                   float max_ratio, double* __restrict__ partial) {
    __shared__ double s_red[SR_THREADS / 32];
    double acc = 0.0;
    for (int c = blockIdx.x; c < num_chunks; c += gridDim.x) {
        const sgn_segment& sg = segs[sr_segment_of(segs, nseg, c)];
        const int row = (c - sg.chunk0) * SR_CHUNK + (int)threadIdx.x;
        if (row < sg.count) {
            const float* x = sg.scales + (size_t)row * 3;
            const float s0 = expf(x[0]), s1 = expf(x[1]), s2 = expf(x[2]);
            const float mx = fmaxf(fmaxf(s0, s1), s2), mn = fminf(fminf(s0, s1), s2);
            const float r = __fdiv_rn(mx, mn);
            acc += (double)__fsub_rn(fmaxf(r, max_ratio), max_ratio);
        }
    }
    const double b = sr_block_sum(acc, s_red);
    if (threadIdx.x == 0) partial[blockIdx.x] = b;
}

__global__ void __launch_bounds__(SR_THREADS) scale_reg_finish_kernel(const double* __restrict__ partial, int nblocks, int N,
                                                                      float* __restrict__ out) {
    __shared__ double s_red[SR_THREADS / 32];
    double s = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += partial[i];
    const double tot = sr_block_sum(s, s_red);
    if (threadIdx.x == 0) out[0] = __fmul_rn((float)(tot / (double)N), 0.1f);  // 0 / 0 = NaN for zero rows, as torch's mean
}

__global__ void __launch_bounds__(SR_THREADS) scale_reg_bwd_kernel(const sgn_segment* __restrict__ segs,
                                                                   const sgn_segment_grads* __restrict__ grads, int nseg, float inv_n,
                                                                   float max_ratio, const float* __restrict__ v_out) {
    const int c = blockIdx.x;
    const int k = sr_segment_of(segs, nseg, c);
    const sgn_segment& sg = segs[k];
    const int row = (c - sg.chunk0) * SR_CHUNK + (int)threadIdx.x;
    if (row >= sg.count) return;
    const float* x = sg.scales + (size_t)row * 3;
    const float s[3] = {expf(x[0]), expf(x[1]), expf(x[2])};
    const float mx = fmaxf(fmaxf(s[0], s[1]), s[2]), mn = fminf(fminf(s[0], s[1]), s[2]);
    const float r = __fdiv_rn(mx, mn);
    if (r < max_ratio) return;  // max(r, max_ratio) does not depend on r: no gradient
    float g = __fmul_rn(__fmul_rn(*v_out, 0.1f), inv_n);
    if (r == max_ratio) g = __fmul_rn(g, 0.5f);  // torch.maximum sends half of the gradient to each side of a tie
    const float g_mx = __fdiv_rn(g, mn);
    const float g_mn = __fmul_rn(-g, __fdiv_rn(r, mn));
    const float n_mx = (float)((s[0] == mx) + (s[1] == mx) + (s[2] == mx));
    const float n_mn = (float)((s[0] == mn) + (s[1] == mn) + (s[2] == mn));
    const float d_mx = __fdiv_rn(g_mx, n_mx), d_mn = __fdiv_rn(g_mn, n_mn);
    float* gs = grads[k].scales + (size_t)row * 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float d = 0.f;
        if (s[j] == mx) d = d_mx;
        if (s[j] == mn) d = s[j] == mx ? __fadd_rn(d, d_mn) : d_mn;
        gs[j] = __fadd_rn(gs[j], __fmul_rn(d, s[j]));
    }
}

extern "C" size_t sgn_scale_reg_scratch_bytes(void) { return sizeof(double) * SR_BLOCKS; }

extern "C" int sgn_scale_reg_fwd(const sgn_segment* table_dev, int nseg, int N, int num_chunks, float max_ratio, float* out, void* scratch,
                                 size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_scale_reg_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(out && scratch, "sgn_scale_reg_fwd: null output or scratch");
    SGN_REQUIRE(N >= 0 && nseg >= 0 && num_chunks >= 0, "sgn_scale_reg_fwd: negative N / nseg / num_chunks");
    SGN_REQUIRE(table_dev || nseg == 0, "sgn_scale_reg_fwd: null segment table with nseg = %d", nseg);
    SGN_REQUIRE(nseg > 0 || num_chunks == 0, "sgn_scale_reg_fwd: num_chunks = %d without segments", num_chunks);
    if (scratch_bytes < sgn_scale_reg_scratch_bytes()) {
        sgn_set_error("sgn_scale_reg_fwd: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_scale_reg_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    scale_reg_fwd_kernel<<<SR_BLOCKS, SR_THREADS, 0, stream>>>(table_dev, nseg, num_chunks, max_ratio, (double*)scratch);
    SGN_CHECK_LAUNCH("scale_reg_fwd_kernel");
    scale_reg_finish_kernel<<<1, SR_THREADS, 0, stream>>>((const double*)scratch, SR_BLOCKS, N, out);
    SGN_CHECK_LAUNCH("scale_reg_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_scale_reg_bwd(const sgn_segment* table_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                                 float max_ratio, const float* v_out, void* stream_) {
    SGN_RANGE("sgn_scale_reg_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(v_out, "sgn_scale_reg_bwd: null cotangent");
    SGN_REQUIRE(N >= 0 && nseg >= 0 && num_chunks >= 0, "sgn_scale_reg_bwd: negative N / nseg / num_chunks");
    SGN_REQUIRE((table_dev && grads_dev) || nseg == 0, "sgn_scale_reg_bwd: null segment or gradient table with nseg = %d", nseg);
    SGN_REQUIRE(nseg > 0 || num_chunks == 0, "sgn_scale_reg_bwd: num_chunks = %d without segments", num_chunks);
    if (num_chunks == 0) return SGN_OK;
    const float inv_n = 1.0f / (float)N;
    scale_reg_bwd_kernel<<<num_chunks, SR_THREADS, 0, stream>>>(table_dev, grads_dev, nseg, inv_n, max_ratio, v_out);
    SGN_CHECK_LAUNCH("scale_reg_bwd_kernel");
    return SGN_OK;
}
