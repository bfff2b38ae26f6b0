// Per-step training metrics (the reference's SplatfactoModel.get_metrics_dict, street_gaussians_ns/sgn_splatfacto.py:1015-1040,
// inherited by the scene graph) in one HBM-bound pass: PSNR of rgb against gt (torchmetrics PeakSignalNoiseRatio,
// data_range 1), and the means of exp(scales), scales, sigmoid(opacities) and radii over the visible sub-models.  The reference
// reads the last four from the torch.cat of the visible sub-models built in get_outputs (scene graph :354-360); here they are
// read through the frame's device segment table, in place, in the 128-row chunks project.cu uses.  Eval's
// get_image_metrics_and_images (:1109-1187) takes its PSNR from the same pass, with the mask.
//
// Arithmetic: gt*mask and rgb*mask rounded separately (as loss.cu: an exact tie gives a zero difference under any mask), the
// difference squared in fp32, expf and 1 / (1 + expf(-x)) in fp32 with IEEE division.  Every term is summed in fp64 per thread,
// then per block, and the per-block partials are added in a fixed order by a one-block finish kernel: the results are
// bit-identical from run to run.  The radii sum is an int64.
#include "sgn_common.cuh"

#define MET_THREADS 256
#define MET_BLOCKS 1056       // 132 SMs (H100 SXM) x 8 resident blocks of 256 threads
#define MET_CHUNK 128         // rows per chunk of the segment table (sgn_segment.chunk0)
#define MET_MAX_SEGMENTS 1024 // as project.cu

struct MetricsParams {
    long long P;  // pixels; 0 = no image term
    const float* rgb;
    const uint8_t* gt_u8;
    const float* gt_f32;
    const float* mask;  // [P] or null
    const sgn_segment* segs;  // null = no parameter terms
    int nseg, num_chunks;
    long long N;  // rows of the frame
    const int32_t* radii;  // [N] or null
};

__device__ __forceinline__ float gt_at(const MetricsParams& p, long long e) {
    return p.gt_u8 ? (float)p.gt_u8[e] / 255.0f : p.gt_f32[e];
}

__device__ __forceinline__ float sq_diff(float g, float r, float m) {
    const float d = __fsub_rn(__fmul_rn(g, m), __fmul_rn(r, m));
    return __fmul_rn(d, d);
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < MET_THREADS / 32) t = smem[threadIdx.x];
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// partial: double[4][gridDim.x] = {sse, sum exp(scale), sum scale, sum sigmoid(opacity)}, then int64[gridDim.x] = sum radii
__global__ void __launch_bounds__(MET_THREADS) metrics_kernel(const MetricsParams p, double* __restrict__ partial) {
    __shared__ int s_chunk0[MET_MAX_SEGMENTS];
    __shared__ double s_red[MET_THREADS / 32];
    __shared__ long long s_red_i[MET_THREADS / 32];
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double s_sse = 0.0, s_exp = 0.0, s_log = 0.0, s_sig = 0.0;
    long long s_rad = 0;

    if (p.rgb) {
        const long long n3 = p.P * 3;
        const bool vec = (n3 % 4 == 0) && sgn_aligned16(p.rgb) && (p.gt_u8 ? ((uintptr_t)p.gt_u8 % 4 == 0) : sgn_aligned16(p.gt_f32));
        if (vec) {
            for (long long q = tid; q < n3 / 4; q += stride) {
                const float4 r = reinterpret_cast<const float4*>(p.rgb)[q];
                float4 g;
                if (p.gt_u8) {
                    const uchar4 u = reinterpret_cast<const uchar4*>(p.gt_u8)[q];
                    g = make_float4((float)u.x / 255.0f, (float)u.y / 255.0f, (float)u.z / 255.0f, (float)u.w / 255.0f);
                } else {
                    g = reinterpret_cast<const float4*>(p.gt_f32)[q];
                }
                float m0 = 1.f, m1 = 1.f, m2 = 1.f, m3 = 1.f;
                if (p.mask) {
                    const long long e = 4 * q;
                    m0 = p.mask[e / 3]; m1 = p.mask[(e + 1) / 3]; m2 = p.mask[(e + 2) / 3]; m3 = p.mask[(e + 3) / 3];
                }
                // fp32 squares, one fp64 add per element
                s_sse += (double)sq_diff(g.x, r.x, m0);
                s_sse += (double)sq_diff(g.y, r.y, m1);
                s_sse += (double)sq_diff(g.z, r.z, m2);
                s_sse += (double)sq_diff(g.w, r.w, m3);
            }
        } else {
            for (long long e = tid; e < n3; e += stride)
                s_sse += (double)sq_diff(gt_at(p, e), p.rgb[e], p.mask ? p.mask[e / 3] : 1.f);
        }
    }

    if (p.segs && p.num_chunks > 0) {
        for (int i = threadIdx.x; i < p.nseg; i += blockDim.x) s_chunk0[i] = p.segs[i].chunk0;
        __syncthreads();
        for (int c = blockIdx.x; c < p.num_chunks; c += gridDim.x) {
            // the last segment whose first chunk is <= c (a zero-row segment shares its chunk0 with the next one)
            int lo = 0, hi = p.nseg - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (s_chunk0[mid] <= c) lo = mid; else hi = mid - 1;
            }
            const sgn_segment& sg = p.segs[lo];
            const int r0 = (c - sg.chunk0) * MET_CHUNK;
            const int rows = min(MET_CHUNK, sg.count - r0);
            const float* sc = sg.scales + (size_t)r0 * 3;
            for (int k = threadIdx.x; k < rows * 3; k += blockDim.x) {
                const float x = sc[k];
                s_exp += (double)expf(x);
                s_log += (double)x;
            }
            if ((int)threadIdx.x < rows) {
                const float x = sg.opacities[r0 + threadIdx.x];
                s_sig += (double)(1.0f / (1.0f + expf(-x)));
            }
        }
    }

    if (p.radii)
        for (long long i = tid; i < p.N; i += stride) s_rad += p.radii[i];

    const double a = block_sum(s_sse, s_red), b = block_sum(s_exp, s_red), c = block_sum(s_log, s_red), d = block_sum(s_sig, s_red);
    const long long e = block_sum(s_rad, s_red_i);
    if (threadIdx.x == 0) {
        const int nb = gridDim.x;
        partial[blockIdx.x] = a;
        partial[nb + blockIdx.x] = b;
        partial[2 * nb + blockIdx.x] = c;
        partial[3 * nb + blockIdx.x] = d;
        reinterpret_cast<long long*>(partial + 4 * nb)[blockIdx.x] = e;
    }
}

// out[5] = {psnr, scale_mean, log_scale_mean, sigmoid_opacity, radii_mean}, each rounded once to fp32; a term without inputs is NaN
__global__ void __launch_bounds__(MET_THREADS) metrics_finish_kernel(const MetricsParams p, const double* __restrict__ partial, int nblocks,
                                                                     float* __restrict__ out) {
    __shared__ double s_red[MET_THREADS / 32];
    __shared__ long long s_red_i[MET_THREADS / 32];
    double tot[4];
    for (int term = 0; term < 4; ++term) {
        double s = 0.0;
        for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += partial[term * nblocks + i];
        tot[term] = block_sum(s, s_red);
    }
    long long r = 0;
    const long long* pr = reinterpret_cast<const long long*>(partial + 4 * nblocks);
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) r += pr[i];
    r = block_sum(r, s_red_i);
    if (threadIdx.x == 0) {
        const double nan = __longlong_as_double(0x7ff8000000000000ULL);
        const double n = (double)p.N;
        // 10 log10(1 / mse) = -10 log10(sse / 3P): +inf when the images are equal
        out[0] = p.rgb ? (float)(-10.0 * log10(tot[0] / (3.0 * (double)p.P))) : (float)nan;
        out[1] = p.segs ? (float)(tot[1] / (3.0 * n)) : (float)nan;  // 0 / 0 = NaN for zero rows, as torch.mean of an empty tensor
        out[2] = p.segs ? (float)(tot[2] / (3.0 * n)) : (float)nan;
        out[3] = p.segs ? (float)(tot[3] / n) : (float)nan;
        out[4] = p.radii ? (float)((double)r / n) : (float)nan;
    }
}

extern "C" size_t sgn_metrics_scratch_bytes(void) { return (4 * sizeof(double) + sizeof(long long)) * MET_BLOCKS; }

extern "C" int sgn_metrics(int H, int W, const sgn_loss_in* image, const sgn_segment* table_dev, int nseg, int N, int num_chunks,
                           const int32_t* radii, float* out, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_metrics");
    cudaStream_t stream = (cudaStream_t)stream_;
    MetricsParams p = {};
    SGN_REQUIRE(out && scratch, "sgn_metrics: null output or scratch");
    SGN_REQUIRE(N >= 0 && nseg >= 0 && num_chunks >= 0, "sgn_metrics: negative N / nseg / num_chunks");
    SGN_REQUIRE(table_dev || nseg == 0, "sgn_metrics: null segment table with nseg = %d", nseg);
    SGN_REQUIRE(nseg <= MET_MAX_SEGMENTS, "sgn_metrics: %d segments (at most %d)", nseg, MET_MAX_SEGMENTS);
    SGN_REQUIRE(!table_dev || nseg > 0 || num_chunks == 0, "sgn_metrics: num_chunks = %d without segments", num_chunks);
    if (image && image->rgb) {
        SGN_REQUIRE(H > 0 && W > 0, "sgn_metrics: empty image");
        SGN_REQUIRE((image->gt_u8 != nullptr) != (image->gt_f32 != nullptr), "sgn_metrics: exactly one of gt_u8 / gt_f32 must be given with rgb");
        p.P = (long long)H * W;
        p.rgb = image->rgb; p.gt_u8 = image->gt_u8; p.gt_f32 = image->gt_f32; p.mask = image->mask;
    }
    if (scratch_bytes < sgn_metrics_scratch_bytes()) {
        sgn_set_error("sgn_metrics: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_metrics_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    p.segs = table_dev; p.nseg = nseg; p.num_chunks = table_dev ? num_chunks : 0; p.N = N; p.radii = radii;
    metrics_kernel<<<MET_BLOCKS, MET_THREADS, 0, stream>>>(p, (double*)scratch);
    SGN_CHECK_LAUNCH("metrics_kernel");
    metrics_finish_kernel<<<1, MET_THREADS, 0, stream>>>(p, (const double*)scratch, MET_BLOCKS, out);
    SGN_CHECK_LAUNCH("metrics_finish_kernel");
    return SGN_OK;
}
