// Loss epilogue (SURVEY.md 8f rank 2): the image-space terms of the reference's get_loss_dict that re-read
// the rasterizer's outputs straight after the render -- L1 (street_gaussians_ns/sgn_splatfacto.py:1079-1084),
// sky accumulation (:1090-1093) and the object-accumulation entropy (sgn_splatfacto_scene_graph.py:386-389) --
// and their cotangents, in two HBM-bound passes (forward sums, backward cotangents) instead of ~25 torch
// elementwise / reduction launches.  The SSIM term (:1085-1087) has its own kernels (ssim.cu).  The ground truth may be the
// uint8 image the data loader holds (gt = u8 / 255, as the reference's `.float() / 255`).
//
// Arithmetic follows torch: gt*mask and rgb*mask rounded separately (no fma: an exact tie gt == rgb gives a zero difference
// and a zero gradient under any mask), |a - b|, clamp(x, 1e-5, 1 - 1e-5) with pass-through gradient inside the closed
// interval, natural log, means as sum / count (fp32 sums of per-block partials, summed in a fixed order: the
// result is deterministic run to run).
#include "sgn_common.cuh"

#define LOSS_THREADS 256
#define LOSS_BLOCKS 1056  // 132 SMs (H100 SXM) x 8 resident blocks of 256 threads

struct LossParams {
    long long P;  // pixels
    const float* rgb;
    const uint8_t* gt_u8;
    const float* gt_f32;
    const float* mask;          // [P] or null: gt*mask vs rgb*mask (sgn_splatfacto.py:1073-1076)
    const float* accumulation;  // [P] or null
    const uint8_t* sky_mask;    // [P] (1 = sky) or null
    const float* object_acc;    // [P] or null
    float w_l1, w_sky, w_ent;
};

__device__ __forceinline__ float gt_at(const LossParams& p, long long e) {
    return p.gt_u8 ? (float)p.gt_u8[e] / 255.0f : p.gt_f32[e];
}

__device__ __forceinline__ float block_sum(float v, float* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < LOSS_THREADS / 32) t = smem[threadIdx.x];
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// partial[3][gridDim.x]: per-block sums of |gt - rgb|, sky*accumulation, entropy
__global__ void __launch_bounds__(LOSS_THREADS) loss_fwd_kernel(const LossParams p, float* __restrict__ partial) {
    __shared__ float smem[LOSS_THREADS / 32];
    const long long n3 = p.P * 3, stride = (long long)gridDim.x * blockDim.x;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float s_l1 = 0.f, s_sky = 0.f, s_ent = 0.f;
    if (p.rgb) {
        const bool vec = !p.mask && (n3 % 4 == 0) && sgn_aligned16(p.rgb) && (p.gt_u8 ? ((uintptr_t)p.gt_u8 % 4 == 0) : sgn_aligned16(p.gt_f32));
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
                s_l1 += fabsf(g.x - r.x) + fabsf(g.y - r.y) + fabsf(g.z - r.z) + fabsf(g.w - r.w);
            }
        } else {
            for (long long e = tid; e < n3; e += stride) {
                const float m = p.mask ? p.mask[e / 3] : 1.f;
                s_l1 += fabsf(__fmul_rn(gt_at(p, e), m) - __fmul_rn(p.rgb[e], m));
            }
        }
    }
    for (long long i = tid; i < p.P; i += stride) {
        if (p.sky_mask && p.accumulation) s_sky += p.sky_mask[i] ? p.accumulation[i] : 0.f;
        if (p.object_acc) {
            const float oa = fminf(fmaxf(p.object_acc[i], 1e-5f), 1.f - 1e-5f);
            s_ent += -(oa * logf(oa) + (1.f - oa) * logf(1.f - oa));
        }
    }
    const float a = block_sum(s_l1, smem), b = block_sum(s_sky, smem), c = block_sum(s_ent, smem);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = a;
        partial[gridDim.x + blockIdx.x] = b;
        partial[2 * gridDim.x + blockIdx.x] = c;
    }
}

// losses[3] = weight * mean, in a fixed summation order
__global__ void __launch_bounds__(LOSS_THREADS) loss_finish_kernel(const LossParams p, const float* __restrict__ partial, int nblocks,
                                                                   float* __restrict__ losses) {
    __shared__ float smem[LOSS_THREADS / 32];
    for (int term = 0; term < 3; ++term) {
        float s = 0.f;
        for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += partial[term * nblocks + i];
        const float tot = block_sum(s, smem);
        if (threadIdx.x == 0) {
            const float count = term == 0 ? (float)(p.P * 3) : (float)p.P;
            const float w = term == 0 ? p.w_l1 : (term == 1 ? p.w_sky : p.w_ent);
            losses[term] = w * (tot / count);
        }
    }
}

// cotangents of the three weighted means, scaled by the incoming gradients g[3] (device scalars; null = 1)
__global__ void __launch_bounds__(LOSS_THREADS) loss_bwd_kernel(const LossParams p, const float* __restrict__ g, float* __restrict__ v_rgb,
                                                                float* __restrict__ v_acc, float* __restrict__ v_obj) {
    const long long n3 = p.P * 3, stride = (long long)gridDim.x * blockDim.x;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const float g0 = g ? g[0] : 1.f, g1 = g ? g[1] : 1.f, g2 = g ? g[2] : 1.f;
    if (v_rgb && p.rgb) {
        const float k = g0 * p.w_l1 / (float)n3;
        const bool vec = !p.mask && (n3 % 4 == 0) && sgn_aligned16(p.rgb) && sgn_aligned16(v_rgb) &&
                         (p.gt_u8 ? ((uintptr_t)p.gt_u8 % 4 == 0) : sgn_aligned16(p.gt_f32));
        auto sgn = [](float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f); };
        if (vec) {
            for (long long q = tid; q < n3 / 4; q += stride) {
                const float4 r = reinterpret_cast<const float4*>(p.rgb)[q];
                float4 t;
                if (p.gt_u8) {
                    const uchar4 u = reinterpret_cast<const uchar4*>(p.gt_u8)[q];
                    t = make_float4((float)u.x / 255.0f, (float)u.y / 255.0f, (float)u.z / 255.0f, (float)u.w / 255.0f);
                } else {
                    t = reinterpret_cast<const float4*>(p.gt_f32)[q];
                }
                // d|gt - rgb| / d rgb = -sign(gt - rgb)
                reinterpret_cast<float4*>(v_rgb)[q] = make_float4(-k * sgn(t.x - r.x), -k * sgn(t.y - r.y), -k * sgn(t.z - r.z), -k * sgn(t.w - r.w));
            }
        } else {
            for (long long e = tid; e < n3; e += stride) {
                const float m = p.mask ? p.mask[e / 3] : 1.f;
                v_rgb[e] = -k * sgn(__fmul_rn(gt_at(p, e), m) - __fmul_rn(p.rgb[e], m)) * m;
            }
        }
    }
    for (long long i = tid; i < p.P; i += stride) {
        if (v_acc) v_acc[i] = (p.sky_mask && p.sky_mask[i]) ? g1 * p.w_sky / (float)p.P : 0.f;
        if (v_obj && p.object_acc) {
            const float x = p.object_acc[i];
            const bool inside = (x >= 1e-5f) && (x <= 1.f - 1e-5f);  // torch.clamp passes the gradient on the closed interval
            const float oa = fminf(fmaxf(x, 1e-5f), 1.f - 1e-5f);
            // d/d oa [-(oa log oa + (1 - oa) log(1 - oa))] = log(1 - oa) - log(oa)
            v_obj[i] = inside ? g2 * p.w_ent / (float)p.P * (logf(1.f - oa) - logf(oa)) : 0.f;
        }
    }
}

static int fill(LossParams& p, int H, int W, const sgn_loss_in* in) {
    SGN_REQUIRE(H > 0 && W > 0 && in, "sgn_loss: empty image or null input");
    SGN_REQUIRE(!in->rgb || (in->gt_u8 != nullptr) != (in->gt_f32 != nullptr), "sgn_loss: exactly one of gt_u8 / gt_f32 must be given with rgb");
    p.P = (long long)H * W;
    p.rgb = in->rgb; p.gt_u8 = in->gt_u8; p.gt_f32 = in->gt_f32; p.mask = in->mask;
    p.accumulation = in->accumulation; p.sky_mask = in->sky_mask; p.object_acc = in->object_acc;
    p.w_l1 = in->w_l1; p.w_sky = in->w_sky; p.w_ent = in->w_entropy;
    return SGN_OK;
}

extern "C" size_t sgn_loss_scratch_bytes(void) { return sizeof(float) * 3 * LOSS_BLOCKS; }

extern "C" int sgn_loss_fwd(int H, int W, const sgn_loss_in* in, float* losses, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_loss_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    LossParams p;
    if (int rc = fill(p, H, W, in)) return rc;
    SGN_REQUIRE(losses && scratch, "sgn_loss_fwd: null output");
    if (scratch_bytes < sgn_loss_scratch_bytes()) {
        sgn_set_error("sgn_loss_fwd: scratch too small");
        return SGN_ERR_WORKSPACE;
    }
    loss_fwd_kernel<<<LOSS_BLOCKS, LOSS_THREADS, 0, stream>>>(p, (float*)scratch);
    SGN_CHECK_LAUNCH("loss_fwd_kernel");
    loss_finish_kernel<<<1, LOSS_THREADS, 0, stream>>>(p, (const float*)scratch, LOSS_BLOCKS, losses);
    SGN_CHECK_LAUNCH("loss_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_loss_bwd(int H, int W, const sgn_loss_in* in, const float* grad_losses, float* v_rgb, float* v_accumulation,
                            float* v_object_acc, void* stream_) {
    SGN_RANGE("sgn_loss_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    LossParams p;
    if (int rc = fill(p, H, W, in)) return rc;
    loss_bwd_kernel<<<LOSS_BLOCKS, LOSS_THREADS, 0, stream>>>(p, grad_losses, v_rgb, v_accumulation, v_object_acc);
    SGN_CHECK_LAUNCH("loss_bwd_kernel");
    return SGN_OK;
}
