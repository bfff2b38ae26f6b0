// SSIM loss term of the reference's get_loss_dict (street_gaussians_ns/sgn_splatfacto.py:1085-1087, ssim_lambda = 0.2 at
// :200): loss = weight * (1 - SSIM(gt*mask, rgb*mask)) with pytorch_msssim.SSIM(data_range=1, size_average=True,
// channel=3) -- an 11-tap separable Gaussian window (sigma 1.5), VALID padding, C1 = 0.01^2, C2 = 0.03^2, the mean of the
// (H-10) x (W-10) x 3 map -- and its cotangent for rgb (the gradient reaches the render only through rgb).
//
// Forward: a CTA owns a 32 x 16 tile of the output map for all three channels.  It stages the tile plus the 10-pixel halo
// of x = gt*mask and y = rgb*mask (interleaved, as [H,W,3] holds them), then per channel a horizontal pass and a vertical
// pass give the five moments mu_x, mu_y, E[x^2], E[y^2], E[xy] of every output pixel.  It evaluates the SSIM map there and
// writes, per valid pixel and channel, a = dS/dmu_y, b = dS/dE[y^2], c = dS/dE[xy] (each with the other moments held
// fixed) to the workspace (planar [3 channels][3 maps][Hv][Wv], 36 B per valid pixel), and one partial sum of the map per
// channel per CTA.  A one-CTA finish kernel adds the partials in a fixed order and writes weight * (1 - mean).
//
// Backward, a gather (no atomics; v_rgb is bit-reproducible):
//   dL/dy(q) = k * [ (G^T a)(q) + 2 y(q) (G^T b)(q) + x(q) (G^T c)(q) ] * mask(q),   k = -weight * g / (3 Hv Wv)
// where G^T is the transposed (full) separable filter over the valid-region maps, zero outside them.
//
// Arithmetic follows torch's fp32 statement of the same expressions (model.ssim): products x*x, y*y, x*y are rounded
// before they are filtered; divisions are IEEE (no fast math); FMA contraction is allowed.
#include "sgn_common.cuh"

#define SSIM_TW 32                 // output tile width (one warp row)
#define SSIM_TH 16                 // output tile height
#define SSIM_THREADS 256           // 32 x 8: each thread owns two adjacent output rows of its column
#define SSIM_R (SSIM_TH + 10)      // staged rows
#define SSIM_C (SSIM_TW + 10)      // staged columns
#define SSIM_FINISH_THREADS 1024

// _gauss_window(11, 1.5) in fp32, as torch computes it (exp, then division by the sum); symmetric.  The unrolled filter
// loops index it with constants: the taps are constant-bank operands of the FMAs
__constant__ float kTaps[11] = {0x1.0d957p-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c3ep-3f, 0x1.10656p-2f,
                             0x1.b43c3ep-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f, 0x1.0d957p-10f};
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

struct SsimParams {
    int H, W, Hv, Wv;  // image; valid map (H - 10) x (W - 10)
    const float* rgb;  // [H,W,3]
    const uint8_t* gt_u8;
    const float* gt_f32;
    const float* mask;  // [H,W,1] or null
};

__device__ __forceinline__ float ssim_gt(const SsimParams& p, long long e) {
    return p.gt_u8 ? (float)p.gt_u8[e] / 255.0f : p.gt_f32[e];
}

static __device__ __forceinline__ float ssim_block_sum(float v, float* smem, int nthreads) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 32) {
        t = threadIdx.x < nthreads / 32 ? smem[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// partial[3][nblocks]: per-CTA sums of the SSIM map per channel; maps: a, b, c per channel
__global__ void __launch_bounds__(SSIM_THREADS) ssim_fwd_kernel(const SsimParams p, float* __restrict__ maps, float* __restrict__ partial) {
    __shared__ float sx[SSIM_R][SSIM_C * 3], sy[SSIM_R][SSIM_C * 3];
    __shared__ float sh[5][SSIM_R][SSIM_TW];
    __shared__ float red[SSIM_THREADS / 32];
    const int ox0 = blockIdx.x * SSIM_TW, oy0 = blockIdx.y * SSIM_TH;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;

    // tile + halo of x = gt*mask and y = rgb*mask, channels interleaved; zero outside the image (never read by a valid output)
    for (int e = threadIdx.x; e < SSIM_R * SSIM_C * 3; e += SSIM_THREADS) {
        const int r = e / (SSIM_C * 3), k = e - r * (SSIM_C * 3);
        const int gy = oy0 + r, gx = ox0 + k / 3;
        float x = 0.f, y = 0.f;
        if (gy < p.H && gx < p.W) {
            const long long pix = (long long)gy * p.W + gx;
            const long long i = (long long)gy * p.W * 3 + (long long)ox0 * 3 + k;
            x = ssim_gt(p, i);
            y = p.rgb[i];
            if (p.mask) {
                const float m = p.mask[pix];
                x *= m;
                y *= m;
            }
        }
        sx[r][k] = x;
        sy[r][k] = y;
    }
    __syncthreads();

    const long long plane = (long long)p.Hv * p.Wv;
    float tot[3];
#pragma unroll 1
    for (int c = 0; c < 3; ++c) {
        // horizontal pass over every staged row
        for (int e = threadIdx.x; e < SSIM_R * SSIM_TW; e += SSIM_THREADS) {
            const int r = e / SSIM_TW, j = e - r * SSIM_TW;
            float m1 = 0.f, m2 = 0.f, m11 = 0.f, m22 = 0.f, m12 = 0.f;
#pragma unroll
            for (int t = 0; t < 11; ++t) {
                const float x = sx[r][(j + t) * 3 + c], y = sy[r][(j + t) * 3 + c];
                const float xx = x * x, yy = y * y, xy = x * y;
                m1 = fmaf(kTaps[t], x, m1);
                m2 = fmaf(kTaps[t], y, m2);
                m11 = fmaf(kTaps[t], xx, m11);
                m22 = fmaf(kTaps[t], yy, m22);
                m12 = fmaf(kTaps[t], xy, m12);
            }
            sh[0][r][j] = m1;
            sh[1][r][j] = m2;
            sh[2][r][j] = m11;
            sh[3][r][j] = m22;
            sh[4][r][j] = m12;
        }
        __syncthreads();
        // vertical pass: the thread's two adjacent output rows read the 12 staged rows they share once
        float mom[2][5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            float o0 = 0.f, o1 = 0.f;
#pragma unroll
            for (int u = 0; u < 12; ++u) {
                const float v = sh[k][2 * ty + u][tx];
                if (u < 11) o0 = fmaf(kTaps[u], v, o0);
                if (u > 0) o1 = fmaf(kTaps[u - 1], v, o1);
            }
            mom[0][k] = o0;
            mom[1][k] = o1;
        }
        float s_sum = 0.f;
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int i = oy0 + 2 * ty + s, j = ox0 + tx;
            if (i < p.Hv && j < p.Wv) {
                const float mu1 = mom[s][0], mu2 = mom[s][1], e11 = mom[s][2], e22 = mom[s][3], e12 = mom[s][4];
                const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
                const float s1 = e11 - mu1_sq, s2 = e22 - mu2_sq, s12 = e12 - mu12;
                const float A = 2.f * mu12 + kC1, B = mu1_sq + mu2_sq + kC1;
                const float Cn = 2.f * s12 + kC2, D = s1 + s2 + kC2;
                const float cs = Cn / D, l = A / B;
                s_sum += l * cs;
                // S = l * cs with l = A / B, cs = Cn / D; sigma_y^2 = E[y^2] - mu_y^2, sigma_xy = E[xy] - mu_x mu_y
                const float dl = (2.f * mu1 - 2.f * mu2 * l) / B;     // dl / dmu_y
                const float dcs = (2.f * mu2 * cs - 2.f * mu1) / D;   // dcs / dmu_y
                const long long o = (long long)i * p.Wv + j;
                float* mc = maps + (long long)(3 * c) * plane;
                mc[o] = dl * cs + l * dcs;          // a
                mc[plane + o] = -l * cs / D;        // b = dS / dE[y^2] = -l Cn / D^2
                mc[2 * plane + o] = 2.f * l / D;    // c = dS / dE[xy]
            }
        }
        tot[c] = ssim_block_sum(s_sum, red, SSIM_THREADS);  // its barriers also free sh for the next channel
    }
    if (threadIdx.x == 0) {
        const int nb = gridDim.x * gridDim.y, b = blockIdx.y * gridDim.x + blockIdx.x;
        partial[b] = tot[0];
        partial[nb + b] = tot[1];
        partial[2 * nb + b] = tot[2];
    }
}

// *loss = weight * (1 - mean): the per-channel means of the map, then their mean (torch: map.flatten(2).mean(-1).mean())
__global__ void __launch_bounds__(SSIM_FINISH_THREADS) ssim_finish_kernel(const float* __restrict__ partial, int nblocks, long long count,
                                                                          float weight, float* __restrict__ loss) {
    __shared__ float smem[SSIM_FINISH_THREADS / 32];
    float s[3] = {0.f, 0.f, 0.f};
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
        s[0] += partial[i];
        s[1] += partial[nblocks + i];
        s[2] += partial[2 * nblocks + i];
    }
    float m[3];
    for (int c = 0; c < 3; ++c) m[c] = ssim_block_sum(s[c], smem, SSIM_FINISH_THREADS) / (float)count;
    if (threadIdx.x == 0) *loss = weight * (1.f - (m[0] + m[1] + m[2]) / 3.f);
}

// v_rgb[H,W,3]: a CTA owns a 32 x 16 tile of image pixels and gathers the maps from the 10 rows / columns above and left of it
__global__ void __launch_bounds__(SSIM_THREADS) ssim_bwd_kernel(const SsimParams p, const float* __restrict__ maps, float weight,
                                                                const float* __restrict__ g, float* __restrict__ v_rgb) {
    __shared__ float sm[3][SSIM_R][SSIM_C];
    __shared__ float sh[3][SSIM_R][SSIM_TW];
    const int qx0 = blockIdx.x * SSIM_TW, qy0 = blockIdx.y * SSIM_TH;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const long long plane = (long long)p.Hv * p.Wv;
    const float k = -weight * (g ? g[0] : 1.f) / (3.f * (float)plane);
    float v[2][3];
#pragma unroll 1
    for (int c = 0; c < 3; ++c) {
        const float* mc = maps + (long long)(3 * c) * plane;
        for (int e = threadIdx.x; e < 3 * SSIM_R * SSIM_C; e += SSIM_THREADS) {
            const int m = e / (SSIM_R * SSIM_C), rem = e - m * (SSIM_R * SSIM_C);
            const int r = rem / SSIM_C, cc = rem - r * SSIM_C;
            const int py = qy0 - 10 + r, px = qx0 - 10 + cc;
            sm[m][r][cc] = (py >= 0 && py < p.Hv && px >= 0 && px < p.Wv) ? mc[m * plane + (long long)py * p.Wv + px] : 0.f;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < 3 * SSIM_R * SSIM_TW; e += SSIM_THREADS) {
            const int m = e / (SSIM_R * SSIM_TW), rem = e - m * (SSIM_R * SSIM_TW);
            const int r = rem / SSIM_TW, j = rem - r * SSIM_TW;
            float s = 0.f;
#pragma unroll
            for (int t = 0; t < 11; ++t) s = fmaf(kTaps[t], sm[m][r][j + 10 - t], s);
            sh[m][r][j] = s;
        }
        __syncthreads();
        // vertical pass: the thread's two adjacent rows read the 12 staged rows they share once
        float gm[2][3];
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            float o0 = 0.f, o1 = 0.f;
#pragma unroll
            for (int u = 0; u < 12; ++u) {
                const float x = sh[m][2 * ty + u][tx];
                if (u < 11) o0 = fmaf(kTaps[10 - u], x, o0);
                if (u > 0) o1 = fmaf(kTaps[11 - u], x, o1);
            }
            gm[0][m] = o0;
            gm[1][m] = o1;
        }
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int qy = qy0 + 2 * ty + s, qx = qx0 + tx;
            v[s][c] = 0.f;
            if (qy < p.H && qx < p.W) {
                const float ga = gm[s][0], gb = gm[s][1], gc = gm[s][2];
                const long long pix = (long long)qy * p.W + qx;
                const float m = p.mask ? p.mask[pix] : 1.f;
                const float x = ssim_gt(p, pix * 3 + c) * m, y = p.rgb[pix * 3 + c] * m;
                v[s][c] = k * fmaf(x, gc, fmaf(2.f * y, gb, ga)) * m;
            }
        }
        __syncthreads();  // sm / sh are restaged for the next channel
    }
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int qy = qy0 + 2 * ty + s, qx = qx0 + tx;
        if (qy < p.H && qx < p.W) {
            float* o = v_rgb + ((long long)qy * p.W + qx) * 3;
            o[0] = v[s][0];
            o[1] = v[s][1];
            o[2] = v[s][2];
        }
    }
}

static dim3 ssim_fwd_grid(int H, int W) { return dim3((W - 10 + SSIM_TW - 1) / SSIM_TW, (H - 10 + SSIM_TH - 1) / SSIM_TH); }

static size_t ssim_partial_bytes(int H, int W) {
    const dim3 g = ssim_fwd_grid(H, W);
    return ((sizeof(float) * 3 * g.x * g.y) + 255) / 256 * 256;  // the maps start 256-byte aligned
}

static int ssim_fill(SsimParams& p, int H, int W, const sgn_loss_in* in, const char* who) {
    SGN_REQUIRE(in, "%s: null input", who);
    SGN_REQUIRE(H >= 11 && W >= 11, "%s: the 11 x 11 SSIM window needs an image of at least 11 x 11 pixels, got %d x %d", who, H, W);
    SGN_REQUIRE(in->rgb, "%s: rgb is null", who);
    SGN_REQUIRE((in->gt_u8 != nullptr) != (in->gt_f32 != nullptr), "%s: exactly one of gt_u8 / gt_f32 must be given", who);
    p.H = H; p.W = W; p.Hv = H - 10; p.Wv = W - 10;
    p.rgb = in->rgb; p.gt_u8 = in->gt_u8; p.gt_f32 = in->gt_f32; p.mask = in->mask;
    return SGN_OK;
}

extern "C" size_t sgn_ssim_workspace_bytes(int H, int W) {
    if (H < 11 || W < 11) return 0;
    return ssim_partial_bytes(H, W) + sizeof(float) * 9 * (size_t)(H - 10) * (size_t)(W - 10);
}

extern "C" int sgn_ssim_fwd(int H, int W, const sgn_loss_in* in, float weight, float* loss, void* workspace, size_t workspace_bytes,
                            void* stream_) {
    SGN_RANGE("sgn_ssim_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SsimParams p;
    if (int rc = ssim_fill(p, H, W, in, "sgn_ssim_fwd")) return rc;
    SGN_REQUIRE(loss && workspace, "sgn_ssim_fwd: null output or workspace");
    if (workspace_bytes < sgn_ssim_workspace_bytes(H, W)) {
        sgn_set_error("sgn_ssim_fwd: workspace too small (%zu bytes, needs %zu)", workspace_bytes, sgn_ssim_workspace_bytes(H, W));
        return SGN_ERR_WORKSPACE;
    }
    const dim3 grid = ssim_fwd_grid(H, W);
    float* partial = (float*)workspace;
    float* maps = (float*)((char*)workspace + ssim_partial_bytes(H, W));
    ssim_fwd_kernel<<<grid, SSIM_THREADS, 0, stream>>>(p, maps, partial);
    SGN_CHECK_LAUNCH("ssim_fwd_kernel");
    ssim_finish_kernel<<<1, SSIM_FINISH_THREADS, 0, stream>>>(partial, (int)(grid.x * grid.y), (long long)p.Hv * p.Wv, weight, loss);
    SGN_CHECK_LAUNCH("ssim_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_ssim_bwd(int H, int W, const sgn_loss_in* in, float weight, const float* grad_loss, const void* workspace, float* v_rgb,
                            void* stream_) {
    SGN_RANGE("sgn_ssim_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SsimParams p;
    if (int rc = ssim_fill(p, H, W, in, "sgn_ssim_bwd")) return rc;
    SGN_REQUIRE(workspace && v_rgb, "sgn_ssim_bwd: null workspace or output");
    const float* maps = (const float*)((const char*)workspace + ssim_partial_bytes(H, W));
    const dim3 grid((W + SSIM_TW - 1) / SSIM_TW, (H + SSIM_TH - 1) / SSIM_TH);
    ssim_bwd_kernel<<<grid, SSIM_THREADS, 0, stream>>>(p, maps, weight, grad_loss, v_rgb);
    SGN_CHECK_LAUNCH("ssim_bwd_kernel");
    return SGN_OK;
}
