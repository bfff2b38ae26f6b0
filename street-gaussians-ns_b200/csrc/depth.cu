// Lidar depth supervision: a sweep projected into a sparse depth map for one camera, the L1 depth term on the rendered depth
// and its cotangent, and the depth metrics of eval.  Street Gaussians supervises the rendered depth with lidar; the
// reference's datamanager carries the target as batch["depth_image"] (sgn_datamanager.py:360-361) and its eval asks for a
// depth_result (sgn_splatfacto.py:1160-1168) that it never defines.
//
// Map: a point's camera-space position, depth and pixel centre are the projection's own arithmetic (sgn_exact.cuh: pv, then
// rw = 1 / (z + 1e-6), u = (pv.x * rw) * fx + cx), through the never-contracted xf operations: a point at a Gaussian's mean
// lands on that Gaussian's xy with that Gaussian's depth record.  The nearest return of a pixel wins, by atomicMin on the bits
// of a positive float (the order of the points does not change the minimum: the map is the same bits every run).
//
// Loss and metrics: per-block partials summed in fp64 (the pixel counts as int64), then added in a fixed order by a one-block
// finish kernel, as loss.cu / metrics.cu: deterministic run to run.  The valid-pixel count stays on the device.
#include <math.h>

#include <algorithm>

#include "sgn_exact.cuh"

#define DEPTH_THREADS 256
#define DEPTH_BLOCKS 1056  // 132 SMs (H100 SXM) x 8 resident blocks of 256 threads
#define DEPTH_EMPTY 0x7f800000u  // +inf: above the bits of every finite positive depth

__global__ void __launch_bounds__(DEPTH_THREADS) depth_fill_kernel(unsigned* __restrict__ map, long long P) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
        map[i] = DEPTH_EMPTY;
}

// A[12]: the camera-from-point 3x4, row-major (the viewmat, or the viewmat composed with the sweep's to_world)
struct LidarParams {
    float A[12];
    float fx, fy, cx, cy, clip_thresh;
    int width, height;
};

__global__ void __launch_bounds__(DEPTH_THREADS) lidar_scatter_kernel(const LidarParams p, const float* __restrict__ points, long long M,
                                                                      unsigned* __restrict__ map) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
        const xf m[3] = {xf(points[3 * i]), xf(points[3 * i + 1]), xf(points[3 * i + 2])};
        xf pv[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) pv[r] = ((xf(p.A[4 * r]) * m[0] + xf(p.A[4 * r + 1]) * m[1]) + xf(p.A[4 * r + 2]) * m[2]) + xf(p.A[4 * r + 3]);
        const float z = pv[2].v;
        if (!(z > p.clip_thresh)) continue;  // also drops NaN
        const xf rw = xf(1.f) / (pv[2] + xf(1e-6f));
        const float u = ((pv[0] * rw) * xf(p.fx) + xf(p.cx)).v;
        const float v = ((pv[1] * rw) * xf(p.fy) + xf(p.cy)).v;
        if (!(u >= 0.f && u < (float)p.width && v >= 0.f && v < (float)p.height)) continue;
        const long long pix = (long long)(int)floorf(v) * p.width + (int)floorf(u);
        atomicMin(map + pix, __float_as_uint(z));  // z > clip_thresh >= 0: unsigned order of the bits = order of the depths
    }
}

__global__ void __launch_bounds__(DEPTH_THREADS) depth_finish_map_kernel(unsigned* __restrict__ map, long long P) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
        if (map[i] == DEPTH_EMPTY) map[i] = 0u;  // 0.0f: no return
}

extern "C" int sgn_lidar_depth_map(const float* points, int64_t M, const sgn_camera* cam, const float* to_world, float* depth_map,
                                   void* stream_) {
    SGN_RANGE("sgn_lidar_depth_map");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(cam && depth_map, "sgn_lidar_depth_map: null camera or output");
    SGN_REQUIRE(cam->width > 0 && cam->height > 0, "sgn_lidar_depth_map: empty image %dx%d", cam->width, cam->height);
    SGN_REQUIRE(M >= 0 && (M == 0 || points), "sgn_lidar_depth_map: null points with M = %lld", (long long)M);
    SGN_REQUIRE(cam->clip_thresh >= 0.f, "sgn_lidar_depth_map: clip_thresh %g < 0 (the nearest return is chosen on the bits of a positive float)",
                (double)cam->clip_thresh);
    LidarParams p;
    if (to_world) {  // camera-from-sweep = viewmat * [to_world; 0 0 0 1], composed in fp64 and rounded once
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c) {
                double s = c == 3 ? (double)cam->viewmat[4 * r + 3] : 0.0;
                for (int k = 0; k < 3; ++k) s += (double)cam->viewmat[4 * r + k] * (double)to_world[4 * k + c];
                p.A[4 * r + c] = (float)s;
            }
    } else {
        for (int k = 0; k < 12; ++k) p.A[k] = cam->viewmat[k];
    }
    p.fx = cam->fx; p.fy = cam->fy; p.cx = cam->cx; p.cy = cam->cy; p.clip_thresh = cam->clip_thresh;
    p.width = cam->width; p.height = cam->height;
    const long long P = (long long)cam->width * cam->height;
    unsigned* map = reinterpret_cast<unsigned*>(depth_map);
    const int fill_blocks = (int)std::min<long long>((P + DEPTH_THREADS - 1) / DEPTH_THREADS, DEPTH_BLOCKS);
    depth_fill_kernel<<<fill_blocks, DEPTH_THREADS, 0, stream>>>(map, P);
    SGN_CHECK_LAUNCH("depth_fill_kernel");
    if (M > 0) {
        const int blocks = (int)std::min<long long>((M + DEPTH_THREADS - 1) / DEPTH_THREADS, 4 * DEPTH_BLOCKS);
        lidar_scatter_kernel<<<blocks, DEPTH_THREADS, 0, stream>>>(p, points, M, map);
        SGN_CHECK_LAUNCH("lidar_scatter_kernel");
    }
    depth_finish_map_kernel<<<fill_blocks, DEPTH_THREADS, 0, stream>>>(map, P);
    SGN_CHECK_LAUNCH("depth_finish_map_kernel");
    return SGN_OK;
}

// ---- loss and metrics ------------------------------------------------------------------------------------------------

struct DepthParams {
    long long P;
    const float* depth;
    const float* target;
    const float* mask;  // [P] or null
};

__device__ __forceinline__ bool depth_valid(const DepthParams& p, long long i) {
    return p.target[i] > 0.f && (!p.mask || p.mask[i] != 0.f);
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < DEPTH_THREADS / 32) t = smem[threadIdx.x];
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

// partial: double[gridDim.x] = sum |D - T| over the valid pixels, then int64[gridDim.x] = their count
__global__ void __launch_bounds__(DEPTH_THREADS) depth_loss_fwd_kernel(const DepthParams p, double* __restrict__ partial) {
    __shared__ double s_red[DEPTH_THREADS / 32];
    __shared__ long long s_red_i[DEPTH_THREADS / 32];
    double s = 0.0;
    long long n = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        if (depth_valid(p, i)) {
            s += (double)fabsf(__fsub_rn(p.depth[i], p.target[i]));
            ++n;
        }
    }
    const double a = block_sum(s, s_red);
    const long long b = block_sum(n, s_red_i);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = a;
        reinterpret_cast<long long*>(partial + gridDim.x)[blockIdx.x] = b;
    }
}

// loss = w * sum / n_valid (exactly 0 when n_valid = 0)
__global__ void __launch_bounds__(DEPTH_THREADS) depth_loss_finish_kernel(const double* __restrict__ partial, int nblocks, float w,
                                                                          float* __restrict__ loss, int* __restrict__ n_valid) {
    __shared__ double s_red[DEPTH_THREADS / 32];
    __shared__ long long s_red_i[DEPTH_THREADS / 32];
    double s = 0.0;
    long long n = 0;
    const long long* pn = reinterpret_cast<const long long*>(partial + nblocks);
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { s += partial[i]; n += pn[i]; }
    s = block_sum(s, s_red);
    n = block_sum(n, s_red_i);
    if (threadIdx.x == 0) {
        *loss = n > 0 ? (float)((double)w * (s / (double)n)) : 0.f;
        *n_valid = (int)n;
    }
}

// v_depth = g * w * sign(D - T) / n_valid on the valid pixels, 0 elsewhere
__global__ void __launch_bounds__(DEPTH_THREADS) depth_loss_bwd_kernel(const DepthParams p, float w, const int* __restrict__ n_valid,
                                                                       const float* __restrict__ g, float* __restrict__ v_depth) {
    const int n = *n_valid;
    const float k = n > 0 ? (g ? *g : 1.f) * w / (float)n : 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        float v = 0.f;
        if (n > 0 && depth_valid(p, i)) {
            const float d = __fsub_rn(p.depth[i], p.target[i]);
            v = d > 0.f ? k : (d < 0.f ? -k : 0.f);
        }
        v_depth[i] = v;
    }
}

static int fill(DepthParams& p, int H, int W, const float* depth, const float* target, const float* mask, const char* who) {
    SGN_REQUIRE(H > 0 && W > 0, "%s: empty image %dx%d", who, H, W);
    SGN_REQUIRE(depth && target, "%s: null depth or target", who);
    p.P = (long long)H * W;
    p.depth = depth; p.target = target; p.mask = mask;
    return SGN_OK;
}

extern "C" size_t sgn_depth_scratch_bytes(void) { return (4 * sizeof(double) + 4 * sizeof(long long)) * DEPTH_BLOCKS; }

extern "C" int sgn_depth_loss_fwd(int H, int W, const float* depth, const float* target, const float* mask, float weight, float* loss,
                                  int32_t* n_valid, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_depth_loss_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    DepthParams p;
    if (int rc = fill(p, H, W, depth, target, mask, "sgn_depth_loss_fwd")) return rc;
    SGN_REQUIRE(loss && n_valid && scratch, "sgn_depth_loss_fwd: null output or scratch");
    if (scratch_bytes < sgn_depth_scratch_bytes()) {
        sgn_set_error("sgn_depth_loss_fwd: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_depth_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    depth_loss_fwd_kernel<<<DEPTH_BLOCKS, DEPTH_THREADS, 0, stream>>>(p, (double*)scratch);
    SGN_CHECK_LAUNCH("depth_loss_fwd_kernel");
    depth_loss_finish_kernel<<<1, DEPTH_THREADS, 0, stream>>>((const double*)scratch, DEPTH_BLOCKS, weight, loss, n_valid);
    SGN_CHECK_LAUNCH("depth_loss_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_depth_loss_bwd(int H, int W, const float* depth, const float* target, const float* mask, float weight,
                                  const int32_t* n_valid, const float* grad_loss, float* v_depth, void* stream_) {
    SGN_RANGE("sgn_depth_loss_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    DepthParams p;
    if (int rc = fill(p, H, W, depth, target, mask, "sgn_depth_loss_bwd")) return rc;
    SGN_REQUIRE(n_valid && v_depth, "sgn_depth_loss_bwd: null n_valid or output");
    depth_loss_bwd_kernel<<<DEPTH_BLOCKS, DEPTH_THREADS, 0, stream>>>(p, weight, n_valid, grad_loss, v_depth);
    SGN_CHECK_LAUNCH("depth_loss_bwd_kernel");
    return SGN_OK;
}

// partial: double[4][gridDim.x] = {sum |d-t|/t, sum (d-t)^2/t, sum (d-t)^2, sum (log d - log t)^2}, then
// int64[4][gridDim.x] = {n(r < 1.25), n(r < 1.25^2), n(r < 1.25^3), n_valid}; d = max(D, 1e-3f), r = max(d/t, t/d)
__global__ void __launch_bounds__(DEPTH_THREADS) depth_metrics_kernel(const DepthParams p, double* __restrict__ partial) {
    __shared__ double s_red[DEPTH_THREADS / 32];
    __shared__ long long s_red_i[DEPTH_THREADS / 32];
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    long long c[4] = {0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.P; i += (long long)gridDim.x * blockDim.x) {
        if (!depth_valid(p, i)) continue;
        const double d = (double)fmaxf(p.depth[i], 1e-3f), t = (double)p.target[i];
        const double e = d - t, lg = log(d) - log(t), r = fmax(d / t, t / d);
        s[0] += fabs(e) / t;
        s[1] += e * e / t;
        s[2] += e * e;
        s[3] += lg * lg;
        c[0] += r < 1.25;
        c[1] += r < 1.5625;
        c[2] += r < 1.953125;
        c[3] += 1;
    }
    double a[4];
    long long b[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = block_sum(s[k], s_red);
#pragma unroll
    for (int k = 0; k < 4; ++k) b[k] = block_sum(c[k], s_red_i);
    if (threadIdx.x == 0) {
        const int nb = gridDim.x;
        long long* pi = reinterpret_cast<long long*>(partial + 4 * nb);
        for (int k = 0; k < 4; ++k) {
            partial[k * nb + blockIdx.x] = a[k];
            pi[k * nb + blockIdx.x] = b[k];
        }
    }
}

// out[8] = {abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3, n_valid}, each rounded once to fp32; the means are NaN when n_valid = 0
__global__ void __launch_bounds__(DEPTH_THREADS) depth_metrics_finish_kernel(const double* __restrict__ partial, int nblocks,
                                                                             float* __restrict__ out) {
    __shared__ double s_red[DEPTH_THREADS / 32];
    __shared__ long long s_red_i[DEPTH_THREADS / 32];
    double s[4];
    long long c[4];
    const long long* pi = reinterpret_cast<const long long*>(partial + 4 * nblocks);
    for (int k = 0; k < 4; ++k) {
        double x = 0.0;
        long long y = 0;
        for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { x += partial[k * nblocks + i]; y += pi[k * nblocks + i]; }
        s[k] = block_sum(x, s_red);
        c[k] = block_sum(y, s_red_i);
    }
    if (threadIdx.x == 0) {
        const double n = (double)c[3];  // 0 / 0 = NaN
        out[0] = (float)(s[0] / n);
        out[1] = (float)(s[1] / n);
        out[2] = (float)sqrt(s[2] / n);
        out[3] = (float)sqrt(s[3] / n);
        out[4] = (float)((double)c[0] / n);
        out[5] = (float)((double)c[1] / n);
        out[6] = (float)((double)c[2] / n);
        out[7] = (float)c[3];
    }
}

extern "C" int sgn_depth_metrics(int H, int W, const float* depth, const float* target, const float* mask, float* out, void* scratch,
                                 size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_depth_metrics");
    cudaStream_t stream = (cudaStream_t)stream_;
    DepthParams p;
    if (int rc = fill(p, H, W, depth, target, mask, "sgn_depth_metrics")) return rc;
    SGN_REQUIRE(out && scratch, "sgn_depth_metrics: null output or scratch");
    if (scratch_bytes < sgn_depth_scratch_bytes()) {
        sgn_set_error("sgn_depth_metrics: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_depth_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    depth_metrics_kernel<<<DEPTH_BLOCKS, DEPTH_THREADS, 0, stream>>>(p, (double*)scratch);
    SGN_CHECK_LAUNCH("depth_metrics_kernel");
    depth_metrics_finish_kernel<<<1, DEPTH_THREADS, 0, stream>>>((const double*)scratch, DEPTH_BLOCKS, out);
    SGN_CHECK_LAUNCH("depth_metrics_finish_kernel");
    return SGN_OK;
}
