// Mip-Splatting's 3D smoothing filter sizes (Yu et al. 2024, eq. 7 and the reference implementation's compute_3D_filter):
//
//   nu_i    = max over the views v that sample row i of max(fx_v, fy_v) / z_v(i)
//   sigma_i = sqrt(variance) / nu_i
//
// where view v samples row i when its camera-space depth z = (A_vm mu_i + b_vm).z exceeds `near` and its projection lands
// inside the image with a 15 % margin, u in [-0.15 W, 1.15 W] and w in [-0.15 H, 1.15 H] (bounds inclusive).  A_vm, b_vm is
// the view composed with the sub-model's object->world pose at the view's timestamp; (v, m) rows that are absent (an actor
// without a box at that timestamp) are skipped.  Rows no view samples take the largest sigma of the sampled rows (the lowest
// rate), as Mip-Splatting gives unseen points the widest filter; when no row at all is sampled every sigma is 0.
//
// Sweep: one thread per row over all views, blocks of 128 rows that never straddle sub-models (sgn_filter_sub.chunk0), so the
// (view, sub-model) transform a block reads is the same for all its threads.  Views and transforms are staged through shared
// memory in tiles of FT_TILE views.  The transform and the projection are evaluated in fp64: the sampling tests sit on exact
// boundaries, and the float64 statement they are checked against sees the same values.  The rate is reduced in registers;
// the only atomics are integer ones (a row count and the largest sigma's bit pattern, positive floats order like their
// bits), so the result does not depend on the schedule.  A second launch fills the unsampled rows.
#include "sgn_common.cuh"

#define FT_CHUNK 128   // rows per block
#define FT_TILE 64     // views per shared-memory tile

__device__ __forceinline__ int ft_sub_of(const int* s_chunk0, int nsub, int c) {
    int lo = 0, hi = nsub - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_chunk0[mid] <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(FT_CHUNK)
filter3d_sweep_kernel(const sgn_filter_sub* __restrict__ subs, int nsub, const sgn_filter_view* __restrict__ views, int V,
                      const sgn_filter_xform* __restrict__ xforms, double sqrt_var, double near, int32_t* __restrict__ stats) {
    extern __shared__ int s_chunk0[];
    __shared__ double s_A[FT_TILE][12];
    __shared__ double s_in[FT_TILE][5];  // focal = max(fx, fy), fx, fy, cx, cy
    __shared__ double s_lim[FT_TILE][4];  // u lo, u hi, w lo, w hi
    __shared__ int s_present[FT_TILE];
    __shared__ int s_any[FT_CHUNK / 32];
    __shared__ unsigned s_max[FT_CHUNK / 32];
    for (int k = threadIdx.x; k < nsub; k += blockDim.x) s_chunk0[k] = subs[k].chunk0;
    __syncthreads();
    const int si = ft_sub_of(s_chunk0, nsub, blockIdx.x);
    const sgn_filter_sub sb = subs[si];
    const int i = (blockIdx.x - sb.chunk0) * FT_CHUNK + threadIdx.x;
    const bool active = i < sb.count;
    double m[3] = {0.0, 0.0, 0.0};
    if (active) {
#pragma unroll
        for (int k = 0; k < 3; ++k) m[k] = (double)__ldg(sb.means + 3 * (size_t)i + k);
    }
    double nu = 0.0;
    for (int v0 = 0; v0 < V; v0 += FT_TILE) {
        const int nt = min(FT_TILE, V - v0);
        for (int t = threadIdx.x; t < nt; t += blockDim.x) {
            const sgn_filter_xform& x = xforms[(size_t)(v0 + t) * nsub + si];
            s_present[t] = x.present;
#pragma unroll
            for (int k = 0; k < 12; ++k) s_A[t][k] = x.M[k];
            const sgn_filter_view& vw = views[v0 + t];
            s_in[t][0] = (double)fmaxf(vw.fx, vw.fy);
            s_in[t][1] = vw.fx; s_in[t][2] = vw.fy; s_in[t][3] = vw.cx; s_in[t][4] = vw.cy;
            s_lim[t][0] = -0.15 * vw.width;  s_lim[t][1] = 1.15 * vw.width;
            s_lim[t][2] = -0.15 * vw.height; s_lim[t][3] = 1.15 * vw.height;
        }
        __syncthreads();
        for (int t = 0; t < nt; ++t) {
            if (!s_present[t]) continue;  // block-uniform
            const double* A = s_A[t];
            const double z = A[8] * m[0] + A[9] * m[1] + A[10] * m[2] + A[11];
            if (!(z > near)) continue;
            const double x = A[0] * m[0] + A[1] * m[1] + A[2] * m[2] + A[3];
            const double y = A[4] * m[0] + A[5] * m[1] + A[6] * m[2] + A[7];
            const double u = s_in[t][1] * x / z + s_in[t][3];
            const double w = s_in[t][2] * y / z + s_in[t][4];
            if (u >= s_lim[t][0] && u <= s_lim[t][1] && w >= s_lim[t][2] && w <= s_lim[t][3]) nu = fmax(nu, s_in[t][0] / z);
        }
        __syncthreads();
    }
    const bool sampled = active && nu > 0.0;
    float sigma = -1.f;  // marks an unsampled row for the fill launch
    if (sampled) sigma = (float)(sqrt_var / nu);
    if (active) sb.out[i] = sigma;
    // the block's sampled rows and largest sigma, then one integer atomic each
    const unsigned bal = __ballot_sync(0xffffffffu, sampled);
    const unsigned mx = __reduce_max_sync(0xffffffffu, sampled ? __float_as_uint(sigma) : 0u);
    if ((threadIdx.x & 31) == 0) { s_any[threadIdx.x >> 5] = __popc(bal); s_max[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        unsigned b = 0u;
#pragma unroll
        for (int k = 0; k < FT_CHUNK / 32; ++k) { n += s_any[k]; b = max(b, s_max[k]); }
        if (n > 0) {
            atomicAdd(stats, n);
            atomicMax(reinterpret_cast<unsigned*>(stats + 1), b);
        }
    }
}

__global__ void __launch_bounds__(FT_CHUNK)
filter3d_fill_kernel(const sgn_filter_sub* __restrict__ subs, int nsub, const int32_t* __restrict__ stats) {
    extern __shared__ int s_chunk0[];
    for (int k = threadIdx.x; k < nsub; k += blockDim.x) s_chunk0[k] = subs[k].chunk0;
    __syncthreads();
    const int si = ft_sub_of(s_chunk0, nsub, blockIdx.x);
    const sgn_filter_sub sb = subs[si];
    const int i = (blockIdx.x - sb.chunk0) * FT_CHUNK + threadIdx.x;
    if (i >= sb.count) return;
    if (sb.out[i] < 0.f) sb.out[i] = __uint_as_float((unsigned)stats[1]);  // 0 when no row is sampled
}

extern "C" size_t sgn_sizeof_filter_xform(void) { return sizeof(sgn_filter_xform); }

extern "C" int sgn_filter3d(const sgn_filter_sub* subs_dev, int nsub, int num_chunks, const sgn_filter_view* views_dev, int V,
                            const sgn_filter_xform* xforms_dev, double variance, double near, int32_t* stats, void* stream) {
    SGN_RANGE("sgn_filter3d");
    SGN_REQUIRE(subs_dev && stats, "sgn_filter3d: null pointer");
    SGN_REQUIRE(nsub >= 1 && nsub <= 1024, "sgn_filter3d: nsub=%d out of range [1,1024]", nsub);
    SGN_REQUIRE(num_chunks >= 0 && V >= 0, "sgn_filter3d: negative size");
    SGN_REQUIRE(V == 0 || (views_dev && xforms_dev), "sgn_filter3d: null view or transform table");
    SGN_REQUIRE(variance >= 0.0 && near >= 0.0, "sgn_filter3d: variance and near must be >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    SGN_CHECK_CUDA(cudaMemsetAsync(stats, 0, 2 * sizeof(int32_t), st));
    if (num_chunks == 0) return SGN_OK;
    filter3d_sweep_kernel<<<num_chunks, FT_CHUNK, nsub * sizeof(int), st>>>(subs_dev, nsub, views_dev, V, xforms_dev,
                                                                          sqrt(variance), near, stats);
    SGN_CHECK_LAUNCH("filter3d_sweep_kernel");
    filter3d_fill_kernel<<<num_chunks, FT_CHUNK, nsub * sizeof(int), st>>>(subs_dev, nsub, stats);
    SGN_CHECK_LAUNCH("filter3d_fill_kernel");
    return SGN_OK;
}
