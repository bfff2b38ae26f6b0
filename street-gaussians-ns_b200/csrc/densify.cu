// Densification statistics (SURVEY.md 8f rank 3, first half): what every sub-model's `after_train` callback
// accumulates after each backward (street_gaussians_ns/sgn_splatfacto.py:513-541), for all visible sub-models
// of a frame in ONE launch over the frame's row space instead of ~8 torch launches per sub-model (33 sub-models):
//
//   grads = ||xys.grad||                      (pixel-space mean gradient: v_records[:, 0:2]; sgn_densify_stats_abs:
//                                              the absolute one, v_absxy[:, 0:2] of sgn_blend_bwd_absgrad)
//   first call of a sub-model:  xys_grad_norm = grads;  vis_counts = 1 (every row);  max_2Dsize = 0
//   later calls, visible rows:  xys_grad_norm += grads; vis_counts += 1
//   always, visible rows:       max_2Dsize = max(max_2Dsize, radii / max(H, W))
//
// HBM-bound: 12 B read (+12 B read-modify-write) per row.
#include "sgn_common.cuh"

// STRIDE: floats per row of the gradient input (12: v_records, 2: v_absxy); its first two are (v_x, v_y)
template <int STRIDE>
__global__ void __launch_bounds__(256)
densify_stats_kernel(const sgn_densify_segment* __restrict__ table, int nseg, int N, const float2* __restrict__ v_xy,
                     const int32_t* __restrict__ radii, float inv_max_size) {
    extern __shared__ int s_row0[];
    for (int i = threadIdx.x; i < nseg; i += blockDim.x) s_row0[i] = table[i].row0;
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_row0[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const sgn_densify_segment sg = table[lo];
    const int i = g - sg.row0;
    // rows in front of the first segment (a table whose first row0 > 0) give i < 0; rows in a gap give i >= count
    if (i < 0 || i >= sg.count) return;
    const float2 v = __ldg(v_xy + (STRIDE / 2) * (size_t)g);  // (v_x, v_y)
    // torch.linalg.vector_norm over 2 elements: sqrt(x*x + y*y)
    const float gn = sqrtf(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
    const int r = radii[g];
    const bool vis = r > 0;
    if (sg.first) {
        sg.xys_grad_norm[i] = gn;
        sg.vis_counts[i] = 1.f;
        sg.max_2Dsize[i] = vis ? fmaxf(0.f, __fmul_rn((float)r, inv_max_size)) : 0.f;
    } else if (vis) {
        sg.xys_grad_norm[i] = gn + sg.xys_grad_norm[i];
        sg.vis_counts[i] = sg.vis_counts[i] + 1.f;
        sg.max_2Dsize[i] = fmaxf(sg.max_2Dsize[i], __fmul_rn((float)r, inv_max_size));
    }
}

extern "C" size_t sgn_sizeof_densify_segment(void) { return sizeof(sgn_densify_segment); }

template <int STRIDE>
static int densify_stats(const sgn_densify_segment* table_dev, int nseg, int N, const float* v_xy, const int32_t* radii, int height,
                         int width, cudaStream_t stream) {
    SGN_REQUIRE(nseg >= 0 && N >= 0 && height > 0 && width > 0, "sgn_densify_stats: bad sizes");
    if (nseg == 0 || N == 0) return SGN_OK;
    SGN_REQUIRE(table_dev && v_xy && radii, "sgn_densify_stats: null pointer");
    SGN_REQUIRE((reinterpret_cast<uintptr_t>(v_xy) & (STRIDE == 12 ? 15u : 7u)) == 0,
                STRIDE == 12 ? "sgn_densify_stats: v_records must be 16-byte aligned" : "sgn_densify_stats_abs: v_absxy must be 8-byte aligned");
    // torch divides a CUDA tensor by a host scalar as a multiplication with the scalar's fp32 reciprocal
    // (BinaryDivTrueKernel): radii / float(max(H, W)) in the reference is radii * (1.f / max(H, W))
    const float inv_max_size = 1.0f / (float)(height > width ? height : width);
    densify_stats_kernel<STRIDE><<<(N + 255) / 256, 256, sizeof(int) * nseg, stream>>>(table_dev, nseg, N,
                                                                                     reinterpret_cast<const float2*>(v_xy), radii, inv_max_size);
    SGN_CHECK_LAUNCH("densify_stats_kernel");
    return SGN_OK;
}

extern "C" int sgn_densify_stats(const sgn_densify_segment* table_dev, int nseg, int N, const float* v_records, const int32_t* radii,
                                 int height, int width, void* stream) {
    SGN_RANGE("sgn_densify_stats");
    return densify_stats<SGN_RECORD_FLOATS>(table_dev, nseg, N, v_records, radii, height, width, (cudaStream_t)stream);
}

extern "C" int sgn_densify_stats_abs(const sgn_densify_segment* table_dev, int nseg, int N, const float* v_absxy, const int32_t* radii,
                                     int height, int width, void* stream) {
    SGN_RANGE("sgn_densify_stats_abs");
    return densify_stats<2>(table_dev, nseg, N, v_absxy, radii, height, width, (cudaStream_t)stream);
}
