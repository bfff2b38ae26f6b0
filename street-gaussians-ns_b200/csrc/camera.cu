// Camera pose correction (nerfstudio CameraOptimizer, mode "SO3xR3"): pose_adjustment row -> device view, the regulariser
// and the two metrics forward; the view cotangent and the regulariser's gradient back to every row.  One launch each way in
// place of the few dozen small torch launches the same terms take as tensor ops.
#include "sgn_common.cuh"

struct C2W {
    float m[12];  // camera_to_worlds 3x4, row-major
};

// R_a, t_a of x (lie_groups.exp_map_SO3xR3) and the intermediate values the backward needs
struct Adjust {
    float w[3], theta, f1, f2, K[9], Ra[9], ta[3];
};

__device__ __forceinline__ void exp_map_so3xr3(const float* __restrict__ x, Adjust& a) {
    for (int k = 0; k < 3; ++k) { a.ta[k] = x[k]; a.w[k] = x[3 + k]; }
    const float nrms = (a.w[0] * a.w[0] + a.w[1] * a.w[1]) + a.w[2] * a.w[2];
    a.theta = sqrtf(fmaxf(nrms, 1e-4f));
    const float inv = 1.f / a.theta;
    a.f1 = inv * sinf(a.theta);
    a.f2 = (inv * inv) * (1.f - cosf(a.theta));
    const float K[9] = {0.f, -a.w[2], a.w[1], a.w[2], 0.f, -a.w[0], -a.w[1], a.w[0], 0.f};
    for (int k = 0; k < 9; ++k) a.K[k] = K[k];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const float k2 = (K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j]) + K[3 * i + 2] * K[6 + j];
            a.Ra[3 * i + j] = (a.f1 * K[3 * i + j] + a.f2 * k2) + (i == j ? 1.f : 0.f);
        }
}

// c2w' = c2w [R_a t_a; 0 1]: R' = R0 R_a, t' = R0 t_a + t0
__device__ __forceinline__ void corrected_pose(const C2W& c, const Adjust& a, float Rp[9], float tp[3]) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            Rp[3 * i + j] = (c.m[4 * i] * a.Ra[j] + c.m[4 * i + 1] * a.Ra[3 + j]) + c.m[4 * i + 2] * a.Ra[6 + j];
        tp[i] = ((c.m[4 * i] * a.ta[0] + c.m[4 * i + 1] * a.ta[1]) + c.m[4 * i + 2] * a.ta[2]) + c.m[4 * i + 3];
    }
}

// One block.  Every thread sums, over its rows of pose_adjustment in ascending order, |x_t|, |x_r| (the rows' norms) and
// |x_t|^2, |x_r|^2; the block then adds the threads' sums in a fixed tree: reg = mean |x_t| w_t + mean |x_r| w_r,
// norms = {sqrt(sum |x_t|^2), sqrt(sum |x_r|^2)} -- the same bits on every run.  Thread 0 also writes the view when cam_idx >= 0.
#define CAM_THREADS 256
__device__ __forceinline__ void row_norms(const float* __restrict__ x, float& t2, float& r2) {
    t2 = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2];
    r2 = (x[3] * x[3] + x[4] * x[4]) + x[5] * x[5];
}

__global__ void __launch_bounds__(CAM_THREADS)
camera_adjust_fwd_kernel(const float* __restrict__ pose_adjustment, int num_cameras, int cam_idx, const C2W c, float* __restrict__ view,
                         float* __restrict__ reg, float* __restrict__ norms, float w_t, float w_r) {
    __shared__ float s_sum[4][CAM_THREADS];
    const int tid = threadIdx.x;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};  // sum |x_t|, sum |x_r|, sum |x_t|^2, sum |x_r|^2
    for (int r = tid; r < num_cameras; r += CAM_THREADS) {
        float t2, r2;
        row_norms(pose_adjustment + 6 * (size_t)r, t2, r2);
        acc[0] += sqrtf(t2);
        acc[1] += sqrtf(r2);
        acc[2] += t2;
        acc[3] += r2;
    }
    for (int k = 0; k < 4; ++k) s_sum[k][tid] = acc[k];
    __syncthreads();
    for (int h = CAM_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h)
            for (int k = 0; k < 4; ++k) s_sum[k][tid] += s_sum[k][tid + h];
        __syncthreads();
    }
    if (tid != 0) return;
    const float n = (float)num_cameras;
    reg[0] = (s_sum[0][0] / n) * w_t + (s_sum[1][0] / n) * w_r;
    norms[0] = sqrtf(s_sum[2][0]);
    norms[1] = sqrtf(s_sum[3][0]);
    if (cam_idx < 0) return;

    Adjust a;
    exp_map_so3xr3(pose_adjustment + 6 * (size_t)cam_idx, a);
    float Rp[9], tp[3];
    corrected_pose(c, a, Rp, tp);
    // Camera._viewmat: R = R' diag(1,-1,-1), W = R^T, c = -W t'
    for (int i = 0; i < 3; ++i) {
        const float d = i == 0 ? 1.f : -1.f;
        float W[3];
        for (int j = 0; j < 3; ++j) W[j] = Rp[3 * j + i] * d;
        for (int j = 0; j < 3; ++j) view[4 * i + j] = W[j];
        view[4 * i + 3] = ((-W[0]) * tp[0] + (-W[1]) * tp[1]) + (-W[2]) * tp[2];
        view[12 + i] = tp[i];
    }
}

// the view cotangent -> the gradient of row cam_idx (into chain[6])
__device__ void view_chain_bwd(const float* __restrict__ pose_adjustment, int cam_idx, const C2W& c, const float* __restrict__ v_view,
                               float* chain) {
    Adjust a;
    exp_map_so3xr3(pose_adjustment + 6 * (size_t)cam_idx, a);
    float Rp[9], tp[3];
    corrected_pose(c, a, Rp, tp);
    float gW[9], gc[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) gW[3 * i + j] = v_view[4 * i + j];
        gc[i] = v_view[4 * i + 3];
    }
    // c = -W t':  v_W -= v_c t'^T,  v_t' = -W^T v_c   (W[i][j] = d_i R'[j][i])
    float gtp[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < 3; ++i) {
        const float d = i == 0 ? 1.f : -1.f;
        for (int j = 0; j < 3; ++j) {
            gW[3 * i + j] -= gc[i] * tp[j];
            gtp[j] -= d * Rp[3 * j + i] * gc[i];
        }
    }
    // W[i][j] = d_i R'[j][i]  ->  v_R'[j][i] = d_i v_W[i][j];  R' = R0 R_a  ->  v_Ra = R0^T v_R';  t' = R0 t_a + t0  ->  v_ta = R0^T v_t'
    float gRp[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) gRp[3 * j + i] = (i == 0 ? 1.f : -1.f) * gW[3 * i + j];
    float gRa[9], gta[3];
    for (int p = 0; p < 3; ++p) {
        for (int q = 0; q < 3; ++q) gRa[3 * p + q] = c.m[p] * gRp[q] + c.m[4 + p] * gRp[3 + q] + c.m[8 + p] * gRp[6 + q];
        gta[p] = c.m[p] * gtp[0] + c.m[4 + p] * gtp[1] + c.m[8 + p] * gtp[2];
    }
    // R_a = I + f1 K + f2 K^2:  v_f1 = <v_Ra, K>, v_f2 = <v_Ra, K^2>, v_K = f1 v_Ra + f2 (v_Ra K^T + K^T v_Ra)
    const float* K = a.K;
    float gf1 = 0.f, gf2 = 0.f, gK[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const float k2 = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
            gf1 += gRa[3 * i + j] * K[3 * i + j];
            gf2 += gRa[3 * i + j] * k2;
            float s = 0.f;
            for (int k = 0; k < 3; ++k) s += gRa[3 * i + k] * K[3 * j + k] + K[3 * k + i] * gRa[3 * k + j];
            gK[3 * i + j] = a.f1 * gRa[3 * i + j] + a.f2 * s;
        }
    float gw[3] = {gK[7] - gK[5], gK[2] - gK[6], gK[3] - gK[1]};
    // theta = sqrt(max(|w|^2, 1e-4)): below the clamp f1, f2 are constants and w gets nothing through them
    const float nrms = (a.w[0] * a.w[0] + a.w[1] * a.w[1]) + a.w[2] * a.w[2];
    if (nrms >= 1e-4f) {
        const float t = a.theta, s = sinf(t), co = cosf(t);
        const float df1 = (t * co - s) / (t * t), df2 = (t * s - 2.f * (1.f - co)) / (t * t * t);
        const float gt = gf1 * df1 + gf2 * df2;
        for (int k = 0; k < 3; ++k) gw[k] += gt * a.w[k] / t;
    }
    for (int k = 0; k < 3; ++k) { chain[k] = gta[k]; chain[3 + k] = gw[k]; }
}

// One block writes every row of v_x: the regulariser's share g_reg (w_t / n x_t / |x_t| and w_r / n x_r / |x_r|, zero for a
// zero norm, as torch's norm backward gives) plus, in row cam_idx, the chain from v_view.  g_reg / v_view NULL: no share.
__global__ void __launch_bounds__(CAM_THREADS)
camera_adjust_bwd_kernel(const float* __restrict__ pose_adjustment, int num_cameras, int cam_idx, const C2W c,
                         const float* __restrict__ v_view, const float* __restrict__ g_reg, float w_t, float w_r,
                         float* __restrict__ v_x) {
    __shared__ float s_chain[6];
    const int tid = threadIdx.x;
    if (tid == 0) {
        if (cam_idx >= 0 && v_view) view_chain_bwd(pose_adjustment, cam_idx, c, v_view, s_chain);
        else for (int k = 0; k < 6; ++k) s_chain[k] = 0.f;
    }
    __syncthreads();
    const float g = g_reg ? g_reg[0] : 0.f;
    const float gt = g * w_t / (float)num_cameras, gr = g * w_r / (float)num_cameras;
    for (int r = tid; r < num_cameras; r += CAM_THREADS) {
        const float* x = pose_adjustment + 6 * (size_t)r;
        float t2, r2;
        row_norms(x, t2, r2);
        const float nt = sqrtf(t2), nr = sqrtf(r2);
        const float ft = nt > 0.f ? gt / nt : 0.f, fr = nr > 0.f ? gr / nr : 0.f;
        float* out = v_x + 6 * (size_t)r;
        for (int k = 0; k < 3; ++k) {
            out[k] = ft * x[k] + (r == cam_idx ? s_chain[k] : 0.f);
            out[3 + k] = fr * x[3 + k] + (r == cam_idx ? s_chain[3 + k] : 0.f);
        }
    }
}

static int adjust_args(const char* who, const float* pose_adjustment, int num_cameras, int cam_idx, const float* c2w, C2W& c) {
    SGN_REQUIRE(pose_adjustment, "%s: null pose_adjustment", who);
    SGN_REQUIRE(num_cameras >= 1, "%s: %d cameras", who, num_cameras);
    SGN_REQUIRE(cam_idx >= -1 && cam_idx < num_cameras, "%s: camera index %d outside [0, %d) (or -1: no view)", who, cam_idx, num_cameras);
    SGN_REQUIRE(cam_idx < 0 || c2w, "%s: null c2w", who);
    for (int k = 0; k < 12; ++k) c.m[k] = cam_idx >= 0 ? c2w[k] : 0.f;
    return SGN_OK;
}

extern "C" int sgn_camera_adjust_fwd(const float* pose_adjustment, int num_cameras, int cam_idx, const float* c2w, float w_t, float w_r,
                                     float* view, float* reg, float* norms, void* stream) {
    SGN_RANGE("sgn_camera_adjust_fwd");
    C2W c;
    if (int rc = adjust_args("sgn_camera_adjust_fwd", pose_adjustment, num_cameras, cam_idx, c2w, c)) return rc;
    SGN_REQUIRE(reg && norms && (cam_idx < 0 || view), "sgn_camera_adjust_fwd: null view, reg or norms");
    camera_adjust_fwd_kernel<<<1, CAM_THREADS, 0, (cudaStream_t)stream>>>(pose_adjustment, num_cameras, cam_idx, c, view, reg, norms, w_t,
                                                                          w_r);
    SGN_CHECK_LAUNCH("camera_adjust_fwd_kernel");
    return SGN_OK;
}

extern "C" int sgn_camera_adjust_bwd(const float* pose_adjustment, int num_cameras, int cam_idx, const float* c2w, float w_t, float w_r,
                                     const float* v_view, const float* g_reg, float* v_pose_adjustment, void* stream) {
    SGN_RANGE("sgn_camera_adjust_bwd");
    C2W c;
    if (int rc = adjust_args("sgn_camera_adjust_bwd", pose_adjustment, num_cameras, cam_idx, c2w, c)) return rc;
    SGN_REQUIRE(v_pose_adjustment, "sgn_camera_adjust_bwd: null v_pose_adjustment");
    camera_adjust_bwd_kernel<<<1, CAM_THREADS, 0, (cudaStream_t)stream>>>(pose_adjustment, num_cameras, cam_idx, c, v_view, g_reg, w_t, w_r,
                                                                          v_pose_adjustment);
    SGN_CHECK_LAUNCH("camera_adjust_bwd_kernel");
    return SGN_OK;
}
