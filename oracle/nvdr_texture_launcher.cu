// Launcher for nvdiffrast's own cube-map texture kernels, built into oracle/_ref/libnvdr_texture.so by oracle/nvdr_texture.py
// from a checkout of the reference (its vendored nvdiffrast, dependencies/nvdiffrast/nvdiffrast/common/texture.cu, is compiled
// in this translation unit with -DNVDR_TORCH -lineinfo, as nvdiffrast's torch plugin compiles it).  Test infrastructure only:
// the parity tests compare csrc/sky.cu with these kernels on the same directions.
//
// dr.texture(tex[None], uv, filter_mode='linear', boundary_mode='cube') with tex [6,R,R,3] and uv [1,H,W,3]: one forward
// launch of TextureFwdKernelCubeLinear1, and for the gradient one launch of TextureGradKernelCubeLinear (which also writes the
// uv gradient, hence the caller's grad_uv buffer), with the plugin's thread-block shapes (at most 8 x 8 threads).
#include "texture.cu"

static TextureKernelParams nvdr_params(const float* tex, int R, const float* uv, int H, int W) {
    TextureKernelParams p;
    memset(&p, 0, sizeof(p));
    p.tex[0] = tex;
    p.uv = uv;
    p.filterMode = TEX_MODE_LINEAR;
    p.boundaryMode = TEX_BOUNDARY_MODE_CUBE;
    p.channels = 3;
    p.imgWidth = W;
    p.imgHeight = H;
    p.texWidth = R;
    p.texHeight = R;
    p.texDepth = 1;
    p.n = 1;
    return p;
}

// the plugin's launch shapes: getLaunchBlockSize / getLaunchGridSize of the checkout's common/common.cpp, compiled into the
// same library (oracle/nvdr_texture.py), with the texture kernels' limit of 8 x 8 threads
static dim3 nvdr_block(int H, int W) { return getLaunchBlockSize(TEX_FWD_MAX_KERNEL_BLOCK_WIDTH, TEX_FWD_MAX_KERNEL_BLOCK_HEIGHT, W, H); }

static dim3 nvdr_grad_block(int H, int W) {
    return getLaunchBlockSize(TEX_GRAD_MAX_KERNEL_BLOCK_WIDTH, TEX_GRAD_MAX_KERNEL_BLOCK_HEIGHT, W, H);
}

extern "C" int nvdr_cube_linear_fwd(const float* tex, int R, const float* uv, int H, int W, float* out, void* stream) {
    TextureKernelParams p = nvdr_params(tex, R, uv, H, W);
    p.out = out;
    const dim3 b = nvdr_block(H, W);
    TextureFwdKernelCubeLinear1<<<getLaunchGridSize(b, W, H, 1), b, 0, (cudaStream_t)stream>>>(p);
    return (int)cudaGetLastError();
}

// grad_tex [6,R,R,3] is accumulated into (zero it first); grad_uv [H,W,3] is written
extern "C" int nvdr_cube_linear_grad(const float* tex, int R, const float* uv, int H, int W, const float* dy, float* grad_tex,
                                     float* grad_uv, void* stream) {
    TextureKernelParams p = nvdr_params(tex, R, uv, H, W);
    p.dy = dy;
    p.gradTex[0] = grad_tex;
    p.gradUV = grad_uv;
    const dim3 b = nvdr_grad_block(H, W);
    TextureGradKernelCubeLinear<<<getLaunchGridSize(b, W, H, 1), b, 0, (cudaStream_t)stream>>>(p);
    return (int)cudaGetLastError();
}
