// Per-image bilateral grids (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH 2024; gsplat's
// use_bilateral_grid): the slice that applies one image's grid to a rendered image, its gradient, and the grids' total
// variation.  The statement is in bilagrid.py's docstring.
//
// A grid is [12, L, Hg, Wg] float32: a 3x4 affine per node, coefficient-major.  Pixel (i, j) of an H x W image samples it at
//   gx = (j + 0.5) / W * (Wg - 1),  gy = (i + 0.5) / H * (Hg - 1),  gz = clamp(0.299 r + 0.587 g + 0.114 b, 0, 1) * (L - 1)
// trilinearly (F.grid_sample, align_corners=True, padding_mode="border"), and out = A c + t with M = [A | t].
//
// Work split (slice forward and backward): a "cell" is the set of pixels whose floor(gx), floor(gy) (clamped to Wg - 2,
// Hg - 2) are (cx, cy); its pixels read only the 4 xy-nodes of the cell, at every level: 4 x L x 12 floats, staged in shared
// memory.  One block takes a chunk of BG_TX columns x BG_RB rows of a superset of one cell's pixel rectangle (every pixel tests
// its own cell, so each pixel is taken by exactly one block); a thread owns one column.
//
// Backward: no float atomics.  Each thread accumulates its column's grid contributions serially into its own slice of
// shared memory, [y-corner][level][coefficient] without the x weight, which is constant along the column.  The block then
// sums the threads' slices times their x weights in thread order into a per-block partial [4][L][12], and a second kernel
// adds, for every grid element, the partials of the blocks whose cells touch its node in a fixed order.  Every run gives the
// same bits.  The per-thread slices bound the depth: L <= BG_MAX_L.
//
// Total variation: tv = (1 / N) sum over the three axes of mean((forward difference along the axis)^2), each mean over all
// images and coefficients; an axis of size 1 has no differences and adds 0.  Squares are summed in fp64 per thread, per block,
// then over the blocks in a fixed order (as scale_reg.cu does).  The backward is elementwise in fp64, rounded once.
#include "sgn_common.cuh"

#define BG_TX 64         // slice: columns per block, one per thread
#define BG_RB 32         // slice: rows per block
#define BG_FWD_TY 4      // slice forward: row lanes per block
#define BG_MAX_L 32      // backward: 2 x L x 12 floats of shared memory per thread
#define BG_TV_BLOCKS 1056
#define BG_TV_THREADS 256

struct BgGeom {
    int L, Hg, Wg, H, W;
    int ncx, ncy;      // cells per axis: max(Wg - 1, 1), max(Hg - 1, 1)
    int spanx, spany;  // columns / rows of a cell's superset rectangle
    int nchx, nchy;    // blocks per cell along each axis
};

static BgGeom bg_geom(int L, int Hg, int Wg, int H, int W) {
    BgGeom g;
    g.L = L; g.Hg = Hg; g.Wg = Wg; g.H = H; g.W = W;
    g.ncx = Wg > 1 ? Wg - 1 : 1;
    g.ncy = Hg > 1 ? Hg - 1 : 1;
    // a cell's pixels lie in [floor(c n / nc) - 1, that + ceil(n / nc) + 3)
    g.spanx = (W + g.ncx - 1) / g.ncx + 3;
    g.spany = (H + g.ncy - 1) / g.ncy + 3;
    g.nchx = (g.spanx + BG_TX - 1) / BG_TX;
    g.nchy = (g.spany + BG_RB - 1) / BG_RB;
    return g;
}

// (p + 0.5) / n * (g - 1), each operation rounded once
__device__ __forceinline__ float bg_coord(int p, int n, int g) {
    return __fmul_rn(__fdiv_rn(__fadd_rn((float)p, 0.5f), (float)n), (float)(g - 1));
}
// the lower corner: floor, clamped so that the upper one (lower + 1, itself clamped to g - 1) is on the grid
__device__ __forceinline__ int bg_lower(float c, int g) { return min((int)floorf(c), max(g - 2, 0)); }

__device__ __forceinline__ float bg_gray(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(0.299f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// the block's cell and the first column / row of its chunk
struct BgBlock {
    int cx, cy, j0, j1, i0, i1;
};
__device__ __forceinline__ BgBlock bg_block(const BgGeom& g) {
    BgBlock b;
    b.cx = blockIdx.x / g.nchx;
    b.cy = blockIdx.y / g.nchy;
    const int basex = max(0, (int)(((long long)b.cx * g.W) / g.ncx) - 1);
    const int basey = max(0, (int)(((long long)b.cy * g.H) / g.ncy) - 1);
    b.j0 = basex + (blockIdx.x % g.nchx) * BG_TX;
    b.j1 = min(min(b.j0 + BG_TX, basex + g.spanx), g.W);
    b.i0 = basey + (blockIdx.y % g.nchy) * BG_RB;
    b.i1 = min(min(b.i0 + BG_RB, basey + g.spany), g.H);
    return b;
}

// the cell's 4 xy-nodes (q = dy * 2 + dx) at every level: s[(q * L + l) * 12 + c]
__device__ __forceinline__ void bg_stage(const float* __restrict__ grid, const BgGeom& g, int cx, int cy, float* s, int tid,
                                         int nthreads) {
    const int n = 4 * g.L * 12;
    for (int e = tid; e < n; e += nthreads) {
        const int c = e % 12, l = (e / 12) % g.L, q = e / (12 * g.L);
        const int x = min(cx + (q & 1), g.Wg - 1), y = min(cy + (q >> 1), g.Hg - 1);
        s[e] = grid[(((size_t)c * g.L + l) * g.Hg + y) * g.Wg + x];
    }
}

// M (the interpolated affine) and dM = dM/dgz at one pixel of the staged cell
__device__ __forceinline__ void bg_interp(const float* s, int L, float fx, float fy, int z0, int z1, float fz, float M[12],
                                          float dM[12]) {
    const float w[4] = {(1.f - fy) * (1.f - fx), (1.f - fy) * fx, fy * (1.f - fx), fy * fx};
#pragma unroll
    for (int c = 0; c < 12; ++c) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            a += w[q] * s[(q * L + z0) * 12 + c];
            b += w[q] * s[(q * L + z1) * 12 + c];
        }
        M[c] = (1.f - fz) * a + fz * b;
        dM[c] = b - a;
    }
}

struct BgZ {
    float gray, fz;
    int z0, z1;
};
__device__ __forceinline__ BgZ bg_z(float r, float gg, float b, int L) {
    BgZ z;
    z.gray = bg_gray(r, gg, b);
    const float gz = __fmul_rn(fminf(fmaxf(z.gray, 0.f), 1.f), (float)(L - 1));
    z.z0 = bg_lower(gz, L);
    z.z1 = min(z.z0 + 1, L - 1);
    z.fz = gz - (float)z.z0;
    return z;
}

__global__ void __launch_bounds__(BG_TX * BG_FWD_TY) bilagrid_slice_fwd_kernel(const float* __restrict__ grid, BgGeom g,
                                                                                const float* __restrict__ rgb, float* __restrict__ out) {
    extern __shared__ float s_cell[];
    const BgBlock bk = bg_block(g);
    const int tid = threadIdx.y * BG_TX + threadIdx.x;
    bg_stage(grid, g, bk.cx, bk.cy, s_cell, tid, BG_TX * BG_FWD_TY);
    __syncthreads();
    const int j = bk.j0 + threadIdx.x;
    if (j >= bk.j1) return;
    const float gx = bg_coord(j, g.W, g.Wg);
    const int x0 = bg_lower(gx, g.Wg);
    if (x0 != bk.cx) return;
    const float fx = gx - (float)x0;
    for (int i = bk.i0 + threadIdx.y; i < bk.i1; i += BG_FWD_TY) {
        const float gy = bg_coord(i, g.H, g.Hg);
        const int y0 = bg_lower(gy, g.Hg);
        if (y0 != bk.cy) continue;
        const size_t p = ((size_t)i * g.W + j) * 3;
        const float r = rgb[p], gg = rgb[p + 1], b = rgb[p + 2];
        const BgZ z = bg_z(r, gg, b, g.L);
        float M[12], dM[12];
        bg_interp(s_cell, g.L, fx, gy - (float)y0, z.z0, z.z1, z.fz, M, dM);
#pragma unroll
        for (int k = 0; k < 3; ++k) out[p + k] = M[4 * k] * r + M[4 * k + 1] * gg + M[4 * k + 2] * b + M[4 * k + 3];
    }
}

__global__ void __launch_bounds__(BG_TX) bilagrid_slice_bwd_kernel(const float* __restrict__ grid, BgGeom g, const float* __restrict__ rgb,
                                                                   const float* __restrict__ d_out, float* __restrict__ d_rgb,
                                                                   float* __restrict__ partial) {
    extern __shared__ float s_mem[];
    const int L = g.L;
    float* s_cell = s_mem;                  // [4][L][12]
    float* s_acc = s_cell + 4 * L * 12;     // [2][L][12][BG_TX]: this thread's column, without its x weight
    float* s_wx = s_acc + 2 * L * 12 * BG_TX;  // [2][BG_TX]
    const BgBlock bk = bg_block(g);
    const int t = threadIdx.x;
    bg_stage(grid, g, bk.cx, bk.cy, s_cell, t, BG_TX);
    for (int e = 0; e < 2 * L * 12; ++e) s_acc[e * BG_TX + t] = 0.f;
    const int j = bk.j0 + t;
    float gx = 0.f;
    bool col = j < bk.j1;
    if (col) {
        gx = bg_coord(j, g.W, g.Wg);
        col = bg_lower(gx, g.Wg) == bk.cx;
    }
    const float fx = col ? gx - (float)bk.cx : 0.f;
    s_wx[t] = col ? 1.f - fx : 0.f;
    s_wx[BG_TX + t] = col ? fx : 0.f;
    __syncthreads();
    if (col) {
        for (int i = bk.i0; i < bk.i1; ++i) {
            const float gy = bg_coord(i, g.H, g.Hg);
            const int y0 = bg_lower(gy, g.Hg);
            if (y0 != bk.cy) continue;
            const float fy = gy - (float)y0;
            const size_t p = ((size_t)i * g.W + j) * 3;
            const float cin[4] = {rgb[p], rgb[p + 1], rgb[p + 2], 1.f};
            const float d[3] = {d_out[p], d_out[p + 1], d_out[p + 2]};
            const BgZ z = bg_z(cin[0], cin[1], cin[2], L);
            float M[12], dM[12];
            bg_interp(s_cell, L, fx, fy, z.z0, z.z1, z.fz, M, dM);
            // d c = A^T d_out, plus the guidance term where gray is strictly inside (0, 1) (grid_sample's border clip passes no
            // gradient on or beyond the border)
            float dc[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) dc[k] = M[k] * d[0] + M[4 + k] * d[1] + M[8 + k] * d[2];
            if (z.gray > 0.f && z.gray < 1.f) {
                float dg = 0.f;
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    dg += d[r] * (dM[4 * r] * cin[0] + dM[4 * r + 1] * cin[1] + dM[4 * r + 2] * cin[2] + dM[4 * r + 3]);
                dg *= (float)(L - 1);
                dc[0] += dg * 0.299f;
                dc[1] += dg * 0.587f;
                dc[2] += dg * 0.114f;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) d_rgb[p + k] = dc[k];
            // d grid: the trilinear scatter of d_out (x) (c, 1); the x weight is applied in the block reduction
            const float wz[2] = {1.f - z.fz, z.fz};
            const float wy[2] = {1.f - fy, fy};
            const int zl[2] = {z.z0, z.z1};
#pragma unroll
            for (int c = 0; c < 12; ++c) {
                const float gc = d[c >> 2] * cin[c & 3];
#pragma unroll
                for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                    for (int dz = 0; dz < 2; ++dz) {
                        float* a = s_acc + ((size_t)((dy * L + zl[dz]) * 12 + c)) * BG_TX + t;
                        *a += (wy[dy] * wz[dz]) * gc;
                    }
            }
        }
    }
    __syncthreads();
    // the block's partial [q = dy * 2 + dx][L][12]: the threads' columns times their x weights, summed in thread order
    const int n = 4 * L * 12;
    float* dst = partial + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * n;
    for (int o = t; o < n; o += BG_TX) {
        const int c = o % 12, l = (o / 12) % L, q = o / (12 * L);
        const float* a = s_acc + (size_t)(((q >> 1) * L + l) * 12 + c) * BG_TX;
        const float* w = s_wx + (q & 1) * BG_TX;
        float sum = 0.f;
        for (int k = 0; k < BG_TX; ++k) sum += w[k] * a[k];
        dst[o] = sum;
    }
}

// d_grid[c, l, y, x] = the partials of every block whose cell has node (x, y) as a corner, in a fixed order
__global__ void __launch_bounds__(256) bilagrid_grid_reduce_kernel(const float* __restrict__ partial, BgGeom g,
                                                                   float* __restrict__ d_grid) {
    const int total = 12 * g.L * g.Hg * g.Wg;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int x = e % g.Wg, y = (e / g.Wg) % g.Hg, l = (e / (g.Wg * g.Hg)) % g.L, c = e / (g.Wg * g.Hg * g.L);
    const int n = 4 * g.L * 12, bx = g.ncx * g.nchx;
    double acc = 0.0;
    // a node is corner dy = 1 of cell y - 1 and corner dy = 0 of cell y; on a grid of one node it is both corners of cell 0
    for (int py = 0; py < 2; ++py) {
        const int cy = g.Hg == 1 ? 0 : y - 1 + py, dy = g.Hg == 1 ? py : 1 - py;
        if (cy < 0 || cy >= g.ncy) continue;
        for (int px = 0; px < 2; ++px) {
            const int cx = g.Wg == 1 ? 0 : x - 1 + px, dx = g.Wg == 1 ? px : 1 - px;
            if (cx < 0 || cx >= g.ncx) continue;
            const float* src = partial + (size_t)((cy * g.nchy) * bx + cx * g.nchx) * n + ((dy * 2 + dx) * g.L + l) * 12 + c;
#pragma unroll 1
            for (int hy = 0; hy < g.nchy; ++hy)
#pragma unroll 1
                for (int hx = 0; hx < g.nchx; ++hx) acc += (double)src[((size_t)hy * bx + hx) * n];
        }
    }
    d_grid[e] = (float)acc;
}

template <typename T>
__device__ __forceinline__ T bg_block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < BG_TV_THREADS / 32 ? smem[threadIdx.x] : T(0);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

__global__ void __launch_bounds__(BG_TV_THREADS) bilagrid_tv_fwd_kernel(const float* __restrict__ x, long long total, int L, int Hg,
                                                                        int Wg, double* __restrict__ partial) {
    __shared__ double s_red[BG_TV_THREADS / 32];
    const long long plane = (long long)Hg * Wg;
    double s[3] = {0.0, 0.0, 0.0};  // along Wg, Hg, L
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int xi = (int)(e % Wg), yi = (int)((e / Wg) % Hg), li = (int)((e / plane) % L);
        const double v = x[e];
        if (xi + 1 < Wg) { const double d = (double)x[e + 1] - v; s[0] += d * d; }
        if (yi + 1 < Hg) { const double d = (double)x[e + Wg] - v; s[1] += d * d; }
        if (li + 1 < L) { const double d = (double)x[e + plane] - v; s[2] += d * d; }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double b = bg_block_sum(s[a], s_red);
        if (threadIdx.x == 0) partial[blockIdx.x * 3 + a] = b;
    }
}

// the number of forward differences along each axis, over all images and coefficients
static void bg_tv_counts(int N, int L, int Hg, int Wg, double cnt[3]) {
    const double m = 12.0 * N;
    cnt[0] = m * L * Hg * (Wg - 1);
    cnt[1] = m * L * (Hg - 1) * Wg;
    cnt[2] = m * (L - 1) * Hg * Wg;
}

__global__ void __launch_bounds__(BG_TV_THREADS) bilagrid_tv_finish_kernel(const double* __restrict__ partial, int nblocks, double c0,
                                                                           double c1, double c2, int N, float* __restrict__ out) {
    __shared__ double s_red[BG_TV_THREADS / 32];
    const double cnt[3] = {c0, c1, c2};
    double tv = 0.0;
    for (int a = 0; a < 3; ++a) {
        double s = 0.0;
        for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += partial[i * 3 + a];
        const double tot = bg_block_sum(s, s_red);
        if (cnt[a] > 0.0) tv += tot / cnt[a];  // an axis of size 1 has no differences
    }
    if (threadIdx.x == 0) out[0] = (float)(tv / (double)N);
}

__global__ void __launch_bounds__(BG_TV_THREADS) bilagrid_tv_bwd_kernel(const float* __restrict__ x, long long total, int L, int Hg,
                                                                        int Wg, double k0, double k1, double k2,
                                                                        const float* __restrict__ v_out, float* __restrict__ dx) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const long long plane = (long long)Hg * Wg;
    const int xi = (int)(e % Wg), yi = (int)((e / Wg) % Hg), li = (int)((e / plane) % L);
    const double v = x[e];
    double g = 0.0;
    if (xi > 0) g += k0 * (v - (double)x[e - 1]);
    if (xi + 1 < Wg) g -= k0 * ((double)x[e + 1] - v);
    if (yi > 0) g += k1 * (v - (double)x[e - Wg]);
    if (yi + 1 < Hg) g -= k1 * ((double)x[e + Wg] - v);
    if (li > 0) g += k2 * (v - (double)x[e - plane]);
    if (li + 1 < L) g -= k2 * ((double)x[e + plane] - v);
    dx[e] = (float)((double)v_out[0] * g);
}

static int bg_check_grid(const char* fn, int L, int Hg, int Wg) {
    SGN_REQUIRE(L >= 1 && Hg >= 1 && Wg >= 1, "%s: grid shape L = %d, Hg = %d, Wg = %d must be positive", fn, L, Hg, Wg);
    SGN_REQUIRE((long long)12 * L * Hg * Wg < (1ll << 31), "%s: grid of %d x %d x %d nodes is too large", fn, L, Hg, Wg);
    return SGN_OK;
}

static int bg_check_slice(const char* fn, int L, int Hg, int Wg, int H, int W) {
    const int rc = bg_check_grid(fn, L, Hg, Wg);
    if (rc != SGN_OK) return rc;
    SGN_REQUIRE(H >= 1 && W >= 1 && (long long)H * W < (1ll << 31) / 3, "%s: image %d x %d out of range", fn, H, W);
    return SGN_OK;
}

static size_t bg_bwd_smem(int L) { return sizeof(float) * ((size_t)4 * L * 12 + (size_t)2 * L * 12 * BG_TX + 2 * BG_TX); }

extern "C" int sgn_bilagrid_slice_fwd(const float* grid, int L, int Hg, int Wg, const float* rgb, int H, int W, float* out, void* stream_) {
    SGN_RANGE("sgn_bilagrid_slice_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(grid && rgb && out, "sgn_bilagrid_slice_fwd: null grid, rgb or out");
    const int rc = bg_check_slice("sgn_bilagrid_slice_fwd", L, Hg, Wg, H, W);
    if (rc != SGN_OK) return rc;
    const BgGeom g = bg_geom(L, Hg, Wg, H, W);
    const size_t smem = sizeof(float) * 4 * L * 12;
    if (smem > 48 * 1024) SGN_CHECK_CUDA(cudaFuncSetAttribute(bilagrid_slice_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bilagrid_slice_fwd_kernel<<<dim3(g.ncx * g.nchx, g.ncy * g.nchy), dim3(BG_TX, BG_FWD_TY), smem, stream>>>(grid, g, rgb, out);
    SGN_CHECK_LAUNCH("bilagrid_slice_fwd_kernel");
    return SGN_OK;
}

extern "C" size_t sgn_bilagrid_slice_bwd_scratch_bytes(int L, int Hg, int Wg, int H, int W) {
    if (L < 1 || Hg < 1 || Wg < 1 || H < 1 || W < 1) return 0;
    const BgGeom g = bg_geom(L, Hg, Wg, H, W);
    return sizeof(float) * (size_t)(g.ncx * g.nchx) * (size_t)(g.ncy * g.nchy) * 4 * L * 12;
}

extern "C" int sgn_bilagrid_slice_bwd(const float* grid, int L, int Hg, int Wg, const float* rgb, const float* d_out, int H, int W,
                                      float* d_rgb, float* d_grid, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_bilagrid_slice_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(grid && rgb && d_out && d_rgb && d_grid && scratch, "sgn_bilagrid_slice_bwd: null pointer argument");
    const int rc = bg_check_slice("sgn_bilagrid_slice_bwd", L, Hg, Wg, H, W);
    if (rc != SGN_OK) return rc;
    SGN_REQUIRE(L <= BG_MAX_L, "sgn_bilagrid_slice_bwd: grid depth L = %d above the supported %d", L, BG_MAX_L);
    const size_t need = sgn_bilagrid_slice_bwd_scratch_bytes(L, Hg, Wg, H, W);
    if (scratch_bytes < need) {
        sgn_set_error("sgn_bilagrid_slice_bwd: scratch too small (%zu < %zu bytes)", scratch_bytes, need);
        return SGN_ERR_WORKSPACE;
    }
    const BgGeom g = bg_geom(L, Hg, Wg, H, W);
    const size_t smem = bg_bwd_smem(L);
    if (smem > 48 * 1024) SGN_CHECK_CUDA(cudaFuncSetAttribute(bilagrid_slice_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bilagrid_slice_bwd_kernel<<<dim3(g.ncx * g.nchx, g.ncy * g.nchy), BG_TX, smem, stream>>>(grid, g, rgb, d_out, d_rgb, (float*)scratch);
    SGN_CHECK_LAUNCH("bilagrid_slice_bwd_kernel");
    const int total = 12 * L * Hg * Wg;
    bilagrid_grid_reduce_kernel<<<(total + 255) / 256, 256, 0, stream>>>((const float*)scratch, g, d_grid);
    SGN_CHECK_LAUNCH("bilagrid_grid_reduce_kernel");
    return SGN_OK;
}

extern "C" size_t sgn_bilagrid_tv_scratch_bytes(void) { return sizeof(double) * 3 * BG_TV_BLOCKS; }

extern "C" int sgn_bilagrid_tv_fwd(const float* grids, int N, int L, int Hg, int Wg, float* out, void* scratch, size_t scratch_bytes,
                                   void* stream_) {
    SGN_RANGE("sgn_bilagrid_tv_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(grids && out && scratch, "sgn_bilagrid_tv_fwd: null grids, out or scratch");
    SGN_REQUIRE(N >= 1, "sgn_bilagrid_tv_fwd: N = %d grids", N);
    const int rc = bg_check_grid("sgn_bilagrid_tv_fwd", L, Hg, Wg);
    if (rc != SGN_OK) return rc;
    if (scratch_bytes < sgn_bilagrid_tv_scratch_bytes()) {
        sgn_set_error("sgn_bilagrid_tv_fwd: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_bilagrid_tv_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    const long long total = 12ll * N * L * Hg * Wg;
    double cnt[3];
    bg_tv_counts(N, L, Hg, Wg, cnt);
    bilagrid_tv_fwd_kernel<<<BG_TV_BLOCKS, BG_TV_THREADS, 0, stream>>>(grids, total, L, Hg, Wg, (double*)scratch);
    SGN_CHECK_LAUNCH("bilagrid_tv_fwd_kernel");
    bilagrid_tv_finish_kernel<<<1, BG_TV_THREADS, 0, stream>>>((const double*)scratch, BG_TV_BLOCKS, cnt[0], cnt[1], cnt[2], N, out);
    SGN_CHECK_LAUNCH("bilagrid_tv_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_bilagrid_tv_bwd(const float* grids, int N, int L, int Hg, int Wg, const float* v_out, float* d_grids, void* stream_) {
    SGN_RANGE("sgn_bilagrid_tv_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(grids && v_out && d_grids, "sgn_bilagrid_tv_bwd: null grids, cotangent or gradient");
    SGN_REQUIRE(N >= 1, "sgn_bilagrid_tv_bwd: N = %d grids", N);
    const int rc = bg_check_grid("sgn_bilagrid_tv_bwd", L, Hg, Wg);
    if (rc != SGN_OK) return rc;
    const long long total = 12ll * N * L * Hg * Wg;
    double cnt[3], k[3];
    bg_tv_counts(N, L, Hg, Wg, cnt);
    for (int a = 0; a < 3; ++a) k[a] = cnt[a] > 0.0 ? 2.0 / (cnt[a] * N) : 0.0;
    bilagrid_tv_bwd_kernel<<<(unsigned)((total + BG_TV_THREADS - 1) / BG_TV_THREADS), BG_TV_THREADS, 0, stream>>>(
        grids, total, L, Hg, Wg, k[0], k[1], k[2], v_out, d_grids);
    SGN_CHECK_LAUNCH("bilagrid_tv_bwd_kernel");
    return SGN_OK;
}
