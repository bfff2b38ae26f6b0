// Learnable sky of the reference (EnvLight, street_gaussians_ns/sgn_splatfacto.py:109-150; use_sky_sphere = True by
// default): one world direction per pixel, looked up in a [6,R,R,3] cube map with nvdiffrast's
// dr.texture(filter_mode='linear', boundary_mode='cube'), and the gradient of that lookup for the cube map.
//
// Directions: pixel (x = column, y = row), jitter (ju, jv) = (0.5, 0.5) in eval, two torch.rand draws in training:
//   d = normalize(((x - cx + ju) / fx, (y - cy + jv) / fy, 1)),  d = c2w[:3,:3] @ d,  l = (d.x, d.z, -d.y)   (to_opengl)
// c2w[:3,:3] is recovered exactly from the camera's viewmat (transpose, negate columns 1 and 2).  Divisions and the square
// root are IEEE (no fast math): the directions follow torch's fp32 statement of the same expressions.
//
// Cube lookup (the OpenGL cube map convention): the major axis picks the face (|z| > max(|x|,|y|): 4/5, else |y| > |x|:
// 2/3, else 0/1; +1 when the major component is negative).  With face basis (N, U, V) below, a direction d on face f has
// face coordinates s = <d,U> / (2|<d,N>|) + 1/2, t = <d,V> / (2|<d,N>|) + 1/2, clamped to [0,1]; texel space is
// s * R - 1/2.  Bilinear taps that fall off the face are taken from the adjacent face: the off-face texel centre is
// carried across the edge onto the neighbouring face, where it lands on the texel derived in cube_wrap.  At a cube corner
// the fourth tap has no texel: it takes the mean of the other three (a sum times 0.33333333f), and in the gradient each
// of the three receives its own weight plus a third of the missing one.  A non-finite face coordinate (zero or NaN
// direction) samples 0 and contributes no gradient.
//
// The face coordinate arithmetic follows the sampler it stands in for operation by operation (__frcp_rz, separately rounded
// product and add, a fused s * R - 1/2, fused lerps).  Against that sampler's own kernels on the same directions most
// lookups come out bit-equal and the rest differ within the fp32 bar of the tests (tests/test_gpu_sky.py).
//
// Forward: one thread per pixel, a warp on 32 consecutive pixels of a row; the texels a camera reads stay in L2.
// Backward: a CTA owns a 32 x 32 pixel tile (each thread four rows).  It reduces the texel box its in-face lookups touch on
// the face of the tile's first pixel; when that box fits in shared memory the contributions are accumulated there and
// each touched texel is flushed with one global RED.  Contributions of other faces, wrapped edges and corners, or of a
// tile whose box is too large, go straight to global REDs.  Float atomics: this gradient is not bit-reproducible.
//
// Deterministic backward (sgn_sky_bwd_det / sgn_cube_texture_bwd_det, cube_bwd_kernel<CAM, true>): the same tiles and
// boxes, but every addend is rounded once to 64-bit fixed point and added as an integer, in the shared box and on the
// global path alike.  Integer addition is associative, so the sums are bit-identical whatever the order in which blocks,
// warps and atomics run; one conversion kernel then adds them to v_tex.  The grid is 2^32 units per unit of max|v_out|
// (cot_max_kernel + fixed_scale_kernel, sgn_fixed.cuh: a power of two, so scaling an addend is exact).  A lookup gives a
// texel at most one addend (its taps are four distinct texels, the missing corner tap's share folded into the other three),
// of |w v| <= 4/3 max|v_out|, i.e. at most 4/3 2^32 units; an int64 holds 2^30 such addends, while a camera of 32-bit
// indexable size has fewer than 2^30 pixels (1920 x 1280: 2^21.2) and a uv array fewer than 2^29.5 lookups (3 P <= INT_MAX).
// So, unlike the blend's conic components, no texel needs a coarser grid.  Halving the box capacity keeps the int64 box at
// the float box's 24 KB of static shared memory.
#include <limits.h>

#include <type_traits>

#include "sgn_common.cuh"
#include "sgn_fixed.cuh"

#define SKY_THREADS 256
#define SKY_TILE 32                                   // backward tile: 32 x 32 pixels (camera) or 1024 items (uv array)
#define SKY_ITEMS (SKY_TILE * SKY_TILE / SKY_THREADS) // items per thread in the backward
#define SKY_BOX_TEXELS 2048                           // shared-memory box capacity (x 3 channels: 24 KB)
#define SKY_DET_BOX_TEXELS 1024                       // the deterministic backward's int64 box (x 3 channels: 24 KB)

// gradient accumulator of the backward: float (atomics in any order) or fixed point (deterministic)
template <bool DET>
using SkyAcc = typename std::conditional<DET, unsigned long long, float>::type;

// face basis (N, U, V) of faces 0..5 = +x, -x, +y, -y, +z, -z: direction = N + a U + b V with a = 2s - 1, b = 2t - 1
__constant__ int8_t kCubeBasis[6][3][3] = {
    {{1, 0, 0}, {0, 0, -1}, {0, -1, 0}},  {{-1, 0, 0}, {0, 0, 1}, {0, -1, 0}}, {{0, 1, 0}, {1, 0, 0}, {0, 0, 1}},
    {{0, -1, 0}, {1, 0, 0}, {0, 0, -1}},  {{0, 0, 1}, {1, 0, 0}, {0, -1, 0}},  {{0, 0, -1}, {-1, 0, 0}, {0, -1, 0}},
};
constexpr float kThird = 0.33333333f;

struct SkyCam {
    float R[9];  // c2w[:3,:3], row-major
    float fx, fy, cx, cy;
    int W, H;
};

static __device__ __forceinline__ int dot3(const int8_t* a, const int8_t* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// Texel reached by the off-face texel (i, j) of `face` when exactly one of i, j lies outside [0, R).  The texel centre lies
// just beyond one edge: direction N + o + (along-edge part), o the outward axis.  The neighbouring face g has N_g = o; on
// it the coordinate along an axis that is +-N_f is pinned to the far / near border, the other follows the along-edge index.
static __device__ int cube_wrap(int face, int i, int j, int R) {
    const int8_t* B = kCubeBasis[face][0];
    int k;
    const int8_t* e = (i < 0 || i >= R) ? kCubeBasis[face][1] : kCubeBasis[face][2];  // U or V: the axis that was left
    const int8_t* a = (i < 0 || i >= R) ? kCubeBasis[face][2] : kCubeBasis[face][1];
    const int sgn = (i < 0 || j < 0) ? -1 : 1;
    k = (i < 0 || i >= R) ? j : i;
    int g = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int o = sgn * e[c];
        if (o != 0) g = 2 * c + (o < 0);  // the face whose N is the outward axis
    }
    int coord[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const int8_t* Bg = kCubeBasis[g][1 + c];
        const int dn = dot3(B, Bg);
        coord[c] = dn > 0 ? R - 1 : dn < 0 ? 0 : (dot3(a, Bg) > 0 ? k : R - 1 - k);
    }
    return (g * R + coord[1]) * R + coord[0];
}

static __device__ __forceinline__ int cube_texel(int face, int i, int j, int R) {
    const bool oi = (unsigned)i >= (unsigned)R, oj = (unsigned)j >= (unsigned)R;
    if (!oi && !oj) return (face * R + j) * R + i;
    if (oi && oj) return -1;  // the missing corner texel
    return cube_wrap(face, i, j, R);
}

struct Quad {
    int idx[4];      // texel indices of taps (i,j), (i+1,j), (i,j+1), (i+1,j+1); -1 = missing corner tap (all -1: invalid)
    float fu, fv;    // bilinear weights
    int i0, j0;
    int own_face;    // the face when all four taps lie on it, else -1 (a tap wraps onto a neighbour, or the lookup is invalid)
};

static __device__ __forceinline__ bool quad_corner(const Quad& q) { return (q.idx[0] | q.idx[1] | q.idx[2] | q.idx[3]) < 0; }

static __device__ __forceinline__ void cube_quad(float3 l, int R, Quad& q) {
    // major axis: z when |z| beats both others, else y when |y| beats |x|, else x (ties fall through in that order)
    const float mx = fabsf(l.x), my = fabsf(l.y), mz = fabsf(l.z);
    const int axis = mz > fmaxf(mx, my) ? 2 : my > mx ? 1 : 0;
    const float major = axis == 2 ? l.z : axis == 1 ? l.y : l.x;
    const int face = 2 * axis + (major < 0.f);
    // s = <l,U> / (2|<l,N>|) + 1/2: the reciprocal rounded toward zero, then a separately rounded product and add
    const float half_inv = __frcp_rz(fabsf(major)) * 0.5f;
    // <l,U> and <l,V>: each basis axis has one non-zero entry (+-1), taken from x or z for U and from y or z for V; selecting
    // the component keeps an infinite one from meeting a zero, and the +-1 factor is an exact sign
    const int iu = axis == 0 ? 2 : 0, iv = axis == 1 ? 2 : 1;
    const float lu = (iu == 2 ? l.z : l.x) * (float)kCubeBasis[face][1][iu];
    const float lv = (iv == 2 ? l.z : l.y) * (float)kCubeBasis[face][2][iv];
    float s = __fadd_rn(__fmul_rn(lu, half_inv), 0.5f);
    float t = __fadd_rn(__fmul_rn(lv, half_inv), 0.5f);
    if (!isfinite(s) || !isfinite(t)) {
        q.idx[0] = q.idx[1] = q.idx[2] = q.idx[3] = -1;
        q.fu = q.fv = 0.f;
        q.i0 = q.j0 = 0;
        q.own_face = -1;
        return;
    }
    s = fminf(fmaxf(s, 0.f), 1.f);
    t = fminf(fmaxf(t, 0.f), 1.f);
    const float u = fmaf(s, (float)R, -0.5f), v = fmaf(t, (float)R, -0.5f);
    const int i0 = __float2int_rd(u), j0 = __float2int_rd(v);
    q.fu = u - (float)i0;
    q.fv = v - (float)j0;
    q.i0 = i0;
    q.j0 = j0;
    const bool wrapped = i0 < 0 || j0 < 0 || i0 + 1 >= R || j0 + 1 >= R;
    q.own_face = wrapped ? -1 : face;
    if (!wrapped) {
        const int b = (face * R + j0) * R + i0;
        q.idx[0] = b;
        q.idx[1] = b + 1;
        q.idx[2] = b + R;
        q.idx[3] = b + R + 1;
    } else {
        q.idx[0] = cube_texel(face, i0, j0, R);
        q.idx[1] = cube_texel(face, i0 + 1, j0, R);
        q.idx[2] = cube_texel(face, i0, j0 + 1, R);
        q.idx[3] = cube_texel(face, i0 + 1, j0 + 1, R);
    }
}

static __device__ __forceinline__ float lerpf(float a, float b, float c) { return fmaf(c, b - a, a); }

static __device__ __forceinline__ void cube_sample(const Quad& q, const float* __restrict__ tex, float* o) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float a[4];
        if (quad_corner(q)) {
            float avg = 0.f;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (q.idx[k] >= 0) avg += (a[k] = __ldg(tex + 3 * q.idx[k] + ch));
            avg *= kThird;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (q.idx[k] < 0) a[k] = avg;
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) a[k] = __ldg(tex + 3 * q.idx[k] + ch);
        }
        o[ch] = lerpf(lerpf(a[0], a[1], q.fu), lerpf(a[2], a[3], q.fu), q.fv);
    }
}

// bilinear weights of taps (i,j), (i+1,j), (i,j+1), (i+1,j+1): the corner product fu fv once, the two edge weights as a
// fraction minus it, and the first tap as the remainder (1 - fu) - fv (1 - fu)
static __device__ __forceinline__ void quad_weights(const Quad& q, float w[4]) {
    w[3] = q.fu * q.fv;
    w[2] = q.fv - w[3];
    w[1] = q.fu - w[3];
    w[0] = 1.f - q.fu - w[2];
}

// the same weights with every operation rounded on its own (no contraction): the deterministic backward forms each
// addend by one fixed sequence of roundings wherever the lookup is accumulated (shared box or global path)
static __device__ __forceinline__ void quad_weights_rn(const Quad& q, float w[4]) {
    w[3] = __fmul_rn(q.fu, q.fv);
    w[2] = __fsub_rn(q.fv, w[3]);
    w[1] = __fsub_rn(q.fu, w[3]);
    w[0] = __fsub_rn(__fsub_rn(1.f, q.fu), w[2]);
}

// an addend on the fixed-point grid: the scale is a power of two (the product is exact), then one rounding to an integer
static __device__ __forceinline__ unsigned long long to_fixed(float a, float fscale) {
    return (unsigned long long)__float2ll_rn(__fmul_rn(a, fscale));
}

// every tap of the lookup straight to global memory, with the corner rule
static __device__ __forceinline__ void quad_red_global(const Quad& q, const float vy[3], float* __restrict__ v_tex) {
    float w[4];
    quad_weights(q, w);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float cw[4], cb = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            cw[k] = w[k] * vy[ch];
            if (q.idx[k] < 0) cb = cw[k];
        }
        const bool corner = quad_corner(q);
        if (corner) cb *= kThird;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (q.idx[k] >= 0) atomicAdd(v_tex + 3 * q.idx[k] + ch, corner ? cw[k] + cb : cw[k]);
    }
}

// the deterministic form: the same addends w v and, at a corner, w v + (w_missing v) kThird, each rounded on its own and
// then once to fixed point
static __device__ __forceinline__ void quad_red_global(const Quad& q, const float vy[3], unsigned long long* __restrict__ v_fx,
                                                       float fscale) {
    float w[4];
    quad_weights_rn(q, w);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float cw[4], cb = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            cw[k] = __fmul_rn(w[k], vy[ch]);
            if (q.idx[k] < 0) cb = cw[k];
        }
        const bool corner = quad_corner(q);
        if (corner) cb = __fmul_rn(cb, kThird);
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (q.idx[k] >= 0) atomicAdd(v_fx + 3 * q.idx[k] + ch, to_fixed(corner ? __fadd_rn(cw[k], cb) : cw[k], fscale));
    }
}

static __device__ __forceinline__ float3 sky_direction(const SkyCam& c, int x, int y, float ju, float jv) {
    const float dx = __fdiv_rn(__fadd_rn(__fsub_rn((float)x, c.cx), ju), c.fx);
    const float dy = __fdiv_rn(__fadd_rn(__fsub_rn((float)y, c.cy), jv), c.fy);
    const float n = fmaxf(__fsqrt_rn(__fadd_rn(__fmaf_rn(dy, dy, __fmul_rn(dx, dx)), 1.f)), 1e-12f);
    const float ux = __fdiv_rn(dx, n), uy = __fdiv_rn(dy, n), uz = __fdiv_rn(1.f, n);
    const float w0 = __fmaf_rn(c.R[2], uz, __fmaf_rn(c.R[1], uy, __fmul_rn(c.R[0], ux)));
    const float w1 = __fmaf_rn(c.R[5], uz, __fmaf_rn(c.R[4], uy, __fmul_rn(c.R[3], ux)));
    const float w2 = __fmaf_rn(c.R[8], uz, __fmaf_rn(c.R[7], uy, __fmul_rn(c.R[6], ux)));
    return make_float3(w0, w2, -w1);  // to_opengl
}

// the lookup direction of item p (pixel p = y * W + x of the camera, or row p of the uv array)
template <bool CAM>
static __device__ __forceinline__ float3 item_direction(const SkyCam& c, const float* __restrict__ ju, const float* __restrict__ jv,
                                                        const float* __restrict__ uv, int p) {
    if (CAM) {
        const int y = p / c.W, x = p - y * c.W;
        return sky_direction(c, x, y, ju ? ju[p] : 0.5f, jv ? jv[p] : 0.5f);
    }
    return make_float3(uv[3 * p], uv[3 * p + 1], uv[3 * p + 2]);
}

template <bool CAM>
__global__ void __launch_bounds__(SKY_THREADS) cube_fwd_kernel(const SkyCam c, const float* __restrict__ ju, const float* __restrict__ jv,
                                                               const float* __restrict__ uv, int P, const float* __restrict__ tex, int R,
                                                               float* __restrict__ out, float* __restrict__ dirs) {
    const int p = blockIdx.x * SKY_THREADS + threadIdx.x;
    if (p >= P) return;
    const float3 l = item_direction<CAM>(c, ju, jv, uv, p);
    if (CAM && dirs) {
        dirs[3 * p] = l.x;
        dirs[3 * p + 1] = l.y;
        dirs[3 * p + 2] = l.z;
    }
    Quad q;
    cube_quad(l, R, q);
    float o[3];
    cube_sample(q, tex, o);
    out[3 * p] = o[0];
    out[3 * p + 1] = o[1];
    out[3 * p + 2] = o[2];
}

// DET = false: float atomics into v_tex.  DET = true: v_tex is the fixed-point scratch, int64 [6,R,R,3] followed by the
// grid scale (one float), and the box holds int64 (SKY_DET_BOX_TEXELS).  The float instantiations carry no fixed-point code.
template <bool CAM, bool DET>
__global__ void __launch_bounds__(SKY_THREADS) cube_bwd_kernel(const SkyCam c, const float* __restrict__ ju, const float* __restrict__ jv,
                                                               const float* __restrict__ uv, int P, int R, const float* __restrict__ v_out,
                                                               SkyAcc<DET>* __restrict__ v_tex) {
    constexpr int BOX_TEXELS = DET ? SKY_DET_BOX_TEXELS : SKY_BOX_TEXELS;
    __shared__ SkyAcc<DET> box[BOX_TEXELS * 3];
    __shared__ int s_dom, s_lo[2], s_hi[2];
    float fscale = 0.f;
    if constexpr (DET) fscale = __ldg(reinterpret_cast<const float*>(v_tex + 18LL * R * R));
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_dom = -1;
        s_lo[0] = s_lo[1] = INT_MAX;
        s_hi[0] = s_hi[1] = INT_MIN;
    }
    Quad q[SKY_ITEMS];
    int item[SKY_ITEMS];
#pragma unroll
    for (int k = 0; k < SKY_ITEMS; ++k) {
        int p = -1;
        if (CAM) {
            const int x = blockIdx.x * SKY_TILE + (tid & (SKY_TILE - 1));
            const int y = blockIdx.y * SKY_TILE + (tid / SKY_TILE) + k * (SKY_THREADS / SKY_TILE);
            if (x < c.W && y < c.H) p = y * c.W + x;
        } else {
            const int pp = blockIdx.x * (SKY_TILE * SKY_TILE) + tid + k * SKY_THREADS;
            if (pp < P) p = pp;
        }
        item[k] = p;
        if (p >= 0) cube_quad(item_direction<CAM>(c, ju, jv, uv, p), R, q[k]);
    }
    __syncthreads();
    if (tid == 0 && item[0] >= 0) s_dom = q[0].own_face;  // the tile's first pixel names the privatised face
    __syncthreads();
    const int dom = s_dom;
    int lo0 = INT_MAX, lo1 = INT_MAX, hi0 = INT_MIN, hi1 = INT_MIN;
#pragma unroll
    for (int k = 0; k < SKY_ITEMS; ++k) {
        if (dom >= 0 && item[k] >= 0 && q[k].own_face == dom) {
            lo0 = min(lo0, q[k].i0);
            hi0 = max(hi0, q[k].i0);
            lo1 = min(lo1, q[k].j0);
            hi1 = max(hi1, q[k].j0);
        }
    }
    lo0 = __reduce_min_sync(0xffffffffu, lo0);
    lo1 = __reduce_min_sync(0xffffffffu, lo1);
    hi0 = __reduce_max_sync(0xffffffffu, hi0);
    hi1 = __reduce_max_sync(0xffffffffu, hi1);
    if ((tid & 31) == 0 && lo0 != INT_MAX) {
        atomicMin(&s_lo[0], lo0);
        atomicMin(&s_lo[1], lo1);
        atomicMax(&s_hi[0], hi0);
        atomicMax(&s_hi[1], hi1);
    }
    __syncthreads();
    const int bi0 = s_lo[0], bj0 = s_lo[1];
    const bool some = dom >= 0 && s_hi[0] >= bi0;  // block-uniform: some lookup lies on the privatised face
    const int bw = some ? s_hi[0] - bi0 + 2 : 0, bh = some ? s_hi[1] - bj0 + 2 : 0;  // a quad spans two texels per axis
    const bool priv = some && bw * bh <= BOX_TEXELS;
    if (priv) {
        for (int e = tid; e < bw * bh * 3; e += SKY_THREADS) box[e] = 0;
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < SKY_ITEMS; ++k) {
        const int p = item[k];
        if (p < 0) continue;
        const float vy[3] = {v_out[3 * p], v_out[3 * p + 1], v_out[3 * p + 2]};
        if (vy[0] == 0.f && vy[1] == 0.f && vy[2] == 0.f) continue;
        if (priv && q[k].own_face == dom) {
            if constexpr (DET) {
                float w[4];
                quad_weights_rn(q[k], w);
                unsigned long long* b = box + 3 * ((q[k].j0 - bj0) * bw + (q[k].i0 - bi0));
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    atomicAdd(b + ch, to_fixed(__fmul_rn(w[0], vy[ch]), fscale));
                    atomicAdd(b + 3 + ch, to_fixed(__fmul_rn(w[1], vy[ch]), fscale));
                    atomicAdd(b + 3 * bw + ch, to_fixed(__fmul_rn(w[2], vy[ch]), fscale));
                    atomicAdd(b + 3 * bw + 3 + ch, to_fixed(__fmul_rn(w[3], vy[ch]), fscale));
                }
            } else {
                float w[4];
                quad_weights(q[k], w);
                float* b = box + 3 * ((q[k].j0 - bj0) * bw + (q[k].i0 - bi0));
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    atomicAdd(b + ch, w[0] * vy[ch]);
                    atomicAdd(b + 3 + ch, w[1] * vy[ch]);
                    atomicAdd(b + 3 * bw + ch, w[2] * vy[ch]);
                    atomicAdd(b + 3 * bw + 3 + ch, w[3] * vy[ch]);
                }
            }
        } else {
            if constexpr (DET) quad_red_global(q[k], vy, v_tex, fscale);
            else quad_red_global(q[k], vy, v_tex);
        }
    }
    if (priv) {
        __syncthreads();
        for (int e = tid; e < bw * bh * 3; e += SKY_THREADS) {
            const SkyAcc<DET> g = box[e];
            if (g != 0) {
                const int t = e / 3, ch = e - 3 * t;
                const int jj = t / bw, ii = t - jj * bw;
                atomicAdd(v_tex + 3 * ((dom * R + bj0 + jj) * R + bi0 + ii) + ch, g);
            }
        }
    }
}

static int sky_cam(SkyCam& c, const sgn_camera* cam, const char* who) {
    SGN_REQUIRE(cam, "%s: null camera", who);
    SGN_REQUIRE(cam->width >= 1 && cam->height >= 1, "%s: empty image (%d x %d)", who, cam->width, cam->height);
    SGN_REQUIRE((long long)cam->width * cam->height * 3 <= INT_MAX, "%s: %d x %d pixels overflow 32-bit indexing", who, cam->width,
                cam->height);
    // viewmat[:3,:3] = (c2w[:3,:3] diag(1,-1,-1))^T: transpose back and negate columns 1 and 2 (exact)
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c.R[3 * i + j] = j == 0 ? cam->viewmat[4 * j + i] : -cam->viewmat[4 * j + i];
    c.fx = cam->fx;
    c.fy = cam->fy;
    c.cx = cam->cx;
    c.cy = cam->cy;
    c.W = cam->width;
    c.H = cam->height;
    return SGN_OK;
}

static int check_res(int R, const char* who) {
    SGN_REQUIRE(R >= 1, "%s: cube map resolution must be >= 1, got %d", who, R);
    SGN_REQUIRE(18LL * R * R <= INT_MAX, "%s: a [6,%d,%d,3] cube map overflows 32-bit indexing", who, R, R);
    return SGN_OK;
}

static int check_jitter(const float* ju, const float* jv, const char* who) {
    SGN_REQUIRE((ju == nullptr) == (jv == nullptr), "%s: give both jitter arrays (training) or neither (eval)", who);
    return SGN_OK;
}

extern "C" int sgn_sky_fwd(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, const float* tex, int R, float* sky,
                           float* dirs, void* stream) {
    SGN_RANGE("sgn_sky_fwd");
    SkyCam c;
    if (int rc = sky_cam(c, cam, "sgn_sky_fwd")) return rc;
    if (int rc = check_res(R, "sgn_sky_fwd")) return rc;
    if (int rc = check_jitter(jitter_u, jitter_v, "sgn_sky_fwd")) return rc;
    SGN_REQUIRE(tex && sky, "sgn_sky_fwd: null texture or output");
    const int P = c.W * c.H;
    cube_fwd_kernel<true><<<(P + SKY_THREADS - 1) / SKY_THREADS, SKY_THREADS, 0, (cudaStream_t)stream>>>(c, jitter_u, jitter_v, nullptr, P, tex,
                                                                                                          R, sky, dirs);
    SGN_CHECK_LAUNCH("cube_fwd_kernel<camera>");
    return SGN_OK;
}

extern "C" int sgn_sky_bwd(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, int R, const float* v_sky, float* v_tex,
                           void* stream) {
    SGN_RANGE("sgn_sky_bwd");
    SkyCam c;
    if (int rc = sky_cam(c, cam, "sgn_sky_bwd")) return rc;
    if (int rc = check_res(R, "sgn_sky_bwd")) return rc;
    if (int rc = check_jitter(jitter_u, jitter_v, "sgn_sky_bwd")) return rc;
    SGN_REQUIRE(v_sky && v_tex, "sgn_sky_bwd: null v_sky or v_tex");
    const dim3 grid((c.W + SKY_TILE - 1) / SKY_TILE, (c.H + SKY_TILE - 1) / SKY_TILE);
    cube_bwd_kernel<true, false><<<grid, SKY_THREADS, 0, (cudaStream_t)stream>>>(c, jitter_u, jitter_v, nullptr, c.W * c.H, R, v_sky, v_tex);
    SGN_CHECK_LAUNCH("cube_bwd_kernel<camera>");
    return SGN_OK;
}

// ---- deterministic backward: zero the scratch, the grid from max|v_out|, the kernel into the int64 sums, then v_tex += sums
__global__ void __launch_bounds__(256)
sky_fixed_add_kernel(const long long* __restrict__ fx, const float* __restrict__ scale, float* __restrict__ v_tex, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v_tex[i] += (float)((double)fx[i] / (double)scale[0]);
}

extern "C" size_t sgn_sky_det_scratch_bytes(int R) {
    if (R < 1 || 18LL * R * R > INT_MAX) return 0;
    return (size_t)18 * R * R * sizeof(long long) + 16;  // the int64 sums, then the grid scale (one float, padded)
}

static int check_det_scratch(const void* scratch, size_t scratch_bytes, int R, const char* who) {
    SGN_REQUIRE(scratch, "%s: null scratch", who);
    SGN_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0, "%s: scratch must be 8-byte aligned", who);
    const size_t need = sgn_sky_det_scratch_bytes(R);
    SGN_REQUIRE(scratch_bytes >= need, "%s: scratch of %zu bytes, sgn_sky_det_scratch_bytes(%d) = %zu", who, scratch_bytes, R, need);
    return SGN_OK;
}

template <bool CAM>
static int launch_bwd_det(const SkyCam& c, const float* ju, const float* jv, const float* uv, int P, int R, const float* v_out,
                          float* v_tex, void* scratch, dim3 grid, cudaStream_t stream) {
    const long long n = 18LL * R * R;
    unsigned long long* fx = reinterpret_cast<unsigned long long*>(scratch);
    float* scale = reinterpret_cast<float*>(fx + n);
    SGN_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)n * sizeof(long long) + sizeof(float), stream));
    cot_max_kernel<<<296, 256, 0, stream>>>(v_out, 3LL * P, reinterpret_cast<unsigned*>(scale));
    SGN_CHECK_LAUNCH("cot_max_kernel");
    fixed_scale_kernel<<<1, 1, 0, stream>>>(scale);
    SGN_CHECK_LAUNCH("fixed_scale_kernel");
    cube_bwd_kernel<CAM, true><<<grid, SKY_THREADS, 0, stream>>>(c, ju, jv, uv, P, R, v_out, fx);
    SGN_CHECK_LAUNCH(CAM ? "cube_bwd_kernel<camera, det>" : "cube_bwd_kernel<uv, det>");
    sky_fixed_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const long long*>(fx), scale, v_tex, n);
    SGN_CHECK_LAUNCH("sky_fixed_add_kernel");
    return SGN_OK;
}

extern "C" int sgn_sky_bwd_det(const sgn_camera* cam, const float* jitter_u, const float* jitter_v, int R, const float* v_sky, float* v_tex,
                               void* scratch, size_t scratch_bytes, void* stream) {
    SGN_RANGE("sgn_sky_bwd_det");
    SkyCam c;
    if (int rc = sky_cam(c, cam, "sgn_sky_bwd_det")) return rc;
    if (int rc = check_res(R, "sgn_sky_bwd_det")) return rc;
    if (int rc = check_jitter(jitter_u, jitter_v, "sgn_sky_bwd_det")) return rc;
    SGN_REQUIRE(v_sky && v_tex, "sgn_sky_bwd_det: null v_sky or v_tex");
    if (int rc = check_det_scratch(scratch, scratch_bytes, R, "sgn_sky_bwd_det")) return rc;
    const dim3 grid((c.W + SKY_TILE - 1) / SKY_TILE, (c.H + SKY_TILE - 1) / SKY_TILE);
    return launch_bwd_det<true>(c, jitter_u, jitter_v, nullptr, c.W * c.H, R, v_sky, v_tex, scratch, grid, (cudaStream_t)stream);
}

static int check_items(int P, const char* who) {
    SGN_REQUIRE(P >= 0 && 3LL * P <= INT_MAX, "%s: %d lookups overflow 32-bit indexing", who, P);
    return SGN_OK;
}

extern "C" int sgn_cube_texture_fwd(int P, const float* uv, const float* tex, int R, float* out, void* stream) {
    SGN_RANGE("sgn_cube_texture_fwd");
    if (int rc = check_items(P, "sgn_cube_texture_fwd")) return rc;
    if (int rc = check_res(R, "sgn_cube_texture_fwd")) return rc;
    SGN_REQUIRE(uv && tex && out, "sgn_cube_texture_fwd: null uv, texture or output");
    if (P == 0) return SGN_OK;
    const SkyCam c{};
    cube_fwd_kernel<false><<<(P + SKY_THREADS - 1) / SKY_THREADS, SKY_THREADS, 0, (cudaStream_t)stream>>>(c, nullptr, nullptr, uv, P, tex, R,
                                                                                                           out, nullptr);
    SGN_CHECK_LAUNCH("cube_fwd_kernel<uv>");
    return SGN_OK;
}

extern "C" int sgn_cube_texture_bwd(int P, const float* uv, int R, const float* v_out, float* v_tex, void* stream) {
    SGN_RANGE("sgn_cube_texture_bwd");
    if (int rc = check_items(P, "sgn_cube_texture_bwd")) return rc;
    if (int rc = check_res(R, "sgn_cube_texture_bwd")) return rc;
    SGN_REQUIRE(uv && v_out && v_tex, "sgn_cube_texture_bwd: null uv, v_out or v_tex");
    if (P == 0) return SGN_OK;
    const SkyCam c{};
    const int tile = SKY_TILE * SKY_TILE;
    cube_bwd_kernel<false, false><<<(P + tile - 1) / tile, SKY_THREADS, 0, (cudaStream_t)stream>>>(c, nullptr, nullptr, uv, P, R, v_out, v_tex);
    SGN_CHECK_LAUNCH("cube_bwd_kernel<uv>");
    return SGN_OK;
}

extern "C" int sgn_cube_texture_bwd_det(int P, const float* uv, int R, const float* v_out, float* v_tex, void* scratch, size_t scratch_bytes,
                                        void* stream) {
    SGN_RANGE("sgn_cube_texture_bwd_det");
    if (int rc = check_items(P, "sgn_cube_texture_bwd_det")) return rc;
    if (int rc = check_res(R, "sgn_cube_texture_bwd_det")) return rc;
    SGN_REQUIRE(uv && v_out && v_tex, "sgn_cube_texture_bwd_det: null uv, v_out or v_tex");
    if (int rc = check_det_scratch(scratch, scratch_bytes, R, "sgn_cube_texture_bwd_det")) return rc;
    if (P == 0) return SGN_OK;
    const SkyCam c{};
    const int tile = SKY_TILE * SKY_TILE;
    return launch_bwd_det<false>(c, nullptr, nullptr, uv, P, R, v_out, v_tex, scratch, dim3((P + tile - 1) / tile), (cudaStream_t)stream);
}
