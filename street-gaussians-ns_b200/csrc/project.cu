// Fused scene-graph compose + EWA projection + SH colour + sigmoid, forward and backward.
// One thread per Gaussian over the concatenated row space; HBM-bound (SURVEY.md 8d).
// Compiled with --fmad=false (see sgn_exact.cuh).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "sgn_exact.cuh"
#include "sgn_touch.cuh"

// ------------------------------------------------------------------------------------------------
// error plumbing + tiny ABI helpers
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void sgn_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
#include <atomic>
static std::atomic<long long> g_launches{0};
void sgn_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long sgn_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" const char* sgn_last_error(void) { return g_err; }
extern "C" int sgn_abi_version(void) { return SGN_ABI_VERSION; }
extern "C" size_t sgn_sizeof_segment(void) { return sizeof(sgn_segment); }
extern "C" size_t sgn_sizeof_segment_grads(void) { return sizeof(sgn_segment_grads); }
extern "C" size_t sgn_sizeof_camera(void) { return sizeof(sgn_camera); }

extern "C" int sgn_upload(const void* host, size_t bytes, void* dev, void* stream) {
    SGN_RANGE("sgn_upload");
    SGN_REQUIRE(host && dev, "sgn_upload: null pointer");
    SGN_CHECK_CUDA(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return SGN_OK;
}

// ------------------------------------------------------------------------------------------------
// Work decomposition: 128-row chunks that never straddle a sub-model (sgn_segment.chunk0 = first chunk
// of the segment).  A chunk's slice of every parameter tensor is CONTIGUOUS in HBM (rows*12 B of means,
// rows*180 B of features_rest, ...), so the block stages it into shared memory with coalesced 128-bit
// loads and each thread then walks its own row at a bank-conflict-free odd word stride; the backward
// stages the dense gradient rows the same way in the other direction.
// ------------------------------------------------------------------------------------------------
#define SGN_MAX_SEGMENTS 1024
#define PROJ_THREADS 256  // Level-1 kernels
#define CH 128            // rows per chunk == threads per block of the fused kernels
#define MAX_REST 45       // (4^2 - 1) * 3
#define MAX_DC (3 * SGN_MAX_FOURIER)

// the camera struct with its view (viewmat[12], then cam_pos[3]) replaced by the 15 floats at `view` (device memory)
__device__ __forceinline__ sgn_camera sgn_camera_with_view(const sgn_camera& c, const float* __restrict__ view) {
    sgn_camera o = c;
#pragma unroll
    for (int k = 0; k < 12; ++k) o.viewmat[k] = __ldg(view + k);
#pragma unroll
    for (int k = 0; k < 3; ++k) o.cam_pos[k] = __ldg(view + 12 + k);
    return o;
}

__device__ __forceinline__ int find_segment_by_chunk(const int* s_chunk0, int nseg, int c) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_chunk0[mid] <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// global -> shared, n floats, all threads of the block participate
__device__ __forceinline__ void coop_load(float* __restrict__ dst, const float* __restrict__ src, int n) {
    if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
        const int n4 = n >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) d4[i] = __ldg(s4 + i);
        for (int i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) dst[i] = __ldg(src + i);
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = __ldg(src + i);
    }
}
// shared -> global
__device__ __forceinline__ void coop_store(float* __restrict__ dst, const float* __restrict__ src, int n) {
    if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
        const int n4 = n >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) d4[i] = s4[i];
        for (int i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    }
}

// Forward: one thread per row, direct loads (independent per-thread loads keep more requests in flight
// than a stage-sync-compute split; measured).  Rows the camera does not see skip the colour work:
// nothing downstream ever reads the colour of an invisible Gaussian.
// VIEW: the world->camera view (viewmat[12], cam_pos[3]) is read from the device (`view`) instead of the camera struct --
// a view computed on the device (camera pose optimisation) reaches the kernel without a host read-back.
template <bool VIEW>
__global__ void __launch_bounds__(CH)
project_fwd_direct_kernel(const sgn_segment* __restrict__ segs, int nseg, const sgn_camera cam_arg,
                   float4* __restrict__ records, int32_t* __restrict__ radii, int32_t* __restrict__ num_tiles_hit,
                   ushort4* __restrict__ tile_bbox, int32_t* __restrict__ tiles_touched, uint32_t* __restrict__ touch_mask,
                   const float* __restrict__ view) {
    sgn_camera cam_view;
    if constexpr (VIEW) cam_view = sgn_camera_with_view(cam_arg, view);
    const sgn_camera& cam = VIEW ? cam_view : cam_arg;
    extern __shared__ int s_chunk0[];
    for (int i = threadIdx.x; i < nseg; i += blockDim.x) s_chunk0[i] = segs[i].chunk0;
    __syncthreads();
    const int si = find_segment_by_chunk(s_chunk0, nseg, blockIdx.x);
    const sgn_segment& sg = segs[si];
    const int i = (blockIdx.x - sg.chunk0) * CH + threadIdx.x;
    const bool active = i < sg.count;  // idle lanes of a tail chunk still take part in the warp-collective tile count
    const size_t g = (size_t)sg.row0 + i;
    const int K = (cam.sh_degree + 1) * (cam.sh_degree + 1);
    bool vis = false;
    ushort4 bb = make_ushort4(0, 0, 0, 0);
    TouchCtx tc = {};
    if (active) {

    float m[3], ls[3], q[4];
#pragma unroll
    for (int k = 0; k < 3; ++k) { m[k] = __ldg(sg.means + 3 * (size_t)i + k); ls[k] = __ldg(sg.scales + 3 * (size_t)i + k); }
    {
        const float4 qq = __ldg(reinterpret_cast<const float4*>(sg.quats) + i);
        q[0] = qq.x; q[1] = qq.y; q[2] = qq.z; q[3] = qq.w;
    }
    const bool filt = cam.filter_3d != nullptr;  // uniform: the 3D smoothing filter
    const float sigma = filt ? __ldg(cam.filter_3d[si] + i) : 0.f;
    SgnProj st;
    vis = sgn_project_exact(sg, cam, m, ls, q, st, true, 1.f, cam.antialiased != 0, filt, sigma);

    float rgb[3] = {0.f, 0.f, 0.f};
    float opac = 0.f, comp = 0.f;
    int aux = 0;
    if (vis) {
        // colour: Fourier DC (scene graph :239-247), SH (sgn_splatfacto.py:933-940)
        float c0[3] = {0.f, 0.f, 0.f};
        for (int f = 0; f < sg.F; ++f) {
            const float w = sg.idft[f];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) c0[ch] += __ldg(sg.features_dc + ((size_t)i * sg.F + f) * 3 + ch) * w;
        }
        if (cam.sh_degree > 0) {
            float d[3] = {st.mw[0] - cam.cam_pos[0], st.mw[1] - cam.cam_pos[1], st.mw[2] - cam.cam_pos[2]};
            const float n = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            d[0] /= n; d[1] /= n; d[2] /= n;
            float Y[16];
            sgn_sh_basis(cam.sh_degree_to_use, d[0], d[1], d[2], Y);
            const int Kuse = min((cam.sh_degree_to_use + 1) * (cam.sh_degree_to_use + 1), K);
            float acc[3] = {Y[0] * c0[0], Y[0] * c0[1], Y[0] * c0[2]};
            const float* rest = sg.features_rest + (size_t)i * (K - 1) * 3;
            for (int k = 1; k < Kuse; ++k) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) acc[ch] += Y[k] * __ldg(rest + (k - 1) * 3 + ch);
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float pre = acc[ch] + 0.5f;
                if (pre >= 0.f) aux |= (1 << ch);
                rgb[ch] = pre > 0.f ? pre : 0.f;
            }
        } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) { rgb[ch] = 1.f / (1.f + expf(-c0[ch])); aux |= (1 << ch); }
        }
        opac = 1.f / (1.f + expf(-__ldg(sg.opacities + i)));
        if (filt) opac = opac * st.coef;
        if (cam.antialiased) {  // warp-uniform
            comp = st.comp;
            opac = opac * comp;
        }
        aux |= SGN_AUX_VISIBLE;
    }
    if (sg.cls == 1) aux |= SGN_AUX_OBJECT;

    float4* rec = records + 3 * g;
    rec[0] = make_float4(st.xy[0], st.xy[1], st.conic[0], st.conic[1]);
    rec[1] = make_float4(st.conic[2], opac, rgb[0], rgb[1]);
    rec[2] = make_float4(rgb[2], vis ? st.pv[2] : 0.f, __int_as_float(aux), comp);
    radii[g] = st.radius;
    num_tiles_hit[g] = vis ? (st.tmax[0] - st.tmin[0]) * (st.tmax[1] - st.tmin[1]) : 0;
    bb = make_ushort4((unsigned short)st.tmin[0], (unsigned short)st.tmin[1],
                      (unsigned short)st.tmax[0], (unsigned short)st.tmax[1]);
    tile_bbox[g] = bb;
    if (vis) tc = make_touch_ctx(make_float4(st.xy[0], st.xy[1], st.conic[0], st.conic[1]), make_float4(st.conic[2], opac, 0.f, 0.f));
    }  // active
    // tiles the Gaussian can really reach (exact ellipse-vs-tile test, sgn_touch.cuh) with the opacity the blend draws --
    // compensated in the antialiased mode, where comp == 0 gives tau = -inf and no tile; binning lists only those
    uint32_t mask;
    const int nt = count_touched_tiles(vis, tc, bb, cam.width, cam.height, cam.block_width, mask);
    if (active) {
        tiles_touched[g] = nt;
        touch_mask[g] = mask;
    }
}

// Forward, two phases per 128-row chunk (the one-phase form runs with few active lanes per
// instruction -- visible and invisible rows mixed in every warp -- with 45 row-strided scalar loads per thread):
//   A  every thread projects its row (exact section); invisible rows write their record and leave;
//   -  the chunk's visible rows are compacted (stable), and ONLY their colour parameters (features_rest: 180 B per row,
//      features_dc) are gathered into shared memory with coalesced loads: consecutive threads read consecutive words;
//   B  thread c takes visible row c: view direction, SH, Fourier DC, sigmoid, record, exact tile count -- full warps.
__global__ void __launch_bounds__(CH)
project_fwd_staged_kernel(const sgn_segment* __restrict__ segs, int nseg, const sgn_camera cam,
                   float4* __restrict__ records, int32_t* __restrict__ radii, int32_t* __restrict__ num_tiles_hit,
                   ushort4* __restrict__ tile_bbox, int32_t* __restrict__ tiles_touched, uint32_t* __restrict__ touch_mask) {
    extern __shared__ int s_chunk0[];
    __shared__ __align__(16) float s_rest[CH * MAX_REST];
    __shared__ __align__(16) float s_dc[CH * MAX_DC];
    __shared__ __align__(16) float s_means[CH * 3];
    __shared__ __align__(16) float s_scales[CH * 3];
    __shared__ float s_geo[CH][11];  // per visible row (compact index): xy, conic, depth, world mean, comp, filter coef
    __shared__ int s_row[CH];       // compact index -> row of the chunk
    __shared__ int s_warp_base[CH / 32 + 1];
    for (int i = threadIdx.x; i < nseg; i += blockDim.x) s_chunk0[i] = segs[i].chunk0;
    __syncthreads();
    const int si = find_segment_by_chunk(s_chunk0, nseg, blockIdx.x);
    const sgn_segment& sg = segs[si];
    const int r0 = (blockIdx.x - sg.chunk0) * CH;
    const int rows = min(CH, sg.count - r0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = (cam.sh_degree + 1) * (cam.sh_degree + 1);
    const int nrest = (K - 1) * 3, ndc = sg.F * 3;
    coop_load(s_means, sg.means + 3 * (size_t)r0, rows * 3);
    coop_load(s_scales, sg.scales + 3 * (size_t)r0, rows * 3);
    __syncthreads();

    // ---- phase A: projection of every row
    const bool active = tid < rows;
    const size_t g = (size_t)sg.row0 + r0 + tid;
    const int cls_bit = sg.cls == 1 ? SGN_AUX_OBJECT : 0;
    bool vis = false;
    SgnProj st;
    if (active) {
        const float m[3] = {s_means[3 * tid], s_means[3 * tid + 1], s_means[3 * tid + 2]};
        const float ls[3] = {s_scales[3 * tid], s_scales[3 * tid + 1], s_scales[3 * tid + 2]};
        const float4 qq = __ldg(reinterpret_cast<const float4*>(sg.quats) + r0 + tid);
        const float q[4] = {qq.x, qq.y, qq.z, qq.w};
        const bool filt = cam.filter_3d != nullptr;  // uniform: the 3D smoothing filter
        const float sigma = filt ? __ldg(cam.filter_3d[si] + r0 + tid) : 0.f;
        vis = sgn_project_exact(sg, cam, m, ls, q, st, true, 1.f, cam.antialiased != 0, filt, sigma);
        radii[g] = st.radius;
        num_tiles_hit[g] = vis ? (st.tmax[0] - st.tmin[0]) * (st.tmax[1] - st.tmin[1]) : 0;
        tile_bbox[g] = make_ushort4((unsigned short)st.tmin[0], (unsigned short)st.tmin[1],
                                    (unsigned short)st.tmax[0], (unsigned short)st.tmax[1]);
        float4* rec = records + 3 * g;
        rec[0] = make_float4(st.xy[0], st.xy[1], st.conic[0], st.conic[1]);
        if (!vis) {  // nothing downstream reads the colour of a Gaussian the camera does not see
            rec[1] = make_float4(st.conic[2], 0.f, 0.f, 0.f);
            rec[2] = make_float4(0.f, 0.f, __int_as_float(cls_bit), 0.f);
            tiles_touched[g] = 0;
            touch_mask[g] = 0u;
        }
    }
    // stable compaction of the visible rows
    const unsigned bal = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) s_warp_base[warp + 1] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
        s_warp_base[0] = 0;
#pragma unroll
        for (int w = 0; w < CH / 32; ++w) s_warp_base[w + 1] += s_warp_base[w];
    }
    __syncthreads();
    const int nvis = s_warp_base[CH / 32];
    if (vis) {
        const int c = s_warp_base[warp] + __popc(bal & ((1u << lane) - 1u));
        s_row[c] = tid;
        float* ge = s_geo[c];
        ge[0] = st.xy[0]; ge[1] = st.xy[1]; ge[2] = st.conic[0]; ge[3] = st.conic[1]; ge[4] = st.conic[2];
        ge[5] = st.pv[2]; ge[6] = st.mw[0]; ge[7] = st.mw[1]; ge[8] = st.mw[2];
        ge[9] = st.comp;
        ge[10] = st.coef;
    }
    __syncthreads();
    if (nvis == 0) return;

    // ---- gather the colour parameters of the visible rows (word e of the compacted block: row e / width, column e % width)
    {
        const unsigned inv_rest = nrest > 0 ? (0xffffffffu / (unsigned)nrest) + 1u : 0u;  // e / nrest == umulhi(e, inv) for e < 2^16
        const float* __restrict__ rest = sg.features_rest + (size_t)r0 * nrest;
        const int n_rest = nvis * nrest;
        for (int e0 = tid; e0 < n_rest; e0 += 4 * CH) {  // four independent requests per thread in flight
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int e = e0 + u * CH;
                if (e < n_rest) {
                    const int r = (int)__umulhi((unsigned)e, inv_rest);
                    v[u] = __ldg(rest + s_row[r] * nrest + (e - r * nrest));
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int e = e0 + u * CH;
                if (e < n_rest) s_rest[e] = v[u];
            }
        }
        const unsigned inv_dc = (0xffffffffu / (unsigned)ndc) + 1u;
        const float* __restrict__ dc = sg.features_dc + (size_t)r0 * ndc;
        for (int e = tid; e < nvis * ndc; e += CH) {
            const int r = (int)__umulhi((unsigned)e, inv_dc);
            s_dc[e] = __ldg(dc + s_row[r] * ndc + (e - r * ndc));
        }
    }
    __syncthreads();

    // ---- phase B: colour, opacity, record and tile count of visible row c = tid
    const bool mine = tid < nvis;
    ushort4 bb = make_ushort4(0, 0, 0, 0);
    TouchCtx tc = {};
    size_t gb = 0;
    if (mine) {
        const int row = s_row[tid];
        gb = (size_t)sg.row0 + r0 + row;
        const float* ge = s_geo[tid];
        // colour: Fourier DC (scene graph :239-247), SH (sgn_splatfacto.py:933-940)
        float c0[3] = {0.f, 0.f, 0.f};
        const float* dcr = s_dc + tid * ndc;
        for (int f = 0; f < sg.F; ++f) {
            const float w = sg.idft[f];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) c0[ch] += dcr[f * 3 + ch] * w;
        }
        float rgb[3];
        int aux = SGN_AUX_VISIBLE | cls_bit;
        if (cam.sh_degree > 0) {
            float d[3] = {ge[6] - cam.cam_pos[0], ge[7] - cam.cam_pos[1], ge[8] - cam.cam_pos[2]};
            const float n = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            d[0] /= n; d[1] /= n; d[2] /= n;
            float Y[16];
            sgn_sh_basis(cam.sh_degree_to_use, d[0], d[1], d[2], Y);
            const int Kuse = min((cam.sh_degree_to_use + 1) * (cam.sh_degree_to_use + 1), K);
            float acc[3] = {Y[0] * c0[0], Y[0] * c0[1], Y[0] * c0[2]};
            const float* rr = s_rest + tid * nrest;
            for (int k = 1; k < Kuse; ++k) {
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) acc[ch] += Y[k] * rr[(k - 1) * 3 + ch];
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float pre = acc[ch] + 0.5f;
                if (pre >= 0.f) aux |= (1 << ch);
                rgb[ch] = pre > 0.f ? pre : 0.f;
            }
        } else {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) { rgb[ch] = 1.f / (1.f + expf(-c0[ch])); aux |= (1 << ch); }
        }
        float opac = 1.f / (1.f + expf(-__ldg(sg.opacities + r0 + row)));
        if (cam.filter_3d) opac = opac * ge[10];   // uniform
        if (cam.antialiased) opac = opac * ge[9];  // warp-uniform
        float4* rec = records + 3 * gb;
        rec[1] = make_float4(ge[4], opac, rgb[0], rgb[1]);
        rec[2] = make_float4(rgb[2], ge[5], __int_as_float(aux), ge[9]);
        bb = tile_bbox[gb];  // written by this block in phase A (visible to the block after the barriers above)
        tc = make_touch_ctx(make_float4(ge[0], ge[1], ge[2], ge[3]), make_float4(ge[4], opac, 0.f, 0.f));
    }
    // tiles the Gaussian can really reach (exact ellipse-vs-tile test, sgn_touch.cuh); binning lists only those.
    // Warp-collective: whole warps without a visible row skip it together.
    if ((warp << 5) >= nvis) return;
    uint32_t mask;
    const int nt = count_touched_tiles(mine, tc, bb, cam.width, cam.height, cam.block_width, mask);
    if (mine) {
        tiles_touched[gb] = nt;
        touch_mask[gb] = mask;
    }
}

static int project_fwd_check(const char* what, const sgn_segment* segs_dev, int nseg, int N, int num_chunks, const sgn_camera* cam,
                             float* records, int32_t* radii, int32_t* num_tiles_hit, uint16_t* tile_bbox,
                             int32_t* tiles_touched, uint32_t* touch_mask) {
    SGN_REQUIRE(segs_dev && cam && records && radii && num_tiles_hit && tile_bbox && tiles_touched && touch_mask,
                "%s: null pointer", what);
    SGN_REQUIRE(nseg >= 1 && nseg <= SGN_MAX_SEGMENTS, "%s: nseg=%d out of range [1,%d]", what, nseg, SGN_MAX_SEGMENTS);
    SGN_REQUIRE(N >= 0 && num_chunks >= 0, "%s: negative size", what);
    SGN_REQUIRE(cam->block_width >= 2 && cam->block_width <= 16, "block_width must be between 2 and 16 (got %d)", cam->block_width);
    SGN_REQUIRE(cam->sh_degree >= 0 && cam->sh_degree <= 3 && cam->sh_degree_to_use >= 0 && cam->sh_degree_to_use <= cam->sh_degree,
                "sh_degree must be in [0,3] and sh_degree_to_use <= sh_degree");
    SGN_REQUIRE((cam->width + cam->block_width - 1) / cam->block_width < 65536 && (cam->height + cam->block_width - 1) / cam->block_width < 65536,
                "image too large for 16-bit tile coordinates");
    SGN_REQUIRE(sgn_aligned16(records), "records must be 16-byte aligned");
    return SGN_OK;
}

extern "C" int sgn_project_fwd_view(const sgn_segment* segs_dev, int nseg, int N, int num_chunks, const sgn_camera* cam,
                                    const float* view, float* records, int32_t* radii, int32_t* num_tiles_hit, uint16_t* tile_bbox,
                                    int32_t* tiles_touched, uint32_t* touch_mask, void* stream) {
    SGN_RANGE("sgn_project_fwd_view");
    if (int rc = project_fwd_check("sgn_project_fwd_view", segs_dev, nseg, N, num_chunks, cam, records, radii, num_tiles_hit, tile_bbox,
                                   tiles_touched, touch_mask)) return rc;
    SGN_REQUIRE(view, "sgn_project_fwd_view: null view");
    if (N == 0 || num_chunks == 0) return SGN_OK;
    project_fwd_direct_kernel<true><<<num_chunks, CH, nseg * sizeof(int), (cudaStream_t)stream>>>(
        segs_dev, nseg, *cam, reinterpret_cast<float4*>(records), radii, num_tiles_hit,
        reinterpret_cast<ushort4*>(tile_bbox), tiles_touched, touch_mask, view);
    SGN_CHECK_LAUNCH("project_fwd_kernel<view>");
    return SGN_OK;
}

extern "C" int sgn_project_fwd(const sgn_segment* segs_dev, int nseg, int N, int num_chunks, const sgn_camera* cam,
                               float* records, int32_t* radii, int32_t* num_tiles_hit, uint16_t* tile_bbox,
                               int32_t* tiles_touched, uint32_t* touch_mask, void* stream) {
    SGN_RANGE("sgn_project_fwd");
    if (int rc = project_fwd_check("sgn_project_fwd", segs_dev, nseg, N, num_chunks, cam, records, radii, num_tiles_hit, tile_bbox,
                                   tiles_touched, touch_mask)) return rc;
    if (N == 0 || num_chunks == 0) return SGN_OK;
    // SGN_PROJECT_STAGED=1: the two-phase form (compaction + shared-memory staging of the visible rows' colour parameters);
    // the direct form is the default.  Read on every call (one getenv per frame), so one process can run both forms.
    const char* staged_env = getenv("SGN_PROJECT_STAGED");
    if (staged_env && staged_env[0] == '1')
        project_fwd_staged_kernel<<<num_chunks, CH, nseg * sizeof(int), (cudaStream_t)stream>>>(
            segs_dev, nseg, *cam, reinterpret_cast<float4*>(records), radii, num_tiles_hit,
            reinterpret_cast<ushort4*>(tile_bbox), tiles_touched, touch_mask);
    else
        project_fwd_direct_kernel<false><<<num_chunks, CH, nseg * sizeof(int), (cudaStream_t)stream>>>(
            segs_dev, nseg, *cam, reinterpret_cast<float4*>(records), radii, num_tiles_hit,
            reinterpret_cast<ushort4*>(tile_bbox), tiles_touched, touch_mask, nullptr);
    SGN_CHECK_LAUNCH("project_fwd_kernel");
    return SGN_OK;
}

// geometry backward shared by the fused and the Level-1 kernels: cotangents of (xy, depth, conic) ->
// (world mean, scale as used [st.s], composed quaternion qr).
// VIEW: also this row's cotangent of the view [W | c] (viewmat[12] row-major) into vview.  With the camera-space mean
// p_c = W p_w + c and covariance S_c = W S_w W^T: v_W = v_pc p_w^T + 2 G W S_w, v_c = v_pc, where v_pc (vpv below) is the
// complete cotangent of p_c (xy, depth and the Jacobian's dependence on p_c) and G = J^T g J that of S_c; 2 G W S_w = J^T vT
// since T = J W and vT = 2 g T S_w.
// with_comp (a warp-uniform flag): also the cotangent v_comp of comp (the forward's sgn_compensation), through cov2d.  Its
// un-blurred diagonal is rebuilt from st.T and st.S (the forward's bits), so that it does not stay live from the projection
// to here.
template <bool VIEW = false>
__device__ __forceinline__ void sgn_project_vjp(const sgn_camera& cam, const SgnProj& st, const float v_xy[2], float v_depth,
                                                const float v_conic[3], float vmw[3], float vs[3], float vqr[4],
                                                float* vview = nullptr, bool with_comp = false, float comp = 0.f,
                                                float v_comp = 0.f) {
    const float* W = cam.viewmat;
    const float fx = cam.fx, fy = cam.fy;
    float vpv[3];
    {
        const float rw = 1.f / (st.pv[2] + 1e-6f);
        const float vx = fx * v_xy[0], vy = fy * v_xy[1];
        vpv[0] = vx * rw;
        vpv[1] = vy * rw;
        vpv[2] = -(vx * st.pv[0] + vy * st.pv[1]) * rw * rw + v_depth;
    }
    float vA, vB, vC;
    {
        const float X0 = st.conic[0], X1 = st.conic[1], X2 = st.conic[2];
        const float G0 = v_conic[0], G1 = 0.5f * v_conic[1], G2 = v_conic[2];
        const float a00 = X0 * G0 + X1 * G1, a01 = X0 * G1 + X1 * G2;
        const float a10 = X1 * G0 + X2 * G1, a11 = X1 * G1 + X2 * G2;
        vA = -(a00 * X0 + a01 * X1);
        vB = -(a00 * X1 + a01 * X2) - (a10 * X0 + a11 * X1);
        vC = -(a10 * X1 + a11 * X2);
    }
    if (with_comp) {
        xf T[6], S[6], a, b, c, c00, c11;
#pragma unroll
        for (int k = 0; k < 6; ++k) { T[k] = xf(st.T[k]); S[k] = xf(st.S[k]); }
        sgn_cov2d_blur(T, S, a, b, c, c00, c11);
        sgn_compensation_vjp(c00.v, c11.v, a.v, b.v, c.v, comp, v_comp, vA, vB, vC);
    }
    const float g00 = vA, g01 = 0.5f * vB, g11 = vC;
    const float* T = st.T;
    const float Sf[9] = {st.S[0], st.S[1], st.S[2], st.S[1], st.S[3], st.S[4], st.S[2], st.S[4], st.S[5]};
    float GT[6];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        GT[c] = g00 * T[c] + g01 * T[3 + c];
        GT[3 + c] = g01 * T[c] + g11 * T[3 + c];
    }
    float vS[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) vS[3 * r + c] = T[r] * GT[c] + T[3 + r] * GT[3 + c];
    float vT[6];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            vT[3 * r + c] = 2.f * (GT[3 * r] * Sf[c] + GT[3 * r + 1] * Sf[3 + c] + GT[3 * r + 2] * Sf[6 + c]);
    const float vJ00 = vT[0] * W[0] + vT[1] * W[1] + vT[2] * W[2];
    const float vJ02 = vT[0] * W[8] + vT[1] * W[9] + vT[2] * W[10];
    const float vJ11 = vT[3] * W[4] + vT[4] * W[5] + vT[5] * W[6];
    const float vJ12 = vT[3] * W[8] + vT[4] * W[9] + vT[5] * W[10];
    {
        const float rz = 1.f / st.pv[2], rz2 = rz * rz, rz3 = rz2 * rz;
        const float vtx = -fx * rz2 * vJ02;
        const float vty = -fy * rz2 * vJ12;
        const float vtz = -fx * rz2 * vJ00 - fy * rz2 * vJ11 + 2.f * fx * st.tx * rz3 * vJ02 + 2.f * fy * st.ty * rz3 * vJ12;
        if (st.clampx == 0) vpv[0] += vtx; else vpv[2] += (st.clampx > 0 ? cam.limx : -cam.limx) * vtx;
        if (st.clampy == 0) vpv[1] += vty; else vpv[2] += (st.clampy > 0 ? cam.limy : -cam.limy) * vty;
        vpv[2] += vtz;
        if constexpr (VIEW) {
            const float J00 = fx * rz, J11 = fy * rz, J02 = -fx * st.tx * rz2, J12 = -fy * st.ty * rz2;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                vview[c] = vpv[0] * st.mw[c] + J00 * vT[c];
                vview[4 + c] = vpv[1] * st.mw[c] + J11 * vT[3 + c];
                vview[8 + c] = vpv[2] * st.mw[c] + J02 * vT[c] + J12 * vT[3 + c];
            }
#pragma unroll
            for (int r = 0; r < 3; ++r) vview[4 * r + 3] = vpv[r];
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) vmw[c] = W[c] * vpv[0] + W[4 + c] * vpv[1] + W[8 + c] * vpv[2];
    float M[9], vM[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) M[3 * r + c] = st.Rg[3 * r + c] * st.s[c];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            vM[3 * r + c] = 2.f * (vS[3 * r] * M[c] + vS[3 * r + 1] * M[3 + c] + vS[3 * r + 2] * M[6 + c]);
    float vR[9];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        vs[c] = st.Rg[c] * vM[c] + st.Rg[3 + c] * vM[3 + c] + st.Rg[6 + c] * vM[6 + c];
#pragma unroll
        for (int r = 0; r < 3; ++r) vR[3 * r + c] = vM[3 * r + c] * st.s[c];
    }
    float vqn[4];
    {
        const float w = st.qn[0], x = st.qn[1], y = st.qn[2], z = st.qn[3];
        vqn[0] = 2.f * (x * (vR[7] - vR[5]) + y * (vR[2] - vR[6]) + z * (vR[3] - vR[1]));
        vqn[1] = 2.f * (-2.f * x * (vR[4] + vR[8]) + y * (vR[1] + vR[3]) + z * (vR[2] + vR[6]) + w * (vR[7] - vR[5]));
        vqn[2] = 2.f * (x * (vR[1] + vR[3]) - 2.f * y * (vR[0] + vR[8]) + z * (vR[5] + vR[7]) + w * (vR[2] - vR[6]));
        vqn[3] = 2.f * (x * (vR[2] + vR[6]) + y * (vR[5] + vR[7]) - 2.f * z * (vR[0] + vR[4]) + w * (vR[3] - vR[1]));
    }
    const float dot = vqn[0] * st.qn[0] + vqn[1] * st.qn[1] + vqn[2] * st.qn[2] + vqn[3] * st.qn[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) vqr[k] = (vqn[k] - st.qn[k] * dot) / st.qnorm;
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
// POSE: a block whose segment has an object->world pose also reduces the cotangents of that pose over its rows --
// v_R[r][c] = sum vmw[r] m[c] (means_w = R m + t), v_t = sum vmw, v_a = sum vqr (x) conj(q) (q_w = a (x) q, q un-normalised) --
// and stores the 16 sums to pose_partials[chunk]: warp shuffles, then the four warps in fixed order; no atomics, so the
// sums do not depend on the run.  Colour contributes nothing (the SH view direction is taken from detached means).
// VIEW: the view is read from the device (`view`, as in the forward) and every block also reduces the rows' cotangents of
// it (sgn_project_vjp<true>) the same way, storing SGN_VIEW_FLOATS sums to view_partials[chunk].
template <bool POSE, bool VIEW = false>
__global__ void __launch_bounds__(CH)
project_bwd_kernel(const sgn_segment* __restrict__ segs, const sgn_segment_grads* __restrict__ grads, int nseg,
                   const sgn_camera cam_arg, const float4* __restrict__ records, const int32_t* __restrict__ radii,
                   const float4* __restrict__ v_records, const int chunk_begin, float* __restrict__ pose_partials,
                   const float* __restrict__ view, float* __restrict__ view_partials) {
    sgn_camera cam_view;
    if constexpr (VIEW) cam_view = sgn_camera_with_view(cam_arg, view);
    const sgn_camera& cam = VIEW ? cam_view : cam_arg;
    extern __shared__ int s_chunk0[];
    __shared__ __align__(16) float s_rest[CH * MAX_REST];   // out: features_rest gradient rows
    __shared__ __align__(16) float s_dc[CH * MAX_DC];       // out: features_dc gradient rows
    __shared__ __align__(16) float s_means[CH * 3];         // in: means, then out: means gradient
    __shared__ __align__(16) float s_scales[CH * 3];        // in: scales, then out: scales gradient
    for (int i = threadIdx.x; i < nseg; i += blockDim.x) s_chunk0[i] = segs[i].chunk0;
    __syncthreads();
    const int chunk = chunk_begin + (int)blockIdx.x;
    const int si = find_segment_by_chunk(s_chunk0, nseg, chunk);
    const sgn_segment& sg = segs[si];
    const sgn_segment_grads& gr = grads[si];
    const int r0 = (chunk - sg.chunk0) * CH;
    const int rows = min(CH, sg.count - r0);
    const int K = (cam.sh_degree + 1) * (cam.sh_degree + 1);
    const int nrest = (K - 1) * 3, ndc = sg.F * 3;
    coop_load(s_means, sg.means + 3 * (size_t)r0, rows * 3);
    coop_load(s_scales, sg.scales + 3 * (size_t)r0, rows * 3);
    __syncthreads();
    const int tid = threadIdx.x;
    float gm[3] = {0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f};
    float vp[POSE ? SGN_POSE_FLOATS : 1] = {};  // this row's share of (v_R 9, v_t 3, v_a 4)
    float vv[VIEW ? SGN_VIEW_FLOATS : 1] = {};  // this row's share of v_view
    const bool row_vis = (tid < rows) && radii[(size_t)sg.row0 + r0 + tid] > 0;
    if (tid < rows && !row_vis) {
        // the rasterizer never touched this Gaussian: every cotangent is zero, so is every gradient
        const int i = r0 + tid;
        gr.opacities[i] = 0.f;
        reinterpret_cast<float4*>(gr.quats)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        float* grest = s_rest + tid * nrest;
        for (int k = 0; k < nrest; ++k) grest[k] = 0.f;
        float* gdc = s_dc + tid * ndc;
        for (int k = 0; k < ndc; ++k) gdc[k] = 0.f;
    }
    if (row_vis) {
        const int i = r0 + tid;
        const size_t g = (size_t)sg.row0 + i;
        const float4 v0 = v_records[3 * g], v1 = v_records[3 * g + 1], v2 = v_records[3 * g + 2];
        const float v_xy[2] = {v0.x, v0.y};
        const float v_conic[3] = {v0.z, v0.w, v1.x};
        const float v_opac = v1.y;
        const float v_rgb[3] = {v1.z, v1.w, v2.x};
        const float v_depth = v2.y;
        const float4 r1 = records[3 * g + 1], r2 = records[3 * g + 2];
        const int aux = __float_as_int(r2.z);
        const bool filt = cam.filter_3d != nullptr;  // uniform: the 3D smoothing filter
        if (!cam.antialiased && !filt) {  // opacity: sigmoid backward (the antialiased mode's and the filter's below)
            const float o = r1.y;
            gr.opacities[i] = v_opac * o * (1.f - o);
        }
        const float m[3] = {s_means[3 * tid], s_means[3 * tid + 1], s_means[3 * tid + 2]};
        const float ls[3] = {s_scales[3 * tid], s_scales[3 * tid + 1], s_scales[3 * tid + 2]};
        float q[4];
        {
            const float4 qq = __ldg(reinterpret_cast<const float4*>(sg.quats) + i);
            q[0] = qq.x; q[1] = qq.y; q[2] = qq.z; q[3] = qq.w;
        }
        const float sigma = filt ? __ldg(cam.filter_3d[si] + i) : 0.f;
        SgnProj st;
        const bool vis = sgn_project_exact(sg, cam, m, ls, q, st, true, 1.f, false, filt, sigma);
        // colour backward (compute_sh_backward + clamp mask + Fourier DC) into the staging rows
        {
            float vc[3];
            float* grest = s_rest + tid * nrest;
            if (cam.sh_degree > 0) {
                float d[3] = {st.mw[0] - cam.cam_pos[0], st.mw[1] - cam.cam_pos[1], st.mw[2] - cam.cam_pos[2]};
                const float n = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
                d[0] /= n; d[1] /= n; d[2] /= n;
                float Y[16];
                sgn_sh_basis(cam.sh_degree_to_use, d[0], d[1], d[2], Y);
                const int Kuse = (cam.sh_degree_to_use + 1) * (cam.sh_degree_to_use + 1);
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) vc[ch] = (aux & (1 << ch)) ? v_rgb[ch] : 0.f;
                for (int k = 1; k < K; ++k) {
                    const float y = (k < Kuse) ? Y[k] : 0.f;
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) grest[(k - 1) * 3 + ch] = y * vc[ch];
                }
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) vc[ch] *= Y[0];
            } else {
                const float rgb[3] = {r1.z, r1.w, r2.x};
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) vc[ch] = v_rgb[ch] * rgb[ch] * (1.f - rgb[ch]);
                for (int k = 0; k < nrest; ++k) grest[k] = 0.f;
            }
            float* gdc = s_dc + tid * ndc;
            for (int f = 0; f < sg.F; ++f) {
                const float w = sg.idft[f];
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) gdc[f * 3 + ch] = w * vc[ch];
            }
        }
        // antialiased mode: record [5] = s comp with s = sigmoid(logit) and comp in record [11]; v_comp = v_opac s goes on
        // through cov2d (sgn_project_vjp)
        // 3D filter: record [5] = s coef [comp]; v_coef = v_opac s [comp] reaches the log-scales through coef, and the scales'
        // cotangent passes d s' / d log s = r s' (coef and r recomputed from the parameters and sigma, as the forward has them)
        float v_comp = 0.f, comp = 0.f, v_coef = 0.f;
        if (cam.antialiased || filt) {  // warp-uniform
            const float s = 1.f / (1.f + expf(-__ldg(sg.opacities + i)));  // the forward's sigmoid, not record [5]
            float f = 1.f;  // the factors of the opacity beyond the sigmoid
            if (cam.antialiased) {
                v_comp = v_opac * s;
                f = r2.w;
                comp = __ldg(reinterpret_cast<const float*>(records) + 12 * g + 11);  // read again here: nothing stays live
            }
            if (filt) {
                v_coef = v_opac * s * f;
                v_comp = v_comp * st.coef;
                f = f * st.coef;
            }
            gr.opacities[i] = v_opac * f * s * (1.f - s);
        }
        if (vis && radii[g] > 0) {
            float vmw[3], vs[3], vqr[4];
            sgn_project_vjp<VIEW>(cam, st, v_xy, v_depth, v_conic, vmw, vs, vqr, vv, cam.antialiased != 0, comp, v_comp);
#pragma unroll
            for (int c = 0; c < 3; ++c) gs[c] = vs[c] * st.s[c];  // through exp
            if (filt) {
                float r[3];
                sgn_filter_ratios(ls, sigma, r);
                const float vc = v_coef * st.coef;
#pragma unroll
                for (int c = 0; c < 3; ++c) gs[c] = gs[c] * r[c] + vc * (1.f - r[c]);
            }
            if (sg.has_pose) {
                const float* R = sg.R;
#pragma unroll
                for (int c = 0; c < 3; ++c) gm[c] = R[c] * vmw[0] + R[3 + c] * vmw[1] + R[6 + c] * vmw[2];
                const float aw = sg.q[0], ax = sg.q[1], ay = sg.q[2], az = sg.q[3];
                gq[0] = aw * vqr[0] + ax * vqr[1] + ay * vqr[2] + az * vqr[3];
                gq[1] = -ax * vqr[0] + aw * vqr[1] + az * vqr[2] - ay * vqr[3];
                gq[2] = -ay * vqr[0] - az * vqr[1] + aw * vqr[2] + ax * vqr[3];
                gq[3] = -az * vqr[0] + ay * vqr[1] - ax * vqr[2] + aw * vqr[3];
                if constexpr (POSE) {
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
#pragma unroll
                        for (int c = 0; c < 3; ++c) vp[3 * r + c] = vmw[r] * m[c];
                        vp[9 + r] = vmw[r];
                    }
                    vp[12] = vqr[0] * q[0] + vqr[1] * q[1] + vqr[2] * q[2] + vqr[3] * q[3];
                    vp[13] = -vqr[0] * q[1] + vqr[1] * q[0] - vqr[2] * q[3] + vqr[3] * q[2];
                    vp[14] = -vqr[0] * q[2] + vqr[1] * q[3] + vqr[2] * q[0] - vqr[3] * q[1];
                    vp[15] = -vqr[0] * q[3] - vqr[1] * q[2] + vqr[2] * q[1] + vqr[3] * q[0];
                }
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) gm[c] = vmw[c];
#pragma unroll
                for (int k = 0; k < 4; ++k) gq[k] = vqr[k];
            }
        }
        reinterpret_cast<float4*>(gr.quats)[i] = make_float4(gq[0], gq[1], gq[2], gq[3]);
    }
    if constexpr (POSE) {
        __shared__ float s_pose[(CH / 32) * SGN_POSE_FLOATS];
        if (sg.has_pose) {  // block-uniform: a chunk never straddles segments
#pragma unroll
            for (int k = 0; k < SGN_POSE_FLOATS; ++k) {
                float x = vp[k];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
                if ((tid & 31) == 0) s_pose[(tid >> 5) * SGN_POSE_FLOATS + k] = x;
            }
            __syncthreads();
            if (tid < SGN_POSE_FLOATS) {
                float x = s_pose[tid];
#pragma unroll
                for (int w = 1; w < CH / 32; ++w) x += s_pose[w * SGN_POSE_FLOATS + tid];
                pose_partials[(size_t)chunk * SGN_POSE_FLOATS + tid] = x;
            }
        }
    }
    if constexpr (VIEW) {
        __shared__ float s_view[(CH / 32) * SGN_VIEW_FLOATS];
#pragma unroll
        for (int k = 0; k < SGN_VIEW_FLOATS; ++k) {
            float x = vv[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
            if ((tid & 31) == 0) s_view[(tid >> 5) * SGN_VIEW_FLOATS + k] = x;
        }
        __syncthreads();
        if (tid < SGN_VIEW_FLOATS) {
            float x = s_view[tid];
#pragma unroll
            for (int w = 1; w < CH / 32; ++w) x += s_view[w * SGN_VIEW_FLOATS + tid];
            view_partials[(size_t)chunk * SGN_VIEW_FLOATS + tid] = x;
        }
    }
    __syncthreads();  // every thread has consumed its means / scales inputs
    if (tid < rows) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { s_means[3 * tid + k] = gm[k]; s_scales[3 * tid + k] = gs[k]; }
    }
    __syncthreads();
    coop_store(gr.means + 3 * (size_t)r0, s_means, rows * 3);
    coop_store(gr.scales + 3 * (size_t)r0, s_scales, rows * 3);
    coop_store(gr.features_dc + (size_t)r0 * ndc, s_dc, rows * ndc);
    if (nrest > 0) coop_store(gr.features_rest + (size_t)r0 * nrest, s_rest, rows * nrest);
}

static int project_bwd_launch(const char* what, const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                              const sgn_camera* cam, const float* records, const int32_t* radii, const float* v_records,
                              int chunk_begin, int chunk_end, float* pose_partials, bool pose, void* stream,
                              const float* view = nullptr, float* view_partials = nullptr) {
    SGN_REQUIRE(segs_dev && grads_dev && cam && records && radii && v_records, "%s: null pointer", what);
    SGN_REQUIRE(!pose || pose_partials, "%s: null pose_partials", what);
    SGN_REQUIRE((view == nullptr) == (view_partials == nullptr), "%s: give both view and view_partials, or neither", what);
    SGN_REQUIRE(nseg >= 1 && nseg <= SGN_MAX_SEGMENTS, "%s: nseg=%d out of range", what, nseg);
    SGN_REQUIRE(sgn_aligned16(records) && sgn_aligned16(v_records), "records / v_records must be 16-byte aligned");
    SGN_REQUIRE(chunk_begin >= 0 && chunk_begin <= chunk_end && chunk_end <= num_chunks, "%s: chunk range [%d, %d) outside [0, %d)",
                what, chunk_begin, chunk_end, num_chunks);
    if (N == 0 || chunk_end == chunk_begin) return SGN_OK;
    auto kernel = view ? (pose ? project_bwd_kernel<true, true> : project_bwd_kernel<false, true>)
                       : (pose ? project_bwd_kernel<true, false> : project_bwd_kernel<false, false>);
    kernel<<<chunk_end - chunk_begin, CH, nseg * sizeof(int), (cudaStream_t)stream>>>(
        segs_dev, grads_dev, nseg, *cam, reinterpret_cast<const float4*>(records), radii,
        reinterpret_cast<const float4*>(v_records), chunk_begin, pose_partials, view, view_partials);
    SGN_CHECK_LAUNCH("project_bwd_kernel");
    return SGN_OK;
}

extern "C" int sgn_project_bwd_range(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                                     const sgn_camera* cam, const float* records, const int32_t* radii,
                                     const float* v_records, int chunk_begin, int chunk_end, void* stream) {
    SGN_RANGE("sgn_project_bwd");
    return project_bwd_launch("sgn_project_bwd", segs_dev, grads_dev, nseg, N, num_chunks, cam, records, radii, v_records, chunk_begin,
                              chunk_end, nullptr, false, stream);
}

extern "C" int sgn_project_bwd(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                               const sgn_camera* cam, const float* records, const int32_t* radii,
                               const float* v_records, void* stream) {
    return sgn_project_bwd_range(segs_dev, grads_dev, nseg, N, num_chunks, cam, records, radii, v_records, 0, num_chunks > 0 ? num_chunks : 0, stream);
}

extern "C" int sgn_project_bwd_pose(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                                    const sgn_camera* cam, const float* records, const int32_t* radii, const float* v_records,
                                    int chunk_begin, int chunk_end, float* pose_partials, void* stream) {
    SGN_RANGE("sgn_project_bwd_pose");
    return project_bwd_launch("sgn_project_bwd_pose", segs_dev, grads_dev, nseg, N, num_chunks, cam, records, radii, v_records,
                              chunk_begin, chunk_end, pose_partials, true, stream);
}

extern "C" int sgn_project_bwd_view(const sgn_segment* segs_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                                    const sgn_camera* cam, const float* view, const float* records, const int32_t* radii,
                                    const float* v_records, int chunk_begin, int chunk_end, float* pose_partials, float* view_partials,
                                    void* stream) {
    SGN_RANGE("sgn_project_bwd_view");
    SGN_REQUIRE(view && view_partials, "sgn_project_bwd_view: null view or view_partials");
    return project_bwd_launch("sgn_project_bwd_view", segs_dev, grads_dev, nseg, N, num_chunks, cam, records, radii, v_records,
                              chunk_begin, chunk_end, pose_partials, pose_partials != nullptr, stream, view, view_partials);
}

// One block of VR_THREADS = 80 x SGN_VIEW_FLOATS threads: thread t sums the floats t, t + VR_THREADS, ... of view_partials
// (all of one value k = t % 12, coalesced), in ascending order; then thread k < 12 sums the 80 partial sums of value k in
// ascending order.  A fixed order throughout: v_view is the same bits on every run.
#define VR_THREADS (80 * SGN_VIEW_FLOATS)
__global__ void __launch_bounds__(VR_THREADS)
view_reduce_kernel(int num_chunks, const float* __restrict__ view_partials, float* __restrict__ v_view) {
    __shared__ float s_sum[VR_THREADS];
    const int tid = threadIdx.x;
    const long long n = (long long)num_chunks * SGN_VIEW_FLOATS;
    float x = 0.f;
    for (long long e = tid; e < n; e += VR_THREADS) x += __ldg(view_partials + e);
    s_sum[tid] = x;
    __syncthreads();
    if (tid < SGN_VIEW_FLOATS) {
        float y = 0.f;
        for (int j = tid; j < VR_THREADS; j += SGN_VIEW_FLOATS) y += s_sum[j];
        v_view[tid] = y;
    }
}

extern "C" int sgn_view_grad_reduce(int num_chunks, const float* view_partials, float* v_view, void* stream) {
    SGN_RANGE("sgn_view_grad_reduce");
    SGN_REQUIRE(v_view, "sgn_view_grad_reduce: null v_view");
    SGN_REQUIRE(num_chunks >= 0 && (num_chunks == 0 || view_partials), "sgn_view_grad_reduce: null view_partials for %d chunks", num_chunks);
    view_reduce_kernel<<<1, VR_THREADS, 0, (cudaStream_t)stream>>>(num_chunks, view_partials, v_view);
    SGN_CHECK_LAUNCH("view_reduce_kernel");
    return SGN_OK;
}

// One warp per segment: the sums of pose_partials over the segment's chunks, in a fixed order (lane = value + 16 x chunk
// parity, chunks ascending, then the two parities) -> v_pose[segment]; zeros for a segment without a pose.
__global__ void __launch_bounds__(CH)
pose_reduce_kernel(const sgn_segment* __restrict__ segs, int nseg, const float* __restrict__ pose_partials, float* __restrict__ v_pose) {
    const int si = blockIdx.x * (CH / 32) + (threadIdx.x >> 5);
    if (si >= nseg) return;
    const int lane = threadIdx.x & 31, k = lane & (SGN_POSE_FLOATS - 1);
    float x = 0.f;
    if (segs[si].has_pose) {
        const int chunk0 = segs[si].chunk0, n = (segs[si].count + CH - 1) / CH;
        for (int c = lane >> 4; c < n; c += 2) x += pose_partials[(size_t)(chunk0 + c) * SGN_POSE_FLOATS + k];
    }
    x += __shfl_down_sync(0xffffffffu, x, 16);
    if (lane < SGN_POSE_FLOATS) v_pose[(size_t)si * SGN_POSE_FLOATS + lane] = x;
}

extern "C" int sgn_pose_grad_reduce(const sgn_segment* segs_dev, int nseg, int num_chunks, const float* pose_partials, float* v_pose,
                                    void* stream) {
    SGN_RANGE("sgn_pose_grad_reduce");
    SGN_REQUIRE(segs_dev && v_pose, "sgn_pose_grad_reduce: null pointer");
    SGN_REQUIRE(nseg >= 1 && nseg <= SGN_MAX_SEGMENTS, "sgn_pose_grad_reduce: nseg=%d out of range", nseg);
    SGN_REQUIRE(num_chunks >= 0 && (num_chunks == 0 || pose_partials), "sgn_pose_grad_reduce: null pose_partials for %d chunks", num_chunks);
    pose_reduce_kernel<<<(nseg + CH / 32 - 1) / (CH / 32), CH, 0, (cudaStream_t)stream>>>(segs_dev, nseg, pose_partials, v_pose);
    SGN_CHECK_LAUNCH("pose_reduce_kernel");
    return SGN_OK;
}

// ================================================================================================
// Level-1 entry points: gsplat 0.1.x function API (project_gaussians / spherical_harmonics) on plain
// tensors, for the reference's unmodified model code (street_gaussians_ns/sgn_splatfacto.py:11-14,
// 860-873, 939).  Same device functions as the fused path.
// ================================================================================================
__global__ void __launch_bounds__(PROJ_THREADS)
l1_project_fwd_kernel(int N, const float* __restrict__ means, const float* __restrict__ scales, float glob_scale,
                      const float* __restrict__ quats, const sgn_camera cam, float* __restrict__ xys,
                      float* __restrict__ depths, int32_t* __restrict__ radii, float* __restrict__ conics,
                      float* __restrict__ comp, int32_t* __restrict__ num_tiles_hit, float* __restrict__ cov3d) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    sgn_segment sg;
    sg.has_pose = 0;
    const float m[3] = {means[3 * g], means[3 * g + 1], means[3 * g + 2]};
    const float sc[3] = {scales[3 * g], scales[3 * g + 1], scales[3 * g + 2]};
    const float q[4] = {quats[4 * g], quats[4 * g + 1], quats[4 * g + 2], quats[4 * g + 3]};
    SgnProj st;
    const bool vis = sgn_project_exact(sg, cam, m, sc, q, st, false, glob_scale, true);
    const bool clipped = st.pv[2] <= cam.clip_thresh;
    xys[2 * g] = st.xy[0]; xys[2 * g + 1] = st.xy[1];
    depths[g] = vis ? st.pv[2] : 0.f;
    radii[g] = st.radius;
    conics[3 * g] = st.conic[0]; conics[3 * g + 1] = st.conic[1]; conics[3 * g + 2] = st.conic[2];
    num_tiles_hit[g] = vis ? (st.tmax[0] - st.tmin[0]) * (st.tmax[1] - st.tmin[1]) : 0;
    comp[g] = vis ? st.comp : 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) cov3d[6 * g + k] = clipped ? 0.f : st.S[k];
}

extern "C" int sgn_l1_project_fwd(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                                  const sgn_camera* cam, float* xys, float* depths, int32_t* radii, float* conics,
                                  float* compensation, int32_t* num_tiles_hit, float* cov3d, void* stream) {
    SGN_RANGE("sgn_l1_project_fwd");
    SGN_REQUIRE(means && scales && quats && cam && xys && depths && radii && conics && compensation && num_tiles_hit && cov3d,
                "sgn_l1_project_fwd: null pointer");
    SGN_REQUIRE(cam->block_width >= 2 && cam->block_width <= 16, "block_width must be between 2 and 16 (got %d)", cam->block_width);
    if (N == 0) return SGN_OK;
    l1_project_fwd_kernel<<<(N + PROJ_THREADS - 1) / PROJ_THREADS, PROJ_THREADS, 0, (cudaStream_t)stream>>>(
        N, means, scales, glob_scale, quats, *cam, xys, depths, radii, conics, compensation, num_tiles_hit, cov3d);
    SGN_CHECK_LAUNCH("l1_project_fwd_kernel");
    return SGN_OK;
}

__global__ void __launch_bounds__(PROJ_THREADS)
l1_project_bwd_kernel(int N, const float* __restrict__ means, const float* __restrict__ scales, float glob_scale,
                      const float* __restrict__ quats, const sgn_camera cam, const int32_t* __restrict__ radii,
                      const float* __restrict__ v_xys, const float* __restrict__ v_depths, const float* __restrict__ v_conics,
                      const float* __restrict__ v_comp, float* __restrict__ v_means, float* __restrict__ v_scales,
                      float* __restrict__ v_quats) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    float gm[3] = {0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f};
    if (radii[g] > 0) {
        sgn_segment sg;
        sg.has_pose = 0;
        const float m[3] = {means[3 * g], means[3 * g + 1], means[3 * g + 2]};
        const float sc[3] = {scales[3 * g], scales[3 * g + 1], scales[3 * g + 2]};
        const float q[4] = {quats[4 * g], quats[4 * g + 1], quats[4 * g + 2], quats[4 * g + 3]};
        SgnProj st;
        if (sgn_project_exact(sg, cam, m, sc, q, st, false, glob_scale, v_comp != nullptr)) {
            const float vxy[2] = {v_xys ? v_xys[2 * g] : 0.f, v_xys ? v_xys[2 * g + 1] : 0.f};
            const float vc[3] = {v_conics ? v_conics[3 * g] : 0.f, v_conics ? v_conics[3 * g + 1] : 0.f,
                                 v_conics ? v_conics[3 * g + 2] : 0.f};
            float vs[3];
            const bool with_comp = v_comp != nullptr;  // uniform: a NULL cotangent is sgn_l1_project_bwd, unchanged
            sgn_project_vjp(cam, st, vxy, v_depths ? v_depths[g] : 0.f, vc, gm, vs, gq, nullptr, with_comp, st.comp,
                            with_comp ? v_comp[g] : 0.f);
#pragma unroll
            for (int k = 0; k < 3; ++k) gs[k] = vs[k] * glob_scale;
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { v_means[3 * g + k] = gm[k]; v_scales[3 * g + k] = gs[k]; }
#pragma unroll
    for (int k = 0; k < 4; ++k) v_quats[4 * g + k] = gq[k];
}

static int l1_project_bwd_launch(const char* what, int N, const float* means, const float* scales, float glob_scale,
                                 const float* quats, const sgn_camera* cam, const int32_t* radii, const float* v_xys,
                                 const float* v_depths, const float* v_conics, const float* v_comp, float* v_means,
                                 float* v_scales, float* v_quats, void* stream) {
    SGN_REQUIRE(means && scales && quats && cam && radii && v_means && v_scales && v_quats, "%s: null pointer", what);
    if (N == 0) return SGN_OK;
    l1_project_bwd_kernel<<<(N + PROJ_THREADS - 1) / PROJ_THREADS, PROJ_THREADS, 0, (cudaStream_t)stream>>>(
        N, means, scales, glob_scale, quats, *cam, radii, v_xys, v_depths, v_conics, v_comp, v_means, v_scales, v_quats);
    SGN_CHECK_LAUNCH("l1_project_bwd_kernel");
    return SGN_OK;
}

extern "C" int sgn_l1_project_bwd(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                                  const sgn_camera* cam, const int32_t* radii, const float* v_xys, const float* v_depths,
                                  const float* v_conics, float* v_means, float* v_scales, float* v_quats, void* stream) {
    SGN_RANGE("sgn_l1_project_bwd");
    return l1_project_bwd_launch("sgn_l1_project_bwd", N, means, scales, glob_scale, quats, cam, radii, v_xys, v_depths,
                                 v_conics, nullptr, v_means, v_scales, v_quats, stream);
}

extern "C" int sgn_l1_project_bwd_comp(int N, const float* means, const float* scales, float glob_scale, const float* quats,
                                       const sgn_camera* cam, const int32_t* radii, const float* v_xys, const float* v_depths,
                                       const float* v_conics, const float* v_compensation, float* v_means, float* v_scales,
                                       float* v_quats, void* stream) {
    SGN_RANGE("sgn_l1_project_bwd_comp");
    return l1_project_bwd_launch("sgn_l1_project_bwd_comp", N, means, scales, glob_scale, quats, cam, radii, v_xys, v_depths,
                                 v_conics, v_compensation, v_means, v_scales, v_quats, stream);
}

// gsplat spherical_harmonics(degrees_to_use, viewdirs[N,3], coeffs[N,K,3]) -> colors[N,3]
__global__ void __launch_bounds__(PROJ_THREADS)
l1_sh_kernel(int N, int K, int degree, const float* __restrict__ viewdirs, const float* __restrict__ coeffs,
             const float* __restrict__ v_colors, float* __restrict__ colors, float* __restrict__ v_coeffs) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    float Y[16];
    sgn_sh_basis(degree, viewdirs[3 * g], viewdirs[3 * g + 1], viewdirs[3 * g + 2], Y);
    const int Kuse = min((degree + 1) * (degree + 1), K);
    if (colors) {
        float acc[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < Kuse; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) acc[ch] += Y[k] * coeffs[((size_t)g * K + k) * 3 + ch];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) colors[3 * g + ch] = acc[ch];
    }
    if (v_coeffs) {
        for (int k = 0; k < K; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) v_coeffs[((size_t)g * K + k) * 3 + ch] = (k < Kuse) ? Y[k] * v_colors[3 * g + ch] : 0.f;
    }
}

extern "C" int sgn_l1_sh(int N, int K, int degree, const float* viewdirs, const float* coeffs, const float* v_colors,
                         float* colors, float* v_coeffs, void* stream) {
    SGN_RANGE("sgn_l1_sh");
    SGN_REQUIRE(viewdirs && (colors || v_coeffs), "sgn_l1_sh: null pointer");
    SGN_REQUIRE(degree >= 0 && degree <= 3 && K >= 1 && K <= 16, "sgn_l1_sh: degree must be in [0,3], K in [1,16]");
    SGN_REQUIRE(!colors || coeffs, "sgn_l1_sh: forward needs coeffs");
    SGN_REQUIRE(!v_coeffs || v_colors, "sgn_l1_sh: backward needs v_colors");
    if (N == 0) return SGN_OK;
    l1_sh_kernel<<<(N + PROJ_THREADS - 1) / PROJ_THREADS, PROJ_THREADS, 0, (cudaStream_t)stream>>>(
        N, K, degree, viewdirs, coeffs, v_colors, colors, v_coeffs);
    SGN_CHECK_LAUNCH("l1_sh_kernel");
    return SGN_OK;
}
