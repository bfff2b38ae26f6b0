// Front-to-back alpha compositing, forward and backward, for 16x16 tiles.
//
// One traversal of each tile's depth-sorted list produces what the reference obtains from two gsplat
// rasterize_gaussians calls (street_gaussians_ns/sgn_splatfacto.py:954-996: rgb+alpha and the depth
// pass), with gsplat's skip and termination rules (SURVEY.md Appendix A.6).  The objects-only and
// background-only accumulations (street_gaussians_ns/sgn_splatfacto_scene_graph.py:364-366) see the
// compacted per-tile class sub-lists (binning.cu), which is what the reference's subset re-renders see.
// The objects-only one rides along in the main traversal (same alphas, a second transmittance advanced
// by the object entries only) and finishes on the object sub-list where the main streams ended; its
// gradient is folded into the main backward's reduction.  The background-only one is a separate
// accumulation-only traversal of the pixels an object entry took part in.  The reference's post-ops
// (:968-975, :995) run in the epilogue.
//
// Execution shape (H100): the loops are FP32/MUFU issue-bound, not HBM-bound, so the
// design minimises instructions per (pixel, Gaussian) pair:
//   * a warp owns a 16-column strip of a tile and each lane PPL pixels of one column (rows two apart):
//     dx and the dx-terms of the quadratic form are computed once per lane and shared by its pixels;
//     the per-Gaussian gradient reduction (10 values x 5 shuffle levels) is paid once per 32*PPL
//     pixels; the geometric gradients are accumulated per lane as three moments (S0, Sy, Syy);
//   * PPL = 8 (one warp per tile) is the throughput shape; tiles with long lists are split into
//     2/4/8 independent strips (PPL 4/2/1) so that no single warp's serial traversal becomes the
//     kernel's tail (per-tile lists reach thousands of entries behind dense actors);
//   * exp(-sigma) is one MUFU.EX2: the conic is pre-scaled by log2(e) when an entry is staged;
//   * entries are staged through a double-buffered shared-memory ring by the warp itself, the next
//     batch's gathers are in flight while the current batch is blended (no block-wide barriers);
//   * tiles are pre-culled exactly at binning time (binning.cu), so most staged entries are useful.
//
// Sorted payloads carry the Gaussian row in bits 0-30 and the object-class flag in bit 31.
#include "sgn_common.cuh"
#include "sgn_fixed.cuh"

#include <type_traits>

// Resident CTAs per SM the compiler must leave room for (register budget = 65536 / (32 * N) per thread); one warp per CTA, at
// most 32 CTAs per SM.  -maxrregcount is ignored for kernels with launch bounds, so the occupancy experiments go through these.
#ifndef BLEND_FWD_MIN_BLOCKS
#define BLEND_FWD_MIN_BLOCKS 16  // 128 registers: the objects-only stream would otherwise take the main forward to ~150
#endif
#ifndef BLEND_BWD_MIN_BLOCKS
#define BLEND_BWD_MIN_BLOCKS 12  // 168 registers: the folded objects-only gradient would otherwise take it to 178 (11 CTAs)
#endif
#ifndef BLEND_ACC_MIN_BLOCKS
#define BLEND_ACC_MIN_BLOCKS 1
#endif

#define ALPHA_MIN (1.f / 255.f)
#define T_STOP 1e-4f
#define ID_MASK 0x7fffffff
#define FULL 0xffffffffu
#define LOG2E 1.4426950408889634f
#define LN2 0.6931471805599453f
#define LOG2_255 7.994353436858858f

// saved per-pixel state is planar: slot 0 main, 1 object, 2 background
#define SLOT_MAIN 0
#define SLOT_OBJ 1
#define SLOT_BG 2
// background slot of final_idx: a pixel whose main stream met no valid object entry has a background
// accumulation bit-identical to its main accumulation (same alphas, same order, same products)
#define BG_SAME_AS_MAIN (-2)  // written by the main forward: T/idx/background_acc already final
#define BG_TODO (-3)          // an object entry took part: the background pass must traverse this pixel

struct BlendFwdParams {
    int width, height, tiles_x, tiles;
    int split_main, split_acc;  // list length up to which a tile is one strip (doubles per extra split)
    int32_t* tile_depth;  // [3][tiles] entries traversed per tile by the main / object / background pass (atomicMax)
    const int32_t* sched;  // heavy-first work lists (sched_kernel) or null
    float clamp_fwd;
    int has_sky, eval_clamp, raw_mode;
    float bg[4];
    const float4* records;
    const float4* staged;  // experiment (SGN_TUNE_FWD_TMA): the lists materialised as staged entries, 48 B each, in list order
    const int32_t* sorted_ids;
    const int2* tile_bins;
    const int32_t* cls_ids[2];  // class sub-lists: [0] background, [1] object
    const int2* cls_bins[2];
    const float* sky;
    float* rgb;
    float* acc;
    float* depth;
    float* obj_acc;
    float* bg_acc;
    float4* raw;
    float* final_T;      // [3][H*W]
    int32_t* final_idx;  // [3][H*W]
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ int warp_max(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(FULL, v, o));
    return v;
}

// Sums N per-lane values over the warp with N/2 + N/4 + ... shuffles instead of 5*N: at each butterfly
// level a lane keeps one half of its values and ships the other half to its partner, so the values end
// up spread over the lanes -- which is where the per-component atomics want them.  SHFL issues at a
// quarter of the FP32 rate, and the backward's 10 x 5 shuffles per entry were its largest single cost.
// Returns the warp total of the component multi_reduce_slot<N>(lane) names.
template <int N>
__device__ __forceinline__ float warp_multi_reduce(float (&v)[N], int lane) {
    int n = N;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        if (n == 1) {
            v[0] += __shfl_xor_sync(FULL, v[0], off);
        } else {
            const int half = (n + 1) / 2;
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < half; ++i) {
                const float hi = (i + half < n) ? v[i + half] : 0.f;
                const float send = up ? v[i] : hi;
                const float keep = up ? hi : v[i];
                v[i] = keep + __shfl_xor_sync(FULL, send, off);
            }
            n = half;
        }
    }
    return v[0];
}
// component (0..N-1) whose total warp_multi_reduce leaves in this lane; -1 for a padding slot and for the
// lanes that hold a duplicate of another lane's total (levels reached with one value left are plain sums)
template <int N>
__device__ __forceinline__ int multi_reduce_slot(int lane) {
    int sizes[6];
    sizes[0] = N;
#pragma unroll
    for (int l = 0; l < 5; ++l) sizes[l + 1] = sizes[l] > 1 ? (sizes[l] + 1) / 2 : 1;
    int idx = 0;
    bool ok = true;
#pragma unroll
    for (int l = 4; l >= 0; --l) {  // level l exchanges across lane bit (16 >> l)
        if (sizes[l] > 1) {
            if (lane & (16 >> l)) idx += sizes[l + 1];
            ok = ok && (idx < sizes[l]);
        } else if (lane & (16 >> l)) {
            ok = false;
        }
    }
    return ok ? idx : -1;
}

// One staged entry: A = (gx, gy, 0.5*a*log2e, b*log2e)  B = (0.5*c*log2e, log2(opacity), r, g)
//                   C = (b, depth, id bits, opacity)
// With sg = sigma*log2e:  o*exp(-sigma) = 2^(log2(o) - sg);  sigma >= 0 <=> sg >= 0;
// alpha >= 1/255 <=> sg <= log2(255 o).  Both tests only need sg, so validity is known before the MUFU result.
struct Staged {
    float4 A, B, C;
};

__device__ __forceinline__ Staged gather_entry(const float4* __restrict__ records, int id) {
    const float4* rec = records + 3 * (size_t)(id & ID_MASK);
    const float4 r0 = __ldg(rec), r1 = __ldg(rec + 1), r2 = __ldg(rec + 2);
    Staged s;
    s.A = make_float4(r0.x, r0.y, 0.5f * LOG2E * r0.z, LOG2E * r0.w);
    // an opacity that is not a positive number (NaN logits upstream) gets log2 = -inf: no pixel accepts the entry
    s.B = make_float4(0.5f * LOG2E * r1.x, r1.y > 0.f ? __log2f(r1.y) : __int_as_float(0xff800000) /* -inf */, r1.z, r1.w);
    s.C = make_float4(r2.x, r2.y, __int_as_float(id), r1.y);
    return s;
}

// Row reach of a staged entry: the largest |dy| (pixels) at which alpha >= 1/255 is still possible for
// SOME dx, i.e. min_dx sigma(dx,dy) <= ln(255 o).  In staged units: dy^2 * (hc - bb^2/(4 ha)) <= log2(255 o).
// Rows further away are skipped (warp-uniformly) by the accumulation kernels: a provable no-op.
__device__ __forceinline__ float row_reach(const Staged& e) {
    const float tau2 = LOG2_255 + e.B.y;
    const float den = e.B.x - (e.A.w * e.A.w) / (4.f * e.A.z);
    if (!(e.A.z > 0.f) || !(den > 0.f) || !(tau2 == tau2)) return 3.0e38f;  // degenerate conic: never cull
    if (tau2 < 0.f) return -1.f;                                             // opacity < 1/255: no row can accept it
    return sqrtf(tau2 / den) * 1.0001f + 0.01f;
}

// Pins an alpha clamp (a kernel parameter in [0.5, 1]) in a register: ptxas otherwise re-reads it from the
// constant bank (one LDC issue slot) inside every predicated slot body.  1 - (1 - x) is exact for
// 0.5 <= x <= 2 (Sterbenz) and is not something ptxas rematerialises.
__device__ __forceinline__ float in_register(float x) {
    float y;
    asm volatile("{.reg .f32 t; sub.rn.f32 t, 0f3F800000, %1; sub.rn.f32 %0, 0f3F800000, t;}" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float fast_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float fast_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ---- bulk-asynchronous staging (experiment, SGN_TUNE_FWD_TMA) --------------------------------------------------------
// The north-star names "TMA / shared-memory staging of per-tile sorted Gaussian records".  With the lists materialised as
// 48-byte staged entries in list order (sgn_blend_stage_entries), a batch of 32 entries is ONE contiguous 1.5 KB run, which
// the copy engine moves with cp.async.bulk (SASS: UBLKCP) and signals on an mbarrier -- no per-lane gathers, no log2 /
// rescale in the consumer.  The gathers cost < 1 instruction of a ~180-instruction entry, and materialising costs a 48 B
// write + read per entry: kept as a switchable variant, off by default.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

// Row-slot pairs (2p, 2p+1) of a lane, updated together: two independent IEEE fp32 operations per helper, which the
// scheduler dual-issues on Hopper's FP32 pipes.  Explicit .rn without .ftz: this file is built with --use_fast_math, and
// these bodies keep denormals and never contract, so the paired (PACKED) kernels round exactly as specified here.
struct f2 {
    float x, y;
};
__device__ __forceinline__ float fma_rn(float a, float b, float c) {
    float d;
    asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(d) : "f"(a), "f"(b), "f"(c));
    return d;
}
__device__ __forceinline__ float mul_rn(float a, float b) {
    float d;
    asm("mul.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
    return d;
}
__device__ __forceinline__ float add_rn(float a, float b) {
    float d;
    asm("add.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
    return d;
}
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return f2{fma_rn(a.x, b.x, c.x), fma_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{mul_rn(a.x, b.x), mul_rn(a.y, b.y)}; }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return f2{add_rn(a.x, b.x), add_rn(a.y, b.y)}; }
__device__ __forceinline__ f2 dup2(float v) { return f2{v, v}; }

// number of strips (warps) a tile is split into, from the length of the list it has to traverse
__device__ __forceinline__ int strips_for(int len, int t1) { return len <= t1 ? 1 : (len <= 2 * t1 ? 2 : (len <= 4 * t1 ? 4 : 8)); }

// ---- heavy-first scheduling ------------------------------------------------------------------
// Per-tile lists range from empty to thousands of entries (behind dense actors) and a blend kernel ends
// when its slowest warp does: with CTAs in raster order many SMs idle through the kernel's tail.  One block per list kind (0 main, 1 object, 2
// background: the slot numbering of final_T / tile_depth) counting-sorts the (tile, strip) work items
// into 64 half-octave length buckets, longest first, with no empty items; CTA b takes item b and the
// CTAs past the item count exit.  The order inside a bucket is arbitrary: it changes scheduling, never results.
// Layout per kind: [0] item count, [1 + i] = tile << 3 | strip.
#define SCHED_STRIDE(tiles) ((size_t)(tiles) * 8 + 1)
extern "C" size_t sgn_blend_sched_ints(int tiles) { return 3 * SCHED_STRIDE(tiles > 0 ? tiles : 0); }

__global__ void __launch_bounds__(1024)
sched_kernel(int tiles, const int2* __restrict__ tile_bins, const int2* __restrict__ cls_bins0,
             const int32_t* __restrict__ tile_depth /* backward: lengths come from here */, int fuse_obj, int split_main,
             int split_acc, int32_t* __restrict__ sched) {
    const int kind = blockIdx.x ? SLOT_BG : SLOT_MAIN;  // the objects-only pass is part of the main one
    const int2* bins = kind == SLOT_MAIN ? tile_bins : cls_bins0;
    const int split = kind == SLOT_MAIN ? split_main : split_acc;
    int32_t* out = sched + kind * SCHED_STRIDE(tiles);
    // per-warp histograms / cursors: the tiles of a frame fall into a handful of length buckets, and 9600 shared-memory
    // atomics on ~10 addresses serialise (15 us); privatised per warp they contend 32-way at most
    __shared__ int hist[32][64];
    __shared__ int start[64];
    const int warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) (&hist[0][0])[i] = 0;
    __syncthreads();
    // every forward pass and the main backward write per-pixel results for tiles with empty lists too (background
    // colour, zero accumulation, v_sky); only the accumulation backward has nothing to do there
    const bool visit_empty = !tile_depth || kind == SLOT_MAIN;
    auto length = [&](int t) {
        if (tile_depth) {  // backward: with fuse_obj the main traversal also walks the objects-only streams' residual
            const int d = tile_depth[(size_t)kind * tiles + t];
            return kind == SLOT_MAIN && fuse_obj ? d + tile_depth[(size_t)SLOT_OBJ * tiles + t] : d;
        }
        const int2 r = bins[t];
        return r.y - r.x;
    };
    auto bucket = [](int len) {
        if (len <= 0) return 63;
        const int lg = 31 - __clz(len);                          // floor(log2 len), len >= 1
        const int half = lg > 0 ? ((len >> (lg - 1)) & 1) : 0;  // upper half of the octave?
        return 62 - min(2 * lg + half, 62);                     // longest lists -> bucket 0
    };
    for (int t = threadIdx.x; t < tiles; t += blockDim.x) {
        const int len = length(t);
        if (len > 0 || visit_empty) atomicAdd(&hist[warp][bucket(len)], len > 0 ? strips_for(len, split) : 1);
    }
    __syncthreads();
    if (threadIdx.x < 64) {  // bucket b: exclusive offsets of the warps inside the bucket, bucket total in start[b]
        int acc = 0;
        for (int w = 0; w < 32; ++w) { const int c = hist[w][threadIdx.x]; hist[w][threadIdx.x] = acc; acc += c; }
        start[threadIdx.x] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < 64; ++b) { const int c = start[b]; start[b] = acc; acc += c; }
        out[0] = acc;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < tiles; t += blockDim.x) {
        const int len = length(t);
        if (!(len > 0 || visit_empty)) continue;
        const int W = len > 0 ? strips_for(len, split) : 1;
        const int bk = bucket(len);
        const int pos = start[bk] + atomicAdd(&hist[warp][bk], W);
        for (int s = 0; s < W; ++s) out[1 + pos + s] = (t << 3) | s;
    }
}

// CTA -> (tile, strip); false when there is nothing to do.  Without a schedule: strip-major raster order over
// the tiles x 8 grid.  (A persistent form -- CTAs looping over the list -- was measured slower: the loop makes
// ptxas hoist every parameter-derived value out of it, +35 registers.)
__device__ __forceinline__ bool take_work(const int32_t* __restrict__ sched, int kind, int tiles, int& tile, int& strip) {
    if (!sched) {
        tile = blockIdx.x % tiles; strip = blockIdx.x / tiles;
        return true;
    }
    const int32_t* w = sched + kind * SCHED_STRIDE(tiles);
    if ((int)blockIdx.x >= w[0]) return false;
    const int item = w[1 + blockIdx.x];
    tile = item >> 3; strip = item & 7;
    return true;
}

// Accumulation-only traversal of the class sub-list positions [range.x, range.y) (objects-only / background-only render).
// Carries each pixel's transmittance T and last-entry index idx (a sub-list position); yoff = 2s for a pixel whose stream is
// still live, DEAD for one that has terminated or is not rendered.
template <int PPL, bool SKIP>
__device__ __forceinline__ void acc_fwd_traverse(const BlendFwdParams& p, const int32_t* __restrict__ ids, int tile, int strip,
                                                 const int2 range, float (&T)[PPL], int (&idx)[PPL], float (&yoff)[PPL],
                                                 float4 (*sA)[32], float4 (*sB)[32]) {
    const float yc0 = (float)((tile / p.tiles_x) * SGN_TILE + strip * (2 * PPL)) + 1.0f;
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    const float px = (float)j + 0.5f, py0 = (float)i0 + 0.5f;
    constexpr float DEAD = 1e18f;  // row offset of a terminated / skipped pixel (see blend_fwd_strip)
    const float clampf = in_register(p.clamp_fwd), nclampf = in_register(-p.clamp_fwd);
    Staged nxt;
    if (range.x + lane < range.y) nxt = gather_entry(p.records, ids[range.x + lane]);
    int buf = 0;
    bool finished = false;
    for (int base = range.x; base < range.y && !finished; base += 32) {
        sA[buf][lane] = nxt.A; sB[buf][lane] = make_float4(nxt.B.x, nxt.B.y, row_reach(nxt) + 0.5f, 0.f);
        __syncwarp();
        if (base + 32 + lane < range.y) nxt = gather_entry(p.records, ids[base + 32 + lane]);
        const int n = min(32, range.y - base);
        // strips of long lists (PPL <= 2) are the kernel's critical path, and one entry is a ~70-cycle dependency
        // chain: unrolled, consecutive entries (independent but for the one-FMA T chain) overlap
#pragma unroll(PPL <= 2 ? 4 : 1)
        for (int t = 0; t < n; ++t) {
            if ((t & 7) == 0) {
                float ymin = DEAD;
#pragma unroll
                for (int s = 0; s < PPL; ++s) ymin = fminf(ymin, yoff[s]);
                if (__all_sync(FULL, ymin >= 0.5f * DEAD)) { finished = true; break; }
            }
            const float4 A = sA[buf][t];
            const float4 B = sB[buf][t];
            const float dx = A.x - px;
            const float bdx = A.w * dx, ax2 = A.z * dx * dx;
            const float dy0 = A.y - py0;
            const float dyc = A.y - yc0;  // distance to the centre line of slot 0's row pair (warp-uniform)
            const float span = LOG2_255 + B.y;
            const unsigned lim1 = (unsigned)(max(__float_as_int(span), -1) + 1);  // 0 when span < 0 (negative floats are negative ints)
            const int k = base + t;
            if constexpr (PPL >= 2) {
                // row-slot pairs (2q, 2q+1) updated together (f2), as in the main kernels
#pragma unroll
                for (int q = 0; q < PPL / 2; ++q) {
                    if (SKIP && fabsf(dyc - (float)(4 * q + 1)) > B.z + 1.f) continue;  // the entry reaches neither row pair
                    const f2 dy = f2{dy0 - yoff[2 * q], dy0 - yoff[2 * q + 1]};
                    const f2 sg = fma2(dy, fma2(dup2(B.x), dy, dup2(bdx)), dup2(ax2));
                    const bool v0 = __float_as_uint(sg.x) < lim1, v1 = __float_as_uint(sg.y) < lim1;
                    const f2 nam = f2{v0 ? fmaxf(nclampf, -fast_ex2(B.y - sg.x)) : 0.f, v1 ? fmaxf(nclampf, -fast_ex2(B.y - sg.y)) : 0.f};
                    const f2 Tq = f2{T[2 * q], T[2 * q + 1]};
                    const f2 nT = fma2(nam, Tq, Tq);
                    const bool st0 = nT.x <= T_STOP, st1 = nT.y <= T_STOP;
                    T[2 * q] = st0 ? Tq.x : nT.x; T[2 * q + 1] = st1 ? Tq.y : nT.y;
                    yoff[2 * q] = st0 ? DEAD : yoff[2 * q]; yoff[2 * q + 1] = st1 ? DEAD : yoff[2 * q + 1];
                    idx[2 * q] = (v0 && !st0) ? k : idx[2 * q];
                    idx[2 * q + 1] = (v1 && !st1) ? k : idx[2 * q + 1];
                }
            } else {
#pragma unroll
            for (int s = 0; s < PPL; ++s) {
                if (SKIP && fabsf(dyc - (float)(2 * s)) > B.z) continue;  // the entry cannot reach this row pair
                const float dy = dy0 - yoff[s];
                const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                const bool valid = __float_as_uint(sg) < lim1;
                const float am = valid ? fminf(clampf, fast_ex2(B.y - sg)) : 0.f;
                const float nT = __fmaf_rn(-am, T[s], T[s]);
                const bool stop = nT <= T_STOP;
                T[s] = stop ? T[s] : nT;
                yoff[s] = stop ? DEAD : yoff[s];
                idx[s] = (valid && !stop) ? k : idx[s];
            }
            }
        }
        buf ^= 1;
    }
}

// The main pass.  CLS: the per-tile list carries object entries (payload bit 31), and the strip also renders the
// objects-only accumulation: a second transmittance To per pixel, advanced with the SAME alpha by the object entries
// only (a warp-uniform branch), with its last-entry index recorded as a position in the object sub-list -- the object
// entries of the list in list order.  When every pixel's main stream has terminated, the objects-only streams that are
// still live continue on the object sub-list from the first object entry not yet passed (acc_fwd_traverse).
template <int PPL, bool CLS, bool SKIP, bool PACK, bool TMA = false>
__device__ __forceinline__ void blend_fwd_strip(const BlendFwdParams& p, int tile, int strip, const int2 range,
                                                float4 (*sA)[32], float4 (*sB)[32], float4 (*sC)[32],
                                                float4 (*sE)[96] = nullptr, uint64_t* mbar = nullptr) {
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    const float px = (float)j + 0.5f, py0 = (float)i0 + 0.5f;
    // The slot loop is bound by the half-rate ALU pipe (compares, selects, min/max, bit logic), not by FMA:
    // its bookkeeping is therefore arithmetic wherever possible.
    //   * liveness lives in the sign of the stream's transmittance: a stream that has terminated (or a pixel outside
    //     the image) holds -|T|, for which the next T is never above T_STOP, so nothing more is blended into it and
    //     there is no per-slot `done` test.  The alpha itself stays live for the other stream of the pixel;
    //   * validity (0 <= sigma*log2e <= log2(255 o)) is ONE unsigned compare of the float's bits;
    //   * an invalid slot is masked once (alpha = 0): T and the sums then pass through unchanged.
    float T[PPL], pr[PPL], pg[PPL], pb[PPL], pd[PPL], osum[PPL], To[PPL];
    int idx[PPL], idxo[PPL];
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        pr[s] = pg[s] = pb[s] = pd[s] = 0.f; osum[s] = 0.f;
        idx[s] = idxo[s] = -1;
        const bool inside = (j < p.width) && (i0 + 2 * s < p.height);
        T[s] = To[s] = inside ? 1.f : -1.f;
    }
    // object sub-list position of the next object entry of the list (warp-uniform)
    int orank = CLS ? p.cls_bins[1][tile].x : 0;

    Staged nxt;
    unsigned parity = 0;    // TMA: phase parity of the two mbarriers (bit b = buffer b)
    int pending_buf = -1;   // TMA: buffer with a bulk copy in flight that nobody has waited for yet
    if constexpr (TMA) {
        if (lane == 0) {
            mbar_init(&mbar[0], 1);
            mbar_init(&mbar[1], 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            if (range.x < range.y) {
                const uint32_t bytes = (uint32_t)min(32, range.y - range.x) * 48u;
                mbar_expect_tx(&mbar[0], bytes);
                bulk_g2s(sE[0], p.staged + 3 * (size_t)range.x, bytes, &mbar[0]);
            }
        }
        __syncwarp();
    } else {
        if (range.x + lane < range.y) nxt = gather_entry(p.records, p.sorted_ids[range.x + lane]);
    }
    int buf = 0;
    bool finished = false;
    const float yc0 = (float)((tile / p.tiles_x) * SGN_TILE + strip * (2 * PPL)) + 1.0f;
    unsigned slot_live = (1u << PPL) - 1u;  // warp-uniform: row pairs that still have a live stream (refreshed per batch)
    constexpr bool PK = PACK && PPL >= 2;
    constexpr int NP = PK ? PPL / 2 : 1;
    f2 T2[NP], pr2[NP], pg2[NP], pb2[NP], pd2[NP], osum2[NP], To2[NP];
#pragma unroll
    for (int q = 0; q < NP; ++q) {
        pr2[q] = pg2[q] = pb2[q] = pd2[q] = osum2[q] = dup2(0.f);
        if (PK) { T2[q] = f2{T[2 * q], T[2 * q + 1]}; To2[q] = f2{To[2 * q], To[2 * q + 1]}; }
    }
    const float clampf = in_register(p.clamp_fwd), nclamp = in_register(-p.clamp_fwd);
    for (int base = range.x; base < range.y && !finished; base += 32) {
        if constexpr (TMA) {
            __syncwarp();  // every lane has finished reading the other buffer (previous batch)
            pending_buf = -1;
            if (base + 32 < range.y) {
                if (lane == 0) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    const uint32_t bytes = (uint32_t)min(32, range.y - base - 32) * 48u;
                    mbar_expect_tx(&mbar[buf ^ 1], bytes);
                    bulk_g2s(sE[buf ^ 1], p.staged + 3 * (size_t)(base + 32), bytes, &mbar[buf ^ 1]);
                }
                pending_buf = buf ^ 1;
            }
            mbar_wait(&mbar[buf], (parity >> buf) & 1u);
            parity ^= 1u << buf;
        } else {
        sA[buf][lane] = nxt.A; sB[buf][lane] = nxt.B;
        sC[buf][lane] = make_float4(nxt.C.x, nxt.C.y, nxt.C.z, SKIP ? row_reach(nxt) + 0.5f : 0.f);
        __syncwarp();
        if (base + 32 + lane < range.y) nxt = gather_entry(p.records, p.sorted_ids[base + 32 + lane]);
        }
        if (SKIP) {
            slot_live = 0;
#pragma unroll
            for (int s = 0; s < PPL; ++s) {
                const float Ts = PK ? ((s & 1) ? T2[s / 2].y : T2[s / 2].x) : T[s];
                const float Tos = PK ? ((s & 1) ? To2[s / 2].y : To2[s / 2].x) : To[s];
                slot_live |= __any_sync(FULL, (CLS ? fmaxf(Ts, Tos) : Ts) > 0.f) ? (1u << s) : 0u;
            }
        }
        const int n = min(32, range.y - base);
        // strips of long lists (PPL <= 2) are the kernel's critical path, and one entry is a ~70-cycle dependency
        // chain: unrolled, consecutive entries (independent but for the one-FMA T chain) overlap
#pragma unroll(PPL <= 2 ? 4 : 1)
        for (int t = 0; t < n; ++t) {
            if ((t & 7) == 0) {  // every pixel's main stream terminated: stop traversing (checked every 8 entries)
                float tmax = -1.f;
#pragma unroll
                for (int s = 0; s < PPL; ++s) tmax = fmaxf(tmax, PK ? ((s & 1) ? T2[s / 2].y : T2[s / 2].x) : T[s]);
                if (__all_sync(FULL, tmax < 0.f)) { finished = true; break; }
            }
            const float4 A = TMA ? sE[buf][3 * t] : sA[buf][t];
            const float4 B = TMA ? sE[buf][3 * t + 1] : sB[buf][t];
            const float4 Cc = TMA ? sE[buf][3 * t + 2] : sC[buf][t];
            const float dyc = A.y - yc0;
            const float dx = A.x - px;
            const float bdx = A.w * dx, ax2 = A.z * dx * dx;
            const float dy0 = A.y - py0;
            // valid  <=>  0 <= sg <= log2(255 o)  <=>  bits(sg) < lim1   (sg = sigma*log2e; negative and NaN have huge bits)
            const float span = LOG2_255 + B.y;
            const unsigned lim1 = (unsigned)(max(__float_as_int(span), -1) + 1);  // 0 when span < 0 (negative floats are negative ints)
            const int k = base + t;
            // OBJ (warp-uniform): an object entry, which the objects-only stream takes as well
            auto blend_entry = [&](auto obj_tag) {
                constexpr bool OBJ = decltype(obj_tag)::value;
                if constexpr (PK) {
                    // paired row slots (f2); weights and the blended channels are kept negated (nw = -alpha*T)
#pragma unroll
                    for (int q = 0; q < NP; ++q) {
                        if (SKIP) {
                            if (!((slot_live >> (2 * q)) & 3u) || fabsf(dyc - (float)(4 * q + 1)) > Cc.w + 1.f) continue;
                        }
                        const f2 dy = f2{dy0 - (float)(4 * q), dy0 - (float)(4 * q + 2)};
                        const f2 sg = fma2(dy, fma2(dup2(B.x), dy, dup2(bdx)), dup2(ax2));
                        const bool v0 = __float_as_uint(sg.x) < lim1, v1 = __float_as_uint(sg.y) < lim1;
                        const f2 nam = f2{v0 ? fmaxf(nclamp, -fast_ex2(B.y - sg.x)) : 0.f, v1 ? fmaxf(nclamp, -fast_ex2(B.y - sg.y)) : 0.f};
                        const f2 nT = fma2(nam, T2[q], T2[q]);
                        const bool st0 = nT.x <= T_STOP, st1 = nT.y <= T_STOP;
                        const f2 nau = f2{st0 ? 0.f : nam.x, st1 ? 0.f : nam.y};
                        const f2 nw = mul2(nau, T2[q]);
                        if (OBJ) {  // an object entry took part in the main stream (the background pass needs this pixel)
                            osum2[q].x = T2[q].x > 0.f ? osum2[q].x + nam.x : osum2[q].x;
                            osum2[q].y = T2[q].y > 0.f ? osum2[q].y + nam.y : osum2[q].y;
                        }
                        T2[q].x = st0 ? -fabsf(T2[q].x) : nT.x; T2[q].y = st1 ? -fabsf(T2[q].y) : nT.y;
                        idx[2 * q] = (nau.x < 0.f) ? k : idx[2 * q];
                        idx[2 * q + 1] = (nau.y < 0.f) ? k : idx[2 * q + 1];
                        pr2[q] = fma2(dup2(B.z), nw, pr2[q]); pg2[q] = fma2(dup2(B.w), nw, pg2[q]);
                        pb2[q] = fma2(dup2(Cc.x), nw, pb2[q]); pd2[q] = fma2(dup2(Cc.y), nw, pd2[q]);
                        if (OBJ) {
                            const f2 nTo = fma2(nam, To2[q], To2[q]);
                            const bool so0 = nTo.x <= T_STOP, so1 = nTo.y <= T_STOP;
                            idxo[2 * q] = (v0 && !so0) ? orank : idxo[2 * q];
                            idxo[2 * q + 1] = (v1 && !so1) ? orank : idxo[2 * q + 1];
                            To2[q].x = so0 ? -fabsf(To2[q].x) : nTo.x; To2[q].y = so1 ? -fabsf(To2[q].y) : nTo.y;
                        }
                    }
                } else {
                    // straight-line, predicated: the PPL pixel chains are independent and interleave (ILP)
#pragma unroll
                    for (int s = 0; s < PPL; ++s) {
                        if (SKIP) {  // warp-uniform: the entry cannot reach this row pair, or all its pixels terminated
                            if (!((slot_live >> s) & 1u) || fabsf(dyc - (float)(2 * s)) > Cc.w) continue;
                        }
                        const float dy = dy0 - (float)(2 * s);
                        const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                        const bool valid = __float_as_uint(sg) < lim1;
                        const float am = valid ? fminf(clampf, fast_ex2(B.y - sg)) : 0.f;
                        const float nT = __fmaf_rn(-am, T[s], T[s]);
                        const bool stop = nT <= T_STOP;
                        const float au = stop ? 0.f : am;
                        const float w = au * T[s];
                        if (OBJ) osum[s] = T[s] > 0.f ? osum[s] + am : osum[s];
                        T[s] = stop ? -fabsf(T[s]) : nT;
                        idx[s] = (au > 0.f) ? k : idx[s];
                        pr[s] = __fmaf_rn(B.z, w, pr[s]); pg[s] = __fmaf_rn(B.w, w, pg[s]);
                        pb[s] = __fmaf_rn(Cc.x, w, pb[s]); pd[s] = __fmaf_rn(Cc.y, w, pd[s]);
                        if (OBJ) {
                            const float nTo = __fmaf_rn(-am, To[s], To[s]);
                            const bool so = nTo <= T_STOP;
                            idxo[s] = (valid && !so) ? orank : idxo[s];
                            To[s] = so ? -fabsf(To[s]) : nTo;
                        }
                    }
                }
                if (OBJ) ++orank;
            };
            if (CLS && __float_as_int(Cc.z) < 0) blend_entry(std::true_type{});
            else blend_entry(std::false_type{});
        }
        buf ^= 1;
    }
    if constexpr (TMA) {  // a copy issued for a batch the traversal never reached must land before the CTA may exit
        if (pending_buf >= 0) mbar_wait(&mbar[pending_buf], (parity >> pending_buf) & 1u);
    }
    if constexpr (PK) {
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            T[2 * q] = T2[q].x; T[2 * q + 1] = T2[q].y;
            To[2 * q] = To2[q].x; To[2 * q + 1] = To2[q].y;
            pr[2 * q] = -pr2[q].x; pr[2 * q + 1] = -pr2[q].y; pg[2 * q] = -pg2[q].x; pg[2 * q + 1] = -pg2[q].y;
            pb[2 * q] = -pb2[q].x; pb[2 * q + 1] = -pb2[q].y; pd[2 * q] = -pd2[q].x; pd[2 * q + 1] = -pd2[q].y;
            osum[2 * q] = -osum2[q].x; osum[2 * q + 1] = -osum2[q].y;
        }
    }
    const size_t P = (size_t)p.width * p.height;
    {   // how deep this tile was traversed: the backward sizes its strips from it
        int kdeep = -1;
#pragma unroll
        for (int s = 0; s < PPL; ++s) kdeep = max(kdeep, idx[s]);
        kdeep = warp_max(kdeep);
        if (lane == 0 && kdeep >= 0) atomicMax(p.tile_depth + tile, kdeep + 1 - range.x);
    }
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        const int i = i0 + 2 * s;
        if (j >= p.width || i >= p.height) continue;
        T[s] = fabsf(T[s]);
        const size_t pid = (size_t)i * p.width + j;
        const float alpha = 1.f - T[s];
        p.raw[pid] = make_float4(pr[s], pg[s], pb[s], pd[s]);
        if (p.raw_mode) {  // gsplat rasterize_gaussians: out = blended + T_final * background
            p.rgb[3 * pid] = pr[s] + T[s] * p.bg[0]; p.rgb[3 * pid + 1] = pg[s] + T[s] * p.bg[1];
            p.rgb[3 * pid + 2] = pb[s] + T[s] * p.bg[2];
            p.depth[pid] = pd[s] + T[s] * p.bg[3];
            p.acc[pid] = alpha;
            p.final_T[SLOT_MAIN * P + pid] = T[s];
            p.final_idx[SLOT_MAIN * P + pid] = idx[s];
            continue;
        }
        // post-ops (sgn_splatfacto.py:968-975): clamp(max=1), sky blend (premultiplied rgb times alpha again), eval clamp
        float r = fminf(pr[s], 1.f), g = fminf(pg[s], 1.f), bl = fminf(pb[s], 1.f);
        if (p.has_sky) {
            const float* sk = p.sky + 3 * pid;
            r = r * alpha + sk[0] * (1.f - alpha);
            g = g * alpha + sk[1] * (1.f - alpha);
            bl = bl * alpha + sk[2] * (1.f - alpha);
        }
        if (p.eval_clamp) {
            r = fminf(fmaxf(r, 0.f), 1.f); g = fminf(fmaxf(g, 0.f), 1.f); bl = fminf(fmaxf(bl, 0.f), 1.f);
        }
        p.rgb[3 * pid] = r; p.rgb[3 * pid + 1] = g; p.rgb[3 * pid + 2] = bl;
        p.acc[pid] = alpha;
        p.depth[pid] = alpha > 1e-3f ? pd[s] / alpha : 10.f;  // sgn_splatfacto.py:995
        p.final_T[SLOT_MAIN * P + pid] = T[s];
        p.final_idx[SLOT_MAIN * P + pid] = idx[s];
        if (CLS) {
            const bool hit = osum[s] > 0.f;
            p.final_idx[SLOT_BG * P + pid] = hit ? BG_TODO : BG_SAME_AS_MAIN;
            if (!hit) { p.final_T[SLOT_BG * P + pid] = T[s]; p.bg_acc[pid] = alpha; }
        }
    }
    if constexpr (CLS) {
        // objects-only streams still live: the rest of the object sub-list, from the first object entry not yet passed
        constexpr float DEAD = 1e18f;
        float yo[PPL];
        bool live = false;
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            live = live || To[s] > 0.f;
            yo[s] = To[s] > 0.f ? (float)(2 * s) : DEAD;
            To[s] = fabsf(To[s]);
        }
        const int2 orange = p.cls_bins[1][tile];
        if (__any_sync(FULL, live) && orank < orange.y) {
            if constexpr (TMA) {  // the bulk-copy ring is idle now (every copy has landed): stage through it
                acc_fwd_traverse<PPL, true>(p, p.cls_ids[1], tile, strip, make_int2(orank, orange.y), To, idxo, yo,
                                            reinterpret_cast<float4(*)[32]>(&sE[0][0]), reinterpret_cast<float4(*)[32]>(&sE[0][64]));
            } else {
                acc_fwd_traverse<PPL, true>(p, p.cls_ids[1], tile, strip, make_int2(orank, orange.y), To, idxo, yo, sA, sB);
            }
            // tile_depth[object]: how far this tile's object streams ran past the main traversal (sizes the backward)
            int kdeep = -1;
#pragma unroll
            for (int s = 0; s < PPL; ++s) kdeep = max(kdeep, idxo[s]);
            kdeep = warp_max(kdeep);
            if (lane == 0 && kdeep >= orank) atomicMax(p.tile_depth + (size_t)SLOT_OBJ * p.tiles + tile, kdeep + 1 - orank);
        }
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            const int i = i0 + 2 * s;
            if (j >= p.width || i >= p.height) continue;
            const size_t pid = (size_t)i * p.width + j;
            p.final_T[SLOT_OBJ * P + pid] = To[s];
            p.final_idx[SLOT_OBJ * P + pid] = idxo[s];
            p.obj_acc[pid] = 1.f - To[s];
        }
    }
}

// accumulation-only pass over one class's per-tile sub-lists (the background-only render; the objects-only one is part of
// the main pass)
template <int PPL, bool SKIP>
__device__ __forceinline__ void acc_fwd_strip(const BlendFwdParams& p, int cls, int tile, int strip, const int2 range,
                                              float4 (*sA)[32], float4 (*sB)[32]) {
    const int32_t* __restrict__ ids = p.cls_ids[cls];
    const int slot = cls ? SLOT_OBJ : SLOT_BG;
    float* __restrict__ out_acc = cls ? p.obj_acc : p.bg_acc;
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    constexpr unsigned ALL = (1u << PPL) - 1u;
    constexpr float DEAD = 1e18f;  // row offset of a terminated / skipped pixel
    float T[PPL], yoff[PPL];
    int idx[PPL];
    unsigned skip = 0;
    const size_t P = (size_t)p.width * p.height;
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        T[s] = 1.f; idx[s] = -1; yoff[s] = (float)(2 * s);
        const int i = i0 + 2 * s;
        if (!((j < p.width) && (i < p.height))) { yoff[s] = DEAD; skip |= 1u << s; }
        else if (cls == 0 && p.final_idx[SLOT_BG * P + (size_t)i * p.width + j] != BG_TODO) {
            yoff[s] = DEAD; skip |= 1u << s;  // the main forward already wrote this pixel's background result
        }
    }
    if (__all_sync(FULL, skip == ALL)) return;
    acc_fwd_traverse<PPL, SKIP>(p, ids, tile, strip, range, T, idx, yoff, sA, sB);
    {
        int kdeep = -1;
#pragma unroll
        for (int s = 0; s < PPL; ++s) kdeep = max(kdeep, idx[s]);
        kdeep = warp_max(kdeep);
        if (lane == 0 && kdeep >= 0) atomicMax(p.tile_depth + (size_t)slot * p.tiles + tile, kdeep + 1 - range.x);
    }
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        const int i = i0 + 2 * s;
        if ((skip >> s) & 1u) continue;
        const size_t pid = (size_t)i * p.width + j;
        p.final_T[slot * P + pid] = T[s];
        p.final_idx[slot * P + pid] = idx[s];
        out_acc[pid] = 1.f - T[s];
    }
}

template <bool CLS, bool SKIP, bool PACK>
__global__ void __launch_bounds__(32, BLEND_FWD_MIN_BLOCKS) blend_fwd_kernel(const BlendFwdParams p) {
    __shared__ float4 sA[2][32];
    __shared__ float4 sB[2][32];
    __shared__ float4 sC[2][32];
    int tile, strip;
    if (!take_work(p.sched, SLOT_MAIN, p.tiles, tile, strip)) return;
    const int2 range = p.tile_bins[tile];
    const int W = strips_for(range.y - range.x, p.split_main);
    if (strip >= W) return;
    switch (W) {
        case 1: blend_fwd_strip<8, CLS, SKIP, PACK>(p, tile, strip, range, sA, sB, sC); break;
        case 2: blend_fwd_strip<4, CLS, SKIP, PACK>(p, tile, strip, range, sA, sB, sC); break;
        case 4: blend_fwd_strip<2, CLS, SKIP, PACK>(p, tile, strip, range, sA, sB, sC); break;
        default: blend_fwd_strip<1, CLS, SKIP, PACK>(p, tile, strip, range, sA, sB, sC); break;
    }
}

template <bool CLS>
__global__ void __launch_bounds__(32) blend_fwd_tma_kernel(const BlendFwdParams p) {
    __shared__ __align__(128) float4 sE[2][96];
    __shared__ __align__(8) uint64_t mbar[2];
    int tile, strip;
    if (!take_work(p.sched, SLOT_MAIN, p.tiles, tile, strip)) return;
    const int2 range = p.tile_bins[tile];
    const int W = strips_for(range.y - range.x, p.split_main);
    if (strip >= W) return;
    switch (W) {
        case 1: blend_fwd_strip<8, CLS, false, true, true>(p, tile, strip, range, nullptr, nullptr, nullptr, sE, mbar); break;
        case 2: blend_fwd_strip<4, CLS, false, true, true>(p, tile, strip, range, nullptr, nullptr, nullptr, sE, mbar); break;
        case 4: blend_fwd_strip<2, CLS, false, true, true>(p, tile, strip, range, nullptr, nullptr, nullptr, sE, mbar); break;
        default: blend_fwd_strip<1, CLS, false, true, true>(p, tile, strip, range, nullptr, nullptr, nullptr, sE, mbar); break;
    }
}

// materialises the per-tile lists as staged entries (the TMA experiment's input): entry k of the sorted list -> 48 bytes
__global__ void __launch_bounds__(256)
stage_entries_kernel(long long M, const float4* __restrict__ records, const int32_t* __restrict__ sorted_ids, float4* __restrict__ staged) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= M) return;
    const Staged s = gather_entry(records, sorted_ids[k]);
    staged[3 * k] = s.A; staged[3 * k + 1] = s.B; staged[3 * k + 2] = s.C;
}

template <bool SKIP>
__global__ void __launch_bounds__(32, BLEND_ACC_MIN_BLOCKS) acc_fwd_kernel(const BlendFwdParams p, const int cls) {
    __shared__ float4 sA[2][32];
    __shared__ float4 sB[2][32];
    int tile, strip;
    if (!take_work(p.sched, cls ? SLOT_OBJ : SLOT_BG, p.tiles, tile, strip)) return;
    const int2 range = p.cls_bins[cls][tile];
    const int W = strips_for(range.y - range.x, p.split_acc);
    if (strip >= W) return;
    switch (W) {
        case 1: acc_fwd_strip<8, SKIP>(p, cls, tile, strip, range, sA, sB); break;
        case 2: acc_fwd_strip<4, SKIP>(p, cls, tile, strip, range, sA, sB); break;
        case 4: acc_fwd_strip<2, SKIP>(p, cls, tile, strip, range, sA, sB); break;
        default: acc_fwd_strip<1, SKIP>(p, cls, tile, strip, range, sA, sB); break;
    }
}

// The background-only backward is independent of the main backward (both only RED into v_records), and every
// blend kernel ends in a tail during which most SMs idle.  It is therefore forked onto an auxiliary stream and
// joined back with events: same results, the tails overlap.
#include <mutex>
static cudaStream_t aux_stream() {
    static std::mutex mu;
    static cudaStream_t streams[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    if (!streams[dev]) {
        if (cudaStreamCreateWithFlags(&streams[dev], cudaStreamNonBlocking) != cudaSuccess) streams[dev] = nullptr;
    }
    return streams[dev];
}
// fork / join events are created once per device (event creation + destruction cost ~4 us per blend call on a 2 ms step)
struct ForkJoinEvents {
    cudaEvent_t fork = nullptr, join = nullptr;
};
static ForkJoinEvents* fork_join_events() {
    static thread_local ForkJoinEvents events[64];  // per host thread: a viewer thread rendering next to the trainer has its own pair
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    ForkJoinEvents& e = events[dev];
    if (!e.fork && cudaEventCreateWithFlags(&e.fork, cudaEventDisableTiming) != cudaSuccess) { e.fork = nullptr; return nullptr; }
    if (!e.join && cudaEventCreateWithFlags(&e.join, cudaEventDisableTiming) != cudaSuccess) { e.join = nullptr; return nullptr; }
    return &e;
}
// (re-recording an event that an earlier wait still references is fine: cudaStreamWaitEvent captures the event's state at
// the time of the call)
struct ForkJoin {
    cudaStream_t main, aux;
    ForkJoinEvents* ev = nullptr;
    bool ok = false;
    ForkJoin(cudaStream_t m) : main(m), aux(aux_stream()) {
        if (!aux) return;
        ev = fork_join_events();
        if (!ev) return;
        ok = cudaEventRecord(ev->fork, main) == cudaSuccess && cudaStreamWaitEvent(aux, ev->fork, 0) == cudaSuccess;
    }
    cudaStream_t side() const { return ok ? aux : main; }
    void finish() {
        if (ok) { cudaEventRecord(ev->join, aux); cudaStreamWaitEvent(main, ev->join, 0); }
    }
};

static int check_cam(const sgn_camera* cam) {
    SGN_REQUIRE(cam, "null camera");
    SGN_REQUIRE(cam->block_width == SGN_TILE, "the fused blend kernels require block_width == 16 (got %d)", cam->block_width);
    SGN_REQUIRE(cam->width > 0 && cam->height > 0, "empty image");
    return SGN_OK;
}

template <bool CLS>
static void launch_blend_fwd(const BlendFwdParams& p, int tuning, cudaStream_t stream) {
    const dim3 grid(p.tiles * 8), block(32);
    if ((tuning & SGN_TUNE_FWD_TMA) && p.staged) {
        blend_fwd_tma_kernel<CLS><<<grid, block, 0, stream>>>(p);
        return;
    }
    switch (((tuning & SGN_TUNE_FWD_ROW_SKIP) ? 2 : 0) | ((tuning & SGN_TUNE_FWD_PACKED) ? 1 : 0)) {
        case 0: blend_fwd_kernel<CLS, false, false><<<grid, block, 0, stream>>>(p); break;
        case 1: blend_fwd_kernel<CLS, false, true><<<grid, block, 0, stream>>>(p); break;
        case 2: blend_fwd_kernel<CLS, true, false><<<grid, block, 0, stream>>>(p); break;
        default: blend_fwd_kernel<CLS, true, true><<<grid, block, 0, stream>>>(p); break;
    }
}

extern "C" int sgn_blend_fwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records,
                             const int32_t* sorted_ids, const int32_t* tile_bins, int64_t M, const int32_t* cls_ids,
                             const int32_t* cls_bins, const float* sky, const sgn_blend_fwd_out* out, void* stream) {
    SGN_RANGE("sgn_blend_fwd");
    if (int rc = check_cam(cam)) return rc;
    SGN_REQUIRE(opts && records && tile_bins && out, "sgn_blend_fwd: null pointer");
    SGN_REQUIRE(out->rgb && out->accumulation && out->depth && out->raw && out->final_T && out->final_idx,
                "sgn_blend_fwd: null output");
    SGN_REQUIRE(!opts->class_streams || (out->object_acc && out->background_acc && cls_ids && cls_bins),
                "class_streams needs object_acc/background_acc outputs and the class sub-lists");
    SGN_REQUIRE(!opts->has_sky || sky, "has_sky set but sky is null");
    SGN_REQUIRE(sgn_aligned16(records) && sgn_aligned16(out->raw), "records / raw must be 16-byte aligned");
    BlendFwdParams p;
    p.width = cam->width; p.height = cam->height;
    p.tiles_x = (cam->width + SGN_TILE - 1) / SGN_TILE;
    const int tiles_y = (cam->height + SGN_TILE - 1) / SGN_TILE;
    p.clamp_fwd = opts->alpha_clamp_fwd;
    p.split_main = opts->split_fwd_main > 0 ? opts->split_fwd_main : 768;
    p.split_acc = opts->split_fwd_acc > 0 ? opts->split_fwd_acc : 512;
    p.has_sky = opts->has_sky; p.eval_clamp = opts->eval_clamp; p.raw_mode = opts->raw_mode;
    for (int c = 0; c < 4; ++c) p.bg[c] = opts->background[c];
    p.records = reinterpret_cast<const float4*>(records);
    p.staged = nullptr;
    p.sorted_ids = sorted_ids;
    p.tile_bins = reinterpret_cast<const int2*>(tile_bins);
    const int tiles = p.tiles_x * tiles_y;
    p.tiles = tiles;
    if ((opts->tuning & SGN_TUNE_FWD_TMA) && out->staged && sorted_ids && M > 0) {
        SGN_REQUIRE(sgn_aligned16(out->staged), "staged entries must be 16-byte aligned");
        stage_entries_kernel<<<(unsigned)((M + 255) / 256), 256, 0, (cudaStream_t)stream>>>(M, p.records, sorted_ids, reinterpret_cast<float4*>(out->staged));
        SGN_CHECK_LAUNCH("stage_entries_kernel");
        p.staged = reinterpret_cast<const float4*>(out->staged);
    }
    p.cls_ids[0] = cls_ids; p.cls_ids[1] = cls_ids ? cls_ids + M : nullptr;
    p.cls_bins[0] = reinterpret_cast<const int2*>(cls_bins);
    p.cls_bins[1] = cls_bins ? reinterpret_cast<const int2*>(cls_bins) + tiles : nullptr;
    p.sky = sky;
    p.rgb = out->rgb; p.acc = out->accumulation; p.depth = out->depth;
    p.obj_acc = out->object_acc; p.bg_acc = out->background_acc;
    p.raw = reinterpret_cast<float4*>(out->raw);
    p.final_T = out->final_T; p.final_idx = out->final_idx;
    SGN_REQUIRE(out->tile_depth, "sgn_blend_fwd: tile_depth is null");
    p.tile_depth = out->tile_depth;
    SGN_CHECK_CUDA(cudaMemsetAsync(out->tile_depth, 0, sizeof(int32_t) * 3 * (size_t)tiles, (cudaStream_t)stream));
    p.sched = out->sched;
    if (out->sched) {
        sched_kernel<<<opts->class_streams ? 2 : 1, 1024, 0, (cudaStream_t)stream>>>(tiles, p.tile_bins, p.cls_bins[0], nullptr, 0,
                                                                                  p.split_main, p.split_acc, out->sched);
        SGN_CHECK_LAUNCH("sched_kernel");
    }
    if (opts->class_streams) {
        const bool acc_skip = !(opts->tuning & SGN_TUNE_ACC_NO_ROW_SKIP);
        const unsigned acc_grid = tiles * 8;
        launch_blend_fwd<true>(p, opts->tuning, (cudaStream_t)stream);  // main + objects-only
        SGN_CHECK_LAUNCH("blend_fwd_kernel");
        if (acc_skip) acc_fwd_kernel<true><<<acc_grid, 32, 0, (cudaStream_t)stream>>>(p, 0);  // background: needs the main pass's flags
        else acc_fwd_kernel<false><<<acc_grid, 32, 0, (cudaStream_t)stream>>>(p, 0);
        SGN_CHECK_LAUNCH("acc_fwd_kernel<background>");
    } else {
        launch_blend_fwd<false>(p, opts->tuning, (cudaStream_t)stream);
        SGN_CHECK_LAUNCH("blend_fwd_kernel");
    }
    return SGN_OK;
}

// ------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------
struct BlendBwdParams {
    int width, height, tiles_x, tiles;
    int split_main, split_acc;
    const int32_t* tile_depth;  // [3][tiles]
    const int32_t* sched;  // heavy-first work lists (sched_kernel) or null
    float clamp_bwd;
    int has_sky, eval_clamp, raw_mode;
    float bg[4];
    const float4* records;
    const int32_t* sorted_ids;
    const int2* tile_bins;
    const int32_t* cls_ids[2];
    const int2* cls_bins[2];
    const float* v_rgb;
    const float* v_acc;
    const float* v_depth;
    const float* v_obj;
    const float* v_bg;
    const float4* raw;
    const float* final_T;
    const int32_t* final_idx;
    const float* sky;
    float* v_sky;
    float* v_records;
    long long* v_fixed;        // deterministic mode: [N,12] fixed-point accumulators instead of float atomics (or null)
    const float* fixed_scale;  // device scalar: fixed-point units per unit of gradient
};

// Deterministic mode: how many binary places the fixed-point grid of record component idx (= row * 12 + component) gives
// up, from the Gaussian's own record.  A conic gradient is a sum of 1/2 dx^2 v_sigma (dx dy, 1/2 dy^2) over the pixels the
// Gaussian covers, which grows like o sigma^4 -- about pi/4 E^2 per unit of v_alpha with E = trace of the 2D covariance in
// px^2 (the support ellipse holds ~2 pi sigma^2 pixels).  At sigma = 200 px that is ~4e9, twice the 2^31 units of headroom
// of the grid; the conic components of a Gaussian with E > 2^13 (sigma above ~64 px) are therefore accumulated 2^-(2 ceil(log2
// E) - 26) coarser, which keeps their sums below ~2^26 units per unit of v_alpha.  Smaller Gaussians keep the full grid.
// Exact double operations on the record's floats: the same value wherever it is computed (accumulate_grad and
// fixed_to_float_kernel).
__device__ __forceinline__ int fixed_shift(const float* __restrict__ records, size_t idx) {
    const int comp = (int)(idx % SGN_RECORD_FLOATS);
    if (comp < 2 || comp > 4) return 0;
    const float* r = records + (idx - comp);
    const double a = __ldg(r + 2), b = __ldg(r + 3), c = __ldg(r + 4);
    const double det = __dsub_rn(__dmul_rn(a, c), __dmul_rn(b, b));
    if (!(det > 0.0)) return 0;  // not positive definite (or NaN): such an entry is valid for no pixel or a few
    const double E = __ddiv_rn(__dadd_rn(a, c), det);
    if (!(E > 0.0)) return 0;
    int e;
    frexp(fmin(E, 1e18), &e);  // E < 2^e
    return min(max(2 * e - 26, 0), 100);
}

// Per-Gaussian gradient accumulation.  Default: float RED (summation order varies from run to run).  Deterministic mode
// (sgn_blend_bwd_in.v_fixed): the addend is rounded ONCE to 64-bit fixed point and added as an integer -- integer addition
// is associative, so the total is bit-identical whatever order the tiles and strips arrive in.
// DET is a template parameter of the backward kernels: the float path's instantiations carry no fixed-point code (with the
// shift computation behind a run-time branch, blend_bwd took 0.85 instead of 0.75 ms at config 3).
template <bool DET>
__device__ __forceinline__ void accumulate_grad(const BlendBwdParams& p, float fscale, size_t idx, float v) {
    if constexpr (DET) {
        const int sh = fixed_shift(reinterpret_cast<const float*>(p.records), idx);
        const float m = v * fscale * __int_as_float((127 - sh) << 23);  // times 2^-sh: exact
        atomicAdd(reinterpret_cast<unsigned long long*>(p.v_fixed) + idx, (unsigned long long)__float2ll_rn(m));
    } else {
        atomicAdd(p.v_records + idx, v);
    }
}

// backward of the accumulation-only pass: out = 1 - T_final  =>  v_alpha_k = T_final * ra_k * v_out.  Walks the class
// sub-list positions [range.x, range.y) back to front; tfv = T_final * v_out and idx (a sub-list position) per pixel.
template <int PPL, bool SKIP, bool DET>
__device__ __forceinline__ void acc_bwd_traverse(const BlendBwdParams& p, const int32_t* __restrict__ ids, int tile, int strip,
                                                 const int2 range, const float (&tfv)[PPL], const int (&idx)[PPL],
                                                 float4 (*sA)[32], float4 (*sB)[32], float (*sR)[32]) {
    const float yc0 = (float)((tile / p.tiles_x) * SGN_TILE + strip * (2 * PPL)) + 1.0f;
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    const float px = (float)j + 0.5f, py0 = (float)i0 + 0.5f;
    const int my_comp = multi_reduce_slot<6>(lane);
    const float clampb = in_register(p.clamp_bwd), nclamp = -clampb;
    const float fscale = DET ? __ldg(p.fixed_scale) : 0.f;
    Staged nxt;
    if (range.y - 1 - lane >= range.x) nxt = gather_entry(p.records, ids[range.y - 1 - lane]);
    int buf = 0;
    for (int hi = range.y; hi > range.x; hi -= 32) {
        sA[buf][lane] = nxt.A; sB[buf][lane] = make_float4(nxt.B.x, nxt.B.y, nxt.C.z, nxt.C.w);
        sR[buf][lane] = row_reach(nxt) + 0.5f;
        __syncwarp();
        if (hi - 33 - lane >= range.x) nxt = gather_entry(p.records, ids[hi - 33 - lane]);
        const int n = min(32, hi - range.x);
        for (int t = 0; t < n; ++t) {
            const int k = hi - 1 - t;
            const float4 A = sA[buf][t];
            const float4 B = sB[buf][t];
            const float dx = A.x - px;
            const float bdx = A.w * dx, ax2 = A.z * dx * dx;
            const float dy0 = A.y - py0;
            const float dyc = A.y - yc0, reach = sR[buf][t];
            const unsigned lim1 = (unsigned)(max(__float_as_int(LOG2_255 + B.y), -1) + 1);
            const float o = B.w;
            float S0 = 0.f, Sy = 0.f, Syy = 0.f;
            if constexpr (PPL >= 2) {  // paired row slots (f2), as in blend_bwd_strip
                f2 S0p = dup2(0.f), Syp = dup2(0.f), Syyp = dup2(0.f);
                const f2 dyb = f2{dy0, dy0 - 2.f};
#pragma unroll
                for (int q = 0; q < PPL / 2; ++q) {
                    if (SKIP && fabsf(dyc - (float)(4 * q + 1)) > reach + 1.f) continue;
                    const f2 dy = add2(dyb, dup2(-(float)(4 * q)));
                    const f2 sg = fma2(dy, fma2(dup2(B.x), dy, dup2(bdx)), dup2(ax2));
                    const bool v0 = (__float_as_uint(sg.x) < lim1) && (k <= idx[2 * q]);
                    const bool v1 = (__float_as_uint(sg.y) < lim1) && (k <= idx[2 * q + 1]);
                    const f2 nraw = f2{v0 ? -fast_ex2(B.y - sg.x) : 0.f, v1 ? -fast_ex2(B.y - sg.y) : 0.f};
                    const f2 om = add2(f2{fmaxf(nclamp, nraw.x), fmaxf(nclamp, nraw.y)}, dup2(1.f));
                    const f2 ra = f2{fast_rcp(om.x), fast_rcp(om.y)};
                    const f2 vs = mul2(nraw, mul2(f2{tfv[2 * q], tfv[2 * q + 1]}, ra));
                    S0p = add2(S0p, vs);
                    const f2 vsy = mul2(vs, dy);
                    Syp = add2(Syp, vsy);
                    Syyp = fma2(vsy, dy, Syyp);
                }
                S0 = S0p.x + S0p.y; Sy = Syp.x + Syp.y; Syy = Syyp.x + Syyp.y;
            } else {
#pragma unroll
            for (int s = 0; s < PPL; ++s) {
                if (SKIP && fabsf(dyc - (float)(2 * s)) > reach) continue;
                const float dy = dy0 - (float)(2 * s);
                const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                const bool valid = (__float_as_uint(sg) < lim1) && (k <= idx[s]);
                const float raw = fast_ex2(B.y - sg);
                const float alpha = fminf(clampb, raw);
                const float ra = fast_rcp(1.f - alpha);
                const float vs = valid ? -raw * (tfv[s] * ra) : 0.f;
                S0 += vs;
                const float vsy = vs * dy;
                Sy += vsy;
                Syy = __fmaf_rn(vsy, dy, Syy);
            }
            }
            if (!__any_sync(FULL, S0 != 0.f)) continue;  // every term carries vs: all zero => nothing to add
            const float ca = A.z * (2.f * LN2), cbb = A.w * LN2, cc = B.x * (2.f * LN2);
            float l0 = ca * dx * S0 + cbb * Sy;
            float l1 = cbb * dx * S0 + cc * Sy;
            float l2 = 0.5f * dx * dx * S0;
            float l3 = dx * Sy;
            float l4 = 0.5f * Syy;
            float l5 = -S0 / o;
            float comps[6] = {l0, l1, l2, l3, l4, l5};
            const float mine = warp_multi_reduce<6>(comps, lane);
            if (my_comp >= 0) accumulate_grad<DET>(p, fscale, (size_t)(__float_as_int(B.z) & ID_MASK) * SGN_RECORD_FLOATS + my_comp, mine);
        }
        buf ^= 1;
    }
}

// DEPTHG: the depth output has a cotangent.  OBJ: object_acc has one; its gradient is folded into the main traversal
// (see below).
// (Measured and dropped: software-pipelining the reduction of entry t-1 under the arithmetic of entry t -- it
// has to run unconditionally, which costs more than the overlap gains: 0.87 vs 0.82 ms on cfg3.)
template <int PPL, bool DEPTHG, bool PACK, bool OBJ, bool DET>
__device__ __forceinline__ void blend_bwd_strip(const BlendBwdParams& p, int tile, int strip, const int2 range,
                                                float4 (*sA)[32], float4 (*sB)[32], float4 (*sC)[32]) {
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    const float px = (float)j + 0.5f, py0 = (float)i0 + 0.5f;
    const size_t P = (size_t)p.width * p.height;

    // ---- per-pixel prologue: cotangents of the RAW blend outputs from those of the final outputs
    float T[PPL], tfv[PPL];
    float vr[PPL], vg[PPL], vb[PPL], vd[PPL];
    float bv[PPL];  // running  sum_{later k} (c_k . v_out) * alpha_k * T_k  (gsplat's `buffer` dotted with v_out)
    int idx[PPL];
    float tfo[PPL];  // OBJ: T_final * v_out of the objects-only accumulation
    int idxo[PPL];   // OBJ: its last entry, as an object sub-list position
    int kmax = -1, kmaxo = -1;
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        T[s] = 1.f; tfv[s] = 0.f; vr[s] = vg[s] = vb[s] = vd[s] = 0.f;
        bv[s] = 0.f;
        idx[s] = -1;
        tfo[s] = 0.f; idxo[s] = -1;
        const int i = i0 + 2 * s;
        if (j >= p.width || i >= p.height) continue;
        const size_t pid = (size_t)i * p.width + j;
        const float Tf = p.final_T[SLOT_MAIN * P + pid];
        idx[s] = p.final_idx[SLOT_MAIN * P + pid];
        T[s] = Tf;
        const float alpha = 1.f - Tf;
        const float4 raw = p.raw[pid];
        float voa = p.v_acc ? p.v_acc[pid] : 0.f;
        if (p.v_bg && p.final_idx[SLOT_BG * P + pid] == BG_SAME_AS_MAIN) voa += p.v_bg[pid];  // background_acc == accumulation here
        if (p.raw_mode) {  // out_c = blended_c + (1 - alpha) * bg_c
            if (p.v_rgb) {
                vr[s] = p.v_rgb[3 * pid]; vg[s] = p.v_rgb[3 * pid + 1]; vb[s] = p.v_rgb[3 * pid + 2];
                voa -= p.bg[0] * vr[s] + p.bg[1] * vg[s] + p.bg[2] * vb[s];
            }
            if (DEPTHG) { vd[s] = p.v_depth[pid]; voa -= p.bg[3] * vd[s]; }
        } else if (p.v_rgb) {
            float v[3] = {p.v_rgb[3 * pid], p.v_rgb[3 * pid + 1], p.v_rgb[3 * pid + 2]};
            const float rr[3] = {raw.x, raw.y, raw.z};
            float vraw[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float cl = fminf(rr[c], 1.f);
                float fin = cl;
                float sk = 0.f;
                if (p.has_sky) { sk = p.sky[3 * pid + c]; fin = cl * alpha + sk * (1.f - alpha); }
                if (p.eval_clamp && (fin < 0.f || fin > 1.f)) v[c] = 0.f;
                if (p.has_sky) {
                    voa += v[c] * (cl - sk);
                    if (p.v_sky) p.v_sky[3 * pid + c] = v[c] * (1.f - alpha);
                    vraw[c] = (rr[c] <= 1.f) ? v[c] * alpha : 0.f;
                } else {
                    vraw[c] = (rr[c] <= 1.f) ? v[c] : 0.f;
                }
            }
            vr[s] = vraw[0]; vg[s] = vraw[1]; vb[s] = vraw[2];
        }
        if (DEPTHG && !p.raw_mode) {
            if (alpha > 1e-3f) {
                const float vdep = p.v_depth[pid];
                vd[s] = vdep / alpha;
                voa += -vdep * raw.w / (alpha * alpha);
            }
        }
        tfv[s] = Tf * voa;
        kmax = max(kmax, idx[s]);
        if (OBJ) {
            tfo[s] = p.final_T[SLOT_OBJ * P + pid] * p.v_obj[pid];
            idxo[s] = p.final_idx[SLOT_OBJ * P + pid];
            kmaxo = max(kmaxo, idxo[s]);
        }
    }
    if (range.y <= range.x) return;  // empty tile (after the prologue: v_sky is written for every pixel)
    const int wkmax = warp_max(kmax);
    const int hi0 = min(range.y, wkmax + 1);  // entries at positions >= hi0 matter to no pixel's main stream
    if (!OBJ && hi0 <= range.x) return;

    // OBJ: the objects-only accumulation's gradient, folded into this traversal.  An object entry at list position k < hi0
    // is the object sub-list entry of position orank (counted back to front from the number of object entries in
    // [range.x, hi0)); it adds T_final_o * ra * v_obj to the v_alpha of the pixels whose objects-only stream took it
    // (orank <= idxo), before the one shared reduction.  Object entries at positions >= hi0 are left to acc_bwd_traverse.
    int orank = 0;
    if constexpr (OBJ) {
        int nobj = 0;
#pragma unroll 4
        for (int b = range.x; b < hi0; b += 32) nobj += __popc(__ballot_sync(FULL, b + lane < hi0 && p.sorted_ids[b + lane] < 0));
        orank = p.cls_bins[1][tile].x + nobj;
    }
    const int orest = orank;  // first object sub-list position past this traversal

    Staged nxt;
    if (hi0 - 1 - lane >= range.x) nxt = gather_entry(p.records, p.sorted_ids[hi0 - 1 - lane]);
    int buf = 0;
    constexpr int NV = DEPTHG ? 10 : 9;
    const int my_comp = multi_reduce_slot<NV>(lane);
    const float clampb = in_register(p.clamp_bwd), nclamp = -clampb;
    const float fscale = DET ? __ldg(p.fixed_scale) : 0.f;
    constexpr bool PK = PACK && PPL >= 2;
    constexpr int NP = PK ? PPL / 2 : 1;
    f2 T2[NP], d2[NP], vr2[NP], vg2[NP], vb2[NP], vd2[NP];
    if constexpr (PK) {
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            T2[q] = f2{T[2 * q], T[2 * q + 1]}; d2[q] = f2{tfv[2 * q], tfv[2 * q + 1]};
            vr2[q] = f2{vr[2 * q], vr[2 * q + 1]}; vg2[q] = f2{vg[2 * q], vg[2 * q + 1]};
            vb2[q] = f2{vb[2 * q], vb[2 * q + 1]}; vd2[q] = f2{vd[2 * q], vd[2 * q + 1]};
        }
    }
    for (int hi = hi0; hi > range.x; hi -= 32) {
        sA[buf][lane] = nxt.A; sB[buf][lane] = nxt.B; sC[buf][lane] = nxt.C;
        __syncwarp();
        if (hi - 33 - lane >= range.x) nxt = gather_entry(p.records, p.sorted_ids[hi - 33 - lane]);
        const int n = min(32, hi - range.x);
        for (int t = 0; t < n; ++t) {
            const int k = hi - 1 - t;
            const float4 A = sA[buf][t];
            const float4 B = sB[buf][t];
            const float4 Cc = sC[buf][t];
            const float dx = A.x - px;
            const float bdx = A.w * dx, ax2 = A.z * dx * dx;
            const float dy0 = A.y - py0;
            // valid  <=>  0 <= sg <= log2(255 o)  <=>  bits(sg) < lim1  (see blend_fwd_strip), and k <= idx
            const unsigned lim1 = (unsigned)(max(__float_as_int(LOG2_255 + B.y), -1) + 1);
            const float o = Cc.w;
            float S0 = 0.f, Sy = 0.f, Syy = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, cd = 0.f;
            float activity = 0.f;  // sum of alpha*T over the valid slots: non-zero iff some pixel of this lane took the entry
            // OE (warp-uniform): an object entry, whose objects-only gradient is added here as well
            auto entry = [&](auto obj_tag) {
                constexpr bool OE = decltype(obj_tag)::value;
                if constexpr (PK) {
                    // packed row-slot pairs.  An invalid slot is masked ONCE, at the exponential (raw = 0): then
                    // alpha = 0, 1/(1-alpha) = 1, T and the running sums pass through unchanged and its gradient
                    // terms are exact zeros, so no further selects are needed.  The running value is
                    // d = T_final*v_acc - buffer.v, and the colour sums are kept negated (nfac = -alpha*T).
                    // (OE: a slot valid for the objects-only stream only masks the main terms with selects.)
                    f2 S0p = dup2(0.f), Syp = dup2(0.f), Syyp = dup2(0.f);
                    f2 ncr = dup2(0.f), ncg = dup2(0.f), ncb = dup2(0.f), ncd = dup2(0.f), nact = dup2(0.f);
                    const f2 dyb = f2{dy0, dy0 - 2.f};
#pragma unroll
                    for (int q = 0; q < NP; ++q) {
                        const f2 dy = add2(dyb, dup2(-(float)(4 * q)));
                        const f2 sg = fma2(dy, fma2(dup2(B.x), dy, dup2(bdx)), dup2(ax2));
                        const bool s0 = __float_as_uint(sg.x) < lim1, s1 = __float_as_uint(sg.y) < lim1;
                        const bool v0 = s0 && (k <= idx[2 * q]), v1 = s1 && (k <= idx[2 * q + 1]);
                        const bool o0 = OE && s0 && (orank <= idxo[2 * q]), o1 = OE && s1 && (orank <= idxo[2 * q + 1]);
                        const f2 nraw = f2{(v0 || o0) ? -fast_ex2(B.y - sg.x) : 0.f, (v1 || o1) ? -fast_ex2(B.y - sg.y) : 0.f};  // -o*exp(-sigma)
                        const f2 nal = f2{fmaxf(nclamp, nraw.x), fmaxf(nclamp, nraw.y)};                 // -alpha
                        const f2 om = add2(nal, dup2(1.f));
                        const f2 ra = f2{fast_rcp(om.x), fast_rcp(om.y)};
                        f2 ram = ra, nalm = nal;  // the main stream's
                        if (OE) {
                            ram = f2{v0 ? ra.x : 1.f, v1 ? ra.y : 1.f};
                            nalm = f2{v0 ? nal.x : 0.f, v1 ? nal.y : 0.f};
                        }
                        const f2 Tk = mul2(T2[q], ram);
                        T2[q] = Tk;
                        const f2 nfac = mul2(nalm, Tk);
                        nact = add2(nact, nfac);
                        ncr = fma2(nfac, vr2[q], ncr); ncg = fma2(nfac, vg2[q], ncg); ncb = fma2(nfac, vb2[q], ncb);
                        f2 dotc = fma2(dup2(B.z), vr2[q], fma2(dup2(B.w), vg2[q], mul2(dup2(Cc.x), vb2[q])));
                        if (DEPTHG) {
                            ncd = fma2(nfac, vd2[q], ncd);
                            dotc = fma2(dup2(Cc.y), vd2[q], dotc);
                        }
                        f2 v_alpha = fma2(Tk, dotc, mul2(ram, d2[q]));
                        d2[q] = fma2(nfac, dotc, d2[q]);
                        if (OE) {
                            v_alpha = f2{v0 ? v_alpha.x : 0.f, v1 ? v_alpha.y : 0.f};
                            v_alpha = fma2(ra, f2{o0 ? tfo[2 * q] : 0.f, o1 ? tfo[2 * q + 1] : 0.f}, v_alpha);
                            nact = add2(nact, f2{o0 ? nal.x : 0.f, o1 ? nal.y : 0.f});
                        }
                        const f2 vs = mul2(nraw, v_alpha);  // d/d sigma = -o*vis*v_alpha
                        S0p = add2(S0p, vs);
                        const f2 vsy = mul2(vs, dy);
                        Syp = add2(Syp, vsy);
                        Syyp = fma2(vsy, dy, Syyp);
                    }
                    S0 = S0p.x + S0p.y; Sy = Syp.x + Syp.y; Syy = Syyp.x + Syyp.y;
                    cr = -(ncr.x + ncr.y); cg = -(ncg.x + ncg.y); cb = -(ncb.x + ncb.y);
                    if (DEPTHG) cd = -(ncd.x + ncd.y);
                    activity = nact.x + nact.y;
                } else {
                // straight-line, predicated (see the forward)
#pragma unroll
                for (int s = 0; s < PPL; ++s) {
                    const float dy = dy0 - (float)(2 * s);
                    const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                    const bool sv = __float_as_uint(sg) < lim1;
                    const bool valid = sv && (k <= idx[s]);
                    const bool ov = OE && sv && (orank <= idxo[s]);
                    const float raw = fast_ex2(B.y - sg);       // o * exp(-sigma)
                    const float alpha = fminf(clampb, raw);
                    const float ra = fast_rcp(1.f - alpha);
                    const bool vm = valid;
                    const float Tk = vm ? T[s] * ra : T[s];
                    T[s] = Tk;
                    const float fac = vm ? alpha * Tk : 0.f;
                    activity += fac;
                    cr = __fmaf_rn(fac, vr[s], cr); cg = __fmaf_rn(fac, vg[s], cg); cb = __fmaf_rn(fac, vb[s], cb);
                    // v_alpha = sum_c (c*T - buffer_c*ra) * v_c + T_final*ra*v_acc  =  T*(c.v) + ra*(T_final*v_acc - buffer.v)
                    float dotc = __fmaf_rn(B.z, vr[s], __fmaf_rn(B.w, vg[s], Cc.x * vb[s]));
                    if (DEPTHG) {
                        cd = __fmaf_rn(fac, vd[s], cd);
                        dotc = __fmaf_rn(Cc.y, vd[s], dotc);
                    }
                    float v_alpha = __fmaf_rn(Tk, dotc, ra * (tfv[s] - bv[s]));
                    bv[s] = __fmaf_rn(fac, dotc, bv[s]);
                    if (OE) {
                        v_alpha = valid ? v_alpha : 0.f;
                        v_alpha = ov ? __fmaf_rn(ra, tfo[s], v_alpha) : v_alpha;
                        activity += ov ? alpha : 0.f;
                    }
                    const float vs = (valid || ov) ? -raw * v_alpha : 0.f;   // d/d sigma = -o*vis*v_alpha
                    S0 += vs;
                    const float vsy = vs * dy;
                    Sy += vsy;
                    Syy = __fmaf_rn(vsy, dy, Syy);
                }
                }
            };
            if (OBJ && __float_as_int(Cc.z) < 0) {
                --orank;
                entry(std::true_type{});
            } else {
                entry(std::false_type{});
            }
            if (!__any_sync(FULL, activity != 0.f)) continue;
            // true conic from the staged (log2e-scaled) one
            const float ca = A.z * (2.f * LN2), cbb = A.w * LN2, cc = B.x * (2.f * LN2);
            float l0 = ca * dx * S0 + cbb * Sy;     // v_xy.x
            float l1 = cbb * dx * S0 + cc * Sy;     // v_xy.y
            float l2 = 0.5f * dx * dx * S0;         // v_conic.x
            float l3 = dx * Sy;                     // v_conic.y
            float l4 = 0.5f * Syy;                  // v_conic.z
            float l5 = -S0 / o;                     // v_opacity = sum vis * v_alpha
            // one component of the record-layout gradient per lane pair
            float comps[NV] = {l0, l1, l2, l3, l4, l5, cr, cg, cb};
            if (DEPTHG) comps[NV - 1] = cd;
            const size_t dst = (size_t)(__float_as_int(Cc.z) & ID_MASK) * SGN_RECORD_FLOATS + (my_comp >= 0 ? my_comp : 0);
            const float mine = warp_multi_reduce<NV>(comps, lane);
            if (my_comp >= 0) accumulate_grad<DET>(p, fscale, dst, mine);
        }
        buf ^= 1;
    }
    if constexpr (OBJ) {  // object entries past this traversal: the accumulation-only backward
        const int ohi = min(p.cls_bins[1][tile].y, warp_max(kmaxo) + 1);
        if (ohi > orest) {
            __syncwarp();  // every lane has finished reading the staging ring
            acc_bwd_traverse<PPL, true, DET>(p, p.cls_ids[1], tile, strip, make_int2(orest, ohi), tfo, idxo, sA, sB,
                                        reinterpret_cast<float(*)[32]>(&sC[0][0]));
        }
    }
}

// the prologue (v_sky, cotangent chain) must run for every pixel, so strips are always launched for the
// whole tile: W strips of 16/W rows.  OBJ: the strips are sized from the main depth plus how far the objects-only
// streams run past it (tile_depth[object], see blend_fwd_strip).
template <bool DEPTHG, bool PACK, bool OBJ, bool DET>
__global__ void __launch_bounds__(32, BLEND_BWD_MIN_BLOCKS) blend_bwd_kernel(const BlendBwdParams p) {
    __shared__ float4 sA[2][32];
    __shared__ float4 sB[2][32];
    __shared__ float4 sC[2][32];
    int tile, strip;
    if (!take_work(p.sched, SLOT_MAIN, p.tiles, tile, strip)) return;
    const int2 range = p.tile_bins[tile];
    const int W = strips_for(p.tile_depth[tile] + (OBJ ? p.tile_depth[(size_t)SLOT_OBJ * p.tiles + tile] : 0), p.split_main);
    if (strip >= W) return;
    switch (W) {
        case 1: blend_bwd_strip<8, DEPTHG, PACK, OBJ, DET>(p, tile, strip, range, sA, sB, sC); break;
        case 2: blend_bwd_strip<4, DEPTHG, PACK, OBJ, DET>(p, tile, strip, range, sA, sB, sC); break;
        case 4: blend_bwd_strip<2, DEPTHG, PACK, OBJ, DET>(p, tile, strip, range, sA, sB, sC); break;
        default: blend_bwd_strip<1, DEPTHG, PACK, OBJ, DET>(p, tile, strip, range, sA, sB, sC); break;
    }
}

// the background-only accumulation's backward (the objects-only one is part of blend_bwd_kernel)
template <int PPL, bool SKIP, bool DET>
__device__ __forceinline__ void acc_bwd_strip(const BlendBwdParams& p, int cls, int tile, int strip, const int2 range,
                                              float4 (*sA)[32], float4 (*sB)[32], float (*sR)[32]) {
    const int slot = cls ? SLOT_OBJ : SLOT_BG;
    const float* __restrict__ v_out = cls ? p.v_obj : p.v_bg;
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + strip * (2 * PPL) + (lane >> 4);
    if (range.y <= range.x) return;
    const size_t P = (size_t)p.width * p.height;
    float tfv[PPL];
    int idx[PPL];
    int kmax = -1;
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        tfv[s] = 0.f; idx[s] = -1;
        const int i = i0 + 2 * s;
        if (j >= p.width || i >= p.height) continue;
        const size_t pid = (size_t)i * p.width + j;
        tfv[s] = p.final_T[slot * P + pid] * v_out[pid];
        idx[s] = p.final_idx[slot * P + pid];
        kmax = max(kmax, idx[s]);
    }
    const int wkmax = warp_max(kmax);
    const int hi0 = min(range.y, wkmax + 1);
    if (hi0 <= range.x) return;
    acc_bwd_traverse<PPL, SKIP, DET>(p, p.cls_ids[cls], tile, strip, make_int2(range.x, hi0), tfv, idx, sA, sB, sR);
}

template <bool SKIP, bool DET>
__global__ void __launch_bounds__(32, BLEND_ACC_MIN_BLOCKS) acc_bwd_kernel(const BlendBwdParams p, const int cls) {
    __shared__ float4 sA[2][32];
    __shared__ float4 sB[2][32];
    __shared__ float sR[2][32];
    int tile, strip;
    if (!take_work(p.sched, cls ? SLOT_OBJ : SLOT_BG, p.tiles, tile, strip)) return;
    const int2 range = p.cls_bins[cls][tile];
    const int W = strips_for(p.tile_depth[(size_t)(cls ? SLOT_OBJ : SLOT_BG) * p.tiles + tile], p.split_acc);
    if (strip >= W) return;
    switch (W) {
        case 1: acc_bwd_strip<8, SKIP, DET>(p, cls, tile, strip, range, sA, sB, sR); break;
        case 2: acc_bwd_strip<4, SKIP, DET>(p, cls, tile, strip, range, sA, sB, sR); break;
        case 4: acc_bwd_strip<2, SKIP, DET>(p, cls, tile, strip, range, sA, sB, sR); break;
        default: acc_bwd_strip<1, SKIP, DET>(p, cls, tile, strip, range, sA, sB, sR); break;
    }
}

// ---- deterministic mode: the grid comes from cot_max_kernel + fixed_scale_kernel (sgn_fixed.cuh), then fixed point -> float
__global__ void __launch_bounds__(256)
fixed_to_float_kernel(const long long* __restrict__ fx, const float* __restrict__ scale, const float* __restrict__ records,
                      float* __restrict__ out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)(ldexp((double)fx[i], fixed_shift(records, (size_t)i)) / (double)scale[0]);
}

template <bool DET>
static int launch_blend_bwd(const BlendBwdParams& p, int tuning, cudaStream_t side, cudaStream_t stream) {
    const unsigned acc_grid = p.tiles * 8;
    if (p.v_bg) {
        if (!(tuning & SGN_TUNE_ACC_NO_ROW_SKIP)) acc_bwd_kernel<true, DET><<<acc_grid, 32, 0, side>>>(p, 0);
        else acc_bwd_kernel<false, DET><<<acc_grid, 32, 0, side>>>(p, 0);
        SGN_CHECK_LAUNCH("acc_bwd_kernel<background>");
    }
    const bool pack = (tuning & SGN_TUNE_BWD_PACKED) != 0;
    const dim3 grid(p.tiles * 8), block(32);
    switch ((p.v_obj ? 4 : 0) | (p.v_depth ? 2 : 0) | (pack ? 1 : 0)) {
        case 0: blend_bwd_kernel<false, false, false, DET><<<grid, block, 0, stream>>>(p); break;
        case 1: blend_bwd_kernel<false, true, false, DET><<<grid, block, 0, stream>>>(p); break;
        case 2: blend_bwd_kernel<true, false, false, DET><<<grid, block, 0, stream>>>(p); break;
        case 3: blend_bwd_kernel<true, true, false, DET><<<grid, block, 0, stream>>>(p); break;
        case 4: blend_bwd_kernel<false, false, true, DET><<<grid, block, 0, stream>>>(p); break;
        case 5: blend_bwd_kernel<false, true, true, DET><<<grid, block, 0, stream>>>(p); break;
        case 6: blend_bwd_kernel<true, false, true, DET><<<grid, block, 0, stream>>>(p); break;
        default: blend_bwd_kernel<true, true, true, DET><<<grid, block, 0, stream>>>(p); break;
    }
    SGN_CHECK_LAUNCH("blend_bwd_kernel");
    return SGN_OK;
}

extern "C" int sgn_blend_bwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records,
                             const int32_t* sorted_ids, const int32_t* tile_bins, int64_t M, const int32_t* cls_ids,
                             const int32_t* cls_bins, const sgn_blend_bwd_in* in, float* v_records, void* stream_) {
    SGN_RANGE("sgn_blend_bwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = check_cam(cam)) return rc;
    SGN_REQUIRE(opts && records && tile_bins && in && v_records, "sgn_blend_bwd: null pointer");
    SGN_REQUIRE(in->raw && in->final_T && in->final_idx, "sgn_blend_bwd: saved forward state missing");
    SGN_REQUIRE(!opts->has_sky || in->sky, "has_sky set but sky is null");
    SGN_REQUIRE(!(in->v_object_acc || in->v_background_acc) || opts->class_streams,
                "cotangents for object_acc/background_acc need class_streams");
    SGN_REQUIRE(!(in->v_object_acc || in->v_background_acc) || (cls_ids && cls_bins), "class cotangents need the class sub-lists");
    SGN_REQUIRE(sgn_aligned16(records) && sgn_aligned16(in->raw), "records / raw must be 16-byte aligned");
    BlendBwdParams p;
    p.width = cam->width; p.height = cam->height;
    p.tiles_x = (cam->width + SGN_TILE - 1) / SGN_TILE;
    const int tiles_y = (cam->height + SGN_TILE - 1) / SGN_TILE;
    p.clamp_bwd = opts->alpha_clamp_bwd;
    p.split_main = opts->split_bwd_main > 0 ? opts->split_bwd_main : 384;
    p.split_acc = opts->split_bwd_acc > 0 ? opts->split_bwd_acc : 384;
    p.has_sky = opts->has_sky; p.eval_clamp = opts->eval_clamp; p.raw_mode = opts->raw_mode;
    for (int c = 0; c < 4; ++c) p.bg[c] = opts->background[c];
    p.records = reinterpret_cast<const float4*>(records);
    p.sorted_ids = sorted_ids;
    p.tile_bins = reinterpret_cast<const int2*>(tile_bins);
    const int tiles = p.tiles_x * tiles_y;
    p.tiles = tiles;
    p.cls_ids[0] = cls_ids; p.cls_ids[1] = cls_ids ? cls_ids + M : nullptr;
    p.cls_bins[0] = reinterpret_cast<const int2*>(cls_bins);
    p.cls_bins[1] = cls_bins ? reinterpret_cast<const int2*>(cls_bins) + tiles : nullptr;
    p.v_rgb = in->v_rgb; p.v_acc = in->v_accumulation; p.v_depth = in->v_depth;
    p.v_obj = in->v_object_acc; p.v_bg = in->v_background_acc;
    p.raw = reinterpret_cast<const float4*>(in->raw);
    p.final_T = in->final_T; p.final_idx = in->final_idx;
    p.sky = in->sky; p.v_sky = in->v_sky;
    p.v_records = v_records;
    p.v_fixed = reinterpret_cast<long long*>(in->v_fixed);
    p.fixed_scale = in->fixed_scale;
    const long long P_ = (long long)cam->width * cam->height;
    if (in->v_fixed) {
        SGN_REQUIRE(in->fixed_scale && in->num_gaussians > 0, "deterministic mode needs fixed_scale (1 float) and num_gaussians");
        SGN_CHECK_CUDA(cudaMemsetAsync(in->fixed_scale, 0, sizeof(float), stream));
        const float* cots[5] = {in->v_rgb, in->v_accumulation, in->v_depth, in->v_object_acc, in->v_background_acc};
        for (int c = 0; c < 5; ++c) {
            if (!cots[c]) continue;
            cot_max_kernel<<<296, 256, 0, stream>>>(cots[c], c == 0 ? 3 * P_ : P_, reinterpret_cast<unsigned*>(in->fixed_scale));
            SGN_CHECK_LAUNCH("cot_max_kernel");
        }
        fixed_scale_kernel<<<1, 1, 0, stream>>>(in->fixed_scale);
        SGN_CHECK_LAUNCH("fixed_scale_kernel");
    }
    SGN_REQUIRE(in->tile_depth, "sgn_blend_bwd: tile_depth (saved by the forward) is null");
    p.tile_depth = in->tile_depth;
    p.sched = in->sched;
    if (in->sched) {
        sched_kernel<<<in->v_background_acc ? 2 : 1, 1024, 0, stream>>>(
            tiles, p.tile_bins, p.cls_bins[0], in->tile_depth, in->v_object_acc != nullptr, p.split_main, p.split_acc, in->sched);
        SGN_CHECK_LAUNCH("sched_kernel");
    }
    {
        // all three kernels only accumulate (RED) into v_records: they may run concurrently
        ForkJoin fj(stream);
        const int rc = in->v_fixed ? launch_blend_bwd<true>(p, opts->tuning, fj.side(), stream)
                                   : launch_blend_bwd<false>(p, opts->tuning, fj.side(), stream);
        fj.finish();
        if (rc) return rc;
    }
    if (in->v_fixed) {
        const long long n = (long long)in->num_gaussians * SGN_RECORD_FLOATS;
        fixed_to_float_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const long long*>(in->v_fixed), in->fixed_scale,
                                                                                records, v_records, n);
        SGN_CHECK_LAUNCH("fixed_to_float_kernel");
    }
    return SGN_OK;
}

// ------------------------------------------------------------------------------------------------
// Generic per-Gaussian channels (the north-star's "per-Gaussian 4D-SH semantic logits"; dormant consumer in the reference:
// street_gaussians_ns/scripts/render.py:188,231-236, group `semantic` in sgn_config.py:30): C extra values per Gaussian are
// composited with the SAME weights as the colours -- out[p, c] = sum_k e[k, c] * alpha_k * T_k over the entries the main pass
// blended (it saved, per pixel, the index of the last one) -- EXTRA_CG channels per traversal, forward and backward.
// The weights are recomputed with the main pass's arithmetic (same sigma, same ex2, same FMA for T), bounded by final_idx,
// so every pixel sees exactly the entries and weights of the main render.
// ------------------------------------------------------------------------------------------------
#define EXTRA_CG 8

struct ExtraParams {
    int width, height, tiles_x, tiles, C;
    float clamp_fwd, clamp_bwd;
    const float4* records;
    const int32_t* sorted_ids;
    const int2* tile_bins;
    const float* final_T;      // slot 0 (main)
    const int32_t* final_idx;  // slot 0 (main)
    const float* extra;        // [N, C]
    float* out;                // forward: [H, W, C]
    const float* v_out;        // backward: [H, W, C]
    float* v_extra;            // backward: [N, C] (accumulated)
    float* v_records;          // backward: [N, 12] (geometry part accumulated)
};
// the deterministic backward's own arguments: a separate kernel parameter type, so that the float instantiations keep
// theirs (and their register allocation) unchanged
struct ExtraDetParams {
    ExtraParams p;
    long long* fx_geom;     // [N, 6] fixed-point geometry accumulators (zeroed)
    long long* fx_extra;    // [N, C] fixed-point channel accumulators (zeroed)
    const float* fx_scale;  // units per unit of gradient: [0] geometry, [1] channels
};
template <bool DET>
using ExtraArgs = typename std::conditional<DET, ExtraDetParams, ExtraParams>::type;
__device__ __forceinline__ const ExtraParams& extra_base(const ExtraParams& p) { return p; }
__device__ __forceinline__ const ExtraParams& extra_base(const ExtraDetParams& q) { return q.p; }

// one warp per tile, lane = (column, row parity), 8 pixels per lane (rows two apart); blockIdx.y = channel group.
// DET (backward only): the per-Gaussian sums go to the fixed-point accumulators, one rounding per addend and integer adds,
// as accumulate_grad does for the main backward; the float instantiations carry no fixed-point code.
template <bool BWD, bool DET = false>
__global__ void __launch_bounds__(32) extra_kernel(const ExtraArgs<DET> args) {
    static_assert(BWD || !DET, "the forward has no accumulators");
    const ExtraParams& p = extra_base(args);
    constexpr int PPL = 8;
    __shared__ float4 sA[32], sB[32];
    __shared__ float sX[32][EXTRA_CG + 1];
    __shared__ int sId[32];
    const int tile = blockIdx.x, c0 = blockIdx.y * EXTRA_CG;
    const int nch = min(EXTRA_CG, p.C - c0);
    const int2 range = p.tile_bins[tile];
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    const int lane = threadIdx.x;
    const int j = tx * SGN_TILE + (lane & 15);
    const int i0 = ty * SGN_TILE + (lane >> 4);
    const float px = (float)j + 0.5f, py0 = (float)i0 + 0.5f;
    float T[PPL], acc[PPL][EXTRA_CG], bv[PPL];
    int idx[PPL];
    int kmax = -1;
#pragma unroll
    for (int s = 0; s < PPL; ++s) {
        const int i = i0 + 2 * s;
        const bool inside = j < p.width && i < p.height;
        const size_t pid = (size_t)i * p.width + j;
        idx[s] = inside ? p.final_idx[pid] : -1;
        T[s] = BWD ? (inside ? p.final_T[pid] : 1.f) : 1.f;
        bv[s] = 0.f;
        kmax = max(kmax, idx[s]);
#pragma unroll
        for (int c = 0; c < EXTRA_CG; ++c) acc[s][c] = (BWD && inside && c < nch) ? p.v_out[pid * p.C + c0 + c] : 0.f;  // backward: the cotangents
    }
    const int hi0 = min(range.y, warp_max(kmax) + 1);
    if (!BWD) {
        if (hi0 <= range.x) {
#pragma unroll
            for (int s = 0; s < PPL; ++s) {
                const int i = i0 + 2 * s;
                if (j < p.width && i < p.height)
                    for (int c = 0; c < nch; ++c) p.out[((size_t)i * p.width + j) * p.C + c0 + c] = 0.f;
            }
            return;
        }
    } else if (hi0 <= range.x) {
        return;
    }
    const float clampf = in_register(p.clamp_fwd), clampb = in_register(p.clamp_bwd);
    constexpr int NV = 6 + EXTRA_CG;
    const int my_comp = multi_reduce_slot<NV>(lane);
    const int nbatch = (hi0 - range.x + 31) / 32;
    for (int b = 0; b < nbatch; ++b) {
        // forward walks front to back, backward back to front; entry t of the batch is list position k(t)
        const int first = BWD ? hi0 - 1 - 32 * b : range.x + 32 * b;
        const int n = BWD ? min(32, first - range.x + 1) : min(32, hi0 - first);
        __syncwarp();
        if (lane < n) {
            const int k = BWD ? first - lane : first + lane;
            const int id = p.sorted_ids[k];
            const Staged e = gather_entry(p.records, id);
            sA[lane] = e.A;
            sB[lane] = make_float4(e.B.x, e.B.y, e.C.w /* opacity */, 0.f);
            sId[lane] = id & ID_MASK;
            const float* ex = p.extra + (size_t)(id & ID_MASK) * p.C + c0;
            for (int c = 0; c < EXTRA_CG; ++c) sX[lane][c] = c < nch ? ex[c] : 0.f;
        }
        __syncwarp();
        for (int t = 0; t < n; ++t) {
            const int k = BWD ? first - t : first + t;
            const float4 A = sA[t], B = sB[t];
            const float dx = A.x - px;
            const float bdx = A.w * dx, ax2 = A.z * dx * dx;
            const float dy0 = A.y - py0;
            const unsigned lim1 = (unsigned)(max(__float_as_int(LOG2_255 + B.y), -1) + 1);
            float e[EXTRA_CG];
#pragma unroll
            for (int c = 0; c < EXTRA_CG; ++c) e[c] = sX[t][c];
            if (!BWD) {
#pragma unroll
                for (int s = 0; s < PPL; ++s) {
                    const float dy = dy0 - (float)(2 * s);
                    const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                    const bool valid = (__float_as_uint(sg) < lim1) && (k <= idx[s]);
                    const float am = valid ? fminf(clampf, fast_ex2(B.y - sg)) : 0.f;
                    const float w = am * T[s];
                    T[s] = __fmaf_rn(-am, T[s], T[s]);
#pragma unroll
                    for (int c = 0; c < EXTRA_CG; ++c) acc[s][c] = __fmaf_rn(e[c], w, acc[s][c]);
                }
            } else {
                float S0 = 0.f, Sy = 0.f, Syy = 0.f, ve[EXTRA_CG];
#pragma unroll
                for (int c = 0; c < EXTRA_CG; ++c) ve[c] = 0.f;
                float activity = 0.f;
#pragma unroll
                for (int s = 0; s < PPL; ++s) {
                    const float dy = dy0 - (float)(2 * s);
                    const float sg = __fmaf_rn(dy, __fmaf_rn(B.x, dy, bdx), ax2);
                    const bool valid = (__float_as_uint(sg) < lim1) && (k <= idx[s]);
                    const float raw = fast_ex2(B.y - sg);
                    const float alpha = fminf(clampb, raw);
                    const float ra = fast_rcp(1.f - alpha);
                    const float Tk = valid ? T[s] * ra : T[s];
                    T[s] = Tk;
                    const float fac = valid ? alpha * Tk : 0.f;
                    activity += fac;
                    float dotc = 0.f;
#pragma unroll
                    for (int c = 0; c < EXTRA_CG; ++c) {
                        ve[c] = __fmaf_rn(fac, acc[s][c], ve[c]);
                        dotc = __fmaf_rn(e[c], acc[s][c], dotc);
                    }
                    // v_alpha = sum_c (e_c T_k - buffer_c / (1 - alpha)) v_c, buffer = what lies behind entry k
                    const float v_alpha = __fmaf_rn(Tk, dotc, -ra * bv[s]);
                    bv[s] = __fmaf_rn(fac, dotc, bv[s]);
                    const float vs = valid ? -raw * v_alpha : 0.f;
                    S0 += vs;
                    const float vsy = vs * dy;
                    Sy += vsy;
                    Syy = __fmaf_rn(vsy, dy, Syy);
                }
                if (!__any_sync(FULL, activity != 0.f)) continue;
                const float ca = A.z * (2.f * LN2), cbb = A.w * LN2, cc = B.x * (2.f * LN2);
                float comps[NV];
                comps[0] = ca * dx * S0 + cbb * Sy;
                comps[1] = cbb * dx * S0 + cc * Sy;
                comps[2] = 0.5f * dx * dx * S0;
                comps[3] = dx * Sy;
                comps[4] = 0.5f * Syy;
                comps[5] = -S0 / B.z;
#pragma unroll
                for (int c = 0; c < EXTRA_CG; ++c) comps[6 + c] = ve[c];
                const float mine = warp_multi_reduce<NV>(comps, lane);
                if (my_comp >= 0) {
                    const size_t g = (size_t)sId[t];
                    if constexpr (DET) {
                        if (my_comp < 6) {
                            const int sh = fixed_shift(reinterpret_cast<const float*>(p.records), g * SGN_RECORD_FLOATS + my_comp);
                            const float m = mine * __ldg(args.fx_scale) * __int_as_float((127 - sh) << 23);  // times 2^-sh: exact
                            atomicAdd(reinterpret_cast<unsigned long long*>(args.fx_geom) + g * 6 + my_comp, (unsigned long long)__float2ll_rn(m));
                        } else if (my_comp - 6 < nch) {
                            atomicAdd(reinterpret_cast<unsigned long long*>(args.fx_extra) + g * p.C + c0 + (my_comp - 6),
                                      (unsigned long long)__float2ll_rn(mine * __ldg(args.fx_scale + 1)));
                        }
                    } else {
                        if (my_comp < 6) atomicAdd(p.v_records + g * SGN_RECORD_FLOATS + my_comp, mine);
                        else if (my_comp - 6 < nch) atomicAdd(p.v_extra + g * p.C + c0 + (my_comp - 6), mine);
                    }
                }
            }
        }
    }
    if (!BWD) {
#pragma unroll
        for (int s = 0; s < PPL; ++s) {
            const int i = i0 + 2 * s;
            if (j < p.width && i < p.height)
                for (int c = 0; c < nch; ++c) p.out[((size_t)i * p.width + j) * p.C + c0 + c] = acc[s][c];
        }
    }
}

static int extra_params(ExtraParams& p, const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                        const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C) {
    if (int rc = check_cam(cam)) return rc;
    SGN_REQUIRE(opts && records && sorted_ids && tile_bins && final_T && final_idx && extra, "sgn_blend_extra: null pointer");
    SGN_REQUIRE(C >= 1 && C <= 4096, "sgn_blend_extra: C=%d out of range", C);
    SGN_REQUIRE(sgn_aligned16(records), "records must be 16-byte aligned");
    p.width = cam->width; p.height = cam->height;
    p.tiles_x = (cam->width + SGN_TILE - 1) / SGN_TILE;
    p.tiles = p.tiles_x * ((cam->height + SGN_TILE - 1) / SGN_TILE);
    p.C = C;
    p.clamp_fwd = opts->alpha_clamp_fwd; p.clamp_bwd = opts->alpha_clamp_bwd;
    p.records = reinterpret_cast<const float4*>(records);
    p.sorted_ids = sorted_ids;
    p.tile_bins = reinterpret_cast<const int2*>(tile_bins);
    p.final_T = final_T; p.final_idx = final_idx;
    p.extra = extra;
    p.out = nullptr; p.v_out = nullptr; p.v_extra = nullptr; p.v_records = nullptr;
    return SGN_OK;
}

extern "C" int sgn_blend_extra_fwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                                   const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                                   float* out, void* stream) {
    SGN_RANGE("sgn_blend_extra_fwd");
    ExtraParams p;
    if (int rc = extra_params(p, cam, opts, records, sorted_ids, tile_bins, final_T, final_idx, extra, C)) return rc;
    SGN_REQUIRE(out, "sgn_blend_extra_fwd: null output");
    p.out = out;
    extra_kernel<false><<<dim3(p.tiles, (C + EXTRA_CG - 1) / EXTRA_CG), 32, 0, (cudaStream_t)stream>>>(p);
    SGN_CHECK_LAUNCH("extra_kernel<fwd>");
    return SGN_OK;
}

extern "C" int sgn_blend_extra_bwd(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                                   const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                                   const float* v_out, float* v_extra, float* v_records, void* stream) {
    SGN_RANGE("sgn_blend_extra_bwd");
    ExtraParams p;
    if (int rc = extra_params(p, cam, opts, records, sorted_ids, tile_bins, final_T, final_idx, extra, C)) return rc;
    SGN_REQUIRE(v_out && v_extra && v_records, "sgn_blend_extra_bwd: null pointer");
    p.v_out = v_out; p.v_extra = v_extra; p.v_records = v_records;
    extra_kernel<true><<<dim3(p.tiles, (C + EXTRA_CG - 1) / EXTRA_CG), 32, 0, (cudaStream_t)stream>>>(p);
    SGN_CHECK_LAUNCH("extra_kernel<bwd>");
    return SGN_OK;
}

// ---- deterministic extra backward: the fixed-point grids are powers of two.  An entry's alpha cotangent is
// sum_c extra_c v_c, at most C max|extra| max|v_out|: the geometry grid is 2^32 units per unit of that bound (the
// conic components of wide Gaussians give up fixed_shift places, as in the main backward).  A channel gradient is a sum
// of weights times v_out: its grid is 2^32 units per max|v_out|.  Both keep 2^31 units of headroom.
__global__ void extra_fixed_scale_kernel(float* scale, int C) {
    const float mv = scale[0], me = fmaxf(1.f, scale[1]);  // the bits cot_max_kernel left are the floats themselves
    const double eg = ceil(log2((double)mv * (double)me * (double)C)), ev = ceil(log2((double)mv));
    scale[0] = mv > 0.f ? (float)exp2(32.0 - fmin(eg, 150.0)) : 4294967296.f;
    scale[1] = mv > 0.f ? (float)exp2(32.0 - fmin(ev, 150.0)) : 4294967296.f;
}
__global__ void __launch_bounds__(256)
extra_fixed_add_kernel(const long long* __restrict__ fx_geom, const long long* __restrict__ fx_extra, const float* __restrict__ scale,
                       const float* __restrict__ records, float* __restrict__ v_records, float* __restrict__ v_extra, long long N, int C) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 6 * N) {
        const size_t idx = (size_t)(i / 6) * SGN_RECORD_FLOATS + (size_t)(i % 6);
        v_records[idx] += (float)(ldexp((double)fx_geom[i], fixed_shift(records, idx)) / (double)scale[0]);
    } else if (i < 6 * N + (long long)C * N) {
        const long long k = i - 6 * N;
        v_extra[k] += (float)((double)fx_extra[k] / (double)scale[1]);
    }
}

extern "C" int sgn_blend_extra_bwd_det(const sgn_camera* cam, const sgn_blend_opts* opts, const float* records, const int32_t* sorted_ids,
                                       const int32_t* tile_bins, const float* final_T, const int32_t* final_idx, const float* extra, int C,
                                       int64_t num_gaussians, const float* v_out, float* v_extra, float* v_records, int64_t* fixed_geom,
                                       int64_t* fixed_extra, float* fixed_scale, void* stream_) {
    SGN_RANGE("sgn_blend_extra_bwd_det");
    cudaStream_t stream = (cudaStream_t)stream_;
    ExtraDetParams q;
    ExtraParams& p = q.p;
    if (int rc = extra_params(p, cam, opts, records, sorted_ids, tile_bins, final_T, final_idx, extra, C)) return rc;
    SGN_REQUIRE(v_out && v_extra && v_records && fixed_geom && fixed_extra && fixed_scale, "sgn_blend_extra_bwd_det: null pointer");
    SGN_REQUIRE(num_gaussians > 0, "sgn_blend_extra_bwd_det: num_gaussians=%lld", (long long)num_gaussians);
    p.v_out = v_out; p.v_extra = v_extra; p.v_records = v_records;
    q.fx_geom = reinterpret_cast<long long*>(fixed_geom); q.fx_extra = reinterpret_cast<long long*>(fixed_extra);
    q.fx_scale = fixed_scale;
    SGN_CHECK_CUDA(cudaMemsetAsync(fixed_scale, 0, 2 * sizeof(float), stream));
    cot_max_kernel<<<296, 256, 0, stream>>>(v_out, (long long)p.width * p.height * C, reinterpret_cast<unsigned*>(fixed_scale));
    cot_max_kernel<<<296, 256, 0, stream>>>(extra, (long long)num_gaussians * C, reinterpret_cast<unsigned*>(fixed_scale) + 1);
    SGN_CHECK_LAUNCH("cot_max_kernel");
    extra_fixed_scale_kernel<<<1, 1, 0, stream>>>(fixed_scale, C);
    SGN_CHECK_LAUNCH("extra_fixed_scale_kernel");
    extra_kernel<true, true><<<dim3(p.tiles, (C + EXTRA_CG - 1) / EXTRA_CG), 32, 0, stream>>>(q);
    SGN_CHECK_LAUNCH("extra_kernel<bwd, det>");
    const long long n = (6 + (long long)C) * num_gaussians;
    extra_fixed_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(q.fx_geom, q.fx_extra, fixed_scale, records, v_records, v_extra,
                                                                              num_gaussians, C);
    SGN_CHECK_LAUNCH("extra_fixed_add_kernel");
    return SGN_OK;
}
