// Tile binning: per-Gaussian touched-tile counts -> depth order -> key emit -> stable sort by tile ->
// per-tile bin edges (-> class sub-lists).
// Semantics: gsplat 0.1.x rasterize_gaussians internals (SURVEY.md Appendix A.5): every tile's list is
// ordered like a stable sort of (tile_id << 32 | float_bits(depth)) with emission order (Gaussian index)
// as the tie break.  That order is produced in two cheaper stable steps instead of one 46-bit sort of
// the M intersections:
//   1. the N Gaussians are stably sorted by depth bits (32-bit keys, N elements), carrying their entry payloads;
//   2. intersections are emitted in that order, rank by rank, and stably sorted by their 14-bit tile id only.
// Step 2 moves 12 B per entry twice instead of 24 B six times.
#include <cub/cub.cuh>

#include "sgn_touch.cuh"

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// standalone touched-tile count (the fused path gets it from project_fwd; the Level-1 rasterize path,
// which starts from plain xys/conics tensors, calls this)
__global__ void __launch_bounds__(256)
count_tiles_kernel(int N, int width, int height, int bw, const float4* __restrict__ records, const int32_t* __restrict__ radii,
                   const ushort4* __restrict__ tile_bbox, int32_t* __restrict__ tiles_touched, uint32_t* __restrict__ touch_mask) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    const bool vis = (g < N) && radii[g] > 0;
    ushort4 bb = make_ushort4(0, 0, 0, 0);
    TouchCtx t = {};
    if (vis) {
        bb = tile_bbox[g];
        t = make_touch_ctx(records[3 * (size_t)g], records[3 * (size_t)g + 1]);
    }
    uint32_t mask;
    const int n = count_touched_tiles(vis, t, bb, width, height, bw, mask);
    if (g < N) { tiles_touched[g] = n; touch_mask[g] = mask; }
}

extern "C" int sgn_bin_count(int N, const sgn_camera* cam, const float* records, const int32_t* radii,
                             const uint16_t* tile_bbox, int32_t* tiles_touched, uint32_t* touch_mask, void* stream) {
    SGN_RANGE("sgn_bin_count");
    SGN_REQUIRE(cam && records && radii && tile_bbox && tiles_touched && touch_mask, "sgn_bin_count: null pointer");
    if (N == 0) return SGN_OK;
    count_tiles_kernel<<<(N + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        N, cam->width, cam->height, cam->block_width, reinterpret_cast<const float4*>(records), radii,
        reinterpret_cast<const ushort4*>(tile_bbox), tiles_touched, touch_mask);
    SGN_CHECK_LAUNCH("count_tiles_kernel");
    return SGN_OK;
}

// ------------------------------------------------------------------------------------------------
// step 1: depth order + inclusive scan of the touched-tile counts in that order
__global__ void __launch_bounds__(256)
depth_keys_kernel(int N, const float4* __restrict__ records, const int32_t* __restrict__ radii, uint32_t* __restrict__ keys,
                  int32_t* __restrict__ vals) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    // invisible rows sort last (no positive float has all bits set) and emit nothing
    uint32_t key = 0xffffffffu;
    int32_t payload = g;
    if (radii[g] > 0) {
        const float4 r2 = records[3 * (size_t)g + 2];
        key = (uint32_t)__float_as_int(r2.y);
        // the entry payload travels with the depth key: Gaussian row in the low 31 bits, object-class flag in bit 31
        if (__float_as_int(r2.z) & SGN_AUX_OBJECT) payload |= (int32_t)0x80000000;
    }
    keys[g] = key;
    vals[g] = payload;
}

struct PermutedCount {
    const int32_t* order;
    const int32_t* counts;
    __host__ __device__ int32_t operator()(int i) const { return counts[order[i] & 0x7fffffff]; }
};

__global__ void write_total_kernel(const int32_t* __restrict__ cum, int N, int64_t* __restrict__ total) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *total = (N > 0) ? (int64_t)cum[N - 1] : 0;
}

struct ScanLayout {
    size_t keys_in, keys_out, vals_in, temp, temp_bytes, total;
};
static ScanLayout scan_layout(int N) {
    ScanLayout L;
    const size_t n = (size_t)(N > 0 ? N : 1);
    size_t t1 = 0, t2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                    (int32_t*)nullptr, (int)n, 0, 32);
    cub::DeviceScan::InclusiveSum(nullptr, t2, (const int32_t*)nullptr, (int32_t*)nullptr, (int)n);
    L.keys_in = 0;
    L.keys_out = align_up(n * 4, 256);
    L.vals_in = L.keys_out + align_up(n * 4, 256);
    L.temp = L.vals_in + align_up(n * 4, 256);
    L.temp_bytes = t1 > t2 ? t1 : t2;
    L.total = L.temp + align_up(L.temp_bytes, 256) + 256;
    return L;
}

extern "C" size_t sgn_bin_scan_scratch_bytes(int N) { return scan_layout(N).total; }

extern "C" int sgn_bin_scan(int N, const float* records, const int32_t* radii, const int32_t* tiles_touched,
                            int32_t* order /* out: entry payloads (row | class << 31) in depth order */, int32_t* cum,
                            int64_t* total_dev, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_bin_scan");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(records && radii && tiles_touched && order && cum && total_dev && scratch, "sgn_bin_scan: null pointer");
    const ScanLayout L = scan_layout(N);
    if (scratch_bytes < L.total) {
        sgn_set_error("sgn_bin_scan: scratch too small (%zu < %zu)", scratch_bytes, L.total);
        return SGN_ERR_WORKSPACE;
    }
    if (N > 0) {
        char* base = (char*)scratch;
        uint32_t* keys_in = (uint32_t*)(base + L.keys_in);
        uint32_t* keys_out = (uint32_t*)(base + L.keys_out);
        int32_t* vals_in = (int32_t*)(base + L.vals_in);
        depth_keys_kernel<<<(N + 255) / 256, 256, 0, stream>>>(N, reinterpret_cast<const float4*>(records), radii, keys_in, vals_in);
        SGN_CHECK_LAUNCH("depth_keys_kernel");
        size_t temp = L.temp_bytes;
        SGN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(base + L.temp, temp, keys_in, keys_out, vals_in, order, N, 0, 32, stream));
        sgn_count_launch(1);
        // counts scanned IN DEPTH ORDER: cum[r] = number of entries emitted by the first r+1 rows of that order
        cub::CountingInputIterator<int> idx(0);
        cub::TransformInputIterator<int32_t, PermutedCount, cub::CountingInputIterator<int>> it(idx, PermutedCount{order, tiles_touched});
        temp = L.temp_bytes;
        SGN_CHECK_CUDA(cub::DeviceScan::InclusiveSum(base + L.temp, temp, it, cum, N, stream));
        sgn_count_launch(1);
    }
    // the synchronous path reads the total back before the emit, so it cannot wait for a later kernel
    write_total_kernel<<<1, 32, 0, stream>>>(cum, N, total_dev);
    SGN_CHECK_LAUNCH("write_total_kernel");
    return SGN_OK;
}

// ------------------------------------------------------------------------------------------------
// step 2: key emit in depth order, stable sort by tile, bin edges.
// Thread i handles depth rank i, so the 32 runs of a warp are adjacent in the entry sequence: run i occupies
// [cum[i-1], cum[i]).  Runs of AABBs of at most COOP_AREA tiles are laid end to end and written 32 consecutive
// entries per store: entry f of the warp's flattened sequence belongs to the last lane whose exclusive prefix is <= f
// (as in count_touched_tiles), and is the k-th tile the owner reaches, i.e. the k-th set bit of the touch mask
// project_fwd stored (no re-test).  Larger AABBs are listed and tested by emit_big_kernel.
#define HUGE_AREA 1024  // AABBs above this many tiles are tested by a whole CTA

// position of the k-th (0-based) set bit of m; m has more than k set bits
__device__ __forceinline__ int nth_set_bit(uint32_t m, int k) {
    int pos = 0;
#pragma unroll
    for (int w = 16; w > 0; w >>= 1) {
        const int c = __popc(m & ((1u << w) - 1u));
        if (k >= c) { k -= c; m >>= w; pos += w; }
    }
    return pos;
}

// `end` bounds the buffers (M, or the capacity); with `total` (capped form) the slots [min(*total, end), end) get the
// padding key, which sorts behind every tile
__global__ void __launch_bounds__(256)
emit_keys_kernel(int N, int tiles_x, const ushort4* __restrict__ tile_bbox, const uint32_t* __restrict__ touch_mask,
                 const int32_t* __restrict__ order, const int32_t* __restrict__ cum, int end, const int64_t* __restrict__ total,
                 uint16_t sentinel, uint16_t* __restrict__ keys, int32_t* __restrict__ vals, int32_t* __restrict__ big_ranks,
                 unsigned int* __restrict__ big_count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int start = 0, n = 0;
    int32_t payload = 0;
    if (i < N) {
        const int c = cum[i];
        start = i > 0 ? cum[i - 1] : 0;
        n = c - start;
        payload = order[i];
    }
    if (start >= end) n = 0;  // truncated (capped form): the run lies past the buffers
    // invisible rows come last in depth order and reach no tile: a warp of them has nothing to emit
    if (__ballot_sync(0xffffffffu, n > 0)) {
        const int row = payload & 0x7fffffff;
        ushort4 bb = make_ushort4(0, 0, 0, 0);
        uint32_t mask = 0;
        if (n > 0) {
            bb = tile_bbox[row];
            mask = touch_mask[row];
        }
        const int bwid = bb.z - bb.x, area = bwid * (bb.w - bb.y);
        const int mine = (n > 0 && area <= COOP_AREA) ? __popc(mask) : 0;
        int pre = mine;  // inclusive scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
        }
        const int flat = __shfl_sync(0xffffffffu, pre, 31);
        pre -= mine;  // exclusive
        const int delta = start - pre;  // entry f of this lane's run goes to f + delta
        const int tbase = bb.y * tiles_x + bb.x;
        for (int base = 0; base < flat; base += 32) {
            const int f = base + lane;
            int o = 0;
#pragma unroll
            for (int step = 16; step > 0; step >>= 1) {
                const int cand = o + step;  // <= 31
                const int pc = __shfl_sync(0xffffffffu, pre, cand);
                if (pc <= f) o = cand;
            }
            const int k = f - __shfl_sync(0xffffffffu, pre, o);
            const uint32_t m = __shfl_sync(0xffffffffu, mask, o);
            const int w = __shfl_sync(0xffffffffu, bwid, o);
            const int tb = __shfl_sync(0xffffffffu, tbase, o);
            const int pos = f + __shfl_sync(0xffffffffu, delta, o);
            const int32_t pl = __shfl_sync(0xffffffffu, payload, o);
            if (f < flat && pos < end) {
                const int bit = nth_set_bit(m, k);
                // bit < 32, w in [1, 32]: (bit + 0.5) / w lies at least 1/64 from an integer, far beyond the error of the
                // approximate quotient, so the truncation is exact
                const int r = (int)__fdividef((float)bit + 0.5f, (float)w);
                keys[pos] = (uint16_t)(tb + r * tiles_x + (bit - r * w));
                vals[pos] = pl;
            }
        }
        // AABBs above COOP_AREA tiles go to lists the whole grid works through (emit_big_kernel): the nearest, widest
        // Gaussians come first in depth order, and one warp testing all of them would serialise the kernel's tail.  Runs
        // up to HUGE_AREA tiles are counted from the front of big_ranks, larger ones from the back (each listed run has an
        // entry below `end`, so the two never meet)
        const unsigned big = __ballot_sync(0xffffffffu, n > 0 && area > COOP_AREA && area <= HUGE_AREA);
        const unsigned huge = __ballot_sync(0xffffffffu, n > 0 && area > HUGE_AREA);
        if (big) {
            int at = 0;
            if (lane == 0) at = (int)atomicAdd(&big_count[0], (unsigned)__popc(big));
            at = __shfl_sync(0xffffffffu, at, 0);
            if ((big >> lane) & 1u) big_ranks[at + __popc(big & ((1u << lane) - 1u))] = i;
        }
        if (huge) {
            int at = 0;
            if (lane == 0) at = (int)atomicAdd(&big_count[1], (unsigned)__popc(huge));
            at = __shfl_sync(0xffffffffu, at, 0);
            if ((huge >> lane) & 1u) big_ranks[end - 1 - (at + __popc(huge & ((1u << lane) - 1u)))] = i;
        }
    }
    if (total) {
        const int64_t m = min(*total, (int64_t)end);
        for (int64_t j = m + i; j < end; j += (int64_t)gridDim.x * blockDim.x) {
            keys[j] = sentinel;
            vals[j] = 0;
        }
    }
}

// The runs of the AABBs above COOP_AREA tiles.  The tiles of an AABB are tested in row-major steps, the reached ones written
// contiguously from the run's start, so a run is a serial chain of steps: runs above HUGE_AREA tiles are taken by whole CTAs
// (EMIT_BIG_THREADS tiles per step), the others by single warps (32 tiles per step), the CTAs / warps of the grid taking the
// listed ranks in turn.
#define EMIT_BIG_THREADS 256

struct BigRun {
    TouchCtx c;
    int32_t pl;
    int x0, y0, wd, ar, pos;
};

__device__ __forceinline__ BigRun big_run(int i, const float4* __restrict__ records, const ushort4* __restrict__ tile_bbox,
                                          const int32_t* __restrict__ order, const int32_t* __restrict__ cum) {
    BigRun r;
    r.pl = order[i];
    const int row = r.pl & 0x7fffffff;
    const ushort4 bb = tile_bbox[row];
    r.c = make_touch_ctx(records[3 * (size_t)row], records[3 * (size_t)row + 1]);
    r.x0 = bb.x; r.y0 = bb.y; r.wd = bb.z - bb.x; r.ar = r.wd * (bb.w - bb.y);
    r.pos = i > 0 ? cum[i - 1] : 0;
    return r;
}

__global__ void __launch_bounds__(EMIT_BIG_THREADS)
emit_big_kernel(int tiles_x, int width, int height, int bw, const float4* __restrict__ records, const ushort4* __restrict__ tile_bbox,
                const int32_t* __restrict__ order, const int32_t* __restrict__ cum, int end, const int32_t* __restrict__ big_ranks,
                const unsigned int* __restrict__ big_count, uint16_t* __restrict__ keys, int32_t* __restrict__ vals) {
    constexpr int WARPS = EMIT_BIG_THREADS / 32;
    __shared__ int warp_hits[2][WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    // runs above HUGE_AREA tiles: a CTA per run
    const int huge = (int)big_count[1];
    int buf = 0;
    for (int h = blockIdx.x; h < huge; h += gridDim.x) {
        BigRun r = big_run(big_ranks[end - 1 - h], records, tile_bbox, order, cum);
        for (int b = 0; b < r.ar && r.pos < end; b += EMIT_BIG_THREADS) {
            const int ti = b + threadIdx.x;
            const int tx = r.x0 + ti % r.wd, ty = r.y0 + ti / r.wd;
            const bool ok = (ti < r.ar) && tile_touched(r.c, tx, ty, width, height, bw);
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) warp_hits[buf][warp] = __popc(bal);
            __syncthreads();  // one barrier per step: the counts alternate between two buffers
            int before = 0, all = 0;
#pragma unroll
            for (int k = 0; k < WARPS; ++k) {
                const int c = warp_hits[buf][k];
                before += k < warp ? c : 0;
                all += c;
            }
            const int my = r.pos + before + __popc(bal & lt);
            if (ok && my < end) {
                keys[my] = (uint16_t)(ty * tiles_x + tx);
                vals[my] = r.pl;
            }
            r.pos += all;
            buf ^= 1;
        }
    }
    // the others: a warp per run
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int count = (int)big_count[0];
    for (int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < count; w += warps) {
        BigRun r = big_run(big_ranks[w], records, tile_bbox, order, cum);
        for (int b = 0; b < r.ar && r.pos < end; b += 32) {
            const int ti = b + lane;
            const int tx = r.x0 + ti % r.wd, ty = r.y0 + ti / r.wd;
            const bool ok = (ti < r.ar) && tile_touched(r.c, tx, ty, width, height, bw);
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            const int my = r.pos + __popc(bal & lt);
            if (ok && my < end) {
                keys[my] = (uint16_t)(ty * tiles_x + tx);
                vals[my] = r.pl;
            }
            r.pos += __popc(bal);
        }
    }
}

__global__ void __launch_bounds__(256)
bin_edges_kernel(int64_t M, const uint16_t* __restrict__ keys_sorted, int32_t* __restrict__ tile_bins) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    const int32_t cur = (int32_t)keys_sorted[i];
    if (i == 0) tile_bins[2 * cur] = 0;
    else {
        const int32_t prev = (int32_t)keys_sorted[i - 1];
        if (prev != cur) {
            tile_bins[2 * prev + 1] = (int32_t)i;
            tile_bins[2 * cur] = (int32_t)i;
        }
    }
    if (i == M - 1) tile_bins[2 * cur + 1] = (int32_t)M;
}

// capacity-bounded form: the number of entries stays on the device (no host read-back between the scan and the sort)
__global__ void __launch_bounds__(256)
bin_edges_capped_kernel(int64_t cap, const int64_t* __restrict__ total, const uint16_t* __restrict__ keys_sorted, int32_t* __restrict__ tile_bins,
                        int32_t* __restrict__ overflow) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t M = min(*total, cap);
    if (i == 0 && *total > cap) *overflow = 1;  // the lists of this frame are truncated: the host finds out with the next frame
    if (i >= M) return;
    const int32_t cur = (int32_t)keys_sorted[i];
    if (i == 0) tile_bins[2 * cur] = 0;
    else {
        const int32_t prev = (int32_t)keys_sorted[i - 1];
        if (prev != cur) {
            tile_bins[2 * prev + 1] = (int32_t)i;
            tile_bins[2 * cur] = (int32_t)i;
        }
    }
    if (i == M - 1) tile_bins[2 * cur + 1] = (int32_t)M;
}

struct SortLayout {
    size_t keys_in, keys_out, vals_in, big, temp, temp_bytes, total;
};

static SortLayout sort_layout(int64_t M) {
    SortLayout L;
    const size_t m = (size_t)(M > 0 ? M : 1);
    size_t temp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp, (const uint16_t*)nullptr, (uint16_t*)nullptr, (const int32_t*)nullptr,
                                    (int32_t*)nullptr, (int64_t)m, 0, 16);
    L.keys_in = 0;
    L.keys_out = align_up(L.keys_in + m * 2, 256);
    L.vals_in = align_up(L.keys_out + m * 2, 256);
    L.big = align_up(L.vals_in + m * 4, 256);  // two counts (256 B), then the ranks of the runs above COOP_AREA tiles (each has an entry)
    L.temp = align_up(L.big + 256 + m * 4, 256);
    L.temp_bytes = temp;
    L.total = align_up(L.temp + temp, 256);
    return L;
}

extern "C" size_t sgn_bin_sort_scratch_bytes(int64_t M) { return sort_layout(M).total; }

static int bin_sort_impl(int N, int64_t M, const int64_t* total_dev, int32_t* overflow_dev, const sgn_camera* cam, const float* records,
                         const int32_t* radii, const uint16_t* tile_bbox, const uint32_t* touch_mask, const int32_t* order, const int32_t* cum,
                         int32_t* sorted_ids, int32_t* tile_bins, void* scratch, size_t scratch_bytes, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(cam && records && radii && tile_bbox && touch_mask && order && cum && tile_bins && scratch,
                "sgn_bin_sort: null pointer");
    SGN_REQUIRE(M >= 0 && M < ((int64_t)1 << 31), "sgn_bin_sort: M=%lld out of the int32 range gsplat's cum_tiles_hit supports", (long long)M);
    const int bw = cam->block_width;
    const int tiles_x = (cam->width + bw - 1) / bw, tiles_y = (cam->height + bw - 1) / bw;
    const int tiles = tiles_x * tiles_y;
    SGN_REQUIRE(tiles <= 65536, "sgn_bin_sort: more than 65536 tiles (16-bit tile keys)");
    SGN_CHECK_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)tiles, stream));
    if (M == 0 || N == 0) return SGN_OK;
    SGN_REQUIRE(sorted_ids, "sgn_bin_sort: sorted_ids is null");
    SGN_REQUIRE(!total_dev || overflow_dev, "sgn_bin_sort_capped: overflow flag is null");
    const SortLayout L = sort_layout(M);
    if (scratch_bytes < L.total) {
        sgn_set_error("sgn_bin_sort: scratch too small (%zu < %zu)", scratch_bytes, L.total);
        return SGN_ERR_WORKSPACE;
    }
    char* base = (char*)scratch;
    uint16_t* keys_in = (uint16_t*)(base + L.keys_in);
    uint16_t* keys_out = (uint16_t*)(base + L.keys_out);
    int32_t* vals_in = (int32_t*)(base + L.vals_in);
    unsigned int* big_count = (unsigned int*)(base + L.big);
    int32_t* big_ranks = (int32_t*)(base + L.big + 256);
    SGN_CHECK_CUDA(cudaMemsetAsync(big_count, 0, 2 * sizeof(unsigned int), stream));
    int tile_bits = 1;
    while ((1 << tile_bits) < tiles + (total_dev ? 1 : 0)) ++tile_bits;  // capped: one more key value, the padding sentinel
    SGN_REQUIRE(!total_dev || tile_bits <= 16, "sgn_bin_sort_capped: %d tiles leave no 16-bit key for the padding", tiles);
    emit_keys_kernel<<<(N + 255) / 256, 256, 0, stream>>>(N, tiles_x, reinterpret_cast<const ushort4*>(tile_bbox), touch_mask, order, cum, (int)M,
                                                          total_dev, (uint16_t)((1u << tile_bits) - 1u), keys_in, vals_in, big_ranks,
                                                          big_count);
    SGN_CHECK_LAUNCH("emit_keys_kernel");
    int sms = 0, dev = 0;
    SGN_CHECK_CUDA(cudaGetDevice(&dev));
    SGN_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    emit_big_kernel<<<4 * sms, EMIT_BIG_THREADS, 0, stream>>>(tiles_x, cam->width, cam->height, bw, reinterpret_cast<const float4*>(records),
                                                 reinterpret_cast<const ushort4*>(tile_bbox), order, cum, (int)M, big_ranks, big_count,
                                                 keys_in, vals_in);
    SGN_CHECK_LAUNCH("emit_big_kernel");
    size_t temp = L.temp_bytes;
    SGN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(base + L.temp, temp, keys_in, keys_out, vals_in, sorted_ids, M, 0, tile_bits, stream));
    sgn_count_launch(1);
    if (total_dev) {
        bin_edges_capped_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(M, total_dev, keys_out, tile_bins, overflow_dev);
        SGN_CHECK_LAUNCH("bin_edges_capped_kernel");
    } else {
        bin_edges_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(M, keys_out, tile_bins);
        SGN_CHECK_LAUNCH("bin_edges_kernel");
    }
    return SGN_OK;
}

extern "C" int sgn_bin_sort(int N, int64_t M, const sgn_camera* cam, const float* records, const int32_t* radii,
                            const uint16_t* tile_bbox, const uint32_t* touch_mask, const int32_t* order, const int32_t* cum,
                            int32_t* sorted_ids, int32_t* tile_bins, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_bin_sort");
    return bin_sort_impl(N, M, nullptr, nullptr, cam, records, radii, tile_bbox, touch_mask, order, cum, sorted_ids, tile_bins, scratch,
                         scratch_bytes, stream_);
}

extern "C" int sgn_bin_sort_capped(int N, int64_t capacity, const int64_t* total_dev, int32_t* overflow_dev, const sgn_camera* cam,
                                   const float* records, const int32_t* radii, const uint16_t* tile_bbox, const uint32_t* touch_mask,
                                   const int32_t* order, const int32_t* cum, int32_t* sorted_ids, int32_t* tile_bins, void* scratch,
                                   size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_bin_sort_capped");
    SGN_REQUIRE(total_dev && capacity > 0, "sgn_bin_sort_capped: needs the device-side entry count and a positive capacity");
    return bin_sort_impl(N, capacity, total_dev, overflow_dev, cam, records, radii, tile_bbox, touch_mask, order, cum, sorted_ids, tile_bins,
                         scratch, scratch_bytes, stream_);
}

// ------------------------------------------------------------------------------------------------
// per-tile class sub-lists: stable partition of every tile's list into its object entries and its
// background entries.  The objects-only / background-only accumulation renders of the reference
// (get_submodel_output, scene graph :255-303,364-366) see exactly these entries in exactly this order.
// Layout: class c (0 = background, 1 = object) owns cls_ids[c*M ...) and cls_bins[c][tiles][2]; class c of tile t starts
// at the number of class-c entries in tiles 0..t-1 (also when the tile is empty).
// One launch: a warp per tile, tiles taken in order through a ticket, so every tile a warp looks back at already belongs to a
// running warp.  The warp counts its object entries with ballots, publishes the (background, object) pair, finds the sum over
// the earlier tiles by decoupled look-back, then writes both sub-lists at ballot / popc positions.
// Tile state: flag (bits 62-63: 0 = not yet, 1 = this tile's counts, 2 = inclusive over tiles 0..t) | background << 31 | object;
// both counts are below 2^31.
#define CLS_AGG 1ull
#define CLS_INC 2ull
#define CLS_CHUNK 16  // list entries per lane per step (loads in flight: a long tile list is one warp's serial chain)

__device__ __forceinline__ unsigned long long cls_pack(unsigned long long flag, int bg, int obj) {
    return (flag << 62) | ((unsigned long long)bg << 31) | (unsigned long long)obj;
}

__global__ void __launch_bounds__(256)
class_lists_kernel(int tiles, int64_t M, const int2* __restrict__ tile_bins, const int32_t* __restrict__ sorted_ids,
                   unsigned long long* __restrict__ state, unsigned int* __restrict__ ticket, int32_t* __restrict__ cls_ids,
                   int2* __restrict__ cls_bins) {
    const int lane = threadIdx.x & 31;
    int t = 0;
    if (lane == 0) t = (int)atomicAdd(ticket, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= tiles) return;
    const int2 range = tile_bins[t];
    const unsigned lt = (1u << lane) - 1u;
    int obj = 0;
    for (int k0 = range.x; k0 < range.y; k0 += 32 * CLS_CHUNK) {
        int32_t id[CLS_CHUNK];
#pragma unroll
        for (int j = 0; j < CLS_CHUNK; ++j) {
            const int k = k0 + 32 * j + lane;
            id[j] = k < range.y ? sorted_ids[k] : 0;
        }
#pragma unroll
        for (int j = 0; j < CLS_CHUNK; ++j) obj += __popc(__ballot_sync(0xffffffffu, id[j] < 0));
    }
    const int bg = (range.y - range.x) - obj;
    volatile unsigned long long* vs = state;
    int bg0 = 0, obj0 = 0;  // exclusive prefix over tiles 0..t-1
    if (t == 0) {
        if (lane == 0) vs[0] = cls_pack(CLS_INC, bg, obj);
    } else {
        if (lane == 0) vs[t] = cls_pack(CLS_AGG, bg, obj);
        // look back 32 tiles at a time: lane j reads tile w - j
        for (int w = t - 1; ; w -= 32) {
            unsigned long long s;
            do {
                s = w - lane >= 0 ? vs[w - lane] : cls_pack(CLS_INC, 0, 0);
            } while (__any_sync(0xffffffffu, (s >> 62) == 0));
            const unsigned inc = __ballot_sync(0xffffffffu, (s >> 62) == CLS_INC);
            const int stop = inc ? __ffs(inc) - 1 : 31;  // the nearest inclusive value ends the look-back
            int b = lane <= stop ? (int)((s >> 31) & 0x7fffffffu) : 0;
            int o = lane <= stop ? (int)(s & 0x7fffffffu) : 0;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                b += __shfl_xor_sync(0xffffffffu, b, d);
                o += __shfl_xor_sync(0xffffffffu, o, d);
            }
            bg0 += b;
            obj0 += o;
            if (inc) break;
        }
        if (lane == 0) vs[t] = cls_pack(CLS_INC, bg0 + bg, obj0 + obj);
    }
    if (lane == 0) {
        cls_bins[t] = make_int2(bg0, bg0 + bg);
        cls_bins[tiles + t] = make_int2(obj0, obj0 + obj);
    }
    int32_t* bg_out = cls_ids + bg0;
    int32_t* obj_out = cls_ids + M + obj0;
    for (int k0 = range.x; k0 < range.y; k0 += 32 * CLS_CHUNK) {
        int32_t id[CLS_CHUNK];
#pragma unroll
        for (int j = 0; j < CLS_CHUNK; ++j) {
            const int k = k0 + 32 * j + lane;
            id[j] = k < range.y ? sorted_ids[k] : 0;
        }
#pragma unroll
        for (int j = 0; j < CLS_CHUNK; ++j) {
            const bool in = k0 + 32 * j + lane < range.y;
            const unsigned ob = __ballot_sync(0xffffffffu, in && id[j] < 0);
            const unsigned valid = __ballot_sync(0xffffffffu, in);
            if (in) {
                if (id[j] < 0) obj_out[__popc(ob & lt)] = id[j];
                else bg_out[__popc(valid & ~ob & lt)] = id[j];
            }
            obj_out += __popc(ob);
            bg_out += __popc(valid & ~ob);
        }
    }
}

// tile state, then the ticket counter
extern "C" size_t sgn_bin_class_scratch_bytes(int tiles) {
    return align_up(sizeof(unsigned long long) * (size_t)(tiles > 0 ? tiles : 1), 256) + 256;
}

extern "C" int sgn_bin_class_lists(const sgn_camera* cam, int64_t M, const int32_t* sorted_ids, const int32_t* tile_bins,
                                   int32_t* cls_ids, int32_t* cls_bins, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_bin_class_lists");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(cam && tile_bins && cls_ids && cls_bins && scratch, "sgn_bin_class_lists: null pointer");
    SGN_REQUIRE(M >= 0 && M < ((int64_t)1 << 31), "sgn_bin_class_lists: M=%lld out of the int32 range", (long long)M);
    const int bw = cam->block_width;
    const int tiles = ((cam->width + bw - 1) / bw) * ((cam->height + bw - 1) / bw);
    const size_t bytes = sgn_bin_class_scratch_bytes(tiles);
    if (scratch_bytes < bytes) {
        sgn_set_error("sgn_bin_class_lists: scratch too small");
        return SGN_ERR_WORKSPACE;
    }
    if (tiles == 0) return SGN_OK;
    char* base = (char*)scratch;
    unsigned long long* state = (unsigned long long*)base;
    unsigned int* ticket = (unsigned int*)(base + bytes - 256);
    SGN_CHECK_CUDA(cudaMemsetAsync(scratch, 0, bytes, stream));
    class_lists_kernel<<<(tiles + 7) / 8, 256, 0, stream>>>(tiles, M, reinterpret_cast<const int2*>(tile_bins), sorted_ids, state, ticket,
                                                            cls_ids, reinterpret_cast<int2*>(cls_bins));
    SGN_CHECK_LAUNCH("class_lists_kernel");
    return SGN_OK;
}
