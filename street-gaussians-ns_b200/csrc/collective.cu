// Gradient exchange of the camera-sharded data-parallel step (SURVEY.md 8e) as this library's own kernels over
// peer-mapped ("symmetric") memory, instead of a library all-reduce behind the step:
//
//   * every rank's flat gradient arena lives in a symmetric allocation (torch.distributed._symmetric_memory: the same
//     virtual layout on every GPU, peer pointers and -- behind an NVSwitch -- one multicast address for all replicas);
//   * a two-shot all-reduce in ONE kernel: rank r owns the r-th part of every slice; it pulls the SUM of that part
//       - with `multimem.ld_reduce` through the multicast address (the reduction happens INSIDE the switch: each GPU sends
//         each element once, NVLS), or
//       - without multicast: plain loads from every peer's arena over NVLink, summed in rank order,
//     scales it (1/world for the mean), and pushes the result to every replica (`multimem.st`, or one store per peer);
//   * the call takes a LIST of slices, so the exchange runs range by range behind the project backward that produces the
//     arena (dp.SymmetricExchange.exchange_ranges): the slices of rows [r0, r1) of a sub-model are reduced while the next
//     row range is still being written, and the fused Adam (adam.cu) follows range by range.
//
// Synchronisation between GPUs (all ranks have WRITTEN the slices before anyone reduces; all ranks have PUSHED before anyone
// reads the result) is the caller's: two device-side barriers on the symmetric-memory signal pads, issued on the same stream
// (dp.SymmetricExchange).  The wire floor of this pattern is ~S bytes per GPU and direction (S = arena size), against
// 2 S (g-1)/g for a ring: 0.37 ms for the 330 MB arena of config 3 at NVLink 5's 900 GB/s.
#include "sgn_common.cuh"

#define AR_THREADS 512

__device__ __forceinline__ float4 mc_ld_reduce(const float4* mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mc_st(float4* mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

struct ArSlices {
    int n;
    int64_t off4[SGN_AR_MAX_SLICES];  // slice start, in float4 units from the arena base
    int64_t len4[SGN_AR_MAX_SLICES];  // slice length, float4 units
    int32_t width[SGN_AR_MAX_SLICES]; // > 0: the slice holds rows of `width` floats whose visibility is known (row skipping)
    int64_t row0[SGN_AR_MAX_SLICES];  // index of the slice's first row in the visibility array
    int64_t nrows[SGN_AR_MAX_SLICES]; // rows in the slice (floats behind nrows * width are padding)
};

// this rank's part of a slice: [begin, end) in float4 units
__device__ __forceinline__ void my_part(int64_t len4, int rank, int world, int64_t& b, int64_t& e) {
    const int64_t per = (len4 + world - 1) / world;
    b = min(len4, per * rank);
    e = min(len4, b + per);
}

// Rows no replica saw (radius 0 in every rank's frame) have an all-zero gradient in every replica's arena -- project_bwd
// writes zeros there -- so their sum is what is already stored: they are not exchanged.  In a street scene a camera sees
// about half of the background Gaussians and neighbouring cameras see mostly the same half.
__global__ void __launch_bounds__(256)
visible_union_kernel(const uint64_t* __restrict__ peers, int64_t flags_byte_offset, int world, int64_t n, uint8_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t u = 0;
    for (int p = 0; p < world; ++p) u |= reinterpret_cast<const uint8_t*>(peers[p] + flags_byte_offset)[i];
    out[i] = u;
}
__global__ void __launch_bounds__(256)
visible_flags_kernel(const int32_t* __restrict__ radii, int64_t n, uint8_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = radii[i] > 0 ? 1 : 0;
}

__device__ __forceinline__ bool rows_unseen(const ArSlices& sl, int s, const uint8_t* __restrict__ vis, int64_t i) {
    // float4 i of the slice covers floats [4i, 4i+3]: rows (4i)/w .. (4i+3)/w (one or two rows for w >= 4, up to four for w = 1).
    // 32-bit arithmetic: a slice holds fewer than 2^31 floats (64-bit divisions made this test cost as much as it saved).
    const unsigned w = (unsigned)sl.width[s];
    const unsigned f0 = (unsigned)(4 * i), rows = (unsigned)sl.nrows[s];
    const unsigned ra = f0 / w;
    if (ra >= rows) return true;  // padding behind the last row: zeros on every replica
    const unsigned rem = f0 - ra * w;
    const unsigned more = w >= 4 ? (rem + 3 >= w ? 1u : 0u) : (rem + 3) / w;
    const unsigned rb = min(ra + more, rows - 1);
    const uint8_t* v = vis + sl.row0[s];
    uint8_t seen = v[ra];
    for (unsigned r = ra + 1; r <= rb; ++r) seen |= v[r];
    return !seen;
}

template <bool MC>
__global__ void __launch_bounds__(AR_THREADS)
allreduce_sym_kernel(float4* __restrict__ local, float4* __restrict__ mc, const uint64_t* __restrict__ peers, int rank, int world,
                     const ArSlices sl, float scale, const uint8_t* __restrict__ vis) {
    for (int s = 0; s < sl.n; ++s) {
        int64_t b, e;
        my_part(sl.len4[s], rank, world, b, e);
        const int64_t base = sl.off4[s];
        const bool skipping = vis && sl.width[s] > 0;
        // UNROLL independent requests per thread in flight: a pull through the switch has a multi-microsecond latency, and
        // 900 GB/s x that latency must be covered by outstanding 16-byte requests
        constexpr int UNROLL = 4;
        const int64_t stride = (int64_t)gridDim.x * AR_THREADS;
        for (int64_t i0 = b + (int64_t)blockIdx.x * AR_THREADS + threadIdx.x; i0 < e; i0 += stride * UNROLL) {
            float4 v[UNROLL];
            bool live[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const int64_t i = i0 + u * stride;
                live[u] = i < e && !(skipping && rows_unseen(sl, s, vis, i));
                if (!live[u]) { v[u] = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
                if (MC) {
                    v[u] = mc_ld_reduce(mc + base + i);
                } else {
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                    for (int p = 0; p < world; ++p) {  // rank order: one rank computes each element, every replica gets the same bits
                        const float4 x = __ldcg(reinterpret_cast<const float4*>(peers[p]) + base + i);
                        acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
                    }
                    v[u] = acc;
                }
            }
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const int64_t i = i0 + u * stride;
                if (!live[u]) continue;
                const float4 r = make_float4(v[u].x * scale, v[u].y * scale, v[u].z * scale, v[u].w * scale);
                if (MC) {
                    mc_st(mc + base + i, r);
                } else {
                    for (int p = 0; p < world; ++p) __stcg(reinterpret_cast<float4*>(peers[p]) + base + i, r);
                }
            }
        }
    }
    (void)local;
}

extern "C" int sgn_visible_flags(const int32_t* radii, int64_t n, uint8_t* flags, void* stream) {
    SGN_RANGE("sgn_visible_flags");
    SGN_REQUIRE(radii && flags && n >= 0, "sgn_visible_flags: null pointer");
    if (n == 0) return SGN_OK;
    visible_flags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(radii, n, flags);
    SGN_CHECK_LAUNCH("visible_flags_kernel");
    return SGN_OK;
}

extern "C" int sgn_visible_union(const uint64_t* peer_ptrs_dev, int64_t flags_byte_offset, int world, int64_t n, uint8_t* out, void* stream) {
    SGN_RANGE("sgn_visible_union");
    SGN_REQUIRE(peer_ptrs_dev && out && world >= 1 && n >= 0, "sgn_visible_union: bad argument");
    if (n == 0) return SGN_OK;
    visible_union_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(peer_ptrs_dev, flags_byte_offset, world, n, out);
    SGN_CHECK_LAUNCH("visible_union_kernel");
    return SGN_OK;
}

extern "C" int sgn_allreduce_sym(void* local, void* multicast, const uint64_t* peer_ptrs_dev, int rank, int world, int nslices,
                                 const int64_t* slice_offsets, const int64_t* slice_lengths, const int32_t* slice_widths,
                                 const int64_t* slice_row0, const int64_t* slice_rows, const uint8_t* visible_union, float scale,
                                 int max_ctas, void* stream) {
    SGN_RANGE("sgn_allreduce_sym");
    SGN_REQUIRE(local && (multicast || peer_ptrs_dev), "sgn_allreduce_sym: needs the multicast address or the peer pointer table");
    SGN_REQUIRE(world >= 1 && rank >= 0 && rank < world, "sgn_allreduce_sym: rank %d of %d", rank, world);
    SGN_REQUIRE(nslices >= 0 && nslices <= SGN_AR_MAX_SLICES, "sgn_allreduce_sym: %d slices (at most %d per call)", nslices, SGN_AR_MAX_SLICES);
    SGN_REQUIRE(sgn_aligned16(local) && sgn_aligned16(multicast), "sgn_allreduce_sym: the arena must be 16-byte aligned");
    SGN_REQUIRE(!visible_union || (slice_widths && slice_row0 && slice_rows), "sgn_allreduce_sym: row skipping needs slice_widths, slice_row0 and slice_rows");
    if (nslices == 0) return SGN_OK;
    SGN_REQUIRE(slice_offsets && slice_lengths, "sgn_allreduce_sym: null slice table");
    ArSlices sl;
    sl.n = nslices;
    int64_t total4 = 0;
    for (int s = 0; s < nslices; ++s) {
        SGN_REQUIRE(slice_offsets[s] >= 0 && slice_lengths[s] >= 0 && slice_offsets[s] % 4 == 0 && slice_lengths[s] % 4 == 0,
                    "sgn_allreduce_sym: slice %d (offset %lld, length %lld floats) is not a run of 16-byte units", s,
                    (long long)slice_offsets[s], (long long)slice_lengths[s]);
        sl.off4[s] = slice_offsets[s] / 4;
        sl.len4[s] = slice_lengths[s] / 4;
        sl.width[s] = (visible_union && slice_widths) ? slice_widths[s] : 0;
        sl.row0[s] = (visible_union && slice_row0) ? slice_row0[s] : 0;
        sl.nrows[s] = (visible_union && slice_rows) ? slice_rows[s] : 0;
        SGN_REQUIRE(sl.width[s] >= 0 && sl.width[s] <= 4096 && sl.row0[s] >= 0 && sl.nrows[s] >= 0 &&
                        sl.nrows[s] * (int64_t)sl.width[s] <= slice_lengths[s],
                    "sgn_allreduce_sym: slice %d has a bad row description", s);
        // rows_unseen indexes a row-skipping slice with 32-bit arithmetic
        SGN_REQUIRE(sl.width[s] == 0 || slice_lengths[s] < ((int64_t)1 << 31),
                    "sgn_allreduce_sym: row-skipping slice %d has %lld floats (at most 2^31 - 1)", s, (long long)slice_lengths[s]);
        total4 += sl.len4[s];
    }
    if (total4 == 0) return SGN_OK;
    const int64_t mine = (total4 + world - 1) / world;
    int ctas = (int)((mine + AR_THREADS * 4 - 1) / (AR_THREADS * 4));  // >= 4 float4 per thread
    ctas = ctas < 1 ? 1 : ctas;
    const int cap = max_ctas > 0 ? max_ctas : 132 * 2;  // two CTAs per SM of an H100 SXM
    if (ctas > cap) ctas = cap;
    if (multicast)
        allreduce_sym_kernel<true><<<ctas, AR_THREADS, 0, (cudaStream_t)stream>>>((float4*)local, (float4*)multicast, peer_ptrs_dev, rank, world, sl, scale,
                                                                                   visible_union);
    else
        allreduce_sym_kernel<false><<<ctas, AR_THREADS, 0, (cudaStream_t)stream>>>((float4*)local, nullptr, peer_ptrs_dev, rank, world, sl, scale,
                                                                                    visible_union);
    SGN_CHECK_LAUNCH("allreduce_sym_kernel");
    return SGN_OK;
}
