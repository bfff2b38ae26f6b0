// Exact k-nearest-neighbour search (1 <= k <= 16): the initial scales of SplatfactoModel.populate_modules
// (street_gaussians_ns/sgn_splatfacto.py:260-264, which runs sklearn's NearestNeighbors on the CPU) and the lidar chamfer
// distance (data/utils/geometric_metric.py:59-69, open3d on the CPU).
//
// Shape: a bounding-box reduction; 63-bit Morton keys (21 bits per axis, one isotropic cell size over the box); a CUB radix
// sort of (key, row); the sorted points grouped into leaves of KNN_LEAF and an implicit complete binary tree of axis-aligned
// boxes over the leaves (heap layout, one launch per level); then one thread per query, in Morton order, walking the tree
// depth first, nearer child first, and pruning every subtree whose box is farther than the current k-th best.  The tree
// adapts to the cloud (a dense ground slab, sparse volume and far outliers alike): the search is exact for every point with
// no cap on how far it looks.
//
// Exactness in fp32: a point's squared distance is ((dx*dx + dy*dy) + dz*dz) with each difference, product and sum rounded
// once (explicit _rn intrinsics, no contraction).  A box's squared distance is the same expression over the per-axis gaps
// max(lo - q, q - hi, 0); every operation in it is monotone, so it never exceeds the computed distance of a point inside
// the box and pruning drops no candidate.  Candidates are ordered by (squared distance, row): the smaller row wins a tie,
// and a subtree is also skipped when its box distance equals the k-th best but its smallest row is larger.  The result is
// independent of the visiting order, so it is deterministic; no atomics feed it (the box reduction uses integer min / max).
#include <cub/cub.cuh>

#include "sgn_common.cuh"

#define KNN_LEAF 16
#define KNN_THREADS 128
#define KNN_STACK 32  // > tree depth: log2(2^31 / KNN_LEAF) + 1
#define KNN_MAX_K 16

static inline size_t knn_align(size_t x) { return (x + 255) & ~(size_t)255; }

// float <-> int with the order of the floats (for integer atomic min / max)
__device__ __forceinline__ int ord_of(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float float_of(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__device__ __forceinline__ float sq3(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ bool before(float d, int i, float bd, int bi) { return d < bd || (d == bd && i < bi); }

__global__ void knn_box_init_kernel(int* box) {
    if (threadIdx.x < 3) box[threadIdx.x] = ord_of(__int_as_float(0x7f800000));       // +inf
    else if (threadIdx.x < 6) box[threadIdx.x] = ord_of(__int_as_float(0xff800000)); // -inf
}

__global__ void __launch_bounds__(256) knn_box_kernel(const float* __restrict__ pts, long long n, int* __restrict__ box) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(box + a, ord_of(lo[a]));
            atomicMax(box + 3 + a, ord_of(hi[a]));
        }
    }
}

__device__ __forceinline__ unsigned long long spread21(unsigned int v) {
    unsigned long long x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

// Morton key of each row of xyz (queries outside the box are clamped to it: the key only orders the work)
__global__ void __launch_bounds__(256) knn_keys_kernel(const float* __restrict__ xyz, long long n, const int* __restrict__ box,
                                                       unsigned long long* __restrict__ keys, int* __restrict__ rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float lo[3] = {float_of(box[0]), float_of(box[1]), float_of(box[2])};
    const float ext = fmaxf(fmaxf(float_of(box[3]) - lo[0], float_of(box[4]) - lo[1]), float_of(box[5]) - lo[2]);
    const float s = ext > 0.f ? 2097151.0f / ext : 0.f;
    unsigned long long key = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float c = fminf(fmaxf((xyz[3 * i + a] - lo[a]) * s, 0.f), 2097151.0f);
        key |= spread21((unsigned int)c) << a;
    }
    keys[i] = key;
    rows[i] = (int)i;
}

// sorted points (x, y, z, row) and the leaf boxes: lo = (x, y, z, -), hi = (x, y, z, smallest row as int bits)
__global__ void __launch_bounds__(256) knn_leaves_kernel(const float* __restrict__ pts, int n, const int* __restrict__ order,
                                                         int nleaves_pow2, float4* __restrict__ sorted, float4* __restrict__ nodes) {
    const int leaf = blockIdx.x * blockDim.x + threadIdx.x;
    if (leaf >= nleaves_pow2) return;
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    int rmin = 0x7fffffff;
    for (int s = leaf * KNN_LEAF; s < min(n, (leaf + 1) * KNN_LEAF); ++s) {
        const int r = order[s];
        const float x = pts[3 * (long long)r], y = pts[3 * (long long)r + 1], z = pts[3 * (long long)r + 2];
        sorted[s] = make_float4(x, y, z, __int_as_float(r));
        lo.x = fminf(lo.x, x); lo.y = fminf(lo.y, y); lo.z = fminf(lo.z, z);
        hi.x = fmaxf(hi.x, x); hi.y = fmaxf(hi.y, y); hi.z = fmaxf(hi.z, z);
        rmin = min(rmin, r);
    }
    hi.w = __int_as_float(rmin);
    const long long node = (long long)nleaves_pow2 - 1 + leaf;
    nodes[2 * node] = lo;
    nodes[2 * node + 1] = hi;
}

// one level of the tree: node i in [first, first + count) from its children 2i+1, 2i+2
__global__ void __launch_bounds__(256) knn_level_kernel(long long first, long long count, float4* __restrict__ nodes) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const long long i = first + j, l = 2 * i + 1, r = 2 * i + 2;
    const float4 a = nodes[2 * l], b = nodes[2 * l + 1], c = nodes[2 * r], d = nodes[2 * r + 1];
    nodes[2 * i] = make_float4(fminf(a.x, c.x), fminf(a.y, c.y), fminf(a.z, c.z), 0.f);
    nodes[2 * i + 1] = make_float4(fmaxf(b.x, d.x), fmaxf(b.y, d.y), fmaxf(b.z, d.z),
                                   __int_as_float(min(__float_as_int(b.w), __float_as_int(d.w))));
}

__device__ __forceinline__ float box_d2(const float4* __restrict__ nodes, int node, float qx, float qy, float qz, int* rmin) {
    const float4 lo = __ldg(nodes + 2 * (long long)node), hi = __ldg(nodes + 2 * (long long)node + 1);
    *rmin = __float_as_int(hi.w);
    const float gx = fmaxf(fmaxf(__fsub_rn(lo.x, qx), __fsub_rn(qx, hi.x)), 0.f);
    const float gy = fmaxf(fmaxf(__fsub_rn(lo.y, qy), __fsub_rn(qy, hi.y)), 0.f);
    const float gz = fmaxf(fmaxf(__fsub_rn(lo.z, qz), __fsub_rn(qz, hi.z)), 0.f);
    return sq3(gx, gy, gz);  // +inf for an empty (padding) leaf
}

struct KnnParams {
    const float4* sorted;   // [n] points in Morton order, row in .w
    const float4* nodes;    // [2 * (2P - 1)] boxes, heap layout, leaves at P - 1 ..
    int n, P;
    const float* query;     // [m, 3] or null: the points themselves, each excluding its own row
    const int* qorder;      // [m] query rows in Morton order (null without a query set)
    int m;
    float* dist;            // [m, k] or null
    int* idx;               // [m, k] or null
    float* log_scales;      // [m, 3] or null: log(mean of the k distances), broadcast
};

template <int K>
__global__ void __launch_bounds__(KNN_THREADS) knn_query_kernel(const KnnParams p) {
    __shared__ int s_node[KNN_STACK][KNN_THREADS];
    __shared__ float s_d[KNN_STACK][KNN_THREADS];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.m) return;
    int self, out;
    float qx, qy, qz;
    if (p.query) {
        out = p.qorder[t];
        self = -1;
        qx = p.query[3 * (long long)out]; qy = p.query[3 * (long long)out + 1]; qz = p.query[3 * (long long)out + 2];
    } else {
        const float4 q = p.sorted[t];
        qx = q.x; qy = q.y; qz = q.z;
        out = self = __float_as_int(q.w);
    }
    float bd[K];
    int bi[K];
#pragma unroll
    for (int j = 0; j < K; ++j) { bd[j] = INFINITY; bi[j] = 0x7fffffff; }

    int sp = 0, rmin;
    s_node[0][threadIdx.x] = 0;
    s_d[0][threadIdx.x] = box_d2(p.nodes, 0, qx, qy, qz, &rmin);
    sp = 1;
    const int first_leaf = p.P - 1;
    while (sp > 0) {
        --sp;
        int node = s_node[sp][threadIdx.x];
        const float nd = s_d[sp][threadIdx.x];
        if (nd > bd[K - 1]) continue;
        bool alive = true;
        while (node < first_leaf) {
            const int l = 2 * node + 1, r = 2 * node + 2;
            int ml, mr;
            float dl = box_d2(p.nodes, l, qx, qy, qz, &ml), dr = box_d2(p.nodes, r, qx, qy, qz, &mr);
            int nl = l, nr = r;
            if (dr < dl) { const float td = dl; dl = dr; dr = td; const int tn = nl; nl = nr; nr = tn; const int tm = ml; ml = mr; mr = tm; }
            const float w = bd[K - 1];
            const int wi = bi[K - 1];
            if (dr < w || (dr == w && mr < wi)) {
                s_node[sp][threadIdx.x] = nr;
                s_d[sp][threadIdx.x] = dr;
                ++sp;
            }
            if (dl < w || (dl == w && ml < wi)) {
                node = nl;
            } else {
                alive = false;
                break;
            }
        }
        if (!alive) continue;
        const int s0 = (node - first_leaf) * KNN_LEAF, s1 = min(p.n, s0 + KNN_LEAF);
        for (int s = s0; s < s1; ++s) {
            const float4 c = __ldg(p.sorted + s);
            const int row = __float_as_int(c.w);
            if (row == self) continue;
            float cd = sq3(__fsub_rn(c.x, qx), __fsub_rn(c.y, qy), __fsub_rn(c.z, qz));
            int ci = row;
            if (!before(cd, ci, bd[K - 1], bi[K - 1])) continue;
#pragma unroll
            for (int j = 0; j < K; ++j) {
                if (before(cd, ci, bd[j], bi[j])) {
                    const float td = bd[j]; bd[j] = cd; cd = td;
                    const int ti = bi[j]; bi[j] = ci; ci = ti;
                }
            }
        }
    }

    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        const float d = sqrtf(bd[j]);
        sum += d;
        if (p.dist) p.dist[(long long)out * K + j] = d;
        if (p.idx) p.idx[(long long)out * K + j] = bi[j];
    }
    if (p.log_scales) {
        const float ls = logf(sum / (float)K);
        p.log_scales[3 * (long long)out] = ls;
        p.log_scales[3 * (long long)out + 1] = ls;
        p.log_scales[3 * (long long)out + 2] = ls;
    }
}

struct KnnLayout {
    size_t box, keys_in, keys_out, rows_in, order, qorder, sorted, nodes, temp, temp_bytes, total;
    int P;
};

static KnnLayout knn_layout(long long n, long long m) {
    KnnLayout L;
    const long long nl = (n + KNN_LEAF - 1) / KNN_LEAF;
    long long P = 1;
    while (P < nl) P <<= 1;
    L.P = (int)P;
    const size_t kn = (size_t)(n > m ? n : m) + 1;
    size_t temp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const int*)nullptr, (int*)nullptr, (int)kn, 0, 63);
    L.box = 0;
    L.keys_in = knn_align(6 * sizeof(int));
    L.keys_out = L.keys_in + knn_align(kn * 8);
    L.rows_in = L.keys_out + knn_align(kn * 8);
    L.order = L.rows_in + knn_align(kn * 4);
    L.qorder = L.order + knn_align((size_t)(n + 1) * 4);
    L.sorted = L.qorder + knn_align((size_t)(m + 1) * 4);
    L.nodes = L.sorted + knn_align((size_t)(n + 1) * 16);
    L.temp = L.nodes + knn_align((size_t)(2 * P - 1) * 32);
    L.temp_bytes = temp;
    L.total = L.temp + knn_align(temp);
    return L;
}

extern "C" size_t sgn_knn_scratch_bytes(int64_t n, int64_t m) {
    if (n < 0 || m < 0 || n >= 0x7fffffffLL || m >= 0x7fffffffLL) return 0;
    return knn_layout(n, m).total;
}

template <int K>
static int knn_launch(const KnnParams& p, cudaStream_t stream) {
    knn_query_kernel<K><<<(p.m + KNN_THREADS - 1) / KNN_THREADS, KNN_THREADS, 0, stream>>>(p);
    SGN_CHECK_LAUNCH("knn_query_kernel");
    return SGN_OK;
}

extern "C" int sgn_knn(const float* points, int64_t n, const float* query, int64_t m, int k, float* dist, int32_t* idx,
                       float* log_scales, void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_knn");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(k >= 1 && k <= KNN_MAX_K, "sgn_knn: k = %d outside 1..%d", k, KNN_MAX_K);
    SGN_REQUIRE(points && scratch, "sgn_knn: null points or scratch");
    SGN_REQUIRE(dist || idx || log_scales, "sgn_knn: no output (dist, idx and log_scales are all null)");
    SGN_REQUIRE(n >= 0 && n < 0x7fffffffLL, "sgn_knn: n = %lld outside 0..2^31-2", (long long)n);
    if (query) {
        SGN_REQUIRE(m >= 0 && m < 0x7fffffffLL, "sgn_knn: m = %lld outside 0..2^31-2", (long long)m);
        SGN_REQUIRE(n >= k, "sgn_knn: %lld points cannot give %d neighbours", (long long)n, k);
    } else {
        SGN_REQUIRE(n >= k + 1, "sgn_knn: %lld points cannot give %d neighbours other than the point itself", (long long)n, k);
        m = n;
    }
    const KnnLayout L = knn_layout(n, query ? m : 0);
    if (scratch_bytes < L.total) {
        sgn_set_error("sgn_knn: scratch too small (%zu < %zu bytes)", scratch_bytes, L.total);
        return SGN_ERR_WORKSPACE;
    }
    if (m == 0) return SGN_OK;
    char* base = (char*)scratch;
    int* box = (int*)(base + L.box);
    unsigned long long* keys_in = (unsigned long long*)(base + L.keys_in);
    unsigned long long* keys_out = (unsigned long long*)(base + L.keys_out);
    int* rows_in = (int*)(base + L.rows_in);
    int* order = (int*)(base + L.order);
    int* qorder = (int*)(base + L.qorder);
    float4* sorted = (float4*)(base + L.sorted);
    float4* nodes = (float4*)(base + L.nodes);

    knn_box_init_kernel<<<1, 32, 0, stream>>>(box);
    SGN_CHECK_LAUNCH("knn_box_init_kernel");
    const int nb = (int)((n + 255) / 256 < 132 * 8 ? (n + 255) / 256 : 132 * 8);
    knn_box_kernel<<<nb, 256, 0, stream>>>(points, n, box);
    SGN_CHECK_LAUNCH("knn_box_kernel");

    // (key, row) sorts: the points, then the queries
    const float* xyz[2] = {points, query};
    const long long cnt[2] = {n, m};
    int* dst[2] = {order, qorder};
    for (int pass = 0; pass < (query ? 2 : 1); ++pass) {
        knn_keys_kernel<<<(unsigned)((cnt[pass] + 255) / 256), 256, 0, stream>>>(xyz[pass], cnt[pass], box, keys_in, rows_in);
        SGN_CHECK_LAUNCH("knn_keys_kernel");
        size_t temp = L.temp_bytes;
        SGN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(base + L.temp, temp, keys_in, keys_out, rows_in, dst[pass], (int)cnt[pass], 0, 63,
                                                       stream));
        sgn_count_launch(1);
    }

    knn_leaves_kernel<<<(L.P + 255) / 256, 256, 0, stream>>>(points, (int)n, order, L.P, sorted, nodes);
    SGN_CHECK_LAUNCH("knn_leaves_kernel");
    for (long long count = L.P / 2; count >= 1; count /= 2) {
        knn_level_kernel<<<(unsigned)((count + 255) / 256), 256, 0, stream>>>(count - 1, count, nodes);
        SGN_CHECK_LAUNCH("knn_level_kernel");
    }

    KnnParams p;
    p.sorted = sorted; p.nodes = nodes; p.n = (int)n; p.P = L.P;
    p.query = query; p.qorder = query ? qorder : nullptr; p.m = (int)m;
    p.dist = dist; p.idx = idx; p.log_scales = log_scales;
    switch (k) {
        case 1: return knn_launch<1>(p, stream);
        case 2: return knn_launch<2>(p, stream);
        case 3: return knn_launch<3>(p, stream);
        case 4: return knn_launch<4>(p, stream);
        case 5: return knn_launch<5>(p, stream);
        case 6: return knn_launch<6>(p, stream);
        case 7: return knn_launch<7>(p, stream);
        case 8: return knn_launch<8>(p, stream);
        case 9: return knn_launch<9>(p, stream);
        case 10: return knn_launch<10>(p, stream);
        case 11: return knn_launch<11>(p, stream);
        case 12: return knn_launch<12>(p, stream);
        case 13: return knn_launch<13>(p, stream);
        case 14: return knn_launch<14>(p, stream);
        case 15: return knn_launch<15>(p, stream);
        default: return knn_launch<16>(p, stream);
    }
}
