// Densification by MCMC ("3D Gaussian Splatting as Markov Chain Monte Carlo", Kheradmand et al., NeurIPS 2024; gsplat's
// MCMCStrategy): the per-step position noise, the opacity-weighted sampler, the relocation update rule, the row copy and the
// opacity / scale regularisers.  The statements are in include/sgn_raster.h; the test suite restates them in float64.
//
// Random numbers: Philox4x32-10 keyed by the seed, counter (index, step, sub-model, purpose).  Every draw is a function of its
// own counter, so the bits do not depend on the launch shape.
//
// The sampler's prefix sum is fp64 and deterministic: 4096-row tiles (256 threads x 16 consecutive rows), each thread sums its
// rows serially, one thread per block adds the thread sums serially, and one thread adds the tile sums serially.  Serial sums
// keep the prefix non-decreasing bit for bit across thread and tile boundaries (see mcmc_tile_sums_kernel), which is what keeps
// a zero-weight row from ever being drawn.  No float atomics anywhere in this file; the draw counts use integer atomics.
#include "sgn_common.cuh"

#define MC_CHUNK 128        // rows per chunk of the segment tables (sgn_segment.chunk0, sgn_mcmc_sub.chunk0)
#define MC_SCAN_THREADS 256
#define MC_SCAN_ITEMS 16
#define MC_TILE (MC_SCAN_THREADS * MC_SCAN_ITEMS)
#define MC_REG_BLOCKS 1056  // 132 SMs (H100 SXM) x 8 resident blocks
#define MC_MAX_N 51         // gsplat's n_max: counts above 50 are clamped

// ---- Philox4x32-10 ----------------------------------------------------------------------------------------------
struct mc_u4 { uint32_t x, y, z, w; };

__device__ __forceinline__ mc_u4 mc_philox(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return {c0, c1, c2, c3};
}

// ---- helpers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ float mc_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// the last entry whose first chunk is <= c (a zero-row segment shares its chunk0 with the next one)
template <typename S>
__device__ __forceinline__ int mc_segment_of(const S* __restrict__ segs, int nseg, int c) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (segs[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// in place: sh[k] <- sh[0] + ... + sh[k-1] (exclusive), added serially by thread 0; returns the total to every thread.  Serial, so
// that E[k+1] == E[k] + sh[k] holds bit for bit: the prefix of a thread's last row equals the next thread's starting prefix
template <typename T>
__device__ __forceinline__ T mc_block_exclusive(T* sh, int n) {
    __syncthreads();
    if (threadIdx.x == 0) {
        T s = T(0);
        for (int k = 0; k < n; ++k) {
            const T v = sh[k];
            sh[k] = s;
            s += v;
        }
        sh[n] = s;
    }
    __syncthreads();
    const T tot = sh[n];
    return tot;
}

// ---- noise -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MC_CHUNK) mcmc_noise_kernel(const sgn_mcmc_sub* __restrict__ subs, int nsub, float lr, uint64_t seed, int step,
                                                              const float* __restrict__ normals) {
    const int k = mc_segment_of(subs, nsub, (int)blockIdx.x);
    const sgn_mcmc_sub& sb = subs[k];
    const int row = ((int)blockIdx.x - sb.chunk0) * MC_CHUNK + (int)threadIdx.x;
    if (row >= sb.count) return;
    float e0, e1, e2;
    if (normals) {
        const float* e = normals + (size_t)(sb.row0 + row) * 3;
        e0 = e[0]; e1 = e[1]; e2 = e[2];
    } else {  // Box-Muller on two pairs of 24-bit uniforms, u1 in (0, 1]
        const mc_u4 r = mc_philox(seed, (uint32_t)row, (uint32_t)step, (uint32_t)sb.index, SGN_MCMC_NOISE);
        const float u1 = (float)((r.x >> 8) + 1u) * 5.9604645e-8f, u2 = (float)(r.y >> 8) * 5.9604645e-8f;
        const float u3 = (float)((r.z >> 8) + 1u) * 5.9604645e-8f, u4 = (float)(r.w >> 8) * 5.9604645e-8f;
        const float ra = sqrtf(-2.0f * logf(u1)), rb = sqrtf(-2.0f * logf(u3));
        float sa, ca, sb_;
        sincospif(2.0f * u2, &sa, &ca);
        sb_ = sinpif(2.0f * u4);
        e0 = ra * ca; e1 = ra * sa; e2 = rb * sb_;
    }
    const float o = mc_sigmoid(sb.opacities[row]);
    const float gate = 1.0f / (1.0f + expf(-100.0f * ((1.0f - o) - 0.995f)));
    const float g = gate * (lr * sb.noise_lr);
    const float t0 = e0 * g, t1 = e1 * g, t2 = e2 * g;
    const float* qp = sb.quats + (size_t)row * 4;
    float w = qp[0], x = qp[1], y = qp[2], z = qp[3];
    const float inv = 1.0f / fmaxf(sqrtf(w * w + x * x + y * y + z * z), 1e-12f);  // F.normalize
    w *= inv; x *= inv; y *= inv; z *= inv;
    const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - w * z), R02 = 2.f * (x * z + w * y);
    const float R10 = 2.f * (x * y + w * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - w * x);
    const float R20 = 2.f * (x * z - w * y), R21 = 2.f * (y * z + w * x), R22 = 1.f - 2.f * (x * x + y * y);
    const float* ls = sb.scales + (size_t)row * 3;
    const float s0 = expf(ls[0]), s1 = expf(ls[1]), s2 = expf(ls[2]);
    // Sigma t = R diag(s^2) R^T t
    const float a0 = (R00 * t0 + R10 * t1 + R20 * t2) * (s0 * s0);
    const float a1 = (R01 * t0 + R11 * t1 + R21 * t2) * (s1 * s1);
    const float a2 = (R02 * t0 + R12 * t1 + R22 * t2) * (s2 * s2);
    float* m = sb.means + (size_t)row * 3;
    m[0] += R00 * a0 + R01 * a1 + R02 * a2;
    m[1] += R10 * a0 + R11 * a1 + R12 * a2;
    m[2] += R20 * a0 + R21 * a1 + R22 * a2;
}

// ---- sampler ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double mc_weight(const float* __restrict__ op, int i, float min_opacity, int exclude_dead, int* dead) {
    const float o = mc_sigmoid(op[i]);
    *dead = o <= min_opacity;
    return (exclude_dead && *dead) ? 0.0 : (double)o;
}

// per tile: the sum of its weights and its number of dead rows.  Row i of thread k of tile t has the prefix
//   P_i = T_t + (E_k + L_i),  L_i = the thread's weights up to i added serially, E_k = the thread sums added serially,
// T_t = the tile sums added serially: P is non-decreasing, a zero-weight row repeats its predecessor's P exactly, and the last
// row's P is the total.
__device__ __forceinline__ void mc_thread_weights(const float* __restrict__ op, int n, float min_opacity, int exclude_dead, int i0,
                                                  double* w, double* l, int* dmask) {
    double s = 0.0;
    int m = 0;
#pragma unroll
    for (int j = 0; j < MC_SCAN_ITEMS; ++j) {
        w[j] = 0.0;
        if (i0 + j < n) {
            int dead;
            w[j] = mc_weight(op, i0 + j, min_opacity, exclude_dead, &dead);
            m |= dead << j;
        }
        s += w[j];
        l[j] = s;
    }
    *dmask = m;
}

__global__ void __launch_bounds__(MC_SCAN_THREADS) mcmc_tile_sums_kernel(const float* __restrict__ op, int n, float min_opacity,
                                                                         int exclude_dead, double* __restrict__ tile_w,
                                                                         int* __restrict__ tile_d) {
    __shared__ double sw[MC_SCAN_THREADS + 1];
    __shared__ int sd[MC_SCAN_THREADS + 1];
    const int i0 = (int)blockIdx.x * MC_TILE + (int)threadIdx.x * MC_SCAN_ITEMS;
    double w[MC_SCAN_ITEMS], l[MC_SCAN_ITEMS];
    int dmask;
    mc_thread_weights(op, n, min_opacity, exclude_dead, i0, w, l, &dmask);
    sw[threadIdx.x] = l[MC_SCAN_ITEMS - 1];
    sd[threadIdx.x] = __popc(dmask);
    const double W = mc_block_exclusive(sw, MC_SCAN_THREADS);
    const int D = mc_block_exclusive(sd, MC_SCAN_THREADS);
    if (threadIdx.x == 0) {
        tile_w[blockIdx.x] = W;
        tile_d[blockIdx.x] = D;
    }
}

// one thread: the tile sums and dead counts become exclusive prefixes in place; the total and the number of dead rows
__global__ void mcmc_tile_scan_kernel(double* __restrict__ tile_w, int* __restrict__ tile_d, int ntiles, double* __restrict__ total,
                                      int* __restrict__ num_dead) {
    double s = 0.0;
    int d = 0;
    for (int t = 0; t < ntiles; ++t) {
        const double w = tile_w[t];
        const int c = tile_d[t];
        tile_w[t] = s;
        tile_d[t] = d;
        s += w;
        d += c;
    }
    *total = s;
    *num_dead = d;
}

// per tile: the prefix of every row and the compacted dead rows
__global__ void __launch_bounds__(MC_SCAN_THREADS) mcmc_prefix_kernel(const float* __restrict__ op, int n, float min_opacity,
                                                                      int exclude_dead, const double* __restrict__ tile_w,
                                                                      const int* __restrict__ tile_d, double* __restrict__ prefix,
                                                                      int32_t* __restrict__ dead_rows) {
    __shared__ double sw[MC_SCAN_THREADS + 1];
    __shared__ int sd[MC_SCAN_THREADS + 1];
    const int i0 = (int)blockIdx.x * MC_TILE + (int)threadIdx.x * MC_SCAN_ITEMS;
    double w[MC_SCAN_ITEMS], l[MC_SCAN_ITEMS];
    int dmask;
    mc_thread_weights(op, n, min_opacity, exclude_dead, i0, w, l, &dmask);
    sw[threadIdx.x] = l[MC_SCAN_ITEMS - 1];
    sd[threadIdx.x] = __popc(dmask);
    mc_block_exclusive(sw, MC_SCAN_THREADS);
    mc_block_exclusive(sd, MC_SCAN_THREADS);
    const double T = tile_w[blockIdx.x], E = sw[threadIdx.x];
    int d = tile_d[blockIdx.x] + sd[threadIdx.x];
#pragma unroll
    for (int j = 0; j < MC_SCAN_ITEMS; ++j) {
        if (i0 + j < n) {
            prefix[i0 + j] = T + (E + l[j]);
            if (dead_rows && ((dmask >> j) & 1)) dead_rows[d++] = i0 + j;
        }
    }
}

__global__ void mcmc_draw_kernel(const double* __restrict__ prefix, int n, int max_draws,
                                 const int32_t* __restrict__ num_draws_dev, uint64_t seed, int step, int sub, int purpose,
                                 const double* __restrict__ uniforms, int32_t* __restrict__ draws, int32_t* __restrict__ counts) {
    const int j = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    const int nd = num_draws_dev ? min(*num_draws_dev, max_draws) : max_draws;
    if (j >= nd) return;
    const double T = prefix[n - 1];  // == the total
    if (!(T > 0.0)) {
        draws[j] = -1;
        return;
    }
    double u;
    if (uniforms) {
        u = uniforms[j];
    } else {  // 53 bits
        const mc_u4 r = mc_philox(seed, (uint32_t)j, (uint32_t)step, (uint32_t)sub, (uint32_t)purpose);
        u = (double)(((uint64_t)r.x << 21) ^ (uint64_t)(r.y >> 11)) * 1.1102230246251565e-16;
    }
    const double t = u * T;
    // the first row whose prefix exceeds t: a zero-weight row repeats its predecessor's prefix and is never first
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (prefix[mid] > t) hi = mid; else lo = mid + 1;
    }
    if (!(prefix[lo] > t)) {  // t rounded up to the total: the first row that reaches it
        lo = 0; hi = n - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (prefix[mid] >= T) hi = mid; else lo = mid + 1;
        }
    }
    draws[j] = lo;
    atomicAdd(counts + lo, 1);
}

// ---- relocation update rule ------------------------------------------------------------------------------------
__global__ void mcmc_relocate_kernel(float* __restrict__ op, float* __restrict__ scales, int n, const int32_t* __restrict__ counts,
                                     float min_opacity, sgn_mcmc_tensors zero) {
    const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (i >= n) return;
    const int c = counts[i];
    if (c <= 0) return;
    const int N = min(c + 1, MC_MAX_N);
    const double o = (double)mc_sigmoid(op[i]);
    const double op_ = 1.0 - pow(1.0 - o, 1.0 / (double)N);
    double denom = 0.0, binom = 1.0, pk = 1.0;
    for (int k = 1; k <= N; ++k) {
        binom = binom * (double)(N - k + 1) / (double)k;  // C(N, k), exact in fp64 for N <= 51
        pk *= op_;
        const double term = binom * pk / sqrt((double)k);
        denom += (k & 1) ? term : -term;
    }
    const double ratio = o / denom;
    float* ls = scales + (size_t)i * 3;
#pragma unroll
    for (int a = 0; a < 3; ++a) ls[a] = (float)log(ratio * (double)expf(ls[a]));
    const float onew = fminf(fmaxf((float)op_, min_opacity), 1.0f - 1.1920929e-7f);
    op[i] = (float)log((double)onew / (1.0 - (double)onew));
    for (int t = 0; t < zero.count; ++t) {
        float* z = zero.data[t] + (size_t)i * zero.width[t];
        for (int a = 0; a < zero.width[t]; ++a) z[a] = 0.f;
    }
}

// one warp per row
__global__ void mcmc_copy_rows_kernel(sgn_mcmc_tensors t, const int32_t* __restrict__ dst_rows, int dst_row0,
                                      const int32_t* __restrict__ src_rows, int max_rows, const int32_t* __restrict__ num_rows_dev) {
    const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    const int nr = num_rows_dev ? min(*num_rows_dev, max_rows) : max_rows;
    if (j >= nr) return;
    const int s = src_rows[j];
    if (s < 0) return;
    const size_t d = dst_rows ? (size_t)dst_rows[j] : (size_t)dst_row0 + j;
    for (int k = 0; k < t.count; ++k) {
        const int wdt = t.width[k];
        float* base = t.data[k];
        for (int a = lane; a < wdt; a += 32) base[d * wdt + a] = base[(size_t)s * wdt + a];
    }
}

// ---- regularisers ----------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T mc_block_sum(T v, T* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < MC_CHUNK / 32 ? smem[threadIdx.x] : T(0);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
}

__global__ void __launch_bounds__(MC_CHUNK) mcmc_reg_fwd_kernel(const sgn_segment* __restrict__ segs, int nseg, int num_chunks,
                                                                double* __restrict__ partial) {
    __shared__ double s_red[MC_CHUNK / 32];
    double ao = 0.0, as = 0.0;
    for (int c = blockIdx.x; c < num_chunks; c += gridDim.x) {
        const sgn_segment& sg = segs[mc_segment_of(segs, nseg, c)];
        const int row = (c - sg.chunk0) * MC_CHUNK + (int)threadIdx.x;
        if (row < sg.count) {
            ao += (double)mc_sigmoid(sg.opacities[row]);
            const float* x = sg.scales + (size_t)row * 3;
            as += (double)expf(x[0]) + (double)expf(x[1]) + (double)expf(x[2]);
        }
    }
    const double bo = mc_block_sum(ao, s_red);
    const double bs = mc_block_sum(as, s_red);
    if (threadIdx.x == 0) {
        partial[2 * blockIdx.x] = bo;
        partial[2 * blockIdx.x + 1] = bs;
    }
}

__global__ void __launch_bounds__(MC_CHUNK) mcmc_reg_finish_kernel(const double* __restrict__ partial, int nblocks, int N, float w_o,
                                                                   float w_s, float* __restrict__ out) {
    __shared__ double s_red[MC_CHUNK / 32];
    double so = 0.0, ss = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
        so += partial[2 * i];
        ss += partial[2 * i + 1];
    }
    const double to = mc_block_sum(so, s_red);
    const double ts = mc_block_sum(ss, s_red);
    if (threadIdx.x == 0) {  // 0 / 0 = NaN for zero rows, as torch's mean
        out[0] = __fmul_rn(w_o, (float)(to / (double)N));
        out[1] = __fmul_rn(w_s, (float)(ts / (3.0 * (double)N)));
    }
}

__global__ void __launch_bounds__(MC_CHUNK) mcmc_reg_bwd_kernel(const sgn_segment* __restrict__ segs,
                                                                const sgn_segment_grads* __restrict__ grads, int nseg, float inv_n,
                                                                float inv_3n, float w_o, float w_s, const float* __restrict__ v_o,
                                                                const float* __restrict__ v_s) {
    const int c = blockIdx.x;
    const int k = mc_segment_of(segs, nseg, c);
    const sgn_segment& sg = segs[k];
    const int row = (c - sg.chunk0) * MC_CHUNK + (int)threadIdx.x;
    if (row >= sg.count) return;
    // torch autograd's chain: (v * w) * (1 / N), then sigmoid's backward g (1 - o) o, exp's backward g s
    if (v_o) {
        const float g = __fmul_rn(__fmul_rn(*v_o, w_o), inv_n);
        const float o = mc_sigmoid(sg.opacities[row]);
        float* go = grads[k].opacities + row;
        *go = __fadd_rn(*go, __fmul_rn(__fmul_rn(g, __fsub_rn(1.0f, o)), o));
    }
    if (v_s) {
        const float g = __fmul_rn(__fmul_rn(*v_s, w_s), inv_3n);
        const float* x = sg.scales + (size_t)row * 3;
        float* gs = grads[k].scales + (size_t)row * 3;
#pragma unroll
        for (int a = 0; a < 3; ++a) gs[a] = __fadd_rn(gs[a], __fmul_rn(g, expf(x[a])));
    }
}

// ---- C ABI -----------------------------------------------------------------------------------------------------
extern "C" size_t sgn_sizeof_mcmc_sub(void) { return sizeof(sgn_mcmc_sub); }
extern "C" size_t sgn_sizeof_mcmc_tensors(void) { return sizeof(sgn_mcmc_tensors); }

extern "C" int sgn_mcmc_noise(const sgn_mcmc_sub* subs_dev, int nsub, int num_chunks, float lr, uint64_t seed, int step,
                              const float* normals, void* stream_) {
    SGN_RANGE("sgn_mcmc_noise");
    SGN_REQUIRE(nsub >= 0 && num_chunks >= 0, "sgn_mcmc_noise: negative nsub / num_chunks");
    SGN_REQUIRE(subs_dev || nsub == 0, "sgn_mcmc_noise: null sub-model table with nsub = %d", nsub);
    SGN_REQUIRE(nsub > 0 || num_chunks == 0, "sgn_mcmc_noise: num_chunks = %d without sub-models", num_chunks);
    if (num_chunks == 0) return SGN_OK;
    mcmc_noise_kernel<<<num_chunks, MC_CHUNK, 0, (cudaStream_t)stream_>>>(subs_dev, nsub, lr, seed, step, normals);
    SGN_CHECK_LAUNCH("mcmc_noise_kernel");
    return SGN_OK;
}

static int mc_tiles(int n) { return (n + MC_TILE - 1) / MC_TILE; }

extern "C" size_t sgn_mcmc_sample_scratch_bytes(int n) {
    const size_t nt = (size_t)mc_tiles(n > 0 ? n : 0);
    return sizeof(double) * ((size_t)(n > 0 ? n : 0) + nt + 1) + sizeof(int) * (nt + 1) + 16;
}

extern "C" int sgn_mcmc_sample(const float* opacities, int n, float min_opacity, int exclude_dead, int max_draws,
                               const int32_t* num_draws_dev, uint64_t seed, int step, int sub, int purpose, const double* uniforms,
                               int32_t* draws, int32_t* counts, int32_t* dead_rows, int32_t* num_dead, double* total, void* scratch,
                               size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_mcmc_sample");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(n >= 0 && max_draws >= 0, "sgn_mcmc_sample: negative n / max_draws");
    SGN_REQUIRE(n == 0 || (opacities && counts), "sgn_mcmc_sample: null opacities / counts");
    SGN_REQUIRE(max_draws == 0 || draws, "sgn_mcmc_sample: null draws");
    SGN_REQUIRE(scratch, "sgn_mcmc_sample: null scratch");
    if (scratch_bytes < sgn_mcmc_sample_scratch_bytes(n)) {
        sgn_set_error("sgn_mcmc_sample: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_mcmc_sample_scratch_bytes(n));
        return SGN_ERR_WORKSPACE;
    }
    const int nt = mc_tiles(n);
    double* prefix = (double*)scratch;
    double* tile_w = prefix + n;
    double* tot = tile_w + nt;
    int* tile_d = (int*)(tot + 1);
    int* nd = tile_d + nt;
    if (n > 0) SGN_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * (size_t)n, stream));
    if (n == 0) {  // nothing to draw from
        SGN_CHECK_CUDA(cudaMemsetAsync(tot, 0, sizeof(double), stream));
        SGN_CHECK_CUDA(cudaMemsetAsync(nd, 0, sizeof(int), stream));
    } else {
        mcmc_tile_sums_kernel<<<nt, MC_SCAN_THREADS, 0, stream>>>(opacities, n, min_opacity, exclude_dead, tile_w, tile_d);
        SGN_CHECK_LAUNCH("mcmc_tile_sums_kernel");
        mcmc_tile_scan_kernel<<<1, 1, 0, stream>>>(tile_w, tile_d, nt, tot, nd);
        SGN_CHECK_LAUNCH("mcmc_tile_scan_kernel");
        mcmc_prefix_kernel<<<nt, MC_SCAN_THREADS, 0, stream>>>(opacities, n, min_opacity, exclude_dead, tile_w, tile_d, prefix, dead_rows);
        SGN_CHECK_LAUNCH("mcmc_prefix_kernel");
    }
    if (num_dead) SGN_CHECK_CUDA(cudaMemcpyAsync(num_dead, nd, sizeof(int), cudaMemcpyDeviceToDevice, stream));
    if (total) SGN_CHECK_CUDA(cudaMemcpyAsync(total, tot, sizeof(double), cudaMemcpyDeviceToDevice, stream));
    if (max_draws > 0 && n > 0) {
        mcmc_draw_kernel<<<(max_draws + 255) / 256, 256, 0, stream>>>(prefix, n, max_draws, num_draws_dev, seed, step, sub, purpose,
                                                                      uniforms, draws, counts);
        SGN_CHECK_LAUNCH("mcmc_draw_kernel");
    } else if (max_draws > 0) {
        SGN_CHECK_CUDA(cudaMemsetAsync(draws, 0xff, sizeof(int32_t) * (size_t)max_draws, stream));
    }
    return SGN_OK;
}

static bool mc_tensors_ok(const sgn_mcmc_tensors* t) {
    if (t->count < 0 || t->count > SGN_MCMC_MAX_TENSORS) return false;
    for (int k = 0; k < t->count; ++k)
        if (!t->data[k] || t->width[k] <= 0) return false;
    return true;
}

extern "C" int sgn_mcmc_relocate(float* opacities, float* scales, int n, const int32_t* counts, float min_opacity,
                                 const sgn_mcmc_tensors* zero, void* stream_) {
    SGN_RANGE("sgn_mcmc_relocate");
    SGN_REQUIRE(n >= 0, "sgn_mcmc_relocate: negative n");
    SGN_REQUIRE(n == 0 || (opacities && scales && counts), "sgn_mcmc_relocate: null opacities / scales / counts");
    sgn_mcmc_tensors z = {};
    if (zero) {
        SGN_REQUIRE(mc_tensors_ok(zero), "sgn_mcmc_relocate: bad tensor table (count %d)", zero->count);
        z = *zero;
    }
    if (n == 0) return SGN_OK;
    mcmc_relocate_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(opacities, scales, n, counts, min_opacity, z);
    SGN_CHECK_LAUNCH("mcmc_relocate_kernel");
    return SGN_OK;
}

extern "C" int sgn_mcmc_copy_rows(const sgn_mcmc_tensors* t, const int32_t* dst_rows, int dst_row0, const int32_t* src_rows, int max_rows,
                                  const int32_t* num_rows_dev, void* stream_) {
    SGN_RANGE("sgn_mcmc_copy_rows");
    SGN_REQUIRE(t && mc_tensors_ok(t), "sgn_mcmc_copy_rows: bad tensor table");
    SGN_REQUIRE(max_rows >= 0 && dst_row0 >= 0, "sgn_mcmc_copy_rows: negative max_rows / dst_row0");
    SGN_REQUIRE(max_rows == 0 || src_rows, "sgn_mcmc_copy_rows: null src_rows");
    if (max_rows == 0 || t->count == 0) return SGN_OK;
    const long long threads = (long long)max_rows * 32;
    mcmc_copy_rows_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(*t, dst_rows, dst_row0, src_rows, max_rows,
                                                                                               num_rows_dev);
    SGN_CHECK_LAUNCH("mcmc_copy_rows_kernel");
    return SGN_OK;
}

extern "C" size_t sgn_mcmc_reg_scratch_bytes(void) { return sizeof(double) * 2 * MC_REG_BLOCKS; }

extern "C" int sgn_mcmc_reg_fwd(const sgn_segment* table_dev, int nseg, int N, int num_chunks, float w_opacity, float w_scale, float* out,
                                void* scratch, size_t scratch_bytes, void* stream_) {
    SGN_RANGE("sgn_mcmc_reg_fwd");
    cudaStream_t stream = (cudaStream_t)stream_;
    SGN_REQUIRE(out && scratch, "sgn_mcmc_reg_fwd: null output or scratch");
    SGN_REQUIRE(N >= 0 && nseg >= 0 && num_chunks >= 0, "sgn_mcmc_reg_fwd: negative N / nseg / num_chunks");
    SGN_REQUIRE(table_dev || nseg == 0, "sgn_mcmc_reg_fwd: null segment table with nseg = %d", nseg);
    SGN_REQUIRE(nseg > 0 || num_chunks == 0, "sgn_mcmc_reg_fwd: num_chunks = %d without segments", num_chunks);
    if (scratch_bytes < sgn_mcmc_reg_scratch_bytes()) {
        sgn_set_error("sgn_mcmc_reg_fwd: scratch too small (%zu < %zu bytes)", scratch_bytes, sgn_mcmc_reg_scratch_bytes());
        return SGN_ERR_WORKSPACE;
    }
    mcmc_reg_fwd_kernel<<<MC_REG_BLOCKS, MC_CHUNK, 0, stream>>>(table_dev, nseg, num_chunks, (double*)scratch);
    SGN_CHECK_LAUNCH("mcmc_reg_fwd_kernel");
    mcmc_reg_finish_kernel<<<1, MC_CHUNK, 0, stream>>>((const double*)scratch, MC_REG_BLOCKS, N, w_opacity, w_scale, out);
    SGN_CHECK_LAUNCH("mcmc_reg_finish_kernel");
    return SGN_OK;
}

extern "C" int sgn_mcmc_reg_bwd(const sgn_segment* table_dev, const sgn_segment_grads* grads_dev, int nseg, int N, int num_chunks,
                                float w_opacity, float w_scale, const float* v_opacity, const float* v_scale, void* stream_) {
    SGN_RANGE("sgn_mcmc_reg_bwd");
    SGN_REQUIRE(N >= 0 && nseg >= 0 && num_chunks >= 0, "sgn_mcmc_reg_bwd: negative N / nseg / num_chunks");
    SGN_REQUIRE((table_dev && grads_dev) || nseg == 0, "sgn_mcmc_reg_bwd: null segment or gradient table with nseg = %d", nseg);
    SGN_REQUIRE(nseg > 0 || num_chunks == 0, "sgn_mcmc_reg_bwd: num_chunks = %d without segments", num_chunks);
    if (num_chunks == 0 || (!v_opacity && !v_scale)) return SGN_OK;
    const float inv_n = 1.0f / (float)N, inv_3n = 1.0f / (float)(3 * (long long)N);
    mcmc_reg_bwd_kernel<<<num_chunks, MC_CHUNK, 0, (cudaStream_t)stream_>>>(table_dev, grads_dev, nseg, inv_n, inv_3n, w_opacity, w_scale,
                                                                            v_opacity, v_scale);
    SGN_CHECK_LAUNCH("mcmc_reg_bwd_kernel");
    return SGN_OK;
}
