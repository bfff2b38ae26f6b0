// Exact-section projection math shared by the forward and backward per-Gaussian kernels.
//
// Arithmetic contract: every * + - / sqrt of the exact section goes through the `xf` wrapper below (explicit
// round-to-nearest intrinsics, never contracted), in the order written -- independent of the translation unit's --fmad.
// tests/ compare the integer outputs (radii, tile AABB, num_tiles_hit, sort order) BIT-EXACTLY
// against the CPU oracle, which states the same sequence independently.
//
// Semantics: gsplat 0.1.x project_gaussians (SURVEY.md Appendix A.1-A.4) preceded by the reference's
// compose / pre-ops (street_gaussians_ns/sgn_splatfacto_scene_graph.py:404-417,
// street_gaussians_ns/sgn_splatfacto.py:857,864).
#pragma once
#include "sgn_common.cuh"

struct SgnProj {
    float mw[3];
    float qr[4];
    float qnorm;
    float qn[4];
    float s[3];
    float Rg[9];
    float S[6];
    float pv[3];
    float tx, ty;
    int clampx, clampy;
    float T[6];
    float a, b, c;
    float comp;  // blur compensation (sgn_compensation), when sgn_project_exact was asked for it; 0 otherwise
    float coef;  // opacity factor of the 3D smoothing filter (sgn_filter_coef), when asked for; 1 otherwise
    float conic[3];
    float xy[2];
    int radius;
    int tmin[2], tmax[2];
    bool visible;
};

// xf: a float whose * + - / are the explicit round-to-nearest intrinsics, which the compiler never contracts into an FMA.
// Every operand of the exact section is an xf, so the section is individually rounded in ANY translation unit, whatever
// its --fmad setting (the colour / gradient code around it is free to use FMAs).
struct xf {
    float v;
    __device__ __forceinline__ xf() {}
    __device__ __forceinline__ xf(float x) : v(x) {}
};
__device__ __forceinline__ xf operator*(xf a, xf b) { return xf(__fmul_rn(a.v, b.v)); }
__device__ __forceinline__ xf operator+(xf a, xf b) { return xf(__fadd_rn(a.v, b.v)); }
__device__ __forceinline__ xf operator-(xf a, xf b) { return xf(__fsub_rn(a.v, b.v)); }
__device__ __forceinline__ xf operator/(xf a, xf b) { return xf(__fdiv_rn(a.v, b.v)); }
__device__ __forceinline__ xf operator-(xf a) { return xf(-a.v); }
__device__ __forceinline__ xf xsqrt(xf a) { return xf(__fsqrt_rn(a.v)); }
__device__ __forceinline__ xf xmax(xf a, xf b) { return xf(fmaxf(a.v, b.v)); }

// exp() as a fixed sequence of IEEE operations (same constants as oracle/sgn_oracle.c).
__device__ __forceinline__ float sgn_expf_exact(float x_) {
    const xf x(fminf(fmaxf(x_, -80.0f), 80.0f));
    const xf n(rintf((x * 1.44269504f).v));
    xf r = x - n * 0.693145752f;
    r = r - n * 1.42860677e-6f;
    xf p(1.98412698e-4f);
    p = p * r + 1.38888889e-3f;
    p = p * r + 8.33333333e-3f;
    p = p * r + 4.16666667e-2f;
    p = p * r + 1.66666667e-1f;
    p = p * r + 0.5f;
    p = p * r + 1.0f;
    p = p * r + 1.0f;
    return ldexpf(p.v, (int)n.v);
}

__device__ __forceinline__ int sgn_f2i_sat(float x) {
    if (x != x) return 0;
    if (x >= 1.0e9f) return 1000000000;
    if (x <= -1.0e9f) return -1000000000;
    return (int)x;
}

// The blurred screen covariance [[a, b], [b, c]] = T S T^T + 0.3 I from T = J W (2x3) and S = Sigma3D (upper triangle 00 01 02
// 11 12 22), in the exact section's order, and its un-blurred diagonal c00, c11.  The backward calls it again on SgnProj's
// T and S for the same bits.
__device__ __forceinline__ void sgn_cov2d_blur(const xf T[6], const xf S[6], xf& a, xf& b, xf& c, xf& c00, xf& c11) {
    xf TS[6];
    TS[0] = (T[0] * S[0] + T[1] * S[1]) + T[2] * S[2];
    TS[1] = (T[0] * S[1] + T[1] * S[3]) + T[2] * S[4];
    TS[2] = (T[0] * S[2] + T[1] * S[4]) + T[2] * S[5];
    TS[3] = (T[3] * S[0] + T[4] * S[1]) + T[5] * S[2];
    TS[4] = (T[3] * S[1] + T[4] * S[3]) + T[5] * S[4];
    TS[5] = (T[3] * S[2] + T[4] * S[4]) + T[5] * S[5];
    c00 = (TS[0] * T[0] + TS[1] * T[1]) + TS[2] * T[2];
    const xf c01 = (TS[0] * T[3] + TS[1] * T[4]) + TS[2] * T[5];
    c11 = (TS[3] * T[3] + TS[4] * T[4]) + TS[5] * T[5];
    a = c00 + xf(0.3f);
    b = c01;
    c = c11 + xf(0.3f);
}

__device__ __forceinline__ float sgn_compensation(const SgnProj& st);

// ---- 3D smoothing filter (Mip-Splatting): s' = sqrt(s^2 + sigma^2) on one axis, and r = s^2 / (s^2 + sigma^2) ----------------
// Individually rounded (xf), so that the forward and the backward (which recomputes r from the parameters) get the same bits.
// s^2 + sigma^2 == 0 (sigma 0 and s^2 below the smallest float) keeps r = 1: the filter is then the identity.
__device__ __forceinline__ xf sgn_filter_axis(xf s, xf sigma, xf& r) {
    const xf s2 = s * s;
    const xf v = s2 + sigma * sigma;
    r = v.v > 0.f ? s2 / v : xf(1.f);
    return xsqrt(v);
}

// coef = prod_k sqrt(r_k), the filter's opacity factor, as a product of per-axis ratios: prod s^2 / prod (s^2 + sigma^2)
// underflows in fp32 for small scales
__device__ __forceinline__ float sgn_filter_coef(const float r[3]) {
    return ((xsqrt(xf(r[0])) * xsqrt(xf(r[1]))) * xsqrt(xf(r[2]))).v;
}

// the ratios r_k of the log-scales ls (the model's parameters) under the filter sigma, recomputed as sgn_project_exact does
__device__ __forceinline__ void sgn_filter_ratios(const float ls[3], float sigma, float r[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        xf rk;
        sgn_filter_axis(xf(sgn_expf_exact(ls[k])), xf(sigma), rk);
        r[k] = rk.v;
    }
}

// Returns st.visible.  `m`, `ls`, `q` are this Gaussian's raw parameters.
// log_scales: `ls` holds log-scales (the model's parameters) -> exp is applied here; otherwise `ls` holds
// activated scales (gsplat's project_gaussians argument) multiplied by glob_scale.
// with_comp (warp-uniform): also st.comp = sgn_compensation(st), computed here while its inputs are live.
// with_filter (warp-uniform): the 3D smoothing filter of size `sigma` -- st.s and the covariance use s' = sqrt(s^2 + sigma^2),
// and st.coef = sgn_filter_coef of the ratios (1 otherwise).
__device__ __forceinline__ bool sgn_project_exact(const sgn_segment& sg, const sgn_camera& cam, const float m_[3],
                                                  const float ls[3], const float q_[4], SgnProj& st,
                                                  const bool log_scales = true, const float glob_scale = 1.f,
                                                  const bool with_comp = false, const bool with_filter = false,
                                                  const float sigma = 0.f) {
    xf W[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) W[k] = xf(cam.viewmat[k]);
    st.visible = false;
    st.radius = 0;
    st.xy[0] = st.xy[1] = 0.f;
    st.conic[0] = st.conic[1] = st.conic[2] = 0.f;
    st.tmin[0] = st.tmin[1] = st.tmax[0] = st.tmax[1] = 0;
    st.clampx = st.clampy = 0;
    st.comp = 0.f;
    st.coef = 1.f;
    const xf m[3] = {xf(m_[0]), xf(m_[1]), xf(m_[2])};
    xf mw[3], qr[4];
    if (sg.has_pose) {
        xf R[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) R[k] = xf(sg.R[k]);
        mw[0] = ((R[0] * m[0] + R[1] * m[1]) + R[2] * m[2]) + xf(sg.t[0]);
        mw[1] = ((R[3] * m[0] + R[4] * m[1]) + R[5] * m[2]) + xf(sg.t[1]);
        mw[2] = ((R[6] * m[0] + R[7] * m[1]) + R[8] * m[2]) + xf(sg.t[2]);
        const xf aw(sg.q[0]), ax(sg.q[1]), ay(sg.q[2]), az(sg.q[3]);
        const xf bw(q_[0]), bx(q_[1]), by(q_[2]), bz(q_[3]);
        qr[0] = ((aw * bw - ax * bx) - ay * by) - az * bz;
        qr[1] = ((aw * bx + ax * bw) + ay * bz) - az * by;
        qr[2] = ((aw * by - ax * bz) + ay * bw) + az * bx;
        qr[3] = ((aw * bz + ax * by) - ay * bx) + az * bw;
    } else {
        mw[0] = m[0]; mw[1] = m[1]; mw[2] = m[2];
        qr[0] = xf(q_[0]); qr[1] = xf(q_[1]); qr[2] = xf(q_[2]); qr[3] = xf(q_[3]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) st.mw[k] = mw[k].v;
#pragma unroll
    for (int k = 0; k < 4; ++k) st.qr[k] = qr[k].v;
    xf pv[3];
    pv[0] = ((W[0] * mw[0] + W[1] * mw[1]) + W[2] * mw[2]) + W[3];
    pv[1] = ((W[4] * mw[0] + W[5] * mw[1]) + W[6] * mw[2]) + W[7];
    pv[2] = ((W[8] * mw[0] + W[9] * mw[1]) + W[10] * mw[2]) + W[11];
#pragma unroll
    for (int k = 0; k < 3; ++k) st.pv[k] = pv[k].v;
    if (pv[2].v <= cam.clip_thresh) return false;
    xf qn[4];
    {
        const xf n2 = ((qr[0] * qr[0] + qr[1] * qr[1]) + qr[2] * qr[2]) + qr[3] * qr[3];
        const xf qnorm = xsqrt(n2);
        st.qnorm = qnorm.v;
#pragma unroll
        for (int k = 0; k < 4; ++k) { qn[k] = qr[k] / qnorm; st.qn[k] = qn[k].v; }
    }
    xf sc[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) sc[k] = log_scales ? xf(sgn_expf_exact(ls[k])) : xf(ls[k]) * xf(glob_scale);
    if (with_filter) {
        float r[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            xf rk;
            sc[k] = sgn_filter_axis(sc[k], xf(sigma), rk);
            r[k] = rk.v;
        }
        st.coef = sgn_filter_coef(r);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) st.s[k] = sc[k].v;
    xf S[6];
    {
        const xf w = qn[0], x = qn[1], y = qn[2], z = qn[3];
        xf R[9];
        R[0] = xf(1.f) - xf(2.f) * (y * y + z * z);
        R[1] = xf(2.f) * (x * y - w * z);
        R[2] = xf(2.f) * (x * z + w * y);
        R[3] = xf(2.f) * (x * y + w * z);
        R[4] = xf(1.f) - xf(2.f) * (x * x + z * z);
        R[5] = xf(2.f) * (y * z - w * x);
        R[6] = xf(2.f) * (x * z - w * y);
        R[7] = xf(2.f) * (y * z + w * x);
        R[8] = xf(1.f) - xf(2.f) * (x * x + y * y);
        xf M[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) { st.Rg[3 * r + c] = R[3 * r + c].v; M[3 * r + c] = R[3 * r + c] * sc[c]; }
        S[0] = (M[0] * M[0] + M[1] * M[1]) + M[2] * M[2];
        S[1] = (M[0] * M[3] + M[1] * M[4]) + M[2] * M[5];
        S[2] = (M[0] * M[6] + M[1] * M[7]) + M[2] * M[8];
        S[3] = (M[3] * M[3] + M[4] * M[4]) + M[5] * M[5];
        S[4] = (M[3] * M[6] + M[4] * M[7]) + M[5] * M[8];
        S[5] = (M[6] * M[6] + M[7] * M[7]) + M[8] * M[8];
#pragma unroll
        for (int k = 0; k < 6; ++k) st.S[k] = S[k].v;
    }
    xf a, b, c;
    {
        const xf z = pv[2];
        const xf rz = xf(1.f) / z;
        const xf rz2 = rz * rz;
        xf ux = pv[0] / z, uy = pv[1] / z;
        if (ux.v > cam.limx) { ux = xf(cam.limx); st.clampx = 1; }
        else if (ux.v < -cam.limx) { ux = xf(-cam.limx); st.clampx = -1; }
        if (uy.v > cam.limy) { uy = xf(cam.limy); st.clampy = 1; }
        else if (uy.v < -cam.limy) { uy = xf(-cam.limy); st.clampy = -1; }
        const xf tx = z * ux, ty = z * uy;
        st.tx = tx.v;
        st.ty = ty.v;
        const xf fx(cam.fx), fy(cam.fy);
        const xf J00 = fx * rz, J11 = fy * rz;
        const xf J02 = -((fx * tx) * rz2);
        const xf J12 = -((fy * ty) * rz2);
        xf T[6];
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
            T[cc] = J00 * W[cc] + J02 * W[8 + cc];
            T[3 + cc] = J11 * W[4 + cc] + J12 * W[8 + cc];
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) st.T[k] = T[k].v;
        xf c00, c11;
        sgn_cov2d_blur(T, S, a, b, c, c00, c11);
        st.a = a.v; st.b = b.v; st.c = c.v;
        if (with_comp) st.comp = sgn_compensation(st);
    }
    const xf det = a * c - b * b;
    if (det.v == 0.f) return false;
    {
        const xf inv = xf(1.f) / det;
        st.conic[0] = (c * inv).v;
        st.conic[1] = ((-b) * inv).v;
        st.conic[2] = (a * inv).v;
        const xf bm = xf(0.5f) * (a + c);
        const xf disc = xsqrt(xmax(xf(0.1f), bm * bm - det));
        const xf v1 = bm + disc, v2 = bm - disc;
        st.radius = sgn_f2i_sat(ceilf((xf(3.f) * xsqrt(xmax(v1, v2))).v));
    }
    xf cxp, cyp;
    {
        const xf rw = xf(1.f) / (pv[2] + xf(1e-6f));
        cxp = (pv[0] * rw) * xf(cam.fx) + xf(cam.cx);
        cyp = (pv[1] * rw) * xf(cam.fy) + xf(cam.cy);
        const xf bw((float)cam.block_width);
        const int tiles_x = (cam.width + cam.block_width - 1) / cam.block_width;
        const int tiles_y = (cam.height + cam.block_width - 1) / cam.block_width;
        const xf tcx = cxp / bw, tcy = cyp / bw, tr = xf((float)st.radius) / bw;
        st.tmin[0] = min(max(0, sgn_f2i_sat((tcx - tr).v)), tiles_x);
        st.tmax[0] = min(max(0, sgn_f2i_sat(((tcx + tr) + xf(1.f)).v)), tiles_x);
        st.tmin[1] = min(max(0, sgn_f2i_sat((tcy - tr).v)), tiles_y);
        st.tmax[1] = min(max(0, sgn_f2i_sat(((tcy + tr) + xf(1.f)).v)), tiles_y);
    }
    const int area = (st.tmax[0] - st.tmin[0]) * (st.tmax[1] - st.tmin[1]);
    if (area <= 0) { st.radius = 0; return false; }
    st.xy[0] = cxp.v;
    st.xy[1] = cyp.v;
    st.visible = true;
    return true;
}

// ---- blur compensation (the antialiased rasterize mode, and the Level-1 `compensation` output) ---------------------
// comp = sqrt(max(0, det(cov2d) / det(cov2d + 0.3 I))): the factor by which the 0.3 px^2 blur spreads the Gaussian's
// integrated density, gsplat's antialiased-mode opacity scale.  det(cov2d) of cov2d = P P^T, P = T M (2x3), M = R diag(s), is
// taken as the sum of the squared 2x2 minors of P (Cauchy-Binet): each minor is s_i s_j times a cross product of two
// columns of T R, so it keeps its accuracy for needles and sub-pixel Gaussians, where c00 c11 - c01^2 -- or (a - 0.3)
// (c - 0.3) - b^2 from the blurred entries -- cancels to rounding noise.  A Gaussian of rank one on the screen has comp 0.
// Individually rounded (xf) from SgnProj's T, Rg, s, a, b, c, so the forward and the backward compute the same bits.
__device__ __forceinline__ float sgn_compensation(const SgnProj& st) {
    xf P0[3], P1[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const xf m0 = xf(st.Rg[c]) * xf(st.s[c]), m1 = xf(st.Rg[3 + c]) * xf(st.s[c]), m2 = xf(st.Rg[6 + c]) * xf(st.s[c]);
        P0[c] = (xf(st.T[0]) * m0 + xf(st.T[1]) * m1) + xf(st.T[2]) * m2;
        P1[c] = (xf(st.T[3]) * m0 + xf(st.T[4]) * m1) + xf(st.T[5]) * m2;
    }
    const xf m01 = P0[0] * P1[1] - P0[1] * P1[0], m02 = P0[0] * P1[2] - P0[2] * P1[0], m12 = P0[1] * P1[2] - P0[2] * P1[1];
    const xf det_orig = (m01 * m01 + m02 * m02) + m12 * m12;
    const xf det_blur = xf(st.a) * xf(st.c) - xf(st.b) * xf(st.b);
    return xsqrt(xmax(xf(0.f), det_orig / det_blur)).v;
}

// Cotangent of comp -> cotangents of the blurred a, b (the one off-diagonal parameter), c, ADDED to vA, vB, vC.  With
// r = det_orig / det_blur and det_blur - det_orig = 0.3 (a + c) - 0.09:
//   dr/da = 0.3 (c c11 + b^2) / det_blur^2,  dr/dc = 0.3 (a c00 + b^2) / det_blur^2,
//   dr/db = -2 b (0.3 (a + c) - 0.09) / det_blur^2,  d comp = dr / (2 comp),
// with c00, c11 the un-blurred diagonal (not a - 0.3, c - 0.3, which lose a sub-pixel Gaussian's covariance).  The blur is a
// constant, so these are also the cotangents of the un-blurred cov2d.  comp == 0 (det_orig <= 0, clamped) passes nothing: the
// clamp is flat there, and 1 / (2 comp) would be inf.
__device__ __forceinline__ void sgn_compensation_vjp(float c00, float c11, float a, float b, float c, float comp, float v_comp,
                                                     float& vA, float& vB, float& vC) {
    if (!(comp > 0.f)) return;
    const float inv = 1.f / (a * c - b * b);
    const float w = (0.5f * v_comp) / comp * inv * inv;
    const float b2 = b * b;
    vA += w * (0.3f * (c * c11 + b2));
    vC += w * (0.3f * (a * c00 + b2));
    vB -= w * (2.f * b * (0.3f * (a + c) - 0.09f));
}

// ---- SH basis (gsplat "poly" SH, Appendix A.7); not part of the exact section -------------------
__device__ __forceinline__ void sgn_sh_basis(int deg, float x, float y, float z, float Y[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) Y[k] = 0.f;
    Y[0] = 0.28209479177387814f;
    if (deg < 1) return;
    const float C1 = 0.4886025119029199f;
    Y[1] = -C1 * y; Y[2] = C1 * z; Y[3] = -C1 * x;
    if (deg < 2) return;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    Y[4] = 1.0925484305920792f * xy;
    Y[5] = -1.0925484305920792f * yz;
    Y[6] = 0.31539156525252005f * (2.f * zz - xx - yy);
    Y[7] = -1.0925484305920792f * xz;
    Y[8] = 0.5462742152960396f * (xx - yy);
    if (deg < 3) return;
    Y[9] = -0.5900435899266435f * y * (3.f * xx - yy);
    Y[10] = 2.890611442640554f * xy * z;
    Y[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
    Y[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
    Y[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
    Y[14] = 1.445305721320277f * z * (xx - yy);
    Y[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
}
