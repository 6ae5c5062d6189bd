// polyrigid_math.cuh -- per-ray math of the blended-rigid (skinned) trilinear march (host+device; DESIGN.md 6h).
//
// The rays and samples are the Trilinear renderer's: pix_m = p0 + alpha_m dp (ray_math.cuh: make_pixline, linspace01).  At every
// sample the volume is pulled back through a linear blend of K affine maps M_k (3 x 4, voxel space), the rest of the weight on the
// identity:
//   y_m = x_m + sum_k w_k(x_m) (M_k [x_m; 1] - x_m),      I = L step sum_m tri(V, y_m)
// w_k is a coarse lattice sampled trilinearly (align_corners=False over the volume, zero outside the lattice), stored channel-last
// with the channels padded to KP = 4 or 8 (zero weights, zero matrices), so a lattice corner is KP / 4 float4 reads.
// With M = identity or w = 0 the displacement is exactly 0.0f and the march is trilinear_ray_fwd bit for bit.  The backprojection
// (polyrigid_ray_bproj) is the forward's transpose in the density: 8 scalar reductions per in-volume sample into a volume gradient,
// with no density read.
#pragma once

#include "ray_math.cuh"

namespace b200drr {

// The weight lattice: lattice coordinate u_a = pix_a * sc[a] + of[a] (node i of axis a sits at pix = (i + 1/2) D_a / g_a - 1/2);
// [elo, ehi] is, per axis, the pix interval outside which a sample can contribute nothing: the lattice's support (u in (-1, g))
// united with the zero-padded volume (pix in (-1, D)).  Outside it w = 0, so y = x, and x is outside the padded volume.
struct PolyLattice {
    const float4* w;  // [g0][g1][g2][KP / 4]
    int g[3];
    float sc[3], of[3], elo[3], ehi[3];
};

B200_HD PolyLattice make_lattice(const float* weights, int g0, int g1, int g2, const VolDims& dims)
{
    PolyLattice lat;
    lat.w = reinterpret_cast<const float4*>(weights);
    lat.g[0] = g0;
    lat.g[1] = g1;
    lat.g[2] = g2;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float cell = (float)dims.d[a] / (float)lat.g[a];
        lat.sc[a] = (float)lat.g[a] / (float)dims.d[a];
        lat.of[a] = 0.5f * lat.sc[a] - 0.5f;
        // one voxel of slack on the support: u is evaluated in rounded fp32
        lat.elo[a] = fminf(-1.0f, -1.5f - 0.5f * cell);
        lat.ehi[a] = fmaxf((float)dims.d[a], (float)dims.d[a] + 0.5f + 0.5f * cell);
    }
    return lat;
}

// sample_range (ray_math.cuh) on the box [elo, ehi] instead of the padded volume: the march tests every y_m exactly, so the range
// only has to be a superset of the samples whose x_m lies in the box.  One sample of slack on both sides.
B200_HD void poly_sample_range(const PixLine& pl, const PolyLattice& lat, float amin, float range, int P, int& m_lo, int& m_hi)
{
    float lo = -INFINITY, hi = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float inv = 1.0f / pl.dp[a];
        const float a0 = (lat.elo[a] - pl.p0[a]) * inv, a1 = (lat.ehi[a] - pl.p0[a]) * inv;
        lo = fmaxf(lo, fminf(a0, a1));
        hi = fminf(hi, fmaxf(a0, a1));
    }
    if (!(range > 0.0f)) {  // degenerate range: march everything
        m_lo = 0;
        m_hi = P - 1;
        return;
    }
    if (!(lo <= hi)) {  // the line misses the box
        m_lo = 1;
        m_hi = 0;
        return;
    }
    const float scale = (float)(P - 1) / range;
    const float f_lo = floorf((lo - amin) * scale) - 1.0f, f_hi = ceilf((hi - amin) * scale) + 1.0f;
    m_lo = (int)fmaxf(0.0f, fminf(f_lo, (float)P));
    m_hi = (int)fminf((float)(P - 1), fmaxf(f_hi, -1.0f));
}

B200_HD float4 ldg4(const float4* p)
{
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// value and gradient (w.r.t. the fractions f) of the trilinear interpolant of 8 corner values, corner c = o0 | o1<<1 | o2<<2
B200_HD void tri_value_grad(const float v[8], const float f[3], float& val, float G[3])
{
    const float f0 = f[0], f1 = f[1], f2 = f[2];
    const float e0 = 1.0f - f0, e1 = 1.0f - f1;
    const float c00 = fmaf(f2, v[4] - v[0], v[0]), c10 = fmaf(f2, v[5] - v[1], v[1]);
    const float c01 = fmaf(f2, v[6] - v[2], v[2]), c11 = fmaf(f2, v[7] - v[3], v[3]);
    const float c0 = fmaf(f1, c01 - c00, c00), c1 = fmaf(f1, c11 - c10, c10);
    val = fmaf(f0, c1 - c0, c0);
    G[0] = c1 - c0;
    G[1] = e0 * (c01 - c00) + f0 * (c11 - c10);
    G[2] = e0 * (e1 * (v[4] - v[0]) + f1 * (v[6] - v[2])) + f0 * (e1 * (v[5] - v[1]) + f1 * (v[7] - v[3]));
}

// The KP blend weights at pix, and with GRAD their gradients w.r.t. pix.  false: pix is outside the lattice's support, every
// weight is zero and nothing was written.
template <int KP, bool GRAD>
B200_HD bool poly_weights(const PolyLattice& lat, const float pix[3], float w[KP], float gw[][3])
{
    float f[3];
    int i0[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float u = fmaf(pix[a], lat.sc[a], lat.of[a]);
        if (!(u > -1.0f && u < (float)lat.g[a])) return false;
        const float fl = floorf(u);
        f[a] = u - fl;
        i0[a] = (int)fl;
    }
    constexpr int Q = KP / 4;
    int off[8];  // the C ABI refuses a lattice of 2^31 floats or more
    unsigned mask = 0u;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int x = i0[0] + (c & 1), y = i0[1] + ((c >> 1) & 1), z = i0[2] + ((c >> 2) & 1);
        const bool inb = (unsigned)x < (unsigned)lat.g[0] && (unsigned)y < (unsigned)lat.g[1] && (unsigned)z < (unsigned)lat.g[2];
        off[c] = ((x * lat.g[1] + y) * lat.g[2] + z) * Q;
        mask |= inb ? (1u << c) : 0u;
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        float v[4][8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float4 t;
            t.x = t.y = t.z = t.w = 0.0f;
            if (mask & (1u << c)) t = ldg4(lat.w + off[c] + q);
            v[0][c] = t.x;
            v[1][c] = t.y;
            v[2][c] = t.z;
            v[3][c] = t.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float g[3];
            tri_value_grad(v[j], f, w[4 * q + j], g);
            if (GRAD) {
#pragma unroll
                for (int a = 0; a < 3; ++a) gw[4 * q + j][a] = g[a] * lat.sc[a];
            }
        }
    }
    return true;
}

// M_k [x; 1] - x
B200_HD void poly_offset(const float* Mk, const float x[3], float o[3])
{
#pragma unroll
    for (int i = 0; i < 3; ++i)
        o[i] = fmaf(Mk[4 * i], x[0], fmaf(Mk[4 * i + 1], x[1], fmaf(Mk[4 * i + 2], x[2], Mk[4 * i + 3]))) - x[i];
}

B200_HD bool inside_padded(const float pix[3], const VolDims& dims)
{
    return pix[0] > -1.0f && pix[1] > -1.0f && pix[2] > -1.0f && pix[0] < (float)dims.d[0] && pix[1] < (float)dims.d[1] &&
           pix[2] < (float)dims.d[2];  // false for a NaN, unlike !outside_padded
}

// sum over the samples of tri(V, y_m); multiply by raylen * step outside.  M: [KP][12], rows k >= K zero.
template <int KP, class Gather>
B200_HD float polyrigid_ray_fwd(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const float* M, const Ray& ray,
                                float shift, int P, float amin, float amax)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    const float kb = shift - 0.5f;  // pix = x + kb
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    float acc = 0.0f;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], w[KP];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        if (poly_weights<KP, false>(lat, pix, w, nullptr)) {
            const float x[3] = {pix[0] - kb, pix[1] - kb, pix[2] - kb};
            float disp[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int k = 0; k < KP; ++k) {
                float o[3];
                poly_offset(M + 12 * k, x, o);
#pragma unroll
                for (int a = 0; a < 3; ++a) disp[a] = fmaf(w[k], o[a], disp[a]);
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += disp[a];
        }
        float val = 0.0f;
        if (inside_padded(pix, dims)) val = lerp8(gather(dims, pix));
        acc += val;
    }
    return acc;
}

// Transpose of polyrigid_ray_fwd in the density (DESIGN.md 6o): polyrigid_ray_fwd's samples through the same arithmetic, each adding
//   g_vol[corner] += c tri_weight(corner, y_m)
// to the in-bounds corners of the cell around y_m, for every y_m inside the padded volume.  The cell, the fractions and the weight
// product are deform_ray_bproj's, so with w = 0 or identity maps every add is the Trilinear volume gradient's.  c = gout raylen step;
// no density is read.  M: the pose's K maps [K][12], read from global memory (no shared copy); rows k >= K read as zeros, the
// forward's zero-padded rows, so the blend's arithmetic is the forward's.
template <int KP>
B200_HD void polyrigid_ray_bproj(const VolDims& dims, const PolyLattice& lat, const float* M, int K, const Ray& ray, float shift, int P,
                                 float amin, float amax, float c, float* g_vol)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    const float kb = shift - 0.5f;  // pix = x + kb
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], w[KP];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        if (poly_weights<KP, false>(lat, pix, w, nullptr)) {
            const float x[3] = {pix[0] - kb, pix[1] - kb, pix[2] - kb};
            float disp[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int k = 0; k < KP; ++k) {
                float Mk[12], o[3];
#pragma unroll
                for (int e = 0; e < 12; ++e) Mk[e] = k < K ? ldg(M + 12 * k + e) : 0.0f;
                poly_offset(Mk, x, o);
#pragma unroll
                for (int a = 0; a < 3; ++a) disp[a] = fmaf(w[k], o[a], disp[a]);
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += disp[a];
        }
        if (!inside_padded(pix, dims)) continue;
        float f[3], e[3];
        int i0[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float fl = floorf(pix[a]);
            f[a] = pix[a] - fl;
            e[a] = 1.0f - f[a];
            i0[a] = (int)fl;
        }
        const int64_t base = ((int64_t)i0[0] * dims.d[1] + i0[1]) * dims.d[2] + i0[2];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int x = i0[0] + (q & 1), y = i0[1] + ((q >> 1) & 1), z = i0[2] + ((q >> 2) & 1);
            if ((unsigned)x < (unsigned)dims.d[0] && (unsigned)y < (unsigned)dims.d[1] && (unsigned)z < (unsigned)dims.d[2]) {
                const float wq = ((q & 1) ? f[0] : e[0]) * (((q >> 1) & 1) ? f[1] : e[1]) * (((q >> 2) & 1) ? f[2] : e[2]);
                red_add(g_vol + base + corner_off(dims, q), c * wq);
            }
        }
    }
}

// Closed-form backward of one ray (DESIGN.md 6h).  With G_m the interpolant's gradient at y_m and
//   J_m = 1 + sum_k w_k (R_k - 1) + sum_k (M_k [x_m; 1] - x_m) (x) grad w_k(x_m),          H_m = J_m^T G_m:
//   g_s = g L step sum (1 - alpha_m) H_m,   g_t = g L step sum alpha_m H_m,   g_L = g step sum V_m,
//   g_amin / g_amax: trilinear_ray_bwd_g's with G.dp replaced by H.dp,
//   dI/dM_k = A_k (x) [s; 1] + B_k (x) [d; 0],   A_k = L step sum w_k G_m,   B_k = L step sum alpha_m w_k G_m.
// AG / BG [KP][3] receive g * A_k and g * B_k (overwritten).
template <int KP, class Gather>
B200_HD TriGrad polyrigid_ray_bwd(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const float* M, const Ray& ray,
                                  float shift, int P, float amin, float amax, float g, float L, float AG[][3], float BG[][3])
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float step = range / (float)(P - 1);
    const float lstep = 1.0f / (float)(P - 1);
    const float kb = shift - 0.5f;
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    const float gLs = g * L * step;
    float sumV = 0.0f, S[3] = {0.0f, 0.0f, 0.0f}, T[3] = {0.0f, 0.0f, 0.0f}, E0 = 0.0f, E1 = 0.0f;
#pragma unroll
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) AG[k][a] = BG[k][a] = 0.0f;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float lin = linspace01(m, P, lstep);
        const float alpha = add_rn(mul_rn(lin, range), amin);
        float pix[3], x[3], w[KP], gw[KP][3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
            x[a] = pix[a] - kb;
        }
        const bool blended = poly_weights<KP, true>(lat, pix, w, gw);
        if (blended) {
            float disp[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int k = 0; k < KP; ++k) {
                float o[3];
                poly_offset(M + 12 * k, x, o);
#pragma unroll
                for (int a = 0; a < 3; ++a) disp[a] = fmaf(w[k], o[a], disp[a]);
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += disp[a];
        }
        if (!inside_padded(pix, dims)) continue;
        const Corner8 c8 = gather(dims, pix);
        float val, G[3], Hm[3];
        tri_value_grad(c8.v, c8.f, val, G);
        sumV += val;
#pragma unroll
        for (int a = 0; a < 3; ++a) Hm[a] = G[a];
        if (blended) {
#pragma unroll
            for (int k = 0; k < KP; ++k) {
                const float* Mk = M + 12 * k;
                float o[3];
                poly_offset(Mk, x, o);
                const float oG = o[0] * G[0] + o[1] * G[1] + o[2] * G[2];
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const float RtG = Mk[a] * G[0] + Mk[4 + a] * G[1] + Mk[8 + a] * G[2];
                    Hm[a] += w[k] * (RtG - G[a]) + gw[k][a] * oG;
                    const float wG = w[k] * G[a];
                    AG[k][a] += wG;
                    BG[k][a] = fmaf(alpha, wG, BG[k][a]);
                }
            }
        }
        float Hd = 0.0f;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            S[a] = fmaf(1.0f - alpha, Hm[a], S[a]);
            T[a] = fmaf(alpha, Hm[a], T[a]);
            Hd = fmaf(Hm[a], pl.dp[a], Hd);
        }
        E0 = fmaf(1.0f - lin, Hd, E0);
        E1 = fmaf(lin, Hd, E1);
    }
    TriGrad out;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        out.gs[a] = gLs * S[a];
        out.gt[a] = gLs * T[a];
    }
#pragma unroll
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            AG[k][a] *= gLs;
            BG[k][a] *= gLs;
        }
    out.sumV = sumV;
    const float gLv = g * L * sumV / (float)(P - 1);
    out.ga0 = -gLv + gLs * E0;
    out.ga1 = gLv + gLs * E1;
    return out;
}

// dI/dM_k of one ray from its A_k, B_k: e = 4 i + j -> A[i] [s; 1][j] + B[i] [d; 0][j]
B200_HD float poly_gM_entry(const float A[3], const float Bv[3], const Ray& ray, int e)
{
    const int i = e >> 2, j = e & 3;
    return j < 3 ? fmaf(A[i], ray.s[j], Bv[i] * ray.d[j]) : A[i];
}

// Per-pixel motion Jacobian of one ray (DESIGN.md 6j): polyrigid_ray_fwd's march, the same samples through the same arithmetic,
// so the returned sum is its result bit for bit, that also keeps, per in-volume sample,
//   A_k += w_k G_m,   B_k += alpha_m w_k G_m          (polyrigid_ray_bwd's A_k, B_k without the factor L step)
// and sets bit k of `touched` where w_k != 0.  The rays do not depend on the motions, so there are no camera or range terms.
template <int KP, class Gather>
B200_HD float polyrigid_ray_jac(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const float* M, const Ray& ray,
                                float shift, int P, float amin, float amax, float A[][3], float Bv[][3], unsigned& touched)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    const float kb = shift - 0.5f;
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
#pragma unroll
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) A[k][a] = Bv[k][a] = 0.0f;
    touched = 0u;
    float acc = 0.0f;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], w[KP];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        const bool blended = poly_weights<KP, false>(lat, pix, w, nullptr);
        if (blended) {
            const float x[3] = {pix[0] - kb, pix[1] - kb, pix[2] - kb};
            float disp[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int k = 0; k < KP; ++k) {
                float o[3];
                poly_offset(M + 12 * k, x, o);
#pragma unroll
                for (int a = 0; a < 3; ++a) disp[a] = fmaf(w[k], o[a], disp[a]);
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += disp[a];
        }
        // a sample outside the padded volume adds +0.0f in the forward, which leaves acc unchanged
        if (!inside_padded(pix, dims)) continue;
        const Corner8 c8 = gather(dims, pix);
        acc += lerp8(c8);
        if (!blended) continue;
        float val, G[3];
        tri_value_grad(c8.v, c8.f, val, G);
#pragma unroll
        for (int k = 0; k < KP; ++k) {
            touched |= w[k] != 0.0f ? 1u << k : 0u;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float wG = w[k] * G[a];
                A[k][a] += wG;
                Bv[k][a] = fmaf(alpha, wG, Bv[k][a]);
            }
        }
    }
    return acc;
}

// Column i of structure k for one ray: LS sum_e dI/dM_k[e] T_ki[e], dI/dM_k from A_k, B_k as poly_gM_entry lays it out and
// T_ki [12] = dM_k / d xi_ki (row-major 3 x 4), LS = L step.  So sum_n g_n J_n = g_M : T with g_M b200drr_polyrigid_bwd's.
B200_HD float poly_jac_entry(const float A[3], const float Bv[3], const Ray& ray, const float* Tki, float LS)
{
    float s = 0.0f;
#pragma unroll
    for (int e = 0; e < 12; ++e) s = fmaf(poly_gM_entry(A, Bv, ray, e), Tki[e], s);
    return LS * s;
}

}  // namespace b200drr
