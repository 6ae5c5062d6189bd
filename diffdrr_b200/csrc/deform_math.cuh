// deform_math.cuh -- per-ray math of the deformable (dense displacement field) trilinear march (host+device; DESIGN.md 6i).
//
// The rays and samples are the Trilinear renderer's: pix_m = p0 + alpha_m dp (ray_math.cuh: make_pixline, linspace01).  Every
// sample is pulled back through a displacement field u given on a coarse lattice over the volume (polyrigid_math.cuh's lattice:
// align_corners=False, zero outside the lattice), in voxel-index units:
//   y_m = x_m + u(x_m),      I = L step sum_m tri(V, y_m)
// The field is stored channel-last with 4 channels (u_0, u_1, u_2, 0), so a lattice node is one float4 and poly_weights<4>
// interpolates it.  With u = 0 the displacement is exactly 0.0f and the march is trilinear_ray_fwd bit for bit.
//
// The backward scatters d I / d u into a lattice gradient with one vector reduction per lattice node and flush (deform_red4): the
// field gradient repeats only to fp32 reordering of those adds.  Every other output is a per-ray value.  The tangent march
// (deform_ray_jvp) is the scatter's transpose: the image's derivative along a field direction, one value per ray.  The
// Jacobian march (deform_ray_jac) takes the transpose of that scatter for 6K tangents at once.  The
// backprojection (deform_ray_bproj) is the forward's transpose in the density: 8 scalar reductions per in-volume sample into a
// volume gradient, with no density read.
#pragma once

#include "polyrigid_math.cuh"

namespace b200drr {

// The lattice cell around pix, by poly_weights' own arithmetic: i0 = the cell's lower node per axis (-1 .. g - 1), f = the
// fractions in it.  false: pix is outside the lattice's support and nothing was written.
B200_HD bool deform_cell(const PolyLattice& lat, const float pix[3], int i0[3], float f[3])
{
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float u = fmaf(pix[a], lat.sc[a], lat.of[a]);
        if (!(u > -1.0f && u < (float)lat.g[a])) return false;
        const float fl = floorf(u);
        f[a] = u - fl;
        i0[a] = (int)fl;
    }
    return true;
}

// p[0..2] += (x, y, z): one red.global.add.v4.f32 on the device (p 16-byte aligned; lane 3 adds 0), plain adds in a host build
B200_HD void deform_red4(float* p, float x, float y, float z)
{
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(x), "f"(y), "f"(z), "f"(0.0f) : "memory");
#else
    p[0] += x;
    p[1] += y;
    p[2] += z;
#endif
}

// sum over the samples of tri(V, y_m); multiply by raylen * step outside.  lat.w: this pose's field [g0][g1][g2][4].
template <class Gather>
B200_HD float deform_ray_fwd(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const Ray& ray, float shift, int P,
                             float amin, float amax)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    float acc = 0.0f;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], u[4];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        if (poly_weights<4, false>(lat, pix, u, nullptr)) {
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += u[a];
        }
        float val = 0.0f;
        if (inside_padded(pix, dims)) val = lerp8(gather(dims, pix));
        acc += val;
    }
    return acc;
}

// Adds s * acc[c] to the 8 lattice nodes of the cell with lower node `cell` (the in-lattice ones); cell[0] < -1: nothing held.
B200_HD int deform_flush(const PolyLattice& lat, float* gfield, const int cell[3], const float acc[8][3], float s)
{
    if (cell[0] < -1) return 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int x = cell[0] + (c & 1), y = cell[1] + ((c >> 1) & 1), z = cell[2] + ((c >> 2) & 1);
        if ((unsigned)x < (unsigned)lat.g[0] && (unsigned)y < (unsigned)lat.g[1] && (unsigned)z < (unsigned)lat.g[2])
            deform_red4(gfield + 4 * ((x * lat.g[1] + y) * lat.g[2] + z), s * acc[c][0], s * acc[c][1], s * acc[c][2]);
    }
    return 1;
}

// Closed-form backward of one ray (DESIGN.md 6i).  With G_m the interpolant's gradient at y_m, J_m = 1 + grad u(x_m) and
// H_m = J_m^T G_m:
//   g_s = g L step sum (1 - alpha_m) H_m,   g_t = g L step sum alpha_m H_m,   g_L = g step sum V_m,
//   g_amin / g_amax: trilinear_ray_bwd_g's with G.dp replaced by H.dp,
//   g_u[node] += g L step tri_weight(node, x_m) G_m   for the 8 lattice nodes around x_m.
// The field term is summed in 8 x 3 registers while consecutive samples stay in one lattice cell and added to gfield
// ([g0][g1][g2][4], lane 3 left as it is) when the cell changes and at the end; gfield == nullptr skips it.  flushes: how many
// times the ray added its registers to gfield.
template <class Gather>
B200_HD TriGrad deform_ray_bwd(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const Ray& ray, float shift, int P,
                               float amin, float amax, float g, float L, float* gfield, int& flushes)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float step = range / (float)(P - 1);
    const float lstep = 1.0f / (float)(P - 1);
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    const float gLs = g * L * step;
    float sumV = 0.0f, S[3] = {0.0f, 0.0f, 0.0f}, T[3] = {0.0f, 0.0f, 0.0f}, E0 = 0.0f, E1 = 0.0f;
    float acc[8][3];
    int cell[3] = {-2, 0, 0};
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int a = 0; a < 3; ++a) acc[c][a] = 0.0f;
    flushes = 0;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float lin = linspace01(m, P, lstep);
        const float alpha = add_rn(mul_rn(lin, range), amin);
        float pix[3], u[4], gu[4][3], f[3];
        int i0[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        const bool moved = poly_weights<4, true>(lat, pix, u, gu);
        if (moved && gfield) deform_cell(lat, pix, i0, f);
        if (moved) {
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += u[a];
        }
        if (!inside_padded(pix, dims)) continue;
        const Corner8 c8 = gather(dims, pix);
        float val, G[3], Hm[3];
        tri_value_grad(c8.v, c8.f, val, G);
        sumV += val;
#pragma unroll
        for (int a = 0; a < 3; ++a) Hm[a] = moved ? G[a] + (gu[0][a] * G[0] + gu[1][a] * G[1] + gu[2][a] * G[2]) : G[a];
        float Hd = 0.0f;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            S[a] = fmaf(1.0f - alpha, Hm[a], S[a]);
            T[a] = fmaf(alpha, Hm[a], T[a]);
            Hd = fmaf(Hm[a], pl.dp[a], Hd);
        }
        E0 = fmaf(1.0f - lin, Hd, E0);
        E1 = fmaf(lin, Hd, E1);
        if (moved && gfield) {
            if (i0[0] != cell[0] || i0[1] != cell[1] || i0[2] != cell[2]) {
                flushes += deform_flush(lat, gfield, cell, acc, gLs);
#pragma unroll
                for (int a = 0; a < 3; ++a) cell[a] = i0[a];
#pragma unroll
                for (int c = 0; c < 8; ++c)
#pragma unroll
                    for (int a = 0; a < 3; ++a) acc[c][a] = 0.0f;
            }
            const float e[3] = {1.0f - f[0], 1.0f - f[1], 1.0f - f[2]};
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const float w = ((c & 1) ? f[0] : e[0]) * ((c & 2) ? f[1] : e[1]) * ((c & 4) ? f[2] : e[2]);
#pragma unroll
                for (int a = 0; a < 3; ++a) acc[c][a] = fmaf(w, G[a], acc[c][a]);
            }
        }
    }
    if (gfield) flushes += deform_flush(lat, gfield, cell, acc, gLs);
    TriGrad out;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        out.gs[a] = gLs * S[a];
        out.gt[a] = gLs * T[a];
    }
    out.sumV = sumV;
    const float gLv = g * L * sumV / (float)(P - 1);
    out.ga0 = -gLv + gLs * E0;
    out.ga1 = gLv + gLs * E1;
    return out;
}

// Directional derivative of one ray along a field tangent v (DESIGN.md 6k): deform_ray_fwd's march, the same samples through the
// same arithmetic, that also sums
//   jv = sum_m G_m . v(x_m),      G_m = grad tri(V)(y_m)
// over exactly the samples where deform_ray_bwd adds its field term (x_m inside the lattice's support, y_m inside the padded
// volume), so L step jv is the transpose of that scatter.  tan: lat's geometry, w = this pose's tangent [g0][g1][g2][4] (lane 3
// ignored).  img receives the forward's sum bit for bit (a skipped sample adds +0.0f there, which leaves it unchanged).  Multiply
// both by raylen * step outside.
template <class Gather>
B200_HD float deform_ray_jvp(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const PolyLattice& tan, const Ray& ray,
                             float shift, int P, float amin, float amax, float& img)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    float acc = 0.0f, jv = 0.0f;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], u[4], v[4];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        const bool moved = poly_weights<4, false>(lat, pix, u, nullptr);
        if (moved) {
            poly_weights<4, false>(tan, pix, v, nullptr);
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += u[a];
        }
        if (!inside_padded(pix, dims)) continue;
        const Corner8 c8 = gather(dims, pix);
        acc += lerp8(c8);
        if (!moved) continue;
        float val, G[3];
        tri_value_grad(c8.v, c8.f, val, G);
        jv = fmaf(G[0], v[0], fmaf(G[1], v[1], fmaf(G[2], v[2], jv)));
    }
    img = acc;
    return jv;
}

// Contracts the register accumulator of deform_ray_jac with the tangents at the in-lattice corners of the cell with lower node `cell`:
// Jp[p] += sum_c <acc[c], t_p(c)> for p < 6K, tan = this pose's tangents [g0][g1][g2][6K] float4 (lane 3 ignored), and sets bit k of
// touched when one of structure k's six tangents is nonzero at such a corner.  cell[0] < -1: nothing held.
template <int KP>
B200_HD int deform_jac_flush(const PolyLattice& lat, const float4* tan, int K, const int cell[3], const float acc[8][3],
                             float Jp[KP * 6], unsigned& touched)
{
    if (cell[0] < -1) return 0;
    const int P = 6 * K;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int x = cell[0] + (c & 1), y = cell[1] + ((c >> 1) & 1), z = cell[2] + ((c >> 2) & 1);
        if (!((unsigned)x < (unsigned)lat.g[0] && (unsigned)y < (unsigned)lat.g[1] && (unsigned)z < (unsigned)lat.g[2])) continue;
        const float4* t = tan + (int64_t)((x * lat.g[1] + y) * lat.g[2] + z) * P;
#pragma unroll
        for (int p = 0; p < KP * 6; ++p) {
            if (p >= P) break;
            const float4 v = ldg4(t + p);
            Jp[p] = fmaf(acc[c][0], v.x, fmaf(acc[c][1], v.y, fmaf(acc[c][2], v.z, Jp[p])));
            if (v.x != 0.0f || v.y != 0.0f || v.z != 0.0f) touched |= 1u << (p / 6);
        }
    }
    return 1;
}

// Per-pixel Jacobian of one ray along the 6K field tangents of K structures' motions (DESIGN.md 6p): deform_ray_jvp's samples,
// through the same arithmetic, for all 6K tangents at once,
//   Jp[p] = sum_m G_m . t_p(x_m),      G_m = grad tri(V)(y_m),
// over exactly the samples where deform_ray_jvp adds.  t_p is not interpolated per sample: as deform_ray_bwd's field scatter,
// acc[c] += w_c(x_m) G_m is summed in 8 x 3 registers while consecutive samples stay in one lattice cell, and contracted with the
// tangents at the cell's corners when the cell changes and at the end (deform_jac_flush), so sum_n gout_n L step Jp_n is <g_field
// of deform_ray_bwd, t_p> to fp32 reordering.  touched: bit k set when a contraction met a nonzero tangent of structure k.
// -> deform_ray_fwd's sum bit for bit.  Multiply it and Jp by raylen * step outside.  flushes: the contractions made.
template <int KP, class Gather>
B200_HD float deform_ray_jac(const Gather& gather, const VolDims& dims, const PolyLattice& lat, const float4* tan, int K, const Ray& ray,
                             float shift, int P, float amin, float amax, float Jp[KP * 6], unsigned& touched, int& flushes)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    float img = 0.0f, acc[8][3];
    int cell[3] = {-2, 0, 0};
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int a = 0; a < 3; ++a) acc[c][a] = 0.0f;
#pragma unroll
    for (int p = 0; p < KP * 6; ++p) Jp[p] = 0.0f;
    touched = 0u;
    flushes = 0;
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], u[4], f[3];
        int i0[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        const bool moved = poly_weights<4, false>(lat, pix, u, nullptr);
        if (moved) {
            deform_cell(lat, pix, i0, f);
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += u[a];
        }
        if (!inside_padded(pix, dims)) continue;
        const Corner8 c8 = gather(dims, pix);
        img += lerp8(c8);
        if (!moved) continue;
        float val, G[3];
        tri_value_grad(c8.v, c8.f, val, G);
        if (i0[0] != cell[0] || i0[1] != cell[1] || i0[2] != cell[2]) {
            flushes += deform_jac_flush<KP>(lat, tan, K, cell, acc, Jp, touched);
#pragma unroll
            for (int a = 0; a < 3; ++a) cell[a] = i0[a];
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int a = 0; a < 3; ++a) acc[c][a] = 0.0f;
        }
        const float e[3] = {1.0f - f[0], 1.0f - f[1], 1.0f - f[2]};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float w = ((c & 1) ? f[0] : e[0]) * ((c & 2) ? f[1] : e[1]) * ((c & 4) ? f[2] : e[2]);
#pragma unroll
            for (int a = 0; a < 3; ++a) acc[c][a] = fmaf(w, G[a], acc[c][a]);
        }
    }
    flushes += deform_jac_flush<KP>(lat, tan, K, cell, acc, Jp, touched);
    return img;
}

// Transpose of deform_ray_fwd in the density (DESIGN.md 6l): deform_ray_fwd's samples, through the same arithmetic, each adding
//   g_vol[corner] += c tri_weight(corner, y_m)
// to the in-bounds corners of the cell around y_m, for every y_m inside the padded volume (x_m inside the lattice's support or
// not: u = 0 there and y_m = x_m).  The cell and the fractions are gather8's, the weights trilinear_ray_bwd_g's product, so with
// u = 0 every add is that kernel's volume-gradient add bit for bit.  c = gout raylen step; no density is read.
B200_HD void deform_ray_bproj(const VolDims& dims, const PolyLattice& lat, const Ray& ray, float shift, int P, float amin, float amax,
                              float c, float* g_vol)
{
    const PixLine pl = make_pixline(ray, dims, shift, 0);
    const float range = amax - amin;
    const float lstep = 1.0f / (float)(P - 1);
    int m_lo, m_hi;
    poly_sample_range(pl, lat, amin, range, P, m_lo, m_hi);
    for (int m = m_lo; m <= m_hi; ++m) {
        const float alpha = add_rn(mul_rn(linspace01(m, P, lstep), range), amin);
        float pix[3], u[4];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = fmaf(alpha, pl.dp[a], pl.p0[a]);
        if (poly_weights<4, false>(lat, pix, u, nullptr)) {
#pragma unroll
            for (int a = 0; a < 3; ++a) pix[a] += u[a];
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
        for (int k = 0; k < 8; ++k) {
            const int x = i0[0] + (k & 1), y = i0[1] + ((k >> 1) & 1), z = i0[2] + ((k >> 2) & 1);
            if ((unsigned)x < (unsigned)dims.d[0] && (unsigned)y < (unsigned)dims.d[1] && (unsigned)z < (unsigned)dims.d[2]) {
                const float w = ((k & 1) ? f[0] : e[0]) * (((k >> 1) & 1) ? f[1] : e[1]) * (((k >> 2) & 1) ? f[2] : e[2]);
                red_add(g_vol + base + corner_off(dims, k), c * w);
            }
        }
    }
}

}  // namespace b200drr
