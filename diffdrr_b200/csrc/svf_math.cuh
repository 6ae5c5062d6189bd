// svf_math.cuh -- per-node math of the scaling-and-squaring exponential of a stationary velocity field (host+device; DESIGN.md 6m).
//
// The field is deform_math.cuh's: [Bf][g0][g1][g2][4] fp32, voxel-index units, lane 3 zero, node i of axis a at voxel coordinate
// (i + 1/2) D_a / g_a - 1/2 (make_lattice's sc / of).  One squaring step maps u to
//   u'(x) = s u(x) + s U(y),      y = x + s u(x),
// U the trilinear interpolant of u with lattice coordinates CLAMPED to the node range [0, g_a - 1] per axis (not poly_weights'
// zero outside: a zero lookup beyond the border folds the composed map there).  s = 1 / 2^N on the first step, which folds
// u_0 = v / 2^N into it, and 1 on the others.  At node x the lattice coordinate of y is i_a + s u_a sc_a.
//
// The adjoint of a step, for an upstream gradient g' on u', adds
//   s g'(x) + s^2 J_U(y)^T g'(x)        to node x,
//   s w_c(y) g'(x)                      to each corner node c of the cell around y,
// J_U the interpolant's spatial gradient (voxel units), zero along an axis where the clamp is active.  Every add is a vector
// reduction (deform_red4), so the gradient repeats only to fp32 reordering.
#pragma once

#include "deform_math.cuh"

namespace b200drr {

// The cell of the clamped lookup at lattice coordinate q (per axis): lower node i0, upper node i1 (= i0 when g == 1), fraction f,
// and live[a] = 0 where q lies outside [0, g_a - 1] (the clamp is active and the lookup is constant along that axis).
struct SvfCell {
    int i0[3], i1[3];
    float f[3], live[3];
};

B200_HD SvfCell svf_cell(const PolyLattice& lat, const float q[3])
{
    SvfCell c;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float hi = (float)(lat.g[a] - 1);
        const float qc = fminf(fmaxf(q[a], 0.0f), hi);
        c.live[a] = (q[a] >= 0.0f && q[a] <= hi) ? 1.0f : 0.0f;
        int i0 = (int)floorf(qc);
        if (i0 > lat.g[a] - 2) i0 = lat.g[a] > 1 ? lat.g[a] - 2 : 0;  // q = g - 1 sits in the last cell with f = 1
        c.i0[a] = i0;
        c.i1[a] = i0 + 1 < lat.g[a] ? i0 + 1 : i0;
        c.f[a] = qc - (float)i0;
    }
    return c;
}

B200_HD int64_t svf_node(const PolyLattice& lat, int x, int y, int z) { return ((int64_t)x * lat.g[1] + y) * lat.g[2] + z; }

// U(q) and, with GRAD, J[i][a] = dU_i / dy_a in voxel units (zero along a clamped axis).  lat.w: this pose's field.
template <bool GRAD>
B200_HD void svf_lookup(const PolyLattice& lat, const SvfCell& c, float U[3], float J[3][3])
{
    float v[3][8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float4 t = ldg4(lat.w + svf_node(lat, (k & 1) ? c.i1[0] : c.i0[0], (k & 2) ? c.i1[1] : c.i0[1], (k & 4) ? c.i1[2] : c.i0[2]));
        v[0][k] = t.x;
        v[1][k] = t.y;
        v[2][k] = t.z;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float G[3];
        tri_value_grad(v[i], c.f, U[i], G);
        if (GRAD) {
#pragma unroll
            for (int a = 0; a < 3; ++a) J[i][a] = G[a] * lat.sc[a] * c.live[a];
        }
    }
}

// The lattice coordinate of y = x + s u(x) for node (x0, x1, x2)
B200_HD void svf_target(const PolyLattice& lat, const int node[3], const float4 u, float s, float q[3])
{
    q[0] = fmaf(s * u.x, lat.sc[0], (float)node[0]);
    q[1] = fmaf(s * u.y, lat.sc[1], (float)node[1]);
    q[2] = fmaf(s * u.z, lat.sc[2], (float)node[2]);
}

// One squaring step at one node: -> u'(x) (lane 3 zero)
B200_HD float4 svf_square_node(const PolyLattice& lat, const int node[3], float s)
{
    const float4 u = ldg4(lat.w + svf_node(lat, node[0], node[1], node[2]));
    float q[3], U[3];
    svf_target(lat, node, u, s, q);
    svf_lookup<false>(lat, svf_cell(lat, q), U, nullptr);
    float4 o;
    o.x = s * (u.x + U[0]);
    o.y = s * (u.y + U[1]);
    o.z = s * (u.z + U[2]);
    o.w = 0.0f;
    return o;
}

// The adjoint of one squaring step at one node: adds node (x0, x1, x2)'s share of g'(x) = gp to gin (this pose's [g0][g1][g2][4])
B200_HD void svf_square_node_bwd(const PolyLattice& lat, const int node[3], float s, const float4 gp, float* gin)
{
    const float4 u = ldg4(lat.w + svf_node(lat, node[0], node[1], node[2]));
    float q[3], U[3], J[3][3];
    svf_target(lat, node, u, s, q);
    const SvfCell c = svf_cell(lat, q);
    svf_lookup<true>(lat, c, U, J);
    const float g[3] = {gp.x, gp.y, gp.z};
    const float ss = s * s;
    float h[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) h[a] = fmaf(ss, fmaf(J[0][a], g[0], fmaf(J[1][a], g[1], J[2][a] * g[2])), s * g[a]);
    deform_red4(gin + 4 * svf_node(lat, node[0], node[1], node[2]), h[0], h[1], h[2]);
    const float e[3] = {1.0f - c.f[0], 1.0f - c.f[1], 1.0f - c.f[2]};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float w = s * ((k & 1) ? c.f[0] : e[0]) * ((k & 2) ? c.f[1] : e[1]) * ((k & 4) ? c.f[2] : e[2]);
        if (w == 0.0f) continue;  // an exact zero adds nothing
        const int64_t n = svf_node(lat, (k & 1) ? c.i1[0] : c.i0[0], (k & 2) ? c.i1[1] : c.i0[1], (k & 4) ? c.i1[2] : c.i0[2]);
        deform_red4(gin + 4 * n, w * g[0], w * g[1], w * g[2]);
    }
}

// The tangent of one squaring step at one node: for a tangent t on u (lat_t: this pose's tangent, lat_u's geometry), -> t'(x) =
//   s t(x) + s^2 J_U(y) t(x) + s sum_c w_c(y) t(c)          (lane 3 zero),
// y, its cell and J_U those of svf_square_node_bwd, one cell for u and for t: term by term the transpose of that adjoint, and no
// reductions, so the tangent repeats bit for bit.  out_u (nullable) receives u'(x) by svf_square_node's own arithmetic.
B200_HD float4 svf_square_node_jvp(const PolyLattice& lat_u, const PolyLattice& lat_t, const int node[3], float s, float4* out_u)
{
    const int64_t x = svf_node(lat_u, node[0], node[1], node[2]);
    const float4 u = ldg4(lat_u.w + x);
    const float4 tx = ldg4(lat_t.w + x);
    float q[3], U[3], J[3][3], T[3];
    svf_target(lat_u, node, u, s, q);
    const SvfCell c = svf_cell(lat_u, q);
    svf_lookup<true>(lat_u, c, U, J);
    svf_lookup<false>(lat_t, c, T, nullptr);   // sum_c w_c(y) t(c)
    if (out_u) *out_u = svf_square_node(lat_u, node, s);
    const float t[3] = {tx.x, tx.y, tx.z};
    const float ss = s * s;
    float o[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) o[i] = fmaf(ss, fmaf(J[i][0], t[0], fmaf(J[i][1], t[1], J[i][2] * t[2])), s * (t[i] + T[i]));
    float4 r;
    r.x = o[0];
    r.y = o[1];
    r.z = o[2];
    r.w = 0.0f;
    return r;
}

// svf_square_node_jvp for P tangents at once (DESIGN.md 6p).  tan: this pose's tangents, node-major [g0][g1][g2][P] float4; tout
// receives node x's P results [P] float4.  y, its cell and J_U depend only on u, so they are formed once per node; the per-tangent
// arithmetic is svf_square_node_jvp's in the same order, so slice p equals that function on tangent p bit for bit.  out_u as there.
B200_HD void svf_square_node_tangents(const PolyLattice& lat_u, const float4* tan, int P, const int node[3], float s, float4* tout,
                                      float4* out_u)
{
    const int64_t x = svf_node(lat_u, node[0], node[1], node[2]);
    const float4 u = ldg4(lat_u.w + x);
    float q[3], U[3], J[3][3];
    svf_target(lat_u, node, u, s, q);
    const SvfCell c = svf_cell(lat_u, q);
    svf_lookup<true>(lat_u, c, U, J);
    if (out_u) *out_u = svf_square_node(lat_u, node, s);
    int64_t corner[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
        corner[k] = svf_node(lat_u, (k & 1) ? c.i1[0] : c.i0[0], (k & 2) ? c.i1[1] : c.i0[1], (k & 4) ? c.i1[2] : c.i0[2]) * P;
    const float ss = s * s;
    for (int p = 0; p < P; ++p) {
        const float4 tx = ldg4(tan + x * P + p);
        float v[3][8], T[3], G[3];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float4 t = ldg4(tan + corner[k] + p);
            v[0][k] = t.x;
            v[1][k] = t.y;
            v[2][k] = t.z;
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) tri_value_grad(v[i], c.f, T[i], G);
        const float t[3] = {tx.x, tx.y, tx.z};
        float o[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) o[i] = fmaf(ss, fmaf(J[i][0], t[0], fmaf(J[i][1], t[1], J[i][2] * t[2])), s * (t[i] + T[i]));
        float4 r;
        r.x = o[0];
        r.y = o[1];
        r.z = o[2];
        r.w = 0.0f;
        tout[p] = r;
    }
}

}  // namespace b200drr
