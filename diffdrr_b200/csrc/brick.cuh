// brick.cuh -- per-(ray, brick) logic of the brick-major Siddon kernels (siddon_brick.cu).
//
// Brick-major scheduling: a CTA owns one BX x BY x BZ voxel brick, staged in shared memory by ONE TMA box copy
// (cp.async.bulk.tensor.3d, zero fill outside the volume), and integrates over it every ray of every pose of the batch
// whose line crosses it; the partial line integrals are combined with red.global.add.  A voxel fetched once from L2
// then serves ~0.4 visits per pose x all poses of the batch from shared memory, instead of one 32-byte sector per
// visit from L1/L2 (the limit of the slab-major kernels, DESIGN.md 4.1).
//
// Everything in this header is host+device code so tests/hostemu can run the same decomposition (brick loop, detector
// rectangle of a brick, hit test, per-pair walk) on the CPU against the oracle; the TMA / mbarrier / sorting machinery
// is device-only and lives in siddon_brick.cu.  Replaces reference renderers.py:94-113 (+156-169) on this path.
#pragma once

#include "ray_math.cuh"

namespace b200drr {

// Per-pose detector geometry in voxel-index space, derived from three corner rays of the full H x W grid (the grid is
// affine in the pixel indices: detector.py:105-132 builds it as a cartesian product).  For a point X, the line
// source->X meets the detector plane at pixel (u, v):  t = num / (n . (X - S)),  rel = (S - O) + t (X - S),
// u = rel . A,  v = rel . Bv.
struct PoseGeo {
    float S[3];   // source
    float n[3];   // eu x ev (plane normal, not normalised)
    float num;    // n . (O - S);  NaN marks a degenerate grid (H or W == 1): no rectangle can be derived
    float A[3];   // (ev x n) / |n|^2
    float Bv[3];  // (n x eu) / |n|^2
    float O[3];   // target of pixel (0, 0)
};

B200_HD void cross3(const float a[3], const float b[3], float c[3])
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// t00 / t0w / th0: targets of pixels (row 0, col 0), (row 0, col W-1), (row H-1, col 0)
B200_HD PoseGeo make_pose_geo(const float s[3], const float t00[3], const float t0w[3], const float th0[3], int H, int W)
{
    PoseGeo g;
    float eu[3], ev[3], os[3];
    const float iu = W > 1 ? 1.0f / (float)(W - 1) : 0.0f, iv = H > 1 ? 1.0f / (float)(H - 1) : 0.0f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        eu[a] = (t0w[a] - t00[a]) * iu;
        ev[a] = (th0[a] - t00[a]) * iv;
        g.S[a] = s[a];
        g.O[a] = t00[a];
        os[a] = t00[a] - s[a];
    }
    cross3(eu, ev, g.n);
    const float nn = g.n[0] * g.n[0] + g.n[1] * g.n[1] + g.n[2] * g.n[2];
    g.num = g.n[0] * os[0] + g.n[1] * os[1] + g.n[2] * os[2];
    float en[3], ne[3];
    cross3(ev, g.n, en);
    cross3(g.n, eu, ne);
    const float inn = 1.0f / nn;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        g.A[a] = en[a] * inn;
        g.Bv[a] = ne[a] * inn;
    }
    if (!(nn > 0.0f) || H < 2 || W < 2) g.num = NAN;
    return g;
}

// Projection of one brick corner: pixel coordinates (u, v) and the denominator n . (X - S).
B200_HD void project_corner(const PoseGeo& g, const float X[3], float& u, float& v, float& den)
{
    float w[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) w[a] = X[a] - g.S[a];
    den = g.n[0] * w[0] + g.n[1] * w[1] + g.n[2] * w[2];
    const float t = g.num / den;
    float rel[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) rel[a] = (g.S[a] - g.O[a]) + t * w[a];
    u = rel[0] * g.A[0] + rel[1] * g.A[1] + rel[2] * g.A[2];
    v = rel[0] * g.Bv[0] + rel[1] * g.Bv[1] + rel[2] * g.Bv[2];
}

struct PixRect {
    int x0, y0, x1, y1;  // inclusive; x0 > x1 = empty
};

// Pixel rectangle that certainly contains every pixel whose LINE (quirk Q1: Siddon integrates the infinite line,
// renderers.py:97-113) meets the box: bounding box of the 8 projected corners +- 1 pixel when the box stays on one
// side of the plane through the source parallel to the detector (a projective map keeps a convex set convex there);
// otherwise -- or when a corner comes close to that plane -- the whole detector.
B200_HD PixRect rect_from_extents(float umin, float umax, float vmin, float vmax, float dmin, float dmax, int H, int W)
{
    PixRect r;
    const float lo = fminf(fabsf(dmin), fabsf(dmax)), hi = fmaxf(fabsf(dmin), fabsf(dmax));
    const bool one_side = (dmin > 0.0f) || (dmax < 0.0f);
    const bool ok = one_side && (lo >= 1e-3f * hi) && (umin <= umax) && (vmin <= vmax);  // false for NaN as well
    if (!ok) {
        r.x0 = 0; r.y0 = 0; r.x1 = W - 1; r.y1 = H - 1;
        return r;
    }
    const float fx0 = floorf(umin) - 1.0f, fx1 = ceilf(umax) + 1.0f, fy0 = floorf(vmin) - 1.0f, fy1 = ceilf(vmax) + 1.0f;
    if (fx1 < 0.0f || fy1 < 0.0f || fx0 > (float)(W - 1) || fy0 > (float)(H - 1)) {
        r.x0 = 1; r.x1 = 0; r.y0 = 1; r.y1 = 0;  // projects off the detector
        return r;
    }
    r.x0 = (int)fmaxf(fx0, 0.0f);
    r.y0 = (int)fmaxf(fy0, 0.0f);
    r.x1 = (int)fminf(fx1, (float)(W - 1));
    r.y1 = (int)fminf(fy1, (float)(H - 1));
    return r;
}

B200_HD PixRect brick_rect(const PoseGeo& g, const int lo_v[3], const int hi_v[3], float shift, int H, int W)
{
    float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY, dmin = INFINITY, dmax = -INFINITY;
    for (int c = 0; c < 8; ++c) {
        const float X[3] = {(float)((c & 1) ? hi_v[0] : lo_v[0]) - shift, (float)((c & 2) ? hi_v[1] : lo_v[1]) - shift,
                            (float)((c & 4) ? hi_v[2] : lo_v[2]) - shift};
        float u, v, den;
        project_corner(g, X, u, v, den);
        // NaN-propagating min / max: a NaN corner must invalidate the rectangle (fminf would drop it)
        umin = (u < umin || u != u) ? u : umin;
        umax = (u > umax || u != u) ? u : umax;
        vmin = (v < vmin || v != v) ? v : vmin;
        vmax = (v > vmax || v != v) ? v : vmax;
        dmin = (den < dmin || den != den) ? den : dmin;
        dmax = (den > dmax || den != den) ? den : dmax;
    }
    return rect_from_extents(umin, umax, vmin, vmax, dmin, dmax, H, W);
}

// Column range [umin, umax] of the brick's projected outline inside the pixel-row band [vb0, vb1] (already widened by
// the caller's margin): the outline is the convex hull of the 8 projected corners and its edges are projections of box
// edges, so the extent over a band is attained at a corner inside the band or where one of the 12 box edges meets a band
// boundary.  uv = {u0, v0, u1, v1, ...} in corner order (bit 0/1/2 of the index = high face of axis 0/1/2).
// Returns false when the band misses the outline.
B200_HD bool band_extent(const float* uv, float vb0, float vb1, float& umin, float& umax)
{
    umin = INFINITY;
    umax = -INFINITY;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float u = uv[2 * c], v = uv[2 * c + 1];
        if (v >= vb0 && v <= vb1) {
            umin = fminf(umin, u);
            umax = fmaxf(umax, u);
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
#pragma unroll
        for (int bit = 1; bit < 8; bit <<= 1) {
            if (c & bit) continue;  // each edge once: c has the bit clear, its partner has it set
            const float u1 = uv[2 * c], v1 = uv[2 * c + 1], u2 = uv[2 * (c | bit)], v2 = uv[2 * (c | bit) + 1];
            const float dv = v2 - v1;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float vb = k == 0 ? vb0 : vb1;
                if ((v1 - vb) * (v2 - vb) <= 0.0f && dv != 0.0f) {
                    const float t = (vb - v1) / dv;
                    const float u = fmaf(t, u2 - u1, u1);
                    umin = fminf(umin, u);
                    umax = fmaxf(umax, u);
                }
            }
        }
    }
    return umin <= umax;
}

// Pixel columns [px_lo, px_hi] of the 4-row tile band starting at row py0 that can hold hits of the brick: the outline's
// extent over rows [py0 - 1, py0 + 4] (one pixel of margin, as for the rectangle) widened by one pixel and clipped to the
// rectangle; the whole rectangle width when the projection is not valid (`outline_ok` false).  False = no candidates.
B200_HD bool row_span(const float* uv, bool outline_ok, const PixRect& rc, int py0, int& px_lo, int& px_hi)
{
    px_lo = rc.x0;
    px_hi = rc.x1;
    if (!outline_ok) return true;
    float umin, umax;
    if (!band_extent(uv, (float)(py0 - 1), (float)(py0 + 4), umin, umax)) return false;
    const float flo = fmaxf(floorf(umin) - 1.0f, (float)rc.x0), fhi = fminf(ceilf(umax) + 1.0f, (float)rc.x1);
    if (!(flo <= fhi)) return false;
    px_lo = (int)flo;
    px_hi = (int)fhi;
    return true;
}

// True when rect_from_extents derived the rectangle from the projected corners (false = whole-detector fallback).
B200_HD bool outline_valid(float umin, float umax, float vmin, float vmax, float dmin, float dmax)
{
    const float lo = fminf(fabsf(dmin), fabsf(dmax)), hi = fmaxf(fabsf(dmin), fabsf(dmax));
    const bool one_side = (dmin > 0.0f) || (dmax < 0.0f);
    return one_side && (lo >= 1e-3f * hi) && (umin <= umax) && (vmin <= vmax);
}

// Conservative (ray, box) test from the ray-table entry: the same expressions as box_surely_missed with the
// per-(pose, box) constants clo = (lo - shift) - s, chi = (hi - shift) - s hoisted.  Returns false only when the line
// certainly misses; a_in / a_out feed the step estimate the work list is sorted by.
B200_HD bool brick_maybe_hit(const float inv[3], const float clo[3], const float chi[3], float& a_in, float& a_out)
{
    a_in = -INFINITY;
    a_out = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float a0 = clo[a] * inv[a], a1 = chi[a] * inv[a];
        a_in = fmaxf(a_in, fminf(a0, a1));
        a_out = fminf(a_out, fmaxf(a0, a1));
    }
    const float margin = 1e-4f * (1.0f + fabsf(a_in) + fabsf(a_out));
    return !(a_in > a_out + margin);
}

// Work item: bin (5 bits) | pose within the chunk (5 bits) | ray index within the pose (22 bits: up to 2048 x 2048 rays).
// Band descriptor (same word layout, different fields): pose (5 bits) | first row (11 bits) | first column (11 bits).
constexpr int kBrickPoseChunk = 32;
constexpr int kBrickMaxSide = 2048;
constexpr int kBrickBins = 32;
B200_HD unsigned pack_item(int bin, int bl, int n) { return ((unsigned)bin << 27) | ((unsigned)bl << 22) | (unsigned)n; }
B200_HD int item_bin(unsigned it) { return (int)(it >> 27); }
B200_HD int item_pose(unsigned it) { return (int)((it >> 22) & 31u); }
B200_HD int item_ray(unsigned it) { return (int)(it & 0x3fffffu); }
B200_HD unsigned pack_band(int bl, int py, int px) { return ((unsigned)bl << 22) | ((unsigned)py << 11) | (unsigned)px; }
B200_HD int band_row(unsigned it) { return (int)((it >> 11) & 2047u); }
B200_HD int band_col(unsigned it) { return (int)(it & 2047u); }

// Estimated number of voxels a hit visits inside the box -> sort bin (longest first keeps the lanes of a warp alike)
B200_HD int step_bin(float a_in, float a_out, float sumabs_d, float inv_width)
{
    float est = (a_out - a_in) * sumabs_d;      // L1 length of the chord in voxels
    est = fminf(fmaxf(est, 0.0f), 4096.0f);     // NaN -> 0
    const int b = (int)(est * inv_width);
    return b < kBrickBins - 1 ? b : kBrickBins - 1;
}

// Host emulation loader: the brick is a plain array, offsets are element offsets.
// V = the staged voxel type (float, or a 16-bit VoxF16 / VoxBF16 widened by ldg).
template <class V>
struct LdHostT {
    const V* brick;
    static constexpr int kScale = 1;
    B200_HD int base() const { return 0; }
    B200_HD float operator()(int off) const { return ldg(brick + off); }
};
using LdHost = LdHostT<float>;

// Line integral (sum of v * dalpha) of one ray over the voxels [lo_v, hi_v) of a brick whose voxel (org) sits at element
// 0 of the staged copy with element strides (st0, st1, st2).  Same walk, same order, same rounding as
// siddon_ray_lean_box; only the loads differ (shared memory instead of global).
template <int U, class Ld>
B200_HD float brick_pair_fwd(const Ld& ld, const Ray& ray, const int lo_v[3], const int hi_v[3], const int org[3], int st0,
                             int st1, int st2, float shift)
{
    const Walk w = start_walk_box(ray, lo_v, hi_v, shift);
    if (!w.hit) return 0.0f;
    LeanConst k;
    LeanState s;
    lean_init(w, st0 * Ld::kScale, st1 * Ld::kScale, st2 * Ld::kScale, s, k);
    s.off += ld.base() - (org[0] * st0 + org[1] * st1 + org[2] * st2) * Ld::kScale;
    float acc = 0.0f;
    while (s.acur < k.a_out) {
        float len[U], v[U];
        int offs[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
            offs[j] = s.off;
            len[j] = lean_step(s, k);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) v[j] = ld(offs[j]);
#pragma unroll
        for (int j = 0; j < U; ++j) acc = fmaf(len[j], v[j], acc);
    }
    return acc;
}


// ---- lean per-pair path (production): set-up without the entry-voxel fix-ups, accumulated crossing alphas ---------------
// A slimmer set-up than start_walk_box: the start voxel is floor(position), corrected by at most one step so that it
// agrees with the order of the crossing alphas (see below); ties within one ulp of alpha may fall either way -- that only
// re-attributes a segment of ~1e-7 in alpha in the forward sum (the backward pass needs start_walk_frame's exact order).
// Crossing alphas are accumulated with ROUND-UP additions (an = add.rp(an, |1/d|)) from an anchor that is exact per
// brick, and the stop alpha is the exit plane's alpha ROUNDED DOWN (fma.rm): by induction the accumulated alpha of the
// exit plane can never fall below it, so the walk never steps out of the staged brick and no tolerance window is needed.
// The remainder of the chord [acur, a_out] is given to the last voxel, so every brick integrates exactly its
// [a_in, a_out] whatever the accumulated drift (<= 32 additions deep, ~1e-7 in alpha).
B200_HD float add_rp(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_ru(a, b);
#else
    const double x = (double)a + (double)b;
    float f = (float)x;
    if ((double)f < x) f = nextafterf(f, INFINITY);
    return f;
#endif
}
B200_HD float fma_rm(float a, float b, float c)
{
#if defined(__CUDA_ARCH__)
    return __fmaf_rd(a, b, c);
#else
    const double x = (double)a * (double)b + (double)c;
    float f = (float)x;
    if ((double)f > x) f = nextafterf(f, -INFINITY);
    return f;
#endif
}

struct AccState {
    float an0, an1, an2, acur;
    int off;
};
struct AccConst {
    float da0, da1, da2, a_stop;
    int so0, so1, so2;
};

B200_HD float acc_step(AccState& s, const AccConst& k)
{
    float len;
#if defined(__CUDA_ARCH__)
    asm("{\n\t"
        ".reg .pred q, p0, p1, p2;\n\t"
        ".reg .f32 nx;\n\t"
        "min.f32 nx, %0, %1;\n\t"
        "min.f32 nx, nx, %2;\n\t"
        "sub.f32 %5, nx, %3;\n\t"
        "mov.f32 %3, nx;\n\t"
        "setp.lt.f32 q, nx, %6;\n\t"
        "setp.eq.and.f32 p0, %0, nx, q;\n\t"
        "setp.eq.and.f32 p1, %1, nx, q;\n\t"
        "setp.eq.and.f32 p2, %2, nx, q;\n\t"
        "@p0 add.rp.f32 %0, %0, %7;\n\t"
        "@p1 add.rp.f32 %1, %1, %8;\n\t"
        "@p2 add.rp.f32 %2, %2, %9;\n\t"
        "@p0 add.s32 %4, %4, %10;\n\t"
        "@p1 add.s32 %4, %4, %11;\n\t"
        "@p2 add.s32 %4, %4, %12;\n\t"
        "}"
        : "+f"(s.an0), "+f"(s.an1), "+f"(s.an2), "+f"(s.acur), "+r"(s.off), "=f"(len)
        : "f"(k.a_stop), "f"(k.da0), "f"(k.da1), "f"(k.da2), "r"(k.so0), "r"(k.so1), "r"(k.so2));
#else
    const float nx = fminf(fminf(s.an0, s.an1), s.an2);
    len = nx - s.acur;
    s.acur = nx;
    const bool q = nx < k.a_stop;
    const bool p0 = q && s.an0 == nx, p1 = q && s.an1 == nx, p2 = q && s.an2 == nx;
    if (p0) { s.an0 = add_rp(s.an0, k.da0); s.off += k.so0; }
    if (p1) { s.an1 = add_rp(s.an1, k.da1); s.off += k.so1; }
    if (p2) { s.an2 = add_rp(s.an2, k.da2); s.off += k.so2; }
#endif
    return len;
}

#if !defined(__CUDACC__)
static float g_emu_rcp_perturb = 0.0f;  // host emulation only
#endif
B200_HD float approx_rcp(float x)
{
#if defined(__CUDA_ARCH__)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#elif defined(__CUDACC__)
    return 1.0f / x;
#else
    return (1.0f / x) * (1.0f + g_emu_rcp_perturb);  // tests can model the 1-ulp error of MUFU.RCP
#endif
}

// s = source, inv = 1/d from the ray table, clo / chi = (box face - shift) - s per axis (the hit test's constants).
// The direction d is only needed for the entry voxel (a floor that the clamp / entry-face select make robust), so it is
// re-formed as 1/inv (MUFU.RCP, 1 ulp) instead of being fetched: the ray table is 16 bytes per ray.
template <int U, class Ld, bool ACC = true, bool PIPE = true>
B200_HD float brick_pair_fwd_lean(const Ld& ld, const float s[3], const float inv[3], const float clo[3],
                                  const float chi[3], const int lo_v[3], const int hi_v[3], const int org[3], int st0, int st1,
                                  int st2, float shift)
{
    float lo[3], a_in = -INFINITY, a_hi = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float a0 = clo[a] * inv[a], a1 = chi[a] * inv[a];  // == plane_alpha_acc of the two faces
        lo[a] = fminf(a0, a1);
        a_in = fmaxf(a_in, lo[a]);
        a_hi = fminf(a_hi, fmaxf(a0, a1));
    }
    if (!(a_in < a_hi)) return 0.0f;
    const int st[3] = {st0 * Ld::kScale, st1 * Ld::kScale, st2 * Ld::kScale};
    AccState w;
    AccConst k;
    float an[3], da[3], nxc[3], a_out = INFINITY;
    int so[3];
    w.off = ld.base();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const bool fwd = inv[a] > 0.0f;
        const int lo_i = lo_v[a], hi_i = hi_v[a] - 1;
        int i = (int)floorf(fmaf(a_in, approx_rcp(inv[a]), s[a] + shift));
        i = i < lo_i ? lo_i : (i > hi_i ? hi_i : i);
        i = (lo[a] >= a_in) ? (fwd ? lo_i : hi_i) : i;  // entering through a face of this axis
        float p0 = (float)(fwd ? i + 1 : i);
        da[a] = fabsf(inv[a]);
        an[a] = ((p0 - shift) - s[a]) * inv[a];
        // Make the start voxel agree with the ORDER of the alphas: the floor() above sees the position to ~1e-4 voxel,
        // which for a ray nearly parallel to this axis' planes (|d_a| << 1) is a long stretch of alpha (round-off / |d_a|).
        // One step forward if the plane "ahead" is already behind a_in, one step back if the plane behind is not.
        const bool ahead = (an[a] < a_in) && (fwd ? i < hi_i : i > lo_i);
        const bool back = !ahead && (an[a] - da[a] >= a_in) && (fwd ? i > lo_i : i < hi_i);
        const int dstep = ahead ? 1 : (back ? -1 : 0);  // along the direction of travel
        i += fwd ? dstep : -dstep;
        p0 += (float)(fwd ? dstep : -dstep);
        an[a] = dstep == 0 ? an[a] : ((p0 - shift) - s[a]) * inv[a];
        const float nx = fwd ? (float)hi_v[a] - p0 : p0 - (float)lo_v[a];
        nxc[a] = nx;
        a_out = fminf(a_out, fmaf(nx, da[a], an[a]));
        so[a] = fwd ? st[a] : -st[a];
        w.off += (i - org[a]) * st[a];
    }
    if (!ACC) {  // exact crossing alphas (fma from a counter), for A/B comparison with the accumulated form
        LeanState ls;
        LeanConst lk;
        lk.da0 = da[0]; lk.da1 = da[1]; lk.da2 = da[2];
        lk.a00 = an[0]; lk.a01 = an[1]; lk.a02 = an[2];
        lk.a_out = a_out;
        lk.so0 = so[0]; lk.so1 = so[1]; lk.so2 = so[2];
        ls.an0 = an[0]; ls.an1 = an[1]; ls.an2 = an[2];
        ls.nf0 = ls.nf1 = ls.nf2 = 0.0f;
        ls.acur = a_in;
        ls.off = w.off;
        float acc = 0.0f;
        while (ls.acur < lk.a_out) {
            float len[U], v[U];
            int offs[U];
#pragma unroll
            for (int j = 0; j < U; ++j) {
                offs[j] = ls.off;
                len[j] = lean_step(ls, lk);
            }
#pragma unroll
            for (int j = 0; j < U; ++j) v[j] = ld(offs[j]);
#pragma unroll
            for (int j = 0; j < U; ++j) acc = fmaf(len[j], v[j], acc);
        }
        return acc;
    }
    // accumulate in the pair's own frame beta = alpha - a_in: values of ~0..0.03 instead of ~0.5..1, i.e. additions that
    // round at ~2e-9 instead of 6e-8 -- 32 of them drift less than ONE rounding of an absolute alpha
    w.an0 = an[0] - a_in; w.an1 = an[1] - a_in; w.an2 = an[2] - a_in;
    w.acur = 0.0f;
    k.da0 = da[0]; k.da1 = da[1]; k.da2 = da[2];
    k.so0 = so[0]; k.so1 = so[1]; k.so2 = so[2];
    a_out = fminf(fminf(fma_rm(nxc[0], da[0], w.an0), fma_rm(nxc[1], da[1], w.an1)), fma_rm(nxc[2], da[2], w.an2));
    k.a_stop = a_out;
    float acc = 0.0f;
    if (PIPE) {
        // software-pipelined: the products of one group of U steps are formed while the NEXT group's loads are in flight
        float len[U], v[U];
#pragma unroll
        for (int j = 0; j < U; ++j) len[j] = v[j] = 0.0f;
        while (w.acur < k.a_stop) {
            float lenn[U];
            int offs[U];
#pragma unroll
            for (int j = 0; j < U; ++j) {
                offs[j] = w.off;
                lenn[j] = acc_step(w, k);
            }
#pragma unroll
            for (int j = 0; j < U; ++j) acc = fmaf(len[j], v[j], acc);
#pragma unroll
            for (int j = 0; j < U; ++j) {
                v[j] = ld(offs[j]);
                len[j] = lenn[j];
            }
        }
#pragma unroll
        for (int j = 0; j < U; ++j) acc = fmaf(len[j], v[j], acc);
    } else {
        while (w.acur < k.a_stop) {
            float len[U], v[U];
            int offs[U];
#pragma unroll
            for (int j = 0; j < U; ++j) {
                offs[j] = w.off;
                len[j] = acc_step(w, k);
            }
#pragma unroll
            for (int j = 0; j < U; ++j) v[j] = ld(offs[j]);
#pragma unroll
            for (int j = 0; j < U; ++j) acc = fmaf(len[j], v[j], acc);
        }
    }
    return fmaf(a_out - w.acur, ld(w.off), acc);  // the rest of the chord belongs to the last voxel
}


// ---- two rays per thread (instruction-level parallelism for the issue-bound walk) -------------------------------------------
// Same set-up and step as brick_pair_fwd_lean<ACC>, split so that one thread can interleave the dependent chains of TWO
// independent (ray, brick) pairs: the walk is bound by instruction issue with ~1.8 eligible warps per cycle, and a second
// chain per thread hides the fixed ALU / shared-memory latencies that an extra warp (no registers left) cannot.
template <class Ld>
B200_HD bool brick_pair_setup_acc(const Ld& ld, bool valid, const float s[3], const float inv[3], const float clo[3],
                                  const float chi[3], const int lo_v[3], const int hi_v[3], const int org[3], int st0, int st1,
                                  int st2, float shift, AccState& w, AccConst& k)
{
    float lo[3], a_in = -INFINITY, a_hi = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float a0 = clo[a] * inv[a], a1 = chi[a] * inv[a];
        lo[a] = fminf(a0, a1);
        a_in = fmaxf(a_in, lo[a]);
        a_hi = fminf(a_hi, fmaxf(a0, a1));
    }
    const bool hit = valid && (a_in < a_hi);
    const int st[3] = {st0 * Ld::kScale, st1 * Ld::kScale, st2 * Ld::kScale};
    float an[3], da[3], nxc[3];
    int so[3];
    w.off = ld.base();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const bool fwd = inv[a] > 0.0f;
        const int lo_i = lo_v[a], hi_i = hi_v[a] - 1;
        int i = (int)floorf(fmaf(a_in, approx_rcp(inv[a]), s[a] + shift));
        i = i < lo_i ? lo_i : (i > hi_i ? hi_i : i);
        i = (lo[a] >= a_in) ? (fwd ? lo_i : hi_i) : i;
        float p0 = (float)(fwd ? i + 1 : i);
        da[a] = fabsf(inv[a]);
        an[a] = ((p0 - shift) - s[a]) * inv[a];
        const bool ahead = (an[a] < a_in) && (fwd ? i < hi_i : i > lo_i);
        const bool back = !ahead && (an[a] - da[a] >= a_in) && (fwd ? i > lo_i : i < hi_i);
        const int dstep = ahead ? 1 : (back ? -1 : 0);
        i += fwd ? dstep : -dstep;
        p0 += (float)(fwd ? dstep : -dstep);
        an[a] = dstep == 0 ? an[a] : ((p0 - shift) - s[a]) * inv[a];
        nxc[a] = fwd ? (float)hi_v[a] - p0 : p0 - (float)lo_v[a];
        so[a] = fwd ? st[a] : -st[a];
        w.off += hit ? (i - org[a]) * st[a] : 0;
    }
    // a miss / an empty slot is a walk that is already finished: every quantity zero, the offset on the brick's first voxel
    w.an0 = hit ? an[0] - a_in : 0.0f;
    w.an1 = hit ? an[1] - a_in : 0.0f;
    w.an2 = hit ? an[2] - a_in : 0.0f;
    w.acur = 0.0f;
    k.da0 = hit ? da[0] : 0.0f;
    k.da1 = hit ? da[1] : 0.0f;
    k.da2 = hit ? da[2] : 0.0f;
    k.so0 = hit ? so[0] : 0;
    k.so1 = hit ? so[1] : 0;
    k.so2 = hit ? so[2] : 0;
    const float a_out = fminf(fminf(fma_rm(nxc[0], da[0], w.an0), fma_rm(nxc[1], da[1], w.an1)), fma_rm(nxc[2], da[2], w.an2));
    k.a_stop = hit ? a_out : 0.0f;
    return hit;
}

template <int U, class Ld>
B200_HD void brick_pair2_walk(const Ld& ld, AccState& wa, const AccConst& ka, AccState& wb, const AccConst& kb, float& part_a,
                              float& part_b)
{
    float acc_a = 0.0f, acc_b = 0.0f;
    while (wa.acur < ka.a_stop || wb.acur < kb.a_stop) {
        float la[U], lb[U], va[U], vb[U];
        int oa[U], ob[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
            oa[j] = wa.off;
            la[j] = acc_step(wa, ka);
            ob[j] = wb.off;
            lb[j] = acc_step(wb, kb);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
            va[j] = ld(oa[j]);
            vb[j] = ld(ob[j]);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
            acc_a = fmaf(la[j], va[j], acc_a);
            acc_b = fmaf(lb[j], vb[j], acc_b);
        }
    }
    part_a = fmaf(ka.a_stop - wa.acur, ld(wa.off), acc_a);
    part_b = fmaf(kb.a_stop - wb.acur, ld(wb.off), acc_b);
}

// ---- volume gradient (transpose of the walk): the same chord lengths scattered into a brick of accumulators -------------------
// d(out[ray]) / d(vol[voxel]) = L * len(ray, voxel), so g_vol[voxel] += sum over rays of (gout * L) * len: the pair's walk with
// the load replaced by an add of len * wgt into the staged brick (`st.add`: shared-memory atomic on the device, += in the host
// emulation).  Same set-up (brick_pair_setup_acc), same steps, same tail term as brick_pair_fwd_lean<ACC = true>.
struct StHost {
    float* brick;
    static constexpr int kScale = 1;
    B200_HD int base() const { return 0; }
    B200_HD void add(int off, float v) const { brick[off] += v; }
};

template <int U, class St>
B200_HD void brick_pair_bwd_lean(const St& st, float wgt, const float s[3], const float inv[3], const float clo[3],
                                 const float chi[3], const int lo_v[3], const int hi_v[3], const int org[3], int st0, int st1,
                                 int st2, float shift)
{
    AccState w;
    AccConst k;
    if (!brick_pair_setup_acc(st, true, s, inv, clo, chi, lo_v, hi_v, org, st0, st1, st2, shift, w, k)) return;
    while (w.acur < k.a_stop) {
        float len[U];
        int offs[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
            offs[j] = w.off;
            len[j] = acc_step(w, k);
        }
#pragma unroll
        for (int j = 0; j < U; ++j)
            if (len[j] != 0.0f) st.add(offs[j], len[j] * wgt);
    }
    const float rest = k.a_stop - w.acur;  // the rest of the chord belongs to the last voxel (<= 0 when the last step overshot)
    if (rest != 0.0f) st.add(w.off, rest * wgt);
}

// ---- per-ray sensitivities (training step) over a staged brick ------------------------------------------------------------
// The pair runs the slab kernels' exact-frame sensitivities walk (siddon_ray_sens_box, CUT = true: every brick face inside the
// volume is a cut on its own axis, so a tie of a crossing with a brick edge or corner goes to the same axis as in the un-cut
// walk) on the ray rebuilt bit-identically to the slab kernel.  Only the voxel fetch differs: the walk's offsets are formed
// with the brick's strides scaled to the loader's units (kScale), and `bias` moves them onto the staged copy.
template <class Ld>
struct BrickLoad {
    Ld ld;
    int bias;  // ld.base() - (org . strides) * kScale
    template <int U>
    B200_HD void batch(const float*, const int (&offs)[U], float (&v)[U]) const
    {
#pragma unroll
        for (int j = 0; j < U; ++j) v[j] = ld(offs[j] + bias);
    }
    B200_HD float at(const float*, int off) const { return ld(off + bias); }
};

// A, C accumulated INTO (see siddon_ray_sens_box_m); returns sum v * dalpha over the brick's voxels [lo_v, hi_v).
// The framed pair starts from the ray's volume frame f (volume_frame), its source s and direction d: what siddon_ray_sens_box
// does for the ray, without re-deriving the frame.
template <int U, class Ld>
B200_HD float brick_pair_sens_framed(const Ld& ld, const VolFrame& f, const float s[3], const float d[3], const VolDims& dims,
                                     const int lo_v[3], const int hi_v[3], const int org[3], int st0, int st1, int st2, float shift,
                                     float A[3], float C[3])
{
    const int s0 = st0 * Ld::kScale, s1 = st1 * Ld::kScale, s2 = st2 * Ld::kScale;
    const BrickLoad<Ld> load{ld, ld.base() - (org[0] * s0 + org[1] * s1 + org[2] * s2)};
    const Walk w = start_walk_in_frame<true>(f, s, d, dims, lo_v, hi_v, shift);
    const float* vol = nullptr;
    const float m0 = fabsf(d[0]), m1 = fabsf(d[1]), m2 = fabsf(d[2]);
    if (m0 >= m1 && m0 >= m2) return siddon_ray_sens_walk_m<U, 0>(vol, w, s0, s1, s2, A, C, load);
    if (m1 >= m2) return siddon_ray_sens_walk_m<U, 1>(vol, w, s0, s1, s2, A, C, load);
    return siddon_ray_sens_walk_m<U, 2>(vol, w, s0, s1, s2, A, C, load);
}

template <int U, class Ld>
B200_HD float brick_pair_sens(const Ld& ld, const Ray& ray, const VolDims& dims, const int lo_v[3], const int hi_v[3],
                              const int org[3], int st0, int st1, int st2, float shift, float A[3], float C[3])
{
    return brick_pair_sens_framed<U>(ld, volume_frame(ray, dims, shift), ray.s, ray.d, dims, lo_v, hi_v, org, st0, st1, st2, shift, A,
                                     C);
}

// ---- per-ray frame record of the sensitivities mode ----------------------------------------------------------------------------
// A ray is cut into ~20-30 (ray, brick) pairs, and every part of a pair's set-up that depends on the ray alone -- rebuilding the
// ray, its volume frame, its length L -- is the same for all of them.  brick_prep_kernel builds it once per launch into this record,
// so a pair only clips the frame to its brick (start_walk_in_frame).  The stored values are the ones the pair would compute, so
// every brick of a ray still sees bit-identical alphas.  32 bytes, one L2 sector: 1/d comes from the ray table, s from the pose,
// and the frame's entry voxel index i_a (pref_a = i_a + 1 when d_a > 0, else i_a) takes 10 bits per axis -- which limits the
// volume's sides to kSensFrameMaxSide voxels (larger volumes take the slab kernels, siddon_sens_brick_route).
//   f0 = (a0[0], a0[1], a0[2], L),   f1 = (d[0], d[1], d[2], bits of i_0 | i_1 << 10 | i_2 << 20 | hit << 30)
struct SensFrameRec {
    float4 f0, f1;
};
constexpr int kSensFrameMaxSide = 1024;

B200_HD SensFrameRec pack_sens_frame(const VolFrame& f, const float d[3], float L)
{
    uint32_t bits = f.hit ? 1u << 30 : 0u;
#pragma unroll
    for (int a = 0; a < 3; ++a) bits |= (uint32_t)((int)f.pref[a] - (f.sti[a] > 0 ? 1 : 0)) << (10 * a);
    SensFrameRec r;
    r.f0.x = f.a0[0];
    r.f0.y = f.a0[1];
    r.f0.z = f.a0[2];
    r.f0.w = L;
    r.f1.x = d[0];
    r.f1.y = d[1];
    r.f1.z = d[2];
    r.f1.w = f32_from_bits(bits);
    return r;
}

// inv = the ray's 1/d (ray table); d and L are read back from the record
B200_HD VolFrame unpack_sens_frame(const SensFrameRec& r, const float inv[3], float d[3], float& L)
{
    VolFrame f;
    const uint32_t bits = f32_bits(r.f1.w);
    const float a0[3] = {r.f0.x, r.f0.y, r.f0.z};
    d[0] = r.f1.x;
    d[1] = r.f1.y;
    d[2] = r.f1.z;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        f.inv[a] = inv[a];
        f.da[a] = fabsf(inv[a]);
        f.sti[a] = d[a] > 0.0f ? 1 : -1;
        f.a0[a] = a0[a];
        const int i = (int)((bits >> (10 * a)) & 1023u);
        f.pref[a] = (float)(f.sti[a] > 0 ? i + 1 : i);
    }
    f.hit = ((bits >> 30) & 1u) != 0u;
    L = r.f0.w;
    return f;
}

// Sort key of the sensitivities mode: the walk branches three ways on the ray's major axis M, and a warp's 32 items mix poses,
// so M goes into the key (bin = M * 10 + one of 10 length bins, longest first within each M): warps are M-uniform except at
// the group boundaries.  M comes from the ray table's 1/d (largest |d| = smallest |1/d|, ties to the lower axis as in
// siddon_ray_sens_box); a rounding near 45 degrees only costs a divergent warp, the walk itself decides on d.
// A length bin is U voxels of the chord's L1 length wide, the length of one walk group of U steps: a pair visits about one voxel
// per unit of L1 length, so the pairs of a bin mostly run the same number of groups, and a 32-item chunk, which runs until its
// longest pair is done, pads few of its lanes (CPU emulation of the bench's lists, DESIGN.md 4.2b).
constexpr int kSensLenBins = 10;
template <int U>
B200_HD int sens_bin(const float inv[3], float a_in, float a_out, float sumabs_d)
{
    const float i0 = fabsf(inv[0]), i1 = fabsf(inv[1]), i2 = fabsf(inv[2]);
    const int M = (i0 <= i1 && i0 <= i2) ? 0 : (i1 <= i2 ? 1 : 2);
    const int b = step_bin(a_in, a_out, sumabs_d, 1.0f / (float)U);
    return M * kSensLenBins + (b < kSensLenBins - 1 ? b : kSensLenBins - 1);
}

}  // namespace b200drr
