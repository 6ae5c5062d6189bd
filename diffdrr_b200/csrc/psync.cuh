// psync.cuh -- plane-synchronous Siddon walk (the production forward path).
//
// Why: with one lane per ray, the lanes of a warp that advance "one voxel per step" drift apart in depth (each
// ray interleaves its minor-axis crossings differently), so a warp-wide gather touches ~one 32-byte sector PER
// LANE and the L1 wavefront / miss-request pipes saturate (many sectors and wavefronts per request).  Here every lane advances exactly one plane of its MAJOR axis (argmax |d|) per iteration, so the
// 32 lanes of an 8x4 ray bundle always read from the same voxel plane and share sectors.
//
// Inside one major slab (between two consecutive major planes) a ray with minor slopes |d_u/d_m|, |d_v/d_m| <= 1
// crosses at most one u-plane and one v-plane, i.e. it visits 1..3 voxels:
//     A = (iu0, iv0)   for t in [0, t1]          t1 = min(tu, tv)
//     M = (iu1, iv0) or (iu0, iv1)   [t1, t2]    t2 = max(tu, tv)   (whichever minor plane comes first)
//     D = (iu1, iv1)   for t in [t2, 1]
// with tu, tv the crossing fractions (1 when there is no crossing -- then the "other" voxel coincides, so any
// value in [0,1] gives the same sum).  These are exactly Siddon's segments: same voxels, same lengths.
// The first and last (partial) major slabs of a ray are walked with the generic lean step (ray_math.cuh).
#pragma once

#include "ray_math.cuh"

namespace b200drr {

constexpr float kMagic = 12582912.0f;       // 1.5 * 2^23: (x + kMagic) rounds x to the nearest integer ...
constexpr unsigned kMagicBits = 0x4B400000u;  // ... which then sits in the low mantissa bits: bits = kMagicBits + n

B200_HD unsigned f2u(float x)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(x);
#else
    unsigned u;
    memcpy(&u, &x, 4);
    return u;
#endif
}

B200_HD float sat_fma(float a, float b, float c)
{
#if defined(__CUDA_ARCH__)
    float r;
    asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
#else
    const float r = fmaf(a, b, c);
    return r != r ? 0.0f : (r < 0.0f ? 0.0f : (r > 1.0f ? 1.0f : r));
#endif
}

B200_HD float sat_add(float a, float b)
{
#if defined(__CUDA_ARCH__)
    float r;
    asm("add.sat.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
#else
    const float r = a + b;
    return r != r ? 0.0f : (r < 0.0f ? 0.0f : (r > 1.0f ? 1.0f : r));
#endif
}

B200_HD float pick3(const float v[3], int a) { return a == 0 ? v[0] : (a == 1 ? v[1] : v[2]); }
B200_HD int pick3i(const int v[3], int a) { return a == 0 ? v[0] : (a == 1 ? v[1] : v[2]); }

// `align(m, sigma_positive, p_start, active)` returns how many iterations this lane must idle so that all lanes
// of its warp sit on the same major plane in the same iteration (0 on the host / when the warp is mixed).
template <int U, class Align>
B200_HD float siddon_ray_psync(const float* vol, unsigned nvox, const int lo_v[3], const int hi_v[3], int st0, int st1,
                               int st2, const Ray& ray, float shift, Align align)
{
    const Walk w = start_walk_box(ray, lo_v, hi_v, shift);
    const int st[3] = {st0, st1, st2};
    LeanConst k;
    LeanState s;
    lean_init(w, st0, st1, st2, s, k);

    // ---- major axis m and the two minor axes u, v -----------------------------------------------------
    const float ad0 = fabsf(ray.d[0]), ad1 = fabsf(ray.d[1]), ad2 = fabsf(ray.d[2]);
    const int m = (ad0 >= ad1 && ad0 >= ad2) ? 0 : (ad1 >= ad2 ? 1 : 2);
    const int u = m == 2 ? 0 : m + 1, v = m == 0 ? 2 : (m == 1 ? 0 : 1);
    const float da_m = pick3(w.da, m), a0_m = pick3(w.a0, m);

    // ---- prologue: generic steps until the first major plane is crossed ---------------------------------
    float acc = 0.0f;
    float nfm = 0.0f;  // index of the major crossing the ray sits on after the prologue
    bool at_plane = false;
    while (s.acur < k.a_out && !at_plane) {
        const float before = m == 0 ? s.nf0 : (m == 1 ? s.nf1 : s.nf2);
        const int off = s.off;
        const float len = lean_step(s, k);
        acc = fmaf(len, ldg(vol + off), acc);
        const float after = m == 0 ? s.nf0 : (m == 1 ? s.nf1 : s.nf2);
        if (after != before) {
            at_plane = true;
            nfm = before;
        }
    }
    const float a_start = s.acur;  // == fma(nfm, da_m, a0_m) when at_plane

    // ---- how many FULL major slabs follow: crossings nfm+1 .. nfm+n with alpha <= a_out -----------------------
    const float adm = 1.0f / da_m;  // |d_m|: alpha -> slab units
    int n_full = 0;
    if (at_plane) {
        const int n_max = (int)(pick3(w.nx, m) - nfm);
        int n = (int)floorf((k.a_out - a_start) * adm + 0.5f);
        n = n < 0 ? 0 : (n > n_max ? n_max : n);
        if (n > 0 && fmaf(nfm + (float)n, da_m, a0_m) > k.a_out) --n;
        if (n > 0 && fmaf(nfm + (float)n, da_m, a0_m) > k.a_out) --n;
        if (n < n_max && fmaf(nfm + (float)(n + 1), da_m, a0_m) <= k.a_out) ++n;
        n_full = n;
    }
    const bool pos = pick3i(w.sti, m) > 0;
    const int p_start = (int)pick3(w.p0, m) + (pos ? (int)nfm : -(int)nfm);
    const int delay = align(m, pos, p_start, n_full > 0);

    // ---- closed-form main loop over the full slabs, in SLAB UNITS ------------------------------------------
    // Measure alpha in units of one major slab (|1/d_m|) from the start plane: slab j spans [j, j+1] and the next
    // crossing of minor axis u (crossing count nu) sits at  T_u = (alpha_u(nu) - a_start)*|d_m| = fma(nu, Ku, Cu),
    // so its position inside slab j is tu = sat(T_u - j) (1 = "not in this slab").  Same conditioning as the
    // reference's own alphas, unlike positions formed from absolute fp32 coordinates.
    const float Ku = pick3(w.da, u) * adm, Kv = pick3(w.da, v) * adm;
    const float Cu = (pick3(w.a0, u) - a_start) * adm, Cv = (pick3(w.a0, v) - a_start) * adm;
    const unsigned ssu = (unsigned)(pick3i(w.sti, u) * pick3i(st, u)), ssv = (unsigned)(pick3i(w.sti, v) * pick3i(st, v));
    const unsigned ssm = (unsigned)(pick3i(w.sti, m) * pick3i(st, m));
    float nu = u == 0 ? s.nf0 : (u == 1 ? s.nf1 : s.nf2);  // minor crossing counters, straight from the generic walk
    float nv = v == 0 ? s.nf0 : (v == 1 ? s.nf1 : s.nf2);
    unsigned oA = (unsigned)s.off;
    float jf = 0.0f;
    float accm = 0.0f;
    const int total = delay + n_full;
    for (int j = 0; j < total; j += U) {
        float wA[U], wM[U], wD[U];
        unsigned oa[U], om[U], od[U];
#pragma unroll
        for (int q = 0; q < U; ++q) {
            const bool act = (j + q >= delay) && (j + q < total);
            wA[q] = 0.0f;
            wM[q] = 0.0f;
            wD[q] = 0.0f;
            oa[q] = om[q] = od[q] = oA;
            if (act) {
                const float tu = sat_add(fmaf(nu, Ku, Cu), -jf), tv = sat_add(fmaf(nv, Kv, Cv), -jf);
                const bool cu = tu < 1.0f, cv = tv < 1.0f;
                nu = cu ? nu + 1.0f : nu;
                nv = cv ? nv + 1.0f : nv;
                const unsigned du = cu ? ssu : 0u, dv = cv ? ssv : 0u;
                const float t1 = fminf(tu, tv), t2 = fmaxf(tu, tv);
                wA[q] = t1;
                wM[q] = t2 - t1;
                wD[q] = 1.0f - t2;
                om[q] = oA + (tu < tv ? du : dv);
                od[q] = oA + du + dv;
                oA = od[q] + ssm;
                jf += 1.0f;
            }
        }
        float vA[U], vM[U], vD[U];
#pragma unroll
        for (int q = 0; q < U; ++q) {
            // (offset < nvox) guards the rare ray whose minor crossing rounds across a face of the box
            vA[q] = (wA[q] > 0.0f && oa[q] < nvox) ? ldg(vol + oa[q]) : 0.0f;
            vM[q] = (wM[q] > 0.0f && om[q] < nvox) ? ldg(vol + om[q]) : 0.0f;
            vD[q] = (wD[q] > 0.0f && od[q] < nvox) ? ldg(vol + od[q]) : 0.0f;
        }
#pragma unroll
        for (int q = 0; q < U; ++q) accm = fmaf(wA[q], vA[q], fmaf(wM[q], vM[q], fmaf(wD[q], vD[q], accm)));
    }
    acc = fmaf(accm, da_m, acc);  // every full slab spans |1/d_m| in alpha

    // ---- epilogue: generic steps from the last full plane to the exit ------------------------------------
    if (at_plane && n_full > 0) {
        const float nm_last = nfm + (float)n_full;
        const float nm_next = nm_last + 1.0f;
        s.nf0 = m == 0 ? nm_next : (u == 0 ? nu : nv);
        s.nf1 = m == 1 ? nm_next : (u == 1 ? nu : nv);
        s.nf2 = m == 2 ? nm_next : (u == 2 ? nu : nv);
        s.an0 = fmaf(s.nf0, k.da0, k.a00);
        s.an1 = fmaf(s.nf1, k.da1, k.a01);
        s.an2 = fmaf(s.nf2, k.da2, k.a02);
        s.acur = fmaf(nm_last, da_m, a0_m);
        s.off = (int)oA;
    }
    while (s.acur < k.a_out) {
        const int off = s.off;
        const float len = lean_step(s, k);
        acc = fmaf(len, (unsigned)off < nvox ? ldg(vol + off) : 0.0f, acc);
    }
    return acc;
}

struct NoAlign {
    B200_HD int operator()(int, bool, int, bool) const { return 0; }
};

}  // namespace b200drr
