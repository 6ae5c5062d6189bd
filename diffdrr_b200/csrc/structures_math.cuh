// structures_math.cuh -- per-thread math of the piecewise-rigid renders (structures.cu; DESIGN.md 6f), host+device so that
// tests/hostemu compiles the same source: the gated voxel load, the detector footprint of a box, the label runs of a row.
#pragma once

#include "ray_math.cuh"

namespace b200drr {

B200_HD int ldg_u8(const uint8_t* p)
{
#if defined(__CUDA_ARCH__)
    return (int)__ldg(p);
#else
    return (int)*p;
#endif
}

// Voxel load policy of the walks (LoadPlain's interface): the voxels whose label belongs to this slot (mine[label] != 0), every
// other voxel read as 0.  `mine` is the slot's 256-entry label table (shared memory in the kernel).  The walk's closed forms
// telescope per voxel, so walking the slot's box with this policy gives exactly the image and sensitivities of a whole-volume walk
// of density * (label in slot).
struct LoadGated {
    const uint8_t* label;
    const uint8_t* mine;
    template <int U, class V>
    B200_HD void batch(const V* vol, const int (&offs)[U], float (&v)[U])
    {
        int l[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
            l[j] = ldg_u8(label + offs[j]);
            v[j] = ldg(vol + offs[j]);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) v[j] = mine[l[j]] ? v[j] : 0.0f;
    }
    template <class V>
    B200_HD float at(const V* vol, int off) const { return mine[ldg_u8(label + off)] ? ldg(vol + off) : 0.0f; }
};

// A gated walk runs over a label box, whose faces are interior planes on every axis: its sensitivities walk takes the CUT entry
// rule, so a crossing that ties with the box's entry face, and a ray that only touches the box along an edge or at a corner, are
// booked as the un-cut walk of density * (label in slot) books them (DESIGN.md 6f).
template <>
struct load_cut<LoadGated> {
    static constexpr bool value = true;
};

// Detector footprint of a box.  The pose-in ray of detector point (u, v) is x = src + t (G0 u + G1 v + c), c = G2 + G3 - src (G
// row-major [3][4], columns G0..G3).  Corner x of the box then projects to (u, v) = (y0, y1) / y2 with y = M^-1 (x - src), M = [G0 |
// G1 | c], and t = y2.  t is affine in x, so when every corner has t > 0 the whole box lies in front of the source and every line
// through the box hits the detector plane inside the hull of the corners' projections.
// box_corner_uv: corner k (bit a = high face on axis a) of the box [lo - shift, hi - shift] -> (u, v); false when t <= 0 or the
// system is degenerate (the caller then takes the whole detector).
B200_HD bool box_corner_uv(const float* G, const float* src, const int lo_v[3], const int hi_v[3], float shift, int k, float& u,
                           float& v)
{
    float a[3], b[3], c[3], x[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        a[i] = G[i * 4];
        b[i] = G[i * 4 + 1];
        c[i] = G[i * 4 + 2] + G[i * 4 + 3] - src[i];
        x[i] = (float)(((k >> i) & 1) ? hi_v[i] : lo_v[i]) - shift - src[i];
    }
    // Cramer's rule: y0 = x.(b x c) / det, y1 = x.(c x a) / det, y2 = x.(a x b) / det, det = a.(b x c)
    const float bc[3] = {b[1] * c[2] - b[2] * c[1], b[2] * c[0] - b[0] * c[2], b[0] * c[1] - b[1] * c[0]};
    const float ca[3] = {c[1] * a[2] - c[2] * a[1], c[2] * a[0] - c[0] * a[2], c[0] * a[1] - c[1] * a[0]};
    const float ab[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    const float det = a[0] * bc[0] + a[1] * bc[1] + a[2] * bc[2];
    const float y0 = x[0] * bc[0] + x[1] * bc[1] + x[2] * bc[2];
    const float y1 = x[0] * ca[0] + x[1] * ca[1] + x[2] * ca[2];
    const float y2 = x[0] * ab[0] + x[1] * ab[1] + x[2] * ab[2];
    const float t = y2 / det;
    if (!(t > 0.0f) || !isfinite(t)) return false;
    u = y0 / y2;
    v = y1 / y2;
    return isfinite(u) && isfinite(v);
}

// Pixel rectangle {w0, w1, h0, h1} (inclusive) covering detector coordinates [umin, umax] x [vmin, vmax], widened by one pixel
// and clamped; empty (w0 > w1 or h0 > h1) when the range misses the detector.  cols / rows are the detector's pixel coordinates,
// evenly spaced (either direction).  ok = false: the whole detector.
B200_HD void footprint_rect(bool ok, float umin, float umax, float vmin, float vmax, float c0, float c1, int W, float r0, float r1,
                            int H, int rect[4])
{
    rect[0] = 0;
    rect[1] = W - 1;
    rect[2] = 0;
    rect[3] = H - 1;
    if (!ok) return;
    if (W > 1) {
        const float dc = (c1 - c0) / (float)(W - 1);
        const float p = (umin - c0) / dc, q = (umax - c0) / dc;
        if (isfinite(p) && isfinite(q)) {
            rect[0] = (int)fmaxf(-1.0f, fminf((float)W, floorf(fminf(p, q)) - 1.0f));
            rect[1] = (int)fmaxf(-1.0f, fminf((float)W, ceilf(fmaxf(p, q)) + 1.0f));
        }
    }
    if (H > 1) {
        const float dr = (r1 - r0) / (float)(H - 1);
        const float p = (vmin - r0) / dr, q = (vmax - r0) / dr;
        if (isfinite(p) && isfinite(q)) {
            rect[2] = (int)fmaxf(-1.0f, fminf((float)H, floorf(fminf(p, q)) - 1.0f));
            rect[3] = (int)fmaxf(-1.0f, fminf((float)H, ceilf(fmaxf(p, q)) + 1.0f));
        }
    }
    rect[0] = rect[0] < 0 ? 0 : rect[0];
    rect[1] = rect[1] > W - 1 ? W - 1 : rect[1];
    rect[2] = rect[2] < 0 ? 0 : rect[2];
    rect[3] = rect[3] > H - 1 ? H - 1 : rect[3];
    if (rect[1] < 0 || rect[0] > W - 1) rect[0] = 1, rect[1] = 0;  // left or right of the detector
    if (rect[3] < 0 || rect[2] > H - 1) rect[2] = 1, rect[3] = 0;
}

// The label runs of one row of n voxels: flush(label, i_begin, i_end) once per maximal run of equal labels.
template <class F>
B200_HD void label_row_runs(const uint8_t* row, int n, F&& flush)
{
    int cur = ldg_u8(row), start = 0;
    for (int i = 1; i < n; ++i) {
        const int l = ldg_u8(row + i);
        if (l != cur) {
            flush(cur, start, i);
            cur = l;
            start = i;
        }
    }
    flush(cur, start, n);
}

}  // namespace b200drr
