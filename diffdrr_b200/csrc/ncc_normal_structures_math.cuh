// ncc_normal_structures_math.cuh -- global-NCC normal equations of a piecewise-rigid composite image, block by block
// (host+device; ncc_normal_structures.cu wraps these functions, tests/hostemu compiles the same source).  DESIGN.md 6g.
//
// One pose: the composite image x (the sum of the render_structures channels), the target t, and per structure k = 0..K-1 the
// H*W x 6 Jacobian J_k of x with respect to that structure's motion increment.  The P = 6K unknowns are the K blocks.  The global
// mode of ncc_normal_math.cuh needs
//   the scalar moments {S x, S x^2, S t, S t^2, S x t} over the whole image,
//   S J_k, S x J_k, S t J_k per structure, and S J_j J_k^T per pair of structures,
// and J_k is zero outside structure k's detector footprint (the render culls to it).  So the moments of k run over footprint k,
// and block (j, k) of S J J^T over the intersection of footprints j and k: a pair whose footprints miss each other reads no
// pixel.  Each summation task (a pair j <= k, or the scalar moments) covers a rectangle, split into `chunks` row bands; the
// partial sums of a band are products of two staged rows {1, x, t, J_j[0..5], J_k[0..5]}, summed in double.  ne_window then turns
// the moments into the window terms a, b, g and 1/s^2, and A = S J J^T / s^2 - a a^T - b b^T.
#pragma once

#include "ncc_normal_math.cuh"
#include "structures_math.cuh"

namespace b200drr {

constexpr int kNsDof = 6;                                  // motion parameters per structure: (omega, v)
constexpr int kNsRows = 3 + 2 * kNsDof;                    // staged rows {1, x, t, J_j, J_k}
constexpr int kNsEntries = 3 * kNsDof + kNsDof * kNsDof;   // per task and band: S {1, x, t} J_k, then S J_j J_k^T
constexpr int kNsMaxK = 255;
constexpr int kNsMaxChunks = 32;
constexpr int kNsChunkTarget = 8192;                       // (task, band) pairs one call aims at

B200_HD int ns_pairs(int K) { return ne_tri(K); }

// task index of the pair j <= k (ne_tri_index's row-major upper triangle)
B200_HD int ns_pair(int j, int k, int K) { return j * K - j * (j - 1) / 2 + (k - j); }

// row bands per task: fewer as the task count grows, so the partials stay small
B200_HD int ns_chunks(int B, int K, int H)
{
    const int64_t tasks = (int64_t)B * (ns_pairs(K) + 1);
    int64_t c = kNsChunkTarget / tasks;
    c = c < 1 ? 1 : (c > kNsMaxChunks ? kNsMaxChunks : c);
    return (int)(c < H ? c : H);
}

// intersection of two pixel rectangles {w0, w1, h0, h1} (inclusive); false when empty
B200_HD bool ns_overlap(const int* a, const int* b, int out[4])
{
    out[0] = a[0] > b[0] ? a[0] : b[0];
    out[1] = a[1] < b[1] ? a[1] : b[1];
    out[2] = a[2] > b[2] ? a[2] : b[2];
    out[3] = a[3] < b[3] ? a[3] : b[3];
    return out[0] <= out[1] && out[2] <= out[3];
}

// rows [r0, r1) of band c of the rows h0..h1
B200_HD void ns_band(int h0, int h1, int c, int chunks, int& r0, int& r1)
{
    const int64_t n = (int64_t)h1 - h0 + 1;
    r0 = h0 + (int)(n * c / chunks);
    r1 = h0 + (int)(n * (c + 1) / chunks);
}

// entry e of a task -> the two staged rows it multiplies.  Scalar task: e < 5, the five image moments (ne_global_pair's order);
// pair task: e < 18 the moments S {1, x, t} J_k (used for j == k only), then S J_j[a] J_k[b] at 18 + 6 a + b.  -> false: unused.
B200_HD bool ns_entry_rows(int e, bool scalar, bool diag, int& ra, int& rb)
{
    ra = rb = 0;
    if (scalar) {
        if (e >= 5) return false;
        ne_global_pair(e, 1, ra, rb);
        return true;
    }
    if (e < 3 * kNsDof) {
        ra = e / kNsDof;
        rb = 3 + kNsDof + e % kNsDof;
        return diag;
    }
    if (e >= kNsEntries) return false;
    ra = 3 + (e - 3 * kNsDof) / kNsDof;
    rb = 3 + kNsDof + (e - 3 * kNsDof) % kNsDof;
    return true;
}

// staged row r of one pixel: Jj, Jk point at the pixel's 6 parameters of structures j and k, parameter i at [i * sk]
B200_HD double ns_row(int r, float x, float t, const float* Jj, const float* Jk, int64_t sk)
{
    if (r == 0) return 1.0;
    if (r == 1) return (double)x;
    if (r == 2) return (double)t;
    return r < 3 + kNsDof ? (double)ldg(Jj + (r - 3) * sk) : (double)ldg(Jk + (r - 3 - kNsDof) * sk);
}

// the moment vector T [5 + 3P] of one pose, element e, from the summed partials: sum(task, entry) is the band sum of that task's
// entry.  T is in ne_window's layout: the scalars, then S J, S x J, S t J over the P = 6K parameters.
template <class Sum>
B200_HD double ns_moment(int e, int K, Sum&& sum)
{
    const int P = kNsDof * K;
    if (e < 5) return sum(ns_pairs(K), e);
    const int f = (e - 5) / P, q = (e - 5) - f * P, k = q / kNsDof;
    return sum(ns_pair(k, k, K), f * kNsDof + q % kNsDof);
}

// entry (i, l) of S J J^T: block (i / 6, l / 6), summed by the pair task of the lower index first
template <class Sum>
B200_HD double ns_jj(int i, int l, int K, Sum&& sum)
{
    const int sj = i / kNsDof, sl = l / kNsDof, a = i % kNsDof, b = l % kNsDof;
    return sj <= sl ? sum(ns_pair(sj, sl, K), 3 * kNsDof + a * kNsDof + b) : sum(ns_pair(sl, sj, K), 3 * kNsDof + b * kNsDof + a);
}

// The footprint rectangle the structures render culls slot (pose b, slot s) to (structures.cu: the box's 8 corners through
// box_corner_uv, their hull through footprint_rect; the whole detector when a corner is not in front of the source).
B200_HD void structure_footprint(const float* G, const float* src, const int* box, float shift, const float* rows,
                                 const float* cols, int H, int W, int rect[4])
{
    int lo_v[3], hi_v[3];
    for (int a = 0; a < 3; ++a) {
        lo_v[a] = box[a];
        hi_v[a] = box[3 + a];
    }
    bool all_ok = true;
    float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
    for (int k = 0; k < 8; ++k) {
        float u = 0.0f, v = 0.0f;
        all_ok = box_corner_uv(G, src, lo_v, hi_v, shift, k, u, v) && all_ok;
        umin = fminf(umin, u);
        umax = fmaxf(umax, u);
        vmin = fminf(vmin, v);
        vmax = fmaxf(vmax, v);
    }
    footprint_rect(all_ok, umin, umax, vmin, vmax, ldg(cols), ldg(cols + W - 1), W, ldg(rows), ldg(rows + H - 1), H, rect);
}

}  // namespace b200drr
