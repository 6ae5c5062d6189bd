// local_ncc_math.cuh -- patch-wise (local) zero-normalised cross correlation and its closed-form gradient, one output per call
// (host+device; the kernels of local_ncc.cu are thin wrappers over these functions, tests/hostemu compiles the same source).
//
// Replaces reference diffdrr/metrics.py:16-44 with patch_size = p: every stride-1 p x p window w of every channel is
// normalised on its own (mean, population variance + eps), L_w = cov_w r1_w r2_w with r = 1/sqrt(var + eps), and
//   score[b] = mean of L_w over the C * H' * W' windows,   H' = H - p + 1,  W' = W - p + 1.
// The reference unfolds every window into its own channel (a (B, C H' W' p^2) copy); here a window's five moments are box
// sums, separable into a vertical p-row sum per column (pass 1) and a horizontal p-column sum of those (pass 2): O(p) work
// per output.  Moments are summed in double, as in ncc_math.cuh: the one-pass variance cancels in fp32.
//
// Gradient.  With k = gscore[b] / (C H' W' p^2) and the sums running over the windows w that contain pixel q:
//   d score / d x2_q = k sum_w r2 ((x1_q - mu1) r1 - (x2_q - mu2) r2 L) = k (x1_q A - B2 - x2_q C2 + D2)
//   A = sum r1 r2,  B2 = sum mu1 r1 r2,  C2 = sum L r2^2,  D2 = sum L mu2 r2^2     (and 1 <-> 2 swapped for x1; A is shared).
// The window sums are the adjoint of the forward's box sums: a "full" p x p box sum of the per-window maps, zero outside the
// H' x W' window grid -- the same two passes, vertical then horizontal.
//
// Layouts (per image pair; planes are contiguous):
//   V     [5][H'][W]  double   vertical sums {x1, x2, x1^2, x2^2, x1 x2} of rows i .. i+p-1 at column x
//   stats [5][H'][W'] float    per-window {mu1, r1, mu2, r2, L}, kept for the backward pass
//   VB    [7][H][W']  double   vertical adjoint sums of the maps {A, B1, B2, C1, D1, C2, D2} over the windows rows covering y
#pragma once

#include "ncc_math.cuh"

namespace b200drr {

constexpr int kLnccStats = 5;  // stats planes
constexpr int kLnccMaps = 7;   // VB planes

// pass 1: V[:, i, x] = moments of x1, x2 over rows i .. i+p-1 of column x
B200_HD void lncc_vertical(const float* x1, const float* x2, int H, int W, int p, int i, int x, double* V)
{
    NccSums s = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int r = 0; r < p; ++r) ncc_accumulate(s, ldg(x1 + (int64_t)(i + r) * W + x), ldg(x2 + (int64_t)(i + r) * W + x));
    const int64_t plane = (int64_t)(H - p + 1) * W, o = (int64_t)i * W + x;
    V[o] = s.s1;
    V[plane + o] = s.s2;
    V[2 * plane + o] = s.q1;
    V[3 * plane + o] = s.q2;
    V[4 * plane + o] = s.p;
}

// pass 2: window (i, j) = columns j .. j+p-1 of V row i -> stats[:, i, j]; returns L of the window (for the score)
B200_HD double lncc_window(const double* V, int H, int W, int p, float eps, int i, int j, float* stats)
{
    const int Hp = H - p + 1, Wp = W - p + 1;
    const int64_t plane = (int64_t)Hp * W;
    const double* v = V + (int64_t)i * W + j;
    NccSums s = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int c = 0; c < p; ++c) {
        s.s1 += v[c];
        s.s2 += v[plane + c];
        s.q1 += v[2 * plane + c];
        s.q2 += v[3 * plane + c];
        s.p += v[4 * plane + c];
    }
    const double inv_n = 1.0 / ((double)p * (double)p);
    const double mu1 = s.s1 * inv_n, mu2 = s.s2 * inv_n;
    double v1 = s.q1 * inv_n - mu1 * mu1, v2 = s.q2 * inv_n - mu2 * mu2;
    v1 = v1 > 0.0 ? v1 : 0.0;  // a constant window: the cancellation may leave -1e-17
    v2 = v2 > 0.0 ? v2 : 0.0;
    const double r1 = 1.0 / sqrt(v1 + (double)eps), r2 = 1.0 / sqrt(v2 + (double)eps);
    const double L = (s.p * inv_n - mu1 * mu2) * r1 * r2;
    const int64_t splane = (int64_t)Hp * Wp, o = (int64_t)i * Wp + j;
    stats[o] = (float)mu1;
    stats[splane + o] = (float)r1;
    stats[2 * splane + o] = (float)mu2;
    stats[3 * splane + o] = (float)r2;
    stats[4 * splane + o] = (float)L;
    return L;
}

// backward pass 1: VB[:, y, j] = sums of the window maps over the window rows i in [y-p+1, y] that exist (0 <= i < H')
B200_HD void lncc_bwd_vertical(const float* stats, int H, int W, int p, int y, int j, double* VB)
{
    const int Hp = H - p + 1, Wp = W - p + 1;
    const int64_t splane = (int64_t)Hp * Wp;
    const int lo = y - p + 1 > 0 ? y - p + 1 : 0, hi = y < Hp - 1 ? y : Hp - 1;
    double m[kLnccMaps] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = lo; i <= hi; ++i) {
        const float* s = stats + (int64_t)i * Wp + j;
        const double mu1 = ldg(s), r1 = ldg(s + splane), mu2 = ldg(s + 2 * splane), r2 = ldg(s + 3 * splane), L = ldg(s + 4 * splane);
        const double a = r1 * r2, c1 = L * r1 * r1, c2 = L * r2 * r2;
        m[0] += a;         // A
        m[1] += mu2 * a;   // B1 = mu2 r1 r2
        m[2] += mu1 * a;   // B2 = mu1 r1 r2
        m[3] += c1;        // C1 = L r1^2
        m[4] += mu1 * c1;  // D1 = L mu1 r1^2
        m[5] += c2;        // C2 = L r2^2
        m[6] += mu2 * c2;  // D2 = L mu2 r2^2
    }
    const int64_t bplane = (int64_t)H * Wp, o = (int64_t)y * Wp + j;
#pragma unroll
    for (int t = 0; t < kLnccMaps; ++t) VB[t * bplane + o] = m[t];
}

// a product rounded on its own, never fused into the following subtraction: x1 A - B2 then vanishes exactly where it should
// (p = 1: mu1 = x1 and B2 = mu1 A, and the reference's gradient is exactly 0)
B200_HD double dmul_rn(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// backward pass 2: the window columns j in [x-p+1, x] that exist, then the closed form at pixel (y, x).  k as above.
B200_HD void lncc_bwd_pixel(const double* VB, int H, int W, int p, int y, int x, float x1, float x2, double k, float& g1, float& g2)
{
    const int Wp = W - p + 1;
    const int64_t bplane = (int64_t)H * Wp;
    const int lo = x - p + 1 > 0 ? x - p + 1 : 0, hi = x < Wp - 1 ? x : Wp - 1;
    const double* v = VB + (int64_t)y * Wp;
    double m[kLnccMaps] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = lo; j <= hi; ++j) {
#pragma unroll
        for (int t = 0; t < kLnccMaps; ++t) m[t] += v[t * bplane + j];
    }
    const double u = (double)x1, w = (double)x2;
    g1 = (float)(k * ((dmul_rn(w, m[0]) - m[1]) - (dmul_rn(u, m[3]) - m[4])));
    g2 = (float)(k * ((dmul_rn(u, m[0]) - m[2]) - (dmul_rn(w, m[5]) - m[6])));
}

}  // namespace b200drr
