// ncc_normal_math.cuh -- Gauss-Newton normal equations of the global and patch-wise NCC losses from box sums of per-pixel
// moments (host+device; the kernels of ncc_normal.cu are thin wrappers over these functions, tests/hostemu compiles the same
// source).
//
// One pose, one channel, one window w of n pixels (n = p^2, or H W for the global NCC); x the rendered image, t the target, J_q
// the P-vector of pose derivatives of pixel q.  With the population variance and eps as in metrics.py:
//   mu = Sx/n, v = Sxx/n - mu^2, s = sqrt(v + eps), z = (x - mu)/s, kappa = v/(v + eps)   (mu_t, s_t, z_t likewise)
//   L = mean(z z_t),  m = S_J/n,  c = (S_xJ/n - mu m)/s,  u = (S_tJ - mu_t S_J)/s_t
// The window's residual r = z - z_t has Jacobian Jz_q = (J_q - m - z_q c)/s, and
//   A_w = sum_q Jz_q Jz_q^T = (1/s^2) [sum_q J_q J_q^T - n m m^T - n (2 - kappa) c c^T] = (1/s^2) sum_q J_q J_q^T - a a^T - b b^T
//   g_w = sum_q Jz_q r_q   = (1/s) [n c (1 - kappa + L) - u]
// with a = sqrt(n) m / s and b = sqrt(n (2 - kappa)) c / s.  So a window needs the box sums of K = 5 + 3P channels
//   {x, x^2, t, t^2, x t, J_0..J_{P-1}, x J_0.., t J_0..}
// and the P x P term needs none: sum_w (1/s_w^2) sum_{q in w} J_q J_q^T = sum_q beta_q J_q J_q^T with beta_q = sum_{w contains q}
// 1/s_w^2, the adjoint box sum of one scalar map (the backward pass of local_ncc_math.cuh does the same for its maps).
// Every channel value is a product of at most two fp32 numbers: exact in double.  All sums run in double.
#pragma once

#include "common.cuh"

namespace b200drr {

constexpr int kNeMaxP = 16;  // pose parameters (kJacMaxP)

B200_HD int ne_channels(int P) { return 5 + 3 * P; }
B200_HD int ne_tri(int P) { return P * (P + 1) / 2; }

// channel k of one pixel: Jq is the pixel's J, parameter k at Jq[k * sk]
B200_HD double ne_channel(int k, int P, float x, float t, const float* Jq, int64_t sk)
{
    const double u = (double)x, v = (double)t;
    switch (k) {
        case 0: return u;
        case 1: return u * u;
        case 2: return v;
        case 3: return v * v;
        case 4: return u * v;
        default: break;
    }
    const int f = (k - 5) / P, q = (k - 5) - f * P;
    const double j = (double)ldg(Jq + q * sk);
    return f == 0 ? j : (f == 1 ? u : v) * j;
}

// vertical pass: channel k of column `col` summed over rows i .. i+p-1.  x, t: one image plane [H][W]; J: that (pose, channel)'s
// base, pixel n at J[n * sn]
B200_HD double ne_vertical(const float* x, const float* t, const float* J, int64_t sk, int64_t sn, int W, int p, int P, int k, int i,
                           int col)
{
    double s = 0.0;
    for (int r = 0; r < p; ++r) {
        const int64_t n = (int64_t)(i + r) * W + col;
        s += ne_channel(k, P, ldg(x + n), ldg(t + n), J + n * sn, sk);
    }
    return s;
}

// horizontal pass: columns j .. j+p-1 of one channel's vertical sums
B200_HD double ne_horizontal(const double* Vk, int p, int j)
{
    double s = 0.0;
    for (int c = 0; c < p; ++c) s += Vk[j + c];
    return s;
}

// The K window sums at S[k * st] -> in place: a at S[(5 + k) st], b at S[(5 + P + k) st], g_w at S[(5 + 2P + k) st].  Returns 1/s^2.
B200_HD double ne_window(double* S, int64_t st, int P, double n, double eps)
{
    const double inv_n = 1.0 / n;
    const double mu = S[0] * inv_n, mt = S[2 * st] * inv_n;
    double v = S[st] * inv_n - mu * mu, vt = S[3 * st] * inv_n - mt * mt;
    v = v > 0.0 ? v : 0.0;  // a constant window: the cancellation may leave -1e-17
    vt = vt > 0.0 ? vt : 0.0;
    const double s = sqrt(v + eps), s_t = sqrt(vt + eps);
    const double kappa = v / (v + eps);
    const double L = (S[4 * st] * inv_n - mu * mt) / (s * s_t);
    const double fa = sqrt(n) / s, fb = sqrt(n * (2.0 - kappa)) / s, fg = n * (1.0 - kappa + L);
    for (int k = 0; k < P; ++k) {
        double* SJ = S + (5 + k) * st;
        double* SxJ = S + (5 + P + k) * st;
        double* StJ = S + (5 + 2 * P + k) * st;
        const double m = *SJ * inv_n, c = (*SxJ * inv_n - mu * m) / s, u = (*StJ - mt * *SJ) / s_t;
        *SJ = fa * m;
        *SxJ = fb * c;
        *StJ = (fg * c - u) / s;
    }
    return 1.0 / (v + eps);
}

// a_k a_l + b_k b_l of one transformed window (ne_window's layout)
B200_HD double ne_ab(const double* S, int64_t st, int P, int k, int l)
{
    return S[(5 + k) * st] * S[(5 + l) * st] + S[(5 + P + k) * st] * S[(5 + P + l) * st];
}

// entry e < P(P+1)/2 of the upper triangle, row-major -> (k, l), k <= l
B200_HD void ne_tri_index(int e, int P, int& k, int& l)
{
    k = 0;
    while (e >= P - k) {
        e -= P - k;
        ++k;
    }
    l = k + e;
}

// adjoint vertical pass: 1/s^2 of the windows (i, j) with rows i in [y-p+1, y] that exist (0 <= i < H'); rs2 [H'][W']
B200_HD double ne_beta_vertical(const double* rs2, int H, int W, int p, int y, int j)
{
    const int Hp = H - p + 1, Wp = W - p + 1;
    const int lo = y - p + 1 > 0 ? y - p + 1 : 0, hi = y < Hp - 1 ? y : Hp - 1;
    double s = 0.0;
    for (int i = lo; i <= hi; ++i) s += rs2[(int64_t)i * Wp + j];
    return s;
}

// adjoint horizontal pass: beta at pixel (y, x) from VB [H][W'], columns j in [x-p+1, x] that exist
B200_HD double ne_beta(const double* VB, int W, int p, int y, int x)
{
    const int Wp = W - p + 1;
    const int lo = x - p + 1 > 0 ? x - p + 1 : 0, hi = x < Wp - 1 ? x : Wp - 1;
    const double* v = VB + (int64_t)y * Wp;
    double s = 0.0;
    for (int j = lo; j <= hi; ++j) s += v[j];
    return s;
}

// Global mode: one window per channel, reduced as products of two staged rows {1, x, t, J_0 .. J_{P-1}}.  Entry e < K + P(P+1)/2:
// the K channel sums in ne_channel's order, then sum J_k J_l over the upper triangle.  -> the two staged rows it multiplies.
B200_HD void ne_global_pair(int e, int P, int& a, int& b)
{
    const int K = ne_channels(P);
    if (e >= K) {
        int k, l;
        ne_tri_index(e - K, P, k, l);
        a = 3 + k;
        b = 3 + l;
        return;
    }
    switch (e) {
        case 0: a = 0; b = 1; return;
        case 1: a = 1; b = 1; return;
        case 2: a = 0; b = 2; return;
        case 3: a = 2; b = 2; return;
        case 4: a = 1; b = 2; return;
        default: break;
    }
    const int f = (e - 5) / P, q = (e - 5) - f * P;
    a = f;  // 0: one, 1: x, 2: t
    b = 3 + q;
}

}  // namespace b200drr
