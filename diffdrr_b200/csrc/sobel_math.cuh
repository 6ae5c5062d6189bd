// sobel_math.cuh -- Gaussian blur (reflect padding) + 3x3 Sobel of one-channel images and the exact adjoint, one output per call
// (host+device; the kernels of sobel.cu are thin wrappers over these functions, tests/hostemu compiles the same source).
//
// Replaces reference diffdrr/metrics.py:69-93 (Sobel, the front end of GradientNormalizedCrossCorrelation2d):
//   blur   only when sigma > 0: torchvision gaussian_blur, k = int(6 sigma + 1) | 1, the outer product of the normalised 1-D
//          Gaussian w[0..k) applied after REFLECT padding of R = k // 2 (torch's "reflect": index -1 -> 1, H -> H - 2).
//          Separable: Bl[y][x] = sum_{a,b} w[a] w[b] x[refl(y + a - R)][refl(x + b - R)].  k = 1, w = {1} is the identity.
//   Sobel  Conv2d(1 -> 2, 3x3, padding 1): cross-correlation of Bl (ZERO outside the image) with
//          Gx = [[1,0,-1],[2,0,-2],[1,0,-1]] (channel 0) and Gy = [[1,2,1],[0,0,0],[-1,-2,-1]] (channel 1).
// Adjoint: g_bl = the Sobel stencils transposed (zero padding), then the blur transposed.  A blur tap that read a reflected
// position refl(i) adds its gradient to the mirrored interior pixel:  for the 1-D pass along an axis of length n,
//   g[m] = sum_a w[a] (G(m - a + R) + [m > 0] G(-m - a + R) + [m < n-1] G(2n - 2 - m - a + R)),   G = 0 outside [0, n).
// The single fold is exact because R < n (reflect padding requires it).
#pragma once

#include "common.cuh"

namespace b200drr {

// torch "reflect" padding index for -n < i < 2n - 1 (single fold); clamped so that a halo position that is never used stays in
// bounds
B200_HD int reflect_index(int i, int n)
{
    i = i < 0 ? -i : i;
    i = i > n - 1 ? 2 * (n - 1) - i : i;
    return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
}

// horizontal blur of image row `row` (already a valid row index) at column x (0 <= x < W)
B200_HD float sobel_blur_row(const float* img, int W, int row, int x, const float* w, int k)
{
    const int R = k >> 1;
    const float* r = img + (int64_t)row * W;
    float acc = 0.0f;
    for (int a = 0; a < k; ++a) acc += w[a] * ldg(r + reflect_index(x + a - R, W));
    return acc;
}

// vertical blur from a column of horizontally blurred rows: col[a * stride] holds the row refl(y + a - R)
B200_HD float sobel_blur_col(const float* col, int64_t stride, const float* w, int k)
{
    float acc = 0.0f;
    for (int a = 0; a < k; ++a) acc += w[a] * col[a * stride];
    return acc;
}

// Sobel at one pixel from the 3x3 neighbourhood b[r][c] = Bl[y + r - 1][x + c - 1] (zero outside the image)
B200_HD void sobel_stencil(const float b[3][3], float& gx, float& gy)
{
    gx = (b[0][0] - b[0][2]) + 2.0f * (b[1][0] - b[1][2]) + (b[2][0] - b[2][2]);
    gy = (b[0][0] + 2.0f * b[0][1] + b[0][2]) - (b[2][0] + 2.0f * b[2][1] + b[2][2]);
}

// transposed Sobel at pixel (y, x): gradient reaching Bl[y][x] from both output channels g0 = d/d gx, g1 = d/d gy [H][W]
B200_HD float sobel_stencil_adjoint(const float* g0, const float* g1, int H, int W, int y, int x)
{
    // out[oy][ox] reads Bl[oy + r - 1][ox + c - 1] with weight G[r][c]  =>  Bl[y][x] feeds out[y - r + 1][x - c + 1]
    float acc = 0.0f;
    for (int r = 0; r < 3; ++r) {
        const int oy = y - r + 1;
        if (oy < 0 || oy >= H) continue;
        for (int c = 0; c < 3; ++c) {
            const int ox = x - c + 1;
            if (ox < 0 || ox >= W) continue;
            const float wx = (c == 1) ? 0.0f : (c == 0 ? 1.0f : -1.0f) * (r == 1 ? 2.0f : 1.0f);
            const float wy = (r == 1) ? 0.0f : (r == 0 ? 1.0f : -1.0f) * (c == 1 ? 2.0f : 1.0f);
            const int64_t o = (int64_t)oy * W + ox;
            acc += wx * ldg(g0 + o) + wy * ldg(g1 + o);
        }
    }
    return acc;
}

// transposed 1-D blur along an axis of length n at index m: G(i) = src[(i - base) * stride] for 0 <= i < n, else 0.  Every
// index read lies in [m - R, m + R] (the folds land there too), so `src` only has to cover that range around m.
B200_HD float sobel_blur_adjoint(const float* src, int64_t stride, int base, int n, int m, const float* w, int k)
{
    const int R = k >> 1;
    float acc = 0.0f;
    for (int a = 0; a < k; ++a) {
        const int d = a - R;
        float t = 0.0f;
        int i = m - d;
        if (i >= 0 && i < n) t += src[(int64_t)(i - base) * stride];
        i = -m - d;
        if (m > 0 && i >= 0 && i < n) t += src[(int64_t)(i - base) * stride];
        i = 2 * n - 2 - m - d;
        if (m < n - 1 && i >= 0 && i < n) t += src[(int64_t)(i - base) * stride];
        acc += w[a] * t;
    }
    return acc;
}

}  // namespace b200drr
