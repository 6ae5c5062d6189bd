// hostemu_metrics.cpp -- TEST INFRASTRUCTURE: compiles the product's image-loss math (local_ncc_math.cuh, sobel_math.cuh) with
// g++ and loops over outputs on the CPU in the order the kernels of local_ncc.cu / sobel.cu use, so that the CPU-only build
// container can check the kernels' arithmetic against the reference goldens before any GPU time is spent.
// Never linked into libb200drr.so and never imported by the product package.
#include <vector>

#include "../../diffdrr_b200/csrc/local_ncc_math.cuh"
#include "../../diffdrr_b200/csrc/sobel_math.cuh"

using namespace b200drr;

extern "C" {
// local_ncc.cu on the CPU: the same passes (vertical moments -> windows -> fixed-order score; vertical + horizontal adjoint).
void emu_local_ncc_fwd(const float* x1, const float* x2, int B, int C, int H, int W, int p, float eps, float* stats, float* score)
{
    const int Hp = H - p + 1, Wp = W - p + 1;
    std::vector<double> V((size_t)kLnccStats * Hp * W);
    for (int b = 0; b < B; ++b) {
        double total = 0.0;
        for (int c = 0; c < C; ++c) {
            const long img = (long)b * C + c;
            for (int i = 0; i < Hp; ++i)
                for (int x = 0; x < W; ++x) lncc_vertical(x1 + img * H * W, x2 + img * H * W, H, W, p, i, x, V.data());
            for (int i = 0; i < Hp; ++i)
                for (int j = 0; j < Wp; ++j) total += lncc_window(V.data(), H, W, p, eps, i, j, stats + img * kLnccStats * Hp * Wp);
        }
        score[b] = (float)(total / ((double)C * Hp * Wp));
    }
}

void emu_local_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2, int B,
                       int C, int H, int W, int p)
{
    const int Hp = H - p + 1, Wp = W - p + 1;
    std::vector<double> VB((size_t)kLnccMaps * H * Wp);
    for (long img = 0; img < (long)B * C; ++img) {
        for (int y = 0; y < H; ++y)
            for (int j = 0; j < Wp; ++j) lncc_bwd_vertical(stats + img * kLnccStats * Hp * Wp, H, W, p, y, j, VB.data());
        const double k = (double)gscore[img / C] / ((double)C * Hp * Wp * p * p);
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) {
                const long q = img * H * W + (long)y * W + x;
                lncc_bwd_pixel(VB.data(), H, W, p, y, x, x1[q], x2[q], k, g_x1[q], g_x2[q]);
            }
    }
}

// sobel.cu on the CPU: horizontal blur (reflect) -> vertical blur -> Sobel stencils, and the adjoint in reverse.
void emu_sobel_fwd(const float* x, float* out, int B, int H, int W, const float* w, int k)
{
    const int R = k >> 1;
    const long n = (long)H * W;
    std::vector<float> hb((size_t)n), bl((size_t)(H + 2) * (W + 2), 0.0f);  // bl: 1-pixel zero border
    for (int b = 0; b < B; ++b) {
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) hb[(long)y * W + xx] = sobel_blur_row(x + b * n, W, y, xx, w, k);
        std::vector<float> col(k);
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) {
                for (int a = 0; a < k; ++a) col[a] = hb[(long)reflect_index(y + a - R, H) * W + xx];
                bl[(long)(y + 1) * (W + 2) + xx + 1] = sobel_blur_col(col.data(), 1, w, k);
            }
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) {
                float s[3][3];
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j) s[i][j] = bl[(long)(y + i) * (W + 2) + xx + j];
                sobel_stencil(s, out[b * 2 * n + (long)y * W + xx], out[b * 2 * n + n + (long)y * W + xx]);
            }
    }
}

void emu_sobel_bwd(const float* gout, float* g_x, int B, int H, int W, const float* w, int k)
{
    const long n = (long)H * W;
    std::vector<float> gbl((size_t)n), th((size_t)n);
    for (int b = 0; b < B; ++b) {
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) gbl[(long)y * W + xx] = sobel_stencil_adjoint(gout + b * 2 * n, gout + b * 2 * n + n, H, W, y, xx);
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) th[(long)y * W + xx] = sobel_blur_adjoint(gbl.data() + (long)y * W, 1, 0, W, xx, w, k);
        for (int y = 0; y < H; ++y)
            for (int xx = 0; xx < W; ++xx) g_x[b * n + (long)y * W + xx] = sobel_blur_adjoint(th.data() + xx, W, 0, H, y, w, k);
    }
}
}
