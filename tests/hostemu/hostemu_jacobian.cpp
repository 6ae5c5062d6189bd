// hostemu_jacobian.cpp -- TEST INFRASTRUCTURE: compiles the product's per-pixel pose-Jacobian math (jacobian_math.cuh) with g++
// and runs it over the pixels in the order of jacobian.cu's kernels, so that the CPU-only build container can check the kernels'
// arithmetic before any GPU time is spent.  Never linked into libb200drr.so and never imported by the product package.
#include <vector>

#include "../../diffdrr_b200/csrc/jacobian_math.cuh"

using namespace b200drr;

extern "C" {
// jac_sens_pose_kernel<tri> on the CPU: J [B][H*W][P] from sens [B][H*W][8 | 12] and the per-pose tangents
void emu_jac_sens_pose(int tri, const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                       const float* rows, const float* cols, const float* drange, float* J, int B, int H, int W, int P, int stop_grad)
{
    const long N = (long)H * W;
    const int nv = tri ? 12 : 8;
    std::vector<float> tan((size_t)P * kJacStride);
    float coef[kJacTermsTrilinear];
    for (int b = 0; b < B; ++b) {
        for (int k = 0; k < P; ++k) {
            const long bk = (long)b * P + k;
            jac_fold_tangent(dsrc + bk * 3, dG + bk * 12, dWd + bk * 12, tri ? drange[(long)b * 2 * P + k] : 0.0f,
                             tri ? drange[((long)b * 2 + 1) * P + k] : 0.0f, &tan[(size_t)k * kJacStride]);
        }
        for (long n = 0; n < N; ++n) {
            const float* s = sens + ((long)b * N + n) * nv;
            const float c = cols[n % W], r = rows[n / W];
            float* out = J + ((long)b * N + n) * P;
            if (tri) {
                jac_coeffs<true>(s, c, r, Wd + b * 12, false, coef);
                for (int k = 0; k < P; ++k) out[k] = jac_dot<kJacTermsTrilinear>(coef, &tan[(size_t)k * kJacStride]);
            } else {
                jac_coeffs<false>(s, c, r, Wd + b * 12, stop_grad != 0, coef);
                for (int k = 0; k < P; ++k) out[k] = jac_dot<kJacTermsSiddon>(coef, &tan[(size_t)k * kJacStride]);
            }
        }
    }
}
}
