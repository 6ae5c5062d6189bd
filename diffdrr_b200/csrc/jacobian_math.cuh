// jacobian_math.cuh -- per-pixel pose Jacobian from the saved per-ray sensitivities (host+device; the kernels of jacobian.cu are
// thin wrappers, tests/hostemu compiles the same source).
//
// The pose-in kernels generate pixel (h, w)'s ray from three per-pose matrices: with p = (cols[w], rows[h], 1, 1)
//   target = G.p (voxel space),   world ray dl = Wd.p,   ray length L = |dl|,   source = src.
// The sensitivities walk saved dI/dtarget, dI/dL (= I / L) and dI/dsource per pixel (Trilinear also the two sampling-range
// partials), so along a tangent (dsrc, dG, dWd, drange) of those inputs
//   dI = dI/dtgt . dG p + dI/dL (dl . dWd p) / L + dI/dsrc . dsrc  [+ dI/dalphamin drange0 + dI/dalphamax drange1]
// (the dWd term is dropped for stop_gradients_through_grid_sample, as the Siddon backward drops it).  dI is linear in the
// tangent: dI = sum_i coef_i tan_i, and the coefficients are exactly the per-pixel terms that sens_bwd_pose_kernel (siddon.cu) and
// trilinear_sens_bwd_pose_kernel (trilinear.cu) multiply by the upstream gradient and sum -- this is the forward twin of those
// reductions, so sum_n g_n dI_n = <their reduced gradients, tangent>.
//
// Folded tangent layout (the homogeneous 1 multiplies columns 2 and 3 alike, so their tangents are summed once per pose):
//   [0..8]   dG[a][0], dG[a][1], dG[a][2] + dG[a][3]     a = 0, 1, 2
//   [9..17]  dWd, likewise
//   [18..20] dsrc
//   [21, 22] drange {alphamin, alphamax}                  (Trilinear only)
#pragma once

#include "common.cuh"

namespace b200drr {

constexpr int kJacTermsSiddon = 21;
constexpr int kJacTermsTrilinear = 23;
constexpr int kJacStride = 24;  // floats per folded tangent in shared memory
constexpr int kJacMaxP = 16;    // pose parameters per pose

B200_HD float jac_rsqrt(float x)
{
#if defined(__CUDA_ARCH__)
    return rsqrtf(x);
#else
    return 1.0f / sqrtf(x);
#endif
}

// The folded tangent of one (pose, parameter): dsrc [3], dG [3][4], dWd [3][4], drange {d alphamin, d alphamax}.
B200_HD void jac_fold_tangent(const float* dsrc, const float* dG, const float* dWd, float dr0, float dr1, float* tan)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        tan[a * 3 + 0] = dG[a * 4 + 0];
        tan[a * 3 + 1] = dG[a * 4 + 1];
        tan[a * 3 + 2] = dG[a * 4 + 2] + dG[a * 4 + 3];
        tan[9 + a * 3 + 0] = dWd[a * 4 + 0];
        tan[9 + a * 3 + 1] = dWd[a * 4 + 1];
        tan[9 + a * 3 + 2] = dWd[a * 4 + 2] + dWd[a * 4 + 3];
        tan[18 + a] = dsrc[a];
    }
    tan[21] = dr0;
    tan[22] = dr1;
    tan[23] = 0.0f;
}

// The coefficients of one pixel.  sens: Siddon { dI/dtgt[3], S | dI/dsrc[3], 0 }, Trilinear additionally
// { .., dI/dalphamin | dI/dalphamax, 0, 0, 0 } (include/b200drr.h); wd = the pose's Wd [3][4]; (c, r) = cols[w], rows[h].
template <bool TRI>
B200_HD void jac_coeffs(const float* sens, float c, float r, const float* wd, bool stop_grad, float* coef)
{
    float dl[3], l2 = 0.0f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        dl[a] = fmaf(wd[a * 4], c, fmaf(wd[a * 4 + 1], r, wd[a * 4 + 2] + wd[a * 4 + 3]));
        l2 = fmaf(dl[a], dl[a], l2);
    }
    const float gl = stop_grad ? 0.0f : sens[3] * jac_rsqrt(fmaxf(l2, 1e-30f));
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float t = sens[a], u = gl * dl[a];
        coef[a * 3 + 0] = t * c;
        coef[a * 3 + 1] = t * r;
        coef[a * 3 + 2] = t;
        coef[9 + a * 3 + 0] = u * c;
        coef[9 + a * 3 + 1] = u * r;
        coef[9 + a * 3 + 2] = u;
        coef[18 + a] = sens[4 + a];
    }
    if (TRI) {
        coef[21] = sens[7];
        coef[22] = sens[8];
    }
}

// J = sum_i coef_i tan_i in a fixed order
template <int TERMS>
B200_HD float jac_dot(const float* coef, const float* tan)
{
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < TERMS; ++i) acc = fmaf(coef[i], tan[i], acc);
    return acc;
}

}  // namespace b200drr
