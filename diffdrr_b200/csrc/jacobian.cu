// jacobian.cu -- per-pixel pose Jacobians J [B][H*W][P] from the sensitivities the pose-in training walk saves (sm_90a).
//
// Forward mode of the pose-in renderers: every pixel depends on one ray, and the walk already stored that ray's end-point
// partials, so J[b][n][k] = sum_i coef_i(n) tan_i(b, k) (jacobian_math.cuh) -- no walk, no reduction.  One thread per pixel;
// pose b's P folded tangents sit in shared memory (every thread reads the same one: a broadcast); the block's J rows are staged
// in shared memory and written back as one contiguous run.  Each pixel reads 32 B (Siddon) or 48 B (Trilinear) of
// sensitivities and writes 4P B: bandwidth-bound by construction.
#include "jacobian_math.cuh"
#include "kernels.h"

namespace b200drr {

namespace {

constexpr int kJacThreads = 256;

template <bool TRI>
__global__ void __launch_bounds__(kJacThreads) jac_sens_pose_kernel(const float4* __restrict__ sens, const float* __restrict__ dsrc,
                                                                    const float* __restrict__ dG, const float* __restrict__ dWd,
                                                                    const float* __restrict__ Wd, const float* __restrict__ rows,
                                                                    const float* __restrict__ cols,
                                                                    const float* __restrict__ drange, float* __restrict__ J, int H,
                                                                    int W, int P, int stop_grad)
{
    constexpr int kTerms = TRI ? kJacTermsTrilinear : kJacTermsSiddon;
    constexpr int kVec = TRI ? 3 : 2;  // float4 of sensitivities per pixel
    __shared__ float tan[kJacMaxP][kJacStride];
    __shared__ float wd[12];
    __shared__ float stage[kJacThreads * (kJacMaxP + 1)];
    const int b = blockIdx.y;
    const int Pp = P | 1;  // odd row pitch: the per-thread rows of `stage` fall in distinct banks
    for (int k = threadIdx.x; k < P; k += kJacThreads) {
        const int64_t bk = (int64_t)b * P + k;
        jac_fold_tangent(dsrc + bk * 3, dG + bk * 12, dWd + bk * 12, TRI ? drange[(int64_t)b * 2 * P + k] : 0.0f,
                         TRI ? drange[((int64_t)b * 2 + 1) * P + k] : 0.0f, tan[k]);
    }
    if (threadIdx.x < 12) wd[threadIdx.x] = Wd[b * 12 + threadIdx.x];
    __syncthreads();

    const int64_t N = (int64_t)H * W;
    const int64_t n0 = (int64_t)blockIdx.x * kJacThreads;
    const int64_t n = n0 + threadIdx.x;
    if (n < N) {
        const int h = (int)(n / W), w = (int)(n % W);
        float s[kVec * 4];
#pragma unroll
        for (int v = 0; v < kVec; ++v) {
            const float4 q = __ldg(sens + ((int64_t)b * N + n) * kVec + v);
            s[v * 4 + 0] = q.x;
            s[v * 4 + 1] = q.y;
            s[v * 4 + 2] = q.z;
            s[v * 4 + 3] = q.w;
        }
        float coef[kTerms];
        jac_coeffs<TRI>(s, __ldg(cols + w), __ldg(rows + h), wd, stop_grad != 0, coef);
        for (int k = 0; k < P; ++k) stage[threadIdx.x * Pp + k] = jac_dot<kTerms>(coef, tan[k]);
    }
    __syncthreads();
    const int cnt = (int)min((int64_t)kJacThreads, N - n0) * P;
    float* dst = J + ((int64_t)b * N + n0) * P;
    for (int i = threadIdx.x; i < cnt; i += kJacThreads) {
        const int row = i / P;
        dst[i] = stage[row * Pp + (i - row * P)];
    }
}

template <bool TRI>
cudaError_t launch_jac(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd, const float* rows,
                       const float* cols, const float* drange, float* J, int B, int H, int W, int P, int stop_grad,
                       cudaStream_t stream)
{
    const int64_t blocks = ((int64_t)H * W + kJacThreads - 1) / kJacThreads;
    jac_sens_pose_kernel<TRI><<<dim3((unsigned)blocks, (unsigned)B), kJacThreads, 0, stream>>>(
        (const float4*)sens, dsrc, dG, dWd, Wd, rows, cols, drange, J, H, W, P, stop_grad);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_siddon_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                        const float* rows, const float* cols, float* J, int B, int H, int W, int P, int stop_grad,
                                        cudaStream_t stream)
{
    return launch_jac<false>(sens, dsrc, dG, dWd, Wd, rows, cols, nullptr, J, B, H, W, P, stop_grad, stream);
}

cudaError_t launch_trilinear_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                           const float* rows, const float* cols, const float* drange, float* J, int B, int H, int W,
                                           int P, cudaStream_t stream)
{
    return launch_jac<true>(sens, dsrc, dG, dWd, Wd, rows, cols, drange, J, B, H, W, P, 0, stream);
}

}  // namespace b200drr
