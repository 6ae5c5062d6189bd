// local_ncc.cu -- patch-wise (local) zero-normalised cross correlation of two image stacks and its gradient (sm_90a).
//
// Replaces the patch mode of reference diffdrr/metrics.py:16-44 (NormalizedCrossCorrelation2d(patch_size=p)), which unfolds
// every stride-1 p x p window into its own channel: a (B, C H' W' p^2) copy (40 MB per 256^2 image at p = 13) that autograd
// keeps several of.  The math is in local_ncc_math.cuh; the launches are
//   forward   lncc_vertical_kernel   vertical p-row sums of the five moments per column          -> V  (workspace, double)
//             lncc_window_kernel     horizontal p-column sums -> per-window stats + one partial score per CTA
//             lncc_finalize_kernel   one CTA per batch element, partials summed in a fixed order (no atomics: deterministic)
//   backward  lncc_bwd_vertical_kernel  vertical adjoint box sums of the seven window maps      -> VB (workspace, double)
//             lncc_bwd_pixel_kernel     horizontal adjoint box sums + closed-form gradient, fp32 out
// Every pass is O(p) per output, for any 1 <= p <= min(H, W).
#include "kernels.h"
#include "local_ncc_math.cuh"

namespace b200drr {

namespace {

constexpr int kLnccThreads = 256;

__device__ __forceinline__ double lncc_block_sum(double v)
{
    __shared__ double red[kLnccThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // `red` may still be read by the previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
#pragma unroll
        for (int w = 0; w < kLnccThreads / 32; ++w) t += red[w];  // fixed order
    return t;  // valid in thread 0
}

struct LnccShape {
    int B, C, H, W, p, Hp, Wp;
    int64_t v_elems, s_elems, b_elems;  // per image pair: V, stats, VB
    int win_blocks;                     // CTAs of lncc_window_kernel per image pair
};

LnccShape lncc_shape(int B, int C, int H, int W, int p)
{
    LnccShape s;
    s.B = B;
    s.C = C;
    s.H = H;
    s.W = W;
    s.p = p;
    s.Hp = H - p + 1;
    s.Wp = W - p + 1;
    s.v_elems = (int64_t)kLnccStats * s.Hp * W;
    s.s_elems = (int64_t)kLnccStats * s.Hp * s.Wp;
    s.b_elems = (int64_t)kLnccMaps * H * s.Wp;
    s.win_blocks = (int)(((int64_t)s.Hp * s.Wp + kLnccThreads - 1) / kLnccThreads);
    return s;
}

inline unsigned blocks_for(int64_t n) { return (unsigned)((n + kLnccThreads - 1) / kLnccThreads); }

}  // namespace

// grid (blocks over H' x W, B*C)
__global__ void __launch_bounds__(kLnccThreads) lncc_vertical_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                                                     int H, int W, int p, double* __restrict__ V)
{
    const int64_t img = blockIdx.y, t = (int64_t)blockIdx.x * kLnccThreads + threadIdx.x;
    const int Hp = H - p + 1;
    if (t >= (int64_t)Hp * W) return;
    const int64_t n = (int64_t)H * W;
    lncc_vertical(x1 + img * n, x2 + img * n, H, W, p, (int)(t / W), (int)(t % W), V + img * kLnccStats * Hp * (int64_t)W);
}

// grid (win_blocks, B*C).  partial[img * win_blocks + blockIdx.x] = sum of L over this CTA's windows
__global__ void __launch_bounds__(kLnccThreads) lncc_window_kernel(const double* __restrict__ V, int H, int W, int p, float eps,
                                                                   float* __restrict__ stats, double* __restrict__ partial)
{
    const int64_t img = blockIdx.y, t = (int64_t)blockIdx.x * kLnccThreads + threadIdx.x;
    const int Hp = H - p + 1, Wp = W - p + 1;
    double L = 0.0;
    if (t < (int64_t)Hp * Wp)
        L = lncc_window(V + img * kLnccStats * Hp * (int64_t)W, H, W, p, eps, (int)(t / Wp), (int)(t % Wp),
                        stats + img * kLnccStats * Hp * (int64_t)Wp);
    L = lncc_block_sum(L);
    if (threadIdx.x == 0) partial[img * gridDim.x + blockIdx.x] = L;
}

// grid (B).  score[b] = sum over the C channels and their partials / (C H' W')
__global__ void __launch_bounds__(kLnccThreads) lncc_finalize_kernel(const double* __restrict__ partial, int C, int blocks,
                                                                     int64_t windows, float* __restrict__ score)
{
    const int b = blockIdx.x;
    const double* q = partial + (int64_t)b * C * blocks;
    double acc = 0.0;
    for (int64_t k = threadIdx.x; k < (int64_t)C * blocks; k += kLnccThreads) acc += q[k];
    acc = lncc_block_sum(acc);
    if (threadIdx.x == 0) score[b] = (float)(acc / ((double)C * (double)windows));
}

// grid (blocks over H x W', B*C)
__global__ void __launch_bounds__(kLnccThreads) lncc_bwd_vertical_kernel(const float* __restrict__ stats, int H, int W, int p,
                                                                         double* __restrict__ VB)
{
    const int64_t img = blockIdx.y, t = (int64_t)blockIdx.x * kLnccThreads + threadIdx.x;
    const int Hp = H - p + 1, Wp = W - p + 1;
    if (t >= (int64_t)H * Wp) return;
    lncc_bwd_vertical(stats + img * kLnccStats * Hp * (int64_t)Wp, H, W, p, (int)(t / Wp), (int)(t % Wp),
                      VB + img * kLnccMaps * H * (int64_t)Wp);
}

// grid (blocks over H x W, B*C).  g_x1 / g_x2 may be null (that input needs no gradient).
__global__ void __launch_bounds__(kLnccThreads) lncc_bwd_pixel_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                                                      const double* __restrict__ VB, const float* __restrict__ gscore,
                                                                      float* __restrict__ g_x1, float* __restrict__ g_x2, int C,
                                                                      int H, int W, int p)
{
    const int64_t img = blockIdx.y, t = (int64_t)blockIdx.x * kLnccThreads + threadIdx.x;
    const int64_t n = (int64_t)H * W;
    if (t >= n) return;
    const int Hp = H - p + 1, Wp = W - p + 1;
    const double k = (double)__ldg(gscore + img / C) / ((double)C * (double)Hp * (double)Wp * (double)p * (double)p);
    float g1, g2;
    lncc_bwd_pixel(VB + img * kLnccMaps * H * (int64_t)Wp, H, W, p, (int)(t / W), (int)(t % W), __ldg(x1 + img * n + t),
                   __ldg(x2 + img * n + t), k, g1, g2);
    if (g_x1) g_x1[img * n + t] = g1;
    if (g_x2) g_x2[img * n + t] = g2;
}

int64_t local_ncc_workspace_bytes(int B, int C, int H, int W, int p)
{
    const LnccShape s = lncc_shape(B, C, H, W, p);
    const int64_t fwd = (int64_t)B * C * (s.v_elems + s.win_blocks), bwd = (int64_t)B * C * s.b_elems;
    return (fwd > bwd ? fwd : bwd) * (int64_t)sizeof(double);
}

cudaError_t launch_local_ncc_fwd(const float* x1, const float* x2, int B, int C, int H, int W, int p, float eps, void* workspace,
                                 float* stats, float* score, cudaStream_t stream)
{
    if ((int64_t)B * C > 65535 || p < 1 || p > H || p > W) return cudaErrorInvalidValue;
    const LnccShape s = lncc_shape(B, C, H, W, p);
    double* V = (double*)workspace;
    double* partial = V + (int64_t)B * C * s.v_elems;
    const unsigned imgs = (unsigned)(B * C);
    lncc_vertical_kernel<<<dim3(blocks_for((int64_t)s.Hp * W), imgs), kLnccThreads, 0, stream>>>(x1, x2, H, W, p, V);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    lncc_window_kernel<<<dim3((unsigned)s.win_blocks, imgs), kLnccThreads, 0, stream>>>(V, H, W, p, eps, stats, partial);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    lncc_finalize_kernel<<<(unsigned)B, kLnccThreads, 0, stream>>>(partial, C, s.win_blocks, (int64_t)s.Hp * s.Wp, score);
    return cudaGetLastError();
}

cudaError_t launch_local_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2,
                                 int B, int C, int H, int W, int p, void* workspace, cudaStream_t stream)
{
    if ((int64_t)B * C > 65535 || p < 1 || p > H || p > W) return cudaErrorInvalidValue;
    const LnccShape s = lncc_shape(B, C, H, W, p);
    double* VB = (double*)workspace;
    const unsigned imgs = (unsigned)(B * C);
    lncc_bwd_vertical_kernel<<<dim3(blocks_for((int64_t)H * s.Wp), imgs), kLnccThreads, 0, stream>>>(stats, H, W, p, VB);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    lncc_bwd_pixel_kernel<<<dim3(blocks_for((int64_t)H * W), imgs), kLnccThreads, 0, stream>>>(x1, x2, VB, gscore, g_x1, g_x2, C, H,
                                                                                               W, p);
    return cudaGetLastError();
}

}  // namespace b200drr
