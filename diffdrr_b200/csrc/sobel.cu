// sobel.cu -- Gaussian blur + Sobel gradients of one-channel image stacks and the exact adjoint (sm_90a).
//
// Replaces reference diffdrr/metrics.py:69-93 (Sobel: torchvision gaussian_blur with reflect padding, then a 3x3 Conv2d with
// zero padding), the front end of GradientNormalizedCrossCorrelation2d.  The math is in sobel_math.cuh; the launches are
//   forward   sobel_fwd_kernel          one CTA per 32 x 32 output tile: horizontal blur of the tile + (1 + R)-pixel halo into
//                                       shared memory, vertical blur of the tile + 1-pixel halo, both Sobel stencils -> [B][2][H][W]
//   backward  sobel_adjoint_kernel      transposed Sobel (zero padding)                          -> g_bl [B][H][W] (workspace)
//             blur_adjoint_kernel       one CTA per 32 x 32 tile: transposed horizontal blur of the tile's rows + R-row halo
//                                       into shared memory, then the transposed vertical blur; reflected taps fold back
// The 1-D Gaussian weights w[k] are a device array the caller computes (the host computes them with torchvision's own ops).
#include "kernels.h"
#include "sobel_math.cuh"

namespace b200drr {

namespace {

constexpr int kSobelTile = 32;
constexpr int kSobelThreads = 256;

inline int64_t sobel_fwd_smem(int k)
{
    const int R = k >> 1, hw = kSobelTile + 2;
    return ((int64_t)k + (int64_t)(hw + 2 * R) * hw + (int64_t)hw * hw) * (int64_t)sizeof(float);
}

inline int64_t blur_adjoint_smem(int k)
{
    const int R = k >> 1;
    return ((int64_t)k + (int64_t)(kSobelTile + 2 * R) * kSobelTile) * (int64_t)sizeof(float);
}

constexpr int64_t kSmemDefault = 48 * 1024;
constexpr int64_t kSmemMax = 227 * 1024;  // Hopper opt-in limit per CTA

}  // namespace

// grid (tiles over W, tiles over H, B).  x [B][H][W] -> out [B][2][H][W]
__global__ void __launch_bounds__(kSobelThreads) sobel_fwd_kernel(const float* __restrict__ x, float* __restrict__ out, int H, int W,
                                                                  const float* __restrict__ wts, int k)
{
    extern __shared__ float sm[];
    const int R = k >> 1, hw = kSobelTile + 2, hr = hw + 2 * R;
    float* w = sm;
    float* hb = w + k;        // [hr][hw]  rows y0-1-R .., columns x0-1 ..
    float* bl = hb + hr * hw;  // [hw][hw]  rows y0-1 .., columns x0-1 ..  (zero outside the image)
    const int64_t n = (int64_t)H * W;
    const float* im = x + blockIdx.z * n;
    const int y0 = blockIdx.y * kSobelTile, x0 = blockIdx.x * kSobelTile;
    for (int i = threadIdx.x; i < k; i += kSobelThreads) w[i] = __ldg(wts + i);
    __syncthreads();
    for (int e = threadIdx.x; e < hr * hw; e += kSobelThreads) {
        const int gy = y0 - 1 - R + e / hw, gx = x0 - 1 + e % hw;
        hb[e] = (gx >= 0 && gx < W) ? sobel_blur_row(im, W, reflect_index(gy, H), gx, w, k) : 0.0f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < hw * hw; e += kSobelThreads) {
        const int r = e / hw, c = e % hw, gy = y0 - 1 + r, gx = x0 - 1 + c;
        bl[e] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? sobel_blur_col(hb + r * hw + c, hw, w, k) : 0.0f;
    }
    __syncthreads();
    float* o = out + blockIdx.z * 2 * n;
    for (int e = threadIdx.x; e < kSobelTile * kSobelTile; e += kSobelThreads) {
        const int r = e / kSobelTile, c = e % kSobelTile, y = y0 + r, xx = x0 + c;
        if (y >= H || xx >= W) continue;
        float b[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) b[i][j] = bl[(r + i) * hw + c + j];
        float gx, gy;
        sobel_stencil(b, gx, gy);
        o[(int64_t)y * W + xx] = gx;
        o[n + (int64_t)y * W + xx] = gy;
    }
}

// grid (blocks over H x W, B).  gout [B][2][H][W] -> g_bl [B][H][W]
__global__ void __launch_bounds__(kSobelThreads) sobel_adjoint_kernel(const float* __restrict__ gout, float* __restrict__ g_bl, int H,
                                                                      int W)
{
    const int64_t n = (int64_t)H * W, t = (int64_t)blockIdx.x * kSobelThreads + threadIdx.x;
    if (t >= n) return;
    const float* g0 = gout + blockIdx.y * 2 * n;
    g_bl[blockIdx.y * n + t] = sobel_stencil_adjoint(g0, g0 + n, H, W, (int)(t / W), (int)(t % W));
}

// grid (tiles over W, tiles over H, B).  g_bl [B][H][W] -> g_x [B][H][W]
__global__ void __launch_bounds__(kSobelThreads) blur_adjoint_kernel(const float* __restrict__ g_bl, float* __restrict__ g_x, int H,
                                                                     int W, const float* __restrict__ wts, int k)
{
    extern __shared__ float sm[];
    const int R = k >> 1, T = kSobelTile, hr = T + 2 * R;
    float* w = sm;
    float* th = w + k;  // [hr][T]  rows m0-R .., columns n0 ..  (the horizontal adjoint)
    const int64_t n = (int64_t)H * W;
    const float* g = g_bl + blockIdx.z * n;
    const int m0 = blockIdx.y * T, n0 = blockIdx.x * T;
    for (int i = threadIdx.x; i < k; i += kSobelThreads) w[i] = __ldg(wts + i);
    __syncthreads();
    for (int e = threadIdx.x; e < hr * T; e += kSobelThreads) {
        const int gy = m0 - R + e / T, gx = n0 + e % T;
        th[e] = (gy >= 0 && gy < H && gx < W) ? sobel_blur_adjoint(g + (int64_t)gy * W, 1, 0, W, gx, w, k) : 0.0f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < T * T; e += kSobelThreads) {
        const int r = e / T, c = e % T, m = m0 + r, nn = n0 + c;
        if (m >= H || nn >= W) continue;
        g_x[blockIdx.z * n + (int64_t)m * W + nn] = sobel_blur_adjoint(th + c, T, m0 - R, H, m, w, k);
    }
}

int64_t sobel_workspace_bytes(int B, int H, int W) { return (int64_t)B * H * W * (int64_t)sizeof(float); }

bool sobel_kernel_fits(int k) { return sobel_fwd_smem(k) <= kSmemMax && blur_adjoint_smem(k) <= kSmemMax; }

static cudaError_t smem_opt_in(const void* fn, int64_t bytes)
{
    if (bytes <= kSmemDefault) return cudaSuccess;
    return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

static inline dim3 tiles(int B, int H, int W)
{
    return dim3((unsigned)((W + kSobelTile - 1) / kSobelTile), (unsigned)((H + kSobelTile - 1) / kSobelTile), (unsigned)B);
}

cudaError_t launch_sobel_fwd(const float* x, float* out, int B, int H, int W, const float* weights, int k, cudaStream_t stream)
{
    if (B > 65535 || !sobel_kernel_fits(k)) return cudaErrorInvalidValue;
    const int64_t smem = sobel_fwd_smem(k);
    cudaError_t e = smem_opt_in((const void*)sobel_fwd_kernel, smem);
    if (e != cudaSuccess) return e;
    sobel_fwd_kernel<<<tiles(B, H, W), kSobelThreads, (size_t)smem, stream>>>(x, out, H, W, weights, k);
    return cudaGetLastError();
}

cudaError_t launch_sobel_bwd(const float* gout, float* g_x, int B, int H, int W, const float* weights, int k, void* workspace,
                             cudaStream_t stream)
{
    if (B > 65535 || !sobel_kernel_fits(k)) return cudaErrorInvalidValue;
    const int64_t smem = blur_adjoint_smem(k);
    cudaError_t e = smem_opt_in((const void*)blur_adjoint_kernel, smem);
    if (e != cudaSuccess) return e;
    float* g_bl = (float*)workspace;
    sobel_adjoint_kernel<<<dim3((unsigned)(((int64_t)H * W + kSobelThreads - 1) / kSobelThreads), (unsigned)B), kSobelThreads, 0,
                           stream>>>(gout, g_bl, H, W);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    blur_adjoint_kernel<<<tiles(B, H, W), kSobelThreads, (size_t)smem, stream>>>(g_bl, g_x, H, W, weights, k);
    return cudaGetLastError();
}

}  // namespace b200drr
