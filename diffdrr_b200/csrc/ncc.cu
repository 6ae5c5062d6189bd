// ncc.cu -- zero-normalised cross correlation of two image stacks and its gradient, three launches per training step (sm_90a).
//
// Replaces reference diffdrr/metrics.py:21-44 (NormalizedCrossCorrelation2d, patch_size = None) on the registration loop
// (registration.py:14-50 + the loss): ~40 ATen launches per step of a loop whose renderer takes 0.14 ms -- at one pose per
// step the loop is launch-bound, not bandwidth-bound, so the metric is collapsed to
//   ncc_partial_kernel   one pass over both images: 5 moments per (image pair, 2048-pixel chunk), double accumulation,
//                        written to a workspace in a fixed order (no atomics: the result is run-to-run deterministic)
//   ncc_finalize_kernel  one CTA per batch element: chunk partials -> NccStats per channel, score[b] = mean_c L_c
//   ncc_bwd_kernel       elementwise closed-form gradient (ncc_math.cuh), float4 in / float4 out
// Every image is read once forward and once backward: 8 B/pixel + 8 (or 16) B/pixel -- HBM/L2-bound by construction.
#include "kernels.h"
#include "ncc_math.cuh"

namespace b200drr {

namespace {

constexpr int kNccThreads = 256;

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// block-wide sum of the five moments; the result is valid in thread 0
__device__ __forceinline__ NccSums block_sum(NccSums a)
{
    __shared__ double red[5][kNccThreads / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    a.s1 = warp_sum(a.s1);
    a.s2 = warp_sum(a.s2);
    a.q1 = warp_sum(a.q1);
    a.q2 = warp_sum(a.q2);
    a.p = warp_sum(a.p);
    __syncthreads();  // `red` may still be read by the previous call
    if (lane == 0) {
        red[0][warp] = a.s1;
        red[1][warp] = a.s2;
        red[2][warp] = a.q1;
        red[3][warp] = a.q2;
        red[4][warp] = a.p;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        NccSums t = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int w = 0; w < kNccThreads / 32; ++w) {  // fixed order
            t.s1 += red[0][w];
            t.s2 += red[1][w];
            t.q1 += red[2][w];
            t.q2 += red[3][w];
            t.p += red[4][w];
        }
        a = t;
    }
    return a;
}

}  // namespace

// grid (chunks, B*C).  `vec` = both images 16-byte aligned and N % 4 == 0.
__global__ void __launch_bounds__(kNccThreads) ncc_partial_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                                                  int64_t N, int vec, double* __restrict__ partial)
{
    const int64_t img = blockIdx.y;
    const int64_t lo = (int64_t)blockIdx.x * kNccChunk;
    const int64_t hi = lo + kNccChunk < N ? lo + kNccChunk : N;
    const float* a = x1 + img * N;
    const float* b = x2 + img * N;
    NccSums acc = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (vec) {
        const float4* a4 = reinterpret_cast<const float4*>(a);
        const float4* b4 = reinterpret_cast<const float4*>(b);
        for (int64_t i = (lo >> 2) + threadIdx.x; i < (hi >> 2); i += kNccThreads) {
            const float4 u = __ldg(a4 + i), v = __ldg(b4 + i);
            ncc_accumulate(acc, u.x, v.x);
            ncc_accumulate(acc, u.y, v.y);
            ncc_accumulate(acc, u.z, v.z);
            ncc_accumulate(acc, u.w, v.w);
        }
    } else {
        for (int64_t i = lo + threadIdx.x; i < hi; i += kNccThreads) ncc_accumulate(acc, __ldg(a + i), __ldg(b + i));
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) {
        double* o = partial + (img * gridDim.x + blockIdx.x) * 5;
        o[0] = acc.s1;
        o[1] = acc.s2;
        o[2] = acc.q1;
        o[3] = acc.q2;
        o[4] = acc.p;
    }
}

// grid (B).  stats[(b*C + c)] = NccStats of the pair, score[b] = mean over the C channels.
__global__ void __launch_bounds__(kNccThreads) ncc_finalize_kernel(const double* __restrict__ partial, int chunks, int C, int64_t N,
                                                                   float eps, NccStats* __restrict__ stats, float* __restrict__ score)
{
    const int b = blockIdx.x;
    double total = 0.0;  // thread 0 only
    for (int c = 0; c < C; ++c) {
        const double* p = partial + ((int64_t)(b * C + c) * chunks) * 5;
        NccSums acc = {0.0, 0.0, 0.0, 0.0, 0.0};
        for (int k = threadIdx.x; k < chunks; k += kNccThreads) {
            acc.s1 += p[k * 5 + 0];
            acc.s2 += p[k * 5 + 1];
            acc.q1 += p[k * 5 + 2];
            acc.q2 += p[k * 5 + 3];
            acc.p += p[k * 5 + 4];
        }
        acc = block_sum(acc);
        if (threadIdx.x == 0) {
            const NccStats s = ncc_finalize(acc, N, eps);
            stats[b * C + c] = s;
            total += (double)s.score;
        }
    }
    if (threadIdx.x == 0) score[b] = (float)(total / (double)C);
}

// grid (chunks, B*C).  g_x1 / g_x2 may be null (that input needs no gradient).
__global__ void __launch_bounds__(kNccThreads) ncc_bwd_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                                              const NccStats* __restrict__ stats, const float* __restrict__ gscore,
                                                              float* __restrict__ g_x1, float* __restrict__ g_x2, int C, int64_t N,
                                                              int vec)
{
    const int64_t img = blockIdx.y;
    const int64_t lo = (int64_t)blockIdx.x * kNccChunk;
    const int64_t hi = lo + kNccChunk < N ? lo + kNccChunk : N;
    const NccStats s = stats[img];
    const float k = __ldg(gscore + img / C) / ((float)C * (float)N);
    const float* a = x1 + img * N;
    const float* b = x2 + img * N;
    float* ga = g_x1 ? g_x1 + img * N : nullptr;
    float* gb = g_x2 ? g_x2 + img * N : nullptr;
    if (vec) {
        const float4* a4 = reinterpret_cast<const float4*>(a);
        const float4* b4 = reinterpret_cast<const float4*>(b);
        for (int64_t i = (lo >> 2) + threadIdx.x; i < (hi >> 2); i += kNccThreads) {
            const float4 u = __ldg(a4 + i), v = __ldg(b4 + i);
            float4 gu, gv;
            ncc_grad(s, k, u.x, v.x, gu.x, gv.x);
            ncc_grad(s, k, u.y, v.y, gu.y, gv.y);
            ncc_grad(s, k, u.z, v.z, gu.z, gv.z);
            ncc_grad(s, k, u.w, v.w, gu.w, gv.w);
            if (ga) reinterpret_cast<float4*>(ga)[i] = gu;
            if (gb) reinterpret_cast<float4*>(gb)[i] = gv;
        }
    } else {
        for (int64_t i = lo + threadIdx.x; i < hi; i += kNccThreads) {
            float gu, gv;
            ncc_grad(s, k, __ldg(a + i), __ldg(b + i), gu, gv);
            if (ga) ga[i] = gu;
            if (gb) gb[i] = gv;
        }
    }
}

static inline int ncc_chunks(int64_t N) { return (int)((N + kNccChunk - 1) / kNccChunk); }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int64_t ncc_workspace_bytes(int B, int C, int64_t N) { return (int64_t)B * C * ncc_chunks(N) * 5 * (int64_t)sizeof(double); }

cudaError_t launch_ncc_fwd(const float* x1, const float* x2, int B, int C, int64_t N, float eps, void* workspace, float* stats,
                           float* score, cudaStream_t stream)
{
    const int chunks = ncc_chunks(N);
    if ((int64_t)B * C > 65535 || N > ((int64_t)1 << 40)) return cudaErrorInvalidValue;
    const int vec = (N % 4 == 0) && aligned16(x1) && aligned16(x2);
    ncc_partial_kernel<<<dim3((unsigned)chunks, (unsigned)(B * C)), kNccThreads, 0, stream>>>(x1, x2, N, vec, (double*)workspace);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ncc_finalize_kernel<<<(unsigned)B, kNccThreads, 0, stream>>>((const double*)workspace, chunks, C, N, eps, (NccStats*)stats, score);
    return cudaGetLastError();
}

cudaError_t launch_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2,
                           int B, int C, int64_t N, cudaStream_t stream)
{
    if ((int64_t)B * C > 65535) return cudaErrorInvalidValue;
    const int vec = (N % 4 == 0) && aligned16(x1) && aligned16(x2) && (!g_x1 || aligned16(g_x1)) && (!g_x2 || aligned16(g_x2));
    ncc_bwd_kernel<<<dim3((unsigned)ncc_chunks(N), (unsigned)(B * C)), kNccThreads, 0, stream>>>(
        x1, x2, (const NccStats*)stats, gscore, g_x1, g_x2, C, N, vec);
    return cudaGetLastError();
}

}  // namespace b200drr
