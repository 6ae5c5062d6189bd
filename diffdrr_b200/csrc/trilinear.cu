// trilinear.cu -- fixed-step trilinear ray-marching DRR kernels for sm_90a (forward + backward).
// One thread marches one ray (ray_math.cuh); blockIdx.y is the pose, blockIdx.x tiles the rays of that pose.
#include "kernels.h"
#include "ray_math.cuh"

namespace b200drr {

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) trilinear_fwd_kernel(const float* __restrict__ vol, VolDims dims,
                                                                 const float* __restrict__ src,
                                                                 const float* __restrict__ tgt,
                                                                 const float* __restrict__ raylen,
                                                                 float* __restrict__ out, int64_t N, float shift,
                                                                 float eps, int P,
                                                                 const float* __restrict__ alpha_range, int reduce,
                                                                 int align_corners)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    const float acc = trilinear_ray_fwd(vol, dims, ray, shift, P, amin, amax, reduce, align_corners);
    // reference order is (L * v_m) * step per sample; L and step are per-ray constants and are factored out
    out[r] = acc * (__ldg(raylen + r) * step);
}

__global__ void __launch_bounds__(kThreads) trilinear_bwd_kernel(
    const float* __restrict__ vol, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, const float* __restrict__ gout, float* __restrict__ g_src,
    float* __restrict__ g_tgt, float* __restrict__ g_raylen, float* __restrict__ g_vol,
    float* __restrict__ g_alpha_range, int64_t N, float shift, float eps, int P,
    const float* __restrict__ alpha_range, int align_corners, int reduce)
{
    __shared__ float red[32];
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const bool active = n < N;
    float gs[3] = {0.0f, 0.0f, 0.0f}, ga0 = 0.0f, ga1 = 0.0f;
    if (active) {
        const int64_t r = (int64_t)b * N + n;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        const TriGrad tg = reduce == 0
                               ? trilinear_ray_bwd(vol, dims, ray, shift, P, amin, amax, align_corners, g, L, g_vol)
                               : trilinear_ray_bwd_max(vol, dims, ray, shift, P, amin, amax, align_corners, g, L, g_vol);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            gs[a] = tg.gs[a];
            if (g_tgt) g_tgt[r * 3 + a] = tg.gt[a];
        }
        if (g_raylen) g_raylen[r] = g * step * tg.sumV;
        ga0 = tg.ga0;
        ga1 = tg.ga1;
    }
    if (g_src) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float tot = block_sum(gs[a], red);
            if (threadIdx.x == 0) atomicAdd(g_src + b * 3 + a, tot);
        }
    }
    if (g_alpha_range) {
        const float t0 = block_sum(ga0, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range, t0);
        const float t1 = block_sum(ga1, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range + 1, t1);
    }
}

// ---------------------------------------------------------------------------------------------------
// Detector-grid variants: CTA = TW x TH pixel tile, warp = 8 x 4 sub-tile (see siddon.cu).  Fixed-step marching is
// plane-synchronous by construction (every lane is at the same alpha in the same iteration), so the ray bundle of a
// warp shares sectors among its 8 corner gathers.
// ---------------------------------------------------------------------------------------------------
template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_fwd_grid_kernel(const float* __restrict__ vol, VolDims dims,
                                                                    const float* __restrict__ src,
                                                                    const float* __restrict__ tgt,
                                                                    const float* __restrict__ raylen,
                                                                    float* __restrict__ out, int H, int W, float shift,
                                                                    float eps, int P, const float* __restrict__ alpha_range)
{
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW;
    const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    if (px >= W || py >= H) return;
    const int b = blockIdx.y;
    const int64_t r = ((int64_t)b * H + py) * W + px;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    out[r] = trilinear_ray_fwd(vol, dims, ray, shift, P, amin, amax, 0, 0) * (__ldg(raylen + r) * step);
}

template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_bwd_grid_kernel(
    const float* __restrict__ vol, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, const float* __restrict__ gout, float* __restrict__ g_src,
    float* __restrict__ g_tgt, float* __restrict__ g_raylen, float* __restrict__ g_vol,
    float* __restrict__ g_alpha_range, int H, int W, float shift, float eps, int P,
    const float* __restrict__ alpha_range)
{
    __shared__ float red[32];
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW;
    const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    const int b = blockIdx.y;
    float gs[3] = {0.0f, 0.0f, 0.0f}, ga0 = 0.0f, ga1 = 0.0f;
    if (px < W && py < H) {
        const int64_t r = ((int64_t)b * H + py) * W + px;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        const TriGrad tg = trilinear_ray_bwd(vol, dims, ray, shift, P, amin, amax, 0, g, L, g_vol);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            gs[a] = tg.gs[a];
            if (g_tgt) g_tgt[r * 3 + a] = tg.gt[a];
        }
        if (g_raylen) g_raylen[r] = g * step * tg.sumV;
        ga0 = tg.ga0;
        ga1 = tg.ga1;
    }
    if (g_src) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float tot = block_sum(gs[a], red);
            if (threadIdx.x == 0) atomicAdd(g_src + b * 3 + a, tot);
        }
    }
    if (g_alpha_range) {
        const float t0 = block_sum(ga0, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range, t0);
        const float t1 = block_sum(ga1, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range + 1, t1);
    }
}

// Forward / backward from the packed-corner copy of the volume (ray_math.cuh: GatherPacked): one aligned 32-byte read
// per sample instead of 8 scalar gathers.  ncu: the scalar-gather kernel is 99 % L1-bound; this one reaches 65 % of the
// HBM roofline on BASELINE config 3's shape.
template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_fwd_packed_kernel(const float4* __restrict__ packed, VolDims dims,
                                                                      const float* __restrict__ src,
                                                                      const float* __restrict__ tgt,
                                                                      const float* __restrict__ raylen,
                                                                      float* __restrict__ out, int H, int W, float shift,
                                                                      float eps, int P, const float* __restrict__ alpha_range)
{
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW;
    const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    if (px >= W || py >= H) return;
    const int b = blockIdx.y;
    const int64_t r = ((int64_t)b * H + py) * W + px;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    out[r] = trilinear_ray_fwd_packed(packed, dims, ray, shift, P, amin, amax) * (__ldg(raylen + r) * step);
}

template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_bwd_packed_kernel(
    const float4* __restrict__ packed, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, const float* __restrict__ gout, float* __restrict__ g_src,
    float* __restrict__ g_tgt, float* __restrict__ g_raylen, float* __restrict__ g_alpha_range, int H, int W, float shift,
    float eps, int P, const float* __restrict__ alpha_range)
{
    __shared__ float red[32];
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW;
    const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    const int b = blockIdx.y;
    float gs[3] = {0.0f, 0.0f, 0.0f}, ga0 = 0.0f, ga1 = 0.0f;
    if (px < W && py < H) {
        const int64_t r = ((int64_t)b * H + py) * W + px;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        const TriGrad tg = trilinear_ray_bwd_packed(packed, dims, ray, shift, P, amin, amax, g, L);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            gs[a] = tg.gs[a];
            if (g_tgt) g_tgt[r * 3 + a] = tg.gt[a];
        }
        if (g_raylen) g_raylen[r] = g * step * tg.sumV;
        ga0 = tg.ga0;
        ga1 = tg.ga1;
    }
    if (g_src) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float tot = block_sum(gs[a], red);
            if (threadIdx.x == 0) atomicAdd(g_src + b * 3 + a, tot);
        }
    }
    if (g_alpha_range) {
        const float t0 = block_sum(ga0, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range, t0);
        const float t1 = block_sum(ga1, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range + 1, t1);
    }
}

// Slab-major packed kernels: blockIdx.x = (slab, pose, tile) with the slab slowest.  A slab is `slab` planes of base
// voxels along axis 0 (slab * (D1+1)*(D2+1)*32 bytes of the packed copy, sized to sit in L2), so the poses of a batch
// share the packed cells through L2 instead of each streaming the 8x volume from HBM.  Partial sums are combined
// with red.global.add (outputs zero-filled by the launcher).
template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_fwd_packed_slab_kernel(
    const float4* __restrict__ packed, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, float* __restrict__ out, int B, int H, int W, int slab, float shift, float eps, int P,
    const float* __restrict__ alpha_range)
{
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW, tiles = tiles_x * ((H + TH - 1) / TH);
    int id = blockIdx.x;
    const int tile = id % tiles;
    id /= tiles;
    const int b = id % B, sl = id / B;
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    if (px >= W || py >= H) return;
    const int64_t r = ((int64_t)b * H + py) * W + px;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    const float s_lo = (float)(sl * slab - 1), s_hi = (float)((sl + 1) * slab - 1);
    const float part = trilinear_ray_fwd_packed(packed, dims, ray, shift, P, amin, amax, s_lo, s_hi);
    if (part != 0.0f) red_add(out + r, part * (__ldg(raylen + r) * step));
}

template <int TW, int TH>
__global__ void __launch_bounds__(TW* TH) trilinear_bwd_packed_slab_kernel(
    const float4* __restrict__ packed, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, const float* __restrict__ gout, float* __restrict__ g_src,
    float* __restrict__ g_tgt, float* __restrict__ g_raylen, float* __restrict__ g_alpha_range, int B, int H, int W,
    int slab, float shift, float eps, int P, const float* __restrict__ alpha_range)
{
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW, tiles = tiles_x * ((H + TH - 1) / TH);
    int id = blockIdx.x;
    const int tile = id % tiles;
    id /= tiles;
    const int b = id % B, sl = id / B;
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    float gs[3] = {0.0f, 0.0f, 0.0f}, ga0 = 0.0f, ga1 = 0.0f;
    if (px < W && py < H) {
        const int64_t r = ((int64_t)b * H + py) * W + px;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        const float s_lo = (float)(sl * slab - 1), s_hi = (float)((sl + 1) * slab - 1);
        const TriGrad tg = trilinear_ray_bwd_packed(packed, dims, ray, shift, P, amin, amax, g, L, s_lo, s_hi);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            gs[a] = tg.gs[a];
            if (g_tgt && tg.gt[a] != 0.0f) red_add(g_tgt + r * 3 + a, tg.gt[a]);
        }
        if (g_raylen && tg.sumV != 0.0f) red_add(g_raylen + r, g * step * tg.sumV);
        ga0 = tg.ga0;
        ga1 = tg.ga1;
    }
    // warp-level reductions, one atomic per warp (no block barrier)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float tot = warp_sum(gs[a]);
        if (g_src && lane == 0 && tot != 0.0f) atomicAdd(g_src + b * 3 + a, tot);
    }
    const float t0 = warp_sum(ga0), t1 = warp_sum(ga1);
    if (g_alpha_range && lane == 0) {
        if (t0 != 0.0f) atomicAdd(g_alpha_range, t0);
        if (t1 != 0.0f) atomicAdd(g_alpha_range + 1, t1);
    }
}

// packed[(i0+1)][(i1+1)][(i2+1)][c] = V[i0+o0][i1+o1][i2+o2] (0 outside), c = o0 | o1<<1 | o2<<2, i in [-1, D-1].
__global__ void __launch_bounds__(256) pack_corners_kernel(const float* __restrict__ vol, VolDims dims,
                                                           float4* __restrict__ packed)
{
    const int64_t n1 = dims.d[1] + 1, n2 = dims.d[2] + 1;
    const int64_t cells = (int64_t)(dims.d[0] + 1) * n1 * n2;
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (int64_t)gridDim.x * blockDim.x) {
        const int i2 = (int)(c % n2) - 1, i1 = (int)((c / n2) % n1) - 1, i0 = (int)(c / (n2 * n1)) - 1;
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int x = i0 + (k & 1), y = i1 + ((k >> 1) & 1), z = i2 + ((k >> 2) & 1);
            const bool inb = (unsigned)x < (unsigned)dims.d[0] && (unsigned)y < (unsigned)dims.d[1] &&
                             (unsigned)z < (unsigned)dims.d[2];
            v[k] = inb ? __ldg(vol + ((int64_t)x * dims.d[1] + y) * dims.d[2] + z) : 0.0f;
        }
        packed[2 * c] = make_float4(v[0], v[1], v[2], v[3]);
        packed[2 * c + 1] = make_float4(v[4], v[5], v[6], v[7]);
    }
}

cudaError_t launch_pack_corners(const float* vol, VolDims dims, float* packed, cudaStream_t stream)
{
    pack_corners_kernel<<<current_sm_count() * 16, 256, 0, stream>>>(vol, dims, (float4*)packed);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_fwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream)
{
    if (slab > 0) {
        const int n_slabs = (dims.d[0] + 1 + slab - 1) / slab;
        const int64_t blocks = (int64_t)((W + 15) / 16) * ((H + 15) / 16) * B * n_slabs;
        if (blocks > INT32_MAX) return cudaErrorInvalidValue;
        cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B * H * W, stream);
        if (e != cudaSuccess) return e;
        trilinear_fwd_packed_slab_kernel<16, 16><<<(unsigned)blocks, 256, 0, stream>>>(
            (const float4*)packed, dims, src, tgt, raylen, out, B, H, W, slab, shift, eps, n_points, alpha_range);
        return cudaGetLastError();
    }
    const dim3 grid((unsigned)(((W + 15) / 16) * ((H + 15) / 16)), (unsigned)B, 1);
    trilinear_fwd_packed_kernel<16, 16><<<grid, 256, 0, stream>>>((const float4*)packed, dims, src, tgt, raylen, out, H, W,
                                                                   shift, eps, n_points, alpha_range);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_bwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                        float* g_raylen, float* g_alpha_range, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream)
{
    if (g_src) {
        cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    if (slab > 0) {
        const int n_slabs = (dims.d[0] + 1 + slab - 1) / slab;
        const int64_t blocks = (int64_t)((W + 15) / 16) * ((H + 15) / 16) * B * n_slabs;
        if (blocks > INT32_MAX) return cudaErrorInvalidValue;
        const size_t n = (size_t)B * H * W;
        cudaError_t e = cudaSuccess;
        if (g_tgt) e = cudaMemsetAsync(g_tgt, 0, sizeof(float) * 3 * n, stream);
        if (e == cudaSuccess && g_raylen) e = cudaMemsetAsync(g_raylen, 0, sizeof(float) * n, stream);
        if (e != cudaSuccess) return e;
        trilinear_bwd_packed_slab_kernel<16, 16><<<(unsigned)blocks, 256, 0, stream>>>(
            (const float4*)packed, dims, src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_alpha_range, B, H, W, slab, shift,
            eps, n_points, alpha_range);
        return cudaGetLastError();
    }
    const dim3 grid((unsigned)(((W + 15) / 16) * ((H + 15) / 16)), (unsigned)B, 1);
    trilinear_bwd_packed_kernel<16, 16><<<grid, 256, 0, stream>>>((const float4*)packed, dims, src, tgt, raylen, gout, g_src,
                                                                   g_tgt, g_raylen, g_alpha_range, H, W, shift, eps, n_points,
                                                                   alpha_range);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// Forward WITH per-ray sensitivities from the packed copy (the training-step fast path; siddon.cu has the Siddon
// twin).  Every sample's 8 corners are in registers anyway, so the interpolant's gradient costs no extra traffic, and
// everything the closed-form backward accumulates is linear in the upstream gradient g.  One march with g = 1 yields
//   out[r] = L * step * sum V     and     sens[r] = { dI/dtgt[3], step*sum V | dI/dsrc[3], dI/dalphamin | dI/dalphamax, 0, 0, 0 }
// and the backward pass is the elementwise trilinear_sens_bwd_kernel.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void red_add4(float* addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <int TW, int TH, bool SLAB>
__global__ void __launch_bounds__(TW* TH) trilinear_sens_packed_kernel(
    const float4* __restrict__ packed, VolDims dims, const float* __restrict__ src, const float* __restrict__ tgt,
    const float* __restrict__ raylen, float* __restrict__ out, float* __restrict__ sens, int B, int H, int W, int slab,
    float shift, float eps, int P, const float* __restrict__ alpha_range, PoseRays pr)
{
    constexpr int WX = TW / 8;
    const int tiles_x = (W + TW - 1) / TW, tiles = tiles_x * ((H + TH - 1) / TH);
    int id = blockIdx.x;
    const int tile = id % tiles;
    id /= tiles;
    const int b = id % B, sl = id / B;  // sl == 0 when not slabbed
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    if (px >= W || py >= H) return;
    const int64_t r = ((int64_t)b * H + py) * W + px;
    float L;
    const Ray ray = make_ray(pr, src, tgt, raylen, b, r, px, py, eps, L);  // pr.G != nullptr: rays generated here (pose-in)
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    const float s_lo = SLAB ? (float)(sl * slab - 1) : -INFINITY, s_hi = SLAB ? (float)((sl + 1) * slab - 1) : INFINITY;
    const TriGrad tg = trilinear_ray_bwd_packed(packed, dims, ray, shift, P, amin, amax, 1.0f, L, s_lo, s_hi);
    const float sv = step * tg.sumV;
    float* sr = sens + r * 12;
    if (SLAB) {
        if (tg.sumV != 0.0f || tg.gt[0] != 0.0f || tg.gt[1] != 0.0f || tg.gt[2] != 0.0f || tg.ga0 != 0.0f || tg.ga1 != 0.0f) {
            red_add4(sr, tg.gt[0], tg.gt[1], tg.gt[2], sv);
            red_add4(sr + 4, tg.gs[0], tg.gs[1], tg.gs[2], tg.ga0);
            red_add(sr + 8, tg.ga1);
            red_add(out + r, tg.sumV * (L * step));  // bitwise the forward kernel's expression
        }
    } else {
        reinterpret_cast<float4*>(sr)[0] = make_float4(tg.gt[0], tg.gt[1], tg.gt[2], sv);
        reinterpret_cast<float4*>(sr)[1] = make_float4(tg.gs[0], tg.gs[1], tg.gs[2], tg.ga0);
        reinterpret_cast<float4*>(sr)[2] = make_float4(tg.ga1, 0.0f, 0.0f, 0.0f);
        out[r] = tg.sumV * (L * step);  // bitwise the forward kernel's expression
    }
}

// Forward with sensitivities from the PLAIN volume (8 scalar gathers per sample): arbitrary ray sets (H == 0: ray n of
// pose b, one thread per ray in row order) or the full detector grid (H > 0: 16x16 pixel tiles, 8x4 ray bundle per warp).
// Same sens layout as the packed kernel; align_corners supported (arbitrary-ray form only).
__global__ void __launch_bounds__(256) trilinear_sens_kernel(const float* __restrict__ vol, VolDims dims,
                                                             const float* __restrict__ src, const float* __restrict__ tgt,
                                                             const float* __restrict__ raylen, float* __restrict__ out,
                                                             float* __restrict__ sens, int64_t N, int H, int W, float shift,
                                                             float eps, int P, const float* __restrict__ alpha_range,
                                                             int align_corners)
{
    const int b = blockIdx.y;
    int64_t n;
    if (H > 0) {
        const int tiles_x = (W + 15) / 16;
        const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int px = tile_x * 16 + (warp % 2) * 8 + (lane & 7);
        const int py = tile_y * 16 + (warp / 2) * 4 + (lane >> 3);
        if (px >= W || py >= H) return;
        n = (int64_t)py * W + px;
    } else {
        n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= N) return;
    }
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    const float L = __ldg(raylen + r);
    const TriGrad tg = trilinear_ray_bwd(vol, dims, ray, shift, P, amin, amax, align_corners, 1.0f, L, nullptr);
    float* sr = sens + r * 12;
    reinterpret_cast<float4*>(sr)[0] = make_float4(tg.gt[0], tg.gt[1], tg.gt[2], step * tg.sumV);
    reinterpret_cast<float4*>(sr)[1] = make_float4(tg.gs[0], tg.gs[1], tg.gs[2], tg.ga0);
    reinterpret_cast<float4*>(sr)[2] = make_float4(tg.ga1, 0.0f, 0.0f, 0.0f);
    out[r] = tg.sumV * (L * step);  // bitwise the forward kernels' expression
}

cudaError_t launch_trilinear_fwd_sens(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                      float* out, float* sens, int B, int64_t N, int H, int W, float shift, float eps,
                                      int n_points, const float* alpha_range, int align_corners, cudaStream_t stream)
{
    if (H > 0 && ((int64_t)H * W != N || align_corners)) return cudaErrorInvalidValue;
    const int64_t blocks = H > 0 ? (int64_t)((W + 15) / 16) * ((H + 15) / 16) : (N + 255) / 256;
    if (blocks > INT32_MAX || B > 65535) return cudaErrorInvalidValue;
    trilinear_sens_kernel<<<dim3((unsigned)blocks, (unsigned)B), 256, 0, stream>>>(vol, dims, src, tgt, raylen, out, sens, N, H,
                                                                                 W, shift, eps, n_points, alpha_range,
                                                                                 align_corners);
    return cudaGetLastError();
}

// mask_to_channels backward (autograd of renderers.py:242-252): gout [B][C][N]; sample m carries the gradient of the
// channel its nearest label routed it to.  g_alpha_range accumulated into (caller zero-fills).
__global__ void __launch_bounds__(kThreads) trilinear_bwd_mask_kernel(
    const float* __restrict__ vol, const float* __restrict__ mask, VolDims dims, const float* __restrict__ src,
    const float* __restrict__ tgt, const float* __restrict__ raylen, const float* __restrict__ gout,
    float* __restrict__ g_src, float* __restrict__ g_tgt, float* __restrict__ g_raylen, float* __restrict__ g_vol,
    float* __restrict__ g_alpha_range, int64_t N, int C, float shift, float eps, int P,
    const float* __restrict__ alpha_range, int align_corners, int W)
{
    __shared__ float red[32];
    const int64_t n = tiled_ray_index(N, W);  // W > 0: full detector grid, threads in pixel tiles
    const int b = blockIdx.y;
    float gs[3] = {0.0f, 0.0f, 0.0f}, ga0 = 0.0f, ga1 = 0.0f;
    if (n >= 0) {
        const int64_t r = (int64_t)b * N + n;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r);
        const SampleGradMasked sg{mask, gout + (int64_t)b * C * N + n, N, C};
        const TriGrad tg = trilinear_ray_bwd_g(GatherPlain{vol}, dims, ray, shift, P, amin, amax, align_corners, 1.0f, L,
                                               g_vol, -INFINITY, INFINITY, sg);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            gs[a] = tg.gs[a];
            if (g_tgt) g_tgt[r * 3 + a] = tg.gt[a];
        }
        if (g_raylen) g_raylen[r] = step * tg.sumV;
        ga0 = tg.ga0;
        ga1 = tg.ga1;
    }
    if (g_src) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float tot = block_sum(gs[a], red);
            if (threadIdx.x == 0) atomicAdd(g_src + b * 3 + a, tot);
        }
    }
    if (g_alpha_range) {
        const float t0 = block_sum(ga0, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range, t0);
        const float t1 = block_sum(ga1, red);
        if (threadIdx.x == 0) atomicAdd(g_alpha_range + 1, t1);
    }
}

cudaError_t launch_trilinear_bwd_mask(const float* vol, const float* mask, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                      float* g_vol, float* g_alpha_range, int B, int64_t N, int C, float shift, float eps,
                                      int n_points, const float* alpha_range, int align_corners, cudaStream_t stream, int W)
{
    if (g_src) {
        const cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    trilinear_bwd_mask_kernel<<<tiled_ray_grid(B, N, W), kThreads, 0, stream>>>(
        vol, mask, dims, src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, g_alpha_range, N, C, shift, eps, n_points,
        alpha_range, align_corners, W);
    return cudaGetLastError();
}

static cudaError_t launch_sens_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                      float eps, int n_points, const float* alpha_range, int slab, cudaStream_t stream,
                                      PoseRays pr)
{
    const int64_t tiles = (int64_t)((W + 15) / 16) * ((H + 15) / 16);
    if (slab > 0) {
        const int n_slabs = (dims.d[0] + 1 + slab - 1) / slab;
        const int64_t blocks = tiles * B * n_slabs;
        if (blocks > INT32_MAX) return cudaErrorInvalidValue;
        const size_t n = (size_t)B * H * W;
        cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * n, stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(sens, 0, sizeof(float) * 12 * n, stream);
        if (e != cudaSuccess) return e;
        trilinear_sens_packed_kernel<16, 16, true><<<(unsigned)blocks, 256, 0, stream>>>(
            (const float4*)packed, dims, src, tgt, raylen, out, sens, B, H, W, slab, shift, eps, n_points, alpha_range, pr);
        return cudaGetLastError();
    }
    if (tiles * B > INT32_MAX) return cudaErrorInvalidValue;
    trilinear_sens_packed_kernel<16, 16, false><<<(unsigned)(tiles * B), 256, 0, stream>>>(
        (const float4*)packed, dims, src, tgt, raylen, out, sens, B, H, W, 0, shift, eps, n_points, alpha_range, pr);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_fwd_sens_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                             const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                             float eps, int n_points, const float* alpha_range, int slab,
                                             cudaStream_t stream)
{
    return launch_sens_packed(packed, dims, src, tgt, raylen, out, sens, B, H, W, shift, eps, n_points, alpha_range, slab, stream,
                              PoseRays{nullptr, nullptr, nullptr, nullptr});
}

// ---- pose-in entry (SURVEY 8f-2 for the trilinear renderer) -----------------------------------------------------------------
// The batch-global sampling range of renderers.py:217-222 (min over ALL rays of the slab-entry alpha, max of the slab-exit
// alpha, `_get_alpha_minmax` renderers.py:124-140 incl. its dims + 1 far plane) from in-kernel rays: values AND the ray that
// attains each, so that the host can rebuild the two scalars differentiably from the pose of those two rays alone.
__device__ __forceinline__ unsigned int ordered_bits(float f)
{
    const unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(unsigned int k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(256) alpha_range_pose_kernel(VolDims dims, const float* __restrict__ src, PoseRays pr,
                                                               unsigned long long* __restrict__ keys, int H, int W, float shift,
                                                               float eps)
{
    const int b = blockIdx.y;
    const int64_t N = (int64_t)H * W;
    unsigned long long kmin = ~0ull, kmax = 0ull;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (int64_t)gridDim.x * blockDim.x) {
        const int py = (int)(n / W), px = (int)(n % W);
        float L;
        const Ray ray = make_ray(pr, src, nullptr, nullptr, b, 0, px, py, eps, L);
        float lo = -INFINITY, hi = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float a0 = ((-shift) - ray.s[a]) / ray.d[a];
            const float a1 = (((float)dims.d[a] + (1.0f - shift)) - ray.s[a]) / ray.d[a];
            lo = fmaxf(lo, fminf(a0, a1));
            hi = fminf(hi, fmaxf(a0, a1));
        }
        lo = fmaxf(lo, 0.0f);
        hi = fminf(hi, 1.0f);
        const unsigned long long idx = (unsigned long long)((int64_t)b * N + n) & 0xffffffffull;
        const unsigned long long k0 = ((unsigned long long)ordered_bits(lo) << 32) | idx;
        const unsigned long long k1 = ((unsigned long long)ordered_bits(hi) << 32) | idx;
        kmin = k0 < kmin ? k0 : kmin;
        kmax = k1 > kmax ? k1 : kmax;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long m0 = __shfl_xor_sync(0xffffffffu, kmin, o), m1 = __shfl_xor_sync(0xffffffffu, kmax, o);
        kmin = m0 < kmin ? m0 : kmin;
        kmax = m1 > kmax ? m1 : kmax;
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(keys, kmin);
        atomicMax(keys + 1, kmax);
    }
}

__global__ void alpha_range_decode_kernel(const unsigned long long* __restrict__ keys, float* __restrict__ range,
                                          int64_t* __restrict__ arg)
{
    if (threadIdx.x < 2) {
        const unsigned long long k = keys[threadIdx.x];
        range[threadIdx.x] = from_ordered_bits((unsigned int)(k >> 32));
        arg[threadIdx.x] = (int64_t)(k & 0xffffffffull);
    }
}

cudaError_t launch_trilinear_alpha_range_pose(VolDims dims, const float* src, const float* G, const float* Wd, const float* rows,
                                              const float* cols, float* range, int64_t* arg, void* keys, int B, int H, int W,
                                              float shift, float eps, cudaStream_t stream)
{
    if ((int64_t)B * H * W > 0xffffffffll) return cudaErrorInvalidValue;
    unsigned long long* k = (unsigned long long*)keys;
    cudaError_t e = cudaMemsetAsync(k, 0xff, sizeof(unsigned long long), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(k + 1, 0, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const int chunks = (int)min((int64_t)64, ((int64_t)H * W + 255) / 256);
    alpha_range_pose_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, stream>>>(dims, src, PoseRays{G, Wd, rows, cols}, k, H, W,
                                                                                   shift, eps);
    alpha_range_decode_kernel<<<1, 32, 0, stream>>>(k, range, arg);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_fwd_sens_pose(const float* packed, VolDims dims, const float* src, const float* G, const float* Wd,
                                           const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                           float shift, float eps, int n_points, const float* alpha_range, int slab,
                                           cudaStream_t stream)
{
    return launch_sens_packed(packed, dims, src, nullptr, nullptr, out, sens, B, H, W, shift, eps, n_points, alpha_range, slab,
                              stream, PoseRays{G, Wd, rows, cols});
}

// gradients of the pose-in form reduced to the per-pose matrices (the trilinear twin of sens_bwd_pose_kernel, siddon.cu):
// target(h,w) = G.p and raylen = |Wd.p| with p = (cols[w], rows[h], 1, 1)  =>  g_G = sum g dI/dtgt p^T, g_Wd = sum g (dI/dL) (Wd.p / L) p^T
__global__ void __launch_bounds__(256) trilinear_sens_bwd_pose_kernel(const float4* __restrict__ sens, const float* __restrict__ gout,
                                                                      const float* __restrict__ Wd, const float* __restrict__ rows,
                                                                      const float* __restrict__ cols, float* __restrict__ g_src,
                                                                      float* __restrict__ g_G, float* __restrict__ g_Wd,
                                                                      float* __restrict__ g_alpha_range, int H, int W)
{
    __shared__ float red[32];
    const int b = blockIdx.y;
    const int64_t N = (int64_t)H * W;
    float acc[23];
#pragma unroll
    for (int i = 0; i < 23; ++i) acc[i] = 0.0f;
    const float* wd = Wd + b * 12;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (int64_t)gridDim.x * blockDim.x) {
        const int h = (int)(n / W), w = (int)(n % W);
        const float c = __ldg(cols + w), r = __ldg(rows + h);
        const int64_t ray = (int64_t)b * N + n;
        const float g = __ldg(gout + ray);
        const float4 t = __ldg(sens + ray * 3), s = __ldg(sens + ray * 3 + 1), u = __ldg(sens + ray * 3 + 2);
        float dl[3], l2 = 0.0f;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            dl[a] = fmaf(__ldg(wd + a * 4), c, fmaf(__ldg(wd + a * 4 + 1), r, __ldg(wd + a * 4 + 2) + __ldg(wd + a * 4 + 3)));
            l2 = fmaf(dl[a], dl[a], l2);
        }
        const float gl = g * t.w * rsqrtf(fmaxf(l2, 1e-30f));
        const float gt[3] = {g * t.x, g * t.y, g * t.z};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = gl * dl[a];
            acc[a * 3 + 0] = fmaf(gt[a], c, acc[a * 3 + 0]);
            acc[a * 3 + 1] = fmaf(gt[a], r, acc[a * 3 + 1]);
            acc[a * 3 + 2] += gt[a];
            acc[9 + a * 3 + 0] = fmaf(v, c, acc[9 + a * 3 + 0]);
            acc[9 + a * 3 + 1] = fmaf(v, r, acc[9 + a * 3 + 1]);
            acc[9 + a * 3 + 2] += v;
        }
        acc[18] = fmaf(g, s.x, acc[18]);
        acc[19] = fmaf(g, s.y, acc[19]);
        acc[20] = fmaf(g, s.z, acc[20]);
        acc[21] = fmaf(g, s.w, acc[21]);
        acc[22] = fmaf(g, u.x, acc[22]);
    }
#pragma unroll
    for (int i = 0; i < 23; ++i) {
        const float tot = block_sum(acc[i], red);
        if (threadIdx.x == 0) {
            if (i >= 21) {
                if (g_alpha_range) atomicAdd(g_alpha_range + (i - 21), tot);
            } else if (i >= 18) {
                atomicAdd(g_src + b * 3 + (i - 18), tot);
            } else {
                float* dst = (i < 9 ? g_G : g_Wd) + b * 12;
                const int a = (i % 9) / 3, k = i % 3;
                atomicAdd(dst + a * 4 + k, tot);
                if (k == 2) atomicAdd(dst + a * 4 + 3, tot);  // the homogeneous 1 multiplies column 3 as well
            }
        }
    }
}

cudaError_t launch_trilinear_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows,
                                           const float* cols, float* g_src, float* g_G, float* g_Wd, float* g_alpha_range, int B,
                                           int H, int W, cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(g_G, 0, sizeof(float) * 12 * (size_t)B, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(g_Wd, 0, sizeof(float) * 12 * (size_t)B, stream);
    if (e != cudaSuccess) return e;
    const int chunks = (int)min((int64_t)64, ((int64_t)H * W + 255) / 256);
    trilinear_sens_bwd_pose_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, stream>>>((const float4*)sens, gout, Wd, rows, cols,
                                                                                          g_src, g_G, g_Wd, g_alpha_range, H, W);
    return cudaGetLastError();
}

// g_tgt = g * dI/dtgt, g_raylen = g * step*sumV, g_src[b] = sum_n g * dI/dsrc, g_alpha_range += sum g * dI/d(alphamin, alphamax)
__global__ void __launch_bounds__(256) trilinear_sens_bwd_kernel(const float4* __restrict__ sens, const float* __restrict__ gout,
                                                                 float* __restrict__ g_src, float* __restrict__ g_tgt,
                                                                 float* __restrict__ g_raylen,
                                                                 float* __restrict__ g_alpha_range, int64_t N)
{
    __shared__ float red[32];
    const int b = blockIdx.y;
    float acc[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = (int64_t)b * N + n;
        const float g = __ldg(gout + r);
        const float4 t = __ldg(sens + r * 3), s = __ldg(sens + r * 3 + 1), u = __ldg(sens + r * 3 + 2);
        if (g_tgt) {
            g_tgt[r * 3 + 0] = g * t.x;
            g_tgt[r * 3 + 1] = g * t.y;
            g_tgt[r * 3 + 2] = g * t.z;
        }
        if (g_raylen) g_raylen[r] = g * t.w;
        acc[0] = fmaf(g, s.x, acc[0]);
        acc[1] = fmaf(g, s.y, acc[1]);
        acc[2] = fmaf(g, s.z, acc[2]);
        acc[3] = fmaf(g, s.w, acc[3]);
        acc[4] = fmaf(g, u.x, acc[4]);
    }
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        const float tot = block_sum(acc[i], red);
        if (threadIdx.x == 0) {
            if (i < 3) {
                if (g_src) atomicAdd(g_src + b * 3 + i, tot);
            } else if (g_alpha_range) {
                atomicAdd(g_alpha_range + (i - 3), tot);
            }
        }
    }
}

cudaError_t launch_trilinear_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                      float* g_alpha_range, int B, int64_t N, cudaStream_t stream)
{
    if (g_src) {
        const cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    const int chunks = (int)min((int64_t)64, (N + 255) / 256);
    trilinear_sens_bwd_kernel<<<dim3((unsigned)chunks, (unsigned)B), 256, 0, stream>>>((const float4*)sens, gout, g_src, g_tgt,
                                                                                     g_raylen, g_alpha_range, N);
    return cudaGetLastError();
}

template <int TW, int TH>
static cudaError_t tri_fwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                float* out, int B, int H, int W, float shift, float eps, int P, const float* ar,
                                cudaStream_t stream)
{
    const dim3 grid((unsigned)(((W + TW - 1) / TW) * ((H + TH - 1) / TH)), (unsigned)B, 1);
    trilinear_fwd_grid_kernel<TW, TH><<<grid, TW * TH, 0, stream>>>(vol, dims, src, tgt, raylen, out, H, W, shift, eps, P, ar);
    return cudaGetLastError();
}

template <int TW, int TH>
static cudaError_t tri_bwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_vol, float* g_ar,
                                int B, int H, int W, float shift, float eps, int P, const float* ar, cudaStream_t stream)
{
    if (g_src) {
        cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    const dim3 grid((unsigned)(((W + TW - 1) / TW) * ((H + TH - 1) / TH)), (unsigned)B, 1);
    trilinear_bwd_grid_kernel<TW, TH><<<grid, TW * TH, 0, stream>>>(vol, dims, src, tgt, raylen, gout, g_src, g_tgt, g_raylen,
                                                                   g_vol, g_ar, H, W, shift, eps, P, ar);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_fwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                      int n_points, const float* alpha_range, int variant, cudaStream_t stream)
{
    switch (variant) {
        case 0: return tri_fwd_grid<16, 8>(vol, dims, src, tgt, raylen, out, B, H, W, shift, eps, n_points, alpha_range, stream);
        case 1: return tri_fwd_grid<16, 16>(vol, dims, src, tgt, raylen, out, B, H, W, shift, eps, n_points, alpha_range, stream);
        case 2: return tri_fwd_grid<8, 8>(vol, dims, src, tgt, raylen, out, B, H, W, shift, eps, n_points, alpha_range, stream);
        case 3: return tri_fwd_grid<32, 8>(vol, dims, src, tgt, raylen, out, B, H, W, shift, eps, n_points, alpha_range, stream);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_trilinear_bwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                      float* g_raylen, float* g_vol, float* g_alpha_range, int B, int H, int W, float shift,
                                      float eps, int n_points, const float* alpha_range, int variant, cudaStream_t stream)
{
#define TB(TW, TH) \
    tri_bwd_grid<TW, TH>(vol, dims, src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, g_alpha_range, B, H, W, shift, eps, \
                         n_points, alpha_range, stream)
    switch (variant) {
        case 0: return TB(16, 8);
        case 1: return TB(16, 16);
        case 2: return TB(8, 8);
        case 3: return TB(32, 8);
        default: return cudaErrorInvalidValue;
    }
#undef TB
}

__global__ void __launch_bounds__(kThreads) trilinear_fwd_mask_kernel(const float* __restrict__ vol,
                                                                      const float* __restrict__ mask, VolDims dims,
                                                                      const float* __restrict__ src,
                                                                      const float* __restrict__ tgt,
                                                                      const float* __restrict__ raylen, float* out,
                                                                      int64_t N, int C, float shift, float eps, int P,
                                                                      const float* __restrict__ alpha_range,
                                                                      int align_corners, int W)
{
    const int64_t n = tiled_ray_index(N, W);
    if (n < 0) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    trilinear_ray_fwd_mask(vol, mask, dims, ray, shift, P, amin, amax, align_corners, __ldg(raylen + r) * step,
                           out + (int64_t)b * C * N + n, N, C);
}

cudaError_t launch_trilinear_fwd_mask(const float* vol, const float* mask, VolDims dims, const float* src,
                                      const float* tgt, const float* raylen, float* out, int B, int64_t N, int C,
                                      float shift, float eps, int n_points, const float* alpha_range, int align_corners,
                                      cudaStream_t stream, int W)
{
    static_assert(kThreads == 128, "tiled_ray_index assumes 128-thread CTAs");
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B * C * N, stream);
    if (e != cudaSuccess) return e;
    trilinear_fwd_mask_kernel<<<tiled_ray_grid(B, N, W), kThreads, 0, stream>>>(
        vol, mask, dims, src, tgt, raylen, out, N, C, shift, eps, n_points, alpha_range, align_corners, W);
    return cudaGetLastError();
}

static inline dim3 ray_grid(int B, int64_t N) { return dim3((unsigned)((N + kThreads - 1) / kThreads), (unsigned)B, 1); }

cudaError_t launch_trilinear_fwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int reduce, int align_corners,
                                 cudaStream_t stream)
{
    trilinear_fwd_kernel<<<ray_grid(B, N), kThreads, 0, stream>>>(vol, dims, src, tgt, raylen, out, N, shift, eps,
                                                                  n_points, alpha_range, reduce, align_corners);
    return cudaGetLastError();
}

cudaError_t launch_trilinear_bwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                 float* g_vol, float* g_alpha_range, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int align_corners, cudaStream_t stream,
                                 int reduce)
{
    if (g_src) {
        cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(float) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    trilinear_bwd_kernel<<<ray_grid(B, N), kThreads, 0, stream>>>(vol, dims, src, tgt, raylen, gout, g_src, g_tgt,
                                                                  g_raylen, g_vol, g_alpha_range, N, shift, eps,
                                                                  n_points, alpha_range, align_corners, reduce);
    return cudaGetLastError();
}

}  // namespace b200drr
