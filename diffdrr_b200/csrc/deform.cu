// deform.cu -- deformable (dense displacement field) trilinear DRR kernels for sm_90a (forward + backward; math in deform_math.cuh).
// One thread marches one ray; blockIdx.y is the pose, blockIdx.x a 16 x 8 pixel tile of a full detector grid (W > 0) or 128
// consecutive rays of any ray set (W == 0), as tiled_ray_index lays them out.
// g_src and the range partials go through one row of partial sums per backward CTA, added in a fixed order by
// polyrigid_finish_kernel (polyrigid.cu), and g_tgt / g_raylen are per ray, so all of them repeat bit for bit.  The field gradient
// is the one output accumulated with atomics (vector reductions, one per lattice node and flush): it repeats to fp32 reordering.
// The tangent (JVP) kernel writes one image value and one directional derivative per ray, with no shared memory and no atomics,
// so both repeat bit for bit.  The Jacobian kernel (DESIGN.md 6p) writes each pixel's 6K columns from one thread and grows the
// footprints with integer min / max atomics, which do not depend on order, so every output repeats bit for bit.  The backprojection kernel (the forward's transpose in the density) scatters into one volume gradient
// with scalar reductions, shared and per-pose fields alike: it repeats to fp32 reordering.
#include <climits>

#include "deform_math.cuh"
#include "kernels.h"

namespace b200drr {

constexpr int kDeformThreads = 128;
constexpr int kDeformWarps = kDeformThreads / 32;
constexpr int kDeformRow = 5;  // partial sums one backward CTA writes: g_src [3], g_alpha_range [2]

template <class Gather>
__global__ void __launch_bounds__(kDeformThreads, 6) deform_fwd_kernel(Gather gather, VolDims dims, PolyLattice lat, int Bf,
                                                                     const float* __restrict__ src, const float* __restrict__ tgt,
                                                                     const float* __restrict__ raylen, float* __restrict__ out,
                                                                     int64_t N, int W, float shift, float eps, int P,
                                                                     const float* __restrict__ alpha_range)
{
    const int b = blockIdx.y;
    const int64_t n = tiled_ray_index(N, W);
    if (n < 0) return;
    if (Bf != 1) lat.w += (int64_t)b * lat.g[0] * lat.g[1] * lat.g[2];
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    out[r] = deform_ray_fwd(gather, dims, lat, ray, shift, P, amin, amax) * (__ldg(raylen + r) * step);
}

template <class Gather>
__global__ void __launch_bounds__(kDeformThreads) deform_bwd_kernel(Gather gather, VolDims dims, PolyLattice lat, int Bf,
                                                                    const float* __restrict__ src, const float* __restrict__ tgt,
                                                                    const float* __restrict__ raylen, const float* __restrict__ gout,
                                                                    float* __restrict__ g_tgt, float* __restrict__ g_raylen,
                                                                    float* g_field, float* __restrict__ partial, int64_t N, int W,
                                                                    float shift, float eps, int P, const float* __restrict__ alpha_range)
{
    __shared__ float red[kDeformWarps][kDeformRow];
    const int b = blockIdx.y;
    const int64_t n = tiled_ray_index(N, W);
    float tail[kDeformRow] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    if (n >= 0) {
        const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
        if (Bf != 1) {
            lat.w += b * nodes;
            if (g_field) g_field += b * nodes * 4;
        }
        const int64_t r = (int64_t)b * N + n;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        int flushes;
        const TriGrad tg = deform_ray_bwd(gather, dims, lat, ray, shift, P, amin, amax, g, L, g_field, flushes);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            tail[a] = tg.gs[a];
            if (g_tgt) g_tgt[r * 3 + a] = tg.gt[a];
        }
        if (g_raylen) g_raylen[r] = g * step * tg.sumV;
        tail[3] = tg.ga0;
        tail[4] = tg.ga1;
    }
    // CTA sums in a fixed order: xor-shuffle tree within a warp, then the warps in index order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < kDeformRow; ++i) {
        const float v = warp_sum(tail[i]);
        if (lane == 0) red[warp][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < kDeformRow) {
        float v = red[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < kDeformWarps; ++w) v += red[w][threadIdx.x];
        partial[((int64_t)b * gridDim.x + blockIdx.x) * kDeformRow + threadIdx.x] = v;
    }
}

// jv[r] = L step sum_m G_m . v(x_m) along the tangent `tan` (deform_ray_jvp); img (may be null) = deform_fwd_kernel's out bit for bit
template <class Gather>
__global__ void __launch_bounds__(kDeformThreads) deform_jvp_kernel(Gather gather, VolDims dims, PolyLattice lat, PolyLattice tan,
                                                                    int Bf, const float* __restrict__ src, const float* __restrict__ tgt,
                                                                    const float* __restrict__ raylen, float* __restrict__ img,
                                                                    float* __restrict__ jv, int64_t N, int W, float shift, float eps,
                                                                    int P, const float* __restrict__ alpha_range)
{
    const int b = blockIdx.y;
    const int64_t n = tiled_ray_index(N, W);
    if (n < 0) return;
    if (Bf != 1) {
        const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
        lat.w += b * nodes;
        tan.w += b * nodes;
    }
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    float acc;
    const float d = deform_ray_jvp(gather, dims, lat, tan, ray, shift, P, amin, amax, acc);
    const float Ls = __ldg(raylen + r) * step;
    jv[r] = d * Ls;
    if (img) img[r] = acc * Ls;
}

// Per-pixel Jacobian along the 6K tangents `tan` [Bf][g0][g1][g2][6K] float4 (deform_ray_jac), full H x W grids only: img [B][H*W]
// (deform_fwd_kernel's bits), J [B][K][H*W][6] with column p = 6k + i, and rects [B][K][4] {w0, w1, h0, h1} grown with one integer
// atomicMin / atomicMax per (CTA, k) over the pixels whose ray touched structure k (polyrigid_rects_empty_kernel runs first).  The
// footprint reduction and the staged stores of each warp's 8 x 4 pixel bundle are polyrigid_jac_kernel's.
template <int KP, class Gather>
__global__ void __launch_bounds__(kDeformThreads) deform_jac_kernel(Gather gather, VolDims dims, PolyLattice lat, const float4* __restrict__ tan,
                                                                    int K, int Bf, const float* __restrict__ src,
                                                                    const float* __restrict__ tgt, const float* __restrict__ raylen,
                                                                    float* __restrict__ img, float* __restrict__ J, int* __restrict__ rects,
                                                                    int H, int W, float shift, float eps, int P,
                                                                    const float* __restrict__ alpha_range)
{
    __shared__ float2 stage[kDeformWarps][32 * 3];
    __shared__ int red[kDeformWarps][KP][4];
    const int b = blockIdx.y;
    const int64_t N = (int64_t)H * W;
    const int64_t n = tiled_ray_index(N, W);
    float Jp[KP * 6];
    unsigned touched = 0u;
#pragma unroll
    for (int p = 0; p < KP * 6; ++p) Jp[p] = 0.0f;
    if (n >= 0) {
        if (Bf != 1) {
            const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
            lat.w += b * nodes;
            tan += b * nodes * 6 * K;
        }
        const int64_t r = (int64_t)b * N + n;
        const Ray ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float Ls = __ldg(raylen + r) * step;
        int flushes;
        const float acc = deform_ray_jac<KP>(gather, dims, lat, tan, K, ray, shift, P, amin, amax, Jp, touched, flushes);
        img[r] = acc * Ls;
#pragma unroll
        for (int p = 0; p < KP * 6; ++p) Jp[p] *= Ls;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tiles_x = (W + 15) / 16;
    const int px0 = (blockIdx.x % tiles_x) * 16 + (warp & 1) * 8, py0 = (int)(blockIdx.x / tiles_x) * 8 + (warp >> 1) * 4;
    const int px = px0 + (lane & 7), py = py0 + (lane >> 3);
#pragma unroll
    for (int k = 0; k < KP; ++k) {
        const bool hit = n >= 0 && ((touched >> k) & 1u);
        const int w0 = __reduce_min_sync(0xffffffffu, hit ? px : INT_MAX), w1 = __reduce_max_sync(0xffffffffu, hit ? px : -1);
        const int h0 = __reduce_min_sync(0xffffffffu, hit ? py : INT_MAX), h1 = __reduce_max_sync(0xffffffffu, hit ? py : -1);
        if (lane == 0) {
            red[warp][k][0] = w0;
            red[warp][k][1] = w1;
            red[warp][k][2] = h0;
            red[warp][k][3] = h1;
        }
    }
    // stage[warp] holds the bundle's 4 rows x 8 pixels x 6 floats of one k: float2 j = row * 24 + pixel * 3 + i / 2
    float* st = reinterpret_cast<float*>(stage[warp]);
#pragma unroll
    for (int k = 0; k < KP; ++k) {
        if (k >= K) break;
#pragma unroll
        for (int i = 0; i < 6; ++i) st[lane * 6 + i] = Jp[k * 6 + i];
        __syncwarp();
        float* Jk = J + ((int64_t)b * K + k) * N * 6;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const int j = lane + 32 * q, row = j / 24, c = j % 24;
            const int x = px0 + c / 3, y = py0 + row;
            if (x < W && y < H) reinterpret_cast<float2*>(Jk + ((int64_t)y * W + x) * 6)[c % 3] = stage[warp][j];
        }
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x < K) {
        const int k = threadIdx.x;
        int r[4] = {red[0][k][0], red[0][k][1], red[0][k][2], red[0][k][3]};
#pragma unroll
        for (int w = 1; w < kDeformWarps; ++w) {
            r[0] = min(r[0], red[w][k][0]);
            r[1] = max(r[1], red[w][k][1]);
            r[2] = min(r[2], red[w][k][2]);
            r[3] = max(r[3], red[w][k][3]);
        }
        if (r[0] <= r[1]) {
            int* rk = rects + ((int64_t)b * K + k) * 4;
            atomicMin(rk, r[0]);
            atomicMax(rk + 1, r[1]);
            atomicMin(rk + 2, r[2]);
            atomicMax(rk + 3, r[3]);
        }
    }
}

// g_vol [D0][D1][D2] += the transpose of deform_fwd_kernel in the density, for upstream gradient gout (deform_ray_bproj)
__global__ void __launch_bounds__(kDeformThreads) deform_bproj_kernel(VolDims dims, PolyLattice lat, int Bf, const float* __restrict__ src,
                                                                      const float* __restrict__ tgt, const float* __restrict__ raylen,
                                                                      const float* __restrict__ gout, float* g_vol, int64_t N, int W,
                                                                      float shift, float eps, int P, const float* __restrict__ alpha_range)
{
    const int b = blockIdx.y;
    const int64_t n = tiled_ray_index(N, W);
    if (n < 0) return;
    const int64_t r = (int64_t)b * N + n;
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    const float c = __ldg(gout + r) * __ldg(raylen + r) * step;
    if (c == 0.0f) return;  // every add would be a zero
    if (Bf != 1) lat.w += (int64_t)b * lat.g[0] * lat.g[1] * lat.g[2];
    const Ray ray = load_ray(src, tgt, b, r, eps);
    deform_ray_bproj(dims, lat, ray, shift, P, amin, amax, c, g_vol);
}

int64_t deform_scratch_floats(int B, int64_t N, int W)
{
    const dim3 grid = tiled_ray_grid(B, N, W);
    return (int64_t)grid.x * grid.y * kDeformRow;
}

namespace {

struct DeformCall {
    VolDims dims;
    const float *src, *tgt, *raylen, *field;
    int Bf, g0, g1, g2, B;
    int64_t N;
    int W;
    float shift, eps;
    int P;
    const float* alpha_range;
    cudaStream_t stream;
};

template <class Gather>
cudaError_t run_fwd(const Gather& gather, const DeformCall& c, float* out)
{
    const PolyLattice lat = make_lattice(c.field, c.g0, c.g1, c.g2, c.dims);
    deform_fwd_kernel<Gather><<<tiled_ray_grid(c.B, c.N, c.W), kDeformThreads, 0, c.stream>>>(
        gather, c.dims, lat, c.Bf, c.src, c.tgt, c.raylen, out, c.N, c.W, c.shift, c.eps, c.P, c.alpha_range);
    return cudaGetLastError();
}

template <class Gather>
cudaError_t run_jvp(const Gather& gather, const DeformCall& c, const float* tangent, float* img, float* jv)
{
    const PolyLattice lat = make_lattice(c.field, c.g0, c.g1, c.g2, c.dims);
    const PolyLattice tan = make_lattice(tangent, c.g0, c.g1, c.g2, c.dims);
    deform_jvp_kernel<Gather><<<tiled_ray_grid(c.B, c.N, c.W), kDeformThreads, 0, c.stream>>>(
        gather, c.dims, lat, tan, c.Bf, c.src, c.tgt, c.raylen, img, jv, c.N, c.W, c.shift, c.eps, c.P, c.alpha_range);
    return cudaGetLastError();
}

template <int KP, class Gather>
cudaError_t run_jac(const Gather& gather, const DeformCall& c, const float* tangents, int K, float* img, float* J, int* rects, int H)
{
    const PolyLattice lat = make_lattice(c.field, c.g0, c.g1, c.g2, c.dims);
    const int n = c.B * K;
    polyrigid_rects_empty_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(rects, n, H, c.W);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    deform_jac_kernel<KP, Gather><<<tiled_ray_grid(c.B, c.N, c.W), kDeformThreads, 0, c.stream>>>(
        gather, c.dims, lat, (const float4*)tangents, K, c.Bf, c.src, c.tgt, c.raylen, img, J, rects, H, c.W, c.shift, c.eps, c.P,
        c.alpha_range);
    return cudaGetLastError();
}

template <class Gather>
cudaError_t run_bwd(const Gather& gather, const DeformCall& c, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                    float* g_field, float* g_alpha_range, float* scratch)
{
    const PolyLattice lat = make_lattice(c.field, c.g0, c.g1, c.g2, c.dims);
    const dim3 grid = tiled_ray_grid(c.B, c.N, c.W);
    if (g_field) {
        const size_t bytes = sizeof(float) * 4 * (size_t)c.Bf * c.g0 * c.g1 * c.g2;
        const cudaError_t e = cudaMemsetAsync(g_field, 0, bytes, c.stream);
        if (e != cudaSuccess) return e;
    }
    deform_bwd_kernel<Gather><<<grid, kDeformThreads, 0, c.stream>>>(gather, c.dims, lat, c.Bf, c.src, c.tgt, c.raylen, gout, g_tgt,
                                                                     g_raylen, g_field, scratch, c.N, c.W, c.shift, c.eps, c.P,
                                                                     c.alpha_range);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // the finish of the blended-rigid backward with no maps: its columns are then g_src [3] and g_alpha_range [2]
    polyrigid_finish_kernel<<<(unsigned)(3 * c.B + 2), 256, 0, c.stream>>>(scratch, kDeformRow, 0, c.B, (int)grid.x, 1, 0, nullptr,
                                                                         g_src, g_alpha_range);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_deform_fwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, float* out, int B, int64_t N,
                              int W, float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream)
{
    const DeformCall c{dims, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) { return run_fwd(gather, c, out); });
}

cudaError_t launch_deform_bwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* gout, float* g_src,
                              float* g_tgt, float* g_raylen, float* g_field, float* g_alpha_range, float* scratch, int B, int64_t N,
                              int W, float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream)
{
    const DeformCall c{dims, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) {
        return run_bwd(gather, c, gout, g_src, g_tgt, g_raylen, g_field, g_alpha_range, scratch);
    });
}

cudaError_t launch_deform_jvp(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangent, float* img,
                              float* jv, int B, int64_t N, int W, float shift, float eps, int n_points, const float* alpha_range,
                              cudaStream_t stream)
{
    const DeformCall c{dims, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) { return run_jvp(gather, c, tangent, img, jv); });
}

cudaError_t launch_deform_jac(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangents, int K,
                              float* img, float* J, int* rects, int B, int H, int W, float shift, float eps, int n_points,
                              const float* alpha_range, cudaStream_t stream)
{
    const DeformCall c{dims, src, tgt, raylen, field, Bf, g0, g1, g2, B, (int64_t)H * W, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) {
        return K <= 4 ? run_jac<4>(gather, c, tangents, K, img, J, rects, H) : run_jac<8>(gather, c, tangents, K, img, J, rects, H);
    });
}

cudaError_t launch_deform_bproj(VolDims dims, const float* src, const float* tgt, const float* raylen, const float* field, int Bf, int g0,
                                int g1, int g2, const float* gout, float* g_vol, int B, int64_t N, int W, float shift, float eps,
                                int n_points, const float* alpha_range, cudaStream_t stream)
{
    const size_t bytes = sizeof(float) * (size_t)dims.d[0] * dims.d[1] * dims.d[2];
    const cudaError_t e = cudaMemsetAsync(g_vol, 0, bytes, stream);
    if (e != cudaSuccess) return e;
    const PolyLattice lat = make_lattice(field, g0, g1, g2, dims);
    deform_bproj_kernel<<<tiled_ray_grid(B, N, W), kDeformThreads, 0, stream>>>(dims, lat, Bf, src, tgt, raylen, gout, g_vol, N, W, shift,
                                                                                eps, n_points, alpha_range);
    return cudaGetLastError();
}

}  // namespace b200drr
