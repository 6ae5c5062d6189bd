// polyrigid.cu -- blended-rigid (skinned) trilinear DRR kernels for sm_90a (forward, backward and per-pixel motion Jacobian; math
// in polyrigid_math.cuh).  One thread marches one ray; blockIdx.y is the pose, blockIdx.x a 16 x 8 pixel tile of a full detector
// grid (W > 0) or 128 consecutive rays of any ray set (W == 0), as tiled_ray_index lays them out.  The pose's K affine maps sit in
// shared memory.  The forward and backward write every output from exactly one thread and use no atomics: the backward kernel
// writes one row of partial sums per CTA and polyrigid_finish_kernel adds the rows in a fixed order, so repeated calls give
// identical bits.  The Jacobian's footprints use integer min / max atomics, which do not depend on order.  The backprojection kernel
// (the forward's transpose in the density) reads the maps from global memory, with no shared memory, and scatters into one volume
// gradient with scalar reductions, shared and per-pose maps alike: it repeats to fp32 reordering.
#include <climits>

#include "kernels.h"
#include "polyrigid_math.cuh"

namespace b200drr {

constexpr int kPolyThreads = 128;
constexpr int kPolyWarps = kPolyThreads / 32;

// partial sums one backward CTA writes: g_M [KP][12], g_src [3], g_alpha_range [2]
template <int KP>
constexpr int kPolyRow = KP * 12 + 5;

template <int KP>
__device__ __forceinline__ void load_maps(float* sM, const float* __restrict__ M, int Bm, int K, int b)
{
    const float* Mb = M + (Bm == 1 ? 0 : (int64_t)b * K * 12);
    for (int i = threadIdx.x; i < KP * 12; i += blockDim.x) sM[i] = i < K * 12 ? __ldg(Mb + i) : 0.0f;
    __syncthreads();
}

template <int KP, class Gather>
__global__ void __launch_bounds__(kPolyThreads, 6) polyrigid_fwd_kernel(Gather gather, VolDims dims, PolyLattice lat,
                                                                     const float* __restrict__ M, int Bm, int K,
                                                                     const float* __restrict__ src, const float* __restrict__ tgt,
                                                                     const float* __restrict__ raylen, float* __restrict__ out,
                                                                     int64_t N, int W, float shift, float eps, int P,
                                                                     const float* __restrict__ alpha_range)
{
    __shared__ float sM[KP * 12];
    const int b = blockIdx.y;
    load_maps<KP>(sM, M, Bm, K, b);
    const int64_t n = tiled_ray_index(N, W);
    if (n < 0) return;
    const int64_t r = (int64_t)b * N + n;
    const Ray ray = load_ray(src, tgt, b, r, eps);
    const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
    const float step = (amax - amin) / (float)(P - 1);
    out[r] = polyrigid_ray_fwd<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax) * (__ldg(raylen + r) * step);
}

// g_vol [D0][D1][D2] += the transpose of polyrigid_fwd_kernel in the density, for upstream gradient gout (polyrigid_ray_bproj)
template <int KP>
__global__ void __launch_bounds__(kPolyThreads) polyrigid_bproj_kernel(VolDims dims, PolyLattice lat, const float* __restrict__ M,
                                                                       int Bm, int K, const float* __restrict__ src,
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
    const float* Mb = M + (Bm == 1 ? 0 : (int64_t)b * K * 12);
    const Ray ray = load_ray(src, tgt, b, r, eps);
    polyrigid_ray_bproj<KP>(dims, lat, Mb, K, ray, shift, P, amin, amax, c, g_vol);
}

template <int KP, class Gather>
__global__ void __launch_bounds__(kPolyThreads) polyrigid_bwd_kernel(Gather gather, VolDims dims, PolyLattice lat,
                                                                     const float* __restrict__ M, int Bm, int K,
                                                                     const float* __restrict__ src, const float* __restrict__ tgt,
                                                                     const float* __restrict__ raylen, const float* __restrict__ gout,
                                                                     float* __restrict__ g_tgt, float* __restrict__ g_raylen,
                                                                     float* __restrict__ partial, int64_t N, int W, float shift,
                                                                     float eps, int P, const float* __restrict__ alpha_range)
{
    constexpr int ROW = kPolyRow<KP>;
    __shared__ float sM[KP * 12];
    __shared__ float red[kPolyWarps][ROW];
    const int b = blockIdx.y;
    load_maps<KP>(sM, M, Bm, K, b);
    const int64_t n = tiled_ray_index(N, W);
    float AG[KP][3], BG[KP][3], tail[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    Ray ray;
#pragma unroll
    for (int a = 0; a < 3; ++a) ray.s[a] = ray.d[a] = ray.inv[a] = 0.0f;
#pragma unroll
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) AG[k][a] = BG[k][a] = 0.0f;
    if (n >= 0) {
        const int64_t r = (int64_t)b * N + n;
        ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r), g = __ldg(gout + r);
        const TriGrad tg = polyrigid_ray_bwd<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax, g, L, AG, BG);
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
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int e = 0; e < 12; ++e) {
            const float v = warp_sum(poly_gM_entry(AG[k], BG[k], ray, e));
            if (lane == 0) red[warp][k * 12 + e] = v;
        }
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        const float v = warp_sum(tail[i]);
        if (lane == 0) red[warp][KP * 12 + i] = v;
    }
    __syncthreads();
    float* row = partial + ((int64_t)b * gridDim.x + blockIdx.x) * ROW;
    for (int i = threadIdx.x; i < ROW; i += blockDim.x) {
        float v = red[0][i];
#pragma unroll
        for (int w = 1; w < kPolyWarps; ++w) v += red[w][i];
        row[i] = v;
    }
}

// Per-pixel motion Jacobian (DESIGN.md 6j), full H x W grids only: img [B][H*W] (polyrigid_fwd_kernel's bits), J [B][K][H*W][6]
// with J[b][k][n][i] = poly_jac_entry of ray n against T [Bm][K][6][12] (the tangents dM_k / d xi_ki), and rects [B][K][4] int32
// {w0, w1, h0, h1}: the bounding rectangle of the pixels whose ray had an in-volume sample with w_k != 0, grown with one integer
// atomicMin / atomicMax per (CTA, k) (order-free, so every output repeats bit for bit; polyrigid_rects_empty_kernel runs first).
// Each warp's 8 x 4 pixel bundle (tiled_ray_index) stages its J rows of one k in shared memory, so that the stores are runs of
// 8 consecutive pixels (192 B) instead of 24 B per thread.
template <int KP, class Gather>
__global__ void __launch_bounds__(kPolyThreads) polyrigid_jac_kernel(Gather gather, VolDims dims, PolyLattice lat,
                                                                     const float* __restrict__ M, const float* __restrict__ T, int Bm,
                                                                     int K, const float* __restrict__ src, const float* __restrict__ tgt,
                                                                     const float* __restrict__ raylen, float* __restrict__ img,
                                                                     float* __restrict__ J, int* __restrict__ rects, int H, int W,
                                                                     float shift, float eps, int P, const float* __restrict__ alpha_range)
{
    __shared__ float sM[KP * 12];
    __shared__ float sT[KP * 72];
    __shared__ float2 stage[kPolyWarps][32 * 3];
    __shared__ int red[kPolyWarps][KP][4];
    const int b = blockIdx.y;
    const float* Tb = T + (Bm == 1 ? 0 : (int64_t)b * K * 72);
    for (int i = threadIdx.x; i < KP * 72; i += blockDim.x) sT[i] = i < K * 72 ? __ldg(Tb + i) : 0.0f;
    load_maps<KP>(sM, M, Bm, K, b);   // its __syncthreads covers sT too
    const int64_t N = (int64_t)H * W;
    const int64_t n = tiled_ray_index(N, W);
    float A[KP][3], Bv[KP][3];
    unsigned touched = 0u;
    float LS = 0.0f;
    Ray ray;
#pragma unroll
    for (int a = 0; a < 3; ++a) ray.s[a] = ray.d[a] = ray.inv[a] = 0.0f;
#pragma unroll
    for (int k = 0; k < KP; ++k)
#pragma unroll
        for (int a = 0; a < 3; ++a) A[k][a] = Bv[k][a] = 0.0f;
    if (n >= 0) {
        const int64_t r = (int64_t)b * N + n;
        ray = load_ray(src, tgt, b, r, eps);
        const float amin = __ldg(alpha_range), amax = __ldg(alpha_range + 1);
        const float step = (amax - amin) / (float)(P - 1);
        const float L = __ldg(raylen + r);
        img[r] = polyrigid_ray_jac<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax, A, Bv, touched) * (L * step);
        LS = L * step;
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
        for (int i = 0; i < 6; ++i) st[lane * 6 + i] = poly_jac_entry(A[k], Bv[k], ray, sT + (k * 6 + i) * 12, LS);
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
        for (int w = 1; w < kPolyWarps; ++w) {
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

// every rectangle empty: {W, -1, H, -1}
__global__ void __launch_bounds__(256) polyrigid_rects_empty_kernel(int* __restrict__ rects, int n, int H, int W)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) reinterpret_cast<int4*>(rects)[i] = make_int4(W, -1, H, -1);
}

// One CTA per output value: g_M [Bm][K][12], then g_src [B][3], then g_alpha_range [2].  Each adds its column of the partial rows
// (the rows of one pose, or of every pose for shared motions and the alpha range) strided over the threads, then block_sum: the
// order depends on the launch shape only.
__global__ void __launch_bounds__(256) polyrigid_finish_kernel(const float* __restrict__ partial, int row, int KP, int B, int T, int Bm,
                                                               int K, float* __restrict__ g_M, float* __restrict__ g_src,
                                                               float* __restrict__ g_alpha_range)
{
    __shared__ float red[32];
    const int nM = Bm * K * 12;
    int o = blockIdx.x, col, b0 = 0, b1 = B;
    float* dst;
    if (o < nM) {
        const int bm = o / (K * 12);
        col = o % (K * 12);
        if (Bm != 1) b0 = bm, b1 = bm + 1;
        dst = g_M ? g_M + o : nullptr;
    } else if (o < nM + 3 * B) {
        o -= nM;
        b0 = o / 3;
        b1 = b0 + 1;
        col = KP * 12 + o % 3;
        dst = g_src ? g_src + o : nullptr;
    } else {
        o -= nM + 3 * B;
        col = KP * 12 + 3 + o;
        dst = g_alpha_range ? g_alpha_range + o : nullptr;
    }
    if (!dst) return;
    float v = 0.0f;
    for (int64_t i = (int64_t)b0 * T + threadIdx.x; i < (int64_t)b1 * T; i += blockDim.x) v += __ldg(partial + i * row + col);
    v = block_sum(v, red);
    if (threadIdx.x == 0) *dst = v;
}

__global__ void __launch_bounds__(256) polyrigid_pack_weights_kernel(const float* __restrict__ weights, int K, int KP, int64_t nodes,
                                                                     float* __restrict__ packed)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nodes * KP) return;
    const int64_t node = i / KP;
    const int k = (int)(i % KP);
    packed[i] = k < K ? __ldg(weights + (int64_t)k * nodes + node) : 0.0f;
}

int polyrigid_channels(int K) { return K <= 4 ? 4 : 8; }

cudaError_t launch_polyrigid_pack_weights(const float* weights, int K, int g0, int g1, int g2, float* packed, cudaStream_t stream)
{
    const int KP = polyrigid_channels(K);
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    polyrigid_pack_weights_kernel<<<(unsigned)((nodes * KP + 255) / 256), 256, 0, stream>>>(weights, K, KP, nodes, packed);
    return cudaGetLastError();
}

int64_t polyrigid_scratch_floats(int B, int64_t N, int W, int K)
{
    const dim3 grid = tiled_ray_grid(B, N, W);
    return (int64_t)grid.x * grid.y * (polyrigid_channels(K) * 12 + 5);
}

namespace {

struct PolyCall {
    VolDims dims;
    const float *src, *tgt, *raylen, *M;
    int Bm, K;
    const float* weights;
    int g0, g1, g2, B;
    int64_t N;
    int W;
    float shift, eps;
    int P;
    const float* alpha_range;
    cudaStream_t stream;
};

template <int KP, class Gather>
cudaError_t run_fwd(const Gather& gather, const PolyCall& c, float* out)
{
    const PolyLattice lat = make_lattice(c.weights, c.g0, c.g1, c.g2, c.dims);
    polyrigid_fwd_kernel<KP, Gather><<<tiled_ray_grid(c.B, c.N, c.W), kPolyThreads, 0, c.stream>>>(
        gather, c.dims, lat, c.M, c.Bm, c.K, c.src, c.tgt, c.raylen, out, c.N, c.W, c.shift, c.eps, c.P, c.alpha_range);
    return cudaGetLastError();
}

template <int KP, class Gather>
cudaError_t run_bwd(const Gather& gather, const PolyCall& c, const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_M,
                    float* g_alpha_range, float* scratch)
{
    const PolyLattice lat = make_lattice(c.weights, c.g0, c.g1, c.g2, c.dims);
    const dim3 grid = tiled_ray_grid(c.B, c.N, c.W);
    polyrigid_bwd_kernel<KP, Gather><<<grid, kPolyThreads, 0, c.stream>>>(gather, c.dims, lat, c.M, c.Bm, c.K, c.src, c.tgt, c.raylen,
                                                                        gout, g_tgt, g_raylen, scratch, c.N, c.W, c.shift, c.eps,
                                                                        c.P, c.alpha_range);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const unsigned outputs = (unsigned)(c.Bm * c.K * 12 + 3 * c.B + 2);
    polyrigid_finish_kernel<<<outputs, 256, 0, c.stream>>>(scratch, kPolyRow<KP>, KP, c.B, (int)grid.x, c.Bm, c.K, g_M, g_src,
                                                          g_alpha_range);
    return cudaGetLastError();
}

template <int KP, class Gather>
cudaError_t run_jac(const Gather& gather, const PolyCall& c, const float* T, float* img, float* J, int* rects, int H)
{
    const PolyLattice lat = make_lattice(c.weights, c.g0, c.g1, c.g2, c.dims);
    const int n = c.B * c.K;
    polyrigid_rects_empty_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(rects, n, H, c.W);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    polyrigid_jac_kernel<KP, Gather><<<tiled_ray_grid(c.B, c.N, c.W), kPolyThreads, 0, c.stream>>>(
        gather, c.dims, lat, c.M, T, c.Bm, c.K, c.src, c.tgt, c.raylen, img, J, rects, H, c.W, c.shift, c.eps, c.P, c.alpha_range);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_polyrigid_fwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 float* out, int B, int64_t N, int W, float shift, float eps, int n_points, const float* alpha_range,
                                 cudaStream_t stream)
{
    const PolyCall c{dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, N, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) {
        return K <= 4 ? run_fwd<4>(gather, c, out) : run_fwd<8>(gather, c, out);
    });
}

cudaError_t launch_polyrigid_bwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_M, float* g_alpha_range,
                                 float* scratch, int B, int64_t N, int W, float shift, float eps, int n_points,
                                 const float* alpha_range, cudaStream_t stream)
{
    const PolyCall c{dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, N, W, shift, eps, n_points, alpha_range, stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) {
        return K <= 4 ? run_bwd<4>(gather, c, gout, g_src, g_tgt, g_raylen, g_M, g_alpha_range, scratch)
                      : run_bwd<8>(gather, c, gout, g_src, g_tgt, g_raylen, g_M, g_alpha_range, scratch);
    });
}

cudaError_t launch_polyrigid_jac(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 const float* T, float* img, float* J, int* rects, int B, int H, int W, float shift, float eps,
                                 int n_points, const float* alpha_range, cudaStream_t stream)
{
    const PolyCall c{dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, (int64_t)H * W, W, shift, eps, n_points, alpha_range,
                     stream};
    return with_gather(vol, packed, vol_type, [&](auto gather) {
        return K <= 4 ? run_jac<4>(gather, c, T, img, J, rects, H) : run_jac<8>(gather, c, T, img, J, rects, H);
    });
}

cudaError_t launch_polyrigid_bproj(VolDims dims, const float* src, const float* tgt, const float* raylen, const float* M, int Bm, int K,
                                   const float* weights, int g0, int g1, int g2, const float* gout, float* g_vol, int B, int64_t N, int W,
                                   float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream)
{
    const size_t bytes = sizeof(float) * (size_t)dims.d[0] * dims.d[1] * dims.d[2];
    const cudaError_t e = cudaMemsetAsync(g_vol, 0, bytes, stream);
    if (e != cudaSuccess) return e;
    const PolyLattice lat = make_lattice(weights, g0, g1, g2, dims);
    const dim3 grid = tiled_ray_grid(B, N, W);
    if (K <= 4)
        polyrigid_bproj_kernel<4><<<grid, kPolyThreads, 0, stream>>>(dims, lat, M, Bm, K, src, tgt, raylen, gout, g_vol, N, W, shift, eps,
                                                                     n_points, alpha_range);
    else
        polyrigid_bproj_kernel<8><<<grid, kPolyThreads, 0, stream>>>(dims, lat, M, Bm, K, src, tgt, raylen, gout, g_vol, N, W, shift, eps,
                                                                     n_points, alpha_range);
    return cudaGetLastError();
}

}  // namespace b200drr
