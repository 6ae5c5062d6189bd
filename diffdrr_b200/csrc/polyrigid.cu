// polyrigid.cu -- blended-rigid (skinned) trilinear DRR kernels for sm_90a (forward + backward; math in polyrigid_math.cuh).
// One thread marches one ray; blockIdx.y is the pose, blockIdx.x a 16 x 8 pixel tile of a full detector grid (W > 0) or 128
// consecutive rays of any ray set (W == 0), as tiled_ray_index lays them out.  The pose's K affine maps sit in shared memory.
// Every output is written by exactly one thread and no atomics are used: the backward kernel writes one row of partial sums per
// CTA and polyrigid_finish_kernel adds the rows in a fixed order, so repeated calls give identical bits.
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

// f(gather) with the gather policy of the volume the caller gave: the packed-corner copy when there is one, the plain volume
// otherwise; vol_type 0 = fp32, B200DRR_VOL_F16, B200DRR_VOL_BF16
template <class F>
cudaError_t with_gather(const void* vol, const void* packed, int vol_type, F&& f)
{
    switch (vol_type) {
    case 0: return packed ? f(GatherPacked{(const float4*)packed}) : f(GatherPlainT<float>{(const float*)vol});
    case 1:
        return packed ? f(GatherPacked16<VoxF16>{(const Cell16<VoxF16>*)packed}) : f(GatherPlainT<VoxF16>{(const VoxF16*)vol});
    case 2:
        return packed ? f(GatherPacked16<VoxBF16>{(const Cell16<VoxBF16>*)packed}) : f(GatherPlainT<VoxBF16>{(const VoxBF16*)vol});
    }
    return cudaErrorInvalidValue;
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

}  // namespace b200drr
