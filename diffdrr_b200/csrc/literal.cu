// literal.cu -- reference-literal Siddon / trilinear renderers for sm_90a, templated on the real type.
//
// Two uses, both off the fast paths:
//   * fp64: the reference reaches double precision through `drr.to(torch.float64)` (drr.py:75 comment, utils.py:110);
//   * callable `reducefn` (renderers.py:175-183: `reducefn(img)` on the (B, N, M-1) per-segment / (B, N, P) per-sample tensor):
//     the kernels can write that tensor instead of reducing it, and their backward takes a per-segment upstream gradient.
// One thread per ray, no tiling (accuracy / generality paths), same closed-form backward as the tuned kernels (SURVEY.md 8a-G):
//   Siddon    renderers.py:34-76 + 94-113 + 143-169: every plane alpha of the three axes, merged ascending, midpoint ->
//             nearest voxel (half-to-even, zero padding), L * v * (alpha_{j+1} - alpha_j), sum or max (or the segments);
//   Trilinear renderers.py:205-240: alpha_m = linspace(0,1,P)[m] * (amax - amin) + amin (the linspace is built in fp32 by
//             the reference even in the fp64 run, renderers.py:224), 8-corner interpolation with per-corner zero padding,
//             L * value * step, sum or max (or the samples).
#include <math.h>

#include "kernels.h"

namespace b200drr {

namespace {

template <typename R>
struct RayL {
    R s[3], d[3];
};

template <typename R>
__device__ __forceinline__ RayL<R> load_ray_l(const R* src, const R* tgt, int b, int64_t r, R eps)
{
    RayL<R> ray;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray.s[a] = src[b * 3 + a];
        ray.d[a] = (tgt[r * 3 + a] - ray.s[a]) + eps;  // renderers.py:104-106: eps is added to the direction
    }
    return ray;
}

__device__ __forceinline__ double rint_he(double x) { return nearbyint(x); }
__device__ __forceinline__ float rint_he(float x) { return nearbyintf(x); }
__device__ __forceinline__ double floor_r(double x) { return floor(x); }
__device__ __forceinline__ float floor_r(float x) { return floorf(x); }

// continuous voxel coordinate grid_sample sees for the point s + alpha * d (renderers.py:148-152 + ATen un-normalisation)
template <typename R>
__device__ __forceinline__ R pix_at(R alpha, R s, R d, R shift, int D, int align_corners)
{
    const R g = R(2) * ((s + alpha * d) + shift) / (R)D - R(1);
    return align_corners ? (g + R(1)) * R(0.5) * (R)(D - 1) : ((g + R(1)) * (R)D - R(1)) * R(0.5);
}

// ascending merge of the three per-axis plane sequences alpha_a(i) = ((i - shift) - s_a) / d_a, i = 0..D_a
template <typename R>
struct PlaneMerge {
    R cur[3];
    int i[3], step[3], left[3];
    R shift;
    __device__ void init(const RayL<R>& ray, const VolDims& dims, R sh)
    {
        shift = sh;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const bool up = ray.d[a] > R(0);
            i[a] = up ? 0 : dims.d[a];
            step[a] = up ? 1 : -1;
            left[a] = dims.d[a] + 1;
            cur[a] = (((R)i[a] - shift) - ray.s[a]) / ray.d[a];
        }
    }
    __device__ bool pop(const RayL<R>& ray, R& alpha, int& axis)
    {
        axis = -1;
        R best = R(0);
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (left[a] > 0 && (axis < 0 || cur[a] < best)) {
                best = cur[a];
                axis = a;
            }
        if (axis < 0) return false;
        alpha = best;
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (a == axis) {
                i[a] += step[a];
                --left[a];
                cur[a] = (((R)i[a] - shift) - ray.s[a]) / ray.d[a];
            }
        return true;
    }
};

template <typename R>
__device__ __forceinline__ int64_t nearest_voxel(const RayL<R>& ray, const VolDims& dims, R mid, R shift, int align_corners)
{
    int64_t flat = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const R r = rint_he(pix_at<R>(mid, ray.s[a], ray.d[a], shift, dims.d[a], align_corners));  // half to even
        if (!(r >= R(0) && r < (R)dims.d[a])) return -1;                                            // zero padding
        flat = flat * dims.d[a] + (int64_t)r;
    }
    return flat;
}

// reduce: 0 = sum, 1 = max -> out [B][N];  2 = keep the segments -> out [B][N][D0+D1+D2+2] in the reference's sorted order
template <typename R>
__global__ void __launch_bounds__(128) siddon_fwd_l_kernel(const R* __restrict__ vol, VolDims dims, const R* __restrict__ src,
                                                           const R* __restrict__ tgt, const R* __restrict__ raylen,
                                                           R* __restrict__ out, int64_t N, R shift, R eps, int reduce,
                                                           int align_corners)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const RayL<R> ray = load_ray_l<R>(src, tgt, b, r, eps);
    const R L = raylen[r];
    const int64_t M1 = (int64_t)dims.d[0] + dims.d[1] + dims.d[2] + 2;
    PlaneMerge<R> pm;
    pm.init(ray, dims, shift);
    R prev, alpha, acc = R(0);
    int axis;
    int64_t j = 0;
    pm.pop(ray, prev, axis);
    while (pm.pop(ray, alpha, axis)) {
        const int64_t v = nearest_voxel<R>(ray, dims, R(0.5) * (prev + alpha), shift, align_corners);
        const R term = (L * (v >= 0 ? vol[v] : R(0))) * (alpha - prev);
        if (reduce == 2) out[r * M1 + j] = term;
        else if (reduce == 0) acc += term;
        else if (j == 0 || term > acc) acc = term;
        ++j;
        prev = alpha;
    }
    if (reduce != 2) out[r] = acc;
}

// closed form: dI/dalpha_m = L (g_{m-1} v_{m-1} - g_m v_m), dalpha/ds_a = (alpha - 1)/d_a, dalpha/dt_a = -alpha/d_a
// (SURVEY 8a-G).  gseg != nullptr: per-segment upstream gradient [B][N][M1] (callable reducefn); else gout [B][N].
template <typename R>
__global__ void __launch_bounds__(128) siddon_bwd_l_kernel(const R* __restrict__ vol, VolDims dims, const R* __restrict__ src,
                                                           const R* __restrict__ tgt, const R* __restrict__ raylen,
                                                           const R* __restrict__ gout, const R* __restrict__ gseg,
                                                           R* __restrict__ g_src, R* __restrict__ g_tgt, R* __restrict__ g_raylen,
                                                           R* __restrict__ g_vol, int64_t N, R shift, R eps, int stop_grad,
                                                           int align_corners)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const RayL<R> ray = load_ray_l<R>(src, tgt, b, r, eps);
    const R L = raylen[r];
    const int64_t M1 = (int64_t)dims.d[0] + dims.d[1] + dims.d[2] + 2;
    PlaneMerge<R> pm;
    pm.init(ray, dims, shift);
    R A[3] = {R(0), R(0), R(0)}, C[3] = {R(0), R(0), R(0)};
    R prev, alpha, wprev = R(0), acc = R(0);   // wprev = g_{j-1} v_{j-1}
    int axprev, axis;
    int64_t j = 0;
    pm.pop(ray, prev, axprev);
    while (pm.pop(ray, alpha, axis)) {
        const int64_t v = nearest_voxel<R>(ray, dims, R(0.5) * (prev + alpha), shift, align_corners);
        const R val = v >= 0 ? vol[v] : R(0);
        const R gj = gseg ? gseg[r * M1 + j] : gout[r];
        const R len = alpha - prev;
        acc += gj * val * len;
        if (g_vol && !stop_grad && v >= 0) atomicAdd(g_vol + v, gj * L * len);
        const R w = gj * val;
        const R coef = L * (wprev - w);  // the crossing at `prev` (axis axprev) separates segment j-1 from segment j
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (a == axprev) {
                A[a] += coef * prev;
                C[a] += coef;
            }
        wprev = w;
        prev = alpha;
        axprev = axis;
        ++j;
    }
    {  // the last plane: beyond it the volume is zero padding
        const R coef = L * wprev;
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (a == axprev) {
                A[a] += coef * prev;
                C[a] += coef;
            }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (g_tgt) g_tgt[r * 3 + a] = -A[a] / ray.d[a];
        if (g_src) atomicAdd(g_src + b * 3 + a, (A[a] - C[a]) / ray.d[a]);
    }
    if (g_raylen) g_raylen[r] = stop_grad ? R(0) : acc;
}

// ATen's fp32 linspace(0, 1, P)[m] (symmetric about the midpoint, the second half as end - step * k), then cast
__device__ __forceinline__ float linspace01_f32(int m, int P)
{
    const float step = 1.0f / (float)(P - 1);
    if (m < P / 2) return __fmul_rn(step, (float)m);
    return fmaf(-step, (float)(P - 1 - m), 1.0f);
}

// 8-corner interpolation with per-corner zero padding; optionally the analytic gradient w.r.t. pix and a volume scatter
template <typename R>
__device__ __forceinline__ R trilerp_l(const R* __restrict__ vol, const VolDims& dims, const R pix[3], R grad[3], R* g_vol, R g_scale)
{
    R f[3];
    int64_t i0[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const R fl = floor_r(pix[a]);
        i0[a] = (int64_t)fl;
        f[a] = pix[a] - fl;
    }
    R val = R(0);
    if (grad) grad[0] = grad[1] = grad[2] = R(0);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int o[3] = {c & 1, (c >> 1) & 1, (c >> 2) & 1};
        R w[3];
        int64_t id[3];
        bool inb = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            id[a] = i0[a] + o[a];
            w[a] = o[a] ? f[a] : R(1) - f[a];
            inb = inb && id[a] >= 0 && id[a] < dims.d[a];
        }
        if (!inb) continue;
        const int64_t flat = (id[0] * dims.d[1] + id[1]) * dims.d[2] + id[2];
        const R v = vol[flat];
        val += v * w[0] * w[1] * w[2];
        if (grad) {
            grad[0] += v * (o[0] ? R(1) : R(-1)) * w[1] * w[2];
            grad[1] += v * (o[1] ? R(1) : R(-1)) * w[0] * w[2];
            grad[2] += v * (o[2] ? R(1) : R(-1)) * w[0] * w[1];
        }
        if (g_vol) atomicAdd(g_vol + flat, g_scale * w[0] * w[1] * w[2]);
    }
    return val;
}

// reduce: 0 = sum, 1 = max -> out [B][N];  2 = keep the samples -> out [B][N][P]
template <typename R>
__global__ void __launch_bounds__(128) trilinear_fwd_l_kernel(const R* __restrict__ vol, VolDims dims, const R* __restrict__ src,
                                                              const R* __restrict__ tgt, const R* __restrict__ raylen,
                                                              R* __restrict__ out, int64_t N, R shift, R eps, int P,
                                                              const R* __restrict__ alpha_range, int reduce, int align_corners)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const RayL<R> ray = load_ray_l<R>(src, tgt, b, r, eps);
    const R L = raylen[r], amin = alpha_range[0], amax = alpha_range[1];
    const R step = (amax - amin) / (R)(P - 1);
    R acc = R(0);
    for (int m = 0; m < P; ++m) {
        const R alpha = (R)linspace01_f32(m, P) * (amax - amin) + amin;
        R pix[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = pix_at<R>(alpha, ray.s[a], ray.d[a], shift, dims.d[a], align_corners);
        const R term = (L * trilerp_l<R>(vol, dims, pix, nullptr, nullptr, R(0))) * step;
        if (reduce == 2) out[r * P + m] = term;
        else if (reduce == 0) acc += term;
        else if (m == 0 || term > acc) acc = term;
    }
    if (reduce != 2) out[r] = acc;
}

// gsmp != nullptr: per-sample upstream gradient [B][N][P] (callable reducefn); else gout [B][N]
template <typename R>
__global__ void __launch_bounds__(128) trilinear_bwd_l_kernel(const R* __restrict__ vol, VolDims dims, const R* __restrict__ src,
                                                              const R* __restrict__ tgt, const R* __restrict__ raylen,
                                                              const R* __restrict__ gout, const R* __restrict__ gsmp,
                                                              R* __restrict__ g_src, R* __restrict__ g_tgt, R* __restrict__ g_raylen,
                                                              R* __restrict__ g_vol, R* __restrict__ g_alpha_range, int64_t N,
                                                              R shift, R eps, int P, const R* __restrict__ alpha_range,
                                                              int align_corners)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int b = blockIdx.y;
    const int64_t r = (int64_t)b * N + n;
    const RayL<R> ray = load_ray_l<R>(src, tgt, b, r, eps);
    const R L = raylen[r], amin = alpha_range[0], amax = alpha_range[1];
    const R range = amax - amin, step = range / (R)(P - 1);
    R scale[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) scale[a] = align_corners ? (R)(dims.d[a] - 1) / (R)dims.d[a] : R(1);  // dpix/dx
    R gs[3] = {R(0), R(0), R(0)}, gt[3] = {R(0), R(0), R(0)}, sumv = R(0), d_amin = R(0), d_amax = R(0);
    for (int m = 0; m < P; ++m) {
        const R lin = (R)linspace01_f32(m, P), alpha = lin * range + amin;
        const R gm = gsmp ? gsmp[r * P + m] : gout[r];
        R pix[3], G[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) pix[a] = pix_at<R>(alpha, ray.s[a], ray.d[a], shift, dims.d[a], align_corners);
        sumv += gm * trilerp_l<R>(vol, dims, pix, G, g_vol, gm * L * step);
        R gd = R(0);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const R ga = gm * G[a] * scale[a];
            gs[a] += (R(1) - alpha) * ga;
            gt[a] += alpha * ga;
            gd += ga * ray.d[a];
        }
        d_amin += (R(1) - lin) * gd;
        d_amax += lin * gd;
    }
    const R k = L * step;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (g_tgt) g_tgt[r * 3 + a] = k * gt[a];
        if (g_src) atomicAdd(g_src + b * 3 + a, k * gs[a]);
    }
    if (g_raylen) g_raylen[r] = step * sumv;
    if (g_alpha_range) {
        atomicAdd(g_alpha_range + 0, L * (-sumv / (R)(P - 1) + step * d_amin));
        atomicAdd(g_alpha_range + 1, L * (sumv / (R)(P - 1) + step * d_amax));
    }
}

inline dim3 grid_l(int B, int64_t N) { return dim3((unsigned)((N + 127) / 128), (unsigned)B, 1); }

}  // namespace

template <typename R>
cudaError_t launch_siddon_fwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, R* out, int B,
                                      int64_t N, R shift, R eps, int reduce, int align_corners, cudaStream_t stream)
{
    siddon_fwd_l_kernel<R><<<grid_l(B, N), 128, 0, stream>>>(vol, dims, src, tgt, raylen, out, N, shift, eps, reduce, align_corners);
    return cudaGetLastError();
}

template <typename R>
cudaError_t launch_siddon_bwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, const R* gout,
                                      const R* gseg, R* g_src, R* g_tgt, R* g_raylen, R* g_vol, int B, int64_t N, R shift, R eps,
                                      int stop_grad, int align_corners, cudaStream_t stream)
{
    if (g_src) {
        cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(R) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    siddon_bwd_l_kernel<R><<<grid_l(B, N), 128, 0, stream>>>(vol, dims, src, tgt, raylen, gout, gseg, g_src, g_tgt, g_raylen, g_vol,
                                                            N, shift, eps, stop_grad, align_corners);
    return cudaGetLastError();
}

template <typename R>
cudaError_t launch_trilinear_fwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, R* out, int B,
                                         int64_t N, R shift, R eps, int n_points, const R* alpha_range, int reduce,
                                         int align_corners, cudaStream_t stream)
{
    trilinear_fwd_l_kernel<R><<<grid_l(B, N), 128, 0, stream>>>(vol, dims, src, tgt, raylen, out, N, shift, eps, n_points,
                                                               alpha_range, reduce, align_corners);
    return cudaGetLastError();
}

template <typename R>
cudaError_t launch_trilinear_bwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, const R* gout,
                                         const R* gsmp, R* g_src, R* g_tgt, R* g_raylen, R* g_vol, R* g_alpha_range, int B,
                                         int64_t N, R shift, R eps, int n_points, const R* alpha_range, int align_corners,
                                         cudaStream_t stream)
{
    if (g_src) {
        cudaError_t e = cudaMemsetAsync(g_src, 0, sizeof(R) * 3 * (size_t)B, stream);
        if (e != cudaSuccess) return e;
    }
    trilinear_bwd_l_kernel<R><<<grid_l(B, N), 128, 0, stream>>>(vol, dims, src, tgt, raylen, gout, gsmp, g_src, g_tgt, g_raylen,
                                                               g_vol, g_alpha_range, N, shift, eps, n_points, alpha_range,
                                                               align_corners);
    return cudaGetLastError();
}

#define B200_INSTANTIATE(R)                                                                                                          \
    template cudaError_t launch_siddon_fwd_literal<R>(const R*, VolDims, const R*, const R*, const R*, R*, int, int64_t, R, R, int,  \
                                                      int, cudaStream_t);                                                            \
    template cudaError_t launch_siddon_bwd_literal<R>(const R*, VolDims, const R*, const R*, const R*, const R*, const R*, R*, R*,   \
                                                      R*, R*, int, int64_t, R, R, int, int, cudaStream_t);                           \
    template cudaError_t launch_trilinear_fwd_literal<R>(const R*, VolDims, const R*, const R*, const R*, R*, int, int64_t, R, R,    \
                                                         int, const R*, int, int, cudaStream_t);                                     \
    template cudaError_t launch_trilinear_bwd_literal<R>(const R*, VolDims, const R*, const R*, const R*, const R*, const R*, R*,    \
                                                         R*, R*, R*, R*, int, int64_t, R, R, int, const R*, int, cudaStream_t);
B200_INSTANTIATE(float)
B200_INSTANTIATE(double)
#undef B200_INSTANTIATE

}  // namespace b200drr
