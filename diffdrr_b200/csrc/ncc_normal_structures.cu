// ncc_normal_structures.cu -- global-NCC normal equations A [B][6K][6K], g [B][6K] of a piecewise-rigid composite image, summed
// block by block over the structures' detector footprints (sm_90a; math in ncc_normal_structures_math.cuh, DESIGN.md 6g).
//
//   footprints  structure_footprints_kernel  a thread per (pose, slot): the rectangle the structures render culls to
//   sums        ns_sum_kernel                per (band, task, pose): a task is a pair of structures j <= k (S J_j J_k^T over
//                                            the intersection of their footprints, and for j == k the moments S {1, x, t} J_k)
//                                            or the scalar moments over the whole image; a pair that does not overlap writes
//                                            zeros and reads no pixel
//           ns_moments_kernel            one CTA per pose: band sums of the moments in ne_window's layout, then ne_window
//           ns_fill_kernel               per (entry tile, pose): A += weight (S J J^T / s^2 - a a^T - b b^T), g += weight g_w
// Every sum is a per-thread loop in a fixed order followed by fixed-order sums over the bands (no atomics): repeated calls give
// identical bits.  The workspace holds per-(task, band) partials of 54 doubles and one moment vector per pose: nothing of size
// pixels x P^2 or pairs x pixels.
#include "kernels.h"
#include "ncc_normal_structures_math.cuh"

namespace b200drr {

namespace {

constexpr int kNsThreads = 256;
constexpr int kNsStage = 256;  // pixels staged per step of ns_sum_kernel

struct NsShape {
    int P, pairs, tasks, chunks, moments;
    int64_t part_off, T_off, rs2_off, total;  // in doubles
};

NsShape ns_shape(int B, int K, int H)
{
    NsShape s;
    s.P = kNsDof * K;
    s.pairs = ns_pairs(K);
    s.tasks = s.pairs + 1;
    s.chunks = ns_chunks(B, K, H);
    s.moments = ne_channels(s.P);
    s.part_off = 0;                                                                 // [B][tasks][chunks][kNsEntries]
    s.T_off = s.part_off + (int64_t)B * s.tasks * s.chunks * kNsEntries;            // [B][5 + 3P]
    s.rs2_off = s.T_off + (int64_t)B * s.moments;                                   // [B]
    s.total = s.rs2_off + B;
    return s;
}

__global__ void __launch_bounds__(128) structure_footprints_kernel(const float* __restrict__ src, const float* __restrict__ G,
                                                                   const float* __restrict__ rows, const float* __restrict__ cols,
                                                                   const int* __restrict__ box, int* __restrict__ rects, int BS,
                                                                   int S, int H, int W, float shift)
{
    const int bs = blockIdx.x * 128 + threadIdx.x;
    if (bs >= BS) return;
    int box_s[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) box_s[a] = __ldg(box + (bs % S) * 6 + a);
    int r[4];
    structure_footprint(G + (int64_t)bs * 12, src + (int64_t)bs * 3, box_s, shift, rows, cols, H, W, r);
    reinterpret_cast<int4*>(rects)[bs] = make_int4(r[0], r[1], r[2], r[3]);
}

// grid (chunks, tasks, B), static shared kNsRows x kNsStage doubles
__global__ void __launch_bounds__(kNsThreads) ns_sum_kernel(const float* __restrict__ x, const float* __restrict__ t, int64_t st,
                                                            const float* __restrict__ J, int64_t sb, int64_t ss, int64_t sn, int64_t sk,
                                                            const int* __restrict__ rects, int K, int S, int H, int W,
                                                            double* __restrict__ part)
{
    __shared__ double stage[kNsRows * kNsStage];
    const int c = blockIdx.x, task = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
    const int pairs = ns_pairs(K);
    const bool scalar = task == pairs;
    int j = 0, k = 0, rect[4] = {0, W - 1, 0, H - 1};
    bool any = true;
    if (!scalar) {
        ne_tri_index(task, K, j, k);
        int rj[4], rk[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            rj[a] = __ldg(rects + ((int64_t)b * S + j) * 4 + a);
            rk[a] = __ldg(rects + ((int64_t)b * S + k) * 4 + a);
        }
        any = ns_overlap(rj, rk, rect);
    }
    double* out = part + (((int64_t)b * gridDim.y + task) * gridDim.x + c) * kNsEntries;
    int ra, rb;
    const bool active = tid < kNsEntries && ns_entry_rows(tid, scalar, j == k, ra, rb) && any;
    double acc = 0.0;
    if (any) {
        int r0, r1;
        ns_band(rect[2], rect[3], c, gridDim.x, r0, r1);
        const int w = rect[1] - rect[0] + 1;
        const int64_t n = (int64_t)(r1 - r0) * w, HW = (int64_t)H * W;
        const float* xb = x + b * HW;
        const float* tb = t + b * st;
        const float* Jj = J + b * sb + j * ss;
        const float* Jk = J + b * sb + k * ss;
        for (int64_t i0 = 0; i0 < n; i0 += kNsStage) {
            const int nq = n - i0 < kNsStage ? (int)(n - i0) : kNsStage;
            for (int e = tid; e < (scalar ? 3 : kNsRows) * kNsStage; e += kNsThreads) {
                const int r = e / kNsStage, qq = e - r * kNsStage;
                if (qq >= nq) continue;
                const int64_t i = i0 + qq, q = (int64_t)(r0 + i / w) * W + rect[0] + i % w;
                stage[e] = r == 0 ? 1.0 : r == 1 ? (double)__ldg(xb + q) : r == 2 ? (double)__ldg(tb + q)
                                                                     : ns_row(r, 0.0f, 0.0f, Jj + q * sn, Jk + q * sn, sk);
            }
            __syncthreads();
            if (active) {
                const double* a = stage + ra * kNsStage;
                const double* bb = stage + rb * kNsStage;
                for (int qq = 0; qq < nq; ++qq) acc += a[qq] * bb[qq];
            }
            __syncthreads();
        }
    }
    if (tid < kNsEntries) out[tid] = active ? acc : 0.0;
}

// grid (B): the moment vector of each pose from the band sums, then ne_window in place (a, b, g_w; 1/s^2 -> rs2[b])
__global__ void __launch_bounds__(kNsThreads) ns_moments_kernel(const double* __restrict__ part, int K, int chunks, int64_t HW,
                                                                double eps, double* __restrict__ T, double* __restrict__ rs2)
{
    const int b = blockIdx.x, P = kNsDof * K, tasks = ns_pairs(K) + 1, M = ne_channels(P);
    double* Tb = T + (int64_t)b * M;
    const double* pb = part + (int64_t)b * tasks * chunks * kNsEntries;
    auto sum = [&](int task, int e) {
        const double* q = pb + (int64_t)task * chunks * kNsEntries + e;
        double s = 0.0;
        for (int c = 0; c < chunks; ++c) s += q[(int64_t)c * kNsEntries];
        return s;
    };
    for (int e = threadIdx.x; e < M; e += kNsThreads) Tb[e] = ns_moment(e, K, sum);
    __syncthreads();
    if (threadIdx.x == 0) rs2[b] = ne_window(Tb, 1, P, (double)HW, eps);
}

// grid (entry tiles over P^2 + P, B)
__global__ void __launch_bounds__(kNsThreads) ns_fill_kernel(const double* __restrict__ part, const double* __restrict__ T,
                                                             const double* __restrict__ rs2, int K, int chunks, double weight,
                                                             double* __restrict__ A, double* __restrict__ g)
{
    const int b = blockIdx.y, P = kNsDof * K, tasks = ns_pairs(K) + 1;
    const int64_t e = (int64_t)blockIdx.x * kNsThreads + threadIdx.x, PP = (int64_t)P * P;
    if (e >= PP + P) return;
    const double* Tb = T + (int64_t)b * ne_channels(P);
    if (e >= PP) {
        g[(int64_t)b * P + (e - PP)] += weight * Tb[5 + 2 * P + (e - PP)];
        return;
    }
    const double* pb = part + (int64_t)b * tasks * chunks * kNsEntries;
    auto sum = [&](int task, int en) {
        const double* q = pb + (int64_t)task * chunks * kNsEntries + en;
        double s = 0.0;
        for (int c = 0; c < chunks; ++c) s += q[(int64_t)c * kNsEntries];
        return s;
    };
    const int i = (int)(e / P), l = (int)(e - (int64_t)i * P);
    A[(int64_t)b * PP + e] += weight * (rs2[b] * ns_jj(i, l, K, sum) - ne_ab(Tb, 1, P, i, l));
}

}  // namespace

cudaError_t launch_structure_footprints(const float* src, const float* G, const float* rows, const float* cols, const int32_t* box,
                                        int32_t* rects, int B, int S, int H, int W, float shift, cudaStream_t stream)
{
    const int BS = B * S;
    structure_footprints_kernel<<<(unsigned)((BS + 127) / 128), 128, 0, stream>>>(src, G, rows, cols, box, rects, BS, S, H, W, shift);
    return cudaGetLastError();
}

int64_t ncc_normal_structures_workspace_bytes(int B, int K, int H)
{
    return ns_shape(B, K, H).total * (int64_t)sizeof(double);
}

cudaError_t launch_ncc_normal_structures(const float* x, const float* t, int t_batch, const float* J, int64_t sb, int64_t ss,
                                         int64_t sn, int64_t sk, const int32_t* rects, int B, int K, int S, int H, int W, double eps,
                                         double weight, void* workspace, double* A, double* g, cudaStream_t stream)
{
    if (K < 1 || K > kNsMaxK || S < K || B < 1 || B > 65535) return cudaErrorInvalidValue;
    const NsShape s = ns_shape(B, K, H);
    double* ws = (double*)workspace;
    const int64_t HW = (int64_t)H * W, st = t_batch == 1 ? 0 : HW;
    ns_sum_kernel<<<dim3((unsigned)s.chunks, (unsigned)s.tasks, (unsigned)B), kNsThreads, 0, stream>>>(
        x, t, st, J, sb, ss, sn, sk, rects, K, S, H, W, ws + s.part_off);
    cudaError_t e;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ns_moments_kernel<<<(unsigned)B, kNsThreads, 0, stream>>>(ws + s.part_off, K, s.chunks, HW, eps, ws + s.T_off, ws + s.rs2_off);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int64_t entries = (int64_t)s.P * s.P + s.P;
    ns_fill_kernel<<<dim3((unsigned)((entries + kNsThreads - 1) / kNsThreads), (unsigned)B), kNsThreads, 0, stream>>>(
        ws + s.part_off, ws + s.T_off, ws + s.rs2_off, K, s.chunks, weight, A, g);
    return cudaGetLastError();
}

}  // namespace b200drr
