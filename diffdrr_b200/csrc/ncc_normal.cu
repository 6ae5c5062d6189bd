// ncc_normal.cu -- Gauss-Newton normal equations A [B][P][P], g [B][P] of the global and patch-wise NCC losses (sm_90a).
//
// The Levenberg-Marquardt step of registration.py models 1 - NCC as |r|^2 / 2N with the z-normalised residual of every window.
// The torch statement of that model needs the normalised Jacobian per (window, pixel): 480 MB per pose and channel at 256^2,
// p = 13, P = 6.  The math in ncc_normal_math.cuh reduces every window to box sums of 5 + 3P channels plus one adjoint box sum
// of a scalar map, and the launches are
//   patch   ne_window_kernel         per window row: vertical p-row sums of the K channels into the CTA's own row buffer, then
//                                    per 64-window tile the horizontal sums, the window terms (a, b, g_w, 1/s^2) and the
//                                    CTA's partial of -sum (a a^T + b b^T) and sum g_w
//           ne_beta_vertical_kernel  vertical adjoint sums of 1/s^2
//           ne_pixel_kernel          beta_q per pixel, then the CTA's partial of sum beta_q J_q J_q^T
//           ne_finalize_kernel       one CTA per pose: partials of every channel summed in a fixed order, A, g += weight * ...
//   global  ne_global_kernel         per (image, pixel chunk): the K channel sums and sum J J^T, spread over the SMs
//           ne_global_finalize_kernel  one CTA per pose: chunk sums, window terms per channel, A, g += weight * ...
// Every reduction is a per-thread loop in a fixed order followed by fixed-order sums of per-CTA partials (no atomics): repeated
// runs are bitwise identical.  The workspace holds no (window x pixel) or (pixel x P^2) array: the vertical sums live in one
// K x W row buffer per CTA, and the CTA count per image falls as the batch grows (ne_shape).
#include "kernels.h"
#include "ncc_normal_math.cuh"

namespace b200drr {

namespace {

constexpr int kNeThreads = 256;
constexpr int kNeTile = 64;      // windows per horizontal tile of ne_window_kernel
constexpr int kNeChunk = 256;    // pixels staged per step of ne_pixel_kernel / ne_global_kernel
constexpr int kNeCtaTarget = 512;  // CTAs one launch aims at: the per-image split shrinks as B * C grows

struct NeShape {
    int imgs, K, tri, Ep, Eg, Hp, Wp;
    int nbw, nbp;          // patch: window-row CTAs, pixel CTAs per image
    int chunks;            // global: pixel chunks per image
    int64_t chunk_pix;     // global: pixels per chunk (a multiple of kNeChunk)
    int64_t v_off, r_off, b_off, p_off, total;  // workspace layout, in doubles
};

int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

NeShape ne_shape(int B, int C, int H, int W, int p, int P)
{
    NeShape s;
    s.imgs = B * C;
    s.K = ne_channels(P);
    s.tri = ne_tri(P);
    s.Ep = s.tri + P;
    s.Eg = s.K + s.tri;
    const int per_img = kNeCtaTarget / s.imgs > 1 ? kNeCtaTarget / s.imgs : 1;
    const int64_t HW = (int64_t)H * W, pix_tiles = cdiv(HW, kNeChunk);
    s.nbp = (int)(pix_tiles < per_img ? pix_tiles : per_img);
    if (p == 0) {  // global
        s.Hp = s.Wp = 1;
        s.nbw = 0;
        s.chunk_pix = cdiv(pix_tiles, s.nbp) * kNeChunk;
        s.chunks = (int)cdiv(HW, s.chunk_pix);
        s.v_off = s.r_off = s.b_off = s.p_off = 0;
        s.total = (int64_t)s.imgs * s.chunks * s.Eg;
        return s;
    }
    s.Hp = H - p + 1;
    s.Wp = W - p + 1;
    s.nbw = s.Hp < per_img ? s.Hp : per_img;
    s.chunks = 0;
    s.chunk_pix = 0;
    s.v_off = 0;                                                       // V   [imgs][nbw][K][W]
    s.r_off = s.v_off + (int64_t)s.imgs * s.nbw * s.K * W;             // rs2 [imgs][H'][W']
    s.b_off = s.r_off + (int64_t)s.imgs * s.Hp * s.Wp;                 // VB  [imgs][H][W']
    s.p_off = s.b_off + (int64_t)s.imgs * H * s.Wp;                    // partials [imgs][nbw + nbp][Ep]
    s.total = s.p_off + (int64_t)s.imgs * (s.nbw + s.nbp) * s.Ep;
    return s;
}

}  // namespace

// grid (nbw, B*C), dynamic shared K x kNeTile doubles.  Window rows i = blockIdx.x, blockIdx.x + nbw, ...
__global__ void __launch_bounds__(kNeThreads) ne_window_kernel(const float* __restrict__ x, const float* __restrict__ t,
                                                               const float* __restrict__ J, int64_t sb, int64_t sc, int64_t sk,
                                                               int64_t sn, int C, int H, int W, int p, int P, double eps,
                                                               double* V, double* __restrict__ rs2, double* __restrict__ part,
                                                               int nbt)
{
    extern __shared__ double stage[];  // [K][kNeTile]
    const int img = blockIdx.y, b = img / C, c = img - b * C, tid = threadIdx.x;
    const int K = ne_channels(P), tri = ne_tri(P), Hp = H - p + 1, Wp = W - p + 1;
    const int64_t HW = (int64_t)H * W;
    const float* xi = x + img * HW;
    const float* ti = t + img * HW;
    const float* Ji = J + b * sb + c * sc;
    double* v = V + ((int64_t)img * gridDim.x + blockIdx.x) * K * W;  // this CTA's row buffer (written and read by it alone)
    double* r2 = rs2 + (int64_t)img * Hp * Wp;
    int ek = 0, el = 0;
    if (tid < tri) ne_tri_index(tid, P, ek, el);
    const double n = (double)p * (double)p;
    double acc = 0.0;
    for (int i = blockIdx.x; i < Hp; i += gridDim.x) {
        for (int e = tid; e < K * W; e += kNeThreads) {
            const int k = e / W, col = e - k * W;
            v[e] = ne_vertical(xi, ti, Ji, sk, sn, W, p, P, k, i, col);
        }
        __syncthreads();
        for (int j0 = 0; j0 < Wp; j0 += kNeTile) {
            const int nw = Wp - j0 < kNeTile ? Wp - j0 : kNeTile;
            for (int e = tid; e < K * kNeTile; e += kNeThreads) {
                const int k = e / kNeTile, jj = e - k * kNeTile;
                stage[e] = jj < nw ? ne_horizontal(v + (int64_t)k * W, p, j0 + jj) : 0.0;
            }
            __syncthreads();
            if (tid < nw) r2[(int64_t)i * Wp + j0 + tid] = ne_window(stage + tid, kNeTile, P, n, eps);
            __syncthreads();
            if (tid < tri) {
                for (int jj = 0; jj < nw; ++jj) acc -= ne_ab(stage + jj, kNeTile, P, ek, el);
            } else if (tid < tri + P) {
                const double* gw = stage + (5 + 2 * P + (tid - tri)) * kNeTile;
                for (int jj = 0; jj < nw; ++jj) acc += gw[jj];
            }
            __syncthreads();
        }
    }
    if (tid < tri + P) part[((int64_t)img * nbt + blockIdx.x) * (tri + P) + tid] = acc;
}

// grid (blocks over H x W', B*C)
__global__ void __launch_bounds__(kNeThreads) ne_beta_vertical_kernel(const double* __restrict__ rs2, int H, int W, int p,
                                                                      double* __restrict__ VB)
{
    const int64_t img = blockIdx.y, e = (int64_t)blockIdx.x * kNeThreads + threadIdx.x;
    const int Hp = H - p + 1, Wp = W - p + 1;
    if (e >= (int64_t)H * Wp) return;
    VB[img * H * Wp + e] = ne_beta_vertical(rs2 + img * Hp * Wp, H, W, p, (int)(e / Wp), (int)(e % Wp));
}

// grid (nbp, B*C), dynamic shared (1 + P) x kNeChunk doubles.  Pixel chunks blockIdx.x, blockIdx.x + nbp, ...
__global__ void __launch_bounds__(kNeThreads) ne_pixel_kernel(const float* __restrict__ J, int64_t sb, int64_t sc, int64_t sk,
                                                              int64_t sn, int C, int H, int W, int p, int P,
                                                              const double* __restrict__ VB, double* __restrict__ part, int nbw,
                                                              int nbt)
{
    extern __shared__ double stage[];  // [0]: beta, [1 + k]: J_k
    const int img = blockIdx.y, b = img / C, c = img - b * C, tid = threadIdx.x;
    const int tri = ne_tri(P), Wp = W - p + 1;
    const int64_t HW = (int64_t)H * W;
    const float* Ji = J + b * sb + c * sc;
    const double* vb = VB + (int64_t)img * H * Wp;
    int ek = 0, el = 0;
    if (tid < tri) ne_tri_index(tid, P, ek, el);
    double acc = 0.0;
    for (int64_t q0 = (int64_t)blockIdx.x * kNeChunk; q0 < HW; q0 += (int64_t)gridDim.x * kNeChunk) {
        const int nq = HW - q0 < kNeChunk ? (int)(HW - q0) : kNeChunk;
        if (tid < nq) {
            const int64_t q = q0 + tid;
            stage[tid] = ne_beta(vb, W, p, (int)(q / W), (int)(q % W));
        }
        for (int e = tid; e < P * kNeChunk; e += kNeThreads) {
            const int k = e / kNeChunk, qq = e - k * kNeChunk;
            stage[kNeChunk + e] = qq < nq ? (double)__ldg(Ji + (q0 + qq) * sn + k * sk) : 0.0;
        }
        __syncthreads();
        if (tid < tri) {
            const double* a = stage + (1 + ek) * kNeChunk;
            const double* bb = stage + (1 + el) * kNeChunk;
            for (int qq = 0; qq < nq; ++qq) acc += stage[qq] * a[qq] * bb[qq];
        }
        __syncthreads();
    }
    if (tid < tri + P) part[((int64_t)img * nbt + nbw + blockIdx.x) * (tri + P) + tid] = tid < tri ? acc : 0.0;
}

// grid (B).  A[b] += weight * (sum of the partials' triangle, mirrored), g[b] += weight * (sum of their g entries)
__global__ void __launch_bounds__(kNeThreads) ne_finalize_kernel(const double* __restrict__ part, int C, int nbt, int P,
                                                                 double weight, double* __restrict__ A, double* __restrict__ g)
{
    const int b = blockIdx.x, tid = threadIdx.x, tri = ne_tri(P), Ep = tri + P;
    if (tid >= Ep) return;
    double acc = 0.0;
    for (int c = 0; c < C; ++c) {
        const double* q = part + (int64_t)(b * C + c) * nbt * Ep + tid;
        for (int k = 0; k < nbt; ++k) acc += q[(int64_t)k * Ep];
    }
    acc *= weight;
    if (tid < tri) {
        int k, l;
        ne_tri_index(tid, P, k, l);
        A[((int64_t)b * P + k) * P + l] += acc;
        if (k != l) A[((int64_t)b * P + l) * P + k] += acc;
    } else {
        g[(int64_t)b * P + (tid - tri)] += acc;
    }
}

// grid (chunks, B*C), dynamic shared (3 + P) x kNeChunk doubles (rows {1, x, t, J_k}).  part [img][chunk][K + tri]
__global__ void __launch_bounds__(kNeThreads) ne_global_kernel(const float* __restrict__ x, const float* __restrict__ t,
                                                               const float* __restrict__ J, int64_t sb, int64_t sc, int64_t sk,
                                                               int64_t sn, int C, int64_t HW, int P, int64_t chunk_pix,
                                                               double* __restrict__ part)
{
    extern __shared__ double stage[];
    const int img = blockIdx.y, b = img / C, c = img - b * C, tid = threadIdx.x;
    const int Eg = ne_channels(P) + ne_tri(P);
    const float* xi = x + img * HW;
    const float* ti = t + img * HW;
    const float* Ji = J + b * sb + c * sc;
    int ra = 0, rb = 0;
    if (tid < Eg) ne_global_pair(tid, P, ra, rb);
    const int64_t lo = (int64_t)blockIdx.x * chunk_pix, hi = lo + chunk_pix < HW ? lo + chunk_pix : HW;
    double acc = 0.0;
    for (int64_t q0 = lo; q0 < hi; q0 += kNeChunk) {
        const int nq = hi - q0 < kNeChunk ? (int)(hi - q0) : kNeChunk;
        if (tid < nq) {
            stage[tid] = 1.0;
            stage[kNeChunk + tid] = (double)__ldg(xi + q0 + tid);
            stage[2 * kNeChunk + tid] = (double)__ldg(ti + q0 + tid);
        }
        for (int e = tid; e < P * kNeChunk; e += kNeThreads) {
            const int k = e / kNeChunk, qq = e - k * kNeChunk;
            if (qq < nq) stage[3 * kNeChunk + e] = (double)__ldg(Ji + (q0 + qq) * sn + k * sk);
        }
        __syncthreads();
        if (tid < Eg) {
            const double* a = stage + ra * kNeChunk;
            const double* bb = stage + rb * kNeChunk;
            for (int qq = 0; qq < nq; ++qq) acc += a[qq] * bb[qq];
        }
        __syncthreads();
    }
    if (tid < Eg) part[((int64_t)img * gridDim.x + blockIdx.x) * Eg + tid] = acc;
}

// grid (B).  Per channel: chunk sums -> window terms (ne_window) -> A_c = S_JJ / s^2 - a a^T - b b^T and g_c; summed over C.
__global__ void __launch_bounds__(kNeThreads) ne_global_finalize_kernel(const double* __restrict__ part, int C, int chunks, int64_t HW,
                                                                        int P, double eps, double weight, double* __restrict__ A,
                                                                        double* __restrict__ g)
{
    __shared__ double T[kNeMaxP * (kNeMaxP + 1) / 2 + 5 + 3 * kNeMaxP];
    __shared__ double rs2;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int K = ne_channels(P), tri = ne_tri(P), Eg = K + tri;
    int ek = 0, el = 0;
    if (tid < tri) ne_tri_index(tid, P, ek, el);
    double acc = 0.0;
    for (int c = 0; c < C; ++c) {
        if (tid < Eg) {
            const double* q = part + (int64_t)(b * C + c) * chunks * Eg + tid;
            double s = 0.0;
            for (int k = 0; k < chunks; ++k) s += q[(int64_t)k * Eg];
            T[tid] = s;
        }
        __syncthreads();
        if (tid == 0) rs2 = ne_window(T, 1, P, (double)HW, eps);
        __syncthreads();
        if (tid < tri) acc += rs2 * T[K + tid] - ne_ab(T, 1, P, ek, el);
        else if (tid < tri + P) acc += T[5 + 2 * P + (tid - tri)];
        __syncthreads();
    }
    acc *= weight;
    if (tid < tri) {
        A[((int64_t)b * P + ek) * P + el] += acc;
        if (ek != el) A[((int64_t)b * P + el) * P + ek] += acc;
    } else if (tid < tri + P) {
        g[(int64_t)b * P + (tid - tri)] += acc;
    }
}

int64_t ncc_normal_workspace_bytes(int B, int C, int H, int W, int p, int P)
{
    return ne_shape(B, C, H, W, p, P).total * (int64_t)sizeof(double);
}

cudaError_t launch_ncc_normal(const float* x, const float* t, const float* J, int64_t sb, int64_t sc, int64_t sk, int64_t sn, int B,
                              int C, int H, int W, int p, int P, double eps, double weight, void* workspace, double* A, double* g,
                              cudaStream_t stream)
{
    if ((int64_t)B * C > 65535 || P < 1 || P > kNeMaxP || p < 0 || p > H || p > W) return cudaErrorInvalidValue;
    if (p == 1) return cudaSuccess;  // one-pixel windows: z = 0 and Jz = 0 exactly, the system is zero
    const NeShape s = ne_shape(B, C, H, W, p, P);
    double* ws = (double*)workspace;
    const unsigned imgs = (unsigned)s.imgs;
    cudaError_t e;
    if (p == 0) {
        ne_global_kernel<<<dim3((unsigned)s.chunks, imgs), kNeThreads, (size_t)(3 + P) * kNeChunk * sizeof(double), stream>>>(
            x, t, J, sb, sc, sk, sn, C, (int64_t)H * W, P, s.chunk_pix, ws);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        ne_global_finalize_kernel<<<(unsigned)B, kNeThreads, 0, stream>>>(ws, C, s.chunks, (int64_t)H * W, P, eps, weight, A, g);
        return cudaGetLastError();
    }
    const int nbt = s.nbw + s.nbp;
    ne_window_kernel<<<dim3((unsigned)s.nbw, imgs), kNeThreads, (size_t)s.K * kNeTile * sizeof(double), stream>>>(
        x, t, J, sb, sc, sk, sn, C, H, W, p, P, eps, ws + s.v_off, ws + s.r_off, ws + s.p_off, nbt);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ne_beta_vertical_kernel<<<dim3((unsigned)cdiv((int64_t)H * s.Wp, kNeThreads), imgs), kNeThreads, 0, stream>>>(ws + s.r_off, H, W,
                                                                                                                  p, ws + s.b_off);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ne_pixel_kernel<<<dim3((unsigned)s.nbp, imgs), kNeThreads, (size_t)(1 + P) * kNeChunk * sizeof(double), stream>>>(
        J, sb, sc, sk, sn, C, H, W, p, P, ws + s.b_off, ws + s.p_off, s.nbw, nbt);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ne_finalize_kernel<<<(unsigned)B, kNeThreads, 0, stream>>>(ws + s.p_off, C, nbt, P, weight, A, g);
    return cudaGetLastError();
}

}  // namespace b200drr
