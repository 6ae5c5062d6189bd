// structures.cu -- piecewise-rigid DRRs (DESIGN.md 6f): every labelled structure rendered under its own pose in one launch.
//
// Slot s of pose b is an ordinary pose-in render (src, G, Wd of index b*S + s) of the voxels whose label belongs to s, walked over
// the slot's box only.  A thread per (pixel, b, s); per (b, s) the CTA first projects the box's 8 corners onto the detector and
// the pixels outside that footprint write zeros without walking, so the cost follows the structures' footprints.  Every output
// element is written by exactly one thread: no atomics, repeated calls give identical bits.
#include <algorithm>
#include <climits>

#include "kernels.h"
#include "structures_math.cuh"

namespace b200drr {

namespace {

constexpr int kBoxThreads = 256;

__global__ void label_boxes_init_kernel(int* __restrict__ boxes, VolDims dims)
{
    const int l = threadIdx.x;  // 256 labels
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        boxes[l * 6 + a] = dims.d[a];  // empty: lo = D > hi = 0
        boxes[l * 6 + 3 + a] = 0;
    }
}

// A thread per row (i0, i1) of the label volume; the label runs of the row go into the CTA's shared boxes, which leave with one
// global atomic min / max per (CTA, present label).
__global__ void __launch_bounds__(kBoxThreads) label_boxes_kernel(const uint8_t* __restrict__ labels, VolDims dims,
                                                                   int* __restrict__ boxes)
{
    __shared__ int sb[256 * 6];
    for (int i = threadIdx.x; i < 256 * 6; i += kBoxThreads) sb[i] = (i % 6) < 3 ? INT_MAX : INT_MIN;
    __syncthreads();
    const int64_t n_rows = (int64_t)dims.d[0] * dims.d[1];
    for (int64_t row = (int64_t)blockIdx.x * kBoxThreads + threadIdx.x; row < n_rows; row += (int64_t)gridDim.x * kBoxThreads) {
        const int i0 = (int)(row / dims.d[1]), i1 = (int)(row % dims.d[1]);
        label_row_runs(labels + row * dims.d[2], dims.d[2], [&](int l, int b, int e) {
            int* q = sb + l * 6;
            atomicMin(q + 0, i0);
            atomicMin(q + 1, i1);
            atomicMin(q + 2, b);
            atomicMax(q + 3, i0 + 1);
            atomicMax(q + 4, i1 + 1);
            atomicMax(q + 5, e);
        });
    }
    __syncthreads();
    for (int l = threadIdx.x; l < 256; l += kBoxThreads) {
        const int* q = sb + l * 6;
        if (q[0] == INT_MAX) continue;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(boxes + l * 6 + a, q[a]);
            atomicMax(boxes + l * 6 + 3 + a, q[3 + a]);
        }
    }
}

// Pixel tiles of TW x TH made of 8 x 4 warp bundles, as the slab-major sensitivities kernel (siddon.cu).  SENS = false: the image
// only, through the forward walk (no crossing coefficients are accumulated).
template <int TW, int TH, int U, bool SENS, class V>
__global__ void __launch_bounds__(TW* TH, 8) siddon_structures_kernel(const V* __restrict__ vol, const uint8_t* __restrict__ labels,
                                                                      VolDims dims, const float* __restrict__ src,
                                                                      const float* __restrict__ G, const float* __restrict__ Wd,
                                                                      const float* __restrict__ rows, const float* __restrict__ cols,
                                                                      const int* __restrict__ slot_of_label,
                                                                      const int* __restrict__ box, float* __restrict__ out,
                                                                      float* __restrict__ sens, int S, int H, int W, float shift,
                                                                      float eps)
{
    constexpr int WX = TW / 8;
    __shared__ uint8_t mine[256];
    __shared__ int rect[4];
    const int tiles_x = (W + TW - 1) / TW, tiles_y = (H + TH - 1) / TH;
    const int tiles = tiles_x * tiles_y;
    const int tile = blockIdx.x % tiles;
    const int bs = blockIdx.x / tiles;  // b * S + s
    const int s = bs % S;
    int lo_v[3], hi_v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo_v[a] = __ldg(box + s * 6 + a);
        hi_v[a] = __ldg(box + s * 6 + 3 + a);
    }
    for (int i = threadIdx.x; i < 256; i += TW * TH) mine[i] = __ldg(slot_of_label + i) == s;
    if (threadIdx.x < 8) {  // one box corner per lane, then min / max over the 8 lanes
        float u = 0.0f, v = 0.0f;
        const bool ok = box_corner_uv(G + (int64_t)bs * 12, src + (int64_t)bs * 3, lo_v, hi_v, shift, threadIdx.x, u, v);
        const bool all_ok = __all_sync(0xffu, ok);
        float umin = u, umax = u, vmin = v, vmax = v;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            umin = fminf(umin, __shfl_xor_sync(0xffu, umin, o));
            umax = fmaxf(umax, __shfl_xor_sync(0xffu, umax, o));
            vmin = fminf(vmin, __shfl_xor_sync(0xffu, vmin, o));
            vmax = fmaxf(vmax, __shfl_xor_sync(0xffu, vmax, o));
        }
        if (threadIdx.x == 0) {
            int r[4];
            footprint_rect(all_ok, umin, umax, vmin, vmax, __ldg(cols), __ldg(cols + W - 1), W, __ldg(rows), __ldg(rows + H - 1), H, r);
            rect[0] = r[0]; rect[1] = r[1]; rect[2] = r[2]; rect[3] = r[3];
        }
    }
    __syncthreads();
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * TW + (warp % WX) * 8 + (lane & 7);
    const int py = tile_y * TH + (warp / WX) * 4 + (lane >> 3);
    if (px >= W || py >= H) return;
    const int64_t r = ((int64_t)bs * H + py) * W + px;
    float S_ = 0.0f, L = 0.0f, jt[3] = {0.0f, 0.0f, 0.0f}, js[3] = {0.0f, 0.0f, 0.0f};
    const bool inside = px >= rect[0] && px <= rect[1] && py >= rect[2] && py <= rect[3] && lo_v[0] < hi_v[0] && lo_v[1] < hi_v[1] &&
                        lo_v[2] < hi_v[2];
    if (inside) {
        const Ray ray = make_ray(PoseRays{G, Wd, rows, cols}, src, nullptr, nullptr, bs, r, px, py, eps, L);
        if (!box_surely_missed(ray, lo_v, hi_v, shift)) {
            const LoadGated ld{labels, mine};
            if constexpr (SENS) {
                // the CUT entry rule of gated walks (load_cut<LoadGated>, structures_math.cuh): ties at the label box's faces are
                // booked as the un-cut walk of density * (label in slot) books them
                float A[3] = {0.0f, 0.0f, 0.0f}, C[3] = {0.0f, 0.0f, 0.0f};
                S_ = siddon_ray_sens_box<U, LoadGated>(vol, dims, lo_v, hi_v, dims.d[1] * dims.d[2], dims.d[2], 1, ray, shift, A, C, ld);
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const float k = L * ray.inv[a];
                    jt[a] = -k * A[a];
                    js[a] = k * (A[a] - C[a]);
                }
            } else {
                S_ = siddon_ray_lean_box<U, V, LoadGated>(vol, lo_v, hi_v, dims.d[1] * dims.d[2], dims.d[2], 1, ray, shift, ld);
            }
        }
    }
    out[r] = L * S_;
    if constexpr (SENS) {
        reinterpret_cast<float4*>(sens)[r * 2] = make_float4(jt[0], jt[1], jt[2], S_);
        reinterpret_cast<float4*>(sens)[r * 2 + 1] = make_float4(js[0], js[1], js[2], 0.0f);
    }
}

}  // namespace

cudaError_t launch_label_boxes(const uint8_t* labels, VolDims dims, int32_t* boxes, cudaStream_t stream)
{
    label_boxes_init_kernel<<<1, 256, 0, stream>>>(boxes, dims);
    const int64_t n_rows = (int64_t)dims.d[0] * dims.d[1];
    const int64_t blocks = std::min<int64_t>((n_rows + kBoxThreads - 1) / kBoxThreads, (int64_t)current_sm_count() * 8);
    label_boxes_kernel<<<(unsigned)blocks, kBoxThreads, 0, stream>>>(labels, dims, boxes);
    return cudaGetLastError();
}

template <class V>
cudaError_t launch_siddon_fwd_sens_structures(const V* vol, const uint8_t* labels, VolDims dims, const float* src, const float* G,
                                              const float* Wd, const float* rows, const float* cols, const int32_t* slot_of_label,
                                              const int32_t* box, float* out, float* sens, int B, int S, int H, int W, float shift,
                                              float eps, cudaStream_t stream)
{
    // sensitivities walk unrolled by 4 (64 registers at 8 CTAs per SM), the image-only walk by 8 (56 registers; 4 % faster than 4 at
    // 512^3 -> 256^2, 16 poses on the H100)
    constexpr int TW = 8, TH = 16, U_SENS = 4, U_FWD = 8;
    const int64_t blocks = (int64_t)((W + TW - 1) / TW) * ((H + TH - 1) / TH) * B * S;
    if (blocks > INT32_MAX) return cudaErrorInvalidValue;
    if (sens != nullptr)
        siddon_structures_kernel<TW, TH, U_SENS, true, V><<<(unsigned)blocks, TW * TH, 0, stream>>>(
            vol, labels, dims, src, G, Wd, rows, cols, slot_of_label, box, out, sens, S, H, W, shift, eps);
    else
        siddon_structures_kernel<TW, TH, U_FWD, false, V><<<(unsigned)blocks, TW * TH, 0, stream>>>(
            vol, labels, dims, src, G, Wd, rows, cols, slot_of_label, box, out, nullptr, S, H, W, shift, eps);
    return cudaGetLastError();
}
#define B200DRR_STRUCTURES(V)                                                                                                       \
    template cudaError_t launch_siddon_fwd_sens_structures<V>(const V*, const uint8_t*, VolDims, const float*, const float*,        \
                                                              const float*, const float*, const float*, const int32_t*,            \
                                                              const int32_t*, float*, float*, int, int, int, int, float, float,    \
                                                              cudaStream_t);
B200DRR_STRUCTURES(float)
B200DRR_STRUCTURES(VoxF16)
B200DRR_STRUCTURES(VoxBF16)
#undef B200DRR_STRUCTURES

}  // namespace b200drr
