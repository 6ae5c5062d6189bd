// common.cuh -- shared helpers for the sm_90a DRR kernels.
//
// The per-ray math (ray_math.cuh) is written as host+device functions so that tests/hostemu can compile the very
// same source with g++ and check it against the oracle in the CPU-only container.  That emulation is test
// infrastructure; the product library contains device code only and has no CPU path.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
struct float4 {  // host emulation only (tests/hostemu): the CUDA headers provide it for device builds
    float x, y, z, w;
};
struct uint4 {
    unsigned x, y, z, w;
};
#endif

namespace b200drr {

constexpr int kWarp = 32;

struct VolDims {
    int d[3];
};

B200_HD float ldg(const float* p)
{
#if defined(__CUDA_ARCH__)
    return __ldg(p);  // (an L2::256B prefetch hint was tried: no effect)
#else
    return *p;
#endif
}

// 16-bit voxel storage (DESIGN.md 4.5): the volume may be stored as IEEE binary16 or bfloat16; every voxel read widens it to fp32
// and all geometry and accumulation stay fp32.  The kernels take the voxel type V = float | VoxF16 | VoxBF16 as a template
// parameter and read through ldg(vol + off), so the fp32 instantiations are the unchanged fp32 kernels.
struct VoxF16 {
    uint16_t bits;
    static constexpr bool kBF16 = false;
};
struct VoxBF16 {
    uint16_t bits;
    static constexpr bool kBF16 = true;
};

B200_HD float f32_from_bits(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    __builtin_memcpy(&f, &u, 4);
    return f;
#endif
}

B200_HD uint32_t f32_bits(float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    __builtin_memcpy(&u, &f, 4);
    return u;
#endif
}

// The one 16-bit -> fp32 conversion (exact: both formats are subsets of fp32).  bf16 is the top half of an fp32; binary16 is
// decoded by hand on the host (subnormals, infinities and NaN payloads as numpy's float16 -> float32) and by cvt on the device.
B200_HD float vox16_to_f32(uint16_t h, bool bf16)
{
    if (bf16) return f32_from_bits((uint32_t)h << 16);
#if defined(__CUDA_ARCH__)
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
#else
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
    if (e == 0x1fu) return f32_from_bits(sign | 0x7f800000u | (m << 13));  // inf / NaN
    if (e == 0) {
        if (m == 0) return f32_from_bits(sign);
        e = 113;  // subnormal m * 2^-24: normalise the mantissa
        while ((m & 0x400u) == 0) {
            m <<= 1;
            --e;
        }
        return f32_from_bits(sign | (e << 23) | ((m & 0x3ffu) << 13));
    }
    return f32_from_bits(sign | ((e + 112) << 23) | (m << 13));
#endif
}

B200_HD float ldg(const VoxF16* p)
{
#if defined(__CUDA_ARCH__)
    return vox16_to_f32(__ldg(reinterpret_cast<const unsigned short*>(p)), false);
#else
    return vox16_to_f32(p->bits, false);
#endif
}
B200_HD float ldg(const VoxBF16* p)
{
#if defined(__CUDA_ARCH__)
    return vox16_to_f32(__ldg(reinterpret_cast<const unsigned short*>(p)), true);
#else
    return vox16_to_f32(p->bits, true);
#endif
}

// single-rounding multiply / add that the compiler may not contract into an fma
B200_HD float mul_rn(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b;
    return r;
#endif
}
B200_HD float add_rn(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b;
    return r;
#endif
}

// accumulate into the volume gradient: red.global.add.f32 on the device, plain add in the host emulation
B200_HD void red_add(float* addr, float v)
{
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
#else
    *addr += v;
#endif
}

// four consecutive floats (16-byte aligned) in one red.global.add.v4.f32
B200_HD void red_add4(float* addr, float a, float b, float c, float d)
{
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
#else
    addr[0] += a; addr[1] += b; addr[2] += c; addr[3] += d;
#endif
}

#if defined(__CUDACC__)
// SMs of the current device: the grid-stride launches size their grids from it
inline int current_sm_count()
{
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return 1;
    return sms;
}
#endif

// One ray: d = (target - source) + eps (renderers.py:104-106), inv = 1/d.
struct Ray {
    float s[3];
    float d[3];
    float inv[3];
};

B200_HD Ray load_ray(const float* src, const float* tgt, int b, int64_t r, float eps)
{
    Ray ray;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        ray.s[a] = ldg(src + b * 3 + a);
        ray.d[a] = (ldg(tgt + r * 3 + a) - ray.s[a]) + eps;
        ray.inv[a] = 1.0f / ray.d[a];
    }
    return ray;
}

// alpha of plane i on axis a with the reference's own rounding sequence ((i - shift) - s) / d
B200_HD float plane_alpha(const Ray& ray, int a, float i, float shift) { return ((i - shift) - ray.s[a]) / ray.d[a]; }

// Optional in-kernel ray generation ("pose-in" entry points): when G != nullptr the rays of pose b are made from
//   target_voxel(h, w) = G[b] . (cols[w], rows[h], 1, 1),   raylen(h, w) = | Wd[b] . (cols[w], rows[h], 1, 1) |
// (G = affine_inverse . extrinsic . reorient . calibration, Wd = the same without affine_inverse and with the source
// subtracted; reference detector.py:144-154 + drr.py:201-205 collapsed into two 3x4 matrices per pose), so the
// (B, N, 3) target tensor and the ray-length image never exist in HBM.
struct PoseRays {
    const float* G;     // [B][3][4]
    const float* Wd;    // [B][3][4]
    const float* rows;  // [H]  canonical detector y of image row h   (detector.py:114-126)
    const float* cols;  // [W]  canonical detector x of image column w
};

// The pose-in ray of pixel (px, py) of pose b and its length L (host+device: tests/hostemu builds this same source).
B200_HD Ray pose_ray(const float* G, const float* Wd, const float* rows, const float* cols, const float* src, int b, int px, int py,
                     float eps, float& L)
{
    const float c = ldg(cols + px), rr = ldg(rows + py);
    const float* g = G + b * 12;
    const float* wd = Wd + b * 12;
    Ray ray;
    float l2 = 0.0f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float t = fmaf(ldg(g + a * 4), c, fmaf(ldg(g + a * 4 + 1), rr, ldg(g + a * 4 + 2) + ldg(g + a * 4 + 3)));
        const float dw = fmaf(ldg(wd + a * 4), c, fmaf(ldg(wd + a * 4 + 1), rr, ldg(wd + a * 4 + 2) + ldg(wd + a * 4 + 3)));
        l2 = fmaf(dw, dw, l2);
        ray.s[a] = ldg(src + b * 3 + a);
        ray.d[a] = (t - ray.s[a]) + eps;
        ray.inv[a] = 1.0f / ray.d[a];
    }
    L = sqrtf(l2);
    return ray;
}

#if defined(__CUDACC__)
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of `v` (blockDim.x multiple of 32, <= 1024); result valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* smem /* >= 32 floats */)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();  // protect smem reuse between consecutive calls
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    const int nwarp = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nwarp) ? smem[threadIdx.x] : 0.0f;
    if (warp == 0) v = warp_sum(v);
    return v;
}

// Ray handled by this thread of a 128-thread CTA: row order (W == 0, any ray set) or, for a full detector grid of width W,
// a 16 x 8 pixel tile made of four 8 x 4 warp bundles (neighbouring rays gather neighbouring voxels).  -1 = no ray.
__device__ __forceinline__ int64_t tiled_ray_index(int64_t N, int W)
{
    if (W <= 0) {
        const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
        return n < N ? n : -1;
    }
    const int H = (int)(N / W), tiles_x = (W + 15) / 16;
    const int tile_x = blockIdx.x % tiles_x, tile_y = blockIdx.x / tiles_x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int px = tile_x * 16 + (warp & 1) * 8 + (lane & 7), py = tile_y * 8 + (warp >> 1) * 4 + (lane >> 3);
    return (px < W && py < H) ? (int64_t)py * W + px : -1;
}
inline dim3 tiled_ray_grid(int B, int64_t N, int W)
{
    if (W <= 0) return dim3((unsigned)((N + 127) / 128), (unsigned)B, 1);
    const int64_t H = N / W;
    return dim3((unsigned)(((W + 15) / 16) * ((H + 7) / 8)), (unsigned)B, 1);
}

__device__ __forceinline__ Ray make_ray(const PoseRays& pr, const float* __restrict__ src, const float* __restrict__ tgt,
                                        const float* __restrict__ raylen, int b, int64_t r, int px, int py, float eps,
                                        float& L)
{
    if (pr.G == nullptr) {
        L = __ldg(raylen + r);
        return load_ray(src, tgt, b, r, eps);
    }
    return pose_ray(pr.G, pr.Wd, pr.rows, pr.cols, src, b, px, py, eps, L);
}
#endif

}  // namespace b200drr
