// hostemu_volume16.cpp -- TEST INFRASTRUCTURE: the 16-bit voxel reads of the Siddon kernels (common.cuh: vox16_to_f32, ldg;
// brick.cuh: LdHostT) compiled for the CPU.  The same walks run on a volume stored as fp32 (vol_type 0), IEEE binary16 (1) or
// bfloat16 (2): the whole-volume lean walk and sensitivities walk of the slab kernels, and the brick decomposition (a zero-filled
// copy of every brick in the volume's own type, then brick_pair_fwd_lean / brick_pair_sens per (ray, brick) pair, as the brick
// kernel runs them).  Never linked into libb200drr.so.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../diffdrr_b200/csrc/brick.cuh"

using namespace b200drr;

namespace {

template <class V>
void walks(const V* vol, const VolDims& dims, const float* src, const float* tgt, int B, long N, float shift, float eps, int BX,
           int BY, int BZ, float* lean, float* sens, float* brick_fwd, float* brick_sens)
{
    const int D0 = dims.d[0], D1 = dims.d[1], D2 = dims.d[2];
    const int lo0[3] = {0, 0, 0};
    std::vector<Ray> rays((size_t)B * N);
    for (int b = 0; b < B; ++b)
        for (long n = 0; n < N; ++n) {
            const long r = (long)b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            rays[r] = ray;
            lean[r] = siddon_ray_lean_box<4>(vol, lo0, dims.d, D1 * D2, D2, 1, ray, shift);
            float A[3] = {0, 0, 0}, C[3] = {0, 0, 0};
            const float S = siddon_ray_sens_box<8>(vol, dims, lo0, dims.d, D1 * D2, D2, 1, ray, shift, A, C);
            float* o = sens + r * 7;
            o[0] = S;
            for (int a = 0; a < 3; ++a) {
                o[1 + a] = A[a];
                o[4 + a] = C[a];
            }
        }
    std::memset(brick_fwd, 0, sizeof(float) * (size_t)B * N);
    std::memset(brick_sens, 0, sizeof(float) * 7 * (size_t)B * N);
    std::vector<V> brick((size_t)BX * BY * BZ);
    for (int i0 = 0; i0 < D0; i0 += BX)
        for (int i1 = 0; i1 < D1; i1 += BY)
            for (int i2 = 0; i2 < D2; i2 += BZ) {
                const int org[3] = {i0, i1, i2};
                const int hi_v[3] = {std::min(i0 + BX, D0), std::min(i1 + BY, D1), std::min(i2 + BZ, D2)};
                for (int x = 0; x < BX; ++x)
                    for (int y = 0; y < BY; ++y)
                        for (int z = 0; z < BZ; ++z) {
                            const bool in = i0 + x < D0 && i1 + y < D1 && i2 + z < D2;  // TMA zero fill: +0.0 in every type
                            V v;
                            std::memset(&v, 0, sizeof(V));
                            if (in) v = vol[((size_t)(i0 + x) * D1 + (i1 + y)) * D2 + (i2 + z)];
                            brick[((size_t)x * BY + y) * BZ + z] = v;
                        }
                const LdHostT<V> ld{brick.data()};
                for (long r = 0; r < (long)B * N; ++r) {
                    const Ray& ray = rays[r];
                    float clo[3], chi[3], a_in, a_out;
                    for (int a = 0; a < 3; ++a) {
                        clo[a] = ((float)org[a] - shift) - ray.s[a];
                        chi[a] = ((float)hi_v[a] - shift) - ray.s[a];
                    }
                    if (!brick_maybe_hit(ray.inv, clo, chi, a_in, a_out)) continue;
                    // the production forward pair walk (siddon_fwd_brick_kernel, variant 0: U = 2, accumulated alphas, no pipelining)
                    brick_fwd[r] += brick_pair_fwd_lean<2, LdHostT<V>, true, false>(ld, ray.s, ray.inv, clo, chi, org, hi_v, org,
                                                                                    BY * BZ, BZ, 1, shift);
                    float A[3] = {0, 0, 0}, C[3] = {0, 0, 0};
                    float* o = brick_sens + r * 7;
                    o[0] += brick_pair_sens<8>(ld, ray, dims, org, hi_v, org, BY * BZ, BZ, 1, shift, A, C);
                    for (int a = 0; a < 3; ++a) {
                        o[1 + a] += A[a];
                        o[4 + a] += C[a];
                    }
                }
            }
}

}  // namespace

extern "C" {

void emu_vox16_to_f32(const uint16_t* bits, float* out, long n, int bf16)
{
    for (long i = 0; i < n; ++i) out[i] = vox16_to_f32(bits[i], bf16 != 0);
}

// lean [B][N]; sens [B][N][7] = (S, A[3], C[3]); the same two from the brick decomposition with BX x BY x BZ bricks.
int emu_siddon_walks16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt, int B, long N,
                       float shift, float eps, int BX, int BY, int BZ, float* lean, float* sens, float* brick_fwd, float* brick_sens)
{
    VolDims dims;
    dims.d[0] = D0;
    dims.d[1] = D1;
    dims.d[2] = D2;
    if (vol_type == 0)
        walks((const float*)vol, dims, src, tgt, B, N, shift, eps, BX, BY, BZ, lean, sens, brick_fwd, brick_sens);
    else if (vol_type == 1)
        walks((const VoxF16*)vol, dims, src, tgt, B, N, shift, eps, BX, BY, BZ, lean, sens, brick_fwd, brick_sens);
    else if (vol_type == 2)
        walks((const VoxBF16*)vol, dims, src, tgt, B, N, shift, eps, BX, BY, BZ, lean, sens, brick_fwd, brick_sens);
    else
        return -1;
    return 0;
}

}  // extern "C"
