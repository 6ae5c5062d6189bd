// hostemu_brick_sens.cpp -- TEST INFRASTRUCTURE: the brick decomposition of the training step's sensitivities walk
// (siddon_brick.cu, SENS mode) compiled for the CPU.  Per brick a zero-filled copy of the voxels, per (ray, brick) pair the
// kernel's conservative hit test and brick_pair_sens on the copy (brick-local loads), the pair flushed into sens / out as the
// kernel does; then the elementwise backward of sens_bwd_kernel.  Never linked into libb200drr.so.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../diffdrr_b200/csrc/brick.cuh"

using namespace b200drr;

extern "C" {

// sens [B][N][8] and out [B][N] are overwritten; g_src [B][3], g_tgt [B][N][3], g_raylen [B][N] from gout.  Returns the number
// of (ray, brick) pairs that were walked.
long emu_siddon_sens_brick(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                           const float* gout, float* out, float* sens, float* g_src, float* g_tgt, float* g_raylen, int B, long N,
                           float shift, float eps, int BX, int BY, int BZ)
{
    VolDims dims;
    dims.d[0] = D0;
    dims.d[1] = D1;
    dims.d[2] = D2;
    std::memset(out, 0, sizeof(float) * (size_t)B * N);
    std::memset(sens, 0, sizeof(float) * 8 * (size_t)B * N);
    std::vector<Ray> rays((size_t)B * N);
    for (int b = 0; b < B; ++b)
        for (long n = 0; n < N; ++n) rays[(size_t)b * N + n] = load_ray(src, tgt, b, (long)b * N + n, eps);
    std::vector<float> brick((size_t)BX * BY * BZ);
    long pairs = 0;
    for (int i0 = 0; i0 < D0; i0 += BX)
        for (int i1 = 0; i1 < D1; i1 += BY)
            for (int i2 = 0; i2 < D2; i2 += BZ) {
                const int org[3] = {i0, i1, i2};
                const int lo_v[3] = {i0, i1, i2};
                const int hi_v[3] = {std::min(i0 + BX, D0), std::min(i1 + BY, D1), std::min(i2 + BZ, D2)};
                for (int x = 0; x < BX; ++x)
                    for (int y = 0; y < BY; ++y)
                        for (int z = 0; z < BZ; ++z) {
                            const bool in = i0 + x < D0 && i1 + y < D1 && i2 + z < D2;  // TMA zero fill outside the volume
                            brick[((size_t)x * BY + y) * BZ + z] = in ? vol[((size_t)(i0 + x) * D1 + (i1 + y)) * D2 + (i2 + z)] : 0.0f;
                        }
                const LdHost ld{brick.data()};
                for (int b = 0; b < B; ++b)
                    for (long n = 0; n < N; ++n) {
                        const long r = (long)b * N + n;
                        const Ray& ray = rays[r];
                        float clo[3], chi[3], a_in, a_out;
                        for (int a = 0; a < 3; ++a) {
                            clo[a] = ((float)lo_v[a] - shift) - ray.s[a];
                            chi[a] = ((float)hi_v[a] - shift) - ray.s[a];
                        }
                        if (!brick_maybe_hit(ray.inv, clo, chi, a_in, a_out)) continue;
                        ++pairs;
                        float A[3] = {0, 0, 0}, C[3] = {0, 0, 0};
                        const float S = brick_pair_sens<8>(ld, ray, dims, lo_v, hi_v, org, BY * BZ, BZ, 1, shift, A, C);
                        const float L = raylen[r];
                        float jt[3], js[3];
                        bool any = S != 0.0f;
                        for (int a = 0; a < 3; ++a) {
                            const float k = L * ray.inv[a];
                            jt[a] = -k * A[a];
                            js[a] = k * (A[a] - C[a]);
                            any = any || jt[a] != 0.0f || js[a] != 0.0f;
                        }
                        if (any) {
                            red_add4(sens + r * 8, jt[0], jt[1], jt[2], S);
                            red_add4(sens + r * 8 + 4, js[0], js[1], js[2], 0.0f);
                            red_add(out + r, L * S);
                        }
                    }
            }
    std::memset(g_src, 0, sizeof(float) * 3 * B);
    for (int b = 0; b < B; ++b)
        for (long n = 0; n < N; ++n) {
            const long r = (long)b * N + n;
            for (int a = 0; a < 3; ++a) {
                g_tgt[r * 3 + a] = gout[r] * sens[r * 8 + a];
                g_src[b * 3 + a] += gout[r] * sens[r * 8 + 4 + a];
            }
            g_raylen[r] = gout[r] * sens[r * 8 + 3];
        }
    return pairs;
}

}  // extern "C"
