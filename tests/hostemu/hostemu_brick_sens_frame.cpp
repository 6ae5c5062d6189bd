// hostemu_brick_sens_frame.cpp -- TEST INFRASTRUCTURE: the per-ray frame record of the brick kernel's sensitivities mode
// (brick.cuh, SensFrameRec) compiled for the CPU.  For every (ray, brick) pair that passes the kernel's hit test it runs the pair
// twice: brick_pair_sens on the freshly built ray, and brick_pair_sens_framed on the frame read back from the record that
// brick_prep_kernel writes (pack_sens_frame / unpack_sens_frame, 1/d from the ray table entry, s from the pose).  Never linked
// into libb200drr.so.
#include <algorithm>
#include <vector>

#include "../../diffdrr_b200/csrc/brick.cuh"

using namespace b200drr;

extern "C" {

// fresh / framed [max_pairs][8]: S, A[3], C[3], L per pair.  Returns the number of pairs (more than max_pairs: only the first
// max_pairs are written).
long emu_brick_sens_frame_pairs(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                                int B, long N, float shift, float eps, int BX, int BY, int BZ, float* fresh, float* framed,
                                long max_pairs)
{
    VolDims dims;
    dims.d[0] = D0;
    dims.d[1] = D1;
    dims.d[2] = D2;
    std::vector<SensFrameRec> recs((size_t)B * N);
    for (int b = 0; b < B; ++b)
        for (long n = 0; n < N; ++n) {
            const long r = (long)b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            recs[r] = pack_sens_frame(volume_frame(ray, dims, shift), ray.d, raylen[r]);
        }
    std::vector<float> brick((size_t)BX * BY * BZ);
    long pairs = 0;
    for (int i0 = 0; i0 < D0; i0 += BX)
        for (int i1 = 0; i1 < D1; i1 += BY)
            for (int i2 = 0; i2 < D2; i2 += BZ) {
                const int org[3] = {i0, i1, i2};
                const int hi_v[3] = {std::min(i0 + BX, D0), std::min(i1 + BY, D1), std::min(i2 + BZ, D2)};
                for (int x = 0; x < BX; ++x)
                    for (int y = 0; y < BY; ++y)
                        for (int z = 0; z < BZ; ++z) {
                            const bool in = i0 + x < D0 && i1 + y < D1 && i2 + z < D2;
                            brick[((size_t)x * BY + y) * BZ + z] = in ? vol[((size_t)(i0 + x) * D1 + (i1 + y)) * D2 + (i2 + z)] : 0.0f;
                        }
                const LdHost ld{brick.data()};
                for (int b = 0; b < B; ++b)
                    for (long n = 0; n < N; ++n) {
                        const long r = (long)b * N + n;
                        const Ray ray = load_ray(src, tgt, b, r, eps);
                        float clo[3], chi[3], a_in, a_out;
                        for (int a = 0; a < 3; ++a) {
                            clo[a] = ((float)org[a] - shift) - ray.s[a];
                            chi[a] = ((float)hi_v[a] - shift) - ray.s[a];
                        }
                        if (!brick_maybe_hit(ray.inv, clo, chi, a_in, a_out)) continue;
                        if (pairs < max_pairs) {
                            float* o = fresh + 8 * pairs;
                            float A[3] = {0, 0, 0}, C[3] = {0, 0, 0};
                            o[0] = brick_pair_sens<8>(ld, ray, dims, org, hi_v, org, BY * BZ, BZ, 1, shift, A, C);
                            for (int a = 0; a < 3; ++a) {
                                o[1 + a] = A[a];
                                o[4 + a] = C[a];
                            }
                            o[7] = raylen[r];
                            // the kernel's view: 1/d from the ray table, s from the pose, the rest from the record
                            const float s[3] = {src[b * 3 + 0], src[b * 3 + 1], src[b * 3 + 2]};
                            float d[3], L;
                            const VolFrame f = unpack_sens_frame(recs[r], ray.inv, d, L);
                            float* g = framed + 8 * pairs;
                            float Af[3] = {0, 0, 0}, Cf[3] = {0, 0, 0};
                            g[0] = brick_pair_sens_framed<8>(ld, f, s, d, dims, org, hi_v, org, BY * BZ, BZ, 1, shift, Af, Cf);
                            for (int a = 0; a < 3; ++a) {
                                g[1 + a] = Af[a];
                                g[4 + a] = Cf[a];
                            }
                            g[7] = L;
                        }
                        ++pairs;
                    }
            }
    return pairs;
}

}  // extern "C"
