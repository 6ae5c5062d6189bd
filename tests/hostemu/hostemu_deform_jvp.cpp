// hostemu_deform_jvp.cpp -- TEST INFRASTRUCTURE: the field-tangent (JVP) march of csrc/deform.cu (deform_jvp_kernel) compiled for
// the CPU.  Per ray the B200_HD function the kernel calls (deform_ray_jvp).  It builds on hostemu_deform.cpp (included whole: its
// volume packing, and emu_deform, whose forward and field scatter the JVP is compared with).  Never linked into libb200drr.so.
#include "hostemu_deform.cpp"

namespace {

template <class Gather>
void run_jvp(const Gather& gather, const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* field,
             const float* tangent, int Bf, int g0, int g1, int g2, float* img, float* jv, int B, long N, float shift, float eps, int P,
             float amin, float amax)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    const float step = (amax - amin) / (float)(P - 1);
    for (int b = 0; b < B; ++b) {
        const int64_t fo = Bf == 1 ? 0 : b * nodes * 4;
        const PolyLattice lat = make_lattice(field + fo, g0, g1, g2, dims);
        const PolyLattice tan = make_lattice(tangent + fo, g0, g1, g2, dims);
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            float acc;
            const float d = deform_ray_jvp(gather, dims, lat, tan, ray, shift, P, amin, amax, acc);
            const float Ls = raylen[r] * step;
            jv[r] = d * Ls;
            img[r] = acc * Ls;
        }
    }
}

}  // namespace

extern "C" {

// field, tangent [Bf][g0][g1][g2][4]; img, jv [B][N] overwritten.  packed != 0 marches the packed-corner copy.
void emu_deform_jvp(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                    const float* field, const float* tangent, int Bf, int g0, int g1, int g2, float* img, float* jv, int B, long N,
                    float shift, float eps, int P, float amin, float amax, int packed)
{
    const VolDims dims = mk(D0, D1, D2);
    std::vector<float4> pk;
    if (packed) pk = pack_corners(vol, dims);
    auto go = [&](auto gather) {
        run_jvp(gather, dims, src, tgt, raylen, field, tangent, Bf, g0, g1, g2, img, jv, B, N, shift, eps, P, amin, amax);
    };
    if (packed) go(GatherPacked{pk.data()});
    else go(GatherPlainT<float>{vol});
}

}  // extern "C"
