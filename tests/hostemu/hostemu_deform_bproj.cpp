// hostemu_deform_bproj.cpp -- TEST INFRASTRUCTURE: the density backprojection of csrc/deform.cu (deform_bproj_kernel) compiled for
// the CPU.  Per ray the B200_HD function the kernel calls (deform_ray_bproj), whose reductions are plain adds in a host build.  It
// builds on hostemu_deform.cpp (included whole: emu_deform, whose forward the backprojection is the transpose of).  Never linked
// into libb200drr.so.
#include "hostemu_deform.cpp"

extern "C" {

// field [Bf][g0][g1][g2][4]; gout [B][N]; g_vol [D0][D1][D2] overwritten with sum over rays of gout * d out / d V.
void emu_deform_bproj(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* field, int Bf, int g0,
                      int g1, int g2, const float* gout, float* g_vol, int B, long N, float shift, float eps, int P, float amin,
                      float amax)
{
    const VolDims dims = mk(D0, D1, D2);
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    const float step = (amax - amin) / (float)(P - 1);
    std::memset(g_vol, 0, sizeof(float) * (size_t)D0 * D1 * D2);
    for (int b = 0; b < B; ++b) {
        const PolyLattice lat = make_lattice(field + (Bf == 1 ? 0 : b * nodes * 4), g0, g1, g2, dims);
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const float c = gout[r] * raylen[r] * step;
            if (c == 0.0f) continue;
            deform_ray_bproj(dims, lat, load_ray(src, tgt, b, r, eps), shift, P, amin, amax, c, g_vol);
        }
    }
}

}  // extern "C"
