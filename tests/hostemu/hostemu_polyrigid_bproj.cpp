// hostemu_polyrigid_bproj.cpp -- TEST INFRASTRUCTURE: the density backprojection of csrc/polyrigid.cu (polyrigid_bproj_kernel)
// compiled for the CPU.  Per ray the B200_HD function the kernel calls (polyrigid_ray_bproj, on the pose's unpadded maps as the
// kernel reads them), whose reductions are plain adds in a host build.  It builds on hostemu_polyrigid.cpp (included whole:
// emu_polyrigid, whose forward the backprojection is the transpose of).  Never linked into libb200drr.so.
#include "hostemu_polyrigid.cpp"

namespace {

template <int KP>
void run_bproj(const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* M, int Bm, int K,
               const float* weights, int g0, int g1, int g2, const float* gout, float* g_vol, int B, long N, float shift, float eps, int P,
               float amin, float amax)
{
    const std::vector<float4> wp = pack_weights(weights, K, KP, (int64_t)g0 * g1 * g2);
    const PolyLattice lat = make_lattice(reinterpret_cast<const float*>(wp.data()), g0, g1, g2, dims);
    const float step = (amax - amin) / (float)(P - 1);
    for (int b = 0; b < B; ++b) {
        const float* Mb = M + (Bm == 1 ? 0 : (long)b * K * 12);
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const float c = gout[r] * raylen[r] * step;
            if (c == 0.0f) continue;
            polyrigid_ray_bproj<KP>(dims, lat, Mb, K, load_ray(src, tgt, b, r, eps), shift, P, amin, amax, c, g_vol);
        }
    }
}

}  // namespace

extern "C" {

// M [Bm][K][12]; weights (K, g0, g1, g2) unpacked; gout [B][N]; g_vol [D0][D1][D2] overwritten with sum over rays of gout * d out / d V.
void emu_polyrigid_bproj(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* M, int Bm, int K,
                         const float* weights, int g0, int g1, int g2, const float* gout, float* g_vol, int B, long N, float shift,
                         float eps, int P, float amin, float amax)
{
    const VolDims dims = mk(D0, D1, D2);
    std::memset(g_vol, 0, sizeof(float) * (size_t)D0 * D1 * D2);
    if (K <= 4)
        run_bproj<4>(dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, g_vol, B, N, shift, eps, P, amin, amax);
    else
        run_bproj<8>(dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, g_vol, B, N, shift, eps, P, amin, amax);
}

}  // extern "C"
