// hostemu_polyrigid_jac.cpp -- TEST INFRASTRUCTURE: the per-pixel motion Jacobian of csrc/polyrigid.cu (polyrigid_jac_kernel)
// compiled for the CPU.  Per ray the B200_HD functions the kernel calls (polyrigid_ray_jac, poly_jac_entry) with the kernel's
// channel padding; the footprints are plain min / max loops.  It builds on hostemu_polyrigid.cpp (included whole: its volume and
// lattice packing, and emu_polyrigid, whose forward the Jacobian's image is compared with).  Never linked into libb200drr.so.
#include <algorithm>

#include "hostemu_polyrigid.cpp"

namespace {

template <int KP, class Gather>
void run_jac(const Gather& gather, const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* M, int Bm,
             int K, const float* weights, int g0, int g1, int g2, const float* T, float* img, float* J, int* rects, int B, int H, int W,
             float shift, float eps, int P, float amin, float amax)
{
    const std::vector<float4> wp = pack_weights(weights, K, KP, (int64_t)g0 * g1 * g2);
    const PolyLattice lat = make_lattice(reinterpret_cast<const float*>(wp.data()), g0, g1, g2, dims);
    const float step = (amax - amin) / (float)(P - 1);
    const long N = (long)H * W;
    for (int b = 0; b < B; ++b) {
        float sM[KP * 12];
        for (int i = 0; i < KP * 12; ++i) sM[i] = i < K * 12 ? M[(Bm == 1 ? 0 : (long)b * K * 12) + i] : 0.0f;
        const float* Tb = T + (Bm == 1 ? 0 : (long)b * K * 72);
        for (int k = 0; k < K; ++k) {
            int* rk = rects + ((long)b * K + k) * 4;
            rk[0] = W, rk[1] = -1, rk[2] = H, rk[3] = -1;
        }
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            float A[KP][3], Bv[KP][3];
            unsigned touched;
            img[r] = polyrigid_ray_jac<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax, A, Bv, touched) * (raylen[r] * step);
            const float LS = raylen[r] * step;
            const int px = (int)(n % W), py = (int)(n / W);
            for (int k = 0; k < K; ++k) {
                for (int i = 0; i < 6; ++i) J[(((long)b * K + k) * N + n) * 6 + i] = poly_jac_entry(A[k], Bv[k], ray, Tb + (k * 6 + i) * 12, LS);
                if (!((touched >> k) & 1u)) continue;
                int* rk = rects + ((long)b * K + k) * 4;
                rk[0] = std::min(rk[0], px), rk[1] = std::max(rk[1], px), rk[2] = std::min(rk[2], py), rk[3] = std::max(rk[3], py);
            }
        }
    }
}

}  // namespace

extern "C" {

// The per-pixel motion Jacobian of b200drr_polyrigid_jac on a full H x W grid: img [B][H*W], J [B][K][H*W][6], rects [B][K][4];
// T [Bm][K][6][12].  packed as in emu_polyrigid.
void emu_polyrigid_jac(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* M,
                       int Bm, int K, const float* weights, int g0, int g1, int g2, const float* T, float* img, float* J, int* rects,
                       int B, int H, int W, float shift, float eps, int P, float amin, float amax, int packed)
{
    const VolDims dims = mk(D0, D1, D2);
    std::vector<float4> pk;
    if (packed) pk = pack_corners(vol, dims);
    auto go = [&](auto gather) {
        if (K <= 4)
            run_jac<4>(gather, dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, T, img, J, rects, B, H, W, shift, eps, P, amin, amax);
        else
            run_jac<8>(gather, dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, T, img, J, rects, B, H, W, shift, eps, P, amin, amax);
    };
    if (packed) go(GatherPacked{pk.data()});
    else go(GatherPlainT<float>{vol});
}

}  // extern "C"
