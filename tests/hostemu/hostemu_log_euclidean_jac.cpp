// hostemu_log_euclidean_jac.cpp -- TEST INFRASTRUCTURE: the P-tangent squaring step (svf_square_tangents_kernel of csrc/svf.cu) and
// the Jacobian march (deform_jac_kernel of csrc/deform.cu) compiled for the CPU.  Per node and per ray the B200_HD functions the
// kernels call (svf_square_node_tangents, deform_ray_jac); the loops are the launch grids, and the footprints are grown by plain
// min / max.  It builds on hostemu_deform.cpp (included whole: its volume packing and gathers).  Never linked into libb200drr.so.
#include "hostemu_deform.cpp"
#include "../../diffdrr_b200/csrc/svf_math.cuh"

namespace {

template <int KP, class Gather>
void run_jac(const Gather& gather, const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* field,
             const float* tangents, int Bf, int g0, int g1, int g2, int K, float* img, float* J, int* rects, int* flushes, int B, int H,
             int W, float shift, float eps, int P, float amin, float amax)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2, N = (int64_t)H * W;
    const float step = (amax - amin) / (float)(P - 1);
    for (int i = 0; i < B * K; ++i) {
        rects[4 * i] = W;
        rects[4 * i + 1] = -1;
        rects[4 * i + 2] = H;
        rects[4 * i + 3] = -1;
    }
    for (int b = 0; b < B; ++b) {
        const int64_t fb = Bf == 1 ? 0 : b;
        const PolyLattice lat = make_lattice(field + fb * nodes * 4, g0, g1, g2, dims);
        const float4* tan = reinterpret_cast<const float4*>(tangents) + fb * nodes * 6 * K;
        for (int64_t n = 0; n < N; ++n) {
            const int64_t r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            float Jp[KP * 6];
            unsigned touched;
            const float acc = deform_ray_jac<KP>(gather, dims, lat, tan, K, ray, shift, P, amin, amax, Jp, touched, flushes[r]);
            const float Ls = raylen[r] * step;
            img[r] = acc * Ls;
            const int x = (int)(n % W), y = (int)(n / W);
            for (int k = 0; k < K; ++k) {
                for (int i = 0; i < 6; ++i) J[((b * K + k) * N + n) * 6 + i] = Jp[k * 6 + i] * Ls;
                if ((touched >> k) & 1u) {
                    int* rk = rects + 4 * (b * K + k);
                    rk[0] = std::min(rk[0], x);
                    rk[1] = std::max(rk[1], x);
                    rk[2] = std::min(rk[2], y);
                    rk[3] = std::max(rk[3], y);
                }
            }
        }
    }
}

}  // namespace

extern "C" {

// field [Bf][g0][g1][g2][4], tangents and tout [Bf][g0][g1][g2][P][4]; out (may be null) (b200drr_svf_square_tangents)
void emu_svf_square_tangents(const float* field, const float* tangents, float* tout, float* out, int Bf, int P, int g0, int g1, int g2,
                             int D0, int D1, int D2, float s)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    for (int b = 0; b < Bf; ++b) {
        const PolyLattice lat = make_lattice(field + 4 * b * nodes, g0, g1, g2, mk(D0, D1, D2));
        const float4* tan = reinterpret_cast<const float4*>(tangents) + b * nodes * P;
        for (int x = 0; x < g0; ++x)
            for (int y = 0; y < g1; ++y)
                for (int z = 0; z < g2; ++z) {
                    const int node[3] = {x, y, z};
                    const int64_t i = b * nodes + svf_node(lat, x, y, z);
                    svf_square_node_tangents(lat, tan, P, node, s, reinterpret_cast<float4*>(tout) + i * P,
                                             out ? reinterpret_cast<float4*>(out) + i : nullptr);
                }
    }
}

// b200drr_deform_jac on a full H x W grid: img [B][H*W], J [B][K][H*W][6], rects [B][K][4], flushes [B][H*W] overwritten.
// packed != 0 marches the packed-corner copy.
void emu_deform_jac(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* field,
                    const float* tangents, int Bf, int g0, int g1, int g2, int K, float* img, float* J, int* rects, int* flushes, int B,
                    int H, int W, float shift, float eps, int P, float amin, float amax, int packed)
{
    const VolDims dims = mk(D0, D1, D2);
    std::vector<float4> pk;
    if (packed) pk = pack_corners(vol, dims);
    auto go = [&](auto gather) {
        if (K <= 4)
            run_jac<4>(gather, dims, src, tgt, raylen, field, tangents, Bf, g0, g1, g2, K, img, J, rects, flushes, B, H, W, shift, eps, P,
                       amin, amax);
        else
            run_jac<8>(gather, dims, src, tgt, raylen, field, tangents, Bf, g0, g1, g2, K, img, J, rects, flushes, B, H, W, shift, eps, P,
                       amin, amax);
    };
    if (packed) go(GatherPacked{pk.data()});
    else go(GatherPlainT<float>{vol});
}

}  // extern "C"
