// hostemu_polyrigid.cpp -- TEST INFRASTRUCTURE: the blended-rigid march of csrc/polyrigid.cu compiled for the CPU.  Per ray the
// B200_HD functions the kernels call (polyrigid_ray_fwd / polyrigid_ray_bwd, poly_gM_entry) with the kernels' channel padding; the
// sums over rays are plain loops.  Also trilinear_ray_fwd on the same rays, for the identities.  Never linked into libb200drr.so.
#include <cstring>
#include <vector>

#include "../../diffdrr_b200/csrc/polyrigid_math.cuh"

using namespace b200drr;

namespace {

VolDims mk(int D0, int D1, int D2)
{
    VolDims d;
    d.d[0] = D0;
    d.d[1] = D1;
    d.d[2] = D2;
    return d;
}

// the packed-corner copy of ray_math.cuh's GatherPacked: cell (i0+1, i1+1, i2+1) holds the 8 corners of base voxel (i0, i1, i2)
std::vector<float4> pack_corners(const float* vol, const VolDims& dims)
{
    const int64_t p2 = dims.d[2] + 1, p1 = dims.d[1] + 1, p0 = dims.d[0] + 1;
    std::vector<float4> packed((size_t)(2 * p0 * p1 * p2));
    for (int64_t i = 0; i < p0; ++i)
        for (int64_t j = 0; j < p1; ++j)
            for (int64_t k = 0; k < p2; ++k) {
                float v[8];
                for (int c = 0; c < 8; ++c) {
                    const int64_t x = i - 1 + (c & 1), y = j - 1 + ((c >> 1) & 1), z = k - 1 + ((c >> 2) & 1);
                    const bool inb = x >= 0 && x < dims.d[0] && y >= 0 && y < dims.d[1] && z >= 0 && z < dims.d[2];
                    v[c] = inb ? vol[(x * dims.d[1] + y) * dims.d[2] + z] : 0.0f;
                }
                float4* cell = &packed[(size_t)(2 * ((i * p1 + j) * p2 + k))];
                cell[0] = float4{v[0], v[1], v[2], v[3]};
                cell[1] = float4{v[4], v[5], v[6], v[7]};
            }
    return packed;
}

// weights (K, g0, g1, g2) -> channel-last, K padded to KP (polyrigid_pack_weights_kernel)
std::vector<float4> pack_weights(const float* weights, int K, int KP, int64_t nodes)
{
    std::vector<float4> out((size_t)(nodes * KP / 4));
    float* o = reinterpret_cast<float*>(out.data());
    for (int64_t n = 0; n < nodes; ++n)
        for (int k = 0; k < KP; ++k) o[n * KP + k] = k < K ? weights[(int64_t)k * nodes + n] : 0.0f;
    return out;
}

template <int KP, class Gather>
void run(const Gather& gather, const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* M, int Bm,
         int K, const float* weights, int g0, int g1, int g2, const float* gout, float* out, float* g_src, float* g_tgt,
         float* g_raylen, float* g_M, float* g_alpha, int B, long N, float shift, float eps, int P, float amin, float amax)
{
    const std::vector<float4> wp = pack_weights(weights, K, KP, (int64_t)g0 * g1 * g2);
    const PolyLattice lat = make_lattice(reinterpret_cast<const float*>(wp.data()), g0, g1, g2, dims);
    const float step = (amax - amin) / (float)(P - 1);
    if (gout) {
        std::memset(g_src, 0, sizeof(float) * 3 * B);
        std::memset(g_M, 0, sizeof(float) * 12 * K * Bm);
        g_alpha[0] = g_alpha[1] = 0.0f;
    }
    for (int b = 0; b < B; ++b) {
        float sM[KP * 12];
        for (int i = 0; i < KP * 12; ++i) sM[i] = i < K * 12 ? M[(Bm == 1 ? 0 : (long)b * K * 12) + i] : 0.0f;
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            out[r] = polyrigid_ray_fwd<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax) * (raylen[r] * step);
            if (!gout) continue;
            float AG[KP][3], BG[KP][3];
            const TriGrad tg = polyrigid_ray_bwd<KP>(gather, dims, lat, sM, ray, shift, P, amin, amax, gout[r], raylen[r], AG, BG);
            for (int a = 0; a < 3; ++a) {
                g_src[b * 3 + a] += tg.gs[a];
                g_tgt[r * 3 + a] = tg.gt[a];
            }
            g_raylen[r] = gout[r] * step * tg.sumV;
            g_alpha[0] += tg.ga0;
            g_alpha[1] += tg.ga1;
            float* gm = g_M + (Bm == 1 ? 0 : (long)b * K * 12);
            for (int k = 0; k < K; ++k)
                for (int e = 0; e < 12; ++e) gm[k * 12 + e] += poly_gM_entry(AG[k], BG[k], ray, e);
        }
    }
}

}  // namespace

extern "C" {

// out [B][N] overwritten; with gout != NULL also g_src [B][3], g_tgt [B][N][3], g_raylen [B][N], g_M [Bm][K][12], g_alpha [2].
// packed != 0 marches the packed-corner copy (GatherPacked) instead of the plain volume (GatherPlainT<float>).
void emu_polyrigid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* M,
                   int Bm, int K, const float* weights, int g0, int g1, int g2, const float* gout, float* out, float* g_src,
                   float* g_tgt, float* g_raylen, float* g_M, float* g_alpha, int B, long N, float shift, float eps, int P, float amin,
                   float amax, int packed)
{
    const VolDims dims = mk(D0, D1, D2);
    std::vector<float4> pk;
    if (packed) pk = pack_corners(vol, dims);
    auto go = [&](auto gather) {
        if (K <= 4)
            run<4>(gather, dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, out, g_src, g_tgt, g_raylen, g_M, g_alpha, B, N,
                   shift, eps, P, amin, amax);
        else
            run<8>(gather, dims, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, out, g_src, g_tgt, g_raylen, g_M, g_alpha, B, N,
                   shift, eps, P, amin, amax);
    };
    if (packed) go(GatherPacked{pk.data()});
    else go(GatherPlainT<float>{vol});
}

// the Trilinear renderer's forward on the same rays (reduce = sum, align_corners = 0)
void emu_polyrigid_trilinear(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                             float* out, int B, long N, float shift, float eps, int P, float amin, float amax)
{
    const VolDims dims = mk(D0, D1, D2);
    const float step = (amax - amin) / (float)(P - 1);
    for (int b = 0; b < B; ++b)
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            out[r] = trilinear_ray_fwd(vol, dims, ray, shift, P, amin, amax, 0, 0) * (raylen[r] * step);
        }
}

}  // extern "C"
