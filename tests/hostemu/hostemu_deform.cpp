// hostemu_deform.cpp -- TEST INFRASTRUCTURE: the deformable march of csrc/deform.cu compiled for the CPU.  Per ray the B200_HD
// functions the kernels call (deform_ray_fwd / deform_ray_bwd), whose field scatter is a plain add in a host build; the sums over
// rays are plain loops.  Never linked into libb200drr.so.
#include <cstring>
#include <vector>

#include "../../diffdrr_b200/csrc/deform_math.cuh"

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

template <class Gather>
void run(const Gather& gather, const VolDims& dims, const float* src, const float* tgt, const float* raylen, const float* field, int Bf,
         int g0, int g1, int g2, const float* gout, float* out, float* g_src, float* g_tgt, float* g_raylen, float* g_field,
         float* g_alpha, int* flushes, int B, long N, float shift, float eps, int P, float amin, float amax)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    const float step = (amax - amin) / (float)(P - 1);
    if (gout) {
        std::memset(g_src, 0, sizeof(float) * 3 * B);
        if (g_field) std::memset(g_field, 0, sizeof(float) * 4 * nodes * Bf);
        g_alpha[0] = g_alpha[1] = 0.0f;
    }
    for (int b = 0; b < B; ++b) {
        const int64_t fo = Bf == 1 ? 0 : b * nodes * 4;
        const PolyLattice lat = make_lattice(field + fo, g0, g1, g2, dims);
        for (long n = 0; n < N; ++n) {
            const long r = b * N + n;
            const Ray ray = load_ray(src, tgt, b, r, eps);
            out[r] = deform_ray_fwd(gather, dims, lat, ray, shift, P, amin, amax) * (raylen[r] * step);
            if (!gout) continue;
            int fl = 0;
            const TriGrad tg = deform_ray_bwd(gather, dims, lat, ray, shift, P, amin, amax, gout[r], raylen[r],
                                              g_field ? g_field + fo : nullptr, fl);
            if (flushes) flushes[r] = fl;
            for (int a = 0; a < 3; ++a) {
                g_src[b * 3 + a] += tg.gs[a];
                g_tgt[r * 3 + a] = tg.gt[a];
            }
            g_raylen[r] = gout[r] * step * tg.sumV;
            g_alpha[0] += tg.ga0;
            g_alpha[1] += tg.ga1;
        }
    }
}

}  // namespace

extern "C" {

// field [Bf][g0][g1][g2][4].  out [B][N] overwritten; with gout != NULL also g_src [B][3], g_tgt [B][N][3], g_raylen [B][N],
// g_alpha [2], g_field (the field's layout; NULL skips the scatter) and flushes [B][N] (may be NULL).  packed != 0 marches the
// packed-corner copy (GatherPacked) instead of the plain volume (GatherPlainT<float>).
void emu_deform(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* field,
                int Bf, int g0, int g1, int g2, const float* gout, float* out, float* g_src, float* g_tgt, float* g_raylen,
                float* g_field, float* g_alpha, int* flushes, int B, long N, float shift, float eps, int P, float amin, float amax,
                int packed)
{
    const VolDims dims = mk(D0, D1, D2);
    std::vector<float4> pk;
    if (packed) pk = pack_corners(vol, dims);
    auto go = [&](auto gather) {
        run(gather, dims, src, tgt, raylen, field, Bf, g0, g1, g2, gout, out, g_src, g_tgt, g_raylen, g_field, g_alpha, flushes, B, N,
            shift, eps, P, amin, amax);
    };
    if (packed) go(GatherPacked{pk.data()});
    else go(GatherPlainT<float>{vol});
}

}  // extern "C"
