// hostemu_svf.cpp -- TEST INFRASTRUCTURE: the scaling-and-squaring step of csrc/svf.cu and its adjoint compiled for the CPU.  Per
// node the B200_HD functions the kernels call (svf_square_node / svf_square_node_bwd), whose vector reductions are plain adds in a
// host build; the loop over the nodes is the launch grid.  Never linked into libb200drr.so.
#include <cstring>

#include "../../diffdrr_b200/csrc/svf_math.cuh"

using namespace b200drr;

namespace {

PolyLattice lattice(const float* field, int g0, int g1, int g2, int D0, int D1, int D2)
{
    VolDims d;
    d.d[0] = D0;
    d.d[1] = D1;
    d.d[2] = D2;
    return make_lattice(field, g0, g1, g2, d);
}

}  // namespace

extern "C" {

// field, out [Bf][g0][g1][g2][4]: out = one squaring step of field with scale s (b200drr_svf_square)
void emu_svf_square(const float* field, float* out, int Bf, int g0, int g1, int g2, int D0, int D1, int D2, float s)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    for (int b = 0; b < Bf; ++b) {
        const PolyLattice lat = lattice(field + 4 * b * nodes, g0, g1, g2, D0, D1, D2);
        for (int x = 0; x < g0; ++x)
            for (int y = 0; y < g1; ++y)
                for (int z = 0; z < g2; ++z) {
                    const int node[3] = {x, y, z};
                    const float4 o = svf_square_node(lat, node, s);
                    float* p = out + 4 * (b * nodes + svf_node(lat, x, y, z));
                    p[0] = o.x;
                    p[1] = o.y;
                    p[2] = o.z;
                    p[3] = o.w;
                }
    }
}

// gin = the adjoint of the step applied to gout (b200drr_svf_square_bwd), all [Bf][g0][g1][g2][4]; gin is zeroed here
void emu_svf_square_bwd(const float* field, const float* gout, float* gin, int Bf, int g0, int g1, int g2, int D0, int D1, int D2,
                        float s)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    std::memset(gin, 0, sizeof(float) * 4 * Bf * nodes);
    for (int b = 0; b < Bf; ++b) {
        const PolyLattice lat = lattice(field + 4 * b * nodes, g0, g1, g2, D0, D1, D2);
        for (int x = 0; x < g0; ++x)
            for (int y = 0; y < g1; ++y)
                for (int z = 0; z < g2; ++z) {
                    const int node[3] = {x, y, z};
                    const float* g = gout + 4 * (b * nodes + svf_node(lat, x, y, z));
                    if (g[0] == 0.0f && g[1] == 0.0f && g[2] == 0.0f) continue;   // as the kernel
                    svf_square_node_bwd(lat, node, s, float4{g[0], g[1], g[2], g[3]}, gin + 4 * b * nodes);
                }
    }
}

}  // extern "C"
