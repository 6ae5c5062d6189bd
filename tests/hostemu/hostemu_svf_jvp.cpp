// hostemu_svf_jvp.cpp -- TEST INFRASTRUCTURE: the tangent of one scaling-and-squaring step (svf_square_jvp_kernel of csrc/svf.cu)
// compiled for the CPU.  Per node the B200_HD function the kernel calls (svf_square_node_jvp); the loop over the nodes is the
// launch grid.  Never linked into libb200drr.so.
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

void put(float* p, const float4& o)
{
    p[0] = o.x;
    p[1] = o.y;
    p[2] = o.z;
    p[3] = o.w;
}

}  // namespace

extern "C" {

// field, tangent, tout, out [Bf][g0][g1][g2][4]: tout = the step's tangent along `tangent`, out (may be null) = the step
// (b200drr_svf_square_jvp)
void emu_svf_square_jvp(const float* field, const float* tangent, float* tout, float* out, int Bf, int g0, int g1, int g2, int D0,
                        int D1, int D2, float s)
{
    const int64_t nodes = (int64_t)g0 * g1 * g2;
    for (int b = 0; b < Bf; ++b) {
        const PolyLattice lat = lattice(field + 4 * b * nodes, g0, g1, g2, D0, D1, D2);
        const PolyLattice tan = lattice(tangent + 4 * b * nodes, g0, g1, g2, D0, D1, D2);
        for (int x = 0; x < g0; ++x)
            for (int y = 0; y < g1; ++y)
                for (int z = 0; z < g2; ++z) {
                    const int node[3] = {x, y, z};
                    const int64_t n = 4 * (b * nodes + svf_node(lat, x, y, z));
                    float4 o;
                    put(tout + n, svf_square_node_jvp(lat, tan, node, s, out ? &o : nullptr));
                    if (out) put(out + n, o);
                }
    }
}

}  // extern "C"
