// svf.cu -- scaling-and-squaring steps of a stationary velocity field and their adjoint for sm_90a (math in svf_math.cuh).
// One thread per lattice node and pose, 256 threads per CTA over the flattened [Bf][g0][g1][g2] nodes, so a warp reads 32
// consecutive float4 nodes along axis 2.  The forward and the tangent write each node once (bit for bit repeatable); the adjoint
// adds 9 vector reductions per node into a gradient the launcher zeroes first, so it repeats to fp32 reordering.  The P-tangent step
// (DESIGN.md 6p) keeps one thread per node and loops over the node's P tangents, which are contiguous in the node-major layout.
#include "kernels.h"
#include "svf_math.cuh"

namespace b200drr {

constexpr int kSvfThreads = 256;

namespace {

// node index t of the flattened [Bf][g0][g1][g2] -> (pose, node coordinates); false past the end
__device__ __forceinline__ bool svf_index(const PolyLattice& lat, int64_t total, int64_t& pose, int node[3])
{
    const int64_t t = (int64_t)blockIdx.x * kSvfThreads + threadIdx.x;
    if (t >= total) return false;
    const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
    pose = t / nodes;
    const int r = (int)(t - pose * nodes);
    node[2] = r % lat.g[2];
    node[1] = (r / lat.g[2]) % lat.g[1];
    node[0] = r / (lat.g[2] * lat.g[1]);
    return true;
}

}  // namespace

__global__ void __launch_bounds__(kSvfThreads) svf_square_kernel(PolyLattice lat, int64_t total, float s, float4* __restrict__ out)
{
    int64_t b;
    int node[3];
    if (!svf_index(lat, total, b, node)) return;
    const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
    lat.w += b * nodes;
    out[b * nodes + svf_node(lat, node[0], node[1], node[2])] = svf_square_node(lat, node, s);
}

__global__ void __launch_bounds__(kSvfThreads) svf_square_bwd_kernel(PolyLattice lat, int64_t total, float s,
                                                                      const float4* __restrict__ gout, float* gin)
{
    int64_t b;
    int node[3];
    if (!svf_index(lat, total, b, node)) return;
    const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
    lat.w += b * nodes;
    const float4 gp = __ldg(gout + b * nodes + svf_node(lat, node[0], node[1], node[2]));
    if (gp.x == 0.0f && gp.y == 0.0f && gp.z == 0.0f) return;  // every add would be a zero
    svf_square_node_bwd(lat, node, s, gp, gin + 4 * b * nodes);
}

__global__ void __launch_bounds__(kSvfThreads) svf_square_jvp_kernel(PolyLattice lat, PolyLattice tan, int64_t total, float s,
                                                                      float4* __restrict__ tout, float4* __restrict__ out)
{
    int64_t b;
    int node[3];
    if (!svf_index(lat, total, b, node)) return;
    const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
    lat.w += b * nodes;
    tan.w += b * nodes;
    const int64_t x = b * nodes + svf_node(lat, node[0], node[1], node[2]);
    tout[x] = svf_square_node_jvp(lat, tan, node, s, out ? out + x : nullptr);
}

// P tangents per node ([Bf][g0][g1][g2][P] float4 in and out): one thread per node forms y, its cell and J_U once for all P
__global__ void __launch_bounds__(kSvfThreads) svf_square_tangents_kernel(PolyLattice lat, const float4* __restrict__ tan, int P,
                                                                           int64_t total, float s, float4* __restrict__ tout,
                                                                           float4* __restrict__ out)
{
    int64_t b;
    int node[3];
    if (!svf_index(lat, total, b, node)) return;
    const int64_t nodes = (int64_t)lat.g[0] * lat.g[1] * lat.g[2];
    lat.w += b * nodes;
    const int64_t x = b * nodes + svf_node(lat, node[0], node[1], node[2]);
    svf_square_node_tangents(lat, tan + b * nodes * P, P, node, s, tout + x * P, out ? out + x : nullptr);
}

cudaError_t launch_svf_square(const float* field, float* out, int Bf, int g0, int g1, int g2, VolDims dims, float scale,
                              cudaStream_t stream)
{
    const PolyLattice lat = make_lattice(field, g0, g1, g2, dims);
    const int64_t total = (int64_t)Bf * g0 * g1 * g2;
    svf_square_kernel<<<(unsigned)((total + kSvfThreads - 1) / kSvfThreads), kSvfThreads, 0, stream>>>(lat, total, scale,
                                                                                                        (float4*)out);
    return cudaGetLastError();
}

cudaError_t launch_svf_square_bwd(const float* field, const float* gout, float* gin, int Bf, int g0, int g1, int g2, VolDims dims,
                                  float scale, cudaStream_t stream)
{
    const int64_t total = (int64_t)Bf * g0 * g1 * g2;
    const cudaError_t e = cudaMemsetAsync(gin, 0, sizeof(float) * 4 * (size_t)total, stream);
    if (e != cudaSuccess) return e;
    const PolyLattice lat = make_lattice(field, g0, g1, g2, dims);
    svf_square_bwd_kernel<<<(unsigned)((total + kSvfThreads - 1) / kSvfThreads), kSvfThreads, 0, stream>>>(lat, total, scale,
                                                                                                            (const float4*)gout, gin);
    return cudaGetLastError();
}

cudaError_t launch_svf_square_jvp(const float* field, const float* tangent, float* tout, float* out, int Bf, int g0, int g1, int g2,
                                  VolDims dims, float scale, cudaStream_t stream)
{
    const PolyLattice lat = make_lattice(field, g0, g1, g2, dims);
    const PolyLattice tan = make_lattice(tangent, g0, g1, g2, dims);
    const int64_t total = (int64_t)Bf * g0 * g1 * g2;
    svf_square_jvp_kernel<<<(unsigned)((total + kSvfThreads - 1) / kSvfThreads), kSvfThreads, 0, stream>>>(lat, tan, total, scale,
                                                                                                            (float4*)tout, (float4*)out);
    return cudaGetLastError();
}

cudaError_t launch_svf_square_tangents(const float* field, const float* tangents, float* tout, float* out, int Bf, int P, int g0, int g1,
                                       int g2, VolDims dims, float scale, cudaStream_t stream)
{
    const PolyLattice lat = make_lattice(field, g0, g1, g2, dims);
    const int64_t total = (int64_t)Bf * g0 * g1 * g2;
    svf_square_tangents_kernel<<<(unsigned)((total + kSvfThreads - 1) / kSvfThreads), kSvfThreads, 0, stream>>>(
        lat, (const float4*)tangents, P, total, scale, (float4*)tout, (float4*)out);
    return cudaGetLastError();
}

}  // namespace b200drr
