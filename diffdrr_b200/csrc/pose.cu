// pose.cu -- the per-pose algebra either side of the pose-in kernels, one kernel each way (sm_90a).
//
// DRR.forward turns pose parameters into the (src, G, Wd) triple of b200drr_siddon_fwd_pose through ~95 tiny ATen kernels per
// training step (cos/sin/stack/bmm/cat and their autograd twins): 0.25 ms of a 1.6 ms step.  Here the same algebra is
// one thread per pose:
//   euler_pose_*  : reference pose.py `convert(rot, xyz, "euler_angles", convention)`  -> 4x4 pose matrix
//                   R = R_c0(a0) R_c1(a1) R_c2(a2),  P = [[R, R t], [0 0 0 1]]
//   pose_rays_*   : detector.py:144-154 + drr.py:201-205 collapsed (see b200drr_siddon_fwd_pose in include/b200drr.h)
//                   T = P Q,  G = Ainv T (rows 0..2),  src = Ainv (P r),  Wd = [T[:3,:3] | T[:3,3] - (P r)[:3]]
//                   with Q = reorient . calibration, r = reorient[:, 3], Ainv = affine_inverse.
#include "kernels.h"

namespace b200drr {

namespace {

__device__ __forceinline__ void axis_rotation(int axis, float c, float s, float R[9])
{
    // reference pose.py `_axis_angle_rotation` / pytorch3d convention
    if (axis == 0) { R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = c; R[5] = -s; R[6] = 0; R[7] = s; R[8] = c; }
    else if (axis == 1) { R[0] = c; R[1] = 0; R[2] = s; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = -s; R[7] = 0; R[8] = c; }
    else { R[0] = c; R[1] = -s; R[2] = 0; R[3] = s; R[4] = c; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1; }
}

__device__ __forceinline__ void mat3_mul(const float A[9], const float B[9], float C[9])
{
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = fmaf(A[i * 3 + 2], B[6 + j], fmaf(A[i * 3 + 1], B[3 + j], A[i * 3] * B[j]));
}

__device__ __forceinline__ float mat3_dot(const float A[9], const float B[9])
{
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < 9; ++i) acc = fmaf(A[i], B[i], acc);
    return acc;
}

}  // namespace

__global__ void euler_pose_fwd_kernel(const float* __restrict__ rot, const float* __restrict__ xyz, int c0, int c1, int c2,
                                      float scale, float* __restrict__ P, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int conv[3] = {c0, c1, c2};
    float R[3][9];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float s, c;
        sincosf(rot[b * 3 + i] * scale, &s, &c);
        axis_rotation(conv[i], c, s, R[i]);
    }
    float R01[9], Rm[9];
    mat3_mul(R[0], R[1], R01);
    mat3_mul(R01, R[2], Rm);
    const float t[3] = {xyz[b * 3], xyz[b * 3 + 1], xyz[b * 3 + 2]};
    float* p = P + b * 16;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        p[i * 4 + 0] = Rm[i * 3 + 0];
        p[i * 4 + 1] = Rm[i * 3 + 1];
        p[i * 4 + 2] = Rm[i * 3 + 2];
        p[i * 4 + 3] = fmaf(Rm[i * 3 + 2], t[2], fmaf(Rm[i * 3 + 1], t[1], Rm[i * 3] * t[0]));
    }
    p[12] = 0.0f; p[13] = 0.0f; p[14] = 0.0f; p[15] = 1.0f;
}

__global__ void euler_pose_bwd_kernel(const float* __restrict__ rot, const float* __restrict__ xyz, int c0, int c1, int c2,
                                      float scale, const float* __restrict__ gP, float* __restrict__ g_rot,
                                      float* __restrict__ g_xyz, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int conv[3] = {c0, c1, c2};
    float R[3][9], dR[3][9];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float s, c;
        sincosf(rot[b * 3 + i] * scale, &s, &c);
        axis_rotation(conv[i], c, s, R[i]);
        axis_rotation(conv[i], -s, c, dR[i]);  // d/da of (c, s) is (-s, c) ...
        dR[i][conv[i] * 4] = 0.0f;             // ... and the constant 1 on the rotation axis differentiates to 0
    }
    const float t[3] = {xyz[b * 3], xyz[b * 3 + 1], xyz[b * 3 + 2]};
    const float* g = gP + b * 16;
    // centre = R t  =>  gR += gcentre t^T,  g_t = R^T gcentre
    float gR[9], Rm[9], R01[9], tmp[9], tmp2[9];
    mat3_mul(R[0], R[1], R01);
    mat3_mul(R01, R[2], Rm);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) gR[i * 3 + j] = fmaf(g[i * 4 + 3], t[j], g[i * 4 + j]);
    if (g_xyz) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            g_xyz[b * 3 + j] = fmaf(Rm[6 + j], g[11], fmaf(Rm[3 + j], g[7], Rm[j] * g[3]));
    }
    if (g_rot) {
        mat3_mul(dR[0], R[1], tmp);
        mat3_mul(tmp, R[2], tmp2);
        g_rot[b * 3 + 0] = mat3_dot(gR, tmp2) * scale;
        mat3_mul(R[0], dR[1], tmp);
        mat3_mul(tmp, R[2], tmp2);
        g_rot[b * 3 + 1] = mat3_dot(gR, tmp2) * scale;
        mat3_mul(R01, dR[2], tmp2);
        g_rot[b * 3 + 2] = mat3_dot(gR, tmp2) * scale;
    }
}

__global__ void pose_rays_fwd_kernel(const float* __restrict__ P, const float* __restrict__ Q, const float* __restrict__ r,
                                     const float* __restrict__ Ainv, float* __restrict__ src, float* __restrict__ G,
                                     float* __restrict__ Wd, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float* p = P + b * 16;
    float T[16], Pr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc = fmaf(p[i * 4 + k], __ldg(Q + k * 4 + j), acc);
            T[i * 4 + j] = acc;
        }
        float acc = 0.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(p[i * 4 + k], __ldg(r + k), acc);
        Pr[i] = acc;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc = fmaf(__ldg(Ainv + i * 4 + k), T[k * 4 + j], acc);
            G[b * 12 + i * 4 + j] = acc;
        }
        float acc = 0.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc = fmaf(__ldg(Ainv + i * 4 + k), Pr[k], acc);
        src[b * 3 + i] = acc;
        Wd[b * 12 + i * 4 + 0] = T[i * 4 + 0];
        Wd[b * 12 + i * 4 + 1] = T[i * 4 + 1];
        Wd[b * 12 + i * 4 + 2] = T[i * 4 + 2];
        Wd[b * 12 + i * 4 + 3] = T[i * 4 + 3] - Pr[i];
    }
}

__global__ void pose_rays_bwd_kernel(const float* __restrict__ Q, const float* __restrict__ r, const float* __restrict__ Ainv,
                                     const float* __restrict__ g_src, const float* __restrict__ g_G,
                                     const float* __restrict__ g_Wd, float* __restrict__ gP, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float gT[16], gPr[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float acc = 0.0f;
#pragma unroll
            for (int i = 0; i < 3; ++i) acc = fmaf(__ldg(Ainv + i * 4 + k), g_G[b * 12 + i * 4 + j], acc);
            if (k < 3) acc += g_Wd[b * 12 + k * 4 + j];
            gT[k * 4 + j] = acc;
        }
        float acc = 0.0f;
#pragma unroll
        for (int i = 0; i < 3; ++i) acc = fmaf(__ldg(Ainv + i * 4 + k), g_src[b * 3 + i], acc);
        if (k < 3) acc -= g_Wd[b * 12 + k * 4 + 3];
        gPr[k] = acc;
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float acc = gPr[a] * __ldg(r + c);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc = fmaf(gT[a * 4 + j], __ldg(Q + c * 4 + j), acc);
            gP[b * 16 + a * 4 + c] = acc;
        }
}

cudaError_t launch_euler_pose_fwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, float* P, int B,
                                  cudaStream_t stream)
{
    euler_pose_fwd_kernel<<<(B + 63) / 64, 64, 0, stream>>>(rot, xyz, c0, c1, c2, scale, P, B);
    return cudaGetLastError();
}

cudaError_t launch_euler_pose_bwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, const float* gP,
                                  float* g_rot, float* g_xyz, int B, cudaStream_t stream)
{
    euler_pose_bwd_kernel<<<(B + 63) / 64, 64, 0, stream>>>(rot, xyz, c0, c1, c2, scale, gP, g_rot, g_xyz, B);
    return cudaGetLastError();
}

cudaError_t launch_pose_rays_fwd(const float* P, const float* Q, const float* r, const float* Ainv, float* src, float* G,
                                 float* Wd, int B, cudaStream_t stream)
{
    pose_rays_fwd_kernel<<<(B + 63) / 64, 64, 0, stream>>>(P, Q, r, Ainv, src, G, Wd, B);
    return cudaGetLastError();
}

cudaError_t launch_pose_rays_bwd(const float* Q, const float* r, const float* Ainv, const float* g_src, const float* g_G,
                                 const float* g_Wd, float* gP, int B, cudaStream_t stream)
{
    pose_rays_bwd_kernel<<<(B + 63) / 64, 64, 0, stream>>>(Q, r, Ainv, g_src, g_G, g_Wd, gP, B);
    return cudaGetLastError();
}

}  // namespace b200drr
