// kernels.h -- internal launcher prototypes shared by the .cu files and the C ABI (capi.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace b200drr {

cudaError_t launch_siddon_fwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, float* out, int B, int64_t N, float shift, float eps, int reduce,
                              int align_corners, cudaStream_t stream);
cudaError_t launch_siddon_fwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                   const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                   int variant, cudaStream_t stream);
cudaError_t launch_siddon_bwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                   const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                   float* g_vol, int B, int H, int W, float shift, float eps, int stop_grad, int variant,
                                   cudaStream_t stream);
cudaError_t launch_siddon_visits(VolDims dims, const float* src, const float* tgt, int32_t* visits, int B, int64_t N,
                                 float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                              float* g_vol, int B, int64_t N, float shift, float eps, int stop_grad,
                              cudaStream_t stream);
cudaError_t launch_trilinear_fwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int reduce, int align_corners,
                                 cudaStream_t stream);
cudaError_t launch_trilinear_bwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                 float* g_vol, float* g_alpha_range, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int align_corners, cudaStream_t stream,
                                 int reduce = 0);

cudaError_t launch_trilinear_fwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                      int n_points, const float* alpha_range, int variant, cudaStream_t stream);
cudaError_t launch_trilinear_bwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                      float* g_raylen, float* g_vol, float* g_alpha_range, int B, int H, int W, float shift,
                                      float eps, int n_points, const float* alpha_range, int variant, cudaStream_t stream);

cudaError_t launch_siddon_fwd_pose(const float* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                   const float* rows, const float* cols, float* out, int B, int H, int W, float shift,
                                   float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd_pose(const float* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                   const float* rows, const float* cols, const float* gout, float* g_src, float* g_G,
                                   float* g_Wd, float* g_vol, float* ws_tgt, float* ws_len, int B, int H, int W, float shift,
                                   float eps, int stop_grad, cudaStream_t stream);

// forward with per-ray end-point sensitivities (sens: 8 floats per ray) and the backward that consumes them
cudaError_t launch_siddon_fwd_sens(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                   float* out, float* sens, int B, int64_t N, float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_fwd_sens_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                        float eps, int variant, cudaStream_t stream);
cudaError_t launch_siddon_fwd_sens_pose(const float* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                        const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                        float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                   int B, int64_t N, int stop_grad, cudaStream_t stream);
cudaError_t launch_siddon_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows,
                                        const float* cols, float* g_src, float* g_G, float* g_Wd, int B, int H, int W,
                                        int stop_grad, cudaStream_t stream);

cudaError_t launch_trilinear_fwd_sens(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                      float* out, float* sens, int B, int64_t N, int H, int W, float shift, float eps,
                                      int n_points, const float* alpha_range, int align_corners, cudaStream_t stream);
cudaError_t launch_trilinear_fwd_sens_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                             const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                             float eps, int n_points, const float* alpha_range, int slab,
                                             cudaStream_t stream);
cudaError_t launch_trilinear_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                      float* g_alpha_range, int B, int64_t N, cudaStream_t stream);
// pose-in forms of the trilinear training path (rays generated in-kernel from per-pose 3x4 matrices)
cudaError_t launch_trilinear_alpha_range_pose(VolDims dims, const float* src, const float* G, const float* Wd, const float* rows,
                                              const float* cols, float* range, int64_t* arg, void* keys, int B, int H, int W,
                                              float shift, float eps, cudaStream_t stream);
cudaError_t launch_trilinear_fwd_sens_pose(const float* packed, VolDims dims, const float* src, const float* G, const float* Wd,
                                           const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                           float shift, float eps, int n_points, const float* alpha_range, int slab,
                                           cudaStream_t stream);
cudaError_t launch_trilinear_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows,
                                           const float* cols, float* g_src, float* g_G, float* g_Wd, float* g_alpha_range, int B,
                                           int H, int W, cudaStream_t stream);

cudaError_t launch_siddon_bwd_general(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                      const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_vol, int B,
                                      int64_t N, float shift, float eps, int stop_grad, int reduce, int align_corners,
                                      int mode, cudaStream_t stream);
cudaError_t launch_siddon_fwd_general(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                      float* out, int B, int64_t N, float shift, float eps, int reduce, int align_corners,
                                      int mode, cudaStream_t stream);
cudaError_t launch_siddon_bwd_mask(const float* vol, const float* mask, VolDims dims, const float* src, const float* tgt,
                                   const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                   float* g_vol, int B, int64_t N, int C, float shift, float eps, int stop_grad,
                                   cudaStream_t stream, int W = 0);  // W > 0: full row-major grid of width W (tile-ordered threads)
cudaError_t launch_trilinear_bwd_mask(const float* vol, const float* mask, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                      float* g_vol, float* g_alpha_range, int B, int64_t N, int C, float shift, float eps,
                                      int n_points, const float* alpha_range, int align_corners, cudaStream_t stream,
                                      int W = 0);

// reference-literal kernels (literal.cu), R = float | double: fp64 path and per-segment / per-sample outputs (reduce == 2)
template <typename R>
cudaError_t launch_siddon_fwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, R* out, int B,
                                      int64_t N, R shift, R eps, int reduce, int align_corners, cudaStream_t stream);
template <typename R>
cudaError_t launch_siddon_bwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, const R* gout,
                                      const R* gseg, R* g_src, R* g_tgt, R* g_raylen, R* g_vol, int B, int64_t N, R shift, R eps,
                                      int stop_grad, int align_corners, cudaStream_t stream);
template <typename R>
cudaError_t launch_trilinear_fwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, R* out, int B,
                                         int64_t N, R shift, R eps, int n_points, const R* alpha_range, int reduce,
                                         int align_corners, cudaStream_t stream);
template <typename R>
cudaError_t launch_trilinear_bwd_literal(const R* vol, VolDims dims, const R* src, const R* tgt, const R* raylen, const R* gout,
                                         const R* gsmp, R* g_src, R* g_tgt, R* g_raylen, R* g_vol, R* g_alpha_range, int B,
                                         int64_t N, R shift, R eps, int n_points, const R* alpha_range, int align_corners,
                                         cudaStream_t stream);

// arbitrary ray sets in a caller-provided locality order (slab-major, thread i = ray i)
cudaError_t launch_siddon_fwd_sorted(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                     float* out, int B, int64_t N, float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_fwd_sens_sorted(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                          float* out, float* sens, int B, int64_t N, float shift, float eps, cudaStream_t stream);

// brick-major Siddon forward (siddon_brick.cu): TMA-staged voxel bricks in shared memory; G == nullptr -> rays from tgt/raylen
size_t siddon_brick_workspace_bytes(int B, int H, int W);
bool siddon_brick_supported(VolDims dims, int H, int W);
cudaError_t launch_siddon_fwd_brick(const float* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                    const float* G, const float* Wd, const float* rows, const float* cols, float* out,
                                    void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                    int variant, cudaStream_t stream, const int* pix_index = nullptr,
                                    const float* corners = nullptr, int64_t Nsub = 0);

cudaError_t launch_siddon_bwd_vol_brick(const float* gout, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                        const float* G, const float* Wd, const float* rows, const float* cols, float* g_vol,
                                        void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                        cudaStream_t stream);

// experiments (b200drr_x_*): chunk-reuse forward over a major-axis-fastest copy
cudaError_t launch_x_transpose_volume(const float* vol, VolDims dims, int axis, float* out, cudaStream_t stream);
cudaError_t launch_x_siddon_fwd_chunk(const float* volT, VolDims dims, int axis, const float* src, const float* tgt,
                                      const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                      int variant, cudaStream_t stream);

cudaError_t launch_x_siddon_sens_chunk(const float* volT, VolDims dims, int axis, const float* src, const float* tgt,
                                       const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                       float eps, int variant, cudaStream_t stream);

// per-pose algebra around the pose-in kernels (pose.cu)
cudaError_t launch_euler_pose_fwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, float* P, int B,
                                  cudaStream_t stream);
cudaError_t launch_euler_pose_bwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, const float* gP,
                                  float* g_rot, float* g_xyz, int B, cudaStream_t stream);
cudaError_t launch_pose_rays_fwd(const float* P, const float* Q, const float* r, const float* Ainv, float* src, float* G,
                                 float* Wd, int B, cudaStream_t stream);
cudaError_t launch_pose_rays_bwd(const float* Q, const float* r, const float* Ainv, const float* g_src, const float* g_G,
                                 const float* g_Wd, float* gP, int B, cudaStream_t stream);

cudaError_t launch_siddon_fwd_mask(const float* vol, const float* mask, VolDims dims, const float* src, const float* tgt,
                                   const float* raylen, float* out, int B, int64_t N, int C, float shift, float eps,
                                   cudaStream_t stream, int W = 0);  // W > 0: the rays are a full row-major grid of width W
cudaError_t launch_trilinear_fwd_mask(const float* vol, const float* mask, VolDims dims, const float* src,
                                      const float* tgt, const float* raylen, float* out, int B, int64_t N, int C,
                                      float shift, float eps, int n_points, const float* alpha_range, int align_corners,
                                      cudaStream_t stream, int W = 0);

cudaError_t launch_pack_corners(const float* vol, VolDims dims, float* packed, cudaStream_t stream);
cudaError_t launch_trilinear_fwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream);
cudaError_t launch_trilinear_bwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                        float* g_raylen, float* g_alpha_range, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream);

// image similarity of the registration loop (ncc.cu)
int64_t ncc_workspace_bytes(int B, int C, int64_t N);
cudaError_t launch_ncc_fwd(const float* x1, const float* x2, int B, int C, int64_t N, float eps, void* workspace, float* stats,
                           float* score, cudaStream_t stream);
cudaError_t launch_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2,
                           int B, int C, int64_t N, cudaStream_t stream);

// patch-wise NCC (local_ncc.cu)
int64_t local_ncc_workspace_bytes(int B, int C, int H, int W, int p);
cudaError_t launch_local_ncc_fwd(const float* x1, const float* x2, int B, int C, int H, int W, int p, float eps, void* workspace,
                                 float* stats, float* score, cudaStream_t stream);
cudaError_t launch_local_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2,
                                 int B, int C, int H, int W, int p, void* workspace, cudaStream_t stream);

// blur + Sobel front end of the gradient NCC (sobel.cu)
int64_t sobel_workspace_bytes(int B, int H, int W);
bool sobel_kernel_fits(int k);
cudaError_t launch_sobel_fwd(const float* x, float* out, int B, int H, int W, const float* weights, int k, cudaStream_t stream);
cudaError_t launch_sobel_bwd(const float* gout, float* g_x, int B, int H, int W, const float* weights, int k, void* workspace,
                             cudaStream_t stream);

}  // namespace b200drr
