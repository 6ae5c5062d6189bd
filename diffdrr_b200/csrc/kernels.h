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
template <class V>  // V = float | VoxF16 | VoxBF16
cudaError_t launch_trilinear_fwd(const V* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int reduce, int align_corners,
                                 cudaStream_t stream);
cudaError_t launch_trilinear_bwd(const float* vol, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                 float* g_vol, float* g_alpha_range, int B, int64_t N, float shift, float eps,
                                 int n_points, const float* alpha_range, int align_corners, cudaStream_t stream,
                                 int reduce = 0);

template <class V>
cudaError_t launch_trilinear_fwd_grid(const V* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                      int n_points, const float* alpha_range, int variant, cudaStream_t stream);
cudaError_t launch_trilinear_bwd_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                      const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                      float* g_raylen, float* g_vol, float* g_alpha_range, int B, int H, int W, float shift,
                                      float eps, int n_points, const float* alpha_range, int variant, cudaStream_t stream);

template <class V>  // V = float | VoxF16 | VoxBF16 (common.cuh) here and below where marked
cudaError_t launch_siddon_fwd_pose(const V* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                   const float* rows, const float* cols, float* out, int B, int H, int W, float shift,
                                   float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd_pose(const float* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                   const float* rows, const float* cols, const float* gout, float* g_src, float* g_G,
                                   float* g_Wd, float* g_vol, float* ws_tgt, float* ws_len, int B, int H, int W, float shift,
                                   float eps, int stop_grad, cudaStream_t stream);

// forward with per-ray end-point sensitivities (sens: 8 floats per ray) and the backward that consumes them
template <class V>
cudaError_t launch_siddon_fwd_sens(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                   float* out, float* sens, int B, int64_t N, float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_fwd_sens_grid(const float* vol, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, float* out, float* sens, int B, int H, int W, float shift,
                                        float eps, int variant, cudaStream_t stream);
template <class V>
cudaError_t launch_siddon_fwd_sens_pose(const V* vol, VolDims dims, const float* src, const float* G, const float* Wd,
                                        const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                        float shift, float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                   int B, int64_t N, int stop_grad, cudaStream_t stream);
// piecewise-rigid renders (structures.cu): label boxes, and one gated pose-in walk per (pixel, pose, slot); sens may be NULL
cudaError_t launch_label_boxes(const uint8_t* labels, VolDims dims, int32_t* boxes, cudaStream_t stream);
template <class V>
cudaError_t launch_siddon_fwd_sens_structures(const V* vol, const uint8_t* labels, VolDims dims, const float* src, const float* G,
                                              const float* Wd, const float* rows, const float* cols, const int32_t* slot_of_label,
                                              const int32_t* box, float* out, float* sens, int B, int S, int H, int W, float shift,
                                              float eps, cudaStream_t stream);
cudaError_t launch_siddon_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows,
                                        const float* cols, float* g_src, float* g_G, float* g_Wd, int B, int H, int W,
                                        int stop_grad, cudaStream_t stream);

template <class V>
cudaError_t launch_trilinear_fwd_sens(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
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
template <class V>
cudaError_t launch_siddon_fwd_sorted(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                     float* out, int B, int64_t N, float shift, float eps, cudaStream_t stream);
template <class V>
cudaError_t launch_siddon_fwd_sens_sorted(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                          float* out, float* sens, int B, int64_t N, float shift, float eps, cudaStream_t stream);

// brick-major Siddon forward (siddon_brick.cu): TMA-staged voxel bricks in shared memory; G == nullptr -> rays from tgt/raylen
size_t siddon_brick_workspace_bytes(int B, int H, int W);
size_t siddon_sens_brick_scratch_bytes(int B, int H, int W);  // the sensitivities mode's own scratch (+ per-ray frame records)
bool siddon_brick_supported(VolDims dims, int H, int W, int elem_bytes = 4);  // 16-byte global strides for the TMA map
template <class V>
cudaError_t launch_siddon_fwd_brick(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                    const float* G, const float* Wd, const float* rows, const float* cols, float* out,
                                    void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                    int variant, cudaStream_t stream, const int* pix_index = nullptr,
                                    const float* corners = nullptr, int64_t Nsub = 0);

cudaError_t launch_siddon_bwd_vol_brick(const float* gout, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                        const float* G, const float* Wd, const float* rows, const float* cols, float* g_vol,
                                        void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                        cudaStream_t stream);
// training step through the brick kernel's sensitivities mode (full detector grids; scratch from cudaMallocAsync on `stream`;
// G == nullptr -> rays from tgt/raylen)
template <class V>
cudaError_t launch_siddon_fwd_sens_brick(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                         const float* G, const float* Wd, const float* rows, const float* cols, float* out,
                                         float* sens, int B, int H, int W, float shift, float eps, cudaStream_t stream);
bool siddon_sens_brick_route(VolDims dims, int B, int H, int W, const void* vol, const float* sens, int elem_bytes = 4);

// the library's default routes, shared by the fp32 entry points (variant 0 / default options) and the 16-bit twins
template <class V>
cudaError_t launch_siddon_fwd_fast(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen, float* out,
                                   int B, int64_t N, float shift, float eps, cudaStream_t stream);
template <class V>
cudaError_t launch_siddon_fwd_grid_default(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                           float* out, int B, int H, int W, float shift, float eps, cudaStream_t stream);
template <class V>
cudaError_t launch_siddon_fwd_sens_grid_default(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                                float* out, float* sens, int B, int H, int W, float shift, float eps,
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
// 16-bit volumes: packed cells of 8 corners in the volume's own type (ray_math.cuh: Cell16); G == nullptr -> rays from tgt/raylen
template <class V>
struct Cell16;
template <class V>
cudaError_t launch_pack_corners16(const V* vol, VolDims dims, Cell16<V>* packed, cudaStream_t stream);
template <class PK>
cudaError_t launch_trilinear_fwd_packed_t(const PK* packed, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                          float* out, int B, int H, int W, float shift, float eps, int n_points,
                                          const float* alpha_range, int slab, cudaStream_t stream);
template <class V>
cudaError_t launch_trilinear_fwd_sens_packed16(const Cell16<V>* packed, VolDims dims, const float* src, const float* tgt,
                                               const float* raylen, const float* G, const float* Wd, const float* rows,
                                               const float* cols, float* out, float* sens, int B, int H, int W, float shift,
                                               float eps, int n_points, const float* alpha_range, int slab, cudaStream_t stream);
cudaError_t launch_trilinear_fwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, float* out, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream);
cudaError_t launch_trilinear_bwd_packed(const float* packed, VolDims dims, const float* src, const float* tgt,
                                        const float* raylen, const float* gout, float* g_src, float* g_tgt,
                                        float* g_raylen, float* g_alpha_range, int B, int H, int W, float shift, float eps,
                                        int n_points, const float* alpha_range, int slab, cudaStream_t stream);

// per-pixel pose Jacobians from the saved sensitivities (jacobian.cu)
cudaError_t launch_siddon_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                        const float* rows, const float* cols, float* J, int B, int H, int W, int P, int stop_grad,
                                        cudaStream_t stream);
cudaError_t launch_trilinear_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                           const float* rows, const float* cols, const float* drange, float* J, int B, int H, int W,
                                           int P, cudaStream_t stream);

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

// Gauss-Newton normal equations of the global / patch-wise NCC (ncc_normal.cu); p = 0 is the global NCC
int64_t ncc_normal_workspace_bytes(int B, int C, int H, int W, int p, int P);
cudaError_t launch_ncc_normal(const float* x, const float* t, const float* J, int64_t sb, int64_t sc, int64_t sk, int64_t sn, int B,
                              int C, int H, int W, int p, int P, double eps, double weight, void* workspace, double* A, double* g,
                              cudaStream_t stream);

// global-NCC normal equations of a piecewise-rigid composite, block-sparse over the structures' footprints, and the footprints
// themselves (ncc_normal_structures.cu)
cudaError_t launch_structure_footprints(const float* src, const float* G, const float* rows, const float* cols, const int32_t* box,
                                        int32_t* rects, int B, int S, int H, int W, float shift, cudaStream_t stream);
int64_t ncc_normal_structures_workspace_bytes(int B, int K, int H);
cudaError_t launch_ncc_normal_structures(const float* x, const float* t, int t_batch, const float* J, int64_t sb, int64_t ss,
                                         int64_t sn, int64_t sk, const int32_t* rects, int B, int K, int S, int H, int W, double eps,
                                         double weight, void* workspace, double* A, double* g, cudaStream_t stream);

// blur + Sobel front end of the gradient NCC (sobel.cu)
int64_t sobel_workspace_bytes(int B, int H, int W);
bool sobel_kernel_fits(int k);
cudaError_t launch_sobel_fwd(const float* x, float* out, int B, int H, int W, const float* weights, int k, cudaStream_t stream);
cudaError_t launch_sobel_bwd(const float* gout, float* g_x, int B, int H, int W, const float* weights, int k, void* workspace,
                             cudaStream_t stream);

// mutual information from Parzen joint histograms (mutual_info.cu)
int64_t mi_workspace_bytes(int B, int64_t N, int nb);
cudaError_t launch_mi_fwd(const float* x1, const float* x2, int B, int64_t N, const float* bins, const float* sigma, int nb,
                          double eps, int normalize, void* workspace, float* stats, float* score, cudaStream_t stream);
cudaError_t launch_mi_bwd(const float* x1, const float* x2, const float* bins, const float* sigma, const float* stats,
                          const float* gscore, float* g_x1, float* g_x2, int B, int64_t N, int nb, cudaStream_t stream);

// blended-rigid (skinned) trilinear render (polyrigid.cu).  Exactly one of vol / packed is given; vol_type 0 = fp32, else
// B200DRR_VOL_F16 / B200DRR_VOL_BF16.  W > 0: the N rays of a pose are a full row-major grid of width W.
int polyrigid_channels(int K);  // K padded to the 4 or 8 channels the packed weight lattice stores
int64_t polyrigid_scratch_floats(int B, int64_t N, int W, int K);
cudaError_t launch_polyrigid_pack_weights(const float* weights, int K, int g0, int g1, int g2, float* packed, cudaStream_t stream);
cudaError_t launch_polyrigid_fwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 float* out, int B, int64_t N, int W, float shift, float eps, int n_points, const float* alpha_range,
                                 cudaStream_t stream);
cudaError_t launch_polyrigid_bwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_M, float* g_alpha_range,
                                 float* scratch, int B, int64_t N, int W, float shift, float eps, int n_points,
                                 const float* alpha_range, cudaStream_t stream);
// per-pixel motion Jacobian on a full H x W grid: T [Bm][K][6][12], img [B][H*W], J [B][K][H*W][6], rects [B][K][4] (set empty first)
cudaError_t launch_polyrigid_jac(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                                 const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                                 const float* T, float* img, float* J, int* rects, int B, int H, int W, float shift, float eps,
                                 int n_points, const float* alpha_range, cudaStream_t stream);
// the forward's transpose in the density: g_vol [D0][D1][D2], zeroed here, += sum over the rays of gout * d out / d V
cudaError_t launch_polyrigid_bproj(VolDims dims, const float* src, const float* tgt, const float* raylen, const float* M, int Bm, int K,
                                   const float* weights, int g0, int g1, int g2, const float* gout, float* g_vol, int B, int64_t N, int W,
                                   float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream);
// the fixed-order finish of the blended-rigid backward's per-CTA partial rows; deform.cu launches it too
__global__ void __launch_bounds__(256) polyrigid_finish_kernel(const float* __restrict__ partial, int row, int KP, int B, int T, int Bm,
                                                               int K, float* __restrict__ g_M, float* __restrict__ g_src,
                                                               float* __restrict__ g_alpha_range);

// every rectangle of polyrigid_jac's footprint format empty, {W, -1, H, -1}; deform.cu launches it too
__global__ void __launch_bounds__(256) polyrigid_rects_empty_kernel(int* __restrict__ rects, int n, int H, int W);

// deformable (dense displacement field) trilinear render (deform.cu).  Arguments as the polyrigid ones; field: [Bf][g0][g1][g2][4]
// voxel-index displacements, lane 3 zero; g_field: the same layout, zeroed here before the scatter.
int64_t deform_scratch_floats(int B, int64_t N, int W);
cudaError_t launch_deform_fwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, float* out, int B, int64_t N,
                              int W, float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream);
cudaError_t launch_deform_bwd(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* gout, float* g_src,
                              float* g_tgt, float* g_raylen, float* g_field, float* g_alpha_range, float* scratch, int B, int64_t N,
                              int W, float shift, float eps, int n_points, const float* alpha_range, cudaStream_t stream);
// the image's derivative along a field tangent [Bf][g0][g1][g2][4] (voxel units): jv [B][N]; img [B][N] (may be null) = the forward
cudaError_t launch_deform_jvp(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangent, float* img,
                              float* jv, int B, int64_t N, int W, float shift, float eps, int n_points, const float* alpha_range,
                              cudaStream_t stream);
// per-pixel Jacobian along P = 6K field tangents [Bf][g0][g1][g2][P][4] on a full H x W grid: img [B][H*W] (the forward's),
// J [B][K][H*W][6], rects [B][K][4] (set empty first)
cudaError_t launch_deform_jac(const void* vol, const void* packed, int vol_type, VolDims dims, const float* src, const float* tgt,
                              const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangents, int K,
                              float* img, float* J, int* rects, int B, int H, int W, float shift, float eps, int n_points,
                              const float* alpha_range, cudaStream_t stream);
// the forward's transpose in the density: g_vol [D0][D1][D2], zeroed here, += sum over the rays of gout * d out / d V
cudaError_t launch_deform_bproj(VolDims dims, const float* src, const float* tgt, const float* raylen, const float* field, int Bf, int g0,
                                int g1, int g2, const float* gout, float* g_vol, int B, int64_t N, int W, float shift, float eps,
                                int n_points, const float* alpha_range, cudaStream_t stream);

// scaling-and-squaring steps of a stationary velocity field (svf.cu).  field / out / gout / gin: [Bf][g0][g1][g2][4], 16-byte
// aligned; out = one squaring step of field with scale s, gin = its adjoint applied to gout (zeroed on the stream first)
cudaError_t launch_svf_square(const float* field, float* out, int Bf, int g0, int g1, int g2, VolDims dims, float scale,
                              cudaStream_t stream);
cudaError_t launch_svf_square_bwd(const float* field, const float* gout, float* gin, int Bf, int g0, int g1, int g2, VolDims dims,
                                  float scale, cudaStream_t stream);
// tout = the step's tangent along `tangent` (same layout); out (may be null) = the step itself, launch_svf_square's out bit for bit
cudaError_t launch_svf_square_jvp(const float* field, const float* tangent, float* tout, float* out, int Bf, int g0, int g1, int g2,
                                  VolDims dims, float scale, cudaStream_t stream);
// the step's tangents along P tangents at once, node-major [Bf][g0][g1][g2][P][4] in tangents and tout; out (may be null) as above
cudaError_t launch_svf_square_tangents(const float* field, const float* tangents, float* tout, float* out, int Bf, int P, int g0, int g1,
                                       int g2, VolDims dims, float scale, cudaStream_t stream);

}  // namespace b200drr
