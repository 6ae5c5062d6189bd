/*
 * b200drr.h -- C ABI of the H100-native (sm_90a) DRR projector (libb200drr.so).
 *
 * This is the drop-in boundary for DiffDRR's renderer slot.  The reference is pure Python/PyTorch, so
 * the "FFI" a maintainer binds is a ctypes stub (INTEGRATION.md); every entry point below names the
 * reference interface it replaces (paths relative to /root/reference/diffdrr/).
 *
 * Conventions
 *   - All pointers are DEVICE pointers to caller-owned, contiguous, row-major fp32 (unless noted).
 *   - vol is the CT density [D0][D1][D2], axis 2 fastest (reference drr.py:81-85 `density`).
 *   - src [B][3], tgt [B][N][3] are ray end points in VOXEL-INDEX coordinates, raylen [B][N] the ray
 *     lengths in world units: exactly the tensors reference drr.py:201-216 hands to the renderer
 *     (`source (B,1,3)`, `target (B,N,3)`, `img (B,1,N)`).
 *   - Launches are asynchronous on `stream` (a cudaStream_t passed as void*; NULL = legacy default
 *     stream).  No entry point allocates, frees or synchronises, except where stated.
 *   - Return value: 0 on success, a negative B200DRR_E* code for bad arguments, or a positive
 *     cudaError_t value if a launch failed.  Nothing throws; nothing falls back to the CPU.
 *   - reduce: 0 = "sum", 1 = "max" (reference renderers.py:175-183).
 */
#ifndef B200DRR_H
#define B200DRR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200DRR_VERSION 200 /* major*10000 + minor*100 + patch */

#define B200DRR_EINVAL (-1)      /* null pointer / non-positive size / bad enum */
#define B200DRR_EUNSUPPORTED (-2) /* combination the kernels do not implement (documented per call) */

int b200drr_version(void);
/* Human-readable text for a return code of any function below (static storage). */
const char *b200drr_error_string(int code);
/* Number of SMs / compute capability (major*10+minor) of the current device; 0 if there is no device. */
int b200drr_device_sm_count(void);
int b200drr_device_cc(void);

/*
 * Siddon forward: replaces Siddon.forward with mask=None (renderers.py:34-76) = _get_alphas (94-113)
 * + _get_xyzs (143-153) + _get_voxel / grid_sample(mode="nearest") (156-169) + diff*mul + reduce (70-76).
 *   out[b][n] = reduce_j  raylen[b][n] * V[nearest(s + mid_j * (t - s + eps))] * (alpha_{j+1} - alpha_j)
 * over ALL D0+D1+D2+3 plane intersections of the infinite line (no clipping to [0,1]; quirk Q1).
 * align_corners as in grid_sample.  Fast path: reduce=0 && align_corners=0; anything else takes the
 * plane-by-plane general kernel (same results, slower).
 */
int b200drr_siddon_fwd(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps,
                       int reduce, int align_corners, void *stream);

/*
 * Siddon forward for a FULL detector grid: the N = H*W rays of every pose are the row-major detector
 * pixels (n = h*W + w; reference detector.py:126), which lets the kernel map compact pixel tiles onto
 * warps/CTAs for cache locality.  Same result as b200drr_siddon_fwd(reduce=0, align_corners=0).
 * variant: 0 = tuned default -- up to 16 poses of 256^2 rays (volumes >= 384 voxels; smaller ones up to 4) every ray is cut into
 * pieces along its own major axis with a thread per (ray, piece), beyond that the volume is cut into 16-plane slabs that the poses
 * of the batch share through L2 (DESIGN.md 4.1 / 4.1c).  The other ids run the same kernels for benchmarking, whatever the batch
 * size: 46 / 47 / 15 = the slab-major kernel with 16- / 24- / 32-plane slabs, 100+K (K = 1..64) = K major-axis pieces.  Any other
 * id returns cudaErrorInvalidValue.
 */
int b200drr_siddon_fwd_grid(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                            const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps,
                            int variant, void *stream);

/*
 * Siddon backward: replaces the autograd graph of Siddon.forward (sum-backward, diff-backward,
 * sort-backward, grid_sampler_3d_backward; SURVEY.md 8a-G) with one closed-form pass.
 *   gout [B][N] = dLoss/dout.
 *   g_src [B][3]        overwritten (zero-filled inside, then accumulated)      -- may be NULL
 *   g_tgt [B][N][3]     overwritten                                             -- may be NULL
 *   g_raylen [B][N]     overwritten (zeros when stop_grad)                      -- may be NULL
 *   g_vol [D0][D1][D2]  ACCUMULATED into with red.global.add (caller zero-fills); NULL = not wanted;
 *                       ignored when stop_grad
 * stop_grad != 0 restates stop_gradients_through_grid_sample=True (renderers.py:63-65).
 * Only reduce="sum", align_corners=0 (B200DRR_EUNSUPPORTED otherwise).
 */
int b200drr_siddon_bwd(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                       float *g_vol, int B, int64_t N, float voxel_shift, float eps, int stop_grad,
                       int align_corners, void *stream);

/*
 * Siddon backward for a FULL detector grid (see b200drr_siddon_fwd_grid): same outputs and conventions as
 * b200drr_siddon_bwd (g_src / g_tgt / g_raylen overwritten, g_vol accumulated into), computed slab-major with
 * red.global.add partial sums.  align_corners=0 only.  variant: 0 (64-plane slabs); any other id returns cudaErrorInvalidValue.
 */
int b200drr_siddon_bwd_grid(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                            const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                            float *g_vol, int B, int H, int W, float voxel_shift, float eps, int stop_grad,
                            int variant, void *stream);

/*
 * "Pose-in" Siddon: the rays of the full H x W detector grid are generated inside the kernel from two 3x4 matrices
 * per pose, replacing Detector.forward (detector.py:144-154) + the ray-length / affine_inverse lines of DRR.render
 * (drr.py:201-205) + Siddon.forward, so no (B, N, 3) tensor exists in HBM:
 *   target_voxel(h, w) = G[b]  . (cols[w], rows[h], 1, 1)      G  = affine_inverse . extrinsic . reorient . calibration
 *   raylen(h, w)       = |Wd[b] . (cols[w], rows[h], 1, 1)|     Wd = extrinsic . reorient . calibration, source subtracted
 *   src [B][3] = source in voxel coordinates; rows [H] / cols [W] = canonical detector coordinates (detector.py:114-126)
 * out [B][H*W].  Same line integrals as b200drr_siddon_fwd(reduce=0, align_corners=0) on those rays.
 */
int b200drr_siddon_fwd_pose(const float *vol, int D0, int D1, int D2, const float *src, const float *G, const float *Wd,
                            const float *rows, const float *cols, float *out, int B, int H, int W, float voxel_shift,
                            float eps, void *stream);

/*
 * Backward of b200drr_siddon_fwd_pose: g_src [B][3], g_G [B][3][4], g_Wd [B][3][4] overwritten; g_vol accumulated into
 * (NULL = not wanted).  ws_tgt [B][H*W][3] and ws_len [B][H*W] are caller-provided scratch (per-ray gradients before
 * they are reduced to the matrices).  stop_grad as in b200drr_siddon_bwd.
 */
int b200drr_siddon_bwd_pose(const float *vol, int D0, int D1, int D2, const float *src, const float *G, const float *Wd,
                            const float *rows, const float *cols, const float *gout, float *g_src, float *g_G,
                            float *g_Wd, float *g_vol, float *ws_tgt, float *ws_len, int B, int H, int W,
                            float voxel_shift, float eps, int stop_grad, void *stream);

/*
 * Siddon forward WITH per-ray sensitivities (the training-step fast path).  Every pixel depends on ONE ray, so the whole
 * Jacobian of Siddon.forward (renderers.py:40-86) w.r.t. the ray end points is 6 numbers per ray, and the crossing
 * coefficients of the closed-form backward (SURVEY.md 8a-G) do not depend on the incoming gradient: ONE walk yields
 *   out  [B][H*W]     the same line integrals as b200drr_siddon_fwd_grid
 *   sens [B][H*W][8]  { dI/dtgt0, dI/dtgt1, dI/dtgt2, S = out/raylen, dI/dsrc0, dI/dsrc1, dI/dsrc2, 0 }
 * and autograd's backward (what torch derives for renderers.py:40-86 given g = dLoss/dout) is the elementwise
 * b200drr_siddon_bwd_sens below.  Replaces a forward walk + a backward walk by one.  No volume gradient on this path
 * (use b200drr_siddon_bwd_grid when the volume requires grad).  variant 0 = tuned default: the brick-major kernel (id 42) when
 * the shape allows it -- at least 4 poses, >= 2048 bricks of 24x32x32 voxels, sparse rays (H*W <= half the voxels of a volume
 * cross-section), D2 % 4 == 0, H, W in [2, 2048], 16-byte aligned vol and sens -- else major-axis pieces up to 6 poses of
 * 256^2 rays, 16-plane slabs beyond.  b200drr_siddon_fwd_sens_pose follows the same rule.  The other ids run the same kernels for
 * benchmarking, whatever the batch size: 41 / 40 / 39 / 38 / 37 / 35 / 33 / 36 / 34 = the slab-major kernel with 16- / 24- / 32- /
 * 48- / 64- / 96- / 128- / 256- / 512-plane slabs (41 = the default's slab height); 42 = the brick-major kernel (TMA-staged
 * 24x32x32 bricks, the slab kernels' sensitivities walk per (ray, brick); ~20 B per ray of scratch from a stream-ordered memory
 * pool of the library that keeps its memory between calls; cudaErrorNotSupported outside the brick kernel's range); 100+K
 * (K = 1..64) = K major-axis pieces.  Any other id returns cudaErrorInvalidValue.
 */
int b200drr_siddon_fwd_sens(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                            const float *raylen, float *out, float *sens, int B, int64_t N, float voxel_shift, float eps,
                            void *stream); /* arbitrary ray sets (sub-sampled / patched rays); same out / sens layout */
int b200drr_siddon_fwd_sens_grid(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                                 const float *raylen, float *out, float *sens, int B, int H, int W, float voxel_shift,
                                 float eps, int variant, void *stream);

/* g_tgt [B][N][3] = g * dI/dtgt, g_raylen [B][N] = g * S (0 when stop_grad), g_src [B][3] = sum_n g * dI/dsrc;
 * any of the three may be NULL. */
int b200drr_siddon_bwd_sens(const float *sens, const float *gout, float *g_src, float *g_tgt, float *g_raylen, int B,
                            int64_t N, int stop_grad, void *stream);

/* Pose-in forms (rays generated in-kernel as in b200drr_siddon_fwd_pose; gradients reduced to the 3x4 matrices). */
int b200drr_siddon_fwd_sens_pose(const float *vol, int D0, int D1, int D2, const float *src, const float *G,
                                 const float *Wd, const float *rows, const float *cols, float *out, float *sens, int B,
                                 int H, int W, float voxel_shift, float eps, void *stream);
int b200drr_siddon_bwd_sens_pose(const float *sens, const float *gout, const float *Wd, const float *rows,
                                 const float *cols, float *g_src, float *g_G, float *g_Wd, int B, int H, int W,
                                 int stop_grad, void *stream);

/*
 * Per-pose algebra either side of the pose-in entry points, one thread per pose (replaces ~95 tiny ATen kernels per
 * training step; everything is [B] x a few floats):
 *   b200drr_euler_pose_fwd: reference pose.py `convert(rot, xyz, parameterization="euler_angles", convention)`:
 *     R = R_c0(a0) R_c1(a1) R_c2(a2) (c = 0/1/2 for X/Y/Z; angles = rot * scale, scale = pi/180 for degrees=True),
 *     P [B][4][4] = [[R, R.xyz], [0 0 0 1]].   _bwd: gP -> g_rot [B][3], g_xyz [B][3] (either may be NULL).
 *   b200drr_pose_rays_fwd: detector.py:144-154 + drr.py:201-205 collapsed into the inputs of b200drr_siddon_fwd_pose:
 *     T = P.Q, G = Ainv.T (rows 0..2), src = Ainv.(P.r), Wd = [T[:3,:3] | T[:3,3] - (P.r)[:3]] with
 *     Q [4][4] = reorient . calibration, r [4] = reorient[:, 3], Ainv [4][4] = affine_inverse (all row-major, device).
 *     _bwd: (g_src, g_G, g_Wd) -> gP [B][4][4].
 */
int b200drr_euler_pose_fwd(const float *rot, const float *xyz, int c0, int c1, int c2, float scale, float *P, int B,
                           void *stream);
int b200drr_euler_pose_bwd(const float *rot, const float *xyz, int c0, int c1, int c2, float scale, const float *gP,
                           float *g_rot, float *g_xyz, int B, void *stream);
int b200drr_pose_rays_fwd(const float *P, const float *Q, const float *r, const float *Ainv, float *src, float *G,
                          float *Wd, int B, void *stream);
int b200drr_pose_rays_bwd(const float *Q, const float *r, const float *Ainv, const float *g_src, const float *g_G,
                          const float *g_Wd, float *gP, int B, void *stream);

/*
 * Trilinear forward: replaces Trilinear.forward with mask=None (renderers.py:205-240) for a given
 * sampling range.  alpha_range is a DEVICE pointer to {alphamin, alphamax} (so that the range computed
 * on the device by _get_alpha_minmax, renderers.py:124-140,221-223, needs no host round trip).
 *   out[b][n] = reduce_m raylen * tri(V, s + alpha_m (t - s + eps)) * step,
 *   alpha_m = linspace(0,1,n_points)[m] * (amax - amin) + amin,  step = (amax - amin)/(n_points - 1)
 */
int b200drr_trilinear_fwd(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                          const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps,
                          int n_points, const float *alpha_range, int reduce, int align_corners, void *stream);

/*
 * Trilinear backward (autograd of Trilinear.forward incl. grid_sampler_3d_backward; SURVEY.md 8a-G).
 * Same output conventions as b200drr_siddon_bwd, plus
 *   g_alpha_range [2]   ACCUMULATED dLoss/d{alphamin, alphamax} (caller zero-fills)  -- may be NULL
 * Only reduce="sum".
 */
int b200drr_trilinear_bwd(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                          const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                          float *g_vol, float *g_alpha_range, int B, int64_t N, float voxel_shift, float eps,
                          int n_points, const float *alpha_range, int align_corners, void *stream);

/*
 * Trilinear forward / backward for a FULL detector grid (n = h*W + w), reduce="sum", align_corners=0: same results
 * as b200drr_trilinear_fwd / _bwd with pixel tiles mapped onto warps/CTAs for cache locality.  variant: 1 (16x16 pixel tiles);
 * any other id returns cudaErrorInvalidValue.
 */
int b200drr_trilinear_fwd_grid(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                               const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps,
                               int n_points, const float *alpha_range, int variant, void *stream);
int b200drr_trilinear_bwd_grid(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                               const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                               float *g_vol, float *g_alpha_range, int B, int H, int W, float voxel_shift, float eps,
                               int n_points, const float *alpha_range, int variant, void *stream);

/*
 * Packed-corner trilinear path.  b200drr_pack_corners writes, for every interpolation cell with base voxel
 * (i0,i1,i2), i in [-1, D-1], its 8 zero-padded corner values contiguously:
 *   packed[(i0+1)][(i1+1)][(i2+1)][c] = V[i0+o0][i1+o1][i2+o2],  c = o0 | o1<<1 | o2<<2
 * into a caller-allocated buffer of b200drr_packed_volume_floats(D0,D1,D2) floats (8x the volume; 32-byte aligned).
 * b200drr_trilinear_fwd_packed / _bwd_packed then read ONE aligned 32-byte cell per sample (the algorithmic byte
 * count) instead of 8 scalar gathers; same results as the *_grid entry points (reduce="sum", align_corners=0).
 * The packed path produces no volume gradient (use b200drr_trilinear_bwd[_grid] when the volume is being optimised)
 * and must be re-packed whenever the volume changes.
 * slab: 0 = one CTA marches whole rays; > 0 = slab-major scheduling over `slab` planes of base voxels along axis 0
 * (the poses of a batch then share the packed cells through L2; partial sums are combined with red.global.add, so
 * results agree with slab = 0 to fp32 round-off).
 */
int64_t b200drr_packed_volume_floats(int D0, int D1, int D2);
int b200drr_pack_corners(const float *vol, int D0, int D1, int D2, float *packed, void *stream);
int b200drr_trilinear_fwd_packed(const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                                 const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps,
                                 int n_points, const float *alpha_range, int slab, void *stream);
int b200drr_trilinear_bwd_packed(const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                                 const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                                 float *g_alpha_range, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                 const float *alpha_range, int slab, void *stream);

/*
 * Trilinear forward WITH per-ray sensitivities from the packed-corner copy (training-step fast path, the twin of
 * b200drr_siddon_fwd_sens_grid): one march yields out [B][H*W] (== b200drr_trilinear_fwd_packed) and
 *   sens [B][H*W][12] = { dI/dtgt[3], out/raylen | dI/dsrc[3], dI/dalphamin | dI/dalphamax, 0, 0, 0 }
 * i.e. everything torch's backward of Trilinear.forward (renderers.py:205-240) needs is linear in g = dLoss/dout, and
 * b200drr_trilinear_bwd_sens applies it: g_tgt [B][N][3], g_raylen [B][N], g_src [B][3] overwritten (NULL = not wanted),
 * g_alpha_range [2] ACCUMULATED INTO (caller zero-fills; NULL = not wanted).  slab as in b200drr_trilinear_fwd_packed.
 */
int b200drr_trilinear_fwd_sens(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                               const float *raylen, float *out, float *sens, int B, int64_t N, int H, int W,
                               float voxel_shift, float eps, int n_points, const float *alpha_range, int align_corners,
                               void *stream); /* from the plain volume: H = W = 0 arbitrary rays, else N == H*W grid tiles */
int b200drr_trilinear_fwd_sens_packed(const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                                      const float *raylen, float *out, float *sens, int B, int H, int W,
                                      float voxel_shift, float eps, int n_points, const float *alpha_range, int slab,
                                      void *stream);
int b200drr_trilinear_bwd_sens(const float *sens, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                               float *g_alpha_range, int B, int64_t N, void *stream);

/*
 * Pose-in forms of the trilinear training path (the twin of b200drr_siddon_fwd_sens_pose; SURVEY.md 8f-2): the rays of the
 * full detector grid are generated in-kernel from src [B][3], G, Wd [B][3][4], rows [H], cols [W]
 * (detector.py:144-154 + drr.py:201-205 collapsed), so neither the (B,N,3) target tensor nor the ray-length image exists.
 *   b200drr_trilinear_alpha_range_pose: the batch-global sampling range of renderers.py:217-222 (`_get_alpha_minmax`,
 *     renderers.py:124-140, min / max over ALL rays): range [2] = {alphamin, alphamax}, arg [2] = the linear ray index
 *     b*H*W + h*W + w attaining each (the host rebuilds the two scalars differentiably from those two rays' pose);
 *     scratch16 = 16 bytes of device scratch.
 *   b200drr_trilinear_fwd_sens_pose: out / sens exactly as b200drr_trilinear_fwd_sens_packed.
 *   b200drr_trilinear_bwd_sens_pose: g_src [B][3], g_G, g_Wd [B][3][4] overwritten; g_alpha_range [2] ACCUMULATED INTO (NULL =
 *     not wanted).
 */
int b200drr_trilinear_alpha_range_pose(int D0, int D1, int D2, const float *src, const float *G, const float *Wd,
                                       const float *rows, const float *cols, float *range, int64_t *arg, void *scratch16,
                                       int B, int H, int W, float voxel_shift, float eps, void *stream);
int b200drr_trilinear_fwd_sens_pose(const float *packed, int D0, int D1, int D2, const float *src, const float *G,
                                    const float *Wd, const float *rows, const float *cols, float *out, float *sens, int B,
                                    int H, int W, float voxel_shift, float eps, int n_points, const float *alpha_range,
                                    int slab, void *stream);
int b200drr_trilinear_bwd_sens_pose(const float *sens, const float *gout, const float *Wd, const float *rows,
                                    const float *cols, float *g_src, float *g_G, float *g_Wd, float *g_alpha_range, int B,
                                    int H, int W, void *stream);

/*
 * Per-pixel pose Jacobians from the sensitivities of a full row-major detector grid (the forward-mode twins of
 * b200drr_siddon_bwd_sens_pose / b200drr_trilinear_bwd_sens_pose).  sens [B][H*W][8] (Siddon) or [B][H*W][12] (Trilinear) from
 * any producer of that layout (*_fwd_sens_pose and their _v16 twins, *_fwd_sens_grid / _sens_packed).  The pose has P
 * parameters (1 <= P <= 16); dsrc [B][P][3], dG [B][P][3][4], dWd [B][P][3][4] are the derivatives of the pose-in inputs src, G,
 * Wd with respect to each of them, and, with p = (cols[w], rows[h], 1, 1) and dl = Wd.p,
 *   J [B][H*W][P] (overwritten) = dI/dtgt . dG_k p + S (dl . dWd_k p) / |dl| + dI/dsrc . dsrc_k
 *                                 [Trilinear: + dI/dalphamin drange[b][0][k] + dI/dalphamax drange[b][1][k]]
 * The ray-length term is dropped when stop_grad != 0, as in b200drr_siddon_bwd_sens_pose.  drange [B][2][P] is the derivative
 * of the batch-global sampling range with respect to pose b's parameters: zero for poses that own neither extreme ray.
 * One thread per pixel; nothing is reduced, so sum_n g_n J[b][n][k] equals the contraction of the *_bwd_sens_pose gradients with
 * tangent k to fp32 round-off.
 */
int b200drr_siddon_jac_sens_pose(const float *sens, const float *dsrc, const float *dG, const float *dWd, const float *Wd,
                                 const float *rows, const float *cols, float *J, int B, int H, int W, int P, int stop_grad,
                                 void *stream);
int b200drr_trilinear_jac_sens_pose(const float *sens, const float *dsrc, const float *dG, const float *dWd, const float *Wd,
                                    const float *rows, const float *cols, const float *drange, float *J, int B, int H, int W,
                                    int P, void *stream);

/*
 * Piecewise-rigid renders (DESIGN.md 6f): every labelled structure of the CT under its own pose, in one launch.
 *   b200drr_label_boxes: one pass over the label volume labels [D0][D1][D2] (uint8) -> boxes [256][6] int32 (overwritten), the
 *     voxel-index box {lo0, lo1, lo2, hi0, hi1, hi2} = [lo, hi) of every label 0..255; an absent label gets lo > hi.
 *   b200drr_siddon_fwd_sens_structures: S slots per pose.  Slot s of pose b renders the voxels whose label l has
 *     slot_of_label[l] == s (slot_of_label [256] int32, -1 = no slot) with the pose-in rays of src [B*S][3], G, Wd [B*S][3][4]
 *     (index b*S + s; rows [H], cols [W] as in b200drr_siddon_fwd_pose), walking only the box box[s] ([S][6] as above; it must
 *     contain every voxel of the slot's labels).  out [B][S][H*W] and sens [B][S][H*W][8] (layout of b200drr_siddon_fwd_sens_pose,
 *     so b200drr_siddon_bwd_sens_pose with batch B*S is the backward) are overwritten; sens = NULL renders the image only.
 *     Equal, to fp32 round-off, to b200drr_siddon_fwd_sens_pose of the density times (label in slot s).  Pixels outside the
 *     detector rectangle that covers the projection of box[s] (one-pixel margin; the whole detector when the box reaches the
 *     source plane) are written as zeros without a walk.  No atomics on the outputs.  1 <= S <= 256, B*S <= 65535.
 */
int b200drr_label_boxes(const uint8_t *labels, int D0, int D1, int D2, int32_t *boxes, void *stream);
int b200drr_siddon_fwd_sens_structures(const float *vol, const uint8_t *labels, int D0, int D1, int D2, const float *src,
                                       const float *G, const float *Wd, const float *rows, const float *cols,
                                       const int32_t *slot_of_label, const int32_t *box, float *out, float *sens, int B, int S,
                                       int H, int W, float voxel_shift, float eps, void *stream);

/*
 * mask_to_channels forward (reference renderers.py:77-89 and 242-252): `mask` is the label volume [D0][D1][D2] stored
 * as fp32 (as DRR registers it, drr.py:86-91); every segment / sample contributes to channel label(voxel), sampled
 * nearest with zero padding.  out [B][C][N] is overwritten.  Siddon: reduce="sum", align_corners=0.
 */
int b200drr_siddon_fwd_mask(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                            const float *tgt, const float *raylen, float *out, int B, int64_t N, int C,
                            float voxel_shift, float eps, void *stream);
int b200drr_trilinear_fwd_mask(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                               const float *tgt, const float *raylen, float *out, int B, int64_t N, int C,
                               float voxel_shift, float eps, int n_points, const float *alpha_range, int align_corners,
                               void *stream);
/* The same for the FULL row-major detector grid (N = H*W): threads are mapped to pixel tiles of 8 x 4 warp bundles so that
 * neighbouring rays gather neighbouring voxels and labels; Siddon additionally runs slab-major over 32-plane slabs of the
 * density AND label volumes (label runs flushed per (ray, slab) with red.global.add: results agree to fp32 round-off). */
int b200drr_siddon_fwd_mask_grid(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                                 const float *tgt, const float *raylen, float *out, int B, int H, int W, int C,
                                 float voxel_shift, float eps, void *stream);
int b200drr_trilinear_fwd_mask_grid(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                                    const float *tgt, const float *raylen, float *out, int B, int H, int W, int C,
                                    float voxel_shift, float eps, int n_points, const float *alpha_range,
                                    int align_corners, void *stream);

/*
 * Backward for the renderer options outside the fast kernels (reference renderers.py:175-183 `reduce`, :40/:161
 * align_corners): Siddon with reducefn="max" (reduce = 1: the first maximal segment carries the whole gradient, as
 * torch.max does) and/or align_corners=1, through the plane-by-plane general walk; Trilinear with reducefn="max" (first
 * maximal sample).  Output conventions of b200drr_siddon_bwd / b200drr_trilinear_bwd.
 */
int b200drr_siddon_bwd_general(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                               const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                               float *g_vol, int B, int64_t N, float voxel_shift, float eps, int stop_grad, int reduce,
                               int align_corners, int mode, void *stream);
/* General walk with the Siddon sampling mode selectable (reference renderers.py:18,66): mode 0 = "nearest" (same result as
 * b200drr_siddon_fwd), mode 1 = "bilinear" = trilinear interpolation at the segment midpoints.  The backward above takes
 * the same `mode` (bilinear: reduce = 0 only, B200DRR_EUNSUPPORTED otherwise; stop_grad then drops the interpolant's
 * gradient terms exactly like stop_gradients_through_grid_sample). */
int b200drr_siddon_fwd_general(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                               const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps, int reduce,
                               int align_corners, int mode, void *stream);
int b200drr_trilinear_bwd_max(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                              const float *raylen, const float *gout, float *g_src, float *g_tgt, float *g_raylen,
                              float *g_vol, float *g_alpha_range, int B, int64_t N, float voxel_shift, float eps,
                              int n_points, const float *alpha_range, int align_corners, void *stream);

/*
 * mask_to_channels backward = what autograd derives for the scatter_add_ routing above: gout [B][C][N]; the segment /
 * sample routed to channel c carries gout[b][c][n], otherwise the closed forms of b200drr_siddon_bwd /
 * b200drr_trilinear_bwd.  Output conventions as there (g_src/g_tgt/g_raylen overwritten, g_vol and g_alpha_range
 * accumulated into, any may be NULL).
 */
int b200drr_siddon_bwd_mask(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                            const float *tgt, const float *raylen, const float *gout, float *g_src, float *g_tgt,
                            float *g_raylen, float *g_vol, int B, int64_t N, int C, float voxel_shift, float eps,
                            int stop_grad, void *stream);
int b200drr_trilinear_bwd_mask(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                               const float *tgt, const float *raylen, const float *gout, float *g_src, float *g_tgt,
                               float *g_raylen, float *g_vol, float *g_alpha_range, int B, int64_t N, int C,
                               float voxel_shift, float eps, int n_points, const float *alpha_range, int align_corners,
                               void *stream);
/* Full row-major detector grid (N = H*W): tile-ordered threads, otherwise identical to the two entries above. */
int b200drr_siddon_bwd_mask_grid(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                                 const float *tgt, const float *raylen, const float *gout, float *g_src, float *g_tgt,
                                 float *g_raylen, float *g_vol, int B, int H, int W, int C, float voxel_shift, float eps,
                                 int stop_grad, void *stream);
int b200drr_trilinear_bwd_mask_grid(const float *vol, const float *mask, int D0, int D1, int D2, const float *src,
                                    const float *tgt, const float *raylen, const float *gout, float *g_src, float *g_tgt,
                                    float *g_raylen, float *g_vol, float *g_alpha_range, int B, int H, int W, int C,
                                    float voxel_shift, float eps, int n_points, const float *alpha_range,
                                    int align_corners, void *stream);

/*
 * Double precision.  The reference reaches fp64 through `drr.to(torch.float64)` (drr.py:75): these entry points take fp64
 * device pointers with the same meaning as their fp32 namesakes (b200drr_siddon_fwd / _bwd, b200drr_trilinear_fwd / _bwd)
 * and restate renderers.py:34-76 / 205-240 literally, one thread per ray (accuracy path: no tiling, no packed copy).
 * reduce = 1 ("max") is forward-only; Siddon is mode="nearest"; g_src is overwritten, g_vol / g_alpha_range are
 * ACCUMULATED into (caller zero-fills), NULL outputs are skipped.
 */
int b200drr_siddon_fwd_f64(const double *vol, int D0, int D1, int D2, const double *src, const double *tgt,
                           const double *raylen, double *out, int B, int64_t N, double voxel_shift, double eps, int reduce,
                           int align_corners, void *stream);
int b200drr_siddon_bwd_f64(const double *vol, int D0, int D1, int D2, const double *src, const double *tgt,
                           const double *raylen, const double *gout, double *g_src, double *g_tgt, double *g_raylen,
                           double *g_vol, int B, int64_t N, double voxel_shift, double eps, int stop_grad, int align_corners,
                           void *stream);
int b200drr_trilinear_fwd_f64(const double *vol, int D0, int D1, int D2, const double *src, const double *tgt,
                              const double *raylen, double *out, int B, int64_t N, double voxel_shift, double eps,
                              int n_points, const double *alpha_range, int reduce, int align_corners, void *stream);
int b200drr_trilinear_bwd_f64(const double *vol, int D0, int D1, int D2, const double *src, const double *tgt,
                              const double *raylen, const double *gout, double *g_src, double *g_tgt, double *g_raylen,
                              double *g_vol, double *g_alpha_range, int B, int64_t N, double voxel_shift, double eps,
                              int n_points, const double *alpha_range, int align_corners, void *stream);

/*
 * Un-reduced renders for a CALLABLE `reducefn` (renderers.py:175-183 calls `reducefn(img)` on the per-segment tensor):
 *   kind = 0 (Siddon):    out [B][N][D0+D1+D2+2] = raylen * v_j * (alpha_{j+1} - alpha_j) for every pair of consecutive plane
 *                         alphas in the reference's sorted order (renderers.py:70-74 before `reduce`);
 *   kind = 1 (trilinear): out [B][N][n_points]   = raylen * sample_m * step (renderers.py:231-236 before `reduce`).
 * b200drr_segments_bwd takes the upstream gradient of that tensor (gseg, same shape) and returns the same gradients as
 * b200drr_siddon_bwd / b200drr_trilinear_bwd (g_src overwritten; g_vol, g_alpha_range ACCUMULATED into; NULL = skipped).
 * is_f64 selects double pointers (and the fp64 kernels) instead of float.  Reference-literal, one thread per ray.
 */
int b200drr_segments_fwd(int kind, int is_f64, const void *vol, int D0, int D1, int D2, const void *src, const void *tgt,
                         const void *raylen, void *out, int B, int64_t N, double voxel_shift, double eps, int n_points,
                         const void *alpha_range, int align_corners, void *stream);
int b200drr_segments_bwd(int kind, int is_f64, const void *vol, int D0, int D1, int D2, const void *src, const void *tgt,
                         const void *raylen, const void *gseg, void *g_src, void *g_tgt, void *g_raylen, void *g_vol,
                         void *g_alpha_range, int B, int64_t N, double voxel_shift, double eps, int n_points,
                         const void *alpha_range, int stop_grad, int align_corners, void *stream);

/*
 * Siddon forward / forward-with-sensitivities for ARBITRARY ray sets that the caller has put in a LOCALITY ORDER
 * (sub-sampled detectors detector.py:134-137, patches drr.py:217-225, user rays): consecutive groups of 32 rays should be
 * spatial neighbours (the module sorts by the Morton code of the target points).  Thread i walks ray i, so a warp's
 * gathers share cache lines like the 8x4-pixel bundles of the *_grid kernels, and the volume is walked slab-major across
 * the batch.  Same results (fp32 round-off: partial sums are combined with red.global.add) and same argument meaning as
 * b200drr_siddon_fwd(reduce=0, align_corners=0) / b200drr_siddon_fwd_sens; any order is CORRECT, a poor one is merely slow.
 */
int b200drr_siddon_fwd_sorted(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                              const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps, void *stream);
int b200drr_siddon_fwd_sens_sorted(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                                   const float *raylen, float *out, float *sens, int B, int64_t N, float voxel_shift,
                                   float eps, void *stream);

/*
 * Brick-major Siddon forward for a FULL detector grid (same result as b200drr_siddon_fwd_grid; replaces
 * renderers.py:94-113 + 156-169): the volume is cut into 24x32x32-voxel bricks, each staged in shared memory by one TMA
 * box copy (cp.async.bulk.tensor.3d behind an mbarrier pipeline) and integrated for every ray of every pose of the
 * batch that crosses it -- L2->SM traffic falls below the algorithmic bytes because a staged voxel serves all poses.
 * Pays off for batches (B >= ~4); needs D2 % 4 == 0, vol 16-byte aligned, 2 <= H, W <= 2048 (B200DRR_EUNSUPPORTED otherwise).
 *   rays: either (tgt, raylen) as in b200drr_siddon_fwd_grid with G = Wd = rows = cols = NULL, or generated in-kernel from
 *   (G, Wd, rows, cols) as in b200drr_siddon_fwd_pose with tgt = raylen = NULL.
 *   workspace: caller-owned scratch of b200drr_siddon_brick_workspace_bytes(B, H, W) bytes, 256-byte aligned (ray table
 *   {1/d, sum|d|, d, L} = 32 B per ray, per-pose detector geometry, the brick work counter); contents are don't-care.
 *   variant: 0 (the production brick shape; the brick_subset form below as well); any other id returns cudaErrorInvalidValue.
 */
int64_t b200drr_siddon_brick_workspace_bytes(int B, int H, int W);
int b200drr_siddon_fwd_brick(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                             const float *raylen, const float *G, const float *Wd, const float *rows, const float *cols,
                             float *out, void *workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift,
                             float eps, int variant, void *stream);

/*
 * Volume gradient of the full-grid Siddon render (what autograd gives for reference renderers.py:40-76 w.r.t. `volume`; the
 * reconstruction path) through the SAME brick-major kernel run as a scatter: the staged brick starts as zeros, every (ray,
 * brick) walk adds gout * raylen * chord length into it in shared memory, and the finished brick leaves with one TMA store --
 * every voxel belongs to exactly one brick, so there are no global atomics.  g_vol [D0][D1][D2] (16-byte aligned) is
 * OVERWRITTEN (unlike the g_vol of b200drr_siddon_bwd[_grid], which is accumulated into).  gout [B][H*W]; rays and workspace as
 * in b200drr_siddon_fwd_brick.  Pose gradients are not produced here (b200drr_siddon_bwd_grid with g_vol = NULL, or the
 * sensitivities of b200drr_siddon_fwd_sens_grid).
 */
int b200drr_siddon_bwd_vol_brick(const float *gout, int D0, int D1, int D2, const float *src, const float *tgt,
                                 const float *raylen, const float *G, const float *Wd, const float *rows, const float *cols,
                                 float *g_vol, void *workspace, int64_t workspace_bytes, int B, int H, int W,
                                 float voxel_shift, float eps, void *stream);

/*
 * The same brick-major kernel for a ray SUBSET of the H x W detector grid (p_subsample, detector.py:134-137): tgt, raylen and
 * out are (B, Nsub) arrays in the caller's order; pix_index [H*W] int32 maps a detector pixel (h*W + w) to its position in that
 * order (-1 = pixel not rendered); corners [B][3][3] are the voxel-space targets of the FULL grid's pixels (0,0), (0,W-1),
 * (H-1,0) of every pose (the kernel derives each pose's detector plane from them).  Shared-memory gathers do not care how far
 * apart the rays are, so the per-ray cost stays close to the full grid's, where the slab-major gather loses its sector sharing.
 * workspace: b200drr_siddon_brick_workspace_bytes(B, 1, Nsub) bytes.
 */
int b200drr_siddon_fwd_brick_subset(const float *vol, int D0, int D1, int D2, const float *src, const float *tgt,
                                    const float *raylen, const int32_t *pix_index, const float *corners, float *out,
                                    void *workspace, int64_t workspace_bytes, int B, int H, int W, int64_t Nsub,
                                    float voxel_shift, float eps, int variant, void *stream);

/*
 * Per-ray voxel-visit count of the Siddon walk (number of voxels the line crosses inside the volume),
 * the unit of the ALGORITHMIC byte count used for roofline accounting (SURVEY.md 8d): visits [B][N]
 * int32.  Measurement helper; not part of the reference surface.
 */
int b200drr_siddon_visits(int D0, int D1, int D2, const float *src, const float *tgt, int32_t *visits, int B,
                          int64_t N, float voxel_shift, float eps, void *stream);

/*
 * Image similarity of the 2D/3D registration loop: zero-normalised cross correlation of two image stacks and its gradient
 * (reference diffdrr/metrics.py:21-44, NormalizedCrossCorrelation2d.forward / .norm with patch_size = None; eps as in the
 * reference's constructor).  x1, x2 [B][C][N] (N = H*W pixels, row-major, device):
 *   norm(x) = (x - mean_N x) / sqrt(var_N x + eps) (population variance),  score[b] = mean_{c,n} norm(x1) norm(x2).
 * b200drr_ncc_fwd: one pass over both stacks (five moments per image pair, accumulated in double, fixed summation order:
 *   deterministic), then score [B] and stats [B*C][8] = {mean1, 1/std1, mean2, 1/std2, ncc of the pair, 0, 0, 0}, the only thing
 *   the backward pass keeps besides the images.  workspace: b200drr_ncc_workspace_bytes(B, C, N) bytes, 8-byte aligned.
 * b200drr_ncc_bwd: gscore [B] -> g_x1, g_x2 [B][C][N] (either may be NULL) by the closed form
 *   d score[b] / d x2[b,c,n] = (n1 - n2 * ncc_bc) / (C N std2)   (and symmetrically for x1) -- one elementwise pass instead of the
 *   ~25 launches of the reference's autograd graph.  B*C <= 65535.
 */
int64_t b200drr_ncc_workspace_bytes(int B, int C, int64_t N);
int b200drr_ncc_fwd(const float *x1, const float *x2, int B, int C, int64_t N, float eps, void *workspace, float *stats,
                    float *score, void *stream);
int b200drr_ncc_bwd(const float *x1, const float *x2, const float *stats, const float *gscore, float *g_x1, float *g_x2, int B,
                    int C, int64_t N, void *stream);

/*
 * Patch-wise (local) NCC (reference diffdrr/metrics.py:16-44, NormalizedCrossCorrelation2d(patch_size = p)).  x1, x2
 * [B][C][H][W] (device, contiguous), 1 <= p <= min(H, W), B*C <= 65535.  Every stride-1 p x p window of every channel is
 * normalised on its own (mean, population variance + eps); with H' = H-p+1, W' = W-p+1:
 *   score[b] = mean over the C*H'*W' windows of  cov_w / sqrt((var1_w + eps)(var2_w + eps)).
 * b200drr_local_ncc_fwd: box sums of the five moments (vertical p-row sums, then horizontal p-column sums; double), written as
 *   stats [B*C][5][H'][W'] = {mean1, 1/std1, mean2, 1/std2, ncc of the window} for the backward pass, and score [B]; the
 *   partial scores are summed in a fixed order (deterministic).
 * b200drr_local_ncc_bwd: gscore [B] -> g_x1, g_x2 [B][C][H][W] (either may be NULL) by the closed form
 *   d score[b] / d x2_q = gscore[b] / (C H' W' p^2) * sum over the windows w containing q of r2 ((x1_q - mu1) r1 - (x2_q - mu2) r2 L)
 *   (symmetrically for x1), evaluated as adjoint box sums of per-window maps.
 * workspace: b200drr_local_ncc_workspace_bytes(B, C, H, W, p) bytes, 8-byte aligned, for either call (0 for bad arguments).
 */
int64_t b200drr_local_ncc_workspace_bytes(int B, int C, int H, int W, int p);
int b200drr_local_ncc_fwd(const float *x1, const float *x2, int B, int C, int H, int W, int p, float eps, void *workspace,
                          float *stats, float *score, void *stream);
int b200drr_local_ncc_bwd(const float *x1, const float *x2, const float *stats, const float *gscore, float *g_x1, float *g_x2, int B,
                          int C, int H, int W, int p, void *workspace, void *stream);

/*
 * Gauss-Newton normal equations of the global (p = 0) or patch-wise (1 <= p <= min(H, W)) NCC between a rendered stack x and a
 * target t, both [B][C][H][W] (device, contiguous), for the pose Jacobian J: fp32, pixel n = h*W + w of parameter k of (pose b,
 * channel c) at J[b*sJb + c*sJc + k*sJk + n*sJn] (element strides >= 0: DRR.jacobian's (B, H*W, P) is {H*W*P, 0, 1, P}, the blur +
 * Sobel of its planes (B, P, 2, H, W) is {2*P*H*W, H*W, 2*H*W, 1}).  1 <= P <= 16, B*C <= 65535, eps >= 0.
 * Every window w (the whole H x W image when p = 0) of every channel is z-normalised as in b200drr_local_ncc_fwd (mean,
 * population variance + eps, clamped at 0); with the window's residual r = z(x) - z(t) and its Jacobian Jz (J through z(x)):
 *   A [B][P][P] += weight * sum_{c,w} sum_q Jz_q Jz_q^T,   g [B][P] += weight * sum_{c,w} sum_q Jz_q r_q   (float64; the caller
 *   zero-fills, so several calls, e.g. one per scale of a multiscale loss, accumulate into one system).
 * Evaluated from box sums of the 5 + 3P channels {x, x^2, t, t^2, x t, J, x J, t J} and an adjoint box sum of 1/(var + eps), all in
 * double, in a fixed order (no atomics: repeated calls give identical bits); nothing of size windows x pixels or pixels x P^2 is
 * formed.  workspace: b200drr_ncc_normal_workspace_bytes(B, C, H, W, p, P) bytes, 8-byte aligned (0 for bad arguments).
 */
int64_t b200drr_ncc_normal_workspace_bytes(int B, int C, int H, int W, int p, int P);
int b200drr_ncc_normal(const float *x, const float *t, const float *J, int64_t sJb, int64_t sJc, int64_t sJk, int64_t sJn, int B,
                       int C, int H, int W, int p, int P, double eps, double weight, void *workspace, double *A, double *g,
                       void *stream);

/*
 * Global-NCC normal equations of a piecewise-rigid composite image, block by block (DESIGN.md 6g).
 *   b200drr_structure_footprints: per (pose b, slot s) of src [B*S][3], G [B*S][3][4] (index b*S + s), rows [H], cols [W] and the
 *     slot boxes box [S][6] (as b200drr_siddon_fwd_sens_structures takes them) -> rects [B*S][4] int32 = {w0, w1, h0, h1}
 *     (inclusive; empty when w0 > w1 or h0 > h1), the pixel rectangle that kernel culls the slot to, or the whole detector when
 *     it walks every pixel.  1 <= S <= 256.
 *   b200drr_ncc_normal_structures: the composite x [B][H][W] (device, contiguous), the target t [t_batch][H][W] (t_batch 1 or B),
 *     and per structure k < K the Jacobian of x with respect to its 6 motion parameters: fp32, pixel n, parameter i of (pose b,
 *     structure k) at J[b*sJb + k*sJs + n*sJn + i*sJk] (element strides >= 0; DRR.structures_jacobian's (B, S, H*W, 6) is
 *     {S*H*W*6, H*W*6, 6, 1}), zero outside rects[b*S + k].  With P = 6K, the global NCC's system of b200drr_ncc_normal (p = 0,
 *     C = 1) is accumulated: A [B][P][P] += weight * sum_q Jz_q Jz_q^T, g [B][P] += weight * sum_q Jz_q r_q (float64).  The image
 *     moments run over the whole image, those of structure k over rects k, and block (j, k) of sum J J^T over the intersection of
 *     rects j and k only.  Fixed-order double sums, no atomics: repeated calls give identical bits.  1 <= K <= 255, K <= S <= 256,
 *     B <= 65535, eps >= 0.  workspace: b200drr_ncc_normal_structures_workspace_bytes(B, K, H, W) bytes, 8-byte aligned (0 for
 *     bad arguments); it holds no pixels x P^2 or pairs x pixels array.
 */
int b200drr_structure_footprints(const float *src, const float *G, const float *rows, const float *cols, const int32_t *box,
                                 int32_t *rects, int B, int S, int H, int W, float voxel_shift, void *stream);
int64_t b200drr_ncc_normal_structures_workspace_bytes(int B, int K, int H, int W);
int b200drr_ncc_normal_structures(const float *x, const float *t, int t_batch, const float *J, int64_t sJb, int64_t sJs, int64_t sJn,
                                  int64_t sJk, const int32_t *rects, int B, int K, int S, int H, int W, double eps, double weight,
                                  void *workspace, double *A, double *g, void *stream);

/*
 * Gaussian blur + Sobel gradients of one-channel images (reference diffdrr/metrics.py:69-93, the Sobel front end of
 * GradientNormalizedCrossCorrelation2d).  x [B][H][W] (device) -> out [B][2][H][W]:
 *   blur   separable, 1-D weights [ksize] (device; torchvision's normalised Gaussian, ksize odd; ksize = 1 with weight 1 is no
 *          blur) after reflect padding of ksize/2, which must be < H and < W;
 *   Sobel  3x3 cross-correlation with zero padding, channel 0 Gx = [[1,0,-1],[2,0,-2],[1,0,-1]], channel 1 Gy = Gx transposed.
 * b200drr_sobel_fwd: one launch.  b200drr_sobel_bwd: gout [B][2][H][W] -> g_x [B][H][W], the exact adjoint (gradient that
 * lands on reflected positions folds back onto the mirrored pixels).  workspace: b200drr_sobel_workspace_bytes(B, H, W) bytes.
 * B <= 65535; ksize is also bounded by the shared-memory tiles (ksize/2 up to about 800).
 */
int64_t b200drr_sobel_workspace_bytes(int B, int H, int W);
int b200drr_sobel_fwd(const float *x, float *out, int B, int H, int W, const float *weights, int ksize, void *stream);
int b200drr_sobel_bwd(const float *gout, float *g_x, int B, int H, int W, const float *weights, int ksize, void *workspace,
                      void *stream);

/*
 * Mutual information of two one-channel image stacks from Parzen (Gaussian kernel) histograms (reference
 * diffdrr/metrics.py:110-139, MutualInformation over kornia's marginal_pdf / joint_pdf).  x1, x2 [B][N] (N = H*W pixels,
 * device), bins [num_bins] and sigma [1] (device fp32: the module's buffers, read on the device), 2 <= num_bins <= 256,
 * N < 2^31, B <= 65535:
 *   k[n,i] = exp(-0.5 ((x_n - bins_i) / sigma)^2)   (fp32, the reference's op order)
 *   p_i = m_i / (sum m + epsilon) with m_i = mean_n k[n,i];   P = J / (sum J + 1e-10) with J[i,j] = sum_n k1[n,i] k2[n,j]
 *   H1 = -sum p1 log2(p1 + epsilon), H2 likewise, H12 = -sum P log2(P + epsilon)
 *   score[b] = H1 + H2 - H12, or 2 (H1 + H2 - H12) / (H1 + H2) when normalize != 0.
 * b200drr_mi_fwd: 3 launches.  The joint histogram is an FP32 register-tiled contraction over pixel chunks with the kernel
 *   values made in shared memory (never in HBM); the chunk partials are summed in a fixed order in double (deterministic), and
 *   the entropies and the unit gradient maps are computed in double: stats [B][num_bins^2 + 2 num_bins + 4] =
 *   {U [nb][nb], u1 [nb], u2 [nb], H1, H2, H12, score} with U = d score / d J and u = d score / d (pixel sum of k).
 *   workspace: b200drr_mi_workspace_bytes(B, N, num_bins) bytes, 8-byte aligned (about 8 MiB per pose at most; 0 for bad
 *   arguments).  It depends on the current device's SM count: query it on the device that runs the call.
 * b200drr_mi_bwd: gscore [B] -> g_x1, g_x2 [B][N] (either may be NULL; one launch):
 *   d score / d x1_n = gscore[b] sum_i (u1_i + sum_j U[i,j] k2[n,j]) k1[n,i] (-(x1_n - bins_i) / sigma^2), x2 with U^T.
 */
int64_t b200drr_mi_workspace_bytes(int B, int64_t N, int num_bins);
int b200drr_mi_fwd(const float *x1, const float *x2, int B, int64_t N, const float *bins, const float *sigma, int num_bins,
                   double epsilon, int normalize, void *workspace, float *stats, float *score, void *stream);
int b200drr_mi_bwd(const float *x1, const float *x2, const float *bins, const float *sigma, const float *stats, const float *gscore,
                   float *g_x1, float *g_x2, int B, int64_t N, int num_bins, void *stream);

/*
 * 16-bit volumes (DESIGN.md 4.5): twins of the Siddon forward entry points for a volume stored as IEEE binary16
 * (vol_type = B200DRR_VOL_F16) or bfloat16 (B200DRR_VOL_BF16).  Only the voxels are 16 bits: every voxel read is widened to
 * fp32 exactly, and the rays, alphas, lengths, sums, outputs and sensitivities are fp32 as in the fp32 entry points, whose
 * arguments follow vol_type unchanged.  Each twin runs the kernel the fp32 call selects with variant 0 / default options, on the
 * widened voxels, so its results equal the fp32 call on the up-cast volume.  The brick kernels need D2 % 8 == 0 (16-byte TMA
 * strides; D2 % 4 for fp32).  Any other vol_type, a nonzero reduce / align_corners or a null pointer returns B200DRR_EINVAL
 * without touching CUDA; so does a variant other than 0 (the tuning variants are fp32-only).  The backward of these forwards is
 * b200drr_siddon_bwd_sens / _bwd_sens_pose (sensitivities only).
 */
#define B200DRR_VOL_F16 1
#define B200DRR_VOL_BF16 2
int b200drr_siddon_fwd_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                           const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps, int reduce,
                           int align_corners, void *stream);
int b200drr_siddon_fwd_sens_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                const float *raylen, float *out, float *sens, int B, int64_t N, float voxel_shift, float eps,
                                void *stream);
int b200drr_siddon_fwd_sorted_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                  const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps, void *stream);
int b200drr_siddon_fwd_sens_sorted_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                       const float *raylen, float *out, float *sens, int B, int64_t N, float voxel_shift, float eps,
                                       void *stream);
int b200drr_siddon_fwd_grid_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps, int variant,
                                void *stream);
int b200drr_siddon_fwd_sens_grid_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                     const float *raylen, float *out, float *sens, int B, int H, int W, float voxel_shift, float eps,
                                     int variant, void *stream);
int b200drr_siddon_fwd_brick_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                 const float *raylen, const float *G, const float *Wd, const float *rows, const float *cols,
                                 float *out, void *workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift,
                                 float eps, int variant, void *stream);
int b200drr_siddon_fwd_brick_subset_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                        const float *raylen, const int32_t *pix_index, const float *corners, float *out,
                                        void *workspace, int64_t workspace_bytes, int B, int H, int W, int64_t Nsub,
                                        float voxel_shift, float eps, int variant, void *stream);
int b200drr_siddon_fwd_pose_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *G,
                                const float *Wd, const float *rows, const float *cols, float *out, int B, int H, int W,
                                float voxel_shift, float eps, void *stream);
int b200drr_siddon_fwd_sens_pose_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *G,
                                     const float *Wd, const float *rows, const float *cols, float *out, float *sens, int B, int H,
                                     int W, float voxel_shift, float eps, void *stream);
int b200drr_siddon_fwd_sens_structures_v16(const void *vol, int vol_type, const uint8_t *labels, int D0, int D1, int D2,
                                           const float *src, const float *G, const float *Wd, const float *rows, const float *cols,
                                           const int32_t *slot_of_label, const int32_t *box, float *out, float *sens, int B,
                                           int S, int H, int W, float voxel_shift, float eps, void *stream);

/*
 * 16-bit volumes, Trilinear (DESIGN.md 4.5): twins of the trilinear entry points with the same fp32 arguments after vol_type.
 * b200drr_pack_corners_v16 writes the packed-corner copy with the 8 corners of each cell in the volume's own 16-bit type:
 * b200drr_packed_volume_floats(D0, D1, D2) * 2 bytes (16 B per base voxel, 16-byte aligned); the *_packed_v16 / _sens_pose_v16
 * twins read that copy (`packed`) and take the volume's vol_type.  reduce and align_corners must be 0; B200DRR_EINVAL otherwise, for
 * a bad vol_type and for null pointers, without touching CUDA.  fwd_grid_v16 takes the fp32 call's variant (1).
 */
int b200drr_pack_corners_v16(const void *vol, int vol_type, int D0, int D1, int D2, void *packed, void *stream);
int b200drr_trilinear_fwd_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                              const float *raylen, float *out, int B, int64_t N, float voxel_shift, float eps, int n_points,
                              const float *alpha_range, int reduce, int align_corners, void *stream);
int b200drr_trilinear_fwd_grid_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                   const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                   const float *alpha_range, int variant, void *stream);
int b200drr_trilinear_fwd_sens_v16(const void *vol, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                   const float *raylen, float *out, float *sens, int B, int64_t N, int H, int W, float voxel_shift,
                                   float eps, int n_points, const float *alpha_range, int align_corners, void *stream);
int b200drr_trilinear_fwd_packed_v16(const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                                     const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                     const float *alpha_range, int slab, void *stream);
int b200drr_trilinear_fwd_sens_packed_v16(const void *packed, int vol_type, int D0, int D1, int D2, const float *src,
                                          const float *tgt, const float *raylen, float *out, float *sens, int B, int H, int W,
                                          float voxel_shift, float eps, int n_points, const float *alpha_range, int slab,
                                          void *stream);
int b200drr_trilinear_fwd_sens_pose_v16(const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *G,
                                        const float *Wd, const float *rows, const float *cols, float *out, float *sens, int B, int H,
                                        int W, float voxel_shift, float eps, int n_points, const float *alpha_range, int slab,
                                        void *stream);

/*
 * Blended-rigid (skinned) trilinear render (DESIGN.md 6h).  The rays and samples are b200drr_trilinear_fwd's (x_m = s + alpha_m d,
 * alpha_range as there, align_corners = 0, reduce = sum); every sample is pulled back through a linear blend of K affine maps,
 * the rest of the weight on the identity:
 *     y_m = x_m + sum_k w_k(x_m) (M_k [x_m; 1] - x_m),      out = raylen * step * sum_m tri(V, y_m).
 * M [Bm][K][12]: row-major 3 x 4 maps in voxel-index coordinates, Bm = 1 (shared by the poses) or B.  K <= 8
 * (B200DRR_EUNSUPPORTED above).  weights: the PACKED lattice b200drr_polyrigid_pack_weights writes from a (K, g0, g1, g2) fp32
 * lattice: channel-last, K padded with zeros to 4 or 8, b200drr_polyrigid_weight_floats(K, g0, g1, g2) floats, 16-byte aligned.
 * The lattice is sampled trilinearly with the align_corners = False convention over the volume (node i of axis a at voxel
 * coordinate (i + 1/2) D_a / g_a - 1/2) and is zero outside itself.
 * The density is read from `vol` (D0 x D1 x D2) or from its packed-corner copy `packed` (b200drr_pack_corners): exactly one of
 * the two is non-NULL; both give the same bits.  The rays of a pose are N arbitrary rays (H = W = 0) or a full row-major
 * H x W grid (N = H * W), marched in 16 x 8 pixel tiles.  out [B][N] is overwritten.
 *
 * b200drr_polyrigid_bwd: gradients of sum(gout * out), every output OVERWRITTEN and NULL where not wanted: g_src [B][3],
 * g_tgt [B][N][3], g_raylen [B][N], g_M [Bm][K][12], g_alpha_range [2] (the partials w.r.t. alpha_range, as
 * b200drr_trilinear_bwd's).  No weight gradient; the volume gradient is b200drr_polyrigid_bproj's.
 * scratch: b200drr_polyrigid_scratch_floats(B, N, H, W, K) floats;
 * the sums over rays are taken from it in a fixed order, so repeated calls return identical bits.  The library allocates
 * nothing.  The _v16 twins read a 16-bit volume (vol_type as above; `packed` from b200drr_pack_corners_v16) and equal the fp32
 * call on the up-cast volume.
 */
int64_t b200drr_polyrigid_weight_floats(int K, int g0, int g1, int g2);
int b200drr_polyrigid_pack_weights(const float *weights, int K, int g0, int g1, int g2, float *packed, void *stream);
int64_t b200drr_polyrigid_scratch_floats(int B, int64_t N, int H, int W, int K);
int b200drr_polyrigid_fwd(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                          const float *raylen, const float *M, int Bm, int K, const float *weights, int g0, int g1, int g2, float *out,
                          int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float *alpha_range,
                          void *stream);
int b200drr_polyrigid_bwd(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                          const float *raylen, const float *M, int Bm, int K, const float *weights, int g0, int g1, int g2,
                          const float *gout, float *g_src, float *g_tgt, float *g_raylen, float *g_M, float *g_alpha_range,
                          float *scratch, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                          const float *alpha_range, void *stream);
int b200drr_polyrigid_fwd_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src,
                              const float *tgt, const float *raylen, const float *M, int Bm, int K, const float *weights, int g0,
                              int g1, int g2, float *out, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                              const float *alpha_range, void *stream);
int b200drr_polyrigid_bwd_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src,
                              const float *tgt, const float *raylen, const float *M, int Bm, int K, const float *weights, int g0,
                              int g1, int g2, const float *gout, float *g_src, float *g_tgt, float *g_raylen, float *g_M,
                              float *g_alpha_range, float *scratch, int B, int64_t N, int H, int W, float voxel_shift, float eps,
                              int n_points, const float *alpha_range, void *stream);

/*
 * Backprojection through the blended-rigid render (DESIGN.md 6o): the transpose of b200drr_polyrigid_fwd in the density, for
 * reconstruction under known (or jointly fitted) articulated motion.  For a fixed camera and fixed maps the render is linear in V:
 *     out = raylen * step * sum_m tri(V, y_m),      y_m = x_m + sum_k w_k(x_m) (M_k [x_m; 1] - x_m),
 * so the gradient of sum(gout * out) with respect to V is
 *     g_vol[corner] = sum over rays and samples of gout * raylen * step * tri_weight(corner, y_m),
 * over every y_m inside the padded volume.  The samples, the maps, the packed lattice `wpacked` and the range are
 * b200drr_polyrigid_fwd's; no density is read, so there is no volume argument and no _v16 twin.  gout [B][N]; g_vol [D0][D1][D2],
 * OVERWRITTEN: the entry zeroes it on the stream, then every pose (shared or per-pose maps) adds into it with scalar atomics, so
 * it repeats only to fp32 reordering.  A NULL gout or g_vol returns B200DRR_EINVAL, and the geometry, lattice and map checks are
 * b200drr_polyrigid_fwd's (with the same return codes), all before touching CUDA.  The library allocates nothing.
 */
int b200drr_polyrigid_bproj(int D0, int D1, int D2, const float *src, const float *tgt, const float *raylen, const float *M, int Bm,
                            int K, const float *wpacked, int g0, int g1, int g2, const float *gout, float *g_vol, int B, int64_t N,
                            int H, int W, float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);

/*
 * Per-pixel motion Jacobian of the blended-rigid render (DESIGN.md 6j), for Gauss-Newton / Levenberg-Marquardt on the motions.
 * Arguments as b200drr_polyrigid_fwd's, on a full row-major H x W grid only (N = H * W, H, W > 0).  Per pose b, structure k,
 * pixel n and parameter i < 6:
 *     J[b][k][n][i] = raylen * step * sum_e dout/dM_k[e] T[bm][k][i][e],
 * dout/dM_k (e = 4 r + c of the row-major 3 x 4 map) the ray's derivative that b200drr_polyrigid_bwd sums into g_M, and
 * T [Bm][K][6][12] fp32 the tangents dM_k / d xi_ki of the caller's parameters (Bm as for M).  So sum_n gout_n J[b][k][n][.] is
 * g_M : T to fp32 reordering.  Outputs, all OVERWRITTEN: img [B][H*W], b200drr_polyrigid_fwd's out bit for bit; J [B][K][H*W][6];
 * rects [B][K][4] int32 {w0, w1, h0, h1} (inclusive; empty as {W, -1, H, -1}), the bounding rectangle of the pixels whose ray had
 * a sample inside the padded volume with w_k != 0: J[b][k] is zero outside it (the contract of
 * b200drr_ncc_normal_structures, which takes J with strides {K*H*W*6, H*W*6, 6, 1} and rects with S = K).  The entry sets the
 * rects empty on the stream, then grows them with integer atomic min / max, which do not depend on order: every output repeats
 * bit for bit.  A null pointer, H * W = 0 or a bad vol_type returns B200DRR_EINVAL, K > 8 B200DRR_EUNSUPPORTED, without touching
 * CUDA.  The _v16 twin reads a 16-bit volume and equals the fp32 call on the up-cast volume.  The library allocates nothing.
 */
int b200drr_polyrigid_jac(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                          const float *raylen, const float *M, int Bm, int K, const float *weights, int g0, int g1, int g2,
                          const float *T, float *img, float *J, int32_t *rects, int B, int H, int W, float voxel_shift, float eps,
                          int n_points, const float *alpha_range, void *stream);
int b200drr_polyrigid_jac_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src,
                              const float *tgt, const float *raylen, const float *M, int Bm, int K, const float *weights, int g0,
                              int g1, int g2, const float *T, float *img, float *J, int32_t *rects, int B, int H, int W,
                              float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);

/*
 * Deformable trilinear render (DESIGN.md 6i).  The rays and samples are b200drr_trilinear_fwd's; every sample is pulled back
 * through a dense displacement field u given in voxel-index units on a lattice over the volume:
 *     y_m = x_m + u(x_m),      out = raylen * step * sum_m tri(V, y_m).
 * field [Bf][g0][g1][g2][4]: channel-last (u_0, u_1, u_2, 0), Bf = 1 (shared by the poses) or B, 16-byte aligned, fewer than 2^31
 * floats per pose (B200DRR_EUNSUPPORTED otherwise).  The lattice convention is b200drr_polyrigid_fwd's (node i of axis a at voxel
 * coordinate (i + 1/2) D_a / g_a - 1/2, trilinear, zero outside the lattice).  vol / packed, the ray sets and out as there.
 *
 * b200drr_deform_bwd: gradients of sum(gout * out), every output OVERWRITTEN and NULL where not wanted: g_src [B][3],
 * g_tgt [B][N][3], g_raylen [B][N], g_alpha_range [2] (as b200drr_polyrigid_bwd's) and g_field, the field's layout, 16-byte
 * aligned; lane 3 is written 0.  The entry zeroes g_field on the stream and then adds every ray's contribution with vector atomics,
 * so g_field repeats only to fp32 reordering; every other output repeats bit for bit (sums over rays taken from scratch,
 * b200drr_deform_scratch_floats(B, N, H, W) floats, in a fixed order).  g_field == NULL skips the scatter.  The volume gradient is
 * b200drr_deform_bproj's.
 * The library allocates nothing.  The _v16 twins read a 16-bit volume and equal the fp32 call on the up-cast volume.
 */
int64_t b200drr_deform_scratch_floats(int B, int64_t N, int H, int W);
int b200drr_deform_fwd(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, const float *field, int Bf, int g0, int g1, int g2, float *out, int B, int64_t N, int H,
                       int W, float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);
int b200drr_deform_bwd(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *gout, float *g_src,
                       float *g_tgt, float *g_raylen, float *g_field, float *g_alpha_range, float *scratch, int B, int64_t N, int H,
                       int W, float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);
int b200drr_deform_fwd_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                           const float *raylen, const float *field, int Bf, int g0, int g1, int g2, float *out, int B, int64_t N, int H,
                           int W, float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);
int b200drr_deform_bwd_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                           const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *gout, float *g_src,
                           float *g_tgt, float *g_raylen, float *g_field, float *g_alpha_range, float *scratch, int B, int64_t N, int H,
                           int W, float voxel_shift, float eps, int n_points, const float *alpha_range, void *stream);

/*
 * Directional derivative of the deformable render along a field tangent (DESIGN.md 6k), for matrix-free Gauss-Newton on the
 * field.  Arguments as b200drr_deform_fwd's, plus tangent [Bf][g0][g1][g2][4] in the field's layout (voxel-index units, the same
 * Bf, 16-byte aligned; lane 3 is ignored).  Per ray, with x_m, y_m = x_m + u(x_m) and step as in b200drr_deform_fwd:
 *     jv = raylen * step * sum_m grad tri(V)(y_m) . v(x_m),
 * summed over the samples whose x_m lies inside the lattice's support and whose y_m lies inside the padded volume: the image's
 * derivative along v with the rays and the sampling range held fixed.  It is the transpose of b200drr_deform_bwd's field scatter:
 * sum_n gout_n jv_n = <g_field, tangent> (lanes 0..2) to fp32 reordering.  Outputs, OVERWRITTEN: jv [B][N]; img [B][N] (NULL
 * skips it), b200drr_deform_fwd's out bit for bit.  One value per ray, no atomics: both repeat bit for bit.  A NULL tangent or
 * jv, a misaligned tangent or a bad vol_type returns B200DRR_EINVAL, and the field and ray checks are b200drr_deform_fwd's.  The
 * library allocates nothing.  The _v16 twin reads a 16-bit volume and equals the fp32 call on the up-cast volume.
 */
int b200drr_deform_jvp(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *tangent, float *img,
                       float *jv, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float *alpha_range,
                       void *stream);
int b200drr_deform_jvp_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                           const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *tangent, float *img,
                           float *jv, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                           const float *alpha_range, void *stream);

/*
 * Per-pixel Jacobian of the deformable render along P = 6K field tangents (DESIGN.md 6p), for Levenberg-Marquardt on the K motions
 * of a log-Euclidean blended-rigid render (the field is the exponential of their blended velocity, the tangents its derivatives
 * along the 6K motion increments).  Arguments as b200drr_deform_fwd's, on a full row-major H x W grid only (N = H * W, H, W > 0),
 * plus tangents [Bf][g0][g1][g2][P][4] fp32, node-major (with P = 1 the field's layout; voxel-index units, lane 3 ignored, the
 * field's Bf, 16-byte aligned, fewer than 2^31 floats per pose).  Per pose b, structure k, pixel n and i < 6, p = 6k + i:
 *     J[b][k][n][i] = raylen * step * sum_m grad tri(V)(y_m) . t_p(x_m),
 * summed over b200drr_deform_jvp's samples: jv of that entry point along tangent p, to fp32 reordering.  t_p is not interpolated
 * per sample: the march sums w_c(x_m) grad tri(V)(y_m) per lattice corner c while the samples stay in one cell and contracts the
 * sums with t_p(c) when the cell changes, so sum_n gout_n J[b][.][n][.] is <g_field of b200drr_deform_bwd, t_p> to fp32 reordering.
 * Outputs, all OVERWRITTEN: img [B][H*W], b200drr_deform_fwd's out bit for bit; J [B][K][H*W][6]; rects [B][K][4] int32
 * {w0, w1, h0, h1} (inclusive; empty as {W, -1, H, -1}), the bounding rectangle of the pixels whose ray contracted a nonzero
 * tangent of one of structure k's six: J[b][k] is exactly zero outside it (the contract of b200drr_ncc_normal_structures with
 * S = K).  The entry sets the rects empty on the stream, then grows them with integer atomic min / max: every output repeats bit
 * for bit.  A null pointer, H * W = 0, P outside 1..48, P != 6 K, a misaligned tangents array, J or img aliasing the tangents or
 * a bad vol_type returns B200DRR_EINVAL; K > 8 or a tangents array of 2^31 floats or more per pose B200DRR_EUNSUPPORTED; the field
 * and ray checks are b200drr_deform_fwd's; all before touching CUDA.  The library allocates nothing.  The _v16 twin reads a 16-bit
 * volume and equals the fp32 call on the up-cast volume.
 */
int b200drr_deform_jac(const float *vol, const float *packed, int D0, int D1, int D2, const float *src, const float *tgt,
                       const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *tangents, int P, int K,
                       float *img, float *J, int32_t *rects, int B, int H, int W, float voxel_shift, float eps, int n_points,
                       const float *alpha_range, void *stream);
int b200drr_deform_jac_v16(const void *vol, const void *packed, int vol_type, int D0, int D1, int D2, const float *src, const float *tgt,
                           const float *raylen, const float *field, int Bf, int g0, int g1, int g2, const float *tangents, int P, int K,
                           float *img, float *J, int32_t *rects, int B, int H, int W, float voxel_shift, float eps, int n_points,
                           const float *alpha_range, void *stream);

/*
 * Backprojection through the deformable render (DESIGN.md 6l): the transpose of b200drr_deform_fwd in the density, for
 * reconstruction through known (or jointly fitted) displacement fields.  For a fixed camera and field the render is linear in V:
 *     out = raylen * step * sum_m tri(V, y_m),      y_m = x_m + u(x_m),
 * so the gradient of sum(gout * out) with respect to V is
 *     g_vol[corner] = sum over rays and samples of gout * raylen * step * tri_weight(corner, y_m),
 * over every y_m inside the padded volume (x_m inside the lattice's support or not).  The samples, the field and the range are
 * b200drr_deform_fwd's; no density is read, so there is no volume argument and no _v16 twin.  gout [B][N]; g_vol [D0][D1][D2],
 * OVERWRITTEN: the entry zeroes it on the stream, then every pose (shared or per-pose field) adds into it with scalar atomics, so
 * it repeats only to fp32 reordering.  A NULL gout or g_vol returns B200DRR_EINVAL, and the field and ray checks are
 * b200drr_deform_fwd's (the field 16-byte aligned, fewer than 2^31 floats per pose), all before touching CUDA.  The library
 * allocates nothing.
 */
int b200drr_deform_bproj(int D0, int D1, int D2, const float *src, const float *tgt, const float *raylen, const float *field, int Bf,
                         int g0, int g1, int g2, const float *gout, float *g_vol, int B, int64_t N, int H, int W, float voxel_shift,
                         float eps, int n_points, const float *alpha_range, void *stream);

/*
 * Scaling and squaring of a stationary velocity field (DESIGN.md 6m): N calls compose exp(v) ~ (id + v / 2^N)^(2^N).
 * field, out: [Bf][g0][g1][g2][4] fp32, channel-last, voxel-index units, lane 3 zero (b200drr_deform_fwd's field layout; node i
 * of axis a at voxel coordinate (i + 1/2) D_a / g_a - 1/2 of a D0 x D1 x D2 volume), 16-byte aligned, not aliased.  One step:
 *     out(x) = s field(x) + s U(x + s field(x)),
 * U the trilinear interpolant of field with lattice coordinates clamped to the node range per axis; s = scale, 1 / 2^N on the
 * first step (folding v / 2^N into it) and 1 on the others.  out is OVERWRITTEN, every node once: it repeats bit for bit.
 *
 * b200drr_svf_square_bwd: the step's adjoint for an upstream gradient gout on out, into gin (the field's layout, OVERWRITTEN: the
 * entry zeroes it on the stream): node x gets s gout(x) + s^2 J_U(y)^T gout(x), y = x + s field(x), J_U the interpolant's spatial
 * gradient (zero along a clamped axis), and each corner node c of y's cell gets s w_c(y) gout(x).  Vector reductions: gin repeats
 * only to fp32 reordering.  gout, gin 16-byte aligned, gin aliasing neither input.
 *
 * A NULL pointer, a non-positive size, a scale that is not positive, a misaligned or aliased array returns B200DRR_EINVAL, and a
 * lattice of 2^31 floats or more per pose B200DRR_EUNSUPPORTED, all before touching CUDA.  The library allocates nothing.
 */
int b200drr_svf_square(const float *field, float *out, int Bf, int g0, int g1, int g2, int D0, int D1, int D2, float scale,
                       void *stream);
int b200drr_svf_square_bwd(const float *field, const float *gout, float *gin, int Bf, int g0, int g1, int g2, int D0, int D1, int D2,
                           float scale, void *stream);

/*
 * Forward-mode derivative of one squaring step (DESIGN.md 6n), for Gauss-Newton on a velocity field: the step's tangent along a
 * tangent t on field (the field's layout and units, the same Bf, lane 3 ignored).  With y = x + s field(x) and its clamped cell as
 * in b200drr_svf_square_bwd,
 *     tout(x) = s t(x) + s^2 J_U(y) t(x) + s sum_c w_c(y) t(c),
 * the exact transpose of that adjoint: <gout, tout> = <gin, t> (lanes 0..2) to fp32 reordering.  out (NULL skips it) receives
 * b200drr_svf_square's out bit for bit, so a chain of calls carries the primal and the tangent together.  tout and out are
 * OVERWRITTEN, every node once, lane 3 zero: both repeat bit for bit.  tangent, tout and out 16-byte aligned, tout and out
 * aliasing neither input nor each other.  The refusals are b200drr_svf_square's, plus a NULL tangent (B200DRR_EINVAL), all before
 * touching CUDA.  The library allocates nothing.
 */
int b200drr_svf_square_jvp(const float *field, const float *tangent, float *tout, float *out /* nullable */, int Bf, int g0, int g1,
                           int g2, int D0, int D1, int D2, float scale, void *stream);

/*
 * b200drr_svf_square_jvp for P tangents at once (DESIGN.md 6p): tangents and tout [Bf][g0][g1][g2][P][4] fp32, node-major (the P
 * tangents of a node are contiguous; with P = 1 the field's layout).  Slice p of tout equals b200drr_svf_square_jvp on slice p of
 * tangents bit for bit: y, its cell and J_U are formed once per node and the per-tangent arithmetic is that entry point's, in the
 * same order.  out (NULL skips it) receives b200drr_svf_square's out bit for bit.  tout and out are OVERWRITTEN, lane 3 zero.
 * tangents, tout and out 16-byte aligned, tout and out aliasing neither input nor each other.  The refusals are
 * b200drr_svf_square_jvp's, plus P outside 1..48 (B200DRR_EINVAL) and a tangents array of 2^31 floats or more per pose
 * (B200DRR_EUNSUPPORTED), all before touching CUDA.  The library allocates nothing.
 */
int b200drr_svf_square_tangents(const float *field, const float *tangents, float *tout, float *out /* nullable */, int Bf, int P,
                                int g0, int g1, int g2, int D0, int D1, int D2, float scale, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B200DRR_H */
