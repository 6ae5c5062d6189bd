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
 * of the batch share through L2 (DESIGN.md 4.1 / 4.1c); other values select kernels for benchmarking: 46 / 47 / 15 = the
 * slab-major kernel with 16- / 24- / 32-plane slabs,
 * 100+K / 200+K / 300+K / 400+K (K = 1..64) = K major-axis pieces with 16x16/U4, 8x16/U8, 16x8/U4, 8x16/U4 tiles, further ids =
 * tile-shape / unroll variants (cudaErrorInvalidValue if unknown).
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
 * red.global.add partial sums.  align_corners=0 only.
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
 * (use b200drr_siddon_bwd_grid when the volume requires grad).  variant 0 = tuned default (major-axis pieces up to 6 poses of
 * 256^2 rays, 16-plane slabs beyond); 41 / 40 / 39 / 38 = the 16- / 24- / 32- / 48-plane-slab kernels; 100+K / 300+K / 400+K = K major-axis pieces (8x16/U8, 16x8/U8,
 * 8x16/U4 tiles); further ids = tile / unroll / slab-height variants for benchmarking.
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
 * as b200drr_trilinear_fwd / _bwd with pixel tiles mapped onto warps/CTAs for cache locality.
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
 *   variant: 0 = tuned default.
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

#ifdef __cplusplus
}
#endif
#endif /* B200DRR_H */
