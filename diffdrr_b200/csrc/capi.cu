// capi.cu -- the C ABI of libb200drr.so (see include/b200drr.h for the contract of every entry point).
#include <cuda_runtime.h>

#include <algorithm>
#include <type_traits>

#include "../../include/b200drr.h"
#ifdef B200DRR_EXPERIMENTS
#include "../../include/b200drr_experimental.h"
#endif
#include "kernels.h"

using namespace b200drr;

namespace {

inline bool bad_dims(int D0, int D1, int D2) { return D0 <= 0 || D1 <= 0 || D2 <= 0; }
inline bool bad_rays(int B, int64_t N) { return B <= 0 || B > 65535 || N <= 0; }
inline bool bad_grid(int B, int H, int W) { return bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0; }  // B detectors of H x W rays
inline bool too_big(int D0, int D1, int D2) { return (int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX; }
inline VolDims mk(int D0, int D1, int D2)
{
    VolDims d;
    d.d[0] = D0;
    d.d[1] = D1;
    d.d[2] = D2;
    return d;
}
inline int ret(cudaError_t e) { return e == cudaSuccess ? 0 : (int)e; }

template <typename R>
int segments_fwd(int kind, const void* vol, int D0, int D1, int D2, const void* src, const void* tgt, const void* raylen, void* out,
                 int B, int64_t N, double shift, double eps, int n_points, const void* alpha_range, int align_corners, void* stream)
{
    const VolDims d = mk(D0, D1, D2);
    if (kind == 0)
        return ret(launch_siddon_fwd_literal<R>((const R*)vol, d, (const R*)src, (const R*)tgt, (const R*)raylen, (R*)out, B, N, (R)shift,
                                                (R)eps, 2, align_corners, (cudaStream_t)stream));
    return ret(launch_trilinear_fwd_literal<R>((const R*)vol, d, (const R*)src, (const R*)tgt, (const R*)raylen, (R*)out, B, N, (R)shift,
                                               (R)eps, n_points, (const R*)alpha_range, 2, align_corners, (cudaStream_t)stream));
}
template <typename R>
int segments_bwd(int kind, const void* vol, int D0, int D1, int D2, const void* src, const void* tgt, const void* raylen,
                 const void* gseg, void* g_src, void* g_tgt, void* g_raylen, void* g_vol, void* g_alpha_range, int B, int64_t N,
                 double shift, double eps, int n_points, const void* alpha_range, int stop_grad, int align_corners, void* stream)
{
    const VolDims d = mk(D0, D1, D2);
    if (kind == 0)
        return ret(launch_siddon_bwd_literal<R>((const R*)vol, d, (const R*)src, (const R*)tgt, (const R*)raylen, nullptr, (const R*)gseg,
                                                (R*)g_src, (R*)g_tgt, (R*)g_raylen, (R*)g_vol, B, N, (R)shift, (R)eps, stop_grad,
                                                align_corners, (cudaStream_t)stream));
    return ret(launch_trilinear_bwd_literal<R>((const R*)vol, d, (const R*)src, (const R*)tgt, (const R*)raylen, nullptr,
                                               (const R*)gseg, (R*)g_src, (R*)g_tgt, (R*)g_raylen, (R*)g_vol, (R*)g_alpha_range, B, N,
                                               (R)shift, (R)eps, n_points, (const R*)alpha_range, align_corners, (cudaStream_t)stream));
}

// Calls f with a value of the voxel type vol_type names (VoxF16 / VoxBF16); B200DRR_EINVAL for anything else.
template <class F>
int with_vox16(int vol_type, F&& f)
{
    if (vol_type == B200DRR_VOL_F16) return f(VoxF16{});
    if (vol_type == B200DRR_VOL_BF16) return f(VoxBF16{});
    return B200DRR_EINVAL;
}
inline bool bad_vol16(int vol_type) { return vol_type != B200DRR_VOL_F16 && vol_type != B200DRR_VOL_BF16; }

// the brick kernels' refusals after the argument checks, in this order: a shape the TMA map cannot take or a volume (or volume
// gradient) off 16 bytes is B200DRR_EUNSUPPORTED, a workspace under `need` bytes or off 256 bytes B200DRR_EINVAL; 0 = go on
int brick_bad(const void* vol, VolDims d, int H, int W, int elem_bytes, const void* workspace, int64_t workspace_bytes, size_t need)
{
    if (!siddon_brick_supported(d, H, W, elem_bytes) || ((uintptr_t)vol & 15u) != 0) return B200DRR_EUNSUPPORTED;
    if (workspace_bytes < (int64_t)need || ((uintptr_t)workspace & 255u) != 0) return B200DRR_EINVAL;
    return 0;
}
}  // namespace

extern "C" {

int b200drr_version(void) { return B200DRR_VERSION; }

const char* b200drr_error_string(int code)
{
    if (code == 0) return "success";
    if (code == B200DRR_EINVAL) return "b200drr: invalid argument (null pointer, non-positive size, B > 65535 or bad enum)";
    if (code == B200DRR_EUNSUPPORTED) return "b200drr: unsupported option combination for this entry point";
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "b200drr: unknown error code";
}

int b200drr_device_sm_count(void)
{
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return n;
}

int b200drr_device_cc(void)
{
    int dev = 0, ma = 0, mi = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&ma, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&mi, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
    return ma * 10 + mi;
}

int b200drr_siddon_fwd_f64(const double* vol, int D0, int D1, int D2, const double* src, const double* tgt, const double* raylen,
                           double* out, int B, int64_t N, double voxel_shift, double eps, int reduce, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || reduce < 0 || reduce > 1)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd_literal<double>(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, reduce, align_corners != 0,
                                     (cudaStream_t)stream));
}

int b200drr_siddon_bwd_f64(const double* vol, int D0, int D1, int D2, const double* src, const double* tgt, const double* raylen,
                           const double* gout, double* g_src, double* g_tgt, double* g_raylen, double* g_vol, int B, int64_t N,
                           double voxel_shift, double eps, int stop_grad, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_literal<double>(vol, mk(D0, D1, D2), src, tgt, raylen, gout, nullptr, g_src, g_tgt, g_raylen, g_vol, B, N, voxel_shift,
                                     eps, stop_grad != 0, align_corners != 0, (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_f64(const double* vol, int D0, int D1, int D2, const double* src, const double* tgt,
                              const double* raylen, double* out, int B, int64_t N, double voxel_shift, double eps, int n_points,
                              const double* alpha_range, int reduce, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) || n_points < 2 ||
        reduce < 0 || reduce > 1)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_literal<double>(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, n_points, alpha_range,
                                        reduce, align_corners != 0, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_f64(const double* vol, int D0, int D1, int D2, const double* src, const double* tgt,
                              const double* raylen, const double* gout, double* g_src, double* g_tgt, double* g_raylen,
                              double* g_vol, double* g_alpha_range, int B, int64_t N, double voxel_shift, double eps,
                              int n_points, const double* alpha_range, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_literal<double>(vol, mk(D0, D1, D2), src, tgt, raylen, gout, nullptr, g_src, g_tgt, g_raylen, g_vol, g_alpha_range, B,
                                        N, voxel_shift, eps, n_points, alpha_range, align_corners != 0, (cudaStream_t)stream));
}

int b200drr_segments_fwd(int kind, int is_f64, const void* vol, int D0, int D1, int D2, const void* src, const void* tgt,
                         const void* raylen, void* out, int B, int64_t N, double voxel_shift, double eps, int n_points,
                         const void* alpha_range, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || kind < 0 || kind > 1 ||
        (kind == 1 && (!alpha_range || n_points < 2)))
        return B200DRR_EINVAL;
    return is_f64 ? segments_fwd<double>(kind, vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, n_points, alpha_range,
                                         align_corners != 0, stream)
                  : segments_fwd<float>(kind, vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, n_points, alpha_range,
                                        align_corners != 0, stream);
}

int b200drr_segments_bwd(int kind, int is_f64, const void* vol, int D0, int D1, int D2, const void* src, const void* tgt,
                         const void* raylen, const void* gseg, void* g_src, void* g_tgt, void* g_raylen, void* g_vol,
                         void* g_alpha_range, int B, int64_t N, double voxel_shift, double eps, int n_points,
                         const void* alpha_range, int stop_grad, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gseg || bad_dims(D0, D1, D2) || bad_rays(B, N) || kind < 0 || kind > 1 ||
        (kind == 1 && (!alpha_range || n_points < 2)))
        return B200DRR_EINVAL;
    return is_f64 ? segments_bwd<double>(kind, vol, D0, D1, D2, src, tgt, raylen, gseg, g_src, g_tgt, g_raylen, g_vol, g_alpha_range,
                                         B, N, voxel_shift, eps, n_points, alpha_range, stop_grad != 0, align_corners != 0, stream)
                  : segments_bwd<float>(kind, vol, D0, D1, D2, src, tgt, raylen, gseg, g_src, g_tgt, g_raylen, g_vol, g_alpha_range,
                                        B, N, voxel_shift, eps, n_points, alpha_range, stop_grad != 0, align_corners != 0, stream);
}

int64_t b200drr_siddon_brick_workspace_bytes(int B, int H, int W)
{
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    return (int64_t)siddon_brick_workspace_bytes(B, H, W);
}

int b200drr_siddon_bwd_vol_brick(const float* gout, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                                 const float* G, const float* Wd, const float* rows, const float* cols, float* g_vol,
                                 void* workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift, float eps,
                                 void* stream)
{
    const bool pose_in = G != nullptr;
    if (!gout || !src || !g_vol || !workspace || bad_dims(D0, D1, D2) || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    if (pose_in ? (!Wd || !rows || !cols) : (!tgt || !raylen)) return B200DRR_EINVAL;
    if (!siddon_brick_supported(mk(D0, D1, D2), H, W) || ((uintptr_t)g_vol & 15u) != 0) return B200DRR_EUNSUPPORTED;
    if (workspace_bytes < (int64_t)siddon_brick_workspace_bytes(B, H, W) || ((uintptr_t)workspace & 255u) != 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_vol_brick(gout, mk(D0, D1, D2), src, tgt, raylen, G, Wd, rows, cols, g_vol, workspace,
                                           (size_t)workspace_bytes, B, H, W, voxel_shift, eps, (cudaStream_t)stream));
}

int b200drr_siddon_bwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                       float* g_vol, int B, int64_t N, float voxel_shift, float eps, int stop_grad, int align_corners,
                       void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if (align_corners) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_bwd(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B, N,
                                 voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_siddon_bwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                            const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                            float* g_vol, int B, int H, int W, float voxel_shift, float eps, int stop_grad, int variant,
                            void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B, H, W,
                                      voxel_shift, eps, stop_grad != 0, variant, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                          const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                          float* g_vol, float* g_alpha_range, int B, int64_t N, float voxel_shift, float eps,
                          int n_points, const float* alpha_range, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol,
                                    g_alpha_range, B, N, voxel_shift, eps, n_points, alpha_range, align_corners != 0,
                                    (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                               float* g_vol, float* g_alpha_range, int B, int H, int W, float voxel_shift, float eps,
                               int n_points, const float* alpha_range, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol,
                                         g_alpha_range, B, H, W, voxel_shift, eps, n_points, alpha_range, variant,
                                         (cudaStream_t)stream));
}

int b200drr_siddon_bwd_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                            const float* rows, const float* cols, const float* gout, float* g_src, float* g_G, float* g_Wd,
                            float* g_vol, float* ws_tgt, float* ws_len, int B, int H, int W, float voxel_shift, float eps,
                            int stop_grad, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !gout || !g_src || !g_G || !g_Wd || !ws_tgt || !ws_len ||
        bad_dims(D0, D1, D2) || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_bwd_pose(vol, mk(D0, D1, D2), src, G, Wd, rows, cols, gout, g_src, g_G, g_Wd, g_vol, ws_tgt,
                                      ws_len, B, H, W, voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_label_boxes(const uint8_t* labels, int D0, int D1, int D2, int32_t* boxes, void* stream)
{
    if (!labels || !boxes || bad_dims(D0, D1, D2)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_label_boxes(labels, mk(D0, D1, D2), boxes, (cudaStream_t)stream));
}

int b200drr_siddon_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen, int B,
                            int64_t N, int stop_grad, void* stream)
{
    if (!sens || !gout || bad_rays(B, N)) return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_sens(sens, gout, g_src, g_tgt, g_raylen, B, N, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_siddon_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows, const float* cols,
                                 float* g_src, float* g_G, float* g_Wd, int B, int H, int W, int stop_grad, void* stream)
{
    if (!sens || !gout || !Wd || !rows || !cols || !g_src || !g_G || !g_Wd || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_sens_pose(sens, gout, Wd, rows, cols, g_src, g_G, g_Wd, B, H, W, stop_grad != 0,
                                           (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_sens(const float* sens, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                               float* g_alpha_range, int B, int64_t N, void* stream)
{
    if (!sens || !gout || bad_rays(B, N)) return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_sens(sens, gout, g_src, g_tgt, g_raylen, g_alpha_range, B, N, (cudaStream_t)stream));
}

int b200drr_trilinear_alpha_range_pose(int D0, int D1, int D2, const float* src, const float* G, const float* Wd, const float* rows,
                                       const float* cols, float* range, int64_t* arg, void* scratch16, int B, int H, int W,
                                       float voxel_shift, float eps, void* stream)
{
    if (!src || !G || !Wd || !rows || !cols || !range || !arg || !scratch16 || bad_dims(D0, D1, D2) ||
        bad_grid(B, H, W))
        return B200DRR_EINVAL;
    return ret(launch_trilinear_alpha_range_pose(mk(D0, D1, D2), src, G, Wd, rows, cols, range, arg, scratch16, B, H, W, voxel_shift,
                                                 eps, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows, const float* cols,
                                    float* g_src, float* g_G, float* g_Wd, float* g_alpha_range, int B, int H, int W, void* stream)
{
    if (!sens || !gout || !Wd || !rows || !cols || !g_src || !g_G || !g_Wd || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_sens_pose(sens, gout, Wd, rows, cols, g_src, g_G, g_Wd, g_alpha_range, B, H, W,
                                              (cudaStream_t)stream));
}

int b200drr_siddon_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                 const float* rows, const float* cols, float* J, int B, int H, int W, int P, int stop_grad,
                                 void* stream)
{
    if (!sens || !dsrc || !dG || !dWd || !Wd || !rows || !cols || !J || bad_grid(B, H, W) || P < 1 ||
        P > 16)
        return B200DRR_EINVAL;
    return ret(launch_siddon_jac_sens_pose(sens, dsrc, dG, dWd, Wd, rows, cols, J, B, H, W, P, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_trilinear_jac_sens_pose(const float* sens, const float* dsrc, const float* dG, const float* dWd, const float* Wd,
                                    const float* rows, const float* cols, const float* drange, float* J, int B, int H, int W, int P,
                                    void* stream)
{
    if (!sens || !dsrc || !dG || !dWd || !Wd || !rows || !cols || !drange || !J || bad_grid(B, H, W) || P < 1 || P > 16)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_jac_sens_pose(sens, dsrc, dG, dWd, Wd, rows, cols, drange, J, B, H, W, P, (cudaStream_t)stream));
}

static bool bad_axes(int c0, int c1, int c2)
{
    return c0 < 0 || c0 > 2 || c1 < 0 || c1 > 2 || c2 < 0 || c2 > 2 || c1 == c0 || c1 == c2;
}

int b200drr_euler_pose_fwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, float* P, int B,
                           void* stream)
{
    if (!rot || !xyz || !P || B <= 0 || bad_axes(c0, c1, c2)) return B200DRR_EINVAL;
    return ret(launch_euler_pose_fwd(rot, xyz, c0, c1, c2, scale, P, B, (cudaStream_t)stream));
}

int b200drr_euler_pose_bwd(const float* rot, const float* xyz, int c0, int c1, int c2, float scale, const float* gP,
                           float* g_rot, float* g_xyz, int B, void* stream)
{
    if (!rot || !xyz || !gP || B <= 0 || bad_axes(c0, c1, c2)) return B200DRR_EINVAL;
    return ret(launch_euler_pose_bwd(rot, xyz, c0, c1, c2, scale, gP, g_rot, g_xyz, B, (cudaStream_t)stream));
}

int b200drr_pose_rays_fwd(const float* P, const float* Q, const float* r, const float* Ainv, float* src, float* G, float* Wd,
                          int B, void* stream)
{
    if (!P || !Q || !r || !Ainv || !src || !G || !Wd || B <= 0) return B200DRR_EINVAL;
    return ret(launch_pose_rays_fwd(P, Q, r, Ainv, src, G, Wd, B, (cudaStream_t)stream));
}

int b200drr_pose_rays_bwd(const float* Q, const float* r, const float* Ainv, const float* g_src, const float* g_G,
                          const float* g_Wd, float* gP, int B, void* stream)
{
    if (!Q || !r || !Ainv || !g_src || !g_G || !g_Wd || !gP || B <= 0) return B200DRR_EINVAL;
    return ret(launch_pose_rays_bwd(Q, r, Ainv, g_src, g_G, g_Wd, gP, B, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_mask(const float* vol, const float* mask, int D0, int D1, int D2, const float* src,
                            const float* tgt, const float* raylen, float* out, int B, int64_t N, int C, float voxel_shift,
                            float eps, void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || C <= 0)
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, out, B, N, C, voxel_shift, eps,
                                      (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_mask(const float* vol, const float* mask, int D0, int D1, int D2, const float* src,
                               const float* tgt, const float* raylen, float* out, int B, int64_t N, int C,
                               float voxel_shift, float eps, int n_points, const float* alpha_range, int align_corners,
                               void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        C <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, out, B, N, C, voxel_shift, eps,
                                         n_points, alpha_range, align_corners != 0, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int H, int W, int C, float voxel_shift, float eps,
                                 void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || C <= 0)
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, out, B, (int64_t)H * W, C, voxel_shift, eps,
                                      (cudaStream_t)stream, W));
}

int b200drr_trilinear_fwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src,
                                    const float* tgt, const float* raylen, float* out, int B, int H, int W, int C,
                                    float voxel_shift, float eps, int n_points, const float* alpha_range, int align_corners,
                                    void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || C <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, out, B, (int64_t)H * W, C, voxel_shift, eps,
                                         n_points, alpha_range, align_corners != 0, (cudaStream_t)stream, W));
}

int b200drr_siddon_bwd_general(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                               float* g_vol, int B, int64_t N, float voxel_shift, float eps, int stop_grad, int reduce,
                               int align_corners, int mode, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_rays(B, N) || reduce < 0 || reduce > 1 ||
        mode < 0 || mode > 1)
        return B200DRR_EINVAL;
    if (mode == 1 && reduce != 0) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_bwd_general(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B, N,
                                         voxel_shift, eps, stop_grad != 0, reduce, align_corners != 0, mode,
                                         (cudaStream_t)stream));
}

int b200drr_siddon_fwd_general(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps, int reduce,
                               int align_corners, int mode, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || reduce < 0 || reduce > 1 ||
        mode < 0 || mode > 1)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd_general(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, reduce,
                                         align_corners != 0, mode, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_max(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                              const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                              float* g_vol, float* g_alpha_range, int B, int64_t N, float voxel_shift, float eps,
                              int n_points, const float* alpha_range, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, g_alpha_range,
                                    B, N, voxel_shift, eps, n_points, alpha_range, align_corners != 0, (cudaStream_t)stream,
                                    1));
}

int b200drr_siddon_bwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_vol,
                                 int B, int H, int W, int C, float voxel_shift, float eps, int stop_grad, void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || C <= 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B,
                                      (int64_t)H * W, C, voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream, W));
}

int b200drr_trilinear_bwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src, const float* tgt,
                                    const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                    float* g_vol, float* g_alpha_range, int B, int H, int W, int C, float voxel_shift, float eps,
                                    int n_points, const float* alpha_range, int align_corners, void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || C <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol,
                                         g_alpha_range, B, (int64_t)H * W, C, voxel_shift, eps, n_points, alpha_range,
                                         align_corners != 0, (cudaStream_t)stream, W));
}

int b200drr_siddon_bwd_mask(const float* vol, const float* mask, int D0, int D1, int D2, const float* src, const float* tgt,
                            const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                            float* g_vol, int B, int64_t N, int C, float voxel_shift, float eps, int stop_grad, void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_rays(B, N) || C <= 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B, N,
                                      C, voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_mask(const float* vol, const float* mask, int D0, int D1, int D2, const float* src,
                               const float* tgt, const float* raylen, const float* gout, float* g_src, float* g_tgt,
                               float* g_raylen, float* g_vol, float* g_alpha_range, int B, int64_t N, int C,
                               float voxel_shift, float eps, int n_points, const float* alpha_range, int align_corners,
                               void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        C <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol,
                                         g_alpha_range, B, N, C, voxel_shift, eps, n_points, alpha_range, align_corners != 0,
                                         (cudaStream_t)stream));
}

}  // extern "C"

// ---- entry points with a 16-bit twin (include/b200drr.h, DESIGN.md 4.5) -----------------------------------------------------------
// One body per fp32 entry point and its `_v16` twin, on the voxel type V: float for the fp32 entry point, VoxF16 / VoxBF16 for the
// twin, which reaches it through with_vox16.  The twins have no tuning variants, and the plain Siddon / Trilinear forward twins
// take only reduce = 0 and align_corners = 0.
namespace {
template <class V>
constexpr bool kF32 = std::is_same<V, float>::value;

template <class V>
int siddon_fwd(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out, int B,
               int64_t N, float voxel_shift, float eps, int reduce, int align_corners, void* stream)
{
    const bool bad_options = kF32<V> ? reduce < 0 || reduce > 1 : reduce != 0 || align_corners != 0;
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || bad_options) return B200DRR_EINVAL;
    if constexpr (kF32<V>)
        return ret(launch_siddon_fwd((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, reduce,
                                     align_corners != 0, (cudaStream_t)stream));
    else
        return ret(launch_siddon_fwd_fast((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps,
                                          (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_sens(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                    float* sens, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, voxel_shift, eps,
                                      (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_sorted(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                      int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sorted((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps,
                                        (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_sens_sorted(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                           float* out, float* sens, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_sorted((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, voxel_shift, eps,
                                             (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_grid(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                    int B, int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_grid(B, H, W)) return B200DRR_EINVAL;
    if constexpr (kF32<V>) {
        return ret(launch_siddon_fwd_grid((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps, variant,
                                          (cudaStream_t)stream));
    } else {
        if (variant != 0) return B200DRR_EUNSUPPORTED;
        return ret(launch_siddon_fwd_grid_default((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps,
                                                  (cudaStream_t)stream));
    }
}

template <class V>
int siddon_fwd_sens_grid(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                         float* out, float* sens, int B, int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_grid(B, H, W)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2) || (!kF32<V> && variant != 0)) return B200DRR_EUNSUPPORTED;
    if constexpr (kF32<V>)
        return ret(launch_siddon_fwd_sens_grid((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps,
                                               variant, (cudaStream_t)stream));
    else
        return ret(launch_siddon_fwd_sens_grid_default((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, H, W,
                                                       voxel_shift, eps, (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_brick(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* G,
                     const float* Wd, const float* rows, const float* cols, float* out, void* workspace, int64_t workspace_bytes, int B,
                     int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    const bool pose_in = G != nullptr;
    if (!vol || !src || !out || !workspace || bad_dims(D0, D1, D2) || bad_grid(B, H, W)) return B200DRR_EINVAL;
    if (pose_in ? (!Wd || !rows || !cols) : (!tgt || !raylen)) return B200DRR_EINVAL;
    if (!kF32<V> && variant != 0) return B200DRR_EUNSUPPORTED;
    if (const int bad =
            brick_bad(vol, mk(D0, D1, D2), H, W, sizeof(V), workspace, workspace_bytes, siddon_brick_workspace_bytes(B, H, W)))
        return bad;
    return ret(launch_siddon_fwd_brick((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, G, Wd, rows, cols, out, workspace,
                                       (size_t)workspace_bytes, B, H, W, voxel_shift, eps, variant, (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_brick_subset(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                            const int32_t* pix_index, const float* corners, float* out, void* workspace, int64_t workspace_bytes, int B,
                            int H, int W, int64_t Nsub, float voxel_shift, float eps, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !pix_index || !corners || !out || !workspace || bad_dims(D0, D1, D2) ||
        bad_rays(B, Nsub) || H <= 0 || W <= 0 || Nsub > (int64_t)H * W)
        return B200DRR_EINVAL;
    if (!kF32<V> && variant != 0) return B200DRR_EUNSUPPORTED;
    if (const int bad = brick_bad(vol, mk(D0, D1, D2), H, W, sizeof(V), workspace, workspace_bytes,
                                  siddon_brick_workspace_bytes(B, 1, (int)Nsub)))
        return bad;
    return ret(launch_siddon_fwd_brick((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, nullptr, nullptr, nullptr, nullptr, out,
                                       workspace, (size_t)workspace_bytes, B, H, W, voxel_shift, eps, variant, (cudaStream_t)stream,
                                       pix_index, corners, Nsub));
}

template <class V>
int siddon_fwd_pose(const void* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd, const float* rows,
                    const float* cols, float* out, int B, int H, int W, float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !out || bad_dims(D0, D1, D2) || bad_grid(B, H, W)) return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_pose((const V*)vol, mk(D0, D1, D2), src, G, Wd, rows, cols, out, B, H, W, voxel_shift, eps,
                                      (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_sens_pose(const void* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                         const float* rows, const float* cols, float* out, float* sens, int B, int H, int W, float voxel_shift,
                         float eps, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !out || !sens || bad_dims(D0, D1, D2) || bad_grid(B, H, W))
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_pose((const V*)vol, mk(D0, D1, D2), src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift,
                                           eps, (cudaStream_t)stream));
}

template <class V>
int siddon_fwd_sens_structures(const void* vol, const uint8_t* labels, int D0, int D1, int D2, const float* src, const float* G,
                               const float* Wd, const float* rows, const float* cols, const int32_t* slot_of_label,
                               const int32_t* box, float* out, float* sens, int B, int S, int H, int W, float voxel_shift,
                               float eps, void* stream)
{
    if (!vol || !labels || !src || !G || !Wd || !rows || !cols || !slot_of_label || !box || !out || bad_dims(D0, D1, D2) ||
        S <= 0 || S > 256 || B <= 0 || bad_rays((int)std::min<int64_t>((int64_t)B * S, INT32_MAX), (int64_t)H * W) || H <= 0 ||
        W <= 0)
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2)) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_structures((const V*)vol, labels, mk(D0, D1, D2), src, G, Wd, rows, cols, slot_of_label, box,
                                                 out, sens, B, S, H, W, voxel_shift, eps, (cudaStream_t)stream));
}

template <class V>
int pack_corners(const void* vol, int D0, int D1, int D2, void* packed, void* stream)
{
    if (!vol || !packed || bad_dims(D0, D1, D2) || (!kF32<V> && ((uintptr_t)packed & 15u) != 0)) return B200DRR_EINVAL;
    if constexpr (kF32<V>)
        return ret(launch_pack_corners((const V*)vol, mk(D0, D1, D2), (float*)packed, (cudaStream_t)stream));
    else
        return ret(launch_pack_corners16((const V*)vol, mk(D0, D1, D2), (Cell16<V>*)packed, (cudaStream_t)stream));
}

template <class V>
int trilinear_fwd(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                  int B, int64_t N, float voxel_shift, float eps, int n_points, const float* alpha_range, int reduce,
                  int align_corners, void* stream)
{
    const bool bad_options = kF32<V> ? reduce < 0 || reduce > 1 : reduce != 0 || align_corners != 0;
    if (!vol || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) || n_points < 2 ||
        bad_options)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, n_points,
                                    alpha_range, reduce, align_corners != 0, (cudaStream_t)stream));
}

template <class V>
int trilinear_fwd_grid(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                       int B, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range, int variant,
                       void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_grid((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points,
                                         alpha_range, variant, (cudaStream_t)stream));
}

template <class V>
int trilinear_fwd_sens(const void* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                       float* sens, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                       const float* alpha_range, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        n_points < 2 || H < 0 || W < 0 || (H > 0 && ((int64_t)H * W != N || align_corners)) || (!kF32<V> && align_corners != 0))
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_sens((const V*)vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, H, W, voxel_shift, eps,
                                         n_points, alpha_range, align_corners != 0, (cudaStream_t)stream));
}

// the packed copy of a 16-bit volume holds cells of its own type (Cell16<V>)
template <class V>
int trilinear_fwd_packed(const void* packed, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                         float* out, int B, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range,
                         int slab, void* stream)
{
    if (!packed || slab < 0 || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) ||
        n_points < 2)
        return B200DRR_EINVAL;
    if constexpr (kF32<V>)
        return ret(launch_trilinear_fwd_packed((const float*)packed, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps,
                                               n_points, alpha_range, slab, (cudaStream_t)stream));
    else
        return ret(launch_trilinear_fwd_packed_t((const Cell16<V>*)packed, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W,
                                                 voxel_shift, eps, n_points, alpha_range, slab, (cudaStream_t)stream));
}

template <class V>
int trilinear_fwd_sens_packed(const void* packed, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                              float* out, float* sens, int B, int H, int W, float voxel_shift, float eps, int n_points,
                              const float* alpha_range, int slab, void* stream)
{
    if (!packed || !src || !tgt || !raylen || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) || bad_grid(B, H, W) ||
        n_points < 2 || slab < 0)
        return B200DRR_EINVAL;
    if constexpr (kF32<V>)
        return ret(launch_trilinear_fwd_sens_packed((const float*)packed, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, H, W,
                                                    voxel_shift, eps, n_points, alpha_range, slab, (cudaStream_t)stream));
    else
        return ret(launch_trilinear_fwd_sens_packed16((const Cell16<V>*)packed, mk(D0, D1, D2), src, tgt, raylen, nullptr, nullptr,
                                                      nullptr, nullptr, out, sens, B, H, W, voxel_shift, eps, n_points, alpha_range,
                                                      slab, (cudaStream_t)stream));
}

template <class V>
int trilinear_fwd_sens_pose(const void* packed, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                            const float* rows, const float* cols, float* out, float* sens, int B, int H, int W, float voxel_shift,
                            float eps, int n_points, const float* alpha_range, int slab, void* stream)
{
    if (!packed || !src || !G || !Wd || !rows || !cols || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_grid(B, H, W) || n_points < 2 || slab < 0)
        return B200DRR_EINVAL;
    if constexpr (kF32<V>)
        return ret(launch_trilinear_fwd_sens_pose((const float*)packed, mk(D0, D1, D2), src, G, Wd, rows, cols, out, sens, B, H, W,
                                                  voxel_shift, eps, n_points, alpha_range, slab, (cudaStream_t)stream));
    else
        return ret(launch_trilinear_fwd_sens_packed16((const Cell16<V>*)packed, mk(D0, D1, D2), src, nullptr, nullptr, G, Wd, rows,
                                                      cols, out, sens, B, H, W, voxel_shift, eps, n_points, alpha_range, slab,
                                                      (cudaStream_t)stream));
}
}  // namespace

extern "C" {

int b200drr_siddon_fwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, float* out,
                       int B, int64_t N, float voxel_shift, float eps, int reduce, int align_corners, void* stream)
{
    return siddon_fwd<float>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, reduce, align_corners, stream);
}

int b200drr_siddon_fwd_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                           const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps, int reduce,
                           int align_corners, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, reduce, align_corners, stream);
    });
}

int b200drr_siddon_fwd_sens(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                            float* out, float* sens, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    return siddon_fwd_sens<float>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_sens_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                const float* raylen, float* out, float* sens, int B, int64_t N, float voxel_shift, float eps,
                                void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sens<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, voxel_shift, eps, stream);
    });
}

int b200drr_siddon_fwd_sorted(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                              float* out, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    return siddon_fwd_sorted<float>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_sorted_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                  const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sorted<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, stream);
    });
}

int b200drr_siddon_fwd_sens_sorted(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                                   const float* raylen, float* out, float* sens, int B, int64_t N, float voxel_shift, float eps,
                                   void* stream)
{
    return siddon_fwd_sens_sorted<float>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_sens_sorted_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                       const float* raylen, float* out, float* sens, int B, int64_t N, float voxel_shift, float eps,
                                       void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sens_sorted<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, voxel_shift, eps, stream);
    });
}

int b200drr_siddon_fwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                            float* out, int B, int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    return siddon_fwd_grid<float>(vol, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, variant, stream);
}

int b200drr_siddon_fwd_grid_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps, int variant,
                                void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_grid<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, variant, stream);
    });
}

int b200drr_siddon_fwd_sens_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                                 float* out, float* sens, int B, int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    return siddon_fwd_sens_grid<float>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps, variant, stream);
}

int b200drr_siddon_fwd_sens_grid_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                     const float* raylen, float* out, float* sens, int B, int H, int W, float voxel_shift, float eps,
                                     int variant, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sens_grid<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps, variant,
                                                 stream);
    });
}

int b200drr_siddon_fwd_brick(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                             const float* G, const float* Wd, const float* rows, const float* cols, float* out, void* workspace,
                             int64_t workspace_bytes, int B, int H, int W, float voxel_shift, float eps, int variant, void* stream)
{
    return siddon_fwd_brick<float>(vol, D0, D1, D2, src, tgt, raylen, G, Wd, rows, cols, out, workspace, workspace_bytes, B, H, W,
                                   voxel_shift, eps, variant, stream);
}

int b200drr_siddon_fwd_brick_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, const float* G, const float* Wd, const float* rows, const float* cols,
                                 float* out, void* workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift,
                                 float eps, int variant, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_brick<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, G, Wd, rows, cols, out, workspace, workspace_bytes, B,
                                             H, W, voxel_shift, eps, variant, stream);
    });
}

int b200drr_siddon_fwd_brick_subset(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                                    const float* raylen, const int32_t* pix_index, const float* corners, float* out,
                                    void* workspace, int64_t workspace_bytes, int B, int H, int W, int64_t Nsub,
                                    float voxel_shift, float eps, int variant, void* stream)
{
    return siddon_fwd_brick_subset<float>(vol, D0, D1, D2, src, tgt, raylen, pix_index, corners, out, workspace, workspace_bytes, B,
                                          H, W, Nsub, voxel_shift, eps, variant, stream);
}

int b200drr_siddon_fwd_brick_subset_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                        const float* raylen, const int32_t* pix_index, const float* corners, float* out,
                                        void* workspace, int64_t workspace_bytes, int B, int H, int W, int64_t Nsub,
                                        float voxel_shift, float eps, int variant, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_brick_subset<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, pix_index, corners, out, workspace,
                                                    workspace_bytes, B, H, W, Nsub, voxel_shift, eps, variant, stream);
    });
}

int b200drr_siddon_fwd_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                            const float* rows, const float* cols, float* out, int B, int H, int W, float voxel_shift,
                            float eps, void* stream)
{
    return siddon_fwd_pose<float>(vol, D0, D1, D2, src, G, Wd, rows, cols, out, B, H, W, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_pose_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* G,
                                const float* Wd, const float* rows, const float* cols, float* out, int B, int H, int W,
                                float voxel_shift, float eps, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_pose<decltype(v)>(vol, D0, D1, D2, src, G, Wd, rows, cols, out, B, H, W, voxel_shift, eps, stream);
    });
}

int b200drr_siddon_fwd_sens_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                                 const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                 float voxel_shift, float eps, void* stream)
{
    return siddon_fwd_sens_pose<float>(vol, D0, D1, D2, src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_sens_pose_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* G,
                                     const float* Wd, const float* rows, const float* cols, float* out, float* sens, int B, int H,
                                     int W, float voxel_shift, float eps, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sens_pose<decltype(v)>(vol, D0, D1, D2, src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps,
                                                 stream);
    });
}

int b200drr_siddon_fwd_sens_structures(const float* vol, const uint8_t* labels, int D0, int D1, int D2, const float* src,
                                       const float* G, const float* Wd, const float* rows, const float* cols,
                                       const int32_t* slot_of_label, const int32_t* box, float* out, float* sens, int B, int S,
                                       int H, int W, float voxel_shift, float eps, void* stream)
{
    return siddon_fwd_sens_structures<float>(vol, labels, D0, D1, D2, src, G, Wd, rows, cols, slot_of_label, box, out, sens, B, S, H,
                                             W, voxel_shift, eps, stream);
}

int b200drr_siddon_fwd_sens_structures_v16(const void* vol, int vol_type, const uint8_t* labels, int D0, int D1, int D2,
                                           const float* src, const float* G, const float* Wd, const float* rows, const float* cols,
                                           const int32_t* slot_of_label, const int32_t* box, float* out, float* sens, int B,
                                           int S, int H, int W, float voxel_shift, float eps, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return siddon_fwd_sens_structures<decltype(v)>(vol, labels, D0, D1, D2, src, G, Wd, rows, cols, slot_of_label, box, out,
                                                       sens, B, S, H, W, voxel_shift, eps, stream);
    });
}

int b200drr_pack_corners(const float* vol, int D0, int D1, int D2, float* packed, void* stream)
{
    return pack_corners<float>(vol, D0, D1, D2, packed, stream);
}

int b200drr_pack_corners_v16(const void* vol, int vol_type, int D0, int D1, int D2, void* packed, void* stream)
{
    return with_vox16(vol_type, [&](auto v) { return pack_corners<decltype(v)>(vol, D0, D1, D2, packed, stream); });
}

int b200drr_trilinear_fwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                          float* out, int B, int64_t N, float voxel_shift, float eps, int n_points, const float* alpha_range,
                          int reduce, int align_corners, void* stream)
{
    return trilinear_fwd<float>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, n_points, alpha_range, reduce,
                                align_corners, stream);
}

int b200drr_trilinear_fwd_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                              const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps, int n_points,
                              const float* alpha_range, int reduce, int align_corners, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, B, N, voxel_shift, eps, n_points, alpha_range,
                                          reduce, align_corners, stream);
    });
}

int b200drr_trilinear_fwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                               float* out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                               const float* alpha_range, int variant, void* stream)
{
    return trilinear_fwd_grid<float>(vol, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points, alpha_range,
                                     variant, stream);
}

int b200drr_trilinear_fwd_grid_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                   const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                   const float* alpha_range, int variant, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd_grid<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points,
                                               alpha_range, variant, stream);
    });
}

int b200drr_trilinear_fwd_sens(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                               float* out, float* sens, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                               const float* alpha_range, int align_corners, void* stream)
{
    return trilinear_fwd_sens<float>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, H, W, voxel_shift, eps, n_points,
                                     alpha_range, align_corners, stream);
}

int b200drr_trilinear_fwd_sens_v16(const void* vol, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                   const float* raylen, float* out, float* sens, int B, int64_t N, int H, int W, float voxel_shift,
                                   float eps, int n_points, const float* alpha_range, int align_corners, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd_sens<decltype(v)>(vol, D0, D1, D2, src, tgt, raylen, out, sens, B, N, H, W, voxel_shift, eps, n_points,
                                               alpha_range, align_corners, stream);
    });
}

int b200drr_trilinear_fwd_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                 const float* alpha_range, int slab, void* stream)
{
    return trilinear_fwd_packed<float>(packed, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points, alpha_range,
                                       slab, stream);
}

int b200drr_trilinear_fwd_packed_v16(const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                                     const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                     const float* alpha_range, int slab, void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd_packed<decltype(v)>(packed, D0, D1, D2, src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points,
                                                 alpha_range, slab, stream);
    });
}

int b200drr_trilinear_fwd_sens_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                      const float* raylen, float* out, float* sens, int B, int H, int W, float voxel_shift,
                                      float eps, int n_points, const float* alpha_range, int slab, void* stream)
{
    return trilinear_fwd_sens_packed<float>(packed, D0, D1, D2, src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps, n_points,
                                            alpha_range, slab, stream);
}

int b200drr_trilinear_fwd_sens_packed_v16(const void* packed, int vol_type, int D0, int D1, int D2, const float* src,
                                          const float* tgt, const float* raylen, float* out, float* sens, int B, int H, int W,
                                          float voxel_shift, float eps, int n_points, const float* alpha_range, int slab,
                                          void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd_sens_packed<decltype(v)>(packed, D0, D1, D2, src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps,
                                                      n_points, alpha_range, slab, stream);
    });
}

int b200drr_trilinear_fwd_sens_pose(const float* packed, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                                    const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                    float voxel_shift, float eps, int n_points, const float* alpha_range, int slab, void* stream)
{
    return trilinear_fwd_sens_pose<float>(packed, D0, D1, D2, src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps,
                                          n_points, alpha_range, slab, stream);
}

int b200drr_trilinear_fwd_sens_pose_v16(const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* G,
                                        const float* Wd, const float* rows, const float* cols, float* out, float* sens, int B, int H,
                                        int W, float voxel_shift, float eps, int n_points, const float* alpha_range, int slab,
                                        void* stream)
{
    return with_vox16(vol_type, [&](auto v) {
        return trilinear_fwd_sens_pose<decltype(v)>(packed, D0, D1, D2, src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps,
                                                    n_points, alpha_range, slab, stream);
    });
}

// ---- blended-rigid (skinned) trilinear render (polyrigid.cu) ----------------------------------------------------------------------
namespace {
// the geometry, lattice and map checks, without the volume
int polyrigid_geom_bad(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* M, int Bm, int K,
                       const float* weights, int g0, int g1, int g2, int B, int64_t N, int H, int W, int n_points,
                       const float* alpha_range)
{
    if (!src || !tgt || !raylen || !M || !weights || !alpha_range || bad_dims(D0, D1, D2) || bad_dims(g0, g1, g2) || bad_rays(B, N) ||
        K <= 0 || (Bm != 1 && Bm != B) || n_points < 2 || H < 0 || W < 0 || ((H > 0 || W > 0) && (int64_t)H * W != N) ||
        ((uintptr_t)weights & 15u) != 0)
        return B200DRR_EINVAL;
    if (K > 8 || too_big(D0, D1, D2) || (int64_t)g0 * g1 * g2 * polyrigid_channels(K) >= (int64_t)INT32_MAX)
        return B200DRR_EUNSUPPORTED;
    return 0;
}

// the checks every polyrigid entry point with a volume shares; 0 = go on
int polyrigid_bad(const void* vol, const void* packed, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                  const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2, int B, int64_t N, int H, int W,
                  int n_points, const float* alpha_range)
{
    if ((vol == nullptr) == (packed == nullptr) || ((uintptr_t)packed & 15u) != 0) return B200DRR_EINVAL;
    return polyrigid_geom_bad(D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, N, H, W, n_points, alpha_range);
}

// one body per fp32 entry point and its 16-bit twin; vol_type is 0 for an fp32 volume, as the launchers take it
int polyrigid_fwd(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                  const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2, float* out, int B,
                  int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!out) return B200DRR_EINVAL;
    if (const int bad = polyrigid_bad(vol, packed, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, N, H, W, n_points,
                                      alpha_range))
        return bad;
    return ret(launch_polyrigid_fwd(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, out, B, N,
                                    W, voxel_shift, eps, n_points, alpha_range, (cudaStream_t)stream));
}

int polyrigid_bwd(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                  const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2, const float* gout,
                  float* g_src, float* g_tgt, float* g_raylen, float* g_M, float* g_alpha_range, float* scratch, int B, int64_t N,
                  int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!gout || !scratch) return B200DRR_EINVAL;
    if (const int bad = polyrigid_bad(vol, packed, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, N, H, W, n_points,
                                      alpha_range))
        return bad;
    return ret(launch_polyrigid_bwd(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, g_src,
                                    g_tgt, g_raylen, g_M, g_alpha_range, scratch, B, N, W, voxel_shift, eps, n_points, alpha_range,
                                    (cudaStream_t)stream));
}

int polyrigid_jac(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                  const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2, const float* T,
                  float* img, float* J, int32_t* rects, int B, int H, int W, float voxel_shift, float eps, int n_points,
                  const float* alpha_range, void* stream)
{
    if (!T || !img || !J || !rects || H <= 0 || W <= 0) return B200DRR_EINVAL;
    if (const int bad = polyrigid_bad(vol, packed, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, B, (int64_t)H * W, H,
                                      W, n_points, alpha_range))
        return bad;
    return ret(launch_polyrigid_jac(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, T, img, J,
                                    rects, B, H, W, voxel_shift, eps, n_points, alpha_range, (cudaStream_t)stream));
}
}  // namespace

int64_t b200drr_polyrigid_weight_floats(int K, int g0, int g1, int g2)
{
    if (K <= 0 || K > 8 || bad_dims(g0, g1, g2)) return 0;
    return (int64_t)g0 * g1 * g2 * polyrigid_channels(K);
}

int b200drr_polyrigid_pack_weights(const float* weights, int K, int g0, int g1, int g2, float* packed, void* stream)
{
    if (!weights || !packed || K <= 0 || bad_dims(g0, g1, g2) || ((uintptr_t)packed & 15u) != 0) return B200DRR_EINVAL;
    if (K > 8 || b200drr_polyrigid_weight_floats(K, g0, g1, g2) >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_polyrigid_pack_weights(weights, K, g0, g1, g2, packed, (cudaStream_t)stream));
}

int64_t b200drr_polyrigid_scratch_floats(int B, int64_t N, int H, int W, int K)
{
    if (bad_rays(B, N) || K <= 0 || K > 8 || H < 0 || W < 0 || ((H > 0 || W > 0) && (int64_t)H * W != N)) return 0;
    return polyrigid_scratch_floats(B, N, W, K);
}

int b200drr_polyrigid_fwd(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                          const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2, float* out,
                          int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range,
                          void* stream)
{
    return polyrigid_fwd(vol, packed, 0, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, out, B, N, H, W, voxel_shift, eps,
                         n_points, alpha_range, stream);
}

int b200drr_polyrigid_fwd_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src,
                              const float* tgt, const float* raylen, const float* M, int Bm, int K, const float* weights, int g0,
                              int g1, int g2, float* out, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                              const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return polyrigid_fwd(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, out, B, N, H, W,
                         voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_polyrigid_bwd(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                          const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                          const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_M, float* g_alpha_range,
                          float* scratch, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                          const float* alpha_range, void* stream)
{
    return polyrigid_bwd(vol, packed, 0, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, g_src, g_tgt, g_raylen, g_M,
                         g_alpha_range, scratch, B, N, H, W, voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_polyrigid_bwd_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src,
                              const float* tgt, const float* raylen, const float* M, int Bm, int K, const float* weights, int g0,
                              int g1, int g2, const float* gout, float* g_src, float* g_tgt, float* g_raylen, float* g_M,
                              float* g_alpha_range, float* scratch, int B, int64_t N, int H, int W, float voxel_shift, float eps,
                              int n_points, const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return polyrigid_bwd(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, gout, g_src, g_tgt,
                         g_raylen, g_M, g_alpha_range, scratch, B, N, H, W, voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_polyrigid_jac(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                          const float* raylen, const float* M, int Bm, int K, const float* weights, int g0, int g1, int g2,
                          const float* T, float* img, float* J, int32_t* rects, int B, int H, int W, float voxel_shift, float eps,
                          int n_points, const float* alpha_range, void* stream)
{
    return polyrigid_jac(vol, packed, 0, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, T, img, J, rects, B, H, W,
                         voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_polyrigid_jac_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src,
                              const float* tgt, const float* raylen, const float* M, int Bm, int K, const float* weights, int g0,
                              int g1, int g2, const float* T, float* img, float* J, int32_t* rects, int B, int H, int W,
                              float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return polyrigid_jac(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, M, Bm, K, weights, g0, g1, g2, T, img, J, rects, B, H, W,
                         voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_polyrigid_bproj(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* M, int Bm,
                            int K, const float* wpacked, int g0, int g1, int g2, const float* gout, float* g_vol, int B, int64_t N,
                            int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!gout || !g_vol) return B200DRR_EINVAL;
    if (const int bad = polyrigid_geom_bad(D0, D1, D2, src, tgt, raylen, M, Bm, K, wpacked, g0, g1, g2, B, N, H, W, n_points,
                                           alpha_range))
        return bad;
    return ret(launch_polyrigid_bproj(mk(D0, D1, D2), src, tgt, raylen, M, Bm, K, wpacked, g0, g1, g2, gout, g_vol, B, N, W,
                                      voxel_shift, eps, n_points, alpha_range, (cudaStream_t)stream));
}

// ---- deformable (dense displacement field) trilinear render (deform.cu) ------------------------------------------------------------
namespace {
// the checks every deform entry point shares; 0 = go on
// the geometry and field checks, without the volume
int deform_geom_bad(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* field, int Bf, int g0,
                    int g1, int g2, int B, int64_t N, int H, int W, int n_points, const float* alpha_range)
{
    if (!src || !tgt || !raylen || !field || !alpha_range || bad_dims(D0, D1, D2) || bad_dims(g0, g1, g2) || bad_rays(B, N) ||
        (Bf != 1 && Bf != B) || n_points < 2 || H < 0 || W < 0 || ((H > 0 || W > 0) && (int64_t)H * W != N) ||
        ((uintptr_t)field & 15u) != 0)
        return B200DRR_EINVAL;
    if (too_big(D0, D1, D2) || (int64_t)g0 * g1 * g2 * 4 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return 0;
}

int deform_bad(const void* vol, const void* packed, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
               const float* field, int Bf, int g0, int g1, int g2, int B, int64_t N, int H, int W, int n_points, const float* alpha_range)
{
    if ((vol == nullptr) == (packed == nullptr) || ((uintptr_t)packed & 15u) != 0) return B200DRR_EINVAL;
    return deform_geom_bad(D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, H, W, n_points, alpha_range);
}

// one body per fp32 entry point and its 16-bit twin; vol_type is 0 for an fp32 volume, as the launchers take it
int deform_fwd(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
               const float* raylen, const float* field, int Bf, int g0, int g1, int g2, float* out, int B, int64_t N, int H, int W,
               float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!out) return B200DRR_EINVAL;
    if (const int bad = deform_bad(vol, packed, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, H, W, n_points, alpha_range))
        return bad;
    return ret(launch_deform_fwd(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, field, Bf, g0, g1, g2, out, B, N, W, voxel_shift,
                                 eps, n_points, alpha_range, (cudaStream_t)stream));
}

int deform_bwd(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
               const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* gout, float* g_src, float* g_tgt,
               float* g_raylen, float* g_field, float* g_alpha_range, float* scratch, int B, int64_t N, int H, int W, float voxel_shift,
               float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!gout || !scratch || ((uintptr_t)g_field & 15u) != 0) return B200DRR_EINVAL;
    if (const int bad = deform_bad(vol, packed, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, H, W, n_points, alpha_range))
        return bad;
    return ret(launch_deform_bwd(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, field, Bf, g0, g1, g2, gout, g_src, g_tgt,
                                 g_raylen, g_field, g_alpha_range, scratch, B, N, W, voxel_shift, eps, n_points, alpha_range,
                                 (cudaStream_t)stream));
}

int deform_jvp(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
               const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangent, float* img, float* jv, int B,
               int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!tangent || !jv || ((uintptr_t)tangent & 15u) != 0) return B200DRR_EINVAL;
    if (const int bad = deform_bad(vol, packed, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, H, W, n_points, alpha_range))
        return bad;
    return ret(launch_deform_jvp(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, field, Bf, g0, g1, g2, tangent, img, jv, B, N,
                                 W, voxel_shift, eps, n_points, alpha_range, (cudaStream_t)stream));
}

int deform_jac(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
               const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangents, int P, int K, float* img,
               float* J, int32_t* rects, int B, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range,
               void* stream)
{
    if (!tangents || !img || !J || !rects || H <= 0 || W <= 0 || P < 1 || P > 48 || P != 6 * K ||
        ((uintptr_t)tangents & 15u) != 0 || (const float*)img == tangents || (const float*)J == tangents)
        return B200DRR_EINVAL;
    if (K > 8 || (int64_t)g0 * g1 * g2 * 4 * P >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    if (const int bad = deform_bad(vol, packed, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, (int64_t)H * W, H, W, n_points,
                                   alpha_range))
        return bad;
    return ret(launch_deform_jac(vol, packed, vol_type, mk(D0, D1, D2), src, tgt, raylen, field, Bf, g0, g1, g2, tangents, K, img, J,
                                 rects, B, H, W, voxel_shift, eps, n_points, alpha_range, (cudaStream_t)stream));
}
}  // namespace

int64_t b200drr_deform_scratch_floats(int B, int64_t N, int H, int W)
{
    if (bad_rays(B, N) || H < 0 || W < 0 || ((H > 0 || W > 0) && (int64_t)H * W != N)) return 0;
    return deform_scratch_floats(B, N, W);
}

int b200drr_deform_fwd(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, const float* field, int Bf, int g0, int g1, int g2, float* out, int B, int64_t N, int H,
                       int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    return deform_fwd(vol, packed, 0, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, out, B, N, H, W, voxel_shift, eps, n_points,
                      alpha_range, stream);
}

int b200drr_deform_fwd_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                           const float* raylen, const float* field, int Bf, int g0, int g1, int g2, float* out, int B, int64_t N, int H,
                           int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return deform_fwd(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, out, B, N, H, W, voxel_shift, eps,
                      n_points, alpha_range, stream);
}

int b200drr_deform_bwd(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* gout, float* g_src,
                       float* g_tgt, float* g_raylen, float* g_field, float* g_alpha_range, float* scratch, int B, int64_t N, int H,
                       int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    return deform_bwd(vol, packed, 0, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, gout, g_src, g_tgt, g_raylen, g_field,
                      g_alpha_range, scratch, B, N, H, W, voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_deform_bwd_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                           const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* gout, float* g_src,
                           float* g_tgt, float* g_raylen, float* g_field, float* g_alpha_range, float* scratch, int B, int64_t N, int H,
                           int W, float voxel_shift, float eps, int n_points, const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return deform_bwd(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, gout, g_src, g_tgt, g_raylen, g_field,
                      g_alpha_range, scratch, B, N, H, W, voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_deform_jvp(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangent, float* img,
                       float* jv, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points, const float* alpha_range,
                       void* stream)
{
    return deform_jvp(vol, packed, 0, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, tangent, img, jv, B, N, H, W, voxel_shift,
                      eps, n_points, alpha_range, stream);
}

int b200drr_deform_jvp_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                           const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangent, float* img,
                           float* jv, int B, int64_t N, int H, int W, float voxel_shift, float eps, int n_points,
                           const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return deform_jvp(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, tangent, img, jv, B, N, H, W,
                      voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_deform_jac(const float* vol, const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangents, int P, int K,
                       float* img, float* J, int32_t* rects, int B, int H, int W, float voxel_shift, float eps, int n_points,
                       const float* alpha_range, void* stream)
{
    return deform_jac(vol, packed, 0, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, tangents, P, K, img, J, rects, B, H, W,
                      voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_deform_jac_v16(const void* vol, const void* packed, int vol_type, int D0, int D1, int D2, const float* src, const float* tgt,
                           const float* raylen, const float* field, int Bf, int g0, int g1, int g2, const float* tangents, int P, int K,
                           float* img, float* J, int32_t* rects, int B, int H, int W, float voxel_shift, float eps, int n_points,
                           const float* alpha_range, void* stream)
{
    if (bad_vol16(vol_type)) return B200DRR_EINVAL;
    return deform_jac(vol, packed, vol_type, D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, tangents, P, K, img, J, rects, B, H, W,
                      voxel_shift, eps, n_points, alpha_range, stream);
}

int b200drr_deform_bproj(int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen, const float* field, int Bf,
                         int g0, int g1, int g2, const float* gout, float* g_vol, int B, int64_t N, int H, int W, float voxel_shift,
                         float eps, int n_points, const float* alpha_range, void* stream)
{
    if (!gout || !g_vol) return B200DRR_EINVAL;
    if (const int bad = deform_geom_bad(D0, D1, D2, src, tgt, raylen, field, Bf, g0, g1, g2, B, N, H, W, n_points, alpha_range))
        return bad;
    return ret(launch_deform_bproj(mk(D0, D1, D2), src, tgt, raylen, field, Bf, g0, g1, g2, gout, g_vol, B, N, W, voxel_shift, eps,
                                   n_points, alpha_range, (cudaStream_t)stream));
}

// ---- scaling and squaring of a stationary velocity field (svf.cu) ------------------------------------------------------------------
namespace {
// the checks every svf entry point shares; 0 = go on
int svf_bad(const float* field, const float* out, int Bf, int g0, int g1, int g2, int D0, int D1, int D2, float scale)
{
    if (!field || !out || Bf <= 0 || bad_dims(g0, g1, g2) || bad_dims(D0, D1, D2) || !(scale > 0.0f) ||
        (((uintptr_t)field | (uintptr_t)out) & 15u) != 0)
        return B200DRR_EINVAL;
    if ((int64_t)g0 * g1 * g2 * 4 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return 0;
}
}  // namespace

int b200drr_svf_square(const float* field, float* out, int Bf, int g0, int g1, int g2, int D0, int D1, int D2, float scale, void* stream)
{
    if (const int bad = svf_bad(field, out, Bf, g0, g1, g2, D0, D1, D2, scale)) return bad;
    if (field == out) return B200DRR_EINVAL;
    return ret(launch_svf_square(field, out, Bf, g0, g1, g2, mk(D0, D1, D2), scale, (cudaStream_t)stream));
}

int b200drr_svf_square_bwd(const float* field, const float* gout, float* gin, int Bf, int g0, int g1, int g2, int D0, int D1, int D2,
                           float scale, void* stream)
{
    if (!gout || (((uintptr_t)gout & 15u) != 0)) return B200DRR_EINVAL;
    if (const int bad = svf_bad(field, gin, Bf, g0, g1, g2, D0, D1, D2, scale)) return bad;
    if (gin == field || gin == gout) return B200DRR_EINVAL;
    return ret(launch_svf_square_bwd(field, gout, gin, Bf, g0, g1, g2, mk(D0, D1, D2), scale, (cudaStream_t)stream));
}

int b200drr_svf_square_jvp(const float* field, const float* tangent, float* tout, float* out, int Bf, int g0, int g1, int g2, int D0,
                           int D1, int D2, float scale, void* stream)
{
    if (!tangent || (((uintptr_t)tangent | (uintptr_t)out) & 15u) != 0) return B200DRR_EINVAL;
    if (const int bad = svf_bad(field, tout, Bf, g0, g1, g2, D0, D1, D2, scale)) return bad;
    if (tout == field || tout == tangent || out == field || out == tangent || out == tout) return B200DRR_EINVAL;
    return ret(launch_svf_square_jvp(field, tangent, tout, out, Bf, g0, g1, g2, mk(D0, D1, D2), scale, (cudaStream_t)stream));
}

int b200drr_svf_square_tangents(const float* field, const float* tangents, float* tout, float* out, int Bf, int P, int g0, int g1, int g2,
                                int D0, int D1, int D2, float scale, void* stream)
{
    if (!tangents || P < 1 || P > 48 || (((uintptr_t)tangents | (uintptr_t)out) & 15u) != 0) return B200DRR_EINVAL;
    if (const int bad = svf_bad(field, tout, Bf, g0, g1, g2, D0, D1, D2, scale)) return bad;
    if (tout == field || tout == tangents || out == field || out == tangents || out == tout) return B200DRR_EINVAL;
    if ((int64_t)g0 * g1 * g2 * 4 * P >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_svf_square_tangents(field, tangents, tout, out, Bf, P, g0, g1, g2, mk(D0, D1, D2), scale, (cudaStream_t)stream));
}

#ifdef B200DRR_EXPERIMENTS
int b200drr_x_transpose_volume(const float* vol, int D0, int D1, int D2, int axis, float* out, void* stream)
{
    if (!vol || !out || bad_dims(D0, D1, D2) || axis < 0 || axis > 2) return B200DRR_EINVAL;
    return ret(launch_x_transpose_volume(vol, mk(D0, D1, D2), axis, out, (cudaStream_t)stream));
}

int b200drr_x_siddon_fwd_chunk(const float* volT, int D0, int D1, int D2, int axis, const float* src, const float* tgt,
                               const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps,
                               int variant, void* stream)
{
    if (!volT || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || axis < 0 || axis > 2 ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_x_siddon_fwd_chunk(volT, mk(D0, D1, D2), axis, src, tgt, raylen, out, B, H, W, voxel_shift, eps, variant,
                                         (cudaStream_t)stream));
}

int b200drr_x_siddon_sens_chunk(const float* volT, int D0, int D1, int D2, int axis, const float* src, const float* tgt,
                                const float* raylen, float* out, float* sens, int B, int H, int W, float voxel_shift,
                                float eps, int variant, void* stream)
{
    if (!volT || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || axis < 0 || axis > 2 ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_x_siddon_sens_chunk(volT, mk(D0, D1, D2), axis, src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps,
                                          variant, (cudaStream_t)stream));
}
#endif  // B200DRR_EXPERIMENTS

int64_t b200drr_packed_volume_floats(int D0, int D1, int D2)
{
    if (bad_dims(D0, D1, D2)) return 0;
    return (int64_t)(D0 + 1) * (D1 + 1) * (D2 + 1) * 8;
}

int b200drr_trilinear_bwd_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                 float* g_alpha_range, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                 const float* alpha_range, int slab, void* stream)
{
    if (!packed || slab < 0 || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_grid(B, H, W) || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_packed(packed, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen,
                                           g_alpha_range, B, H, W, voxel_shift, eps, n_points, alpha_range, slab,
                                           (cudaStream_t)stream));
}

int b200drr_siddon_visits(int D0, int D1, int D2, const float* src, const float* tgt, int32_t* visits, int B,
                          int64_t N, float voxel_shift, float eps, void* stream)
{
    if (!src || !tgt || !visits || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    return ret(launch_siddon_visits(mk(D0, D1, D2), src, tgt, visits, B, N, voxel_shift, eps, (cudaStream_t)stream));
}

int64_t b200drr_ncc_workspace_bytes(int B, int C, int64_t N)
{
    if (B <= 0 || C <= 0 || N <= 0) return 0;
    return ncc_workspace_bytes(B, C, N);
}

int b200drr_ncc_fwd(const float* x1, const float* x2, int B, int C, int64_t N, float eps, void* workspace, float* stats,
                    float* score, void* stream)
{
    if (!x1 || !x2 || !workspace || !stats || !score || B <= 0 || C <= 0 || N <= 0 || (int64_t)B * C > 65535) return B200DRR_EINVAL;
    return ret(launch_ncc_fwd(x1, x2, B, C, N, eps, workspace, stats, score, (cudaStream_t)stream));
}

int b200drr_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2, int B,
                    int C, int64_t N, void* stream)
{
    if (!x1 || !x2 || !stats || !gscore || (!g_x1 && !g_x2) || B <= 0 || C <= 0 || N <= 0 || (int64_t)B * C > 65535)
        return B200DRR_EINVAL;
    return ret(launch_ncc_bwd(x1, x2, stats, gscore, g_x1, g_x2, B, C, N, (cudaStream_t)stream));
}

static bool bad_local_ncc(int B, int C, int H, int W, int p)
{
    return B <= 0 || C <= 0 || H <= 0 || W <= 0 || p < 1 || p > H || p > W || (int64_t)B * C > 65535;
}

int64_t b200drr_local_ncc_workspace_bytes(int B, int C, int H, int W, int p)
{
    if (bad_local_ncc(B, C, H, W, p)) return 0;
    return local_ncc_workspace_bytes(B, C, H, W, p);
}

int b200drr_local_ncc_fwd(const float* x1, const float* x2, int B, int C, int H, int W, int p, float eps, void* workspace,
                          float* stats, float* score, void* stream)
{
    if (!x1 || !x2 || !workspace || !stats || !score || bad_local_ncc(B, C, H, W, p)) return B200DRR_EINVAL;
    return ret(launch_local_ncc_fwd(x1, x2, B, C, H, W, p, eps, workspace, stats, score, (cudaStream_t)stream));
}

int b200drr_local_ncc_bwd(const float* x1, const float* x2, const float* stats, const float* gscore, float* g_x1, float* g_x2, int B,
                          int C, int H, int W, int p, void* workspace, void* stream)
{
    if (!x1 || !x2 || !stats || !gscore || (!g_x1 && !g_x2) || !workspace || bad_local_ncc(B, C, H, W, p)) return B200DRR_EINVAL;
    return ret(launch_local_ncc_bwd(x1, x2, stats, gscore, g_x1, g_x2, B, C, H, W, p, workspace, (cudaStream_t)stream));
}

static bool bad_ncc_normal(int B, int C, int H, int W, int p, int P)
{
    return B <= 0 || C <= 0 || H <= 0 || W <= 0 || p < 0 || p > H || p > W || P < 1 || P > 16 || (int64_t)B * C > 65535;
}

int64_t b200drr_ncc_normal_workspace_bytes(int B, int C, int H, int W, int p, int P)
{
    if (bad_ncc_normal(B, C, H, W, p, P)) return 0;
    return ncc_normal_workspace_bytes(B, C, H, W, p, P);
}

int b200drr_ncc_normal(const float* x, const float* t, const float* J, int64_t sJb, int64_t sJc, int64_t sJk, int64_t sJn, int B,
                       int C, int H, int W, int p, int P, double eps, double weight, void* workspace, double* A, double* g,
                       void* stream)
{
    if (!x || !t || !J || !workspace || !A || !g || sJb < 0 || sJc < 0 || sJk < 0 || sJn < 0 || !(eps >= 0.0) ||
        bad_ncc_normal(B, C, H, W, p, P))
        return B200DRR_EINVAL;
    return ret(launch_ncc_normal(x, t, J, sJb, sJc, sJk, sJn, B, C, H, W, p, P, eps, weight, workspace, A, g, (cudaStream_t)stream));
}

int b200drr_structure_footprints(const float* src, const float* G, const float* rows, const float* cols, const int32_t* box,
                                 int32_t* rects, int B, int S, int H, int W, float voxel_shift, void* stream)
{
    if (!src || !G || !rows || !cols || !box || !rects || B <= 0 || S <= 0 || S > 256 || (int64_t)B * S > INT32_MAX || H <= 0 ||
        W <= 0)
        return B200DRR_EINVAL;
    return ret(launch_structure_footprints(src, G, rows, cols, box, rects, B, S, H, W, voxel_shift, (cudaStream_t)stream));
}

static bool bad_ncc_normal_structures(int B, int K, int H, int W)
{
    return B <= 0 || B > 65535 || K < 1 || K > 255 || H <= 0 || W <= 0;
}

int64_t b200drr_ncc_normal_structures_workspace_bytes(int B, int K, int H, int W)
{
    if (bad_ncc_normal_structures(B, K, H, W)) return 0;
    return ncc_normal_structures_workspace_bytes(B, K, H);
}

int b200drr_ncc_normal_structures(const float* x, const float* t, int t_batch, const float* J, int64_t sJb, int64_t sJs, int64_t sJn,
                                  int64_t sJk, const int32_t* rects, int B, int K, int S, int H, int W, double eps, double weight,
                                  void* workspace, double* A, double* g, void* stream)
{
    if (!x || !t || !J || !rects || !workspace || !A || !g || sJb < 0 || sJs < 0 || sJn < 0 || sJk < 0 || !(eps >= 0.0) ||
        bad_ncc_normal_structures(B, K, H, W) || S < K || S > 256 || (t_batch != 1 && t_batch != B))
        return B200DRR_EINVAL;
    return ret(launch_ncc_normal_structures(x, t, t_batch, J, sJb, sJs, sJn, sJk, rects, B, K, S, H, W, eps, weight, workspace, A, g,
                                            (cudaStream_t)stream));
}

// odd kernel size, blur radius below both image sides (reflect padding), shared-memory tiles that fit
static bool bad_sobel(int B, int H, int W, int ksize)
{
    return B <= 0 || B > 65535 || H <= 0 || W <= 0 || ksize <= 0 || (ksize & 1) == 0 || ksize / 2 >= H || ksize / 2 >= W ||
           !sobel_kernel_fits(ksize);
}

int64_t b200drr_sobel_workspace_bytes(int B, int H, int W)
{
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    return sobel_workspace_bytes(B, H, W);
}

int b200drr_sobel_fwd(const float* x, float* out, int B, int H, int W, const float* weights, int ksize, void* stream)
{
    if (!x || !out || !weights || bad_sobel(B, H, W, ksize)) return B200DRR_EINVAL;
    return ret(launch_sobel_fwd(x, out, B, H, W, weights, ksize, (cudaStream_t)stream));
}

int b200drr_sobel_bwd(const float* gout, float* g_x, int B, int H, int W, const float* weights, int ksize, void* workspace,
                      void* stream)
{
    if (!gout || !g_x || !weights || !workspace || bad_sobel(B, H, W, ksize)) return B200DRR_EINVAL;
    return ret(launch_sobel_bwd(gout, g_x, B, H, W, weights, ksize, workspace, (cudaStream_t)stream));
}

// one-channel images of N < 2^31 pixels, 2 <= num_bins <= 256
static bool bad_mi(int B, int64_t N, int nb) { return B <= 0 || B > 65535 || N <= 0 || N >= ((int64_t)1 << 31) || nb < 2 || nb > 256; }

int64_t b200drr_mi_workspace_bytes(int B, int64_t N, int num_bins)
{
    if (bad_mi(B, N, num_bins)) return 0;
    return mi_workspace_bytes(B, N, num_bins);
}

int b200drr_mi_fwd(const float* x1, const float* x2, int B, int64_t N, const float* bins, const float* sigma, int num_bins,
                   double epsilon, int normalize, void* workspace, float* stats, float* score, void* stream)
{
    if (!x1 || !x2 || !bins || !sigma || !workspace || !stats || !score || bad_mi(B, N, num_bins)) return B200DRR_EINVAL;
    return ret(launch_mi_fwd(x1, x2, B, N, bins, sigma, num_bins, epsilon, normalize, workspace, stats, score, (cudaStream_t)stream));
}

int b200drr_mi_bwd(const float* x1, const float* x2, const float* bins, const float* sigma, const float* stats, const float* gscore,
                   float* g_x1, float* g_x2, int B, int64_t N, int num_bins, void* stream)
{
    if (!x1 || !x2 || !bins || !sigma || !stats || !gscore || (!g_x1 && !g_x2) || bad_mi(B, N, num_bins)) return B200DRR_EINVAL;
    return ret(launch_mi_bwd(x1, x2, bins, sigma, stats, gscore, g_x1, g_x2, B, N, num_bins, (cudaStream_t)stream));
}

}  // extern "C"
