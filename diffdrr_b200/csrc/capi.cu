// capi.cu -- the C ABI of libb200drr.so (see include/b200drr.h for the contract of every entry point).
#include <cuda_runtime.h>

#include "../../include/b200drr.h"
#ifdef B200DRR_EXPERIMENTS
#include "../../include/b200drr_experimental.h"
#endif
#include "kernels.h"

using namespace b200drr;

namespace {

inline bool bad_dims(int D0, int D1, int D2) { return D0 <= 0 || D1 <= 0 || D2 <= 0; }
inline bool bad_rays(int B, int64_t N) { return B <= 0 || B > 65535 || N <= 0; }
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

int b200drr_siddon_fwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                       const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps, int reduce,
                       int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N) || reduce < 0 || reduce > 1)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, reduce,
                                 align_corners != 0, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                            const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps,
                            int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps, variant,
                                      (cudaStream_t)stream));
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

int b200drr_siddon_fwd_sorted(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                              float* out, int B, int64_t N, float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sorted(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_sens_sorted(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                                   const float* raylen, float* out, float* sens, int B, int64_t N, float voxel_shift, float eps,
                                   void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_sorted(vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, voxel_shift, eps,
                                             (cudaStream_t)stream));
}

int64_t b200drr_siddon_brick_workspace_bytes(int B, int H, int W)
{
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    return (int64_t)siddon_brick_workspace_bytes(B, H, W);
}

int b200drr_siddon_fwd_brick(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                             const float* raylen, const float* G, const float* Wd, const float* rows, const float* cols,
                             float* out, void* workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift,
                             float eps, int variant, void* stream)
{
    const bool pose_in = G != nullptr;
    if (!vol || !src || !out || !workspace || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if (pose_in ? (!Wd || !rows || !cols) : (!tgt || !raylen)) return B200DRR_EINVAL;
    if (!siddon_brick_supported(mk(D0, D1, D2), H, W) || ((uintptr_t)vol & 15u) != 0) return B200DRR_EUNSUPPORTED;
    if (workspace_bytes < (int64_t)siddon_brick_workspace_bytes(B, H, W) || ((uintptr_t)workspace & 255u) != 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd_brick(vol, mk(D0, D1, D2), src, tgt, raylen, G, Wd, rows, cols, out, workspace,
                                       (size_t)workspace_bytes, B, H, W, voxel_shift, eps, variant, (cudaStream_t)stream));
}

int b200drr_siddon_bwd_vol_brick(const float* gout, int D0, int D1, int D2, const float* src, const float* tgt, const float* raylen,
                                 const float* G, const float* Wd, const float* rows, const float* cols, float* g_vol,
                                 void* workspace, int64_t workspace_bytes, int B, int H, int W, float voxel_shift, float eps,
                                 void* stream)
{
    const bool pose_in = G != nullptr;
    if (!gout || !src || !g_vol || !workspace || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if (pose_in ? (!Wd || !rows || !cols) : (!tgt || !raylen)) return B200DRR_EINVAL;
    if (!siddon_brick_supported(mk(D0, D1, D2), H, W) || ((uintptr_t)g_vol & 15u) != 0) return B200DRR_EUNSUPPORTED;
    if (workspace_bytes < (int64_t)siddon_brick_workspace_bytes(B, H, W) || ((uintptr_t)workspace & 255u) != 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_vol_brick(gout, mk(D0, D1, D2), src, tgt, raylen, G, Wd, rows, cols, g_vol, workspace,
                                           (size_t)workspace_bytes, B, H, W, voxel_shift, eps, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_brick_subset(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                                    const float* raylen, const int32_t* pix_index, const float* corners, float* out,
                                    void* workspace, int64_t workspace_bytes, int B, int H, int W, int64_t Nsub,
                                    float voxel_shift, float eps, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !pix_index || !corners || !out || !workspace || bad_dims(D0, D1, D2) ||
        bad_rays(B, Nsub) || H <= 0 || W <= 0 || Nsub > (int64_t)H * W)
        return B200DRR_EINVAL;
    if (!siddon_brick_supported(mk(D0, D1, D2), H, W) || ((uintptr_t)vol & 15u) != 0) return B200DRR_EUNSUPPORTED;
    if (workspace_bytes < (int64_t)siddon_brick_workspace_bytes(B, 1, (int)Nsub) || ((uintptr_t)workspace & 255u) != 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_fwd_brick(vol, mk(D0, D1, D2), src, tgt, raylen, nullptr, nullptr, nullptr, nullptr, out, workspace,
                                       (size_t)workspace_bytes, B, H, W, voxel_shift, eps, variant, (cudaStream_t)stream,
                                       pix_index, corners, Nsub));
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
    if (!vol || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B, H, W,
                                      voxel_shift, eps, stop_grad != 0, variant, (cudaStream_t)stream));
}

int b200drr_trilinear_fwd(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                          const float* raylen, float* out, int B, int64_t N, float voxel_shift, float eps,
                          int n_points, const float* alpha_range, int reduce, int align_corners, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        n_points < 2 || reduce < 0 || reduce > 1)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, N, voxel_shift, eps, n_points,
                                    alpha_range, reduce, align_corners != 0, (cudaStream_t)stream));
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

int b200drr_trilinear_fwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps,
                               int n_points, const float* alpha_range, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) ||
        H <= 0 || W <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps, n_points,
                                         alpha_range, variant, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                               float* g_vol, float* g_alpha_range, int B, int H, int W, float voxel_shift, float eps,
                               int n_points, const float* alpha_range, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) ||
        H <= 0 || W <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_grid(vol, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol,
                                         g_alpha_range, B, H, W, voxel_shift, eps, n_points, alpha_range, variant,
                                         (cudaStream_t)stream));
}

int b200drr_siddon_fwd_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                            const float* rows, const float* cols, float* out, int B, int H, int W, float voxel_shift,
                            float eps, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !out || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) ||
        H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_pose(vol, mk(D0, D1, D2), src, G, Wd, rows, cols, out, B, H, W, voxel_shift, eps,
                                      (cudaStream_t)stream));
}

int b200drr_siddon_bwd_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                            const float* rows, const float* cols, const float* gout, float* g_src, float* g_G, float* g_Wd,
                            float* g_vol, float* ws_tgt, float* ws_len, int B, int H, int W, float voxel_shift, float eps,
                            int stop_grad, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !gout || !g_src || !g_G || !g_Wd || !ws_tgt || !ws_len ||
        bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_bwd_pose(vol, mk(D0, D1, D2), src, G, Wd, rows, cols, gout, g_src, g_G, g_Wd, g_vol, ws_tgt,
                                      ws_len, B, H, W, voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_sens(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                            const float* raylen, float* out, float* sens, int B, int64_t N, float voxel_shift, float eps,
                            void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_rays(B, N)) return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens(vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, voxel_shift, eps,
                                      (cudaStream_t)stream));
}

int b200drr_siddon_fwd_sens_grid(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, float* out, float* sens, int B, int H, int W, float voxel_shift,
                                 float eps, int variant, void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || bad_dims(D0, D1, D2) || bad_rays(B, (int64_t)H * W) || H <= 0 ||
        W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_grid(vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps,
                                           variant, (cudaStream_t)stream));
}

int b200drr_siddon_fwd_sens_pose(const float* vol, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                                 const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                 float voxel_shift, float eps, void* stream)
{
    if (!vol || !src || !G || !Wd || !rows || !cols || !out || !sens || bad_dims(D0, D1, D2) ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_sens_pose(vol, mk(D0, D1, D2), src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps,
                                           (cudaStream_t)stream));
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
    if (!sens || !gout || !Wd || !rows || !cols || !g_src || !g_G || !g_Wd || H <= 0 || W <= 0 ||
        bad_rays(B, (int64_t)H * W))
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_sens_pose(sens, gout, Wd, rows, cols, g_src, g_G, g_Wd, B, H, W, stop_grad != 0,
                                           (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_sens(const float* vol, int D0, int D1, int D2, const float* src, const float* tgt,
                               const float* raylen, float* out, float* sens, int B, int64_t N, int H, int W,
                               float voxel_shift, float eps, int n_points, const float* alpha_range, int align_corners,
                               void* stream)
{
    if (!vol || !src || !tgt || !raylen || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) || bad_rays(B, N) ||
        n_points < 2 || H < 0 || W < 0 || (H > 0 && ((int64_t)H * W != N || align_corners)))
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_sens(vol, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, N, H, W, voxel_shift, eps,
                                         n_points, alpha_range, align_corners != 0, (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_sens_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                      const float* raylen, float* out, float* sens, int B, int H, int W, float voxel_shift,
                                      float eps, int n_points, const float* alpha_range, int slab, void* stream)
{
    if (!packed || !src || !tgt || !raylen || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0 || n_points < 2 || slab < 0)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_sens_packed(packed, mk(D0, D1, D2), src, tgt, raylen, out, sens, B, H, W, voxel_shift, eps,
                                                n_points, alpha_range, slab, (cudaStream_t)stream));
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
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_alpha_range_pose(mk(D0, D1, D2), src, G, Wd, rows, cols, range, arg, scratch16, B, H, W, voxel_shift,
                                                 eps, (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_sens_pose(const float* packed, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                                    const float* rows, const float* cols, float* out, float* sens, int B, int H, int W,
                                    float voxel_shift, float eps, int n_points, const float* alpha_range, int slab, void* stream)
{
    if (!packed || !src || !G || !Wd || !rows || !cols || !out || !sens || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0 || n_points < 2 || slab < 0)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_sens_pose(packed, mk(D0, D1, D2), src, G, Wd, rows, cols, out, sens, B, H, W, voxel_shift, eps,
                                              n_points, alpha_range, slab, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_sens_pose(const float* sens, const float* gout, const float* Wd, const float* rows, const float* cols,
                                    float* g_src, float* g_G, float* g_Wd, float* g_alpha_range, int B, int H, int W, void* stream)
{
    if (!sens || !gout || !Wd || !rows || !cols || !g_src || !g_G || !g_Wd || bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_bwd_sens_pose(sens, gout, Wd, rows, cols, g_src, g_G, g_Wd, g_alpha_range, B, H, W,
                                              (cudaStream_t)stream));
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
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
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
    if (!vol || !mask || !src || !tgt || !raylen || !out || bad_dims(D0, D1, D2) || H <= 0 || W <= 0 ||
        bad_rays(B, (int64_t)H * W) || C <= 0)
        return B200DRR_EINVAL;
    if ((int64_t)D0 * D1 * D2 >= (int64_t)INT32_MAX) return B200DRR_EUNSUPPORTED;
    return ret(launch_siddon_fwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, out, B, (int64_t)H * W, C, voxel_shift, eps,
                                      (cudaStream_t)stream, W));
}

int b200drr_trilinear_fwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src,
                                    const float* tgt, const float* raylen, float* out, int B, int H, int W, int C,
                                    float voxel_shift, float eps, int n_points, const float* alpha_range, int align_corners,
                                    void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) || H <= 0 || W <= 0 ||
        bad_rays(B, (int64_t)H * W) || C <= 0 || n_points < 2)
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
    if (!vol || !mask || !src || !tgt || !raylen || !gout || bad_dims(D0, D1, D2) || H <= 0 || W <= 0 ||
        bad_rays(B, (int64_t)H * W) || C <= 0)
        return B200DRR_EINVAL;
    return ret(launch_siddon_bwd_mask(vol, mask, mk(D0, D1, D2), src, tgt, raylen, gout, g_src, g_tgt, g_raylen, g_vol, B,
                                      (int64_t)H * W, C, voxel_shift, eps, stop_grad != 0, (cudaStream_t)stream, W));
}

int b200drr_trilinear_bwd_mask_grid(const float* vol, const float* mask, int D0, int D1, int D2, const float* src, const float* tgt,
                                    const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                    float* g_vol, float* g_alpha_range, int B, int H, int W, int C, float voxel_shift, float eps,
                                    int n_points, const float* alpha_range, int align_corners, void* stream)
{
    if (!vol || !mask || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) || H <= 0 || W <= 0 ||
        bad_rays(B, (int64_t)H * W) || C <= 0 || n_points < 2)
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

int b200drr_pack_corners(const float* vol, int D0, int D1, int D2, float* packed, void* stream)
{
    if (!vol || !packed || bad_dims(D0, D1, D2)) return B200DRR_EINVAL;
    return ret(launch_pack_corners(vol, mk(D0, D1, D2), packed, (cudaStream_t)stream));
}

int b200drr_trilinear_fwd_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, float* out, int B, int H, int W, float voxel_shift, float eps,
                                 int n_points, const float* alpha_range, int slab, void* stream)
{
    if (!packed || slab < 0 || !src || !tgt || !raylen || !out || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0 || n_points < 2)
        return B200DRR_EINVAL;
    return ret(launch_trilinear_fwd_packed(packed, mk(D0, D1, D2), src, tgt, raylen, out, B, H, W, voxel_shift, eps,
                                           n_points, alpha_range, slab, (cudaStream_t)stream));
}

int b200drr_trilinear_bwd_packed(const float* packed, int D0, int D1, int D2, const float* src, const float* tgt,
                                 const float* raylen, const float* gout, float* g_src, float* g_tgt, float* g_raylen,
                                 float* g_alpha_range, int B, int H, int W, float voxel_shift, float eps, int n_points,
                                 const float* alpha_range, int slab, void* stream)
{
    if (!packed || slab < 0 || !src || !tgt || !raylen || !gout || !alpha_range || bad_dims(D0, D1, D2) ||
        bad_rays(B, (int64_t)H * W) || H <= 0 || W <= 0 || n_points < 2)
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

}  // extern "C"
