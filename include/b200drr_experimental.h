/*
 * b200drr_experimental.h -- entry points of REJECTED kernel experiments (prefix b200drr_x_).  They are NOT part of
 * libb200drr.so: build the experimental library with `B200DRR_BUILD_EXPERIMENTS=1 python -m diffdrr_b200.build`
 * (-DB200DRR_EXPERIMENTS) to time them again with scripts/tune_siddon.py.  Measured slower than the
 * production kernels on the predecessor GPU and rejected (not re-measured on the H100); kept as documented negative results.
 */
#ifndef B200DRR_EXPERIMENTAL_H
#define B200DRR_EXPERIMENTAL_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/*
 * EXPERIMENTAL (prefix b200drr_x_: may change or disappear; used by scripts/tune_siddon.py only, never by the module).
 * REJECTED (slower than the production kernels; not re-measured on the H100); kept, like
 * the plane-synchronous walk, as a documented negative result.
 * Chunk-reuse Siddon forward: the lean walk over a copy of the volume whose FASTEST axis is the rays' major axis, so a
 * lane serves several consecutive visits from one LDG.64 / LDG.128 (DESIGN.md 8).  b200drr_x_transpose_volume writes that
 * copy: out [D_p][D_q][D_axis] (p < q the other two axes), D0*D1*D2 + 4 floats (4 floats of padding).  Results are bitwise
 * those of b200drr_siddon_fwd_grid with the same slab height.
 */
int b200drr_x_transpose_volume(const float *vol, int D0, int D1, int D2, int axis, float *out, void *stream);
int b200drr_x_siddon_fwd_chunk(const float *volT, int D0, int D1, int D2, int axis, const float *src, const float *tgt,
                               const float *raylen, float *out, int B, int H, int W, float voxel_shift, float eps,
                               int variant, void *stream);
/* the same for the forward-with-sensitivities walk (outputs as b200drr_siddon_fwd_sens_grid) */
int b200drr_x_siddon_sens_chunk(const float *volT, int D0, int D1, int D2, int axis, const float *src, const float *tgt,
                                const float *raylen, float *out, float *sens, int B, int H, int W, float voxel_shift,
                                float eps, int variant, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* B200DRR_EXPERIMENTAL_H */
