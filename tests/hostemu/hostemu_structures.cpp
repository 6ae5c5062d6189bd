// hostemu_structures.cpp -- TEST INFRASTRUCTURE: the piecewise-rigid render of csrc/structures.cu compiled for the CPU.  Per
// (pose, slot) the footprint rectangle of the slot's box (box_corner_uv + footprint_rect), per pixel the pose-in ray (pose_ray, the
// function make_ray calls) and the gated walk over the box (siddon_ray_sens_box / siddon_ray_lean_box with LoadGated), written as
// the kernel writes it; and the label boxes from the label runs of every row.  Never linked into libb200drr.so.
#include <algorithm>
#include <climits>
#include <cstring>

#include "../../diffdrr_b200/csrc/structures_math.cuh"

using namespace b200drr;

extern "C" {

// out [B*S][H*W], sens [B*S][H*W][8] (NULL: the image only, through the forward walk) overwritten; rects [B*S][4] = the footprint
// rectangles {w0, w1, h0, h1}.  cull = 0 walks every pixel (the reference for the culling).
void emu_structures(const float* vol, const uint8_t* labels, int D0, int D1, int D2, const float* src, const float* G, const float* Wd,
                    const float* rows, const float* cols, const int* slot_of_label, const int* box, float* out, float* sens,
                    int* rects, int B, int S, int H, int W, float shift, float eps, int cull)
{
    VolDims dims;
    dims.d[0] = D0;
    dims.d[1] = D1;
    dims.d[2] = D2;
    uint8_t mine[256];
    for (int bs = 0; bs < B * S; ++bs) {
        const int s = bs % S;
        int lo_v[3], hi_v[3];
        for (int a = 0; a < 3; ++a) {
            lo_v[a] = box[s * 6 + a];
            hi_v[a] = box[s * 6 + 3 + a];
        }
        for (int l = 0; l < 256; ++l) mine[l] = slot_of_label[l] == s;
        bool all_ok = true;
        float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
        for (int k = 0; k < 8; ++k) {
            float u = 0.0f, v = 0.0f;
            all_ok = box_corner_uv(G + bs * 12, src + bs * 3, lo_v, hi_v, shift, k, u, v) && all_ok;
            umin = std::min(umin, u);
            umax = std::max(umax, u);
            vmin = std::min(vmin, v);
            vmax = std::max(vmax, v);
        }
        int* rect = rects + bs * 4;
        footprint_rect(all_ok, umin, umax, vmin, vmax, cols[0], cols[W - 1], W, rows[0], rows[H - 1], H, rect);
        const bool nonempty = lo_v[0] < hi_v[0] && lo_v[1] < hi_v[1] && lo_v[2] < hi_v[2];
        for (int py = 0; py < H; ++py)
            for (int px = 0; px < W; ++px) {
                const long r = ((long)bs * H + py) * W + px;
                float S_ = 0.0f, L = 0.0f, jt[3] = {0, 0, 0}, js[3] = {0, 0, 0};
                const bool inside = !cull || (px >= rect[0] && px <= rect[1] && py >= rect[2] && py <= rect[3]);
                if (inside && nonempty) {
                    const Ray ray = pose_ray(G, Wd, rows, cols, src, bs, px, py, eps, L);   // make_ray's pose-in branch
                    if (!box_surely_missed(ray, lo_v, hi_v, shift)) {
                        const LoadGated ld{labels, mine};
                        if (sens) {
                            float A[3] = {0, 0, 0}, C[3] = {0, 0, 0};
                            S_ = siddon_ray_sens_box<4, LoadGated>(vol, dims, lo_v, hi_v, D1 * D2, D2, 1, ray, shift, A, C, ld);
                            for (int a = 0; a < 3; ++a) {
                                const float k = L * ray.inv[a];
                                jt[a] = -k * A[a];
                                js[a] = k * (A[a] - C[a]);
                            }
                        } else {
                            S_ = siddon_ray_lean_box<8, float, LoadGated>(vol, lo_v, hi_v, D1 * D2, D2, 1, ray, shift, ld);
                        }
                    }
                }
                out[r] = L * S_;
                if (sens) {
                    float* q = sens + r * 8;
                    q[0] = jt[0], q[1] = jt[1], q[2] = jt[2], q[3] = S_;
                    q[4] = js[0], q[5] = js[1], q[6] = js[2], q[7] = 0.0f;
                }
            }
    }
}

// boxes [256][6] = {lo0, lo1, lo2, hi0, hi1, hi2} overwritten; an absent label keeps lo = D > hi = 0.
void emu_label_boxes(const uint8_t* labels, int D0, int D1, int D2, int* boxes)
{
    const int dims[3] = {D0, D1, D2};
    for (int l = 0; l < 256; ++l)
        for (int a = 0; a < 3; ++a) {
            boxes[l * 6 + a] = dims[a];
            boxes[l * 6 + 3 + a] = 0;
        }
    for (long row = 0; row < (long)D0 * D1; ++row) {
        const int i0 = (int)(row / D1), i1 = (int)(row % D1);
        label_row_runs(labels + row * D2, D2, [&](int l, int b, int e) {
            int* q = boxes + l * 6;
            q[0] = std::min(q[0], i0);
            q[1] = std::min(q[1], i1);
            q[2] = std::min(q[2], b);
            q[3] = std::max(q[3], i0 + 1);
            q[4] = std::max(q[4], i1 + 1);
            q[5] = std::max(q[5], e);
        });
    }
}

}  // extern "C"
