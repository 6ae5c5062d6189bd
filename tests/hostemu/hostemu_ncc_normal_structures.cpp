// hostemu_ncc_normal_structures.cpp -- TEST INFRASTRUCTURE: the block-sparse normal equations of ncc_normal_structures.cu
// (ncc_normal_structures_math.cuh) and the structure footprints compiled with g++ and run on the CPU with the kernels' passes:
// per (pose, task, band) the partial sums over the band's pixels in the kernel's order, the moment vector and ne_window per pose,
// then every entry of A and g.  Never linked into libb200drr.so.
#include <vector>

#include "../../diffdrr_b200/csrc/ncc_normal_structures_math.cuh"

using namespace b200drr;

extern "C" {

// rects [B*S][4] overwritten, as b200drr_structure_footprints
void emu_structure_footprints(const float* src, const float* G, const float* rows, const float* cols, const int* box, int* rects,
                              int B, int S, int H, int W, float shift)
{
    for (int bs = 0; bs < B * S; ++bs)
        structure_footprint(G + (long)bs * 12, src + (long)bs * 3, box + (bs % S) * 6, shift, rows, cols, H, W, rects + bs * 4);
}

// A [B][6K][6K] += weight * ..., g [B][6K] += weight * ... as b200drr_ncc_normal_structures
void emu_ncc_normal_structures(const float* x, const float* t, int t_batch, const float* J, long sb, long ss, long sn, long sk,
                               const int* rects, int B, int K, int S, int H, int W, double eps, double weight, double* A, double* g)
{
    const int P = kNsDof * K, pairs = ns_pairs(K), tasks = pairs + 1, chunks = ns_chunks(B, K, H), M = ne_channels(P);
    const long HW = (long)H * W;
    std::vector<double> part((size_t)tasks * chunks * kNsEntries), T(M);
    for (int b = 0; b < B; ++b) {
        const float* xb = x + b * HW;
        const float* tb = t + (t_batch == 1 ? 0 : b * HW);
        for (int task = 0; task < tasks; ++task) {
            const bool scalar = task == pairs;
            int j = 0, k = 0, rect[4] = {0, W - 1, 0, H - 1};
            bool any = true;
            if (!scalar) {
                ne_tri_index(task, K, j, k);
                any = ns_overlap(rects + ((long)b * S + j) * 4, rects + ((long)b * S + k) * 4, rect);
            }
            const float* Jj = J + b * sb + j * ss;
            const float* Jk = J + b * sb + k * ss;
            for (int c = 0; c < chunks; ++c) {
                double* out = &part[((size_t)task * chunks + c) * kNsEntries];
                for (int e = 0; e < kNsEntries; ++e) {
                    int ra, rb;
                    out[e] = 0.0;
                    if (!any || !ns_entry_rows(e, scalar, j == k, ra, rb)) continue;
                    int r0, r1;
                    ns_band(rect[2], rect[3], c, chunks, r0, r1);
                    const int w = rect[1] - rect[0] + 1;
                    double acc = 0.0;
                    for (long i = 0; i < (long)(r1 - r0) * w; ++i) {
                        const long q = (long)(r0 + i / w) * W + rect[0] + i % w;
                        acc += ns_row(ra, xb[q], tb[q], Jj + q * sn, Jk + q * sn, sk) *
                               ns_row(rb, xb[q], tb[q], Jj + q * sn, Jk + q * sn, sk);
                    }
                    out[e] = acc;
                }
            }
        }
        auto sum = [&](int task, int e) {
            double s = 0.0;
            for (int c = 0; c < chunks; ++c) s += part[((size_t)task * chunks + c) * kNsEntries + e];
            return s;
        };
        for (int e = 0; e < M; ++e) T[e] = ns_moment(e, K, sum);
        const double rs2 = ne_window(T.data(), 1, P, (double)HW, eps);
        for (int i = 0; i < P; ++i) {
            for (int l = 0; l < P; ++l)
                A[((long)b * P + i) * P + l] += weight * (rs2 * ns_jj(i, l, K, sum) - ne_ab(T.data(), 1, P, i, l));
            g[(long)b * P + i] += weight * T[5 + 2 * P + i];
        }
    }
}
}
