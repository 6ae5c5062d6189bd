// hostemu_ncc_normal.cpp -- TEST INFRASTRUCTURE: compiles the product's NCC normal-equation math (ncc_normal_math.cuh) with g++
// and runs it over the windows and pixels on the CPU, with the passes of ncc_normal.cu (vertical sums, horizontal sums, window
// terms, adjoint box sum of 1/s^2, per-pixel beta J J^T), so that the CPU-only build container can check the kernels' arithmetic
// before any GPU time is spent.  Never linked into libb200drr.so and never imported by the product package.
#include <vector>

#include "../../diffdrr_b200/csrc/ncc_normal_math.cuh"

using namespace b200drr;

extern "C" {
// A [B][P][P] += weight * ..., g [B][P] += weight * ... as b200drr_ncc_normal (p = 0: global)
void emu_ncc_normal(const float* x, const float* t, const float* J, long sb, long sc, long sk, long sn, int B, int C, int H, int W,
                    int p, int P, double eps, double weight, double* A, double* g)
{
    const int K = ne_channels(P), tri = ne_tri(P);
    const long HW = (long)H * W;
    if (p == 1) return;  // as launch_ncc_normal: one-pixel windows add nothing
    for (int b = 0; b < B; ++b) {
        std::vector<double> acc((size_t)tri + P, 0.0);
        for (int c = 0; c < C; ++c) {
            const long img = (long)b * C + c;
            const float* xi = x + img * HW;
            const float* ti = t + img * HW;
            const float* Ji = J + b * sb + c * sc;
            if (p == 0) {
                std::vector<double> T((size_t)K + tri, 0.0);
                for (long q = 0; q < HW; ++q) {
                    for (int e = 0; e < K + tri; ++e) {
                        int ra, rb;
                        ne_global_pair(e, P, ra, rb);
                        auto row = [&](int r) {
                            return r == 0 ? 1.0 : r == 1 ? (double)xi[q] : r == 2 ? (double)ti[q] : (double)Ji[q * sn + (r - 3) * sk];
                        };
                        T[e] += row(ra) * row(rb);
                    }
                }
                const double rs2 = ne_window(T.data(), 1, P, (double)HW, eps);
                for (int e = 0; e < tri; ++e) {
                    int k, l;
                    ne_tri_index(e, P, k, l);
                    acc[e] += rs2 * T[K + e] - ne_ab(T.data(), 1, P, k, l);
                }
                for (int k = 0; k < P; ++k) acc[tri + k] += T[5 + 2 * P + k];
                continue;
            }
            const int Hp = H - p + 1, Wp = W - p + 1;
            std::vector<double> V((size_t)K * W), S(K), rs2((size_t)Hp * Wp), VB((size_t)H * Wp);
            for (int i = 0; i < Hp; ++i) {
                for (int k = 0; k < K; ++k)
                    for (int col = 0; col < W; ++col) V[(size_t)k * W + col] = ne_vertical(xi, ti, Ji, sk, sn, W, p, P, k, i, col);
                for (int j = 0; j < Wp; ++j) {
                    for (int k = 0; k < K; ++k) S[k] = ne_horizontal(&V[(size_t)k * W], p, j);
                    rs2[(size_t)i * Wp + j] = ne_window(S.data(), 1, P, (double)p * p, eps);
                    for (int e = 0; e < tri; ++e) {
                        int k, l;
                        ne_tri_index(e, P, k, l);
                        acc[e] -= ne_ab(S.data(), 1, P, k, l);
                    }
                    for (int k = 0; k < P; ++k) acc[tri + k] += S[5 + 2 * P + k];
                }
            }
            for (int y = 0; y < H; ++y)
                for (int j = 0; j < Wp; ++j) VB[(size_t)y * Wp + j] = ne_beta_vertical(rs2.data(), H, W, p, y, j);
            for (long q = 0; q < HW; ++q) {
                const double beta = ne_beta(VB.data(), W, p, (int)(q / W), (int)(q % W));
                for (int e = 0; e < tri; ++e) {
                    int k, l;
                    ne_tri_index(e, P, k, l);
                    acc[e] += beta * (double)Ji[q * sn + k * sk] * (double)Ji[q * sn + l * sk];
                }
            }
        }
        for (int e = 0; e < tri; ++e) {
            int k, l;
            ne_tri_index(e, P, k, l);
            A[((long)b * P + k) * P + l] += weight * acc[e];
            if (k != l) A[((long)b * P + l) * P + k] += weight * acc[e];
        }
        for (int k = 0; k < P; ++k) g[(long)b * P + k] += weight * acc[tri + k];
    }
}
}
