// hostemu_brick_sens_refill.cpp -- TEST INFRASTRUCTURE: the work lists of the brick kernel's sensitivities mode
// (csrc/siddon_brick.cu, SENS = 1) rebuilt on the CPU, and two ways of walking them counted.  For every brick, pose chunk and
// round of up to kWarps * K * 32 candidates it builds the round's sorted item list exactly as the kernel does (corner
// projection, 4-row bands, row spans, 8 x 4-pixel tiles, brick_maybe_hit, sens_bin, counting sort with the longest bin first),
// walks every item's (ray, brick) pair to count the U-step groups it runs, and then schedules the list two ways:
//   (a) chunks: a warp takes 32 consecutive items and runs all of them until its longest pair is done;
//   (b) refill: a warp keeps 32 lanes; after every U-step group the lanes whose pair ended flush and, when at least `thresh`
//       lanes are idle (or all are), take the next items of the warp's major-axis group from that group's cursor.
// Warps are simulated as the kernel's kWarps warps of a CTA, each claiming in the order of its own issue clock.  The issue
// cost of a warp is counted in instructions from per-piece weights (set-up, claim, U-step group, exit tail + flush) that the
// caller takes from the SASS of the SENS instantiation.  Never linked into libb200drr.so.
#include <algorithm>
#include <vector>

#include "../../diffdrr_b200/csrc/brick.cuh"

using namespace b200drr;

namespace {

// the SENS instantiation's shape: 512 threads (16 warps), K = 4 tiles per warp and round, two CTAs per SM (256 bands)
constexpr int kWarps = 16, kK = 4, kRowCap = 256;

// groups of U steps the walk of one pair runs, and its major axis (the walk's own choice, from d)
template <int U>
void pair_groups(const VolFrame& f, const float s[3], const float d[3], const VolDims& dims, const int lo_v[3], const int hi_v[3],
                 float shift, int& groups, int& M)
{
    const Walk w = start_walk_in_frame<true>(f, s, d, dims, lo_v, hi_v, shift);
    const float m0 = fabsf(d[0]), m1 = fabsf(d[1]), m2 = fabsf(d[2]);
    M = (m0 >= m1 && m0 >= m2) ? 0 : (m1 >= m2 ? 1 : 2);
    groups = 0;
    if (!w.hit) return;
    LeanConst k;
    LeanState st;
    lean_init(w, 1, 1, 1, st, k);
    while (st.acur < k.a_out) {
        int ax;
        for (int j = 0; j < U; ++j) (void)lean_step_ax(st, k, ax);
        ++groups;
    }
}

struct Cost {
    double setup, claim, group, tail;
};

struct Stats {
    double issue_a, issue_b;         // warp instructions
    double lanesteps_a, lanesteps_b; // 32 * U per group a warp runs
    double setups_a, setups_b;       // set-up passes of a warp (one per chunk / per refill)
    double items, groups, mismatched;
};

// (b) for one round: items [0, n) sorted M-major (M = 2 first); groups[i], bin-M mbin[i].  Returns false if an item was not
// claimed exactly once.
bool schedule_refill(const std::vector<int>& groups, const std::vector<int>& mbin, int thresh, const Cost& c, Stats& st)
{
    const int n = (int)groups.size();
    int beg[3], end[3];
    for (int m = 0; m < 3; ++m) {
        beg[m] = n;
        end[m] = 0;
    }
    for (int i = 0; i < n; ++i) {
        beg[mbin[i]] = std::min(beg[mbin[i]], i);
        end[mbin[i]] = std::max(end[mbin[i]], i + 1);
    }
    int cursor[3];
    for (int m = 0; m < 3; ++m) {
        if (beg[m] >= end[m]) beg[m] = end[m] = 0;
        cursor[m] = beg[m];
    }
    std::vector<int> seen(n, 0);
    struct WarpState {
        double clock = 0.0;
        int M = -1;
        int left[32];
        bool done = false;
    };
    std::vector<WarpState> warps(kWarps);
    for (auto& w : warps) std::fill(w.left, w.left + 32, -1);
    for (;;) {
        int wi = -1;
        for (int i = 0; i < kWarps; ++i)
            if (!warps[i].done && (wi < 0 || warps[i].clock < warps[wi].clock)) wi = i;
        if (wi < 0) break;
        WarpState& w = warps[wi];
        int active = 0;
        for (int l = 0; l < 32; ++l) active += w.left[l] >= 0;
        const int idle = 32 - active;
        if (active == 0) {  // fresh: the first major-axis group with items left
            w.M = -1;
            for (int m = 2; m >= 0; --m)
                if (cursor[m] < end[m]) {
                    w.M = m;
                    break;
                }
            if (w.M < 0) {
                w.done = true;
                continue;
            }
        }
        if (idle > 0 && (idle >= thresh || active == 0) && w.M >= 0 && cursor[w.M] < end[w.M]) {
            const int c0 = cursor[w.M];
            cursor[w.M] += idle;  // one warp-aggregated atomicAdd; indices past the group's end are dropped
            const int got = std::min(c0 + idle, end[w.M]) - c0;
            int g = 0;
            for (int l = 0; l < 32 && g < got; ++l)
                if (w.left[l] < 0) {
                    const int i = c0 + g++;
                    ++seen[i];
                    w.left[l] = groups[i];
                }
            w.clock += c.claim + c.setup;
            st.setups_b += 1.0;
        }
        bool any_walk = false;
        for (int l = 0; l < 32; ++l) any_walk = any_walk || w.left[l] > 0;
        if (any_walk) {
            w.clock += c.group;
            st.lanesteps_b += 32.0;
            for (int l = 0; l < 32; ++l)
                if (w.left[l] > 0) --w.left[l];
        }
        bool fin = false;
        for (int l = 0; l < 32; ++l)
            if (w.left[l] == 0) {
                w.left[l] = -1;
                fin = true;
            }
        if (fin) w.clock += c.tail;
        if (!fin && !any_walk) w.done = true;  // nothing to walk and nothing to claim: drained
    }
    for (auto& w : warps) st.issue_b += w.clock;
    bool ok = true;
    for (int i = 0; i < n; ++i) ok = ok && seen[i] == 1;
    return ok;
}

}  // namespace

extern "C" {

// rays: src [B][3], tgt [B][H*W][3] in voxel-index space, full H x W detector grids.  Volume D0 x D1 x D2 in bricks BX x BY x BZ,
// walk groups of U = 6 steps.  cost = {set-up, claim, group, tail + flush} in warp instructions.  Bricks with index
// brick % brick_step != 0 are skipped (a sample of the volume for quick runs).  out = {issue (a), issue (b), lane-steps (a),
// lane-steps (b), set-ups (a), set-ups (b), items, rounds whose items were all claimed exactly once by (b), rounds, items whose
// walk major axis differs from their sort key's, steps the pairs walk in whole groups}.  Returns 0.
int emu_brick_sens_schedule(const float* src, const float* tgt, int B, int H, int W, int D0, int D1, int D2, float shift, float eps,
                            int BX, int BY, int BZ, const float* cost, int thresh, int brick_step, double* out)
{
    constexpr int U = 6;
    const VolDims dims{{D0, D1, D2}};
    const long N = (long)H * W;
    const Cost c{cost[0], cost[1], cost[2], cost[3]};
    std::vector<PoseGeo> geo(B);
    std::vector<float> raytab((size_t)B * N * 4);
    for (int b = 0; b < B; ++b) {
        for (long n = 0; n < N; ++n) {
            const Ray r = load_ray(src, tgt, b, (long)b * N + n, eps);
            float* q = &raytab[((size_t)b * N + n) * 4];
            q[0] = r.inv[0];
            q[1] = r.inv[1];
            q[2] = r.inv[2];
            q[3] = fabsf(r.d[0]) + fabsf(r.d[1]) + fabsf(r.d[2]);
        }
        const Ray r00 = load_ray(src, tgt, b, (long)b * N, eps), r0w = load_ray(src, tgt, b, (long)b * N + (W - 1), eps),
                  rh0 = load_ray(src, tgt, b, (long)b * N + (long)(H - 1) * W, eps);
        float t00[3], t0w[3], th0[3];
        for (int a = 0; a < 3; ++a) {
            t00[a] = r00.s[a] + r00.d[a];
            t0w[a] = r00.s[a] + r0w.d[a];
            th0[a] = r00.s[a] + rh0.d[a];
        }
        geo[b] = make_pose_geo(r00.s, t00, t0w, th0, H, W);
    }
    Stats st{};
    double rounds = 0.0, rounds_ok = 0.0;
    const int nb0 = (D0 + BX - 1) / BX, nb1 = (D1 + BY - 1) / BY, nb2 = (D2 + BZ - 1) / BZ;
    for (int brick = 0; brick < nb0 * nb1 * nb2; brick += brick_step) {
        const int i2 = brick % nb2, i1 = (brick / nb2) % nb1, i0 = brick / (nb2 * nb1);
        const int org[3] = {i0 * BX, i1 * BY, i2 * BZ};
        const int hi_v[3] = {std::min(org[0] + BX, D0), std::min(org[1] + BY, D1), std::min(org[2] + BZ, D2)};
        int p0 = 0;
        while (p0 < B) {
            const int ntry = std::min(kBrickPoseChunk, B - p0);
            std::vector<float> uv(ntry * 16), clo(ntry * 3), chi(ntry * 3);
            std::vector<PixRect> rect(ntry);
            std::vector<int> flag(ntry), cnt(ntry);
            for (int bl = 0; bl < ntry; ++bl) {
                const PoseGeo& g = geo[p0 + bl];
                float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY, dmin = INFINITY, dmax = -INFINITY;
                bool bad = false;
                for (int k = 0; k < 8; ++k) {
                    const float X[3] = {(float)((k & 1) ? hi_v[0] : org[0]) - shift, (float)((k & 2) ? hi_v[1] : org[1]) - shift,
                                        (float)((k & 4) ? hi_v[2] : org[2]) - shift};
                    float u, v, den;
                    project_corner(g, X, u, v, den);
                    bad = bad || (u != u) || (v != v) || (den != den);
                    uv[bl * 16 + 2 * k] = u;
                    uv[bl * 16 + 2 * k + 1] = v;
                    umin = fminf(umin, u);
                    umax = fmaxf(umax, u);
                    vmin = fminf(vmin, v);
                    vmax = fmaxf(vmax, v);
                    dmin = fminf(dmin, den);
                    dmax = fmaxf(dmax, den);
                }
                if (bad) dmin = NAN;
                rect[bl] = rect_from_extents(umin, umax, vmin, vmax, dmin, dmax, H, W);
                flag[bl] = outline_valid(umin, umax, vmin, vmax, dmin, dmax) ? 1 : 0;
                const PixRect& rc = rect[bl];
                cnt[bl] = (rc.x0 <= rc.x1 && rc.y0 <= rc.y1) ? (rc.y1 - rc.y0) / 4 + 1 : 0;
                for (int a = 0; a < 3; ++a) {
                    clo[bl * 3 + a] = ((float)org[a] - shift) - g.S[a];
                    chi[bl * 3 + a] = ((float)hi_v[a] - shift) - g.S[a];
                }
            }
            std::vector<int> rowbase(ntry + 1, 0);
            int np = 0;
            for (int bl = 0; bl < ntry; ++bl) {
                if (rowbase[bl] + cnt[bl] > kRowCap) break;
                rowbase[bl + 1] = rowbase[bl] + cnt[bl];
                np = bl + 1;
            }
            if (np == 0) {
                np = 1;
                rowbase[1] = cnt[0];
            }
            const int R = rowbase[np];
            std::vector<int> rowpose(R), rowy(R), rowx(R), rowend(R), prefix(R + 1, 0);
            for (int r = 0; r < R; ++r) {
                int bl = 0;
                while (rowbase[bl + 1] <= r) ++bl;
                const PixRect& rc = rect[bl];
                const int py0 = rc.y0 + 4 * (r - rowbase[bl]);
                int px_lo, px_hi, n = 0;
                if (row_span(&uv[bl * 16], flag[bl] != 0, rc, py0, px_lo, px_hi)) n = (px_hi - px_lo) / 8 + 1;
                else px_lo = px_hi = 0;
                rowpose[r] = bl;
                rowy[r] = py0;
                rowx[r] = px_lo;
                rowend[r] = px_hi;
                prefix[r + 1] = prefix[r] + n;
            }
            const int T = prefix[R];
            for (int t0 = 0; t0 < T; t0 += kWarps * kK) {
                // candidates of the round -> hits, in the kernel's candidate order; then the counting sort, longest bin first
                std::vector<std::pair<int, long>> hits;  // (bin, pose * N + ray) ; groups / M alongside
                std::vector<int> hgroups, hm;
                for (int t = t0; t < std::min(T, t0 + kWarps * kK); ++t) {
                    int row = 0;
                    while (prefix[row + 1] <= t) ++row;
                    const int bl = rowpose[row];
                    for (int lane = 0; lane < 32; ++lane) {
                        const int px = rowx[row] + 8 * (t - prefix[row]) + (lane & 7), py = rowy[row] + (lane >> 3);
                        if (px > rowend[row] || py > rect[bl].y1) continue;
                        const long n = (long)py * W + px;
                        const float* q = &raytab[((size_t)(p0 + bl) * N + n) * 4];
                        float a_in, a_out;
                        if (!brick_maybe_hit(q, &clo[bl * 3], &chi[bl * 3], a_in, a_out)) continue;
                        const int bin = sens_bin<U>(q, a_in, a_out, q[3]);
                        const long r = (long)(p0 + bl) * N + n;
                        const Ray ray = load_ray(src, tgt, p0 + bl, r, eps);
                        const VolFrame f = volume_frame(ray, dims, shift);
                        int g, M;
                        pair_groups<U>(f, ray.s, ray.d, dims, org, hi_v, shift, g, M);
                        hits.push_back({bin, r});
                        hgroups.push_back(g);
                        hm.push_back(M);
                    }
                }
                std::vector<int> order(hits.size());
                for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
                std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return hits[a].first > hits[b].first; });
                const int n = (int)order.size();
                std::vector<int> groups(n), mbin(n);
                for (int i = 0; i < n; ++i) {
                    groups[i] = hgroups[order[i]];
                    mbin[i] = hits[order[i]].first / kSensLenBins;
                    st.mismatched += hm[order[i]] != mbin[i];
                    st.groups += groups[i];
                }
                st.items += n;
                // (a) 32-item chunks
                for (int c0 = 0; c0 < n; c0 += 32) {
                    int gmax = 0;
                    for (int i = c0; i < std::min(n, c0 + 32); ++i) gmax = std::max(gmax, groups[i]);
                    st.issue_a += c.claim + c.setup + gmax * c.group + c.tail;
                    st.lanesteps_a += 32.0 * gmax;
                    st.setups_a += 1.0;
                }
                // (b) per-lane refill
                rounds += 1.0;
                rounds_ok += schedule_refill(groups, mbin, thresh, c, st) ? 1.0 : 0.0;
            }
            p0 += np;
        }
    }
    out[0] = st.issue_a;
    out[1] = st.issue_b;
    out[2] = st.lanesteps_a * U;
    out[3] = st.lanesteps_b * U;
    out[4] = st.setups_a;
    out[5] = st.setups_b;
    out[6] = st.items;
    out[7] = rounds_ok;
    out[8] = rounds;
    out[9] = st.mismatched;
    out[10] = st.groups * U;
    return 0;
}

}  // extern "C"
