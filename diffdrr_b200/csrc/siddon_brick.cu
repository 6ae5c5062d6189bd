// siddon_brick.cu -- brick-major Siddon forward for sm_90a: TMA-staged voxel bricks in shared memory.
//
// Persistent CTAs (one per SM).  Each CTA claims bricks from a global counter; a brick (BX x BY x BZ fp32 voxels) is
// brought into shared memory by ONE cp.async.bulk.tensor.3d box copy (zero fill outside the volume) that completes on
// an mbarrier, STAGES deep: the copy of the next brick is in flight while the current one is integrated.  For the
// current brick the CTA
//   1. projects the brick's 8 corners into every pose's detector -> a pixel rectangle per pose (brick.cuh),
//   2. tests the rays of those rectangles against the brick (conservative slab test on a 16-byte ray-table entry),
//   3. counting-sorts the hits by their estimated number of voxel visits (so the 32 lanes of a warp walk chords of
//      similar length) and
//   4. lets the warps pull 32-item chunks, longest first: exact walk set-up (start_walk_box), lean walk with the voxel
//      loads served by ld.shared, one red.global.add of the partial line integral per (ray, brick).
// The (B, N) ray table {1/d, sum|d|} (+ the ray lengths L) is written once per launch by brick_prep_kernel, which also zero-fills
// the output and derives the per-pose detector geometry used in step 1.
// Two more modes of the same kernel: BWD (volume gradient, the staged brick is an accumulator) and SENS (training step: each pair
// runs the exact-frame sensitivities walk of the slab kernels, from a per-ray frame record the prep kernel writes, and adds the
// ray's image and end-point derivatives).
//
// Replaces reference renderers.py:94-113 (alphas + sort) and 156-169 (grid_sample gather) for full detector grids.
#include <cuda.h>  // CUtensorMap + enums only; the encoder is fetched through cudaGetDriverEntryPoint (no -lcuda)

#include <mutex>
#include <type_traits>

#include "brick.cuh"
#include "kernels.h"

namespace b200drr {

namespace {

// ---- PTX helpers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one 3-D box: coordinates are (fastest .. slowest) = (axis 2, axis 1, axis 0) voxel indices of the box origin
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
        "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// one 3-D box shared -> global (clipped to the tensor), bulk async-group completion
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(src), "r"(c0),
                 "r"(c1), "r"(c2)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// volume-gradient mode: the staged brick is an ACCUMULATOR; fp32 add on a byte address in the shared window
// (red.shared.add.f32 = an ATOMS.CAST.SPIN loop on sm_90a: there is no native fp32 shared-memory add)
// SWZ: the brick rows (BZ = 32 floats = 128 B) are stored in TMA's 128-byte swizzle (16-byte chunk index ^= row index & 7, i.e.
// address bits 4-6 ^= bits 7-9; the brick base is 1024-byte aligned), so lanes that share z but differ in y hit different banks
// -- the un-swizzled bank is z mod 32 alone, whatever x and y are.  The TMA store of the finished brick undoes it.
// Faster than the plain layout before the port to Hopper (not re-measured on the H100).  -DB200DRR_BWD_SWIZZLE=0 builds the
// linear layout for A/B runs.
#ifndef B200DRR_BWD_SWIZZLE
#define B200DRR_BWD_SWIZZLE 1
#endif
struct StShared {
    uint32_t base_addr;
    static constexpr int kScale = 4;
    __device__ __forceinline__ int base() const { return (int)base_addr; }
    __device__ __forceinline__ void add(int off, float v) const
    {
#if B200DRR_BWD_SWIZZLE
        off ^= (off >> 3) & 0x70;
#endif
        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(off), "f"(v) : "memory");
    }
};

// ld.shared with a byte address in the shared window.  B200DRR_FWD_SWIZZLE=1 (A/B builds): bricks loaded through a 128-byte
// swizzled tensor map, the address un-swizzled per load (see StShared).
#ifndef B200DRR_FWD_SWIZZLE
#define B200DRR_FWD_SWIZZLE 0
#endif
// V = the staged voxel type: fp32, or a 16-bit VoxF16 / VoxBF16 (ld.shared.u16, widened by vox16_to_f32; unswizzled).
template <class V>
struct LdSharedT {
    uint32_t base_addr;
    static constexpr int kScale = (int)sizeof(V);
    __device__ __forceinline__ int base() const { return (int)base_addr; }
    __device__ __forceinline__ float operator()(int off) const
    {
        if constexpr (sizeof(V) == 4) {
            float v;
#if B200DRR_FWD_SWIZZLE
            off ^= (off >> 3) & 0x70;
#endif
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(off));
            return v;
        } else {
            unsigned short h;
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(off));
            return vox16_to_f32(h, std::is_same<V, VoxBF16>::value);
        }
    }
};

struct PoseRaysB {
    const float* G;
    const float* Wd;
    const float* rows;
    const float* cols;
};

__device__ __forceinline__ Ray make_ray_b(const PoseRaysB& pr, const float* __restrict__ src, const float* __restrict__ tgt,
                                          const float* __restrict__ raylen, int b, int64_t r, int px, int py, float eps,
                                          float& L)
{
    if (pr.G == nullptr) {
        L = __ldg(raylen + r);
        return load_ray(src, tgt, b, r, eps);
    }
    const float c = __ldg(pr.cols + px), rr = __ldg(pr.rows + py);
    const float* g = pr.G + b * 12;
    const float* wd = pr.Wd + b * 12;
    Ray ray;
    float l2 = 0.0f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float t = fmaf(__ldg(g + a * 4), c, fmaf(__ldg(g + a * 4 + 1), rr, __ldg(g + a * 4 + 2) + __ldg(g + a * 4 + 3)));
        const float dw = fmaf(__ldg(wd + a * 4), c, fmaf(__ldg(wd + a * 4 + 1), rr, __ldg(wd + a * 4 + 2) + __ldg(wd + a * 4 + 3)));
        l2 = fmaf(dw, dw, l2);
        ray.s[a] = __ldg(src + b * 3 + a);
        ray.d[a] = (t - ray.s[a]) + eps;
        ray.inv[a] = 1.0f / ray.d[a];
    }
    L = sqrtf(l2);
    return ray;
}

// Sensitivities mode (SENS = 1): the per-ray frame records brick_prep_kernel wrote ([B][Nr], SensFrameRec) and where a pair adds
// its share: sens [B][Nr][8], as b200drr_siddon_fwd_sens_grid lays it out.
struct SensArgs {
    const SensFrameRec* frames;
    float* sens;
};

// ---- ray table + per-pose geometry + zero fill ----------------------------------------------------------------------
__global__ void __launch_bounds__(256) brick_prep_kernel(const float* __restrict__ src, const float* __restrict__ tgt,
                                                         const float* __restrict__ raylen, PoseRaysB pr,
                                                         float4* __restrict__ raytab, float* __restrict__ ltab,
                                                         PoseGeo* __restrict__ geo, float* __restrict__ out,
                                                         unsigned* __restrict__ counter, int H, int W, float eps,
                                                         int64_t Nr /* rays per pose */,
                                                         const float* __restrict__ corners /* [B][3][3] or nullptr */,
                                                         const float* __restrict__ gout /* volume-gradient mode, else nullptr */,
                                                         float* __restrict__ sens = nullptr /* sensitivities mode: zero-filled */,
                                                         SensFrameRec* __restrict__ frames = nullptr /* sensitivities mode */,
                                                         VolDims dims = VolDims{}, float shift = 0.0f)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= Nr) return;
    // full grid: ray n is pixel (n / W, n % W); ray subset (corners != nullptr): n indexes the caller's (B, Nr) ray arrays
    const int py = corners ? 0 : (int)(n / W), px = corners ? 0 : (int)(n - (int64_t)py * W);
    const int64_t r = (int64_t)b * Nr + n;
    float L;
    const Ray ray = make_ray_b(pr, src, tgt, raylen, b, r, px, py, eps, L);
    raytab[r] = make_float4(ray.inv[0], ray.inv[1], ray.inv[2], fabsf(ray.d[0]) + fabsf(ray.d[1]) + fabsf(ray.d[2]));
    ltab[r] = gout ? L * __ldg(gout + r) : L;  // volume-gradient mode: the weight every chord length is scattered with
    if (out) out[r] = 0.0f;
    if (sens) {
        float4* s4 = reinterpret_cast<float4*>(sens) + 2 * r;
        s4[0] = s4[1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    if (frames) frames[r] = pack_sens_frame(volume_frame(ray, dims, shift), ray.d, L);
    if (n == 0) {
        float t00[3], t0w[3], th0[3];
        if (corners) {  // targets of the full grid's pixels (0, 0), (0, W-1), (H-1, 0), handed in by the caller
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                t00[a] = corners[b * 9 + a];
                t0w[a] = corners[b * 9 + 3 + a];
                th0[a] = corners[b * 9 + 6 + a];
            }
        } else {
            float Lx;
            const Ray r0w = make_ray_b(pr, src, tgt, raylen, b, (int64_t)b * Nr + (W - 1), W - 1, 0, eps, Lx);
            const Ray rh0 = make_ray_b(pr, src, tgt, raylen, b, (int64_t)b * Nr + (int64_t)(H - 1) * W, 0, H - 1, eps, Lx);
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                t00[a] = ray.s[a] + ray.d[a];
                t0w[a] = ray.s[a] + r0w.d[a];
                th0[a] = ray.s[a] + rh0.d[a];
            }
        }
        geo[b] = make_pose_geo(ray.s, t00, t0w, th0, H, W);
        if (b == 0) *counter = 0u;
    }
}

// ---- the brick kernel -------------------------------------------------------------------------------------------
struct BrickGrid {
    int nb0, nb1, nb2;  // bricks per axis
};

template <int BX, int BY, int BZ, int STAGES, int THREADS, int K, int U, int CTAS, int PIPE, int RAYS = 1, class V = float>
struct BrickCfg {
    // 4-row tile bands per pose chunk (a chunk takes as many poses as fit); the two-CTA-per-SM shape has less room
    static constexpr int kRowCap = CTAS == 1 ? 512 : 256;
    static constexpr int kBrickElems = BX * BY * BZ;
    static constexpr int kBrickBytes = kBrickElems * (int)sizeof(V);  // 16-bit voxels: half the bytes, same shape
    static constexpr int kWarps = THREADS / 32;
    static constexpr int kCap = kWarps * K * 32;  // items per round (every candidate of a round may hit)
    static constexpr int kPB = kBrickPoseChunk;
    // shared-memory carve-up (bytes)
    static constexpr int oBricks = 0;
    static constexpr int oItems = oBricks + STAGES * kBrickBytes;
    static constexpr int oBar = oItems + kCap * 4;               // STAGES x 8
    static constexpr int oPoseF = oBar + 64;                      // kPB x 12 floats: S[3],-, clo[3],-, chi[3],-
    static constexpr int oUV = oPoseF + kPB * 12 * 4;             // kPB x 16 floats: projected corners (u, v)
    static constexpr int oRect = oUV + kPB * 16 * 4;              // kPB x 4 ints: x0, y0, x1, y1
    static constexpr int oFlag = oRect + kPB * 4 * 4;             // kPB ints: outline valid
    static constexpr int oRowBase = oFlag + kPB * 4;              // kPB + 1 ints (+ pad)
    static constexpr int oRowInfo = oRowBase + (kPB + 4) * 4;     // kRowCap u32: pose | first row | first column
    static constexpr int oRowEnd = oRowInfo + kRowCap * 4;        // kRowCap ints: last column
    static constexpr int oRowPrefix = oRowEnd + kRowCap * 4;      // kRowCap + 1 ints (+ pad): tiles before the band
    static constexpr int oHist = oRowPrefix + (kRowCap + 4) * 4;  // kBrickBins ints
    static constexpr int oCursor = oHist + kBrickBins * 4;        // kBrickBins ints
    static constexpr int oMisc = oCursor + kBrickBins * 4;        // see s_misc
    static constexpr int kSmemBytes = oMisc + 128;
};

// BWD = 1: volume-gradient mode.  `tmap` then describes g_vol, the staged brick starts as zeros instead of a TMA load, every
// pair's walk scatters (gout * L) * chord length into it (brick_pair_bwd_lean; ltab holds gout * L), and the finished brick is
// written with ONE TMA store -- every voxel belongs to exactly one brick, so there is no global atomic and g_vol is overwritten.
// SENS = 1: training-step mode (full detector grids).  Every pair reads its ray's frame record (SensFrameRec) and 1/d, runs the
// exact-frame sensitivities walk over the staged brick (brick_pair_sens_framed) and flushes like siddon_sens_slab_kernel: two
// red.global.add.v4 into sa.sens (dI/dt, S,
// dI/ds) and L * S into out, nothing for an all-zero pair.  The work list is sorted by major axis first (sens_bin).
template <int BX, int BY, int BZ, int STAGES, int THREADS, int K, int U, int CTAS, int PIPE, int RAYS, int BWD = 0, int SENS = 0,
          class V = float>
__global__ void __launch_bounds__(THREADS, CTAS)
    siddon_fwd_brick_kernel(const __grid_constant__ CUtensorMap tmap, VolDims dims, BrickGrid bg,
                            const float4* __restrict__ raytab, const float* __restrict__ ltab,
                            const PoseGeo* __restrict__ geo, float* __restrict__ out, unsigned* __restrict__ counter,
                            const int* __restrict__ pix_index /* [H*W] pixel -> ray index, -1 = no ray; nullptr = full grid */,
                            int Nr /* rays per pose */, int B, int H, int W, float shift, SensArgs sa)
{
    using Cfg = BrickCfg<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, PIPE, RAYS, V>;
    using LdShared = LdSharedT<V>;
    static_assert(BWD == 0 || (STAGES == 1 && RAYS == 1), "volume-gradient mode: single stage, one pair per thread");
    static_assert(BWD == 0 || sizeof(V) == 4, "the volume gradient is fp32");
    static_assert(SENS == 0 || (BWD == 0 && RAYS == 1), "sensitivities mode: forward walk, one pair per thread");
    constexpr int kRowCap = Cfg::kRowCap;
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned* s_items = reinterpret_cast<unsigned*>(smem + Cfg::oItems);
    float* s_posef = reinterpret_cast<float*>(smem + Cfg::oPoseF);
    float* s_uv = reinterpret_cast<float*>(smem + Cfg::oUV);
    int* s_rect = reinterpret_cast<int*>(smem + Cfg::oRect);
    int* s_flag = reinterpret_cast<int*>(smem + Cfg::oFlag);
    int* s_rowbase = reinterpret_cast<int*>(smem + Cfg::oRowBase);
    unsigned* s_rowinfo = reinterpret_cast<unsigned*>(smem + Cfg::oRowInfo);
    int* s_rowend = reinterpret_cast<int*>(smem + Cfg::oRowEnd);
    int* s_rowprefix = reinterpret_cast<int*>(smem + Cfg::oRowPrefix);
    int* s_hist = reinterpret_cast<int*>(smem + Cfg::oHist);
    int* s_cursor = reinterpret_cast<int*>(smem + Cfg::oCursor);
    // s_misc: [0] n_items, [1] chunk counter, [2..3] next brick, [4] poses in this chunk, [5] bands, [6] tiles
    int* s_misc = reinterpret_cast<int*>(smem + Cfg::oMisc);
    const uint32_t bar0 = smem_u32(smem + Cfg::oBar);
    const uint32_t brick0 = smem_u32(smem + Cfg::oBricks);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_bricks = bg.nb0 * bg.nb1 * bg.nb2;
    const float inv_bin_width = (float)kBrickBins / (float)(BX + BY + BZ + 8);

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
        fence_barrier_init();
    }
    if (tid < kBrickBins) s_hist[tid] = 0;
    __syncthreads();

    auto issue = [&](int brick, int stage) {  // thread 0 only
        const int i2 = brick % bg.nb2, i1 = (brick / bg.nb2) % bg.nb1, i0 = brick / (bg.nb2 * bg.nb1);
        fence_proxy_async();  // earlier generic-proxy reads of this stage are ordered before the async-proxy write
        mbar_expect_tx(bar0 + 8 * stage, (uint32_t)Cfg::kBrickBytes);
        tma_load_3d(brick0 + stage * Cfg::kBrickBytes, &tmap, bar0 + 8 * stage, i2 * BZ, i1 * BY, i0 * BX);
    };

    // prologue: claim the first brick (and start its copy)
    if (tid == 0) {
        const int first = (int)atomicAdd(counter, 1u);
        s_misc[2] = first;
        if (BWD == 0 && first < n_bricks) issue(first, 0);
    }
    __syncthreads();
    int cur = s_misc[2];

    for (int it = 0; cur < n_bricks; ++it) {
        const int stage = STAGES == 1 ? 0 : (it & 1);
        const uint32_t parity = STAGES == 1 ? (uint32_t)(it & 1) : (uint32_t)((it >> 1) & 1);
        if (STAGES == 2 && tid == 0) {  // prefetch the next brick into the other stage (free since the last end-of-brick barrier)
            const int nxt = (int)atomicAdd(counter, 1u);
            s_misc[2 + ((it + 1) & 1)] = nxt;
            if (nxt < n_bricks) issue(nxt, stage ^ 1);
        }
        const int i2 = cur % bg.nb2, i1 = (cur / bg.nb2) % bg.nb1, i0 = cur / (bg.nb2 * bg.nb1);
        const int org[3] = {i0 * BX, i1 * BY, i2 * BZ};
        const int lo_v[3] = {org[0], org[1], org[2]};
        const int hi_v[3] = {min(org[0] + BX, dims.d[0]), min(org[1] + BY, dims.d[1]), min(org[2] + BZ, dims.d[2])};
        LdShared ld;
        ld.base_addr = brick0 + stage * Cfg::kBrickBytes;
        if constexpr (BWD != 0) {  // the accumulator brick starts at zero (ordered before the walks by the barriers below)
            float4* z = reinterpret_cast<float4*>(smem + Cfg::oBricks);
            for (int i = tid; i < Cfg::kBrickElems / 4; i += THREADS) z[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }

        int p0 = 0;
        while (p0 < B) {
            const int ntry = min(Cfg::kPB, B - p0);
            __syncthreads();  // the previous chunk's (or brick's) readers of the pose / band tables are done
            // ---- 1a. project the brick's corners per pose: 8 lanes (corners) per pose -----------------------------
            if (warp < (ntry * 8 + 31) / 32) {  // whole warps take part in the shuffles; surplus lanes repeat the last pose
                const int bl_raw = tid >> 3, c = tid & 7;
                const int bl = min(bl_raw, ntry - 1);
                const PoseGeo g = geo[p0 + bl];
                const float X[3] = {(float)((c & 1) ? hi_v[0] : lo_v[0]) - shift, (float)((c & 2) ? hi_v[1] : lo_v[1]) - shift,
                                    (float)((c & 4) ? hi_v[2] : lo_v[2]) - shift};
                float u, v, den;
                project_corner(g, X, u, v, den);
                const bool bad = (u != u) || (v != v) || (den != den);
                float umin = u, umax = u, vmin = v, vmax = v, dmin = den, dmax = den;
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) {
                    umin = fminf(umin, __shfl_xor_sync(0xffffffffu, umin, o));
                    umax = fmaxf(umax, __shfl_xor_sync(0xffffffffu, umax, o));
                    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
                    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
                    dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
                    dmax = fmaxf(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
                }
                const unsigned badmask = __ballot_sync(0xffffffffu, bad);
                if (bl_raw < ntry) {
                    s_uv[bl * 16 + 2 * c] = u;
                    s_uv[bl * 16 + 2 * c + 1] = v;
                    if (c == 0) {
                        const bool anybad = ((badmask >> (lane & 24)) & 0xffu) != 0u;
                        if (anybad) dmin = NAN;  // -> whole detector
                        const PixRect rc = rect_from_extents(umin, umax, vmin, vmax, dmin, dmax, H, W);
                        s_flag[bl] = outline_valid(umin, umax, vmin, vmax, dmin, dmax) ? 1 : 0;
                        s_rect[bl * 4 + 0] = rc.x0;
                        s_rect[bl * 4 + 1] = rc.y0;
                        s_rect[bl * 4 + 2] = rc.x1;
                        s_rect[bl * 4 + 3] = rc.y1;
                        s_rowbase[bl + 1] = (rc.x0 <= rc.x1 && rc.y0 <= rc.y1) ? (rc.y1 - rc.y0) / 4 + 1 : 0;  // band count
#pragma unroll
                        for (int a = 0; a < 3; ++a) {
                            s_posef[bl * 12 + a] = g.S[a];
                            s_posef[bl * 12 + 4 + a] = ((float)lo_v[a] - shift) - g.S[a];
                            s_posef[bl * 12 + 8 + a] = ((float)hi_v[a] - shift) - g.S[a];
                        }
                    }
                }
            }
            __syncthreads();
            // ---- 1b. how many poses fit the band table; first band of every pose --------------------------------------
            if (warp == 0) {
                const int cnt = lane < ntry ? s_rowbase[lane + 1] : 0;
                int incl = cnt;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int up = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += up;
                }
                const unsigned fits = __ballot_sync(0xffffffffu, lane < ntry && incl <= kRowCap);
                const int np = max(1, __popc(fits));  // incl is monotone: the fitting poses are a prefix (one pose always fits)
                if (lane < np) s_rowbase[lane + 1] = incl;
                if (lane == 0) s_rowbase[0] = 0;
                const int R = __shfl_sync(0xffffffffu, incl, np - 1);
                if (lane == 0) {
                    s_misc[4] = np;
                    s_misc[5] = R;
                }
            }
            __syncthreads();
            const int npose = s_misc[4], R = s_misc[5];
            // ---- 1c. column span of every 4-row band inside the projected outline --------------------------------------
            for (int r = tid; r < R; r += THREADS) {
                int bl = 0;
                while (s_rowbase[bl + 1] <= r) ++bl;
                const PixRect rc{s_rect[bl * 4 + 0], s_rect[bl * 4 + 1], s_rect[bl * 4 + 2], s_rect[bl * 4 + 3]};
                const int py0 = rc.y0 + 4 * (r - s_rowbase[bl]);
                int px_lo, px_hi, cnt = 0;
                if (row_span(s_uv + bl * 16, s_flag[bl] != 0, rc, py0, px_lo, px_hi)) cnt = (px_hi - px_lo) / 8 + 1;
                else px_lo = px_hi = 0;
                s_rowinfo[r] = pack_band(bl, py0, px_lo);
                s_rowend[r] = px_hi;
                s_rowprefix[r + 1] = cnt;
            }
            __syncthreads();
            // ---- 1d. tiles before every band (exclusive scan, <= kRowCap entries, 16 per lane) ------------------------
            if (warp == 0) {
                constexpr int PER = kRowCap / 32;
                int c[PER], tot = 0;
#pragma unroll
                for (int i = 0; i < PER; ++i) {
                    const int idx = lane * PER + i;
                    c[i] = idx < R ? s_rowprefix[idx + 1] : 0;
                    tot += c[i];
                }
                int incl = tot;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int up = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += up;
                }
                int run = incl - tot;
#pragma unroll
                for (int i = 0; i < PER; ++i) {
                    const int idx = lane * PER + i;
                    run += c[i];
                    if (idx < R) s_rowprefix[idx + 1] = run;
                }
                if (lane == 0) s_rowprefix[0] = 0;
                if (lane == 31) s_misc[6] = incl;
            }
            if (BWD == 0 && p0 == 0) mbar_wait(bar0 + 8 * stage, parity);  // the brick has landed (first use only)
            __syncthreads();
            const int T = s_misc[6];

            if constexpr (RAYS == 3) {
                // ---- warp-specialised schedule: NPW producer warps test + sort the candidates of round r+1 into one of two
                // work lists while the consumer warps walk the chunks of round r -- no CTA-wide barrier inside a pose chunk
                constexpr int NPW = 4, NCW = Cfg::kWarps - NPW;
                constexpr int LCAP = Cfg::kCap / 2;          // items per list
                constexpr int KP = LCAP / (NPW * 32);        // tiles per producer warp per round
                volatile int* s_ctl = s_misc + 8;            // [0..1] n_items, [2..3] next chunk, [4..5] ready, [6..7] consumers gone
                const int n_rounds = (T + NPW * KP - 1) / (NPW * KP);
                if (tid < 8) s_ctl[tid] = 0;
                __syncthreads();
                if (warp < NPW) {
                    for (int r = 0; r < n_rounds; ++r) {
                        const int slot = r & 1;
                        unsigned items[KP];
#pragma unroll
                        for (int j = 0; j < KP; ++j) items[j] = 0xffffffffu;
                        const int tw0 = (r * NPW + warp) * KP;
                        if (tw0 < T) {
                            int row;
                            {
                                constexpr int STEP = kRowCap / 32;
                                const int probe = min((lane + 1) * STEP, R);
                                const unsigned le = __ballot_sync(0xffffffffu, s_rowprefix[probe] <= tw0);
                                const int coarse = __popc(le) * STEP;
                                const int p2 = min(coarse + lane + 1, R);
                                const unsigned le2 = __ballot_sync(0xffffffffu, lane < STEP && s_rowprefix[p2] <= tw0);
                                row = coarse + __popc(le2);
                            }
#pragma unroll
                            for (int j = 0; j < KP; ++j) {
                                const int t = tw0 + j;
                                if (t < T) {
                                    while (s_rowprefix[row + 1] <= t) ++row;
                                    const unsigned info = s_rowinfo[row];
                                    const int bl = item_pose(info);
                                    const int px = band_col(info) + 8 * (t - s_rowprefix[row]) + (lane & 7);
                                    const int py = band_row(info) + (lane >> 3);
                                    if (px <= s_rowend[row] && py <= s_rect[bl * 4 + 3]) {
                                        const int n = pix_index ? __ldg(pix_index + (py * W + px)) : py * W + px;
                                        if (n < 0) continue;  // pixel not in the caller's ray subset
                                        const float4 q = __ldg(raytab + ((unsigned)(p0 + bl) * (unsigned)Nr + (unsigned)n));
                                        const float4 clo = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 4);
                                        const float4 chi = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 8);
                                        const float inv[3] = {q.x, q.y, q.z};
                                        const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                                        float a_in, a_out;
                                        if (brick_maybe_hit(inv, clo3, chi3, a_in, a_out)) {
                                            const int bin = step_bin(a_in, a_out, q.w, inv_bin_width);
                                            items[j] = pack_item(bin, bl, n);
                                            atomicAdd(&s_hist[bin], 1);
                                        }
                                    }
                                }
                            }
                        }
                        asm volatile("bar.sync 1, %0;" ::"n"(NPW * 32) : "memory");
                        if (warp == 0) {
                            const int h = s_hist[kBrickBins - 1 - lane];
                            int incl = h;
#pragma unroll
                            for (int o = 1; o < 32; o <<= 1) {
                                const int up = __shfl_up_sync(0xffffffffu, incl, o);
                                if (lane >= o) incl += up;
                            }
                            s_cursor[kBrickBins - 1 - lane] = incl - h;
                            s_hist[kBrickBins - 1 - lane] = 0;
                            if (lane == 31) s_misc[0] = incl;
                            // the slot is free once every consumer warp has left the round that used it last
                            if (lane == 0 && r >= 2)
                                while (s_ctl[6 + slot] < NCW * (r / 2)) __nanosleep(40);
                        }
                        asm volatile("bar.sync 1, %0;" ::"n"(NPW * 32) : "memory");
#pragma unroll
                        for (int j = 0; j < KP; ++j)
                            if (items[j] != 0xffffffffu)
                                s_items[slot * LCAP + atomicAdd(&s_cursor[item_bin(items[j])], 1)] = items[j];
                        asm volatile("bar.sync 1, %0;" ::"n"(NPW * 32) : "memory");
                        if (tid == 0) {
                            s_ctl[slot] = s_misc[0];
                            s_ctl[2 + slot] = 0;
                            __threadfence_block();
                            s_ctl[4 + slot] = r + 1;   // publish
                        }
                    }
                } else {
                    for (int r = 0; r < n_rounds; ++r) {
                        const int slot = r & 1;
                        if (lane == 0)
                            while (s_ctl[4 + slot] < r + 1) __nanosleep(40);
                        __syncwarp();
                        __threadfence_block();
                        const int n_items = s_ctl[slot];
                        const int n_chunks = (n_items + 31) >> 5;
                        const unsigned* list = s_items + slot * LCAP;
                        auto claim = [&]() {
                            int c = 0;
                            if (lane == 0) c = atomicAdd(const_cast<int*>(&s_ctl[2 + slot]), 1);
                            return __shfl_sync(0xffffffffu, c, 0);
                        };
                        auto fetch = [&](int c, unsigned& itw, float4& q, float& L) {
                            const int i = c * 32 + lane;
                            itw = 0xffffffffu;
                            if (c < n_chunks && i < n_items) {
                                itw = list[i];
                                const unsigned rr = (unsigned)(p0 + item_pose(itw)) * (unsigned)Nr + (unsigned)item_ray(itw);
                                q = __ldg(raytab + rr);
                                L = __ldg(ltab + rr);
                            }
                        };
                        int c = claim();
                        unsigned itw;
                        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                        float L = 0.0f;
                        fetch(c, itw, q, L);
                        while (c < n_chunks) {
                            const int cn = claim();
                            unsigned itn;
                            float4 qn = make_float4(0.f, 0.f, 0.f, 0.f);
                            float Ln = 0.0f;
                            fetch(cn, itn, qn, Ln);
                            if (itw != 0xffffffffu) {
                                const int bl = item_pose(itw);
                                const float4 S4 = *reinterpret_cast<const float4*>(s_posef + bl * 12);
                                const float4 clo = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 4);
                                const float4 chi = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 8);
                                const float s3[3] = {S4.x, S4.y, S4.z}, inv3[3] = {q.x, q.y, q.z};
                                const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                                const float part = brick_pair_fwd_lean<U, LdShared, true, false>(ld, s3, inv3, clo3, chi3, lo_v, hi_v, org,
                                                                                                 BY * BZ, BZ, 1, shift);
                                if (part != 0.0f)
                                    red_add(out + ((unsigned)(p0 + bl) * (unsigned)Nr + (unsigned)item_ray(itw)), L * part);
                            }
                            c = cn;
                            itw = itn;
                            q = qn;
                            L = Ln;
                        }
                        __syncwarp();
                        if (lane == 0) {
                            __threadfence_block();
                            atomicAdd(const_cast<int*>(&s_ctl[6 + slot]), 1);   // this warp is done with the list
                        }
                    }
                }
                p0 += npose;
                continue;   // next pose chunk (its first statement is the CTA-wide barrier)
            }
            for (int t0 = 0; t0 < T; t0 += Cfg::kWarps * K) {
                // ---- 2. candidates -> hits (kept in registers) + histogram of the sort bins --------------------
                unsigned items[K];
#pragma unroll
                for (int j = 0; j < K; ++j) items[j] = 0xffffffffu;
                const int tw0 = t0 + warp * K;
                if (tw0 < T) {
                    int row;
                    {  // band of the warp's first tile: first index whose prefix exceeds tw0, minus one (two ballots)
                        constexpr int STEP = kRowCap / 32;
                        const int probe = min((lane + 1) * STEP, R);
                        const unsigned le = __ballot_sync(0xffffffffu, s_rowprefix[probe] <= tw0);
                        const int coarse = __popc(le) * STEP;  // prefix[coarse] <= tw0 (or coarse == 0)
                        const int p2 = min(coarse + lane + 1, R);
                        const unsigned le2 = __ballot_sync(0xffffffffu, lane < STEP && s_rowprefix[p2] <= tw0);
                        row = coarse + __popc(le2);
                    }
#pragma unroll
                    for (int j = 0; j < K; ++j) {
                        const int t = tw0 + j;
                        if (t < T) {
                            while (s_rowprefix[row + 1] <= t) ++row;  // warp-uniform, rarely more than one step
                            const unsigned info = s_rowinfo[row];
                            const int bl = item_pose(info);
                            const int px = band_col(info) + 8 * (t - s_rowprefix[row]) + (lane & 7);
                            const int py = band_row(info) + (lane >> 3);
                            if (px <= s_rowend[row] && py <= s_rect[bl * 4 + 3]) {
                                const int n = pix_index ? __ldg(pix_index + (py * W + px)) : py * W + px;
                                if (n < 0) continue;  // pixel not in the caller's ray subset
                                const float4 q = __ldg(raytab + ((unsigned)(p0 + bl) * (unsigned)Nr + (unsigned)n));
                                const float4 clo = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 4);
                                const float4 chi = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 8);
                                const float inv[3] = {q.x, q.y, q.z};
                                const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                                float a_in, a_out;
                                if (brick_maybe_hit(inv, clo3, chi3, a_in, a_out)) {
                                    const int bin = SENS ? sens_bin<U>(inv, a_in, a_out, q.w)
                                                         : step_bin(a_in, a_out, q.w, inv_bin_width);
                                    items[j] = pack_item(bin, bl, n);
                                    atomicAdd(&s_hist[bin], 1);
                                }
                            }
                        }
                    }
                }
                __syncthreads();
                // ---- 3. counting sort, longest bin first ------------------------------------------------------
                if (warp == 0) {
                    const int h = s_hist[kBrickBins - 1 - lane];
                    int incl = h;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int up = __shfl_up_sync(0xffffffffu, incl, o);
                        if (lane >= o) incl += up;
                    }
                    s_cursor[kBrickBins - 1 - lane] = incl - h;
                    s_hist[kBrickBins - 1 - lane] = 0;  // ready for the next round
                    if (lane == 31) {
                        s_misc[0] = incl;
                        s_misc[1] = 0;
                    }
                }
                __syncthreads();
#pragma unroll
                for (int j = 0; j < K; ++j)
                    if (items[j] != 0xffffffffu) s_items[atomicAdd(&s_cursor[item_bin(items[j])], 1)] = items[j];
                __syncthreads();
                // ---- 4. the walks: warps pull 32-item chunks ---------------------------------------------------
                const int n_items = s_misc[0];
                if constexpr (RAYS == 2) {
                    // two (ray, brick) pairs per thread: lane l of chunk c walks items c*64 + l and c*64 + 32 + l
                    const int n_chunks2 = (n_items + 63) >> 6;
                    auto claim2 = [&]() {
                        int c = 0;
                        if (lane == 0) c = atomicAdd(&s_misc[1], 1);
                        return __shfl_sync(0xffffffffu, c, 0);
                    };
                    auto fetch1 = [&](int i, unsigned& itw, float4& q, float& L) {
                        itw = 0xffffffffu;
                        if (i < n_items) {
                            itw = s_items[i];
                            const unsigned r = (unsigned)(p0 + item_pose(itw)) * (unsigned)Nr + (unsigned)item_ray(itw);
                            q = __ldg(raytab + r);
                            L = __ldg(ltab + r);
                        }
                    };
                    int c = claim2();
                    unsigned ita, itb;
                    float4 qa = make_float4(1.f, 1.f, 1.f, 0.f), qb = qa;
                    float La = 0.0f, Lb = 0.0f;
                    if (c < n_chunks2) {
                        fetch1(c * 64 + lane, ita, qa, La);
                        fetch1(c * 64 + 32 + lane, itb, qb, Lb);
                    }
                    while (c < n_chunks2) {
                        const int cn = claim2();
                        unsigned itan = 0xffffffffu, itbn = 0xffffffffu;
                        float4 qan = make_float4(1.f, 1.f, 1.f, 0.f), qbn = qan;
                        float Lan = 0.0f, Lbn = 0.0f;
                        if (cn < n_chunks2) {
                            fetch1(cn * 64 + lane, itan, qan, Lan);
                            fetch1(cn * 64 + 32 + lane, itbn, qbn, Lbn);
                        }
                        if (ita != 0xffffffffu || itb != 0xffffffffu) {
                            const bool va = ita != 0xffffffffu, vb = itb != 0xffffffffu;
                            const int bla = va ? item_pose(ita) : 0, blb = vb ? item_pose(itb) : 0;
                            AccState wa, wb;
                            AccConst ka, kb;
                            {
                                const float4 S4 = *reinterpret_cast<const float4*>(s_posef + bla * 12);
                                const float4 clo = *reinterpret_cast<const float4*>(s_posef + bla * 12 + 4);
                                const float4 chi = *reinterpret_cast<const float4*>(s_posef + bla * 12 + 8);
                                const float s3[3] = {S4.x, S4.y, S4.z}, inv3[3] = {qa.x, qa.y, qa.z};
                                const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                                brick_pair_setup_acc(ld, va, s3, inv3, clo3, chi3, lo_v, hi_v, org, BY * BZ, BZ, 1, shift, wa, ka);
                            }
                            {
                                const float4 S4 = *reinterpret_cast<const float4*>(s_posef + blb * 12);
                                const float4 clo = *reinterpret_cast<const float4*>(s_posef + blb * 12 + 4);
                                const float4 chi = *reinterpret_cast<const float4*>(s_posef + blb * 12 + 8);
                                const float s3[3] = {S4.x, S4.y, S4.z}, inv3[3] = {qb.x, qb.y, qb.z};
                                const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                                brick_pair_setup_acc(ld, vb, s3, inv3, clo3, chi3, lo_v, hi_v, org, BY * BZ, BZ, 1, shift, wb, kb);
                            }
                            float pa, pb;
                            brick_pair2_walk<U>(ld, wa, ka, wb, kb, pa, pb);
                            if (va && pa != 0.0f)
                                red_add(out + ((unsigned)(p0 + bla) * (unsigned)Nr + (unsigned)item_ray(ita)), La * pa);
                            if (vb && pb != 0.0f)
                                red_add(out + ((unsigned)(p0 + blb) * (unsigned)Nr + (unsigned)item_ray(itb)), Lb * pb);
                        }
                        c = cn;
                        ita = itan; itb = itbn;
                        qa = qan; qb = qbn;
                        La = Lan; Lb = Lbn;
                    }
                    continue;  // next round
                }
                const int n_chunks = (n_items + 31) >> 5;
                // (the next chunk's item and ray-table entry are fetched before the current chunk is walked, so the L2
                // latency of the table hides behind a whole walk instead of stalling every chunk's set-up)
                auto claim = [&]() {
                    int c = 0;
                    if (lane == 0) c = atomicAdd(&s_misc[1], 1);
                    return __shfl_sync(0xffffffffu, c, 0);
                };
                auto fetch = [&](int c, unsigned& itw, float4& q, float& L) {
                    const int i = c * 32 + lane;
                    itw = 0xffffffffu;
                    if (c < n_chunks && i < n_items) {
                        itw = s_items[i];
                        if constexpr (SENS == 0) {  // the sensitivities pair loads its ray table entry with its frame record
                            const unsigned r = (unsigned)(p0 + item_pose(itw)) * (unsigned)Nr + (unsigned)item_ray(itw);
                            q = __ldg(raytab + r);
                            L = __ldg(ltab + r);
                        }
                    }
                };
                int c = claim();
                unsigned itw;
                float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                float L = 0.0f;
                fetch(c, itw, q, L);
                while (c < n_chunks) {
                    const int cn = claim();
                    unsigned itn;
                    float4 qn = make_float4(0.f, 0.f, 0.f, 0.f);
                    float Ln = 0.0f;
                    fetch(cn, itn, qn, Ln);
                    if (itw != 0xffffffffu) {
                        const int bl = item_pose(itw);
                        const float4 S4 = *reinterpret_cast<const float4*>(s_posef + bl * 12);
                        const float4 clo = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 4);
                        const float4 chi = *reinterpret_cast<const float4*>(s_posef + bl * 12 + 8);
                        const float s3[3] = {S4.x, S4.y, S4.z}, inv3[3] = {q.x, q.y, q.z};
                        const float clo3[3] = {clo.x, clo.y, clo.z}, chi3[3] = {chi.x, chi.y, chi.z};
                        if constexpr (BWD != 0) {
                            if (L != 0.0f)  // L = gout * raylen here (brick_prep_kernel)
                                brick_pair_bwd_lean<U>(StShared{ld.base_addr}, L, s3, inv3, clo3, chi3, lo_v, hi_v, org, BY * BZ, BZ, 1,
                                                       shift);
                        } else if constexpr (SENS != 0) {
                            const size_t r = (size_t)(p0 + bl) * (size_t)Nr + (size_t)item_ray(itw);
                            const float4* fr = reinterpret_cast<const float4*>(sa.frames + r);
                            const SensFrameRec rec{__ldg(fr), __ldg(fr + 1)};
                            const float4 qi = __ldg(raytab + r);
                            const float inv[3] = {qi.x, qi.y, qi.z};
                            float d[3], Lr;
                            const VolFrame f = unpack_sens_frame(rec, inv, d, Lr);
                            float A[3] = {0.0f, 0.0f, 0.0f}, C[3] = {0.0f, 0.0f, 0.0f};
                            const float S = brick_pair_sens_framed<U>(ld, f, s3, d, dims, lo_v, hi_v, org, BY * BZ, BZ, 1, shift, A, C);
                            float jt[3], js[3];
                            bool any = S != 0.0f;
#pragma unroll
                            for (int a = 0; a < 3; ++a) {
                                const float k = Lr * inv[a];
                                jt[a] = -k * A[a];
                                js[a] = k * (A[a] - C[a]);
                                any = any || jt[a] != 0.0f || js[a] != 0.0f;
                            }
                            if (any) {
                                red_add4(sa.sens + r * 8, jt[0], jt[1], jt[2], S);
                                red_add4(sa.sens + r * 8 + 4, js[0], js[1], js[2], 0.0f);
                                red_add(out + r, Lr * S);
                            }
                        } else {
                            const float part = brick_pair_fwd_lean<U, LdShared, true, PIPE != 0>(ld, s3, inv3, clo3, chi3, lo_v, hi_v, org, BY * BZ, BZ, 1, shift);
                            if (part != 0.0f)
                                red_add(out + ((unsigned)(p0 + bl) * (unsigned)Nr + (unsigned)item_ray(itw)), L * part);
                        }
                    }
                    c = cn;
                    itw = itn;
                    q = qn;
                    L = Ln;
                }
            }
            p0 += npose;
        }
        if constexpr (BWD != 0) fence_proxy_async();  // this thread's scatter adds become visible to the async proxy (TMA store)
        __syncthreads();  // every reader of this stage (and of s_misc[2 + ...]) is done
        if (STAGES == 1) {
            if (tid == 0) {
                if constexpr (BWD != 0) {
                    tma_store_3d(&tmap, brick0, i2 * BZ, i1 * BY, i0 * BX);
                    tma_store_wait_read();  // the brick has been read out: the next zero fill may overwrite it
                }
                const int nxt = (int)atomicAdd(counter, 1u);
                s_misc[2 + ((it + 1) & 1)] = nxt;
                if (BWD == 0 && nxt < n_bricks) issue(nxt, 0);
            }
            __syncthreads();
        }
        cur = s_misc[2 + ((it + 1) & 1)];
    }
    if constexpr (BWD != 0) {
        if (tid == 0) tma_store_wait_all();
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encoder()
{
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

template <class V> constexpr CUtensorMapDataType tmap_type() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }
template <> constexpr CUtensorMapDataType tmap_type<VoxF16>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT16; }
template <> constexpr CUtensorMapDataType tmap_type<VoxBF16>() { return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }

// Out-of-bounds elements are zero-filled (+0.0 in every element type).  The global strides must be multiples of 16 bytes:
// D2 % 4 == 0 for fp32 voxels, D2 % 8 == 0 for 16-bit ones (siddon_brick_supported).
template <class V>
bool make_volume_map(CUtensorMap* map, const V* vol, VolDims dims, int BX, int BY, int BZ, bool swizzle128 = false)
{
    EncodeTiledFn enc = get_encoder();
    if (!enc) return false;
    constexpr cuuint64_t es = sizeof(V);
    const cuuint64_t gdim[3] = {(cuuint64_t)dims.d[2], (cuuint64_t)dims.d[1], (cuuint64_t)dims.d[0]};
    const cuuint64_t gstride[2] = {(cuuint64_t)dims.d[2] * es, (cuuint64_t)dims.d[2] * dims.d[1] * es};
    const cuuint32_t box[3] = {(cuuint32_t)BZ, (cuuint32_t)BY, (cuuint32_t)BX};
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, tmap_type<V>(), 3, const_cast<V*>(vol), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 && es == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <int BX, int BY, int BZ, int STAGES, int THREADS, int K, int U, int CTAS, int PIPE, int RAYS = 1, int BWD = 0, int SENS = 0,
          class V = float>
cudaError_t launch_brick_variant(const CUtensorMap& map, VolDims dims, const float4* raytab, const float* ltab,
                                 const PoseGeo* geo, float* out, unsigned* counter, const int* pix_index, int Nr, int B, int H,
                                 int W, float shift, cudaStream_t stream, const SensArgs& sa = SensArgs{})
{
    using Cfg = BrickCfg<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, PIPE, RAYS, V>;
    auto kern = siddon_fwd_brick_kernel<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, PIPE, RAYS, BWD, SENS, V>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
        if (e != cudaSuccess) return e;
        configured = true;
    }
    BrickGrid bg;
    bg.nb0 = (dims.d[0] + BX - 1) / BX;
    bg.nb1 = (dims.d[1] + BY - 1) / BY;
    bg.nb2 = (dims.d[2] + BZ - 1) / BZ;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    static_assert(Cfg::kSmemBytes <= (233472 - 1024 * CTAS) / CTAS, "shared-memory carve-up exceeds the SM");
    const int ctas_per_sm = CTAS;
    const int grid = min(bg.nb0 * bg.nb1 * bg.nb2, sms * ctas_per_sm);
    kern<<<grid, THREADS, Cfg::kSmemBytes, stream>>>(map, dims, bg, raytab, ltab, geo, out, counter, pix_index, Nr, B, H, W, shift,
                                                     sa);
    return cudaGetLastError();
}

}  // namespace

size_t siddon_brick_workspace_bytes(int B, int H, int W)
{
    return 256 + align_up(sizeof(PoseGeo) * (size_t)B, 256) + (sizeof(float4) + sizeof(float)) * (size_t)B * H * W;
}

// The sensitivities mode's scratch: the forward workspace, then one SensFrameRec per ray (32-byte aligned: one L2 sector each).
size_t siddon_sens_brick_scratch_bytes(int B, int H, int W)
{
    return align_up(siddon_brick_workspace_bytes(B, H, W), 256) + sizeof(SensFrameRec) * (size_t)B * H * W;
}

bool siddon_brick_supported(VolDims dims, int H, int W, int elem_bytes)
{
    return ((int64_t)dims.d[2] * elem_bytes) % 16 == 0 && H <= kBrickMaxSide && W <= kBrickMaxSide && H >= 2 && W >= 2 && get_encoder() != nullptr;
}

// pix_index / corners / Nsub describe a ray SUBSET of the H x W grid (all nullptr / 0 for the full grid): tgt, raylen and out
// are then (B, Nsub) arrays, pix_index [H*W] maps a pixel to its ray (-1: none), corners [B][3][3] are the voxel-space
// targets of the full grid's pixels (0,0), (0,W-1), (H-1,0).
template <class V>
cudaError_t launch_siddon_fwd_brick(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                    const float* G, const float* Wd, const float* rows, const float* cols, float* out,
                                    void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                    int variant, cudaStream_t stream, const int* pix_index, const float* corners, int64_t Nsub)
{
    const bool subset = pix_index != nullptr;
    const int64_t Nr = subset ? Nsub : (int64_t)H * W;
    if (!siddon_brick_supported(dims, H, W, (int)sizeof(V)) || ((uintptr_t)vol & 15u) != 0 || (int64_t)B * Nr >= ((int64_t)1 << 31) || Nr <= 0 ||
        Nr > (int64_t)H * W || (subset && (corners == nullptr || G != nullptr)))
        return cudaErrorNotSupported;
    const size_t need = 256 + align_up(sizeof(PoseGeo) * (size_t)B, 256) + (sizeof(float4) + sizeof(float)) * (size_t)B * Nr;
    if (workspace == nullptr || workspace_bytes < need || ((uintptr_t)workspace & 255u) != 0) return cudaErrorInvalidValue;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    unsigned* counter = reinterpret_cast<unsigned*>(ws);
    PoseGeo* geo = reinterpret_cast<PoseGeo*>(ws + 256);
    float4* raytab = reinterpret_cast<float4*>(ws + 256 + align_up(sizeof(PoseGeo) * (size_t)B, 256));
    float* ltab = reinterpret_cast<float*>(raytab + (size_t)B * Nr);
    PoseRaysB pr{G, Wd, rows, cols};
    brick_prep_kernel<<<dim3((unsigned)((Nr + 255) / 256), (unsigned)B), 256, 0, stream>>>(src, tgt, raylen, pr, raytab, ltab, geo,
                                                                                         out, counter, H, W, eps, Nr,
                                                                                         subset ? corners : nullptr, nullptr);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    CUtensorMap map;
    if (variant == 0) {  // two CTAs per SM, one 96 KB brick each (production shape); 16-bit bricks are staged unswizzled
        if (!make_volume_map(&map, vol, dims, 24, 32, 32, B200DRR_FWD_SWIZZLE != 0 && sizeof(V) == 4)) return cudaErrorNotSupported;
        return launch_brick_variant<24, 32, 32, 1, 512, 4, 2, 2, 0, 1, 0, 0, V>(map, dims, raytab, ltab, geo, out, counter, pix_index,
                                                                                (int)Nr, B, H, W, shift, stream);
    }
#ifdef B200DRR_EXPERIMENTS  // tuning variants, all measured and not chosen; fp32 volumes only, not in the shipped library
#define BV(id, BX, BY, BZ, STAGES, THREADS, K, U, CTAS, PIPE)                                                            \
    case id:                                                                                                             \
        if (!make_volume_map(&map, vol, dims, BX, BY, BZ, B200DRR_FWD_SWIZZLE != 0 && BZ == 32)) return cudaErrorNotSupported;                                 \
        return launch_brick_variant<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, PIPE, 1, 0, 0, V>(map, dims, raytab, ltab, geo, out, counter, \
                                                                                   pix_index, (int)Nr, B, H, W, shift, stream);
#define BV3(id, BX, BY, BZ, STAGES, THREADS, K, U, CTAS)                                                                 \
    case id:                                                                                                             \
        if (!make_volume_map(&map, vol, dims, BX, BY, BZ, B200DRR_FWD_SWIZZLE != 0 && BZ == 32)) return cudaErrorNotSupported;                                 \
        return launch_brick_variant<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, 0, 3, 0, 0, V>(map, dims, raytab, ltab, geo, out, counter, \
                                                                                   pix_index, (int)Nr, B, H, W, shift, stream);
#define BV2(id, BX, BY, BZ, STAGES, THREADS, K, U, CTAS)                                                                 \
    case id:                                                                                                             \
        if (!make_volume_map(&map, vol, dims, BX, BY, BZ, B200DRR_FWD_SWIZZLE != 0 && BZ == 32)) return cudaErrorNotSupported;                                 \
        return launch_brick_variant<BX, BY, BZ, STAGES, THREADS, K, U, CTAS, 0, 2, 0, 0, V>(map, dims, raytab, ltab, geo, out, counter, \
                                                                                   pix_index, (int)Nr, B, H, W, shift, stream);
    if constexpr (sizeof(V) == 4) {
    switch (variant) {
        BV(1, 24, 32, 32, 1, 512, 4, 2, 2, 1)    // the production shape with the software-pipelined walk
        BV(2, 24, 32, 32, 1, 512, 4, 4, 2, 1)
        BV(3, 24, 32, 32, 1, 512, 4, 4, 2, 0)
        BV(4, 22, 32, 32, 1, 512, 8, 2, 2, 1)    // bigger rounds (fewer barriers), slightly smaller brick
        BV(5, 15, 32, 32, 1, 320, 4, 2, 3, 1)    // three CTAs per SM
        BV(6, 15, 32, 32, 1, 320, 4, 2, 3, 0)
        BV(7, 24, 32, 32, 2, 1024, 4, 2, 1, 1)   // one CTA per SM with a two-stage TMA + mbarrier pipeline (slower: CTA-wide barriers)
        BV(8, 24, 32, 32, 2, 1024, 4, 2, 1, 0)
        BV(9, 12, 32, 32, 2, 512, 4, 2, 2, 1)    // two CTAs per SM, each with a two-stage pipeline of 48 KB bricks
        BV(10, 24, 32, 32, 1, 384, 5, 2, 2, 1)
        BV(11, 48, 32, 32, 1, 1024, 4, 2, 1, 0)  // one CTA per SM, one 192 KB brick: fewer (ray, brick) pairs, no second CTA to hide barriers
        BV(12, 32, 32, 32, 1, 1024, 4, 2, 1, 0)
        BV(13, 48, 32, 32, 1, 768, 4, 2, 1, 0)
        BV2(20, 24, 32, 32, 1, 256, 8, 2, 2)     // two rays per thread (ILP), 2 CTAs x 256 threads: 1.28 ms
        BV2(21, 24, 32, 32, 1, 320, 6, 2, 2)
        BV2(22, 24, 32, 32, 1, 384, 5, 2, 2)
        BV2(23, 24, 32, 32, 1, 256, 8, 1, 2)
        BV2(24, 24, 32, 32, 1, 512, 4, 2, 2)     // 1.22 ms
        BV3(30, 24, 32, 32, 1, 512, 4, 2, 2)     // warp-specialised: 4 producer warps (test + sort) / 12 consumer warps (walk): 1.25 ms
        BV3(31, 24, 32, 32, 1, 512, 4, 4, 2)
        default: break;
    }
    }
#undef BV
#undef BV2
#undef BV3
#endif
    return cudaErrorInvalidValue;
}
template cudaError_t launch_siddon_fwd_brick<float>(const float*, VolDims, const float*, const float*, const float*, const float*,
                                                    const float*, const float*, const float*, float*, void*, size_t, int, int, int,
                                                    float, float, int, cudaStream_t, const int*, const float*, int64_t);
template cudaError_t launch_siddon_fwd_brick<VoxF16>(const VoxF16*, VolDims, const float*, const float*, const float*, const float*,
                                                     const float*, const float*, const float*, float*, void*, size_t, int, int, int,
                                                     float, float, int, cudaStream_t, const int*, const float*, int64_t);
template cudaError_t launch_siddon_fwd_brick<VoxBF16>(const VoxBF16*, VolDims, const float*, const float*, const float*,
                                                      const float*, const float*, const float*, const float*, float*, void*, size_t,
                                                      int, int, int, float, float, int, cudaStream_t, const int*, const float*,
                                                      int64_t);

// Volume gradient of the full-grid Siddon render through the brick kernel's BWD mode: g_vol [D0][D1][D2] is OVERWRITTEN with
// sum over poses and rays of gout * raylen * chord length (what autograd gives for renderers.py:40-76 w.r.t. the volume).
cudaError_t launch_siddon_bwd_vol_brick(const float* gout, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                        const float* G, const float* Wd, const float* rows, const float* cols, float* g_vol,
                                        void* workspace, size_t workspace_bytes, int B, int H, int W, float shift, float eps,
                                        cudaStream_t stream)
{
    const int64_t Nr = (int64_t)H * W;
    if (!siddon_brick_supported(dims, H, W, 4) || ((uintptr_t)g_vol & 15u) != 0 || (int64_t)B * Nr >= ((int64_t)1 << 31))
        return cudaErrorNotSupported;
    const size_t need = siddon_brick_workspace_bytes(B, H, W);
    if (workspace == nullptr || workspace_bytes < need || ((uintptr_t)workspace & 255u) != 0) return cudaErrorInvalidValue;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    unsigned* counter = reinterpret_cast<unsigned*>(ws);
    PoseGeo* geo = reinterpret_cast<PoseGeo*>(ws + 256);
    float4* raytab = reinterpret_cast<float4*>(ws + 256 + align_up(sizeof(PoseGeo) * (size_t)B, 256));
    float* ltab = reinterpret_cast<float*>(raytab + (size_t)B * Nr);
    PoseRaysB pr{G, Wd, rows, cols};
    brick_prep_kernel<<<dim3((unsigned)((Nr + 255) / 256), (unsigned)B), 256, 0, stream>>>(src, tgt, raylen, pr, raytab, ltab, geo,
                                                                                         nullptr, counter, H, W, eps, Nr, nullptr,
                                                                                         gout);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    CUtensorMap map;
#ifndef B200DRR_BWD_U
#define B200DRR_BWD_U 4  // steps per group of the scatter walk (4 was the fastest of 1, 2, 4 before the port)
#endif
    // Candidate tiles per warp and round (K): bigger rounds = fewer CTA-wide barriers, at the price of
    // a smaller brick to keep two CTAs per SM.  Tuned before the port (not re-measured on the H100): K = 8
    // with 22-plane bricks was fastest at 16 poses, K = 4 with 24-plane bricks at 4 -- so big batches take K = 8.
    if (B >= 8) {
        if (!make_volume_map(&map, g_vol, dims, 22, 32, 32, B200DRR_BWD_SWIZZLE != 0)) return cudaErrorNotSupported;
        return launch_brick_variant<22, 32, 32, 1, 512, 8, B200DRR_BWD_U, 2, 0, 1, 1>(map, dims, raytab, ltab, geo, nullptr, counter,
                                                                                     nullptr, (int)Nr, B, H, W, shift, stream);
    }
    if (!make_volume_map(&map, g_vol, dims, 24, 32, 32, B200DRR_BWD_SWIZZLE != 0)) return cudaErrorNotSupported;
    return launch_brick_variant<24, 32, 32, 1, 512, 4, B200DRR_BWD_U, 2, 0, 1, 1>(map, dims, raytab, ltab, geo, nullptr, counter,
                                                                                 nullptr, (int)Nr, B, H, W, shift, stream);
}

// ---- training step: image + per-ray sensitivities through the SENS mode ---------------------------------------------------------
#ifndef B200DRR_SENS_U
// Walk steps per group.  Each walk pads its last group to U steps, so a smaller U wastes fewer steps per pair (a pair walks ~30
// voxels) and a larger one keeps more shared-memory loads in flight.  H100 80GB HBM3, 700 W, bench.py, sensitivities launch at 16
// poses: U = 4 2.037 ms, 5 2.023, 6 2.000, 7 2.034, 8 2.044.  All fit the 64 registers of 2 CTAs x 512 threads without spills.
#define B200DRR_SENS_U 6
#endif
// Batches of at least this many poses take the brick path.  H100 80GB HBM3, 700 W, 512^3 -> 256^2 (scripts/sens_brick_sweep.py
// --block 20, median us per launch, brick / best of the others), with the per-ray frame record: 2 poses 373 / 391 (pieces),
// 4: 565 / 628, 8: 1061 / 1268, 16: 2041 / 2396, 32: 4003 / 4491 (slab-major) -- from 4 poses on the brick kernel wins by 11-17 %;
// the 5 % at 2 poses is one sweep (2 % before the record, inside the noise), not yet enough to move the threshold.
constexpr int kSensBrickMinBatch = 4;

// The one routing rule of the training step (b200drr_siddon_fwd_sens_grid variant 0 and b200drr_siddon_fwd_sens_pose): the brick
// kernel can take the shape (siddon_brick_supported, 16-byte aligned volume and sensitivities), the volume has enough bricks for
// the dynamic queue of 2 x 132 resident CTAs to balance (>= 2048 bricks of 24 x 32 x 32), the rays are sparse (detector pixels at
// most half the voxels of a volume cross-section, as the module's forward routing requires: dense rays share L1 sectors and the
// slab-major gather wins), the batch is big enough for the staged bricks to be shared and no side of the volume is longer than the
// per-ray frame record can index (kSensFrameMaxSide).
bool siddon_sens_brick_route(VolDims dims, int B, int H, int W, const void* vol, const float* sens, int elem_bytes)
{
    const int64_t n_bricks = (int64_t)((dims.d[0] + 23) / 24) * ((dims.d[1] + 31) / 32) * ((dims.d[2] + 31) / 32);
    const double nvox = (double)dims.d[0] * dims.d[1] * dims.d[2];
    const bool sparse = (double)H * W <= 0.5 * pow(nvox, 2.0 / 3.0);
    const bool indexable = dims.d[0] <= kSensFrameMaxSide && dims.d[1] <= kSensFrameMaxSide && dims.d[2] <= kSensFrameMaxSide;
    return B >= kSensBrickMinBatch && n_bricks >= 2048 && sparse && indexable && (int64_t)B * H * W < ((int64_t)1 << 31) &&
           ((uintptr_t)vol & 15u) == 0 && ((uintptr_t)sens & 15u) == 0 && siddon_brick_supported(dims, H, W, elem_bytes);
}

// Scratch pool of the sensitivities mode, one per device.  Its release threshold is unlimited: memory freed into it stays
// reserved for the next call, so a training loop that synchronises with the host every step does not hand the ~21 MB back to
// the driver at each synchronisation and map it again on the next call (the default pool's threshold is 0; that cost 20-50 % of
// the eager end-to-end step).  The pool keeps at most the largest scratch one call has needed.
static cudaMemPool_t sens_scratch_pool(int dev)
{
    static cudaMemPool_t pools[64] = {};
    static std::mutex mu;
    if (dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    if (pools[dev] == nullptr) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        cudaMemPool_t pool = nullptr;
        if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
        cuuint64_t keep = ~(cuuint64_t)0;
        if (cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep) != cudaSuccess) {
            cudaMemPoolDestroy(pool);
            return nullptr;
        }
        pools[dev] = pool;
    }
    return pools[dev];
}

// out [B][H*W] and sens [B][H*W][8] are overwritten (zero-filled by brick_prep_kernel, then summed into by the pairs).
template <class V>
cudaError_t launch_siddon_fwd_sens_brick(const V* vol, VolDims dims, const float* src, const float* tgt, const float* raylen,
                                         const float* G, const float* Wd, const float* rows, const float* cols, float* out,
                                         float* sens, int B, int H, int W, float shift, float eps, cudaStream_t stream)
{
    const int64_t Nr = (int64_t)H * W;
    if (!siddon_brick_supported(dims, H, W, (int)sizeof(V)) || ((uintptr_t)vol & 15u) != 0 || ((uintptr_t)sens & 15u) != 0 ||
        (int64_t)B * Nr >= ((int64_t)1 << 31) || dims.d[0] > kSensFrameMaxSide || dims.d[1] > kSensFrameMaxSide ||
        dims.d[2] > kSensFrameMaxSide)
        return cudaErrorNotSupported;
    CUtensorMap map;
    if (!make_volume_map(&map, vol, dims, 24, 32, 32, B200DRR_FWD_SWIZZLE != 0)) return cudaErrorNotSupported;
    // Scratch (claim counter, per-pose geometry, ray table, frame records: ~55 MB at 16 poses of 256^2) from the stream-ordered
    // allocator: no workspace argument, nothing shared across streams, no device-wide sync.  Eager calls take it from
    // sens_scratch_pool; inside CUDA-graph capture the allocation becomes a pair of allocation / free nodes whose memory the graph
    // itself keeps.
    const size_t bytes = siddon_sens_brick_scratch_bytes(B, H, W);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaError_t e = cudaStreamIsCapturing(stream, &cap);
    if (e != cudaSuccess) return e;
    void* ws = nullptr;
    if (cap == cudaStreamCaptureStatusNone) {
        int dev = 0;
        e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        cudaMemPool_t pool = sens_scratch_pool(dev);
        if (pool == nullptr) return cudaErrorMemoryAllocation;
        e = cudaMallocFromPoolAsync(&ws, bytes, pool, stream);
    } else {
        e = cudaMallocAsync(&ws, bytes, stream);
    }
    if (e != cudaSuccess) return e;
    unsigned char* w8 = static_cast<unsigned char*>(ws);
    unsigned* counter = reinterpret_cast<unsigned*>(w8);
    PoseGeo* geo = reinterpret_cast<PoseGeo*>(w8 + 256);
    float4* raytab = reinterpret_cast<float4*>(w8 + 256 + align_up(sizeof(PoseGeo) * (size_t)B, 256));
    float* ltab = reinterpret_cast<float*>(raytab + (size_t)B * Nr);
    SensFrameRec* frames = reinterpret_cast<SensFrameRec*>(w8 + align_up(siddon_brick_workspace_bytes(B, H, W), 256));
    const PoseRaysB pr{G, Wd, rows, cols};
    if (((uintptr_t)ws & 255u) != 0) e = cudaErrorInvalidValue;
    if (e == cudaSuccess) {
        brick_prep_kernel<<<dim3((unsigned)((Nr + 255) / 256), (unsigned)B), 256, 0, stream>>>(
            src, tgt, raylen, pr, raytab, ltab, geo, out, counter, H, W, eps, Nr, nullptr, nullptr, sens, frames, dims, shift);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        const SensArgs sa{frames, sens};
        e = launch_brick_variant<24, 32, 32, 1, 512, 4, B200DRR_SENS_U, 2, 0, 1, 0, 1, V>(map, dims, raytab, ltab, geo, out, counter,
                                                                                      nullptr, (int)Nr, B, H, W, shift, stream, sa);
    }
    const cudaError_t ef = cudaFreeAsync(ws, stream);
    return e != cudaSuccess ? e : ef;
}
#define B200DRR_SENS_BRICK(V)                                                                                                      \
    template cudaError_t launch_siddon_fwd_sens_brick<V>(const V*, VolDims, const float*, const float*, const float*, const float*, \
                                                         const float*, const float*, const float*, float*, float*, int, int, int,   \
                                                         float, float, cudaStream_t);
B200DRR_SENS_BRICK(float)
B200DRR_SENS_BRICK(VoxF16)
B200DRR_SENS_BRICK(VoxBF16)
#undef B200DRR_SENS_BRICK

}  // namespace b200drr
