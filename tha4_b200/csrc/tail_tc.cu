// Fused decoder tail on the tensor cores (default precision mode) -- SURVEY.md section 8 a-T.  From the RAW last feature map of a network (f16, NHWC, written by the
// producing conv's epilogue) to every tensor the network returns, one pass, HBM-bound by design:
//
//   TMA     one 4-D box {C ch, 130 w, TR+2 h, 1 n} = the (TR+2) x 130 pixel HALO of a 128 x TR pixel tile lands in shared
//           memory as 128-byte (C = 64) / 64-byte (C = 32) rows with the matching swizzle; out-of-image pixels are
//           zero-filled = the head conv's zero padding.  The nine 16 x C head-weight tiles come in with one more box.
//   warps   apply the pending GroupNorm / InstanceNorm affine + SiLU / ReLU to the halo IN PLACE (the affine is rebuilt
//           per CTA from the statistics the producing conv accumulated: no finalize kernel, no coefficient tensor).
//   wgmma   the 3x3 head conv is 9 taps x C/16 x 2 wgmma (M = 128 pixels of one tile row as two m64 halves, N = 16 head
//           channels, K = 16) per tile row, straight from the halo: the A descriptor of tap (dy, dx) is the SAME shared-memory
//           image with its start address shifted by (dy * 130 + dx) rows -- the tensor core applies the swizzle on absolute
//           addresses, so any row shift is legal.  Accumulators: TR x 16 columns in registers.
//   drain   the accumulator goes through shared memory (the halo is free by then) so that every thread gets the 16 head
//           outputs of ITS pixel; sigmoid / tanh, affine_grid + grid_sample (4-tap gather from the planar image), blends, and planar NCHW stores
//           where the 32 lanes of a warp write 32 consecutive pixels = one full 128-byte line per channel.
// Reference: morpher_00.py:53-66, upscaler_02.py:84-96, face_morpher_08.py:170-193, eyebrow_morphing_combiner_00.py:51-72,
// eyebrow_decomposer_00.py:49-64.  The fp32 / strict variant is tail.cu.
#include "ops.cuh"
#include "tail_epilogue.cuh"
#include "profiler.cuh"
#include "tc_common.cuh"
#include <cuda.h>
#include <cmath>
#include <map>
#include <mutex>
#include <tuple>

namespace tha4 {
namespace {

using namespace tc;

constexpr int TT_W = 128, TT_HW = TT_W + 2;          // tile / halo width in pixels
constexpr int TT_THREADS = 128;
constexpr int TT_N = 16;                             // head channels of the MMA (TAIL_CO_PAD = 12 real ones at most)

struct TailTcParams {
    int S, N;
    const double* stats; int stats_ld, stats_rep; long stats_rep_stride;   // statistics of the raw feature map
    int groups, act;
    const float* gamma; const float* beta;
    const float* bias;               // [TAIL_CO_PAD]
    float acc_scale;
    ImgView img0, img1;
    const float* g0; int g0_ld; const float* g1; int g1_ld;     // optional interleaved (NHWC) copies of img0 / img1 (tail_epilogue.cuh)
    const float* base;
    float* o[8];
};

template <int C> struct TailCfg {
    static constexpr int ROWB = 2 * C;                // bytes per pixel row of the operand (f16)
    static constexpr int TR = C == 32 ? 4 : 2;        // tile rows per CTA (shared-memory budget: 3 / 2 CTAs per SM)
    static constexpr int HROWS = (TR + 2) * TT_HW;    // halo pixels
    static constexpr int A_BYTES = ((HROWS * ROWB + 1023) / 1024) * 1024;
    static constexpr int B_BYTES = 9 * TT_N * ROWB;
    static constexpr size_t SMEM = 1024 + A_BYTES + B_BYTES + 2 * C * sizeof(float) + 2 * C * sizeof(double) + 16 * sizeof(float) + 64;
};

template <int KIND, int C>
__global__ void __launch_bounds__(TT_THREADS) tail_tc_kernel(const __grid_constant__ CUtensorMap tmF, const __grid_constant__ CUtensorMap tmW,
                                                              const TailTcParams p) {
    using Cfg = TailCfg<C>;
    constexpr int ROWB = Cfg::ROWB, TR = Cfg::TR, NCH = ROWB / 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);      // pointer arithmetic (not an integer round trip) keeps the shared address space: LDS / STS, not generic LD / ST
    uint8_t* smA = smem;
    uint8_t* smB = smem + Cfg::A_BYTES;
    double* chs = reinterpret_cast<double*>(smB + Cfg::B_BYTES);         // [C][2] folded statistics
    float* cA = reinterpret_cast<float*>(chs + 2 * C);                   // [C] affine
    float* cB = cA + C;
    float* sbias = cB + C;                                               // [16]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + 16);            // tma_full

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n = blockIdx.z, x0 = blockIdx.x * TT_W, y0 = blockIdx.y * TR;

    if (tid == 0) {
        mbar_init(smem_u32(bars), 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmF) : "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmW) : "memory");
    }
    __syncthreads();
    pdl_trigger();
    if (tid == 0) {        // the head weights do not depend on the previous kernel: fetch them ahead of the dependency wait
        mbar_expect_tx(smem_u32(bars), Cfg::HROWS * ROWB + Cfg::B_BYTES);
        tma_load_3d(smem_u32(smB), &tmW, 0, 0, 0, smem_u32(bars));
    }
    if (tid < 16) sbias[tid] = tid < TAIL_CO_PAD ? __ldg(p.bias + tid) : 0.0f;
    pdl_wait();
    if (tid == 0) tma_load_4d(smem_u32(smA), &tmF, 0, x0 - 1, y0 - 1, n, smem_u32(bars));

    // ---- per-channel affine of the pending normalisation, from the producer's statistics ----
    const int cpg = p.groups == 0 ? 1 : C / p.groups;
    for (int c = tid; c < C; c += TT_THREADS) {
        const double2 v = fold_stat_replicas(p.stats + ((long)n * p.stats_ld + c) * 2, p.stats_rep_stride, p.stats_rep);
        chs[2 * c] = v.x; chs[2 * c + 1] = v.y;
    }
    __syncthreads();
    const bool silu = p.act == ACT_SILU || p.act == ACT_SILU_FAST;
    for (int c = tid; c < C; c += TT_THREADS) {
        const int g0 = (c / cpg) * cpg;
        double su = 0.0, sq = 0.0;
        for (int j = 0; j < cpg; ++j) { su += chs[2 * (g0 + j)]; sq += chs[2 * (g0 + j) + 1]; }
        const double inv_cnt = 1.0 / ((double)p.S * p.S * cpg);          // fp64 for the sums and the cancelling subtraction only
        const double mean = su * inv_cnt;
        const float var = fmaxf((float)fma(sq, inv_cnt, -mean * mean), 0.0f);
        float A = rsqrtf(var + 1e-5f) * __ldg(p.gamma + c);
        float B = __ldg(p.beta + c) - (float)mean * A;
        if (silu) { A *= 0.5f; B *= 0.5f; }                                // silu(v) = h + h * tanh(h), h = v / 2
        cA[c] = A; cB[c] = B;
    }
    __syncthreads();

    // ---- normalise + activate the halo in place (zero padding stays zero) ----
    mbar_wait(smem_u32(bars), 0);
    for (int row = tid; row < Cfg::HROWS; row += TT_THREADS) {
        const int hy = row / TT_HW, hx = row - hy * TT_HW;
        const int gy = y0 - 1 + hy, gx = x0 - 1 + hx;
        if (gy < 0 || gy >= p.S || gx < 0 || gx >= p.S) continue;
        uint8_t* rowp = smA + row * ROWB;
        const int swz = ROWB == 128 ? (row & 7) : ((row >> 1) & 3);        // smA is 1024-byte aligned: the row's XOR term of the swizzle
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
            uint4* dp = reinterpret_cast<uint4*>(rowp + ((j ^ swz) << 4));
            uint4 d = *dp;
            const float4 a0 = *reinterpret_cast<const float4*>(cA + 8 * j), a1 = *reinterpret_cast<const float4*>(cA + 8 * j + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(cB + 8 * j), b1 = *reinterpret_cast<const float4*>(cB + 8 * j + 4);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            __half2* hp = reinterpret_cast<__half2*>(&d);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 v = __half22float2(hp[e]);
                v.x = fmaf(v.x, av[2 * e], bv[2 * e]); v.y = fmaf(v.y, av[2 * e + 1], bv[2 * e + 1]);
                if (silu) {
                    float tx, ty;
                    asm("tanh.approx.f32 %0, %1;\n" : "=f"(tx) : "f"(v.x));
                    asm("tanh.approx.f32 %0, %1;\n" : "=f"(ty) : "f"(v.y));
                    v.x = fmaf(v.x, tx, v.x); v.y = fmaf(v.y, ty, v.y);
                } else if (p.act == ACT_RELU) {
                    v.x = fmaxf(v.x, 0.0f); v.y = fmaxf(v.y, 0.0f);
                }
                hp[e] = __floats2half2_rn(v.x, v.y);
            }
            *dp = d;
        }
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");          // generic-proxy writes -> the tensor core's async-proxy reads
    __syncthreads();

    // ---- 3x3 head conv: the warpgroup issues TR x 9 x C/16 x 2 wgmma on row-shifted views of the halo ----
    float acc[TR][2][8];
    wg_fence();
#pragma unroll
    for (int r = 0; r < TR; ++r)
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap - 3 * dy;
            const uint32_t a = smem_u32(smA + ((r + dy) * TT_HW + dx) * ROWB), b = smem_u32(smB + tap * TT_N * ROWB);
#pragma unroll
            for (int k = 0; k < C / 16; ++k) {
                const uint64_t bd = make_smem_desc_sw<ROWB>(b + 32 * k);
                Wgmma<TT_N>::f16(acc[r][0], make_smem_desc_sw<ROWB>(a + 32 * k), bd, (tap > 0 || k > 0) ? 1u : 0u);
                Wgmma<TT_N>::f16(acc[r][1], make_smem_desc_sw<ROWB>(a + 64 * ROWB + 32 * k), bd, (tap > 0 || k > 0) ? 1u : 0u);
            }
        }
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int r = 0; r < TR; ++r) { wg_fence_acc(acc[r][0]); wg_fence_acc(acc[r][1]); }

    // ---- drain: thread = pixel column x0 + tid; its 16 head outputs per tile row, transposed through the (now idle) halo ----
    float* stage = reinterpret_cast<float*>(smA);                        // [128][17]
    const int x = x0 + tid;
#pragma unroll
    for (int r = 0; r < TR; ++r) {
        __syncthreads();                                                 // every wgmma has read the halo / the previous row is drained
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int col = 8 * j + 2 * (lane & 3), row = h * 64 + warp * 16 + (lane >> 2);
                stage[row * 17 + col] = acc[r][h][4 * j];           stage[row * 17 + col + 1] = acc[r][h][4 * j + 1];
                stage[(row + 8) * 17 + col] = acc[r][h][4 * j + 2]; stage[(row + 8) * 17 + col + 1] = acc[r][h][4 * j + 3];
            }
        __syncthreads();
        if (x < p.S) {
            float o[TAIL_CO_PAD];
#pragma unroll
            for (int j = 0; j < TAIL_CO_PAD; ++j) o[j] = fmaf(stage[tid * 17 + j], p.acc_scale, sbias[j]);
            tail_epilogue<KIND>(o, n, y0 + r, x, p.S, p.img0, p.img1, p.base, p.o[0], p.o[1], p.o[2], p.o[3], p.o[4], p.o[5], p.o[6], p.o[7]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// PERSISTENT, software-pipelined version (the default).  The kernel above runs one tile per CTA and its phases -- statistics
// fold, halo TMA, in-place normalisation, MMAs, gather / blend / store drain -- are a serial chain, co-resident CTAs all start
// together, so nothing overlaps.  Here ONE CTA per SM walks a contiguous range of tiles with the phases on different warps
// and different tiles:
//   warps 0-3   MMA warpgroup: per tile row 9 x C/16 x 2 wgmma (register accumulator, 16 columns), then the 16 head outputs
//               of every pixel go to one of TWO accumulator slots in shared memory
//   warp 4      TMA producer: halo boxes into an NS-deep ring (the head weights once)
//   warps 5..   workers (4 * TR warps), two stages on the same warps, two tiles apart, the drain split around the transform:
//               drain A(i):       the pixel's grid_change outputs from the slot -> gs_locate -> the four corner pixels requested;
//               transform(i + 2): normalise + activate the landed halo in place (the per-channel affine is rebuilt once per
//                                 SAMPLE, not per tile), every worker thread;
//               drain B(i):       the slot again -> tail_epilogue with the corners that arrived meanwhile (thread = pixel).
// mbarriers: h_full (TMA -> transform), h_xf (transform -> MMA, one arrival per worker thread), h_empty (MMA -> TMA, one
// arrival per MMA thread once its wgmma have completed), acc_full (MMA -> drain, one arrival per MMA thread after its slot
// stores), acc_empty (drain -> MMA, one arrival per drain thread once it has read the slot).
template <int C, int TR> struct TailPCfg {
    static constexpr int ROWB = 2 * C;
    static constexpr int HROWS = (TR + 2) * TT_HW;
    static constexpr int A_BYTES = ((HROWS * ROWB + 1023) / 1024) * 1024;
    static constexpr int NS = C == 32 ? 3 : 2;                              // halo ring depth (32 channels: the transform runs two tiles
                                                                            // ahead of the drain; three 66 KB slots of 64 channels do not fit)
    static constexpr int B_BYTES = 9 * TT_N * ROWB;
    static constexpr int SLOT_FLOATS = TR * TT_W * TT_N;                    // one accumulator slot: [TR rows][128 pixels][16 outputs]
    static constexpr int DRAIN_WARPS = 4 * TR;                              // one thread per output pixel of a tile
    static constexpr int WORKER_WARPS = DRAIN_WARPS;                        // every worker warp transforms AND drains
    static constexpr int THREADS = (5 + WORKER_WARPS) * 32;
    static constexpr int NBARS = 3 * NS + 5;
    static constexpr int MAX_S = 512;                                       // base-grid copy in shared memory
    static constexpr size_t SMEM = 1024 + (size_t)NS * A_BYTES + B_BYTES + 2 * (size_t)SLOT_FLOATS * sizeof(float) + 2 * C * sizeof(double) +
                                   2 * C * sizeof(float) + 16 * sizeof(float) + MAX_S * sizeof(float) + NBARS * sizeof(uint64_t) + 16;
    static_assert(SMEM <= 227 * 1024, "tail_tc: shared memory budget");
};

// position of head output `col` of pixel `px` in a slot row: 16-byte chunks XOR-swizzled so that eight consecutive pixels
// reading the same chunk (LDS.128) hit eight different bank groups
__device__ __forceinline__ int tp_slot_off(int px, int col) { return px * TT_N + (((col >> 2) ^ ((px >> 1) & 3)) << 2) + (col & 3); }

template <int KIND, int C, int TR>
__global__ void __launch_bounds__(TailPCfg<C, TR>::THREADS, 1) tail_tc_persist_kernel(const __grid_constant__ CUtensorMap tmF, const __grid_constant__ CUtensorMap tmW,
                                                                                      const TailTcParams p) {
    using Cfg = TailPCfg<C, TR>;
    constexpr int ROWB = Cfg::ROWB, NCH = ROWB / 16, NS = Cfg::NS;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* smA = smem;
    uint8_t* smB = smem + NS * Cfg::A_BYTES;
    float* slots = reinterpret_cast<float*>(smB + Cfg::B_BYTES);          // [2][SLOT_FLOATS] accumulator slots
    double* chs = reinterpret_cast<double*>(slots + 2 * Cfg::SLOT_FLOATS); // [C][2] folded statistics
    float* cA = reinterpret_cast<float*>(chs + 2 * C);                   // [C] affine
    float* cB = cA + C;
    float* sbias = cB + C;                                               // [16]
    float* sbase = sbias + 16;                                           // [S] affine_grid coordinates (one dependent global round trip less per pixel)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sbase + Cfg::MAX_S);
    uint64_t* h_full = bars, *h_xf = bars + NS, *h_empty = bars + 2 * NS;
    uint64_t* acc_full = bars + 3 * NS, *acc_empty = acc_full + 2, *w_full = acc_empty + 2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tiles_x = (p.S + TT_W - 1) / TT_W, tiles_y = p.S / TR, per_n = tiles_x * tiles_y;
    const int total = per_n * p.N;
    const int t_begin = (int)((long)blockIdx.x * total / gridDim.x);
    const int nt = (int)((long)(blockIdx.x + 1) * total / gridDim.x) - t_begin;       // contiguous tiles of this CTA (>= 1: grid <= total)

    if (tid == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(smem_u32(h_full + s), 1); mbar_init(smem_u32(h_xf + s), Cfg::WORKER_WARPS * 32); mbar_init(smem_u32(h_empty + s), 128); }
        for (int a = 0; a < 2; ++a) { mbar_init(smem_u32(acc_full + a), 128); mbar_init(smem_u32(acc_empty + a), Cfg::DRAIN_WARPS * 32); }
        mbar_init(smem_u32(w_full), 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmF) : "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmW) : "memory");
    }
    if (tid >= 64 && tid < 80) sbias[tid - 64] = (tid - 64) < TAIL_CO_PAD ? __ldg(p.bias + (tid - 64)) : 0.0f;     // weights: independent of the previous kernel
    for (int i = tid; i < p.S; i += Cfg::THREADS) sbase[i] = __ldg(p.base + i);                                     // constant table
    __syncthreads();
    pdl_trigger();
    if (tid == 128) {      // the head weights do not depend on the previous kernel: fetch them ahead of the dependency wait
        mbar_expect_tx(smem_u32(w_full), Cfg::B_BYTES);
        tma_load_3d(smem_u32(smB), &tmW, 0, 0, 0, smem_u32(w_full));
    }
    pdl_wait();

    if (warp == 4) {
        if (lane == 0) {   // ===== TMA producer =====
            for (int i = 0; i < nt; ++i) {
                const int s = i % NS;
                int t = t_begin + i;
                const int n = t / per_n; t -= n * per_n;
                const int ty = t / tiles_x, tx = t - ty * tiles_x;
                mbar_wait(smem_u32(h_empty + s), ((i / NS) & 1) ^ 1);
                mbar_expect_tx(smem_u32(h_full + s), Cfg::HROWS * ROWB);
                tma_load_4d(smem_u32(smA + s * Cfg::A_BYTES), &tmF, 0, tx * TT_W - 1, ty * TR - 1, n, smem_u32(h_full + s));
            }
        }
    } else if (warp < 4) {
        // ===== MMA warpgroup: TR tile rows x 9 taps = row-shifted views of the halo; accumulator -> slot =====
        mbar_wait(smem_u32(w_full), 0);
        for (int i = 0; i < nt; ++i) {
            const int s = i % NS, a = i & 1;
            mbar_wait(smem_u32(acc_empty + a), ((i >> 1) & 1) ^ 1);
            mbar_wait(smem_u32(h_xf + s), (i / NS) & 1);
            const uint8_t* hA = smA + s * Cfg::A_BYTES;
            float* slot = slots + a * Cfg::SLOT_FLOATS;
#pragma unroll 1
            for (int r = 0; r < TR; ++r) {
                float acc[2][8];
                wg_fence();
#pragma unroll
                for (int tap = 0; tap < 9; ++tap) {
                    const int dy = tap / 3, dx = tap - 3 * dy;
                    const uint32_t ap = smem_u32(hA + ((r + dy) * TT_HW + dx) * ROWB), bp = smem_u32(smB + tap * TT_N * ROWB);
#pragma unroll
                    for (int k = 0; k < C / 16; ++k) {
                        const uint64_t bd = make_smem_desc_sw<ROWB>(bp + 32 * k);
                        Wgmma<TT_N>::f16(acc[0], make_smem_desc_sw<ROWB>(ap + 32 * k), bd, (tap > 0 || k > 0) ? 1u : 0u);
                        Wgmma<TT_N>::f16(acc[1], make_smem_desc_sw<ROWB>(ap + 64 * ROWB + 32 * k), bd, (tap > 0 || k > 0) ? 1u : 0u);
                    }
                }
                wg_commit();
                wg_wait<0>();
                wg_fence_acc(acc[0]); wg_fence_acc(acc[1]);
                float* srow = slot + r * (TT_W * TT_N);
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < 2; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int px = h * 64 + warp * 16 + (lane >> 2) + 8 * e, col = 8 * j + 2 * (lane & 3);
                            *reinterpret_cast<float2*>(srow + tp_slot_off(px, col)) = make_float2(acc[h][4 * j + 2 * e], acc[h][4 * j + 2 * e + 1]);
                        }
            }
            mbar_arrive(smem_u32(h_empty + s));          // this thread's wgmma have read the halo slot
            mbar_arrive(smem_u32(acc_full + a));         // and its part of the accumulator slot is written
        }
    } else {
        // ===== worker warps (5 ..): BOTH remaining stages, on every warp =====
        //   transform(i + 1): normalise + activate the landed halo of the NEXT tile in place, all WORKERS threads;
        //   drain(i):         one thread per output pixel of the current tile.
        // A thread owns ONE 16-byte chunk column (8 channels) of the halo rows wt / NCH + k * (WORKERS / NCH): its 16
        // coefficients live in registers, XU rows are in flight at once.
        constexpr int WORKERS = Cfg::WORKER_WARPS * 32;
        constexpr int RSTEP = WORKERS / NCH;
        constexpr int ITEMS = (Cfg::HROWS + RSTEP - 1) / RSTEP, ITERS = (ITEMS + 5) / 6, XU = (ITEMS + ITERS - 1) / ITERS;
        const int wt = tid - 160, wid = warp - 5;
        const int jc = wt % NCH, r_first = wt / NCH;
        const int cpg = p.groups == 0 ? 1 : C / p.groups;
        const bool silu = p.act == ACT_SILU || p.act == ACT_SILU_FAST;
        const bool relu = p.act == ACT_RELU;
        const int q = wid & 3;                                                   // drain: 32-pixel group of the tile row
        const int dr = wid >> 2;                                                 // drain: tile row
        float av[8], bv[8];
        int cur_n = -1;

        auto transform = [&](int i) {
            const int s = i % NS;
            int t = t_begin + i;
            const int n = t / per_n; t -= n * per_n;
            const int ty = t / tiles_x, tx = t - ty * tiles_x;
            const int x0 = tx * TT_W, y0 = ty * TR;
            if (n != cur_n) {            // per-SAMPLE affine of the pending normalisation, from the producer's statistics
                cur_n = n;
                float g1 = 0.0f, b1 = 0.0f;
                if (wt < C) { g1 = __ldg(p.gamma + wt); b1 = __ldg(p.beta + wt); }     // requested ahead of the statistics
                asm volatile("bar.sync 1, %0;\n" :: "n"(WORKERS) : "memory");           // everyone is done with the previous table
                if (wt < C) {
                    const double2 v = fold_stat_replicas16(p.stats + ((long)n * p.stats_ld + wt) * 2, p.stats_rep_stride, p.stats_rep);
                    chs[2 * wt] = v.x; chs[2 * wt + 1] = v.y;
                }
                asm volatile("bar.sync 1, %0;\n" :: "n"(WORKERS) : "memory");
                if (wt < C) {
                    const int g0 = (wt / cpg) * cpg;
                    double su = 0.0, sq = 0.0;
                    for (int j = 0; j < cpg; ++j) { su += chs[2 * (g0 + j)]; sq += chs[2 * (g0 + j) + 1]; }
                    const double inv_cnt = 1.0 / ((double)p.S * p.S * cpg);          // fp64 for the sums and the cancelling subtraction only
                    const double mean = su * inv_cnt;
                    const float var = fmaxf((float)fma(sq, inv_cnt, -mean * mean), 0.0f);
                    float A = rsqrtf(var + 1e-5f) * g1;
                    float B = b1 - (float)mean * A;
                    if (silu) { A *= 0.5f; B *= 0.5f; }                            // silu(v) = h + h * tanh(h), h = v / 2
                    cA[wt] = A; cB[wt] = B;
                }
                asm volatile("bar.sync 1, %0;\n" :: "n"(WORKERS) : "memory");
#pragma unroll
                for (int e = 0; e < 8; ++e) { av[e] = cA[8 * jc + e]; bv[e] = cB[8 * jc + e]; }
            }
            mbar_wait(smem_u32(h_full + s), (i / NS) & 1);
            uint8_t* hbase = smA + s * Cfg::A_BYTES;
#pragma unroll 1
            for (int row0 = r_first; row0 < Cfg::HROWS; row0 += XU * RSTEP) {
                uint4 d[XU];
                uint4* dp[XU];
                bool ok[XU];
#pragma unroll
                for (int u = 0; u < XU; ++u) {
                    const int row = row0 + u * RSTEP;
                    const int hy = row / TT_HW, hx = row - hy * TT_HW;
                    const int gy = y0 - 1 + hy, gx = x0 - 1 + hx;
                    ok[u] = row < Cfg::HROWS && gy >= 0 && gy < p.S && gx >= 0 && gx < p.S;       // zero padding stays zero
                    const int swz = ROWB == 128 ? (row & 7) : ((row >> 1) & 3);
                    dp[u] = reinterpret_cast<uint4*>(hbase + row * ROWB + ((jc ^ swz) << 4));
                    if (ok[u]) d[u] = *dp[u];
                }
#pragma unroll
                for (int u = 0; u < XU; ++u) {
                    if (!ok[u]) continue;
                    __half2* hp = reinterpret_cast<__half2*>(&d[u]);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float2 v = __half22float2(hp[e]);
                        v.x = fmaf(v.x, av[2 * e], bv[2 * e]); v.y = fmaf(v.y, av[2 * e + 1], bv[2 * e + 1]);
                        if (silu) {
                            float tx2, ty2;
                            asm("tanh.approx.f32 %0, %1;\n" : "=f"(tx2) : "f"(v.x));
                            asm("tanh.approx.f32 %0, %1;\n" : "=f"(ty2) : "f"(v.y));
                            v.x = fmaf(v.x, tx2, v.x); v.y = fmaf(v.y, ty2, v.y);
                        } else if (relu) {
                            v.x = fmaxf(v.x, 0.0f); v.y = fmaxf(v.y, 0.0f);
                        }
                        hp[e] = __floats2half2_rn(v.x, v.y);
                    }
                }
#pragma unroll
                for (int u = 0; u < XU; ++u)
                    if (ok[u]) *dp[u] = d[u];
            }
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic-proxy writes -> the tensor core's async-proxy reads
            mbar_arrive(smem_u32(h_xf + s));
        };

        // The drain of a tile is split around the transform of the next one: phase A reads the two grid_change outputs of the
        // pixel and REQUESTS the four corner pixels of its sampling tap; the transform runs while they travel; phase B reads
        // the accumulator again (cheap: shared memory) and finishes.  Unsplit, every tile paid one exposed global round trip with all
        // sixteen drain warps waiting on it together.
        // Every drain warp polls acc_full itself: a common named barrier made fifteen warps wait for the slowest (23 % of all
        // samples); with the drain behind the transform the accumulator has usually been complete for a while.
        float4 pre[4];
        bool have_pre = false;
        auto tile_xy = [&](int i, int& n, int& x, int& y) {
            int t = t_begin + i;
            n = t / per_n; t -= n * per_n;
            const int ty = t / tiles_x, tx = t - ty * tiles_x;
            x = tx * TT_W + q * 32 + lane; y = ty * TR + dr;
        };
        auto load_acc = [&](int a, float (&o)[TAIL_CO_PAD]) {
            const float* srow = slots + a * Cfg::SLOT_FLOATS + dr * (TT_W * TT_N);
            const int px = q * 32 + lane;
            float acc[16];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 v = *reinterpret_cast<const float4*>(srow + tp_slot_off(px, 4 * j));
                acc[4 * j] = v.x; acc[4 * j + 1] = v.y; acc[4 * j + 2] = v.z; acc[4 * j + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < TAIL_CO_PAD; ++j) o[j] = fmaf(acc[j], p.acc_scale, sbias[j]);
        };
        auto drain_issue = [&](int i) {
            const int a = i & 1;
            int n, x, y;
            tile_xy(i, n, x, y);
            mbar_wait(smem_u32(acc_full + a), (i >> 1) & 1);
            have_pre = false;
            if (KIND != TAIL_DECOMPOSER && p.g0 != nullptr) {           // warp-uniform
                float o[TAIL_CO_PAD];
                load_acc(a, o);
                if (x < p.S) have_pre = tail_gather_issue<KIND>(o, n, y, x, p.S, sbase, p.g0, p.g0_ld, pre);
            }
        };
        auto drain_finish = [&](int i) {
            const int a = i & 1;
            int n, x, y;
            tile_xy(i, n, x, y);
            float o[TAIL_CO_PAD];
            load_acc(a, o);
            mbar_arrive(smem_u32(acc_empty + a));                                // this thread is done with the accumulator slot
            if (x < p.S)
                tail_epilogue<KIND>(o, n, y, x, p.S, p.img0, p.img1, sbase, p.o[0], p.o[1], p.o[2], p.o[3], p.o[4], p.o[5], p.o[6], p.o[7],
                                    p.g0, p.g0_ld, p.g1, p.g1_ld, have_pre ? &pre : nullptr);
        };

        // The transform runs TWO tiles ahead of the drain (the halo ring is three deep): the MMAs of tile i + 1 then have the
        // whole of drain(i) and transform(i + 2) to complete in.  One tile ahead, with the drain split around the transform,
        // they had only the second half of drain(i): 31 % of all samples were drain warps polling acc_full.
        transform(0);
        if (nt > 1) transform(1);
        for (int i = 0; i < nt; ++i) {
            drain_issue(i);
            if (i + 2 < nt) transform(i + 2);
            drain_finish(i);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tail_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        THA4_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q));
        THA4_REQUIRE(ptr != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled unavailable");
        fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

using TKey = std::tuple<int, const void*, long, long, long, long, int>;
std::map<TKey, CUtensorMap> g_tail_maps;
std::mutex g_tail_maps_mu;

const CUtensorMap& feature_map(const View& f, int TR) {
    TKey key{current_device(), f.p, f.N, f.H, f.C, f.ld, TR};
    std::lock_guard<std::mutex> lock(g_tail_maps_mu);
    auto it = g_tail_maps.find(key);
    if (it != g_tail_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[4] = {(cuuint64_t)f.C, (cuuint64_t)f.W, (cuuint64_t)f.H, (cuuint64_t)f.N};
    cuuint64_t strides[3] = {(cuuint64_t)f.ld * 2, (cuuint64_t)f.W * f.ld * 2, (cuuint64_t)f.H * f.W * f.ld * 2};
    cuuint32_t box[4] = {(cuuint32_t)f.C, (cuuint32_t)TT_HW, (cuuint32_t)(TR + 2), 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = tail_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, f.p, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               f.C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tail feature map) failed: " + std::to_string((int)r));
    return g_tail_maps.emplace(key, m).first->second;
}

const CUtensorMap& head_weight_map(const TailWeights& tw) {
    TKey key{current_device(), tw.w16, tw.C, 0, 0, 0, -1};
    std::lock_guard<std::mutex> lock(g_tail_maps_mu);
    auto it = g_tail_maps.find(key);
    if (it != g_tail_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)tw.C, (cuuint64_t)TT_N, 9};
    cuuint64_t strides[2] = {(cuuint64_t)tw.C * 2, (cuuint64_t)TT_N * tw.C * 2};
    cuuint32_t box[3] = {(cuuint32_t)tw.C, (cuuint32_t)TT_N, 9};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = tail_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, tw.w16, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               tw.C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(tail head weights) failed: " + std::to_string((int)r));
    return g_tail_maps.emplace(key, m).first->second;
}

// [9][C][TAIL_CO_PAD] fp32 -> [9][16][C] f16 (K-major B operand: one row per head channel), scaled by a power of two
__global__ void tail_pack_half_kernel(const float* __restrict__ w, __half* __restrict__ h, int C, float scale) {
    const int total = 9 * TT_N * C;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int c = i % C, nn = (i / C) % TT_N, tap = i / (C * TT_N);
        h[i] = __float2half_rn(nn < TAIL_CO_PAD ? w[(tap * C + c) * TAIL_CO_PAD + nn] * scale : 0.0f);
    }
}
__global__ void tail_absmax_kernel(const float* __restrict__ w, int n, unsigned* __restrict__ out) {
    float m = 0.0f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

template <int KIND, int C>
void launch_tail_tc(const TailWeights& tw, const View& f, const NormSpecTail& ns, const ImgView& i0, const ImgView& i1, float* const* o,
                    cudaStream_t s) {
    using Cfg = TailCfg<C>;
    TailTcParams p{};
    p.S = f.H; p.N = f.N;
    p.stats = f.stats; p.stats_ld = f.stats_ld; p.stats_rep = std::max(1, f.stats_rep); p.stats_rep_stride = f.stats_rep_stride;
    p.groups = ns.groups; p.act = ns.act; p.gamma = ns.gamma; p.beta = ns.beta;
    p.bias = tw.bias; p.acc_scale = 1.0f / tw.w16_scale;
    p.img0 = i0; p.img1 = i1; p.base = base_grid_table(f.H);
    for (int i = 0; i < 8; ++i) p.o[i] = i < TAIL_OUTPUTS[KIND].count ? o[i] : nullptr;
    THA4_ENSURE_SMEM((tail_tc_kernel<KIND, C>), Cfg::SMEM);
    dim3 grid(ceil_div(f.W, TT_W), f.H / Cfg::TR, f.N);
    ProfScope prof(PROF_TAIL, s);
    {   // compulsory traffic as SURVEY 8d defines it (fp32 element size): feature map + image(s) read once, every returned tensor written once
        const int img_ch = (KIND == TAIL_COMBINER) ? 8 : 4;
        prof_add_work(PROF_TAIL, 2.0 * f.pixels() * 9 * tw.C * tw.CO, (double)f.pixels() * (f.C + img_ch + TAIL_OUTPUTS[KIND].channels()) * 4);
    }
    launch_pdl(tail_tc_kernel<KIND, C>, grid, dim3(TT_THREADS), Cfg::SMEM, s, 1, feature_map(f, Cfg::TR), head_weight_map(tw), p);
    THA4_LAUNCH_CHECK();
}

template <int KIND, int C, int TR>
void launch_tail_persist(const TailWeights& tw, const View& f, const NormSpecTail& ns, const ImgView& i0, const ImgView& i1, float* const* o,
                         cudaStream_t s, const View* g0, const View* g1) {
    using Cfg = TailPCfg<C, TR>;
    TailTcParams p{};
    p.S = f.H; p.N = f.N;
    p.stats = f.stats; p.stats_ld = f.stats_ld; p.stats_rep = std::max(1, f.stats_rep); p.stats_rep_stride = f.stats_rep_stride;
    p.groups = ns.groups; p.act = ns.act; p.gamma = ns.gamma; p.beta = ns.beta;
    p.bias = tw.bias; p.acc_scale = 1.0f / tw.w16_scale;
    p.img0 = i0; p.img1 = i1; p.base = base_grid_table(f.H);
    auto gather_ok = [&](const View* g) {      // fp32 NHWC view of the same geometry, four channels 16-byte aligned, offsets within 32 bits
        return g && g->p && !g->f16 && g->N == f.N && g->H == f.H && g->W == f.W && g->ld % 4 == 0 && (reinterpret_cast<uintptr_t>(g->p) & 15) == 0 &&
               (size_t)f.H * f.W * g->ld < (size_t)1 << 30;
    };
    if (gather_ok(g0)) { p.g0 = g0->p; p.g0_ld = g0->ld; }
    if (gather_ok(g1)) { p.g1 = g1->p; p.g1_ld = g1->ld; }
    for (int i = 0; i < 8; ++i) p.o[i] = i < TAIL_OUTPUTS[KIND].count ? o[i] : nullptr;
    THA4_REQUIRE(f.H <= Cfg::MAX_S, "tail_tc: image size");
    THA4_ENSURE_SMEM((tail_tc_persist_kernel<KIND, C, TR>), Cfg::SMEM);
    const long total = (long)ceil_div(f.W, TT_W) * (f.H / TR) * f.N;
    dim3 grid((unsigned)std::min<long>(total, num_sms()));
    ProfScope prof(PROF_TAIL, s);
    {   // compulsory traffic as SURVEY 8d defines it (fp32 element size): feature map + image(s) read once, every returned tensor written once
        const int img_ch = (KIND == TAIL_COMBINER) ? 8 : 4;
        prof_add_work(PROF_TAIL, 2.0 * f.pixels() * 9 * tw.C * tw.CO, (double)f.pixels() * (f.C + img_ch + TAIL_OUTPUTS[KIND].channels()) * 4);
    }
    launch_pdl(tail_tc_persist_kernel<KIND, C, TR>, grid, dim3(Cfg::THREADS), Cfg::SMEM, s, 1, feature_map(f, TR), head_weight_map(tw), p);
    THA4_LAUNCH_CHECK();
}

template <int KIND>
void launch_tail_tc_c(const TailWeights& tw, const View& f, const NormSpecTail& ns, const ImgView& i0, const ImgView& i1, float* const* o,
                      cudaStream_t s, const View* g0, const View* g1) {
    if (opts().tail_persist) {
        // tile rows per step (32-channel sites): 4 when that still gives every SM two tiles or more, else 2 (more, smaller tiles:
        // the small sites at B = 1 are one latency chain per CTA)
        const long tiles4 = (long)ceil_div(f.W, TT_W) * (f.H / 4) * f.N;
        const bool tr4 = tiles4 >= 2L * num_sms();
        if (tw.C == 32) { if (tr4) launch_tail_persist<KIND, 32, 4>(tw, f, ns, i0, i1, o, s, g0, g1); else launch_tail_persist<KIND, 32, 2>(tw, f, ns, i0, i1, o, s, g0, g1); }
        else            launch_tail_persist<KIND, 64, 2>(tw, f, ns, i0, i1, o, s, g0, g1);        // two halo slots of 66 KB
        return;
    }
    if (tw.C == 32) launch_tail_tc<KIND, 32>(tw, f, ns, i0, i1, o, s);
    else launch_tail_tc<KIND, 64>(tw, f, ns, i0, i1, o, s);
}

}  // namespace

void tail_make_half(TailWeights& tw, cudaStream_t s) {
    if (tw.w16 || !tw.w) return;
    const int nw = 9 * tw.C * TAIL_CO_PAD;
    __half* h = reinterpret_cast<__half*>(tracked_malloc((size_t)9 * TT_N * tw.C * sizeof(__half)));
    unsigned* dmax = reinterpret_cast<unsigned*>(h);
    THA4_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned), s));
    tail_absmax_kernel<<<8, 256, 0, s>>>(tw.w, nw, dmax);
    THA4_LAUNCH_CHECK();
    unsigned hmax = 0;
    THA4_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    float mx; memcpy(&mx, &hmax, sizeof(float));
    float scale = 1.0f;
    if (mx > 0.0f && std::isfinite(mx)) {
        int e = 0; frexpf(mx, &e);
        e = std::max(-24, std::min(8, e));
        scale = ldexpf(1.0f, -e);
    }
    tail_pack_half_kernel<<<16, 256, 0, s>>>(tw.w, h, tw.C, scale);
    THA4_LAUNCH_CHECK();
    tw.w16 = h; tw.w16_scale = scale;
}

bool tail_tc_supported(const TailWeights& tw, const View& feature) {
    return feature.f16 && feature.stats != nullptr && (tw.C == 32 || tw.C == 64) && feature.C == tw.C && feature.ld == tw.C &&
           feature.H == feature.W && feature.H % 4 == 0 && tw.w16 != nullptr && (((uintptr_t)feature.p) & 15) == 0;
}

void tail_tc_forward(TailKind kind, const TailWeights& tw, const View& feature, const NormSpecTail& ns, const ImgView& image0,
                     const ImgView& image1, float* const* outputs, cudaStream_t s, const View* g0, const View* g1) {
    THA4_REQUIRE(tail_tc_supported(tw, feature), "tail_tc: unsupported configuration");
    THA4_REQUIRE(image0.H == feature.H && image0.W == feature.W && image0.C == 4, "tail_tc: image dims");
    THA4_REQUIRE(ns.groups == 0 || tw.C % ns.groups == 0, "tail_tc: groups");
    switch (kind) {
        case TAIL_UNET: launch_tail_tc_c<TAIL_UNET>(tw, feature, ns, image0, image1, outputs, s, g0, g1); break;
        case TAIL_DECOMPOSER: launch_tail_tc_c<TAIL_DECOMPOSER>(tw, feature, ns, image0, image1, outputs, s, g0, g1); break;
        case TAIL_COMBINER: launch_tail_tc_c<TAIL_COMBINER>(tw, feature, ns, image0, image1, outputs, s, g0, g1); break;
        case TAIL_FACE: launch_tail_tc_c<TAIL_FACE>(tw, feature, ns, image0, image1, outputs, s, g0, g1); break;
    }
}

}  // namespace tha4
