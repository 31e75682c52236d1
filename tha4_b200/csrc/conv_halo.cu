// 3x3 (stride 1, pad 1) convolution on wgmma with HALO REUSE -- the kernel behind most of the teacher's FLOPs in the
// default mode (both 3x3 convs of every U-Net ResBlock, the eleven 512 -> 512 bottleneck convs of the encoder-decoder nets).
//
// conv_tc.cu fetches one 128-pixel x 64-channel activation box PER TAP (9 boxes per channel chunk) and, with the fused
// input normalisation, transforms each of them.  Here the CTA tile is 8 x 16 pixels and one TMA box {64 ch, 10 w, 18 h}
// brings in the tile's 10 x 18 HALO once per channel chunk; the nine taps are nine VIEWS of that shared-memory image:
// the wgmma A-descriptor start address is shifted by ((dy + 1) * 10 + (dx + 1)) pixel rows and the stride between 8-row
// groups (SBO) is the halo pitch (10 rows) -- the tensor core applies the 128-/64-byte swizzle on absolute shared-memory
// addresses, so row-shifted views of a TMA-written image are legal.
//   * activation traffic L2 -> shared memory per channel chunk: 180 rows instead of 9 x 128 (6.4x less);
//   * the pending normalisation (XF: GroupNorm / InstanceNorm affine + FiLM + SiLU / ReLU of the RAW f16 input) is
//     applied to 180 rows once instead of 1152 rows, by the consumer warpgroup that issues the MMAs;
//   * weights stream per (chunk, tap) through their own TMA ring, pre-issued ahead of the programmatic-dependency wait;
//   * K (channel chunks) can be split over a thread-block cluster, partials meeting in distributed shared memory
//     (same epilogues as conv_tc.cu: conv_tc_device.cuh).
// The four-phase layers (CONV_UP2_3x3, CONVT_4x4_S2: 4 output phases x 2x2 taps, tap offsets in {-1, 0, 1} on the
// low-resolution input) run on the same halo: one 8 x 16 low-resolution tile per CTA, its 10 x 18 halo loaded and
// normalised once per chunk instead of once per (phase, tap) -- 180 rows instead of 16 x 128.  Consumer warpgroup py holds
// the accumulators of phases (py, 0) and (py, 1); the 16 weight tiles of a chunk alternate between the two warpgroups.
// Folded 1x1 skip (SK, the second conv of a U-Net ResBlock whose input and output widths differ): conv1(n1(h0)) + skip(x)
// is one GEMM over a longer K.  The chunk list is the cpt chunks of h0 (halo through tmA, XF transform, nine weight tiles
// from tmB) followed by the cpt2 chunks of x (halo through tmA2, no transform, the centre-tap view and one weight tile from
// tmB2).  Each weight segment keeps the power-of-two scale of its f16 copy: after its last 3x3 chunk a CTA multiplies the
// accumulator by acc_rescale (exact), so the products and their sums are those of the separate convs, in the skip weights'
// units.  Summation order: within a CTA, chunk by chunk in list order (tap by tap inside a 3x3 chunk); a cluster split
// gives rank r the contiguous chunks [halo_fold_c0(r), halo_fold_c0(r + 1)), balanced by weight tiles, and its partials
// meet in the reduction of the unsplit kernel (rank order, conv_tc_device.cuh).
#include "conv.cuh"
#include "profiler.cuh"
#include "conv_tc_device.cuh"
#include <cuda.h>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>

namespace tha4 {
static long long* g_dbg_buf = nullptr;   // THA4_HALO_DEBUG phase stamps

namespace {

using namespace tc;
using namespace tcdev;

// CTA tile: 8 x 16 = 128 output pixels per consumer warpgroup; WG = 2 consumer warpgroups stack two of them vertically
// (8 x 32 = 256 pixels) and share every weight tile: half the weight traffic L2 -> shared memory per FLOP, half the
// CTA start-up cost (barriers, PDL wait, statistic fold of the normalisation table) per pixel.
constexpr int HT_W = 8, HT_H = 16;
constexpr int HALO_W = HT_W + 2;
__host__ __device__ constexpr int halo_h(int wg) { return HT_H * wg + 2; }                  // 18 / 34
__host__ __device__ constexpr int halo_rows(int wg) { return HALO_W * halo_h(wg); }         // 180 / 340 pixel rows
__host__ __device__ constexpr int halo_a_bytes(int rowb, int wg) { return ((halo_rows(wg) * rowb + 1023) / 1024) * 1024; }
// + the TMA producer warp, except in the two-warpgroup CTAs built to run two per SM (ctas = 2, see conv_halo_kernel)
__host__ __device__ constexpr int halo_threads(int wg, int ctas = 1) { return 128 * wg + (ctas == 2 ? 0 : 32); }
// warpgroup 1 reads the halo 16 pixel rows (160 halo rows) further on: a multiple of 1024 bytes at both row widths, so
// its descriptors see the same swizzle phase as warpgroup 0's
static_assert((HT_H * HALO_W * 64) % 1024 == 0, "second warpgroup's halo offset keeps the swizzle phase");

// SA / SB: stages of the activation-halo ring / of the weight-tile ring.  OP: OP_F16 (64 channels per chunk, 128-byte rows)
// or OP_F16N (32 channels, 64-byte rows).  p.ksplit = cluster size CS (split over channel chunks), p.cpt = chunks.
// MINB: resident CTAs per SM the register allocation must allow (4 for the single-chunk unsplit variants, whose small
// rings fit four times: the layers at 256x256 / 512x512 are chains of dependent latencies, more CTAs = more overlap).
// Two-warpgroup CTAs (BN <= 64): two with BN = 32, as many consumer warps per SM as four one-warpgroup CTAs; one with
// BN = 64 (two would cap the 288 threads at 96 registers, which spills the 64-column accumulator's epilogue).  Four-phase
// CTAs (two 32-column accumulators per warpgroup) count as BN = 64.  ctas = 2: the 256-thread variant of those two, without
// the producer warp: 2 x 8 warps put 4 warps on each SM sub-partition, and each thread keeps 128 registers.
__host__ __device__ constexpr int halo_min_ctas(int bn, int sa, int cs, int op, int wg, int ph = 1, int ctas = 1) {
    return ctas == 2 ? 2 : wg > 1 ? (bn * (ph == 4 ? 2 : 1) <= 32 ? 2 : 1) : cs > 1 || bn >= 128 ? 1 : ((sa == (op == OP_F16N ? 2 : 1) && bn <= 32) ? 4 : 2);
}
// Weight tile j of a channel chunk, as the third coordinate of the [phase * tap][cout][cin] weight map.  3x3: tap j.
// Four phases: j = 2 (2 tap + px) + py, so the tiles of the two warpgroups (py) alternate in the ring.
template <int PH>
__host__ __device__ constexpr int halo_wtile(int j) { return PH == 1 ? j : ((j & 1) * 2 + ((j >> 1) & 1)) * 4 + (j >> 2); }
// First chunk of rank r of a cluster split of a folded-skip chunk list (cpt 3x3 chunks of nine weight tiles, then cpt2
// skip chunks of one): the chunk boundary nearest to r / cs of the weight tiles.  Rank cs ends the list.
__host__ __device__ constexpr int halo_fold_c0(int r, int cs, int cpt, int cpt2) {
    const int target = (r * (9 * cpt + cpt2) + cs / 2) / cs;
    return target <= 9 * cpt ? (target + 4) / 9 : cpt + target - 9 * cpt;
}

// every thread of every CTA of the cluster arrives; release / acquire order the shared-memory writes around it
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// Row-owning cluster pair (WG = 2, CS = 2): the accumulators of one warpgroup as 16-byte chunks [k][128 threads], chunk k of
// thread t at (k * 128 + t) * 16 bytes.  Sender and receiver thread t hold the same fragment, so the receiver adds chunk k
// to registers without a transpose, and a warp's 32 chunks fill 512 consecutive bytes (no bank conflicts either side).
template <int BN, int NACC>
__device__ __forceinline__ void halo_push_rows(const Acc<BN> (&acc)[NACC], uint32_t remote, int t) {
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; j += 4) {
                const uint32_t addr = remote + (uint32_t)((((a * 2 + h) * (BN / 8) + j / 4) * 128 + t) * 16);
                asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};\n" :: "r"(addr), "f"(acc[a].d[h][j]),
                             "f"(acc[a].d[h][j + 1]), "f"(acc[a].d[h][j + 2]), "f"(acc[a].d[h][j + 3]) : "memory");
            }
}
template <int BN, int NACC>
__device__ __forceinline__ void halo_add_rows(Acc<BN> (&acc)[NACC], const uint8_t* recv, int t) {
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; j += 4) {
                const float4 v = *reinterpret_cast<const float4*>(recv + (((a * 2 + h) * (BN / 8) + j / 4) * 128 + t) * 16);
                acc[a].d[h][j] += v.x; acc[a].d[h][j + 1] += v.y; acc[a].d[h][j + 2] += v.z; acc[a].d[h][j + 3] += v.w;
            }
}

// WG: consumer warpgroups (1: 128-pixel tiles, 160 threads; 2: 256-pixel tiles, 288 threads)
// PH: output phases (1: 3x3; 4: four-phase layers, two warpgroups on one 8 x 16 low-resolution tile)
// WG = 2 with CS = 2 (one CTA per SM only): a cluster pair splits the channel chunks, and rank r finishes the rows of
// warpgroup r (3x3: tile rows 16 r .. 16 r + 15; four phases: phases (r, 0) and (r, 1)).  After the MMAs warpgroup 1 - r
// pushes its accumulators into the peer's idle half of the ring; warpgroup r adds them and runs the unsplit epilogue.
// CTAS: resident CTAs per SM a two-warpgroup CTA is built for.  1: a TMA producer warp (288 threads, one CTA per SM for
// 256 x 64 and four-phase tiles).  2: no producer warp (256 threads, two CTAs per SM with rings of at most ~113 KB): thread
// 0 of the consumers issues the loads from inside the MMA loop, and while one CTA transforms a chunk, starts up or drains
// its accumulator, the other one's MMAs keep the tensor pipe busy.
// SK: a folded 1x1 skip (see the header): tmA2 / tmB2 are the skip input's halo map and the skip weights (else unused)
template <int BN, int SA, int SB, int CS, int OP, int XF, int WG, int PH = 1, int CTAS = 1, int SK = 0>
__global__ void __launch_bounds__(halo_threads(WG, CTAS), halo_min_ctas(BN, SA, CS, OP, WG, PH, CTAS)) conv_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                const __grid_constant__ CUtensorMap tmO32, const __grid_constant__ CUtensorMap tmO16,
                                                                const __grid_constant__ CUtensorMap tmR, const TcParams p,
                                                                const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2) {
    static_assert(OP != OP_TF32, "halo kernel: f16 operands");
    static_assert(BN <= 128, "the accumulator of one warpgroup: BN registers per thread");
    static_assert(WG == 1 || (WG == 2 && (CS == 1 || (CS == 2 && CTAS == 1)) && BN <= 64),
                  "two consumer warpgroups: unsplit launches or a row-owning pair, two accumulators of at most 64 columns");
    constexpr bool ROW_SPLIT = WG == 2 && CS == 2;
    // four phases: two 128-row accumulators per warpgroup, no more registers than one 128 x 64 accumulator
    static_assert(PH == 1 || (PH == 4 && WG == 2 && BN <= 32), "four-phase layers: two warpgroups, two 128 x 32 accumulators each");
    constexpr bool SELF_LOAD = CTAS == 2;                                // consumer thread 0 issues the TMA loads
    static_assert(CTAS == 1 || (CTAS == 2 && WG == 2), "two CTAs per SM: the two-warpgroup tiles");
    // in-loop loads (below): at step i thread 0 issues the weight tiles up to i + SB - 2 (four phases: 2 i + SB - 3), and the
    // tiles of step i + 1 must be out before thread 0 waits for them
    static_assert(!SELF_LOAD || SB >= (PH == 1 ? 3 : 6), "weight ring too shallow for loads issued by a consumer");
    static_assert(!SK || (PH == 1 && XF), "folded skip: the second conv of a ResBlock (3x3, normalised input)");
    constexpr int SLABS = PH == 1 ? WG : 1;                              // 16-row slabs of the tile (8 x 16 pixels each)
    constexpr int NACC = PH == 1 ? 1 : 2;                                // accumulators per warpgroup
    constexpr int TPC = PH == 1 ? 9 : 16;                                // weight tiles per channel chunk
    constexpr int ROWB = op_row_bytes(OP);
    constexpr int KCE = op_kch(OP);
    constexpr int HALO_ROWS = halo_rows(SLABS);
    constexpr int A_BYTES = halo_a_bytes(ROWB, SLABS);
    constexpr int B_BYTES = BN * ROWB;
    constexpr int PRODUCER_WARP = 4 * WG;
    constexpr int EPI_BYTES = (int)(((size_t)SA * A_BYTES + (size_t)SB * B_BYTES) / WG) & ~1023;      // idle ring per warpgroup in the epilogue
    // TMA-store staging slots of the unsplit epilogue (none for the phase-strided outputs of the four-phase layers)
    constexpr int NSLOT = (CS == 1 || ROW_SPLIT) && PH == 1 ? epi_nslot(BN, EPI_BYTES) : 0;
    // ROW_SPLIT: the peer's partial lands in the other warpgroup's half of the ring, the owner's staging slots lie in its own
    constexpr int RECV_BYTES = NACC * 128 * BN * 4;
    static_assert(!ROW_SPLIT || (RECV_BYTES <= EPI_BYTES && (PH == 4 || NSLOT > 0)), "row-owning pair: receive slot and staging slot in the idle ring");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);      // pointer arithmetic (not an integer round trip) keeps the shared address space: LDS / STS, not generic LD / ST
    uint8_t* smA = smem;
    uint8_t* smB = smem + SA * A_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smB + SB * B_BYTES);
    uint64_t* a_full = bars, *a_empty = bars + SA;
    uint64_t* b_full = bars + 2 * SA, *b_empty = b_full + SB;
    uint64_t* res_bars = b_empty + SB;                                   // [4 per warpgroup]: residual tiles of the unsplit epilogue (epi_direct)
    float* xf_A = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(res_bars + 4 * WG) + ((16u - (tc::smem_u32(res_bars + 4 * WG) & 15u)) & 15u));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // developer timing: CTA `slot` of every 97 records clock64 at its phase boundaries (8 stamps per role: dbg[slot][role][8])
    auto dbg_slot = [&]() -> long long* {
        const bool dbg_on = p.dbg != nullptr && (blockIdx.x % 97) == 0 && blockIdx.y == 0 && (blockIdx.x / 97) * CS + blockIdx.z < 32;
        return dbg_on ? p.dbg + ((blockIdx.x / 97) * CS + blockIdx.z) * 32 : nullptr;
    };
    // the two-CTA variant recomputes the slot at each stamp and has none from the MMA loop on: with 128 registers, a
    // pointer held through the loop and the epilogue costs it a spill
    long long* dbg = SELF_LOAD ? nullptr : dbg_slot();
#define HSTAMP(role, i) do { long long* d_ = SELF_LOAD ? dbg_slot() : dbg; if (d_) d_[(role) * 8 + (i)] = clock64(); } while (0)
#define HSTAMP_END(role, i) do { if (!SELF_LOAD) HSTAMP(role, i); } while (0)
    if (threadIdx.x == 0) HSTAMP(0, 0);
    int tile = blockIdx.x;
    const int tx = tile % p.tiles_x; tile /= p.tiles_x;
    const int ty = tile % p.tiles_y;
    const int n = tile / p.tiles_y;
    const int x0 = tx * HT_W, y0 = ty * (HT_H * SLABS);
    const int n0 = blockIdx.y * BN;
    const int split = blockIdx.z;                                        // rank in the cluster (CS == gridDim.z)
    const int c_per = (p.cpt + CS - 1) / CS;
    const int cb0 = SK ? halo_fold_c0(split, CS, p.cpt, p.cpt2) : split * c_per;
    const int nc = SK ? halo_fold_c0(split + 1, CS, p.cpt, p.cpt2) - cb0 : max(0, min(p.cpt, cb0 + c_per) - cb0);   // channel chunks of this CTA
    const int nconv = SK ? max(0, min(nc, p.cpt - cb0)) : nc;            // of them 3x3 chunks (the rest: skip chunks)
    const int nb = SK ? nconv * TPC + nc - nconv : nc * TPC;             // weight tiles of this CTA
    // weight tile j of this CTA: tap j % TPC of chunk j / TPC, then (SK) the one tile of each skip chunk
    auto load_wtile = [&](int j, uint32_t dst, uint32_t full) {
        if (SK && j >= nconv * TPC) tma_load_3d(dst, &tmB2, (cb0 + j - nconv * (TPC - 1) - p.cpt) * KCE, n0, 0, full);
        else tma_load_3d(dst, &tmB, (cb0 + j / TPC) * KCE, n0, halo_wtile<PH>(j % TPC), full);
    };
    // the halo of chunk ci of this CTA
    auto load_halo = [&](int ci, uint32_t dst, uint32_t full) {
        if (SK && cb0 + ci >= p.cpt) tma_load_4d(dst, &tmA2, (cb0 + ci - p.cpt) * KCE, x0 - 1, y0 - 1, n, full);
        else tma_load_4d(dst, &tmA, (cb0 + ci) * KCE, x0 - 1, y0 - 1, n, full);
    };

    if (threadIdx.x == 0) {
        // the empty barriers take one arrival per consumer thread: every thread arrives once its own wgmma wait has returned
        // (a four-phase weight tile is read by one warpgroup)
        for (int s = 0; s < SA; ++s) { mbar_init(smem_u32(a_full + s), 1); mbar_init(smem_u32(a_empty + s), 128 * WG); }
        for (int s = 0; s < SB; ++s) { mbar_init(smem_u32(b_full + s), 1); mbar_init(smem_u32(b_empty + s), PH == 1 ? 128 * WG : 128); }
        for (int s = 0; s < 4 * WG; ++s) mbar_init(smem_u32(res_bars + s), 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmB) : "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) HSTAMP(0, 1);
    pdl_trigger();
    // weight tiles of the first ring pass do not depend on the previous kernel: fetch them ahead of the dependency wait
    const int npre = p.pre_b ? min(nb, SB) : 0;
    if (SELF_LOAD ? threadIdx.x == 0 : (warp == PRODUCER_WARP && lane == 0)) {
        for (int i = 0; i < npre; ++i) {
            const uint32_t full = smem_u32(b_full + i);
            mbar_expect_tx(full, B_BYTES);
            if constexpr (SK) load_wtile(i, smem_u32(smB + i * B_BYTES), full);
            else tma_load_3d(smem_u32(smB + i * B_BYTES), &tmB, (cb0 + i / TPC) * KCE, n0, halo_wtile<PH>(i % TPC), full);
        }
    }
    pdl_wait();
    if (threadIdx.x == 0) HSTAMP(0, 2);

    Acc<BN> acc[NACC];
    if (nc > 0) {
        if (!SELF_LOAD && warp == PRODUCER_WARP) {
            if (lane == 0) {   // ===== TMA producer: one halo box per chunk, nine (four-phase: sixteen) weight tiles per chunk =====
                int bi = 0;
                for (int ci = 0; ci < nc; ++ci) {
                    const int sa = ci % SA;
                    mbar_wait(smem_u32(a_empty + sa), ((ci / SA) & 1) ^ 1);
                    mbar_expect_tx(smem_u32(a_full + sa), HALO_ROWS * ROWB);
                    if constexpr (SK) load_halo(ci, smem_u32(smA + sa * A_BYTES), smem_u32(a_full + sa));
                    else tma_load_4d(smem_u32(smA + sa * A_BYTES), &tmA, (cb0 + ci) * KCE, x0 - 1, y0 - 1, n, smem_u32(a_full + sa));
                    const int ntile = SK && ci >= nconv ? 1 : TPC;
                    for (int tap = 0; tap < ntile; ++tap, ++bi) {
                        if (bi < npre) continue;
                        const int sb = bi % SB;
                        mbar_wait(smem_u32(b_empty + sb), ((bi / SB) & 1) ^ 1);
                        mbar_expect_tx(smem_u32(b_full + sb), B_BYTES);
                        if constexpr (SK) load_wtile(bi, smem_u32(smB + sb * B_BYTES), smem_u32(b_full + sb));
                        else tma_load_3d(smem_u32(smB + sb * B_BYTES), &tmB, (cb0 + ci) * KCE, n0, halo_wtile<PH>(tap), smem_u32(b_full + sb));
                    }
                }
            }
            if constexpr (ROW_SPLIT) {      // the consumers' cluster barriers A and B (every thread of the cluster arrives)
                __syncwarp();
                cluster_sync_all();
                cluster_sync_all();
            }
        } else {
            // ===== consumer warpgroup(s): normalise each chunk's halo ONCE, in place (XF); 9 taps = 9 row-shifted views of
            // the halo through wgmma; then the epilogue.  With WG = 2 both warpgroups consume every weight stage; warpgroup
            // wg computes tile rows 16 wg .. 16 wg + 15 =====
            const int te = threadIdx.x;                                          // 0 .. 128 WG - 1
            const int wg = WG == 1 ? 0 : te >> 7;
            constexpr int XBAR = WG == 1 ? 1 : 3;                                // named barrier of all consumer threads
            __half* hA = reinterpret_cast<__half*>(xf_A);
            __half* hB = hA + p.xf_C;
            const bool silu = p.xf_act == ACT_SILU || p.xf_act == ACT_SILU_FAST;
            // SELF_LOAD: thread 0 (warpgroup 0) issues every TMA load, in consumption order.  Weight tile j + SB goes out
            // once stage j % SB has been released by both warpgroups, the halo of chunk ci + SA once both have finished
            // chunk ci.  Why no wait can be circular: at MMA step i (its own tile of step i committed), thread 0 waits only
            // for releases the other warpgroup makes at its steps < i -- the tiles of step i - 2 -- and, after the last step
            // of a chunk, for the other warpgroup's end of that same chunk.  For that, the other warpgroup needs the weight
            // tiles of its steps <= i and the chunk's halo.  The tiles of step i + 1 go out at thread 0's step i, before
            // either wait (3x3: tiles up to i + SB - 2, SB >= 3; four phases, two tiles per step: up to 2 i + SB - 3,
            // SB >= 6); the halo at the end of an earlier chunk or before the loop.  The other warpgroup's only other wait
            // is the transform barrier of a chunk, which thread 0 has passed.
            auto load_b = [&](int j) {                           // weight tile j (those of the first ring pass go out before the loop)
                if (j < SB || j >= nb) return;
                const int sb = j % SB;
                mbar_wait(smem_u32(b_empty + sb), ((j / SB) & 1) ^ 1);
                mbar_expect_tx(smem_u32(b_full + sb), B_BYTES);
                if constexpr (SK) load_wtile(j, smem_u32(smB + sb * B_BYTES), smem_u32(b_full + sb));
                else tma_load_3d(smem_u32(smB + sb * B_BYTES), &tmB, (cb0 + j / TPC) * KCE, n0, halo_wtile<PH>(j % TPC), smem_u32(b_full + sb));
            };
            auto load_a = [&](int ci) {                          // the halo of chunk ci
                if (ci >= nc) return;
                const int sa = ci % SA;
                mbar_wait(smem_u32(a_empty + sa), ((ci / SA) & 1) ^ 1);
                mbar_expect_tx(smem_u32(a_full + sa), HALO_ROWS * ROWB);
                if constexpr (SK) load_halo(ci, smem_u32(smA + sa * A_BYTES), smem_u32(a_full + sa));
                else tma_load_4d(smem_u32(smA + sa * A_BYTES), &tmA, (cb0 + ci) * KCE, x0 - 1, y0 - 1, n, smem_u32(a_full + sa));
            };
            if (SELF_LOAD && te == 0) {                          // the first ring pass: nothing to wait for
                for (int ci = 0; ci < SA; ++ci) load_a(ci);
                for (int j = npre; j < min(nb, SB); ++j) {
                    mbar_expect_tx(smem_u32(b_full + j), B_BYTES);
                    if constexpr (SK) load_wtile(j, smem_u32(smB + j * B_BYTES), smem_u32(b_full + j));
                    else tma_load_3d(smem_u32(smB + j * B_BYTES), &tmB, (cb0 + j / TPC) * KCE, n0, halo_wtile<PH>(j % TPC), smem_u32(b_full + j));
                }
            }
            if (XF) {
                double2* chs = reinterpret_cast<double2*>(xf_A + 2 * p.xf_C);
                // SK: the table covers the 3x3 chunks (the skip input is read raw)
                xf_build_coef<128 * WG, XBAR>(p, n, te, hA, hB, chs, (SK ? min(cb0, p.cpt) : cb0) * KCE, (cb0 + nconv) * KCE);
                if (te == 0) HSTAMP_END(2, 0);
            }
            int bi = 0;
            for (int ci = 0; ci < nc; ++ci) {
                const int sa = ci % SA;
                mbar_wait(smem_u32(a_full + sa), (ci / SA) & 1);
                if (te == 0 && ci == 0) HSTAMP_END(2, 1);
                const bool skip_chunk = SK && ci >= nconv;
                if (XF && !skip_chunk) {
                    const int c0 = (cb0 + ci) * KCE;
                    // items = (halo row, half row): 360 / 680 items over 128 / 256 threads; the rows both warpgroups read
                    // are transformed once
                    constexpr int HC = ROWB / 32;                                             // chunks per half row
                    for (int it = te; it < 2 * HALO_ROWS; it += 128 * WG) {
                        const int row = it >> 1, half = it & 1;
                        const int hy = row / HALO_W, hx = row - hy * HALO_W;
                        const int iy = y0 - 1 + hy, ix = x0 - 1 + hx;
                        if (iy < 0 || iy >= p.inH || ix < 0 || ix >= p.inW) continue;      // zero padding stays zero
                        const int swz = ROWB == 128 ? (row & 7) : ((row >> 1) & 3);
                        xf_chunks<HC>(smA + sa * A_BYTES + row * ROWB, swz, half * HC, c0, p, hA, hB, silu);
                    }
                    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // generic-proxy writes -> wgmma's async-proxy reads
                    asm volatile("bar.sync %0, %1;\n" :: "n"(XBAR), "n"(128 * WG) : "memory");
                    if (te == 0 && ci == nc - 1) HSTAMP_END(2, 2);
                }
                const uint32_t a_base = smem_u32(smA + sa * A_BYTES) + (uint32_t)(SLABS > 1 ? wg * HT_H * HALO_W * ROWB : 0);
                if constexpr (PH == 4) {
                    // warpgroup py: steps s = 2 tap + px into the accumulator of phase (py, px); its weight tile is tile
                    // 2 s + py of the chunk.  K order per phase: chunk, then tap (conv_tc: tap, then chunk)
#pragma unroll
                    for (int s = 0; s < 8; ++s) {
                        const int tap = s >> 1, px = s & 1, phase = 2 * wg + px;
                        const int bj = ci * 16 + 2 * s + wg;
                        const int sb = bj % SB;
                        mbar_wait(smem_u32(b_full + sb), (bj / SB) & 1);
                        const int shift = (p.dy[phase][tap] + 1) * HALO_W + (p.dx[phase][tap] + 1);
                        const uint32_t a0 = a_base + shift * ROWB, a1 = a0 + 8 * HALO_W * ROWB;
                        const uint32_t b_addr = smem_u32(smB + sb * B_BYTES);
                        wg_fence();
#pragma unroll
                        for (int k = 0; k < ROWB / 32; ++k) {
                            const uint64_t bd = make_smem_desc_sw<ROWB>(b_addr + 32 * k);
                            const uint32_t accum = (ci > 0 || tap > 0 || k > 0) ? 1u : 0u;
                            Wgmma<BN>::f16(acc[px].d[0], make_desc_sbo<ROWB>(a0 + 32 * k, HALO_W * ROWB), bd, accum);
                            Wgmma<BN>::f16(acc[px].d[1], make_desc_sbo<ROWB>(a1 + 32 * k, HALO_W * ROWB), bd, accum);
                        }
                        wg_commit();
                        if (s < 7) {
                            wg_wait<1>();                                       // the previous step's weight tile has been read
                            if (s > 0) mbar_arrive(smem_u32(b_empty + (bj - 2) % SB));
                        } else {
                            wg_wait<0>();                                       // the chunk's halo and this warpgroup's last two tiles are free
                            mbar_arrive(smem_u32(b_empty + (bj - 2) % SB));
                            mbar_arrive(smem_u32(b_empty + sb));
                            mbar_arrive(smem_u32(a_empty + sa));
                        }
                        if (SELF_LOAD && te == 0) {             // tiles up to bj - 3 (warpgroup 1's, step s - 2) are released
                            load_b(bj + SB - 4);
                            load_b(bj + SB - 3);
                            if (s == 7) load_a(ci + SA);
                        }
                    }
                } else if (skip_chunk) {
                    // a chunk of the folded skip: the centre-tap view of the raw input's halo, one weight tile
                    const int sb = bi % SB;
                    mbar_wait(smem_u32(b_full + sb), (bi / SB) & 1);
                    const uint32_t a0 = a_base + (HALO_W + 1) * ROWB, a1 = a0 + 8 * HALO_W * ROWB;
                    const uint32_t b_addr = smem_u32(smB + sb * B_BYTES);
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < ROWB / 32; ++k) {
                        const uint64_t bd = make_smem_desc_sw<ROWB>(b_addr + 32 * k);
                        const uint32_t accum = (ci > 0 || k > 0) ? 1u : 0u;
                        Wgmma<BN>::f16(acc[0].d[0], make_desc_sbo<ROWB>(a0 + 32 * k, HALO_W * ROWB), bd, accum);
                        Wgmma<BN>::f16(acc[0].d[1], make_desc_sbo<ROWB>(a1 + 32 * k, HALO_W * ROWB), bd, accum);
                    }
                    wg_commit();
                    wg_wait<0>();                                               // the chunk's halo and its weight tile are free
                    mbar_arrive(smem_u32(b_empty + sb));
                    mbar_arrive(smem_u32(a_empty + sa));
                    if (SELF_LOAD && te == 0) {                 // tiles up to bi - 1 are released
                        load_b(bi + SB - 2);
                        load_a(ci + SA);
                    }
                    ++bi;
                } else {
                    // unrolled: the wait depth and the arrivals below depend on the tap only, so no branch separates wgmma issue
                    // from its wait (a data-dependent one makes ptxas serialise the wgmma)
#pragma unroll
                    for (int tap = 0; tap < 9; ++tap, ++bi) {
                        const int sb = bi % SB;
                        mbar_wait(smem_u32(b_full + sb), (bi / SB) & 1);
                        const int shift = (p.dy[0][tap] + 1) * HALO_W + (p.dx[0][tap] + 1);
                        // rows 0-63 of the tile are tile rows 0-7 (halo rows from `shift`), rows 64-127 tile rows 8-15 (8 halo pitches on)
                        const uint32_t a0 = a_base + shift * ROWB, a1 = a0 + 8 * HALO_W * ROWB;
                        const uint32_t b_addr = smem_u32(smB + sb * B_BYTES);
                        wg_fence();
#pragma unroll
                        for (int k = 0; k < ROWB / 32; ++k) {
                            const uint64_t bd = make_smem_desc_sw<ROWB>(b_addr + 32 * k);
                            const uint32_t accum = (ci > 0 || tap > 0 || k > 0) ? 1u : 0u;
                            Wgmma<BN>::f16(acc[0].d[0], make_desc_sbo<ROWB>(a0 + 32 * k, HALO_W * ROWB), bd, accum);
                            Wgmma<BN>::f16(acc[0].d[1], make_desc_sbo<ROWB>(a1 + 32 * k, HALO_W * ROWB), bd, accum);
                        }
                        wg_commit();
                        if (tap < 8) {
                            wg_wait<1>();                                           // the previous tap's weight tile has been read
                            if (tap > 0) mbar_arrive(smem_u32(b_empty + (bi - 1) % SB));
                        } else {
                            wg_wait<0>();                                           // the chunk's halo and its last two weight tiles are free
                            mbar_arrive(smem_u32(b_empty + (bi - 1) % SB));
                            mbar_arrive(smem_u32(b_empty + bi % SB));
                            mbar_arrive(smem_u32(a_empty + sa));
                        }
                        if (SELF_LOAD && te == 0) {             // tiles up to bi - 2 are released
                            load_b(bi + SB - 2);
                            if (tap == 8) load_a(ci + SA);
                        }
                    }
                    if (SK && ci == nconv - 1) {                // the 3x3 sum in the skip weights' units (a power of two: exact)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int j = 0; j < BN / 2; ++j) acc[0].d[h][j] *= p.acc_rescale;
                    }
                }
            }
#pragma unroll
            for (int a = 0; a < NACC; ++a) { wg_fence_acc(acc[a].d[0]); wg_fence_acc(acc[a].d[1]); }
            if (te == 0) { HSTAMP_END(1, 1); HSTAMP_END(2, 3); }
            if constexpr (ROW_SPLIT) {
                // barrier A: both CTAs' MMAs have retired, their rings are idle.  Warpgroup wg = 1 - split pushes its rows to
                // their owner, rank wg, into the half of the ring the owner's epilogue (warpgroup wg there) leaves alone: half
                // 1 - wg.  Barrier B: the pushes are visible; nobody touches a peer's memory afterwards.
                cluster_sync_all();
                if (wg != split) {
                    uint32_t remote;
                    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(smem_u32(smem + (1 - wg) * EPI_BYTES)), "r"(wg));
                    halo_push_rows<BN, NACC>(acc, remote, te & 127);
                }
                cluster_sync_all();
                if (wg == split) halo_add_rows<BN, NACC>(acc, smem + (1 - wg) * EPI_BYTES, te & 127);
            } else if constexpr (WG > 1) {
                // the epilogue reuses the ring: with two warpgroups, the other one may still be reading its last stages
                asm volatile("bar.sync 3, 256;\n" ::: "memory");
            }
            if (!ROW_SPLIT || wg == split) {
                if constexpr (PH == 4) {
                    // phase (wg, px) of the low-resolution tile: output pixels (2 y + wg, 2 x + px), plain stores
#pragma unroll
                    for (int px = 0; px < 2; ++px) {
                        // the statistics fold of the first call reads both warpgroups' partials before the second rewrites them
                        if (px > 0 && !ROW_SPLIT) asm volatile("bar.sync 3, 256;\n" ::: "memory");
                        epi_direct<BN, HT_W, 0, WG, !ROW_SPLIT>(p, acc[px], smem + wg * EPI_BYTES, n, y0, x0, n0, 2 * wg + px, 0, warp, lane,
                                                                nullptr, nullptr, nullptr, nullptr, wg, EPI_BYTES);
                    }
                } else if (CS == 1 || ROW_SPLIT) {
                    epi_direct<BN, HT_W, NSLOT, WG, !ROW_SPLIT>(p, acc[0], smem + wg * EPI_BYTES, n, y0 + wg * HT_H, x0, n0, 0, 0, warp, lane,
                                                                &tmO32, &tmO16, &tmR, res_bars + 4 * wg, wg, EPI_BYTES);
                }
            }
            if (te == 0) HSTAMP_END(2, 4);
        }
    }
    if constexpr (CS > 1 && !ROW_SPLIT) {
        // barrier A: every CTA of the cluster has its accumulator and idle pipeline buffers -> peers may write into them
        asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
        if (threadIdx.x == 0) HSTAMP(2, 5);
        if (warp < PRODUCER_WARP && nc > 0) epi_push_partial<BN, CS>(acc[0], smem, split, warp, lane);
        // barrier B: the pushed slices are visible to their owners; nobody touches a peer's memory afterwards
        asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
        if (threadIdx.x == 0) HSTAMP(2, 7);
        if (warp < PRODUCER_WARP) epi_cluster_reduce<BN, CS, HT_W>(p, smem, n, y0, x0, n0, 0, split, warp, dbg);
        if (threadIdx.x == 0) HSTAMP(2, 6);
    }
    __syncthreads();
    if (threadIdx.x == 0) HSTAMP_END(0, 3);
#undef HSTAMP_END
#undef HSTAMP
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn halo_encode() {
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

using HKey = std::tuple<int, const void*, long, long, long, long, long, int>;
std::map<HKey, CUtensorMap> g_halo_maps;
std::mutex g_halo_mu;

const CUtensorMap& halo_activation_map(const View& v, int op, int wg) {
    HKey key{current_device(), v.p, v.N, v.H, v.W, v.C, v.ld, op + 16 * wg};
    std::lock_guard<std::mutex> lock(g_halo_mu);
    auto it = g_halo_maps.find(key);
    if (it != g_halo_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[4] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)v.N};
    cuuint64_t strides[3] = {(cuuint64_t)v.ld * 2, (cuuint64_t)v.W * v.ld * 2, (cuuint64_t)v.H * v.W * v.ld * 2};
    cuuint32_t box[4] = {(cuuint32_t)op_kch(op), (cuuint32_t)HALO_W, (cuuint32_t)halo_h(wg), 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = halo_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, v.p, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               op == OP_F16N ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(halo activation) failed: " + std::to_string((int)r));
    return g_halo_maps.emplace(key, m).first->second;
}

const CUtensorMap& halo_weight_map(const ConvWeights& cw, int bn, int op) {
    HKey key{current_device(), cw.w16, cw.cin_pad, cw.cout_pad, cw.ntaps * cw.nphase, bn, -1, op};
    std::lock_guard<std::mutex> lock(g_halo_mu);
    auto it = g_halo_maps.find(key);
    if (it != g_halo_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)cw.cin_pad, (cuuint64_t)cw.cout_pad, (cuuint64_t)cw.ntaps * cw.nphase};
    cuuint64_t strides[2] = {(cuuint64_t)cw.cin_pad * 2, (cuuint64_t)cw.cout_pad * cw.cin_pad * 2};
    cuuint32_t box[3] = {(cuuint32_t)op_kch(op), (cuuint32_t)bn, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = halo_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, cw.w16, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               op == OP_F16N ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(halo weights) failed: " + std::to_string((int)r));
    return g_halo_maps.emplace(key, m).first->second;
}

// Output tile of the unsplit epilogue: box {32 channels, 16 x 8 pixels}, rows of 128 bytes (fp32) / 64 bytes (f16), swizzled
// like the staging writes of epi_direct.  Returns false when the view cannot be described (alignment).
bool halo_store_map(const View& v, bool f16, const CUtensorMap** out) {
    const int es = f16 ? 2 : 4;
    if (!v.p || (reinterpret_cast<uintptr_t>(v.p) & 15) || ((long)v.ld * es) % 16 != 0) return false;
    HKey key{current_device(), v.p, v.N, v.H, v.W, v.C, v.ld, f16 ? -2 : -3};
    std::lock_guard<std::mutex> lock(g_halo_mu);
    auto it = g_halo_maps.find(key);
    if (it == g_halo_maps.end()) {
        CUtensorMap m;
        cuuint64_t dims[4] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)v.N};
        cuuint64_t strides[3] = {(cuuint64_t)v.ld * es, (cuuint64_t)v.W * v.ld * es, (cuuint64_t)v.H * v.W * v.ld * es};
        cuuint32_t box[4] = {32, (cuuint32_t)HT_W, (cuuint32_t)HT_H, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = halo_encode()(&m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, v.p, dims, strides, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, f16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return false;
        it = g_halo_maps.emplace(key, m).first;
    }
    *out = &it->second;
    return true;
}

// Shared memory of a CTA: the rings, the barriers, the alignment slack (the XF table comes on top)
constexpr size_t halo_ring(int op, int bn, int sa, int sb, int wg, int ph) {
    return (size_t)sa * halo_a_bytes(op_row_bytes(op), ph == 1 ? wg : 1) + (size_t)sb * bn * op_row_bytes(op);
}
constexpr size_t halo_smem0(int op, int bn, int sa, int sb, int wg, int ph) {
    return 1024 + halo_ring(op, bn, sa, sb, wg, ph) + (2 * sa + 2 * sb + 4 * wg) * 8 + 16;
}

// wg: consumer warpgroups per CTA (1: 128-pixel tiles; 2: 256-pixel tiles, unsplit launches only)
// ctas: resident CTAs per SM of a two-warpgroup launch with 256 x 64 or four-phase tiles (conv_halo_kernel's CTAS)
struct HaloPlan { int bn, tiles_x, tiles_y, tiles_m, tiles_n, cs, chunks, wg, ctas; };

// Weight stages of a two-warpgroup CTA: at least sb_min, and enough that each warpgroup's half of the idle ring holds the
// epilogue scratch and one TMA-store staging slot.
constexpr int halo_sb_wg2(int op, int bn, int sa, int sb_min) {
    const size_t a = (size_t)sa * halo_a_bytes(op_row_bytes(op), 2), b = (size_t)bn * op_row_bytes(op);
    int sb = sb_min;
    while (a + sb * b < 2 * (size_t)(epi_slot0(bn) + EPI_SLOT_BYTES)) ++sb;
    return sb;
}
// Rings of the 256-thread CTAs, two per SM (<= ~113 KB each with the XF table of up to 512 channels).  256 x 64 tiles: one
// halo stage of 64-channel chunks and six weight stages (two halo stages of 32-channel chunks, and the weight stages the
// epilogue needs); four phases: two halo stages and twelve 32-column weight tiles, three quarters of a chunk.
constexpr int halo2_sa(int op, int ph) { return ph == 4 || op == OP_F16N ? 2 : 1; }
constexpr int halo2_sb(int op, int ph) { return ph == 4 ? 12 : halo_sb_wg2(op, 64, halo2_sa(op, ph), op == OP_F16N ? 12 : 6); }

// Two-warpgroup launches with 256 x 64 or four-phase tiles run two 256-thread CTAs per SM when there are more CTAs than
// SMs and two fit in shared memory (228 KB per SM on sm_90, 1 KB of it reserved per CTA).  With one CTA per SM, each SM
// runs a CTA's start-up, its chunks' operand transforms and its epilogue with the tensor pipe idle; a second CTA's MMAs
// fill those gaps.  Measured alone on an H100 SXM (700 W), every such layer of the teacher frame with 144 - 1024 CTAs ran
// 1.04 - 1.18x faster on two CTAs per SM; with at most one CTA per SM (32 - 128 CTAs) nothing overlaps, and the
// shallower rings made the same layers 1.2 - 1.8x slower.
int halo_plan_ctas(int op, int bn, int ph, long ctas, const ConvArgs& a) {
    if (opts().halo_ctas > 0) return opts().halo_ctas;
    const size_t smem = halo_smem0(op, bn, halo2_sa(op, ph), halo2_sb(op, ph), 2, ph) + (a.nin.on ? (size_t)24 * a.nin.C + 32 : 0);
    return ctas > num_sms() && 2 * (smem + 1024) <= (size_t)228 * 1024 ? 2 : 1;
}

// A two-warpgroup launch of one CTA per SM becomes a row-owning cluster pair (cs = 2, conv_halo_kernel's ROW_SPLIT) when
// twice its CTAs still fit one wave and every rank gets channel chunks: the idle SMs take half of each tile's K.  Measured
// alone on an H100 SXM (700 W), the teacher frame's 64^2 3x3 layers (32 - 64 CTAs, 2 - 8 chunks) ran 1.20 - 1.66x faster
// as pairs (64^2 256 -> 256: 29.0 -> 20.0 us), the four-phase layers from 32^2 and 64^2 (64 CTAs) 1.47x and 1.28x; with
// 72 - 256 CTAs (a second wave) the pairs were 0.60 - 0.87x as fast, and those layers stay unsplit.
int halo_plan_cs(long ctas, int chunks, const ConvArgs& a) {
    const int mode = opts().halo_cs;
    if (mode == 1 || chunks < 2) return 1;
    return mode == 2 || (a.ksplit <= 0 && 2 * ctas <= num_sms()) ? 2 : 1;
}

// Every rank of a cs-way cluster split owns channel chunks (a folded skip's list: halo_fold_c0)
bool halo_ranks_own_chunks(const ConvWeights& cw, int op, int cs) {
    const int cpt = cw.cin_pad / op_kch(op), chunks = cpt + cw.cin2_pad / op_kch(op);
    if (cs > chunks) return false;
    if (cw.cin2 == 0) return ceil_div(chunks, ceil_div(chunks, cs)) == cs;
    for (int r = 0; r < cs; ++r)
        if (halo_fold_c0(r + 1, cs, cpt, chunks - cpt) <= halo_fold_c0(r, cs, cpt, chunks - cpt)) return false;
    return true;
}

HaloPlan halo_plan(const ConvWeights& cw, const ConvArgs& a, int op) {
    HaloPlan pl;
    pl.chunks = (cw.cin_pad + cw.cin2_pad) / op_kch(op);      // a folded skip's chunks included
    if (cw.nphase == 4) {
        // one 8 x 16 low-resolution tile (4 x 128 output pixels) x 32 columns per CTA, unsplit
        pl.tiles_x = ceil_div(a.in.W, HT_W); pl.tiles_y = ceil_div(a.in.H, HT_H);
        pl.tiles_m = pl.tiles_x * pl.tiles_y * a.in.N;
        pl.bn = 32; pl.tiles_n = cw.cout_pad / 32; pl.cs = 1; pl.wg = 2;
        pl.ctas = halo_plan_ctas(op, 32, 4, (long)pl.tiles_m * pl.tiles_n, a);
        if (pl.ctas == 1) pl.cs = halo_plan_cs((long)pl.tiles_m * pl.tiles_n, pl.chunks, a);
        return pl;
    }
    pl.tiles_x = ceil_div(a.out.W, HT_W); pl.tiles_y = ceil_div(a.out.H, HT_H);
    pl.tiles_m = pl.tiles_x * pl.tiles_y * a.in.N;
    // N tile: at most 128 columns, the accumulator of one consumer warpgroup (BN fp32 registers per thread)
    pl.bn = (cw.cout_pad % 128 == 0) ? 128 : (cw.cout_pad % 64 == 0 ? 64 : 32);
    const int sms = num_sms();
    pl.cs = 1;
    long ctas = (long)pl.tiles_m * (cw.cout_pad / pl.bn);
    // 256-pixel tiles (two consumer warpgroups, see below) for every launch of at least an eighth of a wave of 128-pixel
    // tiles, unsplit even when the CTAs do not fill the GPU: measured alone on an H100, every such layer of the teacher
    // frame ran faster than on 128-pixel tiles (1.03 - 1.36x at a 400 W power limit, down to 128 tiles), and the 64 x 64
    // layers with 128 - 512 channels (32 tiles) faster than their cluster split-K launches (1.1 - 2.1x at 700 W).  With fewer tiles (32 x 32 and
    // below) the split-K launches win.
    const int m256_mode = opts().halo_m256;
    const bool m256 = m256_mode > 0 || (m256_mode < 0 && a.ksplit <= 1 && 8L * pl.tiles_m >= sms);
    if (a.ksplit > 1) {
        while (pl.cs * 2 <= std::min(8, a.ksplit)) pl.cs *= 2;
    } else if (a.ksplit <= 0 && ctas < sms * 13 / 16 && !m256) {
        // Too few tiles to fill the GPU.  Narrow the N tiles first (down to 64 columns: more CTAs and nothing to exchange),
        // then split the channel chunks over a cluster.  The DSMEM exchange moves 128 x bn x 4 x (cs-1)/cs bytes per CTA at
        // a few bytes per clock, so a wide split of a wide tile costs more than the MMA phase it parallelises.
        while (pl.bn > 64 && (long)pl.tiles_m * (cw.cout_pad / pl.bn) < sms && cw.cout_pad % (pl.bn / 2) == 0) pl.bn /= 2;
        ctas = (long)pl.tiles_m * (cw.cout_pad / pl.bn);
        const int want = std::max(2, (int)((3 * sms / 2 + ctas - 1) / ctas));       // >= 2: the cluster variants carry the deep weight ring
        while (pl.cs < 8 && pl.cs * 2 <= want && pl.cs * 2 <= pl.chunks) pl.cs *= 2;
        while (pl.bn > 32 && (long)pl.tiles_m * (cw.cout_pad / pl.bn) * pl.cs < 96 && cw.cout_pad % (pl.bn / 2) == 0) pl.bn /= 2;
    }
    while (pl.cs > 1 && !halo_ranks_own_chunks(cw, op, pl.cs)) pl.cs /= 2;
    pl.tiles_n = cw.cout_pad / pl.bn;
    // Unsplit launches with many tiles take 256-pixel tiles: each weight tile then feeds 256 rows instead of 128.  Two
    // 128-column accumulators do not fit the registers of a 288-thread CTA, so 128-column tiles become 256 x 64 (per FLOP:
    // half the weight bytes, twice the halo bytes -- a third less L2 -> shared-memory traffic in all).
    pl.wg = 1;
    if (pl.cs == 1 && m256) {
        pl.wg = 2;
        pl.tiles_y = ceil_div(a.out.H, 2 * HT_H);
        pl.tiles_m = pl.tiles_x * pl.tiles_y * a.in.N;
        pl.bn = std::min(pl.bn, 64);
        pl.tiles_n = cw.cout_pad / pl.bn;
    }
    pl.ctas = pl.wg == 2 && pl.bn == 64 ? halo_plan_ctas(op, 64, 1, (long)pl.tiles_m * pl.tiles_n, a) : 1;
    if (pl.wg == 2 && pl.ctas == 1) pl.cs = halo_plan_cs((long)pl.tiles_m * pl.tiles_n, pl.chunks, a);
    return pl;
}

// The tensor maps of a launch: activation halo, weights, fp32 / f16 output and residual tiles, and a folded skip's input
// halo and weights (placeholders where a launch does not read them)
struct HaloMaps { const CUtensorMap *a, *b, *o32, *o16, *r, *a2, *b2; };

template <int OP, int BN, int SA, int SB, int CS, int XF, int WG = 1, int PH = 1, int CTAS = 1, int SK = 0>
void launch_halo(const HaloMaps& m, const TcParams& p, dim3 grid, cudaStream_t s) {
    constexpr size_t ring = halo_ring(OP, BN, SA, SB, WG, PH);
    constexpr size_t smem0 = halo_smem0(OP, BN, SA, SB, WG, PH);
    static_assert(smem0 <= 227 * 1024, "shared memory budget");
    static_assert(ring / WG >= (size_t)4 * 32 * 33 * 4 + 4 * BN * 8, "epilogue scratch must fit in the pipeline buffers");
    static_assert(WG == 1 || PH == 4 || epi_nslot(BN, (ring / WG) & ~(size_t)1023) > 0, "two warpgroups: a TMA-store staging slot each");
    static_assert(CS == 1 || ring >= (size_t)128 * BN * 4 + 128 * 8 * 4 + 128 * 4 * 4, "partial tile + statistics scratch must fit");
    static_assert(CTAS == 1 || 2 * (smem0 + 1024) <= 228 * 1024, "two CTAs per SM");
    const size_t smem = smem0 + (XF ? (size_t)24 * p.xf_C + 32 : 0);
    THA4_REQUIRE(smem <= 227 * 1024, "conv_halo: shared memory budget (fused input normalisation)");
    THA4_ENSURE_SMEM((conv_halo_kernel<BN, SA, SB, CS, OP, XF, WG, PH, CTAS, SK>), smem);
    launch_pdl(conv_halo_kernel<BN, SA, SB, CS, OP, XF, WG, PH, CTAS, SK>, grid, dim3(halo_threads(WG, CTAS)), smem, s, CS,
               *m.a, *m.b, *m.o32, *m.o16, *m.r, p, *m.a2, *m.b2);
    THA4_LAUNCH_CHECK();
}

// SBD: weight-ring depth of the cluster split-K launches (few CTAs per SM, the ring is what hides the DRAM latency of weights
// that are fetched ahead of the dependency wait); SBS: depth of the unsplit launches (many tiles: a shallow ring keeps
// the CTA small so that 2 - 4 of them share an SM and overlap each other's load -> transform -> MMA -> drain chains).
template <int OP, int BN, int SA, int SBD, int SBS, int XF, int SK>
void launch_halo_cs(int cs, int wg, int ctas, const HaloMaps& m, const TcParams& p, dim3 grid, cudaStream_t s) {
    constexpr int SA1 = OP == OP_F16N ? 2 : 1;
    const int chunks = p.cpt + p.cpt2;
    THA4_REQUIRE(wg == 1 || (BN <= 64 && (cs == 1 || (cs == 2 && ctas == 1 && chunks >= 2))),
                 "conv_halo: 256-pixel tiles need N tiles of at most 64 columns, unsplit or a pair of one-CTA-per-SM ranks with chunks each");
    THA4_REQUIRE(ctas == 1 || (wg == 2 && BN == 64 && cs == 1), "conv_halo: two CTAs per SM are built for unsplit 256 x 64 tiles");
    if constexpr (BN == 64) {
        if (ctas == 2) {     // one chunk or several: the same rings
            launch_halo<OP, 64, halo2_sa(OP, 1), halo2_sb(OP, 1), 1, XF, 2, 1, 2, SK>(m, p, grid, s);
            return;
        }
    }
    if constexpr (BN <= 64) {
        if (!SK && cs == 1 && chunks == 1) {     // one chunk: one halo, ever -> a ring that fits four times per SM (twice with two warpgroups)
            if (wg == 2) launch_halo<OP, BN, SA1, halo_sb_wg2(OP, BN, SA1, BN == 64 ? SBD : SBS), 1, XF, 2>(m, p, grid, s);
            else launch_halo<OP, BN, SA1, SBS, 1, XF>(m, p, grid, s);
            return;
        }
    }
    if constexpr (BN <= 64) {
        if (wg == 2) {
            // BN = 64: one CTA per SM, which takes the deep weight ring; BN = 32: two CTAs per SM.  A row-owning pair keeps the rings
            constexpr int M = OP == OP_F16N ? 2 : 1;
            constexpr int SB2 = halo_sb_wg2(OP, BN, SA, BN == 64 ? SBD : 2 * M);
            if (cs == 2) launch_halo<OP, BN, SA, SB2, 2, XF, 2, 1, 1, SK>(m, p, grid, s);
            else launch_halo<OP, BN, SA, SB2, 1, XF, 2, 1, 1, SK>(m, p, grid, s);
            return;
        }
    }
    if (cs == 8) launch_halo<OP, BN, SA, SBD, 8, XF, 1, 1, 1, SK>(m, p, grid, s);
    else if (cs == 4) launch_halo<OP, BN, SA, SBD, 4, XF, 1, 1, 1, SK>(m, p, grid, s);
    else if (cs == 2) launch_halo<OP, BN, SA, SBD, 2, XF, 1, 1, 1, SK>(m, p, grid, s);
    else if ((long)grid.x * grid.y * grid.z <= num_sms())
        // unsplit and at most one CTA per SM (e.g. 256 -> 256 channels at 128 x 128: 128 tiles): nothing shares the SM, so the
        // CTA takes the deep weight ring: with a two-stage ring the MMAs wait on weight tiles streaming from L2
        launch_halo<OP, BN, SA, SBD, 1, XF, 1, 1, 1, SK>(m, p, grid, s);
    else launch_halo<OP, BN, SA, SBS, 1, XF, 1, 1, 1, SK>(m, p, grid, s);
}

template <int OP, int XF, int SK = 0>
void launch_halo_bn(int bn, int cs, int wg, int ctas, const HaloMaps& m, const TcParams& p, dim3 grid, cudaStream_t s) {
    constexpr int M = OP == OP_F16N ? 2 : 1;        // 64-byte rows: twice the stages for the same bytes in flight
    if (bn == 128) launch_halo_cs<OP, 128, 2 * M, 6 * M, 3 * M, XF, SK>(cs, wg, ctas, m, p, grid, s);        // unsplit:  95 KB
    else if (bn == 64) launch_halo_cs<OP, 64, 2 * M, 8 * M, 3 * M, XF, SK>(cs, wg, ctas, m, p, grid, s);     // unsplit:  71 KB
    else launch_halo_cs<OP, 32, 2 * M, 9 * M, 5 * M, XF, SK>(cs, wg, ctas, m, p, grid, s);                    // unsplit:  67 KB
}

}  // namespace

// One operand format for both sources of a folded skip: 64-channel chunks only when both widths allow them
static int halo_op(const ConvWeights& cw) { return cw.cin_pad % 64 == 0 && cw.cin2_pad % 64 == 0 ? OP_F16 : OP_F16N; }

bool conv_halo_supported(const ConvWeights& cw, const ConvArgs& a) {
    if (!opts().halo_conv || !conv_tc_supported(cw, a)) return false;
    if (!a.in.f16 || cw.stride != 1) return false;
    // a folded 1x1 conv: its f16 input at the output's resolution, TMA-able, on the 3x3 normalised-input kernels
    if (cw.cin2 > 0 && (!cw.w16b || cw.ntaps != 9 || cw.nphase != 1 || !a.nin.on || a.res.p || !a.in2.f16 || !a.in2.p || a.in2.C != cw.cin2 ||
                        a.in2.N != a.out.N || a.in2.H != a.out.H || a.in2.W != a.out.W || a.in2.ld % 8 != 0 || (((uintptr_t)a.in2.p) & 15) != 0))
        return false;
    const bool four_phase = cw.nphase == 4 && cw.ntaps == 4 && cw.out_mul == 2;
    if (!four_phase && (cw.ntaps != 9 || cw.nphase != 1 || cw.out_mul != 1)) return false;
    for (int ph = 0; ph < cw.nphase; ++ph)
        for (int t = 0; t < cw.ntaps; ++t)
            if (cw.dy[ph][t] < -1 || cw.dy[ph][t] > 1 || cw.dx[ph][t] < -1 || cw.dx[ph][t] > 1) return false;
    if (!four_phase) return a.in.H == a.out.H && a.in.W == a.out.W;
    // four phases: 64-channel chunks only (the layers of the networks), unsplit.  An explicit split goes to conv_tc.cu
    if (cw.cin_pad % 64 != 0 || a.ksplit > 1 || a.out.H != 2 * a.in.H || a.out.W != 2 * a.in.W) return false;
    // The automatic plan takes the halo kernel from 64 CTAs (8 x 16 x 32 tiles) up.  Measured alone on an H100 SXM (132 SMs)
    // it ran 1.1 - 2.5x faster than conv_tc.cu's launches on every such layer of the teacher frame and at batch 32; with
    // 16 - 48 CTAs (the 16^2 - 32^2 low-resolution layers of 256 - 512 channels) conv_tc.cu's cluster split-K was as fast
    // or faster (0.55 - 1.02x).
    const HaloPlan pl = halo_plan(cw, a, OP_F16);
    return a.ksplit == 1 || (long)pl.tiles_m * pl.tiles_n >= 64;
}

bool conv_halo_fuses_stats(const ConvWeights&, const ConvArgs&) { return true; }       // unsplit or cluster split: always final

// Which outputs of a launch with plan `pl` leave through TMA stores (bit 0 fp32, bit 1 f16) and whether the residual arrives
// through the same box (bit 2); the maps of those that do
static int halo_st_tma(const ConvWeights& cw, const ConvArgs& a, const HaloPlan& pl, const CUtensorMap** mo32, const CUtensorMap** mo16,
                       const CUtensorMap** mr) {
    int st = 0;
    if ((pl.cs == 1 || pl.wg == 2) && opts().tma_store && cw.nphase == 1) {
        if (a.out.p && halo_store_map(a.out, false, mo32)) st |= 1;
        if (a.out16.p && halo_store_map(a.out16, true, mo16)) st |= 2;
        // the residual of a ResBlock's second conv has the geometry of the fp32 output: it arrives through the same box
        if ((st & 1) && a.res.p && a.res_mode == RES_SAME && !a.res.f16 && a.res.N == a.out.N && a.res.H == a.out.H &&
            a.res.W == a.out.W && a.res.C >= a.out.C && halo_store_map(a.res, false, mr)) st |= 4;
    }
    return st;
}

bool conv_halo_plan_info(const ConvWeights& cw, const ConvArgs& a, int* info) {
    if (!conv_halo_supported(cw, a)) return false;
    const HaloPlan pl = halo_plan(cw, a, halo_op(cw));
    const CUtensorMap *m32 = nullptr, *m16 = nullptr, *mr = nullptr;
    info[0] = pl.bn; info[1] = pl.cs; info[2] = pl.wg; info[3] = pl.ctas; info[4] = cw.nphase;
    info[5] = halo_st_tma(cw, a, pl, &m32, &m16, &mr); info[6] = pl.chunks;
    return true;
}

void conv_halo_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s) {
    THA4_REQUIRE(conv_halo_supported(cw, a), "conv_halo: unsupported configuration");
    THA4_REQUIRE(a.in.C == cw.cin && a.out.C == cw.cout && a.in.N == a.out.N, "conv_halo: shapes");
    const int op = halo_op(cw);
    TcParams p{};
    p.out = a.out.p; p.outH = a.out.H; p.outW = a.out.W; p.outC = a.out.C; p.out_ld = a.out.ld;
    p.out16 = a.out16.p ? a.out16.hp() : nullptr; p.out16_ld = a.out16.ld;
    if (a.out16.p) THA4_REQUIRE(a.out16.f16 && a.out16.N == a.out.N && a.out16.H == a.out.H && a.out16.W == a.out.W && a.out16.C == a.out.C, "conv_halo: f16 output copy geometry");
    p.inH = a.in.H; p.inW = a.in.W; p.inC = a.in.C;
    if (a.nin.on) {
        const ConvNormIn& ni = a.nin;
        THA4_REQUIRE(ni.stats != nullptr && ni.gamma != nullptr && ni.beta != nullptr, "conv_halo: fused input normalisation needs statistics and affine parameters");
        THA4_REQUIRE(ni.C > 0 && ni.C <= a.in.C && ni.C % 8 == 0 && ni.C <= 1024, "conv_halo: normalised channel count");
        THA4_REQUIRE(ni.groups == 0 || (ni.C == a.in.C && ni.C % ni.groups == 0), "conv_halo: GroupNorm spans the whole input");
        p.in_stats = ni.stats; p.in_stats_ld = ni.stats_ld; p.in_stats_rep = std::max(1, ni.stats_rep); p.in_stats_rep_stride = ni.stats_rep_stride;
        p.xf_C = ni.C; p.xf_groups = ni.groups; p.xf_act = ni.act;
        p.xf_inv_cnt = 1.0 / ((double)a.in.H * a.in.W * (ni.groups == 0 ? 1 : ni.C / ni.groups));
        p.xf_gamma = ni.gamma; p.xf_beta = ni.beta; p.xf_film0 = ni.film0; p.xf_film1 = ni.film1; p.xf_film1_ld = ni.film1_ld;
    }
    p.bias = cw.bias;
    p.res = a.res.p; p.res_mode = a.res.p ? a.res_mode : RES_NONE;
    p.resH = a.res.H; p.resW = a.res.W; p.res_ld = a.res.ld;
    p.N = a.in.N; p.out_mul = cw.out_mul; p.in_mul = 1;
    const HaloPlan pl = halo_plan(cw, a, op);
    p.MH = a.out.H / cw.out_mul; p.MW = a.out.W / cw.out_mul; p.tiles_x = pl.tiles_x; p.tiles_y = pl.tiles_y;
    p.pre_b = cw.dynamic ? 0 : 1;
    p.ntaps = cw.ntaps; p.cpt = cw.cin_pad / op_kch(op); p.cpt2 = cw.cin2_pad / op_kch(op);
    if (!cw.w16) { conv_make_half(cw, s); p.pre_b = 0; }
    p.acc_scale = 1.0f / cw.w16_scale;
    for (int ph = 0; ph < cw.nphase; ++ph) {
        p.ph_oy[ph] = cw.ph_oy[ph]; p.ph_ox[ph] = cw.ph_ox[ph];
        for (int t = 0; t < cw.ntaps; ++t) { p.dy[ph][t] = cw.dy[ph][t]; p.dx[ph][t] = cw.dx[ph][t]; }
    }
    p.ksplit = 1;                                    // the epilogues' "split-K through a workspace / atomics" modes are not used here
    p.ws = nullptr;
    p.stats = a.out.stats; p.stats_ld = a.out.stats_ld;
    p.stats_rep = std::max(1, a.out.stats_rep); p.stats_rep_stride = a.out.stats_rep_stride;
    static const bool dbg_env = getenv("THA4_HALO_DEBUG") != nullptr;
    if (dbg_env) {
        if (!g_dbg_buf) { THA4_CUDA_CHECK(cudaMalloc(&g_dbg_buf, 32 * 32 * sizeof(long long))); }
        THA4_CUDA_CHECK(cudaMemsetAsync(g_dbg_buf, 0, 32 * 32 * sizeof(long long), s));
        p.dbg = g_dbg_buf;
    }
    ProfScope prof(PROF_CONV, s);
    prof_add_work(PROF_CONV, 2.0 * (double)p.N * p.MH * p.MW * cw.cout * (cw.cin * cw.ntaps * cw.nphase + cw.cin2), 0.0);
    const CUtensorMap& ma = halo_activation_map(a.in, op, cw.nphase == 1 ? pl.wg : 1);
    const CUtensorMap& mb = halo_weight_map(cw, pl.bn, op);
    const CUtensorMap* mo32 = &ma;                   // placeholders when an output does not leave through TMA
    const CUtensorMap* mo16 = &ma;
    const CUtensorMap* mr = &ma;
    const CUtensorMap* ma2 = &ma;
    const CUtensorMap* mb2 = &mb;
    if (cw.cin2 > 0) {                               // the folded skip: its input's halo and the weight segment after the taps
        ConvWeights seg = cw;
        seg.w16 = cw.w16b; seg.cin_pad = cw.cin2_pad; seg.ntaps = 1;
        ma2 = &halo_activation_map(a.in2, op, pl.wg);
        mb2 = &halo_weight_map(seg, pl.bn, op);
        p.acc_scale = 1.0f / cw.w16b_scale;
        p.acc_rescale = cw.w16b_scale / cw.w16_scale;
    }
    p.st_tma = halo_st_tma(cw, a, pl, &mo32, &mo16, &mr);
    p.vec4 = ((!cw.bias || (reinterpret_cast<uintptr_t>(cw.bias) & 15) == 0) &&
              (!a.res.p || ((reinterpret_cast<uintptr_t>(a.res.p) & 15) == 0 && a.res.ld % 4 == 0))) ? 1 : 0;
    dim3 grid(pl.tiles_m, pl.tiles_n, pl.cs);
    const HaloMaps m{&ma, &mb, mo32, mo16, mr, ma2, mb2};
    if (cw.cin2 > 0) {
        if (op == OP_F16) launch_halo_bn<OP_F16, 1, 1>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
        else launch_halo_bn<OP_F16N, 1, 1>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
    } else if (cw.nphase == 4) {
        // OP_F16 (conv_halo_supported).  One CTA per SM: the ring takes two halo stages and a whole chunk of weight tiles;
        // two: see halo2_sb
        constexpr int SA2 = halo2_sa(OP_F16, 4), SB2 = halo2_sb(OP_F16, 4);
        if (pl.ctas == 2) {
            if (a.nin.on) launch_halo<OP_F16, 32, SA2, SB2, 1, 1, 2, 4, 2>(m, p, grid, s);
            else launch_halo<OP_F16, 32, SA2, SB2, 1, 0, 2, 4, 2>(m, p, grid, s);
        } else if (pl.cs == 2) {         // a row-owning pair: the one-CTA-per-SM rings
            THA4_REQUIRE(pl.chunks >= 2, "conv_halo: a row-owning pair needs a channel chunk per rank");
            if (a.nin.on) launch_halo<OP_F16, 32, 2, 16, 2, 1, 2, 4>(m, p, grid, s);
            else launch_halo<OP_F16, 32, 2, 16, 2, 0, 2, 4>(m, p, grid, s);
        } else if (a.nin.on) launch_halo<OP_F16, 32, 2, 16, 1, 1, 2, 4>(m, p, grid, s);
        else launch_halo<OP_F16, 32, 2, 16, 1, 0, 2, 4>(m, p, grid, s);
    } else if (op == OP_F16) {
        if (a.nin.on) launch_halo_bn<OP_F16, 1>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
        else launch_halo_bn<OP_F16, 0>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
    } else {
        if (a.nin.on) launch_halo_bn<OP_F16N, 1>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
        else launch_halo_bn<OP_F16N, 0>(pl.bn, pl.cs, pl.wg, pl.ctas, m, p, grid, s);
    }
    static const bool dbg_all = dbg_env && !strcmp(getenv("THA4_HALO_DEBUG"), "2");
    if (dbg_all) {       // developer: stamps of every launch of a real forward (serialises the stream)
        fprintf(stderr, "halo launch: N %d %dx%d cin %d cout %d | bn %d cs %d wg %d chunks %d grid %d x %d | xf %d groups %d act %d res %d out32 %d out16 %d st_tma %d | phases %d ctas %d | cin2 %d\n",
                p.N, p.MH, p.MW, cw.cin, cw.cout, pl.bn, pl.cs, pl.wg, pl.chunks, pl.tiles_m, pl.tiles_n, a.nin.on ? 1 : 0, p.xf_groups, p.xf_act,
                p.res_mode, p.out ? 1 : 0, p.out16 ? 1 : 0, p.st_tma, cw.nphase, pl.ctas, cw.cin2);
        conv_halo_debug_dump();
    }
}

// developer helper: prints the phase stamps of the last launch (THA4_HALO_DEBUG=1)
void conv_halo_debug_dump() {
    if (!g_dbg_buf) return;
    std::vector<long long> h(32 * 32);
    THA4_CUDA_CHECK(cudaDeviceSynchronize());
    THA4_CUDA_CHECK(cudaMemcpy(h.data(), g_dbg_buf, h.size() * sizeof(long long), cudaMemcpyDeviceToHost));
    for (int c = 0; c < 32; ++c) {
        const long long* d = h.data() + c * 32;
        if (!d[0]) continue;
        auto rel = [&](long long v) { return v ? (long)(v - d[0]) : -1L; };
        fprintf(stderr, "halo slot %2d: init %ld pdl %ld | coef %ld a_full %ld xf_done %ld | mma_first %ld mma_commit %ld | t_full %ld epi_done %ld | bar_A %ld pushed+bar_B %ld (loads issued %ld stored %ld) reduce_done %ld | end %ld\n",
                c, rel(d[1]), rel(d[2]), rel(d[16]), rel(d[17]), rel(d[18]), rel(d[8]), rel(d[9]), rel(d[19]), rel(d[20]), rel(d[21]), rel(d[23]), rel(d[25]), rel(d[24]), rel(d[22]), rel(d[3]));
    }
}

}  // namespace tha4
