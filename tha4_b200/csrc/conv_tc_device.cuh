// Device-side pieces shared by the wgmma convolution kernels (conv_tc.cu: one TMA box per tap; conv_halo.cu: one halo box
// per channel chunk, taps as row-shifted descriptors): launch parameters, operand formats, the register accumulator of the
// consumer warpgroup, and the three epilogues (direct accumulator -> global; cluster split-K: accumulator -> the owners'
// shared-memory partials, then the DSMEM reduction).
// TW: pixels per tile row of the 128-pixel CTA tile (16 x 8 tiles: 16; 8 x 16 tiles: 8); row r of the accumulator is
// pixel (y0 + r / TW, x0 + r % TW).
#pragma once
#include "conv.cuh"
#include "tc_common.cuh"

namespace tha4 {
namespace tcdev {

using namespace tc;



constexpr int TILE_W = 16, TILE_H = 8;          // 128 output pixels per CTA
constexpr int TC_THREADS = 160;                  // warps 0-3: the consumer warpgroup (operand transform, wgmma, epilogue), warp 4: TMA producer
constexpr int TC_PRODUCER_WARP = 4;

// The 128 x BN fp32 accumulator of a CTA tile, in the registers of the consumer warpgroup: two m64 halves (rows 0-63, 64-127).
template <int BN> struct Acc { float d[2][BN / 2]; };

// Named barrier of one consumer warpgroup.  WG: consumer warpgroups of the CTA; warpgroup wg synchronises on barrier 1 + wg
// (barrier 3 spans all consumer threads of a two-warpgroup CTA).
template <int WG>
__device__ __forceinline__ void wg_bar(int wg) {
    if (WG == 1 || wg == 0) asm volatile("bar.sync 1, 128;\n" ::: "memory");       // immediate ids: ptxas reserves
    else asm volatile("bar.sync 2, 128;\n" ::: "memory");                         // all 16 barriers for a register id
}

// Columns [c0, c0 + 32) of the accumulator, transposed through `stage` ([128][33] floats) so that thread t receives the 32
// values of tile row t (the row-per-thread layout the epilogues are written for).  Called by all 128 threads of consumer
// warpgroup wg with the same c0 (a constant after unrolling: the accumulator stays in registers); t: the thread's index in
// its warpgroup.
template <int BN, int WG = 1>
__device__ __forceinline__ void acc_rows32(const Acc<BN>& acc, int c0, float* stage, uint32_t (&r)[32], int t, int wg) {
    const int w = t >> 5, l = t & 31;
    wg_bar<WG>(wg);                                              // earlier readers of the stage are done
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int g = c0 / 8 + j;
            const int col = 8 * j + 2 * (l & 3), row = h * 64 + w * 16 + (l >> 2);
            stage[row * 33 + col] = acc.d[h][4 * g];             stage[row * 33 + col + 1] = acc.d[h][4 * g + 1];
            stage[(row + 8) * 33 + col] = acc.d[h][4 * g + 2];   stage[(row + 8) * 33 + col + 1] = acc.d[h][4 * g + 3];
        }
    wg_bar<WG>(wg);
#pragma unroll
    for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(stage[t * 33 + j]);
}

struct TcParams {
    float* out; int outH, outW, outC, out_ld;
    const float* bias;
    const float* res; int resH, resW, res_ld, res_mode;
    int N, MH, MW, tiles_x, tiles_y;
    int ntaps, cpt, ksplit, out_mul, in_mul;       // in_mul: input stride (2 for the 4x4 stride-2 conv: element-strided TMA boxes)
    int pre_b;                                     // weight tiles may be fetched before the programmatic-dependency wait
    float acc_scale;                               // accumulator scale (undoes the power-of-two normalisation of the f16 weights)
    float* ws; long ws_rows; int ws_ld;            // split-K partials: ws[z][tile*128 + row][cout_pad]
    double* stats; int stats_ld; int stats_rep; long stats_rep_stride;   // per-(n,c) sum / sum-of-squares of the output (optional)
    long long* dbg;                                // developer option: per-phase clock64 stamps of a few CTAs (conv_halo.cu), else null
    int st_tma;                                    // unsplit epilogue: bit 0 / bit 1 = the fp32 / f16 output tile leaves through a TMA store (conv_halo.cu)
    int vec4;                                      // bias / residual rows may be read as float4 (16-byte aligned, ld % 4 == 0)
    __half* out16; int out16_ld;                   // optional f16 copy of the output (the operand format of a consumer conv); out may be null then
    // ---- fused input normalisation (XF kernels): the A operand is the RAW f16 output of the producing conv; its pending
    // InstanceNorm / GroupNorm (+FiLM) affine and activation are applied in shared memory between TMA and wgmma
    const double* in_stats; int in_stats_ld, in_stats_rep; long in_stats_rep_stride;
    int inH, inW, inC;                             // geometry of the input tensor (zero padding must stay zero; statistics count)
    int xf_C;                                      // channels [0, xf_C) are normalised, the rest (pose planes, padding) pass through
    int xf_groups, xf_act;                         // 0: InstanceNorm (one group per channel); activation (ACT_*)
    double xf_inv_cnt;                             // 1 / (inH * inW * channels per group), from the host
    const float* xf_gamma; const float* xf_beta; const float* xf_film0; const float* xf_film1; int xf_film1_ld;
    signed char dy[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char dx[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char ph_oy[CONV_MAX_PHASES], ph_ox[CONV_MAX_PHASES];
    int cpt2;                                      // conv_halo.cu: channel chunks of a folded 1x1 skip's input (after the cpt 3x3 chunks)
    float acc_rescale;                             // conv_halo.cu, folded skip: power of two that takes the 3x3 chunks' sum to the skip weights' scale
};

// CS > 1: the K dimension is split over a thread-block cluster of CS CTAs (cluster dims {1,1,CS} along blockIdx.z); the
// partial accumulators are exchanged through distributed shared memory and every CTA finishes 1/CS of the columns.
// OP selects the operand format of one k-block (one TMA box row per pixel / per cout):
//   OP_TF32: 32 fp32 channels  = 128-byte rows, SWIZZLE_128B, kind::tf32 (4 MMAs of K = 8)
//   OP_F16 : 64 f16 channels   = 128-byte rows, SWIZZLE_128B, kind::f16  (4 MMAs of K = 16)
//   OP_F16N: 32 f16 channels   =  64-byte rows, SWIZZLE_64B,  kind::f16  (2 MMAs of K = 16)  -- Cin % 64 == 32 layers
// f16 operands carry the same 10-bit mantissa as TF32 (the normalisation kernels that produce conv inputs write them),
// so the products are as exact as the TF32 path's while every operand byte count -- HBM, L2 -> smem, smem -> tensor
// core -- is halved, and the tensor pipe runs at twice the TF32 rate.
enum { OP_TF32 = 0, OP_F16 = 1, OP_F16N = 2 };
__host__ __device__ constexpr int op_row_bytes(int op) { return op == OP_F16N ? 64 : 128; }
__host__ __device__ constexpr int op_kch(int op) { return op == OP_TF32 ? 32 : (op == OP_F16 ? 64 : 32); }   // channels per k-block
__host__ __device__ constexpr int op_stages(int op, int stages) { return op == OP_F16N ? 2 * stages : stages; }


// ===== fused input normalisation (XF kernels) =====
// Per-channel affine of sample n's pending normalisation, as packed halves (the operand is f16; HFMA2 / tanh.approx.f16x2
// keep the in-place pass cheap).  Called by the NT consumer threads (te = 0..NT-1), which synchronise on named barrier BAR;
// chs: scratch [xf_C] double2.
// [c_lo, c_hi): the channels this CTA will transform (its K chunks); widened to whole normalisation groups.  A cluster
// split-K CTA builds 1 / CS of the table (the fold of the statistic replicas is the expensive part).
template <int NT = 128, int BAR = 1>
__device__ __forceinline__ void xf_build_coef(const TcParams& p, int n, int te, __half* hA, __half* hB, double2* chs, int c_lo, int c_hi) {
    const int cpg = p.xf_groups == 0 ? 1 : p.xf_C / p.xf_groups;
    c_lo = (c_lo / cpg) * cpg;
    c_hi = min(p.xf_C, ((c_hi + cpg - 1) / cpg) * cpg);
    // The layer constants of this thread's first channel are requested BEFORE the statistics: with the loads behind the
    // barrier below, the table cost three dependent L2 round trips (replicas 0-7, replicas 8-15, constants) in every XF
    // CTA's start-up; now one.
    const int c1 = c_lo + te;
    const bool h1 = c1 < c_hi;
    const float* f1p = p.xf_film1 ? p.xf_film1 + (long)n * p.xf_film1_ld : nullptr;
    const float g1 = h1 ? __ldg(p.xf_gamma + c1) : 0.0f, b1 = h1 ? __ldg(p.xf_beta + c1) : 0.0f;
    const float f0s = (h1 && p.xf_film0) ? __ldg(p.xf_film0 + c1) : 0.0f, f0h = (h1 && p.xf_film0) ? __ldg(p.xf_film0 + p.xf_C + c1) : 0.0f;
    const float f1s = (h1 && f1p) ? __ldg(f1p + c1) : 0.0f, f1h = (h1 && f1p) ? __ldg(f1p + p.xf_C + c1) : 0.0f;
    for (int c = c_lo + te; c < c_hi; c += NT)
        chs[c] = fold_stat_replicas16(p.in_stats + ((long)n * p.in_stats_ld + c) * 2, p.in_stats_rep_stride, p.in_stats_rep);
    asm volatile("bar.sync %0, %1;\n" :: "n"(BAR), "n"(NT) : "memory");
    const bool silu = p.xf_act == ACT_SILU || p.xf_act == ACT_SILU_FAST;
    for (int c = c_lo + te; c < c_hi; c += NT) {
        const int g0 = (c / cpg) * cpg;
        double su = 0.0, sq = 0.0;
        for (int j = 0; j < cpg; ++j) { const double2 v = chs[g0 + j]; su += v.x; sq += v.y; }
        // fp64 only where it matters (the sums and the cancelling subtraction): the divisions and the square root of the
        // first version were a dependent chain of ~100 double-precision instructions per channel -- 3 600 cycles per 128
        // channels of every fused-normalisation CTA's start-up (the coefficient is rounded to fp16 anyway)
        const double mean = su * p.xf_inv_cnt;
        const double vard = fma(sq, p.xf_inv_cnt, -mean * mean);
        const float var = fmaxf((float)vard, 0.0f);
        const bool pre = c == c1;
        float A = rsqrtf(var + 1e-5f) * (pre ? g1 : __ldg(p.xf_gamma + c));
        float B = (pre ? b1 : __ldg(p.xf_beta + c)) - (float)mean * A;
        if (p.xf_film0) { const float sc = 1.0f + (pre ? f0s : __ldg(p.xf_film0 + c)), sh = pre ? f0h : __ldg(p.xf_film0 + p.xf_C + c); A *= sc; B = B * sc + sh; }
        if (f1p) { const float sc = 1.0f + (pre ? f1s : __ldg(f1p + c)), sh = pre ? f1h : __ldg(f1p + p.xf_C + c); A *= sc; B = B * sc + sh; }
        if (silu) { A *= 0.5f; B *= 0.5f; }                      // silu(v) = h + h * tanh(h) with h = v / 2
        hA[c] = __float2half_rn(fminf(fmaxf(A, -65504.0f), 65504.0f)); hB[c] = __float2half_rn(fminf(fmaxf(B, -65504.0f), 65504.0f));
    }
    asm volatile("bar.sync %0, %1;\n" :: "n"(BAR), "n"(NT) : "memory");
}

// NC consecutive 16-byte chunks (8 channels each, logical chunk index j0 .. j0 + NC) of one operand row normalised +
// activated in place.  swz: the row's XOR term of the TMA / UMMA swizzle; c0: the channel of logical chunk 0.
// ALL chunks are loaded before the first is transformed and stored after the last: with one load -> transform -> store per
// chunk the compiler must keep the shared-memory accesses in program order (it cannot prove that the store of chunk j and the
// load of chunk j + 1 do not alias), which made the stage one dependent ~200-cycle chain per chunk on a single warp per
// scheduler .
template <int NC>
__device__ __forceinline__ void xf_chunks(uint8_t* rowp, int swz, int j0, int c0, const TcParams& p, const __half* hA, const __half* hB, bool silu) {
    uint4 d[NC];
#pragma unroll
    for (int j = 0; j < NC; ++j) d[j] = *reinterpret_cast<const uint4*>(rowp + (((j0 + j) ^ swz) << 4));
    const bool relu = p.xf_act == ACT_RELU;
#pragma unroll
    for (int j = 0; j < NC; ++j) {
        const int cb = c0 + (j0 + j) * 8;
        if (cb >= p.xf_C) continue;                      // pass-through channels (pose planes, padding)
        const uint4 a4 = *reinterpret_cast<const uint4*>(hA + cb), b4 = *reinterpret_cast<const uint4*>(hB + cb);
        __half2* x2 = reinterpret_cast<__half2*>(&d[j]);
        const __half2* a2 = reinterpret_cast<const __half2*>(&a4);
        const __half2* b2 = reinterpret_cast<const __half2*>(&b4);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            __half2 h = __hfma2(x2[e], a2[e], b2[e]);
            if (silu) {
                uint32_t hu = *reinterpret_cast<uint32_t*>(&h), tu;
                asm("tanh.approx.f16x2 %0, %1;\n" : "=r"(tu) : "r"(hu));
                h = __hfma2(h, *reinterpret_cast<__half2*>(&tu), h);
            } else if (relu) {
                h = __hmax2(h, __float2half2_rn(0.0f));
            }
            x2[e] = h;
        }
    }
#pragma unroll
    for (int j = 0; j < NC; ++j)
        if (c0 + (j0 + j) * 8 < p.xf_C) *reinterpret_cast<uint4*>(rowp + (((j0 + j) ^ swz) << 4)) = d[j];
}
// whole row
template <int ROWB>
__device__ __forceinline__ void xf_row(uint8_t* rowp, int swz, int c0, const TcParams& p, const __half* hA, const __half* hB, bool silu) {
    xf_chunks<ROWB / 16>(rowp, swz, 0, c0, p, hA, hB, silu);
}

// ===== cluster split-K, step 1 (consumer warpgroup, after a cluster barrier that says every peer's accumulator is complete
// and its pipeline buffers are idle): registers -> the OWNER's shared memory.  Rank r of the cluster finishes columns
// [r * SL, (r + 1) * SL); every CTA PUSHES the slice of its partial that belongs to rank r into slot [sender] of rank r's
// buffer with st.shared::cluster (posted stores).
// Buffer of a CTA: [CS slots][128 rows x SC 16-byte chunks], chunk index L = row * SC + cc stored at L ^ ((L >> 3) & 7)
// (readers -- lanes = consecutive L -- spread over the banks).
template <int BN, int CS>
__device__ __forceinline__ void epi_push_partial(const Acc<BN>& acc, uint8_t* smem, int split, int warp, int lane) {
    constexpr int SL = BN / CS, SC = SL / 4;
    constexpr uint32_t SLOT_BYTES = 128u * SL * 4u;
    const uint32_t base = smem_u32(smem) + (uint32_t)split * SLOT_BYTES;       // slot [sender = this rank] in every owner's buffer
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int g = 0; g < BN / 8; ++g)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int row = h * 64 + warp * 16 + (lane >> 2) + 8 * e;
                const int col = 8 * g + 2 * (lane & 3);
                const int chunk = col >> 2;
                const int owner = chunk / SC, cc = chunk - owner * SC;
                const uint32_t L = (uint32_t)(row * SC + cc);
                const uint32_t addr = base + ((L ^ ((L >> 3) & 7u)) << 4) + (uint32_t)(col & 3) * 4u;
                const float v0 = acc.d[h][4 * g + 2 * e], v1 = acc.d[h][4 * g + 2 * e + 1];
                if (owner == split) {
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" :: "r"(addr), "f"(v0), "f"(v1) : "memory");
                } else {
                    uint32_t remote;
                    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(remote) : "r"(addr), "r"(owner));
                    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};\n" :: "r"(remote), "f"(v0), "f"(v1) : "memory");
                }
            }
}

// ===== unsplit / workspace split-K epilogue (consumer warpgroup): registers -> global (+ statistics) =====
// NSLOT > 0 (and p.st_tma): the finished 128 x 32 tile of each column step is staged in shared memory in the swizzled box
// layout and written by ONE TMA store per output (fp32 / f16) instead of 12 warp-wide stores whose 32 lanes hit 32 different
// lines (32 L1 wavefronts per instruction).  TMA
// clips what lies outside the tensor (partial tiles, channel tails).  Slots live behind the statistics scratch in the idle
// pipeline buffers; a slot is rewritten only after its store has read it (bulk-group wait).
constexpr int EPI_SLOT_BYTES = 128 * 128 + 128 * 64;           // fp32 stage (128-byte rows) + f16 stage (64-byte rows)
__host__ __device__ constexpr int epi_slot0(int bn) { return (4 * 32 * 33 * 4 + 4 * bn * 8 + 1023) & ~1023; }
__host__ __device__ constexpr int epi_nslot(int bn, size_t ring) {
    return ring < (size_t)epi_slot0(bn) + EPI_SLOT_BYTES ? 0
         : ((int)((ring - epi_slot0(bn)) / EPI_SLOT_BYTES) < bn / 32 ? (int)((ring - epi_slot0(bn)) / EPI_SLOT_BYTES) : bn / 32);
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n"
                 :: "l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// WG == 2 (conv_halo.cu's 256-pixel tiles): each consumer warpgroup wg runs this on its own 128 rows, with its own named
// barrier, its own shared-memory region `smem` (warpgroup 1's starts wg_bytes after warpgroup 0's) and its own residual
// barriers; y0 is the first pixel row of the warpgroup's rows.  FOLD: the two warpgroups' channel sums are folded in shared
// memory before the fp64 atomics, one pair per (CTA, channel); without it (a CTA in which only one warpgroup runs the
// epilogue) each warpgroup commits the sums of its own rows.
template <int BN, int TW, int NSLOT = 0, int WG = 1, bool FOLD = true>
__device__ __forceinline__ void epi_direct(const TcParams& p, const Acc<BN>& acc, uint8_t* smem, int n, int y0, int x0,
                                           int n0, int phase, int split, int warp, int lane,
                                           const CUtensorMap* tm32 = nullptr, const CUtensorMap* tm16 = nullptr,
                                           const CUtensorMap* tmR = nullptr, uint64_t* res_bars = nullptr,
                                           int wg = 0, int wg_bytes = 0) {
    static_assert(WG == 1 || WG == 2, "one or two consumer warpgroups");
    const int q = warp & 3;
    const int t = WG == 1 ? (int)threadIdx.x : (int)threadIdx.x & 127;     // index in the warpgroup
    const bool rows_in = WG == 1 || y0 < p.MH;                             // a second warpgroup's rows may all lie below the image
    // p.st_tma bit 2: the residual tile (same geometry as the fp32 output) ARRIVES by TMA as well, into the fp32 stage of
    // the slot it will leave from: 8 conflict-free LDS.128 per thread instead of 8 LDG.128 whose lanes hit 32 different lines
    const bool res_tma = NSLOT > 0 && (p.st_tma & 4) != 0;
    const int nsteps = min(BN / 32, (p.outC - n0 + 31) / 32);
    if (res_tma && t == 0) {
        for (int s = 0; s < NSLOT && s < nsteps; ++s) {
            const uint32_t bar = smem_u32(res_bars + s);
            mbar_expect_tx(bar, 128 * 128);
            tma_load_4d(smem_u32(smem + epi_slot0(BN) + s * EPI_SLOT_BYTES), tmR, n0 + s * 32, x0, y0, n, bar);
        }
    }
    const int row = q * 32 + lane;
    const bool lead = (split == 0);
    float* scratch = reinterpret_cast<float*>(smem) + q * (32 * 33);   // pipeline smem is idle once the last wgmma retired
    const int my = y0 + row / TW, mx = x0 + row % TW;
    const bool valid = my < p.MH && mx < p.MW;
    const int oy = my * p.out_mul + p.ph_oy[phase], ox = mx * p.out_mul + p.ph_ox[phase];
    const long opix = ((long)n * p.outH + oy) * p.outW + ox;
    float* orow = p.out + opix * p.out_ld;
    const int st_tma = NSLOT > 0 ? p.st_tma : 0;
    int step = 0;
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += 32) {
        uint32_t r[32];
        acc_rows32<BN, WG>(acc, c0, reinterpret_cast<float*>(smem), r, t, wg);    // the stage is the statistics scratch: row t at t * 33
        const int cbase = n0 + c0;
        if (cbase >= p.outC) continue;                         // warp-uniform
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]) * p.acc_scale;
        const int cn = min(32, p.outC - cbase);
        const bool to_ws = p.ksplit > 1 && p.ws;
        if (valid) {
            if (lead && !to_ws) {
                const bool v4 = p.vec4 && cn == 32;
                if (p.bias) {
                    if (v4) {
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + cbase + j));
                            v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < cn) v[j] += __ldg(p.bias + cbase + j);
                    }
                }
                if (res_tma) {
                    // added from the staged tile below
                } else if (p.res_mode == RES_SAME || p.res_mode == RES_UP2) {
                    const int ry = p.res_mode == RES_UP2 ? (oy >> 1) : oy, rx = p.res_mode == RES_UP2 ? (ox >> 1) : ox;
                    const float* rr = p.res + (((long)n * p.resH + ry) * p.resW + rx) * p.res_ld + cbase;
                    if (v4) {       // 8 requests of 32 sectors instead of 32 requests of 32 sectors
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            const float4 b = *reinterpret_cast<const float4*>(rr + j);
                            v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < cn) v[j] += rr[j];
                    }
                } else if (p.res_mode == RES_DOWN2) {
                    const float* rr = p.res + (((long)n * p.resH + 2 * oy) * p.resW + 2 * ox) * p.res_ld + cbase;
                    const long dx1 = p.res_ld, dy1 = (long)p.resW * p.res_ld;
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        if (j < cn) v[j] += 0.25f * ((rr[j] + rr[dx1 + j]) + (rr[dy1 + j] + rr[dy1 + dx1 + j]));
                }
            }
            if (to_ws) {
                float* wrow = p.ws + ((long)blockIdx.z * p.ws_rows + (long)blockIdx.x * 128 + row) * p.ws_ld + cbase;
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                    *reinterpret_cast<float4*>(wrow + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            } else if (p.ksplit > 1) {
#pragma unroll
                for (int j = 0; j < 32; ++j) if (j < cn) atomicAdd(orow + cbase + j, v[j]);
            } else {
                if (p.out && !(st_tma & 1)) {
                    if (cn == 32) {
#pragma unroll
                        for (int j = 0; j < 32; j += 4)
                            *reinterpret_cast<float4*>(orow + cbase + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < cn) orow[cbase + j] = v[j];
                    }
                }
                if (p.out16 && !(st_tma & 2)) {          // f16 copy: the operand a consumer conv loads by TMA (raw value; its norm is applied there)
                    __half* hrow = p.out16 + opix * p.out16_ld + cbase;
                    if (cn == 32) {
#pragma unroll
                        for (int j = 0; j < 32; j += 8) {
                            uint4 pk;
                            __half2* h2 = reinterpret_cast<__half2*>(&pk);
                            h2[0] = __floats2half2_rn(v[j], v[j + 1]); h2[1] = __floats2half2_rn(v[j + 2], v[j + 3]);
                            h2[2] = __floats2half2_rn(v[j + 4], v[j + 5]); h2[3] = __floats2half2_rn(v[j + 6], v[j + 7]);
                            *reinterpret_cast<uint4*>(hrow + j) = pk;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (j < cn) hrow[j] = __float2half_rn(v[j]);
                    }
                }
            }
        }
        if (NSLOT > 0 && st_tma) {
            // every row is staged (rows outside the image hold values of zero-padded inputs; the store clips them)
            if (step >= NSLOT && !res_tma) {
                if (t == 0) asm volatile("cp.async.bulk.wait_group.read %0;\n" :: "n"(NSLOT > 0 ? NSLOT - 1 : 0) : "memory");
                wg_bar<WG>(wg);
            }
            uint8_t* slot = smem + epi_slot0(BN) + (NSLOT > 0 ? step % NSLOT : 0) * EPI_SLOT_BYTES;
            if (res_tma) {
                // the residual of this step has landed (its load was issued once the slot's previous stores had been read)
                mbar_wait(smem_u32(res_bars + (NSLOT > 0 ? step % NSLOT : 0)), (uint32_t)((NSLOT > 0 ? step / NSLOT : 0) & 1));
                const uint8_t* rp = slot + row * 128;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float4 t = *reinterpret_cast<const float4*>(rp + ((j ^ (row & 7)) << 4));
                    v[4 * j] += t.x; v[4 * j + 1] += t.y; v[4 * j + 2] += t.z; v[4 * j + 3] += t.w;
                }
            }
            if (st_tma & 1) {
                uint8_t* rp = slot + row * 128;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    *reinterpret_cast<float4*>(rp + ((j ^ (row & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
            if (st_tma & 2) {
                uint8_t* rp = slot + 128 * 128 + row * 64;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    uint4 pk;
                    __half2* h2 = reinterpret_cast<__half2*>(&pk);
                    h2[0] = __floats2half2_rn(v[8 * j], v[8 * j + 1]); h2[1] = __floats2half2_rn(v[8 * j + 2], v[8 * j + 3]);
                    h2[2] = __floats2half2_rn(v[8 * j + 4], v[8 * j + 5]); h2[3] = __floats2half2_rn(v[8 * j + 6], v[8 * j + 7]);
                    *reinterpret_cast<uint4*>(rp + ((j ^ ((row >> 1) & 3)) << 4)) = pk;
                }
            }
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
            wg_bar<WG>(wg);
            if (t == 0) {
                if ((st_tma & 1) && rows_in) tma_store_4d(tm32, smem_u32(slot), cbase, x0, y0, n);
                if ((st_tma & 2) && rows_in) tma_store_4d(tm16, smem_u32(slot + 128 * 128), cbase, x0, y0, n);
                asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
                if (res_tma && step + NSLOT < nsteps) {      // refill the slot with the residual of the step that will use it next
                    asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory");
                    const uint32_t bar = smem_u32(res_bars + (NSLOT > 0 ? step % NSLOT : 0));
                    mbar_expect_tx(bar, 128 * 128);
                    tma_load_4d(smem_u32(slot), tmR, n0 + (step + NSLOT) * 32, x0, y0, n, bar);
                }
            }
            ++step;
        }
        if (p.stats && p.ksplit == 1) {
            // per-channel sum / sum of squares over this warp's 32 pixels: transpose through shared memory,
            // then lane j reduces channel j; one double atomic pair per (warp, channel).
#pragma unroll
            for (int j = 0; j < 32; ++j) scratch[lane * 33 + j] = valid ? v[j] : 0.0f;
            __syncwarp();
            float su = 0.0f, sq = 0.0f;
#pragma unroll 8
            for (int rr = 0; rr < 32; ++rr) { const float t = scratch[rr * 33 + lane]; su += t; sq += t * t; }
            __syncwarp();
            float2* part = reinterpret_cast<float2*>(reinterpret_cast<float*>(smem) + 4 * 32 * 33);   // [4 warps][BN]
            part[q * BN + c0 + lane] = make_float2(su, sq);
        }
    }
    if (p.stats && p.ksplit == 1) {
        // combine the warps' partial sums: one double atomic pair per (tile, channel), spread over replicas
        constexpr bool FOLD2 = WG == 2 && FOLD;
        if constexpr (WG == 1) asm volatile("bar.sync 1, 128;\n" ::: "memory");
        else if constexpr (FOLD2) asm volatile("bar.sync 3, 256;\n" ::: "memory");   // both warpgroups' partials are written
        else wg_bar<WG>(wg);
        const float2* part = reinterpret_cast<const float2*>(reinterpret_cast<float*>(smem - (FOLD2 ? wg * wg_bytes : 0)) + 4 * 32 * 33);
        double* base = p.stats + (long)(blockIdx.x % p.stats_rep) * p.stats_rep_stride + ((long)n * p.stats_ld + n0) * 2;
        for (int c = FOLD2 ? (int)threadIdx.x : t; c < BN; c += FOLD2 ? 128 * WG : 128) {
            if (n0 + c >= p.outC) break;
            const float2 a = part[c], b = part[BN + c], cc = part[2 * BN + c], d = part[3 * BN + c];
            if constexpr (!FOLD2) {
                atomicAdd(base + 2 * c, (double)a.x + (double)b.x + (double)cc.x + (double)d.x);
                atomicAdd(base + 2 * c + 1, (double)a.y + (double)b.y + (double)cc.y + (double)d.y);
            } else {
                const float2* part1 = part + wg_bytes / (int)sizeof(float2);
                const float2 e = part1[c], f = part1[BN + c], g = part1[2 * BN + c], h = part1[3 * BN + c];
                atomicAdd(base + 2 * c, (double)a.x + (double)b.x + (double)cc.x + (double)d.x + (double)e.x + (double)f.x + (double)g.x + (double)h.x);
                atomicAdd(base + 2 * c + 1, (double)a.y + (double)b.y + (double)cc.y + (double)d.y + (double)e.y + (double)f.y + (double)g.y + (double)h.y);
            }
        }
    }
    if (NSLOT > 0 && st_tma && t == 0) asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory");   // the staging slots have been read before the CTA retires (the writes themselves complete with the grid)
}

// ===== cluster split-K, step 2 (consumer warpgroup, after the cluster barrier that publishes the pushes): sum the CS slots of this
// CTA's column slice from its own shared memory, finish the columns =====
template <int BN, int CS, int TW>
__device__ __forceinline__ void epi_cluster_reduce(const TcParams& p, uint8_t* smem, int n, int y0, int x0, int n0, int phase, int split, int warp,
                                                   long long* dbg = nullptr) {
    constexpr int SL = BN / CS, SC = SL / 4;                   // columns / 16-byte chunks finished by this CTA
    static_assert(SL >= 4 && 128 % SC == 0, "cluster slice");
    const int te = threadIdx.x;                                // 0..127
    const int cc = te % SC;
    const int chunk = split * SC + cc;                         // split == rank in the cluster
    const int col = n0 + chunk * 4;
    const uint32_t p_local = smem_u32(smem);
    float su[4] = {0, 0, 0, 0}, sq[4] = {0, 0, 0, 0};
    // A thread finishes SC rows (rows te / SC + i * 128 / SC), U at a time: the slot reads and the residual rows of a batch
    // are all requested before the first is consumed.
    constexpr int RSTEP = 128 / SC;
    constexpr int U = (SC < (16 / CS > 0 ? 16 / CS : 1)) ? SC : (16 / CS > 0 ? 16 / CS : 1);
    static_assert(SC % U == 0, "cluster reduce: batch");
    const int r0 = te / SC;
    const int cn = max(0, min(4, p.outC - col));
    const bool fast = cn == 4 && p.vec4;                       // 16-byte bias / residual reads
    const bool res_direct = p.res_mode == RES_SAME || p.res_mode == RES_UP2, up2 = p.res_mode == RES_UP2;
    const int poy = p.ph_oy[phase], pox = p.ph_ox[phase];
    float bias4[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (p.bias) for (int j = 0; j < cn; ++j) bias4[j] = __ldg(p.bias + col + j);
#pragma unroll 1
    for (int rb = 0; rb < SC; rb += U) {
        float4 part[U][CS];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int row = r0 + (rb + u) * RSTEP;
            const uint32_t L = (uint32_t)(row * SC + cc);
            const uint32_t off = (L ^ ((L >> 3) & 7u)) << 4;
#pragma unroll
            for (int pr = 0; pr < CS; ++pr)          // slot pr = the partial pushed by rank pr (fixed summation order)
                asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n"
                             : "=f"(part[u][pr].x), "=f"(part[u][pr].y), "=f"(part[u][pr].z), "=f"(part[u][pr].w)
                             : "r"(p_local + (uint32_t)pr * (128u * SL * 4u) + off));
        }
        if (dbg && threadIdx.x == 0 && rb == 0) dbg[3 * 8 + 1] = clock64();
        // the residual rows of the batch are requested up front as well (L2 round trips).  Index arithmetic stays in 32 bits up
        // to the one widening multiply by the row stride: with 64-bit products throughout, this loop was ~250 dependent
        // instructions per row on one warp per scheduler.
        float rres[U][4];
        int opix[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            rres[u][0] = rres[u][1] = rres[u][2] = rres[u][3] = 0.0f;
            const int row = r0 + (rb + u) * RSTEP;
            const int my = y0 + row / TW, mx = x0 + row % TW;
            const int oy = my * p.out_mul + poy, ox = mx * p.out_mul + pox;
            ok[u] = my < p.MH && mx < p.MW && col < p.outC;
            opix[u] = (n * p.outH + oy) * p.outW + ox;
            if (res_direct && ok[u]) {
                const int rpix = up2 ? (n * p.resH + (oy >> 1)) * p.resW + (ox >> 1) : (n * p.resH + oy) * p.resW + ox;
                const float* rr = p.res + (long)rpix * p.res_ld + col;
                if (fast) {
                    const float4 t = *reinterpret_cast<const float4*>(rr);
                    rres[u][0] = t.x; rres[u][1] = t.y; rres[u][2] = t.z; rres[u][3] = t.w;
                } else {
                    for (int j = 0; j < cn; ++j) rres[u][j] = rr[j];
                }
            }
        }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float4 acc = part[u][0];
#pragma unroll
        for (int pr = 1; pr < CS; ++pr) { acc.x += part[u][pr].x; acc.y += part[u][pr].y; acc.z += part[u][pr].z; acc.w += part[u][pr].w; }
        if (!ok[u]) continue;
        float v[4] = {acc.x * p.acc_scale + bias4[0], acc.y * p.acc_scale + bias4[1], acc.z * p.acc_scale + bias4[2], acc.w * p.acc_scale + bias4[3]};
        if (res_direct) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] += rres[u][j];
        } else if (p.res_mode == RES_DOWN2) {
            const int row = r0 + (rb + u) * RSTEP;
            const int oy = (y0 + row / TW) * p.out_mul + poy, ox = (x0 + row % TW) * p.out_mul + pox;
            const float* rr = p.res + (long)((n * p.resH + 2 * oy) * p.resW + 2 * ox) * p.res_ld + col;
            const long dx1 = p.res_ld, dy1 = (long)p.resW * p.res_ld;
            if (fast) {       // four 16-byte loads in flight instead of sixteen dependent scalar ones
                const float4 a = *reinterpret_cast<const float4*>(rr), b = *reinterpret_cast<const float4*>(rr + dx1);
                const float4 c = *reinterpret_cast<const float4*>(rr + dy1), d = *reinterpret_cast<const float4*>(rr + dy1 + dx1);
                v[0] += 0.25f * ((a.x + b.x) + (c.x + d.x)); v[1] += 0.25f * ((a.y + b.y) + (c.y + d.y));
                v[2] += 0.25f * ((a.z + b.z) + (c.z + d.z)); v[3] += 0.25f * ((a.w + b.w) + (c.w + d.w));
            } else {
                for (int j = 0; j < cn; ++j) v[j] += 0.25f * ((rr[j] + rr[dx1 + j]) + (rr[dy1 + j] + rr[dy1 + dx1 + j]));
            }
        }
        if (p.out) {
            float* o = p.out + (long)opix[u] * p.out_ld + col;
            if (cn == 4) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
            else for (int j = 0; j < cn; ++j) o[j] = v[j];
        }
        if (p.out16) {
            __half* o16 = p.out16 + (long)opix[u] * p.out16_ld + col;
            if (cn == 4) {
                uint2 pk;
                __half2* h2 = reinterpret_cast<__half2*>(&pk);
                h2[0] = __floats2half2_rn(v[0], v[1]); h2[1] = __floats2half2_rn(v[2], v[3]);
                *reinterpret_cast<uint2*>(o16) = pk;
            } else for (int j = 0; j < cn; ++j) o16[j] = __float2half_rn(v[j]);
        }
        for (int j = 0; j < cn; ++j) { su[j] += v[j]; sq[j] += v[j] * v[j]; }
      }
    }
    if (dbg && threadIdx.x == 0) dbg[3 * 8 + 0] = clock64();
    if (p.stats) {
        // per-column sums of this CTA's slice: thread te holds partials of chunk te % SC; fold the 128 / SC row
        // threads of each chunk in two short steps (8 floats per thread, then <= 16 doubles per output)
        float* red = reinterpret_cast<float*>(smem) + 128 * BN;          // [128][8], behind the partial tile
#pragma unroll
        for (int k = 0; k < 4; ++k) { red[te * 8 + k] = su[k]; red[te * 8 + 4 + k] = sq[k]; }
        asm volatile("bar.sync 1, 128;\n" ::: "memory");
        constexpr int NOUT = SC * 8;                                     // (chunk, {4 sums, 4 sums of squares})
        double* dbase = p.stats + (long)(blockIdx.x % p.stats_rep) * p.stats_rep_stride + ((long)n * p.stats_ld + n0 + split * SL) * 2;
        if constexpr (NOUT <= 128) {
            constexpr int G = 128 / NOUT;                                // threads per output
            constexpr int PER = 128 / SC / G;                            // entries per thread (= 8)
            float* red2 = red + 128 * 8;                                 // [G][NOUT]
            const int o = te % NOUT, g = te / NOUT;
            const int oc = o >> 3, ok = o & 7;
            float acc = 0.0f;
#pragma unroll
            for (int i = 0; i < PER; ++i) acc += red[(oc + SC * (g * PER + i)) * 8 + ok];
            red2[g * NOUT + o] = acc;
            asm volatile("bar.sync 1, 128;\n" ::: "memory");
            if (te < NOUT) {
                const int c = n0 + split * SL + oc * 4 + (ok & 3);
                if (c < p.outC) {
                    double a = 0.0;
#pragma unroll
                    for (int gg = 0; gg < G; ++gg) a += (double)red2[gg * NOUT + o];
                    atomicAdd(dbase + 2 * (oc * 4 + (ok & 3)) + (ok >> 2), a);
                }
            }
        } else {
            for (int o = te; o < NOUT; o += 128) {
                const int oc = o >> 3, ok = o & 7;
                const int c = n0 + split * SL + oc * 4 + (ok & 3);
                if (c >= p.outC) continue;
                double a = 0.0;
                for (int t2 = oc; t2 < 128; t2 += SC) a += (double)red[t2 * 8 + ok];
                atomicAdd(dbase + 2 * (oc * 4 + (ok & 3)) + (ok >> 2), a);
            }
        }
    }
}

}  // namespace tcdev
}  // namespace tha4
