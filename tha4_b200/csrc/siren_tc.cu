// Distilled student networks on the tensor cores: SirenFaceMorpher00 (siren_face_morpher_00.py:28-51) and the three
// levels of SirenMorpher03 (siren_morpher_03.py:107-139) as persistent fused-MLP kernels on TMA + wgmma.
//
// A CTA walks 128-pixel tiles (128 consecutive pixels of one image row).  The activations of a tile live in shared
// memory as the K-major SWIZZLE_128B A operand ([K / 64 chunks][128 rows][128 B]), in two buffers that swap roles per
// layer (a layer reads one and writes the other); every sine layer is
//   TMA     weight tiles W[NB rows x 64 k] (fp16, pre-scaled by omega_0 = 30) stream through a ring that runs ahead of
//           the math across layers and tiles (the weight sequence of a tile is fixed; warp 4 issues them);
//   wgmma   D[128 x NB] (fp32, registers of the consumer warpgroup, two m64 halves) = A[128 x K] . W^T, N in slices of
//           NB <= 96 columns;
//   drain   each thread adds the bias to its accumulator fragment (+ the per-sample pose bias and the two xy terms on a
//           level's first layer: the tiled pose / position planes of siren_morpher_03.py:92-105 are never materialised),
//           takes sin(.) and writes the result into the other A buffer as fp16 -- the layer's output is the next layer's
//           operand, it never leaves the SM.
// Level hand-off (bilinear x2, :121) goes through fp16 NHWC tensors in HBM (it needs a cross-tile halo); level 2 ends in
// the fused tail: 1x1 head (a 16-column MMA) -> grid_sample -> blend -> five NCHW outputs (thread = pixel: the 32 lanes
// of a warp write 32 consecutive pixels = full 128-byte lines).  The mma.sync kernels of siren.cu remain as the
// reference path of the option "siren_tc" = 0 and for the distillation backward (stored-activation forward).
#include "siren.cuh"
#include "gridsample.cuh"
#include "profiler.cuh"
#include "tc_common.cuh"
#include <cuda.h>
#include <map>
#include <mutex>
#include <tuple>

namespace tha4 {
namespace {

using namespace tc;

constexpr int ST_THREADS = 160;            // warps 0-3: the consumer warpgroup (prologue, wgmma, drain), warp 4: TMA producer
constexpr int ST_TILE = 128;
constexpr int ST_MAXL = 8;                 // GEMM layers per kernel (face: 7 sine + head)
enum { SM_BODY0 = 0, SM_BODY1 = 1, SM_BODY2 = 2, SM_FACE = 3 };

struct StLayer {
    int kpad, npad, nb;                    // K (padded, multiple of 16), N (padded), N slice per MMA / per weight tile
    int sine;                              // 1: sin epilogue into the A operand; 0: linear head (N = 16 columns, raw)
    int bias_off;                          // offset of this layer's bias in the staged bias table (floats)
    int first;                             // 1: add the per-sample bias + xy terms (first layer of body levels 1 / 2)
};
struct StMaps { CUtensorMap w[ST_MAXL]; };

struct StParams {
    int R, B, nl;
    StLayer L[ST_MAXL];
    const float* bias_table; int bias_floats;       // all layers' biases, concatenated (pre-scaled)
    // elementwise first layer (body level 0, face): act = sin(pb[n][c] + wx[c] * x + wy[c] * y), c < e_npad
    int e_npad; const float* e_pb; int e_pb_ld; const float* e_wxy;
    // first GEMM layer of body levels 1 / 2: per-sample bias + xy terms
    const float* f_pb; int f_pb_ld; const float* f_wxy;
    const float* base;                              // affine_grid coordinates of this resolution
    const __half* prev; int prev_c;                 // previous level's output [B, R/2, R/2, prev_c] (bilinear x2 prologue)
    __half* out; int out_c;                         // this level's output [B, R, R, out_c] (levels 0 / 1)
    ImgView image; float* o[5]; int o_f16;          // level 2: tail (o_f16: the five outputs are __half planes, io_dtype = f16)
    float* face_out;                                // face: [B, 4, R, R]
    const float* head_bias;
    // character bank (the BANK instantiations): sample n runs on character char_of[n].  The weight maps are 3-D with the
    // character as the outermost coordinate; bias_table, e_wxy / f_wxy and head_bias point at character 0 and the
    // *_cs members are the floats from one character to the next.
    const int* char_of; int bias_cs, wxy_cs, head_cs;
};

// sin(x) WITHOUT the transcendental unit.  The mma.sync student kernels (siren.cu) and the first version of this file used
// rintf + MUFU.SIN: two XU-pipe operations per output -- and ncu showed the XU pipe, not the tensor pipe, bounding every
// level.  Here: k = round(x / pi) by
// the magic-number trick (FMA pipe), r = x - k pi (two-constant Cody-Waite), sin(r) on [-pi/2, pi/2] as the degree-9
// Taylor polynomial (|error| <= 3.6e-6, far below the fp16 the result is stored in), sign (-1)^k from the parity bit.
// 13 FMA / ALU-pipe instructions, 128 lanes / clk / SM.
__device__ __forceinline__ float st_sin(float x) {
    const float kf = fmaf(x, 0.31830988618379067f, 12582912.0f);          // 1.5 * 2^23: the integer k sits in the low mantissa bits
    const float k = kf - 12582912.0f;
    float r = fmaf(-k, 3.1415927410125732f, x);
    r = fmaf(-k, -8.7422776573475858e-8f, r);
    const float r2 = r * r;
    float p = fmaf(r2, 2.7557319223985893e-6f, -1.9841269841269841e-4f);
    p = fmaf(p, r2, 8.3333333333333332e-3f);
    p = fmaf(p, r2, -1.6666666666666666e-1f);
    const float s = fmaf(p * r2, r, r);
    return __uint_as_float(__float_as_uint(s) ^ ((__float_as_uint(kf) & 1u) << 31));
}

// byte offset of the 16-byte chunk holding channels [c8, c8 + 8) of tile row `row` in the swizzled A operand
__device__ __forceinline__ uint32_t a_off(int row, int c8) {
    const int chunk = c8 >> 6, j = (c8 & 63) >> 3;
    return (uint32_t)(chunk * (ST_TILE * 128) + row * 128 + ((j ^ (row & 7)) << 4));
}

// D (+)= A . W^T for one N slice of width nb (a runtime choice among the widths the plans use), K steps of 16 up to ksteps
template <int NBMAX>
__device__ __forceinline__ void st_slice_mma(float (&d)[2][NBMAX / 2], int nb, uint32_t a_addr, uint32_t b_addr, int ksteps, bool acc_in) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (k >= ksteps) break;
        const uint64_t a0 = make_smem_desc_sw<128>(a_addr + 32 * k), a1 = make_smem_desc_sw<128>(a_addr + 64 * 128 + 32 * k);
        const uint64_t bd = make_smem_desc_sw<128>(b_addr + 32 * k);
        const uint32_t accum = (acc_in || k > 0) ? 1u : 0u;
        if (nb == 16) {
            Wgmma<16>::f16(*reinterpret_cast<float(*)[8]>(&d[0][0]), a0, bd, accum);
            Wgmma<16>::f16(*reinterpret_cast<float(*)[8]>(&d[1][0]), a1, bd, accum);
        } else if (nb == 64 && NBMAX >= 64) {
            Wgmma<(NBMAX >= 64 ? 64 : 16)>::f16(*reinterpret_cast<float(*)[NBMAX >= 64 ? 32 : 8]>(&d[0][0]), a0, bd, accum);
            Wgmma<(NBMAX >= 64 ? 64 : 16)>::f16(*reinterpret_cast<float(*)[NBMAX >= 64 ? 32 : 8]>(&d[1][0]), a1, bd, accum);
        } else if (NBMAX >= 96) {
            Wgmma<(NBMAX >= 96 ? 96 : 16)>::f16(*reinterpret_cast<float(*)[NBMAX >= 96 ? 48 : 8]>(&d[0][0]), a0, bd, accum);
            Wgmma<(NBMAX >= 96 ? 96 : 16)>::f16(*reinterpret_cast<float(*)[NBMAX >= 96 ? 48 : 8]>(&d[1][0]), a1, bd, accum);
        }
    }
    wg_commit();
    wg_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h) wg_fence_acc(d[h]);
}

// BANK: per-sample weights (see StParams::char_of).  A tile is one sample's, so its character selects the weight tiles the
// producer fetches (third TMA coordinate), the biases staged in sbias (re-staged when the CTA's next tile is another
// character's), the first layer's wxy and the head bias; everything else is the one-character kernel.
template <int ACH, int NBMAX, int SB, int MODE, bool BANK>
__global__ void __launch_bounds__(ST_THREADS) siren_tc_kernel(const __grid_constant__ StMaps maps, const StParams p) {
    constexpr int A_BYTES = ACH * ST_TILE * 128;
    constexpr int B_STAGE = NBMAX * 128;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);      // pointer arithmetic (not an integer round trip) keeps the shared address space: LDS / STS, not generic LD / ST
    uint8_t* smAbuf[2] = {smem, smem + A_BYTES};
    uint8_t* smB = smem + 2 * A_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smB + SB * B_STAGE);      // b_full[SB], b_empty[SB]
    uint64_t* b_full = bars, *b_empty = bars + SB;
    float* sbias = reinterpret_cast<float*>(bars + 2 * SB);                // [bias_floats]
    float* sfirst = sbias + ((p.bias_floats + 3) & ~3);                    // per-tile first-layer bias [npad] + wxy [2 * npad]
    float* sx = sfirst + 3 * 384;                                          // x coordinate of every tile pixel [128]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_row = p.R / ST_TILE;
    const long ntiles = (long)p.B * p.R * tiles_per_row;

    if (threadIdx.x == 0) {
        for (int s = 0; s < SB; ++s) { mbar_init(smem_u32(b_full + s), 1); mbar_init(smem_u32(b_empty + s), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        for (int l = 0; l < p.nl; ++l) asm volatile("prefetch.tensormap [%0];\n" :: "l"(&maps.w[l]) : "memory");
    }
    if constexpr (!BANK)
        for (int i = threadIdx.x; i < p.bias_floats; i += ST_THREADS) sbias[i] = __ldg(p.bias_table + i);
    __syncthreads();

    if (warp == 4) {
        if (lane == 0) {       // ===== TMA producer: the weight tiles of every layer of every tile, in order =====
            uint32_t it = 0;
            for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                int ch = 0;
                if constexpr (BANK) ch = __ldg(p.char_of + (int)(tile / ((long)p.R * tiles_per_row)));
                for (int l = 0; l < p.nl; ++l) {
                    const StLayer& L = p.L[l];
                    const int nsl = L.npad / L.nb, nkc = (L.kpad + 63) >> 6;
                    for (int ns = 0; ns < nsl; ++ns)
                        for (int kc = 0; kc < nkc; ++kc, ++it) {
                            const int s = it % SB;
                            mbar_wait(smem_u32(b_empty + s), ((it / SB) & 1) ^ 1);
                            mbar_expect_tx(smem_u32(b_full + s), L.nb * 128);
                            if constexpr (BANK)
                                asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n"
                                             :: "r"(smem_u32(smB + s * B_STAGE)), "l"(&maps.w[l]), "r"(smem_u32(b_full + s)), "r"(kc * 64), "r"(ns * L.nb), "r"(ch) : "memory");
                            else
                                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n"
                                             :: "r"(smem_u32(smB + s * B_STAGE)), "l"(&maps.w[l]), "r"(smem_u32(b_full + s)), "r"(kc * 64), "r"(ns * L.nb) : "memory");
                        }
                }
            }
        }
    } else {                   // ===== consumer warpgroup: thread te = pixel (tile row) of the prologue / head; fragments for the MMAs =====
        const int te = threadIdx.x;                                        // 0..127
        const int fr = warp * 16 + (lane >> 2);                            // first accumulator row of this thread (+8, +64, +72)
        uint32_t it = 0;
        int cur = 0;                                                       // A buffer holding the current layer's operand
        int staged = -1;                                                   // BANK: the character whose biases sbias holds
        for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int n = (int)(tile / ((long)p.R * tiles_per_row));
            const int rem = (int)(tile - (long)n * p.R * tiles_per_row);
            const int y = rem / tiles_per_row, x0 = (rem - y * tiles_per_row) * ST_TILE;
            const float yv = __ldg(p.base + y);
            sx[te] = __ldg(p.base + x0 + te);
            int ch = 0;
            if constexpr (BANK) {
                ch = __ldg(p.char_of + n);
                if (ch != staged) {        // the previous tile's readers of sbias are past the barrier that ended it
                    for (int i = te; i < p.bias_floats; i += 128) sbias[i] = __ldg(p.bias_table + (size_t)ch * p.bias_cs + i);
                    staged = ch;
                }
            }
            {   // this tile's per-sample first-layer terms: bias (b + Wpose . pose[n]) and the xy weights
                const bool elementwise = (MODE == SM_BODY0 || MODE == SM_FACE);
                const int np = elementwise ? p.e_npad : p.L[0].npad;
                const float* pb = elementwise ? p.e_pb + (size_t)n * p.e_pb_ld : p.f_pb + (size_t)n * p.f_pb_ld;
                const float* wxy = elementwise ? p.e_wxy : p.f_wxy;
                if constexpr (BANK) wxy += (size_t)ch * p.wxy_cs;
                for (int i = te; i < np; i += 128) {
                    sfirst[i] = __ldg(pb + i);
                    sfirst[384 + 2 * i] = __ldg(wxy + 2 * i); sfirst[384 + 2 * i + 1] = __ldg(wxy + 2 * i + 1);
                }
            }
            asm volatile("bar.sync 1, 128;\n" ::: "memory");
            // ---- prologue: the tile's first operand ----
            uint8_t* smA = smAbuf[cur];
            if (MODE == SM_BODY0 || MODE == SM_FACE) {
                const int groups = p.e_npad >> 3;
                for (int i = te; i < ST_TILE * groups; i += 128) {
                    const int r = i / groups, c8 = (i - r * groups) << 3;
                    const float xv = sx[r];
                    uint4 pk;
                    __half2* h2 = reinterpret_cast<__half2*>(&pk);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int c = c8 + 2 * e;
                        const float v0 = sfirst[c] + sfirst[384 + 2 * c] * xv + sfirst[384 + 2 * c + 1] * yv;
                        const float v1 = sfirst[c + 1] + sfirst[384 + 2 * c + 2] * xv + sfirst[384 + 2 * c + 3] * yv;
                        h2[e] = __floats2half2_rn(st_sin(v0), st_sin(v1));
                    }
                    *reinterpret_cast<uint4*>(smA + a_off(r, c8)) = pk;
                }
            } else {
                // bilinear x2 of the previous level (align_corners = False).  Thread = tile pixel: ONE horizontal tap pair, four corner
                // row pointers and four packed-half weights per thread and tile, then per 8-channel group four 16-byte loads,
                // 1 HMUL2 + 3 HFMA2 per channel pair, one 16-byte store into the swizzled operand.
                // The taps 0 / 0.25 / 0.75 / 1 and their products are exact in fp16; the weighted sum is rounded per operation
                // (<= 2 ulp of the fp16 operand it becomes) instead of once.
                const int Rh = p.R >> 1, CP = p.prev_c, groups = CP >> 3;
                const __half* prev = p.prev + (size_t)n * Rh * Rh * CP;
                const LerpTap ty = lerp_locate(y, 0.5f, Rh);
                const LerpTap tx = lerp_locate(x0 + te, 0.5f, Rh);
                const uint4* pa = reinterpret_cast<const uint4*>(prev + ((size_t)ty.i0 * Rh + tx.i0) * CP);
                const uint4* pb = reinterpret_cast<const uint4*>(prev + ((size_t)ty.i0 * Rh + tx.i1) * CP);
                const uint4* pc = reinterpret_cast<const uint4*>(prev + ((size_t)ty.i1 * Rh + tx.i0) * CP);
                const uint4* pd = reinterpret_cast<const uint4*>(prev + ((size_t)ty.i1 * Rh + tx.i1) * CP);
                const __half2 w00 = __float2half2_rn(ty.l0 * tx.l0), w01 = __float2half2_rn(ty.l0 * tx.l1);
                const __half2 w10 = __float2half2_rn(ty.l1 * tx.l0), w11 = __float2half2_rn(ty.l1 * tx.l1);
#pragma unroll 1
                for (int cg0 = 0; cg0 < groups; cg0 += 4) {
                    uint4 va[4], vb[4], vc[4], vd[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int cg = min(cg0 + u, groups - 1);
                        va[u] = __ldg(pa + cg); vb[u] = __ldg(pb + cg); vc[u] = __ldg(pc + cg); vd[u] = __ldg(pd + cg);
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        if (cg0 + u >= groups) break;
                        const __half2* ah = reinterpret_cast<const __half2*>(&va[u]); const __half2* bh = reinterpret_cast<const __half2*>(&vb[u]);
                        const __half2* ch = reinterpret_cast<const __half2*>(&vc[u]); const __half2* dh = reinterpret_cast<const __half2*>(&vd[u]);
                        uint4 o;
                        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            oh[k] = __hfma2(w11, dh[k], __hfma2(w10, ch[k], __hfma2(w01, bh[k], __hmul2(w00, ah[k]))));
                        *reinterpret_cast<uint4*>(smA + a_off(te, (cg0 + u) * 8)) = o;
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");     // generic-proxy writes -> wgmma's async-proxy reads
            asm volatile("bar.sync 1, 128;\n" ::: "memory");
            // ---- the layer chain ----
            for (int l = 0; l < p.nl; ++l) {
                const StLayer& L = p.L[l];
                const int nsl = L.npad / L.nb, nkc = (L.kpad + 63) >> 6;
                const uint8_t* src = smAbuf[cur];
                uint8_t* dst = smAbuf[cur ^ 1];
                const float* lb = sbias + L.bias_off;
                for (int ns = 0; ns < nsl; ++ns) {
                    float d[2][NBMAX / 2];
                    for (int kc = 0; kc < nkc; ++kc, ++it) {
                        const int s = it % SB;
                        mbar_wait(smem_u32(b_full + s), (it / SB) & 1);
                        const int ksteps = min(4, (L.kpad - kc * 64) >> 4);       // K tail: columns beyond kpad hold stale operand data
                        st_slice_mma<NBMAX>(d, L.nb, smem_u32(src + kc * (ST_TILE * 128)), smem_u32(smB + s * B_STAGE), ksteps, kc > 0);
                        if (te == 0) mbar_arrive(smem_u32(b_empty + s));
                    }
                    if (L.sine) {
                        // fragment (row, column pair) -> bias / first-layer terms -> sin -> the other A buffer (fp16)
#pragma unroll
                        for (int g = 0; g < NBMAX / 8; ++g) {
                            if (g * 8 >= L.nb) break;
#pragma unroll
                            for (int h = 0; h < 2; ++h)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int row = h * 64 + fr + 8 * e;
                                    const int c = ns * L.nb + 8 * g + 2 * (lane & 3);
                                    float v0 = d[h][4 * g + 2 * e], v1 = d[h][4 * g + 2 * e + 1];
                                    if (L.first) {
                                        const float xv = sx[row];
                                        v0 += sfirst[c] + sfirst[384 + 2 * c] * xv + sfirst[384 + 2 * c + 1] * yv;
                                        v1 += sfirst[c + 1] + sfirst[384 + 2 * c + 2] * xv + sfirst[384 + 2 * c + 3] * yv;
                                    } else {
                                        v0 += lb[c]; v1 += lb[c + 1];
                                    }
                                    *reinterpret_cast<__half2*>(dst + a_off(row, c & ~7) + (c & 7) * 2) = __floats2half2_rn(st_sin(v0), st_sin(v1));
                                }
                        }
                    } else {
                        // linear head: 16 accumulator columns, transposed through the idle A buffer so that thread = pixel
                        float* stage = reinterpret_cast<float*>(dst);              // [128][17]
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int j = 0; j < 2; ++j) {
                                const int col = 8 * j + 2 * (lane & 3), row = h * 64 + fr;
                                stage[row * 17 + col] = d[h][4 * j];           stage[row * 17 + col + 1] = d[h][4 * j + 1];
                                stage[(row + 8) * 17 + col] = d[h][4 * j + 2]; stage[(row + 8) * 17 + col + 1] = d[h][4 * j + 3];
                            }
                        asm volatile("bar.sync 1, 128;\n" ::: "memory");
                        const float* acc = stage + te * 17;
                        const int x = x0 + te;
                        const float* head_bias = p.head_bias;
                        if constexpr (BANK) head_bias += ch * p.head_cs;
                        if (MODE == SM_FACE) {
#pragma unroll
                            for (int c = 0; c < 4; ++c)
                                p.face_out[(((size_t)n * 4 + c) * p.R + y) * p.R + x] = acc[c] + __ldg(head_bias + c);
                        } else {
                            float o[7];
#pragma unroll
                            for (int c = 0; c < 7; ++c) o[c] = acc[c] + __ldg(head_bias + c);   // grid_change(0,1) alpha(2) colour(3..6)
                            const GsTap t = gs_locate(sx[te], yv, o[0], o[1], p.R, p.R);
                            float w[4];
                            gs_sample<4>(p.image.p + n * p.image.sn, p.image.sc, p.image.sh, p.R, p.R, t, w);
                            const size_t plane = (size_t)p.R * p.R, pix = (size_t)y * p.R + x;
                            const float alpha = o[2];
                            if (p.o_f16) {
                                __half* const* oh = reinterpret_cast<__half* const*>(p.o);
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    oh[0][((size_t)n * 4 + c) * plane + pix] = __float2half_rn((1.0f - alpha) * w[c] + alpha * o[3 + c]);
                                    oh[2][((size_t)n * 4 + c) * plane + pix] = __float2half_rn(o[3 + c]);
                                    oh[3][((size_t)n * 4 + c) * plane + pix] = __float2half_rn(w[c]);
                                }
                                oh[1][(size_t)n * plane + pix] = __float2half_rn(alpha);
                                oh[4][((size_t)n * 2) * plane + pix] = __float2half_rn(o[0]);
                                oh[4][((size_t)n * 2 + 1) * plane + pix] = __float2half_rn(o[1]);
                            } else {
#pragma unroll
                                for (int c = 0; c < 4; ++c) {
                                    p.o[0][((size_t)n * 4 + c) * plane + pix] = (1.0f - alpha) * w[c] + alpha * o[3 + c];
                                    p.o[2][((size_t)n * 4 + c) * plane + pix] = o[3 + c];
                                    p.o[3][((size_t)n * 4 + c) * plane + pix] = w[c];
                                }
                                p.o[1][(size_t)n * plane + pix] = alpha;
                                p.o[4][((size_t)n * 2) * plane + pix] = o[0];
                                p.o[4][((size_t)n * 2 + 1) * plane + pix] = o[1];
                            }
                        }
                    }
                }
                if (L.sine) {
                    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
                    asm volatile("bar.sync 1, 128;\n" ::: "memory");             // the whole output is written before anyone reads it
                    cur ^= 1;
                    if (l == p.nl - 1) {
                        // levels 0 / 1: the last sine layer's output is the level's output tensor (fp16 NHWC)
                        const int groups = p.out_c >> 3;
                        __half* dstg = p.out + (((size_t)n * p.R + y) * p.R + x0) * p.out_c;
                        for (int i = te; i < ST_TILE * groups; i += 128) {
                            const int r = i / groups, cg = i - r * groups;
                            *reinterpret_cast<uint4*>(dstg + (size_t)r * p.out_c + cg * 8) = *reinterpret_cast<const uint4*>(smAbuf[cur] + a_off(r, cg * 8));
                        }
                    }
                }
            }
            asm volatile("bar.sync 1, 128;\n" ::: "memory");          // sx / sfirst / the operands are rewritten by the next tile
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn st_encode() {
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

// W: [rows][kpad] fp16 K-major; box {64 k, nb rows}; rows beyond `rows` and k beyond kpad are zero-filled by TMA.
// chars > 0: W is [chars][rows][kpad] and the map is 3-D with the character outermost (box {64, nb, 1}), so a tile of one
// character never reads another's rows: rows beyond `rows` are zero-filled per character as in the 2-D map.
CUtensorMap weight_tile_map(const void* W, int rows, int kpad, int nb, int chars) {
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)kpad, (cuuint64_t)rows, (cuuint64_t)chars};
    cuuint64_t strides[2] = {(cuuint64_t)kpad * 2, (cuuint64_t)rows * kpad * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)nb, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = st_encode()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, chars > 0 ? 3 : 2, const_cast<void*>(W), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(siren weights) failed: " + std::to_string((int)r));
    return m;
}

template <int ACH, int NBMAX, int SB, int MODE, bool BANK>
void launch_siren_tc_kernel(const StMaps& maps, const StParams& p, int ctas_per_sm, cudaStream_t s) {
    const size_t smem = 1024 + 2 * (size_t)ACH * ST_TILE * 128 + (size_t)SB * NBMAX * 128 + 2 * SB * 8 +
                        ((size_t)((p.bias_floats + 3) & ~3) + 3 * 384 + 128) * sizeof(float);
    THA4_REQUIRE(smem <= 227 * 1024, "siren_tc: shared memory budget");
    for (int l = 0; l < p.nl; ++l)        // st_slice_mma issues the slice widths up to NBMAX only
        THA4_REQUIRE(p.L[l].nb <= NBMAX && p.L[l].npad % p.L[l].nb == 0, "siren_tc: N slice width of layer " + std::to_string(l));
    THA4_ENSURE_SMEM((siren_tc_kernel<ACH, NBMAX, SB, MODE, BANK>), smem);
    const long ntiles = (long)p.B * p.R * (p.R / ST_TILE);
    const int grid = (int)std::min<long>(ntiles, (long)num_sms() * ctas_per_sm);
    siren_tc_kernel<ACH, NBMAX, SB, MODE, BANK><<<grid, ST_THREADS, smem, s>>>(maps, p);
    THA4_LAUNCH_CHECK();
}

// the bank instantiation for a call that carries per-sample characters, the one-character instantiation for every other
template <int ACH, int NBMAX, int SB, int MODE>
void launch_siren_tc(const StMaps& maps, const StParams& p, int ctas_per_sm, cudaStream_t s) {
    if (p.char_of) launch_siren_tc_kernel<ACH, NBMAX, SB, MODE, true>(maps, p, ctas_per_sm, s);
    else launch_siren_tc_kernel<ACH, NBMAX, SB, MODE, false>(maps, p, ctas_per_sm, s);
}

// per mode: the operand buffers' 64-column chunks (ACH) and the widest weight tile (NBMAX) of the launches in siren_tc_run
constexpr int kStAch[4] = {6, 3, 2, 2};
constexpr int kStNbMax[4] = {96, 96, 96, 64};
constexpr int ST_FIRST_MAX = 384;          // sfirst: per-sample bias + xy weights of up to 384 first-layer columns

__global__ void st_sin_kernel(const float* __restrict__ x, long n, float* __restrict__ y) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = st_sin(x[i]);
}

}  // namespace

void siren_tc_sine(const float* x, long n, float* y, cudaStream_t s) {
    st_sin_kernel<<<(int)std::min<long>(ceil_div(n, 256), 1024), 256, 0, s>>>(x, n, y);
    THA4_LAUNCH_CHECK();
}

std::string siren_tc_plan_error(int mode, const SirenTcPlan& plan, const SirenTcLevel& lv) {
    if (mode < 0 || mode > 3) return "mode " + std::to_string(mode) + " is not 0..3";
    const int ach = kStAch[mode], nbmax = kStNbMax[mode], width = ach * 64;
    const bool elementwise = (mode == SM_BODY0 || mode == SM_FACE);
    const std::string at = " (mode " + std::to_string(mode) + ")";
    if (plan.nl < 1 || plan.nl > ST_MAXL) return "layer count " + std::to_string(plan.nl) + " is not 1.." + std::to_string(ST_MAXL) + at;
    if (lv.R <= 0 || lv.R % ST_TILE != 0) return "R = " + std::to_string(lv.R) + " is not a multiple of 128" + at;
    int produced;                          // columns of the operand the current layer reads that its producer wrote
    if (elementwise) {
        if (lv.e_npad <= 0 || lv.e_npad % 8 != 0) return "first-layer width e_npad = " + std::to_string(lv.e_npad) + " is not a positive multiple of 8" + at;
        if (lv.e_npad > ST_FIRST_MAX) return "first-layer width e_npad = " + std::to_string(lv.e_npad) + " > 384" + at;
        if (lv.e_npad > width) return "first-layer width e_npad = " + std::to_string(lv.e_npad) + " > the operand buffer (" + std::to_string(width) + ")" + at;
        produced = lv.e_npad;
    } else {
        if (lv.prev_c <= 0 || lv.prev_c % 8 != 0) return "prev_c = " + std::to_string(lv.prev_c) + " is not a positive multiple of 8" + at;
        if (lv.prev_c > width) return "prev_c = " + std::to_string(lv.prev_c) + " > the operand buffer (" + std::to_string(width) + ")" + at;
        if (plan.npad[0] > ST_FIRST_MAX) return "first-layer width npad = " + std::to_string(plan.npad[0]) + " > 384" + at;
        produced = lv.prev_c;
    }
    for (int l = 0; l < plan.nl; ++l) {
        const std::string ly = "layer " + std::to_string(l) + ": ";
        const int k = plan.kpad[l], n = plan.npad[l], nb = plan.nb[l];
        const bool last = l == plan.nl - 1;
        if (k <= 0 || k % 16 != 0) return ly + "kpad = " + std::to_string(k) + " is not a positive multiple of 16" + at;
        if (k > width) return ly + "kpad = " + std::to_string(k) + " > the operand buffer (" + std::to_string(width) + ")" + at;
        if (k > produced) return ly + "kpad = " + std::to_string(k) + " > the " + std::to_string(produced) + " columns its producer wrote" + at;
        if (nb != 16 && nb != 64 && nb != 96) return ly + "slice width nb = " + std::to_string(nb) + " is not 16, 64 or 96" + at;
        if (nb > nbmax) return ly + "slice width nb = " + std::to_string(nb) + " > NBMAX = " + std::to_string(nbmax) + at;
        if (n <= 0 || n % nb != 0) return ly + "npad = " + std::to_string(n) + " is not a multiple of nb = " + std::to_string(nb) + at;
        const bool want_first = !elementwise && l == 0;
        if ((plan.first[l] != 0) != want_first)
            return ly + (want_first ? "the first GEMM layer of levels 1 / 2 must take the first-layer terms" : "first-layer terms on a layer that is not the first GEMM layer of level 1 / 2") + at;
        if (plan.sine[l]) {
            if (n > width) return ly + "sine layer npad = " + std::to_string(n) + " > the operand buffer (" + std::to_string(width) + ")" + at;
        } else {
            if (!last) return ly + "the head must be the last layer" + at;
            if (mode != SM_BODY2 && mode != SM_FACE) return ly + "a head on a level without one (modes 2 / 3 only)" + at;
            if (n != 16 || nb != 16) return ly + "head npad = " + std::to_string(n) + ", nb = " + std::to_string(nb) + ": both must be 16" + at;
        }
        produced = n;
    }
    if (plan.sine[plan.nl - 1] && lv.out_c != plan.npad[plan.nl - 1])
        return "out_c = " + std::to_string(lv.out_c) + " is not the last layer's npad = " + std::to_string(plan.npad[plan.nl - 1]) + at;
    return "";
}

void SirenTcPlan::add(const SirenLayer& l, int nb, int sine, int first) {
    THA4_REQUIRE(nl < 8, "siren_tc: too many layers");
    THA4_REQUIRE(nb == 16 || nb == 64 || nb == 96, "siren_tc: N slice width");
    kpad[nl] = l.KPAD; npad[nl] = sine ? l.NPAD : 16; this->nb[nl] = nb; this->sine[nl] = sine; this->first[nl] = first;
    W[nl] = l.W; rows[nl] = l.NPAD; bias[nl] = l.bias;
    ++nl;
}

void siren_tc_run(Runtime& rt, int mode, const SirenTcPlan& plan, const SirenTcLevel& lv) {
    const std::string plan_err = siren_tc_plan_error(mode, plan, lv);
    THA4_REQUIRE(plan_err.empty(), "siren_tc plan: " + plan_err);
    const int chars = lv.char_of ? lv.chars : 0;
    THA4_REQUIRE(!lv.char_of || chars >= 1, "siren_tc: a character bank without characters");
    StParams p{};
    StMaps maps;
    p.R = lv.R; p.B = lv.B; p.nl = plan.nl;
    // bias table (device, rebuilt per call from the layers' bias vectors: tiny); a bank's is [chars][all layers' biases]
    int off = 0;
    for (int l = 0; l < plan.nl; ++l) {
        p.L[l].kpad = plan.kpad[l]; p.L[l].npad = plan.npad[l]; p.L[l].nb = plan.nb[l]; p.L[l].sine = plan.sine[l]; p.L[l].first = plan.first[l];
        p.L[l].bias_off = off;
        if (plan.sine[l]) off += plan.npad[l];
        maps.w[l] = weight_tile_map(plan.W[l], plan.rows[l], plan.kpad[l], plan.nb[l], chars);
    }
    p.bias_floats = off;
    float* table = rt.persist->alloc((size_t)std::max(off, 4) * std::max(chars, 1));
    for (int l = 0; l < plan.nl; ++l)
        if (plan.sine[l]) {
            if (chars)      // a sine layer's biases lie npad floats apart from character to character
                THA4_CUDA_CHECK(cudaMemcpy2DAsync(table + p.L[l].bias_off, off * sizeof(float), plan.bias[l], plan.npad[l] * sizeof(float),
                                                  plan.npad[l] * sizeof(float), chars, cudaMemcpyDeviceToDevice, rt.stream));
            else
                THA4_CUDA_CHECK(cudaMemcpyAsync(table + p.L[l].bias_off, plan.bias[l], plan.npad[l] * sizeof(float), cudaMemcpyDeviceToDevice, rt.stream));
        }
    p.bias_table = table;
    p.char_of = lv.char_of; p.bias_cs = off; p.head_cs = lv.head_cs;
    p.wxy_cs = 2 * ((mode == SM_BODY0 || mode == SM_FACE) ? lv.e_npad : plan.npad[0]);
    p.e_npad = lv.e_npad; p.e_pb = lv.e_pb; p.e_pb_ld = lv.e_pb_ld; p.e_wxy = lv.e_wxy;
    p.f_pb = lv.f_pb; p.f_pb_ld = lv.f_pb_ld; p.f_wxy = lv.f_wxy;
    p.base = base_grid_table(lv.R);
    p.prev = lv.prev; p.prev_c = lv.prev_c; p.out = lv.out; p.out_c = lv.out_c;
    p.image = lv.image;
    for (int i = 0; i < 5; ++i) p.o[i] = lv.o[i];
    p.o_f16 = lv.o_f16 ? 1 : 0;
    p.face_out = lv.face_out; p.head_bias = lv.head_bias;
    cudaStream_t s = rt.stream;
    ProfScope prof(PROF_SIREN, s);
    //                         A chunks, widest weight tile, ring
    if (mode == SM_BODY0) launch_siren_tc<kStAch[0], kStNbMax[0], 2, SM_BODY0>(maps, p, 1, s);          // two 96 KB operand buffers
    else if (mode == SM_BODY1) launch_siren_tc<kStAch[1], kStNbMax[1], 4, SM_BODY1>(maps, p, 1, s);
    else if (mode == SM_BODY2) launch_siren_tc<kStAch[2], kStNbMax[2], 2, SM_BODY2>(maps, p, 2, s);
    else launch_siren_tc<kStAch[3], kStNbMax[3], 2, SM_FACE>(maps, p, 2, s);
}

}  // namespace tha4
