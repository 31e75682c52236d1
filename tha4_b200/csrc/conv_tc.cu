// Implicit-GEMM convolution on the Hopper tensor cores: TMA-staged operands, wgmma (f16 operands at K = 16, fp32 operands
// as TF32 at K = 8) with the accumulator in the registers of one consumer warpgroup, and a TMA producer warp.
//
// GEMM view per CTA: D[128 pixels x BN couts] += A[128 x KC] * B[BN x KC]^T per k-block, k-blocks = taps x (Cin/KC),
// KC = 64 f16 / 32 f16 / 32 fp32 channels (128- or 64-byte rows, see OP_* below).
//  * A (activations, NHWC): one 4-D TMA box {KC ch, 16 w, 8 h, 1 n} per (tap, channel chunk).  The box lands in shared
//    memory as 128 rows with the 128-byte (64-byte) swizzle, which is exactly the K-major wgmma operand layout; the
//    tap offset (dy,dx) is just a shift of the box origin, and TMA's out-of-bounds zero fill *is* the convolution's
//    zero padding (and the channel / edge-tile padding).  No im2col buffer, no index arithmetic.  The 4x4 stride-2
//    conv uses the same box with element strides {1,2,2,1} (a {KC, 32 w, 16 h} window sampled every other pixel).
//  * B (weights, packed [phase*tap][cout_pad][cin_pad]): 3-D TMA box {KC cin, BN cout, 1 tap}, same layout.
//  * D: fp32 accumulator, 128 x BN (BN <= 128: BN registers per thread), two m64 wgmmas per K step; bias / residual fused
//    into the epilogue, NHWC stores + per-channel statistics for the normalisation that follows.
//  * K can be split over a thread-block cluster (partials meet in distributed shared memory), launches use
//    programmatic dependent launch with the weight tiles fetched ahead of the dependency wait.
// Handles every tap table of conv.cuh (3x3, 1x1, 4x4 stride 2, the four phases of the transposed 4x4 and of the
// nearest-x2-upsample + 3x3); strict mode (3xTF32) and non-TMA-able views stay on the mma.sync kernel in conv.cu.
#include "conv.cuh"
#include "profiler.cuh"
#include "conv_tc_device.cuh"
#include <cuda.h>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <map>
#include <mutex>
#include <tuple>

namespace tha4 {
namespace {

using namespace tc;
using namespace tcdev;

template <int BN, int STAGES_, int CS, int OP, int XF>
__global__ void __launch_bounds__(TC_THREADS) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB, const TcParams p) {
    static_assert(BN <= 128, "the accumulator of one warpgroup: BN registers per thread");
    constexpr int STAGES = op_stages(OP, STAGES_);
    constexpr int ROWB = op_row_bytes(OP);
    constexpr int KCE = op_kch(OP);
    constexpr int A_BYTES = 128 * ROWB;
    constexpr int B_BYTES = BN * ROWB;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);      // pointer arithmetic (not an integer round trip) keeps the shared address space: LDS / STS, not generic LD / ST
    uint8_t* smA = smem;
    uint8_t* smB = smem + STAGES * A_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smB + STAGES * B_BYTES);   // full[STAGES], empty[STAGES]
    float* xf_A = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars + 2 * STAGES) + ((16u - (tc::smem_u32(bars + 2 * STAGES) & 15u)) & 15u));   // XF: per-channel affine y = act(A * x + B), [xf_C] each
    static_assert(XF == 0 || OP != OP_TF32, "the fused input normalisation works on f16 operands");

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // tile coordinates
    int tile = blockIdx.x;
    const int tx = tile % p.tiles_x; tile /= p.tiles_x;
    const int ty = tile % p.tiles_y;
    const int n = tile / p.tiles_y;
    const int x0 = tx * TILE_W, y0 = ty * TILE_H;
    const int n0 = blockIdx.y * BN;
    const int phase = blockIdx.z / p.ksplit, split = blockIdx.z % p.ksplit;
    const int KT = p.ntaps * p.cpt;
    const int k_per = (KT + p.ksplit - 1) / p.ksplit;
    const int kb = split * k_per;
    const int nk = max(0, min(KT, kb + k_per) - kb);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(bars + s), 1); mbar_init(smem_u32(bars + STAGES + s), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];\n" :: "l"(&tmB) : "memory");
    }
    __syncthreads();
    // resources are held: let the next kernel of the stream start its prologue, then wait for our own producers.
    // The WEIGHT tiles of the first ring pass do not depend on the previous kernel: their TMA loads are issued before
    // the dependency wait, so the DRAM round trip of the weights overlaps the predecessor's tail instead of following it.
    pdl_trigger();
    const int npre = p.pre_b ? min(nk, STAGES) : 0;
    if (warp == TC_PRODUCER_WARP && lane == 0) {
        for (int i = 0; i < npre; ++i) {
            const uint32_t full = smem_u32(bars + i);
            mbar_expect_tx(full, A_BYTES + B_BYTES);
            const int kt = kb + i;
            const int tap = kt / p.cpt;
            tma_load_3d(smem_u32(smB + i * B_BYTES), &tmB, (kt - tap * p.cpt) * KCE, n0, phase * p.ntaps + tap, full);
        }
    }
    pdl_wait();

    Acc<BN> acc;
    if (nk > 0) {
        if (warp == TC_PRODUCER_WARP) {
            if (lane == 0) {   // ===== TMA producer =====
                for (int i = 0; i < nk; ++i) {
                    const int s = i % STAGES;
                    const uint32_t full = smem_u32(bars + s);
                    const int kt = kb + i;
                    const int tap = kt / p.cpt;
                    const int c0 = (kt - tap * p.cpt) * KCE;
                    if (i >= npre) {
                        mbar_wait(smem_u32(bars + STAGES + s), ((i / STAGES) & 1) ^ 1);
                        mbar_expect_tx(full, A_BYTES + B_BYTES);
                        tma_load_3d(smem_u32(smB + s * B_BYTES), &tmB, c0, n0, phase * p.ntaps + tap, full);
                    }
                    tma_load_4d(smem_u32(smA + s * A_BYTES), &tmA, c0, x0 * p.in_mul + p.dx[phase][tap], y0 * p.in_mul + p.dy[phase][tap], n, full);
                }
            }
        } else {
            // ===== consumer warpgroup: (XF: normalise the A operand of the k-block in place), wgmma, then the epilogue =====
            const int te = threadIdx.x;                                   // 0..127 = tile row (pixel) this thread owns
            __half* hA = reinterpret_cast<__half*>(xf_A);
            __half* hB = hA + p.xf_C;
            const bool silu = p.xf_act == ACT_SILU || p.xf_act == ACT_SILU_FAST;
            const int ry = te / TILE_W, rx = te % TILE_W;
            const int swz = ROWB == 128 ? (te & 7) : ((te >> 1) & 3);    // the row's XOR term of the TMA swizzle (stage bases are 1024-aligned)
            if (XF) {
                // the affine is applied with packed half2 arithmetic (HFMA2, tanh.approx.f16x2): the operand is f16 anyway
                double2* chs = reinterpret_cast<double2*>(xf_A + 2 * p.xf_C); // per-channel (sum, sum of squares) folded over the replicas
                int c_lo = 0, c_hi = p.xf_C;
                { const int f = kb % p.cpt; if (f + nk <= p.cpt) { c_lo = f * KCE; c_hi = (f + nk) * KCE; } }   // k-blocks of one tap: a chunk range
                xf_build_coef(p, n, te, hA, hB, chs, c_lo, c_hi);
            }
            for (int i = 0; i < nk; ++i) {
                const int s = i % STAGES;
                mbar_wait(smem_u32(bars + s), (i / STAGES) & 1);          // TMA bytes of this stage have landed
                if (XF) {
                    const int kt = kb + i;
                    const int tap = kt / p.cpt;
                    const int c0 = (kt - tap * p.cpt) * KCE;
                    const int iy = (y0 + ry) * p.in_mul + p.dy[phase][tap], ix = (x0 + rx) * p.in_mul + p.dx[phase][tap];
                    // rows outside the image are the convolution's zero padding (TMA filled them with zeros): they stay zero
                    if (iy >= 0 && iy < p.inH && ix >= 0 && ix < p.inW) xf_row<ROWB>(smA + s * A_BYTES + te * ROWB, swz, c0, p, hA, hB, silu);
                    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");   // generic-proxy writes -> visible to wgmma's async-proxy reads
                    asm volatile("bar.sync 1, 128;\n" ::: "memory");
                }
                const uint32_t a_addr = smem_u32(smA + s * A_BYTES), b_addr = smem_u32(smB + s * B_BYTES);
                wg_fence();
#pragma unroll
                for (int k = 0; k < ROWB / 32; ++k) {   // one wgmma consumes 32 bytes of K per row (8 tf32 / 16 f16): advance the start address by 32
                    const uint64_t a0 = make_smem_desc_sw<ROWB>(a_addr + 32 * k), a1 = make_smem_desc_sw<ROWB>(a_addr + 64 * ROWB + 32 * k);
                    const uint64_t bd = make_smem_desc_sw<ROWB>(b_addr + 32 * k);
                    const uint32_t accum = (i > 0 || k > 0) ? 1u : 0u;
                    if (OP == OP_TF32) { Wgmma<BN>::tf32(acc.d[0], a0, bd, accum); Wgmma<BN>::tf32(acc.d[1], a1, bd, accum); }
                    else { Wgmma<BN>::f16(acc.d[0], a0, bd, accum); Wgmma<BN>::f16(acc.d[1], a1, bd, accum); }
                }
                wg_commit();
                wg_wait<1>();                                              // the k-block before this one has been read
                if (i > 0 && te == 0) mbar_arrive(smem_u32(bars + STAGES + (i - 1) % STAGES));
            }
            wg_wait<0>();
            wg_fence_acc(acc.d[0]); wg_fence_acc(acc.d[1]);
            if (CS == 1) epi_direct<BN, TILE_W>(p, acc, smem, n, y0, x0, n0, phase, split, warp, lane);
        }
    }
    if (CS > 1) {
        // ---- cluster split-K reduction through distributed shared memory (conv_tc_device.cuh) ----
        // barrier A: every CTA of the cluster has its accumulator and idle pipeline buffers -> peers may write into them
        asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
        if (warp < TC_PRODUCER_WARP && nk > 0) epi_push_partial<BN, CS>(acc, smem, split, warp, lane);
        // barrier B: the pushed slices are visible to their owners; nobody touches a peer's memory afterwards
        asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
        asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
        if (warp < TC_PRODUCER_WARP) epi_cluster_reduce<BN, CS, TILE_W>(p, smem, n, y0, x0, n0, phase, split, warp);
    }
}

// out = sum_splits ws + bias + res  (deterministic split-K reduction; replaces fp32 atomics), plus the per-(n,c)
// statistics of the result.  grid = (pixel slabs, N * nphase); thread (pl, q) walks pixels pl, pl + PL, ... of its slab.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const TcParams p, int nphase, int ppt) {
    __shared__ float red[256][9];
    const int cq = (p.outC + 3) >> 2;
    const int PL = 256 / cq;
    const int tid = threadIdx.x;
    const int pl = tid / cq, q = tid - pl * cq;
    const int n = blockIdx.y / nphase, phase = blockIdx.y % nphase;
    const bool active = pl < PL;
    const int c = 4 * q;
    const int cn = min(4, p.outC - c);
    float su[4] = {0, 0, 0, 0}, sq[4] = {0, 0, 0, 0};
    if (active) {
        const long MHW = (long)p.MH * p.MW;
        const long base = (long)blockIdx.x * PL * ppt;
        for (int i = 0; i < ppt; ++i) {
            const long m = base + (long)i * PL + pl;
            if (m >= MHW) break;
            const int my = (int)(m / p.MW), mx = (int)(m - (long)my * p.MW);
            const long tile = ((long)n * p.tiles_y + my / TILE_H) * p.tiles_x + mx / TILE_W;
            const int row = (my % TILE_H) * TILE_W + mx % TILE_W;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int s = 0; s < p.ksplit; ++s) {
                const float4 v = *reinterpret_cast<const float4*>(p.ws + ((long)(phase * p.ksplit + s) * p.ws_rows + tile * 128 + row) * p.ws_ld + c);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            const int oy = my * p.out_mul + p.ph_oy[phase], ox = mx * p.out_mul + p.ph_ox[phase];
            float v[4] = {acc.x, acc.y, acc.z, acc.w};      // partials were scaled (acc_scale) by the producing CTAs
            if (p.bias) for (int j = 0; j < cn; ++j) v[j] += __ldg(p.bias + c + j);
            if (p.res_mode == RES_SAME || p.res_mode == RES_UP2) {
                const int ry = p.res_mode == RES_UP2 ? (oy >> 1) : oy, rx = p.res_mode == RES_UP2 ? (ox >> 1) : ox;
                const float* rr = p.res + (((long)n * p.resH + ry) * p.resW + rx) * p.res_ld + c;
                for (int j = 0; j < cn; ++j) v[j] += rr[j];
            } else if (p.res_mode == RES_DOWN2) {
                const float* rr = p.res + (((long)n * p.resH + 2 * oy) * p.resW + 2 * ox) * p.res_ld + c;
                const long dx1 = p.res_ld, dy1 = (long)p.resW * p.res_ld;
                for (int j = 0; j < cn; ++j) v[j] += 0.25f * ((rr[j] + rr[dx1 + j]) + (rr[dy1 + j] + rr[dy1 + dx1 + j]));
            }
            const long opix = ((long)n * p.outH + oy) * p.outW + ox;
            if (p.out) {
                float* o = p.out + opix * p.out_ld + c;
                if (cn == 4) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
                else for (int j = 0; j < cn; ++j) o[j] = v[j];
            }
            if (p.out16) {
                __half* o16 = p.out16 + opix * p.out16_ld + c;
                for (int j = 0; j < cn; ++j) o16[j] = __float2half_rn(v[j]);
            }
            for (int j = 0; j < cn; ++j) { su[j] += v[j]; sq[j] += v[j] * v[j]; }
        }
    }
    if (!p.stats) return;
#pragma unroll
    for (int k = 0; k < 4; ++k) { red[tid][k] = su[k]; red[tid][4 + k] = sq[k]; }
    __syncthreads();
    if (active && pl == 0) {
        double acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0;
        for (int j = 0; j < PL; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += (double)red[j * cq + q][k];
        double* d = p.stats + (long)(blockIdx.x % p.stats_rep) * p.stats_rep_stride + ((long)n * p.stats_ld + c) * 2;
        for (int k = 0; k < cn; ++k) { atomicAdd(d + 2 * k, acc[k]); atomicAdd(d + 2 * k + 1, acc[4 + k]); }
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
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

// Encoded tensor maps are cached process-wide, keyed by (device, base pointer, geometry); the cache is shared by every
// context of the process (contexts may be driven from different host threads: ctypes releases the GIL), hence the lock.
// std::map nodes are stable, so the returned references stay valid after the lock is dropped.
using MapKey = std::tuple<int, const void*, long, long, long, long, long, int>;
std::map<MapKey, CUtensorMap> g_maps;
std::mutex g_maps_mu;

const CUtensorMap& activation_map(const View& v, int op, int stride) {
    MapKey key{current_device(), v.p, v.N, v.H, v.W, v.C, v.ld, -(1 + 4 * op + 16 * stride)};
    std::lock_guard<std::mutex> lock(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[4] = {(cuuint64_t)v.C, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)v.N};
    const cuuint64_t eb = op == OP_TF32 ? 4 : 2;
    THA4_REQUIRE((op != OP_TF32) == (v.f16 != 0), "conv_tc: operand format does not match the activation view");
    cuuint64_t strides[3] = {(cuuint64_t)v.ld * eb, (cuuint64_t)v.W * v.ld * eb, (cuuint64_t)v.H * v.W * v.ld * eb};
    // stride 2: the box spans 2x the pixels and is traversed with element stride 2, so it still delivers 16 x 8 pixels
    cuuint32_t box[4] = {(cuuint32_t)op_kch(op), (cuuint32_t)(TILE_W * stride), (cuuint32_t)(TILE_H * stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = get_encode()(&m, op == OP_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, v.p, dims, strides, box, es,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, op == OP_F16N ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(activation) failed: " + std::to_string((int)r));
    return g_maps.emplace(key, m).first->second;
}

const CUtensorMap& weight_map(const ConvWeights& cw, int bn, int op) {
    const void* wp = op == OP_TF32 ? (const void*)cw.w : (const void*)cw.w16;
    MapKey key{current_device(), wp, cw.cin_pad, cw.cout_pad, cw.ntaps, cw.nphase, op, bn};
    std::lock_guard<std::mutex> lock(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) return it->second;
    CUtensorMap m;
    cuuint64_t dims[3] = {(cuuint64_t)cw.cin_pad, (cuuint64_t)cw.cout_pad, (cuuint64_t)cw.ntaps * cw.nphase};
    const cuuint64_t eb = op == OP_TF32 ? 4 : 2;
    cuuint64_t strides[2] = {(cuuint64_t)cw.cin_pad * eb, (cuuint64_t)cw.cout_pad * cw.cin_pad * eb};
    cuuint32_t box[3] = {(cuuint32_t)op_kch(op), (cuuint32_t)bn, 1};
    cuuint32_t es[3] = {1, 1, 1};
    CUresult r = get_encode()(&m, op == OP_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(wp), dims, strides, box, es,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, op == OP_F16N ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    THA4_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r));
    return g_maps.emplace(key, m).first->second;
}

template <int OP, int BN, int STAGES_, int CS = 1, int XF = 0>
void launch_tc(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, dim3 grid, cudaStream_t s) {
    constexpr int STAGES = op_stages(OP, STAGES_);
    constexpr int STAGE_BYTES = (128 + BN) * op_row_bytes(OP);
    constexpr size_t smem0 = 1024 + (size_t)STAGES * STAGE_BYTES + 2 * STAGES * 8 + 16;
    static_assert(smem0 <= 227 * 1024, "shared memory budget");
    // XF: per-channel affine (2 floats) + folded statistics (1 double2) of the normalised input channels
    const size_t smem = smem0 + (XF ? (size_t)24 * p.xf_C + 32 : 0);
    THA4_REQUIRE(smem <= 227 * 1024, "conv_tc: shared memory budget (fused input normalisation)");
    static_assert((size_t)STAGES * STAGE_BYTES >= (size_t)4 * 32 * 33 * 4 + 4 * BN * 8, "epilogue scratch must fit in the pipeline buffers");
    static_assert(CS == 1 || (size_t)STAGES * STAGE_BYTES >= (size_t)128 * BN * 4 + 128 * 8 * 4 + 128 * 4, "partial tile + statistics scratch must fit");
    THA4_ENSURE_SMEM((conv_tc_kernel<BN, STAGES_, CS, OP, XF>), smem);
    launch_pdl(conv_tc_kernel<BN, STAGES_, CS, OP, XF>, grid, dim3(TC_THREADS), smem, s, CS, ma, mb, p);
    THA4_LAUNCH_CHECK();
}

template <int OP, int BN, int STAGES, int XF>
void launch_tc_cluster(int cs, const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, dim3 grid, cudaStream_t s) {
    if (cs == 8) launch_tc<OP, BN, STAGES, 8, XF>(ma, mb, p, grid, s);
    else if (cs == 4) launch_tc<OP, BN, STAGES, 4, XF>(ma, mb, p, grid, s);
    else launch_tc<OP, BN, STAGES, 2, XF>(ma, mb, p, grid, s);
}

// all launch shapes of one operand format: cluster split-K, deep / mid / shallow TMA rings
template <int OP, int XF>
void launch_variants(bool cluster, int stages_mode, int bn, int ksplit, const CUtensorMap& ma, const CUtensorMap& mb,
                     const TcParams& p, dim3 grid, cudaStream_t s) {
    if (cluster) {
        if (bn == 128) launch_tc_cluster<OP, 128, 6, XF>(ksplit, ma, mb, p, grid, s);
        else if (bn == 64) launch_tc_cluster<OP, 64, 8, XF>(ksplit, ma, mb, p, grid, s);
        else launch_tc_cluster<OP, 32, 8, XF>(ksplit, ma, mb, p, grid, s);
    } else if (stages_mode == 0) {
        if (bn == 128) launch_tc<OP, 128, 6, 1, XF>(ma, mb, p, grid, s);
        else if (bn == 64) launch_tc<OP, 64, 8, 1, XF>(ma, mb, p, grid, s);
        else launch_tc<OP, 32, 8, 1, XF>(ma, mb, p, grid, s);
    } else if (stages_mode == 1) {
        if (bn == 128) launch_tc<OP, 128, 3, 1, XF>(ma, mb, p, grid, s);
        else if (bn == 64) launch_tc<OP, 64, 4, 1, XF>(ma, mb, p, grid, s);
        else launch_tc<OP, 32, 5, 1, XF>(ma, mb, p, grid, s);
    } else {
        if (bn == 128) launch_tc<OP, 128, 2, 1, XF>(ma, mb, p, grid, s);
        else if (bn == 64) launch_tc<OP, 64, 2, 1, XF>(ma, mb, p, grid, s);
        else launch_tc<OP, 32, 3, 1, XF>(ma, mb, p, grid, s);
    }
}

// fp32 packed weights -> f16, scaled by a power of two chosen so that max |w| lands in [0.5, 1): the scaling is exact,
// keeps a layer of small weights out of f16's subnormal range (|w| < 6.1e-5 would lose mantissa bits) and is undone
// on the fp32 accumulator (TcParams::acc_scale).  The packed values were already rounded to 10 mantissa bits.
__global__ void pack_half_kernel(const float* __restrict__ w, __half* __restrict__ h, long n, float scale) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) h[i] = __float2half_rn(w[i] * scale);
}
__global__ void absmax_kernel(const float* __restrict__ w, long n, unsigned* __restrict__ out) {
    float m = 0.0f;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));          // non-negative floats order like their bit patterns
}

int op_for(const ConvWeights& cw, const ConvArgs& a) {
    if (!a.in.f16) return OP_TF32;
    return cw.cin_pad % 64 == 0 ? OP_F16 : OP_F16N;
}

}  // namespace

namespace {
struct TcPlan { int bn, tiles_x, tiles_y, tiles_m, tiles_n, ksplit, MH, MW; bool cluster; };
TcPlan tc_plan(const ConvWeights& cw, const ConvArgs& a) {
    TcPlan pl;
    pl.MH = a.out.H / cw.out_mul; pl.MW = a.out.W / cw.out_mul;
    pl.tiles_x = ceil_div(pl.MW, TILE_W); pl.tiles_y = ceil_div(pl.MH, TILE_H);
    // N tile: at most 128 columns, the accumulator of one consumer warpgroup (BN fp32 registers per thread)
    pl.bn = (cw.cout_pad % 128 == 0) ? 128 : (cw.cout_pad % 64 == 0 ? 64 : 32);
    const int sms = num_sms();
    pl.tiles_m = pl.tiles_x * pl.tiles_y * a.in.N;
    pl.tiles_n = cw.cout_pad / pl.bn;
    const int KT = cw.ntaps * (cw.cin_pad / op_kch(op_for(cw, a)));
    int ksplit = a.ksplit;
    if (ksplit <= 0) {
        // few tiles: narrow the N tiles first (nothing to exchange), split K only for what is still missing -- the DSMEM
        // exchange of a cluster split grows with bn (conv_halo.cu, halo_plan)
        while (pl.bn > 64 && (long)pl.tiles_m * (cw.cout_pad / pl.bn) * cw.nphase < sms && cw.cout_pad % (pl.bn / 2) == 0) pl.bn /= 2;
        pl.tiles_n = cw.cout_pad / pl.bn;
        const long ctas = (long)pl.tiles_m * pl.tiles_n * cw.nphase;
        ksplit = 1;
        if (ctas < sms * 13 / 16) {
            ksplit = (int)((sms + ctas - 1) / ctas);
            ksplit = std::min(ksplit, std::max(1, KT / 4));
            ksplit = std::min(ksplit, 32);
        }
    }
    ksplit = std::max(1, std::min(ksplit, KT));
    const int k_per = (KT + ksplit - 1) / ksplit;
    pl.ksplit = (KT + k_per - 1) / k_per;          // every split owns at least one k-block
    if (a.ksplit <= 0 && pl.ksplit == 1) {
        // tiny GEMMs whose K is too short to split (the 1x1 qkv / proj convs at 16^2: 12 CTAs with BN = 128): narrower N
        // tiles put more SMs to work and shorten each CTA's weight fetch and epilogue
        while (pl.bn > 32 && (long)pl.tiles_m * (cw.cout_pad / pl.bn) * cw.nphase < 64 && cw.cout_pad % (pl.bn / 2) == 0) pl.bn /= 2;
        pl.tiles_n = cw.cout_pad / pl.bn;
    }
    pl.cluster = false;
    if (opts().cluster_splitk && pl.ksplit > 1 && KT >= 2) {
        // Split K over a thread-block cluster instead (partials meet in distributed shared memory, no workspace, no
        // second kernel).  Cluster size 2/4/8; narrower N tiles buy back the CTA count the smaller split gives up.
        int cs = 2;
        while (cs < 8 && cs * 2 <= pl.ksplit && cs * 2 <= KT) cs *= 2;
        int bn = pl.bn;
        while (bn > 32 && (long)pl.tiles_m * (cw.cout_pad / bn) * cw.nphase * cs < 96 && cw.cout_pad % (bn / 2) == 0) bn /= 2;
        const int kp = (KT + cs - 1) / cs;
        if ((KT + kp - 1) / kp == cs) {            // every rank of the cluster must own k-blocks
            pl.cluster = true; pl.ksplit = cs; pl.bn = bn; pl.tiles_n = cw.cout_pad / bn;
        }
    }
    return pl;
}
}  // namespace

size_t conv_workspace_floats(const ConvWeights& cw, const ConvArgs& a) {
    if (!conv_tc_supported(cw, a) || conv_halo_supported(cw, a)) return 0;
    const TcPlan pl = tc_plan(cw, a);
    if (pl.ksplit <= 1 || pl.cluster) return 0;
    return (size_t)cw.nphase * pl.ksplit * pl.tiles_m * 128 * cw.cout_pad;
}

int conv_tc_split_plan(const ConvWeights& cw, const ConvArgs& a) {
    if (!opts().tcgen05 || !conv_tc_supported(cw, a) || conv_halo_supported(cw, a)) return 0;
    const TcPlan pl = tc_plan(cw, a);
    if (pl.ksplit <= 1) return 0;
    if (pl.cluster) return 1;
    return a.ws && a.ws_floats >= (size_t)cw.nphase * pl.ksplit * pl.tiles_m * 128 * cw.cout_pad ? 2 : 3;
}

void conv_make_half(const ConvWeights& cw, cudaStream_t s) {
    if (cw.w16 || !cw.w) return;
    const long nw = (long)conv_packed_floats(cw);
    __half* h = reinterpret_cast<__half*>(tracked_malloc(nw * sizeof(__half)));
    const int blocks = (int)std::min<long>((nw + 255) / 256, 1184);
    unsigned* dmax = reinterpret_cast<unsigned*>(h);                          // scratch: the first word of the (not yet written) copy
    THA4_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned), s));
    absmax_kernel<<<blocks, 256, 0, s>>>(cw.w, nw, dmax);
    THA4_LAUNCH_CHECK();
    unsigned hmax = 0;
    THA4_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));                                // load time (or the first call of a test conv)
    float mx; memcpy(&mx, &hmax, sizeof(float));
    float scale = 1.0f;
    if (mx > 0.0f && std::isfinite(mx)) {
        int e = 0; frexpf(mx, &e);                                             // mx = f * 2^e, f in [0.5, 1)
        e = std::max(-24, std::min(8, e));
        scale = ldexpf(1.0f, -e);
    }
    pack_half_kernel<<<blocks, 256, 0, s>>>(cw.w, h, nw, scale);
    THA4_LAUNCH_CHECK();
    cw.w16 = h; cw.w16_scale = scale;
}

__global__ void bias_sum_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ b, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = (a ? a[i] : 0.0f) + (b ? b[i] : 0.0f);
}

void conv_make_fold(ConvWeights& fold, const ConvWeights& conv3, const ConvWeights& conv1x1, cudaStream_t s) {
    THA4_REQUIRE(conv3.ntaps == 9 && conv3.nphase == 1 && conv1x1.ntaps == 1 && conv1x1.nphase == 1 && conv3.cout_pad == conv1x1.cout_pad &&
                 conv3.w16 && conv1x1.w16, "conv_make_fold: a 3x3 and a 1x1 conv of the same width, with f16 copies");
    float* bias = reinterpret_cast<float*>(tracked_malloc(conv3.cout * sizeof(float)));
    bias_sum_kernel<<<ceil_div(conv3.cout, 128), 128, 0, s>>>(bias, conv3.bias, conv1x1.bias, conv3.cout);
    THA4_LAUNCH_CHECK();
    fold = conv3;
    fold.w = nullptr;                                                          // f16 only: the halo kernel's operands
    fold.bias = bias;
    fold.cin2 = conv1x1.cin; fold.cin2_pad = conv1x1.cin_pad;
    fold.w16b = conv1x1.w16; fold.w16b_scale = conv1x1.w16_scale;
}

bool conv_tc_fuses_stats(const ConvWeights& cw, const ConvArgs& a) {
    const TcPlan pl = tc_plan(cw, a);
    if (pl.ksplit == 1 || pl.cluster) return true;
    return a.ws && a.ws_floats >= (size_t)cw.nphase * pl.ksplit * pl.tiles_m * 128 * cw.cout_pad;
}

bool conv_tc_supported(const ConvWeights& cw, const ConvArgs& a) {
    if (a.in_up || a.strict) return false;
    // 4x4 stride-2 convs read their taps through element-strided TMA boxes
    if (cw.stride != 1 && !(cw.stride == 2 && cw.nphase == 1 && a.in.H % 2 == 0 && a.in.W % 2 == 0)) return false;
    if (a.in.ld % (a.in.f16 ? 8 : 4) != 0 || (((uintptr_t)a.in.p) & 15) != 0) return false;
    if (a.out.p && (a.out.ld % 4 != 0 || (((uintptr_t)a.out.p) & 15) != 0)) return false;
    if (a.out16.p && (a.out16.ld % 8 != 0 || (((uintptr_t)a.out16.p) & 15) != 0)) return false;
    if (!a.out.p && !a.out16.p) return false;
    if (a.nin.on && !a.in.f16) return false;       // the fused input normalisation transforms f16 operand tiles
    if (cw.cout_pad % 32 != 0) return false;
    return true;
}

void conv_tc_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s) {
    THA4_REQUIRE(conv_tc_supported(cw, a), "conv_tc: unsupported configuration");
    THA4_REQUIRE(a.in.C == cw.cin && a.out.C == cw.cout && a.in.N == a.out.N, "conv_tc: shapes");
    TcParams p{};
    p.out = a.out.p; p.outH = a.out.H; p.outW = a.out.W; p.outC = a.out.C; p.out_ld = a.out.ld;
    p.out16 = a.out16.p ? a.out16.hp() : nullptr; p.out16_ld = a.out16.ld;
    if (a.out16.p) THA4_REQUIRE(a.out16.f16 && a.out16.N == a.out.N && a.out16.H == a.out.H && a.out16.W == a.out.W && a.out16.C == a.out.C, "conv_tc: f16 output copy geometry");
    p.inH = a.in.H; p.inW = a.in.W; p.inC = a.in.C;
    if (a.nin.on) {
        const ConvNormIn& ni = a.nin;
        THA4_REQUIRE(ni.stats != nullptr && ni.gamma != nullptr && ni.beta != nullptr, "conv_tc: fused input normalisation needs statistics and affine parameters");
        THA4_REQUIRE(ni.C > 0 && ni.C <= a.in.C && ni.C % 8 == 0 && ni.C <= 1024, "conv_tc: normalised channel count");
        THA4_REQUIRE(ni.groups == 0 || (ni.C == a.in.C && ni.C % ni.groups == 0), "conv_tc: GroupNorm spans the whole input");
        p.in_stats = ni.stats; p.in_stats_ld = ni.stats_ld; p.in_stats_rep = std::max(1, ni.stats_rep); p.in_stats_rep_stride = ni.stats_rep_stride;
        p.xf_C = ni.C; p.xf_groups = ni.groups; p.xf_act = ni.act;
        p.xf_inv_cnt = 1.0 / ((double)a.in.H * a.in.W * (ni.groups == 0 ? 1 : ni.C / ni.groups));
        p.xf_gamma = ni.gamma; p.xf_beta = ni.beta; p.xf_film0 = ni.film0; p.xf_film1 = ni.film1; p.xf_film1_ld = ni.film1_ld;
    }
    p.bias = cw.bias;
    p.res = a.res.p; p.res_mode = a.res.p ? a.res_mode : RES_NONE;
    p.vec4 = ((!cw.bias || (reinterpret_cast<uintptr_t>(cw.bias) & 15) == 0) &&
              (!a.res.p || ((reinterpret_cast<uintptr_t>(a.res.p) & 15) == 0 && a.res.ld % 4 == 0))) ? 1 : 0;
    p.resH = a.res.H; p.resW = a.res.W; p.res_ld = a.res.ld;
    p.N = a.in.N;
    p.out_mul = cw.out_mul;
    const TcPlan pl = tc_plan(cw, a);
    p.MH = pl.MH; p.MW = pl.MW;
    p.in_mul = cw.stride;
    THA4_REQUIRE(p.MH * cw.stride == a.in.H && p.MW * cw.stride == a.in.W, "conv_tc: geometry");
    p.tiles_x = pl.tiles_x; p.tiles_y = pl.tiles_y;
    const int op = op_for(cw, a);
    p.pre_b = cw.dynamic ? 0 : 1;            // static (loaded once) weights only
    p.ntaps = cw.ntaps; p.cpt = cw.cin_pad / op_kch(op);
    p.acc_scale = 1.0f;
    if (op != OP_TF32 && !cw.w16) {          // first use with f16 activations and no copy made at load time
        conv_make_half(cw, s);
        p.pre_b = 0;                          // written by the kernel just launched: order through the dependency wait
    }
    if (op != OP_TF32) p.acc_scale = 1.0f / cw.w16_scale;
    for (int ph = 0; ph < CONV_MAX_PHASES; ++ph) {
        p.ph_oy[ph] = cw.ph_oy[ph]; p.ph_ox[ph] = cw.ph_ox[ph];
        for (int t = 0; t < CONV_MAX_TAPS; ++t) { p.dy[ph][t] = cw.dy[ph][t]; p.dx[ph][t] = cw.dx[ph][t]; }
    }
    const int bn = pl.bn, tiles_m = pl.tiles_m, tiles_n = pl.tiles_n, ksplit = pl.ksplit;
    p.ksplit = ksplit;
    const size_t ws_need = (size_t)cw.nphase * ksplit * tiles_m * 128 * cw.cout_pad;
    const bool use_ws = !pl.cluster && ksplit > 1 && a.ws && a.ws_floats >= ws_need;
    p.ws = use_ws ? a.ws : nullptr; p.ws_rows = (long)tiles_m * 128; p.ws_ld = cw.cout_pad;
    // statistics: fused when the result is final in this launch sequence (single pass, or split-K with workspace)
    p.stats = (ksplit == 1 || use_ws || pl.cluster) ? a.out.stats : nullptr; p.stats_ld = a.out.stats_ld;
    p.stats_rep = std::max(1, a.out.stats_rep); p.stats_rep_stride = a.out.stats_rep_stride;
    ProfScope prof(PROF_CONV, s);
    prof_add_work(PROF_CONV, 2.0 * (double)p.N * p.MH * p.MW * cw.cout * cw.cin * cw.ntaps * cw.nphase, 0.0);
    THA4_REQUIRE(!(ksplit > 1 && !use_ws && !pl.cluster) || (a.out.p && !a.out16.p), "conv_tc: atomic split-K accumulates into an fp32 output only");
    if (ksplit > 1 && !use_ws && !pl.cluster)
        THA4_CUDA_CHECK(cudaMemset2DAsync(a.out.p, (size_t)a.out.ld * sizeof(float), 0, (size_t)a.out.C * sizeof(float), a.out.pixels(), s));
    const CUtensorMap& ma = activation_map(a.in, op, cw.stride);
    const CUtensorMap& mb = weight_map(cw, bn, op);
    dim3 grid(tiles_m, tiles_n, cw.nphase * ksplit);
    // Pipeline depth: grids that cannot even fill the GPU once (the B=1 bottleneck layers, which stream their weights
    // from HBM with one CTA per SM) get a deep TMA ring to hide DRAM latency; large grids get a shallow ring so that
    // 2-3 CTAs share an SM and overlap each other's prologue / epilogue.  THA4_TC_STAGES=deep|mid|shallow overrides.
    static int forced = -2;
    if (forced == -2) {
        const char* e = getenv("THA4_TC_STAGES");
        forced = !e ? -1 : (!strcmp(e, "deep") ? 0 : (!strcmp(e, "mid") ? 1 : 2));
    }
    const long total_ctas = (long)grid.x * grid.y * grid.z;
    const int stages_mode = forced >= 0 ? forced : (total_ctas <= 160 ? 0 : 2);
    if (op == OP_TF32) launch_variants<OP_TF32, 0>(pl.cluster, stages_mode, bn, ksplit, ma, mb, p, grid, s);
    else if (op == OP_F16) {
        if (a.nin.on) launch_variants<OP_F16, 1>(pl.cluster, stages_mode, bn, ksplit, ma, mb, p, grid, s);
        else launch_variants<OP_F16, 0>(pl.cluster, stages_mode, bn, ksplit, ma, mb, p, grid, s);
    } else {
        if (a.nin.on) launch_variants<OP_F16N, 1>(pl.cluster, stages_mode, bn, ksplit, ma, mb, p, grid, s);
        else launch_variants<OP_F16N, 0>(pl.cluster, stages_mode, bn, ksplit, ma, mb, p, grid, s);
    }
    if (use_ws) {
        const int cq = (p.outC + 3) / 4;
        THA4_REQUIRE(cq <= 256, "split-K reduce: Cout <= 1024");
        const int PL = 256 / cq;
        const long MHW = (long)p.MH * p.MW;
        // pixels per thread: enough CTAs to fill the GPU on the small layers split-K exists for
        const int ppt = (int)std::max<long>(1, std::min<long>(16, MHW * p.N * cw.nphase / ((long)PL * 296)));
        dim3 rgrid(ceil_div(MHW, (long)PL * ppt), p.N * cw.nphase);
        splitk_reduce_kernel<<<rgrid, 256, 0, s>>>(p, cw.nphase, ppt);
        THA4_LAUNCH_CHECK();
    }
}

}  // namespace tha4
