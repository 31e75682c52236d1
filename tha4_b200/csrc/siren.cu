// Distilled student networks: SirenFaceMorpher00 (siren_face_morpher_00.py:28-51) and SirenMorpher03
// (siren_morpher_03.py:42-145) as fused per-level MLP kernels.
//
// A CTA owns 64 consecutive pixels of one image row and runs the whole layer chain of its level on them; hidden
// activations never leave shared memory (fp16), weights (pre-scaled by omega_0 = 30, fp16, zero-padded to
// multiples of 32) stream from L2 through a cp.async ring, products run on tensor cores (mma.sync m16n8k16, fp32
// accumulate), sin(30 x) is evaluated in registers with a 2-constant Cody-Waite reduction + MUFU.SIN.
// The tiled pose channels and the xy position channels (siren_morpher_03.py:92-105) are never materialised: a 1x1
// conv sees the pose as a per-sample bias (one GEMV per forward), and xy enters as two FMAs per output.
// Level hand-off (bilinear x2, siren_morpher_03.py:121) goes through fp16 NHWC tensors in HBM because it needs a
// cross-tile halo; the 512x512 level ends in the fused tail: 1x1 head -> grid_sample -> blend -> 5 outputs.
#include "siren.cuh"
#include "gridsample.cuh"
#include <cuda_fp16.h>
#include "profiler.cuh"

namespace tha4 {
namespace {

constexpr int TP = 64;          // pixels per CTA
constexpr int NTHREADS = 256;
constexpr int WCH = 32;         // weight K-chunk (halves)
constexpr int WPITCH = WCH + 8; // smem pitch of a staged weight row (halves): conflict-free fragment loads

__device__ __forceinline__ float siren_sin(float x) {
    const float k = rintf(x * 0.15915494309189535f);
    float r = fmaf(-k, 6.2831854820251465f, x);
    r = fmaf(-k, -1.7484555e-7f, r);
    return __sinf(r);
}

__global__ void siren_sin_kernel(const float* __restrict__ x, long n, float* __restrict__ y) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = siren_sin(x[i]);
}

__device__ __forceinline__ void cp_async16h(void* smem_dst, const void* gmem_src) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"(sa), "l"(gmem_src));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" :: "n"(N)); }

__device__ __forceinline__ void mma_f16(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[mt][nt] += actIn[64 x KPAD] * Wg[NPAD x KPAD]^T for this warp's 32 x (NPAD/4) tile.
// Warp layout 2 (M) x 4 (N).  Ends with all cp.async drained and a CTA barrier.
template <int KPAD, int NPAD, int STAGES>
__device__ __forceinline__ void mma_layer(const __half* actIn, const __half* __restrict__ Wg, __half* wst,
                                          float (&acc)[2][NPAD / 32][4]) {
    constexpr int NT = NPAD / 32;
    constexpr int NK = KPAD / WCH;
    constexpr int APITCH = KPAD + 8;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 1, wn = warp >> 1, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[mt][nt][k] = 0.0f;
    auto load_chunk = [&](int stage, int kc) {
        for (int i = tid; i < NPAD * 4; i += NTHREADS) {
            const int n = i >> 2, c = i & 3;
            cp_async16h(wst + ((size_t)stage * NPAD + n) * WPITCH + c * 8, Wg + (size_t)n * KPAD + kc * WCH + c * 8);
        }
    };
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < NK) load_chunk(s, s);
        cp_commit();
    }
#pragma unroll 1
    for (int kc = 0; kc < NK; ++kc) {
        cp_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nxt = kc + STAGES - 1;
            if (nxt < NK) load_chunk(nxt % STAGES, nxt);
            cp_commit();
        }
        const __half* ws = wst + (size_t)(kc % STAGES) * NPAD * WPITCH;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const int k0 = kc * WCH + ks * 16;
            unsigned a[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const __half* ap = actIn + (wm * 32 + mt * 16 + g) * APITCH + k0 + 2 * t;
                a[mt][0] = *reinterpret_cast<const unsigned*>(ap);
                a[mt][1] = *reinterpret_cast<const unsigned*>(ap + 8 * APITCH);
                a[mt][2] = *reinterpret_cast<const unsigned*>(ap + 8);
                a[mt][3] = *reinterpret_cast<const unsigned*>(ap + 8 * APITCH + 8);
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const __half* bp = ws + ((wn * NT + nt) * 8 + g) * WPITCH + ks * 16 + 2 * t;
                const unsigned b0 = *reinterpret_cast<const unsigned*>(bp);
                const unsigned b1 = *reinterpret_cast<const unsigned*>(bp + 8);
                mma_f16(acc[0][nt], a[0], b0, b1);
                mma_f16(acc[1][nt], a[1], b0, b1);
            }
        }
    }
    cp_wait<0>();
    __syncthreads();
}

// actOut[row][col] = half(sin(acc + bias[col] + wxy[col][0]*x(row) + wxy[col][1]*y))
template <int NPAD>
__device__ __forceinline__ void sine_epilogue(const float (&acc)[2][NPAD / 32][4], const float* __restrict__ bias,
                                              const float* __restrict__ wxy, const float* xs, float yv, __half* actOut) {
    constexpr int NT = NPAD / 32;
    constexpr int OPITCH = NPAD + 8;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp & 1, wn = warp >> 1, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int col = (wn * NT + nt) * 8 + 2 * t;
        const float b0 = bias[col], b1 = bias[col + 1];
        float wx0 = 0.f, wy0 = 0.f, wx1 = 0.f, wy1 = 0.f;
        if (wxy) { wx0 = wxy[2 * col]; wy0 = wxy[2 * col + 1]; wx1 = wxy[2 * col + 2]; wy1 = wxy[2 * col + 3]; }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = wm * 32 + mt * 16 + g + h * 8;
                float v0 = acc[mt][nt][2 * h] + b0, v1 = acc[mt][nt][2 * h + 1] + b1;
                if (wxy) {
                    const float xv = xs[row];
                    v0 += wx0 * xv + wy0 * yv;
                    v1 += wx1 * xv + wy1 * yv;
                }
                *reinterpret_cast<__half2*>(actOut + row * OPITCH + col) = __floats2half2_rn(siren_sin(v0), siren_sin(v1));
            }
    }
}

// First layer of a chain whose only inputs are xy + pose (level 0, face): pure elementwise.
template <int NPAD>
__device__ __forceinline__ void first_layer_xy(const float* __restrict__ pb, const float* __restrict__ wxy, const float* xs,
                                               float yv, __half* actOut) {
    constexpr int OPITCH = NPAD + 8;
    for (int i = threadIdx.x; i < TP * (NPAD / 2); i += NTHREADS) {
        const int row = i / (NPAD / 2), col = (i - row * (NPAD / 2)) * 2;
        const float xv = xs[row];
        const float v0 = pb[col] + wxy[2 * col] * xv + wxy[2 * col + 1] * yv;
        const float v1 = pb[col + 1] + wxy[2 * col + 2] * xv + wxy[2 * col + 3] * yv;
        *reinterpret_cast<__half2*>(actOut + row * OPITCH + col) = __floats2half2_rn(siren_sin(v0), siren_sin(v1));
    }
}

// actIn[pix][c] = bilinear x2 upsample (align_corners=False) of prev [R/2][R/2][CP] fp16 NHWC at row y, x0..x0+63
template <int CP>
__device__ __forceinline__ void upsample_prologue(const __half* __restrict__ prev, int R, int y, int x0, __half* actIn) {
    constexpr int APITCH = CP + 8;
    const int Rh = R >> 1;
    const LerpTap ty = lerp_locate(y, 0.5f, Rh);
    for (int i = threadIdx.x; i < TP * (CP / 8); i += NTHREADS) {
        const int px = i / (CP / 8), cg = i - px * (CP / 8);
        const LerpTap tx = lerp_locate(x0 + px, 0.5f, Rh);
        const __half* p00 = prev + ((size_t)ty.i0 * Rh + tx.i0) * CP + cg * 8;
        const __half* p01 = prev + ((size_t)ty.i0 * Rh + tx.i1) * CP + cg * 8;
        const __half* p10 = prev + ((size_t)ty.i1 * Rh + tx.i0) * CP + cg * 8;
        const __half* p11 = prev + ((size_t)ty.i1 * Rh + tx.i1) * CP + cg * 8;
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(p00)), b = __ldg(reinterpret_cast<const uint4*>(p01));
        const uint4 c = __ldg(reinterpret_cast<const uint4*>(p10)), d = __ldg(reinterpret_cast<const uint4*>(p11));
        const __half2* ah = reinterpret_cast<const __half2*>(&a); const __half2* bh = reinterpret_cast<const __half2*>(&b);
        const __half2* ch = reinterpret_cast<const __half2*>(&c); const __half2* dh = reinterpret_cast<const __half2*>(&d);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 fa = __half22float2(ah[k]), fb = __half22float2(bh[k]), fc = __half22float2(ch[k]), fd = __half22float2(dh[k]);
            const float r0 = ty.l0 * (tx.l0 * fa.x + tx.l1 * fb.x) + ty.l1 * (tx.l0 * fc.x + tx.l1 * fd.x);
            const float r1 = ty.l0 * (tx.l0 * fa.y + tx.l1 * fb.y) + ty.l1 * (tx.l0 * fc.y + tx.l1 * fd.y);
            oh[k] = __floats2half2_rn(r0, r1);
        }
        *reinterpret_cast<uint4*>(actIn + px * APITCH + cg * 8) = o;
    }
}

// copy a [64][NPAD] fp16 smem tile (pitch NPAD+8) to NHWC global rows
template <int NPAD>
__device__ __forceinline__ void store_tile(const __half* act, __half* __restrict__ dst) {
    constexpr int OPITCH = NPAD + 8;
    for (int i = threadIdx.x; i < TP * (NPAD / 8); i += NTHREADS) {
        const int px = i / (NPAD / 8), cg = i - px * (NPAD / 8);
        *reinterpret_cast<uint4*>(dst + (size_t)px * NPAD + cg * 8) = *reinterpret_cast<const uint4*>(act + px * OPITCH + cg * 8);
    }
}

// Linear head (no sine): out[64][8] fp32 = act[64 x KPAD] * Wh[8 x KPAD]^T + bias.  Warps 0..3 take one m-tile each.
template <int KPAD>
__device__ __forceinline__ void head_layer(const __half* act, const __half* __restrict__ Wh, const float* __restrict__ bias,
                                           float* outs /*[64][8]*/) {
    constexpr int APITCH = KPAD + 8;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    if (warp < 4) {
        float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k0 = 0; k0 < KPAD; k0 += 16) {
            unsigned a[4];
            const __half* ap = act + (warp * 16 + g) * APITCH + k0 + 2 * t;
            a[0] = *reinterpret_cast<const unsigned*>(ap);
            a[1] = *reinterpret_cast<const unsigned*>(ap + 8 * APITCH);
            a[2] = *reinterpret_cast<const unsigned*>(ap + 8);
            a[3] = *reinterpret_cast<const unsigned*>(ap + 8 * APITCH + 8);
            const __half* bp = Wh + (size_t)g * KPAD + k0 + 2 * t;
            const unsigned b0 = __ldg(reinterpret_cast<const unsigned*>(bp));
            const unsigned b1 = __ldg(reinterpret_cast<const unsigned*>(bp + 8));
            mma_f16(c, a, b0, b1);
        }
        const int row = warp * 16 + g, col = 2 * t;
        outs[row * 8 + col] = c[0] + bias[col];
        outs[row * 8 + col + 1] = c[1] + bias[col + 1];
        outs[(row + 8) * 8 + col] = c[2] + bias[col];
        outs[(row + 8) * 8 + col + 1] = c[3] + bias[col + 1];
    }
    __syncthreads();
}

struct LayerW {
    const __half* W;      // [NPAD][KPAD], x30
    const float* bias;    // [NPAD] (x30) -- or per-sample bias [B][NPAD] for first layers
    const float* wxy;     // [NPAD][2] (x30) or nullptr
};

// dynamic smem layout helper
template <int AMAX, int NMAXW, int STAGES>
struct Smem {
    static constexpr size_t act_halves = (size_t)TP * (AMAX + 8);
    static constexpr size_t w_halves = (size_t)STAGES * NMAXW * WPITCH;
    static constexpr size_t bytes = (2 * act_halves + w_halves) * sizeof(__half) + TP * sizeof(float) + TP * 8 * sizeof(float);
};

// ---------------------------------------------------------------------------------------------- body level 0
// 128x128: (xy,pose) -> 360 -> 360 -> 180, padded 384/384/192.  Output fp16 NHWC [B,128,128,192].
__global__ void __launch_bounds__(NTHREADS, 1) siren_body_l0_kernel(LayerW l0, LayerW l1, LayerW l2, int pb_ld,
                                                                     const float* __restrict__ base, int R,
                                                                     __half* __restrict__ out) {
    using SM = Smem<384, 384, 2>;
    extern __shared__ __align__(16) unsigned char smraw[];
    __half* actA = reinterpret_cast<__half*>(smraw);
    __half* actB = actA + SM::act_halves;
    __half* wst = actB + SM::act_halves;
    float* xs = reinterpret_cast<float*>(wst + SM::w_halves);
    const int tiles_per_row = R / TP;
    const int n = blockIdx.x / (R * tiles_per_row);
    const int rem = blockIdx.x - n * (R * tiles_per_row);
    const int y = rem / tiles_per_row, x0 = (rem - y * tiles_per_row) * TP;
    if (threadIdx.x < TP) xs[threadIdx.x] = base[x0 + threadIdx.x];
    __syncthreads();
    const float yv = base[y];
    first_layer_xy<384>(l0.bias + (size_t)n * pb_ld, l0.wxy, xs, yv, actA);
    {
        float acc[2][12][4];
        mma_layer<384, 384, 2>(actA, l1.W, wst, acc);
        sine_epilogue<384>(acc, l1.bias, nullptr, xs, yv, actB);
    }
    {
        float acc[2][6][4];
        mma_layer<384, 192, 2>(actB, l2.W, wst, acc);
        sine_epilogue<192>(acc, l2.bias, nullptr, xs, yv, actA);
    }
    __syncthreads();
    store_tile<192>(actA, out + (((size_t)n * R + y) * R + x0) * 192);
}

// ---------------------------------------------------------------------------------------------- body level 1
// 256x256: (up(180), xy, pose) -> 180 -> 180 -> 90, padded 192/192/96.  Output fp16 NHWC [B,256,256,96].
__global__ void __launch_bounds__(NTHREADS, 2) siren_body_l1_kernel(LayerW l0, LayerW l1, LayerW l2, int pb_ld,
                                                                     const float* __restrict__ base, int R,
                                                                     const __half* __restrict__ prev, __half* __restrict__ out) {
    using SM = Smem<192, 192, 3>;
    extern __shared__ __align__(16) unsigned char smraw[];
    __half* actA = reinterpret_cast<__half*>(smraw);
    __half* actB = actA + SM::act_halves;
    __half* wst = actB + SM::act_halves;
    float* xs = reinterpret_cast<float*>(wst + SM::w_halves);
    const int tiles_per_row = R / TP;
    const int n = blockIdx.x / (R * tiles_per_row);
    const int rem = blockIdx.x - n * (R * tiles_per_row);
    const int y = rem / tiles_per_row, x0 = (rem - y * tiles_per_row) * TP;
    if (threadIdx.x < TP) xs[threadIdx.x] = base[x0 + threadIdx.x];
    upsample_prologue<192>(prev + (size_t)n * (R / 2) * (R / 2) * 192, R, y, x0, actA);
    __syncthreads();
    const float yv = base[y];
    {
        float acc[2][6][4];
        mma_layer<192, 192, 3>(actA, l0.W, wst, acc);
        sine_epilogue<192>(acc, l0.bias + (size_t)n * pb_ld, l0.wxy, xs, yv, actB);
    }
    {
        float acc[2][6][4];
        mma_layer<192, 192, 3>(actB, l1.W, wst, acc);
        sine_epilogue<192>(acc, l1.bias, nullptr, xs, yv, actA);
    }
    {
        float acc[2][3][4];
        mma_layer<192, 96, 3>(actA, l2.W, wst, acc);
        sine_epilogue<96>(acc, l2.bias, nullptr, xs, yv, actB);
    }
    __syncthreads();
    store_tile<96>(actB, out + (((size_t)n * R + y) * R + x0) * 96);
}

// ---------------------------------------------------------------------------------------------- body level 2 + tail
// 512x512: (up(90), xy, pose) -> 90 -> 90 -> 90 -> head 7 -> grid_sample + blend (siren_morpher_03.py:125-139).
__global__ void __launch_bounds__(NTHREADS, 3) siren_body_l2_kernel(LayerW l0, LayerW l1, LayerW l2, LayerW head, int pb_ld,
                                                                     const float* __restrict__ base, int R,
                                                                     const __half* __restrict__ prev, ImgView image,
                                                                     float* __restrict__ o_blend, float* __restrict__ o_alpha,
                                                                     float* __restrict__ o_color, float* __restrict__ o_warp,
                                                                     float* __restrict__ o_grid) {
    using SM = Smem<96, 96, 3>;
    extern __shared__ __align__(16) unsigned char smraw[];
    __half* actA = reinterpret_cast<__half*>(smraw);
    __half* actB = actA + SM::act_halves;
    __half* wst = actB + SM::act_halves;
    float* xs = reinterpret_cast<float*>(wst + SM::w_halves);
    float* ho = xs + TP;
    const int tiles_per_row = R / TP;
    const int n = blockIdx.x / (R * tiles_per_row);
    const int rem = blockIdx.x - n * (R * tiles_per_row);
    const int y = rem / tiles_per_row, x0 = (rem - y * tiles_per_row) * TP;
    if (threadIdx.x < TP) xs[threadIdx.x] = base[x0 + threadIdx.x];
    upsample_prologue<96>(prev + (size_t)n * (R / 2) * (R / 2) * 96, R, y, x0, actA);
    __syncthreads();
    const float yv = base[y];
    {
        float acc[2][3][4];
        mma_layer<96, 96, 3>(actA, l0.W, wst, acc);
        sine_epilogue<96>(acc, l0.bias + (size_t)n * pb_ld, l0.wxy, xs, yv, actB);
        mma_layer<96, 96, 3>(actB, l1.W, wst, acc);
        sine_epilogue<96>(acc, l1.bias, nullptr, xs, yv, actA);
        mma_layer<96, 96, 3>(actA, l2.W, wst, acc);
        sine_epilogue<96>(acc, l2.bias, nullptr, xs, yv, actB);
    }
    __syncthreads();
    head_layer<96>(actB, head.W, head.bias, ho);
    // tail: thread (c, px) handles channel c of pixel px
    const int px = threadIdx.x & (TP - 1), c = threadIdx.x >> 6;
    const float* o = ho + px * 8;   // grid_change(0,1) alpha(2) colour(3..6)
    const int x = x0 + px;
    const GsTap t = gs_locate(xs[px], yv, o[0], o[1], R, R);
    float w[1];
    gs_sample<1>(image.p + n * image.sn + c * image.sc, 0, image.sh, R, R, t, w);
    const float alpha = o[2], col = o[3 + c];
    const size_t plane = (size_t)R * R, pix = (size_t)y * R + x;
    o_blend[((size_t)n * 4 + c) * plane + pix] = (1.0f - alpha) * w[0] + alpha * col;
    o_color[((size_t)n * 4 + c) * plane + pix] = col;
    o_warp[((size_t)n * 4 + c) * plane + pix] = w[0];
    if (c == 0) o_alpha[(size_t)n * plane + pix] = alpha;
    if (c >= 2) o_grid[((size_t)n * 2 + (c - 2)) * plane + pix] = o[c - 2];
}

// ---------------------------------------------------------------------------------------------- face
// 128x128: (xy, pose39) -> 128 x8 sine layers -> 4.  Output fp32 NCHW [B,4,128,128].
struct FaceLayers { LayerW l[8]; LayerW head; };
__global__ void __launch_bounds__(NTHREADS, 2) siren_face_kernel(FaceLayers L, int pb_ld, const float* __restrict__ base, int R,
                                                                  float* __restrict__ out) {
    using SM = Smem<128, 128, 3>;
    extern __shared__ __align__(16) unsigned char smraw[];
    __half* actA = reinterpret_cast<__half*>(smraw);
    __half* actB = actA + SM::act_halves;
    __half* wst = actB + SM::act_halves;
    float* xs = reinterpret_cast<float*>(wst + SM::w_halves);
    float* ho = xs + TP;
    const int tiles_per_row = R / TP;
    const int n = blockIdx.x / (R * tiles_per_row);
    const int rem = blockIdx.x - n * (R * tiles_per_row);
    const int y = rem / tiles_per_row, x0 = (rem - y * tiles_per_row) * TP;
    if (threadIdx.x < TP) xs[threadIdx.x] = base[x0 + threadIdx.x];
    __syncthreads();
    const float yv = base[y];
    first_layer_xy<128>(L.l[0].bias + (size_t)n * pb_ld, L.l[0].wxy, xs, yv, actA);
    __half* in = actA;
    __half* ot = actB;
    float acc[2][4][4];
#pragma unroll 1
    for (int i = 1; i < 8; ++i) {
        mma_layer<128, 128, 3>(in, L.l[i].W, wst, acc);
        sine_epilogue<128>(acc, L.l[i].bias, nullptr, xs, yv, ot);
        __half* tmp = in; in = ot; ot = tmp;
    }
    __syncthreads();
    head_layer<128>(in, L.head.W, L.head.bias, ho);
    const int px = threadIdx.x & (TP - 1), c = threadIdx.x >> 6;
    out[(((size_t)n * 4 + c) * R + y) * R + x0 + px] = ho[px * 8 + c];
}

// ---------------------------------------------------------------------------------------------- weight packing
// W30[n][k] = half(scale * W[n][k0 + k]) for k < kreal, zero padded to [NPAD][KPAD]
__global__ void pack_w_kernel(const float* __restrict__ W, int cin_total, int k0, int kreal, int nreal, int KPAD, int NPAD,
                              float scale, __half* __restrict__ dst) {
    const int total = NPAD * KPAD;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = i / KPAD, k = i - n * KPAD;
        float v = 0.0f;
        if (n < nreal && k < kreal) v = scale * W[(size_t)n * cin_total + k0 + k];
        dst[i] = __float2half_rn(v);
    }
}
// dst[n][j] = scale * W[n][k0 + j]  (fp32, [NPAD][cols], zero padded rows)
__global__ void pack_cols_kernel(const float* __restrict__ W, int cin_total, int k0, int cols, int nreal, int NPAD, float scale,
                                 float* __restrict__ dst) {
    const int total = NPAD * cols;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = i / cols, j = i - n * cols;
        dst[i] = (n < nreal) ? scale * W[(size_t)n * cin_total + k0 + j] : 0.0f;
    }
}
__global__ void pack_vec_kernel(const float* __restrict__ b, int nreal, int NPAD, float scale, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < NPAD) dst[i] = (i < nreal) ? scale * b[i] : 0.0f;
}

template <typename T> T* dmalloc(size_t n) {      // owned by the loading net (AllocSink)
    return reinterpret_cast<T*>(tracked_malloc(std::max<size_t>(n, 1) * sizeof(T)));
}

const TensorRef& get(const StateDict& sd, const std::string& k) {
    auto it = sd.find(k);
    if (it == sd.end()) throw std::runtime_error("tha4: state_dict is missing key '" + k + "'");
    return it->second;
}

}  // namespace

// Packs one sine layer.  feat: number of leading "feature" input channels that go through the MMA (0: none).
void SirenLayer::pack(const StateDict& sd, const std::string& prefix, int feat, int pose, int kpad, int npad, float scale,
                      cudaStream_t s) {
    const TensorRef& w = get(sd, prefix + ".weight");
    const TensorRef& b = get(sd, prefix + ".bias");
    const int nreal = (int)w.shape[0], cin = (int)w.shape[1];
    const bool first = pose > 0;
    THA4_REQUIRE(cin == feat + (first ? 2 + pose : 0), "siren layer input channels: " + prefix);
    THA4_REQUIRE(nreal <= npad && feat <= kpad, "siren layer padding: " + prefix);
    N = nreal; NPAD = npad; KPAD = kpad; P = pose;
    if (feat > 0) {
        pack_w_kernel<<<64, 256, 0, s>>>(w.p, cin, 0, feat, nreal, kpad, npad, scale, reinterpret_cast<__half*>(W));
        THA4_LAUNCH_CHECK();
    }
    pack_vec_kernel<<<ceil_div(npad, 128), 128, 0, s>>>(b.p, nreal, npad, scale, bias);
    THA4_LAUNCH_CHECK();
    if (first) {
        pack_cols_kernel<<<16, 256, 0, s>>>(w.p, cin, feat, 2, nreal, npad, scale, wxy);
        THA4_LAUNCH_CHECK();
        pack_cols_kernel<<<64, 256, 0, s>>>(w.p, cin, feat + 2, pose, nreal, npad, scale, wpose);
        THA4_LAUNCH_CHECK();
    }
}

// allocates `count` layers' buffers back to back (count = 1: one network; the bank: one per character)
static void alloc_layer(SirenLayer& l, int feat, int pose, int kpad, int npad, size_t count) {
    if (feat > 0) l.W = dmalloc<__half>(count * npad * kpad);
    l.bias = dmalloc<float>(count * npad);
    if (pose > 0) {
        l.wxy = dmalloc<float>(count * npad * 2);
        l.wpose = dmalloc<float>(count * npad * pose);
    }
    l.NPAD = npad; l.KPAD = kpad; l.P = pose;
}

void SirenLayer::load(const StateDict& sd, const std::string& prefix, int feat, int pose, int kpad, int npad, float scale,
                      cudaStream_t s) {
    alloc_layer(*this, feat, pose, kpad, npad, 1);
    pack(sd, prefix, feat, pose, kpad, npad, scale, s);
}

// per-sample bias of a first layer: pb[n][:] = scale*b + (scale*Wpose) . pose[n]
static float* pose_bias(Runtime& rt, const SirenLayer& l, const float* pose, int pose_ld, int B) {
    float* pb = rt.persist->alloc((size_t)B * l.NPAD);
    linear_forward(pose, pose_ld, B, l.P, l.wpose, l.bias, l.NPAD, 0, pb, l.NPAD, rt.stream);
    return pb;
}

// The same for a bank: pb[n][:] = bias[c] + wpose[c] . pose[n] with c = char_of[n].  One block per sample, one warp per
// output at a time, in the summation order of linear_forward (lane-strided FMAs, xor-shuffle tree, bias last), so a
// sample's pb is bit-identical to what its character's own network computes.
__global__ void __launch_bounds__(256) pose_bias_bank_kernel(const float* __restrict__ pose, int pose_ld, int I,
                                                             const float* __restrict__ wpose, const float* __restrict__ bias, int O,
                                                             const int* __restrict__ char_of, float* __restrict__ pb) {
    const int n = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = char_of[n];
    const float* xr = pose + (long)n * pose_ld;
    for (int o = warp; o < O; o += 8) {
        const float* wr = wpose + ((long)c * O + o) * I;
        float acc = 0.0f;
        for (int i = lane; i < I; i += 32) acc = fmaf(xr[i], wr[i], acc);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (lane == 0) pb[(long)n * O + o] = acc + bias[(long)c * O + o];
    }
}
static float* pose_bias_bank(Runtime& rt, const SirenLayer& l, const float* pose, int pose_ld, int B, const int* char_of) {
    float* pb = rt.persist->alloc((size_t)B * l.NPAD);
    pose_bias_bank_kernel<<<B, 256, 0, rt.stream>>>(pose, pose_ld, l.P, l.wpose, l.bias, l.NPAD, char_of, pb);
    THA4_LAUNCH_CHECK();
    return pb;
}

// dst[n] = images[char_of[n]] ([4,512,512] fp32 each); round_f16: through fp16, as an fp16 input image would arrive
__global__ void gather_images_kernel(const float4* __restrict__ images, const int* __restrict__ char_of, long per_image4,
                                     int round_f16, float4* __restrict__ dst) {
    const int n = blockIdx.y;
    const float4* src = images + (long)char_of[n] * per_image4;
    float4* d = dst + (long)n * per_image4;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < per_image4; i += (long)gridDim.x * blockDim.x) {
        float4 v = __ldg(src + i);
        if (round_f16) {
            v.x = __half2float(__float2half_rn(v.x)); v.y = __half2float(__float2half_rn(v.y));
            v.z = __half2float(__float2half_rn(v.z)); v.w = __half2float(__float2half_rn(v.w));
        }
        d[i] = v;
    }
}

static LayerW lw(const SirenLayer& l, const float* bias_override = nullptr) {
    LayerW r;
    r.W = reinterpret_cast<const __half*>(l.W);
    r.bias = bias_override ? bias_override : l.bias;
    r.wxy = l.wxy;
    return r;
}

template <typename K> static void set_smem(K kernel, size_t bytes) {
    THA4_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

void siren_sine(const float* x, long n, float* y, cudaStream_t s) {
    siren_sin_kernel<<<(int)std::min<long>(ceil_div(n, 256), 1024), 256, 0, s>>>(x, n, y);
    THA4_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------------ one level
void siren_level(Runtime& rt, const SirenLevelArgs& a) {
    THA4_REQUIRE(a.mode >= 0 && a.mode <= 3 && a.nl >= 1 && a.L != nullptr, "siren level: mode / layers");
    const SirenLayer* L = a.L;
    const bool elementwise = (a.mode == 0 || a.mode == 3);
    if (a.tc) {       // TMA + wgmma path (siren_tc.cu): one persistent kernel per level
        SirenTcPlan plan;
        int j = 0;
        for (int i = elementwise ? 1 : 0; i < a.nl; ++i, ++j) plan.add(L[i], a.nb[j], 1, (!elementwise && i == 0) ? 1 : 0);
        if (a.head) plan.add(*a.head, a.nb[j], 0, 0);
        SirenTcLevel lv;
        lv.R = a.R; lv.B = a.B;
        if (elementwise) { lv.e_npad = L[0].NPAD; lv.e_pb = a.pb; lv.e_pb_ld = L[0].NPAD; lv.e_wxy = L[0].wxy; }
        else { lv.f_pb = a.pb; lv.f_pb_ld = L[0].NPAD; lv.f_wxy = L[0].wxy; lv.prev = a.prev; lv.prev_c = a.prev_c; }
        lv.out = a.out; lv.out_c = L[a.nl - 1].NPAD;
        lv.image = a.image;
        if (a.outputs) for (int i = 0; i < 5; ++i) lv.o[i] = a.outputs[i];
        lv.o_f16 = a.out_f16;
        lv.face_out = a.face_out;
        lv.head_bias = a.head ? a.head->bias : nullptr;
        lv.char_of = a.char_of; lv.chars = a.chars; lv.head_cs = a.head ? a.head->NPAD : 0;
        siren_tc_run(rt, a.mode, plan, lv);
        return;
    }
    THA4_REQUIRE(a.char_of == nullptr, "siren level: a character bank needs the wgmma kernels (option siren_tc = 1); the mma.sync kernels take one character's weights");
    // mma.sync path: one kernel per level, compiled for the production layer shapes only
    THA4_REQUIRE(!a.out_f16, "siren body: f16 outputs need the tensor-core path (option siren_tc)");
    auto shape = [&](int i, int kpad, int npad) { return a.L[i].KPAD == kpad && a.L[i].NPAD == npad; };
    static const int kR[4] = {128, 256, 512, 128};
    THA4_REQUIRE(a.R == kR[a.mode], "siren level (mma.sync): resolution of mode " + std::to_string(a.mode));
    const int B = a.B, R = a.R;
    cudaStream_t s = rt.stream;
    ProfScope prof(PROF_SIREN, s);
    if (a.mode == 0) {
        THA4_REQUIRE(a.nl == 3 && !a.head && L[0].NPAD == 384 && shape(1, 384, 384) && shape(2, 384, 192) && a.out,
                     "siren level 0 (mma.sync): production shapes only");
        using SM0 = Smem<384, 384, 2>;
        THA4_ENSURE_SMEM(siren_body_l0_kernel, SM0::bytes);
        siren_body_l0_kernel<<<B * R * (R / TP), NTHREADS, SM0::bytes, s>>>(lw(L[0], a.pb), lw(L[1]), lw(L[2]), L[0].NPAD,
                                                                          base_grid_table(R), R, a.out);
    } else if (a.mode == 1) {
        THA4_REQUIRE(a.nl == 3 && !a.head && shape(0, 192, 192) && shape(1, 192, 192) && shape(2, 192, 96) && a.prev_c == 192 && a.out,
                     "siren level 1 (mma.sync): production shapes only");
        using SM1 = Smem<192, 192, 3>;
        THA4_ENSURE_SMEM(siren_body_l1_kernel, SM1::bytes);
        siren_body_l1_kernel<<<B * R * (R / TP), NTHREADS, SM1::bytes, s>>>(lw(L[0], a.pb), lw(L[1]), lw(L[2]), L[0].NPAD,
                                                                          base_grid_table(R), R, a.prev, a.out);
    } else if (a.mode == 2) {
        THA4_REQUIRE(a.nl == 3 && a.head && a.head->KPAD == 96 && a.head->NPAD == 8 && shape(0, 96, 96) && shape(1, 96, 96) &&
                     shape(2, 96, 96) && a.prev_c == 96 && a.outputs, "siren level 2 (mma.sync): production shapes only");
        using SM2 = Smem<96, 96, 3>;
        THA4_ENSURE_SMEM(siren_body_l2_kernel, SM2::bytes);
        siren_body_l2_kernel<<<B * R * (R / TP), NTHREADS, SM2::bytes, s>>>(lw(L[0], a.pb), lw(L[1]), lw(L[2]), lw(*a.head), L[0].NPAD,
                                                                          base_grid_table(R), R, a.prev, a.image, a.outputs[0],
                                                                          a.outputs[1], a.outputs[2], a.outputs[3], a.outputs[4]);
    } else {
        bool ok = a.nl == 8 && a.head && a.head->KPAD == 128 && a.head->NPAD == 8 && L[0].NPAD == 128 && a.face_out;
        for (int i = 1; ok && i < 8; ++i) ok = shape(i, 128, 128);
        THA4_REQUIRE(ok, "siren face (mma.sync): production shapes only");
        FaceLayers FL;
        FL.l[0] = lw(L[0], a.pb);
        for (int i = 1; i < 8; ++i) FL.l[i] = lw(L[i]);
        FL.head = lw(*a.head);
        using SM = Smem<128, 128, 3>;
        THA4_ENSURE_SMEM(siren_face_kernel, SM::bytes);
        siren_face_kernel<<<B * R * (R / TP), NTHREADS, SM::bytes, s>>>(FL, L[0].NPAD, base_grid_table(R), R, a.face_out);
    }
    THA4_LAUNCH_CHECK();
}

void siren_test_level(Runtime& rt, bool tc, int mode, const StateDict& sd, int n_layers, bool has_head, int pose_dim,
                      const int* npad, const int* nb, const float* pose, int pose_ld, int B, const __half* prev, int prev_c,
                      const float* image, bool out_f16, void* const* outputs) {
    THA4_REQUIRE(mode >= 0 && mode <= 3, "siren level: mode must be 0..3");
    THA4_REQUIRE(n_layers >= 1 && n_layers <= 8 && pose_dim >= 1 && pose_ld >= pose_dim && B >= 1, "siren level: arguments");
    static const int kR[4] = {128, 256, 512, 128};
    const bool elementwise = (mode == 0 || mode == 3);
    THA4_REQUIRE(elementwise ? n_layers >= (has_head ? 1 : 2) : (prev != nullptr && prev_c > 0), "siren level: layers / previous level");
    cudaStream_t s = rt.stream;
    AllocSink sink;                        // frees the packed layers on return
    SirenLayer L[8], head;
    {
        SinkScope own(&sink);
        for (int i = 0; i < n_layers; ++i) {
            const std::string key = "layer." + std::to_string(i);
            const int cin = (int)get(sd, key + ".weight").shape[1];
            if (i == 0) L[0].load(sd, key, cin - 2 - pose_dim, pose_dim, elementwise ? 16 : prev_c, npad[0], 30.0f, s);
            else L[i].load(sd, key, cin, 0, npad[i - 1], npad[i], 30.0f, s);
        }
        if (has_head) head.load(sd, "head", (int)get(sd, "head.weight").shape[1], 0, npad[n_layers - 1], 8, 1.0f, s);
    }
    SirenLevelArgs a;
    a.tc = tc; a.mode = mode; a.R = kR[mode]; a.B = B;
    a.L = L; a.nl = n_layers; a.head = has_head ? &head : nullptr; a.nb = nb;
    a.pb = pose_bias(rt, L[0], pose, pose_ld, B);
    a.prev = prev; a.prev_c = prev_c;
    if (!has_head) a.out = reinterpret_cast<__half*>(outputs[0]);
    else if (mode == 3) a.face_out = reinterpret_cast<float*>(outputs[0]);
    else {
        THA4_REQUIRE(mode == 2 && image != nullptr, "siren level: a head needs level 2 (with the image) or the face");
        a.image = make_img(image, B, 4, 512, 512);
        a.outputs = reinterpret_cast<float* const*>(outputs);
        a.out_f16 = out_f16;
    }
    siren_level(rt, a);
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
}

// ------------------------------------------------------------------------------------------------ SirenFaceNet
// The layers of the two students: state_dict prefix, feature / pose input channels, padded K and N, pre-scale.
struct LayerSpec { std::string key; int feat, pose, kpad, npad; float scale; };
static LayerSpec face_layer_spec(int i) {          // i = 8: the head
    if (i == 8) return {"siren.last_linear", 128, 0, 128, 8, 1.0f};
    return {"siren.sine_layers." + std::to_string(i) + ".linear", i == 0 ? 0 : 128, i == 0 ? 39 : 0, 128, 128, 30.0f};
}
static LayerSpec body_layer_spec(int level, int j) {   // level 3: the head
    if (level == 3) return {"last_linear", 90, 0, 96, 8, 1.0f};
    static const int feat[3][3] = {{0, 360, 360}, {180, 180, 180}, {90, 90, 90}};
    static const int kpad[3][3] = {{32, 384, 384}, {192, 192, 192}, {96, 96, 96}};
    static const int npad[3][3] = {{384, 384, 192}, {192, 192, 96}, {96, 96, 96}};
    return {"siren_layers." + std::to_string(level) + "." + std::to_string(j) + ".linear", feat[level][j], j == 0 ? 45 : 0,
            kpad[level][j], npad[level][j], 30.0f};
}
static void load_layer(SirenLayer& l, const StateDict& sd, const LayerSpec& sp, cudaStream_t s) {
    l.load(sd, sp.key, sp.feat, sp.pose, sp.kpad, sp.npad, sp.scale, s);
}

void SirenFaceNet::load(const StateDict& sd, cudaStream_t s) {
    SinkScope own(&owned_);
    for (int i = 0; i < 8; ++i) load_layer(layers_[i], sd, face_layer_spec(i), s);
    load_layer(head_, sd, face_layer_spec(8), s);
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    loaded_ = true;
}

// the face network's one level on pb [B][128]; char_of / chars: see SirenLevelArgs (null / 0: one character)
static void face_levels(Runtime& rt, const SirenLayer* layers, const SirenLayer& head, const float* pb, int B, float* out,
                        const int* char_of, int chars) {
    static const int nb[8] = {64, 64, 64, 64, 64, 64, 64, 16};
    SirenLevelArgs a;
    a.tc = opts().siren_tc; a.mode = 3; a.R = 128; a.B = B;
    a.L = layers; a.nl = 8; a.head = &head; a.nb = nb;
    a.pb = pb;
    a.face_out = out;
    a.char_of = char_of; a.chars = chars;
    siren_level(rt, a);
}

void SirenFaceNet::forward(Runtime& rt, const float* pose, int pose_ld, int B, float* out) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    face_levels(rt, layers_, head_, pose_bias(rt, layers_[0], pose, pose_ld, B), B, out, nullptr, 0);
}

// ------------------------------------------------------------------------------------------------ SirenBodyNet
void SirenBodyNet::load(const StateDict& sd, cudaStream_t s) {
    SinkScope own(&owned_);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) load_layer(l_[i][j], sd, body_layer_spec(i, j), s);
    load_layer(head_, sd, body_layer_spec(3, 0), s);
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    loaded_ = true;
}

// the body network's three levels on the per-level pb; char_of / chars: see SirenLevelArgs (null / 0: one character)
static void body_levels(Runtime& rt, const SirenLayer (*l)[3], const SirenLayer& head, const float* const* pb, const ImgView& image,
                        float* const* outputs, bool outputs_f16, const int* char_of, int chars) {
    THA4_REQUIRE(image.H == 512 && image.W == 512 && image.C == 4, "siren body: image size");
    const int B = image.N;
    __half* f0 = reinterpret_cast<__half*>(rt.persist->alloc((size_t)B * 128 * 128 * 192 / 2));
    __half* f1 = reinterpret_cast<__half*>(rt.persist->alloc((size_t)B * 256 * 256 * 96 / 2));
    const bool tc = opts().siren_tc;
    THA4_REQUIRE(tc || !outputs_f16, "siren body: f16 outputs need the tensor-core path (option siren_tc)");
    static const int nb[4] = {96, 96, 96, 16};      // wgmma slice widths of the GEMM layers (level 2: + the head)
    for (int i = 0; i < 3; ++i) {
        SirenLevelArgs a;
        a.tc = tc; a.mode = i; a.R = 128 << i; a.B = B;
        a.L = l[i]; a.nl = 3; a.nb = nb; a.pb = pb[i];
        if (i > 0) { a.prev = i == 1 ? f0 : f1; a.prev_c = i == 1 ? 192 : 96; }
        if (i < 2) a.out = i == 0 ? f0 : f1;
        else { a.head = &head; a.image = image; a.outputs = outputs; a.out_f16 = outputs_f16; }
        a.char_of = char_of; a.chars = chars;
        siren_level(rt, a);
    }
}

void SirenBodyNet::forward(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, float* const* outputs, bool outputs_f16) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    THA4_REQUIRE(image.H == 512 && image.W == 512 && image.C == 4, "siren body: image size");
    const float* pb[3];
    for (int i = 0; i < 3; ++i) pb[i] = pose_bias(rt, l_[i][0], pose, pose_ld, image.N);
    body_levels(rt, l_, head_, pb, image, outputs, outputs_f16, nullptr, 0);
}

// ------------------------------------------------------------------------------------------------ SirenBank
SirenBank::SirenBank(int capacity) : capacity_(capacity), filled_((size_t)std::max(capacity, 0), 0) {
    THA4_REQUIRE(capacity >= 1 && capacity <= 4096, "character bank: capacity must be 1..4096");
    SinkScope own(&owned_);
    auto alloc = [&](SirenLayer& l, const LayerSpec& sp) { alloc_layer(l, sp.feat, sp.pose, sp.kpad, sp.npad, (size_t)capacity); };
    for (int i = 0; i < 8; ++i) alloc(face_[i], face_layer_spec(i));
    alloc(face_head_, face_layer_spec(8));
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) alloc(body_[i][j], body_layer_spec(i, j));
    alloc(body_head_, body_layer_spec(3, 0));
    images_ = dmalloc<float>((size_t)capacity * 4 * 512 * 512);
}

SirenLayer SirenBank::at(const SirenLayer& base, int slot) const {
    SirenLayer l = base;
    const size_t c = (size_t)slot;
    if (base.W) l.W = reinterpret_cast<__half*>(base.W) + c * base.NPAD * base.KPAD;
    l.bias = base.bias + c * base.NPAD;
    if (base.wxy) { l.wxy = base.wxy + c * base.NPAD * 2; l.wpose = base.wpose + c * base.NPAD * base.P; }
    return l;
}

void SirenBank::set_character(int slot, const StateDict& face, const StateDict& body, const float* image, cudaStream_t s) {
    THA4_REQUIRE(slot >= 0 && slot < capacity_, "character bank: slot " + std::to_string(slot) + " is not 0.." + std::to_string(capacity_ - 1));
    THA4_REQUIRE(image != nullptr, "character bank: the character's image is required");
    filled_[slot] = 0;
    auto pack = [&](const SirenLayer& base, const StateDict& sd, const LayerSpec& sp) {
        at(base, slot).pack(sd, sp.key, sp.feat, sp.pose, sp.kpad, sp.npad, sp.scale, s);
    };
    for (int i = 0; i < 8; ++i) pack(face_[i], face, face_layer_spec(i));
    pack(face_head_, face, face_layer_spec(8));
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) pack(body_[i][j], body, body_layer_spec(i, j));
    pack(body_head_, body, body_layer_spec(3, 0));
    const size_t img = (size_t)4 * 512 * 512;
    THA4_CUDA_CHECK(cudaMemcpyAsync(images_ + (size_t)slot * img, image, img * sizeof(float), cudaMemcpyDeviceToDevice, s));
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    filled_[slot] = 1;
}

void SirenBank::forward(Runtime& rt, const int* char_of_host, const float* pose, int B, void* const* outputs, bool outputs_f16) {
    THA4_REQUIRE(opts().siren_tc, "character bank: needs the wgmma student kernels (option siren_tc = 1); the mma.sync kernels take one character's weights");
    cudaStream_t s = rt.stream;
    int* char_of = reinterpret_cast<int*>(rt.persist->alloc((size_t)B));
    THA4_CUDA_CHECK(cudaMemcpyAsync(char_of, char_of_host, (size_t)B * sizeof(int), cudaMemcpyHostToDevice, s));
    // face SIREN from pose[:, :39] (mode_14.py:64-71), pasted at rows 80:208, cols 192:320 of the character's image (:72-78)
    const long face_n = (long)B * 4 * 128 * 128, per_image4 = 512L * 512;
    float* face = outputs_f16 ? rt.persist->alloc((size_t)face_n) : reinterpret_cast<float*>(outputs[5]);
    face_levels(rt, face_, face_head_, pose_bias_bank(rt, face_[0], pose, 45, B, char_of), B, face, char_of, capacity_);
    float* body_in = rt.persist->alloc((size_t)B * 4 * 512 * 512);
    gather_images_kernel<<<dim3(256, B), 256, 0, s>>>(reinterpret_cast<const float4*>(images_), char_of, per_image4, outputs_f16 ? 1 : 0,
                                                      reinterpret_cast<float4*>(body_in));
    THA4_LAUNCH_CHECK();
    copy_window(make_img(face, B, 4, 128, 128), body_in + 80 * 512 + 192, 4L * 512 * 512, 512L * 512, 512, s);
    if (outputs_f16) convert_flat_f16(face, reinterpret_cast<__half*>(outputs[5]), face_n, s);
    const float* pb[3];
    for (int i = 0; i < 3; ++i) pb[i] = pose_bias_bank(rt, body_[i][0], pose, 45, B, char_of);
    body_levels(rt, body_, body_head_, pb, make_img(body_in, B, 4, 512, 512), reinterpret_cast<float* const*>(outputs), outputs_f16,
                char_of, capacity_);
}

}  // namespace tha4
