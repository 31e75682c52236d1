// Fused "decoder tail" kernels (SURVEY.md section 8 a-T): from the last feature map of a network to every tensor
// that network returns, in one pass:
//   pending norm affine + activation (applied while staging the halo tile; zero padding is applied after it, as
//   the reference pads the activated tensor) -> 3x3 head conv(s) -> channel split -> sigmoid / tanh ->
//   affine_grid + grid_sample index math -> 4-tap bilinear gather of the RGBA image -> alpha blend(s) ->
//   coalesced NCHW stores of all outputs.
// Reference: eyebrow_decomposer_00.py:46-64, eyebrow_morphing_combiner_00.py:51-72, face_morpher_08.py:170-193,
// morpher_00.py:53-66, upscaler_02.py:84-96.
// The 3x3 head conv runs on tensor cores (mma.sync m16n8k8 TF32, M = 16 pixels of one tile row, N = 8 / 16 head
// channels, K = 9 taps x C) straight from the shared-memory halo tile; accumulators are transposed through shared
// memory so that one thread owns all head channels of one pixel for the warp / blend epilogue.  The kernel is
// HBM-bound by design: feature map + image read once, every returned tensor written once.
#include "ops.cuh"
#include "gridsample.cuh"
#include "tail_epilogue.cuh"
#include "profiler.cuh"

namespace tha4 {
namespace {

constexpr int TILE = 16, TILE_H = 8, HALO = TILE + 2, HALO_H = TILE_H + 2;    // 16 x 8 output pixels per CTA (4 warps x 2 rows)
constexpr int TAIL_THREADS = 128;
constexpr int CO_PAD = TAIL_CO_PAD;
constexpr int OPITCH = 17;      // floats per pixel of the transposed accumulators
// floats per (tap, channel) row of the staged weights, chosen for conflict-free B-fragment loads: bank = pitch*t + g
__host__ __device__ constexpr int wpitch(int nt) { return nt == 1 ? 8 : 24; }

__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 3xTF32 split of an fp32 value (hi + lo), so that the head conv keeps fp32 accuracy on the tensor cores
__device__ __forceinline__ void split_tf32(float v, unsigned& hi, unsigned& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(hi) : "f"(v));
    const float r = v - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(lo) : "f"(r));
}

template <int KIND, int NT, bool STRICT>
__global__ void __launch_bounds__(TAIL_THREADS) tail_kernel(const float* __restrict__ feat, int S, int C, int ld,
                                                   const float* __restrict__ coef, int act,
                                                   const float* __restrict__ wg, const float* __restrict__ bg,
                                                   ImgView img0, ImgView img1, const float* __restrict__ base,
                                                   float* o0, float* o1, float* o2, float* o3, float* o4, float* o5,
                                                   float* o6, float* o7) {
    extern __shared__ __align__(16) float sm[];
    constexpr int WPITCH = wpitch(NT);
    const int CP = C + 4;                     // halo pixel pitch: (4*g + t) mod 32 distinct for the A fragments
    float* wsm = sm;                          // [9*C][WPITCH]
    float* fsm = sm + 9 * C * WPITCH;         // [HALO_H*HALO][CP]
    float* osm = fsm;                         // [128][OPITCH], reuses the halo tile after the MMAs
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int n = blockIdx.z;
    const int by0 = blockIdx.y * TILE_H, bx0 = blockIdx.x * TILE;

    constexpr int WQ = NT * 2;                // float4 chunks of head weights actually used (8 or 16 columns; 12..15 are zero)
#pragma unroll 4
    for (int i = tid; i < 9 * C * WQ; i += TAIL_THREADS) {
        const int row = i / WQ, part = i - row * WQ;
        if (4 * part >= CO_PAD) { *reinterpret_cast<float4*>(wsm + row * WPITCH + 4 * part) = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
        float4 wv = *reinterpret_cast<const float4*>(wg + row * CO_PAD + 4 * part);
        if (!STRICT) { wv.x = round_tf32(wv.x); wv.y = round_tf32(wv.y); wv.z = round_tf32(wv.z); wv.w = round_tf32(wv.w); }
        *reinterpret_cast<float4*>(wsm + row * WPITCH + 4 * part) = wv;
    }
    const int cq = C >> 2;
    // halo staging, 4 independent 16-byte loads in flight per thread (a single load per loop trip left the DRAM latency
    // fully exposed: 23 serial round trips per thread at C = 64)
    constexpr int SU = 4;
    const int items = HALO_H * HALO * cq;
    for (int i0 = tid; i0 < items; i0 += SU * TAIL_THREADS) {
        float4 v[SU];
        int hp[SU], q[SU];
        bool in[SU];
#pragma unroll
        for (int u = 0; u < SU; ++u) {
            const int i = i0 + u * TAIL_THREADS;
            const int ii = i < items ? i : 0;
            q[u] = ii % cq; hp[u] = ii / cq;
            const int hy = hp[u] / HALO, hx = hp[u] - hy * HALO;
            const int gy = by0 + hy - 1, gx = bx0 + hx - 1;
            in[u] = i < items && gy >= 0 && gy < S && gx >= 0 && gx < S;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in[u]) v[u] = __ldg(reinterpret_cast<const float4*>(feat + (((long)n * S + gy) * S + gx) * ld + 4 * q[u]));
        }
#pragma unroll
        for (int u = 0; u < SU; ++u) {
            if (i0 + u * TAIL_THREADS >= items) break;
            float4 w = v[u];
            if (in[u]) {
                const float4 c0 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q[u]) * 2);
                const float4 c1 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q[u]) * 2 + 4);
                w.x = act_apply(w.x * c0.x + c0.y, act); w.y = act_apply(w.y * c0.z + c0.w, act);
                w.z = act_apply(w.z * c1.x + c1.y, act); w.w = act_apply(w.w * c1.z + c1.w, act);
            }
            if (!STRICT) { w.x = round_tf32(w.x); w.y = round_tf32(w.y); w.z = round_tf32(w.z); w.w = round_tf32(w.w); }
            *reinterpret_cast<float4*>(fsm + hp[u] * CP + 4 * q[u]) = w;
        }
    }
    __syncthreads();

    // ---- head conv on tensor cores: warp w (of 4) owns tile rows 2w and 2w+1 (16 pixels each = one m16 tile) ----
    float acc[2][NT][4];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[r][nt][k] = 0.0f;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int dy = tap / 3, dx = tap % 3;
        const float* wt = wsm + tap * C * WPITCH;
#pragma unroll 2
        for (int kc = 0; kc < C; kc += 8) {
            if (STRICT) {     // 3xTF32: hi/lo split of both operands, fp32-equivalent products
                unsigned bh[NT][2], bl[NT][2];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    split_tf32(wt[(kc + t) * WPITCH + nt * 8 + g], bh[nt][0], bl[nt][0]);
                    split_tf32(wt[(kc + t + 4) * WPITCH + nt * 8 + g], bh[nt][1], bl[nt][1]);
                }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float* ap = fsm + ((2 * warp + r + dy) * HALO + dx + g) * CP + kc + t;
                    unsigned ah[4], al[4];
                    split_tf32(ap[0], ah[0], al[0]);
                    split_tf32(ap[8 * CP], ah[1], al[1]);
                    split_tf32(ap[4], ah[2], al[2]);
                    split_tf32(ap[8 * CP + 4], ah[3], al[3]);
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        mma_tf32_16x8x8(acc[r][nt], al, bh[nt][0], bh[nt][1]);
                        mma_tf32_16x8x8(acc[r][nt], ah, bl[nt][0], bl[nt][1]);
                        mma_tf32_16x8x8(acc[r][nt], ah, bh[nt][0], bh[nt][1]);
                    }
                }
            } else {          // single TF32: the halo tile and the staged weights were rounded (RNA) when written
                unsigned b[NT][2];
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    b[nt][0] = __float_as_uint(wt[(kc + t) * WPITCH + nt * 8 + g]);
                    b[nt][1] = __float_as_uint(wt[(kc + t + 4) * WPITCH + nt * 8 + g]);
                }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float* ap = fsm + ((2 * warp + r + dy) * HALO + dx + g) * CP + kc + t;
                    unsigned a[4] = {__float_as_uint(ap[0]), __float_as_uint(ap[8 * CP]), __float_as_uint(ap[4]), __float_as_uint(ap[8 * CP + 4])};
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) mma_tf32_16x8x8(acc[r][nt], a, b[nt][0], b[nt][1]);
                }
            }
        }
    }
    __syncthreads();                          // all warps are done reading the halo tile: reuse it for the transpose
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int px0 = (2 * warp + r) * TILE + g;
            osm[px0 * OPITCH + nt * 8 + 2 * t] = acc[r][nt][0];
            osm[px0 * OPITCH + nt * 8 + 2 * t + 1] = acc[r][nt][1];
            osm[(px0 + 8) * OPITCH + nt * 8 + 2 * t] = acc[r][nt][2];
            osm[(px0 + 8) * OPITCH + nt * 8 + 2 * t + 1] = acc[r][nt][3];
        }
    __syncthreads();

    const int ty = tid / TILE, tx = tid % TILE;
    float o[CO_PAD];
#pragma unroll
    for (int j = 0; j < CO_PAD; ++j) o[j] = (j < NT * 8) ? osm[tid * OPITCH + j] + bg[j] : 0.0f;     // 128 threads = 128 pixels

    tail_epilogue<KIND>(o, n, by0 + ty, bx0 + tx, S, img0, img1, base, o0, o1, o2, o3, o4, o5, o6, o7);
}

template <int KIND, int NT, bool STRICT>
void launch_tail(const TailWeights& tw, const View& f, const float* coef, int act, const ImgView& i0, const ImgView& i1,
                 float* const* o, cudaStream_t s) {
    THA4_REQUIRE(tw.C % 8 == 0 && tw.CO <= NT * 8, "tail: head channel layout");
    const size_t halo = (size_t)HALO_H * HALO * (tw.C + 4), outs = (size_t)TILE * TILE_H * OPITCH;
    const size_t smem = ((size_t)9 * tw.C * wpitch(NT) + std::max(halo, outs)) * sizeof(float);
    THA4_ENSURE_SMEM((tail_kernel<KIND, NT, STRICT>), smem);
    float* op[8];
    for (int i = 0; i < 8; ++i) op[i] = i < TAIL_OUTPUTS[KIND].count ? o[i] : nullptr;
    dim3 grid(f.W / TILE, f.H / TILE_H, f.N);
    ProfScope prof(PROF_TAIL, s);
    {   // compulsory traffic: feature map + 4-channel image(s) read once, every returned tensor written once (SURVEY 8d)
        const int img_ch = (KIND == TAIL_COMBINER) ? 8 : 4;
        prof_add_work(PROF_TAIL, 2.0 * f.pixels() * 9 * tw.C * tw.CO, (double)f.pixels() * (f.C + img_ch + TAIL_OUTPUTS[KIND].channels()) * 4);
    }
    tail_kernel<KIND, NT, STRICT><<<grid, TAIL_THREADS, smem, s>>>(f.p, f.H, f.C, f.ld, coef, act, tw.w, tw.bias, i0, i1,
                                             base_grid_table(f.H), op[0], op[1], op[2], op[3], op[4], op[5], op[6], op[7]);
    THA4_LAUNCH_CHECK();
}

__global__ void tail_pack_kernel(float* w, float* b, const float* src_w, const float* src_b, int C, int cout, int co_off) {
    const int total = cout * C * 9;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int tap = i % 9;
        const int c = (i / 9) % C;
        const int co = i / (9 * C);
        w[(tap * C + c) * TAIL_CO_PAD + co_off + co] = src_w[i];
    }
    if (src_b && blockIdx.x == 0 && threadIdx.x < cout) b[co_off + threadIdx.x] = src_b[threadIdx.x];
}

}  // namespace

void tail_init(TailWeights& tw, int C, cudaStream_t s) {
    tw.C = C; tw.CO = 0;
    tw.w = reinterpret_cast<float*>(tracked_malloc((size_t)9 * C * TAIL_CO_PAD * sizeof(float)));
    tw.bias = reinterpret_cast<float*>(tracked_malloc(TAIL_CO_PAD * sizeof(float)));
    THA4_CUDA_CHECK(cudaMemsetAsync(tw.w, 0, (size_t)9 * C * TAIL_CO_PAD * sizeof(float), s));
    THA4_CUDA_CHECK(cudaMemsetAsync(tw.bias, 0, TAIL_CO_PAD * sizeof(float), s));
}

void tail_add(TailWeights& tw, const float* w_ref, const float* b_ref, int cout, cudaStream_t s) {
    THA4_REQUIRE(tw.w != nullptr && tw.CO + cout <= TAIL_CO_PAD, "too many head channels");
    tail_pack_kernel<<<32, 256, 0, s>>>(tw.w, tw.bias, w_ref, b_ref, tw.C, cout, tw.CO);
    THA4_LAUNCH_CHECK();
    tw.CO += cout;
}

void tail_forward(TailKind kind, const TailWeights& tw, const View& feature, const float* coef, int act,
                  const ImgView& image0, const ImgView& image1, float* const* outputs, cudaStream_t s, int strict) {
    THA4_REQUIRE(feature.H == feature.W && feature.H % TILE == 0 && feature.C == tw.C && tw.C % 4 == 0, "tail: feature dims");
    THA4_REQUIRE(image0.H == feature.H && image0.W == feature.W && image0.C == 4, "tail: image dims");
    switch (kind) {
        case TAIL_UNET:
            if (strict) launch_tail<TAIL_UNET, 1, true>(tw, feature, coef, act, image0, image1, outputs, s);
            else launch_tail<TAIL_UNET, 1, false>(tw, feature, coef, act, image0, image1, outputs, s);
            break;
        case TAIL_DECOMPOSER:
            if (strict) launch_tail<TAIL_DECOMPOSER, 2, true>(tw, feature, coef, act, image0, image1, outputs, s);
            else launch_tail<TAIL_DECOMPOSER, 2, false>(tw, feature, coef, act, image0, image1, outputs, s);
            break;
        case TAIL_COMBINER:
            if (strict) launch_tail<TAIL_COMBINER, 1, true>(tw, feature, coef, act, image0, image1, outputs, s);
            else launch_tail<TAIL_COMBINER, 1, false>(tw, feature, coef, act, image0, image1, outputs, s);
            break;
        case TAIL_FACE:
            if (strict) launch_tail<TAIL_FACE, 2, true>(tw, feature, coef, act, image0, image1, outputs, s);
            else launch_tail<TAIL_FACE, 2, false>(tw, feature, coef, act, image0, image1, outputs, s);
            break;
    }
}

}  // namespace tha4
