// Weight gradients of the teacher convolutions on wgmma (TF32, or 3xTF32 in strict mode):
//   dW[d][c][tap] = sum over the batch and the pixels p of the DIRECT operand of  D[p][d] * G[p shifted by tap][c].
// For a Conv2d the direct operand is dz (the gradient at the conv's raw output) and the gathered operand x^ (what the forward
// conv multiplied); for the transposed 4x4 stride-2 conv the roles are exchanged (D = x^ at the input resolution, G = dz at
// the output resolution, gathered at 2 y - 1 + ky exactly like a stride-2 conv's input), so one gather path serves both,
// and the reference layouts ([cout][cin][kh][kw] / [cin][cout][kh][kw]) are both [d][c][tap].  The U-Net's nearest x2 + 3x3
// conv gathers x^ at half resolution: tap (y + ky - 1, x + kx - 1) is checked against the output's bounds, then halved.
//
// GEMM view: M = (tap, c) rows of G in tiles of 64, N = channels d of D in tiles of NT (16 for the 7-12 head channels,
// 64, 128), K = pixels in blocks of 32.  Both NHWC operands are MN-major; the 128 threads of the CTA (one warpgroup) load
// them from global memory, apply the pending normalisation the forward applied (operand transform), zero the padding, and
// store them K-major into 128-byte-swizzled tiles, double-buffered against the asynchronous wgmma.  Pixel-split partials
// go to a workspace and are summed in split order by a second kernel: no float atomics anywhere.
// The U-Net's operand variants (SiLU transforms, the x2 gather) are separate instantiations (EXT); the encoder-decoders'
// instantiations compile to the same SASS as before the variants were added.
#include "conv_wgrad.cuh"
#include "conv_tc_device.cuh"

namespace tha4 {

namespace {

using namespace tc;

constexpr int WG_KB = 32;               // pixels per k-block (one 128-byte row of fp32)

// SiLU as the wgmma convs apply it to an f16 operand (conv_tc_device.cuh, xf_chunks): h + h tanh(h), h = A/2 x + B/2 in f16
__device__ __forceinline__ __half wg_silu_half(__half h) {
    const __half2 h2 = __halves2half2(h, h);
    const uint32_t hu = *reinterpret_cast<const uint32_t*>(&h2);
    uint32_t tu;
    asm("tanh.approx.f16x2 %0, %1;\n" : "=r"(tu) : "r"(hu));
    return __low2half(__hfma2(h2, *reinterpret_cast<const __half2*>(&tu), h2));
}

// the encoder-decoders' operand transforms (the non-EXT kernels): the stored value, the forward's f16 XF transform, or the
// tail's fp32 affine, each + ReLU when act is set
__device__ __forceinline__ float wg_load(const WgradOperand& o, long pix, int n, int c) {
    float v = o.f16 ? __half2float(reinterpret_cast<const __half*>(o.p)[pix * o.ld + c]) : reinterpret_cast<const float*>(o.p)[pix * o.ld + c];
    if (o.xf != WG_XF_NONE && c < o.coef_C) {
        const float2 ab = o.coef[(long)n * o.coef_C + c];
        if (o.xf == WG_XF_HALF) {        // the forward's XF transform: one f16 FMA with f16 coefficients (conv_tc_device.cuh)
            __half h = __hfma(__float2half_rn(v), __float2half_rn(ab.x), __float2half_rn(ab.y));
            if (o.act) h = __hmax(h, __float2half_rn(0.0f));
            v = __half2float(h);
        } else {
            v = fmaf(v, ab.x, ab.y);
            if (o.act) v = fmaxf(v, 0.0f);
            if (o.xf == WG_XF_FLOAT16) v = __half2float(__float2half_rn(v));
        }
    }
    return v;
}

// the U-Net's (EXT kernels): the same with the activation enum -- ReLU, SiLU, or the fast SiLU of the wgmma kernels
__device__ __forceinline__ float wg_load_ext(const WgradOperand& o, long pix, int n, int c) {
    float v = o.f16 ? __half2float(reinterpret_cast<const __half*>(o.p)[pix * o.ld + c]) : reinterpret_cast<const float*>(o.p)[pix * o.ld + c];
    if (o.xf != WG_XF_NONE && c < o.coef_C) {
        const float2 ab = o.coef[(long)n * o.coef_C + c];
        if (o.xf == WG_XF_HALF) {        // the forward's XF transform (conv_tc_device.cuh, xf_chunks)
            __half h = __hfma(__float2half_rn(v), __float2half_rn(ab.x), __float2half_rn(ab.y));
            if (o.act == ACT_RELU) h = __hmax(h, __float2half_rn(0.0f));
            else if (o.act == ACT_SILU_FAST) h = wg_silu_half(h);
            v = __half2float(h);
        } else {                         // the U-Net tails: fp32 affine, SiLU (wgmma tail: tanh.approx.f32 on v / 2)
            if (o.act == ACT_SILU_FAST) {
                float h = fmaf(v, 0.5f * ab.x, 0.5f * ab.y), t;
                asm("tanh.approx.f32 %0, %1;\n" : "=f"(t) : "f"(h));
                v = fmaf(h, t, h);
            } else {
                v = act_apply(fmaf(v, ab.x, ab.y), o.act);
            }
            if (o.xf == WG_XF_FLOAT16) v = __half2float(__float2half_rn(v));
        }
    }
    return v;
}

template <bool EXT>
__device__ __forceinline__ float wg_load_any(const WgradOperand& o, long pix, int n, int c) {
    if constexpr (EXT) return wg_load_ext(o, pix, n, c);
    else return wg_load(o, pix, n, c);
}

// 4 consecutive k values of one K-major row into the 128-byte-swizzled tile (the layout TMA would write)
template <bool STRICT>
__device__ __forceinline__ void wg_store4(uint8_t* hi, uint8_t* lo, int row, int chunk, const float (&v)[4]) {
    const int off = row * 128 + ((chunk ^ (row & 7)) << 4);
    if (STRICT) {
        float h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) { h[e] = __uint_as_float(__float_as_uint(v[e]) & 0xffffe000u); l[e] = v[e] - h[e]; }
        *reinterpret_cast<float4*>(hi + off) = make_float4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<float4*>(lo + off) = make_float4(l[0], l[1], l[2], l[3]);
    } else {
        *reinterpret_cast<float4*>(hi + off) = make_float4(round_tf32(v[0]), round_tf32(v[1]), round_tf32(v[2]), round_tf32(v[3]));
    }
}

template <int NT>
__device__ __forceinline__ void wg_mma(float (&acc)[NT / 2], uint32_t a, uint32_t b) {
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<NT>::tf32(acc, make_smem_desc_sw<128>(a + 32 * k), make_smem_desc_sw<128>(b + 32 * k), 1u);
}

// where row (m = tap * G.C + c, d) of the GEMM lands in the flat parameter buffer (-1: nowhere)
__device__ __forceinline__ long wg_dst(const WgradArgs& a, int m, int d) {
    if (m >= a.M || d >= a.D.C) return -1;
    const int tap = m / a.G.C, c = m - tap * a.G.C;
    if (c >= a.c_real) return -1;
    const long base = a.n_map > 0 ? (d < a.n_map ? a.out_row[d] : -1) : (long)d * a.c_real * a.ntaps;
    return base < 0 ? -1 : base + (long)c * a.ntaps + tap;
}

template <int NT, bool STRICT, bool EXT>
__global__ void __launch_bounds__(128) conv_wgrad_kernel(const WgradArgs a) {
    extern __shared__ uint8_t wg_smem_raw[];
    uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int A_BYTES = 64 * 128, B_BYTES = NT * 128;
    constexpr int OPS = STRICT ? 2 : 1;
    constexpr int STAGE = OPS * (A_BYTES + B_BYTES);
    constexpr int DPIX = NT / 4;                               // direct-operand pixels per thread per k-block
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int m0 = blockIdx.x * 64, n0 = blockIdx.y * NT;
    const int kb0 = blockIdx.z * a.kb_per_split, kb1 = min(a.kblocks, kb0 + a.kb_per_split);
    const int HWd = a.D.H * a.D.W;

    // this thread's gathered row (16 pixels of each k-block) and direct row (DPIX pixels)
    const int gr = t & 63, gh = t >> 6;
    const int gm = m0 + gr;
    const bool g_ok = gm < a.M;
    const int gtap = g_ok ? gm / a.G.C : 0, gc = g_ok ? gm - gtap * a.G.C : 0;
    const int gky = gtap / a.ksz - a.pad, gkx = gtap % a.ksz - a.pad;
    const int dr = t % NT, dg = t / NT;
    const bool d_ok = n0 + dr < a.D.C;

    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.0f;

    for (int kb = kb0; kb < kb1; ++kb) {
        uint8_t* st = sm + ((kb - kb0) & 1) * STAGE;
        uint8_t* Ahi = st; uint8_t* Bhi = st + A_BYTES;
        uint8_t* Alo = st + A_BYTES + B_BYTES; uint8_t* Blo = Alo + A_BYTES;
        const long pix0 = (long)kb * WG_KB;
        const int n = (int)(pix0 / HWd);
        const int rem = (int)(pix0 - (long)n * HWd);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int p = rem + gh * 16 + q * 4 + e;
                const int y = p / a.D.W, x = p - y * a.D.W;
                const int gy = y * a.stride + gky, gx = x * a.stride + gkx;
                // zero padding belongs to the transformed operand: out-of-image taps are zero AFTER the transform.  The x2
                // gather (EXT) checks the tap at D's resolution, then reads the source pixel; written as folded ternaries, not
                // a branch, so the encoder-decoders' kernels compile to the code they had before the EXT variants existed
                const bool up2 = EXT && a.up2;
                const bool in = g_ok && gy >= 0 && gy < (up2 ? a.D.H : a.G.H) && gx >= 0 && gx < (up2 ? a.D.W : a.G.W);
                v[e] = in ? wg_load_any<EXT>(a.G, ((long)n * a.G.H + (up2 ? gy >> 1 : gy)) * a.G.W + (up2 ? gx >> 1 : gx), n, gc) : 0.0f;
            }
            wg_store4<STRICT>(Ahi, Alo, gr, gh * 4 + q, v);
        }
#pragma unroll
        for (int q = 0; q < DPIX / 4; ++q) {
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e)
                v[e] = d_ok ? wg_load_any<EXT>(a.D, pix0 + dg * DPIX + q * 4 + e, n, n0 + dr) : 0.0f;
            wg_store4<STRICT>(Bhi, Blo, dr, (dg * DPIX) / 4 + q, v);
        }
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic-proxy writes -> wgmma's async-proxy reads
        __syncthreads();
        wg_fence();
        wg_mma<NT>(acc, smem_u32(Ahi), smem_u32(Bhi));
        if (STRICT) {
            wg_mma<NT>(acc, smem_u32(Ahi), smem_u32(Blo));
            wg_mma<NT>(acc, smem_u32(Alo), smem_u32(Bhi));
        }
        wg_commit();
        wg_fence_acc(acc);
        wg_wait<1>();                 // the group that read the other stage has retired: the next k-block may overwrite it
        wg_fence_acc(acc);
        __syncthreads();              // ... for every warp of the group before any of them stores into that stage
    }
    wg_wait<0>();
    wg_fence_acc(acc);

    // accumulator fragment: rows 16 warp + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) + {0, 1}
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) {
        const int m = m0 + 16 * warp + (lane >> 2) + ((i & 2) ? 8 : 0);
        const int d = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (a.splits > 1) {
            a.ws[((long)blockIdx.z * a.ws_rows + m) * a.ws_cols + d] = acc[i];
        } else {
            const long o = wg_dst(a, m, d);
            if (o >= 0) a.out[o] = a.accumulate ? a.out[o] + acc[i] : acc[i];
        }
    }
}

// the pixel-split partials summed in split order
__global__ void conv_wgrad_reduce_kernel(const WgradArgs a) {
    const long total = (long)a.ws_rows * a.ws_cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int m = (int)(i / a.ws_cols), d = (int)(i - (long)m * a.ws_cols);
        const long o = wg_dst(a, m, d);
        if (o < 0) continue;
        float s = 0.0f;
        for (int z = 0; z < a.splits; ++z) s += a.ws[(long)z * total + i];
        a.out[o] = a.accumulate ? a.out[o] + s : s;
    }
}

// per-(n, c) coefficients of a pending normalisation, built by the forward's own XF code (f16-rounded, as the forward used them)
__global__ void __launch_bounds__(128) wgrad_xf_coef_kernel(const tcdev::TcParams p, float2* __restrict__ coef) {
    extern __shared__ double2 chs[];
    __half* hA = reinterpret_cast<__half*>(chs + p.xf_C);
    __half* hB = hA + p.xf_C;
    const int n = blockIdx.x;
    tcdev::xf_build_coef<128, 1>(p, n, threadIdx.x, hA, hB, chs, 0, p.xf_C);
    for (int c = threadIdx.x; c < p.xf_C; c += 128) coef[(long)n * p.xf_C + c] = make_float2(__half2float(hA[c]), __half2float(hB[c]));
}

template <int NT, bool STRICT>
size_t wgrad_smem() { return 1024 + 2 * (STRICT ? 2 : 1) * (64 * 128 + NT * 128); }

template <int NT, bool STRICT, bool EXT>
void launch_wgrad(const WgradArgs& a, dim3 grid, cudaStream_t s) {
    const size_t smem = wgrad_smem<NT, STRICT>();
    auto kernel = conv_wgrad_kernel<NT, STRICT, EXT>;
    THA4_ENSURE_SMEM(kernel, smem);
    kernel<<<grid, 128, smem, s>>>(a);
    THA4_LAUNCH_CHECK();
}

}  // namespace

float2* wgrad_xf_coef(const View& raw, const float* gamma, const float* beta, int C, int act, float2* coef, cudaStream_t s,
                      int groups, const float* film0, const float* film1, int film1_ld) {
    THA4_REQUIRE(raw.stats != nullptr && C % 8 == 0 && C <= 1024, "wgrad coefficients: statistics / channels");
    THA4_REQUIRE(groups == 0 || C % groups == 0, "wgrad coefficients: groups");
    tcdev::TcParams p{};
    p.in_stats = raw.stats; p.in_stats_ld = raw.stats_ld; p.in_stats_rep = std::max(1, raw.stats_rep); p.in_stats_rep_stride = raw.stats_rep_stride;
    // the values conv_tc.cu / conv_halo.cu hand xf_build_coef for the same ConvNormIn
    p.xf_C = C; p.xf_groups = groups; p.xf_act = act; p.xf_inv_cnt = 1.0 / ((double)raw.H * raw.W * (groups == 0 ? 1 : C / groups));
    p.xf_gamma = gamma; p.xf_beta = beta; p.xf_film0 = film0; p.xf_film1 = film1; p.xf_film1_ld = film1_ld;
    const size_t smem = (size_t)C * (sizeof(double2) + 2 * sizeof(__half));
    wgrad_xf_coef_kernel<<<raw.N, 128, smem, s>>>(p, coef);
    THA4_LAUNCH_CHECK();
    return coef;
}

WgradPlan conv_wgrad_plan(const WgradArgs& a, int ksplit) {
    WgradPlan pl;
    pl.nt = a.D.C <= 16 ? 16 : (a.D.C <= 64 ? 64 : 128);
    pl.mtiles = ceil_div(a.M, 64);
    pl.ntiles = ceil_div(a.D.C, pl.nt);
    const long pixels = (long)a.D.N * a.D.H * a.D.W;
    pl.kblocks = (int)(pixels / WG_KB);
    const int tiles = pl.mtiles * pl.ntiles;
    int splits = ksplit > 0 ? ksplit : (tiles >= num_sms() ? 1 : ceil_div(2L * num_sms(), tiles));
    splits = std::max(1, std::min(splits, std::max(1, pl.kblocks / 4)));        // at least 4 k-blocks per split
    pl.kb_per_split = ceil_div(pl.kblocks, splits);
    pl.splits = ceil_div(pl.kblocks, pl.kb_per_split);
    return pl;
}

size_t conv_wgrad_workspace_floats(const WgradPlan& pl) {
    return pl.splits > 1 ? (size_t)pl.splits * pl.mtiles * 64 * pl.ntiles * pl.nt : 0;
}

WgradPlan conv_wgrad_layer(ConvKind kind, const WgradOperand& x, const WgradOperand& dz, WgradArgs a, int strict, int ksplit,
                           const std::function<float*(size_t)>& ws_alloc, cudaStream_t s) {
    THA4_REQUIRE(kind == CONV_3x3 || kind == CONV_1x1 || kind == CONV_UP2_3x3 || kind == CONV_4x4_S2 || kind == CONVT_4x4_S2,
                 "conv wgrad: kind");
    a.G = kind == CONVT_4x4_S2 ? dz : x;
    a.D = kind == CONVT_4x4_S2 ? x : dz;
    const bool s1 = kind == CONV_3x3 || kind == CONV_1x1 || kind == CONV_UP2_3x3;
    a.ksz = kind == CONV_1x1 ? 1 : (s1 ? 3 : 4); a.ntaps = a.ksz * a.ksz; a.stride = s1 ? 1 : 2; a.pad = kind == CONV_1x1 ? 0 : 1;
    a.up2 = kind == CONV_UP2_3x3;
    a.M = a.ntaps * a.G.C;
    if (a.c_real == 0) a.c_real = a.G.C;
    if (a.up2) {
        THA4_REQUIRE(a.D.H == 2 * a.G.H && a.D.W == 2 * a.G.W, "conv wgrad: operand geometry (nearest x2)");
    } else {
        const int oh = s1 ? a.G.H : a.G.H / 2;
        THA4_REQUIRE(a.D.H == oh && a.D.W * (a.G.H / oh) == a.G.W, "conv wgrad: operand geometry");
    }
    const WgradPlan pl = conv_wgrad_plan(a, ksplit);
    const size_t ws = conv_wgrad_workspace_floats(pl);
    conv_wgrad(a, pl, strict, ws ? ws_alloc(ws) : nullptr, s);
    return pl;
}

void conv_wgrad(WgradArgs a, const WgradPlan& pl, int strict, float* ws, cudaStream_t s) {
    THA4_REQUIRE(a.ksz == 1 || a.ksz == 3 || a.ksz == 4, "conv wgrad: kernel size");
    THA4_REQUIRE(!a.up2 || (a.ksz == 3 && a.stride == 1 && a.pad == 1), "conv wgrad: nearest x2 gather is a 3x3 conv's");
    THA4_REQUIRE(a.ntaps == a.ksz * a.ksz && a.M == a.ntaps * a.G.C && a.c_real <= a.G.C, "conv wgrad: rows");
    THA4_REQUIRE(a.D.N == a.G.N && ((long)a.D.H * a.D.W) % WG_KB == 0, "conv wgrad: pixels per sample must be a multiple of 32");
    THA4_REQUIRE(a.n_map == 0 || a.n_map <= 16, "conv wgrad: row map");
    a.kblocks = pl.kblocks; a.kb_per_split = pl.kb_per_split; a.splits = pl.splits;
    a.ws_rows = pl.mtiles * 64; a.ws_cols = pl.ntiles * pl.nt;
    if (pl.splits > 1) { THA4_REQUIRE(ws != nullptr, "conv wgrad: workspace"); a.ws = ws; }
    const dim3 grid(pl.mtiles, pl.ntiles, pl.splits);
    // the U-Net's variants: a SiLU operand transform or the x2 gather
    const bool ext = a.up2 || a.G.act == ACT_SILU || a.G.act == ACT_SILU_FAST || a.D.act == ACT_SILU || a.D.act == ACT_SILU_FAST;
    if (ext) {
        if (pl.nt == 16) { if (strict) launch_wgrad<16, true, true>(a, grid, s); else launch_wgrad<16, false, true>(a, grid, s); }
        else if (pl.nt == 64) { if (strict) launch_wgrad<64, true, true>(a, grid, s); else launch_wgrad<64, false, true>(a, grid, s); }
        else { if (strict) launch_wgrad<128, true, true>(a, grid, s); else launch_wgrad<128, false, true>(a, grid, s); }
    } else {
        if (pl.nt == 16) { if (strict) launch_wgrad<16, true, false>(a, grid, s); else launch_wgrad<16, false, false>(a, grid, s); }
        else if (pl.nt == 64) { if (strict) launch_wgrad<64, true, false>(a, grid, s); else launch_wgrad<64, false, false>(a, grid, s); }
        else { if (strict) launch_wgrad<128, true, false>(a, grid, s); else launch_wgrad<128, false, false>(a, grid, s); }
    }
    if (pl.splits > 1) {
        const long total = (long)a.ws_rows * a.ws_cols;
        conv_wgrad_reduce_kernel<<<(int)std::min<long>((total + 255) / 256, 132L * 16), 256, 0, s>>>(a);
        THA4_LAUNCH_CHECK();
    }
}

}  // namespace tha4
