// Implicit-GEMM convolution, NHWC fp32 activations, TF32 tensor-core products with fp32 accumulation.
//
// This is the general-shape kernel (any Cin % 4 == 0, any Cout, all four conv kinds, fused bias / residual /
// nearest-upsample gather / split-K).  A-tiles are gathered straight from the activation tensor with 16-byte
// cp.async (zero-fill implements the conv padding), B-tiles stream from the pre-packed weights; a 3/4-stage
// cp.async ring feeds mma.sync.m16n8k8.tf32.  `strict` switches to 3xTF32 error-compensated products, which
// reproduces fp32 convolution to ~1e-6 relative and is what the tight parity tests use.
#include "conv.cuh"
#include "profiler.cuh"

namespace tha4 {

namespace {

constexpr int BM = 128;
constexpr int BK = 32;
constexpr int PITCH = BK + 4;   // floats; (4*g + t) mod 32 is conflict-free for the mma fragment loads
constexpr int NTHREADS = 256;

struct ConvKernelParams {
    const float* in; int inH, inW, inC, in_ld;   // stored dims
    int LH, LW;                                  // logical input dims (2x stored when in_up)
    int in_up;
    const float* w; const float* bias;
    float* out; int outH, outW, outC, out_ld;
    const float* res; int resH, resW, res_ld, res_mode;
    int N, MH, MW;
    long M_total;
    int stride, out_mul, ntaps, nphase, ksplit;
    int cin_pad, cout_pad;
    int strict;
    signed char dy[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char dx[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char ph_oy[CONV_MAX_PHASES], ph_ox[CONV_MAX_PHASES];
};

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src, bool valid) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" :: "r"(sa), "l"(gmem_src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" :: "n"(N)); }

__device__ __forceinline__ unsigned f2tf32(float f) {
    unsigned r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(f));
    return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const unsigned (&a)[4], const unsigned (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int BN, int WM, int WN, int STAGES>
__global__ void __launch_bounds__(NTHREADS) conv_igemm_kernel(const ConvKernelParams p) {
    constexpr int TM = BM / WM, TN = BN / WN;
    constexpr int MT = TM / 16, NT = TN / 8;
    constexpr int A_FLOATS = BM * PITCH, B_FLOATS = BN * PITCH;
    static_assert(WM * WN == NTHREADS / 32, "warp layout");
    extern __shared__ __align__(16) float smem[];
    float* As = smem;
    float* Bs = smem + STAGES * A_FLOATS;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp % WM, wn = warp / WM;
    const int g = lane >> 2, t = lane & 3;
    const long m0 = (long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int phase = blockIdx.z / p.ksplit;
    const int split = blockIdx.z % p.ksplit;

    // ---- K range of this split ----
    const int cpt = p.cin_pad / BK;                 // K-chunks per tap
    const int KT = p.ntaps * cpt;
    const int k_per = (KT + p.ksplit - 1) / p.ksplit;
    const int kb = split * k_per;
    const int ke = min(KT, kb + k_per);
    const int nk = max(0, ke - kb);

    // ---- per-thread gather rows (fixed for the whole K loop) ----
    const int chunk = tid & 7;                      // 16-byte chunk within the 128-byte K slice
    int row_iy0[4], row_ix0[4];
    long row_base[4];
    bool row_ok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        long m = m0 + (tid >> 3) + 32 * i;
        row_ok[i] = m < p.M_total;
        long mm = row_ok[i] ? m : 0;
        int n = (int)(mm / ((long)p.MH * p.MW));
        int rem = (int)(mm - (long)n * p.MH * p.MW);
        int my = rem / p.MW, mx = rem - my * p.MW;
        row_iy0[i] = my * p.stride;
        row_ix0[i] = mx * p.stride;
        row_base[i] = (long)n * p.inH * p.inW * p.in_ld;
    }
    const float* wph = p.w + (long)phase * p.ntaps * p.cout_pad * p.cin_pad;

    auto load_stage = [&](int slot, int kt) {
        const int tap = kt / cpt;
        const int ci0 = (kt - tap * cpt) * BK;
        const int dy = p.dy[phase][tap], dx = p.dx[phase][tap];
        const int c = ci0 + chunk * 4;
        const bool cok = c < p.inC;
        float* a_dst = As + slot * A_FLOATS + chunk * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int r = (tid >> 3) + 32 * i;
            int iy = row_iy0[i] + dy, ix = row_ix0[i] + dx;
            bool ok = row_ok[i] && cok && iy >= 0 && iy < p.LH && ix >= 0 && ix < p.LW;
            if (p.in_up) { iy >>= 1; ix >>= 1; }
            const float* src = ok ? (p.in + row_base[i] + ((long)iy * p.inW + ix) * p.in_ld + c) : p.in;
            cp_async16(a_dst + r * PITCH, src, ok);
        }
        float* b_dst = Bs + slot * B_FLOATS + chunk * 4;
        const float* wt = wph + (long)tap * p.cout_pad * p.cin_pad + ci0 + chunk * 4;
#pragma unroll
        for (int i = 0; i < BN / 32; ++i) {
            int r = (tid >> 3) + 32 * i;
            int co = n0 + r;
            bool ok = co < p.cout_pad;
            const float* src = ok ? (wt + (long)co * p.cin_pad) : p.w;
            cp_async16(b_dst + r * PITCH, src, ok);
        }
    };

    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.0f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) load_stage(s, kb + s);
        cp_async_commit();
    }

    for (int it = 0; it < nk; ++it) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            int nxt = it + STAGES - 1;
            if (nxt < nk) load_stage(nxt % STAGES, kb + nxt);
            cp_async_commit();
        }
        const float* a_s = As + (it % STAGES) * A_FLOATS + (wm * TM) * PITCH;
        const float* b_s = Bs + (it % STAGES) * B_FLOATS + (wn * TN) * PITCH;
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
            float af[MT][4], bf[NT][2];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                const float* ap = a_s + (mt * 16 + g) * PITCH + ks * 8 + t;
                af[mt][0] = ap[0];
                af[mt][1] = ap[8 * PITCH];
                af[mt][2] = ap[4];
                af[mt][3] = ap[8 * PITCH + 4];
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const float* bp = b_s + (nt * 8 + g) * PITCH + ks * 8 + t;
                bf[nt][0] = bp[0];
                bf[nt][1] = bp[4];
            }
            if (p.strict) {
                unsigned ah[MT][4], al[MT][4], bh[NT][2], bl[NT][2];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        ah[mt][k] = f2tf32(af[mt][k]);
                        al[mt][k] = f2tf32(af[mt][k] - __uint_as_float(ah[mt][k]));
                    }
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int k = 0; k < 2; ++k) {
                        bh[nt][k] = f2tf32(bf[nt][k]);
                        bl[nt][k] = f2tf32(bf[nt][k] - __uint_as_float(bh[nt][k]));
                    }
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        mma_tf32(acc[mt][nt], al[mt], bh[nt]);
                        mma_tf32(acc[mt][nt], ah[mt], bl[nt]);
                        mma_tf32(acc[mt][nt], ah[mt], bh[nt]);
                    }
            } else {
                unsigned au[MT][4], bu[NT][2];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int k = 0; k < 4; ++k) au[mt][k] = f2tf32(af[mt][k]);
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                    for (int k = 0; k < 2; ++k) bu[nt][k] = f2tf32(bf[nt][k]);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) mma_tf32(acc[mt][nt], au[mt], bu[nt]);
            }
        }
    }
    cp_async_wait<0>();

    // ---- epilogue: bias + residual, NHWC store (atomic accumulate when K is split) ----
    if (nk == 0 && p.ksplit > 1) return;
    const bool lead = (split == 0);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            long m = m0 + wm * TM + mt * 16 + g + half * 8;
            if (m >= p.M_total) continue;
            int n = (int)(m / ((long)p.MH * p.MW));
            int rem = (int)(m - (long)n * p.MH * p.MW);
            int my = rem / p.MW, mx = rem - my * p.MW;
            int oy = my * p.out_mul + p.ph_oy[phase], ox = mx * p.out_mul + p.ph_ox[phase];
            float* orow = p.out + (((long)n * p.outH + oy) * p.outW + ox) * p.out_ld;
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                int co = n0 + wn * TN + nt * 8 + 2 * t;
                if (co >= p.outC) continue;
                const bool two = (co + 1) < p.outC;
                float v0 = acc[mt][nt][half * 2 + 0], v1 = acc[mt][nt][half * 2 + 1];
                if (lead) {
                    if (p.bias) { v0 += p.bias[co]; if (two) v1 += p.bias[co + 1]; }
                    if (p.res_mode == RES_SAME) {
                        const float* r = p.res + (((long)n * p.resH + oy) * p.resW + ox) * p.res_ld + co;
                        v0 += r[0]; if (two) v1 += r[1];
                    } else if (p.res_mode == RES_UP2) {
                        const float* r = p.res + (((long)n * p.resH + (oy >> 1)) * p.resW + (ox >> 1)) * p.res_ld + co;
                        v0 += r[0]; if (two) v1 += r[1];
                    } else if (p.res_mode == RES_DOWN2) {
                        const float* r = p.res + (((long)n * p.resH + 2 * oy) * p.resW + 2 * ox) * p.res_ld + co;
                        const long dx1 = p.res_ld, dy1 = (long)p.resW * p.res_ld;
                        v0 += 0.25f * ((r[0] + r[dx1]) + (r[dy1] + r[dy1 + dx1]));
                        if (two) v1 += 0.25f * ((r[1] + r[dx1 + 1]) + (r[dy1 + 1] + r[dy1 + dx1 + 1]));
                    }
                }
                if (p.ksplit > 1) {
                    atomicAdd(orow + co, v0);
                    if (two) atomicAdd(orow + co + 1, v1);
                } else if (two) {
                    *reinterpret_cast<float2*>(orow + co) = make_float2(v0, v1);
                } else {
                    orow[co] = v0;
                }
            }
        }
    }
}

template <int BN, int WM, int WN, int STAGES>
void launch_conv(const ConvKernelParams& p, dim3 grid, cudaStream_t s) {
    constexpr size_t smem = (size_t)STAGES * (BM + BN) * PITCH * sizeof(float);
    THA4_ENSURE_SMEM((conv_igemm_kernel<BN, WM, WN, STAGES>), smem);
    conv_igemm_kernel<BN, WM, WN, STAGES><<<grid, NTHREADS, smem, s>>>(p);
    THA4_LAUNCH_CHECK();
}

// ---- weight packing -------------------------------------------------------------------------------------
__global__ void conv_pack_kernel(float* dst, const float* src, int kind, int w_cin, int cin_offset, int cout,
                                 int cin_pad, int cout_pad, int ntaps, int nphase, int round_w) {
    long total = (long)nphase * ntaps * cout * w_cin;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        int ci = (int)(i % w_cin);
        long r = i / w_cin;
        int co = (int)(r % cout); r /= cout;
        int tap = (int)(r % ntaps);
        int ph = (int)(r / ntaps);
        float v;
        if (kind == CONV_3x3) {
            v = src[(((long)co * w_cin + ci) * 3 + tap / 3) * 3 + tap % 3];
        } else if (kind == CONV_4x4_S2) {
            v = src[(((long)co * w_cin + ci) * 4 + tap / 4) * 4 + tap % 4];
        } else if (kind == CONV_1x1) {
            v = src[(long)co * w_cin + ci];
        } else if (kind == CONV_UP2_3x3) {
            // out[2a+py] = sum_ky up(x)[2a+py+ky-1] w[ky] with up(x)[r] = x[r>>1]:
            //   py=0: ky=0 -> x[a-1];  ky=1,2 -> x[a]        py=1: ky=0,1 -> x[a];  ky=2 -> x[a+1]
            const int py = ph >> 1, px = ph & 1, ty = tap >> 1, tx = tap & 1;
            const int ky0 = (py == 0) ? (ty == 0 ? 0 : 1) : (ty == 0 ? 0 : 2), ky1 = (py == 0) ? (ty == 0 ? 0 : 2) : (ty == 0 ? 1 : 2);
            const int kx0 = (px == 0) ? (tx == 0 ? 0 : 1) : (tx == 0 ? 0 : 2), kx1 = (px == 0) ? (tx == 0 ? 0 : 2) : (tx == 0 ? 1 : 2);
            v = 0.0f;
            for (int ky = ky0; ky <= ky1; ++ky)
                for (int kx = kx0; kx <= kx1; ++kx) v += src[(((long)co * w_cin + ci) * 3 + ky) * 3 + kx];
        } else {  // CONVT_4x4_S2: weight [Cin][Cout][4][4]; phase (py,px), tap (ty,tx): k = (p==0) ? {1,3}[t] : {0,2}[t]
            int py = ph >> 1, px = ph & 1, ty = tap >> 1, tx = tap & 1;
            int ky = (py == 0) ? (ty == 0 ? 1 : 3) : (ty == 0 ? 0 : 2);
            int kx = (px == 0) ? (tx == 0 ? 1 : 3) : (tx == 0 ? 0 : 2);
            v = src[(((long)ci * cout + co) * 4 + ky) * 4 + kx];
        }
        dst[(((long)ph * ntaps + tap) * cout_pad + co) * cin_pad + cin_offset + ci] = round_w ? round_tf32(v) : v;
    }
}

}  // namespace

void conv_describe(ConvWeights& cw, ConvKind kind, int cin, int cout) {
    cw.cin = cin; cw.cout = cout;
    cw.cin_pad = round_up(cin, BK);
    cw.cout_pad = round_up(cout, 32);
    cw.nphase = 1; cw.stride = 1; cw.out_mul = 1;
    for (int ph = 0; ph < CONV_MAX_PHASES; ++ph) {
        cw.ph_oy[ph] = cw.ph_ox[ph] = 0;
        for (int t = 0; t < CONV_MAX_TAPS; ++t) cw.dy[ph][t] = cw.dx[ph][t] = 0;
    }
    if (kind == CONV_3x3) {
        cw.ntaps = 9;
        for (int t = 0; t < 9; ++t) { cw.dy[0][t] = (signed char)(t / 3 - 1); cw.dx[0][t] = (signed char)(t % 3 - 1); }
    } else if (kind == CONV_4x4_S2) {
        cw.ntaps = 16; cw.stride = 2;
        for (int t = 0; t < 16; ++t) { cw.dy[0][t] = (signed char)(t / 4 - 1); cw.dx[0][t] = (signed char)(t % 4 - 1); }
    } else if (kind == CONV_1x1) {
        cw.ntaps = 1;
    } else if (kind == CONV_UP2_3x3) {
        cw.ntaps = 4; cw.nphase = 4; cw.out_mul = 2;
        for (int ph = 0; ph < 4; ++ph) {
            int py = ph >> 1, px = ph & 1;
            cw.ph_oy[ph] = (signed char)py; cw.ph_ox[ph] = (signed char)px;
            for (int t = 0; t < 4; ++t) {
                int ty = t >> 1, tx = t & 1;
                cw.dy[ph][t] = (signed char)((py == 0) ? (ty == 0 ? -1 : 0) : (ty == 0 ? 0 : 1));
                cw.dx[ph][t] = (signed char)((px == 0) ? (tx == 0 ? -1 : 0) : (tx == 0 ? 0 : 1));
            }
        }
    } else {
        // out[2a+py] = sum_ky in[(2a+py+1-ky)/2] w[ky]  (stride 2, pad 1):  py=0: ky=1 -> a, ky=3 -> a-1;
        //                                                                py=1: ky=0 -> a+1, ky=2 -> a.
        cw.ntaps = 4; cw.nphase = 4; cw.out_mul = 2;
        for (int ph = 0; ph < 4; ++ph) {
            int py = ph >> 1, px = ph & 1;
            cw.ph_oy[ph] = (signed char)py; cw.ph_ox[ph] = (signed char)px;
            for (int t = 0; t < 4; ++t) {
                int ty = t >> 1, tx = t & 1;
                cw.dy[ph][t] = (signed char)((py == 0) ? (ty == 0 ? 0 : -1) : (ty == 0 ? 1 : 0));
                cw.dx[ph][t] = (signed char)((px == 0) ? (tx == 0 ? 0 : -1) : (tx == 0 ? 1 : 0));
            }
        }
    }
}

static thread_local bool g_pack_round = true;   // set by the caller right before it packs (tha4_load_net): per thread, not per process
void conv_set_pack_rounding(bool r) { g_pack_round = r; }
bool conv_pack_rounding() { return g_pack_round; }

size_t conv_packed_floats(const ConvWeights& cw) {
    return (size_t)cw.nphase * cw.ntaps * cw.cout_pad * cw.cin_pad;
}

void conv_pack(const ConvWeights& cw, ConvKind kind, const float* w_ref, int w_cin, int cin_offset, cudaStream_t s) {
    THA4_REQUIRE(cin_offset + w_cin <= cw.cin_pad, "conv_pack: cin range");
    long total = (long)cw.nphase * cw.ntaps * cw.cout * w_cin;
    int blocks = (int)std::min<long>(4096, (total + 255) / 256);
    conv_pack_kernel<<<blocks, 256, 0, s>>>(cw.w, w_ref, (int)kind, w_cin, cin_offset, cw.cout, cw.cin_pad,
                                           cw.cout_pad, cw.ntaps, cw.nphase, g_pack_round ? 1 : 0);
    THA4_LAUNCH_CHECK();
}

bool conv_fuses_stats(const ConvWeights& cw, const ConvArgs& a) {
    if (a.out.stats == nullptr || !opts().tcgen05) return false;
    if (conv_halo_supported(cw, a)) return true;
    return conv_tc_supported(cw, a) && conv_tc_fuses_stats(cw, a);
}

void conv_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s) {
    const bool tc = opts().tcgen05;
    if (a.nin.on || a.out16.p || !a.out.p)
        THA4_REQUIRE(tc && conv_tc_supported(cw, a), "conv: fused input normalisation / f16 outputs exist on the wgmma kernel only");
    THA4_REQUIRE(cw.cin2 == 0 || (tc && conv_halo_supported(cw, a)), "conv: a folded 1x1 conv runs on the halo kernel only");
    if (tc && conv_halo_supported(cw, a)) conv_halo_forward(cw, a, s);
    else if (tc && conv_tc_supported(cw, a)) conv_tc_forward(cw, a, s);
    else conv_mma_forward(cw, a, s);
}

void conv_mma_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s) {
    THA4_REQUIRE(!(a.strict && cw.tf32_rounded), "strict mode needs weights packed without TF32 rounding: set the option before loading");
    THA4_REQUIRE(!a.in.f16 && !a.out.f16, "conv (mma.sync path): fp32 activations only");
    ConvKernelParams p{};
    THA4_REQUIRE(a.in.C == cw.cin, "conv: input channels");
    THA4_REQUIRE(a.out.C == cw.cout, "conv: output channels");
    THA4_REQUIRE(a.in.C % 4 == 0 && a.in.ld % 4 == 0 && (((uintptr_t)a.in.p) & 15) == 0, "conv: input alignment");
    THA4_REQUIRE(a.out.ld % 2 == 0 && (((uintptr_t)a.out.p) & 7) == 0, "conv: output alignment");
    p.in = a.in.p; p.inH = a.in.H; p.inW = a.in.W; p.inC = a.in.C; p.in_ld = a.in.ld;
    p.in_up = a.in_up;
    p.LH = a.in_up ? 2 * a.in.H : a.in.H;
    p.LW = a.in_up ? 2 * a.in.W : a.in.W;
    p.w = cw.w; p.bias = cw.bias;
    p.out = a.out.p; p.outH = a.out.H; p.outW = a.out.W; p.outC = a.out.C; p.out_ld = a.out.ld;
    p.N = a.in.N;
    THA4_REQUIRE(a.out.N == a.in.N, "conv: batch");
    p.stride = cw.stride; p.out_mul = cw.out_mul; p.ntaps = cw.ntaps; p.nphase = cw.nphase;
    p.MH = a.out.H / cw.out_mul; p.MW = a.out.W / cw.out_mul;
    if (cw.out_mul == 2) THA4_REQUIRE(p.MH == p.LH && p.MW == p.LW, "convT: geometry");
    else THA4_REQUIRE(p.MH * cw.stride == p.LH && p.MW * cw.stride == p.LW, "conv: geometry");
    p.M_total = (long)p.N * p.MH * p.MW;
    p.cin_pad = cw.cin_pad; p.cout_pad = cw.cout_pad;
    p.strict = a.strict;
    p.res = a.res.p; p.res_mode = a.res.p ? a.res_mode : RES_NONE;
    p.resH = a.res.H; p.resW = a.res.W; p.res_ld = a.res.ld;
    if (p.res_mode == RES_SAME) THA4_REQUIRE(a.res.H == a.out.H && a.res.W == a.out.W && a.res.C == a.out.C, "conv: res dims");
    if (p.res_mode == RES_UP2) THA4_REQUIRE(a.res.H * 2 == a.out.H && a.res.C == a.out.C, "conv: res up dims");
    if (p.res_mode == RES_DOWN2) THA4_REQUIRE(a.res.H == a.out.H * 2 && a.res.C == a.out.C, "conv: res down dims");
    for (int ph = 0; ph < CONV_MAX_PHASES; ++ph) {
        p.ph_oy[ph] = cw.ph_oy[ph]; p.ph_ox[ph] = cw.ph_ox[ph];
        for (int t = 0; t < CONV_MAX_TAPS; ++t) { p.dy[ph][t] = cw.dy[ph][t]; p.dx[ph][t] = cw.dx[ph][t]; }
    }

    const int bn = (cw.cout_pad % 128 == 0) ? 128 : (cw.cout_pad % 64 == 0 ? 64 : 32);
    const int tiles_m = ceil_div(p.M_total, BM);
    const int tiles_n = ceil_div(cw.cout_pad, bn);
    const int KT = cw.ntaps * (cw.cin_pad / BK);
    int ksplit = a.ksplit;
    if (ksplit <= 0) {
        long ctas = (long)tiles_m * tiles_n * cw.nphase;
        ksplit = 1;
        if (ctas < 96) {
            ksplit = (int)((192 + ctas - 1) / ctas);
            ksplit = std::min(ksplit, std::max(1, KT / 8));
            ksplit = std::min(ksplit, 32);
        }
    }
    ksplit = std::max(1, std::min(ksplit, KT));
    p.ksplit = ksplit;
    if (ksplit > 1) {
        THA4_CUDA_CHECK(cudaMemset2DAsync(a.out.p, (size_t)a.out.ld * sizeof(float), 0, (size_t)a.out.C * sizeof(float),
                                          a.out.pixels(), s));
    }
    dim3 grid(tiles_m, tiles_n, cw.nphase * ksplit);
    ProfScope prof(PROF_CONV, s);
    prof_add_work(PROF_CONV, 2.0 * (double)p.M_total * cw.cout * cw.cin * cw.ntaps * cw.nphase, 0.0);
    if (bn == 128) launch_conv<128, 2, 4, 3>(p, grid, s);
    else if (bn == 64) launch_conv<64, 4, 2, 4>(p, grid, s);
    else launch_conv<32, 8, 1, 4>(p, grid, s);
}

}  // namespace tha4
