// Input gradients of the encoder-decoder teacher networks (EyebrowDecomposer00, EyebrowMorphingCombiner00, FaceMorpher08;
// poser_encoder_decoder_00.py:99-121, face_morpher_08.py:158-193): d(image), d(layers) and d(pose) for upstream gradients of
// the outputs.
//
// The forward is recomputed with the inference kernels of the context's precision mode, keeping every raw conv output and its
// statistics (EncDecTape).  The backward then runs, layer by layer:
//   tail: outputs' gradients -> head pre-activation gradients (blends, sigmoid / tanh from the returned values, grid_sample
//         w.r.t. the grid) + the image terms (direct blend terms, grid_sample adjoint scattered into the sampled corners);
//   convs: data gradients on the same conv kernels with adjoint-packed weights (3x3 -> 3x3 with W^T flipped, 4x4 s2 conv <->
//         4x4 s2 transposed conv), fp32 operands (TF32, or 3xTF32 in strict mode), never through f16 storage;
//   InstanceNorm (+ReLU): dz = dy [A x + B > 0];  dx = gamma rstd (dz - mean(dz) - xhat mean(dz xhat)), sums in fp64;
//   pose: spatial sum of the pose channels of the bottleneck entry's data gradient, in a fixed order (no atomics).
#include "nets.cuh"
#include "gridsample.cuh"

namespace tha4 {

namespace {

// adjoint of a 3x3 s1 p1 conv weight [cout][cin][3][3]: dst[ci][co][ky][kx] = src[co][ci][2-ky][2-kx]
__global__ void adjoint3x3_kernel(float* __restrict__ dst, const float* __restrict__ src, int cout, int cin) {
    const long total = (long)cout * cin * 9;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int k = (int)(i % 9);
        const long r = i / 9;
        const int ci = (int)(r % cin), co = (int)(r / cin);
        dst[((long)ci * cout + co) * 9 + 8 - k] = src[i];
    }
}

// adjoint of the fused tail's head conv (tw.w: [9][C][TAIL_CO_PAD]) as a packed 3x3 conv from CO head channels to C:
// dst[tap][c][co] = W[co][c][8 - tap]
__global__ void head_adjoint_pack_kernel(float* __restrict__ dst, const float* __restrict__ tw, int C, int CO, int cin_pad,
                                         int cout_pad, int round_w) {
    const int total = 9 * C * CO;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int co = i % CO, r = i / CO;
        const int c = r % C, t = r / C;
        const float v = tw[((8 - t) * C + c) * TAIL_CO_PAD + co];
        dst[((long)t * cout_pad + c) * cin_pad + co] = round_w ? round_tf32(v) : v;
    }
}

// mean and rstd of channel c of sample n, in the arithmetic of the forward's normalisation kernels
__device__ __forceinline__ float2 in_mean_rstd(const double* __restrict__ stats, int stats_ld, int rep, long rep_stride, int n, int c,
                                               int HW) {
    const double2 v = fold_stat_replicas(stats + ((long)n * stats_ld + c) * 2, rep_stride, rep);
    const double mean = v.x / HW;
    double var = v.y / HW - mean * mean;
    if (var < 0.0) var = 0.0;
    return make_float2((float)mean, (float)(1.0 / sqrt(var + 1e-5)));
}

template <bool F16>
__device__ __forceinline__ float4 load4(const float* p, long off) {
    if (F16) {
        const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(p) + off);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    return *reinterpret_cast<const float4*>(p + off);
}

struct NormBwdArgs {
    const float* x; int x_ld, x_f16;                   // RAW input of the normalisation (NHWC)
    const double* stats; int stats_ld, stats_rep; long stats_rep_stride;
    const float* gamma; const float* beta;
    int act;                                          // ACT_RELU or ACT_NONE
    const float* dy; int dy_ld;                       // gradient of the (activated) output, fp32 NHWC
    float* dx; int dx_ld;
    double* sums;                                     // [N][C][2]: sum dz, sum dz xhat (zero on entry)
    int C, HW;
};

constexpr int NB_PIX_PER_THREAD = 32;

// stage 1: per-(n,c) sums of dz and dz * xhat (fp32 per thread, fp64 across threads and CTAs)
template <bool F16>
__global__ void __launch_bounds__(256) norm_bwd_reduce_kernel(const NormBwdArgs a) {
    __shared__ float red[256][9];
    const int cq = a.C >> 2, PL = 256 / cq;
    const int tid = threadIdx.x, pl = tid / cq, q = tid - pl * cq;
    const int n = blockIdx.y;
    const bool active = pl < PL;
    float s[4] = {0, 0, 0, 0}, sx[4] = {0, 0, 0, 0};
    if (active) {
        float mean[4], rstd[4], A[4], Bc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = 4 * q + k;
            const float2 mr = in_mean_rstd(a.stats, a.stats_ld, a.stats_rep, a.stats_rep_stride, n, c, a.HW);
            mean[k] = mr.x; rstd[k] = mr.y;
            A[k] = mr.y * a.gamma[c]; Bc[k] = a.beta[c] - mr.x * A[k];
        }
        const long base = (long)blockIdx.x * PL * NB_PIX_PER_THREAD;
        for (int i = 0; i < NB_PIX_PER_THREAD; ++i) {
            const long pix = base + (long)i * PL + pl;
            if (pix >= a.HW) break;
            const long p = (long)n * a.HW + pix;
            const float4 xv = load4<F16>(a.x, p * a.x_ld + 4 * q);
            const float4 gv = *reinterpret_cast<const float4*>(a.dy + p * a.dy_ld + 4 * q);
            const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float dz = (a.act == ACT_RELU && !(xs[k] * A[k] + Bc[k] > 0.0f)) ? 0.0f : gs[k];
                s[k] += dz;
                sx[k] += dz * ((xs[k] - mean[k]) * rstd[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { red[tid][k] = s[k]; red[tid][4 + k] = sx[k]; }
    __syncthreads();
    if (active && pl == 0) {
        double acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0;
        for (int j = 0; j < PL; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += (double)red[j * cq + q][k];
        double* dst = a.sums + ((long)n * a.C + 4 * q) * 2;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            atomicAdd(dst + 2 * k, acc[k]);
            atomicAdd(dst + 2 * k + 1, acc[4 + k]);
        }
    }
}

// stage 2: dx = gamma rstd (dz - mean(dz) - xhat mean(dz xhat)), one float4 of channels per thread and step
template <bool F16>
__global__ void __launch_bounds__(256) norm_bwd_apply_kernel(const NormBwdArgs a, long total) {
    const int cq = a.C >> 2;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long p = i / cq;
        const int q = (int)(i - p * cq);
        const int n = (int)(p / a.HW);
        const float4 xv = load4<F16>(a.x, p * a.x_ld + 4 * q);
        const float4 gv = *reinterpret_cast<const float4*>(a.dy + p * a.dy_ld + 4 * q);
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = 4 * q + k;
            const float2 mr = in_mean_rstd(a.stats, a.stats_ld, a.stats_rep, a.stats_rep_stride, n, c, a.HW);
            const float A = mr.y * a.gamma[c], B = a.beta[c] - mr.x * A;
            const float dz = (a.act == ACT_RELU && !(xs[k] * A + B > 0.0f)) ? 0.0f : gs[k];
            const double* sm = a.sums + ((long)n * a.C + c) * 2;
            const float m1 = (float)(sm[0] / a.HW), m2 = (float)(sm[1] / a.HW);
            const float xhat = (xs[k] - mr.x) * mr.y;
            o[k] = A * (dz - m1 - xhat * m2);
        }
        *reinterpret_cast<float4*>(a.dx + p * a.dx_ld + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// d pose[n][k] = sum over the pixels of sample n of d_bin[n, pixel, c0 + k], in pixel order (fp64, no atomics)
__global__ void pose_sum_kernel(const float* __restrict__ dbin, int ld, long hw, int c0, int P, float* __restrict__ dpose, int dpose_ld) {
    const int n = blockIdx.x, k = threadIdx.x;
    if (k >= P) return;
    const float* src = dbin + (long)n * hw * ld + c0 + k;
    double acc = 0.0;
    for (long p = 0; p < hw; ++p) acc += (double)src[p * ld];
    dpose[(long)n * dpose_ld + k] = (float)acc;
}

__device__ __forceinline__ float gv(const float* g, long off) { return g ? g[off] : 0.0f; }

// Tail backward, one thread per pixel.  out[k] / g[k]: the forward's returned tensors and their upstream gradients (NCHW,
// g[k] may be null).  dh: [P][16] gradients of the head pre-activations in the tail's channel order.  d0 / d1 (NHWC, `dld`
// floats per pixel, null = not wanted): d(image0) / d(image1).  Only one kind of term lands on each image, so the direct
// terms are plain stores and the grid_sample adjoint is scattered with atomics (d0 zeroed by the caller when KIND warps).
struct TailBwdArgs {
    const float* out[8];
    const float* g[8];
    ImgView img0, img1;
    const float* base;
    int S, N;
    float* dh;
    float* d0; float* d1; int dld;
};

template <int KIND>
__global__ void __launch_bounds__(256) tail_bwd_kernel(const TailBwdArgs a) {
    const int S = a.S;
    const long hw = (long)S * S, total = (long)a.N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % S), y = (int)((i / S) % S), n = (int)(i / hw);
        const long pp = i - (long)n * hw;
        auto at = [&](int, int c, int ch) { return ((long)n * ch + c) * hw + pp; };
        float dh[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) dh[k] = 0.0f;
        if (KIND == TAIL_DECOMPOSER) {
            // outputs: eb_layer(4) eb_alpha(1) eb_color(4) bg_layer(4) bg_alpha(1) bg_color(4); heads: bg_a(0) bg_c(1..4) eb_a(5) eb_c(6..9)
            const float eba = a.out[1][at(1, 0, 1)], bga = a.out[4][at(4, 0, 1)];
            float deba = gv(a.g[1], at(1, 0, 1)), dbga = gv(a.g[4], at(4, 0, 1)), dimg[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float img = __ldg(a.img0.p + n * a.img0.sn + c * a.img0.sc + (long)y * a.img0.sh + x);
                const float ebc = a.out[2][at(2, c, 4)], bgc = a.out[5][at(5, c, 4)];
                const float g0 = gv(a.g[0], at(0, c, 4)), g3 = gv(a.g[3], at(3, c, 4));
                deba += g0 * (img - ebc);
                dbga += g3 * (bgc - img);
                const float debc = gv(a.g[2], at(2, c, 4)) + g0 * (1.0f - eba);
                const float dbgc = gv(a.g[5], at(5, c, 4)) + g3 * bga;
                dh[6 + c] = debc * (1.0f - ebc * ebc);
                dh[1 + c] = dbgc * (1.0f - bgc * bgc);
                dimg[c] = g0 * eba + g3 * (1.0f - bga);
            }
            dh[0] = dbga * bga * (1.0f - bga);
            dh[5] = deba * eba * (1.0f - eba);
            if (a.d0) *reinterpret_cast<float4*>(a.d0 + i * a.dld) = make_float4(dimg[0], dimg[1], dimg[2], dimg[3]);
        } else {
            // combiner: outputs e0(4) ca(1) e1(4) morphed(4) alpha(1) color(4) warped(4) grid(2); heads grid(0,1) alpha(2) color(3..6) ca(7)
            // face:     outputs out(4) eya(1) eyc(4) im1(4) ima(1) imc(4) im0(4) grid(2);     heads grid(0,1) imc(2..5) ima(6) eyc(7..10) eya(11)
            float dwarp[4];
            if (KIND == TAIL_COMBINER) {
                const float ca = a.out[1][at(1, 0, 1)], alpha = a.out[4][at(4, 0, 1)];
                float m[4], col[4], wp[4], bg[4], dm[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    m[c] = a.out[3][at(3, c, 4)]; col[c] = a.out[5][at(5, c, 4)]; wp[c] = a.out[6][at(6, c, 4)];
                    bg[c] = __ldg(a.img1.p + n * a.img1.sn + c * a.img1.sc + (long)y * a.img1.sh + x);
                    dm[c] = gv(a.g[3], at(3, c, 4));
                }
                const float a2 = (m[3] + 1.0f) / 2.0f;
                float dca = gv(a.g[1], at(1, 0, 1)), da2 = 0.0f, dbg[4];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float g0 = gv(a.g[0], at(0, c, 4)), g2 = gv(a.g[2], at(2, c, 4));
                    dm[c] += g0 * ca + g2 * a2;
                    dca += g0 * (m[c] - bg[c]);
                    da2 += g2 * (m[c] - bg[c]);
                    dbg[c] = g0 * (1.0f - ca) + g2 * (1.0f - a2);
                }
                dbg[3] = gv(a.g[0], at(0, 3, 4)) + gv(a.g[2], at(2, 3, 4));
                dm[3] += da2 * 0.5f;
                float dalpha = gv(a.g[4], at(4, 0, 1));
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float dcol = gv(a.g[5], at(5, c, 4)) + dm[c] * alpha;
                    dalpha += dm[c] * (col[c] - wp[c]);
                    dwarp[c] = gv(a.g[6], at(6, c, 4)) + dm[c] * (1.0f - alpha);
                    dh[3 + c] = dcol * (1.0f - col[c] * col[c]);
                }
                dh[2] = dalpha * alpha * (1.0f - alpha);
                dh[7] = dca * ca * (1.0f - ca);
                if (a.d1) *reinterpret_cast<float4*>(a.d1 + i * a.dld) = make_float4(dbg[0], dbg[1], dbg[2], dbg[3]);
            } else if (KIND == TAIL_UNET) {
                // U-Net: outputs merged(4) alpha(1) warped(4) grid(2) direct(4); heads direct(0..3) grid(4,5) alpha logit(6)
                const float alpha = a.out[1][at(1, 0, 1)];
                float dalpha = gv(a.g[1], at(1, 0, 1));
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float direct = a.out[4][at(4, c, 4)], warped = a.out[2][at(2, c, 4)];
                    const float g0 = gv(a.g[0], at(0, c, 4));
                    dh[c] = gv(a.g[4], at(4, c, 4)) + g0 * alpha;
                    dalpha += g0 * (direct - warped);
                    dwarp[c] = gv(a.g[2], at(2, c, 4)) + g0 * (1.0f - alpha);
                }
                dh[6] = dalpha * alpha * (1.0f - alpha);
            } else {
                const float eya = a.out[1][at(1, 0, 1)], ima = a.out[4][at(4, 0, 1)];
                float deya = gv(a.g[1], at(1, 0, 1)), dima = gv(a.g[4], at(4, 0, 1));
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float eyc = a.out[2][at(2, c, 4)], im1 = a.out[3][at(3, c, 4)];
                    const float imc = a.out[5][at(5, c, 4)], im0 = a.out[6][at(6, c, 4)];
                    const float g0 = gv(a.g[0], at(0, c, 4));
                    const float deyc = gv(a.g[2], at(2, c, 4)) + g0 * eya;
                    deya += g0 * (eyc - im1);
                    const float dim1 = gv(a.g[3], at(3, c, 4)) + g0 * (1.0f - eya);
                    const float dimc = gv(a.g[5], at(5, c, 4)) + dim1 * ima;
                    dima += dim1 * (imc - im0);
                    dwarp[c] = gv(a.g[6], at(6, c, 4)) + dim1 * (1.0f - ima);
                    dh[2 + c] = dimc * (1.0f - imc * imc);
                    dh[7 + c] = deyc * (1.0f - eyc * eyc);
                }
                dh[6] = dima * ima * (1.0f - ima);
                dh[11] = deya * eya * (1.0f - eya);
            }
            // grid_sample(img0, base + grid) w.r.t. the grid (zero where the border clamp is active) and w.r.t. img0
            constexpr int GO = KIND == TAIL_UNET ? 3 : 7, GH = KIND == TAIL_UNET ? 4 : 0;     // grid output, grid head channel
            const float gcx = a.out[GO][at(GO, 0, 2)], gcy = a.out[GO][at(GO, 1, 2)];
            const SampleAt sa = sample_locate(a.base, x, y, gcx, gcy, S);
            float gix = 0.0f, giy = 0.0f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const Corners v = sample_corners(a.img0.p + n * a.img0.sn + c * a.img0.sc, a.img0.sh, sa);
                gix += dwarp[c] * sample_dix(v, sa);
                giy += dwarp[c] * sample_diy(v, sa);
            }
            dh[GH] = gv(a.g[GO], at(GO, 0, 2)) + gix * sa.mx;
            dh[GH + 1] = gv(a.g[GO], at(GO, 1, 2)) + giy * sa.my;
            if (a.d0)        // corners and weights of the inference tail (gs_locate / gs_sample), as image_grad_kernel
                gs_scatter4_nhwc(a.d0 + (long)n * hw * a.dld, a.dld, S, S, gs_locate(a.base[x], a.base[y], gcx, gcy, S, S), dwarp);
        }
        float4* d = reinterpret_cast<float4*>(a.dh + i * 16);
        d[0] = make_float4(dh[0], dh[1], dh[2], dh[3]);
        d[1] = make_float4(dh[4], dh[5], dh[6], dh[7]);
        d[2] = make_float4(dh[8], dh[9], dh[10], dh[11]);
        d[3] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

int grid_for(long n) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, 132L * 16)); }

View fresh(Pool* P, int N, int H, int W, int C) {
    View v; v.N = N; v.H = H; v.W = W; v.C = C; v.ld = C;
    v.p = P->alloc((size_t)N * H * W * C);
    return v;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ shared entry points
void run_dgrad(Runtime& rt, const ConvWeights& cw, const View& dy, const View& dx, const View* add) {
    ConvArgs a;
    a.in = dy; a.out = dx; a.strict = rt.strict;
    if (add) { a.res = *add; a.res_mode = RES_SAME; }
    const size_t ws = conv_workspace_floats(cw, a);
    if (ws) { a.ws = rt.scratch->alloc(ws); a.ws_floats = ws; }
    conv_forward(cw, a, rt.stream);
}

void head_pack_adjoint(ConvWeights& cw, const TailWeights& tw, bool round_w, cudaStream_t s) {
    conv_describe(cw, CONV_3x3, 16, tw.C);
    cw.w = reinterpret_cast<float*>(tracked_malloc(conv_packed_floats(cw) * sizeof(float)));
    THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
    cw.tf32_rounded = round_w;
    head_adjoint_pack_kernel<<<grid_for(9L * tw.C * tw.CO), 256, 0, s>>>(cw.w, tw.w, tw.C, tw.CO, cw.cin_pad, cw.cout_pad, round_w ? 1 : 0);
    THA4_LAUNCH_CHECK();
}

void conv_pack_adjoint(ConvWeights& cw, ConvKind kind, const float* w_ref, int cin, int cout, int cout_kernel, cudaStream_t s) {
    // kind / cin / cout describe the FORWARD conv (w_ref in its reference layout); cw becomes the conv from cout to cin channels
    // (cout_kernel >= cin output channels, the extra ones zero)
    THA4_REQUIRE(kind == CONV_3x3 || kind == CONV_4x4_S2 || kind == CONVT_4x4_S2, "conv adjoint: kind");
    const int oc = std::max(cout_kernel, cin);
    const ConvKind adj = kind == CONV_3x3 ? CONV_3x3 : (kind == CONV_4x4_S2 ? CONVT_4x4_S2 : CONV_4x4_S2);
    conv_describe(cw, adj, round_up(cout, 4), oc);
    cw.w = reinterpret_cast<float*>(tracked_malloc(conv_packed_floats(cw) * sizeof(float)));
    THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
    cw.tf32_rounded = conv_pack_rounding();
    if (kind == CONV_3x3) {
        float* tmp = nullptr;
        const size_t n = (size_t)oc * cout * 9;
        THA4_CUDA_CHECK(cudaMalloc(&tmp, n * sizeof(float)));
        THA4_CUDA_CHECK(cudaMemsetAsync(tmp, 0, n * sizeof(float), s));
        adjoint3x3_kernel<<<grid_for((long)cout * cin * 9), 256, 0, s>>>(tmp, w_ref, cout, cin);
        THA4_LAUNCH_CHECK();
        conv_pack(cw, CONV_3x3, tmp, cout, 0, s);
        THA4_CUDA_CHECK(cudaStreamSynchronize(s));
        cudaFree(tmp);
    } else {
        THA4_REQUIRE(oc == cin, "conv adjoint: padded outputs only for 3x3 convs");
        conv_pack(cw, adj, w_ref, cout, 0, s);       // the same tensor, read in the other kind's layout
    }
}

void norm_backward(const View& x, const float* gamma, const float* beta, int act, const View& dy, const View& dx, double* sums,
                   cudaStream_t s) {
    THA4_REQUIRE(x.stats != nullptr && dy.C == x.C && dx.C == x.C && x.C % 4 == 0 && x.C <= 1024, "norm backward: channels");
    THA4_REQUIRE(!dy.f16 && !dx.f16 && dy.ld % 4 == 0 && dx.ld % 4 == 0 && x.ld % 4 == 0, "norm backward: layouts");
    NormBwdArgs a;
    a.x = x.p; a.x_ld = x.ld; a.x_f16 = x.f16;
    a.stats = x.stats; a.stats_ld = x.stats_ld; a.stats_rep = x.stats_rep; a.stats_rep_stride = x.stats_rep_stride;
    a.gamma = gamma; a.beta = beta; a.act = act;
    a.dy = dy.p; a.dy_ld = dy.ld; a.dx = dx.p; a.dx_ld = dx.ld; a.sums = sums;
    a.C = x.C; a.HW = x.H * x.W;
    const int PL = 256 / (x.C / 4);
    dim3 g1(ceil_div(a.HW, PL * NB_PIX_PER_THREAD), x.N);
    const long total = (long)x.N * a.HW * (x.C / 4);
    if (x.f16) {
        norm_bwd_reduce_kernel<true><<<g1, 256, 0, s>>>(a);
        THA4_LAUNCH_CHECK();
        norm_bwd_apply_kernel<true><<<grid_for(total), 256, 0, s>>>(a, total);
    } else {
        norm_bwd_reduce_kernel<false><<<g1, 256, 0, s>>>(a);
        THA4_LAUNCH_CHECK();
        norm_bwd_apply_kernel<false><<<grid_for(total), 256, 0, s>>>(a, total);
    }
    THA4_LAUNCH_CHECK();
}

void tail_backward(TailKind kind, const float* const* outputs, const float* const* grads, const ImgView& image0, const ImgView& image1,
                   const View& dh, float* d0, float* d1, int dld, cudaStream_t s) {
    THA4_REQUIRE(dh.C == 16 && dh.ld == 16 && dh.H == image0.H && dh.W == image0.W && image0.H == image0.W, "tail backward: dims");
    TailBwdArgs a;
    const int nout = kind == TAIL_UNET ? 5 : (kind == TAIL_DECOMPOSER ? 6 : 8);
    for (int k = 0; k < 8; ++k) { a.out[k] = k < nout ? outputs[k] : nullptr; a.g[k] = (grads && k < nout) ? grads[k] : nullptr; }
    a.img0 = image0; a.img1 = image1; a.base = base_grid_table(image0.H);
    a.S = image0.H; a.N = dh.N; a.dh = dh.p; a.d0 = d0; a.d1 = d1; a.dld = dld;
    const long total = (long)a.N * a.S * a.S;
    if (kind == TAIL_UNET) tail_bwd_kernel<TAIL_UNET><<<grid_for(total), 256, 0, s>>>(a);
    else if (kind == TAIL_DECOMPOSER) tail_bwd_kernel<TAIL_DECOMPOSER><<<grid_for(total), 256, 0, s>>>(a);
    else if (kind == TAIL_COMBINER) tail_bwd_kernel<TAIL_COMBINER><<<grid_for(total), 256, 0, s>>>(a);
    else tail_bwd_kernel<TAIL_FACE><<<grid_for(total), 256, 0, s>>>(a);
    THA4_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------------ EncDecNet
void EncDecNet::load_adjoints(const StateDict& sd, const std::string& p, cudaStream_t s) {
    auto adj = [&](ConvWeights& cw, const std::string& key, ConvKind kind, int cout_kernel = 0) {
        auto it = sd.find(key + ".weight");
        THA4_REQUIRE(it != sd.end(), "state_dict is missing key " + key + ".weight");
        const TensorRef& w = it->second;
        const int cout = (int)(kind == CONVT_4x4_S2 ? w.shape[1] : w.shape[0]);
        const int cin = (int)(kind == CONVT_4x4_S2 ? w.shape[0] : w.shape[1]);
        conv_pack_adjoint(cw, kind, w.p, cin, cout, cout_kernel, s);
    };
    adj(adj_down_[0], p + "downsample_blocks.0.0", CONV_3x3);
    for (int i = 1; i < 4; ++i) adj(adj_down_[i], p + "downsample_blocks." + std::to_string(i) + ".0", CONV_4x4_S2);
    adj(adj_bott0_, p + "bottleneck_blocks.0.0", CONV_3x3, 512 + pose_pad_);
    for (int i = 0; i < 5; ++i) {
        const std::string rp = p + "bottleneck_blocks." + std::to_string(i + 1) + ".resnet_path.";
        adj(adj_res_[i][0], rp + "0", CONV_3x3);
        adj(adj_res_[i][1], rp + "3", CONV_3x3);
    }
    for (int i = 0; i < 3; ++i) adj(adj_up_[i], p + "upsample_blocks." + std::to_string(i) + ".0", CONVT_4x4_S2);
    // the heads: one 3x3 conv from the 16-channel head-gradient tensor to the 64 feature channels
    head_pack_adjoint(adj_head_, tail_, conv_pack_rounding(), s);
}

void EncDecNet::backward(Runtime& rt, const ImgView& image0, const ImgView& image1, const float* pose, int pose_ld, const EncDecGrads& g) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    const bool want_img = g.d_image0 || g.d_image1, want_pose = g.d_pose != nullptr;
    THA4_REQUIRE(want_img || want_pose, "encdec backward: no gradient requested");
    THA4_REQUIRE(!want_pose || pose_ch_ > 0, "encdec backward: this network has no pose input");
    THA4_REQUIRE(!g.d_image1 || kind_ == TAIL_COMBINER, "encdec backward: only the combiner has a second image");
    const int B = image0.N, S = S_, b = S_ / 8;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;

    // forward, keeping the activations (its outputs are what the tail backward differentiates through)
    static const int kChDec[6] = {4, 1, 4, 4, 1, 4}, kCh8[8] = {4, 1, 4, 4, 1, 4, 4, 2};
    const int* ch = kind_ == TAIL_DECOMPOSER ? kChDec : kCh8;
    float* outs[8] = {};
    for (int k = 0; k < num_outputs(); ++k) outs[k] = P->alloc((size_t)B * ch[k] * S * S);
    EncDecTape tape;
    forward(rt, image0, image1, pose, pose_ld, outs, &tape);

    auto nbwd = [&](const View& x, const NormW& nw, int act, const View& dy) {
        THA4_REQUIRE(nw.C == x.C, "norm backward: channel mismatch");
        View dx = fresh(P, x.N, x.H, x.W, x.C);
        norm_backward(x, nw.gamma, nw.beta, act, dy, dx, rt.alloc_stats((size_t)x.N * x.C * 2), s);
        return dx;
    };
    // tail: head pre-activation gradients + the image terms (in the layout of the network input x0)
    View dh = fresh(P, B, S, S, 16);
    View dimg;
    if (want_img) {
        dimg = fresh(P, B, S, S, in_ch_);
        THA4_CUDA_CHECK(cudaMemsetAsync(dimg.p, 0, dimg.pixels() * in_ch_ * sizeof(float), s));
    }
    // combiner: x0 = [background | eyebrow] (image1 | image0)
    float* d0 = want_img ? dimg.p + (kind_ == TAIL_COMBINER ? 4 : 0) : nullptr;
    float* d1 = want_img && kind_ == TAIL_COMBINER ? dimg.p : nullptr;
    tail_backward(kind_, outs, g.grad_outputs, image0, image1, dh, d0, d1, in_ch_, s);
    View df = fresh(P, B, S, S, tail_.C);
    run_dgrad(rt, adj_head_, dh, df);
    // decoder
    View d = nbwd(tape.up[2], up_n_[2], ACT_RELU, df);
    for (int i = 2; i >= 1; --i) {
        View da = fresh(P, B, b << i, b << i, adj_up_[i].cout);
        run_dgrad(rt, adj_up_[i], d, da);
        d = nbwd(tape.up[i - 1], up_n_[i - 1], ACT_RELU, da);
    }
    View gx = fresh(P, B, b, b, 512);
    run_dgrad(rt, adj_up_[0], d, gx);
    // ResnetBlocks: x + IN(conv(relu(IN(conv(x))))): the residual gradient joins in the epilogue of the first conv's adjoint
    for (int i = 4; i >= 0; --i) {
        View d1n = nbwd(tape.res[i][1], res_n_[i][1], ACT_NONE, gx);
        View dh1 = fresh(P, B, b, b, 512);
        run_dgrad(rt, adj_res_[i][1], d1n, dh1);
        View d0n = nbwd(tape.res[i][0], res_n_[i][0], ACT_RELU, dh1);
        View gn = fresh(P, B, b, b, 512);
        run_dgrad(rt, adj_res_[i][0], d0n, gn, &gx);
        gx = gn;
    }
    // bottleneck entry: conv over cat(feature, tiled pose)
    View db = nbwd(tape.bott0, bott0_n_, ACT_RELU, gx);
    View dbin = fresh(P, B, b, b, 512 + pose_pad_);
    run_dgrad(rt, adj_bott0_, db, dbin);
    if (want_pose) {
        pose_sum_kernel<<<B, round_up(pose_ch_, 32), 0, s>>>(dbin.p, dbin.ld, (long)b * b, 512, pose_ch_, g.d_pose, g.d_pose_ld);
        THA4_LAUNCH_CHECK();
    }
    if (!want_img) return;
    // encoder
    d = nbwd(tape.down[3], down_n_[3], ACT_RELU, dbin.slice(0, 512));
    for (int i = 3; i >= 1; --i) {
        View da = fresh(P, B, S >> (i - 1), S >> (i - 1), adj_down_[i].cout);
        run_dgrad(rt, adj_down_[i], d, da);
        d = nbwd(tape.down[i - 1], down_n_[i - 1], ACT_RELU, da);
    }
    View dx0 = fresh(P, B, S, S, in_ch_);
    run_dgrad(rt, adj_down_[0], d, dx0, &dimg);
    if (kind_ == TAIL_COMBINER) {
        if (g.d_image1) nhwc_to_nchw(dx0.slice(0, 4), g.d_image1, s);
        if (g.d_image0) nhwc_to_nchw(dx0.slice(4, 4), g.d_image0, s);
    } else {
        nhwc_to_nchw(dx0, g.d_image0, s);
    }
}

}  // namespace tha4
