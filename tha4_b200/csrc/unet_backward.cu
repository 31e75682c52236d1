// Input gradients of the U-Nets -- the body morpher (Morpher00; morpher_00.py:42-66 on unet.py:531-546): d(image) and d(pose),
// and the upscaler (Upscaler02; upscaler_02.py:59-96 on unet.py:645-658): d(rest image), d(coarse posed image), d(coarse grid
// change) and d(pose) -- for upstream gradients of their five outputs.
//
// The forward is recomputed with the inference kernels of the context's precision mode, keeping a tape (UNetTape): every
// ResBlock's input and raw conv0 output, every attention block's input and qkv, the pose MLP pre-activations and the FiLM
// table, all with the statistics their producers accumulated.  The backward then runs the network in reverse:
//   tail:      outputs' gradients -> d(body output) (direct, grid through grid_sample, alpha logit through the sigmoid of the
//              returned alpha) + the warp's image term; then the last.2 head adjoint (one 3x3 conv);
//   GroupNorm (+FiLM) (+SiLU): one reduction of sum dz, sum dz xhat per (n,c) (fp64), folded per group; the same sums give
//              d(scale1) / d(shift1) of the pose FiLM, written into d(film1) at the block's offset (no atomics on it);
//   convs:     data gradients on the conv kernels with adjoint-packed weights made from the packed forward weights on the
//              first call (3x3 -> 3x3 W^T flipped, 1x1 -> 1x1 W^T, nearest x2 + 3x3 -> 4x4 stride-2 conv W^T);
//   resampling: AvgPool2d(2) -> 1/4 nearest-up read inside the norm backward; nearest x2 residual -> 2x2 sum;
//   attention: P recomputed from the taped qkv, fp32, dK / dV owned by one thread per key (no atomics);
//   skips:     the d(cat) half of a skip tensor is added in the epilogue of its down-path consumer's last adjoint;
//   pose:      d(film1) through the FiLM projection, cond_embed.2 and cond_embed.0 (fixed-order fp64 GEMVs);
//   upscaler:  the fused 16-channel first conv's data gradient goes through the prologue's adjoint (image_ops.cu): identity
//              and warp terms to the rest image (which the tail warps too), the posed / grid terms through the bilinear x2.
#include "nets.cuh"

namespace tha4 {

namespace {

int grid_for(long n) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, 132L * 16)); }

View fresh(Pool* P, int N, int H, int W, int C) {
    View v; v.N = N; v.H = H; v.W = W; v.C = C; v.ld = C;
    v.p = P->alloc((size_t)N * H * W * C);
    return v;
}

// ------------------------------------------------------------------------------------------------ adjoint packing
struct TapMap { int src[CONV_MAX_TAPS]; };    // adjoint tap -> forward (phase * ntaps + tap)

// dst[t][co][ci] (adjoint, packed) = src[map[t]][ci][co] (forward, packed): co = forward input channel, ci = forward output
__global__ void adjoint_from_packed_kernel(float* __restrict__ dst, const float* __restrict__ src, TapMap m, int ntaps, int co_n,
                                           int ci_n, int dst_cout_pad, int dst_cin_pad, int src_cout_pad, int src_cin_pad) {
    const long total = (long)ntaps * co_n * ci_n;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % ci_n);
        const long r = i / ci_n;
        const int co = (int)(r % co_n), t = (int)(r / co_n);
        dst[((long)t * dst_cout_pad + co) * dst_cin_pad + ci] = src[((long)m.src[t] * src_cout_pad + ci) * src_cin_pad + co];
    }
}

// ------------------------------------------------------------------------------------------------ GroupNorm backward
constexpr int GN_MAX_C = 512;
constexpr int GN_PIX_PER_THREAD = 32;

struct GnBwdArgs {
    const float* x; int x_ld, x_f16;                  // RAW input of the normalisation (NHWC, fp32 or f16), at dx's resolution
    const double* stats; int stats_ld, stats_rep; long stats_rep_stride;
    const float* gamma; const float* beta;
    const float* film0;                               // [2C] shared by all samples, or null
    const float* film1; int film1_ld;                 // [N][film1_ld] (this layer's 2C vector), or null
    int act;                                          // ACT_SILU or ACT_NONE
    const float* dy; int dy_ld, dy_pool;              // gradient of the layer output; dy_pool: the output was 2x2-mean-pooled
    const float* res; int res_ld, res_mode;           // + residual gradient: RES_SAME, RES_UP2 (2x2 sum), RES_DOWN2 (1/4 nearest-up)
    const float* add; int add_ld;                     // + same-resolution term
    float* dx; int dx_ld;
    float* dfilm; int dfilm_ld;                       // d(film1): d(scale) at [c], d(shift) at [C + c] of row n
    double* sums;                                     // [N][C][2] zeroed: sum dz, sum dz xhat
    float* coef;                                      // [N][C][8]: A B mean rstd K r1 r2
    int C, H, W, groups;
};

__device__ __forceinline__ float silu_grad(float h) {
    const float sg = 1.0f / (1.0f + expf(-h));
    return sg * (1.0f + h * (1.0f - sg));
}

// per-channel (A, B, mean, rstd) of sample n into sm_ab: the forward's affine y = A x + B (norm.cu, norm_apply_kernel<true>),
// the replicas folded per channel, then the channels of a group summed in order
__device__ void gn_affine_smem(const GnBwdArgs& a, int n, double2* sm_ch, float2* sm_grp, float4* sm_ab) {
    const int C = a.C, ng = a.groups, cpg = C / ng;
    for (int c = threadIdx.x; c < C; c += blockDim.x)
        sm_ch[c] = fold_stat_replicas(a.stats + ((long)n * a.stats_ld + c) * 2, a.stats_rep_stride, a.stats_rep);
    __syncthreads();
    for (int g = threadIdx.x; g < ng; g += blockDim.x) {
        double su = 0.0, sq = 0.0;
        for (int j = 0; j < cpg; ++j) { const double2 v = sm_ch[g * cpg + j]; su += v.x; sq += v.y; }
        const double cnt = (double)a.H * a.W * cpg;
        const double mean = su / cnt;
        double var = sq / cnt - mean * mean;
        if (var < 0.0) var = 0.0;
        sm_grp[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + 1e-5)));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float2 mr = sm_grp[c / cpg];
        float A = mr.y * a.gamma[c];
        float B = a.beta[c] - mr.x * A;
        if (a.film0) { const float sc = 1.0f + a.film0[c], sh = a.film0[C + c]; A *= sc; B = B * sc + sh; }
        if (a.film1) { const float* f = a.film1 + (long)n * a.film1_ld; const float sc = 1.0f + f[c], sh = f[C + c]; A *= sc; B = B * sc + sh; }
        sm_ab[c] = make_float4(A, B, mr.x, mr.y);
    }
    __syncthreads();
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

// the upstream gradient at pixel `pix` of sample n (x's resolution); a pooled output spreads 1/4 of its gradient on each source
__device__ __forceinline__ float4 gn_dy(const GnBwdArgs& a, int n, long pix, int q) {
    if (!a.dy_pool) return *reinterpret_cast<const float4*>(a.dy + ((long)n * a.H * a.W + pix) * a.dy_ld + 4 * q);
    const int y = (int)(pix / a.W), x = (int)(pix - (long)y * a.W);
    const long p = ((long)n * (a.H / 2) + y / 2) * (a.W / 2) + x / 2;
    const float4 v = *reinterpret_cast<const float4*>(a.dy + p * a.dy_ld + 4 * q);
    return make_float4(0.25f * v.x, 0.25f * v.y, 0.25f * v.z, 0.25f * v.w);
}

// stage 1: per-(n,c) sums of dz and dz * xhat, dz = dy * act'(A x + B) (fp32 per thread, fp64 across threads and CTAs)
template <bool F16>
__global__ void __launch_bounds__(256) gn_bwd_reduce_kernel(const GnBwdArgs a) {
    __shared__ double2 sm_ch[GN_MAX_C];
    __shared__ float2 sm_grp[GN_MAX_C];
    __shared__ float4 sm_ab[GN_MAX_C];
    __shared__ float red[256][9];
    const int n = blockIdx.y;
    gn_affine_smem(a, n, sm_ch, sm_grp, sm_ab);
    const int cq = a.C >> 2, PL = 256 / cq;
    const int tid = threadIdx.x, pl = tid / cq, q = tid - pl * cq;
    const bool active = pl < PL;
    const long HW = (long)a.H * a.W;
    float s[4] = {0, 0, 0, 0}, sx[4] = {0, 0, 0, 0};
    if (active) {
        float4 ab[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) ab[k] = sm_ab[4 * q + k];
        const long base = (long)blockIdx.x * PL * GN_PIX_PER_THREAD;
        for (int i = 0; i < GN_PIX_PER_THREAD; ++i) {
            const long pix = base + (long)i * PL + pl;
            if (pix >= HW) break;
            const float4 xv = load4<F16>(a.x, ((long)n * HW + pix) * a.x_ld + 4 * q);
            const float4 gv = gn_dy(a, n, pix, q);
            const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float dz = a.act == ACT_SILU ? gs[k] * silu_grad(xs[k] * ab[k].x + ab[k].y) : gs[k];
                s[k] += dz;
                sx[k] += dz * ((xs[k] - ab[k].z) * ab[k].w);
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

// stage 2 (one CTA per sample): fold the sums per group into the apply coefficients, and d(film1) from the same sums:
//   dx = K dz - r1 - xhat r2,  K = rstd gamma M,  r1 = rstd mean_g(gamma M dz),  r2 = rstd mean_g(gamma M dz xhat),
//   M = (1 + s0)(1 + s1);  d s1 = sum dz h2 = (gamma S2 + beta S1)(1 + s0) + b0 S1,  d b1 = S1
__global__ void __launch_bounds__(256) gn_bwd_finalize_kernel(const GnBwdArgs a) {
    __shared__ double2 sm_ch[GN_MAX_C];
    __shared__ float2 sm_grp[GN_MAX_C];
    __shared__ float4 sm_ab[GN_MAX_C];
    const int n = blockIdx.x, C = a.C, cpg = C / a.groups;
    gn_affine_smem(a, n, sm_ch, sm_grp, sm_ab);
    double2* sm_t = sm_ch;                              // reused: per channel (gamma M S1, gamma M S2)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const double S1 = a.sums[((long)n * C + c) * 2], S2 = a.sums[((long)n * C + c) * 2 + 1];
        const float s0 = a.film0 ? 1.0f + a.film0[c] : 1.0f;
        const float s1 = a.film1 ? 1.0f + a.film1[(long)n * a.film1_ld + c] : 1.0f;
        const double gm = (double)a.gamma[c] * s0 * s1;
        sm_t[c] = make_double2(gm * S1, gm * S2);
        if (a.dfilm) {
            double ds = (double)a.gamma[c] * S2 + (double)a.beta[c] * S1;
            if (a.film0) ds = ds * s0 + (double)a.film0[C + c] * S1;
            a.dfilm[(long)n * a.dfilm_ld + c] = (float)ds;
            a.dfilm[(long)n * a.dfilm_ld + C + c] = (float)S1;
        }
    }
    __syncthreads();
    const double cnt = (double)a.H * a.W * cpg;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g0 = (c / cpg) * cpg;
        double m1 = 0.0, m2 = 0.0;
        for (int j = 0; j < cpg; ++j) { m1 += sm_t[g0 + j].x; m2 += sm_t[g0 + j].y; }
        const float4 ab = sm_ab[c];
        const float s0 = a.film0 ? 1.0f + a.film0[c] : 1.0f;
        const float s1 = a.film1 ? 1.0f + a.film1[(long)n * a.film1_ld + c] : 1.0f;
        float* cf = a.coef + ((long)n * C + c) * 8;
        cf[0] = ab.x; cf[1] = ab.y; cf[2] = ab.z; cf[3] = ab.w;
        cf[4] = ab.w * a.gamma[c] * s0 * s1;
        cf[5] = (float)(ab.w * (m1 / cnt));
        cf[6] = (float)(ab.w * (m2 / cnt));
        cf[7] = 0.0f;
    }
}

// stage 3: dx = K dz - r1 - xhat r2 (+ the residual term, + add), one float4 of channels per thread and step
template <bool F16>
__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const GnBwdArgs a, long total) {
    const int cq = a.C >> 2;
    const long HW = (long)a.H * a.W;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long p = i / cq;
        const int q = (int)(i - p * cq);
        const int n = (int)(p / HW);
        const long pix = p - (long)n * HW;
        const float4 xv = load4<F16>(a.x, p * a.x_ld + 4 * q);
        const float4 gv = gn_dy(a, n, pix, q);
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4* cf = reinterpret_cast<const float4*>(a.coef + ((long)n * a.C + 4 * q + k) * 8);
            const float4 c0 = cf[0], c1 = cf[1];
            const float dz = a.act == ACT_SILU ? gs[k] * silu_grad(xs[k] * c0.x + c0.y) : gs[k];
            const float xhat = (xs[k] - c0.z) * c0.w;
            o[k] = c1.x * dz - c1.y - xhat * c1.z;
        }
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a.res_mode == RES_SAME) {
            r = *reinterpret_cast<const float4*>(a.res + p * a.res_ld + 4 * q);
        } else if (a.res_mode == RES_UP2) {            // the forward added up2(x) to a 2H x 2W output
            const int y = (int)(pix / a.W), x = (int)(pix - (long)y * a.W);
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const float4 v = *reinterpret_cast<const float4*>(a.res + (((long)n * 2 * a.H + 2 * y + dy) * 2 * a.W + 2 * x + dx) * a.res_ld + 4 * q);
                    r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
                }
        } else if (a.res_mode == RES_DOWN2) {          // the forward added AvgPool2d(2)(x) to an H/2 x W/2 output
            const int y = (int)(pix / a.W), x = (int)(pix - (long)y * a.W);
            const float4 v = *reinterpret_cast<const float4*>(a.res + (((long)n * (a.H / 2) + y / 2) * (a.W / 2) + x / 2) * a.res_ld + 4 * q);
            r = make_float4(0.25f * v.x, 0.25f * v.y, 0.25f * v.z, 0.25f * v.w);
        }
        if (a.add) {
            const float4 v = *reinterpret_cast<const float4*>(a.add + p * a.add_ld + 4 * q);
            r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
        }
        *reinterpret_cast<float4*>(a.dx + p * a.dx_ld + 4 * q) = make_float4(o[0] + r.x, o[1] + r.y, o[2] + r.z, o[3] + r.w);
    }
}

// ------------------------------------------------------------------------------------------------ attention backward
constexpr int AB_L = 256, AB_D = 32, AB_Q = 64;      // tokens, head dim, rows (queries or keys) per CTA: one thread each

__device__ __forceinline__ float dot32(const float* a, const float* b) {
    float d = 0.0f;
#pragma unroll
    for (int c = 0; c < AB_D; ++c) d = fmaf(a[c], b[c], d);
    return d;
}

// per query i: m_i, 1/l_i (softmax of S = (s q)(s k)^T, s = D^-1/4), D_i = sum_j P_ij dP_ij (dP = dO V^T) and
// dQ_i = s sum_j dS_ij (s k_j), dS = P (dP - D).  K (scaled) and V of the head in shared memory.
__global__ void __launch_bounds__(AB_Q) attn_bwd_q_kernel(const float* __restrict__ qkv, int qkv_ld, const float* __restrict__ dout,
                                                          int dout_ld, int C, int heads, float* __restrict__ dqkv, int dqkv_ld,
                                                          float4* __restrict__ rowstat) {
    extern __shared__ __align__(16) float sm[];
    float* Ks = sm;
    float* Vs = sm + AB_L * AB_D;
    const int qb = blockIdx.x % (AB_L / AB_Q), nh = blockIdx.x / (AB_L / AB_Q);
    const int n = nh / heads, h = nh % heads, tid = threadIdx.x;
    const float scale = 1.0f / sqrtf(sqrtf((float)AB_D));
    const float* base = qkv + (long)n * AB_L * qkv_ld;
    for (int r = tid; r < AB_L; r += AB_Q)
#pragma unroll
        for (int c = 0; c < AB_D; c += 4) {
            const float4 k = *reinterpret_cast<const float4*>(base + (long)r * qkv_ld + C + h * AB_D + c);
            *reinterpret_cast<float4*>(Ks + r * AB_D + c) = make_float4(k.x * scale, k.y * scale, k.z * scale, k.w * scale);
            *reinterpret_cast<float4*>(Vs + r * AB_D + c) = *reinterpret_cast<const float4*>(base + (long)r * qkv_ld + 2 * C + h * AB_D + c);
        }
    const int i = qb * AB_Q + tid;
    float q[AB_D], go[AB_D];
#pragma unroll
    for (int c = 0; c < AB_D; ++c) {
        q[c] = base[(long)i * qkv_ld + h * AB_D + c] * scale;
        go[c] = dout[((long)n * AB_L + i) * dout_ld + h * AB_D + c];
    }
    __syncthreads();
    float m = -INFINITY, l = 0.0f;
    for (int j = 0; j < AB_L; ++j) {
        const float sc = dot32(q, Ks + j * AB_D);
        const float mn = fmaxf(m, sc);
        l = l * expf(m - mn) + expf(sc - mn);
        m = mn;
    }
    const float il = 1.0f / l;
    float Di = 0.0f;
    for (int j = 0; j < AB_L; ++j) {
        const float p = expf(dot32(q, Ks + j * AB_D) - m) * il;
        Di = fmaf(p, dot32(go, Vs + j * AB_D), Di);
    }
    float dq[AB_D];
#pragma unroll
    for (int c = 0; c < AB_D; ++c) dq[c] = 0.0f;
    for (int j = 0; j < AB_L; ++j) {
        const float p = expf(dot32(q, Ks + j * AB_D) - m) * il;
        const float ds = p * (dot32(go, Vs + j * AB_D) - Di);
#pragma unroll
        for (int c = 0; c < AB_D; ++c) dq[c] = fmaf(ds, Ks[j * AB_D + c], dq[c]);
    }
    float* dst = dqkv + ((long)n * AB_L + i) * dqkv_ld + h * AB_D;
#pragma unroll
    for (int c = 0; c < AB_D; ++c) dst[c] = dq[c] * scale;
    rowstat[(long)nh * AB_L + i] = make_float4(m, il, Di, 0.0f);
}

// per key j: dV_j = sum_i P_ij dO_i, dK_j = s sum_i dS_ij (s q_i), with P and dS recomputed exactly as attn_bwd_q_kernel did
__global__ void __launch_bounds__(AB_Q) attn_bwd_kv_kernel(const float* __restrict__ qkv, int qkv_ld, const float* __restrict__ dout,
                                                           int dout_ld, int C, int heads, float* __restrict__ dqkv, int dqkv_ld,
                                                           const float4* __restrict__ rowstat) {
    extern __shared__ __align__(16) float sm[];
    float* Qs = sm;
    float* Gs = sm + AB_L * AB_D;
    float4* Rs = reinterpret_cast<float4*>(sm + 2 * AB_L * AB_D);
    const int kb = blockIdx.x % (AB_L / AB_Q), nh = blockIdx.x / (AB_L / AB_Q);
    const int n = nh / heads, h = nh % heads, tid = threadIdx.x;
    const float scale = 1.0f / sqrtf(sqrtf((float)AB_D));
    const float* base = qkv + (long)n * AB_L * qkv_ld;
    for (int r = tid; r < AB_L; r += AB_Q) {
#pragma unroll
        for (int c = 0; c < AB_D; c += 4) {
            const float4 v = *reinterpret_cast<const float4*>(base + (long)r * qkv_ld + h * AB_D + c);
            *reinterpret_cast<float4*>(Qs + r * AB_D + c) = make_float4(v.x * scale, v.y * scale, v.z * scale, v.w * scale);
            *reinterpret_cast<float4*>(Gs + r * AB_D + c) = *reinterpret_cast<const float4*>(dout + ((long)n * AB_L + r) * dout_ld + h * AB_D + c);
        }
        Rs[r] = rowstat[(long)nh * AB_L + r];
    }
    const int j = kb * AB_Q + tid;
    float k[AB_D], v[AB_D], dk[AB_D], dv[AB_D];
#pragma unroll
    for (int c = 0; c < AB_D; ++c) {
        k[c] = base[(long)j * qkv_ld + C + h * AB_D + c] * scale;
        v[c] = base[(long)j * qkv_ld + 2 * C + h * AB_D + c];
        dk[c] = dv[c] = 0.0f;
    }
    __syncthreads();
    for (int i = 0; i < AB_L; ++i) {
        const float4 rs = Rs[i];
        const float p = expf(dot32(Qs + i * AB_D, k) - rs.x) * rs.y;
        const float ds = p * (dot32(Gs + i * AB_D, v) - rs.z);
#pragma unroll
        for (int c = 0; c < AB_D; ++c) {
            dv[c] = fmaf(p, Gs[i * AB_D + c], dv[c]);
            dk[c] = fmaf(ds, Qs[i * AB_D + c], dk[c]);
        }
    }
    float* dst = dqkv + ((long)n * AB_L + j) * dqkv_ld + h * AB_D;
#pragma unroll
    for (int c = 0; c < AB_D; ++c) { dst[C + c] = dk[c] * scale; dst[2 * C + c] = dv[c]; }
}

// ------------------------------------------------------------------------------------------------ dense layers
// dx[n][k] = act'(pre[n][k]) * sum_r dy[n][r] W[r][k]; 32 outputs x 8 row slices per CTA, slices summed in order (fp64)
__global__ void __launch_bounds__(256) linear_bwd_kernel(const float* __restrict__ dy, int dy_ld, int R, const float* __restrict__ W, int K,
                                                         const float* __restrict__ pre, int pre_ld, float* __restrict__ dx, int dx_ld) {
    __shared__ double red[8][32];
    const int lane = threadIdx.x & 31, sl = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + lane, n = blockIdx.y;
    double acc = 0.0;
    if (k < K)
        for (int r = sl; r < R; r += 8) acc += (double)dy[(long)n * dy_ld + r] * (double)W[(long)r * K + k];
    red[sl][lane] = acc;
    __syncthreads();
    if (sl == 0 && k < K) {
        double t = 0.0;
        for (int j = 0; j < 8; ++j) t += red[j][lane];
        float v = (float)t;
        if (pre) v *= silu_grad(pre[(long)n * pre_ld + k]);
        dx[(long)n * dx_ld + k] = v;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ entry points
void conv_adjoint_from_packed(ConvWeights& cw, const ConvWeights& fwd, ConvKind kind, cudaStream_t s) {
    THA4_REQUIRE(kind == CONV_3x3 || kind == CONV_1x1 || kind == CONV_UP2_3x3, "conv adjoint (packed): kind");
    THA4_REQUIRE(fwd.cout % 4 == 0 && fwd.w != nullptr, "conv adjoint (packed): forward weights");
    conv_describe(cw, kind == CONV_UP2_3x3 ? CONV_4x4_S2 : kind, fwd.cout, fwd.cin);
    TapMap m;
    for (int t = 0; t < cw.ntaps; ++t) {
        // adjoint tap t reads dy at (stride * o + dy, stride * o + dx); the forward tap that wrote there:
        //   3x3 / 1x1: offset (-dy, -dx);  nearest x2 + 3x3: output phase (py, px) = (dy, dx) mod 2, source offset ((py - dy) / 2, ...)
        const int dy = cw.dy[0][t], dx = cw.dx[0][t];
        const int py = kind == CONV_UP2_3x3 ? (dy & 1) : 0, px = kind == CONV_UP2_3x3 ? (dx & 1) : 0;
        const int fy = kind == CONV_UP2_3x3 ? (py - dy) / 2 : -dy, fx = kind == CONV_UP2_3x3 ? (px - dx) / 2 : -dx;
        const int ph = kind == CONV_UP2_3x3 ? 2 * py + px : 0;
        m.src[t] = -1;
        for (int t2 = 0; t2 < fwd.ntaps; ++t2)
            if (fwd.dy[ph][t2] == fy && fwd.dx[ph][t2] == fx && (kind != CONV_UP2_3x3 || (fwd.ph_oy[ph] == py && fwd.ph_ox[ph] == px)))
                m.src[t] = ph * fwd.ntaps + t2;
        THA4_REQUIRE(m.src[t] >= 0, "conv adjoint (packed): no forward tap for an adjoint tap");
    }
    cw.w = reinterpret_cast<float*>(tracked_malloc(conv_packed_floats(cw) * sizeof(float)));
    THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
    cw.tf32_rounded = fwd.tf32_rounded;
    const long total = (long)cw.ntaps * cw.cout * cw.cin;
    adjoint_from_packed_kernel<<<grid_for(total), 256, 0, s>>>(cw.w, fwd.w, m, cw.ntaps, cw.cout, cw.cin, cw.cout_pad, cw.cin_pad,
                                                              fwd.cout_pad, fwd.cin_pad);
    THA4_LAUNCH_CHECK();
}

void group_norm_backward(const View& x, int groups, const float* gamma, const float* beta, const float* film0, const float* film1,
                         int film1_ld, int act, const View& dy, int dy_pool, const View& dx, float* dfilm, int dfilm_ld,
                         const View* res, int res_mode, const View* add, double* sums, float* coef, cudaStream_t s) {
    THA4_REQUIRE(x.stats != nullptr && x.C % 4 == 0 && x.C <= GN_MAX_C && groups > 0 && x.C % groups == 0, "group norm backward: channels");
    THA4_REQUIRE(dy.C == x.C && dx.C == x.C && !dy.f16 && !dx.f16 && dy.ld % 4 == 0 && dx.ld % 4 == 0 && x.ld % 4 == 0,
                 "group norm backward: layouts");
    THA4_REQUIRE(dy_pool ? (dy.H * 2 == x.H && dy.W * 2 == x.W) : (dy.H == x.H && dy.W == x.W), "group norm backward: dy dims");
    THA4_REQUIRE(dx.H == x.H && dx.W == x.W && dx.N == x.N && dy.N == x.N, "group norm backward: dx dims");
    THA4_REQUIRE(act == ACT_SILU || act == ACT_NONE, "group norm backward: activation");
    THA4_REQUIRE(!dfilm || film1, "group norm backward: d(film) needs the FiLM vector");
    if (res && res_mode != RES_NONE) {
        THA4_REQUIRE(res->C == x.C && !res->f16 && res->ld % 4 == 0, "group norm backward: residual layout");
        if (res_mode == RES_SAME) THA4_REQUIRE(res->H == x.H && res->W == x.W, "group norm backward: residual dims");
        else if (res_mode == RES_UP2) THA4_REQUIRE(res->H == 2 * x.H && res->W == 2 * x.W, "group norm backward: residual dims");
        else THA4_REQUIRE(res_mode == RES_DOWN2 && res->H * 2 == x.H && res->W * 2 == x.W, "group norm backward: residual dims");
    }
    if (add) THA4_REQUIRE(add->C == x.C && add->H == x.H && add->W == x.W && !add->f16 && add->ld % 4 == 0, "group norm backward: added term");
    GnBwdArgs a;
    a.x = x.p; a.x_ld = x.ld; a.x_f16 = x.f16;
    a.stats = x.stats; a.stats_ld = x.stats_ld; a.stats_rep = x.stats_rep; a.stats_rep_stride = x.stats_rep_stride;
    a.gamma = gamma; a.beta = beta; a.film0 = film0; a.film1 = film1; a.film1_ld = film1_ld; a.act = act;
    a.dy = dy.p; a.dy_ld = dy.ld; a.dy_pool = dy_pool;
    a.res = res && res_mode != RES_NONE ? res->p : nullptr; a.res_ld = res ? res->ld : 0; a.res_mode = res ? res_mode : RES_NONE;
    a.add = add ? add->p : nullptr; a.add_ld = add ? add->ld : 0;
    a.dx = dx.p; a.dx_ld = dx.ld; a.dfilm = dfilm; a.dfilm_ld = dfilm_ld; a.sums = sums; a.coef = coef;
    a.C = x.C; a.H = x.H; a.W = x.W; a.groups = groups;
    const int PL = 256 / (x.C / 4);
    const dim3 g1(ceil_div(x.H * x.W, PL * GN_PIX_PER_THREAD), x.N);
    const long total = (long)x.N * x.H * x.W * (x.C / 4);
    if (x.f16) gn_bwd_reduce_kernel<true><<<g1, 256, 0, s>>>(a);
    else gn_bwd_reduce_kernel<false><<<g1, 256, 0, s>>>(a);
    THA4_LAUNCH_CHECK();
    gn_bwd_finalize_kernel<<<x.N, 256, 0, s>>>(a);
    THA4_LAUNCH_CHECK();
    if (x.f16) gn_bwd_apply_kernel<true><<<grid_for(total), 256, 0, s>>>(a, total);
    else gn_bwd_apply_kernel<false><<<grid_for(total), 256, 0, s>>>(a, total);
    THA4_LAUNCH_CHECK();
}

void attention_backward(const View& qkv, const View& dout, int heads, const View& dqkv, float* rowstat, cudaStream_t s) {
    THA4_REQUIRE(qkv.H * qkv.W == AB_L && dout.C * 3 == qkv.C && dout.C / heads == AB_D && dqkv.C == qkv.C, "attention backward: shape (L=256, head dim 32)");
    THA4_REQUIRE(!qkv.f16 && !dout.f16 && !dqkv.f16 && qkv.ld % 4 == 0 && dout.ld % 4 == 0 && dqkv.N == qkv.N && dout.N == qkv.N,
                 "attention backward: layouts");
    const int C = dout.C, ctas = qkv.N * heads * (AB_L / AB_Q);
    const size_t smem_q = 2 * AB_L * AB_D * sizeof(float), smem_kv = smem_q + AB_L * sizeof(float4);
    THA4_ENSURE_SMEM(attn_bwd_q_kernel, smem_q);
    THA4_ENSURE_SMEM(attn_bwd_kv_kernel, smem_kv);
    float4* rs = reinterpret_cast<float4*>(rowstat);
    attn_bwd_q_kernel<<<ctas, AB_Q, smem_q, s>>>(qkv.p, qkv.ld, dout.p, dout.ld, C, heads, dqkv.p, dqkv.ld, rs);
    THA4_LAUNCH_CHECK();
    attn_bwd_kv_kernel<<<ctas, AB_Q, smem_kv, s>>>(qkv.p, qkv.ld, dout.p, dout.ld, C, heads, dqkv.p, dqkv.ld, rs);
    THA4_LAUNCH_CHECK();
}

void linear_backward(const float* dy, int dy_ld, int N, int R, const float* W, int K, const float* pre, int pre_ld, float* dx, int dx_ld,
                     cudaStream_t s) {
    linear_bwd_kernel<<<dim3(ceil_div(K, 32), N), 256, 0, s>>>(dy, dy_ld, R, W, K, pre, pre_ld, dx, dx_ld);
    THA4_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------------ UNetNet
void UNetNet::pack_adjoints(Runtime& rt) {
    SinkScope own(&owned_);
    cudaStream_t s = rt.stream;
    auto res = [&](const ResBlockW& w, bool up) {
        ResAdj& a = adj_res_[&w];
        conv_adjoint_from_packed(a.conv0, w.conv0, up ? CONV_UP2_3x3 : CONV_3x3, s);
        conv_adjoint_from_packed(a.conv1, w.conv1, CONV_3x3, s);
        if (w.has_skip) conv_adjoint_from_packed(a.skip, w.skip, CONV_1x1, s);
    };
    auto attn = [&](const AttnW& w) {
        AttnAdj& a = adj_attn_[&w];
        conv_adjoint_from_packed(a.qkv, w.qkv, CONV_1x1, s);
        conv_adjoint_from_packed(a.proj, w.proj, CONV_1x1, s);
    };
    for (const auto& w : down_res_) res(w, false);
    for (const auto& w : down_ds_) res(w, false);
    for (const auto& w : mid_res_) res(w, false);
    for (const auto& w : up_res_) res(w, false);
    for (const auto& w : up_us_) res(w, true);
    attn(down_attn_);
    for (const auto& w : mid_attn_) attn(w);
    for (const auto& w : up_attn_) attn(w);
    conv_adjoint_from_packed(adj_first_, first_, CONV_3x3, s);
    head_pack_adjoint(adj_head_, tail_, first_.tf32_rounded, s);      // rounded as the network's own weights were
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    adj_ready_ = true;
}

void UNetNet::backward(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                       const float* pose, int pose_ld, const UNetGrads& g) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    THA4_REQUIRE(upscaler_ || (!g.d_coarse_posed && !g.d_coarse_grid), "unet backward: only the upscaler has coarse inputs");
    const bool want_img = g.d_image != nullptr, want_pose = g.d_pose != nullptr;
    const bool want_coarse = g.d_coarse_posed || g.d_coarse_grid;
    const bool want_x0 = want_img || want_coarse;          // gradients that need the first conv's data gradient
    THA4_REQUIRE(want_x0 || want_pose, "unet backward: no gradient requested");
    if (!adj_ready_) pack_adjoints(rt);
    const int B = image.N, S = S_, NH = 2 * L_;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;

    // forward with a tape; its outputs are what the tail backward differentiates through
    static const int kCh[5] = {4, 1, 4, 2, 4};
    float* outs[5];
    for (int k = 0; k < 5; ++k) outs[k] = P->alloc((size_t)B * kCh[k] * S * S);
    UNetTape tape;
    forward(rt, image, coarse_posed, coarse_grid, coarse_size, pose, pose_ld, outs, &tape);
    float* dfilm = P->alloc((size_t)B * film1_total_);

    auto gn = [&](const View& x, const NormW& nw, const float* film0, const float* film1, int act, const View& dy, int dy_pool,
                  const View& dx, const View* res, int res_mode, const View* add) {
        THA4_REQUIRE(nw.C == x.C, "norm backward: channel mismatch");
        group_norm_backward(x, 32, nw.gamma, nw.beta, film0, film1, film1_total_, act, dy, dy_pool, dx,
                            film1 ? dfilm + (film1 - tape.film1) : nullptr, film1_total_, res, res_mode, add,
                            rt.alloc_stats((size_t)B * x.C * 2), rt.scratch->alloc((size_t)B * x.C * 8), s);
    };
    // ResBlock: out = conv1(SiLU(FiLM(GN(h0)))) + skip(resample(x)),  h0 = conv0(resample(SiLU(GN(x)))).  Returns the gradient of x
    // (+ extra); with input_grad false it stops once the block's d(film1) is written.
    auto res_bwd = [&](const ResBlockW& w, int mode, const View& dout, const View* extra, bool input_grad) -> View {
        const UNetTape::Res& t = tape.res.at(&w);
        const ResAdj& A = adj_res_.at(&w);
        View du = fresh(P, B, dout.H, dout.W, w.cout);
        run_dgrad(rt, A.conv1, dout, du);
        View dh0 = fresh(P, B, t.h0.H, t.h0.W, w.cout);
        gn(t.h0, w.norm1, w.film0, tape.film1 + w.film1_off, ACT_SILU, du, 0, dh0, nullptr, RES_NONE, nullptr);
        if (!input_grad) return View{};
        const int th = mode == 2 ? t.x.H / 2 : t.x.H;
        View dt = fresh(P, B, th, th, w.cin);
        run_dgrad(rt, A.conv0, dh0, dt);
        View dx = fresh(P, B, t.x.H, t.x.W, w.cin);
        if (w.has_skip) {
            View dsk = fresh(P, B, t.x.H, t.x.W, w.cin);
            run_dgrad(rt, A.skip, dout, dsk, extra);
            gn(t.x, w.norm0, nullptr, nullptr, ACT_SILU, dt, 0, dx, &dsk, RES_SAME, nullptr);
        } else {
            gn(t.x, w.norm0, nullptr, nullptr, ACT_SILU, dt, mode == 2, dx, &dout, mode == 0 ? RES_SAME : (mode == 1 ? RES_UP2 : RES_DOWN2), extra);
        }
        return dx;
    };
    // AttentionBlock: out = x + proj(attention(qkv(GN(x))))
    auto attn_bwd = [&](const AttnW& w, const View& dout) -> View {
        const UNetTape::Attn& t = tape.attn.at(&w);
        const AttnAdj& A = adj_attn_.at(&w);
        View da = fresh(P, B, dout.H, dout.W, w.C);
        run_dgrad(rt, A.proj, dout, da);
        View dqkv = fresh(P, B, dout.H, dout.W, 3 * w.C);
        attention_backward(t.qkv, da, 8, dqkv, rt.scratch->alloc((size_t)B * 8 * 256 * 4), s);
        View dn = fresh(P, B, dout.H, dout.W, w.C);
        run_dgrad(rt, A.qkv, dqkv, dn);
        View dx = fresh(P, B, dout.H, dout.W, w.C);
        gn(t.x, w.norm, nullptr, nullptr, ACT_NONE, dn, 0, dx, &dout, RES_SAME, nullptr);
        return dx;
    };

    // ---- tail: d(body output) + the warp's image term; last.2 head; last.0 GroupNorm + SiLU ----
    View dh = fresh(P, B, S, S, 16);
    View dimg;
    if (want_img) {
        dimg = fresh(P, B, S, S, 4);
        THA4_CUDA_CHECK(cudaMemsetAsync(dimg.p, 0, dimg.pixels() * 4 * sizeof(float), s));
    }
    tail_backward(TAIL_UNET, outs, g.grad_outputs, image, ImgView{}, dh, want_img ? dimg.p : nullptr, nullptr, 4, s);
    View df = fresh(P, B, S, S, mc_);
    run_dgrad(rt, adj_head_, dh, df);
    View dfeat = fresh(P, B, S, S, mc_);
    gn(tape.feat, last_n_, nullptr, nullptr, ACT_SILU, df, 0, dfeat, nullptr, RES_NONE, nullptr);

    // ---- up path in reverse: dcat[j] = gradient of up ResBlock j's input cat(h_j, hs[NH-1-j]) ----
    std::vector<int> ch_h(NH);
    for (int j = 0; j < NH; ++j) {
        const int lvl = L_ - 1 - j / 2;
        ch_h[j] = (j == 0) ? mc_ * mults_[L_ - 1] : ((j & 1) ? mc_ * mults_[lvl] : mc_ * mults_[lvl + 1]);
    }
    std::vector<View> dcat(NH);
    for (int j = NH - 1; j >= 0; --j) {
        const int lvl = L_ - 1 - j / 2;
        const bool second = (j & 1);
        View d_dst;
        if (!second) d_dst = dcat[j + 1].slice(0, ch_h[j + 1]);
        else if (lvl > 0) d_dst = res_bwd(up_us_[L_ - 1 - lvl], 1, dcat[j + 1].slice(0, ch_h[j + 1]), nullptr, true);
        else d_dst = dfeat;
        if (lvl == L_ - 1) d_dst = attn_bwd(up_attn_[second ? 1 : 0], d_dst);
        dcat[j] = res_bwd(up_res_[j], 0, d_dst, nullptr, true);
    }
    // the cat half of the gradient of skip tensor hs[k] (joined in its down-path consumer's last adjoint)
    auto dhs = [&](int k) { const View& d = dcat[NH - 1 - k]; return d.slice(ch_h[NH - 1 - k], d.C - ch_h[NH - 1 - k]); };

    // ---- middle in reverse: Res, Attn, Res, Attn, Res, Attn, Res ----
    View dm = dcat[0].slice(0, ch_h[0]);
    for (int j = 3; j >= 0; --j) {
        const View extra = dhs(NH - 1);
        dm = res_bwd(mid_res_[j], 0, dm, j == 0 ? &extra : nullptr, true);
        if (j > 0) dm = attn_bwd(mid_attn_[j - 1], dm);
    }
    // ---- down path in reverse: gk = total gradient of hs[2i+1] ----
    View gk = dm;
    for (int i = L_ - 1; i >= 0; --i) {
        const View d_blk = (i == L_ - 1) ? attn_bwd(down_attn_, gk) : gk;
        const View e_in = dhs(2 * i);
        const View g_in = res_bwd(down_res_[i], 0, d_blk, &e_in, i > 0 || want_x0);
        if (i == 0) { gk = g_in; break; }
        const View e_ds = dhs(2 * i - 1);
        gk = res_bwd(down_ds_[i - 1], 2, g_in, &e_ds, true);
    }
    if (want_x0 && !upscaler_) {     // first conv: its data gradient joins the warp's image term in the epilogue
        View dx0 = fresh(P, B, S, S, 4);
        run_dgrad(rt, adj_first_, gk, dx0, &dimg);
        nhwc_to_nchw(dx0, g.d_image, s);
    } else if (want_x0) {            // the fused 16-channel first conv, then the prologue's adjoint (channels 14, 15 are padding)
        View dx0 = fresh(P, B, S, S, 16);
        run_dgrad(rt, adj_first_, gk, dx0);
        upscaler_prologue_backward(image, coarse_grid, coarse_size, dx0, want_img ? dimg.p : nullptr, g.d_coarse_posed,
                                   g.d_coarse_grid, s);
        if (want_img) nhwc_to_nchw(dimg, g.d_image, s);
    }
    if (want_pose) {    // d(film1) -> FiLM projection (SiLU' at c2) -> cond_embed.2 (SiLU' at c1) -> cond_embed.0
        float* dc2 = P->alloc((size_t)B * 256);
        float* dc1 = P->alloc((size_t)B * 256);
        linear_backward(dfilm, film1_total_, B, film1_total_, film1_w_, 256, tape.c2, 256, dc2, 256, s);
        linear_backward(dc2, 256, B, 256, cond_w2_, 256, tape.c1, 256, dc1, 256, s);
        linear_backward(dc1, 256, B, 256, cond_w0_, 6, nullptr, 0, g.d_pose, g.d_pose_ld, s);
    }
}

}  // namespace tha4
