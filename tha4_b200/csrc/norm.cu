// InstanceNorm2d / GroupNorm32 (+FiLM, +activation, +2x2 mean pool, +residual) on NHWC fp32 activations.
// Statistics are per-(n,c) sum / sum-of-squares in double precision, normally accumulated by the producing conv's
// epilogue (conv_tc.cu); norm_stats is the stand-alone fallback.  norm_apply_fused turns them into the per-(n,c)
// affine inside the apply kernel, so a normalisation layer costs exactly one elementwise pass over the tensor.
#include "ops.cuh"
#include "profiler.cuh"

namespace tha4 {
namespace {

constexpr int STAT_PIX_PER_THREAD = 32;

__global__ void __launch_bounds__(256) norm_stats_kernel(const float* __restrict__ x, int HW, int C, int ld,
                                                         double* __restrict__ sums, int stats_ld, int rep, long rep_stride) {
    __shared__ float red[256][9];
    const int cq = C >> 2;
    const int PL = 256 / cq;
    const int tid = threadIdx.x;
    const int pl = tid / cq, q = tid - pl * cq;
    const int n = blockIdx.y;
    const bool active = pl < PL;
    float s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
    if (active) {
        const long base = (long)blockIdx.x * PL * STAT_PIX_PER_THREAD;
        const float* xp = x + (long)n * HW * ld + 4 * q;
#pragma unroll 4
        for (int i = 0; i < STAT_PIX_PER_THREAD; ++i) {
            long pix = base + (long)i * PL + pl;
            if (pix < HW) {
                float4 v = *reinterpret_cast<const float4*>(xp + pix * ld);
                s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
                ss[0] += v.x * v.x; ss[1] += v.y * v.y; ss[2] += v.z * v.z; ss[3] += v.w * v.w;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { red[tid][k] = s[k]; red[tid][4 + k] = ss[k]; }
    __syncthreads();
    if (active && pl == 0) {
        double acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0;
        for (int j = 0; j < PL; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += (double)red[j * cq + q][k];
        double* dst = sums + (long)(blockIdx.x % rep) * rep_stride + ((long)n * stats_ld + 4 * q) * 2;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            atomicAdd(dst + 2 * k, acc[k]);
            atomicAdd(dst + 2 * k + 1, acc[4 + k]);
        }
    }
}

// per-(n,c) affine from the statistics (shared by the finalize kernel and the fused apply kernel)
__device__ __forceinline__ float2 norm_affine(const double* __restrict__ sums, int stats_ld, int rep, long rep_stride,
                                              int n, int c, int C, int HW, int groups, const float* __restrict__ gamma, const float* __restrict__ beta,
                                              const float* __restrict__ film0, const float* __restrict__ film1, int film1_ld) {
    double su = 0.0, sq = 0.0, cnt;
    const int cpg = groups == 0 ? 1 : C / groups, g0 = (c / cpg) * cpg;
    for (int r = 0; r < rep; ++r) {
        const double* sn = sums + r * rep_stride + (long)n * stats_ld * 2;
        for (int j = 0; j < cpg; ++j) { su += sn[2 * (g0 + j)]; sq += sn[2 * (g0 + j) + 1]; }
    }
    cnt = (double)HW * cpg;
    const double mean = su / cnt;
    double var = sq / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + 1e-5));
    float A = rstd * gamma[c];
    float B = beta[c] - (float)mean * A;
    if (film0) { const float sc = 1.0f + film0[c], sh = film0[C + c]; A *= sc; B = B * sc + sh; }
    if (film1) { const float* f = film1 + (long)n * film1_ld; const float sc = 1.0f + f[c], sh = f[C + c]; A *= sc; B = B * sc + sh; }
    return make_float2(A, B);
}

__global__ void norm_finalize_kernel(const double* __restrict__ sums, int stats_ld, int rep, long rep_stride, int C, int HW, int groups,
                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                     const float* __restrict__ film0, const float* __restrict__ film1, int film1_ld,
                                     float* __restrict__ coef) {
    const int n = blockIdx.x;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float2 ab = norm_affine(sums, stats_ld, rep, rep_stride, n, c, C, HW, groups, gamma, beta, film0, film1, film1_ld);
        coef[((long)n * C + c) * 2] = ab.x;
        coef[((long)n * C + c) * 2 + 1] = ab.y;
    }
}

// FUSED == true: coefficients come from shared memory (computed from the statistics by this CTA, grid.y = sample);
// FUSED == false: from the coef array in global memory (grid.y == 1, samples flattened).
template <bool FUSED>
__global__ void __launch_bounds__(256) norm_apply_kernel(const float* __restrict__ x, int xH, int xW, int x_ld,
                                                         const float* __restrict__ coef, int act, int pool,
                                                         const float* __restrict__ res, int res_ld,
                                                         float* __restrict__ y, int yH, int yW, int y_ld,
                                                         __half* __restrict__ yh, int yh_ld, float* __restrict__ xpool, int xpool_ld,
                                                         int C, long total, int round_out,
                                                         const double* __restrict__ sums, int stats_ld, int rep, long rep_stride,
                                                         int HW, int groups,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                                         const float* __restrict__ film0, const float* __restrict__ film1,
                                                         int film1_ld) {
    extern __shared__ __align__(16) float2 sm_coef[];
    const int cq = C >> 2;
    int n_fixed = 0;
    if (FUSED) {
        pdl_trigger();      // launched with programmatic stream serialization: the statistics come from the previous kernel
        pdl_wait();
        // two-step prologue: (1) mean / rstd per statistics group (channel for InstanceNorm, channel group for GroupNorm)
        // into shared memory, (2) per-channel affine incl. gamma/beta and the FiLM scale-shifts.
        n_fixed = blockIdx.y;
        float2* sm_grp = sm_coef + C;                          // [ngroups] (mean, rstd)
        const int ng = groups == 0 ? C : groups, cpg = C / ng;
        double2* sm_ch = reinterpret_cast<double2*>(sm_coef + 2 * C);   // [C] per-channel (sum, sum of squares) over the replicas
        if (cpg > 1) {                                         // GroupNorm: all threads fold the replicas, then one thread per group
            for (int c = threadIdx.x; c < C; c += blockDim.x)
                sm_ch[c] = fold_stat_replicas(sums + ((long)n_fixed * stats_ld + c) * 2, rep_stride, rep);
            __syncthreads();
        }
        for (int g = threadIdx.x; g < ng; g += blockDim.x) {
            double su = 0.0, sq = 0.0;
            if (cpg > 1) {
                for (int j = 0; j < cpg; ++j) { const double2 v = sm_ch[g * cpg + j]; su += v.x; sq += v.y; }
            } else {
                const double2 v = fold_stat_replicas(sums + ((long)n_fixed * stats_ld + g) * 2, rep_stride, rep);
                su = v.x; sq = v.y;
            }
            const double cnt = (double)HW * cpg;
            const double mean = su / cnt;
            double var = sq / cnt - mean * mean;
            if (var < 0.0) var = 0.0;
            sm_grp[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + 1e-5)));
        }
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const float2 mr = sm_grp[c / cpg];
            float A = mr.y * gamma[c];
            float B = beta[c] - mr.x * A;
            if (film0) { const float sc = 1.0f + film0[c], sh = film0[C + c]; A *= sc; B = B * sc + sh; }
            if (film1) { const float* f = film1 + (long)n_fixed * film1_ld; const float sc = 1.0f + f[c], sh = f[C + c]; A *= sc; B = B * sc + sh; }
            sm_coef[c] = make_float2(A, B);
        }
        __syncthreads();
    }
    const unsigned ucq = (unsigned)cq;
    const unsigned utotal = (unsigned)total, stride = gridDim.x * blockDim.x;
    if (!pool) {
        // streaming path: 4 independent float4 items per thread in flight (32-bit index math; total < 2^31 float4s)
        const long nbase = FUSED ? (long)n_fixed * yH * yW : 0;
        for (unsigned i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < utotal; i0 += 4 * stride) {
            float4 v[4], rv[4];
            unsigned q[4]; long pix[4]; bool ok[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const unsigned i = i0 + u * stride;
                ok[u] = i < utotal;
                const unsigned p0 = ok[u] ? i / ucq : 0u;
                q[u] = ok[u] ? i - p0 * ucq : 0u;
                pix[u] = nbase + p0;
                if (ok[u]) {
                    v[u] = *reinterpret_cast<const float4*>(x + pix[u] * x_ld + 4 * q[u]);
                    if (res) rv[u] = *reinterpret_cast<const float4*>(res + pix[u] * res_ld + 4 * q[u]);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (!ok[u]) continue;
                float4 c0, c1;
                if (FUSED) {
                    const float4* sc = reinterpret_cast<const float4*>(sm_coef + 4 * q[u]);
                    c0 = sc[0]; c1 = sc[1];
                } else {
                    const int n = (int)(pix[u] / ((long)yH * yW));
                    c0 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q[u]) * 2);
                    c1 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q[u]) * 2 + 4);
                }
                float4 r;
                r.x = act_apply(v[u].x * c0.x + c0.y, act); r.y = act_apply(v[u].y * c0.z + c0.w, act);
                r.z = act_apply(v[u].z * c1.x + c1.y, act); r.w = act_apply(v[u].w * c1.z + c1.w, act);
                if (res) { r.x += rv[u].x; r.y += rv[u].y; r.z += rv[u].z; r.w += rv[u].w; }
                if (yh) {     // f16 copy for the tensor-core consumer (round to nearest even; same mantissa width as TF32)
                    const __half2 lo = __floats2half2_rn(r.x, r.y), hi = __floats2half2_rn(r.z, r.w);
                    uint2 pk; pk.x = *reinterpret_cast<const unsigned*>(&lo); pk.y = *reinterpret_cast<const unsigned*>(&hi);
                    *reinterpret_cast<uint2*>(yh + pix[u] * yh_ld + 4 * q[u]) = pk;
                }
                if (y) {
                    if (round_out) { r.x = round_tf32(r.x); r.y = round_tf32(r.y); r.z = round_tf32(r.z); r.w = round_tf32(r.w); }
                    *reinterpret_cast<float4*>(y + pix[u] * y_ld + 4 * q[u]) = r;
                }
            }
        }
        return;
    }
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        // pooled path: i enumerates (output pixel, channel quad); samples are folded into `pix` (FUSED: offset by n_fixed)
        const long pix0 = (long)((unsigned long long)i / ucq);
        const int q = (int)(i - pix0 * ucq);
        const long pix = FUSED ? pix0 + (long)n_fixed * yH * yW : pix0;
        const int n = FUSED ? n_fixed : (int)(pix0 / ((long)yH * yW));
        float4 c0, c1;
        if (FUSED) {
            const float4* sc = reinterpret_cast<const float4*>(sm_coef + 4 * q);
            c0 = sc[0]; c1 = sc[1];
        } else {
            c0 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q) * 2);
            c1 = *reinterpret_cast<const float4*>(coef + ((long)n * C + 4 * q) * 2 + 4);
        }
        const long pin = pix0 - (long)(FUSED ? 0 : n) * yH * yW;       // pixel index within the sample
        const int oy = (int)(pin / yW), ox = (int)(pin - (long)oy * yW);
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 raw[4];
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const float4 v = *reinterpret_cast<const float4*>(
                    x + (((long)n * xH + 2 * oy + dy) * xW + 2 * ox + dx) * x_ld + 4 * q);
                raw[2 * dy + dx] = v;
                r.x += act_apply(v.x * c0.x + c0.y, act); r.y += act_apply(v.y * c0.z + c0.w, act);
                r.z += act_apply(v.z * c1.x + c1.y, act); r.w += act_apply(v.w * c1.z + c1.w, act);
            }
        r.x *= 0.25f; r.y *= 0.25f; r.z *= 0.25f; r.w *= 0.25f;
        if (xpool) {
            // 2x2 mean of the RAW input as well (AvgPool2d(2) of the block's skip path, unet.py:58,164), in the order the conv
            // epilogue's RES_DOWN2 used: the consumer then adds it as a same-resolution residual (one TMA tile instead of
            // 128 scalar loads per thread: slow unsplit RES_DOWN2 epilogues)
            float4 m;
            m.x = 0.25f * ((raw[0].x + raw[1].x) + (raw[2].x + raw[3].x)); m.y = 0.25f * ((raw[0].y + raw[1].y) + (raw[2].y + raw[3].y));
            m.z = 0.25f * ((raw[0].z + raw[1].z) + (raw[2].z + raw[3].z)); m.w = 0.25f * ((raw[0].w + raw[1].w) + (raw[2].w + raw[3].w));
            *reinterpret_cast<float4*>(xpool + pix * xpool_ld + 4 * q) = m;
        }
        if (res) {
            const float4 v = *reinterpret_cast<const float4*>(res + pix * res_ld + 4 * q);
            r.x += v.x; r.y += v.y; r.z += v.z; r.w += v.w;
        }
        if (yh) {
            const __half2 lo = __floats2half2_rn(r.x, r.y), hi = __floats2half2_rn(r.z, r.w);
            uint2 pk; pk.x = *reinterpret_cast<const unsigned*>(&lo); pk.y = *reinterpret_cast<const unsigned*>(&hi);
            *reinterpret_cast<uint2*>(yh + pix * yh_ld + 4 * q) = pk;
        }
        if (y) {
            if (round_out) { r.x = round_tf32(r.x); r.y = round_tf32(r.y); r.z = round_tf32(r.z); r.w = round_tf32(r.w); }
            *reinterpret_cast<float4*>(y + pix * y_ld + 4 * q) = r;
        }
    }
}

void check_apply(const View& x, int pool, const View* res, const View& y) {
    THA4_REQUIRE(x.C == y.C && x.C % 4 == 0 && x.ld % 4 == 0 && y.ld % 4 == 0, "norm_apply: channels");
    THA4_REQUIRE(!x.f16 && (!res || !res->f16), "norm_apply: fp32 input / residual");
    if (pool) THA4_REQUIRE(y.H * 2 == x.H && y.W * 2 == x.W, "norm_apply: pool dims");
    else THA4_REQUIRE(y.H == x.H && y.W == x.W, "norm_apply: dims");
    if (res) THA4_REQUIRE(res->H == y.H && res->W == y.W && res->C == y.C && res->ld % 4 == 0, "norm_apply: res dims");
}

}  // namespace

void norm_stats(const View& x, cudaStream_t s) {
    THA4_REQUIRE(x.stats != nullptr, "norm_stats: view has no statistics buffer");
    THA4_REQUIRE(x.C % 4 == 0 && x.C <= 1024 && x.ld % 4 == 0, "norm_stats: channels");
    const int cq = x.C / 4, PL = 256 / cq;
    const int HW = x.H * x.W;
    dim3 grid(ceil_div(HW, PL * STAT_PIX_PER_THREAD), x.N);
    ProfScope prof(PROF_NORM, s);
    prof_add_work(PROF_NORM, 0.0, (double)x.pixels() * x.C * 4);
    norm_stats_kernel<<<grid, 256, 0, s>>>(x.p, HW, x.C, x.ld, x.stats, x.stats_ld, x.stats_rep, x.stats_rep_stride);
    THA4_LAUNCH_CHECK();
}

void norm_finalize(const View& x, int groups, const float* gamma, const float* beta,
                   const float* film0, const float* film1, int film1_ld, float* coef, cudaStream_t s) {
    THA4_REQUIRE(x.stats != nullptr, "norm_finalize: view has no statistics");
    THA4_REQUIRE(groups == 0 || x.C % groups == 0, "norm_finalize: groups");
    norm_finalize_kernel<<<x.N, 256, 0, s>>>(x.stats, x.stats_ld, x.stats_rep, x.stats_rep_stride, x.C, x.H * x.W, groups, gamma, beta, film0, film1, film1_ld, coef);
    THA4_LAUNCH_CHECK();
}

void norm_apply(const View& x, const float* coef, int act, int pool, const View* res, const View& y, cudaStream_t s,
                int round_out) {
    check_apply(x, pool, res, y);
    const long total = (long)y.N * y.H * y.W * (y.C / 4);
    THA4_REQUIRE(total < (1L << 31), "norm_apply: tensor too large for 32-bit indexing");
    const int blocks = (int)std::max<long>(1, std::min<long>((total + 1023) / 1024, 148L * 8));
    ProfScope prof(PROF_NORM, s);
    prof_add_work(PROF_NORM, 0.0, ((double)x.pixels() + y.pixels() + (res ? y.pixels() : 0)) * x.C * 4);
    THA4_REQUIRE(!y.f16, "norm_apply: fp32 output");
    norm_apply_kernel<false><<<blocks, 256, 0, s>>>(x.p, x.H, x.W, x.ld, coef, act, pool, res ? res->p : nullptr,
                                                    res ? res->ld : 0, y.p, y.H, y.W, y.ld, nullptr, 0, nullptr, 0, x.C, total, round_out,
                                                    nullptr, 0, 1, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, 0);
    THA4_LAUNCH_CHECK();
}

void norm_apply_fused(const View& x, int groups, const float* gamma, const float* beta, const float* film0,
                      const float* film1, int film1_ld, int act, int pool, const View* res, const View& y, cudaStream_t s,
                      int round_out, const View* y16, const View* xpool) {
    check_apply(x, pool, res, y);
    if (xpool) THA4_REQUIRE(pool && !xpool->f16 && xpool->N == y.N && xpool->H == y.H && xpool->W == y.W && xpool->C == y.C && xpool->ld % 4 == 0, "norm_apply_fused: pooled raw copy");
    THA4_REQUIRE(x.stats != nullptr, "norm_apply_fused: view has no statistics");
    // outputs: y fp32 (optionally with an extra f16 copy y16), or y itself f16
    float* yf = y.f16 ? nullptr : y.p;
    __half* yh = y.f16 ? y.hp() : (y16 ? y16->hp() : nullptr);
    const int yh_ld = y.f16 ? y.ld : (y16 ? y16->ld : 0);
    if (y16) THA4_REQUIRE(!y.f16 && y16->f16 && y16->C == y.C && y16->H == y.H && y16->W == y.W && y16->N == y.N && y16->ld % 4 == 0, "norm_apply_fused: f16 copy");
    THA4_REQUIRE(groups == 0 || x.C % groups == 0, "norm_apply_fused: groups");
    const long per_sample = (long)y.H * y.W * (y.C / 4);
    THA4_REQUIRE(per_sample < (1L << 31), "norm_apply: tensor too large for 32-bit indexing");
    const int bx = (int)std::max<long>(1, std::min<long>((per_sample + 1023) / 1024, std::max(1, 148 * 8 / y.N)));
    ProfScope prof(PROF_NORM, s);
    prof_add_work(PROF_NORM, 0.0, ((double)x.pixels() * 4 + y.pixels() * (yf ? 4 : 0) + y.pixels() * (yh ? 2 : 0) + (res ? y.pixels() * 4 : 0)) * x.C);
    // per-sample pointers: grid.y selects the sample, the kernel indexes within it
    dim3 grid(bx, y.N);
    launch_pdl(norm_apply_kernel<true>, grid, dim3(256), 2 * x.C * sizeof(float2) + x.C * sizeof(double2), s, 1,
               (const float*)x.p, x.H, x.W, x.ld, (const float*)nullptr, act, pool, (const float*)(res ? res->p : nullptr), res ? res->ld : 0, yf, y.H, y.W, y.ld, yh, yh_ld, xpool ? xpool->p : (float*)nullptr, xpool ? xpool->ld : 0, x.C, per_sample,
               round_out, (const double*)x.stats, x.stats_ld, x.stats_rep, x.stats_rep_stride, x.H * x.W, groups, gamma, beta, film0, film1, film1_ld);
    THA4_LAUNCH_CHECK();
}

}  // namespace tha4
