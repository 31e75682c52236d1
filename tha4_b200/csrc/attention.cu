// Self-attention of the U-Net bottleneck (unet.py:192-202,230-239): 256 tokens (16x16), 8 heads x 32 channels.
// Two kernels: attention_kernel (fp32 CUDA cores; strict mode): K and V of the head live in shared memory (64 KB), each
// thread owns one query row and runs an online softmax over its keys; attention_mma_kernel (default mode): the same math
// on mma.sync with f16 operands.  0.4 GFLOP per network: latency-, not throughput-critical.
#include "ops.cuh"
#include "profiler.cuh"

namespace tha4 {
namespace {

constexpr int L = 256, D = 32;

// grid = N * heads * (L / QPB), block = 256 threads = QPB queries x KSPLIT key splits.  Each thread runs an online softmax
// over its L / KSPLIT keys; the KSPLIT partial (max, sum, acc) triples of a query are merged with warp shuffles.
// Launched as <64, 4, 36>: 4 CTAs per (sample, head); row pitch 36 (16-byte aligned rows): the 4 key-split lanes hit 4 banks.
template <int QPB, int KSPLIT, int DP>
__global__ void __launch_bounds__(QPB * KSPLIT) attention_kernel(const float* __restrict__ qkv, int qkv_ld, int C, int heads,
                                                                 float* __restrict__ out, int out_ld) {
    static_assert(QPB * KSPLIT == L, "one thread per token while staging K / V");
    static_assert(DP % 4 == 0, "K / V rows are staged as float4");
    extern __shared__ __align__(16) float sm[];
    float* Ks = sm;            // [L][DP]
    float* Vs = sm + L * DP;   // [L][DP]
    const int qq = blockIdx.x % (L / QPB);
    const int nh = blockIdx.x / (L / QPB);
    const int n = nh / heads, h = nh % heads;
    const int tid = threadIdx.x;
    const float* base = qkv + (long)n * L * qkv_ld;
    {   // stage K and V of this head: thread tid copies token tid
        const float4* kp = reinterpret_cast<const float4*>(base + (long)tid * qkv_ld + C + h * D);
        const float4* vp = reinterpret_cast<const float4*>(base + (long)tid * qkv_ld + 2 * C + h * D);
#pragma unroll
        for (int j = 0; j < D / 4; ++j) {
            const float4 kv = kp[j], vv = vp[j];
            reinterpret_cast<float4*>(Ks + tid * DP)[j] = kv;
            reinterpret_cast<float4*>(Vs + tid * DP)[j] = vv;
        }
    }
    const int t = qq * QPB + tid / KSPLIT;      // query token
    const int ks = tid % KSPLIT;                // key split: keys ks, ks + 4, ks + 8, ...
    float q[D];
    {
        const float4* qp = reinterpret_cast<const float4*>(base + (long)t * qkv_ld + h * D);
#pragma unroll
        for (int j = 0; j < D / 4; ++j) {
            float4 v = qp[j];
            q[4 * j] = v.x; q[4 * j + 1] = v.y; q[4 * j + 2] = v.z; q[4 * j + 3] = v.w;
        }
    }
    // scale = C_head^-1/4 applied to both q and k (unet.py:197-199)
    const float scale = 1.0f / sqrtf(sqrtf((float)D));
#pragma unroll
    for (int j = 0; j < D; ++j) q[j] *= scale;
    __syncthreads();

    float m = -INFINITY, l = 0.0f, acc[D];
#pragma unroll
    for (int j = 0; j < D; ++j) acc[j] = 0.0f;
    for (int s = ks; s < L; s += KSPLIT) {
        const float* kr = Ks + s * DP;
        float dot = 0.0f;
#pragma unroll
        for (int j = 0; j < D; ++j) dot = fmaf(q[j], kr[j] * scale, dot);
        const float mn = fmaxf(m, dot);
        const float corr = expf(m - mn);
        const float pw = expf(dot - mn);
        l = l * corr + pw;
        const float* vr = Vs + s * DP;
#pragma unroll
        for (int j = 0; j < D; ++j) acc[j] = fmaf(acc[j], corr, pw * vr[j]);
        m = mn;
    }
    // merge the KSPLIT partials of this query (adjacent lanes)
#pragma unroll
    for (int off = 1; off < KSPLIT; off <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, off);
        const float lo = __shfl_xor_sync(0xffffffffu, l, off);
        const float mn = fmaxf(m, mo);
        const float ca = expf(m - mn), cb = expf(mo - mn);
        l = l * ca + lo * cb;
#pragma unroll
        for (int j = 0; j < D; ++j) {
            const float ao = __shfl_xor_sync(0xffffffffu, acc[j], off);
            acc[j] = acc[j] * ca + ao * cb;
        }
        m = mn;
    }
    if (ks == 0) {
        const float inv = 1.0f / l;
        float4* op = reinterpret_cast<float4*>(out + ((long)n * L + t) * out_ld + h * D);
#pragma unroll
        for (int j = 0; j < D / 4; ++j)
            op[j] = make_float4(acc[4 * j] * inv, acc[4 * j + 1] * inv, acc[4 * j + 2] * inv, acc[4 * j + 3] * inv);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Default-mode attention on the tensor cores (mma.sync m16n8k16, f16 operands, fp32 accumulate).  The kernel above is one
// dependent 32-FMA chain per (query, key) with two warps per scheduler, 12 launches per frame for
// 0.07 GFLOP each.  Here a warp owns 16 queries of one (sample, head): S = Q K^T for all 256 keys stays in registers as
// 32 accumulator tiles, the softmax runs on the fragments (row max / sum over the 4 lanes of a quad), and the accumulator
// layout of two adjacent S tiles IS the A-fragment layout of P for the P V product (the FlashAttention-2 register identity).
// K lives in shared memory as f16 [key][32 + 8] (pitch 40 halves: the 8 rows x 4 words a B-fragment load touches fall in 32
// different banks), V transposed as [32][256 + 8] so that a B fragment of P V is one 32-bit load.  q and k are scaled by
// C_head^-1/4 each before they are rounded (unet.py:197-199).  Error class: 10-bit operands, like every conv of the default mode.
constexpr int AT_WARPS = 4;                       // 64 queries per CTA: N * heads * 4 CTAs
constexpr int KH_PITCH = D + 8, VT_PITCH = L + 8;

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(AT_WARPS * 32) attention_mma_kernel(const float* __restrict__ qkv, int qkv_ld, int C, int heads,
                                                                      float* __restrict__ out, int out_ld) {
    __shared__ __align__(16) __half Kh[L * KH_PITCH];       // 20 480 B
    __shared__ __align__(16) __half Vt[D * VT_PITCH];       // 16 896 B
    constexpr int QBLK = L / (AT_WARPS * 16);
    const int qq = blockIdx.x % QBLK;
    const int nh = blockIdx.x / QBLK;
    const int n = nh / heads, h = nh % heads;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* base = qkv + (long)n * L * qkv_ld;
    const float scale = 1.0f / sqrtf(sqrtf((float)D));
    // ---- stage K (scaled, f16) and V^T (f16): a thread takes a PAIR of tokens so that V^T is written as packed halves ----
    for (int pr = tid; pr < L / 2; pr += AT_WARPS * 32) {
        const int t0 = 2 * pr;
        const float4* k0 = reinterpret_cast<const float4*>(base + (long)t0 * qkv_ld + C + h * D);
        const float4* k1 = reinterpret_cast<const float4*>(base + (long)(t0 + 1) * qkv_ld + C + h * D);
        const float4* v0 = reinterpret_cast<const float4*>(base + (long)t0 * qkv_ld + 2 * C + h * D);
        const float4* v1 = reinterpret_cast<const float4*>(base + (long)(t0 + 1) * qkv_ld + 2 * C + h * D);
        float4 ka[D / 4], kb[D / 4], va[D / 4], vb[D / 4];
#pragma unroll
        for (int j = 0; j < D / 4; ++j) { ka[j] = k0[j]; kb[j] = k1[j]; va[j] = v0[j]; vb[j] = v1[j]; }
#pragma unroll
        for (int j = 0; j < D / 8; ++j) {
            uint4 pa, pb;
            pa.x = pack_h2(ka[2 * j].x * scale, ka[2 * j].y * scale); pa.y = pack_h2(ka[2 * j].z * scale, ka[2 * j].w * scale);
            pa.z = pack_h2(ka[2 * j + 1].x * scale, ka[2 * j + 1].y * scale); pa.w = pack_h2(ka[2 * j + 1].z * scale, ka[2 * j + 1].w * scale);
            pb.x = pack_h2(kb[2 * j].x * scale, kb[2 * j].y * scale); pb.y = pack_h2(kb[2 * j].z * scale, kb[2 * j].w * scale);
            pb.z = pack_h2(kb[2 * j + 1].x * scale, kb[2 * j + 1].y * scale); pb.w = pack_h2(kb[2 * j + 1].z * scale, kb[2 * j + 1].w * scale);
            *reinterpret_cast<uint4*>(Kh + t0 * KH_PITCH + 8 * j) = pa;
            *reinterpret_cast<uint4*>(Kh + (t0 + 1) * KH_PITCH + 8 * j) = pb;
        }
        uint32_t* vt = reinterpret_cast<uint32_t*>(Vt);
#pragma unroll
        for (int j = 0; j < D / 4; ++j) {
            vt[((4 * j + 0) * VT_PITCH + t0) >> 1] = pack_h2(va[j].x, vb[j].x);
            vt[((4 * j + 1) * VT_PITCH + t0) >> 1] = pack_h2(va[j].y, vb[j].y);
            vt[((4 * j + 2) * VT_PITCH + t0) >> 1] = pack_h2(va[j].z, vb[j].z);
            vt[((4 * j + 3) * VT_PITCH + t0) >> 1] = pack_h2(va[j].w, vb[j].w);
        }
    }
    // ---- Q fragments of this warp's 16 queries (two k-steps of 16 channels) ----
    const int g = lane >> 2, t = lane & 3;
    const int q0 = (qq * AT_WARPS + warp) * 16;
    uint32_t qa[2][4];
    {
        const float* qlo = base + (long)(q0 + g) * qkv_ld + h * D;
        const float* qhi = base + (long)(q0 + g + 8) * qkv_ld + h * D;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const float2 a = *reinterpret_cast<const float2*>(qlo + 16 * ks + 2 * t), b = *reinterpret_cast<const float2*>(qhi + 16 * ks + 2 * t);
            const float2 c = *reinterpret_cast<const float2*>(qlo + 16 * ks + 2 * t + 8), d = *reinterpret_cast<const float2*>(qhi + 16 * ks + 2 * t + 8);
            qa[ks][0] = pack_h2(a.x * scale, a.y * scale); qa[ks][1] = pack_h2(b.x * scale, b.y * scale);
            qa[ks][2] = pack_h2(c.x * scale, c.y * scale); qa[ks][3] = pack_h2(d.x * scale, d.y * scale);
        }
    }
    __syncthreads();
    // ---- S = Q K^T: 32 tiles of 16 queries x 8 keys ----
    float sc[L / 8][4];
    const uint32_t* kw = reinterpret_cast<const uint32_t*>(Kh);
#pragma unroll
    for (int j = 0; j < L / 8; ++j) {
        sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.0f;
        const int krow = ((8 * j + g) * KH_PITCH) >> 1;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
            mma_16816(sc[j], qa[ks], kw[krow + 8 * ks + t], kw[krow + 8 * ks + t + 4]);
    }
    // ---- softmax over the 256 keys of rows g (c0, c1) and g + 8 (c2, c3) ----
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < L / 8; ++j) { m0 = fmaxf(m0, fmaxf(sc[j][0], sc[j][1])); m1 = fmaxf(m1, fmaxf(sc[j][2], sc[j][3])); }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    float l0 = 0.0f, l1 = 0.0f;
    constexpr float LOG2E = 1.4426950408889634f;
    const float mb0 = m0 * LOG2E, mb1 = m1 * LOG2E;
#pragma unroll
    for (int j = 0; j < L / 8; ++j) {
        sc[j][0] = exp2f(fmaf(sc[j][0], LOG2E, -mb0)); sc[j][1] = exp2f(fmaf(sc[j][1], LOG2E, -mb0));
        sc[j][2] = exp2f(fmaf(sc[j][2], LOG2E, -mb1)); sc[j][3] = exp2f(fmaf(sc[j][3], LOG2E, -mb1));
        l0 += sc[j][0] + sc[j][1]; l1 += sc[j][2] + sc[j][3];
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    // ---- O = P V: 16 k-steps of 16 keys, 4 tiles of 8 channels ----
    float oc[D / 8][4];
#pragma unroll
    for (int nd = 0; nd < D / 8; ++nd) oc[nd][0] = oc[nd][1] = oc[nd][2] = oc[nd][3] = 0.0f;
    const uint32_t* vw = reinterpret_cast<const uint32_t*>(Vt);
#pragma unroll
    for (int kk = 0; kk < L / 16; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_h2(sc[2 * kk][0], sc[2 * kk][1]); pa[1] = pack_h2(sc[2 * kk][2], sc[2 * kk][3]);
        pa[2] = pack_h2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]); pa[3] = pack_h2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
#pragma unroll
        for (int nd = 0; nd < D / 8; ++nd) {
            const int vrow = ((8 * nd + g) * VT_PITCH + 16 * kk) >> 1;
            mma_16816(oc[nd], pa, vw[vrow + t], vw[vrow + t + 4]);
        }
    }
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    float* olo = out + ((long)n * L + q0 + g) * out_ld + h * D;
    float* ohi = out + ((long)n * L + q0 + g + 8) * out_ld + h * D;
#pragma unroll
    for (int nd = 0; nd < D / 8; ++nd) {
        *reinterpret_cast<float2*>(olo + 8 * nd + 2 * t) = make_float2(oc[nd][0] * i0, oc[nd][1] * i0);
        *reinterpret_cast<float2*>(ohi + 8 * nd + 2 * t) = make_float2(oc[nd][2] * i1, oc[nd][3] * i1);
    }
}

}  // namespace

void attention_forward(const View& qkv, int heads, const View& out, cudaStream_t s, bool fast) {
    THA4_REQUIRE(qkv.H * qkv.W == L && out.C * 3 == qkv.C && out.C / heads == D, "attention: shape (L=256, head dim 32)");
    THA4_REQUIRE(qkv.ld % 4 == 0 && out.ld % 4 == 0, "attention: alignment");
    ProfScope prof(PROF_ATTN, s);
    if (fast) {
        attention_mma_kernel<<<qkv.N * heads * (L / (AT_WARPS * 16)), AT_WARPS * 32, 0, s>>>(qkv.p, qkv.ld, out.C, heads, out.p, out.ld);
        THA4_LAUNCH_CHECK();
        return;
    }
    constexpr int QPB = 64, KSPLIT = 4, DP = 36;
    constexpr size_t smem = 2 * L * DP * sizeof(float);
    THA4_ENSURE_SMEM((attention_kernel<QPB, KSPLIT, DP>), smem);
    attention_kernel<QPB, KSPLIT, DP><<<qkv.N * heads * (L / QPB), QPB * KSPLIT, smem, s>>>(qkv.p, qkv.ld, out.C, heads, out.p, out.ld);
    THA4_LAUNCH_CHECK();
}

}  // namespace tha4
